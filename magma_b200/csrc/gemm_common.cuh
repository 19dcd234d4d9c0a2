// magma_b200 — pieces shared by the GEMM core (gemm.cu) and the fused attention kernels (attention.cu): tile
// configuration, kernel parameter block and the fused epilogue applied to wgmma accumulator fragments.
#pragma once
#include "common.cuh"

namespace mb200 {

static constexpr int BM = 128;        // tile M: two consumer warpgroups x wgmma M = 64
static constexpr int BK = 64;         // 64 bf16 = 128 bytes = one SWIZZLE_128B row
static constexpr int WG_K = 16;       // wgmma K for 16-bit inputs
static constexpr int kThreads = 384;  // warpgroup 0 = TMA producer, warpgroups 1, 2 = MMA + epilogue
static constexpr int kSmemBudget = 200 * 1024;  // operand ring; + alignment slack and barriers < 227 KB

template <int BN>
struct Cfg {
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStagesRaw = kSmemBudget / kStageBytes;
  static constexpr int kStages = kStagesRaw > 8 ? 8 : kStagesRaw;
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
};

struct GemmKernelParams {
  int M, N, K;
  int nb0;
  int tiles_m, tiles_n, total_tiles;
  void* C;
  long long ldc, c_bs0, c_bs1;
  float alpha;
  int act, dact, accumulate;
  const bf16* bias;
  bf16* aux_out;
  const bf16* aux_in;
  const bf16* res1;
  const bf16* res2;
  long long ld_res;
  // fused rotary embedding (rotate_every_two) on column pairs: applied when rope_mode != 0
  const float2* rope_tab;  // [rope_S][rope_rot/2] (cos, sin) of the position of row (row % rope_S)
  int rope_mode;           // +1 forward, -1 inverse (transpose rotation)
  int rope_S, rope_hd, rope_rot, rope_ncols;
  int epi_kind;  // EK_GENERIC, or EK_SPLITK for the partial tiles of a split-K GEMM
  int c_f32;     // C is fp32 (else bf16)
  // split-K (small-M / weight-streaming GEMMs, e.g. decode): work item = (tile, k-range); partial tiles are reduced
  // written to splitk_ws [split][M][ld_ws] (fp32) and summed in fixed order, with the fused epilogue, by
  // splitk_finalize_kernel
  int split_k, kb_per_split;
  float* splitk_ws;
  long long ld_ws;
};

__device__ __forceinline__ uint32_t ldg32(const bf16* ptr) {
  uint32_t u;
  asm volatile("ld.global.nc.u32 %0, [%1];" : "=r"(u) : "l"(ptr));
  return u;
}
__device__ __forceinline__ float2 bf16x2_to_f32(uint32_t u) {
  return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u));
}
__device__ __forceinline__ uint32_t f32x2_to_bf16(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

enum { EK_GENERIC = 0, EK_SPLITK };

// ---------------------------------------------------------------------------------------------
// Epilogue on the accumulator fragment of one consumer warpgroup (64 rows x BN columns, wgmma.cuh layout): every thread
// owns column pairs (c, c + 1), c even, of two rows. A pair is also a rotary pair (rotate_every_two), so alpha / bias /
// rotary / saved pre-activation / activation / activation-derivative / residuals / store are all applied in registers
// on 8-byte (fp32) or 4-byte (bf16) chunks without any exchange between threads. All branches on p are warp-uniform.
// Split-K work items store the fp32 partial tile into their slice of the workspace instead (EK_SPLITK).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void epi_pair(const GemmKernelParams& p, long long boff, int row, int col, float v0, float v1,
                                         int ks) {
  if (row >= p.M || col >= p.N) return;
  const bool two = col + 1 < p.N;
  v0 *= p.alpha;
  v1 *= p.alpha;
  if (p.epi_kind == EK_SPLITK) {
    float* w = p.splitk_ws + ((long long)ks * p.M + row) * p.ld_ws + col;  // ld_ws % 4 == 0: the padded column exists
    *reinterpret_cast<float2*>(w) = make_float2(v0, v1);
    return;
  }
  if (p.bias) {
    v0 += __bfloat162float(p.bias[col]);
    if (two) v1 += __bfloat162float(p.bias[col + 1]);
  }
  if (p.rope_mode != 0 && col < p.rope_ncols) {
    const int dim = col % p.rope_hd;
    if (dim < p.rope_rot) {
      const float2 cs = __ldg(p.rope_tab + (long long)(row % p.rope_S) * (p.rope_rot >> 1) + (dim >> 1));
      const float sg = p.rope_mode > 0 ? 1.f : -1.f;
      const float a0 = v0, a1 = v1;
      v0 = a0 * cs.x - a1 * cs.y * sg;
      v1 = a1 * cs.x + a0 * cs.y * sg;
    }
  }
  const long long coff = boff + (long long)row * p.ldc + col;
  if (p.aux_out) {
    if (two) *reinterpret_cast<uint32_t*>(p.aux_out + coff) = f32x2_to_bf16(v0, v1);
    else p.aux_out[coff] = __float2bfloat16(v0);
  }
  if (p.act == MB200_ACT_GELU_NEW) {
    v0 = gelu_new_f(v0);
    v1 = gelu_new_f(v1);
  } else if (p.act == MB200_ACT_QUICK_GELU) {
    v0 = quick_gelu_f(v0);
    v1 = quick_gelu_f(v1);
  } else if (p.act == MB200_ACT_RELU) {
    v0 = fmaxf(v0, 0.f);
    v1 = fmaxf(v1, 0.f);
  }
  if (p.dact) {
    float2 a;
    if (two) a = bf16x2_to_f32(ldg32(p.aux_in + coff));
    else a = make_float2(__bfloat162float(p.aux_in[coff]), 0.f);
    if (p.dact == MB200_DACT_GELU_NEW) {
      v0 *= gelu_new_grad_f(a.x);
      v1 *= gelu_new_grad_f(a.y);
    } else {
      v0 = a.x > 0.f ? v0 : 0.f;
      v1 = a.y > 0.f ? v1 : 0.f;
    }
  }
  const long long roff = boff + (long long)row * p.ld_res + col;
  if (p.res1) {
    if (two) {
      const float2 r = bf16x2_to_f32(ldg32(p.res1 + roff));
      v0 += r.x;
      v1 += r.y;
    } else {
      v0 += __bfloat162float(p.res1[roff]);
    }
  }
  if (p.res2) {
    if (two) {
      const float2 r = bf16x2_to_f32(ldg32(p.res2 + roff));
      v0 += r.x;
      v1 += r.y;
    } else {
      v0 += __bfloat162float(p.res2[roff]);
    }
  }
  if (p.act == MB200_ACT_RELU_POST) {
    v0 = fmaxf(v0, 0.f);
    v1 = fmaxf(v1, 0.f);
  }
  if (p.c_f32) {
    float* dst = reinterpret_cast<float*>(p.C) + coff;
    if (two) {
      float2 o = make_float2(v0, v1);
      if (p.accumulate) {
        const float2 old = *reinterpret_cast<const float2*>(dst);
        o.x += old.x;
        o.y += old.y;
      }
      *reinterpret_cast<float2*>(dst) = o;
    } else {
      dst[0] = p.accumulate ? dst[0] + v0 : v0;
    }
  } else {
    bf16* dst = reinterpret_cast<bf16*>(p.C) + coff;
    if (two) *reinterpret_cast<uint32_t*>(dst) = f32x2_to_bf16(v0, v1);
    else dst[0] = __float2bfloat16(v0);
  }
}

// row0: first row (within the batch) of this warpgroup's 64-row slab; col0: first column of the tile
template <int BN>
__device__ __forceinline__ void epi_fragment(const GemmKernelParams& p, const float (&acc)[BN / 2], long long boff,
                                             int row0, int col0, int ks) {
  const int wt = threadIdx.x & 127;
  const int r = row0 + (wt >> 5) * 16 + ((wt & 31) >> 2);
  const int c = col0 + 2 * (wt & 3);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    if (col0 + 8 * j >= p.N) break;  // warp-uniform
    epi_pair(p, boff, r, c + 8 * j, acc[4 * j], acc[4 * j + 1], ks);
    epi_pair(p, boff, r + 8, c + 8 * j, acc[4 * j + 2], acc[4 * j + 3], ks);
  }
}

// host helper shared by gemm.cu / attention.cu
int make_operand_map(CUtensorMap* out, const mb200_operand& op, int rows, int K, int nb0, int nb1, int box_rows);

}  // namespace mb200
