// magma_b200 — fused causal self-attention for one (batch, head) per CTA when the whole sequence fits one tile
// (S <= 128 — BASELINE.json config 2 has S = 128), head_dim a multiple of 64 up to 256.
//
// Replaces, per layer, the 3 (forward) / 6 (backward) launches of the GEMM-based path of the schedules — QK^T GEMM,
// softmax kernel, PV GEMM; dP, dV, softmax-bwd, dQ, dK GEMMs — which spend most of their time on fixed launch /
// prologue / epilogue cost for 0.5 % of the step's FLOPs. Numerics are those of the reference
// (GPTJAttention._attn, hf:gptj/modeling_gptj.py:136-149): fp32 scores from bf16 q,k, / sqrt(hd), causal mask,
// fp32 softmax, probabilities rounded to bf16 before P*V; the backward uses the saved bf16 P.
//
// 256 threads = two warpgroups; warpgroup w owns rows [64 w, 64 w + 64) of every 128-row product and holds them as a
// wgmma accumulator fragment (wgmma.cuh): a row is spread over the 4 threads of a quad, so row reductions (softmax
// maximum and sum, rowsum(dP * P)) are two quad shuffles.
// Forward:
//   TMA: Q, K ([S, hd] K-major, hd/64 boxes of 128x64) and V -> smem (SWIZZLE_128B)
//   S = Q K^T      wgmma 64x128xhd per warpgroup
//   softmax in registers; P -> bf16 -> smem (K-major operand layout) and -> global
//   O = P V        wgmma 64xhdx128 (V as MN-major B operand: same bytes as its K-major tile) -> bf16 -> global
// Backward:
//   dP = dO V^T ; dS = P*(dP - rowsum(dP*P))/sqrt(hd) ; dV = P^T dO (P, dO as MN-major operands: same smem bytes)
//   dQ = dS K ; dK = dS^T Q, both with the inverse rotary rotation applied on the way out (they are gradients of the
//   rotated q,k), written straight into the fused dqkv buffer.
//   The EXT_DP instantiation adds a gradient that reaches P from outside the block (a loss reading the returned
//   attention probabilities) to dP before the row sum: the same algebra, dP = dO V^T + dP_ext.
#include <stdlib.h>

#include "gemm_common.cuh"

namespace mb200 {

static constexpr int kAttThreads = 256;
static constexpr int kTile = 128 * 64 * 2;  // one 128-row x 64-col bf16 box = 16 KB

struct AttnParams {
  int S, H, hd, rot;
  float scale;
  // forward outputs / backward inputs
  bf16* P;             // [B,H,S,ldP]
  long long ldP;
  bf16* O;             // [B,S,H,hd] (row stride ldo)
  long long ldo;
  // backward outputs: fused dqkv [B*S][3][H][hd]
  bf16* dqkv;
  long long ld_dqkv;
  const float2* rope_tab;  // [S][rot/2] (cos, sin), positions 0..S-1
  // backward input of attn_bwd_tile_kernel<HD, true>: the gradient on P from outside the block, [B,H,S,ld_dpe]
  const bf16* dPe;
  long long ld_dpe;
};

__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// the 128 threads of warpgroup `wg` meet (named barriers 1 and 2; 0 is __syncthreads)
__device__ __forceinline__ void wg_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(wg + 1) : "memory"); }

// byte offset of element (r, c) in a K-major SWIZZLE_128B operand tile made of 16 KB [128 rows x 64 cols] k-blocks
__device__ __forceinline__ uint32_t operand_off(int r, int c) {
  return (uint32_t)((c >> 6) * kTile + r * 128 + ((((c & 63) >> 3) ^ (r & 7)) << 4) + (c & 7) * 2);
}
__device__ __forceinline__ void st_pair(uint32_t saddr, float a, float b) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(saddr), "r"(f32x2_to_bf16(a, b)) : "memory");
}
__device__ __forceinline__ float2 ld_pair(uint32_t saddr) {
  uint32_t u;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(u) : "r"(saddr));
  return bf16x2_to_f32(u);
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// D[64 rows of warpgroup wg] = A * B over nkb k-blocks of 64. A / B tiles are sequences of 16 KB k-blocks (K-major) or of
// 16 KB 64-wide MN chunks holding 128 k-rows each (MN-major). The warpgroup's rows of A are rows 64 wg.. of each k-block
// (K-major) or MN chunk wg (MN-major). Returns with the products complete.
template <int N, bool A_MN, bool B_MN>
__device__ __forceinline__ void wg_mma(float (&d)[N / 2], int wg, uint32_t a_base, uint32_t b_base, int nkb,
                                       uint32_t acc0 = 0u) {
  a_base += A_MN ? (uint32_t)(wg * kTile) : (uint32_t)(wg * 64 * 128);
  wgmma_fence();
  for (int kb = 0; kb < nkb; ++kb) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      // K-major: k-block kb is its own 16 KB tile, +32 B per 16-element k-step.
      // MN-major: every 64-wide MN chunk is one 16 KB tile of 128 k-rows (LBO = 16 KB), +2048 B per 16 k-rows.
      const uint32_t ao = A_MN ? (uint32_t)((kb * 4 + k) * 2048) : (uint32_t)(kb * kTile + k * 32);
      const uint32_t bo = B_MN ? (uint32_t)((kb * 4 + k) * 2048) : (uint32_t)(kb * kTile + k * 32);
      const uint64_t da = make_smem_desc(a_base + ao, A_MN ? (uint32_t)kTile : 0u, 1024);
      const uint64_t db = make_smem_desc(b_base + bo, B_MN ? (uint32_t)kTile : 0u, 1024);
      wgmma_bf16<N, A_MN ? 1 : 0, B_MN ? 1 : 0>(d, da, db, ((kb | k) != 0 ? 1u : 0u) | acc0);
    }
  }
  wgmma_commit();
  wgmma_wait<0>();
}

// fragment coordinates of this thread: rows r0 and r0 + 8 of the warpgroup's 64, columns 8 j + c0 + {0, 1}
struct Frag {
  int wg, r0, c0, quad0;
  __device__ __forceinline__ Frag() {
    const int t = threadIdx.x;
    wg = t >> 7;
    r0 = wg * 64 + ((t & 127) >> 5) * 16 + ((t & 31) >> 2);
    c0 = 2 * (t & 3);
    quad0 = (t & 3) == 0;
  }
};

// store a 64 x HD fragment as bf16 rows dst + row * ld (rows >= nrows skipped), with the inverse rotary rotation of the
// first `rot` columns when tab != nullptr (row r uses position r)
template <int HD>
__device__ __forceinline__ void store_rows(const Frag& f, const float (&d)[HD / 2], bf16* dst, long long ld, int nrows,
                                           const float2* tab, int rot) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = f.r0 + 8 * h;
    if (r >= nrows) continue;
    bf16* row = dst + (long long)r * ld;
#pragma unroll
    for (int j = 0; j < HD / 8; ++j) {
      const int c = 8 * j + f.c0;
      float a0 = d[4 * j + 2 * h], a1 = d[4 * j + 2 * h + 1];
      if (tab != nullptr && c < rot) {
        const float2 cs = __ldg(tab + (long long)r * (rot >> 1) + (c >> 1));
        const float b0 = a0 * cs.x + a1 * cs.y;  // transpose of [[c, -s], [s, c]]
        a1 = a1 * cs.x - a0 * cs.y;
        a0 = b0;
      }
      *reinterpret_cast<uint32_t*>(row + c) = f32x2_to_bf16(a0, a1);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------------
template <int HD>
__global__ void __launch_bounds__(kAttThreads, 1)
attn_fwd_tile_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                     const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int nhb = HD / 64;  // 64-wide head-dim blocks
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + nhb * kTile;
  uint8_t* sV = sK + nhb * kTile;
  uint8_t* sP = sV + nhb * kTile;  // 2 k-blocks
  uint64_t* bars = reinterpret_cast<uint64_t*>(sP + 2 * kTile);
  uint64_t* bar_qk = bars + 0;
  uint64_t* bar_v = bars + 1;

  const int t = threadIdx.x;
  const int h = blockIdx.x % p.H, b = blockIdx.x / p.H;
  const Frag f;

  pdl_trigger();
  if (t == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    for (int i = 0; i < 2; ++i) mbar_init(&bars[i], 1);
    mbar_fence_init();
  }
  __syncthreads();
  pdl_wait();

  if (t == 0) {
    mbar_expect_tx(bar_qk, 2 * nhb * kTile);
    for (int kb = 0; kb < nhb; ++kb) {
      tma_load_4d(sQ + kb * kTile, &tmQ, bar_qk, kb * 64, 0, h, b);
      tma_load_4d(sK + kb * kTile, &tmK, bar_qk, kb * 64, 0, h, b);
    }
    mbar_expect_tx(bar_v, nhb * kTile);
    for (int kb = 0; kb < nhb; ++kb) tma_load_4d(sV + kb * kTile, &tmV, bar_v, kb * 64, 0, h, b);
  }
  mbar_wait(bar_qk, 0);
  float s[64];
  wg_mma<128, false, false>(s, f.wg, smem_u32(sQ), smem_u32(sK), nhb);  // S = Q K^T
  const uint32_t sP_s = smem_u32(sP);
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int q = f.r0 + 8 * hh;
    const int lim = min(p.S, q + 1);  // causal: keys 0..q
    float m = -INFINITY;
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float& v = s[4 * j + 2 * hh + e];
        v *= p.scale;
        if (8 * j + f.c0 + e < lim) m = fmaxf(m, v);
      }
    m = quad_max(m);
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float& v = s[4 * j + 2 * hh + e];
        v = 8 * j + f.c0 + e < lim ? __expf(v - m) : 0.f;
        sum += v;
      }
    sum = quad_sum(sum);
    const float inv = q < p.S ? 1.f / sum : 0.f;
    bf16* prow = p.P + (((long long)b * p.H + h) * p.S + q) * p.ldP;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int c = 8 * j + f.c0;
      const float a0 = s[4 * j + 2 * hh] * inv, a1 = s[4 * j + 2 * hh + 1] * inv;
      st_pair(sP_s + operand_off(q, c), a0, a1);
      if (q < p.S && c < p.ldP) *reinterpret_cast<uint32_t*>(prow + c) = f32x2_to_bf16(a0, a1);  // saved for backward
    }
  }
  fence_async_smem();  // generic-proxy smem writes -> visible to the tensor core (async proxy)
  wg_sync(f.wg);       // this warpgroup's rows of P are complete
  mbar_wait(bar_v, 0);
  float o[HD / 2];
  wg_mma<HD, false, true>(o, f.wg, sP_s, smem_u32(sV), 2);  // O = P V   (K = 128 keys)
  store_rows<HD>(f, o, p.O + (long long)b * p.S * p.ldo + (long long)h * HD, p.ldo, p.S, nullptr, 0);
}

// ---------------------------------------------------------------------------------------------
// backward
// ---------------------------------------------------------------------------------------------
template <int HD, bool EXT_DP>
__global__ void __launch_bounds__(kAttThreads, 1)
attn_bwd_tile_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                     const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO,
                     const __grid_constant__ CUtensorMap tmP, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int nhb = HD / 64;
  uint8_t* R1 = smem;                 // dO, later Q
  uint8_t* R2 = R1 + nhb * kTile;     // V, later K
  uint8_t* R3 = R2 + nhb * kTile;     // P   (2 k-blocks)
  uint8_t* R4 = R3 + 2 * kTile;       // dS  (2 k-blocks)
  uint64_t* bars = reinterpret_cast<uint64_t*>(R4 + 2 * kTile);
  uint64_t* bar_a = bars + 0;   // dO + V landed
  uint64_t* bar_p = bars + 1;   // P landed
  uint64_t* bar_k = bars + 2;   // K landed
  uint64_t* bar_q = bars + 3;   // Q landed

  const int t = threadIdx.x;
  const int h = blockIdx.x % p.H, b = blockIdx.x / p.H;
  const Frag f;

  pdl_trigger();
  if (t == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    tma_prefetch_desc(&tmdO);
    tma_prefetch_desc(&tmP);
    for (int i = 0; i < 4; ++i) mbar_init(&bars[i], 1);
    mbar_fence_init();
  }
  __syncthreads();
  pdl_wait();

  if (t == 0) {
    mbar_expect_tx(bar_a, 2 * nhb * kTile);
    for (int kb = 0; kb < nhb; ++kb) {
      tma_load_4d(R1 + kb * kTile, &tmdO, bar_a, kb * 64, 0, h, b);
      tma_load_4d(R2 + kb * kTile, &tmV, bar_a, kb * 64, 0, h, b);
    }
    mbar_expect_tx(bar_p, 2 * kTile);
    for (int kb = 0; kb < 2; ++kb) tma_load_4d(R3 + kb * kTile, &tmP, bar_p, kb * 64, 0, h, b);
  }
  const uint32_t R3_s = smem_u32(R3), R4_s = smem_u32(R4);
  {
    // dP_ext, read straight into the fragment's layout from global memory and issued before the wgmma so the loads
    // overlap it. Every element is read once by one thread, so a TMA tile (32 KB, which would still fit next to the
    // 193 KB of hd = 256) would buy no reuse. Elements at rows or columns >= S (the caller's row padding) read as zero:
    // P is zero there, but 0 * NaN would not be.
    uint32_t ext[EXT_DP ? 32 : 1];
    if (EXT_DP) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int q = f.r0 + 8 * hh;
        const bf16* erow = p.dPe + (((long long)b * p.H + h) * p.S + q) * p.ld_dpe;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int c = 8 * j + f.c0;
          uint32_t v = 0u;
          if (q < p.S && c < p.S) {
            v = __ldg(reinterpret_cast<const unsigned int*>(erow + c));
            if (c + 1 >= p.S) v &= 0xffffu;  // low half = column c
          }
          ext[16 * hh + j] = v;
        }
      }
    }
    mbar_wait(bar_a, 0);
    float dp[64];
    wg_mma<128, false, false>(dp, f.wg, smem_u32(R1), smem_u32(R2), nhb);  // dP[q,k] = dO V^T
    if (EXT_DP) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float2 e = bf16x2_to_f32(ext[16 * hh + j]);
          dp[4 * j + 2 * hh] += e.x;
          dp[4 * j + 2 * hh + 1] += e.y;
        }
    }
    // ---- dS = P * (dP - rowsum(dP * P)) / sqrt(hd); P as loaded by TMA (zeros beyond S) ----
    mbar_wait(bar_p, 0);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int q = f.r0 + 8 * hh;
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float2 pr = ld_pair(R3_s + operand_off(q, 8 * j + f.c0));
        acc += dp[4 * j + 2 * hh] * pr.x + dp[4 * j + 2 * hh + 1] * pr.y;
      }
      acc = quad_sum(acc);
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const uint32_t off = operand_off(q, 8 * j + f.c0);
        const float2 pr = ld_pair(R3_s + off);
        st_pair(R4_s + off, pr.x * (dp[4 * j + 2 * hh] - acc) * p.scale, pr.y * (dp[4 * j + 2 * hh + 1] - acc) * p.scale);
      }
    }
  }
  const long long HDall = (long long)p.H * HD;
  bf16* gbase = p.dqkv + (long long)b * p.S * p.ld_dqkv + (long long)h * HD;
  {
    float dv[HD / 2];
    wg_mma<HD, true, true>(dv, f.wg, R3_s, smem_u32(R1), 2);  // dV[k,:] = P^T dO  (K = queries)
    store_rows<HD>(f, dv, gbase + 2 * HDall, p.ld_dqkv, p.S, nullptr, 0);
  }
  fence_async_smem();
  __syncthreads();  // dS complete in smem (all rows); dO and V no longer read by either warpgroup
  if (t == 0) {
    mbar_expect_tx(bar_k, nhb * kTile);
    for (int kb = 0; kb < nhb; ++kb) tma_load_4d(R2 + kb * kTile, &tmK, bar_k, kb * 64, 0, h, b);
    mbar_expect_tx(bar_q, nhb * kTile);
    for (int kb = 0; kb < nhb; ++kb) tma_load_4d(R1 + kb * kTile, &tmQ, bar_q, kb * 64, 0, h, b);
  }
  {
    mbar_wait(bar_k, 0);
    float dq[HD / 2];
    wg_mma<HD, false, true>(dq, f.wg, R4_s, smem_u32(R2), 2);  // dQ[q,:] = dS K      (K = keys)
    store_rows<HD>(f, dq, gbase, p.ld_dqkv, p.S, p.rope_tab, p.rot);
  }
  {
    mbar_wait(bar_q, 0);
    float dk[HD / 2];
    wg_mma<HD, true, true>(dk, f.wg, R4_s, smem_u32(R1), 2);  // dK[k,:] = dS^T Q  (K = queries)
    store_rows<HD>(f, dk, gbase + HDall, p.ld_dqkv, p.S, p.rope_tab, p.rot);
  }
}

// ---------------------------------------------------------------------------------------------
// multi-tile forward (any Sq / Sk, causal with a key offset or not): one CTA per (128-query tile, head, batch)
// ---------------------------------------------------------------------------------------------
// Same numerics as the single-tile kernel and as the reference's materialised softmax (fp32 scores from bf16 q,k,
// softmax over the WHOLE key row in fp32, probabilities rounded to bf16 before P*V — hf:gptj/modeling_gptj.py:136-149,
// hf:clip/modeling_clip.py:282-330), obtained with two sweeps over the key tiles instead of an online rescale:
//   sweep 1: S_j = Q K_j^T per 128-key tile, running row maximum m and sum l = sum exp(s - m)          (no V, no O)
//   sweep 2: S_j again, p = bf16(exp(s - m) / l) exactly as the materialised path rounds it, O += P_j V_j in registers
// so O never needs rescaling and P — when the caller wants it for the backward pass — is rounded where
// softmax_fwd_kernel rounds it. The two sum exp(s - m) in different orders (per-tile quad sums with a running rescale
// here, lane-strided warp sums there), so 1 / sum can differ in its last bits and a bf16 rounding can flip: rare
// one-ulp differences (on an H100: 14 of 2.1 M probabilities at the ViT shape, 80 of 16.8 M at GPT-J S = 2048). QK^T is computed twice: +50 % of the attention FLOPs, which are < 1 % of the
// step, in exchange for no [B,H,S,S] fp32 score buffer. K / V tiles are double-buffered (TMA of tile j+1 under the
// softmax of tile j) when head_dim <= 128; at head_dim 256 one buffer each fits next to Q and P (224 KB) and the next
// tile is prefetched into L2 instead.
struct FlashParams {
  int Sq, Sk, H, hd, causal, kv_off;  // key j visible to query i iff j < Sk and (!causal or j <= i + kv_off)
  float scale;
  bf16* O;             // [B,Sq,H,hd], row stride ldo
  long long ldo;
  bf16* P;             // optional [B,H,Sq,ldP] (columns >= Sk up to ldP are written as zeros)
  long long ldP;
  float2* stats;       // optional [B,H,Sq] (row max of the scaled scores, 1 / sum)
};

template <int HD, int NBUF>
__global__ void __launch_bounds__(kAttThreads, 1)
attn_fwd_flash_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                      const __grid_constant__ CUtensorMap tmV, const FlashParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int nhb = HD / 64;
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + nhb * kTile;            // NBUF buffers
  uint8_t* sV = sK + NBUF * nhb * kTile;     // NBUF buffers
  uint8_t* sP = sV + NBUF * nhb * kTile;     // 2 k-blocks of 64 keys
  uint64_t* bars = reinterpret_cast<uint64_t*>(sP + 2 * kTile);
  uint64_t* bar_q = bars + 0;
  uint64_t* bar_k = bars + 1;   // [2]
  uint64_t* bar_v = bars + 3;   // [2]

  const int t = threadIdx.x;
  const int q0 = blockIdx.x * 128, h = blockIdx.y, b = blockIdx.z;
  const Frag f;

  pdl_trigger();
  if (t == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    for (int i = 0; i < 5; ++i) mbar_init(&bars[i], 1);
    mbar_fence_init();
  }
  __syncthreads();
  pdl_wait();

  // key tiles this query tile looks at
  int n_kv = (p.Sk + 127) >> 7;
  if (p.causal) {
    const int last_key = min(p.Sk - 1, q0 + 127 + p.kv_off);
    n_kv = last_key < 0 ? 0 : min(n_kv, (last_key >> 7) + 1);
  }
  int row_lim[2];  // keys [0, row_lim) are visible to this thread's two rows
  bool row_ok[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int qi = q0 + f.r0 + 8 * hh;
    row_lim[hh] = !p.causal ? p.Sk : min(p.Sk, qi + p.kv_off + 1);
    row_ok[hh] = qi < p.Sq;
  }

  uint32_t ph_k[2] = {0, 0}, ph_v[2] = {0, 0};
  auto load_k = [&](int j, int buf) {
    mbar_expect_tx(&bar_k[buf], nhb * kTile);
    for (int kb = 0; kb < nhb; ++kb) tma_load_4d(sK + (buf * nhb + kb) * kTile, &tmK, &bar_k[buf], kb * 64, j * 128, h, b);
  };
  auto load_v = [&](int j, int buf) {
    mbar_expect_tx(&bar_v[buf], nhb * kTile);
    for (int kb = 0; kb < nhb; ++kb) tma_load_4d(sV + (buf * nhb + kb) * kTile, &tmV, &bar_v[buf], kb * 64, j * 128, h, b);
  };

  // ---------------- sweep 1: row maximum and sum ----------------
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  if (t == 0 && n_kv > 0) {
    mbar_expect_tx(bar_q, nhb * kTile);
    for (int kb = 0; kb < nhb; ++kb) tma_load_4d(sQ + kb * kTile, &tmQ, bar_q, kb * 64, q0, h, b);
    load_k(0, 0);
  }
  if (n_kv > 0) mbar_wait(bar_q, 0);
  float s[64];
  for (int j = 0; j < n_kv; ++j) {
    const int buf = NBUF == 2 ? (j & 1) : 0;
    if (t == 0) {
      if (NBUF == 2 && j + 1 < n_kv) load_k(j + 1, (j + 1) & 1);  // its previous user (tile j-1) has completed
      if (NBUF == 1 && j + 1 < n_kv)
        for (int kb = 0; kb < nhb; ++kb) tma_prefetch_4d(&tmK, kb * 64, (j + 1) * 128, h, b);
    }
    mbar_wait(&bar_k[buf], ph_k[buf]);
    ph_k[buf] ^= 1;
    wg_mma<128, false, false>(s, f.wg, smem_u32(sQ), smem_u32(sK + buf * nhb * kTile), nhb);
    __syncthreads();  // both warpgroups are done with K_j
    if (NBUF == 1 && t == 0 && j + 1 < n_kv) load_k(j + 1, 0);
    const int kbase = j * 128;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float cm = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (kbase + 8 * jj + f.c0 + e < row_lim[hh]) cm = fmaxf(cm, s[4 * jj + 2 * hh + e] * p.scale);
      cm = quad_max(cm);
      if (cm > m[hh]) {  // rescale the running sum to the new maximum
        l[hh] *= __expf(m[hh] - cm);
        m[hh] = cm;
      }
      if (m[hh] != -INFINITY) {
        float ls = 0.f;
#pragma unroll
        for (int jj = 0; jj < 16; ++jj)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (kbase + 8 * jj + f.c0 + e < row_lim[hh]) ls += __expf(s[4 * jj + 2 * hh + e] * p.scale - m[hh]);
        l[hh] += quad_sum(ls);
      }
    }
  }
  float inv[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    inv[hh] = (row_ok[hh] && l[hh] > 0.f) ? 1.f / l[hh] : 0.f;
    if (m[hh] == -INFINITY) m[hh] = 0.f;
    if (p.stats != nullptr && row_ok[hh] && f.quad0)
      p.stats[((long long)b * p.H + h) * p.Sq + q0 + f.r0 + 8 * hh] = make_float2(m[hh], inv[hh]);
  }

  // ---------------- sweep 2: probabilities and O = P V ----------------
  const uint32_t sP_s = smem_u32(sP);
  if (t == 0 && n_kv > 0) {
    load_k(0, 0);  // buffer 0's last user completed before the last __syncthreads of sweep 1
    load_v(0, 0);
  }
  float o[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
  for (int j = 0; j < n_kv; ++j) {
    const int buf = NBUF == 2 ? (j & 1) : 0;
    if (t == 0) {
      if (NBUF == 2 && j + 1 < n_kv) {
        load_k(j + 1, (j + 1) & 1);
        load_v(j + 1, (j + 1) & 1);   // V_{j-1} (same buffer) was consumed by the PV of tile j-1 (synchronised below)
      }
      if (NBUF == 1 && j + 1 < n_kv)
        for (int kb = 0; kb < nhb; ++kb) {
          tma_prefetch_4d(&tmK, kb * 64, (j + 1) * 128, h, b);
          tma_prefetch_4d(&tmV, kb * 64, (j + 1) * 128, h, b);
        }
    }
    mbar_wait(&bar_k[buf], ph_k[buf]);
    ph_k[buf] ^= 1;
    wg_mma<128, false, false>(s, f.wg, smem_u32(sQ), smem_u32(sK + buf * nhb * kTile), nhb);
    __syncthreads();  // both warpgroups are done with K_j
    if (NBUF == 1 && t == 0 && j + 1 < n_kv) load_k(j + 1, 0);
    const int kbase = j * 128;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int r = f.r0 + 8 * hh;
      bf16* prow = p.P ? p.P + (((long long)b * p.H + h) * p.Sq + q0 + r) * p.ldP : nullptr;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        const int c = 8 * jj + f.c0;
        float a[2];
#pragma unroll
        for (int e = 0; e < 2; ++e)
          a[e] = kbase + c + e < row_lim[hh] ? __expf(s[4 * jj + 2 * hh + e] * p.scale - m[hh]) * inv[hh] : 0.f;
        st_pair(sP_s + operand_off(r, c), a[0], a[1]);
        if (prow != nullptr && row_ok[hh] && kbase + c < p.ldP)
          *reinterpret_cast<uint32_t*>(prow + kbase + c) = f32x2_to_bf16(a[0], a[1]);
      }
    }
    fence_async_smem();
    wg_sync(f.wg);  // this warpgroup's rows of P_j are complete
    mbar_wait(&bar_v[buf], ph_v[buf]);
    ph_v[buf] ^= 1;
    wg_mma<HD, false, true>(o, f.wg, sP_s, smem_u32(sV + buf * nhb * kTile), 2, 1u);  // O += P_j V_j
    __syncthreads();  // both warpgroups are done with V_j (and with this P_j)
    if (NBUF == 1 && t == 0 && j + 1 < n_kv) load_v(j + 1, 0);
  }
  // ---------------- O -> bf16 -> global ----------------
  store_rows<HD>(f, o, p.O + ((long long)b * p.Sq + q0) * p.ldo + (long long)h * HD, p.ldo, p.Sq - q0, nullptr, 0);
  // rows of P beyond this tile's last key tile (causal) are zeros in the materialised layout
  if (p.P != nullptr && t < 128 && q0 + t < p.Sq) {
    bf16* prow = p.P + (((long long)b * p.H + h) * p.Sq + q0 + t) * p.ldP;
    for (int col = n_kv * 128; col < p.ldP; col += 8) *reinterpret_cast<uint4*>(prow + col) = make_uint4(0, 0, 0, 0);
  }
}

// ---------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------
static int tile_map(CUtensorMap* m, const void* ptr, long long ld, long long bs0, long long bs1, int rows, int cols,
                    int H, int B) {
  mb200_operand op;
  op.ptr = ptr;
  op.ld = ld;
  op.bs0 = bs0;
  op.bs1 = bs1;
  op.mn_major = 0;
  op.static_data = 0;
  return make_operand_map(m, op, rows, cols, H, B, 128);
}

static constexpr int smem_max = 232448;  // 227 KB: the sm_90 per-block opt-in limit

bool attn_tile_supported(int S, int hd) { return S >= 1 && S <= 128 && hd >= 64 && hd <= 256 && hd % 64 == 0; }

int attn_fwd_tile(const bf16* qkv, long long ld_qkv, bf16* P, long long ldP, bf16* O, long long ldo, int B, int S, int H,
                  int hd, cudaStream_t st) {
  MB_REQUIRE(attn_tile_supported(S, hd) && ldP % 8 == 0, MB200_E_SHAPE, "attn_fwd_tile: unsupported S=%d hd=%d", S, hd);
  CUtensorMap tq, tk, tv;
  const long long d = (long long)H * hd;
  int rc;
  if ((rc = tile_map(&tq, qkv, ld_qkv, hd, (long long)S * ld_qkv, S, hd, H, B))) return rc;
  if ((rc = tile_map(&tk, qkv + d, ld_qkv, hd, (long long)S * ld_qkv, S, hd, H, B))) return rc;
  if ((rc = tile_map(&tv, qkv + 2 * d, ld_qkv, hd, (long long)S * ld_qkv, S, hd, H, B))) return rc;
  AttnParams p;
  memset(&p, 0, sizeof(p));
  p.S = S;
  p.H = H;
  p.hd = hd;
  p.scale = 1.0f / sqrtf((float)hd);
  p.P = P;
  p.ldP = ldP;
  p.O = O;
  p.ldo = ldo;
  const int smem = (3 * (hd / 64) + 2) * kTile + 1024 + 128;
#define MB_FWD(HD)                                                                                                   \
  {                                                                                                                  \
    static bool set = false;                                                                                         \
    if (!set) {                                                                                                      \
      MB_CUDA(cudaFuncSetAttribute(attn_fwd_tile_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max)); \
      set = true;                                                                                                    \
    }                                                                                                                \
    MB_CUDA(launch_pdl(attn_fwd_tile_kernel<HD>, dim3(B * H), dim3(kAttThreads), (size_t)smem, st, tq, tk, tv, p));  \
  }
  switch (hd) {
    case 64: MB_FWD(64) break;
    case 128: MB_FWD(128) break;
    case 192: MB_FWD(192) break;
    default: MB_FWD(256) break;
  }
#undef MB_FWD
  count_launch();
  return 0;
}

// dPe (NULL, or the bf16 [B,H,S,ld_dpe] gradient on P) selects the instantiation that adds it to dP
int attn_bwd_tile(const bf16* qkv, long long ld_qkv, const bf16* dO, long long ld_do, const bf16* P, long long ldP,
                  const bf16* dPe, long long ld_dpe, bf16* dqkv, long long ld_dqkv, const float* rope_tab, int rot, int B,
                  int S, int H, int hd, cudaStream_t st) {
  MB_REQUIRE(attn_tile_supported(S, hd) && ldP % 8 == 0, MB200_E_SHAPE, "attn_bwd_tile: unsupported S=%d hd=%d", S, hd);
  MB_REQUIRE(dPe == nullptr || (ld_dpe >= S && ld_dpe % 8 == 0 && (reinterpret_cast<uintptr_t>(dPe) & 3) == 0),
             MB200_E_ALIGN, "attn_bwd_tile_dp: ld_dpe=%lld must be >= S and %%8, dP_ext 4-byte aligned", ld_dpe);
  CUtensorMap tq, tk, tv, tdo, tp;
  const long long d = (long long)H * hd;
  int rc;
  if ((rc = tile_map(&tq, qkv, ld_qkv, hd, (long long)S * ld_qkv, S, hd, H, B))) return rc;
  if ((rc = tile_map(&tk, qkv + d, ld_qkv, hd, (long long)S * ld_qkv, S, hd, H, B))) return rc;
  if ((rc = tile_map(&tv, qkv + 2 * d, ld_qkv, hd, (long long)S * ld_qkv, S, hd, H, B))) return rc;
  if ((rc = tile_map(&tdo, dO, ld_do, hd, (long long)S * ld_do, S, hd, H, B))) return rc;
  if ((rc = tile_map(&tp, P, ldP, (long long)S * ldP, (long long)H * S * ldP, S, S, H, B))) return rc;
  AttnParams p;
  memset(&p, 0, sizeof(p));
  p.S = S;
  p.H = H;
  p.hd = hd;
  p.rot = rot;
  p.scale = 1.0f / sqrtf((float)hd);
  p.P = const_cast<bf16*>(P);
  p.ldP = ldP;
  p.dqkv = dqkv;
  p.ld_dqkv = ld_dqkv;
  p.rope_tab = reinterpret_cast<const float2*>(rope_tab);
  p.dPe = dPe;
  p.ld_dpe = ld_dpe;
  const int smem = (2 * (hd / 64) + 4) * kTile + 1024 + 128;
#define MB_BWD(HD, EXT)                                                                                               \
  {                                                                                                                  \
    static bool set = false;                                                                                         \
    if (!set) {                                                                                                      \
      MB_CUDA(cudaFuncSetAttribute(attn_bwd_tile_kernel<HD, EXT>, cudaFuncAttributeMaxDynamicSharedMemorySize,       \
                                   smem_max));                                                                       \
      set = true;                                                                                                    \
    }                                                                                                                \
    MB_CUDA(launch_pdl(attn_bwd_tile_kernel<HD, EXT>, dim3(B * H), dim3(kAttThreads), (size_t)smem, st, tq, tk, tv,  \
                       tdo, tp, p));                                                                                 \
  }
  if (dPe == nullptr) {
    switch (hd) {
      case 64: MB_BWD(64, false) break;
      case 128: MB_BWD(128, false) break;
      case 192: MB_BWD(192, false) break;
      default: MB_BWD(256, false) break;
    }
  } else {
    switch (hd) {
      case 64: MB_BWD(64, true) break;
      case 128: MB_BWD(128, true) break;
      case 192: MB_BWD(192, true) break;
      default: MB_BWD(256, true) break;
    }
  }
#undef MB_BWD
  count_launch();
  return 0;
}

// Multi-tile forward. q / k / v: element pointers of head 0, batch 0, row 0 with row stride ld*, head stride *_bsh and
// batch stride *_bsb (elements) — the fused qkv buffer (ld = 3d, bsh = hd, bsb = S * 3d) or a KV cache
// [B,H,Smax,hd] (ld = hd, bsh = Smax * hd, bsb = H * Smax * hd). Causal: key j is visible to query i iff
// j <= i + (Sk - Sq) (queries are the LAST Sq positions of the Sk keys — prefill and its continuations).
bool attn_flash_supported(int hd) { return hd >= 64 && hd <= 256 && hd % 64 == 0; }

int attn_fwd_flash(const bf16* q, long long ldq, long long q_bsh, long long q_bsb, const bf16* k, long long ldk,
                   long long k_bsh, long long k_bsb, const bf16* v, long long ldv, long long v_bsh, long long v_bsb,
                   bf16* O, long long ldo, bf16* P, long long ldP, float* stats, int B, int Sq, int Sk, int H, int hd,
                   int causal, cudaStream_t st) {
  MB_REQUIRE(attn_flash_supported(hd) && Sq >= 1 && Sk >= 1 && B >= 1 && H >= 1, MB200_E_SHAPE,
             "attn_fwd_flash: unsupported Sq=%d Sk=%d hd=%d", Sq, Sk, hd);
  MB_REQUIRE(!causal || Sk >= Sq, MB200_E_SHAPE, "attn_fwd_flash: causal needs Sk >= Sq (%d < %d)", Sk, Sq);
  MB_REQUIRE(P == nullptr || (ldP % 8 == 0 && ldP >= Sk), MB200_E_ALIGN, "attn_fwd_flash: ldP=%lld must be >= Sk and %%8",
             ldP);
  MB_REQUIRE(ldo % 8 == 0 && (reinterpret_cast<uintptr_t>(O) & 15) == 0, MB200_E_ALIGN, "attn_fwd_flash: O alignment");
  CUtensorMap tq, tk, tv;
  int rc;
  if ((rc = tile_map(&tq, q, ldq, q_bsh, q_bsb, Sq, hd, H, B))) return rc;
  if ((rc = tile_map(&tk, k, ldk, k_bsh, k_bsb, Sk, hd, H, B))) return rc;  // rows = Sk: cache rows beyond are OOB zeros
  if ((rc = tile_map(&tv, v, ldv, v_bsh, v_bsb, Sk, hd, H, B))) return rc;
  FlashParams p;
  memset(&p, 0, sizeof(p));
  p.Sq = Sq;
  p.Sk = Sk;
  p.H = H;
  p.hd = hd;
  p.causal = causal;
  p.kv_off = Sk - Sq;
  p.scale = 1.0f / sqrtf((float)hd);
  p.O = O;
  p.ldo = ldo;
  p.P = P;
  p.ldP = ldP;
  p.stats = reinterpret_cast<float2*>(stats);
  const dim3 grid((Sq + 127) / 128, H, B);
  // K / V double-buffered up to head_dim 128; one buffer each at 192 / 256 (smem)
#define MB_FLASH(HD, NB)                                                                                             \
  {                                                                                                                  \
    const int smem = ((1 + 2 * NB) * (HD / 64) + 2) * kTile + 1024 + 128;                                           \
    static bool set = false;                                                                                         \
    if (!set) {                                                                                                      \
      MB_CUDA(cudaFuncSetAttribute(attn_fwd_flash_kernel<HD, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize,      \
                                   smem_max));                                                                       \
      set = true;                                                                                                    \
    }                                                                                                                \
    MB_CUDA(launch_pdl(attn_fwd_flash_kernel<HD, NB>, grid, dim3(kAttThreads), (size_t)smem, st, tq, tk, tv, p));    \
  }
  switch (hd) {
    case 64: MB_FLASH(64, 2) break;
    case 128: MB_FLASH(128, 2) break;
    case 192: MB_FLASH(192, 1) break;
    default: MB_FLASH(256, 1) break;
  }
#undef MB_FLASH
  count_launch();
  return 0;
}

}  // namespace mb200

// C ABI (exposed for the parity tests; the engine calls the C++ functions directly)
extern "C" int mb200_attn_fwd_tile(const void* qkv, int64_t ld_qkv, void* P, int64_t ldP, void* O, int64_t ldo, int32_t B,
                                   int32_t S, int32_t H, int32_t hd, void* stream) {
  int rc = mb200::check_arch();
  if (rc) return rc;
  return mb200::attn_fwd_tile((const mb200::bf16*)qkv, ld_qkv, (mb200::bf16*)P, ldP, (mb200::bf16*)O, ldo, B, S, H, hd,
                              (cudaStream_t)stream);
}

extern "C" int mb200_attn_bwd_tile(const void* qkv, int64_t ld_qkv, const void* dO, int64_t ld_do, const void* P,
                                   int64_t ldP, void* dqkv, int64_t ld_dqkv, const float* rope_tab, int32_t rot,
                                   int32_t B, int32_t S, int32_t H, int32_t hd, void* stream) {
  int rc = mb200::check_arch();
  if (rc) return rc;
  return mb200::attn_bwd_tile((const mb200::bf16*)qkv, ld_qkv, (const mb200::bf16*)dO, ld_do, (const mb200::bf16*)P, ldP,
                              nullptr, 0, (mb200::bf16*)dqkv, ld_dqkv, rope_tab, rot, B, S, H, hd, (cudaStream_t)stream);
}

extern "C" int mb200_attn_bwd_tile_dp(const void* qkv, int64_t ld_qkv, const void* dO, int64_t ld_do, const void* P,
                                      int64_t ldP, const void* dP_ext, int64_t ld_dpe, void* dqkv, int64_t ld_dqkv,
                                      const float* rope_tab, int32_t rot, int32_t B, int32_t S, int32_t H, int32_t hd,
                                      void* stream) {
  int rc = mb200::check_arch();
  if (rc) return rc;
  MB_REQUIRE(dP_ext != nullptr, MB200_E_ARG, "attn_bwd_tile_dp: dP_ext is NULL");
  return mb200::attn_bwd_tile((const mb200::bf16*)qkv, ld_qkv, (const mb200::bf16*)dO, ld_do, (const mb200::bf16*)P, ldP,
                              (const mb200::bf16*)dP_ext, ld_dpe, (mb200::bf16*)dqkv, ld_dqkv, rope_tab, rot, B, S, H, hd,
                              (cudaStream_t)stream);
}

extern "C" int mb200_attn_fwd_flash(const void* q, int64_t ldq, int64_t q_bsh, int64_t q_bsb, const void* k, int64_t ldk,
                                    int64_t k_bsh, int64_t k_bsb, const void* v, int64_t ldv, int64_t v_bsh, int64_t v_bsb,
                                    void* O, int64_t ldo, void* P, int64_t ldP, float* stats, int32_t B, int32_t Sq,
                                    int32_t Sk, int32_t H, int32_t hd, int32_t causal, void* stream) {
  int rc = mb200::check_arch();
  if (rc) return rc;
  return mb200::attn_fwd_flash((const mb200::bf16*)q, ldq, q_bsh, q_bsb, (const mb200::bf16*)k, ldk, k_bsh, k_bsb,
                               (const mb200::bf16*)v, ldv, v_bsh, v_bsb, (mb200::bf16*)O, ldo, (mb200::bf16*)P, ldP, stats,
                               B, Sq, Sk, H, hd, causal, (cudaStream_t)stream);
}
