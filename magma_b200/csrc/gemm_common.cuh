// magma_b200 — pieces shared by the GEMM core (gemm.cu) and the fused attention kernels (attention.cu): tile
// configuration, kernel parameter block and the fused epilogue applied to wgmma accumulator fragments.
#pragma once
#include <type_traits>

#include "common.cuh"

namespace mb200 {

static constexpr int BM = 128;        // tile M: two consumer warpgroups x wgmma M = 64
static constexpr int BK = 64;         // 64 bf16 = 128 bytes = one SWIZZLE_128B row
static constexpr int WG_K = 16;       // wgmma K for 16-bit inputs
static constexpr int kThreads = 384;  // warpgroup 0 = TMA producer, warpgroups 1, 2 = MMA + epilogue
static constexpr int kEpiCols = 64;  // epilogue staging chunk: BM x 64 fp32, 64 rows per consumer warpgroup
static constexpr int kEpiBytes = BM * kEpiCols * 4;
static constexpr int kEpiBoxBytes = BM * kEpiCols * 2;  // one TMA box of an [M, N] epilogue input: BM x 64 bf16
static constexpr int kSmemBudget = 192 * 1024;  // operand ring; + staging, alignment slack and barriers <= 227 KB

template <int BN>
struct Cfg {
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStagesRaw = kSmemBudget / kStageBytes;
  static constexpr int kStages = kStagesRaw > 8 ? 8 : kStagesRaw;
  static constexpr int kSmemBytes = kStages * kStageBytes + kEpiBytes + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(kSmemBytes <= 227 * 1024, "GEMM shared memory exceeds the sm_90 per-block limit");
  // Epilogue-input boxes one ring stage holds: the first fills the A slot, the others the B slot.
  static constexpr int kEpiBoxesPerStage = 1 + kBBytes / kEpiBoxBytes;
  static_assert(kABytes == kEpiBoxBytes && kEpiBoxesPerStage * kEpiBoxBytes <= kStageBytes, "epilogue box layout");
  // A tile's three inputs fit in the ring at once, so the producer never waits on a slot the same tile's epilogue
  // still has to release.
  static_assert(3 * (BN / kEpiCols) <= kStages * kEpiBoxesPerStage, "epilogue inputs exceed the operand ring");
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
  // Number of [M, N] epilogue inputs (aux_in when dact, res1, res2, in that order) that the producer stages by TMA
  // through the operand ring after each tile's last k-block; 0: the epilogue reads them from global memory.
  int epi_in;
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

__device__ __forceinline__ float2 bf16x2_to_f32(uint32_t u) {
  return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u));
}
__device__ __forceinline__ uint32_t f32x2_to_bf16(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// n (<= 4) consecutive bf16 -> fp32 (missing elements read as 0): one 8-byte read-only load when all four are in range
// and 8-byte aligned (operand pointers other than C carry no alignment guarantee beyond the element). kVec: the caller
// knows both hold, and only the vector access is compiled.
template <bool kVec = false>
__device__ __forceinline__ void ld_bf16x4(const bf16* src, int n, float (&v)[4]) {
  if (kVec || (n == 4 && (reinterpret_cast<uintptr_t>(src) & 7) == 0)) {
    uint32_t u0, u1;
    asm volatile("ld.global.nc.v2.u32 {%0, %1}, [%2];" : "=r"(u0), "=r"(u1) : "l"(src));
    const float2 a = bf16x2_to_f32(u0), b = bf16x2_to_f32(u1);
    v[0] = a.x;
    v[1] = a.y;
    v[2] = b.x;
    v[3] = b.y;
  } else {
#pragma unroll
    for (int e = 0; e < 4; ++e) v[e] = e < n ? __bfloat162float(src[e]) : 0.f;
  }
}
template <bool kVec = false>
__device__ __forceinline__ void st_bf16x4(bf16* dst, int n, const float (&v)[4]) {
  if (kVec || (n == 4 && (reinterpret_cast<uintptr_t>(dst) & 7) == 0)) {
    *reinterpret_cast<uint2*>(dst) = make_uint2(f32x2_to_bf16(v[0], v[1]), f32x2_to_bf16(v[2], v[3]));
  } else {
#pragma unroll
    for (int e = 0; e < 4; ++e)
      if (e < n) dst[e] = __float2bfloat16(v[e]);
  }
}

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

enum { EK_GENERIC = 0, EK_SPLITK };

// ---------------------------------------------------------------------------------------------
// Epilogue form: which features the epilogue of a kernel instantiation is compiled for. The epilogue code below asks
// the form, not GemmKernelParams, whether a feature is in use. EF_RUNTIME answers every question from the parameters
// (any feature set, any alignment; also what the split-K kernels run). Any other form is a fixed set of EF_ bits and
// answers from constants, so the code of the features it lacks is not generated, every access is a vector (the host
// checks the alignments, epi_form in gemm.cu) and the row loop can be unrolled. Values (alpha, the rotary direction,
// whether an fp32 store accumulates) stay parameters in every form.
// ---------------------------------------------------------------------------------------------
enum : uint32_t {
  EF_BIAS = 1,
  EF_ROPE = 2,
  EF_AUX_OUT = 4,
  EF_GELU = 8,    // act == MB200_ACT_GELU_NEW
  EF_DGELU = 16,  // dact == MB200_DACT_GELU_NEW
  EF_RES1 = 32,
  EF_RES2 = 64,
  EF_F32 = 128,
  EF_QGELU = 256,  // act == MB200_ACT_QUICK_GELU
  EF_RUNTIME = 1u << 31
};

template <uint32_t F>
struct EpiForm {
  static constexpr bool kRuntime = F == EF_RUNTIME;
  // [M, N] inputs (aux_in, res1, res2) of a compiled form; all of them are staged by TMA
  static constexpr int kInputs = kRuntime ? 0 : ((F & EF_DGELU) != 0) + ((F & EF_RES1) != 0) + ((F & EF_RES2) != 0);
  // Rows of a chunk in flight per thread: the accumulators (BN / 2 registers) are live until the last chunk is staged,
  // which leaves room for 8 rows of fp32 values and their inputs at BN = 256.
  static constexpr int kRows = kRuntime ? 1 : 8;
  using P = GemmKernelParams;
  static __device__ __forceinline__ bool bias(const P& p) { return kRuntime ? p.bias != nullptr : (F & EF_BIAS) != 0; }
  static __device__ __forceinline__ bool rope(const P& p) { return kRuntime ? p.rope_mode != 0 : (F & EF_ROPE) != 0; }
  static __device__ __forceinline__ bool aux_out(const P& p) {
    return kRuntime ? p.aux_out != nullptr : (F & EF_AUX_OUT) != 0;
  }
  static __device__ __forceinline__ int act(const P& p) {
    return kRuntime ? p.act
           : (F & EF_GELU) ? MB200_ACT_GELU_NEW
           : (F & EF_QGELU) ? MB200_ACT_QUICK_GELU
                            : MB200_ACT_NONE;
  }
  static __device__ __forceinline__ int dact(const P& p) {
    return kRuntime ? p.dact : (F & EF_DGELU) ? MB200_DACT_GELU_NEW : MB200_DACT_NONE;
  }
  static __device__ __forceinline__ bool res1(const P& p) { return kRuntime ? p.res1 != nullptr : (F & EF_RES1) != 0; }
  static __device__ __forceinline__ bool res2(const P& p) { return kRuntime ? p.res2 != nullptr : (F & EF_RES2) != 0; }
  static __device__ __forceinline__ bool c_f32(const P& p) { return kRuntime ? p.c_f32 != 0 : (F & EF_F32) != 0; }
  static __device__ __forceinline__ bool accumulate(const P& p) { return (kRuntime || (F & EF_F32)) && p.accumulate; }
  static __device__ __forceinline__ bool splitk(const P& p) { return kRuntime && p.epi_kind == EK_SPLITK; }
};

// [M, N] epilogue inputs of one 4-column group: aux_in, res1, res2. A field is filled only when its input is in use.
struct EpiIn {
  float aux[4], res1[4], res2[4];
};

// aux_in / res1 / res2 of columns [col, col + 4) of one row, from global memory
template <class Form>
__device__ __forceinline__ void epi_load_inputs(const GemmKernelParams& p, long long boff, int row, int col,
                                                EpiIn& in) {
  const int n = min(4, p.N - col);
  if (Form::dact(p)) ld_bf16x4(p.aux_in + boff + (long long)row * p.ldc + col, n, in.aux);
  const long long roff = boff + (long long)row * p.ld_res + col;
  if (Form::res1(p)) ld_bf16x4(p.res1 + roff, n, in.res1);
  if (Form::res2(p)) ld_bf16x4(p.res2 + roff, n, in.res2);
}

// 4 bf16 of a TMA-staged epilogue box -> fp32 (8-byte aligned; columns past N were zero-filled by TMA)
__device__ __forceinline__ void ld_smem_bf16x4(const uint8_t* src, float (&v)[4]) {
  const uint2 u = *reinterpret_cast<const uint2*>(src);
  const float2 a = bf16x2_to_f32(u.x), b = bf16x2_to_f32(u.y);
  v[0] = a.x;
  v[1] = a.y;
  v[2] = b.x;
  v[3] = b.y;
}

// ---------------------------------------------------------------------------------------------
// Fused epilogue of columns [col, col + 4) of one output row (col % 4 == 0, col < N, row < M); v holds alpha x the
// accumulators (or the summed split-K partials), `bias` and `in` the group's inputs. Applied in this order: bias, rotary,
// saved pre-activation (aux_out), activation, activation derivative (aux_in), residuals, ReLU-post, store (bf16, fp32 or
// fp32 accumulate). rope_hd, rope_rot and rope_ncols are multiples of 4, so both rotary pairs (col, col + 1),
// (col + 2, col + 3) of the group are rotated or neither is. Every branch on p is uniform across the kernel.
// kVec: all four columns exist and every tensor written is 8-byte aligned at them (see ld_bf16x4).
// ---------------------------------------------------------------------------------------------
template <class Form, bool kVec = false>
__device__ __forceinline__ void epi_store4(const GemmKernelParams& p, long long boff, int row, int col, float (&v)[4],
                                           const float (&bias)[4], const EpiIn& in) {
  const int n = min(4, p.N - col);
  if (Form::bias(p)) {
#pragma unroll
    for (int e = 0; e < 4; ++e) v[e] += bias[e];
  }
  if (Form::rope(p) && col < p.rope_ncols) {
    const int dim = col % p.rope_hd;
    if (dim < p.rope_rot) {
      const float2* tp = p.rope_tab + (long long)(row % p.rope_S) * (p.rope_rot >> 1) + (dim >> 1);
      const float2 cs0 = __ldg(tp), cs1 = __ldg(tp + 1);
      const float sg = p.rope_mode > 0 ? 1.f : -1.f;
      const float a0 = v[0], a1 = v[1], a2 = v[2], a3 = v[3];
      v[0] = a0 * cs0.x - a1 * cs0.y * sg;
      v[1] = a1 * cs0.x + a0 * cs0.y * sg;
      v[2] = a2 * cs1.x - a3 * cs1.y * sg;
      v[3] = a3 * cs1.x + a2 * cs1.y * sg;
    }
  }
  const long long coff = boff + (long long)row * p.ldc + col;
  if (Form::aux_out(p)) st_bf16x4<kVec>(p.aux_out + coff, n, v);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    if (Form::act(p) == MB200_ACT_GELU_NEW) v[e] = gelu_new_f(v[e]);
    else if (Form::act(p) == MB200_ACT_QUICK_GELU) v[e] = quick_gelu_f(v[e]);
    else if (Form::act(p) == MB200_ACT_RELU) v[e] = fmaxf(v[e], 0.f);
  }
  if (Form::dact(p)) {
#pragma unroll
    for (int e = 0; e < 4; ++e)
      v[e] = Form::dact(p) == MB200_DACT_GELU_NEW ? v[e] * gelu_new_grad_f(in.aux[e]) : (in.aux[e] > 0.f ? v[e] : 0.f);
  }
  if (Form::res1(p)) {
#pragma unroll
    for (int e = 0; e < 4; ++e) v[e] += in.res1[e];
  }
  if (Form::res2(p)) {
#pragma unroll
    for (int e = 0; e < 4; ++e) v[e] += in.res2[e];
  }
  if (Form::act(p) == MB200_ACT_RELU_POST) {
#pragma unroll
    for (int e = 0; e < 4; ++e) v[e] = fmaxf(v[e], 0.f);
  }
  if (Form::c_f32(p)) {  // C is 16-byte aligned and ldc, the batch strides and col are multiples of 4
    float* dst = reinterpret_cast<float*>(p.C) + coff;
    if (kVec || n == 4) {
      float4 o = make_float4(v[0], v[1], v[2], v[3]);
      if (Form::accumulate(p)) {
        const float4 old = *reinterpret_cast<const float4*>(dst);
        o.x += old.x;
        o.y += old.y;
        o.z += old.z;
        o.w += old.w;
      }
      *reinterpret_cast<float4*>(dst) = o;
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (e < n) dst[e] = Form::accumulate(p) ? dst[e] + v[e] : v[e];
    }
  } else {
    st_bf16x4<kVec>(reinterpret_cast<bf16*>(p.C) + coff, n, v);
  }
}

// ---------------------------------------------------------------------------------------------
// Epilogue of one consumer warpgroup's 64 x BN accumulator fragment (wgmma.cuh layout), 64 columns at a time. The
// fragment chunk is written to the warpgroup's 64 x 64 fp32 slice of the staging buffer; after a barrier over the
// warpgroup, a rolled loop hands each thread groups of 4 consecutive columns of a row (16 threads per row), so a warp's
// global loads and stores cover two contiguous 128-byte (bf16) or 256-byte (fp32) row segments, and one copy of the
// feature code serves every chunk. In the runtime form that loop takes one row per pass; in a compiled form (EpiForm) it
// takes Form::kRows rows, reading the staged values and inputs of all of them before the arithmetic and the stores, so
// that many independent load -> convert -> store chains are in flight per thread. Staging layout: row-major, 16-byte chunk q of row r stored at q ^ 2 (r & 3). A
// half-warp's 8-byte fragment writes (4 rows x 2 chunks) and a quarter-warp's 16-byte reads (8 chunks of one row) then
// fall on distinct banks.
// Split-K work items store alpha x the fp32 tile into their slice of the workspace instead (EK_SPLITK).
//
// In the EPI_TMA kernels (p.epi_in != 0) the tile's [M, N] inputs arrive through the operand ring (epi_queue_inputs): box b holds chunk
// b / epi_in of input b % epi_in, and ring item j (the j-th stage after the tile's last k-block) holds boxes
// [j kEpiBoxesPerStage, (j + 1) kEpiBoxesPerStage). Each chunk waits for the items holding its boxes and releases the
// items it has finished, so the producer refills them with the next tile's k-blocks while later chunks run.
// row0: first row (within the batch) of this warpgroup's 64-row slab; col0: first column of the tile;
// stage/phase: ring position of the first item, advanced past the tile's items
// ---------------------------------------------------------------------------------------------

// Operand ring as the epilogue sees it
struct EpiRing {
  uint8_t* a;  // A slots, Cfg::kABytes apart
  uint8_t* b;  // B slots, Cfg::kBBytes apart
  uint64_t* full;
  uint64_t* empty;
};

// Column chunks of the tile starting at col0 that hold columns < N; the producer fetches inputs for these only.
template <int BN>
__device__ __forceinline__ int epi_chunks(const GemmKernelParams& p, int col0) {
  return min(BN / kEpiCols, (p.N - col0 + kEpiCols - 1) / kEpiCols);
}

// Box k (< kEpiBoxesPerStage) of ring stage s
template <int BN>
__device__ __forceinline__ uint8_t* epi_box(const EpiRing& ring, int s, int k) {
  return k == 0 ? ring.a + s * Cfg<BN>::kABytes : ring.b + s * Cfg<BN>::kBBytes + (k - 1) * kEpiBoxBytes;
}

template <int BN, bool EPI_TMA, class Form>
__device__ __forceinline__ void epi_tile(const GemmKernelParams& p, const float (&acc)[BN / 2], float* stage,
                                         int bar_id, long long boff, int row0, int col0, int ks, const EpiRing& ring,
                                         int& ring_stage, uint32_t& ring_phase) {
  constexpr int kStages = Cfg<BN>::kStages, kBps = Cfg<BN>::kEpiBoxesPerStage;
  const int wt = threadIdx.x & 127;
  const int fr = (wt >> 5) * 16 + ((wt & 31) >> 2);  // fragment rows fr, fr + 8; column pair 2 (wt % 4) of each 8
  const int fq = wt & 3;
  const int pr = wt >> 4, pc = wt & 15;  // processing: rows pr + 8 i, 16-byte chunk pc
  const int nch = epi_chunks<BN>(p, col0);
  const int nin = !EPI_TMA ? 0 : Form::kRuntime ? p.epi_in : Form::kInputs;
  // cursor over the staged boxes: the next one is slot bk of stage bs (phase bph); stages before rs are released
  int bs = ring_stage, bk = 0, rs = ring_stage;
  uint32_t bph = ring_phase;
  auto next_box = [&]() {
    if (bk == 0) mbar_wait(&ring.full[bs], bph);
    const uint8_t* box = epi_box<BN>(ring, bs, bk);
    if (++bk == kBps) {
      bk = 0;
      if (++bs == kStages) {
        bs = 0;
        bph ^= 1;
      }
    }
    return box;
  };
  // Byte offset of this thread's 8 bytes (columns 4 pc .. 4 pc + 3) of row pr of its warpgroup's half of a box: in a
  // SWIZZLE_128B box, 16-byte unit u of row r sits at u ^ (r & 7); rows pr + 8 i share r & 7 and lie 1024 B apart.
  // A half-warp reads one 128-byte row: no bank conflicts.
  const int box_off = ((row0 % BM) + pr) * 128 + (((pc >> 1) ^ pr) << 4) + ((pc & 1) << 3);
#pragma unroll 1
  for (int ch = 0; ch < nch; ++ch) {
#pragma unroll
    for (int c = 0; c < BN / kEpiCols; ++c) {
      if (c != ch) continue;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int j = c * 8 + jj;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = fr + 8 * h;
          const int q = (2 * jj + (fq >> 1)) ^ ((r & 3) << 1);
          *reinterpret_cast<float2*>(stage + r * kEpiCols + q * 4 + 2 * (fq & 1)) =
              make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
      }
    }
    named_bar_sync(bar_id, 128);
    const int col = col0 + ch * kEpiCols + pc * 4;
    // this chunk's input boxes, in epi_in order: aux_in (dact), res1, res2
    const uint8_t *src_aux = nullptr, *src_res1 = nullptr, *src_res2 = nullptr;
    if (nin) {
      if (Form::dact(p)) src_aux = next_box() + box_off;
      if (Form::res1(p)) src_res1 = next_box() + box_off;
      if (Form::res2(p)) src_res2 = next_box() + box_off;
    }
    const int n = min(4, p.N - col);
    float bias[4];
    if (Form::bias(p) && col < p.N) ld_bf16x4(p.bias + col, n, bias);
    // rows pr + 8 i, i in [i0, i0 + kRows), of this thread's column group
    auto rows = [&](auto rows_c, auto vec_c, int i0) {
      constexpr int kRows = decltype(rows_c)::value;
      constexpr bool kVec = decltype(vec_c)::value;
      float4 s[kRows];
      EpiIn in[kRows];
#pragma unroll
      for (int u = 0; u < kRows; ++u) {
        const int i = i0 + u, r = pr + 8 * i;
        s[u] = *reinterpret_cast<const float4*>(stage + r * kEpiCols + ((pc ^ ((r & 3) << 1)) * 4));
        if (nin) {
          if (Form::dact(p)) ld_smem_bf16x4(src_aux + i * 1024, in[u].aux);
          if (Form::res1(p)) ld_smem_bf16x4(src_res1 + i * 1024, in[u].res1);
          if (Form::res2(p)) ld_smem_bf16x4(src_res2 + i * 1024, in[u].res2);
        }
      }
#pragma unroll
      for (int u = 0; u < kRows; ++u) {
        const int row = row0 + pr + 8 * (i0 + u);
        if (row >= p.M) continue;
        // __fmul_rn: never fused into the add of a following feature, so every form rounds alpha x acc on its own
        float v[4] = {__fmul_rn(s[u].x, p.alpha), __fmul_rn(s[u].y, p.alpha), __fmul_rn(s[u].z, p.alpha),
                      __fmul_rn(s[u].w, p.alpha)};
        if (Form::splitk(p)) {  // ld_ws % 4 == 0: the padded columns of the group exist
          *reinterpret_cast<float4*>(p.splitk_ws + ((long long)ks * p.M + row) * p.ld_ws + col) =
              make_float4(v[0], v[1], v[2], v[3]);
          continue;
        }
        if (!nin) epi_load_inputs<Form>(p, boff, row, col, in[u]);
        epi_store4<Form, kVec>(p, boff, row, col, v, bias, in[u]);
      }
    };
    if (col < p.N) {
      if (Form::kRuntime || n == 4) {
#pragma unroll 1
        for (int i0 = 0; i0 < 64 / 8; i0 += Form::kRows)
          rows(std::integral_constant<int, Form::kRows>(), std::integral_constant<bool, !Form::kRuntime>(), i0);
      } else {  // compiled form, the ragged group at the right edge of an N that is not a multiple of 4: guarded accesses
#pragma unroll 1
        for (int i0 = 0; i0 < 64 / 8; ++i0) rows(std::integral_constant<int, 1>(), std::false_type(), i0);
      }
    }
    named_bar_sync(bar_id, 128);  // the slice is rewritten by the next chunk; the items read so far may be refilled
    if (nin) {
      if (ch + 1 == nch && bk != 0) {  // the tile's last item may be partly filled: it is done too
        bk = 0;
        if (++bs == kStages) {
          bs = 0;
          bph ^= 1;
        }
      }
#pragma unroll 1
      for (; rs != bs; rs = rs + 1 == kStages ? 0 : rs + 1)  // rs trails bs by fewer than kStages items
        if (wt == 0) mbar_arrive(&ring.empty[rs]);
    }
  }
  ring_stage = bs;
  ring_phase = bph;
}

// Producer side: queues the tile's epilogue-input boxes (see epi_tile) as ring items after its last k-block.
// maps: one tensor map per input, in epi_in order; m0: first row, col0: first column of the tile.
template <int BN>
__device__ __forceinline__ void epi_queue_inputs(const GemmKernelParams& p, const CUtensorMap* maps,
                                                 const EpiRing& ring, int& stage, uint32_t& phase, int m0, int col0,
                                                 int z0, int z1) {
  constexpr int kStages = Cfg<BN>::kStages, kBps = Cfg<BN>::kEpiBoxesPerStage;
  const int nbox = p.epi_in * epi_chunks<BN>(p, col0);
  int col = col0, i = 0;  // box: input i, columns [col, col + 64)
#pragma unroll 1
  for (int b0 = 0; b0 < nbox; b0 += kBps) {
    const int nb = min(kBps, nbox - b0);
    mbar_wait(&ring.empty[stage], phase ^ 1);
    mbar_expect_tx(&ring.full[stage], (uint32_t)(nb * kEpiBoxBytes));  // out-of-range parts are zero-filled
#pragma unroll 1
    for (int k = 0; k < nb; ++k) {
      tma_load_4d(epi_box<BN>(ring, stage, k), &maps[i], &ring.full[stage], col, m0, z0, z1);
      if (++i == p.epi_in) {
        i = 0;
        col += kEpiCols;
      }
    }
    if (++stage == kStages) {
      stage = 0;
      phase ^= 1;
    }
  }
}

// host helper shared by gemm.cu / attention.cu
int make_operand_map(CUtensorMap* out, const mb200_operand& op, int rows, int K, int nb0, int nb1, int box_rows);

}  // namespace mb200
