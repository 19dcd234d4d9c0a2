// magma_b200 — bf16 GEMM core for sm_90a (Hopper).
//
//   C[b][M,N] = epilogue(alpha * A[b][M,K] * B[b][N,K]^T)
//
// Design (not a translation of anything in the reference, which only calls cuBLAS through torch.nn.Linear — e.g.
// magma/adapters.py:19-23, magma/image_prefix.py:72):
//   * persistent grid (<= one CTA per SM), static round-robin tile scheduler, m-fastest tile order so
//     CTAs that run concurrently share the same weight (B) tile through L2;
//   * warp-specialised: warpgroup 0 = TMA producer (one lane), warpgroups 1 and 2 = consumers, each owning 64 rows of
//     the 128-row tile: wgmma.mma_async m64nBNk16 with fp32 accumulators in registers, then the fused epilogue
//     straight from the accumulator fragment (gemm_common.cuh);
//   * operands staged by TMA (cp.async.bulk.tensor, 128-byte swizzle) into a multi-stage smem ring,
//     completion tracked with mbarriers; a consumer releases a slot once the wgmma reading it has retired;
//   * both operand majors (K-major and MN-major) are supported through the wgmma shared-memory descriptors and the
//     transpose bits, so dgrad (dY*W) and wgrad (dY^T*X) read the original tensors — no transposes.
#include <mutex>
#include <stdlib.h>

#include "gemm_common.cuh"

namespace mb200 {

template <int BN, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(kThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ GemmKernelParams p) {
  using C_ = Cfg<BN>;
  constexpr int kStages = C_::kStages;

  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B atoms need 1024-byte alignment
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * C_::kABytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kStages * C_::kStageBytes);
  uint64_t* empty_bar = full_bar + kStages;

  const int wg = threadIdx.x >> 7;
  const int num_kb = (p.K + BK - 1) / BK;
  const int items = p.total_tiles * p.split_k;

  pdl_trigger();  // the next kernel may start its prologue on SMs as they become free
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);  // one arrive per consumer warpgroup
    }
    mbar_fence_init();
  }
  __syncthreads();
  pdl_wait();  // everything above overlapped the previous kernel; global memory is touched only from here on

  if (wg == 0) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int w = blockIdx.x; w < items; w += gridDim.x) {
        const int t = w / p.split_k, ks = w - t * p.split_k;
        const int kb0 = ks * p.kb_per_split, kb1 = min(num_kb, kb0 + p.kb_per_split);
        const int tpb = p.tiles_m * p.tiles_n;
        const int z = t / tpb;
        const int r = t - z * tpb;
        const int m_blk = r % p.tiles_m;
        const int n_blk = r / p.tiles_m;
        const int z0 = z % p.nb0, z1 = z / p.nb0;
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_expect_tx(&full_bar[stage], (uint32_t)C_::kStageBytes);
          uint8_t* sa = smem_a + stage * C_::kABytes;
          uint8_t* sb = smem_b + stage * C_::kBBytes;
          const int kc = kb * BK;
          if constexpr (A_MN) {
#pragma unroll
            for (int i = 0; i < BM / 64; ++i)
              tma_load_4d(sa + i * 8192, &tmA, &full_bar[stage], m_blk * BM + i * 64, kc, z0, z1);
          } else {
            tma_load_4d(sa, &tmA, &full_bar[stage], kc, m_blk * BM, z0, z1);
          }
          if constexpr (B_MN) {
#pragma unroll
            for (int i = 0; i < BN / 64; ++i)
              tma_load_4d(sb + i * 8192, &tmB, &full_bar[stage], n_blk * BN + i * 64, kc, z0, z1);
          } else {
            tma_load_4d(sb, &tmB, &full_bar[stage], kc, n_blk * BN, z0, z1);
          }
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ===================== consumers: wgmma + epilogue =====================
    const int cw = wg - 1;  // rows [64 cw, 64 cw + 64) of the tile
    const bool leader = (threadIdx.x & 127) == 0;
    // K-major SW128: 8-row atoms of 128 B rows -> SBO = 1024, LBO unused; advance K by 16 elems = 32 B; this
    //                warpgroup's 64 rows of A start 64 x 128 B into the slot.
    // MN-major SW128: atom = 64 MN-elements (128 B) x 8 k-rows; SBO = 1024 between k-groups of 8,
    //                 LBO = 8192 between 64-wide MN chunks (one TMA box each); advance K by 16 rows = 2048 B;
    //                 this warpgroup's 64 rows of A are the cw-th box.
    constexpr uint32_t b_lbo = B_MN ? 8192u : 0u;
    constexpr uint32_t a_kadv = A_MN ? 2048u : 32u, b_kadv = B_MN ? 2048u : 32u;
    const uint32_t a_off = (uint32_t)cw * 8192u;
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    for (int w = blockIdx.x; w < items; w += gridDim.x) {
      const int t = w / p.split_k, ks = w - t * p.split_k;
      const int kb0 = ks * p.kb_per_split, kb1 = min(num_kb, kb0 + p.kb_per_split);
      const int tpb = p.tiles_m * p.tiles_n;
      const int z = t / tpb;
      const int r = t - z * tpb;
      const int m_blk = r % p.tiles_m;
      const int n_blk = r / p.tiles_m;
      const int z0 = z % p.nb0, z1 = z / p.nb0;
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem_a + stage * C_::kABytes) + a_off;
        const uint32_t sb = smem_u32(smem_b + stage * C_::kBBytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / WG_K; ++k) {
          const uint64_t da = make_smem_desc(sa + k * a_kadv, 0u, 1024);
          const uint64_t db = make_smem_desc(sb + k * b_kadv, b_lbo, 1024);
          wgmma_bf16<BN, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, (kb > kb0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();  // the group of the previous k-block has retired: its slot may be refilled
        if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
      const long long boff = (long long)z0 * p.c_bs0 + (long long)z1 * p.c_bs1;
      epi_fragment<BN>(p, acc, boff, m_blk * BM + cw * 64, n_blk * BN, ks);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// split-K finalize: C = epilogue(sum over splits of ws[split]). One thread per float4 of the output.
// ---------------------------------------------------------------------------------------------
template <typename OutT>
__global__ void splitk_finalize_kernel(const GemmKernelParams p) {
  pdl_trigger();
  pdl_wait();
  const int ncol4 = (p.N + 3) >> 2;
  const long long total = (long long)p.M * ncol4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int row = (int)(i / ncol4);
    const int col = (int)(i - (long long)row * ncol4) * 4;
    const int nvalid = min(4, p.N - col);
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    for (int ks = 0; ks < p.split_k; ++ks) {  // fixed summation order -> bitwise reproducible
      const float4 w4 = *reinterpret_cast<const float4*>(p.splitk_ws + ((long long)ks * p.M + row) * p.ld_ws + col);
      v[0] += w4.x;
      v[1] += w4.y;
      v[2] += w4.z;
      v[3] += w4.w;
    }
    if (p.bias) {
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (e < nvalid) v[e] += __bfloat162float(p.bias[col + e]);
    }
    if (p.rope_mode != 0 && col < p.rope_ncols && (col % p.rope_hd) < p.rope_rot) {
      const int rp = (col % p.rope_hd) >> 1;
      const float2* tp = p.rope_tab + (long long)(row % p.rope_S) * (p.rope_rot >> 1) + rp;
      const float2 cs0 = __ldg(tp), cs1 = __ldg(tp + 1);
      const float sg = p.rope_mode > 0 ? 1.f : -1.f;
      const float a0 = v[0], a1 = v[1], a2 = v[2], a3 = v[3];
      v[0] = a0 * cs0.x - a1 * cs0.y * sg;
      v[1] = a1 * cs0.x + a0 * cs0.y * sg;
      v[2] = a2 * cs1.x - a3 * cs1.y * sg;
      v[3] = a3 * cs1.x + a2 * cs1.y * sg;
    }
    const long long coff = (long long)row * p.ldc + col;
    const long long roff = (long long)row * p.ld_res + col;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (e >= nvalid) continue;
      float x = v[e];
      if (p.aux_out) p.aux_out[coff + e] = __float2bfloat16(x);
      if (p.act == MB200_ACT_GELU_NEW) x = gelu_new_f(x);
      else if (p.act == MB200_ACT_QUICK_GELU) x = quick_gelu_f(x);
      else if (p.act == MB200_ACT_RELU) x = fmaxf(x, 0.f);
      if (p.dact) {
        const float a = __bfloat162float(p.aux_in[coff + e]);
        x = p.dact == MB200_DACT_GELU_NEW ? x * gelu_new_grad_f(a) : (a > 0.f ? x : 0.f);
      }
      if (p.res1) x += __bfloat162float(p.res1[roff + e]);
      if (p.res2) x += __bfloat162float(p.res2[roff + e]);
      if (p.act == MB200_ACT_RELU_POST) x = fmaxf(x, 0.f);
      if constexpr (sizeof(OutT) == 4) {
        float* dst = reinterpret_cast<float*>(p.C) + coff + e;
        *dst = p.accumulate ? *dst + x : x;
      } else {
        reinterpret_cast<bf16*>(p.C)[coff + e] = __float2bfloat16(x);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

// rank-4 bf16 tensor map over an operand. K-major: dims (K, rows, nb0, nb1), box (64, box_rows).
// MN-major: dims (rows, K, nb0, nb1), box (64, 64).
int make_operand_map(CUtensorMap* out, const mb200_operand& op, int rows, int K, int nb0, int nb1,
                            int box_rows) {
  PFN_encodeTiled enc = get_encode_fn();
  MB_REQUIRE(enc != nullptr, MB200_E_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  MB_REQUIRE((reinterpret_cast<uintptr_t>(op.ptr) & 15) == 0, MB200_E_ALIGN, "gemm operand pointer not 16B aligned");
  MB_REQUIRE(op.ld % 8 == 0, MB200_E_ALIGN, "gemm operand ld (%lld) must be a multiple of 8 elements",
             (long long)op.ld);
  MB_REQUIRE((nb0 == 1 || op.bs0 % 8 == 0) && (nb1 == 1 || op.bs1 % 8 == 0), MB200_E_ALIGN,
             "gemm operand batch strides must be multiples of 8 elements");
  cuuint64_t dims[4];
  cuuint64_t strides[3];
  cuuint32_t box[4];
  cuuint32_t estr[4] = {1, 1, 1, 1};
  if (!op.mn_major) {
    dims[0] = (cuuint64_t)K;
    dims[1] = (cuuint64_t)rows;
    box[0] = BK;
    box[1] = (cuuint32_t)box_rows;
  } else {
    dims[0] = (cuuint64_t)rows;
    dims[1] = (cuuint64_t)K;
    box[0] = 64;
    box[1] = BK;
  }
  dims[2] = (cuuint64_t)nb0;
  dims[3] = (cuuint64_t)nb1;
  box[2] = 1;
  box[3] = 1;
  // strides of dims 1..3 in bytes; a size-1 batch dim still needs a legal (16B-multiple) stride
  strides[0] = (cuuint64_t)op.ld * 2;
  strides[1] = (cuuint64_t)(nb0 > 1 ? op.bs0 : op.ld) * 2;
  strides[2] = (cuuint64_t)(nb1 > 1 ? op.bs1 : op.ld) * 2;
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(op.ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  MB_REQUIRE(r == CUDA_SUCCESS, MB200_E_CUDA,
             "cuTensorMapEncodeTiled failed (%d): dims=(%llu,%llu,%llu,%llu) strides=(%llu,%llu,%llu) box=(%u,%u)",
             (int)r, (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2],
             (unsigned long long)dims[3], (unsigned long long)strides[0], (unsigned long long)strides[1],
             (unsigned long long)strides[2], box[0], box[1]);
  return 0;
}

template <int BN, bool A_MN, bool B_MN>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmKernelParams& kp,
                       cudaStream_t stream) {
  auto kern = gemm_wgmma_kernel<BN, A_MN, B_MN>;
  static bool attr_set = false;  // per instantiation
  if (!attr_set) {
    MB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<BN>::kSmemBytes));
    attr_set = true;
  }
  const long long items = (long long)kp.total_tiles * kp.split_k;
  int grid = items < gemm_sms() ? (int)items : gemm_sms();
  {
    const double nb = (double)kp.total_tiles / ((double)kp.tiles_m * kp.tiles_n);
    const double flops = 2.0 * kp.M * (double)kp.N * kp.K * nb;
    const double bytes = nb * (2.0 * ((double)kp.M * kp.K + (double)kp.N * kp.K) + (kp.c_f32 ? 4.0 : 2.0) * kp.M * kp.N);
    GemmProfScope prof(stream, flops, bytes);
    MB_CUDA(launch_pdl(kern, dim3(grid), dim3(kThreads), Cfg<BN>::kSmemBytes, stream, tmA, tmB, kp));
  }
  count_launch();
  MB_CUDA(cudaGetLastError());
  return 0;
}

template <int BN>
static int dispatch_major(bool a_mn, bool b_mn, const CUtensorMap& tmA, const CUtensorMap& tmB,
                          const GemmKernelParams& kp, cudaStream_t s) {
  if (!a_mn && !b_mn) return launch_gemm<BN, false, false>(tmA, tmB, kp, s);
  if (!a_mn && b_mn) return launch_gemm<BN, false, true>(tmA, tmB, kp, s);
  if (a_mn && !b_mn) return launch_gemm<BN, true, false>(tmA, tmB, kp, s);
  return launch_gemm<BN, true, true>(tmA, tmB, kp, s);
}

static int dispatch_bn(int bn, bool a_mn, bool b_mn, const CUtensorMap& tmA, const CUtensorMap& tmB,
                       const GemmKernelParams& kp, cudaStream_t s) {
  switch (bn) {
    case 64: return dispatch_major<64>(a_mn, b_mn, tmA, tmB, kp, s);
    case 128: return dispatch_major<128>(a_mn, b_mn, tmA, tmB, kp, s);
    default: return dispatch_major<256>(a_mn, b_mn, tmA, tmB, kp, s);
  }
}

static int pick_bn(int M, int N, int batches) {
  if (N <= 64) return 64;
  // Model: time ~ waves * (cost of one tile). A wide tile streams A once per BN columns and keeps more MMA work per
  // smem byte; narrower tiles only win when wide tiles leave most SMs idle (few tiles) — e.g. the adapter
  // down-projection (M=1024, N=1024: 64 tiles at BN=128, 128 at BN=64). The relative tile costs are estimates.
  const int tiles_m = (M + BM - 1) / BM;
  const int sms = num_sms();
  double best = 1e300;
  int best_bn = 256;
  const int cands[3] = {256, 128, 64};
  const double tile_cost[3] = {1.0, 0.55, 0.3};  // relative time of one (BM x BN x K) tile
  for (int i = 0; i < 3; ++i) {
    const int bn = cands[i];
    if (bn > 64 && N <= bn / 2) continue;
    const long long t = (long long)tiles_m * ((N + bn - 1) / bn) * batches;
    const long long waves = (t + sms - 1) / sms;
    const double cost = (double)waves * tile_cost[i];
    if (cost < best - 1e-12) {
      best = cost;
      best_bn = bn;
    }
  }
  return best_bn;
}

// Small-M (decode, M = batch <= 32) GEMMs stream their weight matrix once and are HBM-bound: what matters is bytes in
// flight, i.e. every SM pulling weights all the time. The plan picks the tile width and a K split so that
// tiles x splits covers the SMs evenly:
//   t = t_item + waves * bytes_per_item / rate_per_sm + (split > 1 ? t_finalize : 0),
//   rate_per_sm = min(per-SM TMA streaming rate (bytes in flight / latency), all-SM HBM rate / active SMs).
// The HBM rate is the H100 SXM data-sheet figure; the per-SM rates and fixed costs are estimates.
struct SmallPlan {
  int bn, split;
};
static SmallPlan plan_small_m(int N, int K, int M, size_t ws_bytes) {
  const int sms = num_sms();
  const int num_kb = (K + BK - 1) / BK;
  const double kHbmRate = 3.35e12, kItem = 4e-6, kFinalize = 4e-6;
  SmallPlan best{64, 1};
  double best_t = 1e300;
  const int cands[3] = {256, 128, 64};
  for (int i = 0; i < 3; ++i) {
    const int bn = cands[i];
    if (bn > 64 && N <= bn / 2) continue;
    const int tiles = (N + bn - 1) / bn;
    for (int split = 1; split <= 16; ++split) {
      if (split > 1) {
        if (num_kb / split < 8) break;
        if ((size_t)split * M * ((N + 3) / 4 * 4) * sizeof(float) > ws_bytes) break;
      }
      const int kb_per = (num_kb + split - 1) / split;
      const int eff_split = (num_kb + kb_per - 1) / kb_per;
      const long long items = (long long)tiles * eff_split;
      const long long waves = (items + sms - 1) / sms;
      const double active = (double)(items < sms ? items : sms);
      const double sm_rate = bn == 64 ? 40e9 : 50e9;  // more weight bytes in flight per SM with the deeper B ring
      const double rate = sm_rate < kHbmRate / active ? sm_rate : kHbmRate / active;
      const double t = kItem + waves * ((double)kb_per * bn * BK * 2 / rate) + (eff_split > 1 ? kFinalize : 0.0);
      if (t < best_t - 1e-12) {
        best_t = t;
        best = SmallPlan{bn, eff_split};
      }
    }
  }
  return best;
}

int gemm_impl(const mb200_gemm_args* a, cudaStream_t stream) {
  MB_REQUIRE(a != nullptr, MB200_E_ARG, "null gemm args");
  MB_REQUIRE(a->M > 0 && a->N > 0 && a->K > 0 && a->nb0 > 0 && a->nb1 > 0, MB200_E_SHAPE,
             "gemm: bad shape M=%d N=%d K=%d nb=(%d,%d)", a->M, a->N, a->K, a->nb0, a->nb1);
  MB_REQUIRE(a->c_dtype == MB200_BF16 || a->c_dtype == MB200_F32, MB200_E_DTYPE, "gemm: bad c_dtype %d", a->c_dtype);
  MB_REQUIRE(!(a->accumulate && a->c_dtype != MB200_F32), MB200_E_DTYPE, "gemm: accumulate needs f32 output");
  MB_REQUIRE(!(a->dact && !a->aux_in), MB200_E_ARG, "gemm: dact needs aux_in");
  const int celt = a->c_dtype == MB200_F32 ? 4 : 8;
  MB_REQUIRE((reinterpret_cast<uintptr_t>(a->C) & 15) == 0 && a->ldc % celt == 0, MB200_E_ALIGN,
             "gemm: C must be 16B aligned with ldc multiple of %d", celt);
  MB_REQUIRE((a->nb0 == 1 || a->c_bs0 % celt == 0) && (a->nb1 == 1 || a->c_bs1 % celt == 0), MB200_E_ALIGN,
             "gemm: C batch strides must be multiples of %d elements", celt);
  if (a->res1 || a->res2) MB_REQUIRE(a->ld_res % 8 == 0, MB200_E_ALIGN, "gemm: ld_res must be a multiple of 8");
  if (a->aux_in || a->aux_out)
    MB_REQUIRE(a->ldc % 8 == 0, MB200_E_ALIGN, "gemm: aux tensors share ldc, which must be a multiple of 8");
  int rc = check_arch();
  if (rc) return rc;

  int bn = a->force_bn ? a->force_bn : pick_bn(a->M, a->N, a->nb0 * a->nb1);
  MB_REQUIRE(bn == 64 || bn == 128 || bn == 256, MB200_E_ARG, "gemm: force_bn must be 64, 128 or 256");

  CUtensorMap tmA, tmB;
  // small-M problems (decode: M = batch <= 32) are planned for weight streaming (tile width + K split)
  const bool small_m = a->M <= 32 && a->A.mn_major == 0 && a->nb0 * a->nb1 == 1 && a->c_dtype == MB200_BF16;
  int plan_split = 1;
  if (small_m && !a->force_bn) {
    const SmallPlan pl = plan_small_m(a->N, a->K, a->M, a->splitk_ws ? (size_t)a->splitk_ws_bytes : 0);
    bn = pl.bn;
    plan_split = pl.split;
  }
  rc = make_operand_map(&tmA, a->A, a->M, a->K, a->nb0, a->nb1, BM);
  if (rc) return rc;

  GemmKernelParams kp;
  memset(&kp, 0, sizeof(kp));
  kp.M = a->M;
  kp.N = a->N;
  kp.K = a->K;
  kp.nb0 = a->nb0;
  kp.tiles_m = (a->M + BM - 1) / BM;
  kp.C = a->C;
  kp.ldc = a->ldc;
  kp.c_bs0 = a->c_bs0;
  kp.c_bs1 = a->c_bs1;
  kp.alpha = a->alpha;
  kp.act = a->act;
  kp.dact = a->dact;
  kp.accumulate = a->accumulate;
  kp.bias = reinterpret_cast<const bf16*>(a->bias);
  kp.aux_out = reinterpret_cast<bf16*>(a->aux_out);
  kp.aux_in = reinterpret_cast<const bf16*>(a->aux_in);
  kp.res1 = reinterpret_cast<const bf16*>(a->res1);
  kp.res2 = reinterpret_cast<const bf16*>(a->res2);
  kp.ld_res = a->ld_res;
  kp.epi_kind = EK_GENERIC;
  kp.c_f32 = a->c_dtype == MB200_F32 ? 1 : 0;
  kp.rope_tab = reinterpret_cast<const float2*>(a->rope_tab);
  kp.rope_mode = a->rope_tab ? a->rope_mode : 0;
  kp.rope_S = a->rope_S;
  kp.rope_hd = a->rope_hd;
  kp.rope_rot = a->rope_rot;
  kp.rope_ncols = a->rope_ncols;
  if (kp.rope_mode != 0)
    MB_REQUIRE(a->rope_S > 0 && a->rope_hd > 0 && a->rope_rot % 4 == 0 && a->rope_rot <= a->rope_hd &&
                   a->rope_hd % 4 == 0 && a->rope_ncols % 4 == 0,
               MB200_E_ARG, "gemm: bad rope epilogue parameters");

  const bool amn = a->A.mn_major != 0, bmn = a->B.mn_major != 0;
  const bool f32 = a->c_dtype == MB200_F32;
  kp.split_k = 1;
  kp.kb_per_split = (a->K + BK - 1) / BK;
  // Split-K for small M (see plan_small_m; for 32 < M <= 128 only the long-K / narrow-N shape, GPT-J fc_out, is split).
  // Partials go to per-split fp32 slices; a small finalize kernel sums them in fixed order (deterministic) and applies
  // the fused epilogue.
  const bool split_mid = !small_m && a->splitk_ws && a->M <= 128 && a->nb0 * a->nb1 == 1 && a->K >= 8192 &&
                         a->N <= 8192 && !a->force_bn;
  // Larger M with few tiles and a long K (conv-trunk 3x3 convolutions of the late stages: M = 1152, N = 768,
  // K = 6912 -> 27 tiles of 108 k-blocks) leave most SMs idle: split K until tiles x splits covers the machine.
  const int bn_few = a->N >= 256 ? 256 : (a->N > 64 ? 128 : 64);
  const int tiles_m = kp.tiles_m;
  const bool split_few = !small_m && !split_mid && a->splitk_ws && a->M > 128 && a->nb0 * a->nb1 == 1 &&
                         a->K >= 2048 && !a->force_bn && 2 * tiles_m * ((a->N + bn_few - 1) / bn_few) <= num_sms();
  if (plan_split > 1 || split_mid || split_few) {
    const int bn_s = small_m ? bn : bn_few;
    const int tiles = (a->N + bn_s - 1) / bn_s;
    const int num_kb = (a->K + BK - 1) / BK;
    int split = plan_split;
    if (split_mid || split_few) {
      split = num_sms() / (tiles * tiles_m);
      if (split > num_kb / 4) split = num_kb / 4;
    }
    const long long ld_ws = (a->N + 3) / 4 * 4;
    while (split > 1 && (size_t)split * a->M * ld_ws * sizeof(float) > (size_t)a->splitk_ws_bytes) --split;
    if (split > 1) {
      const int kb_per = (num_kb + split - 1) / split;
      split = (num_kb + kb_per - 1) / kb_per;  // every split owns at least one k-block
      bn = bn_s;
      rc = make_operand_map(&tmB, a->B, a->N, a->K, a->nb0, a->nb1, bn);
      if (rc) return rc;
      kp.tiles_n = tiles;
      kp.total_tiles = tiles_m * tiles;
      kp.split_k = split;
      kp.kb_per_split = kb_per;
      kp.splitk_ws = reinterpret_cast<float*>(a->splitk_ws);
      kp.ld_ws = ld_ws;
      GemmKernelParams kg = kp;  // the GEMM itself only writes partials (alpha applied)
      kg.epi_kind = EK_SPLITK;
      rc = dispatch_bn(bn, amn, bmn, tmA, tmB, kg, stream);
      if (rc) return rc;
      const long long n4 = (long long)a->M * ((a->N + 3) / 4);
      const int fgrid = (int)((n4 + 255) / 256 > 2048 ? 2048 : (n4 + 255) / 256);
      kp.alpha = 1.f;  // already applied to the partials
      if (f32) MB_CUDA(launch_pdl(splitk_finalize_kernel<float>, dim3(fgrid), dim3(256), 0, stream, kp));
      else MB_CUDA(launch_pdl(splitk_finalize_kernel<bf16>, dim3(fgrid), dim3(256), 0, stream, kp));
      count_launch();
      return 0;
    }
  }
  rc = make_operand_map(&tmB, a->B, a->N, a->K, a->nb0, a->nb1, bn);
  if (rc) return rc;
  kp.tiles_n = (a->N + bn - 1) / bn;
  kp.total_tiles = tiles_m * kp.tiles_n * a->nb0 * a->nb1;
  return dispatch_bn(bn, amn, bmn, tmA, tmB, kp, stream);
}

}  // namespace mb200

extern "C" int mb200_gemm(const mb200_gemm_args* args, void* stream) {
  return mb200::gemm_impl(args, reinterpret_cast<cudaStream_t>(stream));
}
