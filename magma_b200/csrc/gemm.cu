// magma_b200 — bf16 GEMM core for sm_90a (Hopper).
//
//   C[b][M,N] = epilogue(alpha * A[b][M,K] * B[b][N,K]^T)
//
// Design (not a translation of anything in the reference, which only calls cuBLAS through torch.nn.Linear — e.g.
// magma/adapters.py:19-23, magma/image_prefix.py:72):
//   * persistent grid (<= one CTA per SM), static round-robin tile scheduler, m-fastest tile order so
//     CTAs that run concurrently share the same weight (B) tile through L2;
//   * warp-specialised: warpgroup 0 = TMA producer (one lane, registers handed to the consumers with setmaxnreg),
//     warpgroups 1 and 2 = consumers, each owning 64 rows of the 128-row tile: wgmma.mma_async m64nBNk16 with fp32
//     accumulators in registers, then the fused epilogue, staged through shared memory 64 columns at a time so that
//     one copy of its code, compiled per epilogue form, reads and writes global memory in contiguous row segments
//     (gemm_common.cuh);
//   * operands staged by TMA (cp.async.bulk.tensor, 128-byte swizzle) into a multi-stage smem ring,
//     completion tracked with mbarriers; a consumer releases a slot once the wgmma reading it has retired;
//   * both operand majors (K-major and MN-major) are supported through the wgmma shared-memory descriptors and the
//     transpose bits, so dgrad (dY*W) and wgrad (dY^T*X) read the original tensors — no transposes.
#include <mutex>
#include <stdlib.h>

#include "gemm_common.cuh"

namespace mb200 {

// Tensor maps of the epilogue inputs staged by TMA (GemmKernelParams::epi_in of them, in its order), each a K-major
// [M, N] operand with box (64 columns, BM rows). Kernels without staged inputs take an empty parameter and carry none
// of the staging code: it would cost them instruction fetch in the epilogue loop.
template <bool kOn>
struct EpiMaps {
  CUtensorMap m[3];
};
template <>
struct EpiMaps<false> {};

// FORM: the epilogue form (gemm_common.cuh) the kernel is compiled for.
template <int BN, bool A_MN, bool B_MN, bool EPI_TMA, uint32_t FORM = EF_RUNTIME>
__global__ void __launch_bounds__(kThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ EpiMaps<EPI_TMA> tmE, const __grid_constant__ GemmKernelParams p) {
  using C_ = Cfg<BN>;
  constexpr int kStages = C_::kStages;

  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B atoms need 1024-byte alignment. An offset on the array, not a rounded integer address: the compiler
  // then still knows everything derived from it is shared memory (LDS / STS for the epilogue staging, not generic).
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * C_::kABytes;
  float* epi_stage = reinterpret_cast<float*>(smem + kStages * C_::kStageBytes);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kStages * C_::kStageBytes + kEpiBytes);
  uint64_t* empty_bar = full_bar + kStages;
  const EpiRing ring{smem_a, smem_b, full_bar, empty_bar};

  const int wg = threadIdx.x >> 7;
  const int num_kb = (p.K + BK - 1) / BK;
  const int items = p.total_tiles * p.split_k;

  pdl_trigger();  // the next kernel may start its prologue on SMs as they become free
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if constexpr (EPI_TMA) {
#pragma unroll 1
      for (int i = 0; i < p.epi_in; ++i) tma_prefetch_desc(&tmE.m[i]);
    }
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);  // one arrive per consumer warpgroup
    }
    mbar_fence_init();
  }
  __syncthreads();
  pdl_wait();  // everything above overlapped the previous kernel; global memory is touched only from here on

  // Register split: 128 x 40 (producer) + 256 x 232 (consumers) <= 65536; the launch bound alone caps every thread
  // at 168, which the BN = 256 accumulators (128 registers) leave little room above.
  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
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
        if constexpr (EPI_TMA) epi_queue_inputs<BN>(p, tmE.m, ring, stage, phase, m_blk * BM, n_blk * BN, z0, z1);
      }
    }
  } else {
    // ===================== consumers: wgmma + epilogue =====================
    setmaxnreg_inc<232>();
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
      epi_tile<BN, EPI_TMA, EpiForm<FORM>>(p, acc, epi_stage + cw * 64 * kEpiCols, 1 + cw, boff, m_blk * BM + cw * 64,
                                           n_blk * BN, ks, ring, stage, phase);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// split-K finalize: C = epilogue(sum over splits of ws[split]). One thread per float4 of the output.
// ---------------------------------------------------------------------------------------------
__global__ void splitk_finalize_kernel(const GemmKernelParams p) {
  pdl_trigger();
  pdl_wait();
  const int ncol4 = (p.N + 3) >> 2;
  const long long total = (long long)p.M * ncol4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int row = (int)(i / ncol4);
    const int col = (int)(i - (long long)row * ncol4) * 4;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    for (int ks = 0; ks < p.split_k; ++ks) {  // fixed summation order -> bitwise reproducible
      const float4 w4 = *reinterpret_cast<const float4*>(p.splitk_ws + ((long long)ks * p.M + row) * p.ld_ws + col);
      v[0] += w4.x;
      v[1] += w4.y;
      v[2] += w4.z;
      v[3] += w4.w;
    }
    using Form = EpiForm<EF_RUNTIME>;
    float bias[4];
    EpiIn in;
    if (p.bias) ld_bf16x4(p.bias + col, min(4, p.N - col), bias);
    epi_load_inputs<Form>(p, 0, row, col, in);
    epi_store4<Form>(p, 0, row, col, v, bias, in);
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
  // The encoder is a driver call and needs a current context. A thread whose first CUDA work is a GEMM (an autograd
  // worker thread entering the backward pass with nothing to allocate, say) has none bound yet: one runtime call binds
  // the current device's primary context to it.
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) {
    MB_CUDA(cudaFree(nullptr));
    ctx_bound = true;
  }
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

template <int BN, bool A_MN, bool B_MN, bool EPI_TMA, uint32_t FORM = EF_RUNTIME>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const EpiMaps<true>& tmE,
                       const GemmKernelParams& kp, cudaStream_t stream) {
  auto kern = gemm_wgmma_kernel<BN, A_MN, B_MN, EPI_TMA, FORM>;
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
    if constexpr (EPI_TMA)
      MB_CUDA(launch_pdl(kern, dim3(grid), dim3(kThreads), Cfg<BN>::kSmemBytes, stream, tmA, tmB, tmE, kp));
    else
      MB_CUDA(launch_pdl(kern, dim3(grid), dim3(kThreads), Cfg<BN>::kSmemBytes, stream, tmA, tmB, EpiMaps<false>{}, kp));
  }
  count_launch();
  MB_CUDA(cudaGetLastError());
  return 0;
}

template <int BN, bool EPI_TMA>
static int dispatch_major(bool a_mn, bool b_mn, const CUtensorMap& tmA, const CUtensorMap& tmB,
                          const EpiMaps<true>& tmE, const GemmKernelParams& kp, cudaStream_t s) {
  if (!a_mn && !b_mn) return launch_gemm<BN, false, false, EPI_TMA>(tmA, tmB, tmE, kp, s);
  if (!a_mn && b_mn) return launch_gemm<BN, false, true, EPI_TMA>(tmA, tmB, tmE, kp, s);
  if (a_mn && !b_mn) return launch_gemm<BN, true, false, EPI_TMA>(tmA, tmB, tmE, kp, s);
  return launch_gemm<BN, true, true, EPI_TMA>(tmA, tmB, tmE, kp, s);
}

static int dispatch_bn(int bn, bool a_mn, bool b_mn, const CUtensorMap& tmA, const CUtensorMap& tmB,
                       const EpiMaps<true>& tmE, const GemmKernelParams& kp, cudaStream_t s) {
  const bool epi = kp.epi_in != 0;
  switch (bn) {
    case 64:
      return epi ? dispatch_major<64, true>(a_mn, b_mn, tmA, tmB, tmE, kp, s)
                 : dispatch_major<64, false>(a_mn, b_mn, tmA, tmB, tmE, kp, s);
    case 128:
      return epi ? dispatch_major<128, true>(a_mn, b_mn, tmA, tmB, tmE, kp, s)
                 : dispatch_major<128, false>(a_mn, b_mn, tmA, tmB, tmE, kp, s);
    default:
      return epi ? dispatch_major<256, true>(a_mn, b_mn, tmA, tmB, tmE, kp, s)
                 : dispatch_major<256, false>(a_mn, b_mn, tmA, tmB, tmE, kp, s);
  }
}

// The compiled epilogue forms: the feature sets the GEMMs of a GPT-J training step with MLP adapters and of the ViT-L/14
// forward launch at the 256-wide tile, each for the operand majors it is launched with. Returns false when (form,
// majors) is not one of them; with kp == nullptr only answers whether it is.
template <uint32_t F, bool A_MN, bool B_MN>
static bool launch_form(uint32_t form, bool a_mn, bool b_mn, const CUtensorMap& tmA, const CUtensorMap& tmB,
                        const EpiMaps<true>& tmE, const GemmKernelParams* kp, cudaStream_t s, int* rc) {
  if (form != F || a_mn != A_MN || b_mn != B_MN) return false;
  if (kp) *rc = launch_gemm<256, A_MN, B_MN, EpiForm<F>::kInputs != 0, F>(tmA, tmB, tmE, *kp, s);
  return true;
}
static bool dispatch_form(uint32_t form, bool a_mn, bool b_mn, const CUtensorMap& tmA, const CUtensorMap& tmB,
                          const EpiMaps<true>& tmE, const GemmKernelParams* kp, cudaStream_t s, int* rc) {
#define MB_FORM(F, A_MN, B_MN) launch_form<(F), A_MN, B_MN>(form, a_mn, b_mn, tmA, tmB, tmE, kp, s, rc)
  return MB_FORM(EF_ROPE, false, false) ||                           // qkv forward
         MB_FORM(EF_RES1, false, false) ||                           // attention out forward
         MB_FORM(EF_BIAS | EF_GELU | EF_AUX_OUT, false, false) ||    // fc_in forward
         MB_FORM(EF_BIAS, false, false) ||                           // fc_out forward, LM head, ViT qkv
         MB_FORM(EF_BIAS | EF_RES1 | EF_RES2, false, false) ||       // adapter up
         MB_FORM(EF_BIAS | EF_RES1, false, false) ||                 // ViT out and proj
         MB_FORM(EF_BIAS | EF_QGELU, false, false) ||                // ViT fc
         MB_FORM(EF_DGELU, false, true) ||                           // fc_out dgrad
         MB_FORM(0u, false, true) ||                                 // fc_in, attention out and LM-head dgrad
         MB_FORM(EF_RES1, false, true) ||                            // qkv dgrad, adapter dgrad-down
         MB_FORM(EF_F32, true, true);                                // adapter wgrads
#undef MB_FORM
}

// The compiled form a launch qualifies for at the 256-wide tile, or EF_RUNTIME: its features must all be ones a form
// can express, every [M, N] input staged by TMA (kp.epi_in), and bias and aux_out 8-byte aligned, which with the
// alignment gemm_impl requires of C, ldc and the batch strides makes every 4-column access of a compiled form a vector.
// generic_epilogue is not looked at here: the plan must not depend on it.
static uint32_t epi_form(const mb200_gemm_args* a, const GemmKernelParams& kp) {
  if ((a->act != MB200_ACT_NONE && a->act != MB200_ACT_GELU_NEW && a->act != MB200_ACT_QUICK_GELU) ||
      (a->dact != MB200_DACT_NONE && a->dact != MB200_DACT_GELU_NEW))
    return EF_RUNTIME;
  if (((reinterpret_cast<uintptr_t>(a->bias) | reinterpret_cast<uintptr_t>(a->aux_out)) & 7) != 0) return EF_RUNTIME;
  const uint32_t f = (a->bias ? EF_BIAS : 0u) | (kp.rope_mode ? EF_ROPE : 0u) | (a->aux_out ? EF_AUX_OUT : 0u) |
                     (a->act == MB200_ACT_GELU_NEW ? EF_GELU : 0u) | (a->act == MB200_ACT_QUICK_GELU ? EF_QGELU : 0u) |
                     (a->dact ? EF_DGELU : 0u) | (a->res1 ? EF_RES1 : 0u) | (a->res2 ? EF_RES2 : 0u) |
                     (kp.c_f32 ? EF_F32 : 0u);
  const int inputs = (a->dact != 0) + (a->res1 != nullptr) + (a->res2 != nullptr);
  if (kp.epi_in != inputs) return EF_RUNTIME;
  CUtensorMap unused;  // not read: no launch
  EpiMaps<true> unused_e;
  return dispatch_form(f, a->A.mn_major != 0, a->B.mn_major != 0, unused, unused, unused_e, nullptr, 0, nullptr)
             ? f
             : EF_RUNTIME;
}

// Tensor maps for the epilogue's [M, N] inputs (aux_in when dact, res1, res2), fetched by the producer through the
// operand ring. Used only when every input is TMA-addressable (16-byte base, row and batch strides multiples of 8
// elements); otherwise kp->epi_in stays 0 and the epilogue reads all of them from global memory itself.
static int make_epi_maps(EpiMaps<true>* maps, GemmKernelParams* kp, const mb200_gemm_args* a) {
  const void* ptr[3];
  long long ld[3];
  int n = 0;
  if (a->dact) {
    ptr[n] = a->aux_in;
    ld[n++] = a->ldc;
  }
  if (a->res1) {
    ptr[n] = a->res1;
    ld[n++] = a->ld_res;
  }
  if (a->res2) {
    ptr[n] = a->res2;
    ld[n++] = a->ld_res;
  }
  bool ok = (a->nb0 == 1 || a->c_bs0 % 8 == 0) && (a->nb1 == 1 || a->c_bs1 % 8 == 0);
  for (int i = 0; i < n; ++i) ok = ok && (reinterpret_cast<uintptr_t>(ptr[i]) & 15) == 0 && ld[i] % 8 == 0;
  if (n == 0 || !ok) return 0;
  for (int i = 0; i < n; ++i) {
    mb200_operand op;
    memset(&op, 0, sizeof(op));
    op.ptr = ptr[i];
    op.ld = ld[i];
    op.bs0 = a->c_bs0;
    op.bs1 = a->c_bs1;
    const int rc = make_operand_map(&maps->m[i], op, a->M, a->N, a->nb0, a->nb1, BM);
    if (rc) return rc;
  }
  kp->epi_in = n;
  return 0;
}

// The GEMM's tile width when it is not split along K. Model: time ~ waves x (cost of one tile).
//  * Runtime epilogue form (no compiled form matches the launch): the relative tile costs of the three widths,
//    kTile, independent of K. A wide tile streams A once per BN columns and keeps more MMA work per smem byte; narrower
//    tiles only win when wide tiles leave most SMs idle, e.g. the adapter down-projection (M = 1024, N = 1024: 32 tiles
//    of 256, 128 of 64).
//  * A compiled form exists at BN = 256 and the GEMM has at least 8 row tiles: only 256 has the form, so the epilogue
//    is counted too, in k-blocks of a 128 x 256 tile: num_kb x kTile[bn] + epi, with epi = kEpiForm at 256 and kEpiRuntime x bn / 256 at the narrower widths on
//    the runtime form. The runtime epilogue costs about half a K = 4096 main loop per tile and a compiled one about a
//    quarter of that (README, "Kernels on Hopper"). At short K the runtime
//    epilogue dominates a narrow tile, so the GEMM stays at 256 with a badly filled last wave: ViT-L/14 fc at M = 2056
//    runs 272 tiles in 3 waves instead of 1088 tiles of 64 in 9 waves. With fewer row tiles each weight tile is shared
//    by few CTAs and the GEMM streams its weights from HBM, so filling the SMs matters more than the epilogue: the
//    decode workload, whose GPT-J prompt GEMMs run at M = 256 (qkv: 96 tiles of 256 against 384 of 64), was 6 % slower
//    with them planned this way, so they keep the first model.
static int pick_bn(int M, int N, int K, int batches, bool compiled_form) {
  if (N <= 64) return 64;
  const int tiles_m = (M + BM - 1) / BM;
  const int num_kb = (K + BK - 1) / BK;
  const int sms = num_sms();
  const bool weigh_epi = compiled_form && tiles_m >= 8;
  const double kTile[3] = {1.0, 0.55, 0.3}, kEpiRuntime = 32.0, kEpiForm = 8.0;
  const int cands[3] = {256, 128, 64};
  double best = 1e300;
  int best_bn = 256;
  for (int i = 0; i < 3; ++i) {
    const int bn = cands[i];
    if (bn > 64 && N <= bn / 2) continue;
    const long long t = (long long)tiles_m * ((N + bn - 1) / bn) * batches;
    const long long waves = (t + sms - 1) / sms;
    const double epi = bn == 256 ? kEpiForm : kEpiRuntime * bn / 256;
    const double cost = (double)waves * (weigh_epi ? num_kb * kTile[i] + epi : kTile[i]);
    if (cost < best - 1e-12) {
      best = cost;
      best_bn = bn;
    }
  }
  return best_bn;
}

// The plan of this thread's last successful mb200_gemm call (mb200_gemm_last_plan)
static thread_local int t_plan[2] = {0, 0};

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

  int bn = a->force_bn;  // 0: planned below
  MB_REQUIRE(bn == 0 || bn == 64 || bn == 128 || bn == 256, MB200_E_ARG, "gemm: force_bn must be 64, 128 or 256");

  CUtensorMap tmA, tmB;
  EpiMaps<true> tmE;
  memset(&tmE, 0, sizeof(tmE));
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
      GemmKernelParams kg = kp;  // the GEMM itself only writes partials (alpha applied); no epilogue inputs
      kg.epi_kind = EK_SPLITK;
      rc = dispatch_bn(bn, amn, bmn, tmA, tmB, tmE, kg, stream);
      if (rc) return rc;
      const long long n4 = (long long)a->M * ((a->N + 3) / 4);
      const int fgrid = (int)((n4 + 255) / 256 > 2048 ? 2048 : (n4 + 255) / 256);
      kp.alpha = 1.f;  // already applied to the partials
      MB_CUDA(launch_pdl(splitk_finalize_kernel, dim3(fgrid), dim3(256), 0, stream, kp));
      count_launch();
      t_plan[0] = bn;  // recorded once every launch of the call has succeeded
      t_plan[1] = split;
      return 0;
    }
  }
  rc = make_epi_maps(&tmE, &kp, a);
  if (rc) return rc;
  const uint32_t form = epi_form(a, kp);
  if (bn == 0) bn = pick_bn(a->M, a->N, a->K, a->nb0 * a->nb1, form != EF_RUNTIME);
  rc = make_operand_map(&tmB, a->B, a->N, a->K, a->nb0, a->nb1, bn);
  if (rc) return rc;
  kp.tiles_n = (a->N + bn - 1) / bn;
  kp.total_tiles = tiles_m * kp.tiles_n * a->nb0 * a->nb1;
  if (!(!a->generic_epilogue && bn == 256 && form != EF_RUNTIME &&
        dispatch_form(form, amn, bmn, tmA, tmB, tmE, &kp, stream, &rc)))
    rc = dispatch_bn(bn, amn, bmn, tmA, tmB, tmE, kp, stream);
  if (rc == 0) {
    t_plan[0] = bn;
    t_plan[1] = 1;
  }
  return rc;
}

}  // namespace mb200

extern "C" int mb200_gemm(const mb200_gemm_args* args, void* stream) {
  return mb200::gemm_impl(args, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int mb200_gemm_last_plan(int32_t* bn, int32_t* split_k) {
  if (bn) *bn = mb200::t_plan[0];
  if (split_k) *split_k = mb200::t_plan[1];
  return 0;
}
