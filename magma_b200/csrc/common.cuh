// magma_b200 — shared device/host helpers for the sm_90a kernels.
// Hand-written PTX wrappers for mbarrier and TMA (cp.async.bulk.tensor); warpgroup MMA lives in wgmma.cuh.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/magma_b200.h"

namespace mb200 {

typedef __nv_bfloat16 bf16;

// ---------------------------------------------------------------------------------------------
// error plumbing (thread-local last-error string, returned through mb200_last_error())
// ---------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int check_cuda(cudaError_t e, const char* what);

#define MB_CUDA(expr)                                                   \
  do {                                                                  \
    cudaError_t _e = (expr);                                            \
    if (_e != cudaSuccess) return mb200::check_cuda(_e, #expr);         \
  } while (0)

#define MB_REQUIRE(cond, code, ...)                                     \
  do {                                                                  \
    if (!(cond)) {                                                      \
      mb200::set_error(__VA_ARGS__);                                    \
      return (code);                                                    \
    }                                                                   \
  } while (0)

int num_sms();
int gemm_sms();  // SMs the persistent GEMM grids may use: num_sms() unless limited (mb200_set_gemm_sm_limit / MB200_GEMM_SMS)
int check_arch();  // 0 if the current device is sm_90 (Hopper), else MB200_E_ARCH
bool pdl_enabled();  // env MB200_PDL (default on)

// launch accounting (mb200_launch_count) and optional per-GEMM CUDA-event timing (mb200_prof_*)
void count_launch(int n = 1);
struct GemmProfScope {
  bool on;
  cudaStream_t st;
  int slot;
  GemmProfScope(cudaStream_t s, double flops, double bytes);
  ~GemmProfScope();
};

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
#ifdef __CUDACC__

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier ----
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded spin: a protocol bug traps (launch failure reported to the host) instead of hanging the GPU.
#ifndef MB200_SPIN_LIMIT
#define MB200_SPIN_LIMIT (1u << 26)
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > MB200_SPIN_LIMIT) __trap();
  }
}

// ---- TMA ----
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// rank-4 tiled load: coordinates (c0 = innermost, c1, c2, c3)
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
        "r"(c2), "r"(c3)
      : "memory");
}

// L2 prefetch of a rank-4 tile (no smem destination, no barrier)
__device__ __forceinline__ void tma_prefetch_4d(const CUtensorMap* m, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.prefetch.tensor.4d.L2.global [%0, {%1, %2, %3, %4}];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}

// ---- programmatic dependent launch (PDL) ----
// Kernels of the layer loop are launched with programmaticStreamSerialization: each CTA signals at its start that the
// next kernel in the stream may be scheduled (onto SMs as they free up), and every kernel blocks in pdl_wait() until
// its predecessor has fully completed and flushed before it touches global memory. The prologue of kernel N+1
// (barrier init, descriptor prefetch, launch latency) thereby overlaps the tail of kernel N.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---- per-warpgroup register reallocation (all threads of a warpgroup execute the same one) ----
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// ---- misc math ----
// gelu_new(x) = 0.5 x (1 + tanh(u)), u = sqrt(2/pi) (x + 0.044715 x^3). With 0.5 (1 + tanh(u)) = sigmoid(2u) this is
// x / (1 + exp(-2u)): one ex2 + one rcp on the SFU instead of tanhf's ~25-instruction branchy expansion, which was a
// visible share of the fc_in / fc_out-dgrad epilogues (4 epilogue warps, 256 elements per thread and tile). Relative
// error ~1e-6 (ex2.approx / rcp.approx), far inside the bf16 rounding of the stored result; saturates correctly
// (exp -> inf gives -0, exp -> 0 gives x).
__device__ __forceinline__ float gelu_new_f(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  float u = k0 * (x + k1 * x * x * x);
  return __fdividef(x, 1.f + __expf(-2.f * u));
}
__device__ __forceinline__ float gelu_new_grad_f(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  float u = k0 * (x + k1 * x * x * x);
  float s = __fdividef(1.f, 1.f + __expf(-2.f * u));  // sigmoid(2u) = 0.5 (1 + tanh u);  1 - tanh^2 u = 4 s (1 - s)
  return s + 2.f * x * s * (1.f - s) * k0 * (1.f + 3.f * k1 * x * x);
}
// x * sigmoid(1.702 x) with the approximate divide (rcp.approx + mul, 2 ulp): the IEEE '/' is a ~20-instruction dependent
// chain with a slow-path branch, which at one epilogue warp per scheduler made the ViT c_fc epilogue cost more than its
// mainloop (tools/epi_bench.py: vit fc 48 us against 19 us for the same GEMM with bias only).
__device__ __forceinline__ float quick_gelu_f(float x) { return __fdividef(x, 1.f + __expf(-1.702f * x)); }

#include "warp_helpers.cuh"
#include "wgmma.cuh"

#endif  // __CUDACC__

#ifdef __CUDACC__
// launch with the programmatic-stream-serialization attribute (PDL); falls back to a plain launch when disabled
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                     Args... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
#endif

}  // namespace mb200
