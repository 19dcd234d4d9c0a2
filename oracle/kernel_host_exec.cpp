// TEST INFRASTRUCTURE — executes the CUDA source of the product's HBM-bound operators on the CPU.
//
// This file compiles the kernel fragments and the C-ABI wrapper fragment (elt_abi.cuh) that elementwise.cu includes,
// UNCHANGED, as host C++, and runs them with the CUDA execution model emulated: every thread of a block is an OS thread
// with its own threadIdx, blocks run one after another, `__shared__` is block-shared static storage, `__syncthreads()` a
// block barrier, `__shfl_xor_sync` an exchange through a per-warp buffer, `atomicAdd` a locked add. The library's own
// mb200_* entry points thereby run here with their argument checks, error messages, memsets, launch geometry and launch
// counts, so magma_b200/ops.py can drive this library (tests/conftest.py::kernel_ops) and the EMULATION of each operator
// (cabi_emul.cpp) can be held to the kernel source. Only the number of SMs differs: num_sms() is 1 here.
// What this cannot show: anything the hardware decides — alignment faults, memory ordering, performance.
//
// The hx_* functions at the end are those entry points without their stream argument.
//
// Only tests build this (oracle/build_emul.py -> oracle/_build/libkernel_host_exec.so).
#ifndef _GNU_SOURCE
#define _GNU_SOURCE  // sincosf
#endif
#include <cuda_bf16.h>
// Philox4x32-10 of mb200_sample is plain arithmetic and compiles as host C++; the MTGP32 part of the header declares the
// built-in thread indices, which this file defines itself
#define threadIdx curand_unused_threadIdx
#define blockDim curand_unused_blockDim
#include <curand_kernel.h>
#undef threadIdx
#undef blockDim
#include <math.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <vector_functions.h>
#include <vector_types.h>

#include <condition_variable>
#include <mutex>
#include <thread>
#include <vector>

#include "../include/magma_b200.h"

// ---- the CUDA execution model, emulated -------------------------------------------------------------------------
static thread_local dim3 threadIdx, blockIdx;
static dim3 blockDim, gridDim;

class Barrier {  // reusable barrier for n threads
 public:
  explicit Barrier(int n) : n_(n) {}
  void wait() {
    std::unique_lock<std::mutex> lk(m_);
    const int gen = gen_;
    if (++count_ == n_) {
      count_ = 0;
      ++gen_;
      cv_.notify_all();
    } else {
      cv_.wait(lk, [&] { return gen != gen_; });
    }
  }

 private:
  std::mutex m_;
  std::condition_variable cv_;
  int n_, count_ = 0, gen_ = 0;
};

static Barrier* g_block_barrier = nullptr;
static std::vector<Barrier*> g_warp_barrier;
static float g_xch[1024];
static std::mutex g_atomic;

#define __global__
#define __device__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)
#define __shared__ static
#define __ldg(p) (*(p))
#define __expf expf
static inline void __syncthreads() { g_block_barrier->wait(); }
static inline float __shfl_xor_sync(unsigned, float v, int o) {
  const int t = (int)threadIdx.x, w = t >> 5;
  g_xch[t] = v;
  g_warp_barrier[w]->wait();
  const float r = g_xch[t ^ o];
  g_warp_barrier[w]->wait();
  return r;
}
static unsigned g_ballot[32];  // one word per warp
static inline unsigned __ballot_sync(unsigned, bool pred) {
  const int t = (int)threadIdx.x, w = t >> 5, l = t & 31;
  if (l == 0) g_ballot[w] = 0u;
  g_warp_barrier[w]->wait();
  if (pred) {
    std::lock_guard<std::mutex> lk(g_atomic);
    g_ballot[w] |= 1u << l;
  }
  g_warp_barrier[w]->wait();
  const unsigned r = g_ballot[w];
  g_warp_barrier[w]->wait();
  return r;
}
static int g_and;  // one word for the block
static inline int __syncthreads_and(int pred) {
  if (threadIdx.x == 0) g_and = 1;
  __syncthreads();
  if (!pred) {
    std::lock_guard<std::mutex> lk(g_atomic);
    g_and = 0;
  }
  __syncthreads();
  const int r = g_and;
  __syncthreads();
  return r;
}
static inline int __ffs(unsigned v) { return v ? __builtin_ffs((int)v) : 0; }
static inline int __shfl_xor_sync(unsigned, int v, int o) {
  static int xi[1024];
  const int t = (int)threadIdx.x, w = t >> 5;
  xi[t] = v;
  g_warp_barrier[w]->wait();
  const int r = xi[t ^ o];
  g_warp_barrier[w]->wait();
  return r;
}
template <typename T>
static inline T shfl_up(T v, int o) {  // lanes below o get their own value back, as on the GPU
  static T x[1024];
  const int t = (int)threadIdx.x, w = t >> 5;
  x[t] = v;
  g_warp_barrier[w]->wait();
  const T r = (t & 31) >= o ? x[t - o] : v;
  g_warp_barrier[w]->wait();
  return r;
}
static inline int __shfl_up_sync(unsigned, int v, int o) { return shfl_up(v, o); }
static inline double __shfl_up_sync(unsigned, double v, int o) { return shfl_up(v, o); }
static inline unsigned __float_as_uint(float x) {
  unsigned u;
  memcpy(&u, &x, 4);
  return u;
}
static inline float __uint_as_float(unsigned u) {
  float x;
  memcpy(&x, &u, 4);
  return x;
}
static inline float rsqrtf(float x) { return 1.0f / sqrtf(x); }
template <typename T> static inline T __ldcs(const T* p) { return *p; }             // cache-streaming hints: plain accesses
template <typename T> static inline void __stcs(T* p, const T& v) { *p = v; }
static inline void pdl_trigger() {}
static inline void pdl_wait() {}
static inline float atomicAdd(float* p, float v) {
  std::lock_guard<std::mutex> lk(g_atomic);
  const float old = *p;
  *p = old + v;
  return old;
}
static inline unsigned int atomicAdd(unsigned int* p, unsigned int v) {
  std::lock_guard<std::mutex> lk(g_atomic);
  const unsigned int old = *p;
  *p = old + v;
  return old;
}
static inline double atomicAdd(double* p, double v) {
  std::lock_guard<std::mutex> lk(g_atomic);
  const double old = *p;
  *p = old + v;
  return old;
}
static inline int atomicMin(int* p, int v) {
  std::lock_guard<std::mutex> lk(g_atomic);
  const int old = *p;
  if (v < old) *p = v;
  return old;
}
static inline void __threadfence() {}  // blocks run one after another here, threads of a block meet at barriers
template <typename T>
static inline T min(T a, T b) {
  return a < b ? a : b;
}
template <typename T>
static inline T max(T a, T b) {
  return a > b ? a : b;
}

template <typename F>
static void run_grid(dim3 grid, int threads, F&& body) {
  gridDim = grid;
  blockDim = dim3(threads);
  Barrier bb(threads);
  g_block_barrier = &bb;
  std::vector<Barrier*> wb;
  for (int w = 0; w < (threads + 31) / 32; ++w) {
    const int lanes = (w + 1) * 32 <= threads ? 32 : threads - w * 32;
    wb.push_back(new Barrier(lanes));
  }
  g_warp_barrier = wb;
  for (unsigned by = 0; by < grid.y; ++by)
    for (unsigned bx = 0; bx < grid.x; ++bx) {
      std::vector<std::thread> ts;
      for (int t = 0; t < threads; ++t)
        ts.emplace_back([&, t] {
          threadIdx = dim3(t);
          blockIdx = dim3(bx, by);
          body();
        });
      for (auto& th : ts) th.join();
    }
  for (auto* b : wb) delete b;
}

// ---- the product's kernel source, unchanged ---------------------------------------------------------------------
namespace mb200 {
typedef __nv_bfloat16 bf16;
#include "../magma_b200/csrc/warp_helpers.cuh"
#include "../magma_b200/csrc/elt_helpers.cuh"
#include "../magma_b200/csrc/elt_kernels.cuh"
#include "../magma_b200/csrc/train_kernels.cuh"
#include "../magma_b200/csrc/samp_kernels.cuh"
}  // namespace mb200

// ---- the host names the C-ABI fragment uses: a launch runs the grid above, a memset is memset --------------------
static thread_local char g_err[1024] = "";
namespace mb200 {
static void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
static int check_arch() { return 0; }
static long long g_launches = 0;
static void count_launch(int n = 1) { g_launches += n; }
// one SM: the grid-stride kernels run on 16 blocks of 256 threads, which keeps the OS threads per launch bounded
static int num_sms() { return 1; }
static void co_resident_kernels_init() {}
template <typename... KArgs, typename... Args>
static void launch(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t, cudaStream_t, Args... args) {
  run_grid(grid, (int)block.x, [&] { kern(static_cast<KArgs>(args)...); });
}
template <typename... KArgs, typename... Args>
static cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                              Args... args) {
  launch(kern, grid, block, smem, st, args...);
  return cudaSuccess;
}
}  // namespace mb200

#define MB_CUDA(expr)                               \
  do {                                              \
    if ((expr) != cudaSuccess) return MB200_E_CUDA; \
  } while (0)
#define MB_REQUIRE(cond, code, ...)  \
  do {                               \
    if (!(cond)) {                   \
      mb200::set_error(__VA_ARGS__); \
      return (code);                 \
    }                                \
  } while (0)
// macros, not functions: the CUDA runtime's own declarations of these names are in scope
#define cudaMemsetAsync(p, v, bytes, st) (memset((p), (v), (bytes)), cudaSuccess)
#define cudaGetLastError() cudaSuccess

#include "../magma_b200/csrc/elt_abi.cuh"

extern "C" {
long long mb200_launch_count(void) { return mb200::g_launches; }
const char* mb200_last_error(void) { return g_err; }
int mb200_version(void) { return MB200_VERSION; }
// the training kernels' entry points without their stream argument, as tests/test_kernel_source_cpu.py calls them
int hx_quick_gelu_bwd(const void* dy, const void* pre, void* dx, long long n) {
  return mb200_quick_gelu_bwd(dy, pre, dx, n, nullptr);
}
int hx_scale_add(const void* u, const float* s, const void* r1, const void* r2, void* out, long long n) {
  return mb200_scale_add(u, s, r1, r2, out, n, nullptr);
}
int hx_dot(const void* a, const void* b, long long n, float* out, int accumulate) {
  return mb200_dot(a, b, n, out, accumulate, nullptr);
}
int hx_layernorm_param_grad_rows(const void* dy, long long lddy, const void* x, long long ldx, const float* mean,
                                 const float* rstd, float* dgamma, float* dbeta, int rows, int d, int accumulate) {
  return mb200_layernorm_param_grad_rows(dy, lddy, x, ldx, mean, rstd, dgamma, dbeta, rows, d, accumulate, nullptr);
}
int hx_col_moments(const void* u, long long ldu, const void* v, long long ldv, const void* mask, long long ldm, int rows,
                   int cols, float* out1, float* out2) {
  return mb200_col_moments(u, ldu, v, ldv, mask, ldm, rows, cols, out1, out2, nullptr);
}
int hx_channel_affine(const void* x1, const float* a1, const void* x2, const float* a2, const float* c0, const void* mask,
                      const void* res, int relu, void* y, long long rows, int C) {
  return mb200_channel_affine(x1, a1, x2, a2, c0, mask, res, relu, y, rows, C, nullptr);
}
int hx_col2im3x3(const void* dcols, void* dx, int B, int H, int W, int C, int stride) {
  return mb200_col2im3x3(dcols, dx, B, H, W, C, stride, nullptr);
}
int hx_avgpool_nhwc_bwd(const void* dy, void* dx, int B, int H, int W, int C, int k) {
  return mb200_avgpool_nhwc_bwd(dy, dx, B, H, W, C, k, nullptr);
}
// curand_uniform after curand_init(seed, subsequence, offset), for the Python restatement of the draw in the tests
float hx_curand_uniform(unsigned long long seed, unsigned long long subsequence, unsigned long long offset) {
  curandStatePhilox4_32_10_t st;
  curand_init(seed, subsequence, offset, &st);
  return curand_uniform(&st);
}
}  // extern "C"
