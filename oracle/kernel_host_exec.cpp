// TEST INFRASTRUCTURE — executes CUDA KERNEL SOURCE of the product on the CPU.
//
// The training kernels (magma_b200/csrc/train_kernels.cuh) are checked on the GPU by tests/test_training_paths_gpu.py. Their
// schedules are also dry-run with emulated operators (cabi_emul.cpp), but that says nothing about the kernel code itself.
// This file compiles the kernel source UNCHANGED (the same .cuh fragments elementwise.cu includes) as host C++ and runs
// it with the CUDA execution model emulated: every thread of a block is an OS thread with its own threadIdx, blocks run
// one after another, `__shared__` is block-shared static storage, `__syncthreads()` a block barrier,
// `__shfl_xor_sync` an exchange through a per-warp buffer, `atomicAdd` a locked add. Indexing, vector handling, masks,
// reductions and accumulation logic of the kernels are thereby checked against torch (tests/test_kernel_source_cpu.py).
// What this cannot show: anything the hardware decides — alignment faults, memory ordering, performance.
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
#include <stdint.h>
#include <string.h>
#include <vector_functions.h>
#include <vector_types.h>

#include <condition_variable>
#include <mutex>
#include <thread>
#include <vector>

// ---- the CUDA execution model, emulated -------------------------------------------------------------------------
struct Dim3 {
  unsigned x = 1, y = 1, z = 1;
};
static thread_local Dim3 threadIdx, blockIdx;
static Dim3 blockDim, gridDim;

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
static void run_grid(Dim3 grid, int threads, F&& body) {
  gridDim = grid;
  blockDim = Dim3{(unsigned)threads, 1, 1};
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
          threadIdx = Dim3{(unsigned)t, 1, 1};
          blockIdx = Dim3{bx, by, 1};
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

using namespace mb200;

// ---- launchers: same grids / block sizes as the host wrappers in elementwise.cu ---------------------------------------
static int grid_for(long long n, int threads, int cap = 64) {  // any grid size is legal for the grid-stride kernels
  long long g = (n + threads - 1) / threads;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

extern "C" {

void hx_quick_gelu_bwd(const void* dy, const void* pre, void* dx, long long n) {
  run_grid(Dim3{(unsigned)grid_for(n / 8, 64), 1, 1}, 64,
           [&] { quick_gelu_bwd_kernel((const bf16*)dy, (const bf16*)pre, (bf16*)dx, n / 8); });
}

void hx_scale_add(const void* u, const float* s, const void* r1, const void* r2, void* out, long long n) {
  run_grid(Dim3{(unsigned)grid_for(n / 8, 64), 1, 1}, 64,
           [&] { scale_add_kernel((const bf16*)u, s, (const bf16*)r1, (const bf16*)r2, (bf16*)out, n / 8); });
}

void hx_dot(const void* a, const void* b, long long n, float* out, int accumulate) {
  if (!accumulate) *out = 0.f;
  run_grid(Dim3{(unsigned)grid_for(n / 8, 256, 4), 1, 1}, 256, [&] { dot_kernel((const bf16*)a, (const bf16*)b, n / 8, out); });
}

void hx_layernorm_param_grad_rows(const void* dy, long long lddy, const void* x, long long ldx, const float* mean,
                                  const float* rstd, float* dgamma, float* dbeta, int rows, int d, int accumulate) {
  if (!accumulate) {
    memset(dgamma, 0, (size_t)d * 4);
    memset(dbeta, 0, (size_t)d * 4);
  }
  run_grid(Dim3{(unsigned)((d + 63) / 64), (unsigned)((rows + kLnPgRows - 1) / kLnPgRows), 1}, 256, [&] {
    layernorm_param_grad_rows_kernel((const bf16*)dy, lddy, (const bf16*)x, ldx, mean, rstd, dgamma, dbeta, rows, d);
  });
}

void hx_col_moments(const void* u, long long ldu, const void* v, long long ldv, const void* mask, long long ldm, int rows,
                    int cols, float* out1, float* out2) {
  memset(out1, 0, (size_t)cols * 4);
  memset(out2, 0, (size_t)cols * 4);
  run_grid(Dim3{(unsigned)((cols + 63) / 64), (unsigned)((rows + kMomRows - 1) / kMomRows), 1}, 256, [&] {
    col_moments_kernel((const bf16*)u, ldu, (const bf16*)v, ldv, (const bf16*)mask, ldm, rows, cols, out1, out2);
  });
}

void hx_channel_affine(const void* x1, const float* a1, const void* x2, const float* a2, const float* c0, const void* mask,
                       const void* res, int relu, void* y, long long rows, int C) {
  run_grid(Dim3{(unsigned)grid_for(rows * (C / 8), 64), 1, 1}, 64, [&] {
    channel_affine_kernel((const bf16*)x1, a1, (const bf16*)x2, a2, c0, (const bf16*)mask, (const bf16*)res, relu, (bf16*)y,
                          rows, C);
  });
}

void hx_col2im3x3(const void* dcols, void* dx, int B, int H, int W, int C, int stride) {
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  run_grid(Dim3{(unsigned)grid_for((long long)B * H * W * (C / 8), 64), 1, 1}, 64,
           [&] { col2im3x3_kernel((const bf16*)dcols, (bf16*)dx, B, H, W, C, stride, Ho, Wo); });
}

void hx_avgpool_nhwc_bwd(const void* dy, void* dx, int B, int H, int W, int C, int k) {
  run_grid(Dim3{(unsigned)grid_for((long long)B * H * W * (C / 8), 64), 1, 1}, 64,
           [&] { avgpool_nhwc_bwd_kernel((const bf16*)dy, (bf16*)dx, B, H, W, C, k); });
}

}  // extern "C"


// =====================================================================================================================
// The GPU-verified kernels of elementwise.cu (csrc/elt_kernels.cuh) under the same executor, behind the C ABI's own names
// and with the launch configurations of the host wrappers in elementwise.cu — so magma_b200/ops.py can drive this library
// (tests/conftest.py::kernel_ops) and the EMULATION of each operator (cabi_emul.cpp) can be held to the kernel source.
// =====================================================================================================================
extern "C" {

int mb200_layernorm_fwd(const void* x, int64_t ldx, const void* gamma, const void* beta, void* y, int64_t ldy, float* mean,
                        float* rstd, int32_t rows, int32_t d, float eps, void*) {
  run_grid(Dim3{(unsigned)rows, 1, 1}, kLnThreads, [&] {
    layernorm_fwd_kernel((const bf16*)x, ldx, (const bf16*)gamma, (const bf16*)beta, (bf16*)y, ldy, mean, rstd, d, eps);
  });
  return 0;
}
int mb200_layernorm_bwd(const void* dy, int64_t lddy, const void* x, int64_t ldx, const void* gamma, const float* mean,
                        const float* rstd, const void* res, int64_t ldres, void* dx, int64_t lddx, int32_t rows, int32_t d,
                        void*) {
  run_grid(Dim3{(unsigned)rows, 1, 1}, kLnThreads, [&] {
    layernorm_bwd_kernel((const bf16*)dy, lddy, (const bf16*)x, ldx, (const bf16*)gamma, mean, rstd, (const bf16*)res, ldres,
                         (bf16*)dx, lddx, d);
  });
  return 0;
}
int mb200_layernorm_param_grad(const void* dy, int64_t lddy, const void* x, int64_t ldx, const float* mean,
                               const float* rstd, float* dgamma, float* dbeta, int32_t rows, int32_t d, int32_t accumulate,
                               void*) {
  run_grid(Dim3{(unsigned)((d + 127) / 128), 1, 1}, 128, [&] {
    layernorm_param_grad_kernel((const bf16*)dy, lddy, (const bf16*)x, ldx, mean, rstd, dgamma, dbeta, rows, d, accumulate);
  });
  return 0;
}
int mb200_layernorm_param_grad_rows(const void* dy, int64_t lddy, const void* x, int64_t ldx, const float* mean,
                                    const float* rstd, float* dgamma, float* dbeta, int32_t rows, int32_t d,
                                    int32_t accumulate, void*) {
  hx_layernorm_param_grad_rows(dy, lddy, x, ldx, mean, rstd, dgamma, dbeta, rows, d, accumulate);
  return 0;
}
int mb200_rope(void* qkv, int64_t ld, int32_t rows, int32_t S, int32_t H, int32_t hd, int32_t rot, int32_t pos0,
               int32_t inverse, void*) {
  run_grid(Dim3{(unsigned)grid_for((long long)rows * 2 * H * (rot / 2), 64), 1, 1}, 64,
           [&] { rope_kernel((bf16*)qkv, ld, rows, S, H, hd, rot, pos0, inverse); });
  return 0;
}
int mb200_rope_table(float* tab, int32_t S, int32_t rot, int32_t pos0, void*) {
  const int n = S * (rot / 2);
  run_grid(Dim3{(unsigned)((n + 63) / 64), 1, 1}, 64, [&] { rope_table_kernel((float2*)tab, S, rot / 2, rot, pos0); });
  return 0;
}
int mb200_softmax_fwd(const float* s, int64_t lds, int64_t s_bs, void* p, int64_t ldp, int64_t p_bs, int32_t nz, int32_t Sq,
                      int32_t Sk, float scale, int32_t causal, int32_t koff, void*) {
  const long long warps = (long long)nz * Sq;
  run_grid(Dim3{(unsigned)((warps + 7) / 8), 1, 1}, 256,
           [&] { softmax_fwd_kernel(s, lds, s_bs, (bf16*)p, ldp, p_bs, nz, Sq, Sk, scale, causal, koff); });
  return 0;
}
int mb200_softmax_bwd(const float* dp, int64_t lddp, int64_t dp_bs, const void* p, int64_t ldp, int64_t p_bs, void* ds,
                      int64_t ldds, int64_t ds_bs, int32_t nz, int32_t Sq, int32_t Sk, float scale, void*) {
  const long long warps = (long long)nz * Sq;
  run_grid(Dim3{(unsigned)((warps + 7) / 8), 1, 1}, 256, [&] {
    softmax_bwd_kernel(dp, lddp, dp_bs, (const bf16*)p, ldp, p_bs, (bf16*)ds, ldds, ds_bs, nz, Sq, Sk, scale);
  });
  return 0;
}
int mb200_build_labels(const int64_t* captions, int64_t ldc, int64_t* labels, int32_t B, int32_t S, int32_t L, int64_t eos,
                       void*) {
  run_grid(Dim3{(unsigned)((B * 32 + 127) / 128), 1, 1}, 128,
           [&] { build_labels_kernel((const long long*)captions, ldc, (long long*)labels, B, S, L, eos); });
  return 0;
}
int mb200_embed_assemble(const int64_t* captions, int64_t ldc, const void* wte, const void* prefix, int32_t L, void* x,
                         int32_t B, int32_t S, int32_t d, int32_t vocab, void*) {
  run_grid(Dim3{(unsigned)(B * S), 1, 1}, 64, [&] {
    embed_assemble_kernel((const long long*)captions, ldc, (const bf16*)wte, (const bf16*)prefix, L, (bf16*)x, B, S, d, vocab);
  });
  return 0;
}
int mb200_embed_gather(const int64_t* ids, const void* wte, void* out, int32_t n, int32_t d, int32_t vocab, void*) {
  run_grid(Dim3{(unsigned)n, 1, 1}, 64,
           [&] { embed_gather_kernel((const long long*)ids, (const bf16*)wte, (bf16*)out, d, vocab); });
  return 0;
}
int mb200_cross_entropy(const void* logits, int64_t ldv, const int64_t* labels, int32_t B, int32_t S, int32_t V,
                        float* row_loss, int32_t* n_valid, float* loss, void* dlogits, float grad_scale, void*) {
  run_grid(Dim3{1, 1, 1}, 1024, [&] { ce_count_kernel((const long long*)labels, B, S, V, n_valid); });
  run_grid(Dim3{(unsigned)(B * S), 1, 1}, kCeThreads, [&] {
    ce_row_kernel((const bf16*)logits, ldv, (const long long*)labels, S, V, n_valid, row_loss, (bf16*)dlogits, grad_scale);
  });
  run_grid(Dim3{1, 1, 1}, 1024, [&] { ce_reduce_kernel(row_loss, B * S, n_valid, loss); });
  return 0;
}
int mb200_colsum(const void* x, int64_t ldx, int32_t rows, int32_t cols, float* out, int32_t accumulate, void*) {
  if (!accumulate) memset(out, 0, (size_t)cols * 4);
  run_grid(Dim3{(unsigned)((cols + 63) / 64), (unsigned)((rows + kColsumRows - 1) / kColsumRows), 1}, 256,
           [&] { colsum_kernel((const bf16*)x, ldx, rows, cols, out); });
  return 0;
}
int mb200_dropout_fwd(const void* x, void* y, uint8_t* mask, int64_t n, float p, uint64_t seed, void*) {
  run_grid(Dim3{(unsigned)grid_for(n, 64), 1, 1}, 64,
           [&] { dropout_fwd_kernel((const bf16*)x, (bf16*)y, mask, n, p, (unsigned long long)seed); });
  return 0;
}
int mb200_dropout_apply(const void* x, const uint8_t* mask, void* y, int64_t n, float p, void*) {
  run_grid(Dim3{(unsigned)grid_for(n, 64), 1, 1}, 64, [&] { dropout_apply_kernel((const bf16*)x, mask, (bf16*)y, n, p); });
  return 0;
}
int mb200_patchify(const void* img, void* patches, int64_t ldp, int32_t B, int32_t R, int32_t Pp, void*) {
  const long long total = (long long)B * (R / Pp) * (R / Pp) * 3 * Pp * Pp;
  run_grid(Dim3{(unsigned)grid_for(total, 64), 1, 1}, 64,
           [&] { patchify_kernel((const bf16*)img, (bf16*)patches, ldp, B, R, Pp); });
  return 0;
}
int mb200_vit_assemble(void* x, const void* pe, const void* cls, const void* pos, int32_t B, int32_t T, int32_t w, void*) {
  run_grid(Dim3{(unsigned)grid_for((long long)B * T * w, 64), 1, 1}, 64,
           [&] { vit_assemble_kernel((bf16*)x, (const bf16*)pe, (const bf16*)cls, (const bf16*)pos, B, T, w); });
  return 0;
}
int mb200_nchw_to_nhwc8(const void* src, void* dst, int32_t B, int32_t C, int32_t H, int32_t W, void*) {
  run_grid(Dim3{(unsigned)grid_for((long long)B * H * W, 64), 1, 1}, 64,
           [&] { nchw_to_nhwc8_kernel((const bf16*)src, (bf16*)dst, B, C, H, W); });
  return 0;
}
int mb200_im2col3x3(const void* src, void* dst, int32_t B, int32_t H, int32_t W, int32_t C, int32_t stride, void*) {
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  const long long nvec = (long long)B * Ho * Wo * 9 * (C / 8);
  run_grid(Dim3{(unsigned)grid_for(nvec, 64), 1, 1}, 64,
           [&] { im2col3x3_kernel<unsigned int>((const bf16*)src, (bf16*)dst, B, H, W, C, stride, Ho, Wo); });
  return 0;
}
int mb200_avgpool_nhwc(const void* src, void* dst, int32_t B, int32_t H, int32_t W, int32_t C, int32_t k, void*) {
  run_grid(Dim3{(unsigned)grid_for((long long)B * (H / k) * (W / k) * (C / 8), 64), 1, 1}, 64,
           [&] { avgpool_nhwc_kernel((const bf16*)src, (bf16*)dst, B, H, W, C, k); });
  return 0;
}
int mb200_argmax(const void* x, int64_t ldx, int32_t rows, int32_t V, int64_t* out, void*) {
  run_grid(Dim3{(unsigned)rows, 1, 1}, 512, [&] { argmax_kernel((const bf16*)x, ldx, V, (long long*)out); });
  return 0;
}
int mb200_add(const void* a, const void* b, const void* c, void* y, int64_t n, void*) {
  run_grid(Dim3{(unsigned)grid_for(n / 8, 64), 1, 1}, 64,
           [&] { add_kernel((const bf16*)a, (const bf16*)b, (const bf16*)c, (bf16*)y, n / 8); });
  return 0;
}
int mb200_sumsq(const float* x, int64_t n, float* out, void*) {
  run_grid(Dim3{(unsigned)grid_for(n, 256, 4), 1, 1}, 256, [&] { sumsq_kernel(x, n, out); });
  return 0;
}
int mb200_adamw_step(float* master, float* grad, float* exp_avg, float* exp_avg_sq, void* shadow, int64_t n, float lr,
                     float beta1, float beta2, float eps, float weight_decay, float grad_scale, const float* gnorm_sq,
                     float max_norm, int32_t step, int32_t zero_grad, void*) {
  const float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
  run_grid(Dim3{(unsigned)grid_for(n / 4, 64), 1, 1}, 64, [&] {
    adamw_kernel(master, grad, exp_avg, exp_avg_sq, (bf16*)shadow, n / 4, lr, beta1, beta2, eps, weight_decay, grad_scale,
                 gnorm_sq, max_norm, bc1, bc2, zero_grad);
  });
  return 0;
}
int mb200_cast_f32_to_bf16(const float* src, void* dst, int64_t n, void*) {
  run_grid(Dim3{(unsigned)grid_for(n, 64), 1, 1}, 64, [&] { cast_f32_bf16_kernel(src, (bf16*)dst, n); });
  return 0;
}
int mb200_cast_bf16_to_f32(const void* src, float* dst, int64_t n, void*) {
  run_grid(Dim3{(unsigned)grid_for(n, 64), 1, 1}, 64, [&] { cast_bf16_f32_kernel((const bf16*)src, dst, n); });
  return 0;
}
// the training kernels under their C-ABI names as well
int mb200_quick_gelu_bwd(const void* dy, const void* pre, void* dx, int64_t n, void*) {
  hx_quick_gelu_bwd(dy, pre, dx, n);
  return 0;
}
int mb200_scale_add(const void* u, const float* s, const void* r1, const void* r2, void* out, int64_t n, void*) {
  hx_scale_add(u, s, r1, r2, out, n);
  return 0;
}
int mb200_dot(const void* a, const void* b, int64_t n, float* out, int32_t accumulate, void*) {
  hx_dot(a, b, n, out, accumulate);
  return 0;
}
int mb200_col_moments(const void* u, int64_t ldu, const void* v, int64_t ldv, const void* mask, int64_t ldm, int32_t rows,
                      int32_t cols, float* out1, float* out2, void*) {
  hx_col_moments(u, ldu, v, ldv, mask, ldm, rows, cols, out1, out2);
  return 0;
}
int mb200_channel_affine(const void* x1, const float* a1, const void* x2, const float* a2, const float* c0, const void* mask,
                         const void* res, int32_t relu, void* y, int64_t rows, int32_t C, void*) {
  hx_channel_affine(x1, a1, x2, a2, c0, mask, res, relu, y, rows, C);
  return 0;
}
int mb200_col2im3x3(const void* dcols, void* dx, int32_t B, int32_t H, int32_t W, int32_t C, int32_t stride, void*) {
  hx_col2im3x3(dcols, dx, B, H, W, C, stride);
  return 0;
}
int mb200_avgpool_nhwc_bwd(const void* dy, void* dx, int32_t B, int32_t H, int32_t W, int32_t C, int32_t k, void*) {
  hx_avgpool_nhwc_bwd(dy, dx, B, H, W, C, k);
  return 0;
}
int mb200_bn_finalize_fwd(const float* s1, const float* s2, const float* gamma, const float* beta, int64_t rows, float eps,
                          float momentum, float* running_mean, float* running_var, float* mean, float* rstd, float* scale,
                          float* shift, int32_t C, void*) {
  const float unbias = rows > 1 ? (float)((double)rows / (double)(rows - 1)) : 1.f;
  run_grid(Dim3{(unsigned)((C + 127) / 128), 1, 1}, 128, [&] {
    bn_finalize_fwd_kernel(s1, s2, gamma, beta, (float)(1.0 / (double)rows), unbias, eps, momentum, running_mean, running_var,
                           mean, rstd, scale, shift, C);
  });
  return 0;
}
int mb200_bn_bwd_coeffs(const float* s1, const float* t, const float* mean, const float* rstd, const float* gamma,
                        int64_t rows, float* dgamma, float* dbeta, int32_t accumulate, float* A, float* Bc, float* Cc,
                        int32_t C, void*) {
  run_grid(Dim3{(unsigned)((C + 127) / 128), 1, 1}, 128, [&] {
    bn_bwd_coeffs_kernel(s1, t, mean, rstd, gamma, (float)(1.0 / (double)rows), dgamma, dbeta, accumulate, A, Bc, Cc, C);
  });
  return 0;
}
// curand_uniform after curand_init(seed, subsequence, offset), for the Python restatement of the draw in the tests
float hx_curand_uniform(unsigned long long seed, unsigned long long subsequence, unsigned long long offset) {
  curandStatePhilox4_32_10_t st;
  curand_init(seed, subsequence, offset, &st);
  return curand_uniform(&st);
}
// sampling.cu and the gradient exchange: the kernels only, without the argument checks of the host wrappers
int mb200_sample(const void* logits, int32_t dtype, int64_t ld, int32_t rows, int32_t V, float temperature, int32_t top_k,
                 float top_p, uint64_t seed, uint64_t offset, int64_t* tokens, uint8_t* keep_mask, void*) {
  run_grid(Dim3{(unsigned)rows, 1, 1}, kSampThreads, [&] {
    if (dtype == 1)
      sample_kernel<float>((const float*)logits, ld, V, 1.f / temperature, top_k, top_p, seed, offset, (long long*)tokens,
                           keep_mask);
    else
      sample_kernel<bf16>((const bf16*)logits, ld, V, 1.f / temperature, top_k, top_p, seed, offset, (long long*)tokens,
                          keep_mask);
  });
  return 0;
}
int mb200_peer_reduce_bcast(void* const* bufs, int32_t world, int64_t offset, int64_t n, int32_t max_blocks, void*) {
  if (n == 0) return 0;
  PeerBufs pb;
  for (int r = 0; r < 16; ++r) pb.p[r] = r < world ? reinterpret_cast<float*>(bufs[r]) : nullptr;
  int grid = grid_for(n / 4, 256);
  if (max_blocks > 0 && grid > max_blocks) grid = max_blocks;
  run_grid(Dim3{(unsigned)grid, 1, 1}, 256, [&] { peer_reduce_bcast_kernel(pb, world, offset / 4, n / 4); });
  return 0;
}
const char* mb200_last_error(void) { return ""; }
int mb200_version(void) { return 100; }

}  // extern "C"
