// magma_b200 — error plumbing and device queries shared by all translation units.
#include "common.cuh"
#include "sched_rt.h"

#include <stdarg.h>
#include <stdlib.h>

namespace mb200 {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

const char* last_error() { return g_err; }

int check_cuda(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) at: %s", (int)e, cudaGetErrorString(e), what);
  return MB200_E_CUDA;
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

// SMs the persistent GEMM kernels may occupy (0 = all). Data-parallel training can leave a few SMs to NCCL's CTAs so the
// gradient all-reduce overlaps the backward GEMMs instead of waiting for gaps between them.
static int g_gemm_sm_limit = -1;
int gemm_sms() {
  if (g_gemm_sm_limit < 0) {
    const char* e = getenv("MB200_GEMM_SMS");
    g_gemm_sm_limit = e ? atoi(e) : 0;
    if (g_gemm_sm_limit < 0) g_gemm_sm_limit = 0;
  }
  const int n = num_sms();
  return (g_gemm_sm_limit >= 1 && g_gemm_sm_limit < n) ? g_gemm_sm_limit : n;
}
void set_gemm_sm_limit(int n) { g_gemm_sm_limit = n < 0 ? 0 : n; }

bool pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("MB200_PDL");
    v = e ? atoi(e) : 1;
  }
  return v != 0;
}

int check_arch() {
  static int cached = 1;  // 1 = unknown
  if (cached == 1) {
    int dev = 0, major = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    if (e != cudaSuccess) {
      set_error("no usable CUDA device (%s); magma_b200 has no CPU fallback", cudaGetErrorString(e));
      return MB200_E_ARCH;
    }
    if (major != 9) {
      set_error("device compute capability %d.x is not sm_90; magma_b200 kernels are sm_90a (Hopper) only", major);
      return MB200_E_ARCH;
    }
    cached = 0;
  }
  return cached;
}

// ---------------------------------------------------------------------------------------------
// runtime helpers of the host-only schedule files (sched_rt.h)
// ---------------------------------------------------------------------------------------------
int rt_check_arch() { return check_arch(); }
int rt_copy(void* dst, const void* src, size_t bytes, void* stream) {
  MB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}
int rt_zero(void* dst, size_t bytes, void* stream) {
  MB_CUDA(cudaMemsetAsync(dst, 0, bytes, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}

// ---------------------------------------------------------------------------------------------
// launch counter + per-GEMM event profiler
// ---------------------------------------------------------------------------------------------
static long long g_launches = 0;
void count_launch(int n) { g_launches += n; }
long long launches() { return g_launches; }

static const int kProfMax = 16384;
struct ProfState {
  bool enabled = false;
  int n = 0;
  cudaEvent_t* ev0 = nullptr;
  cudaEvent_t* ev1 = nullptr;
  double* flops = nullptr;
  double* bytes = nullptr;
  int created = 0;
};
static ProfState g_prof;

GemmProfScope::GemmProfScope(cudaStream_t s, double fl, double by) : on(false), st(s), slot(-1) {
  if (!g_prof.enabled || g_prof.n >= kProfMax) return;
  if (!g_prof.ev0) {
    g_prof.ev0 = new cudaEvent_t[kProfMax];
    g_prof.ev1 = new cudaEvent_t[kProfMax];
    g_prof.flops = new double[kProfMax];
    g_prof.bytes = new double[kProfMax];
  }
  slot = g_prof.n++;
  if (slot >= g_prof.created) {
    cudaEventCreate(&g_prof.ev0[slot]);
    cudaEventCreate(&g_prof.ev1[slot]);
    g_prof.created = slot + 1;
  }
  g_prof.flops[slot] = fl;
  g_prof.bytes[slot] = by;
  cudaEventRecord(g_prof.ev0[slot], st);
  on = true;
}
GemmProfScope::~GemmProfScope() {
  if (on) cudaEventRecord(g_prof.ev1[slot], st);
}

void prof_enable(int on) {
  g_prof.enabled = on != 0;
  g_prof.n = 0;
}
int prof_read(double* ms, double* flops, double* bytes, long long* n) {
  double tms = 0, tf = 0, tb = 0;
  for (int i = 0; i < g_prof.n; ++i) {
    float e = 0.f;
    cudaError_t err = cudaEventSynchronize(g_prof.ev1[i]);
    if (err == cudaSuccess) err = cudaEventElapsedTime(&e, g_prof.ev0[i], g_prof.ev1[i]);
    if (err != cudaSuccess) return check_cuda(err, "prof_read");
    tms += e;
    tf += g_prof.flops[i];
    tb += g_prof.bytes[i];
  }
  *ms = tms;
  *flops = tf;
  *bytes = tb;
  *n = g_prof.n;
  g_prof.n = 0;
  return 0;
}

}  // namespace mb200

namespace mb200 {
void set_gemm_sm_limit(int n);
const char* last_error();
long long launches();
void prof_enable(int on);
int prof_read(double* ms, double* flops, double* bytes, long long* n);
}

extern "C" long long mb200_launch_count(void) { return mb200::launches(); }
extern "C" int mb200_prof_enable(int on) {
  mb200::prof_enable(on);
  return 0;
}
extern "C" int mb200_prof_read(double* gemm_ms, double* gemm_flops, double* gemm_bytes, long long* gemm_launches) {
  return mb200::prof_read(gemm_ms, gemm_flops, gemm_bytes, gemm_launches);
}

extern "C" int mb200_set_gemm_sm_limit(int n_sms) {
  mb200::set_gemm_sm_limit(n_sms);
  return mb200::gemm_sms();
}
extern "C" int mb200_version(void) { return MB200_VERSION; }
extern "C" const char* mb200_last_error(void) { return mb200::last_error(); }
extern "C" int mb200_check_device(void) { return mb200::check_arch(); }
