// TEST INFRASTRUCTURE — CPU emulation of the PRIMITIVE operators of the magma_b200 C ABI.
//
// Purpose: the model-level schedules of the product (csrc/vit_sched.cu, csrc/gptj_sched.cu, written against csrc/sched_rt.h) are host
// code that only carves a workspace and issues primitive operators. tests/ compile such a schedule file as plain C++
// together with this file and run it on CPU tensors, so that every pointer offset, leading dimension, operand major,
// batch stride and accumulate flag of the schedule is checked against the oracle (torch autograd of
// oracle/magma_oracle.py) without a GPU. Each function below restates the documented semantics of the primitive it
// stands for (include/magma_b200.h; the kernel it mirrors is named next to it) in scalar C++ with bf16 storage and fp32
// arithmetic, and enforces the same argument rules as the CUDA host wrappers (alignment, leading dimensions), so a
// call the GPU library would reject is rejected here too.
//
// Only tests/ build and load this (oracle/build_emul.py). Nothing under magma_b200/ links, imports or executes it;
// it is not a fallback for anything — the product fails loudly without its CUDA library (magma_b200/_lib.py).
#include <math.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <vector>

#include "../include/magma_b200.h"

extern "C" int mb200_emul_tracing(void);

namespace mb200 {
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int rt_check_arch() { return 0; }
int rt_copy(void* dst, const void* src, size_t bytes, void*) {
  if (mb200_emul_tracing()) return 0;
  memmove(dst, src, bytes);
  return 0;
}
int rt_zero(void* dst, size_t bytes, void*) {
  if (mb200_emul_tracing()) return 0;
  memset(dst, 0, bytes);
  return 0;
}
}  // namespace mb200

#define EM_REQUIRE(cond, code, ...)   \
  do {                                \
    if (!(cond)) {                    \
      mb200::set_error(__VA_ARGS__);  \
      return (code);                  \
    }                                 \
  } while (0)

// ---- launch-plan trace (tools/plan_trace.py): with a trace file open every primitive logs one line — operator, shape,
// algorithmic FLOPs and bytes — and returns WITHOUT touching memory, so a full-size pass (GPT-J-6B at B = 8, S = 128) can be
// "issued" with placeholder pointers in milliseconds and the product's own schedule code writes out its launch plan.
static FILE* g_trace = nullptr;
extern "C" void mb200_emul_trace(const char* path) {
  if (g_trace) fclose(g_trace);
  g_trace = path ? fopen(path, "w") : nullptr;
}
extern "C" int mb200_emul_tracing(void) { return g_trace != nullptr; }
#define EM_TRACE(flops, bytes, ...)                                   \
  do {                                                                \
    if (g_trace) {                                                    \
      fprintf(g_trace, __VA_ARGS__);                                  \
      fprintf(g_trace, "\tflops=%.0f\tbytes=%.0f\n", (double)(flops), (double)(bytes)); \
      return 0;                                                       \
    }                                                                 \
  } while (0)

// ---- launch records (tools/plan_trace.py, tests/test_production_launches_*.py): with a record file open, every
// primitive a schedule issues also writes one JSON line holding every scalar argument its kernel or its plan depends
// on, and every pointer as a raw address (the caller gives each tensor its own placeholder base and resolves the
// address into (region, byte offset)). Written whether or not the trace is on, next to the trace line: after the
// argument checks for mb200_gemm and mb200_layernorm_param_grad_rows (a call they reject leaves no record), before
// them elsewhere, and always before the primitive computes anything.
static FILE* g_rec = nullptr;
extern "C" void mb200_emul_record(const char* path) {
  if (g_rec) fclose(g_rec);
  g_rec = path ? fopen(path, "w") : nullptr;
}
#define EM_RECORD(op, fmt, ...)                                          \
  do {                                                                   \
    if (g_rec) fprintf(g_rec, "{\"op\":\"" op "\"," fmt "}\n", __VA_ARGS__); \
  } while (0)
#define EM_P(p) (unsigned long long)reinterpret_cast<uintptr_t>(p)

typedef uint16_t bf16_t;
static inline float b2f(bf16_t v) {
  uint32_t u = (uint32_t)v << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
static inline bf16_t f2b(float f) {  // round to nearest even, like __float2bfloat16_rn
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (bf16_t)((u >> 16) | 0x40);
  u += 0x7fffu + ((u >> 16) & 1u);
  return (bf16_t)(u >> 16);
}
static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

static inline float gelu_new_f(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  return 0.5f * x * (1.f + tanhf(k0 * (x + k1 * x * x * x)));
}
static inline float gelu_new_grad_f(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  const float t = tanhf(k0 * (x + k1 * x * x * x));
  return 0.5f * (1.f + t) + 0.5f * x * (1.f - t * t) * k0 * (1.f + 3.f * k1 * x * x);
}
static inline float quick_gelu_f(float x) { return x / (1.f + expf(-1.702f * x)); }

extern "C" {

int mb200_version(void) { return MB200_VERSION; }
const char* mb200_last_error(void) { return mb200::g_err; }
int mb200_check_device(void) { return 0; }

// ---- mb200_gemm (csrc/gemm.cu::gemm_impl + the epilogue of csrc/gemm_common.cuh) ----
static int check_operand(const mb200_operand& op, int nb0, int nb1) {
  EM_REQUIRE(op.ptr != nullptr && aligned16(op.ptr), MB200_E_ALIGN, "gemm operand pointer not 16B aligned");
  EM_REQUIRE(op.ld % 8 == 0, MB200_E_ALIGN, "gemm operand ld (%lld) must be a multiple of 8 elements", (long long)op.ld);
  EM_REQUIRE((nb0 == 1 || op.bs0 % 8 == 0) && (nb1 == 1 || op.bs1 % 8 == 0), MB200_E_ALIGN,
             "gemm operand batch strides must be multiples of 8 elements");
  return 0;
}

int mb200_gemm(const mb200_gemm_args* a, void*) {
  EM_REQUIRE(a != nullptr, MB200_E_ARG, "null gemm args");
  EM_REQUIRE(a->M > 0 && a->N > 0 && a->K > 0 && a->nb0 > 0 && a->nb1 > 0, MB200_E_SHAPE, "gemm: bad shape");
  EM_REQUIRE(a->c_dtype == MB200_BF16 || a->c_dtype == MB200_F32, MB200_E_DTYPE, "gemm: bad c_dtype");
  EM_REQUIRE(!(a->accumulate && a->c_dtype != MB200_F32), MB200_E_DTYPE, "gemm: accumulate needs f32 output");
  EM_REQUIRE(!(a->dact && !a->aux_in), MB200_E_ARG, "gemm: dact needs aux_in");
  const int celt = a->c_dtype == MB200_F32 ? 4 : 8;
  EM_REQUIRE(a->C && aligned16(a->C) && a->ldc % celt == 0, MB200_E_ALIGN, "gemm: C must be 16B aligned with ldc %% %d",
             celt);
  EM_REQUIRE((a->nb0 == 1 || a->c_bs0 % celt == 0) && (a->nb1 == 1 || a->c_bs1 % celt == 0), MB200_E_ALIGN,
             "gemm: C batch strides must be multiples of %d elements", celt);
  if (a->res1 || a->res2) EM_REQUIRE(a->ld_res % 8 == 0, MB200_E_ALIGN, "gemm: ld_res must be a multiple of 8");
  if (a->aux_in || a->aux_out) EM_REQUIRE(a->ldc % 8 == 0, MB200_E_ALIGN, "gemm: aux tensors share ldc (must be %%8)");
  int rc = check_operand(a->A, a->nb0, a->nb1);
  if (rc) return rc;
  rc = check_operand(a->B, a->nb0, a->nb1);
  if (rc) return rc;
  const bool rope = a->rope_tab && a->rope_mode != 0;
  if (rope)
    EM_REQUIRE(a->rope_S > 0 && a->rope_hd > 0 && a->rope_rot % 4 == 0 && a->rope_rot <= a->rope_hd &&
                   a->rope_hd % 4 == 0 && a->rope_ncols % 4 == 0,
               MB200_E_ARG, "gemm: bad rope epilogue parameters");
  EM_RECORD("gemm",
            "\"M\":%d,\"N\":%d,\"K\":%d,\"nb0\":%d,\"nb1\":%d,"
            "\"A\":%llu,\"a_ld\":%lld,\"a_bs0\":%lld,\"a_bs1\":%lld,\"a_mn\":%d,"
            "\"B\":%llu,\"b_ld\":%lld,\"b_bs0\":%lld,\"b_bs1\":%lld,\"b_mn\":%d,\"b_static\":%d,"
            "\"c_dtype\":%d,\"C\":%llu,\"ldc\":%lld,\"c_bs0\":%lld,\"c_bs1\":%lld,\"alpha\":%.9g,"
            "\"act\":%d,\"dact\":%d,\"accumulate\":%d,\"bias\":%llu,\"aux_out\":%llu,\"aux_in\":%llu,"
            "\"res1\":%llu,\"res2\":%llu,\"ld_res\":%lld,\"force_bn\":%d,\"generic_epilogue\":%d,"
            "\"rope_mode\":%d,\"rope_tab\":%llu,\"rope_S\":%d,\"rope_hd\":%d,\"rope_rot\":%d,\"rope_ncols\":%d,"
            "\"splitk_ws\":%llu,\"splitk_ws_bytes\":%lld",
            a->M, a->N, a->K, a->nb0, a->nb1, EM_P(a->A.ptr), (long long)a->A.ld, (long long)a->A.bs0,
            (long long)a->A.bs1, a->A.mn_major, EM_P(a->B.ptr), (long long)a->B.ld, (long long)a->B.bs0,
            (long long)a->B.bs1, a->B.mn_major, a->B.static_data, a->c_dtype, EM_P(a->C), (long long)a->ldc,
            (long long)a->c_bs0, (long long)a->c_bs1, (double)a->alpha, a->act, a->dact, a->accumulate, EM_P(a->bias),
            EM_P(a->aux_out), EM_P(a->aux_in), EM_P(a->res1), EM_P(a->res2), (long long)a->ld_res, a->force_bn,
            a->generic_epilogue, a->rope_mode, EM_P(a->rope_tab), a->rope_S, a->rope_hd, a->rope_rot, a->rope_ncols,
            EM_P(a->splitk_ws), (long long)a->splitk_ws_bytes);
  {
    const double nb = (double)a->nb0 * a->nb1, csz = a->c_dtype == MB200_F32 ? 4.0 : 2.0;
    const double MN = (double)a->M * a->N;
    double bytes = nb * (2.0 * ((double)a->M * a->K + (double)a->N * a->K) + csz * MN);
    bytes += nb * 2.0 * MN * ((a->res1 ? 1 : 0) + (a->res2 ? 1 : 0) + (a->aux_in ? 1 : 0) + (a->aux_out ? 1 : 0));
    if (a->accumulate) bytes += nb * 4.0 * MN;
    EM_TRACE(2.0 * MN * a->K * nb, bytes,
             "gemm\tM=%d N=%d K=%d nb=%d a_mn=%d b_mn=%d c=%s bias=%d act=%d dact=%d res=%d aux=%d acc=%d rope=%d", a->M,
             a->N, a->K, a->nb0 * a->nb1, a->A.mn_major, a->B.mn_major, a->c_dtype == MB200_F32 ? "f32" : "bf16",
             a->bias != nullptr, a->act, a->dact, (a->res1 ? 1 : 0) + (a->res2 ? 1 : 0),
             (a->aux_in ? 1 : 0) + (a->aux_out ? 1 : 0), a->accumulate, rope ? a->rope_mode : 0);
  }
  const bf16_t* bias = (const bf16_t*)a->bias;
  const bf16_t* aux_in = (const bf16_t*)a->aux_in;
  bf16_t* aux_out = (bf16_t*)a->aux_out;
  const bf16_t* res1 = (const bf16_t*)a->res1;
  const bf16_t* res2 = (const bf16_t*)a->res2;
  const float* tab = (const float*)a->rope_tab;
  std::vector<float> row(a->N);
  for (int z = 0; z < a->nb0 * a->nb1; ++z) {
    const int z0 = z % a->nb0, z1 = z / a->nb0;
    const bf16_t* A = (const bf16_t*)a->A.ptr + z0 * a->A.bs0 + z1 * a->A.bs1;
    const bf16_t* B = (const bf16_t*)a->B.ptr + z0 * a->B.bs0 + z1 * a->B.bs1;
    const long long coff0 = z0 * a->c_bs0 + z1 * a->c_bs1;
    for (int m = 0; m < a->M; ++m) {
      for (int n = 0; n < a->N; ++n) {
        float acc = 0.f;
        for (int k = 0; k < a->K; ++k) {
          const float av = b2f(a->A.mn_major ? A[(long long)k * a->A.ld + m] : A[(long long)m * a->A.ld + k]);
          const float bv = b2f(a->B.mn_major ? B[(long long)k * a->B.ld + n] : B[(long long)n * a->B.ld + k]);
          acc += av * bv;
        }
        row[n] = a->alpha * acc + (bias ? b2f(bias[n]) : 0.f);
      }
      if (rope) {  // rotate_every_two on adjacent column pairs
        const float sg = a->rope_mode > 0 ? 1.f : -1.f;
        for (int n = 0; n + 1 < a->N && n < a->rope_ncols; n += 2) {
          const int dim = n % a->rope_hd;
          if (dim >= a->rope_rot) continue;
          const float* cs = tab + ((long long)(m % a->rope_S) * (a->rope_rot / 2) + dim / 2) * 2;
          const float x0 = row[n], x1 = row[n + 1];
          row[n] = x0 * cs[0] - x1 * cs[1] * sg;
          row[n + 1] = x1 * cs[0] + x0 * cs[1] * sg;
        }
      }
      for (int n = 0; n < a->N; ++n) {
        float x = row[n];
        const long long coff = coff0 + (long long)m * a->ldc + n;
        if (aux_out) aux_out[coff] = f2b(x);
        if (a->act == MB200_ACT_GELU_NEW) x = gelu_new_f(x);
        else if (a->act == MB200_ACT_QUICK_GELU) x = quick_gelu_f(x);
        else if (a->act == MB200_ACT_RELU) x = fmaxf(x, 0.f);
        if (a->dact) {
          const float p = b2f(aux_in[coff]);
          x = a->dact == MB200_DACT_GELU_NEW ? x * gelu_new_grad_f(p) : (p > 0.f ? x : 0.f);
        }
        const long long roff = coff0 + (long long)m * a->ld_res + n;  // residuals use C's batch offset
        if (res1) x += b2f(res1[roff]);
        if (res2) x += b2f(res2[roff]);
        if (a->act == MB200_ACT_RELU_POST) x = fmaxf(x, 0.f);
        if (a->c_dtype == MB200_F32) {
          float* dst = (float*)a->C + coff;
          *dst = a->accumulate ? *dst + x : x;
        } else {
          ((bf16_t*)a->C)[coff] = f2b(x);
        }
      }
    }
  }
  return 0;
}

// ---- LayerNorm (elementwise.cu: layernorm_fwd_kernel / layernorm_bwd_kernel / layernorm_param_grad*_kernel) ----
int mb200_layernorm_fwd(const void* x_, int64_t ldx, const void* gamma_, const void* beta_, void* y_, int64_t ldy,
                        float* mean, float* rstd, int32_t rows, int32_t d, float eps, void*) {
  EM_RECORD("layernorm_fwd",
            "\"x\":%llu,\"ldx\":%lld,\"gamma\":%llu,\"beta\":%llu,\"y\":%llu,\"ldy\":%lld,\"mean\":%llu,"
            "\"rstd\":%llu,\"rows\":%d,\"d\":%d,\"eps\":%.9g",
            EM_P(x_), (long long)ldx, EM_P(gamma_), EM_P(beta_), EM_P(y_), (long long)ldy, EM_P(mean), EM_P(rstd), rows,
            d, (double)eps);
  EM_TRACE(8.0 * rows * d, (double)rows * d * 4 + (mean ? rows * 8.0 : 0), "layernorm_fwd\trows=%d d=%d", rows, d);
  EM_REQUIRE(rows > 0 && d > 0 && d % 8 == 0 && d <= 8192, MB200_E_SHAPE, "layernorm: bad d=%d", d);
  EM_REQUIRE(ldx % 8 == 0 && ldy % 8 == 0, MB200_E_ALIGN, "layernorm: row strides must be multiples of 8");
  const bf16_t *x = (const bf16_t*)x_, *g = (const bf16_t*)gamma_, *b = (const bf16_t*)beta_;
  bf16_t* y = (bf16_t*)y_;
  std::vector<float> v(d);
  for (int r = 0; r < rows; ++r) {
    float s = 0.f;
    for (int c = 0; c < d; ++c) {
      v[c] = b2f(x[(long long)r * ldx + c]);  // the row is read completely before it is written (in place is legal)
      s += v[c];
    }
    const float mu = s / d;
    float q = 0.f;
    for (int c = 0; c < d; ++c) q += (v[c] - mu) * (v[c] - mu);
    const float rs = 1.f / sqrtf(q / d + eps);
    if (mean) mean[r] = mu;
    if (rstd) rstd[r] = rs;
    for (int c = 0; c < d; ++c) y[(long long)r * ldy + c] = f2b((v[c] - mu) * rs * b2f(g[c]) + b2f(b[c]));
  }
  return 0;
}

int mb200_layernorm_bwd(const void* dy_, int64_t lddy, const void* x_, int64_t ldx, const void* gamma_,
                        const float* mean, const float* rstd, const void* res_, int64_t ldres, void* dx_, int64_t lddx,
                        int32_t rows, int32_t d, void*) {
  EM_RECORD("layernorm_bwd",
            "\"dy\":%llu,\"lddy\":%lld,\"x\":%llu,\"ldx\":%lld,\"gamma\":%llu,\"mean\":%llu,\"rstd\":%llu,"
            "\"res\":%llu,\"ldres\":%lld,\"dx\":%llu,\"lddx\":%lld,\"rows\":%d,\"d\":%d",
            EM_P(dy_), (long long)lddy, EM_P(x_), (long long)ldx, EM_P(gamma_), EM_P(mean), EM_P(rstd), EM_P(res_),
            (long long)ldres, EM_P(dx_), (long long)lddx, rows, d);
  EM_TRACE(12.0 * rows * d, (double)rows * d * (res_ ? 8 : 6), "layernorm_bwd\trows=%d d=%d res=%d", rows, d, res_ != nullptr);
  EM_REQUIRE(rows > 0 && d > 0 && d % 8 == 0 && d <= 8192, MB200_E_SHAPE, "layernorm_bwd: bad d=%d", d);
  EM_REQUIRE(lddy % 8 == 0 && ldx % 8 == 0 && lddx % 8 == 0 && (!res_ || ldres % 8 == 0), MB200_E_ALIGN,
             "layernorm_bwd: row strides must be multiples of 8");
  const bf16_t *dy = (const bf16_t*)dy_, *x = (const bf16_t*)x_, *gm = (const bf16_t*)gamma_, *res = (const bf16_t*)res_;
  bf16_t* dx = (bf16_t*)dx_;
  std::vector<float> g(d), xh(d), rr(d);
  for (int r = 0; r < rows; ++r) {
    float s1 = 0.f, s2 = 0.f;
    for (int c = 0; c < d; ++c) {
      g[c] = b2f(dy[(long long)r * lddy + c]) * b2f(gm[c]);
      xh[c] = (b2f(x[(long long)r * ldx + c]) - mean[r]) * rstd[r];
      rr[c] = res ? b2f(res[(long long)r * ldres + c]) : 0.f;
      s1 += g[c];
      s2 += g[c] * xh[c];
    }
    const float m1 = s1 / d, m2 = s2 / d;
    for (int c = 0; c < d; ++c) dx[(long long)r * lddx + c] = f2b(rstd[r] * (g[c] - m1 - xh[c] * m2) + rr[c]);
  }
  return 0;
}

static int ln_param_grad(const void* dy_, int64_t lddy, const void* x_, int64_t ldx, const float* mean,
                         const float* rstd, float* dgamma, float* dbeta, int32_t rows, int32_t d, int32_t accumulate) {
  EM_TRACE(4.0 * rows * d, (double)rows * d * 4, "layernorm_param_grad\trows=%d d=%d", rows, d);
  const bf16_t *dy = (const bf16_t*)dy_, *x = (const bf16_t*)x_;
  for (int c = 0; c < d; ++c) {
    float sg = 0.f, sb = 0.f;
    for (int r = 0; r < rows; ++r) {
      const float g = b2f(dy[(long long)r * lddy + c]);
      sg += g * (b2f(x[(long long)r * ldx + c]) - mean[r]) * rstd[r];
      sb += g;
    }
    dgamma[c] = accumulate ? dgamma[c] + sg : sg;
    dbeta[c] = accumulate ? dbeta[c] + sb : sb;
  }
  return 0;
}
int mb200_layernorm_param_grad(const void* dy, int64_t lddy, const void* x, int64_t ldx, const float* mean,
                               const float* rstd, float* dgamma, float* dbeta, int32_t rows, int32_t d,
                               int32_t accumulate, void*) {
  EM_RECORD("layernorm_param_grad",
            "\"dy\":%llu,\"lddy\":%lld,\"x\":%llu,\"ldx\":%lld,\"mean\":%llu,\"rstd\":%llu,\"dgamma\":%llu,"
            "\"dbeta\":%llu,\"rows\":%d,\"d\":%d,\"accumulate\":%d",
            EM_P(dy), (long long)lddy, EM_P(x), (long long)ldx, EM_P(mean), EM_P(rstd), EM_P(dgamma), EM_P(dbeta), rows,
            d, accumulate);
  return ln_param_grad(dy, lddy, x, ldx, mean, rstd, dgamma, dbeta, rows, d, accumulate);
}
int mb200_layernorm_param_grad_rows(const void* dy, int64_t lddy, const void* x, int64_t ldx, const float* mean,
                                    const float* rstd, float* dgamma, float* dbeta, int32_t rows, int32_t d,
                                    int32_t accumulate, void*) {
  /* traced in ln_param_grad */
  EM_REQUIRE(rows > 0 && d > 0 && d % 2 == 0 && lddy % 2 == 0 && ldx % 2 == 0, MB200_E_ALIGN,
             "layernorm_param_grad_rows: d and row strides must be even");
  EM_RECORD("layernorm_param_grad_rows",
            "\"dy\":%llu,\"lddy\":%lld,\"x\":%llu,\"ldx\":%lld,\"mean\":%llu,\"rstd\":%llu,\"dgamma\":%llu,"
            "\"dbeta\":%llu,\"rows\":%d,\"d\":%d,\"accumulate\":%d",
            EM_P(dy), (long long)lddy, EM_P(x), (long long)ldx, EM_P(mean), EM_P(rstd), EM_P(dgamma), EM_P(dbeta), rows,
            d, accumulate);
  return ln_param_grad(dy, lddy, x, ldx, mean, rstd, dgamma, dbeta, rows, d, accumulate);
}

// ---- softmax (elementwise.cu: softmax_fwd_kernel / softmax_bwd_kernel) ----
int mb200_softmax_fwd(const float* s, int64_t lds, int64_t s_bs, void* p_, int64_t ldp, int64_t p_bs, int32_t nz,
                      int32_t Sq, int32_t Sk, float scale, int32_t causal, int32_t koff, void*) {
  EM_RECORD("softmax_fwd",
            "\"s\":%llu,\"lds\":%lld,\"s_bs\":%lld,\"p\":%llu,\"ldp\":%lld,\"p_bs\":%lld,\"nz\":%d,\"Sq\":%d,"
            "\"Sk\":%d,\"scale\":%.9g,\"causal\":%d,\"koff\":%d",
            EM_P(s), (long long)lds, (long long)s_bs, EM_P(p_), (long long)ldp, (long long)p_bs, nz, Sq, Sk,
            (double)scale, causal, koff);
  EM_TRACE(5.0 * nz * Sq * Sk, (double)nz * Sq * Sk * 6, "softmax_fwd\tnz=%d Sq=%d Sk=%d causal=%d", nz, Sq, Sk, causal);
  bf16_t* p = (bf16_t*)p_;
  for (int z = 0; z < nz; ++z)
    for (int i = 0; i < Sq; ++i) {
      const float* sr = s + (long long)z * s_bs + (long long)i * lds;
      bf16_t* pr = p + (long long)z * p_bs + (long long)i * ldp;
      int lim = Sk;
      if (causal && i + koff + 1 < Sk) lim = i + koff + 1;
      float m = -INFINITY, sum = 0.f;
      for (int j = 0; j < lim; ++j) m = fmaxf(m, sr[j] * scale);
      for (int j = 0; j < lim; ++j) sum += expf(sr[j] * scale - m);
      for (int j = 0; j < Sk; ++j) pr[j] = f2b(j < lim ? expf(sr[j] * scale - m) / sum : 0.f);  // pad columns untouched
    }
  return 0;
}

int mb200_softmax_bwd(const float* dp, int64_t lddp, int64_t dp_bs, const void* p_, int64_t ldp, int64_t p_bs,
                      void* ds_, int64_t ldds, int64_t ds_bs, int32_t nz, int32_t Sq, int32_t Sk, float scale, void*) {
  EM_RECORD("softmax_bwd",
            "\"dp\":%llu,\"lddp\":%lld,\"dp_bs\":%lld,\"p\":%llu,\"ldp\":%lld,\"p_bs\":%lld,\"ds\":%llu,"
            "\"ldds\":%lld,\"ds_bs\":%lld,\"nz\":%d,\"Sq\":%d,\"Sk\":%d,\"scale\":%.9g",
            EM_P(dp), (long long)lddp, (long long)dp_bs, EM_P(p_), (long long)ldp, (long long)p_bs, EM_P(ds_), (long
            long)ldds, (long long)ds_bs, nz, Sq, Sk, (double)scale);
  EM_TRACE(4.0 * nz * Sq * Sk, (double)nz * Sq * Sk * 8, "softmax_bwd\tnz=%d Sq=%d Sk=%d", nz, Sq, Sk);
  const bf16_t* p = (const bf16_t*)p_;
  bf16_t* ds = (bf16_t*)ds_;
  for (int z = 0; z < nz; ++z)
    for (int i = 0; i < Sq; ++i) {
      const float* dpr = dp + (long long)z * dp_bs + (long long)i * lddp;
      const bf16_t* pr = p + (long long)z * p_bs + (long long)i * ldp;
      bf16_t* dsr = ds + (long long)z * ds_bs + (long long)i * ldds;
      float acc = 0.f;
      for (int j = 0; j < Sk; ++j) acc += dpr[j] * b2f(pr[j]);
      for (int j = 0; j < Sk; ++j) dsr[j] = f2b(b2f(pr[j]) * (dpr[j] - acc) * scale);
    }
  return 0;
}

// ---- reductions / elementwise / ViT front end ----
int mb200_colsum(const void* x_, int64_t ldx, int32_t rows, int32_t cols, float* out, int32_t accumulate, void*) {
  EM_RECORD("colsum",
            "\"x\":%llu,\"ldx\":%lld,\"rows\":%d,\"cols\":%d,\"out\":%llu,\"accumulate\":%d",
            EM_P(x_), (long long)ldx, rows, cols, EM_P(out), accumulate);
  EM_TRACE((double)rows * cols, (double)rows * cols * 2, "colsum\trows=%d cols=%d", rows, cols);
  EM_REQUIRE(cols % 2 == 0 && ldx % 2 == 0, MB200_E_ALIGN, "colsum: cols and ldx must be even");
  const bf16_t* x = (const bf16_t*)x_;
  for (int c = 0; c < cols; ++c) {
    float s = 0.f;
    for (int r = 0; r < rows; ++r) s += b2f(x[(long long)r * ldx + c]);
    out[c] = accumulate ? out[c] + s : s;
  }
  return 0;
}

int mb200_quick_gelu_bwd(const void* dy_, const void* pre_, void* dx_, int64_t n, void*) {
  EM_RECORD("quick_gelu_bwd",
            "\"dy\":%llu,\"pre\":%llu,\"dx\":%llu,\"n\":%lld",
            EM_P(dy_), EM_P(pre_), EM_P(dx_), (long long)n);
  EM_TRACE(8.0 * n, (double)n * 6, "quick_gelu_bwd\tn=%lld", (long long)n);
  EM_REQUIRE(n > 0 && n % 8 == 0, MB200_E_SHAPE, "quick_gelu_bwd: n must be a positive multiple of 8");
  EM_REQUIRE(aligned16(dy_) && aligned16(pre_) && aligned16(dx_), MB200_E_ALIGN, "quick_gelu_bwd: 16B alignment");
  const bf16_t *dy = (const bf16_t*)dy_, *pre = (const bf16_t*)pre_;
  bf16_t* dx = (bf16_t*)dx_;
  for (int64_t i = 0; i < n; ++i) {
    const float x = b2f(pre[i]), s = 1.f / (1.f + expf(-1.702f * x));
    dx[i] = f2b(b2f(dy[i]) * (s + 1.702f * x * s * (1.f - s)));
  }
  return 0;
}

// out = s[0] * u + r1 + r2   (scale_add_kernel)
int mb200_scale_add(const void* u_, const float* s, const void* r1_, const void* r2_, void* out_, int64_t n, void*) {
  EM_RECORD("scale_add",
            "\"u\":%llu,\"s\":%llu,\"r1\":%llu,\"r2\":%llu,\"out\":%llu,\"n\":%lld",
            EM_P(u_), EM_P(s), EM_P(r1_), EM_P(r2_), EM_P(out_), (long long)n);
  EM_TRACE(3.0 * n, (double)n * (4 + (r1_ ? 2 : 0) + (r2_ ? 2 : 0)), "scale_add\tn=%lld", (long long)n);
  EM_REQUIRE(n > 0 && n % 8 == 0, MB200_E_SHAPE, "scale_add: n must be a positive multiple of 8");
  EM_REQUIRE(aligned16(u_) && aligned16(r1_) && aligned16(r2_) && aligned16(out_), MB200_E_ALIGN, "scale_add: alignment");
  const bf16_t *u = (const bf16_t*)u_, *r1 = (const bf16_t*)r1_, *r2 = (const bf16_t*)r2_;
  bf16_t* out = (bf16_t*)out_;
  const float sc = s ? *s : 1.f;
  for (int64_t i = 0; i < n; ++i) out[i] = f2b(b2f(u[i]) * sc + (r1 ? b2f(r1[i]) : 0.f) + (r2 ? b2f(r2[i]) : 0.f));
  return 0;
}

// out[0] (+)= <a, b>   (dot_kernel)
int mb200_dot(const void* a_, const void* b_, int64_t n, float* out, int32_t accumulate, void*) {
  EM_RECORD("dot",
            "\"a\":%llu,\"b\":%llu,\"n\":%lld,\"out\":%llu,\"accumulate\":%d",
            EM_P(a_), EM_P(b_), (long long)n, EM_P(out), accumulate);
  EM_TRACE(2.0 * n, (double)n * 4, "dot\tn=%lld", (long long)n);
  EM_REQUIRE(n > 0 && n % 8 == 0, MB200_E_SHAPE, "dot: n must be a positive multiple of 8");
  EM_REQUIRE(aligned16(a_) && aligned16(b_), MB200_E_ALIGN, "dot: alignment");
  const bf16_t *a = (const bf16_t*)a_, *b = (const bf16_t*)b_;
  double acc = 0.0;
  for (int64_t i = 0; i < n; ++i) acc += (double)b2f(a[i]) * (double)b2f(b[i]);
  out[0] = (accumulate ? out[0] : 0.f) + (float)acc;
  return 0;
}

// (cos, sin) fp32 [S][rot/2][2]   (rope_table_kernel)
int mb200_rope_table(float* tab, int32_t S, int32_t rot, int32_t pos0, void*) {
  EM_RECORD("rope_table", "\"tab\":%llu,\"S\":%d,\"rot\":%d,\"pos0\":%d", EM_P(tab), S, rot, pos0);
  EM_TRACE(0, (double)S * rot * 4, "rope_table\tS=%d rot=%d", S, rot);
  EM_REQUIRE(S > 0 && rot > 0 && rot % 2 == 0, MB200_E_SHAPE, "rope_table: bad S / rot");
  const int half = rot / 2;
  for (int s = 0; s < S; ++s)
    for (int p = 0; p < half; ++p) {
      const float inv_freq = 1.0f / powf(10000.0f, (float)(2 * p) / (float)rot);
      const float ang = (float)(pos0 + s) * inv_freq;
      tab[((long long)s * half + p) * 2] = cosf(ang);
      tab[((long long)s * half + p) * 2 + 1] = sinf(ang);
    }
  return 0;
}

// shifted cross-entropy over bf16 logits, mean over valid targets; dlogits = grad_scale * (softmax - onehot) / n_valid,
// zero rows where the target is ignored; dlogits may alias logits   (ce_count / ce_row / ce_reduce kernels)
int mb200_cross_entropy(const void* logits_, int64_t ldv, const int64_t* labels, int32_t B, int32_t S, int32_t V,
                        float* row_loss, int32_t* n_valid, float* loss, void* dlogits_, float grad_scale, void*) {
  EM_RECORD("cross_entropy",
            "\"logits\":%llu,\"ldv\":%lld,\"labels\":%llu,\"B\":%d,\"S\":%d,\"V\":%d,\"row_loss\":%llu,"
            "\"n_valid\":%llu,\"loss\":%llu,\"dlogits\":%llu,\"grad_scale\":%.9g",
            EM_P(logits_), (long long)ldv, EM_P(labels), B, S, V, EM_P(row_loss), EM_P(n_valid), EM_P(loss),
            EM_P(dlogits_), (double)grad_scale);
  EM_TRACE(6.0 * B * S * V, (double)B * S * V * (dlogits_ ? 4 : 2), "cross_entropy\trows=%d V=%d grad=%d", B * S, V, dlogits_ != nullptr);
  EM_REQUIRE(ldv % 8 == 0 && V <= ldv, MB200_E_ALIGN, "cross_entropy: ldv must be a multiple of 8 and >= V");
  const bf16_t* logits = (const bf16_t*)logits_;
  bf16_t* dlogits = (bf16_t*)dlogits_;
  int nv = 0;
  for (int i = 0; i < B * S; ++i)
    if (i % S + 1 < S && labels[i + 1] >= 0 && labels[i + 1] < V) ++nv;
  *n_valid = nv;
  const float gs = grad_scale / (float)(nv > 0 ? nv : 1);
  double total = 0.0;
  std::vector<float> f(V);
  for (int row = 0; row < B * S; ++row) {
    const int s = row % S;
    const long long tgt = s + 1 < S ? labels[row + 1] : -100;
    const bf16_t* lr = logits + (long long)row * ldv;
    bf16_t* dr = dlogits ? dlogits + (long long)row * ldv : nullptr;
    if (tgt < 0 || tgt >= V) {
      row_loss[row] = 0.f;
      if (dr)
        for (int j = 0; j < V; ++j) dr[j] = f2b(0.f);
      continue;
    }
    float m = -INFINITY, sum = 0.f;
    for (int j = 0; j < V; ++j) {
      f[j] = b2f(lr[j]);
      m = fmaxf(m, f[j]);
    }
    for (int j = 0; j < V; ++j) sum += expf(f[j] - m);
    row_loss[row] = m + logf(sum) - f[tgt];
    total += row_loss[row];
    if (dr)
      for (int j = 0; j < V; ++j) dr[j] = f2b((expf(f[j] - m) / sum - (j == tgt ? 1.f : 0.f)) * gs);
  }
  *loss = (float)(total / (double)(nv > 0 ? nv : 1));
  return 0;
}

// ---- remaining primitives, so that host-side Python schedules (image_prefix.py, adapters.py, the conv trunk of
// image_encoders.py, arena.py) can be dry-run on CPU tensors through magma_b200/ops.py (tests/conftest.py::emul_ops) ----
long long mb200_launch_count(void) { return 0; }
int mb200_prof_enable(int) { return 0; }
int mb200_prof_read(double* a, double* b, double* c, long long* n) {
  *a = *b = *c = 0.0;
  *n = 0;
  return 0;
}
int mb200_set_gemm_sm_limit(int) { return 132; }
int mb200_set_optimizer_grid(int n) { return n; }

int mb200_rope(void* qkv_, int64_t ld, int32_t rows, int32_t S, int32_t H, int32_t hd, int32_t rot, int32_t pos0,
               int32_t inverse, void*) {  // rope_kernel: in place on q and k of a fused [rows][3][H][hd] buffer
  EM_REQUIRE(rot % 2 == 0 && rot <= hd && rows > 0, MB200_E_SHAPE, "rope: bad rot / hd");
  bf16_t* qkv = (bf16_t*)qkv_;
  for (long long r = 0; r < rows; ++r)
    for (int which = 0; which < 2; ++which)
      for (int h = 0; h < H; ++h)
        for (int p = 0; p < rot / 2; ++p) {
          const float inv_freq = 1.0f / powf(10000.0f, (float)(2 * p) / (float)rot);
          const float ang = (float)(pos0 + (int)(r % S)) * inv_freq;
          const float cs = cosf(ang), sn = inverse ? -sinf(ang) : sinf(ang);
          bf16_t* q = qkv + r * ld + (long long)which * H * hd + (long long)h * hd + 2 * p;
          const float x = b2f(q[0]), y = b2f(q[1]);
          q[0] = f2b(x * cs - y * sn);
          q[1] = f2b(y * cs + x * sn);
        }
  return 0;
}

int mb200_build_labels(const int64_t* captions, int64_t ldc, int64_t* labels, int32_t B, int32_t S, int32_t L,
                       int64_t eos, void*) {  // build_labels_kernel
  EM_REQUIRE(B > 0 && S > 0 && L >= 0 && L <= S, MB200_E_SHAPE, "build_labels: need 0 <= L <= S");
  for (int b = 0; b < B; ++b) {
    int first = S;
    for (int s = L; s < S; ++s)
      if (captions[(long long)b * ldc + (s - L)] == eos) {
        first = s;
        break;
      }
    for (int s = 0; s < S; ++s) {
      int64_t v = s < L ? -100 : captions[(long long)b * ldc + (s - L)];
      if (s > first) v = -100;
      labels[(long long)b * S + s] = v;
    }
  }
  return 0;
}

int mb200_embed_assemble(const int64_t* captions, int64_t ldc, const void* wte_, const void* prefix_, int32_t L, void* x_,
                         int32_t B, int32_t S, int32_t d, int32_t vocab, void*) {  // embed_assemble_kernel
  EM_REQUIRE(d % 8 == 0 && L >= 0 && L <= S, MB200_E_SHAPE, "embed_assemble: bad d / L / S");
  const bf16_t *wte = (const bf16_t*)wte_, *prefix = (const bf16_t*)prefix_;
  bf16_t* x = (bf16_t*)x_;
  for (int b = 0; b < B; ++b)
    for (int s = 0; s < S; ++s) {
      const bf16_t* src;
      if (s < L) {
        src = prefix + ((long long)b * L + s) * d;
      } else {
        long long tok = captions[(long long)b * ldc + (s - L)];
        if (tok < 0 || tok >= vocab) tok = 0;
        src = wte + tok * (long long)d;
      }
      memcpy(x + ((long long)b * S + s) * d, src, (size_t)d * 2);
    }
  return 0;
}

int mb200_embed_gather(const int64_t* ids, const void* wte_, void* out_, int32_t n, int32_t d, int32_t vocab, void*) {
  EM_REQUIRE(d % 8 == 0 && n > 0, MB200_E_SHAPE, "embed_gather: bad n / d");
  const bf16_t* wte = (const bf16_t*)wte_;
  bf16_t* out = (bf16_t*)out_;
  for (int r = 0; r < n; ++r) {
    long long tok = ids[r];
    if (tok < 0 || tok >= vocab) tok = 0;
    memcpy(out + (long long)r * d, wte + tok * (long long)d, (size_t)d * 2);
  }
  return 0;
}

static inline uint32_t hash32(uint64_t k) {  // the counter-based hash of dropout_fwd_kernel
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdULL;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ULL;
  k ^= k >> 33;
  return (uint32_t)k;
}
int mb200_dropout_fwd(const void* x_, void* y_, uint8_t* mask, int64_t n, float p, uint64_t seed, void*) {
  EM_REQUIRE(p >= 0.f && p < 1.f, MB200_E_ARG, "dropout: p out of range");
  const bf16_t* x = (const bf16_t*)x_;
  bf16_t* y = (bf16_t*)y_;
  const float scale = 1.f / (1.f - p);
  for (int64_t i = 0; i < n; ++i) {
    const float u = (float)(hash32(seed * 0x9E3779B97F4A7C15ULL + (uint64_t)i) >> 8) * (1.0f / 16777216.0f);
    mask[i] = u >= p ? 1 : 0;
    y[i] = f2b(mask[i] ? b2f(x[i]) * scale : 0.f);
  }
  return 0;
}
int mb200_dropout_apply(const void* x_, const uint8_t* mask, void* y_, int64_t n, float p, void*) {
  const bf16_t* x = (const bf16_t*)x_;
  bf16_t* y = (bf16_t*)y_;
  const float scale = 1.f / (1.f - p);
  for (int64_t i = 0; i < n; ++i) y[i] = f2b(mask[i] ? b2f(x[i]) * scale : 0.f);
  return 0;
}

int mb200_argmax(const void* x_, int64_t ldx, int32_t rows, int32_t V, int64_t* out, void*) {  // lowest index wins ties
  const bf16_t* x = (const bf16_t*)x_;
  for (int r = 0; r < rows; ++r) {
    float best = -INFINITY;
    int bi = 0;
    for (int j = 0; j < V; ++j) {
      const float v = b2f(x[(long long)r * ldx + j]);
      if (v > best) {
        best = v;
        bi = j;
      }
    }
    out[r] = bi;
  }
  return 0;
}

int mb200_peer_reduce_bcast(void* const* bufs, int32_t world, int64_t offset, int64_t n, int32_t, void*) {
  for (int64_t i = offset; i < offset + n; ++i) {
    float acc = reinterpret_cast<float*>(bufs[0])[i];
    for (int r = 1; r < world; ++r) acc += reinterpret_cast<float*>(bufs[r])[i];
    for (int r = 0; r < world; ++r) reinterpret_cast<float*>(bufs[r])[i] = acc;
  }
  return 0;
}
int mb200_add(const void* a_, const void* b_, const void* c_, void* y_, int64_t n, void*) {
  EM_REQUIRE(n % 8 == 0, MB200_E_SHAPE, "add: n must be a multiple of 8");
  const bf16_t *a = (const bf16_t*)a_, *b = (const bf16_t*)b_, *c = (const bf16_t*)c_;
  bf16_t* y = (bf16_t*)y_;
  for (int64_t i = 0; i < n; ++i) y[i] = f2b(b2f(a[i]) + (b2f(b[i]) + (c ? b2f(c[i]) : 0.f)));
  return 0;
}

int mb200_sumsq(const float* x, int64_t n, float* out, void*) {
  double s = 0.0;
  for (int64_t i = 0; i < n; ++i) s += (double)x[i] * x[i];
  out[0] += (float)s;
  return 0;
}

// torch.optim.AdamW semantics with global-norm clipping and the bf16 refresh   (adamw_kernel)
int mb200_adamw_step(float* w, float* g, float* m1, float* m2, void* shadow_, int64_t n, float lr, float b1, float b2,
                     float eps, float wd, float grad_scale, const float* gnorm_sq, float max_norm, int32_t step,
                     int32_t zero_grad, void*) {
  EM_REQUIRE(step >= 1, MB200_E_ARG, "adamw: step must be >= 1");
  EM_REQUIRE(n % 4 == 0, MB200_E_ALIGN, "adamw: n must be a multiple of 4");
  bf16_t* shadow = (bf16_t*)shadow_;
  const float bc1 = 1.f - powf(b1, (float)step), bc2 = 1.f - powf(b2, (float)step);
  float coef = grad_scale;
  if (gnorm_sq != nullptr && max_norm > 0.f) coef *= fminf(1.f, max_norm / (sqrtf(*gnorm_sq) * grad_scale + 1e-6f));
  const float inv_sqrt_bc2 = 1.f / sqrtf(bc2), stp = lr / bc1, decay = 1.f - lr * wd;
  for (int64_t i = 0; i < n; ++i) {
    const float gi = g[i] * coef;
    float wi = w[i] * decay;
    m1[i] = b1 * m1[i] + (1.f - b1) * gi;
    m2[i] = b2 * m2[i] + (1.f - b2) * gi * gi;
    wi -= stp * (m1[i] / (sqrtf(m2[i]) * inv_sqrt_bc2 + eps));
    w[i] = wi;
    if (shadow) shadow[i] = f2b(wi);
    if (zero_grad) g[i] = 0.f;
  }
  return 0;
}

int mb200_cast_f32_to_bf16(const float* src, void* dst_, int64_t n, void*) {
  bf16_t* dst = (bf16_t*)dst_;
  for (int64_t i = 0; i < n; ++i) dst[i] = f2b(src[i]);
  return 0;
}
int mb200_cast_bf16_to_f32(const void* src_, float* dst, int64_t n, void*) {
  const bf16_t* src = (const bf16_t*)src_;
  for (int64_t i = 0; i < n; ++i) dst[i] = b2f(src[i]);
  return 0;
}

// conv-trunk support   (nchw_to_nhwc8_kernel / im2col3x3_kernel / avgpool_nhwc_kernel)
int mb200_nchw_to_nhwc8(const void* src_, void* dst_, int32_t B, int32_t C, int32_t H, int32_t W, void*) {
  EM_REQUIRE(C >= 1 && C <= 8 && B > 0 && H > 0 && W > 0, MB200_E_SHAPE, "nchw_to_nhwc8: bad shape");
  const bf16_t* src = (const bf16_t*)src_;
  bf16_t* dst = (bf16_t*)dst_;
  const long long hw = (long long)H * W;
  for (long long b = 0; b < B; ++b)
    for (long long px = 0; px < hw; ++px)
      for (int c = 0; c < 8; ++c) dst[(b * hw + px) * 8 + c] = c < C ? src[(b * C + c) * hw + px] : f2b(0.f);
  return 0;
}
int mb200_im2col3x3(const void* src_, void* dst_, int32_t B, int32_t H, int32_t W, int32_t C, int32_t stride, void*) {
  EM_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && (stride == 1 || stride == 2), MB200_E_SHAPE,
             "im2col3x3: bad shape / stride");
  const bf16_t* src = (const bf16_t*)src_;
  bf16_t* dst = (bf16_t*)dst_;
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  for (long long b = 0; b < B; ++b)
    for (int ho = 0; ho < Ho; ++ho)
      for (int wo = 0; wo < Wo; ++wo)
        for (int tap = 0; tap < 9; ++tap) {
          const int hi = ho * stride - 1 + tap / 3, wi = wo * stride - 1 + tap % 3;
          bf16_t* d = dst + ((((b * Ho + ho) * Wo + wo) * 9) + tap) * C;
          if (hi >= 0 && hi < H && wi >= 0 && wi < W) memcpy(d, src + ((b * H + hi) * W + wi) * C, (size_t)C * 2);
          else memset(d, 0, (size_t)C * 2);
        }
  return 0;
}
int mb200_avgpool_nhwc(const void* src_, void* dst_, int32_t B, int32_t H, int32_t W, int32_t C, int32_t k, void*) {
  EM_REQUIRE(B > 0 && k >= 1 && H >= k && W >= k && C > 0 && C % 8 == 0, MB200_E_SHAPE, "avgpool_nhwc: bad shape");
  const bf16_t* src = (const bf16_t*)src_;
  bf16_t* dst = (bf16_t*)dst_;
  const int Ho = H / k, Wo = W / k;
  for (long long b = 0; b < B; ++b)
    for (int ho = 0; ho < Ho; ++ho)
      for (int wo = 0; wo < Wo; ++wo)
        for (int c = 0; c < C; ++c) {
          float acc = 0.f;
          for (int dy = 0; dy < k; ++dy)
            for (int dx = 0; dx < k; ++dx) acc += b2f(src[((b * H + ho * k + dy) * W + wo * k + dx) * C + c]);
          dst[((b * Ho + ho) * Wo + wo) * C + c] = f2b(acc / (float)(k * k));
        }
  return 0;
}

// fused causal self-attention of one tile (csrc/attention.cu: attn_fwd_tile_kernel / attn_bwd_tile_kernel): per
// (batch, head) S = Q K^T / sqrt(hd), causal softmax in fp32, P rounded to bf16 (saved, [B,H,S,ldP]), O = P V; backward
// dP = dO V^T, dV = P^T dO, dS = P * (dP - sum(dP * P)) / sqrt(hd), dQ = dS K, dK = dS^T Q with the inverse rotary
// rotation applied to dQ / dK on the way out (rope_tab [S][rot/2] (cos, sin), may be NULL)
static bool tile_supported(int S, int hd) { return S >= 1 && S <= 128 && hd >= 64 && hd <= 256 && hd % 64 == 0; }

int mb200_attn_fwd_tile(const void* qkv_, int64_t ld, void* P_, int64_t ldP, void* O_, int64_t ldo, int32_t B, int32_t S,
                        int32_t H, int32_t hd, void*) {
  EM_RECORD("attn_fwd_tile",
            "\"qkv\":%llu,\"ld\":%lld,\"P\":%llu,\"ldP\":%lld,\"O\":%llu,\"ldo\":%lld,\"B\":%d,\"S\":%d,\"H\":%d,"
            "\"hd\":%d",
            EM_P(qkv_), (long long)ld, EM_P(P_), (long long)ldP, EM_P(O_), (long long)ldo, B, S, H, hd);
  EM_TRACE(4.0 * B * H * S * (double)S * hd, (double)B * S * H * hd * 8 + (double)B * H * S * ldP * 2, "attn_fwd_tile\tB=%d S=%d H=%d hd=%d", B, S, H, hd);
  EM_REQUIRE(tile_supported(S, hd) && ldP % 8 == 0, MB200_E_SHAPE, "attn_fwd_tile: unsupported S=%d hd=%d", S, hd);
  const bf16_t* qkv = (const bf16_t*)qkv_;
  bf16_t *P = (bf16_t*)P_, *O = (bf16_t*)O_;
  const long long d = (long long)H * hd;
  const float scale = 1.f / sqrtf((float)hd);
  std::vector<float> sc(S);
  for (long long b = 0; b < B; ++b)
    for (int h = 0; h < H; ++h)
      for (int i = 0; i < S; ++i) {
        const bf16_t* q = qkv + (b * S + i) * ld + (long long)h * hd;
        float m = -INFINITY, sum = 0.f;
        for (int j = 0; j <= i; ++j) {
          const bf16_t* k = qkv + (b * S + j) * ld + d + (long long)h * hd;
          float acc = 0.f;
          for (int c = 0; c < hd; ++c) acc += b2f(q[c]) * b2f(k[c]);
          sc[j] = acc * scale;
          m = fmaxf(m, sc[j]);
        }
        for (int j = 0; j <= i; ++j) sum += expf(sc[j] - m);
        bf16_t* pr = P + ((b * H + h) * S + i) * ldP;
        // the kernel writes columns [0, min(ldP, 128)): zeros past the diagonal and past S
        for (int j = 0; j < (ldP < 128 ? ldP : 128); ++j) pr[j] = f2b(j <= i ? expf(sc[j] - m) / sum : 0.f);
        bf16_t* o = O + (b * S + i) * ldo + (long long)h * hd;
        for (int c = 0; c < hd; ++c) {
          float acc = 0.f;
          for (int j = 0; j <= i; ++j) acc += b2f(pr[j]) * b2f(qkv[(b * S + j) * ld + 2 * d + (long long)h * hd + c]);
          o[c] = f2b(acc);
        }
      }
  return 0;
}

// multi-tile forward (csrc/attention.cu: attn_fwd_flash_kernel): any Sq / Sk, causal with key offset Sk - Sq or not;
// fp32 scores, softmax over the whole key row, probabilities rounded to bf16 before P V; optional saved P [B,H,Sq,ldP]
// (columns Sk..ldP zero) and per-row (max, 1 / sum) statistics
int mb200_attn_fwd_flash(const void* q_, int64_t ldq, int64_t q_bsh, int64_t q_bsb, const void* k_, int64_t ldk,
                         int64_t k_bsh, int64_t k_bsb, const void* v_, int64_t ldv, int64_t v_bsh, int64_t v_bsb, void* O_,
                         int64_t ldo, void* P_, int64_t ldP, float* stats, int32_t B, int32_t Sq, int32_t Sk, int32_t H,
                         int32_t hd, int32_t causal, void*) {
  EM_RECORD("attn_fwd_flash",
            "\"q\":%llu,\"ldq\":%lld,\"q_bsh\":%lld,\"q_bsb\":%lld,\"k\":%llu,\"ldk\":%lld,\"k_bsh\":%lld,"
            "\"k_bsb\":%lld,\"v\":%llu,\"ldv\":%lld,\"v_bsh\":%lld,\"v_bsb\":%lld,\"O\":%llu,\"ldo\":%lld,"
            "\"P\":%llu,\"ldP\":%lld,\"stats\":%llu,\"B\":%d,\"Sq\":%d,\"Sk\":%d,\"H\":%d,\"hd\":%d,\"causal\":%d",
            EM_P(q_), (long long)ldq, (long long)q_bsh, (long long)q_bsb, EM_P(k_), (long long)ldk, (long long)k_bsh,
            (long long)k_bsb, EM_P(v_), (long long)ldv, (long long)v_bsh, (long long)v_bsb, EM_P(O_), (long long)ldo,
            EM_P(P_), (long long)ldP, EM_P(stats), B, Sq, Sk, H, hd, causal);
  EM_TRACE(4.0 * B * H * Sq * (double)Sk * hd,  // algorithmic count (QK^T once, full rectangle), like attn_fwd_tile
           (double)B * H * (2.0 * Sq + 2.0 * Sk) * hd * 2 + (P_ ? (double)B * H * Sq * ldP * 2 : 0.0),
           "attn_fwd_flash\tB=%d Sq=%d Sk=%d H=%d hd=%d causal=%d", B, Sq, Sk, H, hd, causal);
  EM_REQUIRE(hd >= 64 && hd <= 256 && hd % 64 == 0 && Sq >= 1 && Sk >= 1, MB200_E_SHAPE,
             "attn_fwd_flash: unsupported Sq=%d Sk=%d hd=%d", Sq, Sk, hd);
  EM_REQUIRE(!causal || Sk >= Sq, MB200_E_SHAPE, "attn_fwd_flash: causal needs Sk >= Sq");
  EM_REQUIRE(P_ == nullptr || (ldP % 8 == 0 && ldP >= Sk), MB200_E_ALIGN, "attn_fwd_flash: ldP must be >= Sk and %%8");
  const bf16_t *Q = (const bf16_t*)q_, *K = (const bf16_t*)k_, *V = (const bf16_t*)v_;
  bf16_t *O = (bf16_t*)O_, *P = (bf16_t*)P_;
  const float scale = 1.f / sqrtf((float)hd);
  const int off = Sk - Sq;
  std::vector<float> sc(Sk);
  std::vector<bf16_t> pr(Sk);
  for (long long b = 0; b < B; ++b)
    for (long long h = 0; h < H; ++h)
      for (int i = 0; i < Sq; ++i) {
        const bf16_t* q = Q + b * q_bsb + h * q_bsh + (long long)i * ldq;
        const int lim = causal ? (i + off + 1 < Sk ? i + off + 1 : Sk) : Sk;
        float m = -INFINITY, sum = 0.f;
        for (int j = 0; j < lim; ++j) {
          const bf16_t* k = K + b * k_bsb + h * k_bsh + (long long)j * ldk;
          float acc = 0.f;
          for (int c = 0; c < hd; ++c) acc += b2f(q[c]) * b2f(k[c]);
          sc[j] = acc * scale;
          m = fmaxf(m, sc[j]);
        }
        for (int j = 0; j < lim; ++j) sum += expf(sc[j] - m);
        const float inv = 1.f / sum;
        for (int j = 0; j < Sk; ++j) pr[j] = f2b(j < lim ? expf(sc[j] - m) * inv : 0.f);
        if (P) {
          bf16_t* prow = P + ((b * H + h) * Sq + i) * ldP;
          for (int j = 0; j < ldP; ++j) prow[j] = j < Sk ? pr[j] : f2b(0.f);
        }
        if (stats) {
          stats[2 * ((b * H + h) * Sq + i)] = m;
          stats[2 * ((b * H + h) * Sq + i) + 1] = inv;
        }
        bf16_t* o = O + (b * Sq + i) * ldo + h * hd;
        for (int c = 0; c < hd; ++c) {
          float acc = 0.f;
          for (int j = 0; j < lim; ++j) acc += b2f(pr[j]) * b2f(V[b * v_bsb + h * v_bsh + (long long)j * ldv + c]);
          o[c] = f2b(acc);
        }
      }
  return 0;
}

int mb200_attn_bwd_tile(const void* qkv_, int64_t ld, const void* dO_, int64_t ld_do, const void* P_, int64_t ldP,
                        void* dqkv_, int64_t ldd, const float* rope_tab, int32_t rot, int32_t B, int32_t S, int32_t H,
                        int32_t hd, void*) {
  EM_RECORD("attn_bwd_tile",
            "\"qkv\":%llu,\"ld\":%lld,\"dO\":%llu,\"ld_do\":%lld,\"P\":%llu,\"ldP\":%lld,\"dqkv\":%llu,"
            "\"ldd\":%lld,\"rope_tab\":%llu,\"rot\":%d,\"B\":%d,\"S\":%d,\"H\":%d,\"hd\":%d",
            EM_P(qkv_), (long long)ld, EM_P(dO_), (long long)ld_do, EM_P(P_), (long long)ldP, EM_P(dqkv_), (long
            long)ldd, EM_P(rope_tab), rot, B, S, H, hd);
  EM_TRACE(10.0 * B * H * S * (double)S * hd, (double)B * S * H * hd * 14 + (double)B * H * S * ldP * 2, "attn_bwd_tile\tB=%d S=%d H=%d hd=%d", B, S, H, hd);
  EM_REQUIRE(tile_supported(S, hd) && ldP % 8 == 0, MB200_E_SHAPE, "attn_bwd_tile: unsupported S=%d hd=%d", S, hd);
  const bf16_t *qkv = (const bf16_t*)qkv_, *dO = (const bf16_t*)dO_, *P = (const bf16_t*)P_;
  bf16_t* dqkv = (bf16_t*)dqkv_;
  const long long d = (long long)H * hd;
  const float scale = 1.f / sqrtf((float)hd);
  std::vector<float> dS((size_t)S * S), dq((size_t)S * hd), dk((size_t)S * hd), dv((size_t)S * hd);
  for (long long b = 0; b < B; ++b)
    for (int h = 0; h < H; ++h) {
      auto Q = [&](int i, int c) { return b2f(qkv[(b * S + i) * ld + (long long)h * hd + c]); };
      auto K = [&](int i, int c) { return b2f(qkv[(b * S + i) * ld + d + (long long)h * hd + c]); };
      auto V = [&](int i, int c) { return b2f(qkv[(b * S + i) * ld + 2 * d + (long long)h * hd + c]); };
      auto G = [&](int i, int c) { return b2f(dO[(b * S + i) * ld_do + (long long)h * hd + c]); };
      auto Pr = [&](int i, int j) { return b2f(P[((b * H + h) * S + i) * ldP + j]); };
      for (int i = 0; i < S; ++i) {
        float dot = 0.f;
        for (int j = 0; j < S; ++j) {
          float dp = 0.f;
          for (int c = 0; c < hd; ++c) dp += G(i, c) * V(j, c);
          dS[(size_t)i * S + j] = dp;
          dot += dp * Pr(i, j);
        }
        for (int j = 0; j < S; ++j)  // bf16 like the kernel's dS operand
          dS[(size_t)i * S + j] = b2f(f2b(Pr(i, j) * (dS[(size_t)i * S + j] - dot) * scale));
      }
      for (int i = 0; i < S; ++i)
        for (int c = 0; c < hd; ++c) {
          float aq = 0.f, ak = 0.f, av = 0.f;
          for (int j = 0; j < S; ++j) {
            aq += dS[(size_t)i * S + j] * K(j, c);
            ak += dS[(size_t)j * S + i] * Q(j, c);
            av += Pr(j, i) * G(j, c);
          }
          dq[(size_t)i * hd + c] = aq;
          dk[(size_t)i * hd + c] = ak;
          dv[(size_t)i * hd + c] = av;
        }
      for (int i = 0; i < S; ++i) {
        if (rope_tab)  // inverse rotation (transpose of rotate_every_two) on the first `rot` dims of dQ, dK
          for (int p = 0; p < rot / 2; ++p) {
            const float cs = rope_tab[((long long)i * (rot / 2) + p) * 2], sn = rope_tab[((long long)i * (rot / 2) + p) * 2 + 1];
            for (std::vector<float>* t : {&dq, &dk}) {
              float& x0 = (*t)[(size_t)i * hd + 2 * p];
              float& x1 = (*t)[(size_t)i * hd + 2 * p + 1];
              const float a = x0, c2 = x1;
              x0 = a * cs + c2 * sn;
              x1 = c2 * cs - a * sn;
            }
          }
        for (int c = 0; c < hd; ++c) {
          dqkv[(b * S + i) * ldd + (long long)h * hd + c] = f2b(dq[(size_t)i * hd + c]);
          dqkv[(b * S + i) * ldd + d + (long long)h * hd + c] = f2b(dk[(size_t)i * hd + c]);
          dqkv[(b * S + i) * ldd + 2 * d + (long long)h * hd + c] = f2b(dv[(size_t)i * hd + c]);
        }
      }
    }
  return 0;
}

// KV cache   (kv_attention.cu: kv_append_kernel / attn_decode_kernel)
int mb200_kv_append(const void* qkv_, int64_t ld, void* kc_, void* vc_, int32_t B, int32_t S, int32_t H, int32_t hd,
                    int32_t Smax, int32_t pos0, void*) {
  EM_RECORD("kv_append",
            "\"qkv\":%llu,\"ld\":%lld,\"kc\":%llu,\"vc\":%llu,\"B\":%d,\"S\":%d,\"H\":%d,\"hd\":%d,\"Smax\":%d,"
            "\"pos0\":%d",
            EM_P(qkv_), (long long)ld, EM_P(kc_), EM_P(vc_), B, S, H, hd, Smax, pos0);
  EM_TRACE(0, (double)B * S * H * hd * 8, "kv_append\tB=%d S=%d H=%d hd=%d", B, S, H, hd);
  EM_REQUIRE(hd % 8 == 0 && B > 0 && S > 0 && pos0 >= 0 && pos0 + S <= Smax, MB200_E_SHAPE, "kv_append: bad shape");
  const bf16_t* qkv = (const bf16_t*)qkv_;
  bf16_t *kc = (bf16_t*)kc_, *vc = (bf16_t*)vc_;
  for (long long b = 0; b < B; ++b)
    for (int s = 0; s < S; ++s)
      for (int h = 0; h < H; ++h) {
        const bf16_t* src = qkv + (b * S + s) * ld + (long long)h * hd;
        const long long dst = ((b * H + h) * Smax + (pos0 + s)) * hd;
        memcpy(kc + dst, src + (long long)H * hd, (size_t)hd * 2);
        memcpy(vc + dst, src + 2LL * H * hd, (size_t)hd * 2);
      }
  return 0;
}

// one decode step: append this step's k, v at `pos`, then softmax(q K^T / sqrt(hd)) V over [0, pos], probabilities
// rounded to bf16 before P*V like the prefill path
int mb200_attn_decode(const void* qkv_, int64_t ld_qkv, void* kc_, void* vc_, void* out_, int64_t ld_out, int32_t B,
                      int32_t H, int32_t hd, int32_t Smax, int32_t pos, void*) {
  EM_RECORD("attn_decode",
            "\"qkv\":%llu,\"ld_qkv\":%lld,\"kc\":%llu,\"vc\":%llu,\"out\":%llu,\"ld_out\":%lld,\"B\":%d,\"H\":%d,"
            "\"hd\":%d,\"Smax\":%d,\"pos\":%d",
            EM_P(qkv_), (long long)ld_qkv, EM_P(kc_), EM_P(vc_), EM_P(out_), (long long)ld_out, B, H, hd, Smax, pos);
  EM_TRACE(4.0 * B * H * (double)(pos + 1) * hd, (double)B * H * (pos + 1) * hd * 4, "attn_decode\tB=%d H=%d hd=%d pos=%d", B, H, hd, pos);
  EM_REQUIRE(hd % 8 == 0 && pos >= 0 && pos < Smax, MB200_E_SHAPE, "attn_decode: bad hd / pos");
  const bf16_t* qkv = (const bf16_t*)qkv_;
  bf16_t *kc = (bf16_t*)kc_, *vc = (bf16_t*)vc_, *out = (bf16_t*)out_;
  const float scale = 1.f / sqrtf((float)hd);
  std::vector<float> sc(pos + 1);
  for (long long b = 0; b < B; ++b)
    for (int h = 0; h < H; ++h) {
      const bf16_t* q = qkv + b * ld_qkv + (long long)h * hd;
      bf16_t* kb = kc + ((b * H + h) * (long long)Smax) * hd;
      bf16_t* vb = vc + ((b * H + h) * (long long)Smax) * hd;
      memcpy(kb + (long long)pos * hd, q + (long long)H * hd, (size_t)hd * 2);
      memcpy(vb + (long long)pos * hd, q + 2LL * H * hd, (size_t)hd * 2);
      float m = -INFINITY, sum = 0.f;
      for (int j = 0; j <= pos; ++j) {
        float acc = 0.f;
        for (int c = 0; c < hd; ++c) acc += b2f(kb[(long long)j * hd + c]) * b2f(q[c]);
        sc[j] = acc * scale;
        m = fmaxf(m, sc[j]);
      }
      for (int j = 0; j <= pos; ++j) {
        sc[j] = expf(sc[j] - m);
        sum += sc[j];
      }
      for (int c = 0; c < hd; ++c) {
        float acc = 0.f;
        for (int j = 0; j <= pos; ++j) acc += b2f(f2b(sc[j] / sum)) * b2f(vb[(long long)j * hd + c]);
        out[b * ld_out + (long long)h * hd + c] = f2b(acc);
      }
    }
  return 0;
}

// conv-trunk training   (col_moments_kernel / channel_affine_kernel / col2im3x3_kernel / avgpool_nhwc_bwd_kernel)
int mb200_col_moments(const void* u_, int64_t ldu, const void* v_, int64_t ldv, const void* mask_, int64_t ldm,
                      int32_t rows, int32_t cols, float* out1, float* out2, void*) {
  EM_REQUIRE(rows > 0 && cols > 0 && cols % 2 == 0 && ldu % 2 == 0 && ldv % 2 == 0 && (!mask_ || ldm % 2 == 0),
             MB200_E_ALIGN, "col_moments: cols and row strides must be even");
  const bf16_t *u = (const bf16_t*)u_, *v = (const bf16_t*)v_, *mask = (const bf16_t*)mask_;
  for (int c = 0; c < cols; ++c) {
    double s1 = 0.0, s2 = 0.0;
    for (int r = 0; r < rows; ++r) {
      float x = b2f(u[(long long)r * ldu + c]);
      if (mask && !(b2f(mask[(long long)r * ldm + c]) > 0.f)) x = 0.f;
      s1 += x;
      s2 += (double)x * b2f(v[(long long)r * ldv + c]);
    }
    out1[c] = (float)s1;
    out2[c] = (float)s2;
  }
  return 0;
}

int mb200_channel_affine(const void* x1_, const float* a1, const void* x2_, const float* a2, const float* c0,
                         const void* mask_, const void* res_, int32_t relu, void* y_, int64_t rows, int32_t C, void*) {
  EM_REQUIRE(rows > 0 && C > 0 && C % 8 == 0 && x1_ && a1 && y_ && (!x2_ || a2), MB200_E_ARG, "channel_affine: bad args");
  EM_REQUIRE(aligned16(x1_) && aligned16(x2_) && aligned16(mask_) && aligned16(res_) && aligned16(y_), MB200_E_ALIGN,
             "channel_affine: alignment");
  const bf16_t *x1 = (const bf16_t*)x1_, *x2 = (const bf16_t*)x2_, *mask = (const bf16_t*)mask_, *res = (const bf16_t*)res_;
  bf16_t* y = (bf16_t*)y_;
  for (int64_t r = 0; r < rows; ++r)
    for (int c = 0; c < C; ++c) {
      const int64_t i = r * C + c;
      float f = b2f(x1[i]);
      if (mask && !(b2f(mask[i]) > 0.f)) f = 0.f;
      f = f * a1[c] + (c0 ? c0[c] : 0.f);
      if (x2) f += b2f(x2[i]) * a2[c];
      if (res) f += b2f(res[i]);
      if (relu) f = fmaxf(f, 0.f);
      y[i] = f2b(f);
    }
  return 0;
}

int mb200_bn_finalize_fwd(const float* s1, const float* s2, const float* gamma, const float* beta, int64_t rows, float eps,
                          float momentum, float* running_mean, float* running_var, float* mean, float* rstd, float* scale,
                          float* shift, int32_t C, void*) {
  EM_REQUIRE(rows > 0 && C > 0 && ((running_mean == nullptr) == (running_var == nullptr)), MB200_E_ARG, "bn_finalize_fwd");
  const double unbias = rows > 1 ? (double)rows / (double)(rows - 1) : 1.0;
  for (int c = 0; c < C; ++c) {
    const double m = (double)s1[c] / rows;
    double var = (double)s2[c] / rows - m * m;
    if (var < 0) var = 0;
    const double rs = 1.0 / sqrt(var + eps);
    mean[c] = (float)m;
    rstd[c] = (float)rs;
    scale[c] = (float)(gamma[c] * rs);
    shift[c] = (float)(beta[c] - m * gamma[c] * rs);
    if (running_mean) {
      running_mean[c] = (float)((1.0 - momentum) * running_mean[c] + momentum * m);
      running_var[c] = (float)((1.0 - momentum) * running_var[c] + momentum * var * unbias);
    }
  }
  return 0;
}

int mb200_bn_bwd_coeffs(const float* s1, const float* t, const float* mean, const float* rstd, const float* gamma,
                        int64_t rows, float* dgamma, float* dbeta, int32_t accumulate, float* A, float* Bc, float* Cc,
                        int32_t C, void*) {
  EM_REQUIRE(rows > 0 && C > 0, MB200_E_ARG, "bn_bwd_coeffs");
  for (int c = 0; c < C; ++c) {
    const double s2 = (double)rstd[c] * ((double)t[c] - (double)mean[c] * s1[c]);
    dgamma[c] = (float)((accumulate ? dgamma[c] : 0.f) + s2);
    dbeta[c] = (accumulate ? dbeta[c] : 0.f) + s1[c];
    const double a = (double)gamma[c] * rstd[c];
    const double k2 = a * rstd[c] * s2 / rows;
    A[c] = (float)a;
    Bc[c] = (float)(-k2);
    Cc[c] = (float)(k2 * mean[c] - a * s1[c] / rows);
  }
  return 0;
}

int mb200_col2im3x3(const void* dcols_, void* dx_, int32_t B, int32_t H, int32_t W, int32_t C, int32_t stride, void*) {
  EM_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && (stride == 1 || stride == 2), MB200_E_SHAPE,
             "col2im3x3: bad shape / stride");
  const bf16_t* dcols = (const bf16_t*)dcols_;
  bf16_t* dx = (bf16_t*)dx_;
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  std::vector<float> acc((size_t)B * H * W * C, 0.f);
  for (long long b = 0; b < B; ++b)  // scatter form: the adjoint of the im2col loop above, tap by tap
    for (int ho = 0; ho < Ho; ++ho)
      for (int wo = 0; wo < Wo; ++wo)
        for (int tap = 0; tap < 9; ++tap) {
          const int hi = ho * stride - 1 + tap / 3, wi = wo * stride - 1 + tap % 3;
          if (hi < 0 || hi >= H || wi < 0 || wi >= W) continue;
          const bf16_t* s = dcols + ((((b * Ho + ho) * Wo + wo) * 9) + tap) * C;
          float* d = acc.data() + ((b * H + hi) * W + wi) * C;
          for (int c = 0; c < C; ++c) d[c] += b2f(s[c]);
        }
  for (size_t i = 0; i < acc.size(); ++i) dx[i] = f2b(acc[i]);
  return 0;
}

int mb200_avgpool_nhwc_bwd(const void* dy_, void* dx_, int32_t B, int32_t H, int32_t W, int32_t C, int32_t k, void*) {
  EM_REQUIRE(B > 0 && k >= 1 && H >= k && W >= k && C > 0 && C % 8 == 0, MB200_E_SHAPE, "avgpool_nhwc_bwd: bad shape");
  const bf16_t* dy = (const bf16_t*)dy_;
  bf16_t* dx = (bf16_t*)dx_;
  const int Ho = H / k, Wo = W / k;
  for (long long b = 0; b < B; ++b)
    for (int h = 0; h < H; ++h)
      for (int w = 0; w < W; ++w)
        for (int c = 0; c < C; ++c) {
          float f = 0.f;
          if (h / k < Ho && w / k < Wo) f = b2f(dy[((b * Ho + h / k) * Wo + w / k) * C + c]) / (float)(k * k);
          dx[((b * H + h) * W + w) * C + c] = f2b(f);
        }
  return 0;
}

// images [B,3,R,R] -> patches [B*g*g][ldp], column order (c, py, px)   (patchify_kernel)
int mb200_patchify(const void* img_, void* patches_, int64_t ldp, int32_t B, int32_t R, int32_t P, void*) {
  EM_RECORD("patchify",
            "\"img\":%llu,\"patches\":%llu,\"ldp\":%lld,\"B\":%d,\"R\":%d,\"P\":%d",
            EM_P(img_), EM_P(patches_), (long long)ldp, B, R, P);
  EM_TRACE(0, (double)B * 3 * R * R * 4, "patchify\tB=%d R=%d P=%d", B, R, P);
  EM_REQUIRE(R % P == 0 && ldp >= 3 * P * P, MB200_E_SHAPE, "patchify: bad geometry");
  const bf16_t* img = (const bf16_t*)img_;
  bf16_t* patches = (bf16_t*)patches_;
  const int g = R / P;
  for (int b = 0; b < B; ++b)
    for (int gy = 0; gy < g; ++gy)
      for (int gx = 0; gx < g; ++gx)
        for (int c = 0; c < 3; ++c)
          for (int py = 0; py < P; ++py)
            for (int px = 0; px < P; ++px)
              patches[(((long long)b * g + gy) * g + gx) * ldp + (c * P + py) * P + px] =
                  img[(((long long)b * 3 + c) * R + (gy * P + py)) * R + (gx * P + px)];
  return 0;
}

// x[b,0] = cls + pos[0]; x[b,1+p] = pe[b,p] + pos[1+p]   (vit_assemble_kernel)
int mb200_vit_assemble(void* x_, const void* pe_, const void* cls_, const void* pos_, int32_t B, int32_t T, int32_t w,
                       void*) {
  EM_RECORD("vit_assemble",
            "\"x\":%llu,\"pe\":%llu,\"cls\":%llu,\"pos\":%llu,\"B\":%d,\"T\":%d,\"w\":%d",
            EM_P(x_), EM_P(pe_), EM_P(cls_), EM_P(pos_), B, T, w);
  EM_TRACE((double)B * T * w, (double)B * T * w * 4, "vit_assemble\tB=%d T=%d w=%d", B, T, w);
  bf16_t* x = (bf16_t*)x_;
  const bf16_t *pe = (const bf16_t*)pe_, *cls = (const bf16_t*)cls_, *pos = (const bf16_t*)pos_;
  for (long long b = 0; b < B; ++b)
    for (int t = 0; t < T; ++t)
      for (int c = 0; c < w; ++c) {
        const float base = t == 0 ? b2f(cls[c]) : b2f(pe[(b * (T - 1) + (t - 1)) * w + c]);
        x[(b * T + t) * w + c] = f2b(base + b2f(pos[(long long)t * w + c]));
      }
  return 0;
}

// device-resident decode loop: on the CPU the "device" position is ordinary memory
int mb200_rope_table_dev(float* tab, int32_t S, int32_t rot, const int32_t* pos0_dev, void* st) {
  EM_REQUIRE(pos0_dev != nullptr, MB200_E_ARG, "rope_table_dev: null position");
  return mb200_rope_table(tab, S, rot, *pos0_dev, st);
}
int mb200_attn_decode_dev(const void* qkv, int64_t ld_qkv, void* kc, void* vc, void* out, int64_t ld_out, int32_t B,
                          int32_t H, int32_t hd, int32_t Smax, const int32_t* pos_dev, void* st) {
  EM_REQUIRE(pos_dev != nullptr, MB200_E_ARG, "attn_decode_dev: null position");
  return mb200_attn_decode(qkv, ld_qkv, kc, vc, out, ld_out, B, H, hd, Smax, *pos_dev, st);
}
int mb200_decode_embed(const int64_t* tokens, int64_t ld_tok, const int32_t* pos_dev, const void* wte_, void* x_, int32_t B,
                       int32_t d, int32_t vocab, void*) {
  EM_REQUIRE(d % 8 == 0 && B > 0 && tokens && pos_dev, MB200_E_SHAPE, "decode_embed: bad B / d");
  const bf16_t* wte = (const bf16_t*)wte_;
  bf16_t* x = (bf16_t*)x_;
  for (long long b = 0; b < B; ++b) {
    long long tok = tokens[b * ld_tok + *pos_dev];
    if (tok < 0 || tok >= vocab) tok = 0;
    memcpy(x + b * d, wte + tok * (long long)d, (size_t)d * 2);
  }
  return 0;
}
int mb200_decode_advance(const int64_t* next, int64_t* tokens, int64_t ld_tok, int32_t* pos_dev, int64_t eos,
                         uint8_t* flags, int32_t s0, int32_t n_flags, int32_t B, void*) {
  EM_REQUIRE(B > 0 && next && tokens && pos_dev, MB200_E_ARG, "decode_advance: null argument");
  const int p = *pos_dev;
  int all = 1;
  for (long long b = 0; b < B; ++b) {
    if (p + 1 < ld_tok) tokens[b * ld_tok + p + 1] = next[b];
    all &= next[b] == eos;
  }
  const int i = p + 1 - s0;
  if (flags && i >= 0 && i < n_flags) flags[i] = (uint8_t)all;
  *pos_dev = p + 1;
  return 0;
}

}  // extern "C"
