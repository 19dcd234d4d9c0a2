// magma_b200 — the small runtime interface that HOST-ONLY schedule files (gptj_sched.cu, vit_sched.cu) are written against,
// and the host-side helpers they share: workspace carving, the GEMM call and its split-K scratch, the switch of the fused
// multi-tile attention and the materialised attention (batched GEMMs + softmax kernels) for head dims it does not take.
//
// A schedule file contains no kernels and no CUDA runtime calls: it carves a workspace and issues the primitive
// operators of the C ABI (include/magma_b200.h: mb200_gemm, mb200_layernorm_*, mb200_softmax_*, ...) plus the three
// runtime helpers below. In the product the runtime helpers are CUDA (common.cu). tests/ also compile the same schedule
// file as plain C++ against oracle/cabi_emul.cpp, a CPU emulation of those primitives, to dry-run the schedule (pointer
// arithmetic, leading dimensions, operand majors, accumulate flags) against the oracle without a GPU. That build is test
// infrastructure only; nothing in magma_b200/ loads it.
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/magma_b200.h"

namespace mb200 {
void set_error(const char* fmt, ...);
int rt_check_arch();                                                   // 0 on sm_90, else MB200_E_ARCH
int rt_copy(void* dst, const void* src, size_t bytes, void* stream);   // device-to-device, stream-ordered
int rt_zero(void* dst, size_t bytes, void* stream);                    // stream-ordered memset(0)
}  // namespace mb200

#define MBS_REQUIRE(cond, code, ...)  \
  do {                                \
    if (!(cond)) {                    \
      mb200::set_error(__VA_ARGS__);  \
      return (code);                  \
    }                                 \
  } while (0)

#define MBS_TRY(expr)     \
  do {                    \
    int _rc = (expr);     \
    if (_rc) return _rc;  \
  } while (0)

namespace mb200 {

typedef uint16_t bf16s;  // bf16 storage; the schedules only do pointer arithmetic on it

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

struct Carver {
  uint8_t* base;
  size_t off;
  explicit Carver(void* b) : base(reinterpret_cast<uint8_t*>(b)), off(0) {}
  template <typename T>
  T* take(size_t n) {
    off = align_up(off, 256);
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += n * sizeof(T);
    return p;
  }
};

struct Mat {
  const void* p;
  long long ld, bs0, bs1;
  int mn, frozen;
};
inline Mat mat(const void* p, long long ld, int mn = 0, long long bs0 = 0, long long bs1 = 0) {
  return Mat{p, ld, bs0, bs1, mn, 0};
}
// a frozen weight matrix (never written by a kernel of the stream): the GEMM may fetch its first tiles ahead of the
// programmatic dependency on the previous kernel (mb200_operand.static_data)
inline Mat wmat(const void* p, long long ld, int mn = 0) { return Mat{p, ld, 0, 0, mn, 1}; }
struct Epi {
  float alpha = 1.f;
  const void* bias = nullptr;
  int act = 0;
  void* aux_out = nullptr;
  const void* aux_in = nullptr;
  int dact = 0;
  const void* res1 = nullptr;
  const void* res2 = nullptr;
  long long ld_res = 0;
  int accumulate = 0;
  const float* rope_tab = nullptr;
  int rope_mode = 0, rope_S = 0, rope_hd = 0, rope_rot = 0, rope_ncols = 0;
};

// scratch a pass lends to the GEMM core (mb200_gemm_args.splitk_ws): the fp32 per-split partial slices of the GEMMs
// gemm.cu splits along K (small-M decode GEMMs streaming their weights, the few-tile, long-K wgrads of training); the
// split count shrinks to what fits
const size_t kGemmScratchBytes = (size_t)128 << 20;

// split-K scratch of the pass being issued
inline thread_local void* t_splitk_ws = nullptr;
inline thread_local long long t_splitk_bytes = 0;

struct ScratchScope {  // the scratch is only valid while the pass that owns the workspace is being issued
  ScratchScope(void* w, size_t b) { t_splitk_ws = w; t_splitk_bytes = (long long)b; }
  ~ScratchScope() { t_splitk_ws = nullptr; t_splitk_bytes = 0; }
};

inline int gemm(void* st, int M, int N, int K, Mat A, Mat B, void* C, long long ldc, int c_f32, const Epi& e = Epi(),
                int nb0 = 1, int nb1 = 1, long long c_bs0 = 0, long long c_bs1 = 0) {
  mb200_gemm_args g;
  memset(&g, 0, sizeof(g));
  g.M = M;
  g.N = N;
  g.K = K;
  g.nb0 = nb0;
  g.nb1 = nb1;
  g.c_dtype = c_f32 ? MB200_F32 : MB200_BF16;
  g.A.ptr = A.p;
  g.A.ld = A.ld;
  g.A.bs0 = A.bs0;
  g.A.bs1 = A.bs1;
  g.A.mn_major = A.mn;
  g.B.ptr = B.p;
  g.B.ld = B.ld;
  g.B.bs0 = B.bs0;
  g.B.bs1 = B.bs1;
  g.B.mn_major = B.mn;
  g.B.static_data = B.frozen;
  g.C = C;
  g.ldc = ldc;
  g.c_bs0 = c_bs0;
  g.c_bs1 = c_bs1;
  g.alpha = e.alpha;
  g.act = e.act;
  g.dact = e.dact;
  g.accumulate = e.accumulate;
  g.bias = e.bias;
  g.aux_out = e.aux_out;
  g.aux_in = e.aux_in;
  g.res1 = e.res1;
  g.res2 = e.res2;
  g.ld_res = e.ld_res;
  g.rope_tab = e.rope_tab;
  g.rope_mode = e.rope_mode;
  g.rope_S = e.rope_S;
  g.rope_hd = e.rope_hd;
  g.rope_rot = e.rope_rot;
  g.rope_ncols = e.rope_ncols;
  g.splitk_ws = t_splitk_ws;
  g.splitk_ws_bytes = t_splitk_bytes;
  return mb200_gemm(&g, st);
}

// wgrad of a linear y = x W^T: dW[out, in] (+)= dy^T x, both operands read MN-major from their [rows, features] storage
inline int wgrad(void* st, int out, int in, int rows, const bf16s* dy, long long lddy, const bf16s* x, long long ldx,
                 float* dW, long long ldw, int accumulate) {
  Epi e;
  e.accumulate = accumulate;
  return gemm(st, out, in, rows, mat(dy, lddy, 1), mat(x, ldx, 1), dW, ldw, 1, e);
}

// the fused multi-tile attention forward (csrc/attention.cu) takes head dims in {64, 128, 192, 256} at any sequence
// length; MB200_ATTN_FLASH=0 forces the materialised path below
inline bool flash_ok(int hd) {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("MB200_ATTN_FLASH");
    on = e ? atoi(e) : 1;
  }
  return on != 0 && hd >= 64 && hd <= 256 && hd % 64 == 0;
}

// Materialised attention forward over B x H heads: scores = Q K^T (fp32), P = softmax(scores / sqrt(hd) + mask),
// O = P V. Q, K, V carry their per-head (bs0) and per-batch (bs1) strides; scores and P are [B,H,Sq,ldP]; O is
// [B,Sq,H*hd] with row stride ldo. causal masks key j > i + koff for query i (koff = Sk - Sq over a KV cache).
// ldPo (0: ldP) is P's own row stride, when P is a caller's buffer rather than the scores' twin.
inline int attn_fwd_gemm(void* st, Mat Q, Mat K, Mat V, int Sq, int Sk, int H, int B, int hd, float* scores, bf16s* P,
                         int ldP, bf16s* O, long long ldo, int causal, int koff, int ldPo = 0) {
  const long long pb0 = (long long)Sq * ldP, pb1 = (long long)H * Sq * ldP;
  if (ldPo == 0) ldPo = ldP;
  const long long ob0 = (long long)Sq * ldPo, ob1 = (long long)H * Sq * ldPo;
  MBS_TRY(gemm(st, Sq, Sk, hd, Q, K, scores, ldP, 1, Epi(), H, B, pb0, pb1));
  MBS_TRY(mb200_softmax_fwd(scores, ldP, pb0, P, ldPo, ob0, B * H, Sq, Sk, 1.0f / sqrtf((float)hd), causal, koff, st));
  return gemm(st, Sq, hd, Sk, mat(P, ldPo, 0, ob0, ob1), V, O, ldo, 0, Epi(), H, B, hd, (long long)Sq * ldo);
}

// Materialised attention backward on the fused qkv layout: qkv and dqkv are [B,S,3*H*hd] (q | k | v), dO is [B,S,H*hd],
// P the saved [B,H,S,ldP] probabilities. dP (fp32) and dS are [B,H,S,ldP] scratch. eqk is the epilogue of dQ and dK
// (e.g. the inverse rotary embedding of q and k). dPe (optional, bf16 [B,H,S,ldP]): a gradient on P from outside the
// block, added to dP in its GEMM's epilogue.
inline int attn_bwd_gemm(void* st, const bf16s* qkv, const bf16s* P, const bf16s* dO, bf16s* dqkv, float* dP, bf16s* dS,
                         int ldP, int S, int H, int B, int hd, const Epi& eqk, const bf16s* dPe = nullptr) {
  const int d = H * hd;
  const long long qb0 = hd, qb1 = (long long)S * 3 * d;
  const long long pb0 = (long long)S * ldP, pb1 = (long long)H * S * ldP;
  // dP = dO V^T (+ dPe) ; dV = P^T dO
  Epi edp;
  edp.res1 = dPe;
  edp.ld_res = dPe ? ldP : 0;
  MBS_TRY(gemm(st, S, S, hd, mat(dO, d, 0, hd, (long long)S * d), mat(qkv + 2 * d, 3 * d, 0, qb0, qb1), dP, ldP, 1, edp,
               H, B, pb0, pb1));
  MBS_TRY(gemm(st, S, hd, S, mat(P, ldP, 1, pb0, pb1), mat(dO, d, 1, hd, (long long)S * d), dqkv + 2 * d, 3 * d, 0, Epi(),
               H, B, qb0, qb1));
  // dS = P * (dP - rowsum(dP * P)) / sqrt(hd)
  MBS_TRY(mb200_softmax_bwd(dP, ldP, pb0, P, ldP, pb0, dS, ldP, pb0, B * H, S, S, 1.0f / sqrtf((float)hd), st));
  // dQ = dS K ; dK = dS^T Q
  MBS_TRY(gemm(st, S, hd, S, mat(dS, ldP, 0, pb0, pb1), mat(qkv + d, 3 * d, 1, qb0, qb1), dqkv, 3 * d, 0, eqk, H, B, qb0,
               qb1));
  return gemm(st, S, hd, S, mat(dS, ldP, 1, pb0, pb1), mat(qkv, 3 * d, 1, qb0, qb1), dqkv + d, 3 * d, 0, eqk, H, B, qb0,
              qb1);
}

}  // namespace mb200
