// magma_b200 — CLIP-ViT schedules, host-only: the inference forward (frozen image encoder: the measured path,
// mb200_vit_forward) and the training schedule (forward with saved activations + backward).
//
// `freeze_img_encoder: false` (MAGMA_v1.yml:5; magma/magma.py:98-100 only freezes the encoder when asked to) puts the
// image encoder on the training path: loss.backward() (magma/train_loop.py:18) then runs through
// ImagePrefix.proj into the encoder, and the optimizer gives the encoder its own learning rate
// (magma/utils.py:173-177). The training schedule is the ViT half of that: the inference forward below with every
// layer's activations kept, and the matching backward — dgrad and wgrad of every linear on the GEMM core with
// MN-major operands (no transposed copies), attention backward as strided batched GEMMs on the fused qkv buffer,
// LayerNorm / softmax / QuickGELU backward and the bias / LN-parameter / positional reductions as HBM-bound kernels.
//
// Reference arithmetic (absent openai/CLIP; stand-in hf:clip/modeling_clip.py:138-219,282-386,647-694,1015-1069 —
// the oracle); the backward is the autograd of that forward and is checked against torch autograd of the oracle.
//
// This file contains no kernels and no CUDA calls (see sched_rt.h): tests/ dry-run it on the CPU against
// oracle/cabi_emul.cpp. Attention (T = 257 for ViT-L/14, head_dim 64, no mask) runs in the fused multi-tile kernel
// (mb200_attn_fwd_flash) whenever head_dim is a multiple of 64 — the training forward asks it for the probabilities
// the materialised backward consumes — and as batched GEMMs + softmax otherwise.
#include "sched_rt.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

namespace mb200 {
namespace {

typedef uint16_t bf16s;  // bf16 storage; this file only does pointer arithmetic on it

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
  const void* bias = nullptr;
  int act = 0;
  void* aux_out = nullptr;
  const void* res1 = nullptr;
  long long ld_res = 0;
  int accumulate = 0;
};

// scratch lent to the GEMM core while a pass is being issued (mb200_gemm_args.splitk_ws: stream-K partial tiles of the
// last wave — the M = 2056 GEMMs of ViT-L/14 are 1.5 - 2.9 waves of 256 x 256 tiles — and split-K slices)
const size_t kGemmScratchBytes = (size_t)128 << 20;
thread_local void* t_gemm_ws = nullptr;
thread_local long long t_gemm_ws_bytes = 0;
struct ScratchScope {
  ScratchScope(void* w, size_t b) { t_gemm_ws = w; t_gemm_ws_bytes = (long long)b; }
  ~ScratchScope() { t_gemm_ws = nullptr; t_gemm_ws_bytes = 0; }
};

int gemm(void* st, int M, int N, int K, Mat A, Mat B, void* C, long long ldc, int c_f32, const Epi& e = Epi(),
         int nb0 = 1, int nb1 = 1, long long c_bs0 = 0, long long c_bs1 = 0) {
  mb200_gemm_args g;
  memset(&g, 0, sizeof(g));
  g.splitk_ws = t_gemm_ws;
  g.splitk_ws_bytes = t_gemm_ws_bytes;
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
  g.alpha = 1.f;
  g.act = e.act;
  g.accumulate = e.accumulate;
  g.bias = e.bias;
  g.aux_out = e.aux_out;
  g.res1 = e.res1;
  g.ld_res = e.ld_res;
  return mb200_gemm(&g, st);
}

// wgrad of a linear y = x W^T: dW[out, in] (+)= dy^T x, both operands read MN-major from their [rows, features] storage
int wgrad(void* st, int out, int in, int rows, const bf16s* dy, long long lddy, const bf16s* x, long long ldx, float* dW,
          long long ldw, int accumulate) {
  Epi e;
  e.accumulate = accumulate;
  return gemm(st, out, in, rows, mat(dy, lddy, 1), mat(x, ldx, 1), dW, ldw, 1, e);
}

struct LayerActs {
  bf16s* x_in;    // [M,w] residual stream entering the block
  bf16s* h1;      // [M,w] ln_1 output
  bf16s* qkv;     // [M,3w]
  bf16s* P;       // [B,H,T,ldS] attention probabilities
  bf16s* attn_o;  // [M,w] merged heads, before out_proj
  bf16s* x_mid;   // [M,w] after the attention residual
  bf16s* h2;      // [M,w] ln_2 output
  bf16s* pre;     // [M,mlp] c_fc pre-activation
  bf16s* hact;    // [M,mlp] QuickGELU output
  float *mean1, *rstd1, *mean2, *rstd2;
};

struct Plan {
  int T, M, ldS, ldpatch, g, Kp;
  bf16s *patches, *pe, *xa, *x_out, *pooled;
  float *mean0, *rstd0, *meanp, *rstdp;
  LayerActs acts[64];
  float* scores;  // [B,H,T,ldS] fp32: scores in forward, dP in backward
  // backward temporaries
  bf16s *gA, *gB, *gmid, *dh, *dhact, *dattn_o, *dqkv, *dS, *dpooled, *dpe;
  void* gemm_ws;
  size_t bytes;
};

int make_plan(Plan& P, const mb200_vit_model* m, int B, void* ws) {
  MBS_REQUIRE(m && m->layers && m->n_layer > 0 && m->n_layer <= 64, MB200_E_SHAPE, "vit_train: n_layer out of range");
  MBS_REQUIRE(B > 0 && m->patch > 0 && m->image % m->patch == 0 && m->n_head > 0 && m->width % m->n_head == 0,
              MB200_E_SHAPE, "vit_train: bad geometry");
  MBS_REQUIRE(m->width % 8 == 0 && m->mlp % 8 == 0 && m->out_dim % 8 == 0 && (m->width / m->n_head) % 8 == 0,
              MB200_E_ALIGN, "vit_train: width, mlp, out_dim and head_dim must be multiples of 8");
  Carver c(ws);
  P.g = m->image / m->patch;
  P.T = P.g * P.g + 1;
  P.M = B * P.T;
  P.ldS = (int)align_up(P.T, 8);
  P.Kp = 3 * m->patch * m->patch;
  MBS_REQUIRE(P.Kp % 4 == 0, MB200_E_ALIGN, "vit_train: 3*patch^2 = %d must be a multiple of 4", P.Kp);
  P.ldpatch = (int)align_up(P.Kp, 8);
  const size_t M = P.M, w = m->width, mlp = m->mlp, np = (size_t)B * P.g * P.g;
  const size_t nP = (size_t)B * m->n_head * P.T * P.ldS;
  P.patches = c.take<bf16s>(np * P.ldpatch);
  P.pe = c.take<bf16s>(np * w);
  P.xa = c.take<bf16s>(M * w);
  P.mean0 = c.take<float>(M);
  P.rstd0 = c.take<float>(M);
  for (int l = 0; l < m->n_layer; ++l) {
    LayerActs& a = P.acts[l];
    a.x_in = c.take<bf16s>(M * w);
    a.h1 = c.take<bf16s>(M * w);
    a.qkv = c.take<bf16s>(M * 3 * w);
    a.P = c.take<bf16s>(nP);
    a.attn_o = c.take<bf16s>(M * w);
    a.x_mid = c.take<bf16s>(M * w);
    a.h2 = c.take<bf16s>(M * w);
    a.pre = c.take<bf16s>(M * mlp);
    a.hact = c.take<bf16s>(M * mlp);
    a.mean1 = c.take<float>(M);
    a.rstd1 = c.take<float>(M);
    a.mean2 = c.take<float>(M);
    a.rstd2 = c.take<float>(M);
  }
  P.x_out = c.take<bf16s>(M * w);
  P.pooled = c.take<bf16s>((size_t)B * w);
  P.meanp = c.take<float>(B);
  P.rstdp = c.take<float>(B);
  P.scores = c.take<float>(nP);
  P.gA = c.take<bf16s>(M * w);
  P.gB = c.take<bf16s>(M * w);
  P.gmid = c.take<bf16s>(M * w);
  P.dh = c.take<bf16s>(M * w);
  P.dhact = c.take<bf16s>(M * mlp);
  P.dattn_o = c.take<bf16s>(M * w);
  P.dqkv = c.take<bf16s>(M * 3 * w);
  P.dS = c.take<bf16s>(nP);
  P.dpooled = c.take<bf16s>((size_t)B * w);
  P.dpe = c.take<bf16s>(np * w);
  P.gemm_ws = c.take<uint8_t>(kGemmScratchBytes);
  P.bytes = align_up(c.off, 256);
  return 0;
}

const float kEps = 1e-5f;  // CLIP LayerNorm eps

// head dims the fused multi-tile attention kernel takes (csrc/attention.cu); MB200_ATTN_FLASH=0 forces the GEMM path
inline bool flash_ok(int hd) {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("MB200_ATTN_FLASH");
    on = e ? atoi(e) : 1;
  }
  return on != 0 && hd >= 64 && hd <= 256 && hd % 64 == 0;
}

// ---------------------------------------------------------------------------------------------
// inference forward (the image encoder is frozen on the measured path, magma/magma.py:98-100): one set of activation
// buffers reused by every layer. Arithmetic: hf:clip/modeling_clip.py:138-219 (patch + class + position embeddings),
// :647-694 (pre / post LayerNorm, class-token pooling), :282-386 (blocks), :1015-1069 (projection).
// ---------------------------------------------------------------------------------------------
struct InferPlan {
  int T, M, ldS, ldpatch;
  bf16s *x, *h, *qkv, *P, *attn_o, *hact, *patches, *pooled;
  float* scores;
  void* gemm_ws;
  size_t bytes;
};

int make_infer_plan(InferPlan& P, const mb200_vit_model* m, int B, void* ws) {
  MBS_REQUIRE(m && m->layers && m->n_layer > 0 && B > 0 && m->patch > 0 && m->image % m->patch == 0 && m->n_head > 0 &&
                  m->width % m->n_head == 0,
              MB200_E_SHAPE, "vit: bad geometry");
  const int g = m->image / m->patch;
  Carver c(ws);
  P.T = g * g + 1;
  P.M = B * P.T;
  P.ldS = (int)align_up(P.T, 8);
  P.ldpatch = (int)align_up(3 * m->patch * m->patch, 8);
  const size_t M = P.M, w = m->width;
  const bool fl = flash_ok(m->width / m->n_head);
  const size_t nP = fl ? 8 : (size_t)B * m->n_head * P.T * P.ldS;  // no score / probability buffers with fused attention
  P.x = c.take<bf16s>(M * w);
  P.h = c.take<bf16s>(M * w);
  P.qkv = c.take<bf16s>(M * 3 * w);
  P.scores = c.take<float>(nP);
  P.P = c.take<bf16s>(nP);
  P.attn_o = c.take<bf16s>(M * w);
  P.hact = c.take<bf16s>(M * (size_t)m->mlp);
  P.patches = c.take<bf16s>((size_t)B * g * g * P.ldpatch);
  P.pooled = c.take<bf16s>((size_t)B * w);
  P.gemm_ws = c.take<uint8_t>(kGemmScratchBytes);
  P.bytes = align_up(c.off, 256);
  return 0;
}

int forward_infer(const mb200_vit_model* m, const bf16s* images, bf16s* feats, int B, void* ws, size_t ws_bytes, void* st) {
  InferPlan P;
  MBS_TRY(make_infer_plan(P, m, B, ws));
  MBS_REQUIRE(ws != nullptr && ws_bytes >= P.bytes, MB200_E_ARG, "vit_forward: workspace too small (%zu < %zu)", ws_bytes,
              P.bytes);
  const int w = m->width, H = m->n_head, hd = w / H, T = P.T, M = P.M, g = m->image / m->patch;
  const int Kp = 3 * m->patch * m->patch;
  const float scale = 1.0f / sqrtf((float)hd);
  ScratchScope scratch(P.gemm_ws, kGemmScratchBytes);
  // conv1 as im2col + GEMM (patch embeddings staged in h), then [cls; patches] + positional embedding
  MBS_TRY(rt_zero(P.patches, (size_t)B * g * g * P.ldpatch * sizeof(bf16s), st));
  MBS_TRY(mb200_patchify(images, P.patches, P.ldpatch, B, m->image, m->patch, st));
  MBS_TRY(gemm(st, B * g * g, w, Kp, mat(P.patches, P.ldpatch), wmat(m->w_conv, m->ld_conv), P.h, w, 0));
  MBS_TRY(mb200_vit_assemble(P.x, P.h, m->cls, m->pos, B, T, w, st));
  // ln_pre (in place: each row is cached in registers before it is rewritten)
  MBS_TRY(mb200_layernorm_fwd(P.x, w, m->ln_pre_g, m->ln_pre_b, P.x, w, nullptr, nullptr, M, w, kEps, st));
  const long long qb0 = hd, qb1 = (long long)T * 3 * w;
  const long long pb0 = (long long)T * P.ldS, pb1 = (long long)H * T * P.ldS;
  for (int l = 0; l < m->n_layer; ++l) {
    const mb200_vit_layer& L = m->layers[l];
    MBS_TRY(mb200_layernorm_fwd(P.x, w, L.ln1_g, L.ln1_b, P.h, w, nullptr, nullptr, M, w, kEps, st));
    {
      Epi e;
      e.bias = L.b_qkv;
      MBS_TRY(gemm(st, M, 3 * w, w, mat(P.h, w), wmat(L.w_qkv, w), P.qkv, 3 * w, 0, e));
    }
    if (flash_ok(hd)) {
      MBS_TRY(mb200_attn_fwd_flash(P.qkv, 3 * w, qb0, qb1, P.qkv + w, 3 * w, qb0, qb1, P.qkv + 2 * w, 3 * w, qb0, qb1,
                                   P.attn_o, w, nullptr, 0, nullptr, B, T, T, H, hd, 0, st));
    } else {
      MBS_TRY(gemm(st, T, T, hd, mat(P.qkv, 3 * w, 0, qb0, qb1), mat(P.qkv + w, 3 * w, 0, qb0, qb1), P.scores, P.ldS, 1,
                   Epi(), H, B, pb0, pb1));
      MBS_TRY(mb200_softmax_fwd(P.scores, P.ldS, pb0, P.P, P.ldS, pb0, B * H, T, T, scale, 0, 0, st));
      MBS_TRY(gemm(st, T, hd, T, mat(P.P, P.ldS, 0, pb0, pb1), mat(P.qkv + 2 * w, 3 * w, 1, qb0, qb1), P.attn_o, w, 0,
                   Epi(), H, B, hd, (long long)T * w));
    }
    {
      Epi e;
      e.bias = L.b_out;
      e.res1 = P.x;
      e.ld_res = w;
      MBS_TRY(gemm(st, M, w, w, mat(P.attn_o, w), wmat(L.w_out, w), P.x, w, 0, e));  // x += out_proj(attn)
    }
    MBS_TRY(mb200_layernorm_fwd(P.x, w, L.ln2_g, L.ln2_b, P.h, w, nullptr, nullptr, M, w, kEps, st));
    {
      Epi e;
      e.bias = L.b_fc;
      e.act = MB200_ACT_QUICK_GELU;
      MBS_TRY(gemm(st, M, m->mlp, w, mat(P.h, w), wmat(L.w_fc, w), P.hact, m->mlp, 0, e));
      Epi e2;
      e2.bias = L.b_proj;
      e2.res1 = P.x;
      e2.ld_res = w;
      MBS_TRY(gemm(st, M, w, m->mlp, mat(P.hact, m->mlp), wmat(L.w_proj, m->mlp), P.x, w, 0, e2));  // x += mlp
    }
  }
  // ln_post on the class token, then the visual projection
  MBS_TRY(mb200_layernorm_fwd(P.x, (long long)T * w, m->ln_post_g, m->ln_post_b, P.pooled, w, nullptr, nullptr, B, w, kEps,
                              st));
  return gemm(st, B, m->out_dim, w, mat(P.pooled, w), wmat(m->proj_t, w), feats, m->out_dim, 0);
}

int forward_train(const mb200_vit_model* m, const bf16s* images, bf16s* feats, int B, void* ws, size_t ws_bytes,
                  void* st) {
  Plan P;
  MBS_TRY(make_plan(P, m, B, ws));
  MBS_REQUIRE(ws != nullptr && ws_bytes >= P.bytes, MB200_E_ARG, "vit_forward_train: workspace too small (%zu < %zu)",
              ws_bytes, P.bytes);
  ScratchScope scratch(P.gemm_ws, kGemmScratchBytes);
  MBS_REQUIRE(m->ld_conv % 8 == 0 && m->ld_conv >= P.Kp, MB200_E_ALIGN, "vit_forward_train: bad ld_conv");
  const int w = m->width, H = m->n_head, hd = w / H, T = P.T, M = P.M, np = B * P.g * P.g;
  const float scale = 1.0f / sqrtf((float)hd);
  // conv1 as im2col + GEMM, then [cls; patches] + positional embedding, then ln_pre (input xa kept for its backward)
  MBS_TRY(rt_zero(P.patches, (size_t)np * P.ldpatch * sizeof(bf16s), st));
  MBS_TRY(mb200_patchify(images, P.patches, P.ldpatch, B, m->image, m->patch, st));
  MBS_TRY(gemm(st, np, w, P.Kp, mat(P.patches, P.ldpatch), mat(m->w_conv, m->ld_conv), P.pe, w, 0));
  MBS_TRY(mb200_vit_assemble(P.xa, P.pe, m->cls, m->pos, B, T, w, st));
  MBS_TRY(mb200_layernorm_fwd(P.xa, w, m->ln_pre_g, m->ln_pre_b, P.acts[0].x_in, w, P.mean0, P.rstd0, M, w, kEps, st));
  const long long qb0 = hd, qb1 = (long long)T * 3 * w;
  const long long pb0 = (long long)T * P.ldS, pb1 = (long long)H * T * P.ldS;
  for (int l = 0; l < m->n_layer; ++l) {
    const mb200_vit_layer& L = m->layers[l];
    LayerActs& a = P.acts[l];
    bf16s* x_next = l + 1 < m->n_layer ? P.acts[l + 1].x_in : P.x_out;
    MBS_TRY(mb200_layernorm_fwd(a.x_in, w, L.ln1_g, L.ln1_b, a.h1, w, a.mean1, a.rstd1, M, w, kEps, st));
    {
      Epi e;
      e.bias = L.b_qkv;
      MBS_TRY(gemm(st, M, 3 * w, w, mat(a.h1, w), mat(L.w_qkv, w), a.qkv, 3 * w, 0, e));
    }
    // scores = Q K^T (fp32), P = softmax(scores / sqrt(hd)), O = P V   (no mask: CLIP's image tower attends fully)
    if (flash_ok(hd)) {
      MBS_TRY(mb200_attn_fwd_flash(a.qkv, 3 * w, qb0, qb1, a.qkv + w, 3 * w, qb0, qb1, a.qkv + 2 * w, 3 * w, qb0, qb1,
                                   a.attn_o, w, a.P, P.ldS, nullptr, B, T, T, H, hd, 0, st));
    } else {
      MBS_TRY(gemm(st, T, T, hd, mat(a.qkv, 3 * w, 0, qb0, qb1), mat(a.qkv + w, 3 * w, 0, qb0, qb1), P.scores, P.ldS, 1,
                   Epi(), H, B, pb0, pb1));
      MBS_TRY(mb200_softmax_fwd(P.scores, P.ldS, pb0, a.P, P.ldS, pb0, B * H, T, T, scale, 0, 0, st));
      MBS_TRY(gemm(st, T, hd, T, mat(a.P, P.ldS, 0, pb0, pb1), mat(a.qkv + 2 * w, 3 * w, 1, qb0, qb1), a.attn_o, w, 0,
                   Epi(), H, B, hd, (long long)T * w));
    }
    {
      Epi e;
      e.bias = L.b_out;
      e.res1 = a.x_in;
      e.ld_res = w;
      MBS_TRY(gemm(st, M, w, w, mat(a.attn_o, w), mat(L.w_out, w), a.x_mid, w, 0, e));  // x_mid = x + out_proj(attn)
    }
    MBS_TRY(mb200_layernorm_fwd(a.x_mid, w, L.ln2_g, L.ln2_b, a.h2, w, a.mean2, a.rstd2, M, w, kEps, st));
    {
      Epi e;
      e.bias = L.b_fc;
      e.act = MB200_ACT_QUICK_GELU;
      e.aux_out = a.pre;  // pre-activation kept for the QuickGELU derivative
      MBS_TRY(gemm(st, M, m->mlp, w, mat(a.h2, w), mat(L.w_fc, w), a.hact, m->mlp, 0, e));
      Epi e2;
      e2.bias = L.b_proj;
      e2.res1 = a.x_mid;
      e2.ld_res = w;
      MBS_TRY(gemm(st, M, w, m->mlp, mat(a.hact, m->mlp), mat(L.w_proj, m->mlp), x_next, w, 0, e2));  // x + mlp
    }
  }
  // ln_post on the class token (row b*T of x_out), then the visual projection
  MBS_TRY(mb200_layernorm_fwd(P.x_out, (long long)T * w, m->ln_post_g, m->ln_post_b, P.pooled, w, P.meanp, P.rstdp, B, w,
                              kEps, st));
  MBS_TRY(gemm(st, B, m->out_dim, w, mat(P.pooled, w), mat(m->proj_t, w), feats, m->out_dim, 0));
  return 0;
}

int backward(const mb200_vit_model* m, const mb200_vit_grads* G, const bf16s* dfeats, int acc, int B, void* ws,
             size_t ws_bytes, void* st) {
  Plan P;
  MBS_TRY(make_plan(P, m, B, ws));
  MBS_REQUIRE(ws != nullptr && ws_bytes >= P.bytes, MB200_E_ARG, "vit_backward: workspace too small");
  MBS_REQUIRE(G && G->layers && dfeats, MB200_E_ARG, "vit_backward: null gradient table / dfeats");
  ScratchScope scratch(P.gemm_ws, kGemmScratchBytes);
  const int w = m->width, H = m->n_head, hd = w / H, T = P.T, M = P.M, np = B * P.g * P.g, mlp = m->mlp;
  const float scale = 1.0f / sqrtf((float)hd);
  const long long qb0 = hd, qb1 = (long long)T * 3 * w;
  const long long pb0 = (long long)T * P.ldS, pb1 = (long long)H * T * P.ldS;

  // ---- head: feats = ln_post(x_out[:, 0]) @ proj ----
  // dproj[w, out] (+)= pooled^T dfeats
  MBS_TRY(wgrad(st, w, m->out_dim, B, P.pooled, w, dfeats, m->out_dim, G->proj, m->out_dim, acc));
  // dpooled = dfeats proj^T   (proj_t is [out, w]: element (n = w-index, k = out-index) at k*w + n -> MN-major B)
  MBS_TRY(gemm(st, B, w, m->out_dim, mat(dfeats, m->out_dim), mat(m->proj_t, w, 1), P.dpooled, w, 0));
  MBS_TRY(mb200_layernorm_param_grad(P.dpooled, w, P.x_out, (long long)T * w, P.meanp, P.rstdp, G->ln_post_g,
                                     G->ln_post_b, B, w, acc, st));
  // only the class-token rows of the last block's output receive gradient
  bf16s* g = P.gA;
  bf16s* g_other = P.gB;
  MBS_TRY(rt_zero(g, (size_t)M * w * sizeof(bf16s), st));
  MBS_TRY(mb200_layernorm_bwd(P.dpooled, w, P.x_out, (long long)T * w, m->ln_post_g, P.meanp, P.rstdp, nullptr, 0, g,
                              (long long)T * w, B, w, st));

  for (int l = m->n_layer - 1; l >= 0; --l) {
    const mb200_vit_layer& L = m->layers[l];
    const mb200_vit_layer_grads& GL = G->layers[l];
    LayerActs& a = P.acts[l];
    // ---- MLP: x_next = x_mid + hact Wproj^T + b_proj, hact = quick_gelu(pre), pre = h2 Wfc^T + b_fc ----
    MBS_TRY(wgrad(st, w, mlp, M, g, w, a.hact, mlp, GL.w_proj, mlp, acc));
    MBS_TRY(mb200_colsum(g, w, M, w, GL.b_proj, acc, st));
    MBS_TRY(gemm(st, M, mlp, w, mat(g, w), mat(L.w_proj, mlp, 1), P.dhact, mlp, 0));  // dhact = g Wproj
    MBS_TRY(mb200_quick_gelu_bwd(P.dhact, a.pre, P.dhact, (int64_t)M * mlp, st));     // -> dpre (in place)
    MBS_TRY(wgrad(st, mlp, w, M, P.dhact, mlp, a.h2, w, GL.w_fc, w, acc));
    MBS_TRY(mb200_colsum(P.dhact, mlp, M, mlp, GL.b_fc, acc, st));
    MBS_TRY(gemm(st, M, w, mlp, mat(P.dhact, mlp), mat(L.w_fc, w, 1), P.dh, w, 0));   // dh2 = dpre Wfc
    MBS_TRY(mb200_layernorm_param_grad_rows(P.dh, w, a.x_mid, w, a.mean2, a.rstd2, GL.ln2_g, GL.ln2_b, M, w, acc, st));
    MBS_TRY(mb200_layernorm_bwd(P.dh, w, a.x_mid, w, L.ln2_g, a.mean2, a.rstd2, g, w, P.gmid, w, M, w, st));
    // ---- attention: x_mid = x_in + attn_o Wout^T + b_out ----
    MBS_TRY(wgrad(st, w, w, M, P.gmid, w, a.attn_o, w, GL.w_out, w, acc));
    MBS_TRY(mb200_colsum(P.gmid, w, M, w, GL.b_out, acc, st));
    MBS_TRY(gemm(st, M, w, w, mat(P.gmid, w), mat(L.w_out, w, 1), P.dattn_o, w, 0));  // d(attn_o) = gmid Wout
    {
      Mat dO = mat(P.dattn_o, w, 0, hd, (long long)T * w);
      Mat dO_mn = mat(P.dattn_o, w, 1, hd, (long long)T * w);
      // dP = dO V^T (fp32)
      MBS_TRY(gemm(st, T, T, hd, dO, mat(a.qkv + 2 * w, 3 * w, 0, qb0, qb1), P.scores, P.ldS, 1, Epi(), H, B, pb0, pb1));
      // dV = P^T dO
      MBS_TRY(gemm(st, T, hd, T, mat(a.P, P.ldS, 1, pb0, pb1), dO_mn, P.dqkv + 2 * w, 3 * w, 0, Epi(), H, B, qb0, qb1));
      // dS = P * (dP - rowsum(dP * P)) / sqrt(hd)
      MBS_TRY(mb200_softmax_bwd(P.scores, P.ldS, pb0, a.P, P.ldS, pb0, P.dS, P.ldS, pb0, B * H, T, T, scale, st));
      // dQ = dS K ; dK = dS^T Q
      MBS_TRY(gemm(st, T, hd, T, mat(P.dS, P.ldS, 0, pb0, pb1), mat(a.qkv + w, 3 * w, 1, qb0, qb1), P.dqkv, 3 * w, 0,
                   Epi(), H, B, qb0, qb1));
      MBS_TRY(gemm(st, T, hd, T, mat(P.dS, P.ldS, 1, pb0, pb1), mat(a.qkv, 3 * w, 1, qb0, qb1), P.dqkv + w, 3 * w, 0,
                   Epi(), H, B, qb0, qb1));
    }
    MBS_TRY(wgrad(st, 3 * w, w, M, P.dqkv, 3 * w, a.h1, w, GL.w_qkv, w, acc));
    MBS_TRY(mb200_colsum(P.dqkv, 3 * w, M, 3 * w, GL.b_qkv, acc, st));
    MBS_TRY(gemm(st, M, w, 3 * w, mat(P.dqkv, 3 * w), mat(L.w_qkv, w, 1), P.dh, w, 0));  // dh1 = dqkv Wqkv
    MBS_TRY(mb200_layernorm_param_grad_rows(P.dh, w, a.x_in, w, a.mean1, a.rstd1, GL.ln1_g, GL.ln1_b, M, w, acc, st));
    MBS_TRY(mb200_layernorm_bwd(P.dh, w, a.x_in, w, L.ln1_g, a.mean1, a.rstd1, P.gmid, w, g_other, w, M, w, st));
    bf16s* t = g;
    g = g_other;
    g_other = t;
  }
  // ---- ln_pre, positional / class embeddings, conv1 ----
  MBS_TRY(mb200_layernorm_param_grad_rows(g, w, P.xa, w, P.mean0, P.rstd0, G->ln_pre_g, G->ln_pre_b, M, w, acc, st));
  bf16s* dxa = g_other;
  MBS_TRY(mb200_layernorm_bwd(g, w, P.xa, w, m->ln_pre_g, P.mean0, P.rstd0, nullptr, 0, dxa, w, M, w, st));
  // xa[b, t] = (t == 0 ? cls : pe[b, t-1]) + pos[t]: dpos = sum_b dxa[b], dcls = sum_b dxa[b, 0]
  MBS_TRY(mb200_colsum(dxa, (long long)T * w, B, T * w, G->pos, acc, st));
  MBS_TRY(mb200_colsum(dxa, (long long)T * w, B, w, G->cls, acc, st));
  for (int b = 0; b < B; ++b)  // patch-token rows of image b, made contiguous for the conv1 wgrad
    MBS_TRY(rt_copy(P.dpe + (size_t)b * (T - 1) * w, dxa + ((size_t)b * T + 1) * w, (size_t)(T - 1) * w * sizeof(bf16s),
                    st));
  // dWconv[w, 3P^2] (+)= dpe^T patches
  MBS_TRY(wgrad(st, w, P.Kp, np, P.dpe, w, P.patches, P.ldpatch, G->w_conv, P.Kp, acc));
  return 0;
}

}  // namespace
}  // namespace mb200

extern "C" size_t mb200_vit_workspace_bytes(const mb200_vit_model* m, int32_t B) {
  mb200::InferPlan P;
  if (mb200::make_infer_plan(P, m, B, nullptr)) return 0;
  return P.bytes;
}

extern "C" int mb200_vit_forward(const mb200_vit_model* m, const void* images, void* feats, int32_t B, void* ws,
                                 size_t ws_bytes, void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  return mb200::forward_infer(m, (const mb200::bf16s*)images, (mb200::bf16s*)feats, B, ws, ws_bytes, stream);
}

extern "C" size_t mb200_vit_train_workspace_bytes(const mb200_vit_model* m, int32_t B) {
  mb200::Plan P;
  if (mb200::make_plan(P, m, B, nullptr)) return 0;
  return P.bytes;
}

extern "C" int mb200_vit_forward_train(const mb200_vit_model* m, const void* images, void* feats, int32_t B, void* ws,
                                       size_t ws_bytes, void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  return mb200::forward_train(m, (const mb200::bf16s*)images, (mb200::bf16s*)feats, B, ws, ws_bytes, stream);
}

extern "C" int mb200_vit_backward(const mb200_vit_model* m, const mb200_vit_grads* g, const void* dfeats,
                                  int32_t accumulate, int32_t B, void* ws, size_t ws_bytes, void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  return mb200::backward(m, g, (const mb200::bf16s*)dfeats, accumulate, B, ws, ws_bytes, stream);
}
