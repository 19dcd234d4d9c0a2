// magma_b200 — GPT-J + adapters: THE language-model runtime (training forward with saved activations + backward, or
// with only each block's input saved and the block recomputed in the backward; full-sequence inference, KV-cache
// prefill and decode steps), host-only.
//
// One C call per pass instead of ~1000 Python-level op calls: this file carves the workspace and issues the kernels of a
// pass on one stream. It schedules every adapter form of the reference — plain bottleneck in "normal" or "parallel"
// wiring (what the shipped configurations use), with or without a leading LayerNorm (`add_layernorm`,
// magma/adapters.py:16-17) and the learnable scalar of the parallel forms (`scaled_parallel`, adapters.py:57-66,85-92) —
// on the MLP and / or the attention branch (magma/magma.py:102-174), from the primitive operators of the C ABI only:
//
//   block (hf:gptj/modeling_gptj.py:400-413, parallel residual):  h = ln_1(x);  x' = attn(h) + mlp(h) + x
//   Adapter.forward            adapters.py:38-39    y = A(z) + z            A(z) = Wu relu(Wd LN?(z) + bd) + bu
//   ParallelAdapter.forward    adapters.py:63-66    y = module(h) + s * A(h)
//   AdapterWrapper / ParallelAdapterWrapper         the same two on the attention output / input (:85-92,:109-116)
//   LM head + shifted CE       hf:gptj/modeling_gptj.py:573,623 ; hf:loss/loss_utils.py:28-67
//
// Attention: the fused single-tile kernels when the sequence fits one tile (S <= 128: BASELINE config 2), the fused
// multi-tile forward (mb200_attn_fwd_flash) for longer sequences / prefill over a KV cache — in training it also writes
// the probabilities, and the backward then runs as strided batched GEMMs on the fused qkv buffer + softmax_bwd — and
// batched GEMMs + softmax kernels for head dims the fused kernels do not take. The backward runs dgrad through every
// GEMM, and wgrad for the adapters and for the LM weights m->lm_grads names (none when it is NULL: the LM is frozen).
//
// No kernels and no CUDA calls here (sched_rt.h, which also holds the GEMM helpers and the materialised attention this
// file shares with vit_sched.cu): tests/test_sched_emul_cpu.py compiles this file as plain C++ against
// oracle/cabi_emul.cpp and checks every adapter form against torch autograd of the oracle on the CPU; on the GPU it is
// the path every LM test and the benchmark run.
#include "sched_rt.h"

#include <stdlib.h>

// The two kernels only output_attentions uses are weak references: the CPU build of this file (oracle/build_emul.py)
// links an emulation that may not carry them and must still load. A pass that needs one that is absent fails with
// MB200_E_ARG; the CUDA library always defines both.
#pragma weak mb200_attn_bwd_tile_dp
#pragma weak mb200_attn_decode_probs
// likewise the kernel that joins a loss's gradient on the logits to the cross-entropy gradient
#pragma weak mb200_logits_grad_combine

namespace mb200 {
namespace {

// what one adapter keeps from forward to backward
struct AdapterActs {
  bf16s* zn;    // [M,d] LN(z) when the adapter has a leading LayerNorm
  float* mean;  // [M]
  float* rstd;  // [M]
  bf16s* t;     // [M,r] hidden (post activation)
  bf16s* pre;   // [M,r] pre-activation (GeLU adapters only: ReLU's mask is read off t)
  bf16s* u;     // [M,d] up-projection output before scaling (scaled_parallel only)
};

struct LayerActs {
  bf16s* x_in;     // [M,d] residual stream entering the block
  bf16s* h;        // [M,d] ln_1 output
  float* mean;     // [M]
  float* rstd;     // [M]
  bf16s* qkv;      // [M,3d] after rotary
  bf16s* P;        // [B,H,S,ldP]
  bf16s* attn_o;   // [M,d] merged heads, before out_proj
  bf16s* pre;      // [M,dff] fc_in pre-activation
  bf16s* hact;     // [M,dff] gelu(pre): the plan's shared P.hact, or the layer's own when its fc_out trains (stored path)
  bf16s* mlp_out;  // [M,d] fc_out output (input of a "normal" MLP adapter)
  bf16s* a_out;    // [M,d] out_proj output (input of a "normal" attention adapter)
  AdapterActs am, aa;
};

struct Plan {
  int M, d, dff, H, hd, S, B, ldP;
  long long ldv;
  LayerActs acts[64];
  float* scores;  // [B,H,S,ldP] fp32 (scores in forward, dP in backward)
  bf16s *hact, *ax, *x_final, *xf_ln, *dlogits;
  float *lnf_mean, *lnf_rstd, *row_loss, *rope_tab;
  int* n_valid;
  // backward temporaries
  bf16s *g0, *g1, *gs, *dt, *dzn, *dm, *dhact, *dh_mlp, *dattn_o, *dqkv, *dS, *dh, *da, *dhp;
  void* gemm_ws;  // scratch lent to the GEMM core: split-K slices
  size_t gemm_ws_bytes;
  float* ln_scratch;  // [2d] the half of a LayerNorm's parameter gradient whose parameter is frozen
  size_t bytes;
};

// the fused single-tile attention kernels (csrc/attention.cu) cover S <= 128 with head_dim in {64, 128, 192, 256};
// MB200_ATTN_TILE=0 skips them
inline bool tile_ok(int S, int hd) {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("MB200_ATTN_TILE");
    on = e ? atoi(e) : 1;
  }
  return on != 0 && S >= 1 && S <= 128 && hd >= 64 && hd <= 256 && hd % 64 == 0;
}

// the GEMM epilogue that rotates (mode 1) or inversely rotates (mode -1) the first rot dims of each hd-wide head in
// columns [0, ncols), with the positions of row % S in the rotary table tab
inline Epi rope_epi(const float* tab, int mode, int S, int hd, int rot, int ncols) {
  Epi e;
  e.rope_tab = tab;
  e.rope_mode = mode;
  e.rope_S = S;
  e.rope_hd = hd;
  e.rope_rot = rot;
  e.rope_ncols = ncols;
  return e;
}

inline bool has_ln(const mb200_adapter_ex& a) { return a.ln_g != nullptr; }
inline bool has_scale(const mb200_adapter_ex& a) { return a.scale != nullptr; }
inline const mb200_gptj_layer_grads* layer_grads(const mb200_gptj_model_ex* m, int l) {
  return m->lm_grads && m->lm_grads->layers ? &m->lm_grads->layers[l] : nullptr;
}

void carve_adapter(Carver& c, AdapterActs& a, const mb200_adapter_ex& ad, int kind, size_t M, size_t d, int r,
                   int act = 0, bool training = true) {
  a.zn = nullptr;
  a.mean = a.rstd = nullptr;
  a.t = a.u = a.pre = nullptr;
  if (kind == MB200_ADAPTER_NONE) return;
  if (act != 0 && training) a.pre = c.take<bf16s>(M * (size_t)r);
  if (has_ln(ad)) {
    a.zn = c.take<bf16s>(M * d);
    a.mean = c.take<float>(M);
    a.rstd = c.take<float>(M);
  }
  a.t = c.take<bf16s>(M * (size_t)r);
  if (has_scale(ad)) a.u = c.take<bf16s>(M * d);
}

// recompute: every layer keeps only x_in; its other activations live in one scratch shared by all layers, which
// the backward refills for each layer by rerunning that layer's forward (layer_fwd) from x_in
int make_plan(Plan& P, const mb200_gptj_model_ex* m, int B, int S, void* ws, bool recompute = false) {
  MBS_REQUIRE(m && m->layers && m->n_layer > 0 && m->n_layer <= 64, MB200_E_SHAPE, "gptj_sched: n_layer out of range");
  MBS_REQUIRE(B > 0 && S > 0 && m->n_head > 0 && m->d % m->n_head == 0 && m->d % 8 == 0 && m->d_ff % 8 == 0,
              MB200_E_SHAPE, "gptj_sched: bad d / n_head / d_ff");
  MBS_REQUIRE(m->adapter_act == 0 || m->adapter_act == 1, MB200_E_ARG, "gptj_sched: adapter_act must be 0 (ReLU) or 1 (GeLU)");
  MBS_REQUIRE((m->d / m->n_head) % 8 == 0 && m->rotary_dim % 4 == 0 && m->rotary_dim <= m->d / m->n_head, MB200_E_SHAPE,
              "gptj_sched: head_dim must be a multiple of 8 and rotary_dim a multiple of 4 within it");
  for (int l = 0; l < m->n_layer; ++l) {
    const mb200_gptj_layer_ex& L = m->layers[l];
    MBS_REQUIRE(!(m->mlp_adapter == MB200_ADAPTER_NORMAL && has_scale(L.mlp_ad)) &&
                    !(m->attn_adapter == MB200_ADAPTER_NORMAL && has_scale(L.attn_ad)),
                MB200_E_ARG, "gptj_sched: adapter_scale exists on the parallel adapter forms only (adapters.py:57-61)");
    MBS_REQUIRE((m->mlp_adapter == MB200_ADAPTER_NONE || (m->mlp_adapter_r > 0 && m->mlp_adapter_r % 8 == 0)) &&
                    (m->attn_adapter == MB200_ADAPTER_NONE || (m->attn_adapter_r > 0 && m->attn_adapter_r % 8 == 0)),
                MB200_E_SHAPE, "gptj_sched: adapter bottleneck widths must be positive multiples of 8");
  }
  Carver c(ws);
  P.B = B;
  P.S = S;
  P.M = B * S;
  P.d = m->d;
  P.dff = m->d_ff;
  P.H = m->n_head;
  P.hd = m->d / m->n_head;
  P.ldP = (int)align_up(S, 8);
  P.ldv = (long long)align_up(m->vocab, 64);
  const size_t M = P.M, d = P.d, dff = P.dff;
  const size_t nP = (size_t)B * P.H * S * P.ldP;
  // the shared scratch of the recompute plan holds what any layer's adapters keep
  mb200_adapter_ex um = m->layers[0].mlp_ad, ua = m->layers[0].attn_ad;
  for (int l = 1; recompute && l < m->n_layer; ++l) {
    const mb200_gptj_layer_ex& L = m->layers[l];
    if (has_ln(L.mlp_ad)) um.ln_g = L.mlp_ad.ln_g;
    if (has_scale(L.mlp_ad)) um.scale = L.mlp_ad.scale;
    if (has_ln(L.attn_ad)) ua.ln_g = L.attn_ad.ln_g;
    if (has_scale(L.attn_ad)) ua.scale = L.attn_ad.scale;
  }
  for (int l = 0; l < m->n_layer; ++l) {
    LayerActs& a = P.acts[l];
    a.x_in = c.take<bf16s>(M * d);
    if (recompute && l > 0) {
      bf16s* x_in = a.x_in;
      a = P.acts[0];
      a.x_in = x_in;
      continue;
    }
    a.h = c.take<bf16s>(M * d);
    a.mean = c.take<float>(M);
    a.rstd = c.take<float>(M);
    a.qkv = c.take<bf16s>(M * 3 * d);
    a.P = c.take<bf16s>(nP);
    a.attn_o = c.take<bf16s>(M * d);
    a.pre = c.take<bf16s>(M * dff);
    a.mlp_out = c.take<bf16s>(M * d);
    a.a_out = c.take<bf16s>(M * d);
    carve_adapter(c, a.am, recompute ? um : m->layers[l].mlp_ad, m->mlp_adapter, M, d, m->mlp_adapter_r, m->adapter_act);
    carve_adapter(c, a.aa, recompute ? ua : m->layers[l].attn_ad, m->attn_adapter, M, d, m->attn_adapter_r,
                  m->adapter_act);
  }
  P.scores = c.take<float>(nP);
  P.hact = c.take<bf16s>(M * dff);
  P.ax = c.take<bf16s>(M * d);
  P.x_final = c.take<bf16s>(M * d);
  P.xf_ln = c.take<bf16s>(M * d);
  P.lnf_mean = c.take<float>(M);
  P.lnf_rstd = c.take<float>(M);
  P.row_loss = c.take<float>(M);
  P.n_valid = c.take<int>(4);
  P.rope_tab = c.take<float>((size_t)S * m->rotary_dim);
  P.dlogits = c.take<bf16s>(M * (size_t)P.ldv);
  const int rmax = m->mlp_adapter_r > m->attn_adapter_r ? m->mlp_adapter_r : m->attn_adapter_r;
  P.g0 = c.take<bf16s>(M * d);
  P.g1 = c.take<bf16s>(M * d);
  P.gs = c.take<bf16s>(M * d);
  P.dt = c.take<bf16s>(M * (size_t)(rmax > 0 ? rmax : 8));
  P.dzn = c.take<bf16s>(M * d);
  P.dm = c.take<bf16s>(M * d);
  P.dhact = c.take<bf16s>(M * dff);
  P.dh_mlp = c.take<bf16s>(M * d);
  P.dattn_o = c.take<bf16s>(M * d);
  P.dqkv = c.take<bf16s>(M * 3 * d);
  P.dS = c.take<bf16s>(nP);
  P.dh = c.take<bf16s>(M * d);
  P.da = c.take<bf16s>(M * d);
  P.dhp = c.take<bf16s>(M * d);
  P.gemm_ws_bytes = M > 128 ? kGemmScratchBytes : 0;
  P.gemm_ws = P.gemm_ws_bytes ? c.take<uint8_t>(P.gemm_ws_bytes) : nullptr;
  // what trainable LM weights add, after everything a frozen LM's plan holds: fc_out's wgrad reads gelu(pre), which
  // the next layer's forward overwrites in P.hact on the stored path
  P.ln_scratch = m->lm_grads ? c.take<float>(2 * d) : nullptr;
  for (int l = 0; l < m->n_layer; ++l) {
    const mb200_gptj_layer_grads* G = layer_grads(m, l);
    P.acts[l].hact = G && G->w_fc_out && !recompute ? c.take<bf16s>(M * dff) : P.hact;
  }
  P.bytes = align_up(c.off, 256);
  return 0;
}

// out = s * A(z) + res1 + res2, A(z) = Wu act(Wd LN?(z) + bd) + bu   (s = 1 without adapter_scale; act = ReLU, or the
// tanh GeLU with its pre-activation kept for the backward pass when a.pre is carved)
int adapter_fwd(void* st, const mb200_adapter_ex& ad, AdapterActs& a, int M, int d, int r, float eps, const bf16s* z,
                bf16s* out, const bf16s* res1, const bf16s* res2, int act) {
  const bf16s* zin = z;
  if (has_ln(ad)) {
    MBS_TRY(mb200_layernorm_fwd(z, d, ad.ln_g, ad.ln_b, a.zn, d, a.mean, a.rstd, M, d, eps, st));
    zin = a.zn;
  }
  Epi e1;
  e1.bias = ad.bd;
  e1.act = act ? MB200_ACT_GELU_NEW : MB200_ACT_RELU;
  e1.aux_out = act ? a.pre : nullptr;  // (inference plans carve no pre buffer)
  MBS_TRY(gemm(st, M, r, d, mat(zin, d), mat(ad.wd, d), a.t, r, 0, e1));
  Epi e2;
  e2.bias = ad.bu;
  if (!has_scale(ad)) {
    e2.res1 = res1;
    e2.res2 = res2;
    e2.ld_res = d;
    return gemm(st, M, d, r, mat(a.t, r), mat(ad.wu, r), out, d, 0, e2);
  }
  MBS_TRY(gemm(st, M, d, r, mat(a.t, r), mat(ad.wu, r), a.u, d, 0, e2));
  return mb200_scale_add(a.u, ad.scale, res1, res2, out, (int64_t)M * d, st);
}

// g = dL/d(out) of adapter_fwd. dz_out = res + dL/dz through the adapter; parameter gradients accumulate or overwrite.
int adapter_bwd(void* st, const mb200_adapter_ex& ad, const AdapterActs& a, const Plan& P, int M, int d, int r,
                const bf16s* g, const bf16s* z, bf16s* dz_out, const bf16s* res, int acc, int act) {
  const bf16s* gu = g;  // gradient w.r.t. the up-projection output
  if (has_scale(ad)) {
    if (ad.g_scale) MBS_TRY(mb200_dot(g, a.u, (int64_t)M * d, ad.g_scale, acc, st));  // d s = <g, u>
    MBS_TRY(mb200_scale_add(g, ad.scale, nullptr, nullptr, P.gs, (int64_t)M * d, st));   // gu = s * g
    gu = P.gs;
  }
  const bf16s* zin = has_ln(ad) ? a.zn : z;
  Epi e1;
  e1.dact = act ? MB200_DACT_GELU_NEW : MB200_DACT_RELU;
  e1.aux_in = act ? a.pre : a.t;
  MBS_TRY(gemm(st, M, r, d, mat(gu, d), mat(ad.wu, r, 1), P.dt, r, 0, e1));  // dt = (gu Wu) * act'(pre)   (ReLU: 1[t > 0])
  if (ad.g_wd) {
    MBS_TRY(wgrad(st, d, r, M, gu, d, a.t, r, ad.g_wu, r, acc));    // dWu[d,r] = gu^T t
    MBS_TRY(mb200_colsum(gu, d, M, d, ad.g_bu, acc, st));
    MBS_TRY(wgrad(st, r, d, M, P.dt, r, zin, d, ad.g_wd, d, acc));  // dWd[r,d] = dt^T zin
    MBS_TRY(mb200_colsum(P.dt, r, M, r, ad.g_bd, acc, st));
  }
  if (!has_ln(ad)) {
    Epi e2;
    e2.res1 = res;
    e2.ld_res = d;
    return gemm(st, M, d, r, mat(P.dt, r), mat(ad.wd, d, 1), dz_out, d, 0, e2);  // dz = dt Wd (+ res)
  }
  MBS_TRY(gemm(st, M, d, r, mat(P.dt, r), mat(ad.wd, d, 1), P.dzn, d, 0));  // d LN(z)
  if (ad.g_ln_g)
    MBS_TRY(mb200_layernorm_param_grad_rows(P.dzn, d, z, d, a.mean, a.rstd, ad.g_ln_g, ad.g_ln_b, M, d, acc, st));
  return mb200_layernorm_bwd(P.dzn, d, z, d, ad.ln_g, a.mean, a.rstd, res, d, dz_out, d, M, d, st);
}

// gradients of a LayerNorm's weight and bias when either trains (the kernel writes both: a frozen half goes to scratch)
int ln_param_grad(void* st, const Plan& P, const bf16s* dy, const bf16s* x, const float* mean, const float* rstd,
                  float* g_gamma, float* g_beta, int acc) {
  if (!g_gamma && !g_beta) return 0;
  return mb200_layernorm_param_grad_rows(dy, P.d, x, P.d, mean, rstd, g_gamma ? g_gamma : P.ln_scratch,
                                         g_beta ? g_beta : P.ln_scratch + P.d, P.M, P.d, acc, st);
}

// one block of the training forward: from P.acts[l].x_in to xout, keeping the activations the backward reads in
// P.acts[l]. The forward pass and the recompute backward both issue it, so a recomputed layer is the stored one bit for bit.
int layer_fwd(const mb200_gptj_model_ex* m, Plan& P, int l, bf16s* xout, void* st) {
  const int M = P.M, d = P.d, dff = P.dff, H = P.H, hd = P.hd, B = P.B, S = P.S;
  const long long qb0 = hd, qb1 = (long long)S * 3 * d;
  const mb200_gptj_layer_ex& L = m->layers[l];
  LayerActs& a = P.acts[l];
  const bf16s* xin = a.x_in;
  MBS_TRY(mb200_layernorm_fwd(xin, d, L.ln1_g, L.ln1_b, a.h, d, a.mean, a.rstd, M, d, m->ln_eps, st));
  // fused q/k/v projection, rotary embedding applied to the q and k column ranges in the epilogue
  MBS_TRY(gemm(st, M, 3 * d, d, mat(a.h, d), wmat(L.w_qkv, d), a.qkv, 3 * d, 0,
               rope_epi(P.rope_tab, 1, S, hd, m->rotary_dim, 2 * d)));
  if (tile_ok(S, hd)) {  // whole sequence in one tile: fused QK^T / softmax / PV, one CTA per (batch, head)
    MBS_TRY(mb200_attn_fwd_tile(a.qkv, 3 * d, a.P, P.ldP, a.attn_o, d, B, S, H, hd, st));
  } else if (flash_ok(hd)) {  // any S: fused multi-tile forward; P is written for the materialised backward
    MBS_TRY(mb200_attn_fwd_flash(a.qkv, 3 * d, qb0, qb1, a.qkv + d, 3 * d, qb0, qb1, a.qkv + 2 * d, 3 * d, qb0, qb1,
                                 a.attn_o, d, a.P, P.ldP, nullptr, B, S, S, H, hd, 1, st));
  } else {
    MBS_TRY(attn_fwd_gemm(st, mat(a.qkv, 3 * d, 0, qb0, qb1), mat(a.qkv + d, 3 * d, 0, qb0, qb1),
                          mat(a.qkv + 2 * d, 3 * d, 1, qb0, qb1), S, S, H, B, hd, P.scores, a.P, P.ldP, a.attn_o, d, 1, 0));
  }
  // out_proj; ax = attention branch + residual x
  if (m->attn_adapter == MB200_ADAPTER_NONE) {
    Epi e;
    e.res1 = xin;
    e.ld_res = d;
    MBS_TRY(gemm(st, M, d, d, mat(a.attn_o, d), wmat(L.w_out, d), P.ax, d, 0, e));
  } else if (m->attn_adapter == MB200_ADAPTER_NORMAL) {  // AdapterWrapper: A(attn_out) + attn_out
    MBS_TRY(gemm(st, M, d, d, mat(a.attn_o, d), wmat(L.w_out, d), a.a_out, d, 0));
    MBS_TRY(adapter_fwd(st, L.attn_ad, a.aa, M, d, m->attn_adapter_r, m->ln_eps, a.a_out, P.ax, a.a_out, xin, m->adapter_act));
  } else {  // ParallelAdapterWrapper: attn(h) + s * A(h)
    Epi e;
    e.res1 = xin;
    e.ld_res = d;
    MBS_TRY(gemm(st, M, d, d, mat(a.attn_o, d), wmat(L.w_out, d), a.a_out, d, 0, e));
    MBS_TRY(adapter_fwd(st, L.attn_ad, a.aa, M, d, m->attn_adapter_r, m->ln_eps, a.h, P.ax, a.a_out, nullptr, m->adapter_act));
  }
  {  // fc_in + bias + gelu_new, pre-activation kept
    Epi e;
    e.bias = L.b_fc_in;
    e.act = MB200_ACT_GELU_NEW;
    e.aux_out = a.pre;
    MBS_TRY(gemm(st, M, dff, d, mat(a.h, d), wmat(L.w_fc_in, d), a.hact, dff, 0, e));
  }
  Epi eo;
  eo.bias = L.b_fc_out;
  if (m->mlp_adapter == MB200_ADAPTER_NONE) {
    eo.res1 = P.ax;
    eo.ld_res = d;
    MBS_TRY(gemm(st, M, d, dff, mat(a.hact, dff), wmat(L.w_fc_out, dff), xout, d, 0, eo));
  } else if (m->mlp_adapter == MB200_ADAPTER_NORMAL) {  // Sequential(mlp, Adapter): A(mlp(h)) + mlp(h)
    MBS_TRY(gemm(st, M, d, dff, mat(a.hact, dff), wmat(L.w_fc_out, dff), a.mlp_out, d, 0, eo));
    MBS_TRY(adapter_fwd(st, L.mlp_ad, a.am, M, d, m->mlp_adapter_r, m->ln_eps, a.mlp_out, xout, a.mlp_out, P.ax, m->adapter_act));
  } else {  // ParallelAdapter: mlp(h) + s * A(h)
    eo.res1 = P.ax;
    eo.ld_res = d;
    MBS_TRY(gemm(st, M, d, dff, mat(a.hact, dff), wmat(L.w_fc_out, dff), a.mlp_out, d, 0, eo));
    MBS_TRY(adapter_fwd(st, L.mlp_ad, a.am, M, d, m->mlp_adapter_r, m->ln_eps, a.h, xout, a.mlp_out, nullptr, m->adapter_act));
  }
  return 0;
}

// attn (NULL, or n_layer pointers, each NULL or bf16 [B,H,S,ld_attn]): output_attentions, each block's probabilities
// copied out of P.acts[l].P as soon as the block has run (on the recompute path the next block overwrites them). The
// saved P and the gradients on it share its layout, so ld_attn must be the plan's ldP = S rounded up to 8.
int forward(const mb200_gptj_model_ex* m, const bf16s* x, const int64_t* labels, bf16s* logits, long long ldv,
            float* loss, int B, int S, void* ws, size_t ws_bytes, void* st, bool recompute,
            bf16s* const* attn = nullptr, long long ld_attn = 0) {
  Plan P;
  MBS_TRY(make_plan(P, m, B, S, ws, recompute));
  MBS_REQUIRE(ws != nullptr && ws_bytes >= P.bytes, MB200_E_ARG, "gptj_sched_forward: workspace too small (%zu < %zu)",
              ws_bytes, P.bytes);
  MBS_REQUIRE(!attn || ld_attn == P.ldP, MB200_E_ALIGN, "gptj_sched_forward_attn: ld_attn=%lld must be %d (S rounded up to 8)",
              ld_attn, P.ldP);
  const int M = P.M, d = P.d;
  ScratchScope scratch(P.gemm_ws, P.gemm_ws_bytes);
  MBS_TRY(mb200_rope_table(P.rope_tab, S, m->rotary_dim, 0, st));
  MBS_TRY(rt_copy(P.acts[0].x_in, x, (size_t)M * d * sizeof(bf16s), st));
  for (int l = 0; l < m->n_layer; ++l) {
    MBS_TRY(layer_fwd(m, P, l, l + 1 < m->n_layer ? P.acts[l + 1].x_in : P.x_final, st));
    if (attn && attn[l])
      MBS_TRY(rt_copy(attn[l], P.acts[l].P, (size_t)B * P.H * S * P.ldP * sizeof(bf16s), st));
  }
  // ln_f + LM head (+ shifted cross-entropy; the logits' gradient is written now, scaled in backward)
  MBS_TRY(mb200_layernorm_fwd(P.x_final, d, m->lnf_g, m->lnf_b, P.xf_ln, d, P.lnf_mean, P.lnf_rstd, M, d, m->ln_eps, st));
  bf16s* lg = logits ? logits : P.dlogits;
  const long long ldl = logits ? ldv : P.ldv;
  MBS_REQUIRE(ldl % 8 == 0 && ldl >= m->vocab, MB200_E_ALIGN, "gptj_sched_forward: ldv=%lld must be >= vocab and %%8", ldl);
  {
    Epi e;
    e.bias = m->b_lm;
    MBS_TRY(gemm(st, M, m->vocab, d, mat(P.xf_ln, d), wmat(m->w_lm, d), lg, ldl, 0, e));
  }
  if (labels) {
    MBS_REQUIRE(loss != nullptr, MB200_E_ARG, "gptj_sched_forward: labels given but loss pointer is NULL");
    MBS_REQUIRE(ldl == P.ldv, MB200_E_ARG, "gptj_sched_forward: ldv must be %lld (vocab rounded up to 64)", P.ldv);
    MBS_TRY(mb200_cross_entropy(lg, ldl, labels, B, S, m->vocab, P.row_loss, P.n_valid, loss, P.dlogits, 1.0f, st));
  }
  return 0;
}

// Layers are processed from layer_hi-1 down to layer_lo; the LM-head / CE backward runs when layer_hi == n_layer. The
// residual-stream gradient lives in the workspace between calls, so a caller can split the range and exchange the
// gradients of finished layers while the rest runs (B200Engine.backward).
// recompute: each layer's activations are rebuilt from its x_in first. The rebuilt block output goes to P.dh, which is
// dead at that point, so x_in, x_final and everything else the forward left stay as they were and a second backward
// gives the same result.
// dhid (NULL, or n_layer + 1 pointers, each NULL or bf16 [M,d]): gradients of the hidden states hidden_states() returns.
// Entry l < n_layer is layer l's input, so its gradient joins the residual-stream gradient once layer l's backward has
// produced it (entry 0 thus reaches dx); the ln_f entry joins the LM head's dgrad in that GEMM's epilogue. Each entry is
// added by the one call whose range holds its layer, so a chunked backward adds it once.
// dattn (NULL, or n_layer pointers, each NULL or bf16 [B,H,S,ld_attn] with ld_attn = ldP): gradients of the attention
// probabilities forward() returned. Layer l's joins dP = dO V^T before rowsum(dP * P) — in the tile kernel's fragment
// (mb200_attn_bwd_tile_dp), or as the dP GEMM's residual on the materialised path.
// logits_grad (the backward_range_logits entries): dlg (NULL, or bf16 [M, V] rows of stride ld_dlg) is the gradient of
// a loss on the logits the forward returned. It joins loss_scale * P.dlogits in the caller's dcomb ([M, ldv]), which
// the LM head's dgrad then reads with alpha 1, so P.dlogits is never written and a second backward gives the same
// result. Without dlg and with loss_scale == 0 (a forward without labels, whose P.dlogits was never written) the LM
// head adds nothing and P.dlogits is not read.
// m->lm_grads: the weight gradients of the LM's own parameters join those of the adapters, from the gradients the dgrad
// GEMMs read and the activations the forward kept (each block's on the recompute path once it is rebuilt). A trainable
// LM head needs dcomb: its gradient, loss_scale * P.dlogits (+ dlg), is formed there once and read by all three GEMMs.
int backward(const mb200_gptj_model_ex* m, bf16s* dx, const bf16s* const* dhid, float loss_scale, int layer_hi,
             int layer_lo, int acc, int B, int S, void* ws, size_t ws_bytes, void* st, bool recompute,
             const bf16s* const* dattn = nullptr, long long ld_attn = 0, bool logits_grad = false,
             const bf16s* dlg = nullptr, long long ld_dlg = 0, bf16s* dcomb = nullptr) {
  Plan P;
  MBS_TRY(make_plan(P, m, B, S, ws, recompute));
  MBS_REQUIRE(ws != nullptr && ws_bytes >= P.bytes, MB200_E_ARG, "gptj_sched_backward: workspace too small");
  MBS_REQUIRE(!dattn || ld_attn == P.ldP, MB200_E_ALIGN,
              "gptj_sched_backward_range_attn: ld_attn=%lld must be %d (S rounded up to 8)", ld_attn, P.ldP);
  MBS_REQUIRE(0 <= layer_lo && layer_lo <= layer_hi && layer_hi <= m->n_layer, MB200_E_ARG,
              "gptj_sched_backward: bad layer range [%d,%d)", layer_lo, layer_hi);
  MBS_REQUIRE(!dlg || (dcomb && ld_dlg >= m->vocab), MB200_E_ARG,
              "gptj_sched_backward_range_logits: dlogits needs ld_dlogits=%lld >= vocab=%d and a dlogits_comb buffer",
              ld_dlg, m->vocab);
  const int M = P.M, d = P.d, dff = P.dff, H = P.H, hd = P.hd;
  ScratchScope scratch(P.gemm_ws, P.gemm_ws_bytes);
  // gradient w.r.t. the residual stream entering layer l lives in g[(l) & 1]
  bf16s* gb[2] = {P.g0, P.g1};
  if (layer_hi == m->n_layer) {  // dxf = loss_scale * dlogits Wlm ; g = LN_f backward
    const mb200_gptj_lm_grads* G = m->lm_grads;
    const bool head_trains = G && (G->w_lm || G->b_lm);
    const bf16s* dhf = dhid ? dhid[m->n_layer] : nullptr;
    const bf16s* dxf = P.dh;
    if (logits_grad && !dlg && loss_scale == 0.f) {  // nothing reaches the LM head
      if (dhf) dxf = dhf;
      else MBS_TRY(rt_zero(P.dh, (size_t)M * d * sizeof(bf16s), st));
      if (head_trains && !acc) {
        if (G->w_lm) MBS_TRY(rt_zero(G->w_lm, (size_t)m->vocab * d * sizeof(float), st));
        if (G->b_lm) MBS_TRY(rt_zero(G->b_lm, (size_t)m->vocab * sizeof(float), st));
      }
    } else {
      Epi e;
      e.alpha = loss_scale;
      if (dhf) {
        e.res1 = dhf;
        e.ld_res = d;
      }
      const bf16s* dl = P.dlogits;
      if (dlg) {  // dcomb = loss_scale * dlogits + dlg, read with alpha 1
        MBS_REQUIRE(mb200_logits_grad_combine, MB200_E_ARG, "gptj_sched: mb200_logits_grad_combine is not in this build");
        MBS_TRY(mb200_logits_grad_combine(loss_scale != 0.f ? P.dlogits : nullptr, P.ldv, dlg, ld_dlg, dcomb, M, m->vocab,
                                          loss_scale, st));
        dl = dcomb;
        e.alpha = 1.f;
      } else if (head_trains) {  // dcomb = loss_scale * dlogits, formed as (loss_scale - 1) * dlogits + dlogits
        MBS_REQUIRE(dcomb, MB200_E_ARG,
                    "gptj_sched_backward: a trainable LM head needs the dlogits_comb buffer of the _logits entry points");
        MBS_REQUIRE(mb200_logits_grad_combine, MB200_E_ARG, "gptj_sched: mb200_logits_grad_combine is not in this build");
        MBS_TRY(mb200_logits_grad_combine(P.dlogits, P.ldv, P.dlogits, P.ldv, dcomb, M, m->vocab, loss_scale - 1.f, st));
        dl = dcomb;
        e.alpha = 1.f;
      }
      MBS_TRY(gemm(st, M, d, m->vocab, mat(dl, P.ldv), wmat(m->w_lm, d, 1), P.dh, d, 0, e));
      if (head_trains && G->w_lm) MBS_TRY(wgrad(st, m->vocab, d, M, dl, P.ldv, P.xf_ln, d, G->w_lm, d, acc));  // dl^T xf
      if (head_trains && G->b_lm) MBS_TRY(mb200_colsum(dl, P.ldv, M, m->vocab, G->b_lm, acc, st));
    }
    MBS_TRY(mb200_layernorm_bwd(dxf, d, P.x_final, d, m->lnf_g, P.lnf_mean, P.lnf_rstd, nullptr, 0, gb[m->n_layer & 1], d,
                                M, d, st));
    if (G) MBS_TRY(ln_param_grad(st, P, dxf, P.x_final, P.lnf_mean, P.lnf_rstd, G->lnf_g, G->lnf_b, acc));
  }
  for (int l = layer_hi - 1; l >= layer_lo; --l) {
    if (recompute) MBS_TRY(layer_fwd(m, P, l, P.dh, st));
    const mb200_gptj_layer_ex& L = m->layers[l];
    LayerActs& a = P.acts[l];
    const bf16s* g = gb[(l + 1) & 1];
    bf16s* gout = (l == 0 && dx) ? dx : gb[l & 1];
    const bf16s* dh_acc = nullptr;  // running sum of gradients w.r.t. h = ln_1 output
    // ---- MLP branch ----
    const bf16s* dm = g;
    if (m->mlp_adapter == MB200_ADAPTER_NORMAL) {
      MBS_TRY(adapter_bwd(st, L.mlp_ad, a.am, P, M, d, m->mlp_adapter_r, g, a.mlp_out, P.dm, g, acc, m->adapter_act));
      dm = P.dm;
    } else if (m->mlp_adapter == MB200_ADAPTER_PARALLEL) {
      MBS_TRY(adapter_bwd(st, L.mlp_ad, a.am, P, M, d, m->mlp_adapter_r, g, a.h, P.dm, nullptr, acc, m->adapter_act));
      dh_acc = P.dm;
    }
    {
      Epi e;
      e.dact = MB200_DACT_GELU_NEW;
      e.aux_in = a.pre;
      MBS_TRY(gemm(st, M, dff, d, mat(dm, d), wmat(L.w_fc_out, dff, 1), P.dhact, dff, 0, e));
      Epi e2;
      e2.res1 = dh_acc;
      e2.ld_res = d;
      MBS_TRY(gemm(st, M, d, dff, mat(P.dhact, dff), wmat(L.w_fc_in, d, 1), P.dh_mlp, d, 0, e2));
      dh_acc = P.dh_mlp;
    }
    // ---- attention branch ----
    const bf16s* da = g;
    if (m->attn_adapter == MB200_ADAPTER_NORMAL) {
      MBS_TRY(adapter_bwd(st, L.attn_ad, a.aa, P, M, d, m->attn_adapter_r, g, a.a_out, P.da, g, acc, m->adapter_act));
      da = P.da;
    } else if (m->attn_adapter == MB200_ADAPTER_PARALLEL) {
      MBS_TRY(adapter_bwd(st, L.attn_ad, a.aa, P, M, d, m->attn_adapter_r, g, a.h, P.dhp, dh_acc, acc, m->adapter_act));
      dh_acc = P.dhp;
    }
    MBS_TRY(gemm(st, M, d, d, mat(da, d), wmat(L.w_out, d, 1), P.dattn_o, d, 0));  // d(attn_o) = da Wo
    const bf16s* dPe = dattn ? dattn[l] : nullptr;
    if (tile_ok(S, hd) && dPe) {
      MBS_REQUIRE(mb200_attn_bwd_tile_dp, MB200_E_ARG, "gptj_sched: mb200_attn_bwd_tile_dp is not in this build");
      MBS_TRY(mb200_attn_bwd_tile_dp(a.qkv, 3 * d, P.dattn_o, d, a.P, P.ldP, dPe, ld_attn, P.dqkv, 3 * d, P.rope_tab,
                                     m->rotary_dim, B, S, H, hd, st));
    } else if (tile_ok(S, hd)) {
      MBS_TRY(mb200_attn_bwd_tile(a.qkv, 3 * d, P.dattn_o, d, a.P, P.ldP, P.dqkv, 3 * d, P.rope_tab, m->rotary_dim, B, S, H,
                                  hd, st));
    } else {  // dQ, dK w.r.t. the rotated q, k: inverse rotation in the epilogue
      MBS_TRY(attn_bwd_gemm(st, a.qkv, a.P, P.dattn_o, P.dqkv, P.scores, P.dS, P.ldP, S, H, B, hd,
                            rope_epi(P.rope_tab, -1, S, hd, m->rotary_dim, hd), dPe));
    }
    {
      Epi e;
      e.res1 = dh_acc;
      e.ld_res = d;
      MBS_TRY(gemm(st, M, d, 3 * d, mat(P.dqkv, 3 * d), wmat(L.w_qkv, d, 1), P.dh, d, 0, e));  // dh = dqkv Wqkv + ...
    }
    MBS_TRY(mb200_layernorm_bwd(P.dh, d, a.x_in, d, L.ln1_g, a.mean, a.rstd, g, d, gout, d, M, d, st));
    if (dhid && dhid[l]) MBS_TRY(mb200_add(gout, dhid[l], nullptr, gout, (int64_t)M * d, st));
    if (const mb200_gptj_layer_grads* G = layer_grads(m, l)) {  // the block's own weights: dW = dy^T x of each linear
      if (G->w_qkv) MBS_TRY(wgrad(st, 3 * d, d, M, P.dqkv, 3 * d, a.h, d, G->w_qkv, d, acc));
      if (G->w_out) MBS_TRY(wgrad(st, d, d, M, da, d, a.attn_o, d, G->w_out, d, acc));
      if (G->w_fc_in) MBS_TRY(wgrad(st, dff, d, M, P.dhact, dff, a.h, d, G->w_fc_in, d, acc));
      if (G->b_fc_in) MBS_TRY(mb200_colsum(P.dhact, dff, M, dff, G->b_fc_in, acc, st));
      if (G->w_fc_out) MBS_TRY(wgrad(st, d, dff, M, dm, d, a.hact, dff, G->w_fc_out, dff, acc));
      if (G->b_fc_out) MBS_TRY(mb200_colsum(dm, d, M, d, G->b_fc_out, acc, st));
      MBS_TRY(ln_param_grad(st, P, P.dh, a.x_in, a.mean, a.rstd, G->ln1_g, G->ln1_b, acc));
    }
  }
  return 0;
}

// The hidden states of the forward recorded in `ws` (GPTNeoModel.forward's all_hidden_states): entry l < n_layer is
// layer l's input, entry n_layer the ln_f output. Both stay in the workspace until the next forward, on either path.
int hidden_states(const mb200_gptj_model_ex* m, bf16s* const* hid, int B, int S, void* ws, size_t ws_bytes, void* st,
                  bool recompute) {
  Plan P;
  MBS_TRY(make_plan(P, m, B, S, ws, recompute));
  MBS_REQUIRE(ws != nullptr && ws_bytes >= P.bytes, MB200_E_ARG, "gptj_sched_hidden_states: workspace too small");
  MBS_REQUIRE(hid != nullptr, MB200_E_ARG, "gptj_sched_hidden_states: hidden is NULL");
  const size_t bytes = (size_t)P.M * P.d * sizeof(bf16s);
  for (int l = 0; l <= m->n_layer; ++l)
    if (hid[l]) MBS_TRY(rt_copy(hid[l], l < m->n_layer ? P.acts[l].x_in : P.xf_ln, bytes, st));
  return 0;
}

// ---------------------------------------------------------------------------------------------
// inference (no saved activations): full sequence, prefill into a KV cache, or one decode step
// ---------------------------------------------------------------------------------------------
struct InferPlan {
  int M, d, dff, H, hd, ldS;
  bf16s *xa, *xb, *h, *qkv, *P, *attn_o, *hact, *ax, *a_out, *mlp_out, *xf_ln;
  AdapterActs am, aa;
  float *scores, *rope_tab, *splitk;
  size_t splitk_bytes, bytes;
};

int make_infer_plan(InferPlan& P, const mb200_gptj_model_ex* m, int B, int S, int Skv, void* ws) {
  Plan chk;  // same validation as the training plan
  MBS_TRY(make_plan(chk, m, B, S, nullptr));
  Carver c(ws);
  P.M = B * S;
  P.d = m->d;
  P.dff = m->d_ff;
  P.H = m->n_head;
  P.hd = m->d / m->n_head;
  const int Sk = Skv > S ? Skv : S;
  P.ldS = (int)align_up(Sk, 8);
  // the fp32 score / bf16 probability buffers only exist for head dims the fused attention kernels do not take
  const size_t M = P.M, d = P.d, dff = P.dff, nP = flash_ok(P.hd) ? 8 : (size_t)B * P.H * S * P.ldS;
  P.xa = c.take<bf16s>(M * d);
  P.xb = c.take<bf16s>(M * d);
  P.h = c.take<bf16s>(M * d);
  P.qkv = c.take<bf16s>(M * 3 * d);
  P.P = c.take<bf16s>(nP);
  P.attn_o = c.take<bf16s>(M * d);
  P.hact = c.take<bf16s>(M * dff);
  P.ax = c.take<bf16s>(M * d);
  P.a_out = c.take<bf16s>(M * d);
  P.mlp_out = c.take<bf16s>(M * d);
  P.xf_ln = c.take<bf16s>(M * d);
  carve_adapter(c, P.am, m->layers[0].mlp_ad, m->mlp_adapter, M, d, m->mlp_adapter_r, m->adapter_act, false);
  carve_adapter(c, P.aa, m->layers[0].attn_ad, m->attn_adapter, M, d, m->attn_adapter_r, m->adapter_act, false);
  P.am.mean = P.am.rstd = P.aa.mean = P.aa.rstd = nullptr;  // no backward: LayerNorm statistics are not kept
  P.scores = c.take<float>(nP);
  P.rope_tab = c.take<float>((size_t)S * m->rotary_dim);
  P.splitk_bytes = M <= 128 ? (size_t)16 * M * d * sizeof(float) : kGemmScratchBytes;
  P.splitk = P.splitk_bytes ? c.take<float>(P.splitk_bytes / sizeof(float)) : nullptr;
  P.bytes = align_up(c.off, 256);
  return 0;
}

// pos_dev != NULL: decode step (S == 1) whose cache position is read from DEVICE memory by the kernels that need it
// (rotary table, fused cache attention) — nothing in the launch sequence depends on the position, so the whole step can
// be captured once in a CUDA graph and replayed per token (pos0 is ignored).
// hidden_all != NULL: n_layer + 1 hidden states of the S positions of this call, entry l at hidden_all + l * ld_hidden:
// x, the outputs of blocks 0 .. n_layer-2 (each block writes its output there directly) and ln_f of the last block's
// output over all S rows, also when last_only projects the last row alone.
// attn != NULL: n_layer pointers, each NULL or bf16 [B,H,S,ld_attn] (ld_attn >= Sk = pos0 + S and % 8), which receive
// the probabilities each block multiplies V with: the fused kernels and the softmax write them there in place of
// their own buffer, a decode step through mb200_attn_decode_probs.
int forward_infer(const mb200_gptj_model_ex* m, const bf16s* x, bf16s* logits, long long ldv, int last_only, bf16s* hidden,
                  bf16s* kcache, bf16s* vcache, int Smax, int pos0, int B, int S, void* ws, size_t ws_bytes, void* st,
                  const int32_t* pos_dev = nullptr, bf16s* hidden_all = nullptr, long long ld_hidden = 0,
                  bf16s* const* attn = nullptr, long long ld_attn = 0) {
  InferPlan P;
  MBS_TRY(make_infer_plan(P, m, B, S, kcache ? Smax : S, ws));
  MBS_REQUIRE(ws != nullptr && ws_bytes >= P.bytes, MB200_E_ARG, "gptj_sched_infer: workspace too small (%zu < %zu)",
              ws_bytes, P.bytes);
  MBS_REQUIRE((kcache == nullptr) == (vcache == nullptr), MB200_E_ARG, "gptj_sched_infer: kcache and vcache go together");
  MBS_REQUIRE(!pos_dev || (kcache && S == 1), MB200_E_ARG, "gptj_sched_decode_step: needs a KV cache and S == 1");
  if (pos_dev) pos0 = 0;
  MBS_REQUIRE(pos0 >= 0 && (kcache ? pos0 + S <= Smax : pos0 == 0), MB200_E_SHAPE,
              "gptj_sched_infer: pos0=%d S=%d does not fit the cache (%d) / needs a cache", pos0, S, Smax);
  for (int l = 1; l < m->n_layer; ++l)
    MBS_REQUIRE(has_ln(m->layers[l].mlp_ad) == has_ln(m->layers[0].mlp_ad) &&
                    has_scale(m->layers[l].mlp_ad) == has_scale(m->layers[0].mlp_ad) &&
                    has_ln(m->layers[l].attn_ad) == has_ln(m->layers[0].attn_ad) &&
                    has_scale(m->layers[l].attn_ad) == has_scale(m->layers[0].attn_ad),
                MB200_E_ARG, "gptj_sched_infer: every layer must carry the same adapter options");
  const int M = P.M, d = P.d, dff = P.dff, H = P.H, hd = P.hd;
  MBS_REQUIRE(!hidden_all || (ld_hidden >= (long long)M * d && ld_hidden % 8 == 0), MB200_E_ALIGN,
              "gptj_sched_infer_hidden: ld_hidden=%lld must be >= B*S*d and %%8", ld_hidden);
  const int Sk = kcache ? pos0 + S : S;
  MBS_REQUIRE(!attn || (!pos_dev && ld_attn >= Sk && ld_attn % 8 == 0), MB200_E_ALIGN,
              "gptj_sched_infer_attn: ld_attn=%lld must be >= %d and %%8", ld_attn, Sk);
  const size_t cache_layer = (size_t)B * H * Smax * hd;
  ScratchScope scratch(P.splitk, P.splitk_bytes);
  if (pos_dev) MBS_TRY(mb200_rope_table_dev(P.rope_tab, S, m->rotary_dim, pos_dev, st));
  else MBS_TRY(mb200_rope_table(P.rope_tab, S, m->rotary_dim, pos0, st));
  if (hidden_all) MBS_TRY(rt_copy(hidden_all, x, (size_t)M * d * sizeof(bf16s), st));
  const bf16s* xin = x;
  for (int l = 0; l < m->n_layer; ++l) {
    const mb200_gptj_layer_ex& L = m->layers[l];
    bf16s* xout = (l & 1) ? P.xb : P.xa;
    if (hidden_all && l + 1 < m->n_layer) xout = hidden_all + (size_t)(l + 1) * ld_hidden;
    MBS_TRY(mb200_layernorm_fwd(xin, d, L.ln1_g, L.ln1_b, P.h, d, nullptr, nullptr, M, d, m->ln_eps, st));
    MBS_TRY(gemm(st, M, 3 * d, d, mat(P.h, d), wmat(L.w_qkv, d), P.qkv, 3 * d, 0,
                 rope_epi(P.rope_tab, 1, S, hd, m->rotary_dim, 2 * d)));
    bf16s* kc = kcache ? kcache + (size_t)l * cache_layer : nullptr;
    bf16s* vc = vcache ? vcache + (size_t)l * cache_layer : nullptr;
    bf16s* Pl = attn ? attn[l] : nullptr;  // this block's probabilities, when asked for
    if (kcache && S == 1 && pos_dev) {
      MBS_TRY(mb200_attn_decode_dev(P.qkv, 3 * d, kc, vc, P.attn_o, d, B, H, hd, Smax, pos_dev, st));
    } else if (kcache && S == 1 && Pl) {
      MBS_REQUIRE(mb200_attn_decode_probs, MB200_E_ARG, "gptj_sched: mb200_attn_decode_probs is not in this build");
      MBS_TRY(mb200_attn_decode_probs(P.qkv, 3 * d, kc, vc, P.attn_o, d, Pl, ld_attn, B, H, hd, Smax, pos0, st));
    } else if (kcache && S == 1) {
      MBS_TRY(mb200_attn_decode(P.qkv, 3 * d, kc, vc, P.attn_o, d, B, H, hd, Smax, pos0, st));
    } else if (flash_ok(hd)) {  // prompts of any length and prefill continuations: fused forward over qkv or the cache
      const long long qb0 = hd, qb1 = (long long)S * 3 * d;
      if (kcache) {
        MBS_TRY(mb200_kv_append(P.qkv, 3 * d, kc, vc, B, S, H, hd, Smax, pos0, st));
        const long long cb0 = (long long)Smax * hd, cb1 = (long long)H * Smax * hd;
        MBS_TRY(mb200_attn_fwd_flash(P.qkv, 3 * d, qb0, qb1, kc, hd, cb0, cb1, vc, hd, cb0, cb1, P.attn_o, d, Pl,
                                     Pl ? ld_attn : 0, nullptr, B, S, Sk, H, hd, 1, st));
      } else {
        MBS_TRY(mb200_attn_fwd_flash(P.qkv, 3 * d, qb0, qb1, P.qkv + d, 3 * d, qb0, qb1, P.qkv + 2 * d, 3 * d, qb0, qb1,
                                     P.attn_o, d, Pl, Pl ? ld_attn : 0, nullptr, B, S, S, H, hd, 1, st));
      }
    } else {
      Mat Q = mat(P.qkv, 3 * d, 0, hd, (long long)S * 3 * d), Kk, Vv;
      if (kcache) {
        MBS_TRY(mb200_kv_append(P.qkv, 3 * d, kc, vc, B, S, H, hd, Smax, pos0, st));
        Kk = mat(kc, hd, 0, (long long)Smax * hd, (long long)H * Smax * hd);
        Vv = mat(vc, hd, 1, (long long)Smax * hd, (long long)H * Smax * hd);
      } else {
        Kk = mat(P.qkv + d, 3 * d, 0, hd, (long long)S * 3 * d);
        Vv = mat(P.qkv + 2 * d, 3 * d, 1, hd, (long long)S * 3 * d);
      }
      MBS_TRY(attn_fwd_gemm(st, Q, Kk, Vv, S, Sk, H, B, hd, P.scores, Pl ? Pl : P.P, P.ldS, P.attn_o, d, 1, Sk - S,
                            Pl ? (int)ld_attn : 0));
    }
    if (m->attn_adapter == MB200_ADAPTER_NONE) {
      Epi e;
      e.res1 = xin;
      e.ld_res = d;
      MBS_TRY(gemm(st, M, d, d, mat(P.attn_o, d), wmat(L.w_out, d), P.ax, d, 0, e));
    } else if (m->attn_adapter == MB200_ADAPTER_NORMAL) {
      MBS_TRY(gemm(st, M, d, d, mat(P.attn_o, d), wmat(L.w_out, d), P.a_out, d, 0));
      MBS_TRY(adapter_fwd(st, L.attn_ad, P.aa, M, d, m->attn_adapter_r, m->ln_eps, P.a_out, P.ax, P.a_out, xin, m->adapter_act));
    } else {
      Epi e;
      e.res1 = xin;
      e.ld_res = d;
      MBS_TRY(gemm(st, M, d, d, mat(P.attn_o, d), wmat(L.w_out, d), P.a_out, d, 0, e));
      MBS_TRY(adapter_fwd(st, L.attn_ad, P.aa, M, d, m->attn_adapter_r, m->ln_eps, P.h, P.ax, P.a_out, nullptr, m->adapter_act));
    }
    {
      Epi e;
      e.bias = L.b_fc_in;
      e.act = MB200_ACT_GELU_NEW;
      MBS_TRY(gemm(st, M, dff, d, mat(P.h, d), wmat(L.w_fc_in, d), P.hact, dff, 0, e));
    }
    Epi eo;
    eo.bias = L.b_fc_out;
    if (m->mlp_adapter == MB200_ADAPTER_NONE) {
      eo.res1 = P.ax;
      eo.ld_res = d;
      MBS_TRY(gemm(st, M, d, dff, mat(P.hact, dff), wmat(L.w_fc_out, dff), xout, d, 0, eo));
    } else if (m->mlp_adapter == MB200_ADAPTER_NORMAL) {
      MBS_TRY(gemm(st, M, d, dff, mat(P.hact, dff), wmat(L.w_fc_out, dff), P.mlp_out, d, 0, eo));
      MBS_TRY(adapter_fwd(st, L.mlp_ad, P.am, M, d, m->mlp_adapter_r, m->ln_eps, P.mlp_out, xout, P.mlp_out, P.ax, m->adapter_act));
    } else {
      eo.res1 = P.ax;
      eo.ld_res = d;
      MBS_TRY(gemm(st, M, d, dff, mat(P.hact, dff), wmat(L.w_fc_out, dff), P.mlp_out, d, 0, eo));
      MBS_TRY(adapter_fwd(st, L.mlp_ad, P.am, M, d, m->mlp_adapter_r, m->ln_eps, P.h, xout, P.mlp_out, nullptr, m->adapter_act));
    }
    xin = xout;
  }
  bf16s* xf = P.xf_ln;
  if (hidden_all) {
    bf16s* h_lnf = hidden_all + (size_t)m->n_layer * ld_hidden;
    MBS_TRY(mb200_layernorm_fwd(xin, d, m->lnf_g, m->lnf_b, h_lnf, d, nullptr, nullptr, M, d, m->ln_eps, st));
    if (!last_only) xf = h_lnf;  // the full-sequence logits read the ln_f entry itself
  }
  if (!logits && !hidden) return 0;
  const int rows = last_only ? B : M;
  if (last_only)
    MBS_TRY(mb200_layernorm_fwd(xin + (size_t)(S - 1) * d, (long long)S * d, m->lnf_g, m->lnf_b, P.xf_ln, d, nullptr, nullptr,
                                B, d, m->ln_eps, st));
  else if (xf == P.xf_ln)
    MBS_TRY(mb200_layernorm_fwd(xin, d, m->lnf_g, m->lnf_b, P.xf_ln, d, nullptr, nullptr, M, d, m->ln_eps, st));
  if (hidden) MBS_TRY(rt_copy(hidden, xf, (size_t)rows * d * sizeof(bf16s), st));
  if (logits) {
    MBS_REQUIRE(ldv % 8 == 0 && ldv >= m->vocab, MB200_E_ALIGN, "gptj_sched_infer: ldv=%lld must be >= vocab and %%8", ldv);
    Epi e;
    e.bias = m->b_lm;
    MBS_TRY(gemm(st, rows, m->vocab, d, mat(xf, d), wmat(m->w_lm, d), logits, ldv, 0, e));
  }
  return 0;
}

}  // namespace
}  // namespace mb200

extern "C" size_t mb200_gptj_sched_infer_workspace_bytes(const mb200_gptj_model_ex* m, int32_t B, int32_t S,
                                                         int32_t S_kv_max) {
  mb200::InferPlan P;
  if (mb200::make_infer_plan(P, m, B, S, S_kv_max, nullptr)) return 0;
  return P.bytes;
}

extern "C" int mb200_gptj_sched_infer(const mb200_gptj_model_ex* m, const void* x, void* logits, int64_t ldv,
                                      int32_t last_only, void* hidden, void* kcache, void* vcache, int32_t S_kv_max,
                                      int32_t pos0, int32_t B, int32_t S, void* ws, size_t ws_bytes, void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  return mb200::forward_infer(m, (const mb200::bf16s*)x, (mb200::bf16s*)logits, ldv, last_only, (mb200::bf16s*)hidden,
                              (mb200::bf16s*)kcache, (mb200::bf16s*)vcache, S_kv_max, pos0, B, S, ws, ws_bytes, stream);
}

extern "C" int mb200_gptj_sched_infer_hidden(const mb200_gptj_model_ex* m, const void* x, void* logits, int64_t ldv,
                                             int32_t last_only, void* hidden_all, int64_t ld_hidden, void* kcache,
                                             void* vcache, int32_t S_kv_max, int32_t pos0, int32_t B, int32_t S, void* ws,
                                             size_t ws_bytes, void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  MBS_REQUIRE(hidden_all != nullptr, MB200_E_ARG, "gptj_sched_infer_hidden: hidden_all is NULL");
  return mb200::forward_infer(m, (const mb200::bf16s*)x, (mb200::bf16s*)logits, ldv, last_only, nullptr,
                              (mb200::bf16s*)kcache, (mb200::bf16s*)vcache, S_kv_max, pos0, B, S, ws, ws_bytes, stream,
                              nullptr, (mb200::bf16s*)hidden_all, ld_hidden);
}

extern "C" int mb200_gptj_sched_infer_attn(const mb200_gptj_model_ex* m, const void* x, void* logits, int64_t ldv,
                                           int32_t last_only, void* hidden_all, int64_t ld_hidden, void* const* attn,
                                           int64_t ld_attn, void* kcache, void* vcache, int32_t S_kv_max, int32_t pos0,
                                           int32_t B, int32_t S, void* ws, size_t ws_bytes, void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  MBS_REQUIRE(attn != nullptr, MB200_E_ARG, "gptj_sched_infer_attn: attn is NULL");
  return mb200::forward_infer(m, (const mb200::bf16s*)x, (mb200::bf16s*)logits, ldv, last_only, nullptr,
                              (mb200::bf16s*)kcache, (mb200::bf16s*)vcache, S_kv_max, pos0, B, S, ws, ws_bytes, stream,
                              nullptr, (mb200::bf16s*)hidden_all, ld_hidden, (mb200::bf16s* const*)attn, ld_attn);
}

extern "C" int mb200_gptj_sched_decode_step(const mb200_gptj_model_ex* m, const void* x, void* logits, int64_t ldv,
                                            void* kcache, void* vcache, int32_t S_kv_max, const int32_t* pos_dev,
                                            int32_t B, void* ws, size_t ws_bytes, void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  MBS_REQUIRE(pos_dev != nullptr, MB200_E_ARG, "gptj_sched_decode_step: pos_dev is NULL");
  return mb200::forward_infer(m, (const mb200::bf16s*)x, (mb200::bf16s*)logits, ldv, 1, nullptr, (mb200::bf16s*)kcache,
                              (mb200::bf16s*)vcache, S_kv_max, 0, B, 1, ws, ws_bytes, stream, pos_dev);
}

extern "C" size_t mb200_gptj_sched_workspace_bytes(const mb200_gptj_model_ex* m, int32_t B, int32_t S) {
  mb200::Plan P;
  if (mb200::make_plan(P, m, B, S, nullptr)) return 0;
  return P.bytes;
}

extern "C" int mb200_gptj_sched_forward(const mb200_gptj_model_ex* m, const void* x, const int64_t* labels, void* logits,
                                        int64_t ldv, float* loss, int32_t B, int32_t S, void* ws, size_t ws_bytes,
                                        void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  return mb200::forward(m, (const mb200::bf16s*)x, labels, (mb200::bf16s*)logits, ldv, loss, B, S, ws, ws_bytes, stream,
                        false);
}

extern "C" int mb200_gptj_sched_backward(const mb200_gptj_model_ex* m, void* dx, float loss_scale, int32_t accumulate,
                                         int32_t B, int32_t S, void* ws, size_t ws_bytes, void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  return mb200::backward(m, (mb200::bf16s*)dx, nullptr, loss_scale, m ? m->n_layer : 0, 0, accumulate, B, S, ws, ws_bytes,
                         stream, false);
}

extern "C" int mb200_gptj_sched_backward_range(const mb200_gptj_model_ex* m, void* dx, float loss_scale, int32_t layer_hi,
                                               int32_t layer_lo, int32_t accumulate, int32_t B, int32_t S, void* ws,
                                               size_t ws_bytes, void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  return mb200::backward(m, (mb200::bf16s*)dx, nullptr, loss_scale, layer_hi, layer_lo, accumulate, B, S, ws, ws_bytes,
                         stream, false);
}

extern "C" int mb200_gptj_sched_hidden_states(const mb200_gptj_model_ex* m, void* const* hidden, int32_t B, int32_t S,
                                              void* ws, size_t ws_bytes, void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  return mb200::hidden_states(m, (mb200::bf16s* const*)hidden, B, S, ws, ws_bytes, stream, false);
}

extern "C" int mb200_gptj_sched_backward_range_hidden(const mb200_gptj_model_ex* m, void* dx, void* const* dhidden,
                                                      float loss_scale, int32_t layer_hi, int32_t layer_lo,
                                                      int32_t accumulate, int32_t B, int32_t S, void* ws, size_t ws_bytes,
                                                      void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  return mb200::backward(m, (mb200::bf16s*)dx, (const mb200::bf16s* const*)dhidden, loss_scale, layer_hi, layer_lo,
                         accumulate, B, S, ws, ws_bytes, stream, false);
}

extern "C" size_t mb200_gptj_sched_recompute_workspace_bytes(const mb200_gptj_model_ex* m, int32_t B, int32_t S) {
  mb200::Plan P;
  if (mb200::make_plan(P, m, B, S, nullptr, true)) return 0;
  return P.bytes;
}

extern "C" int mb200_gptj_sched_forward_recompute(const mb200_gptj_model_ex* m, const void* x, const int64_t* labels,
                                                  void* logits, int64_t ldv, float* loss, int32_t B, int32_t S, void* ws,
                                                  size_t ws_bytes, void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  return mb200::forward(m, (const mb200::bf16s*)x, labels, (mb200::bf16s*)logits, ldv, loss, B, S, ws, ws_bytes, stream,
                        true);
}

extern "C" int mb200_gptj_sched_backward_range_recompute(const mb200_gptj_model_ex* m, void* dx, float loss_scale,
                                                         int32_t layer_hi, int32_t layer_lo, int32_t accumulate,
                                                         int32_t B, int32_t S, void* ws, size_t ws_bytes, void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  return mb200::backward(m, (mb200::bf16s*)dx, nullptr, loss_scale, layer_hi, layer_lo, accumulate, B, S, ws, ws_bytes,
                         stream, true);
}

extern "C" int mb200_gptj_sched_hidden_states_recompute(const mb200_gptj_model_ex* m, void* const* hidden, int32_t B,
                                                        int32_t S, void* ws, size_t ws_bytes, void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  return mb200::hidden_states(m, (mb200::bf16s* const*)hidden, B, S, ws, ws_bytes, stream, true);
}

extern "C" int mb200_gptj_sched_backward_range_hidden_recompute(const mb200_gptj_model_ex* m, void* dx,
                                                                void* const* dhidden, float loss_scale, int32_t layer_hi,
                                                                int32_t layer_lo, int32_t accumulate, int32_t B, int32_t S,
                                                                void* ws, size_t ws_bytes, void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  return mb200::backward(m, (mb200::bf16s*)dx, (const mb200::bf16s* const*)dhidden, loss_scale, layer_hi, layer_lo,
                         accumulate, B, S, ws, ws_bytes, stream, true);
}

extern "C" int mb200_gptj_sched_forward_attn(const mb200_gptj_model_ex* m, const void* x, const int64_t* labels,
                                             void* logits, int64_t ldv, float* loss, void* const* attn, int64_t ld_attn,
                                             int32_t B, int32_t S, void* ws, size_t ws_bytes, void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  MBS_REQUIRE(attn != nullptr, MB200_E_ARG, "gptj_sched_forward_attn: attn is NULL");
  return mb200::forward(m, (const mb200::bf16s*)x, labels, (mb200::bf16s*)logits, ldv, loss, B, S, ws, ws_bytes, stream,
                        false, (mb200::bf16s* const*)attn, ld_attn);
}

extern "C" int mb200_gptj_sched_forward_attn_recompute(const mb200_gptj_model_ex* m, const void* x, const int64_t* labels,
                                                       void* logits, int64_t ldv, float* loss, void* const* attn,
                                                       int64_t ld_attn, int32_t B, int32_t S, void* ws, size_t ws_bytes,
                                                       void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  MBS_REQUIRE(attn != nullptr, MB200_E_ARG, "gptj_sched_forward_attn: attn is NULL");
  return mb200::forward(m, (const mb200::bf16s*)x, labels, (mb200::bf16s*)logits, ldv, loss, B, S, ws, ws_bytes, stream,
                        true, (mb200::bf16s* const*)attn, ld_attn);
}

extern "C" int mb200_gptj_sched_backward_range_attn(const mb200_gptj_model_ex* m, void* dx, void* const* dhidden,
                                                    void* const* dattn, int64_t ld_attn, float loss_scale,
                                                    int32_t layer_hi, int32_t layer_lo, int32_t accumulate, int32_t B,
                                                    int32_t S, void* ws, size_t ws_bytes, void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  return mb200::backward(m, (mb200::bf16s*)dx, (const mb200::bf16s* const*)dhidden, loss_scale, layer_hi, layer_lo,
                         accumulate, B, S, ws, ws_bytes, stream, false, (const mb200::bf16s* const*)dattn, ld_attn);
}

extern "C" int mb200_gptj_sched_backward_range_attn_recompute(const mb200_gptj_model_ex* m, void* dx, void* const* dhidden,
                                                              void* const* dattn, int64_t ld_attn, float loss_scale,
                                                              int32_t layer_hi, int32_t layer_lo, int32_t accumulate,
                                                              int32_t B, int32_t S, void* ws, size_t ws_bytes,
                                                              void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  return mb200::backward(m, (mb200::bf16s*)dx, (const mb200::bf16s* const*)dhidden, loss_scale, layer_hi, layer_lo,
                         accumulate, B, S, ws, ws_bytes, stream, true, (const mb200::bf16s* const*)dattn, ld_attn);
}

extern "C" int mb200_gptj_sched_backward_range_logits(const mb200_gptj_model_ex* m, void* dx, void* const* dhidden,
                                                      void* const* dattn, int64_t ld_attn, const void* dlogits,
                                                      int64_t ld_dlogits, void* dlogits_comb, float loss_scale,
                                                      int32_t layer_hi, int32_t layer_lo, int32_t accumulate, int32_t B,
                                                      int32_t S, void* ws, size_t ws_bytes, void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  return mb200::backward(m, (mb200::bf16s*)dx, (const mb200::bf16s* const*)dhidden, loss_scale, layer_hi, layer_lo,
                         accumulate, B, S, ws, ws_bytes, stream, false, (const mb200::bf16s* const*)dattn, ld_attn, true,
                         (const mb200::bf16s*)dlogits, ld_dlogits, (mb200::bf16s*)dlogits_comb);
}

extern "C" int mb200_gptj_sched_backward_range_logits_recompute(const mb200_gptj_model_ex* m, void* dx,
                                                                void* const* dhidden, void* const* dattn, int64_t ld_attn,
                                                                const void* dlogits, int64_t ld_dlogits,
                                                                void* dlogits_comb, float loss_scale, int32_t layer_hi,
                                                                int32_t layer_lo, int32_t accumulate, int32_t B,
                                                                int32_t S, void* ws, size_t ws_bytes, void* stream) {
  int rc = mb200::rt_check_arch();
  if (rc) return rc;
  return mb200::backward(m, (mb200::bf16s*)dx, (const mb200::bf16s* const*)dhidden, loss_scale, layer_hi, layer_lo,
                         accumulate, B, S, ws, ws_bytes, stream, true, (const mb200::bf16s* const*)dattn, ld_attn, true,
                         (const mb200::bf16s*)dlogits, ld_dlogits, (mb200::bf16s*)dlogits_comb);
}
