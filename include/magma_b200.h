/*
 * magma_b200 — C ABI of libmagma_b200.so
 *
 * Hopper-native (sm_90a) re-backing of the MAGMA forward/backward hot path. The reference
 * (Aleph-Alpha/magma) has no FFI layer of its own: its seams are Python factories and nn.Module
 * duck types. Each entry point below names the reference call site whose arithmetic
 * it replaces. All pointers are raw DEVICE pointers into caller-owned (PyTorch-owned) storage; the
 * library never allocates or frees tensor memory. All work is enqueued on the passed CUDA stream
 * (`void* stream` is a cudaStream_t); no entry point synchronises the device unless stated.
 *
 * Return value: 0 on success, negative MB200_E_* on failure; mb200_last_error() returns a
 * thread-local message. Nothing throws across this boundary. There is no CPU fallback: every
 * compute entry point refuses to run (MB200_E_ARCH) unless the current device is sm_90.
 */
#ifndef MAGMA_B200_H_
#define MAGMA_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MB200_VERSION 100

enum {
  MB200_OK = 0,
  MB200_E_SHAPE = -1,
  MB200_E_DTYPE = -2,
  MB200_E_ALIGN = -3,
  MB200_E_ARCH = -4,
  MB200_E_CUDA = -5,
  MB200_E_NCCL = -6,
  MB200_E_ARG = -7
};

enum { MB200_BF16 = 0, MB200_F32 = 1 };

/* epilogue activation (forward) */
enum {
  MB200_ACT_NONE = 0,
  MB200_ACT_GELU_NEW = 1,   /* GPT-J MLP: transformers/activations.py:59-66 (NewGELUActivation) */
  MB200_ACT_QUICK_GELU = 2, /* CLIP ViT MLP: x * sigmoid(1.702 x) */
  MB200_ACT_RELU = 3,       /* magma/adapters.py:11 (Adapter default activation) */
  MB200_ACT_RELU_POST = 4   /* ReLU applied AFTER the residual adds: relu(A.B + bias + res) (CLIP Bottleneck output) */
};
/* epilogue activation-derivative multiplier (backward): out = acc * f'(aux_in) */
enum {
  MB200_DACT_NONE = 0,
  MB200_DACT_GELU_NEW = 1, /* aux_in = pre-activation */
  MB200_DACT_RELU = 3      /* aux_in = relu output (or pre-activation): mask aux_in > 0 */
};

int mb200_version(void);
const char* mb200_last_error(void);
/* 0 when the current CUDA device is sm_90 (H100), MB200_E_ARCH otherwise. */
int mb200_check_device(void);
/* Limit the persistent GEMM grids to n_sms SMs (0 = all, the default; also env MB200_GEMM_SMS). Data-parallel training
 * may leave a few SMs free for NCCL's CTAs so the gradient all-reduce overlaps the backward GEMMs. Returns the limit in
 * effect. */
int mb200_set_gemm_sm_limit(int n_sms);
/* Cap the grids of the optimizer kernels (mb200_sumsq, mb200_adamw_step) at n_blocks blocks of 256 threads (0 = the
 * default, 16 blocks per SM). With 2 blocks per SM they fit in the registers a persistent GEMM CTA leaves free, so an
 * optimizer step issued on a side stream runs BESIDE the next step's frozen-encoder GEMMs instead of owning every SM
 * until it is done (B200Engine). Returns the cap in effect. */
int mb200_set_optimizer_grid(int n_blocks);
/* number of kernels this library has launched since load (bench.py reports the delta as gpu_launches). */
long long mb200_launch_count(void);
/* optional per-launch CUDA-event timing of the GEMM core (used by bench.py for the roofline numbers):
 * enable, run, then read {sum of launch durations in ms, algorithmic FLOPs, algorithmic bytes, launches}. */
int mb200_prof_enable(int on);
int mb200_prof_read(double* gemm_ms, double* gemm_flops, double* gemm_bytes, long long* gemm_launches);

/* -------------------------------------------------------------------------------------------
 * GEMM core (wgmma.mma_async + register accumulators + TMA operand staging, persistent, warp-specialised)
 *
 *   C[b][M,N] = epilogue( alpha * A[b][M,K] * B[b][N,K]^T )
 *
 * Replaces every nn.Linear / torch.matmul on the hot path: GPT-J q/k/v/out/fc_in/fc_out/lm_head
 * (site-packages/transformers/models/gptj/modeling_gptj.py:182-184,222,375-377,623), Adapter
 * down/up projections (magma/adapters.py:19-23), ImagePrefix.proj (magma/image_prefix.py:72,93),
 * CLIP-ViT linears, and their dgrad/wgrad in backward (autograd in train_loop.py:18).
 *
 * Operands are bf16. An operand with mn_major == 0 is stored [rows = M or N][K] (K contiguous);
 * with mn_major == 1 it is stored [K][M or N] (M/N contiguous) — this is what lets dgrad (dY * W)
 * and wgrad (dY^T * X) run on the original tensors without transposed copies. `ld` is the element
 * stride between stored rows, bs0/bs1 the element strides of the two batch indices.
 * Batch index z in [0, nb0*nb1) maps to (z % nb0, z / nb0).
 * Alignment: base pointers 16 B, ld and batch strides multiples of 8 elements.
 *
 * Epilogue order per element (fp32): v = alpha*acc; v += bias[n]; aux_out = v; v = act(v);
 * v *= dact'(aux_in); v += res1 + res2; (accumulate: v += C_old, f32 output only); C = v.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
  const void* ptr;
  int64_t ld;
  int64_t bs0, bs1;
  int32_t mn_major;
  int32_t static_data; /* != 0: no kernel of the surrounding stream writes this operand's memory (frozen weights).
                        * A B operand so marked has its first tiles fetched while the launch is still waiting for its
                        * programmatic dependency (PDL), i.e. under the tail of the previous kernel. 0 is always safe. */
} mb200_operand;

typedef struct {
  int32_t M, N, K;
  int32_t nb0, nb1;
  int32_t c_dtype; /* MB200_BF16 or MB200_F32 */
  mb200_operand A, B;
  void* C;
  int64_t ldc, c_bs0, c_bs1;
  float alpha;
  int32_t act;
  int32_t dact;
  int32_t accumulate;
  const void* bias;   /* bf16 [N] or NULL */
  void* aux_out;      /* bf16, same ld / batch strides as C, or NULL */
  const void* aux_in; /* bf16, same ld / batch strides as C, or NULL (required when dact != 0) */
  const void* res1;   /* bf16 [M,N], row stride ld_res, batch strides as C, or NULL */
  const void* res2;   /* bf16 [M,N], row stride ld_res, batch strides as C, or NULL */
  int64_t ld_res;
  int32_t force_bn;   /* 0 = auto tile width (and split-K plan), else 64, 128 or 256 (no split-K) — testing / tuning */
  int32_t generic_epilogue; /* non-zero: run the runtime epilogue form even when a compiled form matches — testing */
  /* fused rotary embedding (rotate_every_two, hf:gptj/modeling_gptj.py:57-67) applied to adjacent column pairs after
   * the bias: for columns c < rope_ncols with (c % rope_hd) < rope_rot, using (cos, sin) = rope_tab[row % rope_S]
   * [(c % rope_hd)/2] (fp32 pairs, mb200_rope_table). rope_mode +1 = forward, -1 = inverse; rope_tab NULL = off. */
  int32_t rope_mode;
  const void* rope_tab;
  int32_t rope_S, rope_hd, rope_rot, rope_ncols;
  /* optional split-K scratch for small-M (M <= 128, unbatched) long-K GEMMs: fp32, splits * M * round_up(N, 4) * 4
   * bytes are used (the split count adapts to the size given). Contents need no initialisation. NULL = never split. */
  void* splitk_ws;
  int64_t splitk_ws_bytes;
} mb200_gemm_args;

int mb200_gemm(const mb200_gemm_args* args, void* stream);
/* The plan of the calling thread's last successful mb200_gemm: tile width and K splits (1 = none). For tests and tools. */
int mb200_gemm_last_plan(int32_t* bn, int32_t* split_k);


/* -------------------------------------------------------------------------------------------
 * HBM-bound operators (elementwise.cu). bf16 storage, fp32 math. Row strides (`ld*`) in elements.
 * ------------------------------------------------------------------------------------------- */
/* torch.nn.LayerNorm (GPT-J ln_1/ln_f hf:gptj/modeling_gptj.py:401,573; CLIP ln_*; magma/image_prefix.py:106-107).
 * mean/rstd (fp32 [rows]) may be NULL when no backward is needed. */
int mb200_layernorm_fwd(const void* x, int64_t ldx, const void* gamma, const void* beta, void* y, int64_t ldy,
                        float* mean, float* rstd, int32_t rows, int32_t d, float eps, void* stream);
/* dx = res + dLN/dx (res may be NULL). */
int mb200_layernorm_bwd(const void* dy, int64_t lddy, const void* x, int64_t ldx, const void* gamma,
                        const float* mean, const float* rstd, const void* res, int64_t ldres, void* dx, int64_t lddx,
                        int32_t rows, int32_t d, void* stream);
int mb200_layernorm_param_grad(const void* dy, int64_t lddy, const void* x, int64_t ldx, const float* mean,
                               const float* rstd, float* dgamma, float* dbeta, int32_t rows, int32_t d,
                               int32_t accumulate, void* stream);
/* Same result for many rows (ViT training: 2056 rows per LayerNorm): (column strip) x (row chunk) grid with one
 * atomic per (column, chunk) instead of one thread per column walking every row. */
int mb200_layernorm_param_grad_rows(const void* dy, int64_t lddy, const void* x, int64_t ldx, const float* mean,
                                    const float* rstd, float* dgamma, float* dbeta, int32_t rows, int32_t d,
                                    int32_t accumulate, void* stream);
/* rotate_every_two on q,k of a fused [rows][3][H][hd] buffer (hf:gptj/modeling_gptj.py:57-67,190-207). */
int mb200_rope(void* qkv, int64_t ld, int32_t rows, int32_t S, int32_t H, int32_t hd, int32_t rot, int32_t pos0,
               int32_t inverse, void* stream);
/* (cos, sin) table fp32 [S][rot/2][2] for positions pos0 .. pos0+S-1 (create_sinusoidal_positions,
 * hf:gptj/modeling_gptj.py:47-50) consumed by the GEMM's fused rotary epilogue. */
int mb200_rope_table(float* tab, int32_t S, int32_t rot, int32_t pos0, void* stream);
/* softmax(scale*s [+ causal mask]) fp32 -> bf16 (GPTJAttention._attn, hf:gptj/modeling_gptj.py:136-147). Writes
 * columns [0, Sk) of each row (zeros beyond the causal limit); columns [Sk, ldp) are left as they are. */
int mb200_softmax_fwd(const float* s, int64_t lds, int64_t s_bs, void* p, int64_t ldp, int64_t p_bs, int32_t nz,
                      int32_t Sq, int32_t Sk, float scale, int32_t causal, int32_t koff, void* stream);
int mb200_softmax_bwd(const float* dp, int64_t lddp, int64_t dp_bs, const void* p, int64_t ldp, int64_t p_bs,
                      void* ds, int64_t ldds, int64_t ds_bs, int32_t nz, int32_t Sq, int32_t Sk, float scale,
                      void* stream);
/* magma/utils.py:334-364 build_labels — int64, bit-exact. captions [B][ldc], labels [B][S], prefix length L. */
int mb200_build_labels(const int64_t* captions, int64_t ldc, int64_t* labels, int32_t B, int32_t S, int32_t L,
                       int64_t eos, void* stream);
/* magma/magma.py:258-267: x[b,:L] = prefix[b]; x[b,L+s] = wte[captions[b,s]]. */
int mb200_embed_assemble(const int64_t* captions, int64_t ldc, const void* wte, const void* prefix, int32_t L,
                         void* x, int32_t B, int32_t S, int32_t d, int32_t vocab, void* stream);
/* word_embedding(ids) (magma/magma.py:205; sampling.py:88-90 input_ids path). */
int mb200_embed_gather(const int64_t* ids, const void* wte, void* out, int32_t n, int32_t d, int32_t vocab,
                       void* stream);
/* Backward of the two gathers above: dwte[ids[b, j]] += dy[b, j] for b < B, j < T. ids int64 [B][ld_ids]; row (b, j) of
 * dy (bf16, 16-byte aligned rows) at dy + b * dy_bs + j * lddy; dwte fp32 [vocab, d], overwritten (accumulate == 0) or
 * added to. An id outside [0, vocab) counts as 0, as the gathers read row 0 for it. The rows of one id are summed in
 * position order (b * T + j) without atomics, so the result is the same bit for bit from run to run. */
int mb200_embed_grad(const int64_t* ids, int64_t ld_ids, const void* dy, int64_t lddy, int64_t dy_bs, int32_t B, int32_t T,
                     float* dwte, int32_t vocab, int32_t d, int32_t accumulate, void* stream);
/* ForCausalLMLoss (hf:loss/loss_utils.py:28-67): shifted CE over bf16 logits [B*S][ldv], mean over the valid targets.
 * A target is valid when it lies in [0, V); every other label (-100, any other negative value, V..ldv-1 and beyond)
 * is ignored: its row gets zero loss and zero gradient and does not count in n_valid.
 * row_loss fp32 [B*S], n_valid int32 [1], loss fp32 [1] are device scratch/outputs. When dlogits != NULL it
 * receives grad_scale * dloss/dlogits (may alias logits). logits and dlogits must be 16-byte aligned. */
int mb200_cross_entropy(const void* logits, int64_t ldv, const int64_t* labels, int32_t B, int32_t S, int32_t V,
                        float* row_loss, int32_t* n_valid, float* loss, void* dlogits, float grad_scale,
                        void* stream);
int mb200_colsum(const void* x, int64_t ldx, int32_t rows, int32_t cols, float* out, int32_t accumulate,
                 void* stream);
/* nn.Dropout (magma/image_prefix.py:104); mask (1 byte/elt) is saved for backward. */
int mb200_dropout_fwd(const void* x, void* y, uint8_t* mask, int64_t n, float p, uint64_t seed, void* stream);
int mb200_dropout_apply(const void* x, const uint8_t* mask, void* y, int64_t n, float p, void* stream);
/* CLIP conv1 (stride = kernel = P, no bias) as im2col: images [B,3,R,R] -> patches [B*(R/P)^2][ldp]. */
int mb200_patchify(const void* img, void* patches, int64_t ldp, int32_t B, int32_t R, int32_t P, void* stream);
/* x[b,0] = cls + pos[0]; x[b,1+p] = pe[b,p] + pos[1+p]  (CLIP VisionTransformer.forward token assembly). */
int mb200_vit_assemble(void* x, const void* pe, const void* cls, const void* pos, int32_t B, int32_t T, int32_t w,
                       void* stream);
/* Conv-trunk encoders (CLIP ModifiedResNet behind magma/image_encoders.py:65-74), NHWC bf16 activations:
 * images [B,C<=8,H,W] -> [B,H,W,8] (zero-padded channels); 3x3 / pad 1 / stride 1|2 im2col -> [B*Ho*Wo][9*C] in
 * (kh, kw, c) column order; nn.AvgPool2d(k) -> [B,H/k,W/k,C]. C must be a multiple of 8. The convolutions themselves
 * are mb200_gemm calls with the folded BatchNorm as bias (act RELU, or RELU_POST after the residual). */
int mb200_nchw_to_nhwc8(const void* src, void* dst, int32_t B, int32_t C, int32_t H, int32_t W, void* stream);
int mb200_im2col3x3(const void* src, void* dst, int32_t B, int32_t H, int32_t W, int32_t C, int32_t stride,
                    void* stream);
int mb200_avgpool_nhwc(const void* src, void* dst, int32_t B, int32_t H, int32_t W, int32_t C, int32_t k, void* stream);
/* Conv-trunk TRAINING (freeze_img_encoder: false with a CLIP ModifiedResNet — what MAGMA_v1.yml / MAGMA_v2.yml ship):
 * BatchNorm in training mode and the convolution backward pass on NHWC bf16 activations [rows = B*H*W][C].
 *   col_moments   out1[c] = sum_r u', out2[c] = sum_r u' * v, u' = u * 1[mask > 0] (mask optional). Batch statistics with
 *                 u = v = x; the two BatchNorm-backward reductions with u = dy, v = x, mask = the ReLU output.
 *   channel_affine y = relu?(a1[c] * x1 * 1[mask > 0] + a2[c] * x2 + c0[c] + res) with fp32 per-channel coefficients
 *                 (x2 / a2, c0, mask, res optional): BatchNorm forward (+ residual + ReLU), BatchNorm backward, ReLU
 *                 backward.
 *   col2im3x3     adjoint of mb200_im2col3x3: dcols [B*Ho*Wo][9*C] -> dx [B,H,W,C].
 *   avgpool_nhwc_bwd adjoint of mb200_avgpool_nhwc: dy [B,H/k,W/k,C] -> dx [B,H,W,C]. */
int mb200_col_moments(const void* u, int64_t ldu, const void* v, int64_t ldv, const void* mask, int64_t ldm, int32_t rows,
                      int32_t cols, float* out1, float* out2, void* stream);
int mb200_channel_affine(const void* x1, const float* a1, const void* x2, const float* a2, const float* c0,
                         const void* mask, const void* res, int32_t relu, void* y, int64_t rows, int32_t C, void* stream);
/* Per-channel BatchNorm bookkeeping (one thread per channel; all arrays fp32 [C]).
 *   bn_finalize_fwd  (s1 = sum z, s2 = sum z^2 over `rows`) -> mean, rstd, scale = gamma * rstd, shift = beta - mean * scale,
 *                    and nn.BatchNorm2d's running statistics (momentum, unbiased variance; both NULL = no update).
 *   bn_bwd_coeffs    (s1 = sum dy', t = sum dy' * z) -> dgamma, dbeta (written, or added when accumulate != 0) and the
 *                    coefficients of dz = A * dy' + Bc * z + Cc for mb200_channel_affine. */
int mb200_bn_finalize_fwd(const float* s1, const float* s2, const float* gamma, const float* beta, int64_t rows, float eps,
                          float momentum, float* running_mean, float* running_var, float* mean, float* rstd, float* scale,
                          float* shift, int32_t C, void* stream);
int mb200_bn_bwd_coeffs(const float* s1, const float* t, const float* mean, const float* rstd, const float* gamma,
                        int64_t rows, float* dgamma, float* dbeta, int32_t accumulate, float* A, float* Bc, float* Cc,
                        int32_t C, void* stream);
int mb200_col2im3x3(const void* dcols, void* dx, int32_t B, int32_t H, int32_t W, int32_t C, int32_t stride, void* stream);
int mb200_avgpool_nhwc_bwd(const void* dy, void* dx, int32_t B, int32_t H, int32_t W, int32_t C, int32_t k, void* stream);
/* torch.argmax(logits.float(), -1) (magma/sampling.py:92,97): lowest index wins ties. */
int mb200_argmax(const void* x, int64_t ldx, int32_t rows, int32_t V, int64_t* out, void* stream);
/* One sampled token per row for temperature > 0 (magma/sampling.py:97-105): top_k_filter (:22-30, off when top_k == 0),
 * top_p_filter including its inverted-nucleus comparison (:7-19, off when top_p == 0; ties ordered by index = a stable
 * sort), softmax(logits / temperature) and one multinomial draw from Philox(seed, row, offset). logits bf16 or f32
 * [rows, V] with row stride ld; keep_mask (optional, [rows, V] bytes) receives 1 where a token survives both filters.
 * -0 and +0 are equal to the order (a tie, resolved by index). NaN of either sign is read as -inf (the reference's
 * torch.multinomial rejects such rows). A row with no finite entry in the top-k set has no distribution: its token is
 * rank 0 of the order (the lowest index), and keep_mask is the top-k set when top_p == 0, rank 0 alone otherwise. */
int mb200_sample(const void* logits, int32_t dtype, int64_t ld, int32_t rows, int32_t V, float temperature,
                 int32_t top_k, float top_p, uint64_t seed, uint64_t offset, int64_t* tokens, uint8_t* keep_mask,
                 void* stream);
int mb200_add(const void* a, const void* b, const void* c, void* y, int64_t n, void* stream);
/* The gradient the LM head's backward reads when a loss reads the logits: out[r, j] = alpha * dce[r, j] + g[r, j] for
 * r < M, j < V, in fp32 with one rounding to bf16. dce and out are bf16 [M, ldv] (ldv % 8 == 0, 16-byte aligned); g is
 * bf16 with unit column stride and row stride ld_g >= V, 2-byte aligned (rows read with the widest load their
 * alignment allows). Columns from V on are not written. alpha == 0 never reads dce (it may be NULL). */
int mb200_logits_grad_combine(const void* dce, int64_t ldv, const void* g, int64_t ld_g, void* out, int32_t M, int32_t V,
                              float alpha, void* stream);
/* Data-parallel gradient exchange over peer memory (stands where DeepSpeed's gradient all-reduce stood, train.py:103-111).
 * bufs[r], r < world: rank r's fp32 exchange buffer as mapped into THIS process (peer memory for r != own rank; 16-byte
 * aligned, same layout on every rank). Elements [offset, offset + n) — the calling rank's shard — are read from all
 * `world` buffers, summed in rank order and written back into all of them. The caller brackets the launches of all ranks
 * with a device-side barrier on each side. max_blocks caps the grid (0 = default). */
int mb200_peer_reduce_bcast(void* const* bufs, int32_t world, int64_t offset, int64_t n, int32_t max_blocks,
                            void* stream);

/* Fused AdamW over a flat fp32 arena (torch.optim.AdamW(betas=(0.9,0.95)) of train.py:96-101) with global-norm
 * clipping (gradient_clipping, magma/config.py:126) and refresh of the bf16 compute copy. gnorm_sq: device fp32 [1]
 * holding sum(grad^2) (mb200_sumsq accumulates into it; zero it first) or NULL for no clipping. */
int mb200_sumsq(const float* x, int64_t n, float* out, void* stream);
int mb200_adamw_step(float* master, float* grad, float* exp_avg, float* exp_avg_sq, void* shadow_bf16, int64_t n,
                     float lr, float beta1, float beta2, float eps, float weight_decay, float grad_scale,
                     const float* gnorm_sq, float max_norm, int32_t step, int32_t zero_grad, void* stream);
int mb200_cast_f32_to_bf16(const float* src, void* dst, int64_t n, void* stream);
int mb200_cast_bf16_to_f32(const void* src, float* dst, int64_t n, void* stream);

/* -------------------------------------------------------------------------------------------
 * Model-level runtime: the whole GPT-J / CLIP-ViT forward and backward scheduled in C++ (one C call per pass
 * instead of ~1000 Python-level op calls; host-only schedule files csrc/gptj_sched.cu, csrc/vit_sched.cu).
 * All weights bf16; trainable-parameter gradients fp32. Pointers not used by a configuration are NULL.
 * ------------------------------------------------------------------------------------------- */
enum { MB200_ADAPTER_NONE = 0, MB200_ADAPTER_NORMAL = 1, MB200_ADAPTER_PARALLEL = 2 };

/* CLIP VisionTransformer (openai/CLIP model.py; hf:clip/modeling_clip.py:138-219,282-386,647-694). */
typedef struct {
  const void *ln1_g, *ln1_b;
  const void* w_qkv; /* in_proj_weight [3w, w] */
  const void* b_qkv; /* [3w] */
  const void* w_out; /* [w, w] */
  const void* b_out;
  const void *ln2_g, *ln2_b;
  const void* w_fc;  /* [mlp, w] */
  const void* b_fc;
  const void* w_proj; /* [w, mlp] */
  const void* b_proj;
} mb200_vit_layer;

typedef struct {
  int32_t n_layer, width, n_head, patch, image, mlp, out_dim, _pad;
  const void* w_conv;  /* [w, 3*P*P] row stride ld_conv (padded to a multiple of 8) */
  int64_t ld_conv;
  const void* cls;     /* [w] */
  const void* pos;     /* [T, w] */
  const void *ln_pre_g, *ln_pre_b, *ln_post_g, *ln_post_b;
  const void* proj_t;  /* visual projection stored transposed: [out_dim, w] */
  const mb200_vit_layer* layers;
} mb200_vit_model;

size_t mb200_vit_workspace_bytes(const mb200_vit_model* m, int32_t B);
/* images bf16 [B,3,R,R] -> pooled features bf16 [B, out_dim] (ln_post(x[:,0]) @ proj). Inference only
 * (the encoder is frozen on the measured path: magma/magma.py:98-100). */
int mb200_vit_forward(const mb200_vit_model* m, const void* images, void* feats, int32_t B, void* ws,
                      size_t ws_bytes, void* stream);

/* ---- CLIP-ViT training (freeze_img_encoder: false — MAGMA_v1.yml:5; magma/magma.py:98-100 leaves the encoder
 * trainable, and the optimizer gives it its own learning rate, magma/utils.py:173-177). Host-only schedule in
 * csrc/vit_sched.cu over the same primitives as the inference pass; activations of every layer are kept in `ws`
 * (no recomputation: ~85 MB per ViT-L/14 layer at B = 8). Gradient buffers are fp32 with the parameter's own shape. */
typedef struct {
  float *ln1_g, *ln1_b;
  float* w_qkv; /* [3w, w] */
  float* b_qkv;
  float* w_out; /* [w, w] */
  float* b_out;
  float *ln2_g, *ln2_b;
  float* w_fc;  /* [mlp, w] */
  float* b_fc;
  float* w_proj; /* [w, mlp] */
  float* b_proj;
} mb200_vit_layer_grads;

typedef struct {
  float* w_conv; /* [w, 3*P*P] contiguous — conv1.weight.view(w, -1) */
  float* cls;    /* [w] */
  float* pos;    /* [T, w] */
  float *ln_pre_g, *ln_pre_b, *ln_post_g, *ln_post_b;
  float* proj;   /* [w, out_dim] — the parameter's own layout (not proj_t) */
  const mb200_vit_layer_grads* layers; /* host array [n_layer] */
} mb200_vit_grads;

size_t mb200_vit_train_workspace_bytes(const mb200_vit_model* m, int32_t B);
/* Same result as mb200_vit_forward, with every layer's activations saved in `ws` for mb200_vit_backward. */
int mb200_vit_forward_train(const mb200_vit_model* m, const void* images, void* feats, int32_t B, void* ws,
                            size_t ws_bytes, void* stream);
/* Backward of the pass recorded in `ws`. dfeats: bf16 [B, out_dim]. Every parameter gradient is written to `g`
 * (accumulate != 0 adds into the buffers). The gradient w.r.t. the pixels is not produced (images are data). */
int mb200_vit_backward(const mb200_vit_model* m, const mb200_vit_grads* g, const void* dfeats, int32_t accumulate,
                       int32_t B, void* ws, size_t ws_bytes, void* stream);
/* dx = dy * d/dx[x * sigmoid(1.702 x)] at x = pre (CLIP QuickGELU, backward). dx may alias dy. */
int mb200_quick_gelu_bwd(const void* dy, const void* pre, void* dx, int64_t n, void* stream);

/* ---- GPT-J + adapters (csrc/gptj_sched.cu, host-only): GPTJForCausalLM as magma/magma.py:270-274 and
 * magma/sampling.py:81-93 call it, for EVERY adapter form of the reference: normal / parallel / scaled_parallel
 * (learnable scalar adapter_scale, magma/adapters.py:57-61), each with or without the leading LayerNorm
 * (add_layernorm, adapters.py:16-17), on the MLP and / or the attention branch (magma/magma.py:102-174).
 * Block math: hf:gptj/modeling_gptj.py:400-413 (fork GPTNeoBlock with jax=True); LM head + shifted CE:
 * hf:gptj/modeling_gptj.py:573,623, hf:loss/loss_utils.py:28-67. */
/* Adapter bottleneck (magma/adapters.py:6-39): [LayerNorm ->] Linear(d,r) -> ReLU -> Linear(r,d) [* scale]. */
typedef struct {
  const void* wd; /* [r, d] bf16 */
  const void* bd;
  const void* wu; /* [d, r] */
  const void* bu;
  const void* ln_g; /* leading LayerNorm weight / bias [d] bf16, or NULL */
  const void* ln_b;
  const float* scale; /* DEVICE fp32 scalar (adapter_scale) or NULL = 1 */
  float *g_wd, *g_bd, *g_wu, *g_bu; /* fp32 gradients, parameter shapes; g_wd == NULL => adapter frozen */
  float *g_ln_g, *g_ln_b;
  float* g_scale; /* fp32 [1] */
} mb200_adapter_ex;

typedef struct {
  const void* ln1_g;
  const void* ln1_b;
  const void* w_qkv;
  const void* w_out;
  const void* w_fc_in;
  const void* b_fc_in;
  const void* w_fc_out;
  const void* b_fc_out;
  mb200_adapter_ex mlp_ad;
  mb200_adapter_ex attn_ad;
} mb200_gptj_layer_ex;

/* fp32 gradients of GPT-J's own weights (freeze_lm: false, or any subset of them), each with its parameter's shape. A
 * NULL entry is a frozen parameter; the training backward writes (accumulate == 0) or adds into every other one. */
typedef struct {
  float *ln1_g, *ln1_b;
  float* w_qkv; /* [3d, d]: q, k and v train together */
  float* w_out;
  float *w_fc_in, *b_fc_in;
  float *w_fc_out, *b_fc_out;
} mb200_gptj_layer_grads;

/* The word embedding's gradient is not here: the pass never sees the token ids. The caller scatters the input
 * gradient dx into it with mb200_embed_grad. */
typedef struct {
  const mb200_gptj_layer_grads* layers; /* host array [n_layer], or NULL when no block parameter trains */
  float *lnf_g, *lnf_b;
  float *w_lm, *b_lm; /* a trainable LM head needs the dlogits_comb buffer of the _logits backward entry points */
} mb200_gptj_lm_grads;

typedef struct {
  int32_t n_layer, d, n_head, rotary_dim;
  int32_t vocab;
  int32_t d_ff;
  int32_t mlp_adapter; /* MB200_ADAPTER_* */
  int32_t mlp_adapter_r;
  int32_t attn_adapter;
  int32_t attn_adapter_r;
  float ln_eps;
  int32_t adapter_act; /* bottleneck activation of every adapter (magma/adapters.py:11): 0 = ReLU (the reference default),
                        * 1 = GeLU in the tanh form of the GPT-J MLP (hf:activations.py:59-66), pre-activation kept */
  const mb200_gptj_layer_ex* layers;
  const void* lnf_g;
  const void* lnf_b;
  const void* w_lm;
  const void* b_lm;
  const mb200_gptj_lm_grads* lm_grads; /* NULL: the LM is frozen (dgrad through every GEMM, wgrad for adapters only) */
} mb200_gptj_model_ex;

/* bytes of caller-provided workspace for a [B,S] training pass (per-layer activations are kept: 122 MB per GPT-J-6B
 * layer at B = 8, S = 128; nothing is recomputed — see mb200_gptj_sched_forward_recompute for the pass that
 * recomputes, as the reference's gradient checkpointing does, language_model.py:23). */
size_t mb200_gptj_sched_workspace_bytes(const mb200_gptj_model_ex* m, int32_t B, int32_t S);
/* GPTJForCausalLM.forward(inputs_embeds=x, labels=labels) as called from magma/magma.py:270-274.
 * x bf16 [B,S,d]; labels int64 [B,S] or NULL; logits bf16 [B*S][ldv] or NULL (kept in the workspace then);
 * loss fp32 [1] (device, mean CE over the valid shifted labels) when labels != NULL. Activations are saved in `ws`
 * for the backward pass. */
int mb200_gptj_sched_forward(const mb200_gptj_model_ex* m, const void* x, const int64_t* labels, void* logits,
                             int64_t ldv, float* loss, int32_t B, int32_t S, void* ws, size_t ws_bytes, void* stream);
/* Backward of the pass recorded in `ws` (loss.backward() of magma/train_loop.py:18: dgrad through every GEMM, wgrad for
 * the adapters and for every LM weight m->lm_grads names). dx: bf16 [B,S,d] gradient w.r.t. x (or NULL). accumulate != 0
 * adds into the fp32 gradient buffers (gradient accumulation), else overwrites. */
int mb200_gptj_sched_backward(const mb200_gptj_model_ex* m, void* dx, float loss_scale, int32_t accumulate, int32_t B,
                              int32_t S, void* ws, size_t ws_bytes, void* stream);

/* The same in layer ranges: layers layer_hi-1 .. layer_lo per call (LM head / CE backward when layer_hi == n_layer),
 * so the caller can exchange the gradients of finished layers while the rest runs. dx is written when layer_lo == 0. */
int mb200_gptj_sched_backward_range(const mb200_gptj_model_ex* m, void* dx, float loss_scale, int32_t layer_hi,
                                    int32_t layer_lo, int32_t accumulate, int32_t B, int32_t S, void* ws,
                                    size_t ws_bytes, void* stream);

/* The same training pass with activation recomputation, as the reference's get_gptj(gradient_checkpointing=True)
 * (language_model.py:27-37): the workspace keeps each block's input only, and the backward reruns a block's forward
 * (the same kernels in the same order, so bit-identical to what the stored path keeps) right before that block's
 * backward. Loss, logits, dx and the weight gradients equal the stored path's bit for bit; the 1-D gradients (biases,
 * LayerNorm parameters, adapter scale) are fp32 sums combined with atomics, whose last bits vary from run to run on
 * either path. The price is one more forward of the blocks. At GPT-J-6B with MLP adapters, B = 8, S = 2048, the workspace is 13.6 GiB instead of 78.6 GiB.
 * A recompute workspace pairs only with the recompute entry points: its layout differs from the stored one, and nothing
 * in it records which forward filled it. Arguments are those of mb200_gptj_sched_forward / _backward_range. */
size_t mb200_gptj_sched_recompute_workspace_bytes(const mb200_gptj_model_ex* m, int32_t B, int32_t S);
int mb200_gptj_sched_forward_recompute(const mb200_gptj_model_ex* m, const void* x, const int64_t* labels, void* logits,
                                       int64_t ldv, float* loss, int32_t B, int32_t S, void* ws, size_t ws_bytes,
                                       void* stream);
int mb200_gptj_sched_backward_range_recompute(const mb200_gptj_model_ex* m, void* dx, float loss_scale, int32_t layer_hi,
                                              int32_t layer_lo, int32_t accumulate, int32_t B, int32_t S, void* ws,
                                              size_t ws_bytes, void* stream);
/* output_hidden_states of the training pass (GPTNeoModel.forward's all_hidden_states, magma/magma.py:242,270-274):
 * copies the n_layer + 1 hidden states of the forward recorded in `ws` — entry 0 the input x, entry l the output of
 * block l (l = 1 .. n_layer-1), entry n_layer ln_f of the last block's output — to hidden[l] (bf16 [B*S, d]; a NULL
 * entry is skipped). Nothing is recomputed: the workspace holds them until the next forward. The _recompute variant takes
 * a recompute workspace. */
int mb200_gptj_sched_hidden_states(const mb200_gptj_model_ex* m, void* const* hidden, int32_t B, int32_t S, void* ws,
                                   size_t ws_bytes, void* stream);
int mb200_gptj_sched_hidden_states_recompute(const mb200_gptj_model_ex* m, void* const* hidden, int32_t B, int32_t S,
                                             void* ws, size_t ws_bytes, void* stream);
/* mb200_gptj_sched_backward_range(_recompute) of a loss that also reads those hidden states: dhidden holds n_layer + 1
 * pointers, each NULL (no gradient) or the bf16 [B*S, d] gradient of entry l. The gradient of entry l < n_layer joins the
 * residual-stream gradient where the backward crosses the input of layer l (entry 0 thus reaches dx); that of the ln_f
 * entry joins the LM head's dgrad before the ln_f backward. Each entry is added by the call whose layer range holds it.
 * With every pointer NULL the result equals mb200_gptj_sched_backward_range(_recompute). */
int mb200_gptj_sched_backward_range_hidden(const mb200_gptj_model_ex* m, void* dx, void* const* dhidden, float loss_scale,
                                           int32_t layer_hi, int32_t layer_lo, int32_t accumulate, int32_t B, int32_t S,
                                           void* ws, size_t ws_bytes, void* stream);
int mb200_gptj_sched_backward_range_hidden_recompute(const mb200_gptj_model_ex* m, void* dx, void* const* dhidden,
                                                     float loss_scale, int32_t layer_hi, int32_t layer_lo,
                                                     int32_t accumulate, int32_t B, int32_t S, void* ws, size_t ws_bytes,
                                                     void* stream);
/* output_attentions of the training pass (GPTNeoForCausalLM.forward(output_attentions=True) returns one [B, H, S, S]
 * tensor per block, the softmax probabilities that multiply V, hf:gptj/modeling_gptj.py:145-151; the adapter wrappers
 * pass them through, magma/adapters.py:85-92,109-116). mb200_gptj_sched_forward(_recompute) that also writes block l's
 * bf16 probabilities to attn[l] ([B,H,S,ld_attn], NULL entries skipped) as the block runs: zeros above the causal
 * diagonal, the values P V used. They share the layout of the saved probabilities, so ld_attn must be S rounded up to 8
 * (MB200_E_ALIGN otherwise). */
int mb200_gptj_sched_forward_attn(const mb200_gptj_model_ex* m, const void* x, const int64_t* labels, void* logits,
                                  int64_t ldv, float* loss, void* const* attn, int64_t ld_attn, int32_t B, int32_t S,
                                  void* ws, size_t ws_bytes, void* stream);
int mb200_gptj_sched_forward_attn_recompute(const mb200_gptj_model_ex* m, const void* x, const int64_t* labels,
                                            void* logits, int64_t ldv, float* loss, void* const* attn, int64_t ld_attn,
                                            int32_t B, int32_t S, void* ws, size_t ws_bytes, void* stream);
/* The backward of a loss that reads hidden states and / or attention probabilities, in one pass: dhidden as in
 * mb200_gptj_sched_backward_range_hidden (NULL, or n_layer + 1 pointers each NULL or bf16 [B*S, d]); dattn NULL, or
 * n_layer pointers each NULL or the bf16 [B,H,S,ld_attn] gradient of attn[l] (ld_attn = S rounded up to 8). Layer l's
 * attention gradient is added to dP = dO V^T before rowsum(dP * P) (mb200_attn_bwd_tile_dp for S <= 128, the dP GEMM's
 * residual otherwise), by the call whose layer range holds l. With every pointer NULL the result equals
 * mb200_gptj_sched_backward_range(_recompute). */
int mb200_gptj_sched_backward_range_attn(const mb200_gptj_model_ex* m, void* dx, void* const* dhidden, void* const* dattn,
                                         int64_t ld_attn, float loss_scale, int32_t layer_hi, int32_t layer_lo,
                                         int32_t accumulate, int32_t B, int32_t S, void* ws, size_t ws_bytes,
                                         void* stream);
int mb200_gptj_sched_backward_range_attn_recompute(const mb200_gptj_model_ex* m, void* dx, void* const* dhidden,
                                                   void* const* dattn, int64_t ld_attn, float loss_scale,
                                                   int32_t layer_hi, int32_t layer_lo, int32_t accumulate, int32_t B,
                                                   int32_t S, void* ws, size_t ws_bytes, void* stream);
/* The backward of a loss that reads the logits, and / or hidden states and attention probabilities, in one pass:
 * dhidden, dattn and ld_attn as in mb200_gptj_sched_backward_range_attn. dlogits (NULL, or bf16 [B*S, V] with unit
 * column stride and row stride ld_dlogits >= V, any 2-byte alignment) is the gradient of the logits the forward
 * returned. The call whose range holds the LM head (layer_hi == n_layer) writes loss_scale * (the cross-entropy
 * gradient the forward wrote) + dlogits into dlogits_comb (bf16 [B*S, ldv], ldv = vocab rounded up to 64, 16-byte
 * aligned; mb200_logits_grad_combine) and runs the LM head's dgrad on it, so the workspace is not written and a second
 * backward over the same forward gives the same result. Without dlogits and with loss_scale == 0 the LM head adds
 * nothing and the cross-entropy gradient is not read: the backward of a forward without labels. Otherwise, without
 * dlogits, the result equals mb200_gptj_sched_backward_range_attn(_recompute). */
int mb200_gptj_sched_backward_range_logits(const mb200_gptj_model_ex* m, void* dx, void* const* dhidden, void* const* dattn,
                                           int64_t ld_attn, const void* dlogits, int64_t ld_dlogits, void* dlogits_comb,
                                           float loss_scale, int32_t layer_hi, int32_t layer_lo, int32_t accumulate,
                                           int32_t B, int32_t S, void* ws, size_t ws_bytes, void* stream);
int mb200_gptj_sched_backward_range_logits_recompute(const mb200_gptj_model_ex* m, void* dx, void* const* dhidden,
                                                     void* const* dattn, int64_t ld_attn, const void* dlogits,
                                                     int64_t ld_dlogits, void* dlogits_comb, float loss_scale,
                                                     int32_t layer_hi, int32_t layer_lo, int32_t accumulate, int32_t B,
                                                     int32_t S, void* ws, size_t ws_bytes, void* stream);
/* Inference pass (no saved activations) — use_cache=True of magma/sampling.py:81-90: kcache / vcache bf16
 * [n_layer][B][H][S_kv_max][hd] or NULL; the K / V of this call are written at positions [pos0, pos0 + S) and attention
 * runs over [0, pos0 + S) (prefill S > 1 through mb200_attn_fwd_flash, decode S == 1 through mb200_attn_decode).
 * last_only != 0 projects the last position only (logits [B][ldv] — what magma/sampling.py:92 consumes); hidden = ln_f
 * output (bf16 [rows, d]) or NULL. */
size_t mb200_gptj_sched_infer_workspace_bytes(const mb200_gptj_model_ex* m, int32_t B, int32_t S, int32_t S_kv_max);
int mb200_gptj_sched_infer(const mb200_gptj_model_ex* m, const void* x, void* logits, int64_t ldv, int32_t last_only,
                           void* hidden, void* kcache, void* vcache, int32_t S_kv_max, int32_t pos0, int32_t B, int32_t S,
                           void* ws, size_t ws_bytes, void* stream);
/* The same pass with output_hidden_states: hidden_all receives the n_layer + 1 hidden states of the S positions of this
 * call (with a cache, the new positions only, as GPTNeoModel returns them), entry l at hidden_all + l * ld_hidden
 * elements as bf16 [B*S, d] (ld_hidden >= B*S*d and % 8): x, the outputs of blocks 1 .. n_layer-1 (each block writes
 * its output there, no copy) and ln_f of the last block's output over all S rows, also when last_only != 0 projects the
 * last position only. */
int mb200_gptj_sched_infer_hidden(const mb200_gptj_model_ex* m, const void* x, void* logits, int64_t ldv, int32_t last_only,
                                  void* hidden_all, int64_t ld_hidden, void* kcache, void* vcache, int32_t S_kv_max,
                                  int32_t pos0, int32_t B, int32_t S, void* ws, size_t ws_bytes, void* stream);
/* The inference pass with output_attentions (and, when hidden_all != NULL, output_hidden_states as above): attn holds
 * n_layer pointers, each NULL or bf16 [B,H,S,ld_attn] with ld_attn >= S_kv = pos0 + S and % 8. Block l writes the
 * probabilities it multiplies V with there — mb200_attn_fwd_flash's P output, the materialised softmax's output, or
 * mb200_attn_decode_probs for a decode step — zeros above the causal diagonal. Not available with a device-side
 * position (mb200_gptj_sched_decode_step). */
int mb200_gptj_sched_infer_attn(const mb200_gptj_model_ex* m, const void* x, void* logits, int64_t ldv, int32_t last_only,
                                void* hidden_all, int64_t ld_hidden, void* const* attn, int64_t ld_attn, void* kcache,
                                void* vcache, int32_t S_kv_max, int32_t pos0, int32_t B, int32_t S, void* ws,
                                size_t ws_bytes, void* stream);

/* Device-resident decode loop (magma/sampling.py:78-109 issues one LM call per generated token from the host and syncs
 * on `.all()` every step). Here the cache position of the step lives in DEVICE memory (pos_dev, int32[1]): no argument
 * of a decode step changes from token to token, so the caller captures ONE step in a CUDA graph — mb200_decode_embed
 * (input embedding of the token emitted last) -> mb200_gptj_sched_decode_step (= mb200_gptj_sched_infer with S = 1,
 * last_only, position read on the device) -> mb200_argmax (temperature 0) or mb200_sample_dev (temperature > 0) ->
 * mb200_decode_advance (store the new ids at column pos + 1 of the [B, ld_tok] id buffer, record whether every row
 * emitted EOS, pos += 1) — and replays it per token. Token ids are the same as the host-driven loop's (same kernels,
 * same order, same Philox offsets). */
int mb200_gptj_sched_decode_step(const mb200_gptj_model_ex* m, const void* x, void* logits, int64_t ldv, void* kcache,
                                 void* vcache, int32_t S_kv_max, const int32_t* pos_dev, int32_t B, void* ws,
                                 size_t ws_bytes, void* stream);
int mb200_decode_embed(const int64_t* tokens, int64_t ld_tok, const int32_t* pos_dev, const void* wte, void* x, int32_t B,
                       int32_t d, int32_t vocab, void* stream);
int mb200_decode_advance(const int64_t* next, int64_t* tokens, int64_t ld_tok, int32_t* pos_dev, int64_t eos,
                         uint8_t* flags, int32_t s0, int32_t n_flags, int32_t B, void* stream);
/* mb200_sample with the Philox offset read from device memory: offset = *pos_dev - s0 + 1 (as a 64-bit unsigned value),
 * one load in the kernel before the generator is seeded. pos_dev is the decode loop's int32 cache position and s0 the
 * prompt length; at decode step i >= 1 the position holds s0 + i - 1, so the offset is the step index i that the
 * host-driven loop passes to mb200_sample, and the draws are the same for the same (seed, row, offset). Same kernel,
 * arguments and checks as mb200_sample, plus pos_dev != NULL (MB200_E_ARG). */
int mb200_sample_dev(const void* logits, int32_t dtype, int64_t ld, int32_t rows, int32_t V, float temperature,
                     int32_t top_k, float top_p, uint64_t seed, const int32_t* pos_dev, int32_t s0, int64_t* tokens,
                     uint8_t* keep_mask, void* stream);
/* mb200_rope_table / mb200_attn_decode with the position read from device memory (shared memory sized for S_kv_max). */
int mb200_rope_table_dev(float* tab, int32_t S, int32_t rot, const int32_t* pos0_dev, void* stream);
int mb200_attn_decode_dev(const void* qkv, int64_t ld_qkv, void* kcache, void* vcache, void* out, int64_t ld_out,
                          int32_t B, int32_t H, int32_t hd, int32_t S_kv_max, const int32_t* pos_dev, void* stream);

/* out = s[0] * u + r1 + r2 over n bf16 elements (s: DEVICE fp32 scalar or NULL = 1; r1, r2 optional) — the
 * `* adapter_scale` of ParallelAdapter.forward (magma/adapters.py:63-66,85-92) with the residual sum folded in. */
int mb200_scale_add(const void* u, const float* s, const void* r1, const void* r2, void* out, int64_t n, void* stream);
/* out[0] (+)= sum_i a_i * b_i (fp32) over n bf16 elements — d loss / d adapter_scale. */
int mb200_dot(const void* a, const void* b, int64_t n, float* out, int32_t accumulate, void* stream);

/* Fused causal self-attention for sequences that fit one tile (S <= 128, head_dim a multiple of 64, <= 256): one CTA
 * per (batch, head), S = QK^T / softmax / PV entirely on-chip (wgmma register accumulators + smem). qkv is the fused,
 * already-rotated [B*S][3][H][hd] buffer; P (bf16 [B,H,S,ldP]) is saved for the backward pass: columns
 * [0, min(ldP, 128)) of each row are written (zeros beyond S), columns from 128 on are left as they are. O is
 * [B,S,H,hd] with row stride ldo. GPTJAttention._attn, hf:gptj/modeling_gptj.py:136-149. */
int mb200_attn_fwd_tile(const void* qkv, int64_t ld_qkv, void* P, int64_t ldP, void* O, int64_t ldo, int32_t B,
                        int32_t S, int32_t H, int32_t hd, void* stream);
/* Backward of the above: dqkv [B*S][3][H][hd] receives dQ, dK (inverse rotary applied through rope_tab, which may be
 * NULL) and dV. */
int mb200_attn_bwd_tile(const void* qkv, int64_t ld_qkv, const void* dO, int64_t ld_do, const void* P, int64_t ldP,
                        void* dqkv, int64_t ld_dqkv, const float* rope_tab, int32_t rot, int32_t B, int32_t S, int32_t H,
                        int32_t hd, void* stream);
/* mb200_attn_bwd_tile with a gradient on P from outside the block (output_attentions in training; the adapter wrappers
 * pass the probabilities on, magma/adapters.py:85-92,109-116): dP_ext, bf16 [B,H,S,ld_dpe] (ld_dpe >= S and % 8;
 * entries in rows or columns >= S are not read), is added to dP = dO V^T before dS = P * (dP - rowsum(dP * P)) /
 * sqrt(hd). A separate instantiation of the kernel; mb200_attn_bwd_tile is unchanged. */
int mb200_attn_bwd_tile_dp(const void* qkv, int64_t ld_qkv, const void* dO, int64_t ld_do, const void* P, int64_t ldP,
                           const void* dP_ext, int64_t ld_dpe, void* dqkv, int64_t ld_dqkv, const float* rope_tab,
                           int32_t rot, int32_t B, int32_t S, int32_t H, int32_t hd, void* stream);
/* The forward attention for ANY sequence length (multi-tile): one CTA per (128-query tile, head, batch) sweeps the key
 * tiles twice (row max / sum, then bf16 probabilities and O += P V in wgmma register accumulators), so no [B,H,S,S]
 * fp32 score buffer exists and the probabilities are rounded to bf16 where the materialised softmax rounds them (the
 * row sums are taken in a different order, so rare one-ulp differences remain). q / k / v point at head 0,
 * batch 0, row 0 with row stride ld*, head stride *_bsh and batch stride *_bsb in elements: the fused qkv buffer
 * (ld = 3d, bsh = hd, bsb = S * 3d) or a KV cache [B,H,Smax,hd] (ld = hd, bsh = Smax * hd, bsb = H * Smax * hd).
 * causal != 0: key j is visible to query i iff j <= i + (Sk - Sq) (prefill and its continuations). P (optional, bf16
 * [B,H,Sq,ldP], ldP >= Sk and % 8) is written for a materialised backward, every column [0, ldP) (zeros from Sk on); stats (optional, [B,H,Sq][2]) receives the
 * row maximum of the scaled scores and 1 / sum. Replaces, for S > 128 and for the ViT (T = 257), the QK^T GEMM + softmax
 * kernel + PV GEMM of hf:gptj/modeling_gptj.py:136-149 / hf:clip/modeling_clip.py:282-330 (magma/magma.py:44: the
 * reference runs at seq_len 2048). */
int mb200_attn_fwd_flash(const void* q, int64_t ldq, int64_t q_bsh, int64_t q_bsb, const void* k, int64_t ldk,
                         int64_t k_bsh, int64_t k_bsb, const void* v, int64_t ldv, int64_t v_bsh, int64_t v_bsb, void* O,
                         int64_t ldo, void* P, int64_t ldP, float* stats, int32_t B, int32_t Sq, int32_t Sk, int32_t H,
                         int32_t hd, int32_t causal, void* stream);

/* Fused KV-cache attention for one decode step (Sq = 1): q/k/v come from the fused qkv row [B][3][H][hd] (already
 * rotated); k,v are appended to the cache at position `pos`, then softmax(q K^T / sqrt(hd)) V over [0, pos]. The
 * scores live in shared memory, so pos < 51,168 (200 KB; the same limit applies to S_kv_max in mb200_attn_decode_dev).
 * Replaces the torch.cat cache growth + _attn of hf:gptj/modeling_gptj.py:209-214,136-149 per step. */
int mb200_attn_decode(const void* qkv, int64_t ld_qkv, void* kcache, void* vcache, void* out, int64_t ld_out,
                      int32_t B, int32_t H, int32_t hd, int32_t S_kv_max, int32_t pos, void* stream);
/* mb200_attn_decode that also writes the bf16 probabilities it multiplies V with to row b*H + h of probs (row stride
 * ld_probs > pos), zeros in columns pos + 1 .. ld_probs - 1: output_attentions of a decode step, the last query row of
 * hf:gptj/modeling_gptj.py:145-146 over the cache. A separate instantiation; mb200_attn_decode is unchanged. */
int mb200_attn_decode_probs(const void* qkv, int64_t ld_qkv, void* kcache, void* vcache, void* out, int64_t ld_out,
                            void* probs, int64_t ld_probs, int32_t B, int32_t H, int32_t hd, int32_t S_kv_max, int32_t pos,
                            void* stream);
/* K/V of S positions (prefill) from the fused, rotated qkv rows [B*S][3][H][hd] into one layer's static cache
 * [B][H][S_kv_max][hd] at positions [pos0, pos0 + S) — the in-place replacement of the torch.cat cache growth of
 * hf:gptj/modeling_gptj.py:209-214 for S > 1. */
int mb200_kv_append(const void* qkv, int64_t ld_qkv, void* kcache, void* vcache, int32_t B, int32_t S, int32_t H,
                    int32_t hd, int32_t S_kv_max, int32_t pos0, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MAGMA_B200_H_ */
