// magma_b200 — the C ABI of the HBM-bound kernels: argument checks, launch geometry, memsets and launch counts.
// FRAGMENT: included at file scope by elementwise.cu after the kernel fragments, and, unchanged, by
// oracle/kernel_host_exec.cpp, which runs these wrappers on the CPU. Everything the wrappers need from the host side
// goes through a few names the includer defines: launch / launch_pdl, MB_CUDA / MB_REQUIRE, check_arch,
// count_launch, num_sms, co_resident_kernels_init, cudaMemsetAsync and cudaGetLastError.

namespace mb200 {

static inline int grid_for(long long n, int threads) {
  long long g = (n + threads - 1) / threads;
  const long long cap = (long long)num_sms() * 16;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// True when every pointer (null counts as aligned) is a multiple of `bytes`, the width of the kernel's vector accesses.
template <typename... Ptr>
static inline bool aligned_to(uintptr_t bytes, const Ptr*... p) {
  return ((reinterpret_cast<uintptr_t>(p) | ... | uintptr_t{0}) & (bytes - 1)) == 0;
}

static int g_opt_grid = 0;  // mb200_set_optimizer_grid
static inline int opt_grid(int grid) { return (g_opt_grid > 0 && grid > g_opt_grid) ? g_opt_grid : grid; }

}  // namespace mb200

using namespace mb200;

extern "C" int mb200_set_optimizer_grid(int n_blocks) {
  g_opt_grid = n_blocks > 0 ? n_blocks : 0;
  return g_opt_grid;
}

#define MB_ENTER()                 \
  do {                             \
    int _rc = mb200::check_arch(); \
    if (_rc) return _rc;           \
  } while (0)
#define MB_LAUNCH_CHECK()           \
  do {                              \
    mb200::count_launch();          \
    MB_CUDA(cudaGetLastError());    \
  } while (0)
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int mb200_layernorm_fwd(const void* x, int64_t ldx, const void* gamma, const void* beta, void* y,
                                   int64_t ldy, float* mean, float* rstd, int32_t rows, int32_t d, float eps,
                                   void* stream) {
  MB_ENTER();
  MB_REQUIRE(rows > 0 && d > 0 && d % 8 == 0 && d <= kLnThreads * kLnMaxVec * 8, MB200_E_SHAPE,
             "layernorm: d=%d must be a multiple of 8 and <= %d", d, kLnThreads * kLnMaxVec * 8);
  MB_REQUIRE(ldx % 8 == 0 && ldy % 8 == 0, MB200_E_ALIGN, "layernorm: row strides must be multiples of 8");
  MB_REQUIRE(aligned_to(16, x, gamma, beta, y), MB200_E_ALIGN, "layernorm: x, gamma, beta, y must be 16-byte aligned");
  MB_CUDA(launch_pdl(layernorm_fwd_kernel, dim3(rows), dim3(kLnThreads), 0, ST(stream), (const bf16*)x, (long long)ldx,
                     (const bf16*)gamma, (const bf16*)beta, (bf16*)y, (long long)ldy, mean, rstd, (int)d, eps));
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_layernorm_bwd(const void* dy, int64_t lddy, const void* x, int64_t ldx, const void* gamma,
                                   const float* mean, const float* rstd, const void* res, int64_t ldres, void* dx,
                                   int64_t lddx, int32_t rows, int32_t d, void* stream) {
  MB_ENTER();
  MB_REQUIRE(rows > 0 && d > 0 && d % 8 == 0 && d <= kLnThreads * kLnMaxVec * 8, MB200_E_SHAPE,
             "layernorm_bwd: bad d=%d", d);
  MB_REQUIRE(lddy % 8 == 0 && ldx % 8 == 0 && lddx % 8 == 0 && (!res || ldres % 8 == 0), MB200_E_ALIGN,
             "layernorm_bwd: row strides must be multiples of 8");
  MB_REQUIRE(aligned_to(16, dy, x, gamma, res, dx), MB200_E_ALIGN,
             "layernorm_bwd: dy, x, gamma, res, dx must be 16-byte aligned");
  MB_CUDA(launch_pdl(layernorm_bwd_kernel, dim3(rows), dim3(kLnThreads), 0, ST(stream), (const bf16*)dy,
                     (long long)lddy, (const bf16*)x, (long long)ldx, (const bf16*)gamma, mean, rstd, (const bf16*)res,
                     (long long)ldres, (bf16*)dx, (long long)lddx, (int)d));
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_layernorm_param_grad(const void* dy, int64_t lddy, const void* x, int64_t ldx,
                                          const float* mean, const float* rstd, float* dgamma, float* dbeta,
                                          int32_t rows, int32_t d, int32_t accumulate, void* stream) {
  MB_ENTER();
  launch(layernorm_param_grad_kernel, (d + 127) / 128, 128, 0, ST(stream), (const bf16*)dy, lddy, (const bf16*)x, ldx,
         mean, rstd, dgamma, dbeta, rows, d, accumulate);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_layernorm_param_grad_rows(const void* dy, int64_t lddy, const void* x, int64_t ldx,
                                               const float* mean, const float* rstd, float* dgamma, float* dbeta,
                                               int32_t rows, int32_t d, int32_t accumulate, void* stream) {
  MB_ENTER();
  MB_REQUIRE(rows > 0 && d > 0 && d % 2 == 0 && lddy % 2 == 0 && ldx % 2 == 0, MB200_E_ALIGN,
             "layernorm_param_grad_rows: d and row strides must be even");
  MB_REQUIRE(aligned_to(4, dy, x), MB200_E_ALIGN, "layernorm_param_grad_rows: dy, x must be 4-byte aligned");
  {
    // many rows: 2-D decomposition with one atomic per (column, row chunk)
    if (!accumulate) {
      MB_CUDA(cudaMemsetAsync(dgamma, 0, (size_t)d * sizeof(float), ST(stream)));
      MB_CUDA(cudaMemsetAsync(dbeta, 0, (size_t)d * sizeof(float), ST(stream)));
    }
    dim3 grid((d + 63) / 64, (rows + kLnPgRows - 1) / kLnPgRows);
    launch(layernorm_param_grad_rows_kernel, grid, 256, 0, ST(stream), (const bf16*)dy, lddy, (const bf16*)x, ldx, mean,
           rstd, dgamma, dbeta, rows, d);
    MB_LAUNCH_CHECK();
  }
  return 0;
}

extern "C" int mb200_col_moments(const void* u, int64_t ldu, const void* v, int64_t ldv, const void* mask, int64_t ldm,
                                 int32_t rows, int32_t cols, float* out1, float* out2, void* stream) {
  MB_ENTER();
  MB_REQUIRE(rows > 0 && cols > 0 && cols % 2 == 0 && ldu % 2 == 0 && ldv % 2 == 0 && (!mask || ldm % 2 == 0),
             MB200_E_ALIGN, "col_moments: cols and row strides must be even");
  MB_REQUIRE(aligned_to(4, u, v, mask), MB200_E_ALIGN, "col_moments: u, v, mask must be 4-byte aligned");
  MB_CUDA(cudaMemsetAsync(out1, 0, (size_t)cols * sizeof(float), ST(stream)));
  MB_CUDA(cudaMemsetAsync(out2, 0, (size_t)cols * sizeof(float), ST(stream)));
  dim3 grid((cols + 63) / 64, (rows + kMomRows - 1) / kMomRows);
  launch(col_moments_kernel, grid, 256, 0, ST(stream), (const bf16*)u, ldu, (const bf16*)v, ldv, (const bf16*)mask, ldm,
         rows, cols, out1, out2);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_channel_affine(const void* x1, const float* a1, const void* x2, const float* a2, const float* c0,
                                    const void* mask, const void* res, int32_t relu, void* y, int64_t rows, int32_t C,
                                    void* stream) {
  MB_ENTER();
  MB_REQUIRE(rows > 0 && C > 0 && C % 8 == 0 && x1 && a1 && y && (!x2 || a2), MB200_E_ARG,
             "channel_affine: C must be a multiple of 8, x1 / a1 / y non-null, a2 given with x2");
  MB_REQUIRE(((reinterpret_cast<uintptr_t>(x1) | reinterpret_cast<uintptr_t>(x2) | reinterpret_cast<uintptr_t>(mask) |
               reinterpret_cast<uintptr_t>(res) | reinterpret_cast<uintptr_t>(y)) & 15) == 0, MB200_E_ALIGN,
             "channel_affine: pointers must be 16-byte aligned");
  launch(channel_affine_kernel, grid_for(rows * (C / 8), 256), 256, 0, ST(stream), (const bf16*)x1, a1, (const bf16*)x2,
         a2, c0, (const bf16*)mask, (const bf16*)res, relu, (bf16*)y, rows, C);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_col2im3x3(const void* dcols, void* dx, int32_t B, int32_t H, int32_t W, int32_t C, int32_t stride,
                               void* stream) {
  MB_ENTER();
  MB_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && (stride == 1 || stride == 2), MB200_E_SHAPE,
             "col2im3x3: B=%d H=%d W=%d C=%d (multiple of 8) stride=%d (1 or 2)", B, H, W, C, stride);
  MB_REQUIRE(aligned_to(16, dcols, dx), MB200_E_ALIGN, "col2im3x3: dcols, dx must be 16-byte aligned");
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  launch(col2im3x3_kernel, grid_for((long long)B * H * W * (C / 8), 256), 256, 0, ST(stream), (const bf16*)dcols,
         (bf16*)dx, B, H, W, C, stride, Ho, Wo);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_avgpool_nhwc_bwd(const void* dy, void* dx, int32_t B, int32_t H, int32_t W, int32_t C, int32_t k,
                                      void* stream) {
  MB_ENTER();
  MB_REQUIRE(B > 0 && k >= 1 && H >= k && W >= k && C > 0 && C % 8 == 0, MB200_E_SHAPE,
             "avgpool_nhwc_bwd: B=%d H=%d W=%d C=%d k=%d", B, H, W, C, k);
  MB_REQUIRE(aligned_to(16, dy, dx), MB200_E_ALIGN, "avgpool_nhwc_bwd: dy, dx must be 16-byte aligned");
  launch(avgpool_nhwc_bwd_kernel, grid_for((long long)B * H * W * (C / 8), 256), 256, 0, ST(stream), (const bf16*)dy,
         (bf16*)dx, B, H, W, C, k);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_bn_finalize_fwd(const float* s1, const float* s2, const float* gamma, const float* beta, int64_t rows,
                                     float eps, float momentum, float* running_mean, float* running_var, float* mean,
                                     float* rstd, float* scale, float* shift, int32_t C, void* stream) {
  MB_ENTER();
  MB_REQUIRE(rows > 0 && C > 0 && s1 && s2 && gamma && beta && mean && rstd && scale && shift &&
                 ((running_mean == nullptr) == (running_var == nullptr)),
             MB200_E_ARG, "bn_finalize_fwd: bad arguments");
  const float unbias = rows > 1 ? (float)((double)rows / (double)(rows - 1)) : 1.f;
  launch(bn_finalize_fwd_kernel, (C + 127) / 128, 128, 0, ST(stream), s1, s2, gamma, beta, (float)(1.0 / (double)rows),
         unbias, eps, momentum, running_mean, running_var, mean, rstd, scale, shift, C);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_bn_bwd_coeffs(const float* s1, const float* t, const float* mean, const float* rstd, const float* gamma,
                                   int64_t rows, float* dgamma, float* dbeta, int32_t accumulate, float* A, float* Bc,
                                   float* Cc, int32_t C, void* stream) {
  MB_ENTER();
  MB_REQUIRE(rows > 0 && C > 0 && s1 && t && mean && rstd && gamma && dgamma && dbeta && A && Bc && Cc, MB200_E_ARG,
             "bn_bwd_coeffs: bad arguments");
  launch(bn_bwd_coeffs_kernel, (C + 127) / 128, 128, 0, ST(stream), s1, t, mean, rstd, gamma,
         (float)(1.0 / (double)rows), dgamma, dbeta, accumulate, A, Bc, Cc, C);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_scale_add(const void* u, const float* s, const void* r1, const void* r2, void* out, int64_t n,
                               void* stream) {
  MB_ENTER();
  MB_REQUIRE(n > 0 && n % 8 == 0, MB200_E_SHAPE, "scale_add: n=%lld must be a positive multiple of 8", (long long)n);
  MB_REQUIRE(((reinterpret_cast<uintptr_t>(u) | reinterpret_cast<uintptr_t>(r1) | reinterpret_cast<uintptr_t>(r2) |
               reinterpret_cast<uintptr_t>(out)) & 15) == 0, MB200_E_ALIGN, "scale_add: pointers must be 16-byte aligned");
  launch(scale_add_kernel, grid_for(n / 8, 256), 256, 0, ST(stream), (const bf16*)u, s, (const bf16*)r1,
         (const bf16*)r2, (bf16*)out, n / 8);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_dot(const void* a, const void* b, int64_t n, float* out, int32_t accumulate, void* stream) {
  MB_ENTER();
  MB_REQUIRE(n > 0 && n % 8 == 0, MB200_E_SHAPE, "dot: n=%lld must be a positive multiple of 8", (long long)n);
  MB_REQUIRE(((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) & 15) == 0, MB200_E_ALIGN,
             "dot: pointers must be 16-byte aligned");
  if (!accumulate) MB_CUDA(cudaMemsetAsync(out, 0, sizeof(float), ST(stream)));
  const int grid = grid_for(n / 8, 256) > 1024 ? 1024 : grid_for(n / 8, 256);
  launch(dot_kernel, grid, 256, 0, ST(stream), (const bf16*)a, (const bf16*)b, n / 8, out);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_quick_gelu_bwd(const void* dy, const void* pre, void* dx, int64_t n, void* stream) {
  MB_ENTER();
  MB_REQUIRE(n > 0 && n % 8 == 0, MB200_E_SHAPE, "quick_gelu_bwd: n=%lld must be a positive multiple of 8", (long long)n);
  MB_REQUIRE(((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(pre) | reinterpret_cast<uintptr_t>(dx)) & 15) == 0,
             MB200_E_ALIGN, "quick_gelu_bwd: pointers must be 16-byte aligned");
  launch(quick_gelu_bwd_kernel, grid_for(n / 8, 256), 256, 0, ST(stream), (const bf16*)dy, (const bf16*)pre, (bf16*)dx,
         n / 8);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_rope(void* qkv, int64_t ld, int32_t rows, int32_t S, int32_t H, int32_t hd, int32_t rot,
                          int32_t pos0, int32_t inverse, void* stream) {
  MB_ENTER();
  MB_REQUIRE(rot % 2 == 0 && rot <= hd && rows > 0, MB200_E_SHAPE, "rope: bad rot=%d hd=%d", rot, hd);
  const long long total = (long long)rows * 2 * H * (rot / 2);
  launch(rope_kernel, grid_for(total, 256), 256, 0, ST(stream), (bf16*)qkv, ld, rows, S, H, hd, rot, pos0, inverse);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_rope_table(float* tab, int32_t S, int32_t rot, int32_t pos0, void* stream) {
  MB_ENTER();
  MB_REQUIRE(S > 0 && rot > 0 && rot % 2 == 0, MB200_E_SHAPE, "rope_table: bad S=%d rot=%d", S, rot);
  const int n = S * (rot / 2);
  launch(rope_table_kernel, (n + 255) / 256, 256, 0, ST(stream), reinterpret_cast<float2*>(tab), S, rot / 2, rot, pos0);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_softmax_fwd(const float* s, int64_t lds, int64_t s_bs, void* p, int64_t ldp, int64_t p_bs,
                                 int32_t nz, int32_t Sq, int32_t Sk, float scale, int32_t causal, int32_t koff,
                                 void* stream) {
  MB_ENTER();
  const long long warps = (long long)nz * Sq;
  MB_CUDA(launch_pdl(softmax_fwd_kernel, dim3((unsigned)((warps + 7) / 8)), dim3(256), 0, ST(stream), s, (long long)lds,
                     (long long)s_bs, (bf16*)p, (long long)ldp, (long long)p_bs, (int)nz, (int)Sq, (int)Sk, scale,
                     (int)causal, (int)koff));
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_softmax_bwd(const float* dp, int64_t lddp, int64_t dp_bs, const void* p, int64_t ldp,
                                 int64_t p_bs, void* ds, int64_t ldds, int64_t ds_bs, int32_t nz, int32_t Sq,
                                 int32_t Sk, float scale, void* stream) {
  MB_ENTER();
  const long long warps = (long long)nz * Sq;
  MB_CUDA(launch_pdl(softmax_bwd_kernel, dim3((unsigned)((warps + 7) / 8)), dim3(256), 0, ST(stream), dp,
                     (long long)lddp, (long long)dp_bs, (const bf16*)p, (long long)ldp, (long long)p_bs, (bf16*)ds,
                     (long long)ldds, (long long)ds_bs, (int)nz, (int)Sq, (int)Sk, scale));
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_build_labels(const int64_t* captions, int64_t ldc, int64_t* labels, int32_t B, int32_t S,
                                  int32_t L, int64_t eos, void* stream) {
  MB_ENTER();
  MB_REQUIRE(B > 0 && S > 0 && L >= 0 && L <= S, MB200_E_SHAPE, "build_labels: need 0 <= L=%d <= S=%d", L, S);
  launch(build_labels_kernel, (B * 32 + 127) / 128, 128, 0, ST(stream), (const long long*)captions, ldc,
         (long long*)labels, B, S, L, eos);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_embed_assemble(const int64_t* captions, int64_t ldc, const void* wte, const void* prefix,
                                    int32_t L, void* x, int32_t B, int32_t S, int32_t d, int32_t vocab,
                                    void* stream) {
  MB_ENTER();
  MB_REQUIRE(d % 8 == 0 && L >= 0 && L <= S, MB200_E_SHAPE, "embed_assemble: bad d=%d L=%d S=%d", d, L, S);
  MB_REQUIRE(aligned_to(16, wte, prefix, x), MB200_E_ALIGN, "embed_assemble: wte, prefix, x must be 16-byte aligned");
  launch(embed_assemble_kernel, B * S, 256, 0, ST(stream), (const long long*)captions, ldc, (const bf16*)wte,
         (const bf16*)prefix, L, (bf16*)x, B, S, d, vocab);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_embed_gather(const int64_t* ids, const void* wte, void* out, int32_t n, int32_t d,
                                  int32_t vocab, void* stream) {
  MB_ENTER();
  MB_REQUIRE(d % 8 == 0 && n > 0, MB200_E_SHAPE, "embed_gather: bad n=%d d=%d", n, d);
  MB_REQUIRE(aligned_to(16, wte, out), MB200_E_ALIGN, "embed_gather: wte, out must be 16-byte aligned");
  launch(embed_gather_kernel, n, 256, 0, ST(stream), (const long long*)ids, (const bf16*)wte, (bf16*)out, d, vocab);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_cross_entropy(const void* logits, int64_t ldv, const int64_t* labels, int32_t B, int32_t S,
                                   int32_t V, float* row_loss, int32_t* n_valid, float* loss, void* dlogits,
                                   float grad_scale, void* stream) {
  MB_ENTER();
  MB_REQUIRE(ldv % 8 == 0 && V <= ldv, MB200_E_ALIGN, "cross_entropy: ldv=%lld must be a multiple of 8 and >= V",
             (long long)ldv);
  MB_REQUIRE(aligned_to(16, logits, dlogits), MB200_E_ALIGN, "cross_entropy: logits, dlogits must be 16-byte aligned");
  launch(ce_count_kernel, 1, 1024, 0, ST(stream), (const long long*)labels, B, S, V, n_valid);
  launch(ce_row_kernel, B * S, kCeThreads, 0, ST(stream), (const bf16*)logits, ldv, (const long long*)labels, S, V,
         n_valid, row_loss, (bf16*)dlogits, grad_scale);
  launch(ce_reduce_kernel, 1, 1024, 0, ST(stream), row_loss, B * S, n_valid, loss);
  mb200::count_launch(2);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_colsum(const void* x, int64_t ldx, int32_t rows, int32_t cols, float* out, int32_t accumulate,
                            void* stream) {
  MB_ENTER();
  MB_REQUIRE(cols % 2 == 0 && ldx % 2 == 0, MB200_E_ALIGN, "colsum: cols and ldx must be even");
  MB_REQUIRE(aligned_to(4, x), MB200_E_ALIGN, "colsum: x must be 4-byte aligned");
  if (!accumulate) MB_CUDA(cudaMemsetAsync(out, 0, (size_t)cols * sizeof(float), ST(stream)));
  dim3 grid((cols + 63) / 64, (rows + kColsumRows - 1) / kColsumRows);
  MB_CUDA(launch_pdl(colsum_kernel, grid, dim3(256), 0, ST(stream), (const bf16*)x, (long long)ldx, (int)rows, (int)cols,
                     out));
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_dropout_fwd(const void* x, void* y, uint8_t* mask, int64_t n, float p, uint64_t seed,
                                 void* stream) {
  MB_ENTER();
  MB_REQUIRE(p >= 0.f && p < 1.f, MB200_E_ARG, "dropout: p=%f out of range", p);
  launch(dropout_fwd_kernel, grid_for(n, 256), 256, 0, ST(stream), (const bf16*)x, (bf16*)y, mask, n, p, seed);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_dropout_apply(const void* x, const uint8_t* mask, void* y, int64_t n, float p, void* stream) {
  MB_ENTER();
  launch(dropout_apply_kernel, grid_for(n, 256), 256, 0, ST(stream), (const bf16*)x, mask, (bf16*)y, n, p);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_patchify(const void* img, void* patches, int64_t ldp, int32_t B, int32_t R, int32_t P,
                              void* stream) {
  MB_ENTER();
  MB_REQUIRE(R % P == 0 && ldp >= 3 * P * P, MB200_E_SHAPE, "patchify: R=%d P=%d ldp=%lld", R, P, (long long)ldp);
  const long long total = (long long)B * (R / P) * (R / P) * 3 * P * P;
  launch(patchify_kernel, grid_for(total, 256), 256, 0, ST(stream), (const bf16*)img, (bf16*)patches, ldp, B, R, P);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_vit_assemble(void* x, const void* pe, const void* cls, const void* pos, int32_t B, int32_t T,
                                  int32_t w, void* stream) {
  MB_ENTER();
  launch(vit_assemble_kernel, grid_for((long long)B * T * w, 256), 256, 0, ST(stream), (bf16*)x, (const bf16*)pe,
         (const bf16*)cls, (const bf16*)pos, B, T, w);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_nchw_to_nhwc8(const void* src, void* dst, int32_t B, int32_t C, int32_t H, int32_t W,
                                   void* stream) {
  MB_ENTER();
  MB_REQUIRE(C >= 1 && C <= 8 && B > 0 && H > 0 && W > 0, MB200_E_SHAPE, "nchw_to_nhwc8: B=%d C=%d H=%d W=%d", B, C, H, W);
  MB_REQUIRE(aligned_to(16, dst), MB200_E_ALIGN, "nchw_to_nhwc8: dst must be 16-byte aligned");
  launch(nchw_to_nhwc8_kernel, grid_for((long long)B * H * W, 256), 256, 0, ST(stream), (const bf16*)src, (bf16*)dst, B,
         C, H, W);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_im2col3x3(const void* src, void* dst, int32_t B, int32_t H, int32_t W, int32_t C, int32_t stride,
                                void* stream) {
  MB_ENTER();
  MB_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && (stride == 1 || stride == 2), MB200_E_SHAPE,
             "im2col3x3: B=%d H=%d W=%d C=%d (multiple of 8) stride=%d (1 or 2)", B, H, W, C, stride);
  MB_REQUIRE(aligned_to(16, src, dst), MB200_E_ALIGN, "im2col3x3: src, dst must be 16-byte aligned");
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  const long long nvec = (long long)B * Ho * Wo * 9 * (C / 8);
  if (nvec < (1LL << 31) - (1LL << 24))  // headroom for the grid-stride increment
    launch(im2col3x3_kernel<unsigned int>, grid_for(nvec, 256), 256, 0, ST(stream), (const bf16*)src, (bf16*)dst, B, H,
           W, C, stride, Ho, Wo);
  else
    launch(im2col3x3_kernel<long long>, grid_for(nvec, 256), 256, 0, ST(stream), (const bf16*)src, (bf16*)dst, B, H, W,
           C, stride, Ho, Wo);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_avgpool_nhwc(const void* src, void* dst, int32_t B, int32_t H, int32_t W, int32_t C, int32_t k,
                                   void* stream) {
  MB_ENTER();
  MB_REQUIRE(B > 0 && k >= 1 && H >= k && W >= k && C > 0 && C % 8 == 0, MB200_E_SHAPE,
             "avgpool_nhwc: B=%d H=%d W=%d C=%d (multiple of 8) k=%d", B, H, W, C, k);
  MB_REQUIRE(aligned_to(16, src, dst), MB200_E_ALIGN, "avgpool_nhwc: src, dst must be 16-byte aligned");
  launch(avgpool_nhwc_kernel, grid_for((long long)B * (H / k) * (W / k) * (C / 8), 256), 256, 0, ST(stream),
         (const bf16*)src, (bf16*)dst, B, H, W, C, k);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_argmax(const void* x, int64_t ldx, int32_t rows, int32_t V, int64_t* out, void* stream) {
  MB_ENTER();
  MB_REQUIRE(rows > 0 && V > 0 && V <= ldx, MB200_E_SHAPE, "argmax: need rows=%d > 0 and 0 < V=%d <= ldx=%lld", rows, V,
             (long long)ldx);
  launch(argmax_kernel, rows, 512, 0, ST(stream), (const bf16*)x, ldx, V, (long long*)out);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_add(const void* a, const void* b, const void* c, void* y, int64_t n, void* stream) {
  MB_ENTER();
  MB_REQUIRE(n % 8 == 0, MB200_E_ALIGN, "add: n must be a multiple of 8");
  MB_REQUIRE(aligned_to(16, a, b, c, y), MB200_E_ALIGN, "add: a, b, c, y must be 16-byte aligned");
  launch(add_kernel, grid_for(n / 8, 256), 256, 0, ST(stream), (const bf16*)a, (const bf16*)b, (const bf16*)c, (bf16*)y,
         n / 8);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_logits_grad_combine(const void* dce, int64_t ldv, const void* g, int64_t ld_g, void* out, int32_t M,
                                         int32_t V, float alpha, void* stream) {
  MB_ENTER();
  MB_REQUIRE(M > 0 && V > 0 && V <= ldv && V <= ld_g, MB200_E_SHAPE,
             "logits_grad_combine: need M=%d > 0 and 0 < V=%d <= ldv=%lld, ld_g=%lld", M, V, (long long)ldv,
             (long long)ld_g);
  MB_REQUIRE(g && out && (dce || alpha == 0.f), MB200_E_ARG, "logits_grad_combine: g, out (and dce unless alpha == 0) are NULL");
  MB_REQUIRE(ldv % 8 == 0 && aligned_to(16, dce, out) && aligned_to(2, g), MB200_E_ALIGN,
             "logits_grad_combine: ldv must be a multiple of 8, dce and out 16-byte aligned, g 2-byte aligned");
  const int col_blocks = (V / 8 + kLgThreads * kLgChunks - 1) / (kLgThreads * kLgChunks);
  launch(logits_grad_combine_kernel, dim3((unsigned)M, col_blocks > 0 ? col_blocks : 1), kLgThreads, 0, ST(stream), (const bf16*)dce, (long long)ldv, (const bf16*)g,
         (long long)ld_g, (bf16*)out, (int)V, alpha);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_sumsq(const float* x, int64_t n, float* out, void* stream) {
  MB_ENTER();
  int grid = grid_for(n, 256);
  if (grid > kSumsqMaxBlocks) grid = kSumsqMaxBlocks;
  grid = opt_grid(grid);
  co_resident_kernels_init();
  launch(sumsq_kernel, grid, 256, 0, ST(stream), x, n, out);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_peer_reduce_bcast(void* const* bufs, int32_t world, int64_t offset, int64_t n, int32_t max_blocks,
                                       void* stream) {
  MB_ENTER();
  MB_REQUIRE(world >= 1 && world <= 16, MB200_E_ARG, "peer_reduce_bcast: world must be in [1, 16]");
  MB_REQUIRE(offset % 4 == 0 && n % 4 == 0, MB200_E_ALIGN, "peer_reduce_bcast: offset and n must be multiples of 4");
  if (n == 0) return 0;
  PeerBufs pb;
  for (int r = 0; r < 16; ++r) pb.p[r] = r < world ? reinterpret_cast<float*>(bufs[r]) : nullptr;
  for (int r = 0; r < world; ++r)
    MB_REQUIRE(pb.p[r] != nullptr && (reinterpret_cast<uintptr_t>(pb.p[r]) & 15) == 0, MB200_E_ALIGN,
               "peer_reduce_bcast: buffer %d is null or not 16-byte aligned", r);
  int grid = grid_for(n / 4, 256);
  if (max_blocks > 0 && grid > max_blocks) grid = max_blocks;
  co_resident_kernels_init();
  launch(peer_reduce_bcast_kernel, grid, 256, 0, ST(stream), pb, world, offset / 4, n / 4);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_adamw_step(float* master, float* grad, float* exp_avg, float* exp_avg_sq, void* shadow_bf16,
                                int64_t n, float lr, float beta1, float beta2, float eps, float weight_decay,
                                float grad_scale, const float* gnorm_sq, float max_norm, int32_t step,
                                int32_t zero_grad, void* stream) {
  MB_ENTER();
  MB_REQUIRE(step >= 1, MB200_E_ARG, "adamw: step must be >= 1");
  const float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
  MB_REQUIRE(n % 4 == 0, MB200_E_ALIGN, "adamw: n must be a multiple of 4 (the arena pads every tensor to 64)");
  MB_REQUIRE(aligned_to(16, master, grad, exp_avg, exp_avg_sq) && aligned_to(8, shadow_bf16), MB200_E_ALIGN,
             "adamw: master, grad, moments must be 16-byte aligned, the bf16 shadow 8-byte aligned");
  co_resident_kernels_init();
  launch(adamw_kernel, opt_grid(grid_for(n / 4, 256)), 256, 0, ST(stream), master, grad, exp_avg, exp_avg_sq,
         (bf16*)shadow_bf16, n / 4, lr, beta1, beta2, eps, weight_decay, grad_scale, gnorm_sq, max_norm, bc1, bc2,
         zero_grad);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_cast_f32_to_bf16(const float* src, void* dst, int64_t n, void* stream) {
  MB_ENTER();
  launch(cast_f32_bf16_kernel, grid_for(n, 256), 256, 0, ST(stream), src, (bf16*)dst, n);
  MB_LAUNCH_CHECK();
  return 0;
}
extern "C" int mb200_cast_bf16_to_f32(const void* src, float* dst, int64_t n, void* stream) {
  MB_ENTER();
  launch(cast_bf16_f32_kernel, grid_for(n, 256), 256, 0, ST(stream), (const bf16*)src, dst, n);
  MB_LAUNCH_CHECK();
  return 0;
}

// Device-resident decode loop: the step's cache position lives in device memory, so one CUDA graph of the whole decode
// step is replayed per token with no host-side argument changing (kernels in elt_kernels.cuh).
extern "C" int mb200_rope_table_dev(float* tab, int32_t S, int32_t rot, const int32_t* pos0_dev, void* stream) {
  MB_ENTER();
  MB_REQUIRE(S > 0 && rot > 0 && rot % 2 == 0 && pos0_dev != nullptr, MB200_E_SHAPE, "rope_table_dev: bad S=%d rot=%d", S, rot);
  const int n = S * (rot / 2);
  launch(rope_table_dev_kernel, (n + 255) / 256, 256, 0, ST(stream), reinterpret_cast<float2*>(tab), S, rot / 2, rot,
         pos0_dev);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_decode_embed(const int64_t* tokens, int64_t ld_tok, const int32_t* pos_dev, const void* wte, void* x,
                                  int32_t B, int32_t d, int32_t vocab, void* stream) {
  MB_ENTER();
  MB_REQUIRE(d % 8 == 0 && B > 0 && tokens && pos_dev, MB200_E_SHAPE, "decode_embed: bad B=%d d=%d", B, d);
  MB_REQUIRE(aligned_to(16, wte, x), MB200_E_ALIGN, "decode_embed: wte, x must be 16-byte aligned");
  launch(decode_embed_kernel, B, 256, 0, ST(stream), (const long long*)tokens, ld_tok, pos_dev, (const bf16*)wte,
         (bf16*)x, d, vocab);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_decode_advance(const int64_t* next, int64_t* tokens, int64_t ld_tok, int32_t* pos_dev, int64_t eos,
                                    uint8_t* flags, int32_t s0, int32_t n_flags, int32_t B, void* stream) {
  MB_ENTER();
  MB_REQUIRE(B > 0 && next && tokens && pos_dev, MB200_E_ARG, "decode_advance: null argument");
  launch(decode_advance_kernel, 1, 256, 0, ST(stream), (const long long*)next, (long long*)tokens, ld_tok, pos_dev,
         (long long)eos, flags, s0, n_flags, B);
  MB_LAUNCH_CHECK();
  return 0;
}

// Token sampling for temperature > 0 (kernel and method in samp_kernels.cuh). `name` prefixes the error messages; Off is
// the kernel's offset source.
template <typename Off>
static int sample_launch(const char* name, const void* logits, int32_t dtype, int64_t ld, int32_t rows, int32_t V,
                         float temperature, int32_t top_k, float top_p, uint64_t seed, Off offset, int64_t* tokens,
                         uint8_t* keep_mask, void* stream) {
  MB_REQUIRE(rows > 0 && V > 0 && ld >= V, MB200_E_SHAPE, "%s: rows=%d V=%d ld=%lld", name, rows, V, (long long)ld);
  MB_REQUIRE(temperature > 0.f, MB200_E_ARG, "%s: temperature must be > 0 (use mb200_argmax for greedy decoding)", name);
  MB_REQUIRE(top_k >= 0 && top_p >= 0.f && top_p <= 1.f, MB200_E_ARG, "%s: top_k=%d top_p=%f", name, top_k, top_p);
  MB_REQUIRE(dtype == MB200_BF16 || dtype == MB200_F32, MB200_E_DTYPE, "%s: logits must be bf16 or f32", name);
  if (dtype == MB200_F32)
    launch(sample_kernel<float, Off>, rows, kSampThreads, 0, ST(stream), (const float*)logits, ld, V, 1.f / temperature,
           top_k, top_p, seed, offset, (long long*)tokens, keep_mask);
  else
    launch(sample_kernel<bf16, Off>, rows, kSampThreads, 0, ST(stream), (const bf16*)logits, ld, V, 1.f / temperature,
           top_k, top_p, seed, offset, (long long*)tokens, keep_mask);
  MB_LAUNCH_CHECK();
  return 0;
}

extern "C" int mb200_sample(const void* logits, int32_t dtype, int64_t ld, int32_t rows, int32_t V, float temperature,
                            int32_t top_k, float top_p, uint64_t seed, uint64_t offset, int64_t* tokens,
                            uint8_t* keep_mask, void* stream) {
  MB_ENTER();
  return sample_launch<unsigned long long>("sample", logits, dtype, ld, rows, V, temperature, top_k, top_p, seed,
                                           offset, tokens, keep_mask, stream);
}

// The Philox offset is read on the device: pos_dev - s0 + 1, the decode loop's step index (DecodeOffset).
extern "C" int mb200_sample_dev(const void* logits, int32_t dtype, int64_t ld, int32_t rows, int32_t V, float temperature,
                                int32_t top_k, float top_p, uint64_t seed, const int32_t* pos_dev, int32_t s0,
                                int64_t* tokens, uint8_t* keep_mask, void* stream) {
  MB_ENTER();
  MB_REQUIRE(pos_dev != nullptr, MB200_E_ARG, "sample_dev: pos_dev is NULL");
  return sample_launch("sample_dev", logits, dtype, ld, rows, V, temperature, top_k, top_p, seed,
                       DecodeOffset{pos_dev, s0}, tokens, keep_mask, stream);
}
