// magma_b200 — the HBM-bound kernels of the hot path (LayerNorm, rotary, softmax, cross-entropy, gathers, label
// building, reductions, dropout, ViT / conv-trunk layout kernels, argmax, fused AdamW, the decode loop). FRAGMENT:
// included by elementwise.cu inside `namespace mb200` (its C ABI follows in elt_abi.cuh), and, unchanged, by
// oracle/kernel_host_exec.cpp, which executes kernel source on the CPU under an emulated thread model.

// ---------------------------------------------------------------------------------------------
// LayerNorm forward: y = (x - mean) * rstd * gamma + beta ; one CTA per row, row cached in registers.
// (torch.nn.LayerNorm in GPT-J ln_1/ln_f, CLIP ln_*, magma/image_prefix.py:106-107)
// ---------------------------------------------------------------------------------------------
static constexpr int kLnThreads = 256;
static constexpr int kLnMaxVec = 4;  // d <= 256*4*8 = 8192

__global__ void __launch_bounds__(kLnThreads)
layernorm_fwd_kernel(const bf16* __restrict__ x, long long ldx, const bf16* __restrict__ gamma,
                     const bf16* __restrict__ beta, bf16* __restrict__ y, long long ldy, float* __restrict__ mean_out,
                     float* __restrict__ rstd_out, int d, float eps) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[32];
  const long long row = blockIdx.x;
  const int nvec = d >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * ldx);
  float v[kLnMaxVec][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kLnMaxVec; ++i) {
    const int c = threadIdx.x + i * kLnThreads;
    if (c < nvec) {
      unpack8(xr[c], v[i]);
#pragma unroll
      for (int e = 0; e < 8; ++e) s += v[i][e];
    }
  }
  const float mean = block_sum<kLnThreads>(s, red) / (float)d;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < kLnMaxVec; ++i) {
    const int c = threadIdx.x + i * kLnThreads;
    if (c < nvec) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float t = v[i][e] - mean;
        q += t * t;
      }
    }
  }
  const float var = block_sum<kLnThreads>(q, red) / (float)d;
  const float rstd = rsqrtf(var + eps);
  if (threadIdx.x == 0) {
    if (mean_out) mean_out[row] = mean;
    if (rstd_out) rstd_out[row] = rstd;
  }
  uint4* yr = reinterpret_cast<uint4*>(y + row * ldy);
  const uint4* gr = reinterpret_cast<const uint4*>(gamma);
  const uint4* br = reinterpret_cast<const uint4*>(beta);
#pragma unroll
  for (int i = 0; i < kLnMaxVec; ++i) {
    const int c = threadIdx.x + i * kLnThreads;
    if (c < nvec) {
      float g[8], b[8], o[8];
      unpack8(__ldg(gr + c), g);
      unpack8(__ldg(br + c), b);
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = (v[i][e] - mean) * rstd * g[e] + b[e];
      yr[c] = pack8(o);
    }
  }
}

// LayerNorm backward (input gradient): dx = res + rstd * (g - mean(g) - xhat * mean(g * xhat)), g = dy * gamma
__global__ void __launch_bounds__(kLnThreads)
layernorm_bwd_kernel(const bf16* __restrict__ dy, long long lddy, const bf16* __restrict__ x, long long ldx,
                     const bf16* __restrict__ gamma, const float* __restrict__ mean, const float* __restrict__ rstd,
                     const bf16* __restrict__ res, long long ldres, bf16* __restrict__ dx, long long lddx, int d) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[32];
  const long long row = blockIdx.x;
  const int nvec = d >> 3;
  const uint4* dyr = reinterpret_cast<const uint4*>(dy + row * lddy);
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * ldx);
  const uint4* gr = reinterpret_cast<const uint4*>(gamma);
  const float mu = mean[row], rs = rstd[row];
  float g[kLnMaxVec][8], xh[kLnMaxVec][8];
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int i = 0; i < kLnMaxVec; ++i) {
    const int c = threadIdx.x + i * kLnThreads;
    if (c < nvec) {
      float a[8], b[8], gm[8];
      unpack8(dyr[c], a);
      unpack8(xr[c], b);
      unpack8(__ldg(gr + c), gm);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        g[i][e] = a[e] * gm[e];
        xh[i][e] = (b[e] - mu) * rs;
        s1 += g[i][e];
        s2 += g[i][e] * xh[i][e];
      }
    }
  }
  const float m1 = block_sum<kLnThreads>(s1, red) / (float)d;
  const float m2 = block_sum<kLnThreads>(s2, red) / (float)d;
  uint4* dxr = reinterpret_cast<uint4*>(dx + row * lddx);
  const uint4* rr = res ? reinterpret_cast<const uint4*>(res + row * ldres) : nullptr;
#pragma unroll
  for (int i = 0; i < kLnMaxVec; ++i) {
    const int c = threadIdx.x + i * kLnThreads;
    if (c < nvec) {
      float o[8], r[8];
      if (rr) unpack8(rr[c], r);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        o[e] = rs * (g[i][e] - m1 - xh[i][e] * m2);
        if (rr) o[e] += r[e];
      }
      dxr[c] = pack8(o);
    }
  }
}

// LayerNorm parameter gradients for a (small) number of rows: dgamma[c] (+)= sum_r dy*xhat, dbeta[c] (+)= sum_r dy
__global__ void layernorm_param_grad_kernel(const bf16* __restrict__ dy, long long lddy, const bf16* __restrict__ x,
                                            long long ldx, const float* __restrict__ mean,
                                            const float* __restrict__ rstd, float* __restrict__ dgamma,
                                            float* __restrict__ dbeta, int rows, int d, int accumulate) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= d) return;
  float sg = 0.f, sb = 0.f;
  for (int r = 0; r < rows; ++r) {
    const float g = __bfloat162float(dy[(long long)r * lddy + c]);
    const float xh = (__bfloat162float(x[(long long)r * ldx + c]) - mean[r]) * rstd[r];
    sg += g * xh;
    sb += g;
  }
  dgamma[c] = accumulate ? dgamma[c] + sg : sg;
  dbeta[c] = accumulate ? dbeta[c] + sb : sb;
}

// ---------------------------------------------------------------------------------------------
// Rotary embedding, in place on the fused qkv buffer [rows = B*S][3][H][hd] (q and k, first rot dims of each
// head; interleaved pairs — rotate_every_two, modeling_gptj.py:57-67). inverse != 0 applies the transpose
// rotation (backward). position of row r = pos0 + (r % S).
// ---------------------------------------------------------------------------------------------
__global__ void rope_kernel(bf16* __restrict__ qkv, long long ld, int rows, int S, int H, int hd, int rot, int pos0,
                            int inverse) {
  const int half = rot >> 1;
  const long long total = (long long)rows * 2 * H * half;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int p = (int)(i % half);
    long long t = i / half;
    const int h = (int)(t % H);
    t /= H;
    const int which = (int)(t % 2);
    const long long r = t / 2;
    const int pos = pos0 + (int)(r % S);
    // inv_freq = 10000^(-2p/rot); fp32 like create_sinusoidal_positions (modeling_gptj.py:47-50)
    const float inv_freq = 1.0f / powf(10000.0f, (float)(2 * p) / (float)rot);
    float sn, cs;
    sincosf((float)pos * inv_freq, &sn, &cs);
    if (inverse) sn = -sn;
    __nv_bfloat162* ptr =
        reinterpret_cast<__nv_bfloat162*>(qkv + r * ld + (long long)which * H * hd + (long long)h * hd + 2 * p);
    const float2 v = __bfloat1622float2(*ptr);
    *ptr = __floats2bfloat162_rn(v.x * cs - v.y * sn, v.y * cs + v.x * sn);
  }
}

__global__ void rope_table_kernel(float2* __restrict__ tab, int S, int half, int rot, int pos0) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= S * half) return;
  const int p = i % half, s = i / half;
  const float inv_freq = 1.0f / powf(10000.0f, (float)(2 * p) / (float)rot);
  float sn, cs;
  sincosf((float)(pos0 + s) * inv_freq, &sn, &cs);
  tab[i] = make_float2(cs, sn);
}

// ---------------------------------------------------------------------------------------------
// Softmax over fp32 scores -> bf16 probabilities. One warp per row. causal: key j visible iff j <= i + koff.
// (GPTJAttention._attn, modeling_gptj.py:136-147: fp32 scores / sqrt(hd), mask, softmax, cast to value dtype)
// rows are indexed (z, i): z = batch*head, i in [0, Sq).
// ---------------------------------------------------------------------------------------------
__global__ void softmax_fwd_kernel(const float* __restrict__ s, long long lds, long long s_bs, bf16* __restrict__ p,
                                   long long ldp, long long p_bs, int nz, int Sq, int Sk, float scale, int causal,
                                   int koff) {
  pdl_trigger();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const long long wid = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  if (wid >= (long long)nz * Sq) return;
  const int z = (int)(wid / Sq), i = (int)(wid % Sq);
  const float* sr = s + (long long)z * s_bs + (long long)i * lds;
  bf16* pr = p + (long long)z * p_bs + (long long)i * ldp;
  const int lim = causal ? min(Sk, i + koff + 1) : Sk;
  float m = -INFINITY;
  for (int j = lane; j < lim; j += 32) m = fmaxf(m, sr[j] * scale);
  m = warp_max(m);
  float sum = 0.f;
  for (int j = lane; j < lim; j += 32) sum += __expf(sr[j] * scale - m);
  sum = warp_sum(sum);
  const float inv = 1.f / sum;
  for (int j = lane; j < Sk; j += 32) pr[j] = __float2bfloat16(j < lim ? __expf(sr[j] * scale - m) * inv : 0.f);
}

// dS = P * (dP - sum_j dP*P) * scale  (bf16 out)
__global__ void softmax_bwd_kernel(const float* __restrict__ dp, long long lddp, long long dp_bs,
                                   const bf16* __restrict__ p, long long ldp, long long p_bs, bf16* __restrict__ ds,
                                   long long ldds, long long ds_bs, int nz, int Sq, int Sk, float scale) {
  pdl_trigger();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const long long wid = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  if (wid >= (long long)nz * Sq) return;
  const int z = (int)(wid / Sq), i = (int)(wid % Sq);
  const float* dpr = dp + (long long)z * dp_bs + (long long)i * lddp;
  const bf16* pr = p + (long long)z * p_bs + (long long)i * ldp;
  bf16* dsr = ds + (long long)z * ds_bs + (long long)i * ldds;
  float acc = 0.f;
  for (int j = lane; j < Sk; j += 32) acc += dpr[j] * __bfloat162float(pr[j]);
  acc = warp_sum(acc);
  for (int j = lane; j < Sk; j += 32) dsr[j] = __float2bfloat16(__bfloat162float(pr[j]) * (dpr[j] - acc) * scale);
}

// ---------------------------------------------------------------------------------------------
// build_labels (magma/utils.py:334-364), integer kernel, bit-exact:
//   labels[b, s] = -100                      for s < L
//                = captions[b, s - L]        for s >= L           (captions[:, :-L])
//   then every position AFTER the first eos in the row -> -100 (the first eos itself is kept).
// One warp per row; ballot scan for the first eos.
// ---------------------------------------------------------------------------------------------
__global__ void build_labels_kernel(const long long* __restrict__ captions, long long ldc,
                                    long long* __restrict__ labels, int B, int S, int L, long long eos) {
  const int lane = threadIdx.x & 31;
  const int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (b >= B) return;
  int first = S;  // index in label space of the first eos
  for (int base = L; base < S && first == S; base += 32) {
    const int s = base + lane;
    const bool hit = s < S && captions[(long long)b * ldc + (s - L)] == eos;
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if (m) first = base + __ffs(m) - 1;
  }
  for (int s = lane; s < S; s += 32) {
    long long v;
    if (s < L)
      v = -100;
    else
      v = captions[(long long)b * ldc + (s - L)];
    if (s > first) v = -100;
    labels[(long long)b * S + s] = v;
  }
}

// ---------------------------------------------------------------------------------------------
// Input assembly (magma/magma.py:258-267): x[b, 0:L] = prefix[b]; x[b, L+s] = wte[captions[b, s]], s < S-L.
// Gathers straight into the fused [B,S,d] buffer (the reference embeds the full caption then slices).
// ---------------------------------------------------------------------------------------------
__global__ void embed_assemble_kernel(const long long* __restrict__ captions, long long ldc,
                                      const bf16* __restrict__ wte, const bf16* __restrict__ prefix, int L,
                                      bf16* __restrict__ x, int B, int S, int d, int vocab) {
  const int row = blockIdx.x;  // b*S + s
  const int b = row / S, s = row % S;
  const uint4* src;
  if (s < L) {
    src = reinterpret_cast<const uint4*>(prefix + ((long long)b * L + s) * d);
  } else {
    long long tok = captions[(long long)b * ldc + (s - L)];
    if (tok < 0 || tok >= vocab) tok = 0;  // defensive: never read out of bounds
    src = reinterpret_cast<const uint4*>(wte + tok * (long long)d);
  }
  uint4* dst = reinterpret_cast<uint4*>(x + (long long)row * d);
  for (int c = threadIdx.x; c < (d >> 3); c += blockDim.x) dst[c] = __ldg(src + c);
}

// plain row gather: out[r] = wte[ids[r]]  (Magma.embed / decode-step input_ids path)
__global__ void embed_gather_kernel(const long long* __restrict__ ids, const bf16* __restrict__ wte,
                                    bf16* __restrict__ out, int d, int vocab) {
  long long tok = ids[blockIdx.x];
  if (tok < 0 || tok >= vocab) tok = 0;
  const uint4* src = reinterpret_cast<const uint4*>(wte + tok * (long long)d);
  uint4* dst = reinterpret_cast<uint4*>(out + (long long)blockIdx.x * d);
  for (int c = threadIdx.x; c < (d >> 3); c += blockDim.x) dst[c] = __ldg(src + c);
}

// ---------------------------------------------------------------------------------------------
// Shifted cross-entropy over bf16 logits [M = B*S][ldv] (ForCausalLMLoss, loss_utils.py:28-67):
// target of row (b, s) is labels[b, s+1]; the last position and every target outside [0, V) (-100 among them) are
// ignored; mean over valid. Both passes below apply that one rule, so an ignored row never enters n_valid.
// Pass 1 (ce_count): n_valid. Pass 2 (ce_row): per-row loss + in-place dlogits = (softmax - onehot)/n_valid.
// Pass 3 (ce_reduce): deterministic tree sum of row losses -> mean.
// ---------------------------------------------------------------------------------------------
__global__ void ce_count_kernel(const long long* __restrict__ labels, int B, int S, int V, int* __restrict__ n_valid) {
  __shared__ float red[32];
  float c = 0.f;
  for (int i = threadIdx.x; i < B * S; i += blockDim.x) {
    const int s = i % S;
    if (s + 1 < S && labels[i + 1] >= 0 && labels[i + 1] < V) c += 1.f;
  }
  const float t = block_sum<1024>(c, red);
  if (threadIdx.x == 0) *n_valid = (int)(t + 0.5f);
}

static constexpr int kCeThreads = 512;
__global__ void __launch_bounds__(kCeThreads)
ce_row_kernel(const bf16* logits, long long ldv, const long long* __restrict__ labels, int S, int V,
              const int* __restrict__ n_valid, float* __restrict__ row_loss, bf16* dlogits, float grad_scale) {
  __shared__ float red[32];
  const int row = blockIdx.x;
  const int s = row % S;
  long long tgt = (s + 1 < S) ? labels[row + 1] : -100;
  const bf16* lr = logits + (long long)row * ldv;
  bf16* dr = dlogits ? dlogits + (long long)row * ldv : nullptr;
  const int nvec = V >> 3;
  if (tgt < 0 || tgt >= V) {  // the validity rule of ce_count_kernel
    if (threadIdx.x == 0) row_loss[row] = 0.f;
    if (dr) {
      const uint4 z = make_uint4(0, 0, 0, 0);
      for (int c = threadIdx.x; c < nvec; c += kCeThreads) reinterpret_cast<uint4*>(dr)[c] = z;
      for (int j = nvec * 8 + threadIdx.x; j < V; j += kCeThreads) dr[j] = __float2bfloat16(0.f);
    }
    return;
  }
  float m = -INFINITY;
  for (int c = threadIdx.x; c < nvec; c += kCeThreads) {
    float f[8];
    unpack8(reinterpret_cast<const uint4*>(lr)[c], f);
#pragma unroll
    for (int e = 0; e < 8; ++e) m = fmaxf(m, f[e]);
  }
  for (int j = nvec * 8 + threadIdx.x; j < V; j += kCeThreads) m = fmaxf(m, __bfloat162float(lr[j]));
  m = block_max<kCeThreads>(m, red);
  float sum = 0.f;
  for (int c = threadIdx.x; c < nvec; c += kCeThreads) {
    float f[8];
    unpack8(reinterpret_cast<const uint4*>(lr)[c], f);
#pragma unroll
    for (int e = 0; e < 8; ++e) sum += __expf(f[e] - m);
  }
  for (int j = nvec * 8 + threadIdx.x; j < V; j += kCeThreads) sum += __expf(__bfloat162float(lr[j]) - m);
  sum = block_sum<kCeThreads>(sum, red);
  const float lse = m + logf(sum);
  const float tl = __bfloat162float(lr[tgt]);
  __syncthreads();  // every thread has read lr[tgt] before anyone overwrites it (dlogits may alias logits)
  if (threadIdx.x == 0) row_loss[row] = lse - tl;
  if (dr) {
    const float gs = grad_scale / (float)max(*n_valid, 1);
    const float inv = 1.f / sum;
    for (int c = threadIdx.x; c < nvec; c += kCeThreads) {
      float f[8];
      unpack8(reinterpret_cast<const uint4*>(lr)[c], f);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        float pj = __expf(f[e] - m) * inv;
        if (c * 8 + e == tgt) pj -= 1.f;
        f[e] = pj * gs;
      }
      reinterpret_cast<uint4*>(dr)[c] = pack8(f);
    }
    for (int j = nvec * 8 + threadIdx.x; j < V; j += kCeThreads) {
      float pj = __expf(__bfloat162float(lr[j]) - m) * inv;
      if (j == tgt) pj -= 1.f;
      dr[j] = __float2bfloat16(pj * gs);
    }
  }
}

__global__ void ce_reduce_kernel(const float* __restrict__ row_loss, int M, const int* __restrict__ n_valid,
                                 float* __restrict__ loss) {
  __shared__ float red[32];
  float s = 0.f;
  for (int i = threadIdx.x; i < M; i += blockDim.x) s += row_loss[i];
  const float t = block_sum<1024>(s, red);
  if (threadIdx.x == 0) *loss = t / (float)max(*n_valid, 1);
}

// ---------------------------------------------------------------------------------------------
// column sum: out[c] (+)= sum_r x[r, c]   (bias gradients). grid.x covers 64-column strips.
// ---------------------------------------------------------------------------------------------
static constexpr int kColsumRows = 64;  // rows per CTA: grid = (col strips of 64) x (row chunks) for parallelism
__global__ void __launch_bounds__(256)
colsum_kernel(const bf16* __restrict__ x, long long ldx, int rows, int cols, float* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  __shared__ float part[8][64];
  const int cl = threadIdx.x & 31;        // column pair within the strip
  const int rg = threadIdx.x >> 5;        // row group 0..7
  const int c0 = blockIdx.x * 64 + cl * 2;
  const int r0 = blockIdx.y * kColsumRows;
  const int r1 = min(rows, r0 + kColsumRows);
  float a0 = 0.f, a1 = 0.f;
  if (c0 < cols) {
    for (int r = r0 + rg; r < r1; r += 8) {
      const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(x + (long long)r * ldx + c0));
      a0 += v.x;
      a1 += v.y;
    }
  }
  part[rg][cl * 2] = a0;
  part[rg][cl * 2 + 1] = a1;
  __syncthreads();
  if (threadIdx.x < 64) {
    float s = 0.f;
#pragma unroll
    for (int g = 0; g < 8; ++g) s += part[g][threadIdx.x];
    const int c = blockIdx.x * 64 + threadIdx.x;
    if (c < cols) atomicAdd(out + c, s);  // one atomic per (column, row chunk); out is zeroed first unless accumulating
  }
}

// ---------------------------------------------------------------------------------------------
// dropout with a counter-based hash RNG (nn.Dropout in magma/image_prefix.py:104): y = x * mask / (1-p),
// mask saved as bytes for the backward pass. Also used as the backward (same mask, same scale).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t hash32(uint64_t k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdULL;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ULL;
  k ^= k >> 33;
  return (uint32_t)k;
}
__global__ void dropout_fwd_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, uint8_t* __restrict__ mask,
                                   long long n, float p, unsigned long long seed) {
  const float scale = 1.f / (1.f - p);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float u = (float)(hash32(seed * 0x9E3779B97F4A7C15ULL + (uint64_t)i) >> 8) * (1.0f / 16777216.0f);
    const uint8_t keep = u >= p ? 1 : 0;
    mask[i] = keep;
    y[i] = __float2bfloat16(keep ? __bfloat162float(x[i]) * scale : 0.f);
  }
}
__global__ void dropout_apply_kernel(const bf16* __restrict__ x, const uint8_t* __restrict__ mask,
                                     bf16* __restrict__ y, long long n, float p) {
  const float scale = 1.f / (1.f - p);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = __float2bfloat16(mask[i] ? __bfloat162float(x[i]) * scale : 0.f);
}

// ---------------------------------------------------------------------------------------------
// ViT front end: im2col of non-overlapping patches (CLIP conv1, stride = kernel = P, no bias) and the
// [cls; patches] + positional embedding assembly.
// images [B,3,R,R] -> patches [B*g*g][ldp], column order (c, py, px) = conv weight.view(width, 3*P*P) order.
// ---------------------------------------------------------------------------------------------
__global__ void patchify_kernel(const bf16* __restrict__ img, bf16* __restrict__ patches, long long ldp, int B, int R,
                                int P) {
  const int g = R / P;
  const int K = 3 * P * P;
  const long long total = (long long)B * g * g * K;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(i % K);
    const long long pr = i / K;  // patch row index b*g*g + gy*g + gx
    const int gx = (int)(pr % g);
    const int gy = (int)((pr / g) % g);
    const int b = (int)(pr / ((long long)g * g));
    const int px = k % P, py = (k / P) % P, c = k / (P * P);
    patches[pr * ldp + k] = img[(((long long)b * 3 + c) * R + (gy * P + py)) * R + (gx * P + px)];
  }
}
// x[b, 0, :] = cls + pos[0]; x[b, 1+p, :] = pe[b, p, :] + pos[1+p]   (pe = patch embeddings [B, T-1, w])
__global__ void vit_assemble_kernel(bf16* __restrict__ x, const bf16* __restrict__ pe, const bf16* __restrict__ cls,
                                    const bf16* __restrict__ pos, int B, int T, int w) {
  const long long total = (long long)B * T * w;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % w);
    const int t = (int)((i / w) % T);
    const long long b = i / ((long long)w * T);
    const float base = t == 0 ? __bfloat162float(cls[c]) : __bfloat162float(pe[(b * (T - 1) + (t - 1)) * w + c]);
    x[i] = __float2bfloat16(base + __bfloat162float(pos[(long long)t * w + c]));
  }
}

// ---------------------------------------------------------------------------------------------
// Conv-trunk support (CLIP ModifiedResNet, image_encoders.py:65-74). Activations are NHWC bf16, so a 1x1 convolution is
// a plain GEMM over [B*H*W, C]; a 3x3 convolution is im2col (column order (kh, kw, c), matching weights packed as
// [Cout][3][3][Cin]) followed by the same GEMM with the folded BatchNorm as bias. All three kernels move 16-byte
// vectors of 8 channels and are HBM-bound.
// ---------------------------------------------------------------------------------------------
// images [B, C<=8, H, W] bf16 -> [B, H, W, 8] bf16, channels C..7 zero (so that the stem's K = 9*8 is TMA-aligned)
__global__ void nchw_to_nhwc8_kernel(const bf16* __restrict__ src, bf16* __restrict__ dst, int B, int C, int H, int W) {
  const long long hw = (long long)H * W, total = (long long)B * hw;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / hw, px = i - b * hw;
    alignas(16) bf16 v[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) v[c] = c < C ? src[(b * C + c) * hw + px] : __float2bfloat16(0.f);
    *reinterpret_cast<uint4*>(dst + i * 8) = *reinterpret_cast<const uint4*>(v);
  }
}
// src [B,H,W,C] -> dst [B*Ho*Wo][9*C], 3x3 window, padding 1, stride s (Ho = (H-1)/s + 1); out-of-image taps are zero
template <typename Idx>  // 32-bit index arithmetic whenever the vector count allows it (the divisions dominate otherwise)
__global__ void im2col3x3_kernel(const bf16* __restrict__ src, bf16* __restrict__ dst, int B, int H, int W, int C,
                                 int stride, int Ho, int Wo) {
  const Idx cv = (Idx)(C >> 3);
  const Idx total = (Idx)B * Ho * Wo * 9 * cv;
  for (Idx i = blockIdx.x * (Idx)blockDim.x + threadIdx.x; i < total; i += (Idx)gridDim.x * blockDim.x) {
    const Idx t = i / cv;
    const int c8 = (int)(i - t * cv);
    const Idx row = t / 9;
    const int tap = (int)(t - row * 9);
    const Idx r2 = row / Wo;
    const int wo = (int)(row - r2 * Wo);
    const Idx b = r2 / Ho;
    const int ho = (int)(r2 - b * Ho);
    const int hi = ho * stride - 1 + tap / 3, wi = wo * stride - 1 + tap % 3;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (hi >= 0 && hi < H && wi >= 0 && wi < W)
      v = __ldg(reinterpret_cast<const uint4*>(src + (((long long)b * H + hi) * W + wi) * C) + c8);
    reinterpret_cast<uint4*>(dst)[i] = v;  // (row, tap, c8) is exactly the linear index
  }
}
// nn.AvgPool2d(k) on NHWC: dst [B, H/k, W/k, C], fp32 accumulation
__global__ void avgpool_nhwc_kernel(const bf16* __restrict__ src, bf16* __restrict__ dst, int B, int H, int W, int C,
                                    int k) {
  const int cv = C >> 3, Ho = H / k, Wo = W / k;
  const long long total = (long long)B * Ho * Wo * cv;
  const float inv = 1.f / (float)(k * k);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % cv);
    const long long px = i / cv;
    const int wo = (int)(px % Wo);
    const int ho = (int)((px / Wo) % Ho);
    const long long b = px / ((long long)Wo * Ho);
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int dy = 0; dy < k; ++dy)
      for (int dx = 0; dx < k; ++dx) {
        const uint4 u = __ldg(reinterpret_cast<const uint4*>(src + ((b * H + ho * k + dy) * W + wo * k + dx) * C) + c8);
        const bf16* e = reinterpret_cast<const bf16*>(&u);
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[c] += __bfloat162float(e[c]);
      }
    alignas(16) bf16 o[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) o[c] = __float2bfloat16(acc[c] * inv);
    reinterpret_cast<uint4*>(dst)[i] = *reinterpret_cast<const uint4*>(o);
  }
}

// ---------------------------------------------------------------------------------------------
// argmax over the last dim of bf16 rows, compared in fp32 like sampling.py:92,97 (logits.float(); argmax).
// Ties resolve to the LOWEST index (torch.argmax on CPU/CUDA returns the first maximal element).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(512)
argmax_kernel(const bf16* __restrict__ x, long long ldx, int V, long long* __restrict__ out) {
  __shared__ float sv[16];
  __shared__ int si[16];
  const bf16* r = x + (long long)blockIdx.x * ldx;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int j = threadIdx.x; j < V; j += blockDim.x) {
    const float v = __bfloat162float(r[j]);
    if (v > best || (v == best && j < bi)) {
      best = v;
      bi = j;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) {
      best = ov;
      bi = oi;
    }
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) {
    sv[w] = best;
    si[w] = bi;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < (int)(blockDim.x >> 5); ++k)
      if (sv[k] > best || (sv[k] == best && si[k] < bi)) {
        best = sv[k];
        bi = si[k];
      }
    out[blockIdx.x] = bi;
  }
}

// y = a + b (+ c) elementwise, bf16 (gradient joins)
__global__ void add_kernel(const bf16* __restrict__ a, const bf16* __restrict__ b, const bf16* __restrict__ c,
                           bf16* __restrict__ y, long long nvec) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * blockDim.x) {
    float fa[8], fb[8], fc[8];
    unpack8(reinterpret_cast<const uint4*>(a)[i], fa);
    unpack8(reinterpret_cast<const uint4*>(b)[i], fb);
    if (c) unpack8(reinterpret_cast<const uint4*>(c)[i], fc);
#pragma unroll
    for (int e = 0; e < 8; ++e) fa[e] += fb[e] + (c ? fc[e] : 0.f);
    reinterpret_cast<uint4*>(y)[i] = pack8(fa);
  }
}

// ---------------------------------------------------------------------------------------------
// The gradient that enters the LM head's dgrad when a loss reads the logits: out[r, j] = alpha * dce[r, j] + g[r, j]
// for j < V, one fp32 fma and one rounding. dce (the cross-entropy gradient) and out are [M, ldv] with 16-byte aligned
// rows. g is autograd's gradient on the logits: unit column stride, any row stride, so a row may start on any 2-byte
// boundary (ld_g = 50258 gives rows 4-byte aligned only); each row reads g with the widest load its alignment allows.
// alpha == 0 never reads dce, which then may hold anything (no cross-entropy gradient was written).
// grid = (M rows, column blocks of kLgChunks * kLgThreads 8-column chunks); the last column block also does the V % 8
// tail of its row.
// ---------------------------------------------------------------------------------------------
static constexpr int kLgThreads = 256;
static constexpr int kLgChunks = 4;

__device__ __forceinline__ void load8_aligned_to(const bf16* p, int align, float (&f)[8]) {
  if (align == 16) {
    unpack8(*reinterpret_cast<const uint4*>(p), f);
  } else if (align == 4) {
    const uint32_t* q = reinterpret_cast<const uint32_t*>(p);
    const uint4 u = make_uint4(q[0], q[1], q[2], q[3]);
    unpack8(u, f);
  } else {
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = __bfloat162float(p[e]);
  }
}

__global__ void __launch_bounds__(kLgThreads)
logits_grad_combine_kernel(const bf16* __restrict__ dce, long long ldv, const bf16* __restrict__ g, long long ld_g,
                           bf16* __restrict__ out, int V, float alpha) {
  const long long r = blockIdx.x;
  const bf16* gr = g + r * ld_g;
  const bf16* dr = dce + r * ldv;
  bf16* orow = out + r * ldv;
  const uintptr_t a = reinterpret_cast<uintptr_t>(gr);
  const int align = (a & 15) == 0 ? 16 : (a & 3) == 0 ? 4 : 2;  // the same for every chunk of the row
  const int nvec = V >> 3;
  const int c0 = (int)blockIdx.y * kLgThreads * kLgChunks + (int)threadIdx.x;
#pragma unroll
  for (int k = 0; k < kLgChunks; ++k) {
    const int c = c0 + k * kLgThreads;
    if (c < nvec) {
      float f[8];
      load8_aligned_to(gr + 8 * (long long)c, align, f);
      if (alpha != 0.f) {
        float d[8];
        unpack8(reinterpret_cast<const uint4*>(dr)[c], d);
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = fmaf(alpha, d[e], f[e]);
      }
      reinterpret_cast<uint4*>(orow)[c] = pack8(f);
    }
  }
  if (blockIdx.y == gridDim.y - 1)
    for (int j = nvec * 8 + (int)threadIdx.x; j < V; j += kLgThreads) {
      const float gj = __bfloat162float(gr[j]);
      orow[j] = __float2bfloat16(alpha != 0.f ? fmaf(alpha, __bfloat162float(dr[j]), gj) : gj);
    }
}

// ---------------------------------------------------------------------------------------------
// Gradient exchange over NVLink peer memory (data parallelism; replaces the NCCL all-reduce of DeepSpeed's engine,
// train.py:103-111). Every rank owns one shard of the slice: it reads that shard from ALL ranks' exchange buffers
// (peer-mapped pointers: plain loads over NVLink / NVSwitch), adds them in rank order, and stores the sum back into ALL
// ranks' buffers — reduce-scatter and all-gather in one pass, one launch per rank and slice. The ranks touch disjoint
// shards, so the exchange is race-free between a barrier before (every rank's slice is published) and one after (every
// store has landed). Every rank ends with the owner's bits: replicas stay bit-identical. No shared memory and ~40
// registers: its blocks are resident BESIDE the persistent GEMM CTAs of backward (NCCL's CTAs need an SM of their own).
// ---------------------------------------------------------------------------------------------
struct PeerBufs {
  float* p[16];
};
__global__ void peer_reduce_bcast_kernel(PeerBufs bufs, int world, long long off4, long long n4) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 acc = __ldcs(reinterpret_cast<const float4*>(bufs.p[0]) + off4 + i);
    for (int r = 1; r < world; ++r) {
      const float4 v = __ldcs(reinterpret_cast<const float4*>(bufs.p[r]) + off4 + i);
      acc.x += v.x;
      acc.y += v.y;
      acc.z += v.z;
      acc.w += v.w;
    }
    for (int r = 0; r < world; ++r) __stcs(reinterpret_cast<float4*>(bufs.p[r]) + off4 + i, acc);
  }
}

// ---------------------------------------------------------------------------------------------
// Optimizer step for the (small) trainable set: fused AdamW over a flat fp32 arena (torch.optim.AdamW semantics,
// train.py:96-101 betas=(0.9,0.95)), with global-norm gradient clipping (config.py:126 gradient_clipping) folded in
// through a device-side squared-norm, and the bf16 compute copy of the weights refreshed in the same pass.
// HBM-bound: 16 B read + 14 B written per parameter.
// ---------------------------------------------------------------------------------------------
// Deterministic: per-block partial sums land in a fixed slot each and the LAST block to finish adds them in a fixed order
// — every data-parallel rank holds bit-identical gradients after the all-reduce and must derive the bit-identical clipping
// coefficient from them, or the replicas' parameters drift apart by an ulp per step (an atomicAdd of the block sums, the
// previous version, is order-dependent in its last bits; tests/test_dp_gpu.py caught exactly that on 2 GPUs).
static constexpr int kSumsqMaxBlocks = 2048;
__device__ float g_sumsq_part[kSumsqMaxBlocks];
__device__ unsigned int g_sumsq_ticket = 0;

// Deterministic AND grid-independent: the input is cut into kSumsqMaxBlocks logical parts (float4 index / 256 modulo
// kSumsqMaxBlocks); a part is always summed in the same order (per thread over its chunks, then the fixed block tree), the
// parts are added in index order by the last block to finish. A block takes parts blockIdx.x, blockIdx.x + gridDim.x, ...
// so the launch may use any grid (B200Engine caps it at 2 blocks per SM when the optimizer runs beside GEMMs) without
// changing a bit of the result — data-parallel replicas and pipelined / in-stream optimizers stay bit-identical.
__global__ void sumsq_kernel(const float* __restrict__ x, long long n, float* __restrict__ out) {
  __shared__ float red[32];
  __shared__ int is_last;
  const bool vec = (reinterpret_cast<uintptr_t>(x) & 15) == 0;  // unaligned views take the scalar loop below (same parts)
  const long long n4 = vec ? (n >> 2) : 0;
  const float4* x4 = reinterpret_cast<const float4*>(x);
  const long long stride = (long long)kSumsqMaxBlocks * 256;
  for (int part = blockIdx.x; part < kSumsqMaxBlocks; part += gridDim.x) {
    if ((long long)part * 256 >= n4 && (n4 << 2) + (long long)part * 256 >= n) {  // empty part (short inputs)
      if (threadIdx.x == 0) g_sumsq_part[part] = 0.f;
      continue;
    }
    float s = 0.f;
    long long i = (long long)part * 256 + threadIdx.x;
    for (; i + 3 * stride < n4; i += 4 * stride) {  // 4 independent 16-byte loads in flight per thread
      const float4 a = __ldcs(x4 + i), b = __ldcs(x4 + i + stride), c = __ldcs(x4 + i + 2 * stride),
                   d = __ldcs(x4 + i + 3 * stride);
      s += a.x * a.x; s += a.y * a.y; s += a.z * a.z; s += a.w * a.w;
      s += b.x * b.x; s += b.y * b.y; s += b.z * b.z; s += b.w * b.w;
      s += c.x * c.x; s += c.y * c.y; s += c.z * c.z; s += c.w * c.w;
      s += d.x * d.x; s += d.y * d.y; s += d.z * d.z; s += d.w * d.w;
    }
    for (; i < n4; i += stride) {
      const float4 a = x4[i];
      s += a.x * a.x; s += a.y * a.y; s += a.z * a.z; s += a.w * a.w;
    }
    for (long long j = (n4 << 2) + (long long)part * 256 + threadIdx.x; j < n; j += stride) {  // tail / unaligned input
      const float v = x[j];
      s += v * v;
    }
    const float t = block_sum<256>(s, red);
    if (threadIdx.x == 0) g_sumsq_part[part] = t;
    __syncthreads();  // red[] is reused by the next part
  }
  if (threadIdx.x == 0) {
    __threadfence();
    is_last = atomicAdd(&g_sumsq_ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  float a = 0.f;
  for (int i = threadIdx.x; i < kSumsqMaxBlocks; i += 256) a += *((volatile float*)&g_sumsq_part[i]);
  const float total = block_sum<256>(a, red);
  if (threadIdx.x == 0) {
    out[0] += total;
    g_sumsq_ticket = 0;
  }
}

__global__ void adamw_kernel(float* __restrict__ w, float* __restrict__ g, float* __restrict__ m1,
                             float* __restrict__ m2, bf16* __restrict__ shadow, long long n4, float lr, float b1,
                             float b2, float eps, float wd, float grad_scale, const float* __restrict__ gnorm_sq,
                             float max_norm, float bc1, float bc2, int zero_grad) {
  float coef = grad_scale;
  if (gnorm_sq != nullptr && max_norm > 0.f) {
    const float nrm = sqrtf(*gnorm_sq) * grad_scale;
    coef *= fminf(1.f, max_norm / (nrm + 1e-6f));
  }
  const float inv_sqrt_bc2 = rsqrtf(bc2), step = lr / bc1, decay = 1.f - lr * wd;
  float4* w4 = reinterpret_cast<float4*>(w);
  float4* g4 = reinterpret_cast<float4*>(g);
  float4* a4 = reinterpret_cast<float4*>(m1);
  float4* v4 = reinterpret_cast<float4*>(m2);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    // streaming (evict-first) accesses: 7 GB pass once through the L2 beside GEMMs that live on L2-resident tiles
    float4 wv = __ldcs(w4 + i), gv = __ldcs(g4 + i), av = __ldcs(a4 + i), vv = __ldcs(v4 + i);
    float* wp = &wv.x;
    float* gp = &gv.x;
    float* ap = &av.x;
    float* vp = &vv.x;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float gi = gp[e] * coef;
      float wi = wp[e] * decay;
      const float a = b1 * ap[e] + (1.f - b1) * gi;
      const float v = b2 * vp[e] + (1.f - b2) * gi * gi;
      ap[e] = a;
      vp[e] = v;
      wi -= step * (a / (sqrtf(v) * inv_sqrt_bc2 + eps));
      wp[e] = wi;
    }
    __stcs(w4 + i, wv);
    __stcs(a4 + i, av);
    __stcs(v4 + i, vv);
    if (shadow) {
      __nv_bfloat162 h0 = __floats2bfloat162_rn(wv.x, wv.y), h1 = __floats2bfloat162_rn(wv.z, wv.w);
      uint2 u;
      u.x = *reinterpret_cast<uint32_t*>(&h0);
      u.y = *reinterpret_cast<uint32_t*>(&h1);
      reinterpret_cast<uint2*>(shadow)[i] = u;
    }
    if (zero_grad) __stcs(g4 + i, make_float4(0.f, 0.f, 0.f, 0.f));
  }
}

__global__ void cast_f32_bf16_kernel(const float* __restrict__ src, bf16* __restrict__ dst, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    dst[i] = __float2bfloat16(src[i]);
}
__global__ void cast_bf16_f32_kernel(const bf16* __restrict__ src, float* __restrict__ dst, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    dst[i] = __bfloat162float(src[i]);
}


// ---------------------------------------------------------------------------------------------
// Device-resident decode loop (magma/sampling.py:78-109 runs one host-driven LM call per token with an `.all()` sync
// each step): the step's cache position lives in DEVICE memory, so one CUDA graph of the whole decode step is replayed
// per token with no host-side argument changing. These are the three small kernels around the LM call that read /
// advance that position; the LM schedule itself takes it through mb200_gptj_sched_decode_step.
// ---------------------------------------------------------------------------------------------
__global__ void rope_table_dev_kernel(float2* __restrict__ tab, int S, int half, int rot, const int* __restrict__ pos0) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= S * half) return;
  const int p = i % half, s = i / half;
  const float inv_freq = 1.0f / powf(10000.0f, (float)(2 * p) / (float)rot);
  float sn, cs;
  sincosf((float)(*pos0 + s) * inv_freq, &sn, &cs);
  tab[i] = make_float2(cs, sn);
}

// x[b] = wte[tokens[b][pos]] : the input embedding of the decode step at cache position `pos` (the token emitted last)
__global__ void decode_embed_kernel(const long long* __restrict__ tokens, long long ld_tok, const int* __restrict__ pos,
                                    const bf16* __restrict__ wte, bf16* __restrict__ out, int d, int vocab) {
  long long tok = tokens[(long long)blockIdx.x * ld_tok + *pos];
  if (tok < 0 || tok >= vocab) tok = 0;
  const uint4* src = reinterpret_cast<const uint4*>(wte + tok * (long long)d);
  uint4* dst = reinterpret_cast<uint4*>(out + (long long)blockIdx.x * d);
  for (int c = threadIdx.x; c < (d >> 3); c += blockDim.x) dst[c] = __ldg(src + c);
}

// tokens[b][pos + 1] = next[b]; flags[pos + 1 - s0] = every row emitted EOS (sampling.py:109); pos += 1. One CTA.
__global__ void decode_advance_kernel(const long long* __restrict__ next, long long* __restrict__ tokens, long long ld_tok,
                                      int* __restrict__ pos, long long eos, unsigned char* __restrict__ flags, int s0,
                                      int n_flags, int B) {
  const int p = *pos;
  int is_eos = 1;
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    const long long t = next[b];
    if (p + 1 < ld_tok) tokens[(long long)b * ld_tok + p + 1] = t;
    is_eos &= (t == eos);
  }
  const int all = __syncthreads_and(is_eos);
  if (threadIdx.x == 0) {
    const int i = p + 1 - s0;
    if (flags != nullptr && i >= 0 && i < n_flags) flags[i] = (unsigned char)all;
    *pos = p + 1;
  }
}
