// magma_b200 — the kernels added for encoder training and the general adapter schedule (LayerNorm parameter gradients
// over many rows, QuickGELU backward, BatchNorm / ReLU / convolution-adjoint support for the conv trunk, adapter_scale).
// FRAGMENT: included by elementwise.cu inside `namespace mb200`; the host wrappers (C ABI) are in elt_abi.cuh.
// Checked on the GPU by tests/test_training_paths_gpu.py; their SOURCE is also executed on the CPU by oracle/kernel_host_exec.cpp (threads of a
// block as OS threads, __syncthreads / shuffles / atomics emulated) and held to torch in tests/test_kernel_source_cpu.py.
// LayerNorm parameter gradients for MANY rows (ViT training: 2056 rows x 49 LayerNorms; adapters with a leading LN):
// the same (column strip) x (row chunk) decomposition as colsum_kernel. out must be zeroed first unless accumulating.
static constexpr int kLnPgRows = 64;
__global__ void __launch_bounds__(256)
layernorm_param_grad_rows_kernel(const bf16* __restrict__ dy, long long lddy, const bf16* __restrict__ x, long long ldx,
                                 const float* __restrict__ mean, const float* __restrict__ rstd,
                                 float* __restrict__ dgamma, float* __restrict__ dbeta, int rows, int d) {
  __shared__ float pg[8][64], pb[8][64];
  const int cl = threadIdx.x & 31;  // column pair within the strip
  const int rg = threadIdx.x >> 5;  // row group 0..7
  const int c0 = blockIdx.x * 64 + cl * 2;
  const int r0 = blockIdx.y * kLnPgRows;
  const int r1 = min(rows, r0 + kLnPgRows);
  float g0 = 0.f, g1 = 0.f, b0 = 0.f, b1 = 0.f;
  if (c0 < d) {
    for (int r = r0 + rg; r < r1; r += 8) {
      const float2 g = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(dy + (long long)r * lddy + c0));
      const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(x + (long long)r * ldx + c0));
      const float mu = mean[r], rs = rstd[r];
      g0 += g.x * (v.x - mu) * rs;
      g1 += g.y * (v.y - mu) * rs;
      b0 += g.x;
      b1 += g.y;
    }
  }
  pg[rg][cl * 2] = g0;
  pg[rg][cl * 2 + 1] = g1;
  pb[rg][cl * 2] = b0;
  pb[rg][cl * 2 + 1] = b1;
  __syncthreads();
  if (threadIdx.x < 128) {
    const int j = threadIdx.x & 63;
    const int c = blockIdx.x * 64 + j;
    float s = 0.f;
    if (threadIdx.x < 64) {
#pragma unroll
      for (int q = 0; q < 8; ++q) s += pg[q][j];
      if (c < d) atomicAdd(dgamma + c, s);
    } else {
#pragma unroll
      for (int q = 0; q < 8; ++q) s += pb[q][j];
      if (c < d) atomicAdd(dbeta + c, s);
    }
  }
}

// QuickGELU backward (CLIP MLP): dx = dy * (s + 1.702 x s (1 - s)), s = sigmoid(1.702 x). 16-byte vectors; dx may alias dy.
__global__ void quick_gelu_bwd_kernel(const bf16* dy, const bf16* __restrict__ pre, bf16* dx, long long nvec) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float g[8], x[8], o[8];
    unpack8(reinterpret_cast<const uint4*>(dy)[i], g);
    unpack8(reinterpret_cast<const uint4*>(pre)[i], x);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float s = 1.f / (1.f + __expf(-1.702f * x[e]));
      o[e] = g[e] * (s + 1.702f * x[e] * s * (1.f - s));
    }
    reinterpret_cast<uint4*>(dx)[i] = pack8(o);
  }
}

// ---------------------------------------------------------------------------------------------
// Conv-trunk TRAINING support (freeze_img_encoder: false with a CLIP ModifiedResNet — the configuration MAGMA_v1.yml
// and MAGMA_v2.yml ship): BatchNorm in training mode and the convolution backward pass, NHWC bf16, HBM-bound.
//   col_moments_kernel      per-channel sum(u') and sum(u' * v), u' = u * 1[mask > 0]:  batch statistics (u = v = x)
//                           and the two BatchNorm-backward reductions (u = dy, v = x)
//   channel_affine_kernel   y = relu?(a1[c] * x1 * 1[mask > 0] + a2[c] * x2 + c0[c] + res): BatchNorm forward
//                           (+ residual + ReLU), BatchNorm backward, ReLU backward — coefficients are per channel, fp32
//   col2im3x3_kernel        adjoint of im2col3x3_kernel (3x3, padding 1, stride 1|2): gather form, fp32 accumulation
//   avgpool_nhwc_bwd_kernel adjoint of avgpool_nhwc_kernel
// ---------------------------------------------------------------------------------------------
static constexpr int kMomRows = 128;
__global__ void __launch_bounds__(256)
col_moments_kernel(const bf16* __restrict__ u, long long ldu, const bf16* __restrict__ v, long long ldv,
                   const bf16* __restrict__ mask, long long ldm, int rows, int cols, float* __restrict__ out1,
                   float* __restrict__ out2) {
  __shared__ float p1[8][64], p2[8][64];
  const int cl = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int c0 = blockIdx.x * 64 + cl * 2;
  const int r0 = blockIdx.y * kMomRows;
  const int r1 = min(rows, r0 + kMomRows);
  float a0 = 0.f, a1 = 0.f, b0 = 0.f, b1 = 0.f;
  if (c0 < cols) {
    for (int r = r0 + rg; r < r1; r += 8) {
      float2 x = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(u + (long long)r * ldu + c0));
      const float2 y = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(v + (long long)r * ldv + c0));
      if (mask) {
        const float2 m = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(mask + (long long)r * ldm + c0));
        if (!(m.x > 0.f)) x.x = 0.f;
        if (!(m.y > 0.f)) x.y = 0.f;
      }
      a0 += x.x;
      a1 += x.y;
      b0 += x.x * y.x;
      b1 += x.y * y.y;
    }
  }
  p1[rg][cl * 2] = a0;
  p1[rg][cl * 2 + 1] = a1;
  p2[rg][cl * 2] = b0;
  p2[rg][cl * 2 + 1] = b1;
  __syncthreads();
  if (threadIdx.x < 128) {
    const int j = threadIdx.x & 63;
    const int c = blockIdx.x * 64 + j;
    float s = 0.f;
    if (threadIdx.x < 64) {
#pragma unroll
      for (int q = 0; q < 8; ++q) s += p1[q][j];
      if (c < cols) atomicAdd(out1 + c, s);
    } else {
#pragma unroll
      for (int q = 0; q < 8; ++q) s += p2[q][j];
      if (c < cols) atomicAdd(out2 + c, s);
    }
  }
}

__global__ void channel_affine_kernel(const bf16* __restrict__ x1, const float* __restrict__ a1,
                                      const bf16* __restrict__ x2, const float* __restrict__ a2,
                                      const float* __restrict__ c0, const bf16* __restrict__ mask,
                                      const bf16* __restrict__ res, int relu, bf16* __restrict__ y, long long rows, int C) {
  const int cv = C >> 3;
  const long long total = rows * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv) * 8;
    float f[8], t[8];
    unpack8(reinterpret_cast<const uint4*>(x1)[i], f);
    if (mask) {
      unpack8(reinterpret_cast<const uint4*>(mask)[i], t);
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (!(t[e] > 0.f)) f[e] = 0.f;
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = f[e] * __ldg(a1 + c + e) + (c0 ? __ldg(c0 + c + e) : 0.f);
    if (x2) {
      unpack8(reinterpret_cast<const uint4*>(x2)[i], t);
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] += t[e] * __ldg(a2 + c + e);
    }
    if (res) {
      unpack8(reinterpret_cast<const uint4*>(res)[i], t);
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] += t[e];
    }
    if (relu) {
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] = fmaxf(f[e], 0.f);
    }
    reinterpret_cast<uint4*>(y)[i] = pack8(f);
  }
}

// dcols [B*Ho*Wo][9*C] -> dx [B,H,W,C]: dx[b,h,w] = sum over taps (kh,kw) with ho*s - 1 + kh = h, wo*s - 1 + kw = w
__global__ void col2im3x3_kernel(const bf16* __restrict__ dcols, bf16* __restrict__ dx, int B, int H, int W, int C,
                                 int stride, int Ho, int Wo) {
  const int cv = C >> 3;
  const long long total = (long long)B * H * W * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % cv);
    long long t = i / cv;
    const int w = (int)(t % W);
    t /= W;
    const int h = (int)(t % H);
    const long long b = t / H;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int kh = 0; kh < 3; ++kh) {
      const int hn = h + 1 - kh;
      if (hn < 0 || hn % stride != 0 || hn / stride >= Ho) continue;
      for (int kw = 0; kw < 3; ++kw) {
        const int wn = w + 1 - kw;
        if (wn < 0 || wn % stride != 0 || wn / stride >= Wo) continue;
        const long long row = (b * Ho + hn / stride) * Wo + wn / stride;
        float f[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(dcols + (row * 9 + (kh * 3 + kw)) * C) + c8), f);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] += f[e];
      }
    }
    reinterpret_cast<uint4*>(dx)[i] = pack8(acc);
  }
}

__global__ void avgpool_nhwc_bwd_kernel(const bf16* __restrict__ dy, bf16* __restrict__ dx, int B, int H, int W, int C,
                                        int k) {
  const int cv = C >> 3, Ho = H / k, Wo = W / k;
  const long long total = (long long)B * H * W * cv;
  const float inv = 1.f / (float)(k * k);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % cv);
    long long t = i / cv;
    const int w = (int)(t % W);
    t /= W;
    const int h = (int)(t % H);
    const long long b = t / H;
    float f[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (h / k < Ho && w / k < Wo) {
      unpack8(__ldg(reinterpret_cast<const uint4*>(dy + ((b * Ho + h / k) * Wo + w / k) * C) + c8), f);
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] *= inv;
    }
    reinterpret_cast<uint4*>(dx)[i] = pack8(f);
  }
}

// Per-channel BatchNorm bookkeeping, one thread per channel (C is a few thousand at most): these replace ~16 C-element
// framework launches per conv-BN unit and pass.
//   forward : batch statistics from (sum z, sum z^2), the normalisation coefficients channel_affine consumes
//             (scale = gamma * rstd, shift = beta - mean * scale), and nn.BatchNorm2d's running-statistics update
//             (momentum, unbiased variance)
//   backward: dgamma = sum dy' * xhat, dbeta = sum dy' (written or accumulated), and the coefficients of
//             dz = A * dy' + Bc * z + Cc  ==  gamma * rstd * (dy' - mean(dy') - xhat * mean(dy' * xhat))
__global__ void bn_finalize_fwd_kernel(const float* __restrict__ s1, const float* __restrict__ s2,
                                       const float* __restrict__ gamma, const float* __restrict__ beta, float inv_rows,
                                       float unbias, float eps, float momentum, float* __restrict__ running_mean,
                                       float* __restrict__ running_var, float* __restrict__ mean, float* __restrict__ rstd,
                                       float* __restrict__ scale, float* __restrict__ shift, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float m = s1[c] * inv_rows;
  const float var = fmaxf(s2[c] * inv_rows - m * m, 0.f);
  const float rs = rsqrtf(var + eps);
  const float sc = gamma[c] * rs;
  mean[c] = m;
  rstd[c] = rs;
  scale[c] = sc;
  shift[c] = beta[c] - m * sc;
  if (running_mean) {
    running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * m;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * var * unbias;
  }
}

__global__ void bn_bwd_coeffs_kernel(const float* __restrict__ s1, const float* __restrict__ t,
                                     const float* __restrict__ mean, const float* __restrict__ rstd,
                                     const float* __restrict__ gamma, float inv_rows, float* __restrict__ dgamma,
                                     float* __restrict__ dbeta, int accumulate, float* __restrict__ A,
                                     float* __restrict__ Bc, float* __restrict__ Cc, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float s2 = rstd[c] * (t[c] - mean[c] * s1[c]);  // sum dy' * xhat
  dgamma[c] = accumulate ? dgamma[c] + s2 : s2;
  dbeta[c] = accumulate ? dbeta[c] + s1[c] : s1[c];
  const float a = gamma[c] * rstd[c];
  const float k2 = a * rstd[c] * s2 * inv_rows;
  A[c] = a;
  Bc[c] = -k2;
  Cc[c] = k2 * mean[c] - a * s1[c] * inv_rows;
}

// out = s[0] * u + r1 + r2 (r1 / r2 optional; s == nullptr means 1): the `* adapter_scale` of ParallelAdapter.forward
// (magma/adapters.py:63-66,85-92) with the block's residual sum folded in. s is a DEVICE scalar (a trainable parameter).
__global__ void scale_add_kernel(const bf16* __restrict__ u, const float* __restrict__ s, const bf16* __restrict__ r1,
                                 const bf16* __restrict__ r2, bf16* __restrict__ out, long long nvec) {
  const float sc = s ? __ldg(s) : 1.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float a[8], b[8];
    unpack8(reinterpret_cast<const uint4*>(u)[i], a);
#pragma unroll
    for (int e = 0; e < 8; ++e) a[e] *= sc;
    if (r1) {
      unpack8(reinterpret_cast<const uint4*>(r1)[i], b);
#pragma unroll
      for (int e = 0; e < 8; ++e) a[e] += b[e];
    }
    if (r2) {
      unpack8(reinterpret_cast<const uint4*>(r2)[i], b);
#pragma unroll
      for (int e = 0; e < 8; ++e) a[e] += b[e];
    }
    reinterpret_cast<uint4*>(out)[i] = pack8(a);
  }
}

// out[0] += sum_i a_i * b_i (fp32): gradient of the adapter_scale scalar. One atomic per CTA; out zeroed first unless
// accumulating.
__global__ void __launch_bounds__(256)
dot_kernel(const bf16* __restrict__ a, const bf16* __restrict__ b, long long nvec, float* __restrict__ out) {
  __shared__ float red[32];
  float acc = 0.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float x[8], y[8];
    unpack8(reinterpret_cast<const uint4*>(a)[i], x);
    unpack8(reinterpret_cast<const uint4*>(b)[i], y);
#pragma unroll
    for (int e = 0; e < 8; ++e) acc += x[e] * y[e];
  }
  const float t = block_sum<256>(acc, red);
  if (threadIdx.x == 0) atomicAdd(out, t);
}

