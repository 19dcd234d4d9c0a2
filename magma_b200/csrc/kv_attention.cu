// magma_b200 — KV-cache kernels of the decode path (magma/sampling.py:78-109 runs one LM call per generated token with
// `use_cache=True`; HF grows the cache with torch.cat, hf:gptj/modeling_gptj.py:209-214): append of a prefill's K / V rows
// into the static cache, and the fused single-query attention of a decode step. Both are HBM-bound byte movers; the
// schedules that launch them are host-only (csrc/gptj_sched.cu) and call them through the C ABI below.
#include "common.cuh"

#include <math.h>

namespace mb200 {

// ---------------------------------------------------------------------------------------------
// KV-cache append (prefill and decode): cache[b][h][pos0+s][:] = qkv[b*S+s][which][h][:]
// ---------------------------------------------------------------------------------------------
__global__ void kv_append_kernel(const bf16* __restrict__ qkv, long long ld, bf16* __restrict__ kc,
                                 bf16* __restrict__ vc, int B, int S, int H, int hd, int Smax, int pos0) {
  const int vec = hd >> 3;
  const long long total = (long long)B * S * H * vec;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % vec);
    long long t = i / vec;
    const int h = (int)(t % H);
    t /= H;
    const int s = (int)(t % S);
    const int b = (int)(t / S);
    const long long src = ((long long)b * S + s) * ld + (long long)h * hd + c * 8;
    const long long dst = (((long long)b * H + h) * Smax + (pos0 + s)) * hd + c * 8;
    *reinterpret_cast<uint4*>(kc + dst) = *reinterpret_cast<const uint4*>(qkv + src + (long long)H * hd);
    *reinterpret_cast<uint4*>(vc + dst) = *reinterpret_cast<const uint4*>(qkv + src + 2LL * H * hd);
  }
}

// ---------------------------------------------------------------------------------------------
// Fused decode-step attention (Sq = 1) over the KV cache. One CTA per (b, h): scores in shared memory (fp32),
// softmax in fp32, probabilities rounded to bf16 before P*V exactly like the prefill path / the reference
// (`attn_weights.to(value.dtype)`, hf:gptj/modeling_gptj.py:146). HBM-bound: K and V are each read once, with
// 512-byte coalesced rows.
// ---------------------------------------------------------------------------------------------
static constexpr int kDecThreads = 256;
__global__ void __launch_bounds__(kDecThreads)
attn_decode_kernel(const bf16* __restrict__ qkv, long long ld_qkv, bf16* __restrict__ kc, bf16* __restrict__ vc,
                   bf16* __restrict__ out, long long ld_out, int H, int hd, int Smax, int pos_host,
                   const int* __restrict__ pos_dev) {
  extern __shared__ float sc[];  // [pos+1] scores, then [32] reduction scratch
  // the cache position: a kernel argument, or — device-resident decode loop, one replayed CUDA graph per token — read
  // from device memory (shared memory is then sized for Smax by the launch)
  const int pos = pos_dev ? *pos_dev : pos_host;
  if (pos < 0 || pos >= Smax) return;
  const int b = blockIdx.x / H, h = blockIdx.x % H;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nk = pos + 1;
  float* red = sc + ((nk + 31) & ~31);
  const bf16* qrow = qkv + (long long)b * ld_qkv + (long long)h * hd;
  bf16* kbase = kc + ((long long)b * H + h) * (long long)Smax * hd;
  bf16* vbase = vc + ((long long)b * H + h) * (long long)Smax * hd;
  // append this step's k, v
  for (int c = threadIdx.x; c < hd; c += kDecThreads) {
    kbase[(long long)pos * hd + c] = qrow[(long long)H * hd + c];
    vbase[(long long)pos * hd + c] = qrow[2LL * H * hd + c];
  }
  __syncthreads();
  const float scale = rsqrtf((float)hd);
  // scores: one warp per key, lanes stride the head dim in 8-element vectors
  const int vecs = hd >> 3;
  for (int j = warp; j < nk; j += kDecThreads / 32) {
    float acc = 0.f;
    for (int v = lane; v < vecs; v += 32) {
      const uint4 ku = *reinterpret_cast<const uint4*>(kbase + (long long)j * hd + v * 8);
      const uint4 qu = *reinterpret_cast<const uint4*>(qrow + v * 8);
      const __nv_bfloat162* kh = reinterpret_cast<const __nv_bfloat162*>(&ku);
      const __nv_bfloat162* qh = reinterpret_cast<const __nv_bfloat162*>(&qu);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 a = __bfloat1622float2(kh[e]), q2 = __bfloat1622float2(qh[e]);
        acc += a.x * q2.x + a.y * q2.y;
      }
    }
    acc = warp_sum(acc);
    if (lane == 0) sc[j] = acc * scale;
  }
  __syncthreads();
  float m = -INFINITY;
  for (int j = threadIdx.x; j < nk; j += kDecThreads) m = fmaxf(m, sc[j]);
  m = warp_max(m);
  if (lane == 0) red[warp] = m;
  __syncthreads();
  m = red[0];
  for (int w = 1; w < kDecThreads / 32; ++w) m = fmaxf(m, red[w]);
  __syncthreads();
  float sum = 0.f;
  for (int j = threadIdx.x; j < nk; j += kDecThreads) {
    const float e = __expf(sc[j] - m);
    sc[j] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  sum = 0.f;
  for (int w = 0; w < kDecThreads / 32; ++w) sum += red[w];
  const float inv = 1.f / sum;
  // out[c] = sum_j bf16(p_j) * v[j][c]
  for (int c = threadIdx.x; c < hd; c += kDecThreads) {
    float acc = 0.f;
    for (int j = 0; j < nk; ++j) {
      const float pj = __bfloat162float(__float2bfloat16(sc[j] * inv));
      acc += pj * __bfloat162float(vbase[(long long)j * hd + c]);
    }
    out[(long long)b * ld_out + (long long)h * hd + c] = __float2bfloat16(acc);
  }
}

// Dynamic shared memory of a decode launch that scores n_keys keys ([n_keys] fp32 scores padded to 32, then the [32]
// reduction scratch), checked against the 200 KB the kernel is opted in to — beyond the 48 KB default, so caches longer
// than about 12,000 positions can be used.
static int decode_smem(long long n_keys, size_t* smem) {
  *smem = (((size_t)n_keys + 31) & ~(size_t)31) * 4 + 32 * 4;
  MB_REQUIRE(*smem <= 200 * 1024, MB200_E_SHAPE, "attn_decode: %lld keys need %zu bytes of shared memory", n_keys, *smem);
  static bool set = false;
  if (!set) {
    MB_CUDA(cudaFuncSetAttribute(attn_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    set = true;
  }
  return 0;
}

}  // namespace mb200

using namespace mb200;

extern "C" int mb200_attn_decode(const void* qkv, int64_t ld_qkv, void* kcache, void* vcache, void* out,
                                 int64_t ld_out, int32_t B, int32_t H, int32_t hd, int32_t S_kv_max, int32_t pos,
                                 void* stream) {
  int rc = check_arch();
  if (rc) return rc;
  MB_REQUIRE(hd % 8 == 0 && pos >= 0 && pos < S_kv_max, MB200_E_SHAPE, "attn_decode: bad hd=%d pos=%d Smax=%d", hd, pos,
             S_kv_max);
  size_t smem;
  if ((rc = decode_smem((long long)pos + 1, &smem))) return rc;
  attn_decode_kernel<<<B * H, kDecThreads, smem, (cudaStream_t)stream>>>((const bf16*)qkv, ld_qkv, (bf16*)kcache,
                                                                         (bf16*)vcache, (bf16*)out, ld_out, H, hd,
                                                                         S_kv_max, pos, nullptr);
  count_launch();
  MB_CUDA(cudaGetLastError());
  return 0;
}

// the same step with the cache position read from device memory (graph-replayed decode loop)
extern "C" int mb200_attn_decode_dev(const void* qkv, int64_t ld_qkv, void* kcache, void* vcache, void* out,
                                     int64_t ld_out, int32_t B, int32_t H, int32_t hd, int32_t S_kv_max,
                                     const int32_t* pos_dev, void* stream) {
  int rc = check_arch();
  if (rc) return rc;
  MB_REQUIRE(hd % 8 == 0 && S_kv_max > 0 && pos_dev != nullptr, MB200_E_SHAPE, "attn_decode_dev: bad hd=%d Smax=%d", hd,
             S_kv_max);
  size_t smem;
  if ((rc = decode_smem(S_kv_max, &smem))) return rc;
  attn_decode_kernel<<<B * H, kDecThreads, smem, (cudaStream_t)stream>>>((const bf16*)qkv, ld_qkv, (bf16*)kcache,
                                                                         (bf16*)vcache, (bf16*)out, ld_out, H, hd,
                                                                         S_kv_max, 0, pos_dev);
  count_launch();
  MB_CUDA(cudaGetLastError());
  return 0;
}

// K/V rows of a prefill (or any S > 1 continuation) into the static cache — the launch gptj_forward issues, exposed for
// the host-only LM schedule (csrc/gptj_sched.cu).
extern "C" int mb200_kv_append(const void* qkv, int64_t ld_qkv, void* kcache, void* vcache, int32_t B, int32_t S,
                               int32_t H, int32_t hd, int32_t S_kv_max, int32_t pos0, void* stream) {
  int rc = check_arch();
  if (rc) return rc;
  MB_REQUIRE(hd % 8 == 0 && B > 0 && S > 0 && pos0 >= 0 && pos0 + S <= S_kv_max, MB200_E_SHAPE,
             "kv_append: bad hd=%d B=%d S=%d pos0=%d Smax=%d", hd, B, S, pos0, S_kv_max);
  const long long tot = (long long)B * S * H * (hd / 8);
  int grid = (int)((tot + 255) / 256);
  if (grid > num_sms() * 8) grid = num_sms() * 8;
  kv_append_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const bf16*)qkv, ld_qkv, (bf16*)kcache, (bf16*)vcache, B, S, H,
                                                           hd, S_kv_max, pos0);
  count_launch();
  MB_CUDA(cudaGetLastError());
  return 0;
}
