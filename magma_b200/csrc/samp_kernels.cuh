// Token sampling for temperature > 0 (magma/sampling.py:7-30,97-105): top-k filter, the reference's (inverted) nucleus
// filter, softmax(logits / T) and one multinomial draw per row, in ONE kernel launch with no host round trip.
//
// One CTA of 1024 threads per row; thread t owns the contiguous slice [t*C, (t+1)*C) of the vocabulary, so that "the
// first n elements equal to a value, in index order" — how ties are resolved here, = the reference run with a stable
// sort — is a per-thread counter plus one block scan. The row (200 KB at V = 50258) is re-read from L2 in every pass.
//   top-k      : 4-pass radix select (8 bits per pass) of the k-th largest order-preserving key; kept = the k largest.
//   top-p quirk: sampling.py:13-17 removes the sorted ranks j >= 1 whose PRECEDING cumulative probability is below
//                (1 - threshold), i.e. ranks 1..m with m = #{j : cum[j] < 1 - threshold}: the top m+1 tokens except the
//                very first. The boundary rank is found by a radix descent on probability MASS instead of a sort.
//   multinomial: inverse CDF over the surviving weights exp((x - max)/T) in index order, u from Philox(seed, row, offset).
//
// FRAGMENT: the body of mb200_sample and mb200_sample_dev (elt_abi.cuh), included by elementwise.cu inside an anonymous namespace in
// namespace mb200 after <curand_kernel.h>, and, unchanged, by oracle/kernel_host_exec.cpp, which executes it on the CPU.
// Needs bf16 and INFINITY.
constexpr int kSampThreads = 1024;

// larger float <=> larger key (-inf is the smallest). -0 takes the key of +0: the two are one value to the order, as
// to torch.sort / torch.topk, so ties between them go by index like any other tie.
__device__ __forceinline__ uint32_t order_key(float x) {
  const uint32_t u = __float_as_uint(x) == 0x80000000u ? 0u : __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_value(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
// every pass reads the logits through ldf: NaN of either sign reads as -inf, so it is never drawn and poisons no sum
__device__ __forceinline__ float nan_to_ninf(float v) { return fmaxf(v, -INFINITY); }  // fmaxf drops a NaN
template <typename T>
__device__ __forceinline__ float ldf(const T* p, int i);
template <>
__device__ __forceinline__ float ldf<float>(const float* p, int i) { return nan_to_ninf(p[i]); }
template <>
__device__ __forceinline__ float ldf<bf16>(const bf16* p, int i) { return nan_to_ninf(__bfloat162float(p[i])); }

struct Shared {
  unsigned int hcnt[256];
  double hmass[256];
  double dscan[kSampThreads / 32];
  int iscan[kSampThreads / 32];
  float fred[kSampThreads / 32];
  int ired[kSampThreads / 32];
  unsigned int chosen;
  unsigned int remaining;
  double above;
  int winner;
};

// exclusive prefix sum of one int per thread over the block (in thread order); also returns the block total
__device__ __forceinline__ int block_excl_scan(int v, Shared& s, int* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  __syncthreads();
  if (lane == 31) s.iscan[w] = x;
  __syncthreads();
  int base = 0, tot = 0;
  for (int i = 0; i < kSampThreads / 32; ++i) {
    if (i < w) base += s.iscan[i];
    tot += s.iscan[i];
  }
  if (total) *total = tot;
  return base + x - v;
}
__device__ __forceinline__ double block_excl_scan_d(double v, Shared& s, double* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  double x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  __syncthreads();
  if (lane == 31) s.dscan[w] = x;
  __syncthreads();
  double base = 0.0, tot = 0.0;
  for (int i = 0; i < kSampThreads / 32; ++i) {
    if (i < w) base += s.dscan[i];
    tot += s.dscan[i];
  }
  if (total) *total = tot;
  return base + x - v;
}

// "element i is one of the first n_incl elements with key == tie_key (index order), or has a larger key"
struct TopSet {
  uint32_t key;    // boundary key
  int n_incl;      // how many elements equal to the boundary key belong to the set
  int tie_base;    // number of such elements in the slices of lower-numbered threads
  __device__ __forceinline__ bool contains(uint32_t k, int& local_ties) const {
    if (k > key) return true;
    if (k == key) return (tie_base + local_ties++) < n_incl;
    return false;
  }
};

// Where the Philox offset of the draw comes from. mb200_sample passes it by value. mb200_sample_dev reads it from the
// decode loop's cache position in device memory, so a CUDA graph of the decode step draws at a new offset per replay:
// offset = pos - s0 + 1, the step index i of the host-driven loop (at step i >= 1 the position holds s0 + i - 1).
struct DecodeOffset {
  const int* pos;
  int s0;
};
__device__ __forceinline__ unsigned long long philox_offset(unsigned long long offset) { return offset; }
__device__ __forceinline__ unsigned long long philox_offset(DecodeOffset o) {
  return (unsigned long long)((long long)*o.pos - o.s0 + 1);
}

// One block per SM, said explicitly: with the default bound ptxas aims at 32 registers and spills the Philox state.
// Off: unsigned long long (mb200_sample) or DecodeOffset (mb200_sample_dev); the body is the same.
template <typename T, typename Off>
__global__ void __launch_bounds__(kSampThreads, 1)
sample_kernel(const T* __restrict__ logits, long long ld, int V, float inv_temp, int top_k, float top_p,
              unsigned long long seed, Off offset, long long* __restrict__ tokens,
              uint8_t* __restrict__ keep_mask) {
  __shared__ Shared s;
  const T* x = logits + (long long)blockIdx.x * ld;
  const int tid = threadIdx.x;
  const int C = (V + kSampThreads - 1) / kSampThreads;
  const int i0 = min(V, tid * C), i1 = min(V, i0 + C);

  // ---- top-k: the k largest (ties by index) --------------------------------------------------------------------------
  TopSet K{0u, 0x7fffffff, 0};  // default: everything (key >= 0 always true, unlimited ties)
  if (top_k > 0 && top_k < V) {
    uint32_t prefix = 0, mask = 0;
    unsigned int remaining = (unsigned int)top_k;
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int b = tid; b < 256; b += kSampThreads) s.hcnt[b] = 0;
      __syncthreads();
      for (int i = i0; i < i1; ++i) {
        const uint32_t k = order_key(ldf(x, i));
        if ((k & mask) == prefix) atomicAdd(&s.hcnt[(k >> shift) & 255u], 1u);
      }
      __syncthreads();
      if (tid == 0) {
        unsigned int acc = 0, b = 255;
        for (;; --b) {
          if (acc + s.hcnt[b] >= remaining || b == 0) break;
          acc += s.hcnt[b];
        }
        s.chosen = b;
        s.remaining = remaining - acc;  // how many elements of the chosen bin are still inside the top k
      }
      __syncthreads();
      prefix |= s.chosen << shift;
      mask |= 255u << shift;
      remaining = s.remaining;
      __syncthreads();
    }
    int ties = 0;
    for (int i = i0; i < i1; ++i) ties += order_key(ldf(x, i)) == prefix;
    K.key = prefix;
    K.n_incl = (int)remaining;
    K.tie_base = block_excl_scan(ties, s, nullptr);
  }

  // ---- row max over the kept set (rank 0: largest value, lowest index) and softmax denominator at T = 1 --------------
  float best = -INFINITY;
  int bi = 0x7fffffff;
  {
    int lt = 0;
    for (int i = i0; i < i1; ++i) {
      const float v = ldf(x, i);
      if (K.contains(order_key(v), lt) && (v > best || (v == best && i < bi))) {
        best = v;
        bi = i;
      }
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
  if ((tid & 31) == 0) {
    s.fred[tid >> 5] = best;
    s.ired[tid >> 5] = bi;
  }
  __syncthreads();
  for (int i = 0; i < kSampThreads / 32; ++i)
    if (s.fred[i] > best || (s.fred[i] == best && s.ired[i] < bi)) {
      best = s.fred[i];
      bi = s.ired[i];
    }
  const float M = best;
  const int top1 = bi;
  __syncthreads();

  // ---- the reference's nucleus filter: remove ranks 1..m, m = #{j : cum[j] < 1 - top_p} -----------------------------
  TopSet P{0xffffffffu, 0, 0};  // default: empty set (nothing removed)
  if (top_p > 0.f) {
    double zloc = 0.0;
    {
      int lt = 0;
      for (int i = i0; i < i1; ++i) {
        const float v = ldf(x, i);
        if (K.contains(order_key(v), lt)) zloc += (double)expf(v - M);
      }
    }
    double Z;
    block_excl_scan_d(zloc, s, &Z);
    const double thr = (1.0 - (double)top_p) * Z;  // cum[j] < 1 - p  <=>  mass[j] < thr
    uint32_t prefix = 0, mask = 0;
    double above = 0.0;  // mass of all elements with a key above the current prefix range
    for (int shift = 24; shift >= 0; shift -= 8) {
      for (int b = tid; b < 256; b += kSampThreads) s.hmass[b] = 0.0;
      __syncthreads();
      int lt = 0;
      for (int i = i0; i < i1; ++i) {
        const float v = ldf(x, i);
        const uint32_t k = order_key(v);
        if (K.contains(k, lt) && (k & mask) == prefix) atomicAdd(&s.hmass[(k >> shift) & 255u], (double)expf(v - M));
      }
      __syncthreads();
      if (tid == 0) {
        double acc = above;
        unsigned int b = 255;
        for (;; --b) {
          if (acc + s.hmass[b] >= thr || b == 0) break;  // the crossing element lives in bin b
          acc += s.hmass[b];
        }
        s.chosen = b;
        s.above = acc;
      }
      __syncthreads();
      prefix |= s.chosen << shift;
      mask |= 255u << shift;
      above = s.above;
      __syncthreads();
    }
    // elements equal to the boundary key: t of them keep the cumulative mass below thr, the next one is the crossing rank
    const double e = (double)expf(key_value(prefix) - M);
    int ties = 0;
    {
      int lt = 0;
      for (int i = i0; i < i1; ++i) {
        const uint32_t k = order_key(ldf(x, i));
        const bool in_k = K.contains(k, lt);
        ties += (in_k && k == prefix) ? 1 : 0;
      }
    }
    int total_ties;
    const int base = block_excl_scan(ties, s, &total_ties);
    long long t = 0;  // largest t with above + t*e < thr
    if (e > 0.0 && thr > above) {
      t = (long long)ceil((thr - above) / e) - 1;
      while (t > 0 && above + (double)t * e >= thr) --t;
      while (above + (double)(t + 1) * e < thr) ++t;
    }
    if (t > total_ties - 1) t = total_ties - 1;
    if (t < 0) t = 0;
    P.key = prefix;
    P.n_incl = (int)t + 1;  // the top (m + 1) elements
    P.tie_base = base;
  }

  // ---- surviving weights exp((x - M)/T), inverse-CDF draw in index order ---------------------------------------------
  double wloc = 0.0;
  {
    int ltk = 0, ltp = 0;
    for (int i = i0; i < i1; ++i) {
      const float v = ldf(x, i);
      const uint32_t k = order_key(v);
      const bool in_k = K.contains(k, ltk);
      const bool in_p = in_k && k >= P.key && P.contains(k, ltp);  // one of the top (m + 1) elements
      const bool keep = in_k && !(in_p && i != top1);
      if (keep_mask) keep_mask[(long long)blockIdx.x * V + i] = keep ? 1 : 0;
      if (keep) wloc += (double)expf((v - M) * inv_temp);
    }
  }
  double W;
  const double wbase = block_excl_scan_d(wloc, s, &W);
  curandStatePhilox4_32_10_t st;
  curand_init(seed, (unsigned long long)blockIdx.x, philox_offset(offset), &st);
  const double u = (double)curand_uniform(&st) * W;  // (0, W]: identical in every thread of the row
  if (tid == 0) s.winner = 0x7fffffff;
  __syncthreads();
  if (wloc > 0.0 && u > wbase && u <= wbase + wloc) {
    double acc = wbase;
    int pick = -1, last_kept = -1, ltk = 0, ltp = 0;
    for (int i = i0; i < i1; ++i) {
      const float v = ldf(x, i);
      const uint32_t k = order_key(v);
      const bool in_k = K.contains(k, ltk);
      const bool in_p = in_k && k >= P.key && P.contains(k, ltp);
      if (in_k && !(in_p && i != top1)) {
        last_kept = i;
        acc += (double)expf((v - M) * inv_temp);
        if (acc >= u) {
          pick = i;
          break;
        }
      }
    }
    if (pick < 0) pick = last_kept;
    atomicMin(&s.winner, pick);
  }
  __syncthreads();
  if (tid == 0) tokens[blockIdx.x] = s.winner == 0x7fffffff ? top1 : s.winner;  // rounding fallback: the mode
}
