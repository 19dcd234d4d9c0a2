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
#include <curand_kernel.h>

#include "common.cuh"

#define MB_ENTER()                 \
  do {                             \
    int _rc = mb200::check_arch(); \
    if (_rc) return _rc;           \
  } while (0)
#define MB_LAUNCH_CHECK()        \
  do {                           \
    mb200::count_launch();       \
    MB_CUDA(cudaGetLastError()); \
  } while (0)

namespace mb200 {
namespace {

#include "samp_kernels.cuh"

}  // namespace
}  // namespace mb200

using namespace mb200;

extern "C" int mb200_sample(const void* logits, int32_t dtype, int64_t ld, int32_t rows, int32_t V, float temperature,
                            int32_t top_k, float top_p, uint64_t seed, uint64_t offset, int64_t* tokens,
                            uint8_t* keep_mask, void* stream) {
  MB_ENTER();
  MB_REQUIRE(rows > 0 && V > 0 && ld >= V, MB200_E_SHAPE, "sample: rows=%d V=%d ld=%lld", rows, V, (long long)ld);
  MB_REQUIRE(temperature > 0.f, MB200_E_ARG, "sample: temperature must be > 0 (use mb200_argmax for greedy decoding)");
  MB_REQUIRE(top_k >= 0 && top_p >= 0.f && top_p <= 1.f, MB200_E_ARG, "sample: top_k=%d top_p=%f", top_k, top_p);
  MB_REQUIRE(dtype == MB200_BF16 || dtype == MB200_F32, MB200_E_DTYPE, "sample: logits must be bf16 or f32");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == MB200_F32)
    sample_kernel<float><<<rows, kSampThreads, 0, st>>>((const float*)logits, ld, V, 1.f / temperature, top_k, top_p, seed,
                                                         offset, (long long*)tokens, keep_mask);
  else
    sample_kernel<bf16><<<rows, kSampThreads, 0, st>>>((const bf16*)logits, ld, V, 1.f / temperature, top_k, top_p, seed,
                                                        offset, (long long*)tokens, keep_mask);
  MB_LAUNCH_CHECK();
  return 0;
}
