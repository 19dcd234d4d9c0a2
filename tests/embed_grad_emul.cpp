// TEST INFRASTRUCTURE — CPU emulation of mb200_embed_grad (elt_kernels.cuh: embed_grad_kernel), linked by
// tests/test_lm_train_cpu.py next to oracle/cabi_emul.cpp, so the Python training paths that route the input gradient
// into a trainable word embedding run on the CPU. Nothing in magma_b200/ uses it. The kernel source itself is held to
// float64 on the CPU kernel executor in the same test file. Same order of summation as the kernel: position order.
#include <stdint.h>
#include <string.h>

#include "../include/magma_b200.h"

namespace mb200 {
void set_error(const char* fmt, ...);
}

extern "C" int mb200_embed_grad(const int64_t* ids, int64_t ld_ids, const void* dy_, int64_t lddy, int64_t dy_bs,
                                int32_t B, int32_t T, float* dwte, int32_t vocab, int32_t d, int32_t accumulate, void*) {
  if (B < 0 || T < 0 || vocab <= 0 || d % 8 || ld_ids < T || lddy % 8 || dy_bs % 8 || !ids || !dwte) {
    mb200::set_error("embed_grad: bad arguments");
    return MB200_E_ARG;
  }
  if (!accumulate) memset(dwte, 0, (size_t)vocab * d * sizeof(float));
  const uint16_t* dy = (const uint16_t*)dy_;
  for (long long b = 0; b < B; ++b)
    for (long long j = 0; j < T; ++j) {
      long long t = ids[b * ld_ids + j];
      if (t < 0 || t >= vocab) t = 0;
      const uint16_t* row = dy + b * dy_bs + j * lddy;
      for (int c = 0; c < d; ++c) {
        const uint32_t u = (uint32_t)row[c] << 16;
        float f;
        memcpy(&f, &u, 4);
        dwte[t * d + c] += f;
      }
    }
  return 0;
}
