// TEST INFRASTRUCTURE — CPU emulation of mb200_logits_grad_combine (elt_kernels.cuh: logits_grad_combine_kernel), linked
// by tests/test_logits_grad_cpu.py next to oracle/cabi_emul.cpp and tests/attention_emul.cpp, so the schedule's CPU build
// runs the backward of a loss on the logits. Nothing in magma_b200/ uses it. The kernel source itself is held to float64
// on the CPU kernel executor (tests/test_logits_grad_kernel_twin_cpu.py).
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "../include/magma_b200.h"

namespace mb200 {
void set_error(const char* fmt, ...);
}

namespace {

float b2f(uint16_t v) {
  uint32_t u = (uint32_t)v << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}

uint16_t f2b(float f) {  // round to nearest even, like __float2bfloat16_rn
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);
  return (uint16_t)((u + 0x7fffu + ((u >> 16) & 1u)) >> 16);
}

}  // namespace

extern "C" int mb200_logits_grad_combine(const void* dce_, int64_t ldv, const void* g_, int64_t ld_g, void* out_, int32_t M,
                                         int32_t V, float alpha, void*) {
  if (M <= 0 || V <= 0 || V > ldv || V > ld_g || !g_ || !out_ || (!dce_ && alpha != 0.f) || ldv % 8 ||
      ((uintptr_t)dce_ | (uintptr_t)out_) % 16 || (uintptr_t)g_ % 2) {
    mb200::set_error("logits_grad_combine: bad arguments");
    return MB200_E_ARG;
  }
  const uint16_t* dce = (const uint16_t*)dce_;
  const uint16_t* g = (const uint16_t*)g_;
  uint16_t* out = (uint16_t*)out_;
  for (long long r = 0; r < M; ++r)
    for (long long j = 0; j < V; ++j) {
      const float gj = b2f(g[r * ld_g + j]);
      out[r * ldv + j] = f2b(alpha != 0.f ? fmaf(alpha, b2f(dce[r * ldv + j]), gj) : gj);
    }
  return 0;
}
