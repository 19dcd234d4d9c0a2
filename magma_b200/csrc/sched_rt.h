// magma_b200 — the small runtime interface that HOST-ONLY schedule files (gptj_sched.cu, vit_sched.cu) are written against.
//
// A schedule file contains no kernels and no CUDA runtime calls: it carves a workspace and issues the primitive
// operators of the C ABI (include/magma_b200.h: mb200_gemm, mb200_layernorm_*, mb200_softmax_*, ...) plus the three
// helpers below. In the product the helpers are CUDA (common.cu). tests/ also compile the same schedule file as plain
// C++ against oracle/cabi_emul.cpp, a CPU emulation of those primitives, to dry-run the schedule (pointer arithmetic,
// leading dimensions, operand majors, accumulate flags) against the oracle without a GPU. That build is test
// infrastructure only; nothing in magma_b200/ loads it.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "../../include/magma_b200.h"

namespace mb200 {
void set_error(const char* fmt, ...);
int rt_check_arch();                                                   // 0 on sm_90, else MB200_E_ARCH
int rt_copy(void* dst, const void* src, size_t bytes, void* stream);   // device-to-device, stream-ordered
int rt_zero(void* dst, size_t bytes, void* stream);                    // stream-ordered memset(0)
}  // namespace mb200

#define MBS_REQUIRE(cond, code, ...)  \
  do {                                \
    if (!(cond)) {                    \
      mb200::set_error(__VA_ARGS__);  \
      return (code);                  \
    }                                 \
  } while (0)

#define MBS_TRY(expr)     \
  do {                    \
    int _rc = (expr);     \
    if (_rc) return _rc;  \
  } while (0)
