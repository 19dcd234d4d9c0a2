// TEST INFRASTRUCTURE — mb200_logits_grad_combine for the launch trace of the LM-training backward
// (tests/test_lm_train_cpu.py::lm_train_records): linked next to oracle/cabi_emul.cpp in place of
// tests/logits_grad_emul.cpp. While the emulation traces (placeholder pointers, nothing is dereferenced) it writes one
// JSON record per call to its own file and returns; outside a trace it refuses, since the computing emulation is the
// other file's. Nothing in magma_b200/ uses it.
#include <stdint.h>
#include <stdio.h>

#include "../include/magma_b200.h"

namespace mb200 {
void set_error(const char* fmt, ...);
}

extern "C" int mb200_emul_tracing(void);

static FILE* g_lg_rec = nullptr;
extern "C" void mb200_lm_train_record(const char* path) {
  if (g_lg_rec) fclose(g_lg_rec);
  g_lg_rec = path ? fopen(path, "w") : nullptr;
}

extern "C" int mb200_logits_grad_combine(const void* dce, int64_t ldv, const void* g, int64_t ld_g, void* out, int32_t M,
                                         int32_t V, float alpha, void*) {
  if (!mb200_emul_tracing()) {
    mb200::set_error("logits_grad_combine: this build only records launches");
    return MB200_E_ARG;
  }
  if (g_lg_rec)
    fprintf(g_lg_rec,
            "{\"op\":\"logits_grad_combine\",\"dce\":%llu,\"ldv\":%lld,\"g\":%llu,\"ld_g\":%lld,\"out\":%llu,\"M\":%d,"
            "\"V\":%d,\"alpha\":%.9g}\n",
            (unsigned long long)(uintptr_t)dce, (long long)ldv, (unsigned long long)(uintptr_t)g, (long long)ld_g,
            (unsigned long long)(uintptr_t)out, M, V, (double)alpha);
  return 0;
}
