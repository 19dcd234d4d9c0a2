// TEST INFRASTRUCTURE — CPU emulation of the two attention entry points that output_attentions adds to the C ABI,
// linked by tests/test_attentions_cpu.py next to oracle/cabi_emul.cpp (the emulation of every other primitive) and the
// host-only schedules, so the schedule's CPU build runs every output_attentions path. Nothing in magma_b200/ uses it.
//   mb200_attn_bwd_tile_dp   attention.cu: attn_bwd_tile_kernel<HD, true>
//   mb200_attn_decode_probs  kv_attention.cu: attn_decode_kernel<true>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../include/magma_b200.h"

namespace mb200 {
void set_error(const char* fmt, ...);
}

namespace {

typedef uint16_t bf16_t;

float b2f(bf16_t v) {
  uint32_t u = (uint32_t)v << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}

bf16_t f2b(float f) {  // round to nearest even, like __float2bfloat16_rn
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (bf16_t)((u >> 16) | 0x40);
  return (bf16_t)((u + 0x7fffu + ((u >> 16) & 1u)) >> 16);
}

}  // namespace

#define AE_REQUIRE(cond, code, ...) \
  do {                              \
    if (!(cond)) {                  \
      mb200::set_error(__VA_ARGS__); \
      return (code);                \
    }                               \
  } while (0)

extern "C" {

// per (batch, head): dP = dO V^T + dP_ext (rows and columns < S of dP_ext read), D = rowsum(dP * P),
// dS = bf16(P (dP - D) / sqrt(hd)), dQ = dS K, dK = dS^T Q (inverse rotary through rope_tab when given), dV = P^T dO
int mb200_attn_bwd_tile_dp(const void* qkv_, int64_t ld, const void* dO_, int64_t ld_do, const void* P_, int64_t ldP,
                           const void* dPe_, int64_t ld_dpe, void* dqkv_, int64_t ldd, const float* rope_tab, int32_t rot,
                           int32_t B, int32_t S, int32_t H, int32_t hd, void*) {
  AE_REQUIRE(S >= 1 && S <= 128 && hd >= 64 && hd <= 256 && hd % 64 == 0 && ldP % 8 == 0, MB200_E_SHAPE,
             "attn_bwd_tile: unsupported S=%d hd=%d", S, hd);
  AE_REQUIRE(dPe_ != nullptr, MB200_E_ARG, "attn_bwd_tile_dp: dP_ext is NULL");
  AE_REQUIRE(ld_dpe >= S && ld_dpe % 8 == 0, MB200_E_ALIGN, "attn_bwd_tile_dp: ld_dpe=%lld must be >= S and %%8",
             (long long)ld_dpe);
  const bf16_t *qkv = (const bf16_t*)qkv_, *dO = (const bf16_t*)dO_, *P = (const bf16_t*)P_, *dPe = (const bf16_t*)dPe_;
  bf16_t* dqkv = (bf16_t*)dqkv_;
  const long long d = (long long)H * hd;
  const float scale = 1.f / sqrtf((float)hd);
  std::vector<float> dS((size_t)S * S), dq((size_t)S * hd), dk((size_t)S * hd), dv((size_t)S * hd);
  for (long long b = 0; b < B; ++b)
    for (int h = 0; h < H; ++h) {
      auto Q = [&](int i, int c) { return b2f(qkv[(b * S + i) * ld + (long long)h * hd + c]); };
      auto K = [&](int i, int c) { return b2f(qkv[(b * S + i) * ld + d + (long long)h * hd + c]); };
      auto V = [&](int i, int c) { return b2f(qkv[(b * S + i) * ld + 2 * d + (long long)h * hd + c]); };
      auto G = [&](int i, int c) { return b2f(dO[(b * S + i) * ld_do + (long long)h * hd + c]); };
      auto Pr = [&](int i, int j) { return b2f(P[((b * H + h) * S + i) * ldP + j]); };
      for (int i = 0; i < S; ++i) {
        float dot = 0.f;
        for (int j = 0; j < S; ++j) {
          float dp = 0.f;
          for (int c = 0; c < hd; ++c) dp += G(i, c) * V(j, c);
          dp += b2f(dPe[((b * H + h) * S + i) * ld_dpe + j]);
          dS[(size_t)i * S + j] = dp;
          dot += dp * Pr(i, j);
        }
        for (int j = 0; j < S; ++j)
          dS[(size_t)i * S + j] = b2f(f2b(Pr(i, j) * (dS[(size_t)i * S + j] - dot) * scale));
      }
      for (int i = 0; i < S; ++i)
        for (int c = 0; c < hd; ++c) {
          float aq = 0.f, ak = 0.f, av = 0.f;
          for (int j = 0; j < S; ++j) {
            aq += dS[(size_t)i * S + j] * K(j, c);
            ak += dS[(size_t)j * S + i] * Q(j, c);
            av += Pr(j, i) * G(j, c);
          }
          dq[(size_t)i * hd + c] = aq;
          dk[(size_t)i * hd + c] = ak;
          dv[(size_t)i * hd + c] = av;
        }
      for (int i = 0; i < S; ++i) {
        if (rope_tab)
          for (int p = 0; p < rot / 2; ++p) {
            const float cs = rope_tab[((long long)i * (rot / 2) + p) * 2], sn = rope_tab[((long long)i * (rot / 2) + p) * 2 + 1];
            for (std::vector<float>* t : {&dq, &dk}) {
              float& x0 = (*t)[(size_t)i * hd + 2 * p];
              float& x1 = (*t)[(size_t)i * hd + 2 * p + 1];
              const float a = x0, c2 = x1;
              x0 = a * cs + c2 * sn;
              x1 = c2 * cs - a * sn;
            }
          }
        for (int c = 0; c < hd; ++c) {
          dqkv[(b * S + i) * ldd + (long long)h * hd + c] = f2b(dq[(size_t)i * hd + c]);
          dqkv[(b * S + i) * ldd + d + (long long)h * hd + c] = f2b(dk[(size_t)i * hd + c]);
          dqkv[(b * S + i) * ldd + 2 * d + (long long)h * hd + c] = f2b(dv[(size_t)i * hd + c]);
        }
      }
    }
  return 0;
}

// the decode step itself is mb200_attn_decode's (append at pos, softmax over [0, pos], P V); its probabilities
// bf16(exp(s_j - m) / sum) go to row b*H + h of probs, zeros from column pos + 1 on
int mb200_attn_decode_probs(const void* qkv_, int64_t ld_qkv, void* kc_, void* vc_, void* out_, int64_t ld_out,
                            void* probs_, int64_t ld_probs, int32_t B, int32_t H, int32_t hd, int32_t Smax, int32_t pos,
                            void* st) {
  AE_REQUIRE(probs_ != nullptr && ld_probs > pos, MB200_E_ARG, "attn_decode_probs: ld_probs=%lld must be > pos=%d",
             (long long)ld_probs, pos);
  const int rc = mb200_attn_decode(qkv_, ld_qkv, kc_, vc_, out_, ld_out, B, H, hd, Smax, pos, st);
  if (rc) return rc;
  const bf16_t* qkv = (const bf16_t*)qkv_;
  const bf16_t* kc = (const bf16_t*)kc_;
  bf16_t* probs = (bf16_t*)probs_;
  const float scale = 1.f / sqrtf((float)hd);
  std::vector<float> sc(pos + 1);
  for (long long b = 0; b < B; ++b)
    for (int h = 0; h < H; ++h) {
      const bf16_t* q = qkv + b * ld_qkv + (long long)h * hd;
      const bf16_t* kb = kc + ((b * H + h) * (long long)Smax) * hd;
      float m = -INFINITY, sum = 0.f;
      for (int j = 0; j <= pos; ++j) {
        float acc = 0.f;
        for (int c = 0; c < hd; ++c) acc += b2f(kb[(long long)j * hd + c]) * b2f(q[c]);
        sc[j] = acc * scale;
        m = fmaxf(m, sc[j]);
      }
      for (int j = 0; j <= pos; ++j) {
        sc[j] = expf(sc[j] - m);
        sum += sc[j];
      }
      bf16_t* row = probs + (b * H + h) * ld_probs;
      for (long long j = 0; j < ld_probs; ++j) row[j] = f2b(j <= pos ? sc[j] / sum : 0.f);
    }
  return 0;
}

}  // extern "C"
