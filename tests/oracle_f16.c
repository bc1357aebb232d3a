/*
 * oracle_f16.c — CPU restatement of the two fp16 modes of the data plane (include/b200ddp.h: B2_F32_WIRE_F16 = 3,
 * B2_F16 = 4).  TEST INFRASTRUCTURE ONLY, the fp16 twin of oracle/allreduce_oracle.c; loaded through tests/_oracle_f16.py.
 *
 *   mode 3  torch/distributed/algorithms/ddp_comm_hooks/default_hooks.py `fp16_compress_hook` (`_compress_hook`):
 *             compressed = buffer.to(float16).div_(world_size) -> all_reduce(SUM) -> buffer.copy_(compressed)
 *           c_r = f16(float(f16(x)) * scale),  out = float(f16(s))
 *   mode 4  allreduce_hook / the hook-less Reducer on an fp16 bucket:  c_r = f16(float(x) * scale),  out = f16(s)
 *
 * s is the fp32 sum of the c_r in rank order starting from c_0, exactly as in the other modes.  Every fp16 rounding is
 * IEEE binary16 round-to-nearest-even written out by bit manipulation (no compiler _Float16, so the result does not
 * depend on the compiler): subnormals are kept, overflow goes to +-inf, a NaN stays a NaN.
 */
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#define B2O_F32_WIRE_F16 3
#define B2O_F16 4

static inline uint32_t f2u(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
}
static inline float u2f(uint32_t u) {
  float f;
  memcpy(&f, &u, 4);
  return f;
}

/* fp32 -> fp16 bits, round to nearest even.  NaN -> 0x7fff (what `cvt.rn.f16x2.f32` produces; tests compare NaNs as
 * NaNs, not by payload). */
uint16_t b2o_f16_rne(float f) {
  const uint32_t u = f2u(f);
  const uint16_t sign = (uint16_t)((u >> 16) & 0x8000u);
  const uint32_t a = u & 0x7fffffffu;
  if (a > 0x7f800000u) return 0x7fffu;
  if (a >= 0x477ff000u) return sign | 0x7c00u; /* >= 65520 = 65504 + half an ulp (a tie, to the even neighbour 2^16): inf */
  if (a >= 0x38800000u) {                      /* >= 2^-14: an fp16 normal */
    uint32_t h = (a >> 13) - ((uint32_t)(127 - 15) << 10);
    const uint32_t rem = a & 0x1fffu;
    if (rem > 0x1000u || (rem == 0x1000u && (h & 1u))) ++h; /* a carry into the exponent is the right result */
    return sign | (uint16_t)h;
  }
  /* fp16 subnormal (or zero): the result is round(|f| * 2^24) units of 2^-24 */
  const uint32_t e = a >> 23;
  if (e < 102) return sign; /* |f| < 2^-25: below half the smallest subnormal */
  const uint32_t m = (a & 0x7fffffu) | 0x800000u;
  const uint32_t shift = 126 - e; /* 14 .. 24 */
  uint32_t q = m >> shift;
  const uint32_t rem = m & ((1u << shift) - 1u), half = 1u << (shift - 1u);
  if (rem > half || (rem == half && (q & 1u))) ++q; /* q == 0x400 is the smallest normal: also the right encoding */
  return sign | (uint16_t)q;
}

/* fp16 bits -> fp32, exact (a NaN keeps its sign and payload). */
float b2o_f16_to_f32(uint16_t h) {
  const uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
  const uint32_t exp = (h >> 10) & 0x1fu;
  uint32_t man = h & 0x3ffu;
  if (exp == 0x1f) return u2f(sign | 0x7f800000u | (man << 13));
  if (exp == 0) {
    if (man == 0) return u2f(sign);
    int e = -14; /* subnormal: normalise */
    while (!(man & 0x400u)) {
      man <<= 1;
      --e;
    }
    return u2f(sign | ((uint32_t)(e + 127) << 23) | ((man & 0x3ffu) << 13));
  }
  return u2f(sign | ((exp - 15 + 127) << 23) | (man << 13));
}

static inline float f16_round(float f) { return b2o_f16_to_f32(b2o_f16_rne(f)); }

/* wire(scale * x): one rank's contribution as the fp32 value of the fp16 wire element.  `x_bits`: fp32 bits (mode 3) or
 * fp16 bits in the low half (mode 4). */
static inline float compress1(int mode, uint32_t x_bits, float scale) {
  const float a = mode == B2O_F32_WIRE_F16 ? f16_round(u2f(x_bits)) /* the .to(float16) cast */
                                           : b2o_f16_to_f32((uint16_t)x_bits);
  return f16_round(a * scale); /* the div_ result, rounded to fp16 */
}

/* Returns 0, or -1 on a mode that is not one of the two fp16 modes. */
int b2o_f16_compress(int mode, const void* in, size_t n, float scale, float* out_f32) {
  if (mode != B2O_F32_WIRE_F16 && mode != B2O_F16) return -1;
  for (size_t i = 0; i < n; ++i) {
    const uint32_t bits = mode == B2O_F16 ? ((const uint16_t*)in)[i] : ((const uint32_t*)in)[i];
    out_f32[i] = compress1(mode, bits, scale);
  }
  return 0;
}

/* in[r]: rank r's n-element bucket (fp32 for mode 3, fp16 bits for mode 4); out: what every rank ends up with, in the
 * bucket's dtype.  Returns 0, or -1 on a bad mode / world. */
int b2o_f16_allreduce(int mode, int world, const void* const* in, size_t n, float scale, void* out) {
  if ((mode != B2O_F32_WIRE_F16 && mode != B2O_F16) || world < 1) return -1;
  for (size_t i = 0; i < n; ++i) {
    float s = 0.f;
    for (int r = 0; r < world; ++r) {
      const uint32_t bits = mode == B2O_F16 ? ((const uint16_t*)in[r])[i] : ((const uint32_t*)in[r])[i];
      const float c = compress1(mode, bits, scale);
      s = r == 0 ? c : s + c; /* start from rank 0's value: keeps -0.0 */
    }
    if (mode == B2O_F32_WIRE_F16)
      ((float*)out)[i] = f16_round(s);
    else
      ((uint16_t*)out)[i] = b2o_f16_rne(s);
  }
  return 0;
}
