// TEST INFRASTRUCTURE (see cuda_runtime.h in this directory): IEEE binary16 storage type with round-to-nearest-even
// conversions (subnormals, overflow to infinity, NaN), the two the engine's kernels use.
#pragma once
#include <cstdint>
#include <cstring>
struct __half { uint16_t x; };
static inline __half __float2half_rn(float f) {
  uint32_t u; memcpy(&u, &f, 4);
  const uint16_t sign = (uint16_t)((u >> 16) & 0x8000u);
  const uint32_t a = u & 0x7fffffffu;
  __half r;
  if (a > 0x7f800000u) { r.x = (uint16_t)(sign | 0x7e00u); return r; }          // NaN
  if (a >= 0x38800000u) {                                                        // half normal range (|f| >= 2^-14)
    uint32_t m = a - 0x38000000u;                                                // exponent bias 127 -> 15
    m += 0xfffu + ((m >> 13) & 1u);                                              // nearest-even at bit 13
    m >>= 13;
    r.x = (uint16_t)(sign | (m >= 0x7c00u ? 0x7c00u : m));                       // overflow (and inf) -> inf
    return r;
  }
  const int e = (int)(a >> 23);
  if (e < 102) { r.x = sign; return r; }                                         // |f| < 2^-25: rounds to zero
  const uint32_t mant = (a & 0x7fffffu) | 0x800000u;                             // subnormal: units of 2^-24
  const int shift = 126 - e;                                                     // 14 .. 24
  uint32_t q = mant >> shift;
  const uint32_t rem = mant & ((1u << shift) - 1u), halfway = 1u << (shift - 1);
  if (rem > halfway || (rem == halfway && (q & 1u))) ++q;                        // may carry into the smallest normal
  r.x = (uint16_t)(sign | q);
  return r;
}
static inline float __half2float(__half h) {
  const uint32_t s = (uint32_t)(h.x & 0x8000u) << 16;
  uint32_t e = (h.x >> 10) & 0x1fu, m = h.x & 0x3ffu, u;
  if (e == 0x1fu) u = s | 0x7f800000u | (m << 13);                               // inf / NaN
  else if (e != 0) u = s | ((e + 112u) << 23) | (m << 13);
  else if (m == 0) u = s;
  else {                                                                         // subnormal: normalise
    e = 113;
    while (!(m & 0x400u)) { m <<= 1; --e; }
    u = s | (e << 23) | ((m & 0x3ffu) << 13);
  }
  float f; memcpy(&f, &u, 4);
  return f;
}
