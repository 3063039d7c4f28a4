// The block-scale rule of every fp8 producer (K3's pack, the reduce's re-pack, K4's fp8 panel epilogue); bit-exact
// reference: ops/pack.py quantize_blocks.  A block of 32 values with amax a (an fmaxf reduction: NaN dropped) gets
//     e = the smallest integer with a / 2^e <= 448, clamped to [-127, 127]   (scale byte e + 127)
// and each value x becomes cvt.rn.satfinite.e4m3(x * 2^-e), except at e = 120: there codes above 240 would decode to
// 256 * 2^120 = 2^128 or more, which is Inf in fp32, so |x * 2^-e| > 240 saturates to 240 (NaN stays NaN).
#pragma once
#include <stdint.h>

// e from the fp32 bits of v = a * (1/448): exponent(v) + (mantissa(v) != 0).  A nonzero v at or below 2^-127 (fp32
// 0x00400000, a denormal) takes the clamp -127; read as exponent 0 plus a nonzero mantissa it would give -126.
__device__ __forceinline__ int mx_scale_exponent(float amax) {
  const uint32_t vb = __float_as_uint(amax * (1.0f / 448.0f));
  if (vb <= 0x00400000u) return -127;
  const int e = (int)((vb >> 23) & 0xff) - 127 + ((vb & 0x7fffffu) ? 1 : 0);
  return e < 127 ? e : 127;
}

// At e = 120 every scaled value is below 256 in magnitude (a finite fp32 is below 2^128), so the one code that decodes
// past fp32 max is 256 (0x78 / 0xF8), which values from 248 up round to: saturating |x * 2^-e| > 240 to 240 is the same
// as turning that code into 240 (0x77 / 0xF7).  This does it to the 4 codes packed in a word, cheaper in registers than
// clamping each fp32 value; NaN (0x7F / 0xFF) and every other code pass unchanged.
__device__ __forceinline__ uint32_t mx_saturate_codes(uint32_t q, int e) {
  const uint32_t t = (q & 0x7f7f7f7fu) ^ 0x78787878u;                   // a zero byte where the magnitude is 0x78
  const uint32_t z = ~((t + 0x7f7f7f7fu) | t | 0x7f7f7f7fu);            // 0x80 in each zero byte, no carries between bytes
  return e == 120 ? q - (z >> 7) : q;
}
