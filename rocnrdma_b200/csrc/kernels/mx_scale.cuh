// The block-scale rule of every fp8 producer (K3's pack, the reduce's re-pack, K4's fp8 panel epilogue), and the decode
// of every fp8 consumer; bit-exact references: ops/pack.py quantize_blocks and ue8m0.  A block of 32 values with amax a (an fmaxf reduction: NaN dropped) gets
//     e = the smallest integer with a / 2^e <= 448, clamped to [-127, 127]   (scale byte e + 127)
// and each value x becomes cvt.rn.satfinite.e4m3(x * 2^-e), except at e = 120: there codes above 240 would decode to
// 256 * 2^120 = 2^128 or more, which is Inf in fp32, so |x * 2^-e| > 240 saturates to 240 (NaN stays NaN).
#pragma once
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <stdint.h>

// UE8M0 scale byte -> 2^(e - 127); byte 0 is 2^-127, an fp32 denormal (the OCP MX value), 0xFF is Inf
__device__ __forceinline__ float ue8m0(uint32_t e) { return e ? __uint_as_float(e << 23) : __uint_as_float(0x00400000u); }

// One 32-element block: q[i] holds the e4m3 codes of elements 4i..4i+3 (lowest byte first), `scale` its UE8M0 byte;
// out(k, d) takes the decode d of element k, in element order, four at a time as each code word is converted (a
// consumer that takes all 32 before using any holds them all in registers: one reduce variant then spills).  Each code
// is exact in half and in fp32; the one rounding is __fmul_rn by the scale, which the compiler may not contract into an
// FMA with what out() does next.
template <class Out>
__device__ __forceinline__ void mx_decode_block32(const uint32_t (&q)[8], uint32_t scale, Out out) {
  const float sc = ue8m0(scale);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    __half2_raw h0 = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(q[i] & 0xffff), __NV_E4M3);
    __half2_raw h1 = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(q[i] >> 16), __NV_E4M3);
    const float2 f0 = __half22float2(*reinterpret_cast<__half2*>(&h0));
    const float2 f1 = __half22float2(*reinterpret_cast<__half2*>(&h1));
    out(4 * i, __fmul_rn(f0.x, sc));
    out(4 * i + 1, __fmul_rn(f0.y, sc));
    out(4 * i + 2, __fmul_rn(f1.x, sc));
    out(4 * i + 3, __fmul_rn(f1.y, sc));
  }
}

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
