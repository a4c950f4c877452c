// navillm_b200 — fp8 (OCP e4m3fn) weight format of the decode step: one power-of-two scale per weight row.
//
//   W'[n, k] = e4m3(W[n, k] / 2^e_n) * 2^e_n,   e_n = the smallest integer with max_k |W[n, k]| / 2^e_n <= 448
//
// (all-zero row: e_n = 0).  With max|W[n,:]| = m * 2^x, m in [0.5, 1): e_n = x - 9 if m <= 0.875 else x - 8, because
// 448 = 0.875 * 2^9.  e_n is clamped below at NV_FP8_EXP_MIN so that every non-zero W' (>= 2^-9 * 2^e_n) is an fp32 / bf16
// normal number: then the scale is an exact power of two in both directions, W' is exactly representable in bf16, and
// flush-to-zero arithmetic cannot change it.  Only rows with max|W| < 2^-108 are affected by the clamp.
// The quantizer (quant.cu) and the fp8 GEMMs (gemm_skinny.cu, gemm_bf16.cu) expand e4m3 to bf16 with the same function below,
// so a GEMM's bf16 operand is bit for bit the W' the quantizer wrote back.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace nv {

constexpr int NV_FP8_EXP_MIN = -117;

// e_n from the row's amax (a non-negative finite float)
__device__ __forceinline__ int fp8_row_exponent(float amax) {
  const uint32_t b = __float_as_uint(amax);
  if (b == 0u) return 0;
  const uint32_t bexp = b >> 23, mant = b & 0x7FFFFFu;
  if (bexp == 0u) return NV_FP8_EXP_MIN;                     // fp32 subnormal amax: far below the clamp
  const int x = (int)bexp - 126;                             // amax = m * 2^x with m = 1.mant / 2 in [0.5, 1)
  const int e = mant <= 0x600000u ? x - 9 : x - 8;           // m <= 0.875  <=>  1.mant <= 1.75
  return e < NV_FP8_EXP_MIN ? NV_FP8_EXP_MIN : e;
}

// 2^e as a float (e in [NV_FP8_EXP_MIN, 127])
__device__ __forceinline__ float fp8_pow2(int e) { return __uint_as_float((uint32_t)(e + 127) << 23); }

// four fp32 values (already divided by 2^e_n) -> four e4m3 bytes, round to nearest even, saturating; v0 in the lowest
// byte.  The 16-bit halves stay inside the asm: the packed register is what the callers load and store.
__device__ __forceinline__ uint32_t fp8x4_from_f32(float v0, float v1, float v2, float v3) {
  uint32_t r;
  asm("{\n\t.reg .b16 lo, hi;\n\t"
      "cvt.rn.satfinite.e4m3x2.f32 lo, %2, %1;\n\t"        // a -> upper byte, b -> lower byte
      "cvt.rn.satfinite.e4m3x2.f32 hi, %4, %3;\n\t"
      "mov.b32 %0, {lo, hi};\n\t}"
      : "=r"(r) : "f"(v0), "f"(v1), "f"(v2), "f"(v3));
  return r;
}

// four e4m3 bytes (lowest byte = lowest address) -> two bf16x2 words of e4m3 * scale (scale = 2^e_n; exact, see above)
__device__ __forceinline__ void fp8x4_to_bf16x4(uint32_t q, float scale, uint32_t& lo, uint32_t& hi) {
  uint32_t h0, h1;
  asm("{\n\t.reg .b16 a, b;\n\t"
      "mov.b32 {a, b}, %2;\n\t"
      "cvt.rn.f16x2.e4m3x2 %0, a;\n\t"
      "cvt.rn.f16x2.e4m3x2 %1, b;\n\t}"
      : "=r"(h0), "=r"(h1) : "r"(q));
  const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&h0));
  const float2 f1 = __half22float2(*reinterpret_cast<const __half2*>(&h1));
  __nv_bfloat162 v0 = __floats2bfloat162_rn(f0.x * scale, f0.y * scale);
  __nv_bfloat162 v1 = __floats2bfloat162_rn(f1.x * scale, f1.y * scale);
  lo = *reinterpret_cast<uint32_t*>(&v0);
  hi = *reinterpret_cast<uint32_t*>(&v1);
}

// The row-quantize step shared by the weight quantizer (quant.cu) and the fp8 KV cache (decode.cu).
// |x| of eight bf16 values as 15-bit patterns (|x| orders like them): the per-lane part of a row's amax.  The row's amax is
// the max over its lanes, and its exponent is fp8_row_exponent(__uint_as_float(amax_bits << 16)).
__device__ __forceinline__ uint32_t bf16x8_amax_bits(const uint4& v) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
  uint32_t m = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) m = max(m, max(w[j] & 0x7FFFu, (w[j] >> 16) & 0x7FFFu));
  return m;
}

// eight bf16 values of a row with exponent e (inv = 2^-e) -> eight e4m3 bytes (lowest element in the lowest byte)
__device__ __forceinline__ uint2 fp8x8_from_bf16x8(const uint4& v, float inv) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
  uint32_t q[2];
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const uint32_t a = w[2 * j], b = w[2 * j + 1];
    q[j] = fp8x4_from_f32(__uint_as_float(a << 16) * inv, __uint_as_float(a & 0xffff0000u) * inv, __uint_as_float(b << 16) * inv,
                          __uint_as_float(b & 0xffff0000u) * inv);
  }
  return make_uint2(q[0], q[1]);
}

// four e4m3 bytes -> the four fp32 values of e4m3 * scale (scale = 2^e): the values fp8x4_to_bf16x4 rounds to bf16, which
// that rounding keeps exactly (see above), so they equal the fp32 widening of the bf16 W'.
__device__ __forceinline__ void fp8x4_to_f32x4(uint32_t q, float scale, float* f) {
  uint32_t h0, h1;
  asm("{\n\t.reg .b16 a, b;\n\t"
      "mov.b32 {a, b}, %2;\n\t"
      "cvt.rn.f16x2.e4m3x2 %0, a;\n\t"
      "cvt.rn.f16x2.e4m3x2 %1, b;\n\t}"
      : "=r"(h0), "=r"(h1) : "r"(q));
  const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&h0));
  const float2 f1 = __half22float2(*reinterpret_cast<const __half2*>(&h1));
  f[0] = f0.x * scale; f[1] = f0.y * scale; f[2] = f1.x * scale; f[3] = f1.y * scale;
}

}  // namespace nv
