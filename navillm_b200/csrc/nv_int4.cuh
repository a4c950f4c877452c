// navillm_b200 — the 4-bit group-wise weight format (W4A16) of the decode step: rule and packed code layout.
//
// Rule (include/navillm_b200.h, restated in tests/test_int4_quant_cpu.py): one group is a weight row n and 128 consecutive
// columns.  In fp32 from the bf16 values, with IEEE division and round-half-even rint:
//   lo = min(0, min w), hi = max(0, max w), s = max(bf16_rn((hi - lo) / 15), 2^-126), z = clamp(rint(-lo / s), 0, 15),
//   q = clamp(rint(w / s) + z, 0, 15), W' = bf16_rn((q - z) * s)
// (q - z) * s is exact in fp32, so W' is rounded once; |q - z| >= 1 and s >= 2^-126 keep every nonzero W' normal.  The
// library is built with --use_fast_math (subnormals flushed), so the fp32 steps below are inline PTX without .ftz: a
// group holding bf16 subnormals gets the bits of the rule.
// GPTQ (nv_gptq_int4_block) applies the same rule to the fp32 error-updated weights of the group instead of the bf16 ones:
// lo, hi, s and z come from the row's 128 values as they stand when the group's block starts, and each q from the value
// as it stands when its column is reached.
//
// Packed codes (private to csrc/quant.cu and csrc/gemm_skinny.cu): W [N, K] is cut into chunks of 64 rows x 64 columns;
// chunk (rb, kb) = rows 64 rb.., columns 64 kb.. is 2048 bytes at byte offset (rb * K / 64 + kb) * 2048, so the codes of
// weights stacked along N (q|k|v, gate|up) are the concatenation of theirs when each has a multiple of 64 rows.  Inside a
// chunk, bytes 16 t .. 16 t + 15 are what thread t = 32 w + l of the skinny GEMM's consumer warpgroup needs for its four
// m64n16k16 register-A fragments: word j (k16 step j) holds, with r0 = 16 w + l / 4, r1 = r0 + 8, c = 16 j + 2 (l % 4),
// the pairs p = 0: (r0, c), 1: (r1, c), 2: (r0, c + 8), 3: (r1, c + 8) (the order of the fragment registers a[0..3]),
// element e (column + e) of pair p in nibble p + 4 e.  So (word >> 4 p) & 0x000f000f puts pair p's codes in the low
// bits of the two bf16 halves of a register.
#pragma once
#include <stdint.h>

namespace nv {

constexpr uint32_t Q4_GROUP = 128;        // columns per group (one bf16 scale and one 4-bit zero-point each)
constexpr uint32_t Q4_CHUNK_BYTES = 2048; // one 64 x 64 chunk of codes

// ---- the rule, fp32 without flush-to-zero ----
__device__ __forceinline__ float q4_min(float a, float b) { float r; asm("min.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ float q4_max(float a, float b) { float r; asm("max.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ float q4_sub(float a, float b) { float r; asm("sub.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ float q4_div(float a, float b) { float r; asm("div.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ float q4_mul(float a, float b) { float r; asm("mul.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ float q4_fma(float a, float b, float c) { float r; asm("fma.rn.f32 %0, %1, %2, %3;" : "=f"(r) : "f"(a), "f"(b), "f"(c)); return r; }
__device__ __forceinline__ int q4_rint(float a) { int r; asm("cvt.rni.s32.f32 %0, %1;" : "=r"(r) : "f"(a)); return r; }
__device__ __forceinline__ uint16_t q4_bf16_bits(float a) { uint16_t r; asm("cvt.rn.bf16.f32 %0, %1;" : "=h"(r) : "f"(a)); return r; }
__device__ __forceinline__ float q4_bf16_float(uint32_t bits) { return __uint_as_float(bits << 16); }

// scale (as the float value of its bf16) and zero-point of a group with lo = min(0, min w), hi = max(0, max w)
__device__ __forceinline__ void q4_group_params(float lo, float hi, float& s, int& z) {
  s = q4_max(q4_bf16_float(q4_bf16_bits(q4_div(q4_sub(hi, lo), 15.f))), 1.17549435e-38f);   // 2^-126
  z = min(max(-q4_rint(q4_div(lo, s)), 0), 15);            // rint is odd-symmetric: rint(-lo / s) = -rint(lo / s)
}
__device__ __forceinline__ int q4_code(float w, float s, int z) { return min(max(q4_rint(q4_div(w, s)) + z, 0), 15); }
__device__ __forceinline__ uint16_t q4_value_bits(int q, int z, float s) { return q4_bf16_bits(q4_mul((float)(q - z), s)); }

// ---- the one writer of the packed layout ----
// Thread t (0..127) of the quantizer writes bytes 16 t .. 16 t + 15 of both 64-column chunks of one 64-row block and
// 128-column group: chunks chunk0 (columns 0..63) and chunk0 + 1 (64..127) of codes.  code(r, c) is the 4-bit code of
// row r (0..63) and column c (0..127) of the block; thread t reads rows 16 (t / 32) .. 16 (t / 32) + 15 only.
template <class Code>
__device__ __forceinline__ void q4_pack_group(int t, uint8_t* __restrict__ codes, int64_t chunk0, Code code) {
  const int warp = t >> 5, lane = t & 31;
  const int r0 = warp * 16 + (lane >> 2);
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    uint32_t words[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint32_t word = 0;
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        const int r = r0 + 8 * (p & 1);
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = 64 * half + 16 * j + 2 * (lane & 3) + 8 * (p >> 1) + e;
          word |= (uint32_t)code(r, c) << (4 * (p + 4 * e));
        }
      }
      words[j] = word;
    }
    const int64_t chunk = chunk0 + half;
    *reinterpret_cast<uint4*>(codes + chunk * Q4_CHUNK_BYTES + 16 * t) = make_uint4(words[0], words[1], words[2], words[3]);
  }
}

// ---- dequantization into a register-A fragment (skinny GEMM) ----
// sx: the bf16 scale in both halves; zx: bf16(128 + z) in both halves.  0x4300 | q is bf16(128 + q), the subtraction is
// exact and the one rounding is the bf16 multiply's: bf16_rn((q - z) * s), the W' of the rule.
__device__ __forceinline__ uint32_t q4_dequant_pair(uint32_t word, uint32_t shift, uint32_t sx, uint32_t zx) {
  const uint32_t v = ((word >> shift) & 0x000f000fu) | 0x43004300u;
  uint32_t d, r;
  asm("sub.rn.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(v), "r"(zx));
  asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(r) : "r"(d), "r"(sx));
  return r;
}
// the four fragment registers of one k16 step from word j of the thread's 16 bytes (rows r0 / r1: scales s0x / s1x)
__device__ __forceinline__ void q4_dequant_k16(uint32_t word, uint32_t s0x, uint32_t z0x, uint32_t s1x, uint32_t z1x,
                                               uint32_t (&a)[4]) {
  a[0] = q4_dequant_pair(word, 0, s0x, z0x);
  a[1] = q4_dequant_pair(word, 4, s1x, z1x);
  a[2] = q4_dequant_pair(word, 8, s0x, z0x);
  a[3] = q4_dequant_pair(word, 12, s1x, z1x);
}

}  // namespace nv
