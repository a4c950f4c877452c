// navillm_b200 — weight quantizers for the decode step: fp8 (e4m3) rows (format: nv_fp8.cuh) and 4-bit groups
// (format: nv_int4.cuh, below).
//
// fp8: one CTA per weight row: the row's amax (on the bf16 bit patterns: |x| orders like its 15 low bits), the exponent e_n,
// then one more pass that writes the e4m3 bytes and W' = e4m3 * 2^e_n back over the bf16 row, so the model that remains
// is exactly the one the fp8 kernels compute with.
#include "nv_common.cuh"
#include "nv_fp8.cuh"
#include "nv_host.h"
#include "nv_int4.cuh"

namespace nv {

constexpr int QZ_THREADS = 256;

__global__ void __launch_bounds__(QZ_THREADS)
quantize_fp8_rows_kernel(__nv_bfloat16* __restrict__ W, int64_t ldw, uint8_t* __restrict__ Q, int64_t ldq,
                         int8_t* __restrict__ exps, int K) {
  __shared__ uint32_t red[QZ_THREADS / 32];
  const int64_t n = blockIdx.x;
  uint4* wrow = reinterpret_cast<uint4*>(W + n * ldw);
  const int nvec = K >> 3;                                   // 8 bf16 per 16-byte vector
  uint32_t m = 0;
  for (int i = threadIdx.x; i < nvec; i += QZ_THREADS) m = max(m, bf16x8_amax_bits(wrow[i]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = 0;
#pragma unroll
  for (int i = 0; i < QZ_THREADS / 32; ++i) m = max(m, red[i]);
  const int e = fp8_row_exponent(__uint_as_float(m << 16));
  const float inv = fp8_pow2(-e), scale = fp8_pow2(e);
  if (threadIdx.x == 0) exps[n] = (int8_t)e;
  uint2* qrow = reinterpret_cast<uint2*>(Q + n * ldq);
  for (int i = threadIdx.x; i < nvec; i += QZ_THREADS) {
    const uint2 q = fp8x8_from_bf16x8(wrow[i], inv);
    uint32_t o[4];
    fp8x4_to_bf16x4(q.x, scale, o[0], o[1]);
    fp8x4_to_bf16x4(q.y, scale, o[2], o[3]);
    qrow[i] = q;
    wrow[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// int4 groups (nv_int4.cuh): one CTA per 64-row block and 128-column group.  The tile is staged in shared memory; warp w
// reduces rows 16 w .. 16 w + 15 to their (s, z), then thread t builds the two chunks' words it would read in the GEMM
// and overwrites each element with W' (every element is visited by exactly one thread).
constexpr int Q4_THREADS = 128;

__global__ void __launch_bounds__(Q4_THREADS)
quantize_int4_groups_kernel(__nv_bfloat16* __restrict__ W, int64_t ldw, uint8_t* __restrict__ codes,
                            __nv_bfloat16* __restrict__ scales, uint8_t* __restrict__ zeros, int N, int K) {
  __shared__ __align__(16) uint16_t tile[64][Q4_GROUP + 8];
  __shared__ float s_scale[64];
  __shared__ int s_zero[64];
  const int rb = blockIdx.x, g = blockIdx.y, G = K / (int)Q4_GROUP;
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  for (int i = t; i < 64 * 16; i += Q4_THREADS) {           // 16 vectors of 8 bf16 per row
    const int r = i >> 4, c = (i & 15) * 8, n = rb * 64 + r;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (n < N) v = *reinterpret_cast<const uint4*>(W + n * ldw + (int64_t)g * Q4_GROUP + c);
    *reinterpret_cast<uint4*>(&tile[r][c]) = v;
  }
  __syncthreads();
  for (int rr = 0; rr < 16; ++rr) {
    const int r = warp * 16 + rr;
    float lo = 0.f, hi = 0.f;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float x = q4_bf16_float(tile[r][4 * lane + e]);
      lo = q4_min(lo, x);
      hi = q4_max(hi, x);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo = q4_min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
      hi = q4_max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    if (lane == 0) {
      float s;
      int z;
      q4_group_params(lo, hi, s, z);
      s_scale[r] = s;
      s_zero[r] = z;
      const int n = rb * 64 + r;
      if (n < N) {
        scales[(int64_t)n * G + g] = __ushort_as_bfloat16(q4_bf16_bits(s));
        zeros[(int64_t)n * G + g] = (uint8_t)z;
      }
    }
  }
  __syncthreads();
  const int r0 = warp * 16 + (lane >> 2);
#pragma unroll
  for (int half = 0; half < 2; ++half) {                    // the group's two 64-column chunks
    uint32_t words[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint32_t word = 0;
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        const int r = r0 + 8 * (p & 1);
        const float s = s_scale[r];
        const int z = s_zero[r];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = 64 * half + 16 * j + 2 * (lane & 3) + 8 * (p >> 1) + e;
          const int q = q4_code(q4_bf16_float(tile[r][c]), s, z);
          tile[r][c] = q4_value_bits(q, z, s);
          word |= (uint32_t)q << (4 * (p + 4 * e));
        }
      }
      words[j] = word;
    }
    const int64_t chunk = (int64_t)rb * (K / 64) + 2 * g + half;
    *reinterpret_cast<uint4*>(codes + chunk * Q4_CHUNK_BYTES + 16 * t) = make_uint4(words[0], words[1], words[2], words[3]);
  }
  __syncthreads();
  for (int i = t; i < 64 * 16; i += Q4_THREADS) {
    const int r = i >> 4, c = (i & 15) * 8, n = rb * 64 + r;
    if (n < N) *reinterpret_cast<uint4*>(W + n * ldw + (int64_t)g * Q4_GROUP + c) = *reinterpret_cast<const uint4*>(&tile[r][c]);
  }
}

}  // namespace nv

// Quantize the bf16 weight W [N, K] to 4-bit codes in groups of 128 columns (rule and layout: nv_int4.cuh): codes
// (ceil(N / 64) * 64 * K / 2 bytes, packed for the skinny GEMM; rows >= N hold code 0), scales [N, K / 128] bf16 and
// zeros [N, K / 128] uint8 (0..15), and W overwritten in place with W' = bf16((q - z) * s).  K % 128 == 0.
extern "C" int nv_quantize_int4_groups(void* W, int64_t ldw, void* codes, void* scales, void* zeros, int N, int K,
                                       void* stream_) {
  using namespace nv;
  NV_REQUIRE(N > 0 && K > 0 && (K % (int)Q4_GROUP) == 0, "nv_quantize_int4_groups: needs N > 0 and K %% 128 == 0 (got N=%d K=%d)",
             N, K);
  NV_REQUIRE(W && codes && scales && zeros, "nv_quantize_int4_groups: null operand");
  NV_REQUIRE((ldw & 7) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0 && (reinterpret_cast<uintptr_t>(codes) & 15) == 0,
             "nv_quantize_int4_groups: W / codes must be 16-byte aligned with ldw %% 8 == 0");
  quantize_int4_groups_kernel<<<dim3((N + 63) / 64, K / Q4_GROUP), Q4_THREADS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      reinterpret_cast<__nv_bfloat16*>(W), ldw, reinterpret_cast<uint8_t*>(codes), reinterpret_cast<__nv_bfloat16*>(scales),
      reinterpret_cast<uint8_t*>(zeros), N, K);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

// Quantize the bf16 weight W[N, K] (nn.Linear layout) to e4m3 with one power-of-two scale per row: Q[N, K] e4m3 bytes,
// exps[N] = e_n, and W is overwritten in place with W' = e4m3 * 2^e_n (exact in bf16).  K % 8 == 0.
extern "C" int nv_quantize_fp8_rows(void* W, int64_t ldw, void* Q, int64_t ldq, void* exps, int N, int K, void* stream_) {
  using namespace nv;
  NV_REQUIRE(N > 0 && K > 0 && (K % 8) == 0, "nv_quantize_fp8_rows: needs N > 0 and K %% 8 == 0 (got N=%d K=%d)", N, K);
  NV_REQUIRE(W && Q && exps, "nv_quantize_fp8_rows: null operand");
  NV_REQUIRE((ldw & 7) == 0 && (ldq & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(Q) & 15) == 0,
             "nv_quantize_fp8_rows: W / Q must be 16-byte aligned with ldw %% 8 == 0 and ldq %% 16 == 0");
  quantize_fp8_rows_kernel<<<N, QZ_THREADS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      reinterpret_cast<__nv_bfloat16*>(W), ldw, reinterpret_cast<uint8_t*>(Q), ldq, reinterpret_cast<int8_t*>(exps), K);
  NV_LAUNCH_CHECK();
  return NV_OK;
}
