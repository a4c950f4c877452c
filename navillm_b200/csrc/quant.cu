// navillm_b200 — fp8 (e4m3) weight quantizer for the decode step (format: nv_fp8.cuh).
//
// One CTA per weight row: the row's amax (on the bf16 bit patterns: |x| orders like its 15 low bits), the exponent e_n,
// then one more pass that writes the e4m3 bytes and W' = e4m3 * 2^e_n back over the bf16 row, so the model that remains
// is exactly the one the fp8 kernels compute with.
#include "nv_common.cuh"
#include "nv_fp8.cuh"
#include "nv_host.h"

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

}  // namespace nv

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
