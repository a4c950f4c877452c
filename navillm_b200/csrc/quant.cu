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
// (q4_pack_group) and overwrites each element with W' (every element is visited by exactly one thread).
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
  q4_pack_group(t, codes, (int64_t)rb * (K / 64) + 2 * g, [&](int r, int c) {
    const float s = s_scale[r];
    const int z = s_zero[r];
    const int q = q4_code(q4_bf16_float(tile[r][c]), s, z);
    tile[r][c] = q4_value_bits(q, z, s);
    return q;
  });
  __syncthreads();
  for (int i = t; i < 64 * 16; i += Q4_THREADS) {
    const int r = i >> 4, c = (i & 15) * 8, n = rb * 64 + r;
    if (n < N) *reinterpret_cast<uint4*>(W + n * ldw + (int64_t)g * Q4_GROUP + c) = *reinterpret_cast<const uint4*>(&tile[r][c]);
  }
}

// GPTQ, one 128-column group g per launch (nv_gptq_int4_block).  The group is also GPTQ's block, so a row's (s, z) are
// fixed when the block starts.  Work lies only along N, so a warp owns a row: lane l holds the fp32 working values of
// columns l, l + 32, l + 64 and l + 96.  At column j every lane takes w_j by shuffle and computes the same q, W'_j and
// e = (w_j - W'_j) / U_jj, then subtracts e U[j, c] from its own columns (U is upper triangular, so only the columns after
// j change).  A CTA walks 16-row slabs, a quarter of a 64-row code block each: when its 16 warps are done, warp 0 packs the
// slab's codes (q4_pack_group as thread 32 * (slab % 4) + lane).  The diagonal block of U sits in shared memory once per CTA.
constexpr int GQ_WARPS = 16;
constexpr int GQ_SMEM = (Q4_GROUP * Q4_GROUP + Q4_GROUP) * 4;   // U's diagonal block and 1 / U_jj

__global__ void __launch_bounds__(GQ_WARPS * 32, 2)
gptq_int4_block_kernel(const float* __restrict__ Wf, int64_t ldwf, const float* __restrict__ U, int64_t ldu,
                       __nv_bfloat16* __restrict__ W, int64_t ldw, uint8_t* __restrict__ codes,
                       __nv_bfloat16* __restrict__ scales, uint8_t* __restrict__ zeros, float* __restrict__ negE, int64_t lde,
                       int N, int K, int g) {
  extern __shared__ __align__(16) float sU[];
  __shared__ uint8_t s_q[GQ_WARPS][Q4_GROUP];
  float* s_rdiag = sU + Q4_GROUP * Q4_GROUP;
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31, G = K / (int)Q4_GROUP;
  for (int i = t; i < (int)(Q4_GROUP * Q4_GROUP); i += GQ_WARPS * 32) sU[i] = U[(int64_t)(i >> 7) * ldu + (i & 127)];
  if (t < (int)Q4_GROUP) s_rdiag[t] = __frcp_rn(U[(int64_t)t * ldu + t]);
  __syncthreads();
  for (int slab = blockIdx.x; slab < N / 16; slab += gridDim.x) {
    const int64_t n = (int64_t)slab * 16 + warp;
    const float* wrow = Wf + n * ldwf + (int64_t)g * Q4_GROUP;
    float w[4];
    float lo = 0.f, hi = 0.f;
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      w[m] = wrow[lane + 32 * m];
      lo = q4_min(lo, w[m]);
      hi = q4_max(hi, w[m]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo = q4_min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
      hi = q4_max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    float s;
    int z;
    q4_group_params(lo, hi, s, z);
    if (lane == 0) {
      scales[n * G + g] = __ushort_as_bfloat16(q4_bf16_bits(s));
      zeros[n * G + g] = (uint8_t)z;
    }
    int qs[4];
    uint16_t vs[4];
    float es[4];
#pragma unroll
    for (int m = 0; m < 4; ++m) {
#pragma unroll 8
      for (int jj = 0; jj < 32; ++jj) {
        const int j = 32 * m + jj;
        const float x = __shfl_sync(0xffffffffu, w[m], jj);
        const int q = q4_code(x, s, z);
        const uint16_t v = q4_value_bits(q, z, s);
        const float ne = q4_mul(q4_sub(q4_bf16_float(v), x), s_rdiag[j]);     // -e
        if (lane == jj) {
          qs[m] = q;
          vs[m] = v;
          es[m] = ne;
        }
        const float* urow = sU + j * Q4_GROUP + lane;
#pragma unroll
        for (int m2 = m; m2 < 4; ++m2) w[m2] = q4_fma(ne, urow[32 * m2], w[m2]);
      }
    }
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      const int c = lane + 32 * m;
      W[n * ldw + (int64_t)g * Q4_GROUP + c] = __ushort_as_bfloat16(vs[m]);
      negE[n * lde + c] = es[m];
      s_q[warp][c] = (uint8_t)qs[m];
    }
    __syncthreads();
    if (warp == 0) {
      const int quarter = slab & 3;
      q4_pack_group(32 * quarter + lane, codes, (int64_t)(slab >> 2) * (K / 64) + 2 * g,
                    [&](int r, int c) { return (int)s_q[r - 16 * quarter][c]; });
    }
    __syncthreads();
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

// One GPTQ block (include/navillm_b200.h): group g of the fp32 working copy Wf [N, K] against U_gg, the 128 x 128 diagonal
// block of U (row stride ldu).  Writes the group's codes, scales and zeros, W' over columns 128 g .. 128 g + 127 of the
// bf16 W, and -E [N, 128] (row stride lde), the scaled errors whose product with U's rows of the block is added to the
// later columns of Wf.  Wf is only read.  N % 64 == 0, K % 128 == 0, 0 <= g < K / 128.
extern "C" int nv_gptq_int4_block(const void* Wf, int64_t ldwf, const void* U, int64_t ldu, int g, void* W, int64_t ldw,
                                  void* codes, void* scales, void* zeros, void* negE, int64_t lde, int N, int K,
                                  void* stream_) {
  using namespace nv;
  NV_REQUIRE(N > 0 && (N % 64) == 0 && K > 0 && (K % (int)Q4_GROUP) == 0,
             "nv_gptq_int4_block: needs N %% 64 == 0 and K %% 128 == 0 (got N=%d K=%d)", N, K);
  NV_REQUIRE(g >= 0 && g < K / (int)Q4_GROUP, "nv_gptq_int4_block: block %d outside 0..%d", g, K / (int)Q4_GROUP - 1);
  NV_REQUIRE(Wf && U && W && codes && scales && zeros && negE, "nv_gptq_int4_block: null operand");
  NV_REQUIRE(ldwf >= K && ldw >= K && ldu >= (int64_t)Q4_GROUP && lde >= (int64_t)Q4_GROUP,
             "nv_gptq_int4_block: needs ldwf, ldw >= K and ldu, lde >= 128 (got %lld, %lld, %lld, %lld)", (long long)ldwf,
             (long long)ldw, (long long)ldu, (long long)lde);
  NV_REQUIRE((reinterpret_cast<uintptr_t>(codes) & 15) == 0, "nv_gptq_int4_block: codes must be 16-byte aligned");
  static bool attr = false;
  if (!attr) {
    NV_CUDA(cudaFuncSetAttribute(gptq_int4_block_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GQ_SMEM));
    attr = true;
  }
  const int grid = N / 16 < 2 * sm_count() ? N / 16 : 2 * sm_count();   // every CTA loads U_gg once
  gptq_int4_block_kernel<<<grid, GQ_WARPS * 32, GQ_SMEM, reinterpret_cast<cudaStream_t>(stream_)>>>(
      reinterpret_cast<const float*>(Wf), ldwf, reinterpret_cast<const float*>(U), ldu, reinterpret_cast<__nv_bfloat16*>(W),
      ldw, reinterpret_cast<uint8_t*>(codes), reinterpret_cast<__nv_bfloat16*>(scales), reinterpret_cast<uint8_t*>(zeros),
      reinterpret_cast<float*>(negE), lde, N, K, g);
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
