// navillm_b200 — fp32-in / fp32-out GEMM on Hopper tensor cores (wgmma .tf32) for the panorama encoder.
//
// Replaces the cuBLAS GEMMs behind the fp32 nn.Linear / nn.MultiheadAttention projections of the reference's
// image-embedding stack (models/image_embedding.py:51-121, models/detr_transformer.py:170-182; SURVEY.md §8 a2/a3).
// The reference pins torch==1.10.0 (requirements.txt:19), whose default torch.backends.cuda.matmul.allow_tf32 = True
// means those fp32 matmuls already ran with TF32 inputs and fp32 accumulation on the A100s it was trained on; this
// kernel makes the same numerical choice.  The exact-fp32 CUDA-core kernel (nv_sgemm) stays available
// (ops.set_pano_precision("fp32")) and is what the tight-tolerance parity tests use.
//
//   C[M,N] (+)= op(A) · op(B) (+ bias[N])      fp32 operands read as TF32 (10-bit mantissa), fp32 accumulate
//   ta = 0 : A stored [M,K]   ta = 1 : A stored [K,M]      tb = 0 : B stored [N,K]   tb = 1 : B stored [K,N]
//
// The encoder's problems are small (M = B*36 rows): one 128 x 128 tile per CTA, the K range split over blockIdx.y
// so that a few hundred CTAs are in flight.  The splits of a tile form one thread-block cluster and add their partial
// tiles in rank order in the leader's shared memory (distributed shared memory): the result does not depend on timing,
// and no atomics, workspace or memset are needed.
// The tf32 form of wgmma reads both operands K-major from shared memory only, so the two warpgroups stage every
// 32-wide k-block themselves: global -> registers (the next k-block's loads are in flight while the current one is
// multiplied) -> 128-byte-swizzled K-major rows in one of two shared-memory buffers, whatever the HBM layout
// (an MN-major operand is transposed on the way).  Each warpgroup then issues m64n128k8 wgmmas for its 64 rows.
#include "nv_common.cuh"
#include "nv_host.h"

namespace nv {

constexpr uint32_t T32_BM = 128, T32_BN = 128, T32_BK = 32, T32_THREADS = 256;
constexpr uint32_t T32_TILE_BYTES = 128 * T32_BK * 4;            // one operand tile: 128 rows x 128 B
constexpr uint32_t T32_DYN_BYTES = 2 * 2 * T32_TILE_BYTES + 1024;  // two buffers of (A, B)

// One 128-row x 32-k operand tile: 4 x 16 B per thread.  K-major source X[row][k]: a thread loads 4 consecutive k of
// one row.  MN-major source X[k][row]: a thread loads 4 consecutive rows of one k (lanes walk k, so that the transposed
// shared-memory writes of a warp hit 32 different banks).
template <bool MN>
struct T32Tile {
  float4 v[4];
  __device__ __forceinline__ void load(const float* __restrict__ X, int64_t ld, uint32_t row0, uint32_t rows, uint32_t k0,
                                       uint32_t K) {
#pragma unroll
    for (uint32_t i = 0; i < 4; ++i) {
      const uint32_t idx = threadIdx.x + i * T32_THREADS;
      float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
      if constexpr (!MN) {
        const uint32_t r = row0 + (idx >> 3), k = k0 + (idx & 7) * 4;
        if (r < rows) {
          const float* p = X + (int64_t)r * ld + k;
          if (k + 4 <= K) x = *reinterpret_cast<const float4*>(p);
          else {
            if (k < K) x.x = p[0];
            if (k + 1 < K) x.y = p[1];
            if (k + 2 < K) x.z = p[2];
          }
        }
      } else {
        const uint32_t k = k0 + (idx & 31), r = row0 + (idx >> 5) * 4;
        if (k < K) {
          const float* p = X + (int64_t)k * ld + r;
          if (r + 4 <= rows) x = *reinterpret_cast<const float4*>(p);
          else {
            if (r < rows) x.x = p[0];
            if (r + 1 < rows) x.y = p[1];
            if (r + 2 < rows) x.z = p[2];
          }
        }
      }
      v[i] = x;
    }
  }
  // -> K-major 128-byte-swizzled rows (32 k = 128 B per row) at shared address `dst`
  __device__ __forceinline__ void store(uint32_t dst) const {
#pragma unroll
    for (uint32_t i = 0; i < 4; ++i) {
      const uint32_t idx = threadIdx.x + i * T32_THREADS;
      if constexpr (!MN) {
        const uint32_t r = idx >> 3, c = idx & 7;
        sts128(dst + sw128_offset(r, c), __float_as_uint(v[i].x), __float_as_uint(v[i].y), __float_as_uint(v[i].z),
               __float_as_uint(v[i].w));
      } else {
        const uint32_t k = idx & 31, r = (idx >> 5) * 4;
        const float e[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
#pragma unroll
        for (uint32_t j = 0; j < 4; ++j)
          asm volatile("st.shared.f32 [%0], %1;" ::"r"(dst + sw128_offset(r + j, k >> 2) + (k & 3) * 4), "f"(e[j]) : "memory");
      }
    }
  }
};

template <bool A_MN, bool B_MN>
__global__ void __launch_bounds__(T32_THREADS, 1)
gemm_tf32_wgmma(const float* __restrict__ A, int64_t lda, const float* __restrict__ B, int64_t ldb, float* __restrict__ C,
                int64_t ldc, const float* __restrict__ bias, uint32_t M, uint32_t N, uint32_t K, uint32_t num_n,
                uint32_t kb_per_split, uint32_t accumulate) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023) & ~1023u;
  auto sA = [&](uint32_t buf) { return sbase + buf * 2 * T32_TILE_BYTES; };
  auto sB = [&](uint32_t buf) { return sbase + buf * 2 * T32_TILE_BYTES + T32_TILE_BYTES; };

  const uint32_t m_blk = blockIdx.x / num_n, n_blk = blockIdx.x % num_n;
  const uint32_t m0 = m_blk * T32_BM, n0 = n_blk * T32_BN;
  const uint32_t total_kb = ceil_div_u32(K, T32_BK);
  const uint32_t kb0 = blockIdx.y * kb_per_split;
  const uint32_t nkb = min(kb_per_split, total_kb - kb0);   // host guarantees kb0 < total_kb
  const uint32_t wg = threadIdx.x >> 7;

  T32Tile<A_MN> ta;
  T32Tile<B_MN> tb;
  ta.load(A, lda, m0, M, kb0 * T32_BK, K);
  tb.load(B, ldb, n0, N, kb0 * T32_BK, K);
  ta.store(sA(0));
  tb.store(sB(0));
  fence_proxy_async_smem();
  __syncthreads();

  float acc[64];
#pragma unroll
  for (uint32_t i = 0; i < 64; ++i) acc[i] = 0.f;
  for (uint32_t i = 0; i < nkb; ++i) {
    const uint32_t buf = i & 1;
    const bool more = i + 1 < nkb;
    if (more) {                                            // next k-block's loads in flight under this one's wgmmas
      ta.load(A, lda, m0, M, (kb0 + i + 1) * T32_BK, K);
      tb.load(B, ldb, n0, N, (kb0 + i + 1) * T32_BK, K);
    }
    const uint64_t adesc = gmma_desc_sw128(sA(buf) + wg * 8192, 0, 1024);
    const uint64_t bdesc = gmma_desc_sw128(sB(buf), 0, 1024);
    wgmma_fence();
#pragma unroll
    for (uint32_t k = 0; k < T32_BK / 8; ++k) wgmma_ss_tf32_n128(acc, adesc + k * 2, bdesc + k * 2, 1u);
    wgmma_commit();
    if (more) {                                            // the other buffer was released by the previous wait
      ta.store(sA(buf ^ 1));
      tb.store(sB(buf ^ 1));
      fence_proxy_async_smem();
    }
    wgmma_wait<0>();
    __syncthreads();
  }
  reg_fence(acc);

  // ---- split-K: running sum in the leader's operand buffers (64 KB = 64 floats x 256 threads), ranks in order ----
  if (gridDim.y > 1) {
    const uint32_t rank = blockIdx.y;                      // cluster (1, splits, 1): the rank is the split index
    if (rank == 0) {
#pragma unroll
      for (uint32_t i = 0; i < 64; ++i)
        asm volatile("st.shared.f32 [%0], %1;" ::"r"(sbase + (i * T32_THREADS + threadIdx.x) * 4), "f"(acc[i]) : "memory");
    }
    cluster_sync_all();
    for (uint32_t r = 1; r < gridDim.y; ++r) {
      if (rank == r) {
#pragma unroll
        for (uint32_t i = 0; i < 64; ++i) dsmem_add_f32(sbase + (i * T32_THREADS + threadIdx.x) * 4, 0, acc[i]);
      }
      cluster_sync_all();
    }
    if (rank != 0) return;
#pragma unroll
    for (uint32_t i = 0; i < 64; ++i)
      asm volatile("ld.shared.f32 %0, [%1];" : "=f"(acc[i]) : "r"(sbase + (i * T32_THREADS + threadIdx.x) * 4) : "memory");
  }

  // ---- epilogue straight from the accumulator fragment: rows r, r + 8; columns 8 i + 2 (lane % 4) + {0, 1} ----
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t r = m0 + wg * 64 + ((threadIdx.x & 127) >> 5) * 16 + (lane >> 2);
  const bool add_bias = bias != nullptr;
#pragma unroll
  for (uint32_t i = 0; i < 16; ++i) {
    const uint32_t c = n0 + i * 8 + 2 * (lane & 3);
#pragma unroll
    for (uint32_t h = 0; h < 2; ++h) {
      const uint32_t row = r + h * 8;
      if (row >= M) continue;
      float* dst = C + (int64_t)row * ldc + c;
#pragma unroll
      for (uint32_t e = 0; e < 2; ++e) {
        if (c + e < N) {
          float x = acc[4 * i + 2 * h + e];
          if (add_bias) x += bias[c + e];
          if (accumulate) x += dst[e];                     // one writer per element
          dst[e] = x;
        }
      }
    }
  }
}

template <bool A_MN, bool B_MN>
static int launch_tf32(const float* A, int64_t lda, const float* B, int64_t ldb, float* C, int64_t ldc, const float* bias, int M,
                       int N, int K, int accumulate, cudaStream_t stream) {
  auto kern = gemm_tf32_wgmma<A_MN, B_MN>;
  static bool attr_set = false;
  if (!attr_set) {
    NV_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, T32_DYN_BYTES));
    attr_set = true;
  }
  const uint32_t num_m = ceil_div_u32(M, T32_BM), num_n = ceil_div_u32(N, T32_BN);
  const uint32_t tiles = num_m * num_n, total_kb = ceil_div_u32(K, T32_BK);
  // split K until about two CTAs per SM are in flight, keeping at least 8 k-blocks (256 k) per split; the splits of
  // a tile are one cluster (at most 8 CTAs); with g_fixed_splits as far as K allows, whatever the tile count
  uint32_t splits = 1;
  while (splits < 8 && (g_fixed_splits || tiles * splits * 2 <= 2u * (uint32_t)sm_count()) && total_kb / (splits * 2) >= 8)
    splits *= 2;
  const uint32_t kb_per_split = ceil_div_u32(total_kb, splits);
  splits = ceil_div_u32(total_kb, kb_per_split);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(tiles, splits);
  cfg.blockDim = dim3(T32_THREADS);
  cfg.dynamicSmemBytes = T32_DYN_BYTES;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 1;
  attr[0].val.clusterDim.y = splits;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  NV_CUDA(cudaLaunchKernelEx(&cfg, kern, A, lda, B, ldb, C, ldc, bias, (uint32_t)M, (uint32_t)N, (uint32_t)K, num_n,
                             kb_per_split, (uint32_t)(accumulate ? 1 : 0)));
  return NV_OK;
}

}  // namespace nv

// Same contract as nv_sgemm (csrc/pano_ops.cu) with TF32 operand rounding.  Requirements beyond nv_sgemm's: base
// pointers 16-byte aligned and lda/ldb multiples of 4 floats (16-byte loads); returns NV_ERR_BAD_ARG otherwise so that the
// caller can route odd shapes (e.g. the K = 7 location-feature projections) to nv_sgemm.
extern "C" int nv_gemm_tf32(const float* A, int64_t lda, int ta, const float* B, int64_t ldb, int tb, float* C, int64_t ldc,
                            const float* bias, int M, int N, int K, int accumulate, void* stream_) {
  using namespace nv;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M == 0 || N == 0) return NV_OK;
  NV_REQUIRE(M > 0 && N > 0 && K > 0 && A && B && C, "nv_gemm_tf32: bad arguments M=%d N=%d K=%d", M, N, K);
  NV_REQUIRE((lda & 3) == 0 && (ldb & 3) == 0, "nv_gemm_tf32: lda/ldb must be multiples of 4 (got %lld, %lld)",
             (long long)lda, (long long)ldb);
  NV_REQUIRE(((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B)) & 15) == 0,
             "nv_gemm_tf32: A and B must be 16-byte aligned");
  if (!ta && !tb) return launch_tf32<false, false>(A, lda, B, ldb, C, ldc, bias, M, N, K, accumulate, stream);
  if (!ta && tb) return launch_tf32<false, true>(A, lda, B, ldb, C, ldc, bias, M, N, K, accumulate, stream);
  if (ta && tb) return launch_tf32<true, true>(A, lda, B, ldb, C, ldc, bias, M, N, K, accumulate, stream);
  return launch_tf32<true, false>(A, lda, B, ldb, C, ldc, bias, M, N, K, accumulate, stream);
}
