// navillm_b200 — skinny bf16 GEMM for the decode step (M <= 16 activation rows), swap-AB on wgmma.
//
// The per-token GEMMs of greedy/sampled generation (reference: HF GenerationMixin.generate through
// models/modified_lm.py:184-199; SURVEY.md §8 a10, K13) multiply a handful of activation rows by every weight of
// the model: pure HBM weight streaming.  The general kernel (gemm_bf16.cu) puts the activations on the MMA M side,
// so each CTA re-stages a mostly-zero 128-row activation tile per k-block and the N/128 output tiles of a 4096-wide
// projection occupy 32 of 132 SMs.  Here the roles are swapped:
//
//   C^T[n, m] = sum_k W[n, k] * X[m, k]        MMA M = 128 weight rows (A operand), MMA N = 16 activation rows (B)
//
// so a k-block moves 16 KB of weights + 2 KB of activations, and the K range of one weight tile is split over the
// CTAs of a thread-block cluster (S = 1, 2, 4 or 8) whose partial accumulators are reduced through distributed
// shared memory in the leader CTA - no atomics, no workspace, no second kernel.  4-stage rings of 18 KB let three
// CTAs share an SM, so a 4096-column projection runs as 256 CTAs (S = 8) instead of 32.
//   warps 0..7  two consumer warpgroups, m64n16k16 wgmmas over weight rows 0..63 / 64..127 of the tile
//   warp 8      TMA producer
#include <stdlib.h>

#include "nv_common.cuh"
#include "nv_host.h"

namespace nv {

constexpr uint32_t SK_BN = 128;      // weight rows per tile (MMA M)
constexpr uint32_t SK_BM = 16;       // activation rows (MMA N)
constexpr uint32_t SK_BK = 64;
constexpr uint32_t SK_STAGES = 4;
constexpr uint32_t SK_THREADS = 288;
constexpr uint32_t SK_W_BYTES = SK_BN * SK_BK * 2, SK_X_BYTES = SK_BM * SK_BK * 2;
constexpr uint32_t SK_STAGE_BYTES = SK_W_BYTES + SK_X_BYTES;
constexpr uint32_t SK_BAR_OFF = SK_STAGES * SK_STAGE_BYTES;
constexpr uint32_t SK_DYN_BYTES = SK_BAR_OFF + 2 * SK_STAGES * 8 + 1024;
constexpr uint32_t SK_RED_BYTES = SK_BM * SK_BN * 4;   // one partner's partial tile [16 m][128 n] fp32 (8 KB)
static_assert(8 * SK_RED_BYTES <= SK_STAGES * SK_W_BYTES, "reduction buffers and the output tile reuse the weight stages");

__device__ __forceinline__ uint32_t sk_cluster_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void sk_cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void sk_st_remote_f32(float* p, uint32_t cta, float v) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "st.shared::cluster.f32 [ra], %2;\n\t}"
      ::"r"(smem_u32(p)), "r"(cta), "f"(v)
      : "memory");
}

// swiglu_f != 0: W is the fused gate|up weight [2F, K]; tile n_blk stages 64 gate rows n_blk*64.. and the matching 64 up
// rows F + n_blk*64.. (two 64-row TMA boxes), the leader pairs them and writes h[m, n] = bf16(bf16(silu(g)) * u), the
// same rounding points as swiglu_fwd_kernel on the bf16 gate|up buffer (which is not materialised here).
__global__ void __launch_bounds__(SK_THREADS)
gemm_skinny_wgmma(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x,
                  __nv_bfloat16* __restrict__ C, int64_t ldc, const __nv_bfloat16* __restrict__ addend, int64_t ld_add,
                  uint32_t M, uint32_t N, uint32_t K, uint32_t splits, uint32_t swiglu_f) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_w = smem;
  uint8_t* smem_x = smem + SK_STAGES * SK_W_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + SK_BAR_OFF);
  uint64_t* empty_bar = full_bar + SK_STAGES;
  float* red = reinterpret_cast<float*>(smem_w);          // leader: [splits-1][16][128] fp32, valid after the main loop
  float* ex = red + 7 * SK_BM * SK_BN;                    // leader: the reduced tile [16 m][128 n]

  const uint32_t warp = warp_id_uniform(), lane = threadIdx.x & 31;
  const uint32_t rank = splits > 1 ? sk_cluster_rank() : 0u;
  const uint32_t n_blk = blockIdx.x / splits;
  const uint32_t total_kb = ceil_div_u32(K, SK_BK);
  const uint32_t kb_per = ceil_div_u32(total_kb, splits);
  const uint32_t kb0 = min(rank * kb_per, total_kb);
  const uint32_t nkb = min(kb_per, total_kb - kb0);        // may be 0 for a trailing split: contributes zeros

  if (threadIdx.x == 0) {
    for (uint32_t i = 0; i < SK_STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 2); }
    fence_mbar_init();
  }
  __syncthreads();

  griddep_launch();                                        // the next kernel of the stream may start its own prologue
  float acc[8];
#pragma unroll
  for (uint32_t i = 0; i < 8; ++i) acc[i] = 0.f;
  const uint32_t wg = warp >> 2;
  if (warp == 8) {
    tma_prefetch_desc(&tmap_w);
    tma_prefetch_desc(&tmap_x);
    const int32_t n0 = swiglu_f ? n_blk * 64 : n_blk * SK_BN;
    auto load_w = [&](uint32_t stage, int32_t k0) {
      if (swiglu_f) {                                                                   // box {64 k, 64 n}: gate half, up half
        tma_load_2d(smem_w + stage * SK_W_BYTES, &tmap_w, &full_bar[stage], k0, n0);
        tma_load_2d(smem_w + stage * SK_W_BYTES + SK_W_BYTES / 2, &tmap_w, &full_bar[stage], k0, (int32_t)swiglu_f + n0);
      } else {
        tma_load_2d(smem_w + stage * SK_W_BYTES, &tmap_w, &full_bar[stage], k0, n0);   // box {64 k, 128 n}
      }
    };
    // Programmatic dependent launch: the WEIGHTS do not depend on the previous kernel of the stream, so the first ring of
    // weight tiles is requested before waiting for it (weight streaming continues across the kernel boundary); the
    // activations X are its output and are loaded after the wait.
    const uint32_t pre = min(nkb, SK_STAGES);
    if (elect_one()) {
      for (uint32_t i = 0; i < pre; ++i) {
        mbar_arrive_expect_tx(&full_bar[i], SK_STAGE_BYTES);
        load_w(i, (kb0 + i) * SK_BK);
      }
    }
    __syncwarp();
    griddep_wait();
    if (elect_one()) {
      for (uint32_t i = 0; i < pre; ++i)
        tma_load_2d(smem_x + i * SK_X_BYTES, &tmap_x, &full_bar[i], (kb0 + i) * SK_BK, 0);   // box {64 k, 16 m} (rows >= M: zeros)
    }
    __syncwarp();
    for (uint32_t i = pre; i < nkb; ++i) {
      const uint32_t stage = i % SK_STAGES, phase = (i / SK_STAGES) & 1;
      mbar_wait(&empty_bar[stage], phase ^ 1);
      if (elect_one()) {
        mbar_arrive_expect_tx(&full_bar[stage], SK_STAGE_BYTES);
        const int32_t k0 = (kb0 + i) * SK_BK;
        load_w(stage, k0);
        tma_load_2d(smem_x + stage * SK_X_BYTES, &tmap_x, &full_bar[stage], k0, 0);
      }
      __syncwarp();
    }
  } else {
    for (uint32_t i = 0; i < nkb; ++i) {
      const uint32_t stage = i % SK_STAGES, phase = (i / SK_STAGES) & 1;
      mbar_wait(&full_bar[stage], phase);
      const uint64_t wdesc = gmma_desc_sw128(smem_u32(smem_w + stage * SK_W_BYTES + wg * 8192), 0, 1024);
      const uint64_t xdesc = gmma_desc_sw128(smem_u32(smem_x + stage * SK_X_BYTES), 0, 1024);
      wgmma_fence();
#pragma unroll
      for (uint32_t k = 0; k < SK_BK / 16; ++k) wgmma_ss_bf16<16, 0, 0>(acc, wdesc + k * 2, xdesc + k * 2, 1u);
      wgmma_commit();
      wgmma_wait<0>();
      if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[stage]);
    }
    reg_fence(acc);
    griddep_wait();                                        // before the first read of `addend` / write of C
  }

  // ---- this CTA's partial C^T tile: thread holds weight rows nr, nr + 8 and activation rows mc, mc + 1, mc + 8, mc + 9 ----
  const uint32_t nr = wg * 64 + ((threadIdx.x & 127) >> 5) * 16 + (lane >> 2), mc = 2 * (lane & 3);
  auto frag = [&](uint32_t j, uint32_t& m, uint32_t& n) {  // element j of acc[8] -> (m, n) in the tile
    n = nr + ((j >> 1) & 1) * 8;
    m = mc + (j & 1) + (j >> 2) * 8;
  };
  if (splits > 1) {
    sk_cluster_sync();                                     // every CTA of the cluster is past its main loop: stages are free
    if (warp < 8 && rank != 0) {
#pragma unroll
      for (uint32_t j = 0; j < 8; ++j) {
        uint32_t m, n;
        frag(j, m, n);
        if (m < M) sk_st_remote_f32(red + ((rank - 1) * SK_BM + m) * SK_BN + n, 0, acc[j]);
      }
    }
    sk_cluster_sync();                                     // partials visible in the leader
    if (warp < 8 && rank == 0) {
      for (uint32_t r = 0; r + 1 < splits; ++r)
#pragma unroll
        for (uint32_t j = 0; j < 8; ++j) {
          uint32_t m, n;
          frag(j, m, n);
          if (m < M) acc[j] += red[(r * SK_BM + m) * SK_BN + n];
        }
    }
  } else {
    __syncthreads();                                       // both warpgroups are done with the weight stages
  }
  if (rank != 0) return;
  // the reduced tile -> ex[16 m][128 n] (bf16-rounded: every output below rounds the projection first)
  if (warp < 8) {
#pragma unroll
    for (uint32_t j = 0; j < 8; ++j) {
      uint32_t m, n;
      frag(j, m, n);
      ex[m * SK_BN + n] = bf16_round(acc[j]);
    }
  }
  __syncthreads();
  const uint32_t nl = threadIdx.x;                         // weight row inside the tile
  if (nl >= SK_BN) return;
  if (swiglu_f) {
    // pair gate row nl < 64 with up row nl + 64
    if (nl < 64) {
      const uint32_t n = n_blk * 64 + nl;
      if (n < N) {
#pragma unroll
        for (uint32_t m = 0; m < SK_BM; ++m) {
          if (m < M) {
            const float g = ex[m * SK_BN + nl], u = ex[m * SK_BN + nl + 64];
            C[(int64_t)m * ldc + n] = __float2bfloat16_rn(bf16_round(g / (1.f + __expf(-g))) * u);
          }
        }
      }
    }
  } else {
    const uint32_t n = n_blk * SK_BN + nl;
    if (n < N) {
#pragma unroll
      for (uint32_t m = 0; m < SK_BM; ++m) {
        if (m < M) {
          float x = ex[m * SK_BN + nl];
          if (addend) x += __bfloat162float(addend[(int64_t)m * ld_add + n]);
          C[(int64_t)m * ldc + n] = __float2bfloat16_rn(x);
        }
      }
    }
  }
}

}  // namespace nv

static int skinny_launch(const void* X, int64_t ldx, const void* W, int64_t ldw, void* C, int64_t ldc, const void* addend,
                         int64_t ld_add, int M, int N, int K, uint32_t swiglu_f, cudaStream_t stream) {
  using namespace nv;
  CUtensorMap tw, tx;
  int rc;
  const uint64_t w_rows = swiglu_f ? 2ull * swiglu_f : (uint64_t)N;
  if ((rc = make_tmap_2d(&tw, W, 2, (uint64_t)K, w_rows, (uint64_t)ldw * 2, 64, swiglu_f ? 64 : SK_BN))) return rc;
  if ((rc = make_tmap_2d(&tx, X, 2, (uint64_t)K, (uint64_t)M, (uint64_t)ldx * 2, 64, SK_BM))) return rc;
  static bool attr_set = false;
  if (!attr_set) {
    NV_CUDA(cudaFuncSetAttribute(gemm_skinny_wgmma, cudaFuncAttributeMaxDynamicSharedMemorySize, SK_DYN_BYTES));
    attr_set = true;
  }
  const uint32_t tiles = ceil_div_u32(N, swiglu_f ? 64 : SK_BN), total_kb = ceil_div_u32(K, SK_BK);
  // largest power-of-two split (cluster size <= 8) that keeps about three CTAs per SM and >= 8 k-blocks per CTA
  uint32_t splits = 1;
  static int max_splits = -1, min_kb = -1;
  if (max_splits < 0) {                                    // developer knobs for tools/skinny_bench.py sweeps
    const char* e = getenv("NV_SKINNY_MAX_SPLITS");
    max_splits = (e && atoi(e) > 0) ? atoi(e) : 8;
    const char* f = getenv("NV_SKINNY_MIN_KB");
    min_kb = (f && atoi(f) > 0) ? atoi(f) : 8;
  }
  while (splits < (uint32_t)max_splits && tiles * splits * 2 <= 3u * (uint32_t)sm_count() && total_kb / (splits * 2) >= (uint32_t)min_kb)
    splits *= 2;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(tiles * splits);
  cfg.blockDim = dim3(SK_THREADS);
  cfg.dynamicSmemBytes = SK_DYN_BYTES;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = splits;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (g_pdl) {                                             // see griddep_wait() in the kernel
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.numAttrs = 2;
  }
  NV_CUDA(cudaLaunchKernelEx(&cfg, gemm_skinny_wgmma, tw, tx, reinterpret_cast<__nv_bfloat16*>(C), ldc,
                             reinterpret_cast<const __nv_bfloat16*>(addend), ld_add, (uint32_t)M, (uint32_t)N, (uint32_t)K,
                             splits, swiglu_f));
  return NV_OK;
}

// C[M,N] = bf16( bf16(X[M,K] · W[N,K]^T) (+ addend[M,N]) ), M <= 16.  X, W K-major (nn.Linear weight layout).
// Same rounding points as nv_gemm_bf16; the fp32 accumulation is split over `splits` k ranges (chosen here).
extern "C" int nv_gemm_skinny_bf16(const void* X, int64_t ldx, const void* W, int64_t ldw, void* C, int64_t ldc,
                                   const void* addend, int64_t ld_add, int M, int N, int K, void* stream_) {
  using namespace nv;
  NV_REQUIRE(M > 0 && M <= (int)SK_BM && N > 0 && K > 0, "nv_gemm_skinny_bf16: needs 1 <= M <= 16 (got M=%d N=%d K=%d)", M, N, K);
  NV_REQUIRE(X && W && C, "nv_gemm_skinny_bf16: null operand");
  NV_REQUIRE((ldx & 7) == 0 && (ldw & 7) == 0, "nv_gemm_skinny_bf16: ldx/ldw must be multiples of 8");
  return skinny_launch(X, ldx, W, ldw, C, ldc, addend, ld_add, M, N, K, 0u, reinterpret_cast<cudaStream_t>(stream_));
}

// h[M,F] = bf16( bf16(silu(g)) * u ) with [g | u] = bf16(X[M,K] · Wgu[2F,K]^T): the decode step's gate/up projection and
// SwiGLU in one kernel (HF LlamaMLP act_fn(gate_proj(x)) * up_proj(x)); F % 64 == 0.
extern "C" int nv_gemm_skinny_swiglu_bf16(const void* X, int64_t ldx, const void* Wgu, int64_t ldw, void* H, int64_t ldh, int M,
                                          int F, int K, void* stream_) {
  using namespace nv;
  NV_REQUIRE(M > 0 && M <= (int)SK_BM && F > 0 && K > 0 && (F % 64) == 0,
             "nv_gemm_skinny_swiglu_bf16: needs 1 <= M <= 16 and F %% 64 == 0 (got M=%d F=%d K=%d)", M, F, K);
  NV_REQUIRE(X && Wgu && H && (ldx & 7) == 0 && (ldw & 7) == 0, "nv_gemm_skinny_swiglu_bf16: null operand / alignment");
  return skinny_launch(X, ldx, Wgu, ldw, H, ldh, nullptr, 0, M, F, K, (uint32_t)F, reinterpret_cast<cudaStream_t>(stream_));
}
