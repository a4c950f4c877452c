// navillm_b200 — batch-invariant weight-streaming bf16 GEMM for the decode step and lm_head (any M, tuned for M <= 128).
//
// In batch-invariant mode (ModifiedLlamaForCausalLM.set_batch_invariant) every output element must be a function of its
// own activation row and the weights alone, whatever the number of rows that share the launch.  The default decode
// kernels do not give that: at most 16 rows take the swap-AB cluster-split-K kernel of gemm_skinny.cu, whose k ranges
// follow the tile count and sm_count(), and above 16 rows nv_gemm_bf16 picks its tile by M.  This kernel fixes the
// arithmetic of the 128-wide wgmma kernel of gemm_bf16.cu for every element:
//
//   acc = 0;  for kb in 0 .. ceil(K / 64) - 1 (in order):  for k16 in 0..3:  acc += wgmma m64nNk16 (A rows, W rows)
//   C = bf16(acc)  |  bf16(bf16(acc) + addend)  |  SwiGLU: h = bf16(bf16(silu(bf16(g))) * bf16(u))
//
// no split-K, the activations on the MMA M side (rows padded to 64 by TMA zero fill, never swapped), and an epilogue
// straight from the accumulator registers that does not depend on the tile's row count.  Instead of splitting K, N is
// spread over narrow 32-column tiles: a 4096-wide projection runs as 128 CTAs, q|k|v as 384, two CTAs per SM.
//   warps 0..3  one consumer warpgroup: 64 activation rows x 32 weight rows, m64n32k16 wgmmas from the stage ring
//   warp 4      TMA producer: 8-deep ring of 12 KB stages (8 KB activations + 4 KB weights), 128-byte swizzled
// The weights do not depend on the previous kernel of the stream, so with programmatic dependent launch the producer
// requests the first ring of weight tiles before it waits for that kernel (nv_common.cuh griddep_wait).
// SwiGLU form: the weight is the fused gate|up [2F, K]; a tile holds 16 gate rows n0.. and the same 16 up rows F + n0..
// (two 16-row boxes), so accumulator group i (columns 8 i ..) of gate meets group i + 2 of up in the same thread.
#include "nv_common.cuh"
#include "nv_host.h"

namespace nv {

constexpr uint32_t BI_BM = 64;
constexpr uint32_t BI_BN = 32;
constexpr uint32_t BI_BK = 64;
constexpr uint32_t BI_STAGES = 8;
constexpr uint32_t BI_THREADS = 160;
constexpr uint32_t BI_A_BYTES = BI_BM * BI_BK * 2;
constexpr uint32_t BI_B_BYTES = BI_BN * BI_BK * 2;
constexpr uint32_t BI_STAGE_BYTES = BI_A_BYTES + BI_B_BYTES;
constexpr uint32_t BI_BAR_OFF = BI_STAGES * BI_STAGE_BYTES;
constexpr uint32_t BI_DYN_BYTES = BI_BAR_OFF + 2 * BI_STAGES * 8 + 1024;   // + slack for 1024-byte alignment
static_assert(2 * BI_DYN_BYTES <= 232448, "two CTAs per SM");

// swiglu_f != 0: W is the fused gate|up weight [2 swiglu_f, K] and C is h [M, swiglu_f] (N = swiglu_f).
__global__ void __launch_bounds__(BI_THREADS)
gemm_bi_wgmma(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
              __nv_bfloat16* __restrict__ C, int64_t ldc, const __nv_bfloat16* __restrict__ addend, int64_t ld_add,
              uint32_t M, uint32_t N, uint32_t K, uint32_t swiglu_f) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + BI_STAGES * BI_A_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + BI_BAR_OFF);
  uint64_t* empty_bar = full_bar + BI_STAGES;

  const uint32_t warp = warp_id_uniform(), lane = threadIdx.x & 31;
  const uint32_t num_m = ceil_div_u32(M, BI_BM);
  const uint32_t m_blk = blockIdx.x % num_m, n_blk = blockIdx.x / num_m;   // the m-blocks of a weight tile are adjacent
  const uint32_t num_kb = ceil_div_u32(K, BI_BK);
  const uint32_t n0 = n_blk * (swiglu_f ? BI_BN / 2 : BI_BN);               // first weight row (gate row) of the tile

  if (threadIdx.x == 0) {
    for (uint32_t i = 0; i < BI_STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 1); }
    fence_mbar_init();
  }
  __syncthreads();
  griddep_launch();                                        // the next kernel of the stream may start its own prologue

  if (warp == 4) {
    // ===================== TMA producer =====================
    tma_prefetch_desc(&tmap_x);
    tma_prefetch_desc(&tmap_w);
    auto load_w = [&](uint32_t stage, int32_t k0) {
      uint8_t* sb = smem_b + stage * BI_B_BYTES;
      if (swiglu_f) {                                      // box {64 k, 16 n}: gate rows, then the same up rows
        tma_load_2d(sb, &tmap_w, &full_bar[stage], k0, (int32_t)n0);
        tma_load_2d(sb + BI_B_BYTES / 2, &tmap_w, &full_bar[stage], k0, (int32_t)(swiglu_f + n0));
      } else {                                             // box {64 k, 32 n}
        tma_load_2d(sb, &tmap_w, &full_bar[stage], k0, (int32_t)n0);
      }
    };
    const uint32_t pre = min(num_kb, BI_STAGES);
    if (elect_one()) {
      for (uint32_t i = 0; i < pre; ++i) {
        mbar_arrive_expect_tx(&full_bar[i], BI_STAGE_BYTES);
        load_w(i, (int32_t)(i * BI_BK));
      }
    }
    __syncwarp();
    griddep_wait();                                        // the activations are the previous kernel's output
    if (elect_one()) {
      for (uint32_t i = 0; i < pre; ++i)                   // box {64 k, 64 m}; rows >= M read as zeros
        tma_load_2d(smem_a + i * BI_A_BYTES, &tmap_x, &full_bar[i], (int32_t)(i * BI_BK), (int32_t)(m_blk * BI_BM));
    }
    __syncwarp();
    for (uint32_t kb = pre; kb < num_kb; ++kb) {
      const uint32_t stage = kb % BI_STAGES, phase = (kb / BI_STAGES) & 1;
      mbar_wait(&empty_bar[stage], phase ^ 1);
      if (elect_one()) {
        mbar_arrive_expect_tx(&full_bar[stage], BI_STAGE_BYTES);
        const int32_t k0 = (int32_t)(kb * BI_BK);
        load_w(stage, k0);
        tma_load_2d(smem_a + stage * BI_A_BYTES, &tmap_x, &full_bar[stage], k0, (int32_t)(m_blk * BI_BM));
      }
      __syncwarp();
    }
    return;
  }

  // ===================== consumer warpgroup =====================
  float acc[BI_BN / 2];
#pragma unroll
  for (uint32_t i = 0; i < BI_BN / 2; ++i) acc[i] = 0.f;
  // K > 0 (host check): keeps ptxas from a zero-trip path that would serialize the wgmmas (see gemm_bf16.cu)
  __builtin_assume(num_kb > 0);
  for (uint32_t kb = 0; kb < num_kb; ++kb) {
    const uint32_t stage = kb % BI_STAGES, phase = (kb / BI_STAGES) & 1;
    mbar_wait(&full_bar[stage], phase);
    const uint64_t adesc = gmma_desc_sw128(smem_u32(smem_a + stage * BI_A_BYTES), 0, 1024);
    const uint64_t bdesc = gmma_desc_sw128(smem_u32(smem_b + stage * BI_B_BYTES), 0, 1024);
    wgmma_fence();
#pragma unroll
    for (uint32_t k = 0; k < BI_BK / 16; ++k) wgmma_ss_bf16<BI_BN, 0, 0>(acc, adesc + k * 2, bdesc + k * 2, 1u);
    wgmma_commit();
    wgmma_wait<0>();
    if (threadIdx.x == 0) mbar_arrive(&empty_bar[stage]);
  }
  reg_fence(acc);
  griddep_wait();                                          // before the first read of `addend` / write of C

  // ---- epilogue from the fragments: acc[4 i + 2 h + j] is row r0 + 8 h, tile column 8 i + 2 (lane % 4) + j ----
  const uint32_t r0 = m_blk * BI_BM + (warp << 4) + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
  for (uint32_t h = 0; h < 2; ++h) {
    const uint32_t row = r0 + 8 * h;
    if (row >= M) continue;
    __nv_bfloat16* crow = C + (int64_t)row * ldc;
    if (swiglu_f) {
#pragma unroll
      for (uint32_t i = 0; i < 2; ++i)
#pragma unroll
        for (uint32_t j = 0; j < 2; ++j) {
          const uint32_t col = n0 + 8 * i + cq + j;
          const float g = bf16_round(acc[4 * i + 2 * h + j]), u = bf16_round(acc[4 * (i + 2) + 2 * h + j]);
          if (col < N) crow[col] = __float2bfloat16_rn(bf16_round(g / (1.f + __expf(-g))) * u);
        }
    } else {
#pragma unroll
      for (uint32_t i = 0; i < BI_BN / 8; ++i)
#pragma unroll
        for (uint32_t j = 0; j < 2; ++j) {
          const uint32_t col = n0 + 8 * i + cq + j;
          if (col >= N) continue;
          float x = bf16_round(acc[4 * i + 2 * h + j]);
          if (addend) x += __bfloat162float(addend[(int64_t)row * ld_add + col]);
          crow[col] = __float2bfloat16_rn(x);
        }
    }
  }
}

static int bi_launch(const void* X, int64_t ldx, const void* W, int64_t ldw, void* C, int64_t ldc, const void* addend,
                     int64_t ld_add, int M, int N, int K, uint32_t swiglu_f, cudaStream_t stream) {
  CUtensorMap tx, tw;
  int rc;
  const uint64_t w_rows = swiglu_f ? 2ull * swiglu_f : (uint64_t)N;
  if ((rc = make_tmap_2d(&tx, X, 2, (uint64_t)K, (uint64_t)M, (uint64_t)ldx * 2, 64, BI_BM))) return rc;
  if ((rc = make_tmap_2d(&tw, W, 2, (uint64_t)K, w_rows, (uint64_t)ldw * 2, 64, swiglu_f ? BI_BN / 2 : BI_BN))) return rc;
  static bool attr_set = false;
  if (!attr_set) {
    NV_CUDA(cudaFuncSetAttribute(gemm_bi_wgmma, cudaFuncAttributeMaxDynamicSharedMemorySize, BI_DYN_BYTES));
    attr_set = true;
  }
  const uint32_t tiles = ceil_div_u32((uint32_t)N, swiglu_f ? BI_BN / 2 : BI_BN) * ceil_div_u32((uint32_t)M, BI_BM);
  NV_CUDA(launch_pdl(gemm_bi_wgmma, dim3(tiles), dim3(BI_THREADS), BI_DYN_BYTES, stream, tx, tw,
                     reinterpret_cast<__nv_bfloat16*>(C), ldc, reinterpret_cast<const __nv_bfloat16*>(addend), ld_add,
                     (uint32_t)M, (uint32_t)N, (uint32_t)K, swiglu_f));
  return NV_OK;
}

}  // namespace nv

// C[M,N] = bf16( bf16(X[M,K] · W[N,K]^T) (+ addend[M,N]) ): bit for bit nv_gemm_bf16's C for every M (one accumulation
// chain per element, no split), each row independent of the others.  X, W K-major (nn.Linear weight layout).
extern "C" int nv_gemm_bi_bf16(const void* X, int64_t ldx, const void* W, int64_t ldw, void* C, int64_t ldc,
                               const void* addend, int64_t ld_add, int M, int N, int K, void* stream_) {
  using namespace nv;
  NV_REQUIRE(M > 0 && N > 0 && K > 0, "nv_gemm_bi_bf16: needs M, N, K > 0 (got M=%d N=%d K=%d)", M, N, K);
  NV_REQUIRE(X && W && C, "nv_gemm_bi_bf16: null operand");
  NV_REQUIRE((ldx & 7) == 0 && (ldw & 7) == 0, "nv_gemm_bi_bf16: ldx/ldw must be multiples of 8");
  return bi_launch(X, ldx, W, ldw, C, ldc, addend, ld_add, M, N, K, 0u, reinterpret_cast<cudaStream_t>(stream_));
}

// h[M,F] = bf16( bf16(silu(g)) * u ) with [g | u] = bf16(X[M,K] · Wgu[2F,K]^T): the decode step's gate|up projection and
// SwiGLU in one kernel, bit for bit swiglu_fwd(nv_gemm_bf16(X, Wgu)); F % 16 == 0.
extern "C" int nv_gemm_bi_swiglu_bf16(const void* X, int64_t ldx, const void* Wgu, int64_t ldw, void* H, int64_t ldh, int M,
                                      int F, int K, void* stream_) {
  using namespace nv;
  NV_REQUIRE(M > 0 && F > 0 && K > 0 && (F % 16) == 0,
             "nv_gemm_bi_swiglu_bf16: needs M, K > 0 and F %% 16 == 0 (got M=%d F=%d K=%d)", M, F, K);
  NV_REQUIRE(X && Wgu && H && (ldx & 7) == 0 && (ldw & 7) == 0, "nv_gemm_bi_swiglu_bf16: null operand / alignment");
  return bi_launch(X, ldx, Wgu, ldw, H, ldh, nullptr, 0, M, F, K, (uint32_t)F, reinterpret_cast<cudaStream_t>(stream_));
}
