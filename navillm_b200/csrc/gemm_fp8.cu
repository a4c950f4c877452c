// navillm_b200 — W8A8 GEMM on the e4m3 tensor cores for the no-grad prompt forwards, and its activation quantizer.
//
//   C[M,N] = bf16( sum_kb 2^ea[m,kb] * (Aq[m, kb] . Wq[n, kb]) * 2^ew[n] )  (+ bf16 addend: C = bf16(bf16(acc) + addend))
//
// Operands (both K-major, e4m3 bytes): A' = the activation quantized per (row, 128-column block) by nv_quantize_act_fp8 below,
// Aq [M,K] with exponents ea [M, K/128]; W' = the fp8 weight copy of nv_quantize_fp8_rows, Wq [N,K] with one exponent ew[n]
// per row.  Both scales are exact powers of two (nv_fp8.cuh), so C approximates the product of the dequantized operands.
//
// Structure (gemm_bf16_wgmma's): one 128 x 128 output tile per CTA, 288 threads.
//   warp 8 (1 lane)          TMA producer: per 128-deep k-block one 128 x 128-byte tile of Aq and one of Wq, 128-byte
//                            swizzled (the layout of a 64-deep bf16 tile), W8_STAGES-deep mbarrier ring
//   warps 0..7               consumers: warpgroup w computes rows 64 w .. 64 w + 63 with four m64n128k32 e4m3 wgmmas per
//                            k-block into a FRESH fragment, then promotes it: master = fma(part, 2^ea[m,kb], master)
// Hopper's fp8 wgmma accumulates with fewer bits than fp32, so each k-block of 128 is one short chain that ends in an fp32
// register; the k-blocks are added in order.  An output element therefore depends only on its row and column operands: the
// same bits at every M and every packing of the rows.  The warpgroups preload their rows' ea for all k-blocks into shared
// memory at tile start; ew and the addend are applied in the epilogue (fp32 staging through the idle ring, as in
// gemm_bf16_wgmma).  The wgmma wait after every k-block serialises a warpgroup's MMAs with its promotion; the other warpgroup's
// MMAs fill that gap.
#include "nv_common.cuh"
#include "nv_fp8.cuh"
#include "nv_host.h"

namespace nv {

constexpr uint32_t W8_BM = 128, W8_BN = 128, W8_BK = 128;   // BK in e4m3 elements = bytes = one swizzled row
constexpr uint32_t W8_STAGES = 6;
constexpr uint32_t W8_THREADS = 288;
constexpr uint32_t W8_TILE_BYTES = W8_BM * W8_BK;             // 16 KB (A and B tiles are the same size)
constexpr uint32_t W8_STAGE_BYTES = 2 * W8_TILE_BYTES;
constexpr uint32_t W8_EXP_OFF = W8_STAGES * W8_STAGE_BYTES;   // ea[kb][128 rows] int8 after the ring
constexpr uint32_t W8_ACC_LD = W8_BN + 4;                     // staged fp32 row (+16 B: conflict-free)
constexpr uint32_t W8_SMEM_MAX = 232448;
static_assert(W8_BM * W8_ACC_LD * 4 <= W8_EXP_OFF, "accumulator staging reuses the stage ring");

__host__ __device__ constexpr uint32_t w8_exp_bytes(uint32_t num_kb) { return (W8_BM * num_kb + 15u) & ~15u; }
__host__ __device__ constexpr uint32_t w8_smem_bytes(uint32_t num_kb) {
  return W8_EXP_OFF + w8_exp_bytes(num_kb) + 2 * W8_STAGES * 8 + 1024;   // + slack for 1024-byte alignment
}

__global__ void __launch_bounds__(W8_THREADS, 1)
gemm_w8a8_wgmma(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                const int8_t* __restrict__ a_exp, int64_t lde, const int8_t* __restrict__ w_exp, __nv_bfloat16* __restrict__ C,
                int64_t ldc, const __nv_bfloat16* __restrict__ addend, int64_t ld_add, uint32_t M, uint32_t N, uint32_t K) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t num_kb = K / W8_BK;
  int8_t* es = reinterpret_cast<int8_t*>(smem + W8_EXP_OFF);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + W8_EXP_OFF + w8_exp_bytes(num_kb));
  uint64_t* empty_bar = full_bar + W8_STAGES;

  const uint32_t warp = warp_id_uniform();
  const uint32_t num_m = ceil_div_u32(M, W8_BM);
  const uint32_t m_blk = blockIdx.x % num_m, n_blk = blockIdx.x / num_m;   // m fastest: neighbouring CTAs share the W tile
  const uint32_t m0 = m_blk * W8_BM, n0 = n_blk * W8_BN;

  if (threadIdx.x == 0) {
    for (uint32_t i = 0; i < W8_STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);                         // one arrive per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ===================== TMA producer =====================
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    uint32_t stage = 0, phase = 0;
    for (uint32_t kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&empty_bar[stage], phase ^ 1);
      if (elect_one()) {
        mbar_arrive_expect_tx(&full_bar[stage], W8_STAGE_BYTES);
        uint8_t* sa = smem + stage * W8_STAGE_BYTES;
        tma_load_2d(sa, &tmap_a, &full_bar[stage], kb * W8_BK, m0);                  // box {128 k, 128 m}
        tma_load_2d(sa + W8_TILE_BYTES, &tmap_b, &full_bar[stage], kb * W8_BK, n0);  // box {128 k, 128 n}
      }
      __syncwarp();
      if (++stage == W8_STAGES) { stage = 0; phase ^= 1; }
    }
    return;  // the producer takes no part in the epilogue (named barrier 1 counts the 256 consumer threads only)
  }

  // ===================== consumers (warpgroups 0, 1) =====================
  const uint32_t wg = warp >> 2, t = threadIdx.x & 127, lane = threadIdx.x & 31;
  const uint32_t r0 = wg * 64 + (t >> 5) * 16 + (lane >> 2);   // fragment rows r0, r0 + 8 of the tile
  // this warpgroup's 64 rows of ea, all k-blocks (rows past M: exponent 0, their A tile rows are TMA zero fill)
  for (uint32_t idx = t; idx < 64 * num_kb; idx += 128) {
    const uint32_t r = idx / num_kb, kb = idx - r * num_kb, row = m0 + wg * 64 + r;
    es[kb * W8_BM + wg * 64 + r] = row < M ? a_exp[static_cast<int64_t>(row) * lde + kb] : int8_t(0);
  }
  named_bar_sync(2 + wg, 128);

  float acc[W8_BN / 2], part[W8_BN / 2];
#pragma unroll
  for (uint32_t i = 0; i < W8_BN / 2; ++i) { acc[i] = 0.f; part[i] = 0.f; }
  {
    uint32_t stage = 0, phase = 0;
    // K >= 128 (host check): see gemm_bf16_wgmma
    __builtin_assume(num_kb > 0);
    for (uint32_t kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * W8_STAGE_BYTES);
      const uint64_t adesc = gmma_desc_sw128(sa + wg * 8192, 0, 1024);
      const uint64_t bdesc = gmma_desc_sw128(sa + W8_TILE_BYTES, 0, 1024);
      wgmma_fence();
#pragma unroll
      for (uint32_t k = 0; k < W8_BK / 32; ++k)                    // +32 bytes per k32 step inside the swizzle span
        wgmma_ss_e4m3_n128(part, adesc + 2 * k, bdesc + 2 * k, k > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(part);
      if (t == 0) mbar_arrive(&empty_bar[stage]);
      const float s0 = fp8_pow2(es[kb * W8_BM + r0]), s1 = fp8_pow2(es[kb * W8_BM + r0 + 8]);
#pragma unroll
      for (uint32_t i = 0; i < W8_BN / 8; ++i) {
        acc[4 * i + 0] = fmaf(part[4 * i + 0], s0, acc[4 * i + 0]);
        acc[4 * i + 1] = fmaf(part[4 * i + 1], s0, acc[4 * i + 1]);
        acc[4 * i + 2] = fmaf(part[4 * i + 2], s1, acc[4 * i + 2]);
        acc[4 * i + 3] = fmaf(part[4 * i + 3], s1, acc[4 * i + 3]);
      }
      if (++stage == W8_STAGES) { stage = 0; phase ^= 1; }
    }
  }

  // ---- stage acc * 2^ew[n]: [128 rows][W8_BN + 4] fp32 over the (now idle) stage ring ----
  float* acc_s = reinterpret_cast<float*>(smem);
  named_bar_sync(1, 256);                                  // both warpgroups are past their last wgmma
#pragma unroll
  for (uint32_t i = 0; i < W8_BN / 8; ++i) {
    const uint32_t c = i * 8 + 2 * (lane & 3);
    const float w0 = n0 + c < N ? fp8_pow2(w_exp[n0 + c]) : 1.f;
    const float w1 = n0 + c + 1 < N ? fp8_pow2(w_exp[n0 + c + 1]) : 1.f;
    *reinterpret_cast<float2*>(acc_s + r0 * W8_ACC_LD + c) = make_float2(acc[4 * i] * w0, acc[4 * i + 1] * w1);
    *reinterpret_cast<float2*>(acc_s + (r0 + 8) * W8_ACC_LD + c) = make_float2(acc[4 * i + 2] * w0, acc[4 * i + 3] * w1);
  }
  named_bar_sync(1, 256);

  // ---- epilogue: thread = one output row, 32-column chunks split between the two halves of the consumers ----
  const uint32_t rl = threadIdx.x & 127, half = threadIdx.x >> 7;
  const uint32_t row = m0 + rl;
  if (row >= M) return;
  const float* arow = acc_s + rl * W8_ACC_LD;
  const bool do_add = addend != nullptr;
#pragma unroll 1
  for (uint32_t c = half * 32; c < W8_BN; c += 64) {
    const uint32_t col = n0 + c;
    if (col >= N) break;
    __nv_bfloat16* dst = C + static_cast<int64_t>(row) * ldc + col;
    const __nv_bfloat16* add = do_add ? addend + static_cast<int64_t>(row) * ld_add + col : nullptr;
    if (col + 32 <= N && (ldc & 7) == 0 && (!do_add || (ld_add & 7) == 0)) {
#pragma unroll
      for (uint32_t j = 0; j < 32; j += 8) {
        const float4 v0 = *reinterpret_cast<const float4*>(arow + c + j);
        const float4 v1 = *reinterpret_cast<const float4*>(arow + c + j + 4);
        uint4 o = make_uint4(pack_bf16x2(v0.x, v0.y), pack_bf16x2(v0.z, v0.w), pack_bf16x2(v1.x, v1.y), pack_bf16x2(v1.z, v1.w));
        if (do_add) {
          const uint4 a = *reinterpret_cast<const uint4*>(add + j);
          o.x = pack_bf16x2(bf16_lo(o.x) + bf16_lo(a.x), bf16_hi(o.x) + bf16_hi(a.x));
          o.y = pack_bf16x2(bf16_lo(o.y) + bf16_lo(a.y), bf16_hi(o.y) + bf16_hi(a.y));
          o.z = pack_bf16x2(bf16_lo(o.z) + bf16_lo(a.z), bf16_hi(o.z) + bf16_hi(a.z));
          o.w = pack_bf16x2(bf16_lo(o.w) + bf16_lo(a.w), bf16_hi(o.w) + bf16_hi(a.w));
        }
        *reinterpret_cast<uint4*>(dst + j) = o;
      }
    } else {
      for (uint32_t j = 0; j < 32 && col + j < N; ++j) {
        float x = bf16_round(arow[c + j]);
        if (do_add) x = x + __bfloat162float(add[j]);
        dst[j] = __float2bfloat16_rn(x);
      }
    }
  }
}

// ---- activation quantizer: one warp per (row, 128-column block), 4 elements per lane ----
constexpr int QA_THREADS = 256;

__global__ void __launch_bounds__(QA_THREADS)
quantize_act_fp8_kernel(const __nv_bfloat16* __restrict__ X, int64_t ldx, uint8_t* __restrict__ Q, int64_t ldq,
                        int8_t* __restrict__ E, int64_t lde, int M, int KB) {
  const int64_t task = static_cast<int64_t>(blockIdx.x) * (QA_THREADS / 32) + (threadIdx.x >> 5);
  if (task >= static_cast<int64_t>(M) * KB) return;
  const int64_t m = task / KB;
  const int kb = static_cast<int>(task - m * KB);
  const uint32_t lane = threadIdx.x & 31;
  const uint2 v = *reinterpret_cast<const uint2*>(X + m * ldx + kb * 128 + lane * 4);
  // amax on the bf16 bit patterns (bf16x8_amax_bits on four elements), then the exponent rule of the weight format
  uint32_t a = max(max(v.x & 0x7FFFu, (v.x >> 16) & 0x7FFFu), max(v.y & 0x7FFFu, (v.y >> 16) & 0x7FFFu));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a = max(a, __shfl_xor_sync(0xffffffffu, a, o));
  const int e = fp8_row_exponent(__uint_as_float(a << 16));
  const float inv = fp8_pow2(-e);
  // the element arithmetic of fp8x8_from_bf16x8
  const uint32_t q = fp8x4_from_f32(bf16_lo(v.x) * inv, bf16_hi(v.x) * inv, bf16_lo(v.y) * inv, bf16_hi(v.y) * inv);
  *reinterpret_cast<uint32_t*>(Q + m * ldq + kb * 128 + lane * 4) = q;
  if (lane == 0) E[m * lde + kb] = static_cast<int8_t>(e);
}

}  // namespace nv

// Quantize the bf16 activation X [M, K] (row stride ldx) per (row, 128-column block) in the weight format of nv_fp8.cuh:
// Q [M, K] e4m3 bytes (row stride ldq bytes) and E [M, K/128] int8 exponents (row stride lde).
extern "C" int nv_quantize_act_fp8(const void* X, int64_t ldx, void* Q, int64_t ldq, void* E, int64_t lde, int M, int K,
                                   void* stream_) {
  using namespace nv;
  NV_REQUIRE(M > 0 && K > 0 && (K % 128) == 0, "nv_quantize_act_fp8: needs M > 0 and K %% 128 == 0 (got M=%d K=%d)", M, K);
  NV_REQUIRE(X && Q && E, "nv_quantize_act_fp8: null operand");
  NV_REQUIRE((ldx & 7) == 0 && (ldq & 15) == 0 && lde >= K / 128 && (reinterpret_cast<uintptr_t>(X) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(Q) & 15) == 0,
             "nv_quantize_act_fp8: X / Q must be 16-byte aligned with ldx %% 8 == 0, ldq %% 16 == 0 and lde >= K / 128");
  const int64_t tasks = static_cast<int64_t>(M) * (K / 128);
  const int64_t blocks = (tasks + QA_THREADS / 32 - 1) / (QA_THREADS / 32);
  quantize_act_fp8_kernel<<<static_cast<unsigned>(blocks), QA_THREADS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      reinterpret_cast<const __nv_bfloat16*>(X), ldx, reinterpret_cast<uint8_t*>(Q), ldq, reinterpret_cast<int8_t*>(E), lde, M,
      K / 128);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

// C[M,N] = A'[M,K] · W'[N,K]^T (+ addend), A' = (Aq, Ae) from nv_quantize_act_fp8, W' = (Wq, We) from nv_quantize_fp8_rows.
extern "C" int nv_gemm_w8a8_bf16(const void* Aq, int64_t lda, const void* Ae, int64_t lde, const void* Wq, int64_t ldw,
                                 const void* We, void* C, int64_t ldc, const void* addend, int64_t ld_add, int M, int N, int K,
                                 void* stream_) {
  using namespace nv;
  NV_REQUIRE(M > 0 && N > 0 && K > 0 && (K % 128) == 0, "nv_gemm_w8a8_bf16: needs K %% 128 == 0 (got M=%d N=%d K=%d)", M, N, K);
  NV_REQUIRE(Aq && Ae && Wq && We && C, "nv_gemm_w8a8_bf16: null operand");
  NV_REQUIRE((lda & 15) == 0 && (ldw & 15) == 0 && lde >= K / 128 && (ldc & 7) == 0 && (!addend || (ld_add & 7) == 0),
             "nv_gemm_w8a8_bf16: lda / ldw (bytes) must be multiples of 16, ldc / ld_add multiples of 8 and lde >= K / 128");
  const uint32_t num_kb = static_cast<uint32_t>(K) / W8_BK;
  NV_REQUIRE(w8_smem_bytes(num_kb) <= W8_SMEM_MAX, "nv_gemm_w8a8_bf16: K=%d is too deep for the exponent buffer", K);
  CUtensorMap ta, tb;
  int rc = make_tmap_2d(&ta, Aq, 1, (uint64_t)K, (uint64_t)M, (uint64_t)lda, W8_BK, W8_BM);
  if (rc) return rc;
  if ((rc = make_tmap_2d(&tb, Wq, 1, (uint64_t)K, (uint64_t)N, (uint64_t)ldw, W8_BK, W8_BN))) return rc;
  static bool attr_set = false;
  if (!attr_set) {
    NV_CUDA(cudaFuncSetAttribute(gemm_w8a8_wgmma, cudaFuncAttributeMaxDynamicSharedMemorySize, W8_SMEM_MAX));
    attr_set = true;
  }
  const uint32_t tiles = ceil_div_u32(M, W8_BM) * ceil_div_u32(N, W8_BN);
  gemm_w8a8_wgmma<<<tiles, W8_THREADS, w8_smem_bytes(num_kb), reinterpret_cast<cudaStream_t>(stream_)>>>(
      ta, tb, reinterpret_cast<const int8_t*>(Ae), lde, reinterpret_cast<const int8_t*>(We), reinterpret_cast<__nv_bfloat16*>(C),
      ldc, reinterpret_cast<const __nv_bfloat16*>(addend), ld_add, M, N, K);
  NV_LAUNCH_CHECK();
  return NV_OK;
}
