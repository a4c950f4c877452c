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
//
// The kernel is a template on the weight type.  bf16 weights are TMA-loaded straight into the 128-byte-swizzled layout
// wgmma reads.  e4m3 weights (one power-of-two scale per row, nv_fp8.cuh) stream half the bytes: the producer TMA-loads
// the fp8 tile unswizzled (64-byte rows), and each consumer warpgroup expands its 64 rows to bf16 (scale folded in) into a
// private swizzled buffer, then issues the same m64n16k16 SS wgmmas in the same k order over the same per-rank k range as
// the bf16 kernel, followed by the same rank-ordered reduction.  Those bf16 operands are bit for bit the W' the quantizer
// wrote back, so the fp8 kernel's output equals the bf16 kernel's on W'.  The fp8 stages use 10 KB instead of 18 KB; the
// freed shared memory holds the double-buffered bf16 expansion (2 warpgroups x 2 x 8 KB), so both kernels occupy the same
// 73 KB and three CTAs share an SM either way.
// 4-bit group-wise weights (SkInt4, nv_int4.cuh) take the other road: in swap-AB the weights are the wgmma A operand, which
// may come from registers, so each consumer thread dequantizes its pre-shuffled codes straight into m64n16k16 register-A
// fragments (exactly W') and issues register-A wgmmas over the same k range in the same order -- no expansion buffer,
// fence or barrier, and the next k-block's dequantization runs under the current wgmmas.
#include <stdlib.h>

#include "nv_common.cuh"
#include "nv_fp8.cuh"
#include "nv_host.h"
#include "nv_int4.cuh"

namespace nv {

constexpr uint32_t SK_BN = 128;      // weight rows per tile (MMA M)
constexpr uint32_t SK_BM = 16;       // activation rows (MMA N)
constexpr uint32_t SK_BK = 64;
constexpr uint32_t SK_STAGES = 4;
constexpr uint32_t SK_THREADS = 288;
constexpr uint32_t SK_X_BYTES = SK_BM * SK_BK * 2;
constexpr uint32_t SK_RED_BYTES = SK_BM * SK_BN * 4;   // one partner's partial tile [16 m][128 n] fp32 (8 KB)
constexpr uint32_t SK_CVT_BYTES = 64 * SK_BK * 2;      // one warpgroup's bf16 expansion of its 64 fp8 weight rows (8 KB)

// Shared-memory layout per weight type: [weight stages][fp8 only: 2 x 2 expansion buffers][activation stages][barriers]
template <typename WT>
struct SkLayout {
  static constexpr bool kFp8 = sizeof(WT) == 1, kInt4 = false;
  static constexpr uint32_t STAGES = SK_STAGES;
  static constexpr uint32_t W_BYTES = SK_BN * SK_BK * sizeof(WT);
  static constexpr uint32_t STAGE_BYTES = W_BYTES + SK_X_BYTES;            // TMA bytes per stage
  static constexpr uint32_t CVT_OFF = SK_STAGES * W_BYTES;
  static constexpr uint32_t X_OFF = CVT_OFF + (kFp8 ? 4 * SK_CVT_BYTES : 0);
  static constexpr uint32_t BAR_OFF = X_OFF + SK_STAGES * SK_X_BYTES;
  static constexpr uint32_t DYN_BYTES = BAR_OFF + 2 * SK_STAGES * 8 + 1024;
  static_assert(8 * SK_RED_BYTES <= X_OFF, "reduction buffers and the output tile reuse the weight stages (and expansion buffers)");
};

// 4-bit group-wise weights (nv_int4.cuh).  A k-block carries 4 KB of codes (two 2 KB chunks, one per consumer warpgroup),
// so ten 6 KB stages fit where the reduction needs 64 KB anyway; the reduction reuses weight and activation stages (all
// TMA loads have landed when the cluster synchronises after the main loop).  67 KB: three CTAs share an SM, as above.
struct SkInt4 {};
template <>
struct SkLayout<SkInt4> {
  static constexpr bool kFp8 = false, kInt4 = true;
  static constexpr uint32_t STAGES = 10;
  static constexpr uint32_t W_BYTES = 2 * Q4_CHUNK_BYTES;
  static constexpr uint32_t STAGE_BYTES = W_BYTES + SK_X_BYTES;
  static constexpr uint32_t X_OFF = STAGES * W_BYTES;
  static constexpr uint32_t BAR_OFF = X_OFF + STAGES * SK_X_BYTES > 8 * SK_RED_BYTES ? X_OFF + STAGES * SK_X_BYTES : 8 * SK_RED_BYTES;
  static constexpr uint32_t DYN_BYTES = BAR_OFF + 2 * STAGES * 8 + 1024;
};

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
// WT = uint8_t: W holds e4m3 bytes and w_scale the int8 exponent of each weight row (W' = e4m3 * 2^exp); unused for bf16.
// WT = SkInt4: tmap_w maps the packed codes (nv_int4.cuh) as [chunks x 2, 256] words, w_scale is the bf16 scale and w_zero
// the zero-point of each (row, 128-column group) ([rows, K / 128] row-major).
template <typename WT>
__global__ void __launch_bounds__(SK_THREADS)
gemm_skinny_wgmma(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x,
                  __nv_bfloat16* __restrict__ C, int64_t ldc, const __nv_bfloat16* __restrict__ addend, int64_t ld_add,
                  uint32_t M, uint32_t N, uint32_t K, uint32_t splits, uint32_t swiglu_f, const void* __restrict__ w_scale,
                  const uint8_t* __restrict__ w_zero) {
  using L = SkLayout<WT>;
  constexpr uint32_t SK_W_BYTES = L::W_BYTES, SK_STAGE_BYTES = L::STAGE_BYTES, SK_STAGES = L::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_w = smem;
  uint8_t* smem_x = smem + L::X_OFF;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
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
      if constexpr (L::kInt4) {                                                         // box {256 words, 2}: one chunk
        const int32_t kb = k0 / SK_BK, nkb_all = K / SK_BK;
        const int32_t rb0 = swiglu_f ? n_blk : 2 * n_blk, rb1 = swiglu_f ? swiglu_f / 64 + n_blk : 2 * n_blk + 1;
        tma_load_2d(smem_w + stage * SK_W_BYTES, &tmap_w, &full_bar[stage], 0, 2 * (rb0 * nkb_all + kb));
        tma_load_2d(smem_w + stage * SK_W_BYTES + Q4_CHUNK_BYTES, &tmap_w, &full_bar[stage], 0, 2 * (rb1 * nkb_all + kb));
      } else if (swiglu_f) {                                                                   // box {64 k, 64 n}: gate half, up half
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
  } else if constexpr (L::kInt4) {
    // Register-A wgmmas: thread t of the warpgroup dequantizes its 16 code bytes of a k-block (nv_int4.cuh) straight into
    // the A fragments of the four m64n16k16 steps.  While the wgmmas of k-block i run, the codes of k-block i + 1 are read
    // and dequantized into the other fragment set, and the scales / zero-points of k-block i + 2 are requested from global
    // memory.  Same k16 chain, per-rank k range and reduction as the bf16 kernel, on the bf16 values W'.
    const uint32_t t = threadIdx.x & 127;
    const int32_t n0 = swiglu_f ? n_blk * 64 : n_blk * SK_BN;
    const uint32_t w_rows = swiglu_f ? 2 * swiglu_f : N, G = K / Q4_GROUP;
    const __nv_bfloat16* sc = reinterpret_cast<const __nv_bfloat16*>(w_scale);
    int64_t gbase[2];                                        // (row, group 0) of the thread's rows r0, r1; -1: row >= w_rows
#pragma unroll
    for (uint32_t j = 0; j < 2; ++j) {
      const uint32_t tr = wg * 64 + ((t >> 5) << 4) + ((t & 31) >> 2) + 8 * j;
      const uint32_t r = swiglu_f ? (tr < 64 ? n0 + tr : swiglu_f + n0 + tr - 64) : n0 + tr;
      gbase[j] = r < w_rows ? (int64_t)r * G : -1;
    }
    // (s0x, z0x, s1x, z1x) of k-block kb; rows >= w_rows: s = 0 (their codes are TMA zero fill or padding)
    auto params = [&](uint32_t kb, uint32_t (&p)[4]) {
#pragma unroll
      for (uint32_t j = 0; j < 2; ++j) {
        uint32_t s = 0, z = 0;
        if (gbase[j] >= 0) {
          const int64_t gi = gbase[j] + (kb >> 1);
          s = __bfloat16_as_ushort(sc[gi]);
          z = w_zero[gi];
        }
        p[2 * j] = s * 0x10001u;
        p[2 * j + 1] = (0x4300u + z) * 0x10001u;
      }
    };
    auto dequant = [&](uint32_t stage, const uint32_t (&p)[4], uint32_t (&a)[4][4]) {
      const uint4 c = lds128(smem_u32(smem_w + stage * SK_W_BYTES + wg * Q4_CHUNK_BYTES) + 16 * t);
      q4_dequant_k16(c.x, p[0], p[1], p[2], p[3], a[0]);
      q4_dequant_k16(c.y, p[0], p[1], p[2], p[3], a[1]);
      q4_dequant_k16(c.z, p[0], p[1], p[2], p[3], a[2]);
      q4_dequant_k16(c.w, p[0], p[1], p[2], p[3], a[3]);
    };
    uint32_t pa[4], pb[4], fa[4][4], fb[4][4];
    // one k-block: wgmmas on `cur`; under them the next k-block's fragments into `nxt` (with its parameters `puse`) and
    // the request of k-block i + 2's parameters into `pload` (free: they served k-block i)
    auto step = [&](uint32_t i, uint32_t (&cur)[4][4], uint32_t (&nxt)[4][4], const uint32_t (&puse)[4], uint32_t (&pload)[4]) {
      const uint32_t stage = i % SK_STAGES;
      if (i + 2 < nkb) params(kb0 + i + 2, pload);
      const uint64_t xdesc = gmma_desc_sw128(smem_u32(smem_x + stage * SK_X_BYTES), 0, 1024);
      wgmma_fence();
#pragma unroll
      for (uint32_t k = 0; k < SK_BK / 16; ++k) wgmma_rs_bf16<16, 0>(acc, cur[k], xdesc + k * 2, 1u);
      wgmma_commit();
      if (i + 1 < nkb) {
        const uint32_t s1 = (i + 1) % SK_STAGES;
        mbar_wait(&full_bar[s1], ((i + 1) / SK_STAGES) & 1);
        dequant(s1, puse, nxt);
      }
      wgmma_wait<0>();
      if (t == 0) mbar_arrive(&empty_bar[stage]);
    };
    if (nkb > 0) {
      params(kb0, pa);
      if (nkb > 1) params(kb0 + 1, pb);
      mbar_wait(&full_bar[0], 0);
      dequant(0, pa, fa);
    }
    for (uint32_t i = 0; i < nkb; i += 2) {
      step(i, fa, fb, pb, pa);
      if (i + 1 < nkb) step(i + 1, fb, fa, pa, pb);
    }
    reg_fence(acc);
    griddep_wait();                                        // before the first read of `addend` / write of C
  } else if constexpr (L::kFp8) {
    // Expansion: thread t of the warpgroup owns 16-byte fp8 chunks q = t and t + 128 of the warpgroup's 64 x 64-byte rows
    // (row q / 4, k 16 (q % 4) ..+15) and writes them as bf16 chunks 2 (q % 4), 2 (q % 4) + 1 of the swizzled row.
    const uint32_t t = threadIdx.x & 127;
    const int32_t n0 = swiglu_f ? n_blk * 64 : n_blk * SK_BN;
    const uint32_t w_rows = swiglu_f ? 2 * swiglu_f : N;
    float scale[2];
#pragma unroll
    for (uint32_t j = 0; j < 2; ++j) {
      const uint32_t tr = wg * 64 + (t >> 2) + 32 * j;                       // row of the 128-row tile
      const uint32_t r = swiglu_f ? (tr < 64 ? n0 + tr : swiglu_f + n0 + tr - 64) : n0 + tr;
      scale[j] = r < w_rows ? fp8_pow2(reinterpret_cast<const int8_t*>(w_scale)[r]) : 1.f;                    // rows >= w_rows are TMA zero fill
    }
    uint8_t* cvt = smem + L::CVT_OFF + wg * 2 * SK_CVT_BYTES;
    for (uint32_t i = 0; i < nkb; ++i) {
      const uint32_t stage = i % SK_STAGES, phase = (i / SK_STAGES) & 1;
      mbar_wait(&full_bar[stage], phase);
      // buffer i & 1 was last read by the wgmmas of iteration i - 2, which every thread of the warpgroup waited for
      // before the barrier of iteration i - 1
      const uint32_t cb = smem_u32(cvt + (i & 1) * SK_CVT_BYTES);
      const uint32_t src = smem_u32(smem_w + stage * SK_W_BYTES + wg * (SK_W_BYTES / 2));
#pragma unroll
      for (uint32_t j = 0; j < 2; ++j) {
        const uint32_t q = t + 128 * j, row = q >> 2, c = q & 3;
        uint4 v;
        asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(src + q * 16));
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        uint32_t o[8];
#pragma unroll
        for (uint32_t h = 0; h < 4; ++h) fp8x4_to_bf16x4(w[h], scale[j], o[2 * h], o[2 * h + 1]);
        sts128(cb + sw128_offset(row, 2 * c), o[0], o[1], o[2], o[3]);
        sts128(cb + sw128_offset(row, 2 * c + 1), o[4], o[5], o[6], o[7]);
      }
      fence_proxy_async_smem();                            // generic-proxy writes -> wgmma operand reads
      if (wg == 0) asm volatile("bar.sync 1, 128;" ::: "memory");   // the warpgroup's expansion is complete
      else asm volatile("bar.sync 2, 128;" ::: "memory");
      const uint64_t wdesc = gmma_desc_sw128(cb, 0, 1024);
      const uint64_t xdesc = gmma_desc_sw128(smem_u32(smem_x + stage * SK_X_BYTES), 0, 1024);
      wgmma_fence();
#pragma unroll
      for (uint32_t k = 0; k < SK_BK / 16; ++k) wgmma_ss_bf16<16, 0, 0>(acc, wdesc + k * 2, xdesc + k * 2, 1u);
      wgmma_commit();
      wgmma_wait<0>();
      if (t == 0) mbar_arrive(&empty_bar[stage]);
    }
    reg_fence(acc);
    griddep_wait();                                        // before the first read of `addend` / write of C
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

template <typename WT>
static int skinny_launch(const void* X, int64_t ldx, const void* W, int64_t ldw, const void* w_scale, void* C, int64_t ldc,
                         const void* addend, int64_t ld_add, int M, int N, int K, uint32_t swiglu_f, cudaStream_t stream,
                         const uint8_t* w_zero = nullptr) {
  using namespace nv;
  using L = SkLayout<WT>;
  CUtensorMap tw, tx;
  int rc;
  const uint64_t w_rows = swiglu_f ? 2ull * swiglu_f : (uint64_t)N;
  if constexpr (L::kInt4) {
    // the packed codes as rows of 256 words, two per 2 KB chunk: chunks of row blocks past the weight are zero fill
    const uint64_t chunks = (w_rows + 63) / 64 * (uint64_t)(K / SK_BK);
    if ((rc = make_tmap_2d(&tw, W, 4, 256, 2 * chunks, 1024, 256, 2, /*swizzle128=*/false))) return rc;
  } else {
    // bf16: 128-byte swizzled box (wgmma reads it in place); fp8: plain 64-byte rows, expanded by the consumers
    if ((rc = make_tmap_2d(&tw, W, (int)sizeof(WT), (uint64_t)K, w_rows, (uint64_t)ldw * sizeof(WT), 64, swiglu_f ? 64 : SK_BN,
                           /*swizzle128=*/!L::kFp8)))
      return rc;
  }
  if ((rc = make_tmap_2d(&tx, X, 2, (uint64_t)K, (uint64_t)M, (uint64_t)ldx * 2, 64, SK_BM))) return rc;
  static bool attr_set = false;
  if (!attr_set) {
    NV_CUDA(cudaFuncSetAttribute(gemm_skinny_wgmma<WT>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::DYN_BYTES));
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
  cfg.dynamicSmemBytes = L::DYN_BYTES;
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
  NV_CUDA(cudaLaunchKernelEx(&cfg, gemm_skinny_wgmma<WT>, tw, tx, reinterpret_cast<__nv_bfloat16*>(C), ldc,
                             reinterpret_cast<const __nv_bfloat16*>(addend), ld_add, (uint32_t)M, (uint32_t)N, (uint32_t)K,
                             splits, swiglu_f, w_scale, w_zero));
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
  return skinny_launch<__nv_bfloat16>(X, ldx, W, ldw, nullptr, C, ldc, addend, ld_add, M, N, K, 0u,
                                      reinterpret_cast<cudaStream_t>(stream_));
}

// h[M,F] = bf16( bf16(silu(g)) * u ) with [g | u] = bf16(X[M,K] · Wgu[2F,K]^T): the decode step's gate/up projection and
// SwiGLU in one kernel (HF LlamaMLP act_fn(gate_proj(x)) * up_proj(x)); F % 64 == 0.
extern "C" int nv_gemm_skinny_swiglu_bf16(const void* X, int64_t ldx, const void* Wgu, int64_t ldw, void* H, int64_t ldh, int M,
                                          int F, int K, void* stream_) {
  using namespace nv;
  NV_REQUIRE(M > 0 && M <= (int)SK_BM && F > 0 && K > 0 && (F % 64) == 0,
             "nv_gemm_skinny_swiglu_bf16: needs 1 <= M <= 16 and F %% 64 == 0 (got M=%d F=%d K=%d)", M, F, K);
  NV_REQUIRE(X && Wgu && H && (ldx & 7) == 0 && (ldw & 7) == 0, "nv_gemm_skinny_swiglu_bf16: null operand / alignment");
  return skinny_launch<__nv_bfloat16>(X, ldx, Wgu, ldw, nullptr, H, ldh, nullptr, 0, M, F, K, (uint32_t)F,
                                      reinterpret_cast<cudaStream_t>(stream_));
}

// The fp8-weight forms of the two entry points above: Wq holds e4m3 bytes (leading dimension ldw in bytes) and w_exp[r] the
// power-of-two exponent of weight row r, as written by nv_quantize_fp8_rows.  The result is bit-identical to the bf16 kernel
// on W' = e4m3 * 2^w_exp (same cluster split, k ranges, MMA order and reduction).
extern "C" int nv_gemm_skinny_fp8(const void* X, int64_t ldx, const void* Wq, int64_t ldw, const void* w_exp, void* C, int64_t ldc,
                                  const void* addend, int64_t ld_add, int M, int N, int K, void* stream_) {
  using namespace nv;
  NV_REQUIRE(M > 0 && M <= (int)SK_BM && N > 0 && K > 0, "nv_gemm_skinny_fp8: needs 1 <= M <= 16 (got M=%d N=%d K=%d)", M, N, K);
  NV_REQUIRE(X && Wq && w_exp && C, "nv_gemm_skinny_fp8: null operand");
  NV_REQUIRE((ldx & 7) == 0 && (ldw & 15) == 0, "nv_gemm_skinny_fp8: ldx must be a multiple of 8 and ldw (bytes) of 16");
  return skinny_launch<uint8_t>(X, ldx, Wq, ldw, w_exp, C, ldc, addend, ld_add, M, N, K, 0u,
                                reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int nv_gemm_skinny_swiglu_fp8(const void* X, int64_t ldx, const void* Wgu_q, int64_t ldw, const void* w_exp, void* H,
                                         int64_t ldh, int M, int F, int K, void* stream_) {
  using namespace nv;
  NV_REQUIRE(M > 0 && M <= (int)SK_BM && F > 0 && K > 0 && (F % 64) == 0,
             "nv_gemm_skinny_swiglu_fp8: needs 1 <= M <= 16 and F %% 64 == 0 (got M=%d F=%d K=%d)", M, F, K);
  NV_REQUIRE(X && Wgu_q && w_exp && H && (ldx & 7) == 0 && (ldw & 15) == 0,
             "nv_gemm_skinny_swiglu_fp8: null operand / alignment");
  return skinny_launch<uint8_t>(X, ldx, Wgu_q, ldw, w_exp, H, ldh, nullptr, 0, M, F, K,
                                (uint32_t)F, reinterpret_cast<cudaStream_t>(stream_));
}

// The 4-bit forms (W4A16): codes packed by nv_quantize_int4_groups, scales [N, K / 128] bf16 and zeros [N, K / 128] uint8
// (for the SwiGLU form, of the fused [2F, K] gate|up weight).  The result is bit-identical to the bf16 kernel on
// W' = bf16((q - z) * s): same cluster split, k ranges, k16 MMA chain and reduction; a rank's range may start inside a group.
extern "C" int nv_gemm_skinny_int4(const void* X, int64_t ldx, const void* codes, const void* scales, const void* zeros, void* C,
                                   int64_t ldc, const void* addend, int64_t ld_add, int M, int N, int K, void* stream_) {
  using namespace nv;
  NV_REQUIRE(M > 0 && M <= (int)SK_BM && N > 0 && K > 0 && (K % (int)Q4_GROUP) == 0,
             "nv_gemm_skinny_int4: needs 1 <= M <= 16 and K %% 128 == 0 (got M=%d N=%d K=%d)", M, N, K);
  NV_REQUIRE(X && codes && scales && zeros && C, "nv_gemm_skinny_int4: null operand");
  NV_REQUIRE((ldx & 7) == 0, "nv_gemm_skinny_int4: ldx must be a multiple of 8");
  return skinny_launch<SkInt4>(X, ldx, codes, 0, scales, C, ldc, addend, ld_add, M, N, K, 0u,
                               reinterpret_cast<cudaStream_t>(stream_), reinterpret_cast<const uint8_t*>(zeros));
}

extern "C" int nv_gemm_skinny_swiglu_int4(const void* X, int64_t ldx, const void* codes, const void* scales, const void* zeros,
                                          void* H, int64_t ldh, int M, int F, int K, void* stream_) {
  using namespace nv;
  NV_REQUIRE(M > 0 && M <= (int)SK_BM && F > 0 && K > 0 && (F % 64) == 0 && (K % (int)Q4_GROUP) == 0,
             "nv_gemm_skinny_swiglu_int4: needs 1 <= M <= 16, F %% 64 == 0 and K %% 128 == 0 (got M=%d F=%d K=%d)", M, F, K);
  NV_REQUIRE(X && codes && scales && zeros && H && (ldx & 7) == 0, "nv_gemm_skinny_swiglu_int4: null operand / alignment");
  return skinny_launch<SkInt4>(X, ldx, codes, 0, scales, H, ldh, nullptr, 0, M, F, K, (uint32_t)F,
                               reinterpret_cast<cudaStream_t>(stream_), reinterpret_cast<const uint8_t*>(zeros));
}
