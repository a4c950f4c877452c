// navillm_b200 — bf16 GEMM on Hopper warpgroup MMA (wgmma), the >97 %-of-FLOPs kernel of the path.
//
// Replaces the cuBLAS bf16 GEMMs the reference reaches through nn.Linear inside HF LLaMA
// (reference call sites: models/modified_lm.py:112-120 -> LlamaDecoderLayer q/k/v/o/gate/up/down
// projections and lm_head; SURVEY.md §2b K9/K10) and their autograd backward (dgrad / wgrad).
//
//   C[M,N] = A · B  (+ addend),  fp32 accumulation in registers, bf16 output
//
// Operand forms (all row-major bf16 in HBM, leading dimension in elements):
//   a_mn = 0 : A stored [M,K] (K contiguous)      a_mn = 1 : A stored [K,M] (M contiguous)
//   b_mn = 0 : B stored [N,K] (K contiguous)      b_mn = 1 : B stored [K,N] (N contiguous)
// so   linear fwd  Y = X W^T   -> (a_mn=0, b_mn=0),
//      dgrad       dX = dY W   -> (a_mn=0, b_mn=1),
//      wgrad       dW = dY^T X -> (a_mn=1, b_mn=1).
// wgmma reads MN-major bf16 operands directly (transpose bits of the instruction), so all four forms share one kernel.
//
// Structure: one 128 x BLOCK_N output tile per CTA, 288 threads.
//   warps 0..7 (two warpgroups)  consumers: warpgroup w computes rows 64 w .. 64 w + 63 with m64nBLOCK_Nk16 wgmmas
//                                straight from the shared-memory stages, one wgmma group in flight
//   warp 8 (1 lane)              TMA producer: 128-byte-swizzled tiles, STAGES-deep mbarrier ring
// Epilogue: the accumulators go through shared memory (the stage ring is free by then) so that each thread then owns
// one output row and 32 consecutive columns at a time: 16-byte global stores, and the fused epilogues below see whole
// rows (rotate-half pairs, the gate and up halves of SwiGLU, the per-head row sums of the attention backward).
// HBM layout assumptions: base pointers 16-byte aligned, leading dimensions multiples of 8 elements.
// Ragged M/N/K are handled by TMA zero-fill on loads and predicated stores.
#include "nv_common.cuh"
#include "nv_host.h"

namespace nv {

constexpr uint32_t GEMM_BLOCK_M = 128;
constexpr uint32_t GEMM_BLOCK_K = 64;
constexpr uint32_t GEMM_THREADS = 288;
constexpr uint32_t GEMM_CONSUMERS = 256;
constexpr uint32_t GEMM_GROUP_M = 16;  // m-blocks per rasterisation group (L2 reuse of B tiles)

enum GemmFlags : uint32_t {
  GEMM_ADD = 1u,        // C = bf16(bf16(acc) + addend)   (residual add / gradient accumulation)
  GEMM_OUT_F32 = 2u,    // C is fp32 (no bf16 rounding of the accumulator)
  GEMM_NO_GU = 4u,      // SWIGLU epilogue: inference, do not keep g|u
};

// Fused epilogues (EPI):
//   EPI_PLAIN   C = bf16(acc) (+addend) | fp32(acc)
//   EPI_SWIGLU  gate|up projection: the 256 accumulator columns of a tile are 128 gate columns (B rows n..) and the SAME
//               128 up columns (B rows F + n..); writes g,u into the fused [T,2F] buffer (kept for the backward) and
//               h = bf16(bf16(silu(g)) * u) into aux [T,F]   (HF LlamaMLP act_fn(gate)*up)
//   EPI_DSWIGLU down-projection dgrad: acc = dh; reads g,u from aux [T,2F] and writes dg = dh*u*silu'(g),
//               du = dh*silu(g) into C [T,2F] (the separate swiglu_bwd pass and the dh round trip disappear)
//   EPI_ATTND   o_proj dgrad: C = dO (gradient of the attention output) and, per row and 128-column head, the
//               D[h, t] = sum_d dO[t,h,d] * O[t,h,d] vector of the attention backward (aux = O; replaces attn_bwd_prep)
//   EPI_ROPE    fused q|k|v projection: columns < rope_cols get the rotate-half rotary embedding
//               (HF apply_rotary_pos_emb, bf16 rounding points preserved) with cos/sin[pos[row]] before the store
enum { EPI_PLAIN = 0, EPI_SWIGLU = 1, EPI_DSWIGLU = 2, EPI_ROPE = 3, EPI_ATTND = 4 };

struct EpiAux {
  void* aux;            // SWIGLU: h out [T,F];  DSWIGLU: gu in [T,2F];  ATTND: O in [T,D]
  int64_t ld_aux;
  uint32_t F;           // SWIGLU / DSWIGLU: intermediate size (columns of gate and of up)
  float* dvec;          // ATTND: D out [H, T] fp32 (T = M rows)
  const int* pos;       // ROPE
  const __nv_bfloat16* cos_t;
  const __nv_bfloat16* sin_t;
  uint32_t rope_cols;   // ROPE: q and k columns (2 * H * 128)
};

template <uint32_t BLOCK_N, uint32_t STAGES>
struct GemmSmem {
  static constexpr uint32_t A_BYTES = GEMM_BLOCK_M * GEMM_BLOCK_K * 2;
  static constexpr uint32_t B_BYTES = BLOCK_N * GEMM_BLOCK_K * 2;
  static constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr uint32_t BAR_OFF = STAGES * STAGE_BYTES;
  static constexpr uint32_t DYN_BYTES = BAR_OFF + 2 * STAGES * 8 + 1024;  // + slack for manual 1024-byte alignment
  static constexpr uint32_t ACC_LD = BLOCK_N + 4;                         // staged fp32 row (+16 B: conflict-free)
  static_assert(GEMM_BLOCK_M * ACC_LD * 4 <= BAR_OFF, "accumulator staging reuses the stage ring");
  static_assert(DYN_BYTES <= 232448, "shared memory per block");
};

__device__ __forceinline__ void tile_coords(uint32_t tile, uint32_t num_m, uint32_t num_n, uint32_t& m_blk,
                                            uint32_t& n_blk) {
  const uint32_t group_size = GEMM_GROUP_M * num_n;
  const uint32_t g = tile / group_size;
  const uint32_t first_m = g * GEMM_GROUP_M;
  const uint32_t gm = min(num_m - first_m, GEMM_GROUP_M);
  const uint32_t r = tile - g * group_size;
  m_blk = first_m + r % gm;
  n_blk = r / gm;
}

__device__ __forceinline__ float silu_bf16(float g) { return bf16_round(g / (1.f + __expf(-g))); }

// 32 consecutive staged fp32 accumulators of one row (bit patterns, the form the epilogue bodies take)
__device__ __forceinline__ void ld_acc32(const float* p, uint32_t (&v)[32]) {
#pragma unroll
  for (uint32_t j = 0; j < 32; j += 4) {
    const uint4 x = *reinterpret_cast<const uint4*>(p + j);
    v[j] = x.x; v[j + 1] = x.y; v[j + 2] = x.z; v[j + 3] = x.w;
  }
}

template <uint32_t BLOCK_N, uint32_t STAGES, bool A_MN, bool B_MN, int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_wgmma(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                void* __restrict__ Cout, int64_t ldc, const __nv_bfloat16* __restrict__ addend, int64_t ld_add,
                uint32_t M, uint32_t N, uint32_t K, uint32_t flags, EpiAux ea) {
  using L = GemmSmem<BLOCK_N, STAGES>;
  static_assert(EPI == EPI_PLAIN || BLOCK_N == 256, "fused epilogues use the 128 x 256 tile");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * L::A_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* empty_bar = full_bar + STAGES;

  const uint32_t warp = warp_id_uniform();
  // logical output columns per tile: BLOCK_N, except SWIGLU where the 256 accumulator columns are 128 gate + 128 up
  constexpr uint32_t TILE_N = (EPI == EPI_SWIGLU) ? 128u : BLOCK_N;
  const uint32_t num_m = ceil_div_u32(M, GEMM_BLOCK_M);
  const uint32_t num_n = ceil_div_u32(N, TILE_N);
  const uint32_t num_kb = ceil_div_u32(K, GEMM_BLOCK_K);
  uint32_t m_blk, n_blk;
  tile_coords(blockIdx.x, num_m, num_n, m_blk, n_blk);

  if (threadIdx.x == 0) {
    for (uint32_t i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);  // one arrive per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ===================== TMA producer =====================
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    const int32_t m0 = m_blk * GEMM_BLOCK_M;
    uint32_t stage = 0, phase = 0;
    for (uint32_t kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&empty_bar[stage], phase ^ 1);
      if (elect_one()) {
        mbar_arrive_expect_tx(&full_bar[stage], L::STAGE_BYTES);
        const int32_t k0 = kb * GEMM_BLOCK_K;
        uint8_t* sa = smem_a + stage * L::A_BYTES;
        uint8_t* sb = smem_b + stage * L::B_BYTES;
        if constexpr (!A_MN) {
          tma_load_2d(sa, &tmap_a, &full_bar[stage], k0, m0);  // box {64 k, 128 m}
        } else {
#pragma unroll
          for (uint32_t i = 0; i < GEMM_BLOCK_M / 64; ++i)  // box {64 m, 64 k} per 64-wide MN atom
            tma_load_2d(sa + i * (GEMM_BLOCK_K * 128), &tmap_a, &full_bar[stage], m0 + i * 64, k0);
        }
        if constexpr (!B_MN) {
          constexpr uint32_t BOX = BLOCK_N < 128 ? BLOCK_N : 128;  // box {64 k, BOX n}
#pragma unroll
          for (uint32_t i = 0; i < BLOCK_N / BOX; ++i) {
            const int32_t n0 = (EPI == EPI_SWIGLU) ? (int32_t)(n_blk * 128 + i * ea.F) : (int32_t)(n_blk * BLOCK_N + i * BOX);
            tma_load_2d(sb + i * BOX * 128, &tmap_b, &full_bar[stage], k0, n0);
          }
        } else {
#pragma unroll
          for (uint32_t i = 0; i < BLOCK_N / 64; ++i)
            tma_load_2d(sb + i * (GEMM_BLOCK_K * 128), &tmap_b, &full_bar[stage], n_blk * BLOCK_N + i * 64, k0);
        }
      }
      __syncwarp();
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    return;  // the producer takes no part in the epilogue (named barrier 1 counts the 256 consumer threads only)
  }

  // ===================== consumers (warpgroups 0, 1) =====================
  const uint32_t wg = warp >> 2;
  float acc[BLOCK_N / 2];
#pragma unroll
  for (uint32_t i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
  {
    // K-major: +32 B per k16 step inside the 128-byte swizzle span.  MN-major: LBO = one 64-wide MN atom (64 k rows
    // x 128 B), +16 k rows per step.  Warpgroup w's 64 A rows start 8 KB into the tile in both forms.
    constexpr uint32_t A_KADV = A_MN ? (16 * 128) >> 4 : (16 * 2) >> 4;
    constexpr uint32_t B_KADV = B_MN ? (16 * 128) >> 4 : (16 * 2) >> 4;
    constexpr uint32_t A_LBO = A_MN ? GEMM_BLOCK_K * 128 : 0, B_LBO = B_MN ? GEMM_BLOCK_K * 128 : 0;
    uint32_t stage = 0, phase = 0, prev = 0;
    for (uint32_t kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint64_t adesc = gmma_desc_sw128(smem_u32(smem_a + stage * L::A_BYTES + wg * 8192), A_LBO, 1024);
      const uint64_t bdesc = gmma_desc_sw128(smem_u32(smem_b + stage * L::B_BYTES), B_LBO, 1024);
      wgmma_fence();
#pragma unroll
      for (uint32_t k = 0; k < GEMM_BLOCK_K / 16; ++k)
        wgmma_ss_bf16<BLOCK_N, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, adesc + k * A_KADV, bdesc + k * B_KADV, 1u);
      wgmma_commit();
      wgmma_wait<1>();                                    // the previous k-block's wgmmas are done: free its stage
      if (kb > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    reg_fence(acc);
  }

  // ---- stage the accumulators: [128 rows][BLOCK_N + 4] fp32 over the (now idle) stage ring ----
  float* acc_s = reinterpret_cast<float*>(smem);
  named_bar_sync(1, GEMM_CONSUMERS);                      // both warpgroups are past their last wgmma
  {
    const uint32_t t = threadIdx.x & 127, lane = threadIdx.x & 31;
    const uint32_t r0 = wg * 64 + (t >> 5) * 16 + (lane >> 2);
#pragma unroll
    for (uint32_t i = 0; i < BLOCK_N / 8; ++i) {
      const uint32_t c = i * 8 + 2 * (lane & 3);
      *reinterpret_cast<float2*>(acc_s + r0 * L::ACC_LD + c) = make_float2(acc[4 * i], acc[4 * i + 1]);
      *reinterpret_cast<float2*>(acc_s + (r0 + 8) * L::ACC_LD + c) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
    }
  }
  named_bar_sync(1, GEMM_CONSUMERS);

  // ---- epilogue: thread = one output row, column chunks split between the two halves of the consumers ----
  const uint32_t rl = threadIdx.x & 127, half = threadIdx.x >> 7;
  const uint32_t row = m_blk * GEMM_BLOCK_M + rl;
  const uint32_t col0 = n_blk * TILE_N;
  const float* arow = acc_s + rl * L::ACC_LD;
  if (row >= M) return;
  if constexpr (EPI == EPI_SWIGLU) {
    __nv_bfloat16* gu = reinterpret_cast<__nv_bfloat16*>(Cout) + static_cast<int64_t>(row) * ldc;
    __nv_bfloat16* hrow = reinterpret_cast<__nv_bfloat16*>(ea.aux) + static_cast<int64_t>(row) * ea.ld_aux;
#pragma unroll 1
    for (uint32_t c = half * 32; c < 128; c += 64) {
      uint32_t g[32], u[32];
      ld_acc32(arow + c, g);
      ld_acc32(arow + 128 + c, u);
      const uint32_t col = col0 + c;
      if (col < ea.F) {   // F % 128 == 0 is required by the host wrapper
#pragma unroll
        for (uint32_t j = 0; j < 32; j += 8) {
          uint4 og, ou, oh;
          uint32_t* pg = &og.x; uint32_t* pu = &ou.x; uint32_t* ph = &oh.x;
#pragma unroll
          for (uint32_t q = 0; q < 4; ++q) {
            pg[q] = pack_bf16x2(__uint_as_float(g[j + 2 * q]), __uint_as_float(g[j + 2 * q + 1]));
            pu[q] = pack_bf16x2(__uint_as_float(u[j + 2 * q]), __uint_as_float(u[j + 2 * q + 1]));
            ph[q] = pack_bf16x2(silu_bf16(bf16_lo(pg[q])) * bf16_lo(pu[q]), silu_bf16(bf16_hi(pg[q])) * bf16_hi(pu[q]));
          }
          if ((flags & GEMM_NO_GU) == 0) {
            *reinterpret_cast<uint4*>(gu + col + j) = og;
            *reinterpret_cast<uint4*>(gu + ea.F + col + j) = ou;
          }
          *reinterpret_cast<uint4*>(hrow + col + j) = oh;
        }
      }
    }
  } else if constexpr (EPI == EPI_DSWIGLU) {
    __nv_bfloat16* dgu = reinterpret_cast<__nv_bfloat16*>(Cout) + static_cast<int64_t>(row) * ldc;
    const __nv_bfloat16* gu = reinterpret_cast<const __nv_bfloat16*>(ea.aux) + static_cast<int64_t>(row) * ea.ld_aux;
#pragma unroll 1
    for (uint32_t c = half * 32; c < BLOCK_N; c += 64) {
      uint32_t v[32];
      ld_acc32(arow + c, v);
      const uint32_t col = col0 + c;
      if (col < ea.F) {   // F % 32 == 0 is required by the host wrapper
#pragma unroll
        for (uint32_t j = 0; j < 32; j += 8) {
          const uint4 gg = *reinterpret_cast<const uint4*>(gu + col + j);
          const uint4 uu = *reinterpret_cast<const uint4*>(gu + ea.F + col + j);
          const uint32_t* pg = &gg.x; const uint32_t* pu = &uu.x;
          uint4 og, ou;
          uint32_t* qg = &og.x; uint32_t* qu = &ou.x;
#pragma unroll
          for (uint32_t q = 0; q < 4; ++q) {
            float dg[2], du[2];
#pragma unroll
            for (uint32_t e = 0; e < 2; ++e) {
              const float d = bf16_round(__uint_as_float(v[j + 2 * q + e]));   // dh as the unfused path stores it
              const float gv = e ? bf16_hi(pg[q]) : bf16_lo(pg[q]);
              const float uv = e ? bf16_hi(pu[q]) : bf16_lo(pu[q]);
              const float sg = 1.f / (1.f + __expf(-gv));
              dg[e] = d * uv * (sg * (1.f + gv * (1.f - sg)));
              du[e] = d * (gv * sg);
            }
            qg[q] = pack_bf16x2(dg[0], dg[1]);
            qu[q] = pack_bf16x2(du[0], du[1]);
          }
          *reinterpret_cast<uint4*>(dgu + col + j) = og;
          *reinterpret_cast<uint4*>(dgu + ea.F + col + j) = ou;
        }
      }
    }
  } else if constexpr (EPI == EPI_ROPE) {
    __nv_bfloat16* crow = reinterpret_cast<__nv_bfloat16*>(Cout) + static_cast<int64_t>(row) * ldc;
    const int p = ea.pos[row];
    const __nv_bfloat16* cs = ea.cos_t + static_cast<int64_t>(p) * 128;
    const __nv_bfloat16* sn = ea.sin_t + static_cast<int64_t>(p) * 128;
#pragma unroll 1
    for (uint32_t it = half; it < 4; it += 2) {            // two 128-wide heads per tile x two 32-column chunks
      const uint32_t hh = (it >> 1) * 128, c = (it & 1) * 32;   // chunk c pairs with chunk c + 64 (rotate-half)
      uint32_t a[32], b[32];
      ld_acc32(arow + hh + c, a);
      ld_acc32(arow + hh + 64 + c, b);
      const uint32_t col = col0 + hh + c;
      if (col < N) {
        const bool rope = col < ea.rope_cols;
#pragma unroll
        for (uint32_t j = 0; j < 32; j += 8) {
          uint4 o1, o2;
          uint32_t* p1 = &o1.x; uint32_t* p2 = &o2.x;
          uint4 c1 = make_uint4(0, 0, 0, 0), s1 = c1, c2 = c1, s2 = c1;
          if (rope) {
            c1 = *reinterpret_cast<const uint4*>(cs + c + j);      s1 = *reinterpret_cast<const uint4*>(sn + c + j);
            c2 = *reinterpret_cast<const uint4*>(cs + 64 + c + j); s2 = *reinterpret_cast<const uint4*>(sn + 64 + c + j);
          }
          const uint32_t* pc1 = &c1.x; const uint32_t* ps1 = &s1.x; const uint32_t* pc2 = &c2.x; const uint32_t* ps2 = &s2.x;
#pragma unroll
          for (uint32_t q = 0; q < 4; ++q) {
            // projection output rounded to bf16 first (the reference ropes the bf16 q/k)
            const uint32_t xa = pack_bf16x2(__uint_as_float(a[j + 2 * q]), __uint_as_float(a[j + 2 * q + 1]));
            const uint32_t xb = pack_bf16x2(__uint_as_float(b[j + 2 * q]), __uint_as_float(b[j + 2 * q + 1]));
            if (rope) {
              const float y1l = bf16_round(bf16_lo(xa) * bf16_lo(pc1[q])) + bf16_round(-bf16_lo(xb) * bf16_lo(ps1[q]));
              const float y1h = bf16_round(bf16_hi(xa) * bf16_hi(pc1[q])) + bf16_round(-bf16_hi(xb) * bf16_hi(ps1[q]));
              const float y2l = bf16_round(bf16_lo(xb) * bf16_lo(pc2[q])) + bf16_round(bf16_lo(xa) * bf16_lo(ps2[q]));
              const float y2h = bf16_round(bf16_hi(xb) * bf16_hi(pc2[q])) + bf16_round(bf16_hi(xa) * bf16_hi(ps2[q]));
              p1[q] = pack_bf16x2(y1l, y1h);
              p2[q] = pack_bf16x2(y2l, y2h);
            } else {
              p1[q] = xa;
              p2[q] = xb;
            }
          }
          *reinterpret_cast<uint4*>(crow + col + j) = o1;
          *reinterpret_cast<uint4*>(crow + col + 64 + j) = o2;
        }
      }
    }
  } else if constexpr (EPI == EPI_ATTND) {
    // N % 128 == 0 and 16-byte aligned rows are required by the host wrapper; one 128-column head per half
    __nv_bfloat16* drow = reinterpret_cast<__nv_bfloat16*>(Cout) + static_cast<int64_t>(row) * ldc;
    const __nv_bfloat16* orow = reinterpret_cast<const __nv_bfloat16*>(ea.aux) + static_cast<int64_t>(row) * ea.ld_aux;
    const uint32_t hc = col0 + half * 128;
    if (hc < N) {
      float dsum = 0.f;
#pragma unroll 1
      for (uint32_t c = 0; c < 128; c += 32) {
        uint32_t v[32];
        ld_acc32(arow + half * 128 + c, v);
        const uint32_t col = hc + c;
#pragma unroll
        for (uint32_t j = 0; j < 32; j += 8) {
          uint4 o;
          o.x = pack_bf16x2(__uint_as_float(v[j + 0]), __uint_as_float(v[j + 1]));
          o.y = pack_bf16x2(__uint_as_float(v[j + 2]), __uint_as_float(v[j + 3]));
          o.z = pack_bf16x2(__uint_as_float(v[j + 4]), __uint_as_float(v[j + 5]));
          o.w = pack_bf16x2(__uint_as_float(v[j + 6]), __uint_as_float(v[j + 7]));
          const uint4 a = *reinterpret_cast<const uint4*>(orow + col + j);
          dsum += bf16_lo(o.x) * bf16_lo(a.x) + bf16_hi(o.x) * bf16_hi(a.x) + bf16_lo(o.y) * bf16_lo(a.y) + bf16_hi(o.y) * bf16_hi(a.y)
                + bf16_lo(o.z) * bf16_lo(a.z) + bf16_hi(o.z) * bf16_hi(a.z) + bf16_lo(o.w) * bf16_lo(a.w) + bf16_hi(o.w) * bf16_hi(a.w);
          *reinterpret_cast<uint4*>(drow + col + j) = o;
        }
      }
      ea.dvec[static_cast<int64_t>(hc >> 7) * M + row] = dsum;
    }
  } else {
    const bool do_add = (flags & GEMM_ADD) != 0;
    const bool out_f32 = (flags & GEMM_OUT_F32) != 0;
#pragma unroll 1
    for (uint32_t c = half * 32; c < BLOCK_N; c += 64) {
      uint32_t v[32];
      ld_acc32(arow + c, v);
      const uint32_t col = col0 + c;
      if (col >= N) break;
      if (out_f32) {
        float* dst = reinterpret_cast<float*>(Cout) + static_cast<int64_t>(row) * ldc + col;
        if (col + 32 <= N && (ldc & 3) == 0) {
#pragma unroll
          for (uint32_t j = 0; j < 32; j += 4)
            *reinterpret_cast<uint4*>(dst + j) = make_uint4(v[j], v[j + 1], v[j + 2], v[j + 3]);
        } else {
#pragma unroll
          for (uint32_t j = 0; j < 32; ++j)
            if (col + j < N) dst[j] = __uint_as_float(v[j]);
        }
      } else {
        __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(Cout) + static_cast<int64_t>(row) * ldc + col;
        const __nv_bfloat16* add = do_add ? addend + static_cast<int64_t>(row) * ld_add + col : nullptr;
        if (col + 32 <= N && (ldc & 7) == 0 && (!do_add || (ld_add & 7) == 0)) {
#pragma unroll
          for (uint32_t j = 0; j < 32; j += 8) {
            uint4 o;
            o.x = pack_bf16x2(__uint_as_float(v[j + 0]), __uint_as_float(v[j + 1]));
            o.y = pack_bf16x2(__uint_as_float(v[j + 2]), __uint_as_float(v[j + 3]));
            o.z = pack_bf16x2(__uint_as_float(v[j + 4]), __uint_as_float(v[j + 5]));
            o.w = pack_bf16x2(__uint_as_float(v[j + 6]), __uint_as_float(v[j + 7]));
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
#pragma unroll
          for (uint32_t j = 0; j < 32; ++j) {
            if (col + j < N) {
              float x = bf16_round(__uint_as_float(v[j]));
              if (do_add) x = x + __bfloat162float(add[j]);
              dst[j] = __float2bfloat16_rn(x);
            }
          }
        }
      }
    }
  }
}

template <uint32_t BN, uint32_t ST, bool A_MN, bool B_MN, int EPI = EPI_PLAIN>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, void* C, int64_t ldc, const void* addend,
                       int64_t ld_add, uint32_t M, uint32_t N, uint32_t K, uint32_t flags, cudaStream_t stream,
                       EpiAux ea = EpiAux{}) {
  using L = GemmSmem<BN, ST>;
  auto kern = gemm_bf16_wgmma<BN, ST, A_MN, B_MN, EPI>;
  static bool attr_set = false;
  if (!attr_set) {
    NV_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::DYN_BYTES));
    attr_set = true;
  }
  const uint32_t tiles = ceil_div_u32(M, GEMM_BLOCK_M) * ceil_div_u32(N, EPI == EPI_SWIGLU ? 128u : BN);
  kern<<<tiles, GEMM_THREADS, L::DYN_BYTES, stream>>>(ta, tb, C, ldc, reinterpret_cast<const __nv_bfloat16*>(addend), ld_add,
                                                      M, N, K, flags, ea);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

// TMA maps of the two operands for a BLOCK_N-wide tile (B boxes of at most 128 rows when K-major).
static int gemm_tmaps(CUtensorMap* ta, CUtensorMap* tb, const void* A, int64_t lda, int a_mn, const void* B, int64_t ldb,
                      int b_mn, int M, int N, int K, uint32_t block_n, uint64_t b_rows) {
  int rc;
  if (!a_mn) rc = make_tmap_2d(ta, A, 2, (uint64_t)K, (uint64_t)M, (uint64_t)lda * 2, 64, GEMM_BLOCK_M);
  else       rc = make_tmap_2d(ta, A, 2, (uint64_t)M, (uint64_t)K, (uint64_t)lda * 2, 64, GEMM_BLOCK_K);
  if (rc) return rc;
  if (!b_mn) rc = make_tmap_2d(tb, B, 2, (uint64_t)K, b_rows, (uint64_t)ldb * 2, 64, block_n < 128 ? block_n : 128);
  else       rc = make_tmap_2d(tb, B, 2, (uint64_t)N, (uint64_t)K, (uint64_t)ldb * 2, 64, GEMM_BLOCK_K);
  return rc;
}

}  // namespace nv

extern "C" int nv_gemm_bf16(const void* A, int64_t lda, int a_mn, const void* B, int64_t ldb, int b_mn, void* C,
                            int64_t ldc, const void* addend, int64_t ld_add, int M, int N, int K, unsigned flags,
                            int block_n, void* stream_) {
  using namespace nv;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  NV_REQUIRE(M > 0 && N > 0 && K > 0, "nv_gemm_bf16: empty problem M=%d N=%d K=%d", M, N, K);
  NV_REQUIRE(A && B && C, "nv_gemm_bf16: null operand");
  NV_REQUIRE(!(flags & GEMM_ADD) || addend, "nv_gemm_bf16: GEMM_ADD without addend");
  NV_REQUIRE(!((flags & GEMM_ADD) && (flags & GEMM_OUT_F32)), "nv_gemm_bf16: ADD with fp32 output unsupported");
  NV_REQUIRE((lda & 7) == 0 && (ldb & 7) == 0, "nv_gemm_bf16: lda/ldb must be multiples of 8 (got %lld, %lld)",
             (long long)lda, (long long)ldb);
  // auto: the 128 x 256 tile once the problem fills the GPU with it; otherwise 128-wide tiles, whose larger tile count
  // gives mid-sized problems more parallelism.  Skinny activations (M <= 128) against K-major weights stream the weights
  // from HBM: 32-wide tiles put every SM on that stream unless N is so wide that 128-column tiles already do.  Every
  // variant accumulates the k-blocks in the same order, so the choice does not change a single output bit.
  if (block_n == 0) {
    const long wide_tiles = ((long)(M + 127) / 128) * ((long)(N + 255) / 256);
    block_n = (wide_tiles >= sm_count() && M >= 512) ? 256 : 128;
    if (M <= 128 && !a_mn && !b_mn) block_n = N <= 4096 ? 32 : 128;
  }
  NV_REQUIRE(block_n == 32 || block_n == 128 || block_n == 256, "nv_gemm_bf16: block_n must be 32, 128 or 256");
  NV_REQUIRE(!(block_n == 32 && b_mn), "nv_gemm_bf16: block_n = 32 (skinny-M weight streaming) needs a K-major B");

  CUtensorMap ta, tb;
  int rc = gemm_tmaps(&ta, &tb, A, lda, a_mn, B, ldb, b_mn, M, N, K, (uint32_t)block_n, (uint64_t)N);
  if (rc) return rc;

#define NV_GEMM_CASE(BN, ST)                                                                                       \
  do {                                                                                                             \
    if (!a_mn && !b_mn) return launch_gemm<BN, ST, false, false>(ta, tb, C, ldc, addend, ld_add, M, N, K, flags, stream); \
    if (!a_mn && b_mn) return launch_gemm<BN, ST, false, true>(ta, tb, C, ldc, addend, ld_add, M, N, K, flags, stream);   \
    if (a_mn && b_mn) return launch_gemm<BN, ST, true, true>(ta, tb, C, ldc, addend, ld_add, M, N, K, flags, stream);     \
    return launch_gemm<BN, ST, true, false>(ta, tb, C, ldc, addend, ld_add, M, N, K, flags, stream);                      \
  } while (0)

  if (block_n == 256) NV_GEMM_CASE(256, 4);
  if (block_n == 32) {
    // decode / pruned-row GEMMs (M <= 128): HBM-bound weight streaming; 10 stages keep ~40 KB of weights in flight per SM
    if (!a_mn) return launch_gemm<32, 10, false, false>(ta, tb, C, ldc, addend, ld_add, M, N, K, flags, stream);
    return launch_gemm<32, 10, true, false>(ta, tb, C, ldc, addend, ld_add, M, N, K, flags, stream);
  }
  NV_GEMM_CASE(128, 6);
#undef NV_GEMM_CASE
}

// ---- fused-epilogue entry points (K-major activations x nn.Linear weights) -------------------------------------
extern "C" {

// gu[T, 2F] = x[T,K] · Wgu[2F,K]^T  (gate rows then up rows)  and  h[T,F] = silu(g) * u   in one kernel.
int nv_gemm_swiglu_bf16(const void* x, int64_t ldx, const void* Wgu, int64_t ldw, void* gu, int64_t ldgu, void* h,
                        int64_t ldh, int M, int F, int K, int keep_gu, void* stream) {
  using namespace nv;
  NV_REQUIRE(M > 0 && F > 0 && K > 0 && (F % 128) == 0, "nv_gemm_swiglu_bf16: F must be a multiple of 128 (got %d)", F);
  NV_REQUIRE((ldx & 7) == 0 && (ldw & 7) == 0 && (ldgu & 7) == 0 && (ldh & 7) == 0, "nv_gemm_swiglu_bf16: alignment");
  CUtensorMap ta, tb;
  int rc = gemm_tmaps(&ta, &tb, x, ldx, 0, Wgu, ldw, 0, M, 2 * F, K, 256, (uint64_t)2 * F);
  if (rc) return rc;
  EpiAux ea{};
  ea.aux = h; ea.ld_aux = ldh; ea.F = (uint32_t)F;
  return launch_gemm<256, 4, false, false, EPI_SWIGLU>(ta, tb, gu, ldgu, nullptr, 0, M, F, K, keep_gu ? 0u : GEMM_NO_GU,
                                                       reinterpret_cast<cudaStream_t>(stream), ea);
}

// dgu[T,2F] = swiglu'(gu) applied to dh = dx[T,D] · Wd[D,F]   (Wd is the nn.Linear weight [D, F]: B stored [K=D, N=F]).
int nv_gemm_dswiglu_bf16(const void* dx, int64_t lddx, const void* Wd, int64_t ldw, const void* gu, int64_t ldgu, void* dgu,
                         int64_t lddgu, int M, int F, int D, void* stream) {
  using namespace nv;
  NV_REQUIRE(M > 0 && F > 0 && D > 0 && (F % 32) == 0, "nv_gemm_dswiglu_bf16: F %% 32");
  NV_REQUIRE((lddx & 7) == 0 && (ldw & 7) == 0 && (ldgu & 7) == 0 && (lddgu & 7) == 0, "nv_gemm_dswiglu_bf16: alignment");
  CUtensorMap ta, tb;
  int rc = gemm_tmaps(&ta, &tb, dx, lddx, 0, Wd, ldw, 1, M, F, D, 256, (uint64_t)F);
  if (rc) return rc;
  EpiAux ea{};
  ea.aux = const_cast<void*>(gu); ea.ld_aux = ldgu; ea.F = (uint32_t)F;
  return launch_gemm<256, 4, false, true, EPI_DSWIGLU>(ta, tb, dgu, lddgu, nullptr, 0, M, F, D, 0u,
                                                       reinterpret_cast<cudaStream_t>(stream), ea);
}

// dO[T, D] = dY[T, Dout] · Wo[Dout, D]  (o_proj dgrad; Wo is the nn.Linear weight, B stored [K = Dout, N = D]) and, in the
// same epilogue, dvec[h, t] = sum_d bf16(dO[t, h*128+d]) * O[t, h*128+d]: the D vector of the attention backward.
int nv_gemm_attnd_bf16(const void* dy, int64_t lddy, const void* Wo, int64_t ldw, const void* o, int64_t ldo, void* dout,
                       int64_t lddo, float* dvec, int M, int D, int Dout, void* stream) {
  using namespace nv;
  NV_REQUIRE(M > 0 && D > 0 && Dout > 0 && (D % 128) == 0 && o && dvec, "nv_gemm_attnd_bf16: D %% 128 and O / dvec required");
  NV_REQUIRE((lddy & 7) == 0 && (ldw & 7) == 0 && (ldo & 7) == 0 && (lddo & 7) == 0, "nv_gemm_attnd_bf16: alignment");
  CUtensorMap ta, tb;
  int rc = gemm_tmaps(&ta, &tb, dy, lddy, 0, Wo, ldw, 1, M, D, Dout, 256, (uint64_t)D);
  if (rc) return rc;
  EpiAux ea{};
  ea.aux = const_cast<void*>(o); ea.ld_aux = ldo; ea.dvec = dvec;
  return launch_gemm<256, 4, false, true, EPI_ATTND>(ta, tb, dout, lddo, nullptr, 0, M, D, Dout, 0u,
                                                     reinterpret_cast<cudaStream_t>(stream), ea);
}

// qkv[T, N] = x[T,K] · Wqkv[N,K]^T with rotate-half RoPE applied to the first rope_cols columns (q and k heads).
int nv_gemm_rope_bf16(const void* x, int64_t ldx, const void* W, int64_t ldw, void* out, int64_t ldo, const int* pos,
                      const void* cos_t, const void* sin_t, int M, int N, int K, int rope_cols, void* stream) {
  using namespace nv;
  NV_REQUIRE(M > 0 && N > 0 && K > 0 && (N % 128) == 0 && (rope_cols % 128) == 0, "nv_gemm_rope_bf16: head alignment");
  NV_REQUIRE((ldx & 7) == 0 && (ldw & 7) == 0 && (ldo & 7) == 0, "nv_gemm_rope_bf16: alignment");
  CUtensorMap ta, tb;
  int rc = gemm_tmaps(&ta, &tb, x, ldx, 0, W, ldw, 0, M, N, K, 256, (uint64_t)N);
  if (rc) return rc;
  EpiAux ea{};
  ea.pos = pos; ea.cos_t = reinterpret_cast<const __nv_bfloat16*>(cos_t); ea.sin_t = reinterpret_cast<const __nv_bfloat16*>(sin_t);
  ea.rope_cols = (uint32_t)rope_cols;
  return launch_gemm<256, 4, false, false, EPI_ROPE>(ta, tb, out, ldo, nullptr, 0, M, N, K, 0u,
                                                     reinterpret_cast<cudaStream_t>(stream), ea);
}

}  // extern "C"
