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
// The 128 x 256 tile, with the plain and the fused epilogues, is gemm_bf16_wide below: 2-CTA clusters that share the B
// tile by TMA multicast.
// Epilogue: the accumulators go through shared memory (the stage ring is free by then) so that each thread then owns
// one output row and 32 consecutive columns at a time: 16-byte global stores.
// HBM layout assumptions: base pointers 16-byte aligned, leading dimensions multiples of 8 elements.
// Ragged M/N/K are handled by TMA zero-fill on loads and predicated stores.
//
// fp8 weights (WT = uint8_t; EPI_PLAIN, K-major operands, BLOCK_N 32 / 128): B is the e4m3 copy of an nn.Linear weight with
// one power-of-two exponent per row (nv_fp8.cuh).  The producer TMA-loads the e4m3 tile unswizzled (64-byte rows, half the
// bytes of a bf16 stage) next to the bf16 A tile.  A fourth warpgroup (warps 9..12) expands each raw tile with
// fp8x4_to_bf16x4 into a bf16 buffer of its own stage, 128-byte swizzled exactly as the TMA writes a bf16 B tile, and signals
// a third mbarrier per stage; the consumers wait for it and run the unchanged SS wgmmas.  The expansion of stage s + 1
// overlaps the MMAs of stage s.  The k-blocks, the wgmma sequence and the epilogue are those of the bf16 kernel, and the
// expanded operand is bit for bit the W' the quantizer wrote back, so C equals nv_gemm_bf16's C on W'.
#include "nv_common.cuh"
#include "nv_fp8.cuh"
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
  uint32_t F;           // SWIGLU / DSWIGLU: intermediate size (columns of gate and of up); h, g, u, dg, du are TMA maps
  float* dvec;          // ATTND: D out [H, T] fp32 (T = M rows)
  const int* pos;       // ROPE
  const __nv_bfloat16* cos_t;
  const __nv_bfloat16* sin_t;
  uint32_t rope_cols;   // ROPE: q and k columns (2 * H * 128)
  const int8_t* w_exp;  // fp8 weights: w_exp[n] = exponent of weight row n (W' = e4m3 * 2^w_exp)
};

// Shared memory: [A stages][B stages][fp8 only: expanded bf16 B stages][full | empty | fp8 only: expanded barriers]
template <uint32_t BLOCK_N, uint32_t STAGES, typename WT = __nv_bfloat16>
struct GemmSmem {
  static constexpr bool kFp8 = sizeof(WT) == 1;
  static constexpr uint32_t THREADS = kFp8 ? GEMM_THREADS + 128 : GEMM_THREADS;   // + the expansion warpgroup
  static constexpr uint32_t A_BYTES = GEMM_BLOCK_M * GEMM_BLOCK_K * 2;
  static constexpr uint32_t B_BYTES = BLOCK_N * GEMM_BLOCK_K * sizeof(WT);
  static constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;                      // TMA bytes per stage
  static constexpr uint32_t CVT_BYTES = kFp8 ? BLOCK_N * GEMM_BLOCK_K * 2 : 0;
  static constexpr uint32_t CVT_OFF = STAGES * STAGE_BYTES;
  static constexpr uint32_t BAR_OFF = CVT_OFF + STAGES * CVT_BYTES;
  static constexpr uint32_t DYN_BYTES = BAR_OFF + (kFp8 ? 3 : 2) * STAGES * 8 + 1024;  // + slack for 1024-byte alignment
  static_assert(CVT_OFF % 1024 == 0, "the expanded stages are 128-byte-swizzle atoms");
  static constexpr uint32_t ACC_LD = BLOCK_N + 4;                         // staged fp32 row (+16 B: conflict-free)
  static_assert(GEMM_BLOCK_M * ACC_LD * 4 <= BAR_OFF, "accumulator staging reuses the stage ring");
  static_assert(DYN_BYTES <= 232448, "shared memory per block");
};

__device__ __forceinline__ void tile_coords(uint32_t tile, uint32_t num_m, uint32_t num_n, uint32_t& m_blk,
                                            uint32_t& n_blk, uint32_t group_m = GEMM_GROUP_M) {
  const uint32_t group_size = group_m * num_n;
  const uint32_t g = tile / group_size;
  const uint32_t first_m = g * group_m;
  const uint32_t gm = min(num_m - first_m, group_m);
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

template <uint32_t BLOCK_N, uint32_t STAGES, bool A_MN, bool B_MN, typename WT = __nv_bfloat16>
__global__ void __launch_bounds__(GemmSmem<BLOCK_N, STAGES, WT>::THREADS, 1)
gemm_bf16_wgmma(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                void* __restrict__ Cout, int64_t ldc, const __nv_bfloat16* __restrict__ addend, int64_t ld_add,
                uint32_t M, uint32_t N, uint32_t K, uint32_t flags, EpiAux ea) {
  using L = GemmSmem<BLOCK_N, STAGES, WT>;
  static_assert(BLOCK_N <= 128, "the 128 x 256 tile is gemm_bf16_wide");
  static_assert(!L::kFp8 || (!A_MN && !B_MN), "fp8 weights: K-major operands");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * L::A_BYTES;
  uint8_t* smem_cvt = smem + L::CVT_OFF;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* cvt_bar = empty_bar + STAGES;                 // fp8: the expanded bf16 B tile of the stage is complete

  const uint32_t warp = warp_id_uniform();
  const uint32_t num_m = ceil_div_u32(M, GEMM_BLOCK_M);
  const uint32_t num_n = ceil_div_u32(N, BLOCK_N);
  const uint32_t num_kb = ceil_div_u32(K, GEMM_BLOCK_K);
  uint32_t m_blk, n_blk;
  tile_coords(blockIdx.x, num_m, num_n, m_blk, n_blk);

  if (threadIdx.x == 0) {
    for (uint32_t i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      // one arrive per consumer warpgroup (fp8: + one per expansion thread, after its reads of the raw tile)
      mbar_init(&empty_bar[i], L::kFp8 ? 2 + 128 : 2);
      if constexpr (L::kFp8) mbar_init(&cvt_bar[i], 128);
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
        if constexpr (L::kFp8) {
          tma_load_2d(sb, &tmap_b, &full_bar[stage], k0, n_blk * BLOCK_N);   // box {64 k, BLOCK_N n}, unswizzled e4m3
        } else if constexpr (!B_MN) {
          constexpr uint32_t BOX = BLOCK_N < 128 ? BLOCK_N : 128;  // box {64 k, BOX n}
#pragma unroll
          for (uint32_t i = 0; i < BLOCK_N / BOX; ++i) {
            tma_load_2d(sb + i * BOX * 128, &tmap_b, &full_bar[stage], k0, n_blk * BLOCK_N + i * BOX);
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

  if constexpr (L::kFp8) {
    if (warp >= 9) {
      // ===================== fp8 expansion (warps 9..12) =====================
      // thread t owns the 16-byte e4m3 chunks q = t + 128 j of the tile (row q / 4, k 16 (q % 4) ..+15) and writes them as
      // bf16 chunks 2 (q % 4), 2 (q % 4) + 1 of the swizzled row.  Rows >= N are TMA zero fill (scale 1).
      constexpr uint32_t J = BLOCK_N * GEMM_BLOCK_K / 16 / 128;
      const uint32_t t = threadIdx.x - GEMM_THREADS;
      float scale[J];
#pragma unroll
      for (uint32_t j = 0; j < J; ++j) {
        const uint32_t n = n_blk * BLOCK_N + ((t + 128 * j) >> 2);
        scale[j] = n < N ? fp8_pow2(ea.w_exp[n]) : 1.f;
      }
      uint32_t stage = 0, phase = 0;
      for (uint32_t kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        // the consumers released this stage's expanded buffer (empty_bar) before the producer refilled it
        const uint32_t src = smem_u32(smem_b + stage * L::B_BYTES);
        const uint32_t dst = smem_u32(smem_cvt + stage * L::CVT_BYTES);
#pragma unroll
        for (uint32_t j = 0; j < J; ++j) {
          const uint32_t q = t + 128 * j, row = q >> 2, c = q & 3;
          uint4 v;
          asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(src + q * 16));
          uint32_t o[8];
          fp8x4_to_bf16x4(v.x, scale[j], o[0], o[1]);
          fp8x4_to_bf16x4(v.y, scale[j], o[2], o[3]);
          fp8x4_to_bf16x4(v.z, scale[j], o[4], o[5]);
          fp8x4_to_bf16x4(v.w, scale[j], o[6], o[7]);
          sts128(dst + sw128_offset(row, 2 * c), o[0], o[1], o[2], o[3]);
          sts128(dst + sw128_offset(row, 2 * c + 1), o[4], o[5], o[6], o[7]);
        }
        fence_proxy_async_smem();                          // generic-proxy writes -> wgmma operand reads
        mbar_arrive(&cvt_bar[stage]);
        mbar_arrive(&empty_bar[stage]);                    // this thread's part of the raw e4m3 tile has been read
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      return;
    }
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
    // K > 0 (host check): without this ptxas keeps a zero-trip path that writes the accumulators outside the wgmma
    // pipeline and serializes the wgmmas (warning C7515)
    __builtin_assume(num_kb > 0);
    for (uint32_t kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      if constexpr (L::kFp8) mbar_wait(&cvt_bar[stage], phase);
      const uint64_t adesc = gmma_desc_sw128(smem_u32(smem_a + stage * L::A_BYTES + wg * 8192), A_LBO, 1024);
      const uint64_t bdesc = gmma_desc_sw128(smem_u32(L::kFp8 ? smem_cvt + stage * L::CVT_BYTES : smem_b + stage * L::B_BYTES),
                                             B_LBO, 1024);
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
  const uint32_t col0 = n_blk * BLOCK_N;
  const float* arow = acc_s + rl * L::ACC_LD;
  if (row >= M) return;
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

template <uint32_t BN, uint32_t ST, bool A_MN, bool B_MN, typename WT = __nv_bfloat16>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, void* C, int64_t ldc, const void* addend,
                       int64_t ld_add, uint32_t M, uint32_t N, uint32_t K, uint32_t flags, cudaStream_t stream,
                       EpiAux ea = EpiAux{}) {
  using L = GemmSmem<BN, ST, WT>;
  auto kern = gemm_bf16_wgmma<BN, ST, A_MN, B_MN, WT>;
  static bool attr_set = false;
  if (!attr_set) {
    NV_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::DYN_BYTES));
    attr_set = true;
  }
  const uint32_t tiles = ceil_div_u32(M, GEMM_BLOCK_M) * ceil_div_u32(N, BN);
  kern<<<tiles, L::THREADS, L::DYN_BYTES, stream>>>(ta, tb, C, ldc, reinterpret_cast<const __nv_bfloat16*>(addend), ld_add,
                                                      M, N, K, flags, ea);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

// ================================ 128 x 256 tile: 2-CTA clusters sharing B ================================
// The two CTAs of a cluster (ranks 0, 1) compute the M-adjacent tiles (2 mp + rank, n) of one tile pair, pairs in the
// grouped raster order.  Per 64-deep k-block each CTA TMA-loads its own A tile and one half of the shared B tile,
// multicast into the same stage offset of both CTAs: 32 KB from L2 per CTA instead of 48 KB.  Every CTA's full
// barrier expects the whole 48 KB stage; a stage is refilled only after the consumer warpgroups of both CTAs released
// it (each arrives on the empty barrier of both CTAs).  The partner of the last tile of an odd m-block count lies past
// M: it loads its half of B and zero-filled A, and stores nothing.  The accumulator is rounded to bf16 and drained
// through a 32 KB half-tile buffer in two passes.  Each tile still accumulates its k-blocks in one chain, in order,
// with the m64n256k16 sequence, so C is bit for bit that of the 128-wide gemm_bf16_wgmma.  The fused epilogues
// (EPI != EPI_PLAIN) skip the staging buffer: see "fused epilogues of the wide tile" below.
constexpr uint32_t WIDE_N = 256;
constexpr uint32_t WIDE_STAGES = 4;
constexpr uint32_t WIDE_CLUSTER = 2;

struct WideSmem {
  static constexpr uint32_t A_BYTES = GEMM_BLOCK_M * GEMM_BLOCK_K * 2;
  static constexpr uint32_t B_BYTES = WIDE_N * GEMM_BLOCK_K * 2;
  static constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr uint32_t STG_OFF = WIDE_STAGES * STAGE_BYTES;
  static constexpr uint32_t STG_BYTES = GEMM_BLOCK_M * 128 * 2;           // bf16 [128 rows][128 columns]
  static constexpr uint32_t BAR_OFF = STG_OFF + STG_BYTES;
  static constexpr uint32_t DYN_BYTES = BAR_OFF + (2 * WIDE_STAGES + 1) * 8 + 1024;   // + slack for 1024-byte alignment
  static_assert(DYN_BYTES <= 232448, "shared memory per block");
};

// Staging buffer: 16 chunks of 16 bytes (8 columns) per 256-byte row, chunk c of row r stored at chunk c ^ (r % 8):
// the fragment writes (8 rows x 4 lanes) and the row reads (8 threads, one row each) are both conflict-free.
__device__ __forceinline__ uint32_t stg_offset(uint32_t row, uint32_t chunk) {
  return row * 256u + ((chunk ^ (row & 7u)) << 4);
}
// Pass p stages tile columns [64 p, 64 p + 64) in chunks 0..7 and [128 + 64 p, 128 + 64 p + 64) in chunks 8..15.
// Returns the staged chunk of the accumulator's 8-column group i (tile columns 8 i ..), or -1 when pass p does not
// hold it.
__device__ __forceinline__ int stg_chunk(uint32_t i, uint32_t p) {
  return ((i >> 3) & 1) == p ? int(i < 16 ? i - 8 * p : i - 8 - 8 * p) : -1;
}
// 32 staged columns (4 chunks from `chunk`) of row `row` as 16 packed bf16 pairs
__device__ __forceinline__ void ld_stg32(uint32_t stg, uint32_t row, uint32_t chunk, uint32_t (&w)[16]) {
#pragma unroll
  for (uint32_t q = 0; q < 4; ++q) {
    const uint4 x = lds128(stg + stg_offset(row, chunk + q));
    w[4 * q] = x.x; w[4 * q + 1] = x.y; w[4 * q + 2] = x.z; w[4 * q + 3] = x.w;
  }
}

// C[row, col .. col + 31] = w (+ addend), predicated on N
__device__ __forceinline__ void store_plain32(const uint32_t (&w)[16], void* Cout, int64_t ldc, const __nv_bfloat16* addend,
                                              int64_t ld_add, uint32_t row, uint32_t col, uint32_t N, bool do_add) {
  if (col >= N) return;
  __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(Cout) + static_cast<int64_t>(row) * ldc + col;
  const __nv_bfloat16* add = do_add ? addend + static_cast<int64_t>(row) * ld_add + col : nullptr;
  if (col + 32 <= N && (ldc & 7) == 0 && (!do_add || (ld_add & 7) == 0)) {
#pragma unroll
    for (uint32_t j = 0; j < 4; ++j) {
      uint4 o = make_uint4(w[4 * j], w[4 * j + 1], w[4 * j + 2], w[4 * j + 3]);
      if (do_add) {
        const uint4 a = *reinterpret_cast<const uint4*>(add + 8 * j);
        o.x = pack_bf16x2(bf16_lo(o.x) + bf16_lo(a.x), bf16_hi(o.x) + bf16_hi(a.x));
        o.y = pack_bf16x2(bf16_lo(o.y) + bf16_lo(a.y), bf16_hi(o.y) + bf16_hi(a.y));
        o.z = pack_bf16x2(bf16_lo(o.z) + bf16_lo(a.z), bf16_hi(o.z) + bf16_hi(a.z));
        o.w = pack_bf16x2(bf16_lo(o.w) + bf16_lo(a.w), bf16_hi(o.w) + bf16_hi(a.w));
      }
      *reinterpret_cast<uint4*>(dst + 8 * j) = o;
    }
  } else {
#pragma unroll
    for (uint32_t j = 0; j < 32; ++j) {
      if (col + j < N) {
        float x = (j & 1) ? bf16_hi(w[j >> 1]) : bf16_lo(w[j >> 1]);
        if (do_add) x = x + __bfloat162float(add[j]);
        dst[j] = __float2bfloat16_rn(x);
      }
    }
  }
}

// ---- fused epilogues of the wide tile ----
// The accumulator fragments are rounded and combined in registers (SwiGLU pairs accumulator group i with i + 16, RoPE
// with i + 8 in the same 128-column head: the same thread holds both) and written as bf16 into 64-column x 128-row
// boxes, 128-byte swizzled, in the idle stage ring; one thread then TMA-stores the boxes (clipped at M and at the
// column count) and waits only for their reads to finish before the kernel ends.  dSwiGLU and ATTND read an operand
// tile (g and u of gu, or O) that the producer TMA-loads into the ring while the last k-blocks compute.
constexpr uint32_t EPI_BOX_BYTES = GEMM_BLOCK_M * 128;    // one box: 128 rows of 64 bf16

// TMA maps of the fused epilogues: outputs in m[0], m[1], the prefetched operand in m[2], m[3], boxes {64, 128}.
//   SWIGLU  m[0] g -> gu[:, :F]   m[1] u -> gu[:, F:]   m[2] h -> h[T, F]
//   DSWIGLU m[0] dg -> dgu[:, :F] m[1] du -> dgu[:, F:] m[2] g <- gu[:, :F]  m[3] u <- gu[:, F:]
//   ROPE    m[0] q|k|v
//   ATTND   m[0] dO               m[2] O
// The halves of gu / dgu get a map each, so that TMA zero-fills and clips them at F.
struct EpiMaps {
  CUtensorMap m[4];
};

// Epilogue slot v (one box) in the idle stage ring: the stages in the order the producer would refill them after the
// last k-block, three slots per stage (its A tile, then the two halves of its B tile).  Slots 0..8 lie in the stages of
// k-blocks num_kb - 4 .. num_kb - 2 (or stages no k-block used), which are released while the last k-block computes.
__device__ __forceinline__ uint8_t* epi_slot(uint8_t* smem, uint32_t num_kb, uint32_t v) {
  const uint32_t s = (num_kb + v / 3) % WIDE_STAGES, j = v % 3;
  return j == 0 ? smem + s * WideSmem::A_BYTES
                : smem + WIDE_STAGES * WideSmem::A_BYTES + s * WideSmem::B_BYTES + (j - 1) * EPI_BOX_BYTES;
}
// byte offset, inside its box, of the bf16 pair of accumulator group i (tile columns 8 i ..) in row r held by `lane`
__device__ __forceinline__ uint32_t frag_offset(uint32_t r, uint32_t i, uint32_t lane) {
  return sw128_offset(r, i & 7) + 4 * (lane & 3);
}

template <bool A_MN, bool B_MN, int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_wide(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               const __grid_constant__ EpiMaps em, void* __restrict__ Cout, int64_t ldc,
               const __nv_bfloat16* __restrict__ addend, int64_t ld_add, uint32_t M, uint32_t N, uint32_t K,
               uint32_t flags, EpiAux ea) {
  using L = WideSmem;
  static_assert(EPI == EPI_PLAIN || (!A_MN && B_MN == (EPI == EPI_DSWIGLU || EPI == EPI_ATTND)),
                "fused epilogues: the operand forms of their entry points");
  // logical output columns per tile: WIDE_N, except SWIGLU where the 256 accumulator columns are 128 gate + 128 up
  constexpr uint32_t TILE_N = EPI == EPI_SWIGLU ? 128u : WIDE_N;
  // boxes the producer prefetches for the epilogue (g and u, or O)
  constexpr uint32_t PRE_BOXES = EPI == EPI_DSWIGLU ? 8 : EPI == EPI_ATTND ? 4 : 0;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + WIDE_STAGES * L::A_BYTES;
  const uint32_t stg = smem_u32(smem + L::STG_OFF);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* empty_bar = full_bar + WIDE_STAGES;
  uint64_t* epi_full = empty_bar + WIDE_STAGES;          // the prefetched epilogue operand has landed

  const uint32_t warp = warp_id_uniform();
  const uint32_t rank = cluster_ctarank();
  const uint32_t pair = blockIdx.x / WIDE_CLUSTER;
  const uint32_t num_m = ceil_div_u32(M, GEMM_BLOCK_M);
  const uint32_t num_mp = ceil_div_u32(num_m, WIDE_CLUSTER);
  const uint32_t num_n = ceil_div_u32(N, TILE_N);
  const uint32_t num_kb = ceil_div_u32(K, GEMM_BLOCK_K);

  if (threadIdx.x == 0) {
    for (uint32_t i = 0; i < WIDE_STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2 * WIDE_CLUSTER);      // one arrive per consumer warpgroup of every CTA of the cluster
    }
    mbar_init(epi_full, 1);
    fence_mbar_init();
  }
  cluster_sync_all();                                  // the peer's multicasts and arrivals target these barriers

  uint32_t mp, n_blk;
  tile_coords(pair, num_mp, num_n, mp, n_blk, GEMM_GROUP_M / WIDE_CLUSTER);
  const uint32_t m_blk = mp * WIDE_CLUSTER + rank;
  const int32_t m0 = m_blk * GEMM_BLOCK_M;
  const uint32_t col0 = n_blk * TILE_N;

  if (warp == 8) {
    // ===================== TMA producer =====================
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
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
        // B: K-major two boxes {64 k, 128 n} (SWIGLU: the gate rows n.. and the up rows F + n..), MN-major four boxes
        // {64 n, 64 k}; this CTA loads its 1 / WIDE_CLUSTER share of them into every CTA of the cluster
        constexpr uint32_t BOXES = B_MN ? WIDE_N / 64 : 2, BOX_BYTES = L::B_BYTES / BOXES;
#pragma unroll
        for (uint32_t j = 0; j < BOXES / WIDE_CLUSTER; ++j) {
          const uint32_t i = rank * (BOXES / WIDE_CLUSTER) + j;
          int32_t c0, c1;
          if constexpr (B_MN) { c0 = n_blk * WIDE_N + i * 64; c1 = k0; }
          else { c0 = k0; c1 = EPI == EPI_SWIGLU ? col0 + i * ea.F : n_blk * WIDE_N + i * 128; }
          tma_load_2d_multicast(sb + i * BOX_BYTES, &tmap_b, &full_bar[stage], c0, c1, (1u << WIDE_CLUSTER) - 1);
        }
      }
      __syncwarp();
      if (++stage == WIDE_STAGES) { stage = 0; phase ^= 1; }
    }
    if constexpr (PRE_BOXES > 0) {
      // The epilogue operand goes into the slots of the stages the ring would refill next, each as soon as the empty
      // barrier of its stage completes.  This CTA's own empty barrier is enough: it counts the release by the consumers
      // of both CTAs, and the partner's multicast into the stage had landed before this CTA's full barrier of the
      // stage's last k-block flipped; no later k-block writes the stage.  The loads are local, not multicast.
      if (m_blk < num_m) {
        if (elect_one()) mbar_arrive_expect_tx(epi_full, PRE_BOXES * EPI_BOX_BYTES);
        __syncwarp();
#pragma unroll
        for (uint32_t v0 = 0; v0 < PRE_BOXES; v0 += 3) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          if (elect_one()) {
#pragma unroll
            for (uint32_t v = v0; v < v0 + 3 && v < PRE_BOXES; ++v)   // DSWIGLU: g boxes 0..3, u boxes 4..7
              tma_load_2d(epi_slot(smem, num_kb, v), &em.m[2 + v / 4], epi_full, col0 + 64 * (v % 4), m0);
          }
          __syncwarp();
          if (++stage == WIDE_STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers (warpgroups 0, 1) =====================
    const uint32_t wg = warp >> 2, t = threadIdx.x & 127, lane = threadIdx.x & 31;
    const uint32_t r0 = wg * 64 + (t >> 5) * 16 + (lane >> 2);   // fragment rows r0, r0 + 8
    constexpr uint32_t A_KADV = A_MN ? (16 * 128) >> 4 : (16 * 2) >> 4;
    constexpr uint32_t B_KADV = B_MN ? (16 * 128) >> 4 : (16 * 2) >> 4;
    constexpr uint32_t A_LBO = A_MN ? GEMM_BLOCK_K * 128 : 0, B_LBO = B_MN ? GEMM_BLOCK_K * 128 : 0;
    uint32_t stage = 0, phase = 0;
    {
      float acc[WIDE_N / 2];
#pragma unroll
      for (uint32_t i = 0; i < WIDE_N / 2; ++i) acc[i] = 0.f;
      uint32_t prev = 0;
      // K > 0 (host check): see gemm_bf16_wgmma
      __builtin_assume(num_kb > 0);
      for (uint32_t kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint64_t adesc = gmma_desc_sw128(smem_u32(smem_a + stage * L::A_BYTES + wg * 8192), A_LBO, 1024);
        const uint64_t bdesc = gmma_desc_sw128(smem_u32(smem_b + stage * L::B_BYTES), B_LBO, 1024);
        wgmma_fence();
#pragma unroll
        for (uint32_t k = 0; k < GEMM_BLOCK_K / 16; ++k)
          wgmma_ss_bf16<WIDE_N, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, adesc + k * A_KADV, bdesc + k * B_KADV, 1u);
        wgmma_commit();
        wgmma_wait<1>();                                  // the previous k-block's wgmmas are done: free its stage
        if (kb > 0 && t == 0)
          for (uint32_t c = 0; c < WIDE_CLUSTER; ++c) mbar_arrive_cluster(&empty_bar[prev], c);
        prev = stage;
        if (++stage == WIDE_STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      reg_fence(acc);

      if constexpr (EPI == EPI_PLAIN) {
        // ---- epilogue: two passes of 128 bf16 columns; thread = one output row, warpgroup = half of the pass ----
        const bool do_add = (flags & GEMM_ADD) != 0;
        const uint32_t row = m_blk * GEMM_BLOCK_M + t;
#pragma unroll
        for (uint32_t p = 0; p < 2; ++p) {
          named_bar_sync(1, GEMM_CONSUMERS);              // the previous pass has drained the staging buffer
#pragma unroll
          for (uint32_t i = 0; i < WIDE_N / 8; ++i) {
            const int sc = stg_chunk(i, p);
            if (sc < 0) continue;
            sts32(stg + stg_offset(r0, sc) + 4 * (lane & 3), pack_bf16x2(acc[4 * i], acc[4 * i + 1]));
            sts32(stg + stg_offset(r0 + 8, sc) + 4 * (lane & 3), pack_bf16x2(acc[4 * i + 2], acc[4 * i + 3]));
          }
          named_bar_sync(1, GEMM_CONSUMERS);
          if (row >= M) continue;
#pragma unroll 1
          for (uint32_t h = 0; h < 2; ++h) {              // chunks 4 wg + 8 h.. = tile columns 128 h + 64 p + 32 wg ..
            uint32_t v[16];
            ld_stg32(stg, t, 8 * h + 4 * wg, v);
            store_plain32(v, Cout, ldc, addend, ld_add, row, col0 + 128 * h + 64 * p + 32 * wg, N, do_add);
          }
        }
      } else {
        // ---- fused epilogues: bf16 boxes in the stage ring, TMA stores ----
        named_bar_sync(1, GEMM_CONSUMERS);                // both warpgroups are past their last wgmma
        if (m_blk < num_m) {                              // (the partner past M stores nothing)
          uint8_t* slot[8];
#pragma unroll
          for (uint32_t v = 0; v < 8; ++v) slot[v] = epi_slot(smem, num_kb, v);
          // boxes to store: (slot, map, column); DSWIGLU stores in place over g and u
          constexpr uint32_t OUT_BOXES = EPI == EPI_SWIGLU ? 6 : EPI == EPI_DSWIGLU ? 8 : 4;
          constexpr uint32_t OUT_SLOT0 = EPI == EPI_ATTND ? 4 : 0;
          if constexpr (EPI == EPI_SWIGLU) {
            // g in slots 0, 1, u in 2, 3, h in 4, 5:  h = bf16(silu(g) * u) on the bf16 g and u
#pragma unroll
            for (uint32_t i = 0; i < 16; ++i) {
#pragma unroll
              for (uint32_t h = 0; h < 2; ++h) {
                const uint32_t g = pack_bf16x2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
                const uint32_t u = pack_bf16x2(acc[4 * (i + 16) + 2 * h], acc[4 * (i + 16) + 2 * h + 1]);
                const uint32_t off = frag_offset(r0 + 8 * h, i, lane);
                sts32(smem_u32(slot[i / 8]) + off, g);
                sts32(smem_u32(slot[2 + i / 8]) + off, u);
                sts32(smem_u32(slot[4 + i / 8]) + off,
                      pack_bf16x2(silu_bf16(bf16_lo(g)) * bf16_lo(u), silu_bf16(bf16_hi(g)) * bf16_hi(u)));
              }
            }
          } else if constexpr (EPI == EPI_DSWIGLU) {
            // acc = dh; g in slots 0..3 and u in 4..7 are replaced by dg = dh*u*silu'(g) and du = dh*silu(g)
            mbar_wait(epi_full, 0);
#pragma unroll
            for (uint32_t i = 0; i < 32; ++i) {
#pragma unroll
              for (uint32_t h = 0; h < 2; ++h) {
                const uint32_t off = frag_offset(r0 + 8 * h, i, lane);
                const uint32_t ga = smem_u32(slot[i / 8]) + off, ua = smem_u32(slot[4 + i / 8]) + off;
                const uint32_t gp = lds32(ga), up = lds32(ua);
                float dg[2], du[2];
#pragma unroll
                for (uint32_t e = 0; e < 2; ++e) {
                  const float d = bf16_round(acc[4 * i + 2 * h + e]);   // dh as the unfused path stores it
                  const float gv = e ? bf16_hi(gp) : bf16_lo(gp);
                  const float uv = e ? bf16_hi(up) : bf16_lo(up);
                  const float sg = 1.f / (1.f + __expf(-gv));
                  dg[e] = d * uv * (sg * (1.f + gv * (1.f - sg)));
                  du[e] = d * (gv * sg);
                }
                sts32(ga, pack_bf16x2(dg[0], dg[1]));
                sts32(ua, pack_bf16x2(du[0], du[1]));
              }
            }
          } else if constexpr (EPI == EPI_ROPE) {
            // projection output rounded to bf16 first (the reference ropes the bf16 q/k); column c < 64 of a head
            // (group i) pairs with c + 64 (group i + 8).  Both heads of the tile share the cos / sin of a row.
            const bool rope0 = col0 < ea.rope_cols, rope1 = col0 + 128 < ea.rope_cols;
            int p[2];
#pragma unroll
            for (uint32_t h = 0; h < 2; ++h) p[h] = m0 + r0 + 8 * h < M ? ea.pos[m0 + r0 + 8 * h] : 0;
#pragma unroll
            for (uint32_t i = 0; i < 8; ++i) {
#pragma unroll
              for (uint32_t h = 0; h < 2; ++h) {
                const uint32_t c = 8 * i + 2 * (lane & 3), off = frag_offset(r0 + 8 * h, i, lane);
                uint32_t c1 = 0, s1 = 0, c2 = 0, s2 = 0;
                if (rope0) {
                  const int64_t b = static_cast<int64_t>(p[h]) * 128 + c;
                  c1 = *reinterpret_cast<const uint32_t*>(ea.cos_t + b);
                  s1 = *reinterpret_cast<const uint32_t*>(ea.sin_t + b);
                  c2 = *reinterpret_cast<const uint32_t*>(ea.cos_t + b + 64);
                  s2 = *reinterpret_cast<const uint32_t*>(ea.sin_t + b + 64);
                }
#pragma unroll
                for (uint32_t hd = 0; hd < 2; ++hd) {
                  const uint32_t ia = 16 * hd + i, ib = ia + 8;
                  const uint32_t xa = pack_bf16x2(acc[4 * ia + 2 * h], acc[4 * ia + 2 * h + 1]);
                  const uint32_t xb = pack_bf16x2(acc[4 * ib + 2 * h], acc[4 * ib + 2 * h + 1]);
                  uint32_t o1 = xa, o2 = xb;
                  if (hd ? rope1 : rope0) {
                    const float y1l = bf16_round(bf16_lo(xa) * bf16_lo(c1)) + bf16_round(-bf16_lo(xb) * bf16_lo(s1));
                    const float y1h = bf16_round(bf16_hi(xa) * bf16_hi(c1)) + bf16_round(-bf16_hi(xb) * bf16_hi(s1));
                    const float y2l = bf16_round(bf16_lo(xb) * bf16_lo(c2)) + bf16_round(bf16_lo(xa) * bf16_lo(s2));
                    const float y2h = bf16_round(bf16_hi(xb) * bf16_hi(c2)) + bf16_round(bf16_hi(xa) * bf16_hi(s2));
                    o1 = pack_bf16x2(y1l, y1h);
                    o2 = pack_bf16x2(y2l, y2h);
                  }
                  sts32(smem_u32(slot[2 * hd]) + off, o1);
                  sts32(smem_u32(slot[2 * hd + 1]) + off, o2);
                }
              }
            }
          } else {
            // ATTND: bf16 dO in slots 4..7 (O is prefetched into 0..3)
#pragma unroll
            for (uint32_t i = 0; i < 32; ++i) {
#pragma unroll
              for (uint32_t h = 0; h < 2; ++h)
                sts32(smem_u32(slot[4 + i / 8]) + frag_offset(r0 + 8 * h, i, lane),
                      pack_bf16x2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]));
            }
          }
          fence_proxy_async_smem();                       // generic-proxy writes -> TMA store reads
          named_bar_sync(1, GEMM_CONSUMERS);
          if (threadIdx.x == 0) {
            const uint32_t ncols = EPI == EPI_SWIGLU || EPI == EPI_DSWIGLU ? ea.F : N;
#pragma unroll
            for (uint32_t b = 0; b < OUT_BOXES; ++b) {
              // SWIGLU: boxes 0, 1 g, 2, 3 u, 4, 5 h;  DSWIGLU: 0..3 dg, 4..7 du;  ROPE / ATTND: 0..3
              const uint32_t map = EPI == EPI_SWIGLU ? b / 2 : EPI == EPI_DSWIGLU ? b / 4 : 0;
              const uint32_t col = col0 + 64 * (EPI == EPI_SWIGLU ? b % 2 : b % 4);
              if (EPI == EPI_SWIGLU && map < 2 && (flags & GEMM_NO_GU)) continue;
              if (col < ncols) tma_store_2d(&em.m[map], slot[OUT_SLOT0 + b], col, m0);
            }
            tma_store_commit();
          }
          if constexpr (EPI == EPI_ATTND) {
            // D[h, t] = sum_d dO[t, h, d] * O[t, h, d]: thread = one row of the head of its warpgroup, summed in the
            // order of the row kernel (32-column chunks, then 8-element groups)
            mbar_wait(epi_full, 0);
            const uint32_t hc = col0 + wg * 128;
            if (hc < N && m0 + t < M) {
              float dsum = 0.f;
#pragma unroll
              for (uint32_t c = 0; c < 128; c += 32) {
#pragma unroll
                for (uint32_t j = 0; j < 32; j += 8) {
                  const uint32_t bb = (c + j) / 64, off = sw128_offset(t, ((c + j) % 64) / 8);   // box 2 wg + bb
                  const uint4 o = lds128(smem_u32(wg ? slot[6 + bb] : slot[4 + bb]) + off);
                  const uint4 a = lds128(smem_u32(wg ? slot[2 + bb] : slot[bb]) + off);
                  dsum += bf16_lo(o.x) * bf16_lo(a.x) + bf16_hi(o.x) * bf16_hi(a.x) + bf16_lo(o.y) * bf16_lo(a.y) + bf16_hi(o.y) * bf16_hi(a.y)
                        + bf16_lo(o.z) * bf16_lo(a.z) + bf16_hi(o.z) * bf16_hi(a.z) + bf16_lo(o.w) * bf16_lo(a.w) + bf16_hi(o.w) * bf16_hi(a.w);
                }
              }
              ea.dvec[static_cast<int64_t>(hc >> 7) * M + m0 + t] = dsum;
            }
          }
          if (threadIdx.x == 0) tma_store_wait_read<0>();   // the boxes stay in shared memory until the TMA read them
        }
      }
    }
  }
  __syncwarp();
  cluster_sync_all();   // no CTA exits while its peer can still multicast into it or arrive on its barriers
}

template <bool A_MN, bool B_MN, int EPI = EPI_PLAIN>
static int launch_wide(const CUtensorMap& ta, const CUtensorMap& tb, void* C, int64_t ldc, const void* addend,
                       int64_t ld_add, uint32_t M, uint32_t N, uint32_t K, uint32_t flags, cudaStream_t stream,
                       const EpiMaps& em = EpiMaps{}, EpiAux ea = EpiAux{}) {
  auto kern = gemm_bf16_wide<A_MN, B_MN, EPI>;
  cudaLaunchConfig_t cfg = {};
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = WideSmem::DYN_BYTES;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = WIDE_CLUSTER;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  static bool attr_set = false;
  if (!attr_set) {
    NV_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, WideSmem::DYN_BYTES));
    attr_set = true;
  }
  const uint32_t pairs = ceil_div_u32(ceil_div_u32(M, GEMM_BLOCK_M), WIDE_CLUSTER) *
                         ceil_div_u32(N, EPI == EPI_SWIGLU ? 128u : WIDE_N);
  cfg.gridDim = dim3(WIDE_CLUSTER * pairs);
  NV_CUDA(cudaLaunchKernelEx(&cfg, kern, ta, tb, em, C, ldc, reinterpret_cast<const __nv_bfloat16*>(addend), ld_add, M,
                             N, K, flags, ea));
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

  if (block_n == 256 && (flags & GEMM_OUT_F32)) block_n = 128;   // the 256-wide plain epilogue stages bf16 only

  CUtensorMap ta, tb;
  int rc = gemm_tmaps(&ta, &tb, A, lda, a_mn, B, ldb, b_mn, M, N, K, (uint32_t)block_n, (uint64_t)N);
  if (rc) return rc;

  if (block_n == 256) {
    if (!a_mn && !b_mn) return launch_wide<false, false>(ta, tb, C, ldc, addend, ld_add, M, N, K, flags, stream);
    if (!a_mn && b_mn) return launch_wide<false, true>(ta, tb, C, ldc, addend, ld_add, M, N, K, flags, stream);
    if (a_mn && b_mn) return launch_wide<true, true>(ta, tb, C, ldc, addend, ld_add, M, N, K, flags, stream);
    return launch_wide<true, false>(ta, tb, C, ldc, addend, ld_add, M, N, K, flags, stream);
  }

#define NV_GEMM_CASE(BN, ST)                                                                                       \
  do {                                                                                                             \
    if (!a_mn && !b_mn) return launch_gemm<BN, ST, false, false>(ta, tb, C, ldc, addend, ld_add, M, N, K, flags, stream); \
    if (!a_mn && b_mn) return launch_gemm<BN, ST, false, true>(ta, tb, C, ldc, addend, ld_add, M, N, K, flags, stream);   \
    if (a_mn && b_mn) return launch_gemm<BN, ST, true, true>(ta, tb, C, ldc, addend, ld_add, M, N, K, flags, stream);     \
    return launch_gemm<BN, ST, true, false>(ta, tb, C, ldc, addend, ld_add, M, N, K, flags, stream);                      \
  } while (0)

  if (block_n == 32) {
    // decode / pruned-row GEMMs (M <= 128): HBM-bound weight streaming; 10 stages keep ~40 KB of weights in flight per SM
    if (!a_mn) return launch_gemm<32, 10, false, false>(ta, tb, C, ldc, addend, ld_add, M, N, K, flags, stream);
    return launch_gemm<32, 10, true, false>(ta, tb, C, ldc, addend, ld_add, M, N, K, flags, stream);
  }
  NV_GEMM_CASE(128, 6);
#undef NV_GEMM_CASE
}

// C[M,N] = A[M,K] · W'[N,K]^T (+ addend) with W' = Wq * 2^exps given in the fp8 weight format (e4m3 rows, one int8
// exponent per row; ldw in bytes): bit for bit nv_gemm_bf16(A, W', block_n) for every M, N, K, reading half the weight bytes.
extern "C" int nv_gemm_fp8w_bf16(const void* A, int64_t lda, const void* Wq, int64_t ldw, const void* exps, void* C, int64_t ldc,
                                 const void* addend, int64_t ld_add, int M, int N, int K, int block_n, void* stream_) {
  using namespace nv;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  NV_REQUIRE(M > 0 && N > 0 && K > 0, "nv_gemm_fp8w_bf16: empty problem M=%d N=%d K=%d", M, N, K);
  NV_REQUIRE(A && Wq && exps && C, "nv_gemm_fp8w_bf16: null operand");
  NV_REQUIRE((lda & 7) == 0 && (ldw & 15) == 0,
             "nv_gemm_fp8w_bf16: lda must be a multiple of 8 and ldw (bytes) of 16 (got %lld, %lld)", (long long)lda, (long long)ldw);
  // auto: nv_gemm_bf16's choice for K-major operands below M = 512 (the 256-wide tile is not built for fp8 weights)
  if (block_n == 0) block_n = (M <= 128 && N <= 4096) ? 32 : 128;
  NV_REQUIRE(block_n == 32 || block_n == 128, "nv_gemm_fp8w_bf16: block_n must be 0, 32 or 128 (got %d)", block_n);
  CUtensorMap ta, tb;
  int rc = make_tmap_2d(&ta, A, 2, (uint64_t)K, (uint64_t)M, (uint64_t)lda * 2, 64, GEMM_BLOCK_M);
  if (rc) return rc;
  if ((rc = make_tmap_2d(&tb, Wq, 1, (uint64_t)K, (uint64_t)N, (uint64_t)ldw, 64, (uint32_t)block_n, /*swizzle128=*/false)))
    return rc;
  EpiAux ea{};
  ea.w_exp = reinterpret_cast<const int8_t*>(exps);
  const uint32_t flags = addend ? GEMM_ADD : 0u;
  // stages: the bf16 kernel's 10 at BLOCK_N = 32; 5 of 40 KB (A, e4m3 B, expanded B) fit at 128
  if (block_n == 32)
    return launch_gemm<32, 10, false, false, uint8_t>(ta, tb, C, ldc, addend, ld_add, M, N, K, flags, stream, ea);
  return launch_gemm<128, 5, false, false, uint8_t>(ta, tb, C, ldc, addend, ld_add, M, N, K, flags, stream, ea);
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
  EpiMaps em{};
  if (keep_gu) {
    if ((rc = make_tmap_2d(&em.m[0], gu, 2, (uint64_t)F, (uint64_t)M, (uint64_t)ldgu * 2, 64, GEMM_BLOCK_M))) return rc;
    if ((rc = make_tmap_2d(&em.m[1], static_cast<__nv_bfloat16*>(gu) + F, 2, (uint64_t)F, (uint64_t)M, (uint64_t)ldgu * 2, 64,
                           GEMM_BLOCK_M)))
      return rc;
  }
  if ((rc = make_tmap_2d(&em.m[2], h, 2, (uint64_t)F, (uint64_t)M, (uint64_t)ldh * 2, 64, GEMM_BLOCK_M))) return rc;
  EpiAux ea{};
  ea.F = (uint32_t)F;
  return launch_wide<false, false, EPI_SWIGLU>(ta, tb, gu, ldgu, nullptr, 0, M, F, K, keep_gu ? 0u : GEMM_NO_GU,
                                               reinterpret_cast<cudaStream_t>(stream), em, ea);
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
  EpiMaps em{};
  const __nv_bfloat16* halves[4] = {static_cast<const __nv_bfloat16*>(dgu), static_cast<const __nv_bfloat16*>(dgu) + F,
                                    static_cast<const __nv_bfloat16*>(gu), static_cast<const __nv_bfloat16*>(gu) + F};
  for (int i = 0; i < 4; ++i)
    if ((rc = make_tmap_2d(&em.m[i], halves[i], 2, (uint64_t)F, (uint64_t)M, (uint64_t)(i < 2 ? lddgu : ldgu) * 2, 64,
                           GEMM_BLOCK_M)))
      return rc;
  EpiAux ea{};
  ea.F = (uint32_t)F;
  return launch_wide<false, true, EPI_DSWIGLU>(ta, tb, dgu, lddgu, nullptr, 0, M, F, D, 0u,
                                               reinterpret_cast<cudaStream_t>(stream), em, ea);
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
  EpiMaps em{};
  if ((rc = make_tmap_2d(&em.m[0], dout, 2, (uint64_t)D, (uint64_t)M, (uint64_t)lddo * 2, 64, GEMM_BLOCK_M))) return rc;
  if ((rc = make_tmap_2d(&em.m[2], o, 2, (uint64_t)D, (uint64_t)M, (uint64_t)ldo * 2, 64, GEMM_BLOCK_M))) return rc;
  EpiAux ea{};
  ea.dvec = dvec;
  return launch_wide<false, true, EPI_ATTND>(ta, tb, dout, lddo, nullptr, 0, M, D, Dout, 0u,
                                             reinterpret_cast<cudaStream_t>(stream), em, ea);
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
  EpiMaps em{};
  if ((rc = make_tmap_2d(&em.m[0], out, 2, (uint64_t)N, (uint64_t)M, (uint64_t)ldo * 2, 64, GEMM_BLOCK_M))) return rc;
  EpiAux ea{};
  ea.pos = pos; ea.cos_t = reinterpret_cast<const __nv_bfloat16*>(cos_t); ea.sin_t = reinterpret_cast<const __nv_bfloat16*>(sin_t);
  ea.rope_cols = (uint32_t)rope_cols;
  return launch_wide<false, false, EPI_ROPE>(ta, tb, out, ldo, nullptr, 0, M, N, K, 0u,
                                             reinterpret_cast<cudaStream_t>(stream), em, ea);
}

}  // extern "C"
