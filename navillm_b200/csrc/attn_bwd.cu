// navillm_b200 — causal self-attention backward on Hopper wgmma (packed variable-length rows), pipelined.
//
// Hand-written twin of attn_fwd.cu; replaces the autograd backward of HF LLaMA's eager attention
// (reference: loss.backward() call sites tasks/agents/mp3d_agent.py:750-757, tasks/agents/llava.py:38-40
// through models/modified_lm.py:112-116; SURVEY.md §2b K14).
//
// With P = exp(S*scale - LSE), D_i = sum_d dO_id O_id, dS = P o (dP - D) * scale:
//     dV = P^T dO      dK = dS^T Q      dQ = dS K
// Two deterministic passes (no atomics).  Both walk the partner dimension in 64-wide sub-blocks streamed by TMA
// through a 4-stage ring; two warpgroups own 64 rows each of the CTA's 128-row block, keep
// their accumulators in registers and feed P / dS back into the tensor cores from registers (the wgmma
// A-from-registers form: a score accumulator is laid out like an A fragment).
//
//   dq pass   CTA = (128-query block, head).  Q,dO resident; K_n,V_n [64 keys x 128] streamed.
//             S = Q K_n^T, dP = dO V_n^T  [64 q x 64 keys per warpgroup] -> dS (bf16, registers) -> dQ += dS K_n.
//   dkdv pass CTA = (128-key block, head).  K,V resident; Q_n,dO_n [64 queries x 128] streamed.
//             TRANSPOSED scores so that accumulator rows are keys: S^T = K Q_n^T, dP^T = V dO_n^T [64 keys x 64 q]
//             -> P^T, dS^T (bf16, registers) -> dV += P^T dO_n, dK += dS^T Q_n.
// Threads: warps 0..7 (warpgroups 0, 1); thread 0 also issues the TMA loads (a producer warp as a ninth warp would put
// three warps on one SM sub-partition and cap the dk/dv pass below the registers its two accumulators need).  No row
// reductions are needed in the backward: LSE and D are precomputed.  The inverse rotary embedding of dQ / dK is applied in the epilogue (optional).
#include "nv_common.cuh"
#include "nv_host.h"

namespace nv {

constexpr uint32_t AB_THREADS = 256;
constexpr uint32_t AB_T128 = 128 * 128 * 2;  // [128 rows x 128 hd] bf16 = two 16 KB swizzle atoms (hd halves)
constexpr uint32_t AB_A128 = 128 * 128;      // one atom of a 128-row tile
constexpr uint32_t AB_T64 = 64 * 128 * 2;    // [64 rows x 128 hd] bf16 = two 8 KB atoms
constexpr uint32_t AB_A64 = 64 * 128;        // one atom of a 64-row tile
constexpr uint32_t AB_NST = 4;               // streamed sub-block stages
constexpr float LOG2E = 1.4426950408889634f;

__device__ __forceinline__ bool locate_block_bwd(const int* __restrict__ cu, int B, uint32_t blk, int& seq_start,
                                                 int& seq_len, uint32_t& idx) {
  for (int b = 0; b < B; ++b) {
    const int s = cu[b], len = cu[b + 1] - s;
    const uint32_t nb = (len + 127) / 128;
    if (blk < nb) { seq_start = s; seq_len = len; idx = blk; return true; }
    blk -= nb;
  }
  return false;
}

// KV form: the 128-row blocks of sequence b are counted over blk_len[b] rows (kv_len for the key blocks of the dk/dv pass,
// the suffix length for the query blocks of the dq pass); seq is the sequence index.
__device__ __forceinline__ bool locate_block_kv(const int* __restrict__ cu, const int* __restrict__ blk_len, int B,
                                                uint32_t blk, int& seq_start, int& seq_len, uint32_t& idx, int& seq) {
  for (int b = 0; b < B; ++b) {
    const int s = cu[b], len = cu[b + 1] - s;
    const uint32_t n = ((uint32_t)(blk_len != nullptr ? blk_len[b] : len) + 127) / 128;
    if (blk < n) { seq_start = s; seq_len = len; idx = blk; seq = b; return true; }
    blk -= n;
  }
  return false;
}

// D[h, t] = sum_d dO[t, h*128+d] * O[t, h*128+d]   (one warp per (t, h))
__global__ void attn_bwd_prep_kernel(const __nv_bfloat16* __restrict__ O, int64_t ldo,
                                     const __nv_bfloat16* __restrict__ dO, int64_t lddo, float* __restrict__ D, int T,
                                     int H) {
  const int64_t gw = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gw >= (int64_t)T * H) return;
  const int h = gw % H;
  const int64_t t = gw / H;
  const uint2 a = *reinterpret_cast<const uint2*>(O + t * ldo + h * 128 + lane * 4);
  const uint2 b = *reinterpret_cast<const uint2*>(dO + t * lddo + h * 128 + lane * 4);
  float s = bf16_lo(a.x) * bf16_lo(b.x) + bf16_hi(a.x) * bf16_hi(b.x) + bf16_lo(a.y) * bf16_lo(b.y) +
            bf16_hi(a.y) * bf16_hi(b.y);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) D[(int64_t)h * T + t] = s;
}

// Load a [rows x 128 hd] tile as 64-row x 64-col boxes into the two-atom layout (atom = hd half).
template <uint32_t ROWS>
__device__ __forceinline__ void load_tile(uint8_t* dst, const CUtensorMap* m, uint64_t* bar, int32_t col, int32_t row) {
  constexpr uint32_t ATOM = ROWS * 128;
#pragma unroll
  for (uint32_t a = 0; a < 2; ++a)
#pragma unroll
    for (uint32_t r = 0; r < ROWS / 64; ++r)
      tma_load_2d(dst + a * ATOM + r * (64 * 128), m, bar, col + a * 64, row + r * 64);
}

// Epilogue shared by both passes, in two phases so that HBM sees full 256-byte rows (a row-per-thread store would touch
// many rows per instruction, with per-row cos/sin loads for the fused inverse RoPE on top):
//   stage_acc_tile   the warpgroup's 64 x 128 fp32 accumulator, rounded to bf16, into a padded row-major smem tile
//                    (272-byte rows);
//   flush_acc_tile   warp = row: lane l owns columns 4l..4l+3, its rotate-half partner sits in lane l^16; optional
//                    rotation by -theta[pos] with the rounding points of rope_kernel(sign = -1); 8-byte coalesced stores.
// The 8 compute warps synchronise on named barrier 1 before staging (every operand stage is then free) and between
// the phases.
constexpr uint32_t AB_STAGE_LD = 272;                        // bytes per staged row (256 + 16 padding)
constexpr uint32_t AB_STAGE_BYTES = 128 * AB_STAGE_LD;       // 34 816 B per accumulator

__device__ __forceinline__ void compute_warps_sync() { named_bar_sync(1, 256); }

// wg: warpgroup (rows 64 wg ..), acc: its accumulator fragment (rows r, r + 8; columns 8 i + 2 (lane % 4) + {0, 1})
__device__ __forceinline__ void stage_acc_tile(const float (&acc)[64], uint32_t wg, uint8_t* stage) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t r = wg * 64 + ((threadIdx.x & 127) >> 5) * 16 + (lane >> 2);
#pragma unroll
  for (uint32_t i = 0; i < 16; ++i) {
    const uint32_t c = 8 * i + 2 * (lane & 3);
    *reinterpret_cast<uint32_t*>(stage + r * AB_STAGE_LD + c * 2) = pack_bf16x2(acc[4 * i], acc[4 * i + 1]);
    *reinterpret_cast<uint32_t*>(stage + (r + 8) * AB_STAGE_LD + c * 2) = pack_bf16x2(acc[4 * i + 2], acc[4 * i + 3]);
  }
}

// cw: compute-warp index 0..7 (rows cw, cw + 8, ...); rows_valid: real rows of the tile; dst: row 0 of the tile at the
// head's column offset; pos: rotary positions of the tile's rows (null = no rotation).
__device__ __forceinline__ void flush_acc_tile(const uint8_t* stage, uint32_t cw, uint32_t lane, uint32_t rows_valid,
                                               __nv_bfloat16* dst, int64_t ld, const int* __restrict__ pos,
                                               const __nv_bfloat16* __restrict__ cos_t,
                                               const __nv_bfloat16* __restrict__ sin_t) {
  const float sgn = lane < 16 ? 1.f : -1.f;
  for (uint32_t r = cw; r < rows_valid; r += 8) {
    uint2 x = *reinterpret_cast<const uint2*>(stage + r * AB_STAGE_LD + lane * 8);
    if (pos != nullptr) {
      const uint32_t px = __shfl_xor_sync(0xffffffffu, x.x, 16), py = __shfl_xor_sync(0xffffffffu, x.y, 16);
      const int p = pos[r];
      const uint2 c = *reinterpret_cast<const uint2*>(cos_t + (int64_t)p * 128 + lane * 4);
      const uint2 sn = *reinterpret_cast<const uint2*>(sin_t + (int64_t)p * 128 + lane * 4);
      // y[d] = bf16(x[d] cos) + bf16(x[d+64] sin),  y[d+64] = bf16(x[d+64] cos) + bf16(-x[d] sin)
      const float y0 = bf16_round(bf16_lo(x.x) * bf16_lo(c.x)) + bf16_round(sgn * bf16_lo(px) * bf16_lo(sn.x));
      const float y1 = bf16_round(bf16_hi(x.x) * bf16_hi(c.x)) + bf16_round(sgn * bf16_hi(px) * bf16_hi(sn.x));
      const float y2 = bf16_round(bf16_lo(x.y) * bf16_lo(c.y)) + bf16_round(sgn * bf16_lo(py) * bf16_lo(sn.y));
      const float y3 = bf16_round(bf16_hi(x.y) * bf16_hi(c.y)) + bf16_round(sgn * bf16_hi(py) * bf16_hi(sn.y));
      x.x = pack_bf16x2(y0, y1);
      x.y = pack_bf16x2(y2, y3);
    }
    *reinterpret_cast<uint2*>(dst + (int64_t)r * ld + lane * 4) = x;
  }
}

// P / dS fragment for wgmma A operand chunk kk (16 partner columns) from fp32 pairs of a 64-column accumulator
__device__ __forceinline__ void a_frag(const float (&x)[32], uint32_t kk, uint32_t (&a)[4]) {
  a[0] = pack_bf16x2(x[8 * kk], x[8 * kk + 1]);
  a[1] = pack_bf16x2(x[8 * kk + 2], x[8 * kk + 3]);
  a[2] = pack_bf16x2(x[8 * kk + 4], x[8 * kk + 5]);
  a[3] = pack_bf16x2(x[8 * kk + 6], x[8 * kk + 7]);
}

// S (+)= A_rows · B_n^T over hd = 128: A = 64 resident rows (atoms AB_A128 apart, at `a_off` inside them), B = a streamed
// [64 x 128] tile (atoms AB_A64 apart); both K-major over hd.
__device__ __forceinline__ void scores_64x64(float (&acc)[32], uint32_t a_base, uint32_t b_base) {
  const uint64_t ad = gmma_desc_sw128(a_base, 0, 1024), bd = gmma_desc_sw128(b_base, 0, 1024);
#pragma unroll
  for (uint32_t ks = 0; ks < 8; ++ks)
    wgmma_ss_bf16<64, 0, 0>(acc, ad + (ks >> 2) * (AB_A128 >> 4) + (ks & 3) * 2, bd + (ks >> 2) * (AB_A64 >> 4) + (ks & 3) * 2,
                            ks ? 1u : 0u);
}

struct BwdSmem {
  static constexpr uint32_t RES_OFF = 0;                          // two resident [128 x 128] tiles
  static constexpr uint32_t ST_OFF = 2 * AB_T128;                 // AB_NST x two [64 x 128] tiles
  static constexpr uint32_t BAR_OFF = ST_OFF + AB_NST * 2 * AB_T64;
  // res_full, st_full[NST], st_empty[NST]
  static constexpr uint32_t NUM_BARS = 1 + 2 * AB_NST;
  static constexpr uint32_t DYN_BYTES = BAR_OFF + NUM_BARS * 8 + 1024;
};
static_assert(AB_STAGE_BYTES <= 2 * AB_T128, "accumulator staging reuses the resident tiles");
static_assert(BwdSmem::DYN_BYTES <= 232448, "attention backward shared memory");

// TMA issue of both passes, by thread 0: the two resident tiles and the first AB_NST sub-blocks up front ...
__device__ __forceinline__ void bwd_load_prologue(uint8_t* smem, uint64_t* res_full, uint64_t* st_full, const CUtensorMap* r0,
                                                  const CUtensorMap* r1, const CUtensorMap* s0, const CUtensorMap* s1,
                                                  int32_t col, int32_t res_row, int32_t st_row0, uint32_t n_it) {
  using L = BwdSmem;
  mbar_arrive_expect_tx(res_full, 2 * AB_T128);
  load_tile<128>(smem + L::RES_OFF, r0, res_full, col, res_row);
  load_tile<128>(smem + L::RES_OFF + AB_T128, r1, res_full, col, res_row);
  for (uint32_t n = 0; n < min(n_it, AB_NST); ++n) {
    uint8_t* dst = smem + L::ST_OFF + n * 2 * AB_T64;
    mbar_arrive_expect_tx(&st_full[n], 2 * AB_T64);
    load_tile<64>(dst, s0, &st_full[n], col, st_row0 + n * 64);
    load_tile<64>(dst + AB_T64, s1, &st_full[n], col, st_row0 + n * 64);
  }
}
// ... then sub-block n + AB_NST into stage n % AB_NST once both warpgroups have released sub-block n.
__device__ __forceinline__ void bwd_load_refill(uint8_t* smem, uint64_t* st_full, uint64_t* st_empty, const CUtensorMap* s0,
                                                const CUtensorMap* s1, int32_t col, int32_t st_row0, uint32_t n, uint32_t n_it) {
  using L = BwdSmem;
  if (n + AB_NST >= n_it) return;
  const uint32_t st = n % AB_NST;
  mbar_wait(&st_empty[st], (n / AB_NST) & 1);
  uint8_t* dst = smem + L::ST_OFF + st * 2 * AB_T64;
  const int32_t row = st_row0 + (n + AB_NST) * 64;
  mbar_arrive_expect_tx(&st_full[st], 2 * AB_T64);
  load_tile<64>(dst, s0, &st_full[st], col, row);
  load_tile<64>(dst + AB_T64, s1, &st_full[st], col, row);
}

// ======================================================================================================
// dq pass
// ======================================================================================================
// KV = true (nv_attn_bwd_kv): the keys / values of sequence b are rows kv_start[b] .. +kv_len[b] of a cache (tmap_k /
// tmap_v), the queries its last seq_len positions: query i sees keys <= dk + i, dk = kv_len[b] - seq_len (as attn_fwd_kv).
template <bool KV>
__global__ void __launch_bounds__(AB_THREADS, 1)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_do,
                   const __grid_constant__ CUtensorMap tmap_k, const __grid_constant__ CUtensorMap tmap_v,
                   const float* __restrict__ lse, const float* __restrict__ Dvec, __nv_bfloat16* __restrict__ dq,
                   int64_t lddq, const int* __restrict__ cu_seqlens, int B, int T, float scale,
                   const int* __restrict__ rope_pos, const __nv_bfloat16* __restrict__ cos_t,
                   const __nv_bfloat16* __restrict__ sin_t, const int* __restrict__ kv_start, const int* __restrict__ kv_len) {
  using L = BwdSmem;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* res_full = bars;
  uint64_t* st_full = bars + 1;
  uint64_t* st_empty = bars + 1 + AB_NST;

  const uint32_t warp = warp_id_uniform(), lane = threadIdx.x & 31;
  const uint32_t head = blockIdx.y;
  int seq_start = 0, seq_len = 0;
  uint32_t own = 0, dk = 0;
  int kv0 = 0;
  uint32_t n_sub;
  if constexpr (KV) {
    int seq = 0;
    if (!locate_block_kv(cu_seqlens, nullptr, B, gridDim.x - 1 - blockIdx.x, seq_start, seq_len, own, seq)) return;
    dk = (uint32_t)(kv_len[seq] - seq_len);
    kv0 = kv_start[seq];
    // 64-key sub-blocks 0 .. n_sub-1 cover keys [0, dk + min((own+1)*128, len))
    n_sub = (dk + min((own + 1) * 128, (uint32_t)seq_len) + 63) / 64;
  } else {
    if (!locate_block_bwd(cu_seqlens, B, gridDim.x - 1 - blockIdx.x, seq_start, seq_len, own)) return;  // heavy first
    kv0 = seq_start;
    // 64-key sub-blocks 0 .. n_sub-1 cover keys [0, min((own+1)*128, len))
    n_sub = min(2 * own + 2, (uint32_t)(seq_len + 63) / 64);
  }

  if (threadIdx.x == 0) {
    mbar_init(res_full, 1);
    for (uint32_t i = 0; i < AB_NST; ++i) { mbar_init(&st_full[i], 1); mbar_init(&st_empty[i], 2); }
    fence_mbar_init();
  }
  __syncthreads();

  if (threadIdx.x == 0)
    bwd_load_prologue(smem, res_full, st_full, &tmap_q, &tmap_do, &tmap_k, &tmap_v, head * 128, seq_start + own * 128,
                      kv0, n_sub);

  const uint32_t wg = warp >> 2;
  const uint32_t ra = wg * 64 + (warp & 3) * 16 + (lane >> 2);    // rows ra, ra + 8 of the block
  const uint32_t qa = own * 128 + ra, qb = qa + 8;
  const uint32_t cq = 2 * (lane & 3);
  const float sl2 = scale * LOG2E;
  // an invalid row gets LSE = +inf -> p = exp2(-inf) = 0 without a branch
  const float la = qa < (uint32_t)seq_len ? lse[(int64_t)head * T + seq_start + qa] * LOG2E : INFINITY;
  const float lb = qb < (uint32_t)seq_len ? lse[(int64_t)head * T + seq_start + qb] * LOG2E : INFINITY;
  const float da = qa < (uint32_t)seq_len ? Dvec[(int64_t)head * T + seq_start + qa] : 0.f;
  const float db = qb < (uint32_t)seq_len ? Dvec[(int64_t)head * T + seq_start + qb] : 0.f;
  const uint32_t sQ = smem_u32(smem + L::RES_OFF) + wg * 8192, sdO = sQ + AB_T128;
  float dqacc[64];
#pragma unroll
  for (uint32_t i = 0; i < 64; ++i) dqacc[i] = 0.f;
  mbar_wait(res_full, 0);
  for (uint32_t n = 0; n < n_sub; ++n) {
    const uint32_t st = n % AB_NST;
    const uint32_t sKn = smem_u32(smem + L::ST_OFF + st * 2 * AB_T64), sVn = sKn + AB_T64;
    mbar_wait(&st_full[st], (n / AB_NST) & 1);
    float sacc[32], dpacc[32];
    wgmma_fence();
    scores_64x64(sacc, sQ, sKn);
    scores_64x64(dpacc, sdO, sVn);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(sacc);
    reg_fence(dpacc);
    // sub-blocks that touch the diagonal 128x128 block
    const bool diag = KV ? (n * 64 + 63 > dk + own * 128) : (n >= 2 * own);
#pragma unroll
    for (uint32_t i = 0; i < 8; ++i) {
#pragma unroll
      for (uint32_t e = 0; e < 4; ++e) {
        const uint32_t key = n * 64 + 8 * i + cq + (e & 1);
        const uint32_t q = (e & 2) ? qb : qa;
        float p = exp2f(fmaf(sacc[4 * i + e], sl2, -((e & 2) ? lb : la)));
        if (diag && key > dk + q) p = 0.f;
        // dS = P o (dP - D) * scale
        sacc[4 * i + e] = p * ((dpacc[4 * i + e] - ((e & 2) ? db : da)) * scale);
      }
    }
    // dQ += dS K_n : contraction over the 64 keys; B = K_n rows = keys (K dim), hd contiguous (MN-major)
    const uint64_t kd = gmma_desc_sw128(sKn, AB_A64, 1024);
    wgmma_fence();
#pragma unroll
    for (uint32_t kk = 0; kk < 4; ++kk) {
      uint32_t a[4];
      a_frag(sacc, kk, a);
      wgmma_rs_bf16<128, 1>(dqacc, a, kd + kk * ((16 * 128) >> 4), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(dqacc);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&st_empty[st]);
    if (threadIdx.x == 0) bwd_load_refill(smem, st_full, st_empty, &tmap_k, &tmap_v, head * 128, kv0, n, n_sub);
  }
  compute_warps_sync();                                     // every operand stage is free
  uint8_t* stage = smem + L::RES_OFF;
  stage_acc_tile(dqacc, wg, stage);
  compute_warps_sync();
  const uint32_t rows_valid = min(128u, (uint32_t)seq_len - own * 128);
  const int64_t tok0 = (int64_t)seq_start + own * 128;
  flush_acc_tile(stage, warp, lane, rows_valid, dq + tok0 * lddq + head * 128, lddq,
                 rope_pos != nullptr ? rope_pos + tok0 : nullptr, cos_t, sin_t);
}

// ======================================================================================================
// dk/dv pass (transposed scores: accumulator rows = keys)
// ======================================================================================================
// KV = true (nv_attn_bwd_kv): the CTA owns a 128-key block of [0, kv_len[b]) of the cache (tmap_k / tmap_v rows kv_start[b]
// + ...) and streams the suffix queries that see it.  Epilogue by key row j: j < dk (cached rows) -> acc_k / acc_v
// [kv_start[b] + j] += (dK, dV) in fp32 (read-modify-write: each (row, head) slice has one owning CTA, no atomics); j >= dk
// (the suffix's own rows) -> dK + acc_k and dV + acc_v, rounded once, into packed row seq_start + j - dk of dk / dv.
template <bool KV>
__global__ void __launch_bounds__(AB_THREADS, 1)
attn_bwd_dkv_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                    const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_do,
                    const float* __restrict__ lse, const float* __restrict__ Dvec, __nv_bfloat16* __restrict__ dk,
                    int64_t lddk, __nv_bfloat16* __restrict__ dv, int64_t lddv, const int* __restrict__ cu_seqlens,
                    int B, int T, float scale, const int* __restrict__ rope_pos,
                    const __nv_bfloat16* __restrict__ cos_t, const __nv_bfloat16* __restrict__ sin_t,
                    const int* __restrict__ kv_start, const int* __restrict__ kv_len, float* __restrict__ acc_k,
                    float* __restrict__ acc_v, int64_t ldacc) {
  using L = BwdSmem;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* res_full = bars;
  uint64_t* st_full = bars + 1;
  uint64_t* st_empty = bars + 1 + AB_NST;

  const uint32_t warp = warp_id_uniform(), lane = threadIdx.x & 31;
  const uint32_t head = blockIdx.y;
  int seq_start = 0, seq_len = 0;
  uint32_t own = 0, first, cdk = 0, klen = 0;
  int kv0 = 0;
  if constexpr (KV) {
    int seq = 0;
    if (!locate_block_kv(cu_seqlens, kv_len, B, blockIdx.x, seq_start, seq_len, own, seq)) return;
    klen = (uint32_t)kv_len[seq];
    cdk = klen - (uint32_t)seq_len;
    kv0 = kv_start[seq];
    // the first query that sees key own*128 is own*128 - cdk (clamped at 0)
    first = own * 128 > cdk ? (own * 128 - cdk) / 64 : 0u;
  } else {
    if (!locate_block_bwd(cu_seqlens, B, blockIdx.x, seq_start, seq_len, own)) return;   // early key blocks are the heavy ones
    kv0 = seq_start;
    // 64-query sub-blocks first .. n_qsub-1 can see keys of this block (causal): q >= own*128
    first = 2 * own;
  }
  const uint32_t n_qsub = (uint32_t)(seq_len + 63) / 64;
  const uint32_t n_it = n_qsub - first;

  if (threadIdx.x == 0) {
    mbar_init(res_full, 1);
    for (uint32_t i = 0; i < AB_NST; ++i) { mbar_init(&st_full[i], 1); mbar_init(&st_empty[i], 2); }
    fence_mbar_init();
  }
  __syncthreads();

  if (threadIdx.x == 0)
    bwd_load_prologue(smem, res_full, st_full, &tmap_k, &tmap_v, &tmap_q, &tmap_do, head * 128, kv0 + own * 128,
                      seq_start + first * 64, n_it);

  const uint32_t wg = warp >> 2;
  const uint32_t ra = wg * 64 + (warp & 3) * 16 + (lane >> 2);    // key rows ra, ra + 8 of the block
  const uint32_t ka = own * 128 + ra, kb = ka + 8;
  // KV: key rows relative to the cached count (query q sees key k iff q >= k - cdk), and the first query sub-block row
  // past which every key of the block is visible
  const int ea = (int)ka - (int)cdk, eb = ea + 8, dlim = (int)(own * 128 + 127) - (int)cdk;
  const uint32_t cq = 2 * (lane & 3);
  const float sl2 = scale * LOG2E;
  const uint32_t sK = smem_u32(smem + L::RES_OFF) + wg * 8192, sV = sK + AB_T128;
  float dvacc[64], dkacc[64];
#pragma unroll
  for (uint32_t i = 0; i < 64; ++i) { dvacc[i] = 0.f; dkacc[i] = 0.f; }
  mbar_wait(res_full, 0);
  for (uint32_t n = 0; n < n_it; ++n) {
    const uint32_t st = n % AB_NST;
    const uint32_t sQn = smem_u32(smem + L::ST_OFF + st * 2 * AB_T64), sdOn = sQn + AB_T64;
    const uint32_t q0 = (first + n) * 64;
    // -LSE * log2e and -D * scale of the thread's 16 query columns (stored negated: -inf -> p = 0 past the sequence);
    // loaded before the wait so that their latency hides under it
    float nl[16], nd[16];
#pragma unroll
    for (uint32_t i = 0; i < 8; ++i)
#pragma unroll
      for (uint32_t e = 0; e < 2; ++e) {
        const uint32_t q = q0 + 8 * i + cq + e;
        const bool ok = q < (uint32_t)seq_len;
        const int64_t idx = (int64_t)head * T + seq_start + q;
        nl[2 * i + e] = ok ? -lse[idx] * LOG2E : -INFINITY;
        nd[2 * i + e] = ok ? -Dvec[idx] * scale : 0.f;
      }
    mbar_wait(&st_full[st], (n / AB_NST) & 1);
    float sacc[32], dpacc[32];
    wgmma_fence();
    scores_64x64(sacc, sK, sQn);
    scores_64x64(dpacc, sV, sdOn);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(sacc);
    reg_fence(dpacc);
    // query sub-blocks inside the diagonal 128x128 block
    const bool diag = KV ? ((int)q0 < dlim) : ((first + n) < 2 * own + 2);
#pragma unroll
    for (uint32_t i = 0; i < 8; ++i) {
#pragma unroll
      for (uint32_t e = 0; e < 4; ++e) {
        const uint32_t c = 2 * i + (e & 1);
        const uint32_t q = q0 + 8 * i + cq + (e & 1);
        float p = exp2f(fmaf(sacc[4 * i + e], sl2, nl[c]));
        if constexpr (KV) {
          if (diag && (int)q < ((e & 2) ? eb : ea)) p = 0.f;      // query q sees keys <= cdk + q
        } else {
          if (diag && q < ((e & 2) ? kb : ka)) p = 0.f;     // causal: a query sees keys <= itself
        }
        sacc[4 * i + e] = p;
        dpacc[4 * i + e] = p * fmaf(dpacc[4 * i + e], scale, nd[c]);   // dS^T = P^T o (dP^T - D) * scale
      }
    }
    // dV += P^T dO_n, dK += dS^T Q_n: contraction over the 64 queries; B rows = queries, hd contiguous (MN-major)
    const uint64_t qd = gmma_desc_sw128(sQn, AB_A64, 1024), od = gmma_desc_sw128(sdOn, AB_A64, 1024);
    wgmma_fence();
#pragma unroll
    for (uint32_t kk = 0; kk < 4; ++kk) {
      uint32_t a[4];
      a_frag(sacc, kk, a);
      wgmma_rs_bf16<128, 1>(dvacc, a, od + kk * ((16 * 128) >> 4), 1u);
    }
#pragma unroll
    for (uint32_t kk = 0; kk < 4; ++kk) {
      uint32_t a[4];
      a_frag(dpacc, kk, a);
      wgmma_rs_bf16<128, 1>(dkacc, a, qd + kk * ((16 * 128) >> 4), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(dvacc);
    reg_fence(dkacc);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&st_empty[st]);
    if (threadIdx.x == 0)
      bwd_load_refill(smem, st_full, st_empty, &tmap_q, &tmap_do, head * 128, seq_start + first * 64, n, n_it);
  }
  if constexpr (KV) {
    // the thread's key rows ka (fragment elements 4i, 4i+1) and kb (4i+2, 4i+3), columns 8i + cq, +1
#pragma unroll
    for (uint32_t hf = 0; hf < 2; ++hf) {
      const uint32_t j = own * 128 + ra + 8 * hf;
      if (j >= klen) continue;
      const int64_t off = ((int64_t)kv0 + j) * ldacc + head * 128 + cq;
      float* pk = acc_k + off;
      float* pv = acc_v + off;
      const bool cached_row = j < cdk;
#pragma unroll
      for (uint32_t i = 0; i < 16; ++i) {
        float2 a = *reinterpret_cast<const float2*>(pk + 8 * i);
        float2 c = *reinterpret_cast<const float2*>(pv + 8 * i);
        if (cached_row) {
          a.x += dkacc[4 * i + 2 * hf]; a.y += dkacc[4 * i + 2 * hf + 1];
          c.x += dvacc[4 * i + 2 * hf]; c.y += dvacc[4 * i + 2 * hf + 1];
          *reinterpret_cast<float2*>(pk + 8 * i) = a;
          *reinterpret_cast<float2*>(pv + 8 * i) = c;
        } else {
          dkacc[4 * i + 2 * hf] += a.x; dkacc[4 * i + 2 * hf + 1] += a.y;
          dvacc[4 * i + 2 * hf] += c.x; dvacc[4 * i + 2 * hf + 1] += c.y;
        }
      }
    }
  }
  compute_warps_sync();                                     // every operand stage is free
  uint8_t* stage_v = smem + L::RES_OFF;                     // resident K/V and the Q/dO stages are free now
  uint8_t* stage_k = smem + L::ST_OFF;
  stage_acc_tile(dvacc, wg, stage_v);
  stage_acc_tile(dkacc, wg, stage_k);
  compute_warps_sync();
  if constexpr (KV) {
    // block rows r_first .. rows_valid-1 are suffix rows: packed row seq_start + own*128 + r - cdk
    const uint32_t rows_valid = min(128u, klen - own * 128);
    const uint32_t r_first = cdk > own * 128 ? min(cdk - own * 128, 128u) : 0u;
    if (r_first >= rows_valid) return;
    const int64_t tok0 = (int64_t)seq_start + own * 128 + r_first - cdk;
    flush_acc_tile(stage_v + r_first * AB_STAGE_LD, warp, lane, rows_valid - r_first, dv + tok0 * lddv + head * 128, lddv,
                   nullptr, cos_t, sin_t);
    flush_acc_tile(stage_k + r_first * AB_STAGE_LD, warp, lane, rows_valid - r_first, dk + tok0 * lddk + head * 128, lddk,
                   rope_pos != nullptr ? rope_pos + tok0 : nullptr, cos_t, sin_t);
  } else {
    const uint32_t rows_valid = min(128u, (uint32_t)seq_len - own * 128);
    const int64_t tok0 = (int64_t)seq_start + own * 128;
    flush_acc_tile(stage_v, warp, lane, rows_valid, dv + tok0 * lddv + head * 128, lddv, nullptr, cos_t, sin_t);
    flush_acc_tile(stage_k, warp, lane, rows_valid, dk + tok0 * lddk + head * 128, lddk,
                   rope_pos != nullptr ? rope_pos + tok0 : nullptr, cos_t, sin_t);
  }
}

}  // namespace nv

// Developer hook of the in-kernel phase trace.  The sm_90a kernels carry no trace: returns 0 words.
extern "C" int nv_debug_attn_trace(int kernel, unsigned long long* out, int max_words) {
  (void)kernel; (void)out; (void)max_words;
  return 0;
}

// D = rowsum(dO o O) unless o == nullptr: then dvec already holds D (written by the o_proj dgrad epilogue, nv_gemm_attnd_bf16)
static int attn_bwd_prep(const void* o, int64_t ldo, const void* dout, int64_t lddo, float* dvec, int T, int H,
                         cudaStream_t stream) {
  using namespace nv;
  if (o == nullptr) return NV_OK;
  const int64_t threads = (int64_t)T * H * 32;
  attn_bwd_prep_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(o), ldo, reinterpret_cast<const __nv_bfloat16*>(dout), lddo, dvec, T, H);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

// Inputs: q,k,v (post-RoPE) and o, do as bf16 [T, H*128]-column views; lse [H,T] from the forward.
// dvec: fp32 workspace [H, T] (computed here from o and dout; with o == nullptr it must already hold
// D[h,t] = sum_d dout[t,h,d] o[t,h,d]).  Outputs dq, dk, dv: bf16 views with their own leading dimensions.
// rope_pos/cos_t/sin_t (nullable): when given, dq and dk are rotated back by -theta[pos] in the epilogue, i.e. the
// outputs are the gradients w.r.t. the PRE-RoPE q/k (fuses the backward of the rotary embedding).
extern "C" int nv_attn_bwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                           const void* o, int64_t ldo, const void* dout, int64_t lddo, const float* lse, float* dvec,
                           void* dq, int64_t lddq, void* dk, int64_t lddk, void* dv, int64_t lddv,
                           const int* cu_seqlens, int B, int T, int H, int head_dim, int total_blocks, float scale,
                           const int* rope_pos, const void* cos_t, const void* sin_t, void* stream_) {
  using namespace nv;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  NV_REQUIRE(head_dim == 128, "nv_attn_bwd: head_dim must be 128 (got %d)", head_dim);
  NV_REQUIRE(B > 0 && T > 0 && H > 0 && total_blocks > 0, "nv_attn_bwd: empty problem");
  NV_REQUIRE((lddq & 7) == 0 && (lddk & 7) == 0 && (lddv & 7) == 0 && (ldo & 3) == 0 && (lddo & 3) == 0,
             "nv_attn_bwd: leading-dimension alignment");
  CUtensorMap tq, tk, tv, tdo;
  int rc;
  if ((rc = make_tmap_2d(&tq, q, 2, (uint64_t)H * 128, (uint64_t)T, (uint64_t)ldq * 2, 64, 64))) return rc;
  if ((rc = make_tmap_2d(&tk, k, 2, (uint64_t)H * 128, (uint64_t)T, (uint64_t)ldk * 2, 64, 64))) return rc;
  if ((rc = make_tmap_2d(&tv, v, 2, (uint64_t)H * 128, (uint64_t)T, (uint64_t)ldv * 2, 64, 64))) return rc;
  if ((rc = make_tmap_2d(&tdo, dout, 2, (uint64_t)H * 128, (uint64_t)T, (uint64_t)lddo * 2, 64, 64))) return rc;
  static bool attr_set = false;
  if (!attr_set) {
    NV_CUDA(cudaFuncSetAttribute(attn_bwd_dq_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, BwdSmem::DYN_BYTES));
    NV_CUDA(cudaFuncSetAttribute(attn_bwd_dkv_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, BwdSmem::DYN_BYTES));
    attr_set = true;
  }
  if ((rc = attn_bwd_prep(o, ldo, dout, lddo, dvec, T, H, stream))) return rc;
  const __nv_bfloat16* c = reinterpret_cast<const __nv_bfloat16*>(cos_t);
  const __nv_bfloat16* s = reinterpret_cast<const __nv_bfloat16*>(sin_t);
  dim3 grid(total_blocks, H);
  attn_bwd_dkv_kernel<false><<<grid, AB_THREADS, BwdSmem::DYN_BYTES, stream>>>(
      tq, tk, tv, tdo, lse, dvec, reinterpret_cast<__nv_bfloat16*>(dk), lddk, reinterpret_cast<__nv_bfloat16*>(dv), lddv,
      cu_seqlens, B, T, scale, rope_pos, c, s, nullptr, nullptr, nullptr, nullptr, 0);
  NV_LAUNCH_CHECK();
  attn_bwd_dq_kernel<false><<<grid, AB_THREADS, BwdSmem::DYN_BYTES, stream>>>(
      tq, tdo, tk, tv, lse, dvec, reinterpret_cast<__nv_bfloat16*>(dq), lddq, cu_seqlens, B, T, scale, rope_pos, c, s,
      nullptr, nullptr);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

// Backward of nv_attn_fwd_kv.  q, o, dout, lse, dvec, dq, dk, dv: the Tq packed suffix rows (cu_seqlens), as in nv_attn_bwd;
// kcache / vcache: bf16 [Tkv, H*128] (leading dimension ldkv) holding K/V of sequence b at rows kv_start[b] .. +kv_len[b];
// acc_k / acc_v: fp32 [Tkv, >= H*128] (ldacc) gradient accumulators over the cache rows.  Key row j of sequence b:
//   j <  kv_len[b] - q_len[b] (cached):  acc_{k,v}[kv_start[b] + j] += dK_j, dV_j
//   j >= kv_len[b] - q_len[b] (suffix):  dk / dv[packed row of j] = bf16(dK_j + acc_k[...]) (then the inverse RoPE at
//                                        rope_pos when given), bf16(dV_j + acc_v[...]); the accumulator is only read.
// With kv_len == q_len (nothing cached) every row is a suffix row: the accumulated gradient of the cache rows is added to
// the recomputed prefix's own.  Deterministic: each accumulator (row, head) slice has one owning CTA.
// total_qblocks = sum_b ceil(q_len[b]/128), total_kblocks = sum_b ceil(kv_len[b]/128).
extern "C" int nv_attn_bwd_kv(const void* q, int64_t ldq, const void* kcache, const void* vcache, int64_t ldkv, const void* o,
                              int64_t ldo, const void* dout, int64_t lddo, const float* lse, float* dvec, void* dq, int64_t lddq,
                              void* dk, int64_t lddk, void* dv, int64_t lddv, float* acc_k, float* acc_v, int64_t ldacc,
                              const int* cu_seqlens, const int* kv_start, const int* kv_len, int B, int Tq, int Tkv, int H,
                              int head_dim, int total_qblocks, int total_kblocks, float scale, const int* rope_pos,
                              const void* cos_t, const void* sin_t, void* stream_) {
  using namespace nv;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  NV_REQUIRE(head_dim == 128, "nv_attn_bwd_kv: head_dim must be 128 (got %d)", head_dim);
  NV_REQUIRE(B > 0 && Tq > 0 && Tkv > 0 && H > 0 && total_qblocks > 0 && total_kblocks > 0, "nv_attn_bwd_kv: empty problem");
  NV_REQUIRE(q && kcache && vcache && dout && lse && dvec && dq && dk && dv && acc_k && acc_v && cu_seqlens && kv_start && kv_len,
             "nv_attn_bwd_kv: null argument");
  NV_REQUIRE((lddq & 7) == 0 && (lddk & 7) == 0 && (lddv & 7) == 0 && (ldo & 3) == 0 && (lddo & 3) == 0 && (ldacc & 1) == 0 &&
             ldacc >= (int64_t)H * 128, "nv_attn_bwd_kv: leading-dimension alignment");
  CUtensorMap tq, tk, tv, tdo;
  int rc;
  if ((rc = make_tmap_2d(&tq, q, 2, (uint64_t)H * 128, (uint64_t)Tq, (uint64_t)ldq * 2, 64, 64))) return rc;
  if ((rc = make_tmap_2d(&tk, kcache, 2, (uint64_t)H * 128, (uint64_t)Tkv, (uint64_t)ldkv * 2, 64, 64))) return rc;
  if ((rc = make_tmap_2d(&tv, vcache, 2, (uint64_t)H * 128, (uint64_t)Tkv, (uint64_t)ldkv * 2, 64, 64))) return rc;
  if ((rc = make_tmap_2d(&tdo, dout, 2, (uint64_t)H * 128, (uint64_t)Tq, (uint64_t)lddo * 2, 64, 64))) return rc;
  static bool attr_set = false;
  if (!attr_set) {
    NV_CUDA(cudaFuncSetAttribute(attn_bwd_dq_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, BwdSmem::DYN_BYTES));
    NV_CUDA(cudaFuncSetAttribute(attn_bwd_dkv_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, BwdSmem::DYN_BYTES));
    attr_set = true;
  }
  if ((rc = attn_bwd_prep(o, ldo, dout, lddo, dvec, Tq, H, stream))) return rc;
  const __nv_bfloat16* c = reinterpret_cast<const __nv_bfloat16*>(cos_t);
  const __nv_bfloat16* s = reinterpret_cast<const __nv_bfloat16*>(sin_t);
  attn_bwd_dkv_kernel<true><<<dim3(total_kblocks, H), AB_THREADS, BwdSmem::DYN_BYTES, stream>>>(
      tq, tk, tv, tdo, lse, dvec, reinterpret_cast<__nv_bfloat16*>(dk), lddk, reinterpret_cast<__nv_bfloat16*>(dv), lddv,
      cu_seqlens, B, Tq, scale, rope_pos, c, s, kv_start, kv_len, acc_k, acc_v, ldacc);
  NV_LAUNCH_CHECK();
  attn_bwd_dq_kernel<true><<<dim3(total_qblocks, H), AB_THREADS, BwdSmem::DYN_BYTES, stream>>>(
      tq, tdo, tk, tv, lse, dvec, reinterpret_cast<__nv_bfloat16*>(dq), lddq, cu_seqlens, B, Tq, scale, rope_pos, c, s,
      kv_start, kv_len);
  NV_LAUNCH_CHECK();
  return NV_OK;
}
