// navillm_b200 — causal self-attention forward on Hopper wgmma (flash-style, packed variable-length rows).
//
// Replaces HF LLaMA's eager attention (reference call site models/modified_lm.py:112-116 ->
// LlamaAttention: scores = QK^T/sqrt(hd) + causal/left-pad mask, fp32 softmax, P·V; SURVEY.md §2b K9),
// which materialises [B,32,S,S] scores.  Here the sequences of a batch are PACKED (no pad tokens are
// ever computed): row t of the fused qkv buffer belongs to sequence b with cu_seqlens[b] <= t <
// cu_seqlens[b+1]; the reference's left padding is reproduced by the explicit position ids given to
// the rotary kernel, so results at real tokens are identical (pad positions do not exist here).
//
// One CTA = one (128-query block, head).  head_dim = 128.  288 threads:
//   warp 8            TMA producer: Q once; K_j and V_j through a 2-slot ring (separate full barriers, so that the
//                     scores of block j can start while V_j is still in flight)
//   warpgroups 0, 1   query rows 0..63 / 64..127 of the block.  Per key block: S = Q K_j^T with m64n128k16 wgmmas from
//                     shared memory (fp32 in registers), online softmax in registers (row max / sum over the four
//                     threads of a row), P rounded to bf16 and fed to O += P V_j straight from registers (the wgmma
//                     A-from-registers form: the S accumulator layout is the A-fragment layout), V read MN-major.
// The exponent reference is the running row maximum (log2 units); the row sum is taken over the fp32 p before their
// bf16 rounding, and O is normalised once at the end.
// smem: Q 32K + K 2x32K + V 2x32K = 160 KB.
//
// fp8 cache (FP8 = true, nv_attn_fwd_kv_fp8; format: include/navillm_b200.h): the keys / values are e4m3 rows with one int8
// exponent per (position, head) row.  384 threads: warpgroup 2 (warps 8..11) replaces the lone producer warp.  Warp 8
// TMA-loads the e4m3 K_j and V_j tiles (128 keys x 128 B each, unswizzled) into a 2-slot staging ring and copies the tile's
// 128 + 128 exponents of this head beside them (plain loads: the exponents of one head are H bytes apart, which a TMA box
// cannot stride).  All 128 threads of the warpgroup then widen each staged tile with fp8x4_to_bf16x4 into the bf16 slot the
// bf16 kernel's TMA would have filled, 128-byte swizzled the same way, and arrive on that slot's k_full / v_full: so the
// consumers, their wgmmas, the key order, the online softmax and the normalisation are the bf16 kernel's, and since
// e4m3 * 2^e is exact in bf16 (nv_fp8.cuh) the output is bit for bit nv_attn_fwd_kv over a bf16 cache holding K' / V'.
// The staging is double-buffered: tile j + 2 is in flight while tile j + 1 is widened and tile j is multiplied, so neither
// the HBM latency nor the widening sits between two key blocks of the consumers.  That takes 64 KB on top of the 160 KB
// (225.6 KB of the 227 KB an H100 CTA may use); single-buffered staging would leave the load of tile j + 1 exposed
// whenever it has to wait for the widening of tile j.  384 threads leave the consumers 168 registers a thread.
//
// Tree mask (TREE = true, nv_attn_fwd_tree[_fp8]): the query rows of a sequence are the nodes of a tree in DFS preorder, and
// tree_end[j] (int32 [q_len], shared by every sequence) is the first row after node j's subtree, so key dk + j is an ancestor-
// or-self of query i iff j <= i < tree_end[j].  A query sees the dk cached keys and the keys of its ancestors and itself.
// Preorder puts every ancestor before its descendants, so the causal block count still bounds the blocks a query needs; the
// tree test runs on every block that holds keys at or past dk, not only on the diagonal one.
#include "nv_common.cuh"
#include "nv_fp8.cuh"
#include "nv_host.h"

namespace nv {

constexpr uint32_t ATT_TILE_BYTES = 128 * 128 * 2;  // one 128x128 bf16 tile = two 64-wide swizzle atoms
constexpr uint32_t ATT_ATOM_BYTES = 128 * 128;      // 128 rows x 128 B
constexpr uint32_t ATT_TILE8_BYTES = 128 * 128;     // one 128x128 e4m3 tile, unswizzled
constexpr uint32_t ATT_THREADS = 288;
constexpr uint32_t ATT_QROWS = 128;

template <bool FP8>
struct AttnFwdSmem {
  static constexpr uint32_t THREADS = FP8 ? 384 : ATT_THREADS;
  static constexpr uint32_t Q_OFF = 0;
  static constexpr uint32_t K_OFF = Q_OFF + ATT_TILE_BYTES;        // 2 slots
  static constexpr uint32_t V_OFF = K_OFF + 2 * ATT_TILE_BYTES;    // 2 slots
  // fp8 only: staging slot s holds the e4m3 K tile, then the V tile, at STG_OFF + s * 2 * ATT_TILE8_BYTES, and its exponents
  // (128 of K, then 128 of V) at EXP_OFF + s * 256
  static constexpr uint32_t STG_OFF = V_OFF + 2 * ATT_TILE_BYTES;
  static constexpr uint32_t EXP_OFF = STG_OFF + (FP8 ? 2 * 2 * ATT_TILE8_BYTES : 0);
  static constexpr uint32_t BAR_OFF = EXP_OFF + (FP8 ? 2 * 256 : 0);
  // q_full, k_full[2], v_full[2], kv_empty[2] (fp8: + stg_full[2])
  static constexpr uint32_t NUM_BARS = FP8 ? 9 : 7;
  static constexpr uint32_t DYN_BYTES = BAR_OFF + NUM_BARS * 8 + 1024;
  static_assert(DYN_BYTES <= 232448, "shared memory per block");
};

// Widen one staged e4m3 tile (128 rows x 128 B at src, row r scaled by 2^exps[r]) into the 128-byte-swizzled bf16 tile at dst
// (two 64-wide atoms), the layout TMA SWIZZLE_128B writes.  Thread t of the 128 owns the 16-byte chunks q = t + 128 i: row q / 8,
// columns 16 (q % 8) ..+15, which become bf16 chunks 2 (q % 4), 2 (q % 4) + 1 of atom (q % 8) / 4.  The threads of the second
// atom store their two halves in the opposite order, so the eight threads of a quarter-warp hit eight different bank groups.
__device__ __forceinline__ void att_widen_tile(uint32_t src, uint32_t dst, const int8_t* exps, uint32_t t) {
#pragma unroll
  for (uint32_t i = 0; i < 8; ++i) {
    const uint32_t q = t + 128 * i, row = q >> 3, c = q & 7, h = c >> 2;
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(src + q * 16));
    const float s = fp8_pow2(exps[row]);
    uint32_t o[8];
    fp8x4_to_bf16x4(v.x, s, o[0], o[1]);
    fp8x4_to_bf16x4(v.y, s, o[2], o[3]);
    fp8x4_to_bf16x4(v.z, s, o[4], o[5]);
    fp8x4_to_bf16x4(v.w, s, o[6], o[7]);
    const uint32_t base = dst + h * ATT_ATOM_BYTES, ch = 2 * (c & 3);
    sts128(base + sw128_offset(row, ch + h), h ? o[4] : o[0], h ? o[5] : o[1], h ? o[6] : o[2], h ? o[7] : o[3]);
    sts128(base + sw128_offset(row, ch + 1 - h), h ? o[0] : o[4], h ? o[1] : o[5], h ? o[2] : o[6], h ? o[3] : o[7]);
  }
}

// Map a flat block id to (sequence, 128-row query block); heavy (late) blocks are launched first.
__device__ __forceinline__ bool locate_qblock(const int* __restrict__ cu, int B, uint32_t blk, int& seq_start,
                                              int& seq_len, uint32_t& qblk, int& seq_idx) {
  for (int b = 0; b < B; ++b) {
    const int s = cu[b], len = cu[b + 1] - s;
    const uint32_t nb = (len + ATT_QROWS - 1) / ATT_QROWS;
    if (blk < nb) { seq_start = s; seq_len = len; qblk = blk; seq_idx = b; return true; }
    blk -= nb;
  }
  return false;
}

// FP8: tmap_k / tmap_v describe the e4m3 caches and kexp / vexp are their row exponents ([Tkv, H] int8); unused otherwise.
// TREE: tree_end is the subtree table of the tree mask (see above); unused otherwise.
template <bool FP8, bool TREE = false>
__global__ void __launch_bounds__(AttnFwdSmem<FP8>::THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                const __grid_constant__ CUtensorMap tmap_v, __nv_bfloat16* __restrict__ O, int64_t ldo,
                float* __restrict__ lse, const int* __restrict__ cu_seqlens, int B, int T, float scale,
                const int* __restrict__ kv_start, const int* __restrict__ kv_len, const int8_t* __restrict__ kexp,
                const int8_t* __restrict__ vexp, int Tkv, const int* __restrict__ tree_end) {
  using L = AttnFwdSmem<FP8>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem + L::Q_OFF;
  uint8_t* sK = smem + L::K_OFF;
  uint8_t* sV = smem + L::V_OFF;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* q_full = bars + 0;
  uint64_t* k_full = bars + 1;     // [2]
  uint64_t* v_full = bars + 3;     // [2]
  uint64_t* kv_empty = bars + 5;   // [2] both warpgroups are done with K_j and V_j of the slot

  const uint32_t warp = warp_id_uniform(), lane = threadIdx.x & 31;
  const uint32_t head = blockIdx.y;

  int seq_start = 0, seq_len = 0, seq_idx = 0;
  uint32_t qblk = 0;
  if (!locate_qblock(cu_seqlens, B, gridDim.x - 1 - blockIdx.x, seq_start, seq_len, qblk, seq_idx)) return;  // CTA-uniform
  // Keys: by default the sequence's own rows (self-attention over the packed batch).  With kv_start / kv_len the
  // keys of sequence b are rows kv_start[b] .. +kv_len[b] of the K/V tensors (a KV cache holding an already encoded
  // prefix followed by the new rows) and the queries are its LAST seq_len positions: query i sees keys <= dk + i,
  // dk = kv_len - seq_len.
  const int kv0 = kv_start ? kv_start[seq_idx] : seq_start;
  const uint32_t dk = kv_len ? (uint32_t)(kv_len[seq_idx] - seq_len) : 0u;
  const uint32_t q0 = qblk * ATT_QROWS;                                       // first query row (inside the sequence)
  const uint32_t n_blocks = (dk + min(q0 + ATT_QROWS, (uint32_t)seq_len) + 127) / 128;   // key blocks the block sees

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    // fp8: the 128 widening threads fill k_full / v_full, and stg_full is the TMA barrier of a staging slot
    for (int i = 0; i < 2; ++i) {
      mbar_init(&k_full[i], FP8 ? 128 : 1); mbar_init(&v_full[i], FP8 ? 128 : 1); mbar_init(&kv_empty[i], 2);
      if constexpr (FP8) mbar_init(&bars[7 + i], 1);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if constexpr (FP8) {
    if (warp >= 8) {
      // ================================ TMA producer (warp 8) and widening (warps 8..11) ================================
      uint64_t* stg_full = bars + 7;   // [2]
      uint8_t* stg = smem + L::STG_OFF;
      int8_t* sexp = reinterpret_cast<int8_t*>(smem + L::EXP_OFF);
      const uint32_t t = threadIdx.x - 256;
      const int32_t col = head * 128;
      const int64_t H = gridDim.y;
      int8_t ek[4], ev[4];             // warp 8: exponents of keys lane + 32 i of the next tile it stages
      auto load_exps = [&](uint32_t j) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int r = kv0 + (int)(j * 128 + lane + 32 * i);
          ek[i] = r < Tkv ? kexp[r * H + head] : int8_t(0);  // rows past the cache: TMA zero fill, scale 1
          ev[i] = r < Tkv ? vexp[r * H + head] : int8_t(0);
        }
      };
      auto stage = [&](uint32_t j) {   // warp 8: exponents, then the two e4m3 tiles of key block j, into slot j & 1
        const uint32_t s = j & 1;
#pragma unroll
        for (int i = 0; i < 4; ++i) { sexp[s * 256 + lane + 32 * i] = ek[i]; sexp[s * 256 + 128 + lane + 32 * i] = ev[i]; }
        __syncwarp();
        if (elect_one()) {
          const int32_t krow0 = kv0 + j * 128;
          mbar_arrive_expect_tx(&stg_full[s], 2 * ATT_TILE8_BYTES);   // releases the exponent stores of the warp
          tma_load_2d(stg + s * 2 * ATT_TILE8_BYTES, &tmap_k, &stg_full[s], col, krow0);
          tma_load_2d(stg + s * 2 * ATT_TILE8_BYTES + ATT_TILE8_BYTES, &tmap_v, &stg_full[s], col, krow0);
        }
        __syncwarp();
      };
      if (warp == 8) {
        tma_prefetch_desc(&tmap_q); tma_prefetch_desc(&tmap_k); tma_prefetch_desc(&tmap_v);
        if (elect_one()) {
          mbar_arrive_expect_tx(q_full, ATT_TILE_BYTES);
          tma_load_2d(sQ, &tmap_q, q_full, col, seq_start + q0);
          tma_load_2d(sQ + ATT_ATOM_BYTES, &tmap_q, q_full, col + 64, seq_start + q0);
        }
        __syncwarp();
        for (uint32_t j = 0; j < 2 && j < n_blocks; ++j) { load_exps(j); stage(j); }
      }
      for (uint32_t j = 0; j < n_blocks; ++j) {
        const uint32_t slot = j & 1, par = (j >> 1) & 1;
        const bool refill = warp == 8 && j + 2 < n_blocks;
        if (refill) load_exps(j + 2);                                 // in flight while tile j is widened
        mbar_wait(&stg_full[slot], par);
        mbar_wait(&kv_empty[slot], par ^ 1);                          // both warpgroups are done with block j - 2
        const uint32_t src = smem_u32(stg + slot * 2 * ATT_TILE8_BYTES);
        att_widen_tile(src, smem_u32(sK + slot * ATT_TILE_BYTES), sexp + slot * 256, t);
        fence_proxy_async_smem();                                     // generic-proxy writes -> wgmma operand reads
        mbar_arrive(&k_full[slot]);
        att_widen_tile(src + ATT_TILE8_BYTES, smem_u32(sV + slot * ATT_TILE_BYTES), sexp + slot * 256 + 128, t);
        fence_proxy_async_smem();
        mbar_arrive(&v_full[slot]);
        named_bar_sync(4, 128);                                       // every read of staging slot j & 1 is done
        if (refill) stage(j + 2);
      }
      return;
    }
  }

  if (warp == 8) {
    // ================================ TMA producer ================================
    tma_prefetch_desc(&tmap_q); tma_prefetch_desc(&tmap_k); tma_prefetch_desc(&tmap_v);
    const int32_t col = head * 128;
    if (elect_one()) {
      mbar_arrive_expect_tx(q_full, ATT_TILE_BYTES);
      tma_load_2d(sQ, &tmap_q, q_full, col, seq_start + q0);
      tma_load_2d(sQ + ATT_ATOM_BYTES, &tmap_q, q_full, col + 64, seq_start + q0);
    }
    __syncwarp();
    for (uint32_t j = 0; j < n_blocks; ++j) {
      const uint32_t slot = j & 1;
      mbar_wait(&kv_empty[slot], ((j >> 1) & 1) ^ 1);
      if (elect_one()) {
        const int32_t krow0 = kv0 + j * 128;
        mbar_arrive_expect_tx(&k_full[slot], ATT_TILE_BYTES);
        tma_load_2d(sK + slot * ATT_TILE_BYTES, &tmap_k, &k_full[slot], col, krow0);
        tma_load_2d(sK + slot * ATT_TILE_BYTES + ATT_ATOM_BYTES, &tmap_k, &k_full[slot], col + 64, krow0);
        mbar_arrive_expect_tx(&v_full[slot], ATT_TILE_BYTES);
        tma_load_2d(sV + slot * ATT_TILE_BYTES, &tmap_v, &v_full[slot], col, krow0);
        tma_load_2d(sV + slot * ATT_TILE_BYTES + ATT_ATOM_BYTES, &tmap_v, &v_full[slot], col + 64, krow0);
      }
      __syncwarp();
    }
    return;
  }

  // ================================ consumers ================================
  const uint32_t wg = warp >> 2;
  const uint32_t ra = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's rows ra, ra + 8 (inside the block)
  const uint32_t qa = q0 + ra, qb = qa + 8;                       // query index inside the sequence
  const uint32_t cq = 2 * (lane & 3);                             // column offset of the thread's pairs
  const float sl2 = scale * 1.4426950408889634f;
  const uint32_t vis_first = dk + q0 + wg * 64;                   // last key visible to the warpgroup's first row
  float oacc[64];
#pragma unroll
  for (uint32_t i = 0; i < 64; ++i) oacc[i] = 0.f;
  float m_a = -INFINITY, m_b = -INFINITY, l_a = 0.f, l_b = 0.f;   // running max (log2 units) and partial row sums
  const uint64_t qdesc = gmma_desc_sw128(smem_u32(sQ + wg * 8192), 0, 1024);
  mbar_wait(q_full, 0);
  for (uint32_t j = 0; j < n_blocks; ++j) {
    const uint32_t slot = j & 1, par = (j >> 1) & 1;
    float sacc[64];
    mbar_wait(&k_full[slot], par);
    {
      const uint64_t kdesc = gmma_desc_sw128(smem_u32(sK + slot * ATT_TILE_BYTES), 0, 1024);
      wgmma_fence();
#pragma unroll
      for (uint32_t ks = 0; ks < 8; ++ks)   // hd step 16 ks: atom ks / 4, +32 B per step inside it
        wgmma_ss_bf16<128, 0, 0>(sacc, qdesc + (ks >> 2) * (ATT_ATOM_BYTES >> 4) + (ks & 3) * 2,
                                 kdesc + (ks >> 2) * (ATT_ATOM_BYTES >> 4) + (ks & 3) * 2, ks ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(sacc);
    }
    if constexpr (TREE) {
      if (j * 128 + 127 >= dk) {                                   // block holds tree keys: causal and ancestor test
        const int rel0 = (int)(j * 128) - (int)dk;                 // tree row of the block's first key
#pragma unroll
        for (uint32_t i = 0; i < 16; ++i) {
          const int r0 = rel0 + (int)(8 * i + cq), r1 = r0 + 1;
          // cached keys are seen by every row; tree rows past the sequence's exist for no real row
          const int e0 = r0 < 0 ? 0x7fffffff : r0 < seq_len ? __ldg(tree_end + r0) : 0;
          const int e1 = r1 < 0 ? 0x7fffffff : r1 < seq_len ? __ldg(tree_end + r1) : 0;
          if ((int)qa < r0 || (int)qa >= e0) sacc[4 * i] = -INFINITY;
          if ((int)qa < r1 || (int)qa >= e1) sacc[4 * i + 1] = -INFINITY;
          if ((int)qb < r0 || (int)qb >= e0) sacc[4 * i + 2] = -INFINITY;
          if ((int)qb < r1 || (int)qb >= e1) sacc[4 * i + 3] = -INFINITY;
        }
      }
    } else if (j * 128 + 127 > vis_first) {                        // block holds keys some row must not see
      const int lim_a = (int)(dk + qa) - (int)(j * 128), lim_b = lim_a + 8;
#pragma unroll
      for (uint32_t i = 0; i < 16; ++i) {
        const int c = (int)(8 * i + cq);
        if (c > lim_a) sacc[4 * i] = -INFINITY;
        if (c + 1 > lim_a) sacc[4 * i + 1] = -INFINITY;
        if (c > lim_b) sacc[4 * i + 2] = -INFINITY;
        if (c + 1 > lim_b) sacc[4 * i + 3] = -INFINITY;
      }
    }
    float mxa = -INFINITY, mxb = -INFINITY;
#pragma unroll
    for (uint32_t i = 0; i < 16; ++i) {
      mxa = fmaxf(mxa, fmaxf(sacc[4 * i], sacc[4 * i + 1]));
      mxb = fmaxf(mxb, fmaxf(sacc[4 * i + 2], sacc[4 * i + 3]));
    }
    mxa = fmaxf(mxa, __shfl_xor_sync(0xffffffffu, mxa, 1));
    mxa = fmaxf(mxa, __shfl_xor_sync(0xffffffffu, mxa, 2));
    mxb = fmaxf(mxb, __shfl_xor_sync(0xffffffffu, mxb, 1));
    mxb = fmaxf(mxb, __shfl_xor_sync(0xffffffffu, mxb, 2));
    // key 0 is visible to every row (TREE: a cached key, dk >= 1), so the maximum is finite from the first block on
    const float mna = fmaxf(m_a, mxa * sl2), mnb = fmaxf(m_b, mxb * sl2);
    const float alpha_a = exp2f(m_a - mna), alpha_b = exp2f(m_b - mnb);
    m_a = mna; m_b = mnb;
    float rsa = 0.f, rsb = 0.f;
#pragma unroll
    for (uint32_t i = 0; i < 16; ++i) {
      sacc[4 * i] = exp2f(fmaf(sacc[4 * i], sl2, -mna));
      sacc[4 * i + 1] = exp2f(fmaf(sacc[4 * i + 1], sl2, -mna));
      sacc[4 * i + 2] = exp2f(fmaf(sacc[4 * i + 2], sl2, -mnb));
      sacc[4 * i + 3] = exp2f(fmaf(sacc[4 * i + 3], sl2, -mnb));
      rsa += sacc[4 * i] + sacc[4 * i + 1];
      rsb += sacc[4 * i + 2] + sacc[4 * i + 3];
    }
    l_a = l_a * alpha_a + rsa;
    l_b = l_b * alpha_b + rsb;
#pragma unroll
    for (uint32_t i = 0; i < 16; ++i) {
      oacc[4 * i] *= alpha_a; oacc[4 * i + 1] *= alpha_a;
      oacc[4 * i + 2] *= alpha_b; oacc[4 * i + 3] *= alpha_b;
    }
    // O += P V_j: P (bf16) from registers, 16 keys per wgmma; V rows = keys (K dim), hd contiguous (MN-major B)
    mbar_wait(&v_full[slot], par);
    {
      const uint64_t vdesc = gmma_desc_sw128(smem_u32(sV + slot * ATT_TILE_BYTES), ATT_ATOM_BYTES, 1024);
      wgmma_fence();
#pragma unroll
      for (uint32_t kk = 0; kk < 8; ++kk) {
        const uint32_t a[4] = {pack_bf16x2(sacc[8 * kk], sacc[8 * kk + 1]), pack_bf16x2(sacc[8 * kk + 2], sacc[8 * kk + 3]),
                               pack_bf16x2(sacc[8 * kk + 4], sacc[8 * kk + 5]), pack_bf16x2(sacc[8 * kk + 6], sacc[8 * kk + 7])};
        wgmma_rs_bf16<128, 1>(oacc, a, vdesc + kk * ((16 * 128) >> 4), 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(oacc);
    }
    if ((threadIdx.x & 127) == 0) mbar_arrive(&kv_empty[slot]);
  }

  // ---- epilogue ----
  l_a += __shfl_xor_sync(0xffffffffu, l_a, 1);
  l_a += __shfl_xor_sync(0xffffffffu, l_a, 2);
  l_b += __shfl_xor_sync(0xffffffffu, l_b, 1);
  l_b += __shfl_xor_sync(0xffffffffu, l_b, 2);
  // natural-log LSE of the scaled scores: m is in log2 units
  if (lse && (lane & 3) == 0) {
    if (qa < (uint32_t)seq_len) lse[(int64_t)head * T + seq_start + qa] = m_a * 0.6931471805599453f + __logf(l_a);
    if (qb < (uint32_t)seq_len) lse[(int64_t)head * T + seq_start + qb] = m_b * 0.6931471805599453f + __logf(l_b);
  }
  // Two phases so that HBM sees full 256-byte rows: the normalised bf16 O rows of the warpgroup go into its own 16 KB
  // of the K ring (free once both warpgroups are past the last block; 16-byte chunks XOR-swizzled by the row), then each
  // warp streams whole rows out with 8-byte coalesced stores.
  named_bar_sync(1, 256);
  const uint32_t stg = smem_u32(sK + wg * 64 * 256);
  const float inv_a = 1.f / l_a, inv_b = 1.f / l_b;
  const uint32_t rl = ra - wg * 64;
#pragma unroll
  for (uint32_t i = 0; i < 16; ++i) {
    const uint32_t c = 8 * i + cq;
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(stg + rl * 256 + ((((c >> 3) ^ (rl & 15))) << 4) + (c & 7) * 2),
                 "r"(pack_bf16x2(oacc[4 * i] * inv_a, oacc[4 * i + 1] * inv_a)) : "memory");
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(stg + (rl + 8) * 256 + ((((c >> 3) ^ ((rl + 8) & 15))) << 4) + (c & 7) * 2),
                 "r"(pack_bf16x2(oacc[4 * i + 2] * inv_b, oacc[4 * i + 3] * inv_b)) : "memory");
  }
  named_bar_sync(2 + wg, 128);
  const uint32_t r0 = q0 + wg * 64;
  const uint32_t rows_valid = (uint32_t)seq_len > r0 ? min(64u, (uint32_t)seq_len - r0) : 0u;
  __nv_bfloat16* obase = O + ((int64_t)seq_start + r0) * ldo + head * 128;
  for (uint32_t rr = warp & 3; rr < rows_valid; rr += 4) {
    const uint32_t chunk = (lane >> 1) ^ (rr & 15);
    const uint2 x = lds64(stg + rr * 256 + (chunk << 4) + ((lane & 1) << 3));
    *reinterpret_cast<uint2*>(obase + (int64_t)rr * ldo + lane * 4) = x;
  }
}

}  // namespace nv

// q, k, v: bf16 row-major [T, *] views with leading dimensions ldq/ldk/ldv (elements); head h occupies
// columns [h*128, (h+1)*128).  o: [T, H*128] bf16 (ldo).  lse: [H, T] fp32 or null.
// cu_seqlens: device int32 [B+1]; total_qblocks = sum_b ceil(len_b / 128) (the host knows the lengths): one CTA each.
// kexp / vexp (fp8 cache): k / v are e4m3 [Tkv, H*128] caches (ldk = ldv = H*128 bytes) with int8 exponents [Tkv, H].
static int attn_fwd_launch(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o,
                           int64_t ldo, float* lse, const int* cu_seqlens, const int* kv_start, const int* kv_len, int B, int T,
                           int Tkv, int H, int head_dim, int total_qblocks, float scale, void* stream,
                           const void* kexp = nullptr, const void* vexp = nullptr, const int* tree_end = nullptr) {
  using namespace nv;
  NV_REQUIRE(head_dim == 128, "nv_attn_fwd: head_dim must be 128 (got %d)", head_dim);
  NV_REQUIRE(B > 0 && T > 0 && H > 0 && total_qblocks > 0, "nv_attn_fwd: empty problem");
  NV_REQUIRE((ldo & 7) == 0, "nv_attn_fwd: ldo %% 8");
  const bool fp8 = kexp != nullptr;
  CUtensorMap tq, tk, tv;
  int rc;
  if ((rc = make_tmap_2d(&tq, q, 2, (uint64_t)H * 128, (uint64_t)T, (uint64_t)ldq * 2, 64, 128))) return rc;
  if (fp8) {
    if ((rc = make_tmap_2d(&tk, k, 1, (uint64_t)H * 128, (uint64_t)Tkv, (uint64_t)ldk, 128, 128, /*swizzle128=*/false))) return rc;
    if ((rc = make_tmap_2d(&tv, v, 1, (uint64_t)H * 128, (uint64_t)Tkv, (uint64_t)ldv, 128, 128, /*swizzle128=*/false))) return rc;
  } else {
    if ((rc = make_tmap_2d(&tk, k, 2, (uint64_t)H * 128, (uint64_t)Tkv, (uint64_t)ldk * 2, 64, 128))) return rc;
    if ((rc = make_tmap_2d(&tv, v, 2, (uint64_t)H * 128, (uint64_t)Tkv, (uint64_t)ldv * 2, 64, 128))) return rc;
  }
  const bool tree = tree_end != nullptr;
  static bool attr_set[2][2] = {{false, false}, {false, false}};
  if (!attr_set[tree][fp8]) {
    const int bytes = fp8 ? AttnFwdSmem<true>::DYN_BYTES : AttnFwdSmem<false>::DYN_BYTES;
    const void* fn = tree ? (fp8 ? (const void*)attn_fwd_kernel<true, true> : (const void*)attn_fwd_kernel<false, true>)
                          : (fp8 ? (const void*)attn_fwd_kernel<true> : (const void*)attn_fwd_kernel<false>);
    NV_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    attr_set[tree][fp8] = true;
  }
  dim3 grid(total_qblocks, H);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  __nv_bfloat16* O = reinterpret_cast<__nv_bfloat16*>(o);
  const int8_t* ke = reinterpret_cast<const int8_t*>(kexp);
  const int8_t* ve = reinterpret_cast<const int8_t*>(vexp);
  if (fp8 && tree)
    attn_fwd_kernel<true, true><<<grid, AttnFwdSmem<true>::THREADS, AttnFwdSmem<true>::DYN_BYTES, st>>>(
        tq, tk, tv, O, ldo, lse, cu_seqlens, B, T, scale, kv_start, kv_len, ke, ve, Tkv, tree_end);
  else if (fp8)
    attn_fwd_kernel<true><<<grid, AttnFwdSmem<true>::THREADS, AttnFwdSmem<true>::DYN_BYTES, st>>>(
        tq, tk, tv, O, ldo, lse, cu_seqlens, B, T, scale, kv_start, kv_len, ke, ve, Tkv, nullptr);
  else if (tree)
    attn_fwd_kernel<false, true><<<grid, ATT_THREADS, AttnFwdSmem<false>::DYN_BYTES, st>>>(
        tq, tk, tv, O, ldo, lse, cu_seqlens, B, T, scale, kv_start, kv_len, nullptr, nullptr, Tkv, tree_end);
  else
    attn_fwd_kernel<false><<<grid, ATT_THREADS, AttnFwdSmem<false>::DYN_BYTES, st>>>(
        tq, tk, tv, O, ldo, lse, cu_seqlens, B, T, scale, kv_start, kv_len, nullptr, nullptr, Tkv, nullptr);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

extern "C" int nv_attn_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o,
                           int64_t ldo, float* lse, const int* cu_seqlens, int B, int T, int H, int head_dim,
                           int total_qblocks, float scale, void* stream) {
  return attn_fwd_launch(q, ldq, k, ldk, v, ldv, o, ldo, lse, cu_seqlens, nullptr, nullptr, B, T, T, H, head_dim,
                         total_qblocks, scale, stream);
}

// Suffix ("append") attention over a KV cache: the Tq packed query rows of sequence b (cu_seqlens) are the LAST
// positions of a context whose keys/values are rows kv_start[b] .. kv_start[b] + kv_len[b] of the cache tensors
// (Tkv rows in total; kv_len[b] >= query count, already holding the new rows' K/V).  Rows of the cache past kv_len
// must be finite (allocate it zeroed): they are masked, but 0 * NaN would poison the P·V product.
extern "C" int nv_attn_fwd_kv(const void* q, int64_t ldq, const void* kcache, int64_t ldk, const void* vcache, int64_t ldv,
                              void* o, int64_t ldo, float* lse, const int* cu_seqlens, const int* kv_start,
                              const int* kv_len, int B, int Tq, int Tkv, int H, int head_dim, int total_qblocks, float scale,
                              void* stream) {
  using namespace nv;
  NV_REQUIRE(kv_start && kv_len, "nv_attn_fwd_kv: kv_start / kv_len are required");
  return attn_fwd_launch(q, ldq, kcache, ldk, vcache, ldv, o, ldo, lse, cu_seqlens, kv_start, kv_len, B, Tq, Tkv, H,
                         head_dim, total_qblocks, scale, stream);
}

// nv_attn_fwd_kv over an fp8 cache: kq / vq e4m3 [Tkv, H*128] (dense rows), kexp / vexp int8 [Tkv, H].  Rows past kv_len are
// masked and must widen to finite values: a zeroed cache, or rows the store kernel wrote, qualify.
extern "C" int nv_attn_fwd_kv_fp8(const void* q, int64_t ldq, const void* kq, const void* vq, const void* kexp, const void* vexp,
                                  void* o, int64_t ldo, float* lse, const int* cu_seqlens, const int* kv_start, const int* kv_len,
                                  int B, int Tq, int Tkv, int H, int head_dim, int total_qblocks, float scale, void* stream) {
  using namespace nv;
  NV_REQUIRE(head_dim == 128, "nv_attn_fwd_kv_fp8: head_dim must be 128 (got %d)", head_dim);
  NV_REQUIRE(q && kq && vq && kexp && vexp && o && cu_seqlens && kv_start && kv_len, "nv_attn_fwd_kv_fp8: null argument");
  NV_REQUIRE(Tkv > 0 && H > 0, "nv_attn_fwd_kv_fp8: bad sizes (Tkv=%d H=%d)", Tkv, H);
  return attn_fwd_launch(q, ldq, kq, (int64_t)H * 128, vq, (int64_t)H * 128, o, ldo, lse, cu_seqlens, kv_start, kv_len, B, Tq, Tkv,
                         H, head_dim, total_qblocks, scale, stream, kexp, vexp);
}

// nv_attn_fwd_kv with the tree mask: the q_len rows of every sequence are the nodes of one tree in DFS preorder (the same
// tree for every sequence, so Tq = B * q_len), and query i sees the kv_len - q_len >= 1 cached keys and tree key j only when
// j <= i < tree_end[j] (int32 [q_len] on the device: the first row after node j's subtree).  Rows of the cache past kv_len
// must be finite (allocate it zeroed).
extern "C" int nv_attn_fwd_tree(const void* q, int64_t ldq, const void* kcache, int64_t ldk, const void* vcache, int64_t ldv,
                                void* o, int64_t ldo, float* lse, const int* cu_seqlens, const int* kv_start, const int* kv_len,
                                const int* tree_end, int B, int Tq, int Tkv, int H, int head_dim, int total_qblocks, float scale,
                                void* stream) {
  using namespace nv;
  NV_REQUIRE(kv_start && kv_len && tree_end, "nv_attn_fwd_tree: kv_start / kv_len / tree_end are required");
  return attn_fwd_launch(q, ldq, kcache, ldk, vcache, ldv, o, ldo, lse, cu_seqlens, kv_start, kv_len, B, Tq, Tkv, H,
                         head_dim, total_qblocks, scale, stream, nullptr, nullptr, tree_end);
}

// nv_attn_fwd_tree over an fp8 cache (the layout of nv_attn_fwd_kv_fp8): bit for bit nv_attn_fwd_tree over a bf16 cache holding
// the rounded rows K' / V'.
extern "C" int nv_attn_fwd_tree_fp8(const void* q, int64_t ldq, const void* kq, const void* vq, const void* kexp, const void* vexp,
                                    void* o, int64_t ldo, float* lse, const int* cu_seqlens, const int* kv_start, const int* kv_len,
                                    const int* tree_end, int B, int Tq, int Tkv, int H, int head_dim, int total_qblocks, float scale,
                                    void* stream) {
  using namespace nv;
  NV_REQUIRE(head_dim == 128, "nv_attn_fwd_tree_fp8: head_dim must be 128 (got %d)", head_dim);
  NV_REQUIRE(q && kq && vq && kexp && vexp && o && cu_seqlens && kv_start && kv_len && tree_end,
             "nv_attn_fwd_tree_fp8: null argument");
  NV_REQUIRE(Tkv > 0 && H > 0, "nv_attn_fwd_tree_fp8: bad sizes (Tkv=%d H=%d)", Tkv, H);
  return attn_fwd_launch(q, ldq, kq, (int64_t)H * 128, vq, (int64_t)H * 128, o, ldo, lse, cu_seqlens, kv_start, kv_len, B, Tq, Tkv,
                         H, head_dim, total_qblocks, scale, stream, kexp, vexp, tree_end);
}
