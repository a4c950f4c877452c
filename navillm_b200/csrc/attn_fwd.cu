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
#include "nv_common.cuh"
#include "nv_host.h"

namespace nv {

constexpr uint32_t ATT_TILE_BYTES = 128 * 128 * 2;  // one 128x128 bf16 tile = two 64-wide swizzle atoms
constexpr uint32_t ATT_ATOM_BYTES = 128 * 128;      // 128 rows x 128 B
constexpr uint32_t ATT_THREADS = 288;
constexpr uint32_t ATT_QROWS = 128;

struct AttnFwdSmem {
  static constexpr uint32_t Q_OFF = 0;
  static constexpr uint32_t K_OFF = Q_OFF + ATT_TILE_BYTES;        // 2 slots
  static constexpr uint32_t V_OFF = K_OFF + 2 * ATT_TILE_BYTES;    // 2 slots
  static constexpr uint32_t BAR_OFF = V_OFF + 2 * ATT_TILE_BYTES;
  // q_full, k_full[2], v_full[2], kv_empty[2]
  static constexpr uint32_t NUM_BARS = 7;
  static constexpr uint32_t DYN_BYTES = BAR_OFF + NUM_BARS * 8 + 1024;
};

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

__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                const __grid_constant__ CUtensorMap tmap_v, __nv_bfloat16* __restrict__ O, int64_t ldo,
                float* __restrict__ lse, const int* __restrict__ cu_seqlens, int B, int T, float scale,
                const int* __restrict__ kv_start, const int* __restrict__ kv_len) {
  using L = AttnFwdSmem;
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
    for (int i = 0; i < 2; ++i) { mbar_init(&k_full[i], 1); mbar_init(&v_full[i], 1); mbar_init(&kv_empty[i], 2); }
    fence_mbar_init();
  }
  __syncthreads();

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
    if (j * 128 + 127 > vis_first) {                               // block holds keys some row must not see
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
    // key 0 is visible to every row, so the maximum is finite from the first block on
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
static int attn_fwd_launch(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o,
                           int64_t ldo, float* lse, const int* cu_seqlens, const int* kv_start, const int* kv_len, int B, int T,
                           int Tkv, int H, int head_dim, int total_qblocks, float scale, void* stream) {
  using namespace nv;
  NV_REQUIRE(head_dim == 128, "nv_attn_fwd: head_dim must be 128 (got %d)", head_dim);
  NV_REQUIRE(B > 0 && T > 0 && H > 0 && total_qblocks > 0, "nv_attn_fwd: empty problem");
  NV_REQUIRE((ldo & 7) == 0, "nv_attn_fwd: ldo %% 8");
  CUtensorMap tq, tk, tv;
  int rc;
  if ((rc = make_tmap_2d(&tq, q, 2, (uint64_t)H * 128, (uint64_t)T, (uint64_t)ldq * 2, 64, 128))) return rc;
  if ((rc = make_tmap_2d(&tk, k, 2, (uint64_t)H * 128, (uint64_t)Tkv, (uint64_t)ldk * 2, 64, 128))) return rc;
  if ((rc = make_tmap_2d(&tv, v, 2, (uint64_t)H * 128, (uint64_t)Tkv, (uint64_t)ldv * 2, 64, 128))) return rc;
  static bool attr_set = false;
  if (!attr_set) {
    NV_CUDA(cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AttnFwdSmem::DYN_BYTES));
    attr_set = true;
  }
  dim3 grid(total_qblocks, H);
  attn_fwd_kernel<<<grid, ATT_THREADS, AttnFwdSmem::DYN_BYTES, reinterpret_cast<cudaStream_t>(stream)>>>(
      tq, tk, tv, reinterpret_cast<__nv_bfloat16*>(o), ldo, lse, cu_seqlens, B, T, scale, kv_start, kv_len);
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
