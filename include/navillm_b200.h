/* navillm_b200 — C ABI of the native NaviLLM hot path (libnavillm_b200.so, sm_90a / H100 only).
 *
 * The reference (zd11024/NaviLLM) is pure Python/PyTorch and has NO native interface of its own: its
 * "operator API" for this path is the set of torch calls made inside NavModel.forward() and below
 * (SURVEY.md §8b).  Every entry point here replaces a group of those calls; the reference call site each
 * one stands in for is cited as file:line relative to the reference repository root.
 *
 * Conventions
 *   - raw DEVICE pointers (never host pointers, never torch types), explicit sizes and leading dimensions
 *     in ELEMENTS, `stream` = a cudaStream_t passed as void*;
 *   - the library allocates nothing on the device: outputs and workspaces are caller-owned;
 *   - return value: 0 = ok; negative = argument / environment error (NV_ERR_*); positive = cudaError_t.
 *     nv_last_error() returns a thread-local message for the last failure;
 *   - there is NO CPU fallback: without an sm_90 device every compute entry fails (NV_ERR_NO_DEVICE or a
 *     CUDA error), it never computes on the host;
 *   - bf16 tensors are row-major with 16-byte aligned rows (leading dimensions multiples of 8 elements).
 */
#ifndef NAVILLM_B200_H_
#define NAVILLM_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NV_OK 0
#define NV_ERR_BAD_ARG (-1)
#define NV_ERR_NO_DEVICE (-2)
#define NV_ERR_UNSUPPORTED (-3)

#define NV_GEMM_ADD 1u     /* C = bf16(bf16(acc) + addend): residual add / in-place gradient accumulation */
#define NV_GEMM_OUT_F32 2u /* C is fp32 */

/* ---- runtime ---------------------------------------------------------------------------------------- */
const char* nv_last_error(void);
int nv_abi_version(void);
/* Programmatic dependent launch for the decode chain (generate(): HF GenerationMixin greedy loop reached from
 * models/nav_model.py:324-338,388-399): when on, nv_embed_fwd / nv_rmsnorm_fwd / nv_gemm_skinny[_swiglu]_bf16 /
 * nv_decode_rope_kv / nv_decode_attn[_rope[_fp8]] / nv_add_int / nv_argmax_masked / nv_trie_mask are launched with
 * cudaLaunchAttributeProgrammaticStreamSerialization so a kernel's prologue (and the skinny GEMM's first weight tiles)
 * overlaps the tail of its predecessor.  Returns the previous setting.  Process-wide; default off. */
int nv_set_pdl(int on);
/* Batch-invariant split-K for the panorama encoder GEMMs nv_sgemm / nv_gemm_tf32 (NavModel.set_batch_invariant; reference
 * image_embedding.py's nn.Linear / nn.TransformerEncoder layers): when on, the K split count is the largest power of two
 * <= 8 that leaves every split at least 256 k (K alone decides), instead of following the tile count -- the number of
 * views in the batch -- and sm_count().  The splits are added in rank order either way, so an element's bits then depend
 * on its own row alone.  Returns the previous setting.  Process-wide; default off. */
int nv_set_fixed_splits(int on);
int nv_device_check(void); /* NV_OK iff the current device is sm_90 (Hopper) */
int nv_sm_count(void);

/* ---- wgmma bf16 GEMM (csrc/gemm_bf16.cu) -------------------------------------------------------------
 * C[M,N] = A·B (+addend).  a_mn=0: A is [M,K]; a_mn=1: A is [K,M].  b_mn=0: B is [N,K] (nn.Linear weight);
 * b_mn=1: B is [K,N].  Replaces every nn.Linear of the LLaMA block and lm_head and their autograd dgrad /
 * wgrad: models/modified_lm.py:112-116 (HF LlamaDecoderLayer q/k/v/o/gate/up/down_proj) and :120 (lm_head).
 * block_n: 0 (auto), 32 (M <= 128, K-major B), 128 or 256 (output tile 128 x block_n). */
int nv_gemm_bf16(const void* A, int64_t lda, int a_mn, const void* B, int64_t ldb, int b_mn, void* C, int64_t ldc,
                 const void* addend, int64_t ld_add, int M, int N, int K, unsigned flags, int block_n, void* stream);

/* Fused-epilogue forms on the 128 x 256 tile (csrc/gemm_bf16.cu), bit-identical to the unfused sequences:
 *   nv_gemm_swiglu_bf16   gu = x Wgu^T and h = silu(gate)*up        (HF LlamaMLP: act_fn(gate_proj(x)) * up_proj(x))
 *   nv_gemm_dswiglu_bf16  dgu = swiglu'(gu) o (dx Wd)               (autograd of the above through down_proj)
 *   nv_gemm_rope_bf16     qkv = x Wqkv^T with rotate-half RoPE on the q,k columns (HF apply_rotary_pos_emb)
 *   nv_gemm_attnd_bf16    dO = dY Wo (o_proj dgrad) and D[h,t] = sum_d dO O of the attention backward (same values as
 *                         the separate row-sum kernel up to fp32 summation order) */
/* Decode-step GEMM (M <= 16 rows, reference: HF generate through models/modified_lm.py:184-199): swap-AB wgmma
 * kernel with the K range split over a thread-block cluster and reduced through distributed shared memory
 * (csrc/gemm_skinny.cu).  C = bf16(bf16(X W^T) + addend), X [M,K], W [N,K] (nn.Linear layout). */
int nv_gemm_skinny_bf16(const void* X, int64_t ldx, const void* W, int64_t ldw, void* C, int64_t ldc, const void* addend,
                        int64_t ld_add, int M, int N, int K, void* stream);
/* ... with the SwiGLU of HF LlamaMLP fused: h[M,F] = bf16(bf16(silu(g)) * u), [g|u] = bf16(X Wgu^T), Wgu [2F,K] */
int nv_gemm_skinny_swiglu_bf16(const void* X, int64_t ldx, const void* Wgu, int64_t ldw, void* H, int64_t ldh, int M, int F,
                               int K, void* stream);
/* Batch-invariant inference GEMMs (ModifiedLlamaForCausalLM.set_batch_invariant; csrc/gemm_bi.cu).  The invariant
 * arithmetic of an element C[m, n]: acc = 0, then for every 64-deep k-block in k order the four m64nNk16 bf16 wgmma steps
 * (fp32 accumulation, no split-K), then C = bf16(acc) | bf16(bf16(acc) + addend[m, n]) | for SwiGLU
 * h = bf16(bf16(silu(g)) * u) from g = bf16(acc_g), u = bf16(acc_u).  nv_gemm_bf16 computes every element that way with
 * any of its tiles, so a row's bits depend on that row alone.  These kernels give the same bits while streaming the
 * weights over narrow 32-column tiles (64-row activation blocks, rows padded by TMA zero fill), so the decode steps keep
 * weight-streaming rates at every batch size.  X [M,K], W [N,K] (nn.Linear layout), any M.
 * nv_gemm_bi_bf16: the decode step's q|k|v, o_proj (+ residual) and down_proj (+ residual) (LlamaCore.decode_step) and
 *   every inference lm_head (generation.lm_head_rows, the no-grad logits of ModifiedLlamaForCausalLM), each in the mode.
 * nv_gemm_bi_swiglu_bf16: the decode step's gate|up projection with the SwiGLU of HF LlamaMLP fused, Wgu [2F,K], F % 16 == 0. */
int nv_gemm_bi_bf16(const void* X, int64_t ldx, const void* W, int64_t ldw, void* C, int64_t ldc, const void* addend,
                    int64_t ld_add, int M, int N, int K, void* stream);
int nv_gemm_bi_swiglu_bf16(const void* X, int64_t ldx, const void* Wgu, int64_t ldw, void* H, int64_t ldh, int M, int F,
                           int K, void* stream);
/* Opt-in fp8 weight streaming of the same decode-step GEMMs (HF generate through models/modified_lm.py:184-199; no
 * reference counterpart for the number format).  nv_quantize_fp8_rows (csrc/quant.cu) rounds a bf16 weight W [N,K] to
 * e4m3 with one power-of-two scale per row: exps[n] = e_n (int8, the smallest e with max|W[n,:]| / 2^e <= 448, clamped
 * below at -117; 0 for an all-zero row), Q [N,K] = e4m3(W / 2^e_n) (round to nearest even, subnormals kept), and W is
 * overwritten in place with W' = Q * 2^e_n, which bf16 holds exactly.  K % 8 == 0, ldq (bytes) % 16 == 0.
 * nv_gemm_skinny_fp8 / nv_gemm_skinny_swiglu_fp8 are nv_gemm_skinny_bf16 / nv_gemm_skinny_swiglu_bf16 with the weight
 * given as (Q, exps): they stream half the bytes and return bit for bit what the bf16 kernels return on W'.  ldw in bytes. */
int nv_quantize_fp8_rows(void* W, int64_t ldw, void* Q, int64_t ldq, void* exps, int N, int K, void* stream);
int nv_gemm_skinny_fp8(const void* X, int64_t ldx, const void* Wq, int64_t ldw, const void* exps, void* C, int64_t ldc,
                       const void* addend, int64_t ld_add, int M, int N, int K, void* stream);
int nv_gemm_skinny_swiglu_fp8(const void* X, int64_t ldx, const void* Wgu_q, int64_t ldw, const void* exps, void* H,
                              int64_t ldh, int M, int F, int K, void* stream);
/* Opt-in 4-bit group-wise weight streaming (W4A16) of the same decode-step GEMMs (no reference counterpart for the number
 * format; csrc/nv_int4.cuh).  nv_quantize_int4_groups (csrc/quant.cu) rounds a bf16 weight W [N,K], K % 128 == 0, in groups
 * of one row and 128 columns, in fp32 with IEEE division and round-half-even rint: lo = min(0, min w), hi = max(0, max w),
 * s = max(bf16(((hi - lo) / 15)), 2^-126), z = clamp(rint(-lo / s), 0, 15), q = clamp(rint(w / s) + z, 0, 15), and W is
 * overwritten in place with W' = bf16((q - z) * s) (-0 becomes +0; groups with bf16 subnormals follow the rule too).
 * scales [N, K/128] bf16 and zeros [N, K/128] uint8 hold s and z; codes (ceil(N/64) * 64 * K/2 bytes, 16-byte aligned)
 * hold q packed in a layout private to the library.  nv_gemm_skinny_int4 / nv_gemm_skinny_swiglu_int4 are
 * nv_gemm_skinny_bf16 / nv_gemm_skinny_swiglu_bf16 with the weight given as (codes, scales, zeros): they stream a quarter
 * of the bytes and return bit for bit what the bf16 kernels return on W'.  M <= 16, K % 128 == 0. */
int nv_quantize_int4_groups(void* W, int64_t ldw, void* codes, void* scales, void* zeros, int N, int K, void* stream);
/* GPTQ-calibrated form of the same format (Frantar et al., 2022; no act-order, no static groups).  With U the upper
 * Cholesky factor of H^-1 (H = X^T X of the linear's inputs, dampened) the columns are quantized in order and each one's
 * scaled error e_j = (w_j - W'_j) / U_jj is subtracted as e_j U[j, c] from every later column c.  nv_gptq_int4_block runs
 * block g = the 128-column group g: it reads columns 128 g .. 128 g + 127 of the fp32 working copy Wf [N, K] (row stride
 * ldwf) and U_gg, the 128 x 128 diagonal block of U (row stride ldu), applies the rule above to each row's values as they
 * stand (lo, hi, s and z when the block starts, q when the column is reached), and writes the group's codes (same layout),
 * scales and zeros, W' over the group's columns of the bf16 W (row stride ldw) and -E [N, 128] (row stride lde).  The
 * caller then adds -E U[block rows, later columns] to the later columns of Wf (nv_sgemm with accumulate).  Wf is only
 * read.  N % 64 == 0, K % 128 == 0, 0 <= g < K / 128, codes 16-byte aligned; bad arguments return an error before any
 * launch. */
int nv_gptq_int4_block(const void* Wf, int64_t ldwf, const void* U, int64_t ldu, int g, void* W, int64_t ldw, void* codes,
                       void* scales, void* zeros, void* negE, int64_t lde, int N, int K, void* stream);
int nv_gemm_skinny_int4(const void* X, int64_t ldx, const void* codes, const void* scales, const void* zeros, void* C,
                        int64_t ldc, const void* addend, int64_t ld_add, int M, int N, int K, void* stream);
int nv_gemm_skinny_swiglu_int4(const void* X, int64_t ldx, const void* codes, const void* scales, const void* zeros, void* H,
                               int64_t ldh, int M, int F, int K, void* stream);
/* nv_gemm_fp8w_bf16 is nv_gemm_bf16 with K-major operands (a_mn = b_mn = 0) and the weight given as (Wq, exps) in the same
 * format, for the inference GEMMs above 16 rows (prefix-cached navigation suffixes, pruned last layers, decode batches
 * 17..256): C = bf16(bf16(A Wq'^T) + addend) with addend optional, bit for bit nv_gemm_bf16's result on W' at every M, N, K
 * and tile width.  block_n: 0 (auto), 32 or 128.  lda % 8 == 0, ldw (bytes) % 16 == 0. */
int nv_gemm_fp8w_bf16(const void* A, int64_t lda, const void* Wq, int64_t ldw, const void* exps, void* C, int64_t ldc,
                      const void* addend, int64_t ld_add, int M, int N, int K, int block_n, void* stream);
/* nv_gemm_int4w_bf16 is nv_gemm_fp8w_bf16 with the weight given as (codes, scales, zeros) in the 4-bit format above, for
 * the same inference GEMMs above 16 rows (decode batches, beams and samples of 17..64 rows, pruned last layers, small
 * prefix-cached suffixes and prefills; nv_llama_layer_infer and LlamaCore.decode_step): bit for bit nv_gemm_bf16's result
 * on W' at every M, N, K and tile width, reading about a quarter of the weight bytes.  block_n: 0 (auto), 32 or 128.
 * K % 128 == 0, N % 64 == 0, lda % 8 == 0 and lda >= K, ldc (and ld_add) >= N; A, codes, C and addend 16-byte aligned.
 * The codes have no leading dimension: N and K fix their layout. */
int nv_gemm_int4w_bf16(const void* A, int64_t lda, const void* codes, const void* scales, const void* zeros, void* C,
                       int64_t ldc, const void* addend, int64_t ld_add, int M, int N, int K, int block_n, void* stream);
/* Opt-in W8A8 of the no-grad prompt forwards (set_activation_dtype("fp8"); no reference counterpart for the number format;
 * csrc/gemm_fp8.cu).  nv_quantize_act_fp8 quantizes a bf16 activation X [M,K] (row stride ldx) per (row, 128-column block)
 * with the rule of nv_quantize_fp8_rows: Q [M,K] e4m3 bytes (row stride ldq bytes) and E [M, K/128] int8 exponents (row
 * stride lde), so a row's bytes never depend on other rows.  nv_gemm_w8a8_bf16 computes C[M,N] = A'·W'^T (+ addend) on
 * the e4m3 tensor cores: A' = (Aq, Ae) in that format, W' = (Wq, We) in the weight format above; every 128-deep k-block
 * is one e4m3 wgmma chain promoted into an fp32 master with its 2^Ae, in k order, and 2^We and the addend are applied
 * in the epilogue (C = bf16(bf16(acc) + addend)).  An output element's bits do not depend on M or on the other rows.
 * K % 128 == 0 (K <= 34688), ldx % 8, ldq / lda / ldw (bytes) % 16, ldc / ld_add % 8, 16-byte aligned bases. */
int nv_quantize_act_fp8(const void* X, int64_t ldx, void* Q, int64_t ldq, void* E, int64_t lde, int M, int K, void* stream);
int nv_gemm_w8a8_bf16(const void* Aq, int64_t lda, const void* Ae, int64_t lde, const void* Wq, int64_t ldw, const void* We,
                      void* C, int64_t ldc, const void* addend, int64_t ld_add, int M, int N, int K, void* stream);
int nv_gemm_swiglu_bf16(const void* x, int64_t ldx, const void* Wgu, int64_t ldw, void* gu, int64_t ldgu, void* h,
                        int64_t ldh, int M, int F, int K, int keep_gu, void* stream);
int nv_gemm_dswiglu_bf16(const void* dx, int64_t lddx, const void* Wd, int64_t ldw, const void* gu, int64_t ldgu, void* dgu,
                         int64_t lddgu, int M, int F, int D, void* stream);
int nv_gemm_attnd_bf16(const void* dy, int64_t lddy, const void* Wo, int64_t ldw, const void* o, int64_t ldo, void* dout,
                       int64_t lddo, float* dvec, int M, int D, int Dout, void* stream);
int nv_gemm_rope_bf16(const void* x, int64_t ldx, const void* W, int64_t ldw, void* out, int64_t ldo, const int* pos,
                      const void* cos_t, const void* sin_t, int M, int N, int K, int rope_cols, void* stream);
/* Segmented-contraction weight gradient (deferred wgrad of a training rollout, ModifiedLlamaForCausalLM.defer_weight_grads;
 * reference: the wgrad half of loss.backward() at tasks/agents/mp3d_agent.py:750-757, one per step there):
 *   C[M,N] = bf16(bf16(sum_s A_s^T B_s) + addend)      (addend optional; C may alias it)
 * over n_segs row segments given as HOST arrays: A[s] [rows[s], M] with row stride lda[s], B[s] [rows[s], N] with ldb[s].
 * All segments accumulate in one fp32 chain of 64-row k-blocks on the 128 x 256 tile (a segment's last k-block is
 * zero-padded), so C is bit for bit nv_gemm_bf16(a_mn = 1, b_mn = 1) over the row-concatenation of the segments, each
 * zero-padded to a multiple of 64 rows.  1 <= n_segs <= NV_WGRAD_SEG_MAX, rows[s] >= 1, lda[s] >= M and ldb[s] >= N
 * multiples of 8, ldc / ld_add >= N, 16-byte aligned bases; anything else returns NV_ERR_BAD_ARG before touching the
 * device. */
#define NV_WGRAD_SEG_MAX 64
int nv_gemm_wgrad_seg_bf16(const void* const* A, const int64_t* lda, const void* const* B, const int64_t* ldb, const int* rows,
                           int n_segs, void* C, int64_t ldc, const void* addend, int64_t ld_add, int M, int N, void* stream);

/* ---- flash attention on packed rows (csrc/attn_fwd.cu, attn_bwd.cu) ------------------------------------
 * Causal self-attention of HF LlamaAttention (eager softmax(QK^T/sqrt(d)+mask)V; call site
 * models/modified_lm.py:112-116) and its backward (loss.backward(): tasks/agents/mp3d_agent.py:750-757).
 * q,k,v,o,dout,dq,dk,dv: bf16 [T, H*128] column views; lse: fp32 [H,T]; cu_seqlens: int32 [B+1];
 * total_qblocks = sum_b ceil(len_b/128); dvec: fp32 workspace [H*T]. */
int nv_attn_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o, int64_t ldo,
                float* lse, const int* cu_seqlens, int B, int T, int H, int head_dim, int total_qblocks, float scale,
                void* stream);
/* Suffix attention over a KV cache: queries = packed new rows (cu_seqlens), keys/values of sequence b = rows
 * kv_start[b] .. +kv_len[b] of the cache tensors (Tkv rows, zero-initialised); query i of b sees keys <= kv_len[b] -
 * q_len[b] + i.  Same kernel as nv_attn_fwd (which is the kv_len == q_len, kv_start == cu_seqlens case). */
int nv_attn_fwd_kv(const void* q, int64_t ldq, const void* kcache, int64_t ldk, const void* vcache, int64_t ldv, void* o,
                   int64_t ldo, float* lse, const int* cu_seqlens, const int* kv_start, const int* kv_len, int B, int Tq,
                   int Tkv, int H, int head_dim, int total_qblocks, float scale, void* stream);
/* nv_attn_fwd_kv over an fp8 cache in the format of nv_kv_store_prefill_fp8 below (no reference counterpart for the number
 * format): kq / vq e4m3 [Tkv, H*128] with dense rows, kexp / vexp int8 [Tkv, H].  The same kernel with the e4m3 tiles widened
 * to bf16 in shared memory, so the output is bit for bit nv_attn_fwd_kv's on bf16 caches holding K' / V'.  Rows past kv_len
 * must widen to finite values (a zeroed cache or rows the store kernels wrote).  head_dim 128, 16-byte aligned kq / vq. */
int nv_attn_fwd_kv_fp8(const void* q, int64_t ldq, const void* kq, const void* vq, const void* kexp, const void* vexp, void* o,
                       int64_t ldo, float* lse, const int* cu_seqlens, const int* kv_start, const int* kv_len, int B, int Tq,
                       int Tkv, int H, int head_dim, int total_qblocks, float scale, void* stream);
/* nv_attn_fwd_tree[_fp8]: nv_attn_fwd_kv[_fp8] whose Tq = B * q_len query rows are the q_len nodes of one tree per sequence, in
 * DFS preorder (answer scoring: every node of an answer trie over each prompt's cache).  Query i of sequence b sees the
 * kv_len[b] - q_len >= 1 cached keys, and the key of tree row j only when j <= i < tree_end[j]: tree_end (int32 [q_len], device,
 * shared by every sequence) is the first row after node j's subtree, so a query sees its ancestors and itself.  The fp8 form
 * reads the rounded rows K' / V' as nv_attn_fwd_kv_fp8 does. */
int nv_attn_fwd_tree(const void* q, int64_t ldq, const void* kcache, int64_t ldk, const void* vcache, int64_t ldv, void* o,
                     int64_t ldo, float* lse, const int* cu_seqlens, const int* kv_start, const int* kv_len, const int* tree_end,
                     int B, int Tq, int Tkv, int H, int head_dim, int total_qblocks, float scale, void* stream);
int nv_attn_fwd_tree_fp8(const void* q, int64_t ldq, const void* kq, const void* vq, const void* kexp, const void* vexp, void* o,
                         int64_t ldo, float* lse, const int* cu_seqlens, const int* kv_start, const int* kv_len, const int* tree_end,
                         int B, int Tq, int Tkv, int H, int head_dim, int total_qblocks, float scale, void* stream);
int nv_attn_bwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, const void* o,
                int64_t ldo, const void* dout, int64_t lddo, const float* lse, float* dvec, void* dq, int64_t lddq,
                void* dk, int64_t lddk, void* dv, int64_t lddv, const int* cu_seqlens, int B, int T, int H, int head_dim,
                int total_blocks, float scale, const int* rope_pos, const void* cos_t, const void* sin_t, void* stream);
/* Backward of nv_attn_fwd_kv (no reference counterpart: the reference re-encodes every prompt).  q, o, dout, lse, dvec,
 * dq, dk, dv: the Tq packed suffix rows as in nv_attn_bwd; kcache / vcache: bf16 [Tkv, H*128] (leading dimension ldkv),
 * K/V of sequence b at rows kv_start[b] .. +kv_len[b]; acc_k / acc_v: fp32 [Tkv, >= H*128] (ldacc) gradient accumulators
 * over the cache rows.  Key row j of sequence b with c = kv_len[b] - q_len[b]: j < c -> acc[kv_start[b] + j] += (dK, dV);
 * j >= c -> dk / dv at its packed row = bf16(dK + acc_k), bf16(dV + acc_v) (acc only read), dk then rotated back by
 * -theta[rope_pos] when rope_pos is given (as dq).  kv_len == q_len (c = 0) adds the accumulated gradient of cached rows
 * to a recomputed prefix's own.  Deterministic (no atomics).  total_qblocks = sum_b ceil(q_len/128), total_kblocks =
 * sum_b ceil(kv_len/128). */
int nv_attn_bwd_kv(const void* q, int64_t ldq, const void* kcache, const void* vcache, int64_t ldkv, const void* o, int64_t ldo,
                   const void* dout, int64_t lddo, const float* lse, float* dvec, void* dq, int64_t lddq, void* dk, int64_t lddk,
                   void* dv, int64_t lddv, float* acc_k, float* acc_v, int64_t ldacc, const int* cu_seqlens,
                   const int* kv_start, const int* kv_len, int B, int Tq, int Tkv, int H, int head_dim, int total_qblocks,
                   int total_kblocks, float scale, const int* rope_pos, const void* cos_t, const void* sin_t, void* stream);
/* Developer hook (no reference counterpart) for an in-kernel phase trace of the attention kernels.  The sm_90a kernels
 * record none: returns 0 (words copied). */
int nv_debug_attn_trace(int kernel, unsigned long long* out, int max_words);

/* ---- row-wise LM kernels (csrc/lm_ops.cu) ---------------------------------------------------------------
 * LlamaRMSNorm, rotate-half RoPE, SwiGLU (HF LLaMA via models/modified_lm.py:112-116); embedding gather +
 * visual-token scatter-add (models/modified_lm.py:100-110); <cls_1> head (models/nav_model.py:237,445);
 * action-logit scatter (models/nav_model.py:239-242, :446-447); masked token CE (models/modified_lm.py:122-137). */
int nv_rmsnorm_fwd(const void* x, int64_t ldx, const void* w, void* y, int64_t ldy, float* rstd, int T, int D, float eps,
                   void* stream);
int nv_rmsnorm_bwd_partials(void);
int nv_rmsnorm_bwd(const void* x, int64_t ldx, const void* w, const float* rstd, const void* dy, int64_t lddy,
                   const void* dres, int64_t lddres, void* dx, int64_t lddx, void* dw, int accumulate_dw, float* workspace,
                   int T, int D, void* stream);
int nv_rope_inplace(void* qkv, int64_t ld, const int* pos, const void* cos_t, const void* sin_t, int T, int n_heads,
                    int head_dim, int backward, void* stream);
int nv_swiglu_fwd(const void* gu, int64_t ldgu, void* h, int64_t ldh, int T, int F, void* stream);
/* x[rows, cols] (bf16, leading dimension ld, even) *= scale[0] (device fp32 scalar), rounded to bf16: the upstream gradient of
 * the scalar LM loss folded into the stored dlogits (autograd of CrossEntropyLoss, models/modified_lm.py:126-137). */
int nv_scale_bf16(void* x, int64_t ld, int rows, int cols, const float* scale, void* stream);
int nv_swiglu_bwd(const void* gu, int64_t ldgu, const void* dh, int64_t lddh, void* dgu, int64_t lddgu, int T, int F,
                  void* stream);
int nv_embed_fwd(const int* ids, const void* E, int V, const int* vis_src, const float* vis, void* out, int T, int D,
                 void* stream);
int nv_embed_bwd_vis(const void* dx, const int* vis_src, float* dvis, int T, int D, void* stream);
int nv_embed_bwd_weight(const void* dx, const int* order, const int* sorted_ids, void* dE, int T, int D, void* stream);
int nv_gather_rows(const void* src, int64_t lds, const int* rows, void* dst, int64_t ldd, int R, int D, void* stream);
int nv_scatter_rows(const void* src, int64_t lds, const int* rows, void* dst, int64_t ldd, int R, int D, void* stream);
int nv_head_fwd(const void* x, int64_t ldx, const void* W, const void* bias, void* out, int R, int O, int D, void* stream);
int nv_head_bwd(const void* dy, const void* x, int64_t ldx, const void* W, void* dx, int64_t lddx, void* dW, void* db, int R,
                int O, int D, void* stream);
int nv_logit_scatter_fwd(const void* pred, int O, const int* slot, void* out, int B, int G, void* stream);
int nv_logit_scatter_bwd(const void* dout, const int* slot, void* dpred, int O, int B, int G, void* stream);
int nv_ce_fwd_bwd(const void* logits, int64_t ld, const int* labels, const int* special, int n_special, float* row_loss,
                  void* dlogits, int64_t ldd, int N, int V, float grad_scale, void* stream);

/* ---- fp32 panorama encoder / fusion kernels (csrc/pano_ops.cu) --------------------------------------------
 * nn.Linear / LayerNorm / GELU / nn.MultiheadAttention(key_padding_mask) of ImageEmbeddings and the DETR
 * pre-LN encoder (models/image_embedding.py:51-121, models/detr_transformer.py:170-182), and the gather /
 * scatter glue of NavModel.forward_navigation (models/nav_model.py:146-224), forward and backward. */
int nv_sgemm(const float* A, int64_t lda, int ta, const float* B, int64_t ldb, int tb, float* C, int64_t ldc,
             const float* bias, int M, int N, int K, int accumulate, void* stream);
/* Same contract on the tensor cores (wgmma tf32, fp32 accumulate; csrc/gemm_tf32.cu): the numerical mode the
 * reference's pinned torch 1.10 (allow_tf32 = True by default, requirements.txt:19) used for these fp32 nn.Linear
 * layers.  Needs 16-byte aligned bases and lda/ldb % 4 == 0; other shapes go to nv_sgemm. */
int nv_gemm_tf32(const float* A, int64_t lda, int ta, const float* B, int64_t ldb, int tb, float* C, int64_t ldc,
                 const float* bias, int M, int N, int K, int accumulate, void* stream);
int nv_layernorm_fwd(const float* x, int64_t ldx, const float* gamma, const float* beta, const float* addend, int64_t ldadd,
                     float* y, int64_t ldy, float* mean, float* rstd, int R, int D, float eps, void* stream);
int nv_layernorm_bwd_partials(void);
int nv_layernorm_bwd(const float* x, int64_t ldx, const float* gamma, const float* mean, const float* rstd, const float* dy,
                     int64_t lddy, float* dx, int64_t lddx, int accumulate_dx, float* dgamma, float* dbeta, float* workspace,
                     int R, int D, void* stream);
int nv_colsum_f32(const float* src, int64_t ld, int R, int D, float* dst, int accumulate, void* stream);
int nv_gelu_fwd(const float* z, float* a, int64_t n, void* stream);
int nv_gelu_bwd(const float* z, const float* da, float* dz, int64_t n, void* stream);
int nv_mha_fwd(const float* qkv, const int* lens, float* out, float* P, int B, int N, int H, int hd, void* stream);
int nv_mha_bwd(const float* qkv, const float* dout, const float* P, float* dS, float* dqkv, const int* lens, int B, int N,
               int H, int hd, void* stream);
/* Train-mode dropout of the panorama encoder (nn.Dropout(hidden_dropout_prob), models/image_embedding.py:41,72;
 * dropout / dropout1 / dropout2 and nn.MultiheadAttention(dropout=...), models/detr_transformer.py:136-146,170-182).
 * Counter-based RNG: element i is kept iff hash(seed, i) >= p * 2^32, so applying nv_dropout with the same seed to the
 * upstream gradient is the backward.  nv_mha_*_dropout: Pd [B,H,N,N] = dropped attention probabilities. */
int nv_dropout(const float* x, float* out, int64_t n, float p_drop, unsigned long long seed, void* stream);
int nv_mha_fwd_dropout(const float* qkv, const int* lens, float* out, float* P, float* Pd, int B, int N, int H, int hd,
                       float p_drop, unsigned long long seed, void* stream);
int nv_mha_bwd_dropout(const float* qkv, const float* dout, const float* P, const float* Pd, float* dS, float* dqkv,
                       const int* lens, int B, int N, int H, int hd, void* stream);
int nv_rows_combine(float* out, int64_t ldo, const float* A, int64_t lda, const int* ia, float alpha, const float* Bm,
                    int64_t ldb, const int* ib, float beta, int R, int D, int accumulate, void* stream);
int nv_rows_scatter_add(float* dst, int64_t ldd, const int* idx, const float* src, int64_t lds, float alpha, int R, int D,
                        void* stream);

/* ---- decode phase (csrc/decode.cu) --------------------------------------------------------------------------
 * Pre-allocated contiguous KV cache ([B, Smax, H*128] bf16 per layer for K and V) + single-query attention +
 * masked greedy argmax: replaces HF GenerationMixin's per-token torch.cat cache growth and eager attention
 * (models/nav_model.py:324-338,388-399; models/modified_lm.py:184-199).  `lens` lives on the device so one decode
 * step has static launch parameters (CUDA-graph replayable). */
int nv_kv_store_prefill(const void* qkv, int64_t ld, const int* cu_seqlens, void* kcache, void* vcache, int B, int T,
                        int Smax, int HD, void* stream);
int nv_kv_append(const void* qkv, int64_t ld, const int* lens, void* kcache, void* vcache, int B, int Smax, int HD,
                 void* stream);
/* decode step: rotary embedding of the new token's q,k (in place, position = lens[b]) + append of K (rotated) and V */
int nv_decode_rope_kv(void* qkv, int64_t ld, const int* lens, const void* cos_t, const void* sin_t, void* kcache, void* vcache,
                      int B, int Smax, int H, int head_dim, void* stream);
/* Cross-step prefix-KV reuse in rollouts (SURVEY.md §8f n1; caller tasks/agents/mp3d_agent.py:660-726, prompt order
 * tasks/agents/r2r.py:16-31): store the K/V of the NEW rows of each sequence after the cached[b] rows the cache already
 * holds, then attend from the new rows over cached + new keys (nv_attn_fwd_kv). */
int nv_kv_store_suffix(const void* qkv, int64_t ld, const int* cu_seqlens, const int* cached, void* kcache, void* vcache,
                       int B, int T, int Smax, int HD, void* stream);
/* nv_kv_store_suffix into an fp8 cache (format: nv_kv_store_prefill_fp8 below): every stored (token, head) row is quantized,
 * the bytes and exponents nv_quantize_fp8_rows gives for that row.  Rows at p >= Smax are dropped. */
int nv_kv_store_suffix_fp8(const void* qkv, int64_t ld, const int* cu_seqlens, const int* cached, void* kq, void* vq, void* kexp,
                           void* vexp, int B, int T, int Smax, int H, void* stream);
int nv_decode_attn(const void* q, int64_t ldq, const void* kcache, const void* vcache, const int* lens, void* out,
                   int64_t ldo, int B, int Smax, int H, int head_dim, float scale, void* stream);
/* nv_decode_rope_kv + nv_decode_attn in one launch (qkv pre-RoPE, not modified; k / v appended at row lens[b]). */
int nv_decode_attn_rope(const void* qkv, int64_t ld, const int* lens, const void* cos_t, const void* sin_t, void* kcache,
                        void* vcache, void* out, int64_t ldo, int B, int Smax, int H, int head_dim, float scale, void* stream);
/* Opt-in fp8 (e4m3) KV cache of generate()'s decode step (no reference counterpart for the number format).  Per layer,
 * kq / vq [B, Smax, H*128] e4m3 bytes and kexp / vexp [B, Smax, H] int8: every cached (sequence b, position p, head h) row of
 * 128 elements is stored in the weight format of nv_quantize_fp8_rows above,
 *     K'[b,p,h,:] = e4m3(K[b,p,h,:] / 2^e) * 2^e,   e = kexp[b,p,h] = the row exponent of max|K[b,p,h,:]|   (V' alike),
 * i.e. exactly the bytes and exponents nv_quantize_fp8_rows produces on a [B*Smax*H, 128] view of the bf16 cache (amax on the
 * bf16 bit patterns, round to nearest even, saturating).  Half the bytes of the bf16 cache plus 1/256 for the exponents.
 * nv_kv_store_prefill_fp8 is nv_kv_store_prefill (same packing, rows at p >= Smax dropped) into that cache.
 * nv_decode_attn_rope_fp8 is nv_decode_attn_rope over it: the rotated k and the v of the new token are quantized as they are
 * appended at row lens[b], and the attention returns bit for bit what nv_decode_attn_rope returns on a bf16 cache holding
 * K' / V' (scores and P.V in fp32).  head_dim 128, ld % 8 == 0, 16-byte aligned qkv, 8-byte aligned kq / vq. */
int nv_kv_store_prefill_fp8(const void* qkv, int64_t ld, const int* cu_seqlens, void* kq, void* vq, void* kexp, void* vexp, int B,
                            int T, int Smax, int H, void* stream);
int nv_decode_attn_rope_fp8(const void* qkv, int64_t ld, const int* lens, const void* cos_t, const void* sin_t, void* kq, void* vq,
                            void* kexp, void* vexp, void* out, int64_t ldo, int B, int Smax, int H, int head_dim, float scale,
                            void* stream);
/* Beam search (HF beam_search / BeamSearchScorer of transformers 4.28, the version the reference pins), K = 1..8 beams per
 * prompt, R = B * K beam rows, all state on the device so a whole step can be captured.
 * nv_beam_topk: one CTA per prompt b.  Beam k's scores are bf16(log_softmax(logits[b * ld_prompt + k * ld_beam, :])) (special
 * ids -inf, fp32 result rounded once to bf16) + beam_score[b * K + k] in fp32; the 2K best of the K * V scores by (score desc,
 * flat index k * V + c asc) are written in that order to cand_score / cand_tok / cand_parent [B, 2K] (parent = k).
 * nv_beam_select: one CTA per prompt, BeamSearchScorer.process over those candidates (EOS of rank < K -> hypothesis with
 * score sum_logprobs / norm[t] in fp64, norm[t] = (S + t) ** length_penalty for S padded prompt columns and t generated tokens;
 * EOS of rank >= K skipped, the others -> the K running beams; the done rule of BeamHypotheses.is_done), then gathers hist / src [R, G] (generated tokens, KV source rows) by parent and writes
 * next_ids / lens / beam_score [R] and src[r, t] = r.  hyp_score fp64 [B, K + 1] (K kept scores, worst kept score; start
 * 1e9), hyp_meta [B, K, 2] (generated length, insertion number), hyp_tok [B, K, G], prompt_state [B, 5] (tokens generated t,
 * prompt length, hypotheses kept, next insertion number, done).  A done prompt's beams emit pad_id with score 0.
 * nv_decode_attn_rope_beam[_fp8]: nv_decode_attn_rope[_fp8] for beam rows r: keys [0, plens[r / K]) from the prompt cache
 * pk / pv [B, Sp, H*128] the beams of a prompt share, generated key i from row (src[r, i], i) of kgen / vgen [R, G, H*128];
 * the new k / v go to (r, lens[r] - plens[r / K]).  Same keys in the same order as the contiguous kernel: same bits. */
int nv_beam_topk(const void* logits, int64_t ld_prompt, int64_t ld_beam, int V, const int* special, int n_special,
                 const float* beam_score, float* cand_score, int* cand_tok, int* cand_parent, int B, int K, void* stream);
/* HF logits processors of transformers 4.28 (the reference's pin), in its _get_logits_processor order, as generate() reaches them
 * through models/nav_model.py:388-396 -> lang_model.generate(**kwargs) (repetition_penalty, no_repeat_ngram_size, min_length,
 * min_new_tokens).  A row's history is HF's input_ids: its S padded prompt columns (left pads included; S read from the device
 * int *prompt_width) followed by its t generated tokens.  RepetitionPenaltyLogitsProcessor: every distinct history id once,
 * s < 0 -> bf16(s * penalty), else bf16(s / penalty) (IEEE division); NoRepeatNGramLogitsProcessor (ngram = n > 0): every
 * token that completes an n-gram of the history whose first n - 1 tokens equal its last n - 1 -> -inf (nothing while
 * S + t + 1 < n); MinLength / MinNewTokensLength: eos_id -> -inf while S + t < min_length or t < min_new_tokens.  Off:
 * penalty 1, ngram 0, min_length 0, min_new_tokens 0.  V must fit two V-bit bitmaps in 48 KB (three for nv_beam_topk_trie).
 * nv_logits_process: in place on the bf16 logits [R, ld] of the greedy / sampled decode rows, between the lm_head and the trie
 * mask or the pick.  Row r reads prompt_ids[(r / rows_per_prompt) * ld_prompt ...] and hist[r, 0 .. hist_len[r]) ([R, G]); with
 * append non-null, append[r] is first stored at hist[r, hist_len[r]] and hist_len[r] incremented, so a captured step keeps
 * the history itself.  One CTA per row; PDL like the rest of the decode chain.
 * nv_beam_topk_processed: nv_beam_topk with the processors applied to each bf16 log-prob before the fp32 beam-score add (4.28
 * beam_search); beam k of prompt b has the history prompt_ids[b * ld_ids ...] ++ hist[b * K + k, 0 .. t) with
 * t = prompt_state[b, 0], the state nv_beam_select keeps. */
int nv_logits_process(void* logits, int64_t ld, int V, const int* prompt_ids, int64_t ld_prompt, const int* prompt_width,
                      int rows_per_prompt, int* hist, int G, int* hist_len, const int* append, float penalty, int ngram,
                      int min_length, int min_new_tokens, int eos_id, int R, void* stream);
int nv_beam_topk_processed(const void* logits, int64_t ld_prompt, int64_t ld_beam, int V, const int* special, int n_special,
                           const float* beam_score, float* cand_score, int* cand_tok, int* cand_parent, const int* prompt_ids,
                           int64_t ld_ids, const int* prompt_width, const int* hist, int G, const int* prompt_state, float penalty,
                           int ngram, int min_length, int min_new_tokens, int eos_id, int B, int K, void* stream);
/* nv_beam_topk_trie: nv_beam_topk_processed followed by 4.28's PrefixConstrainedLogitsProcessor walking a trie: after the
 * processors, every log-prob of beam k of prompt b outside the allowed set becomes -inf (allowed ones keep their value).  The
 * beam's node is found by walking its generated tokens hist[b * K + k, 0 .. t), t = prompt_state[b, 0], from the root with
 * the rule of nv_trie_mask (a node without children stays; a token that is not a child of a node with children leads to the
 * childless dead node n_nodes); the allowed set is the node's children, or leaf_tok at a childless node.  The trie is the CSR
 * table of nv_trie_mask (node_ptr [n_nodes + 2], child_tok / child_node [E], children ascending).  At the first step
 * (ld_beam = 0, t = 0) every beam is at the root.  The processors' off values (penalty 1, ngram 0, min_length 0,
 * min_new_tokens 0) give trie-only beams.  V must fit three V-bit bitmaps in 48 KB. */
int nv_beam_topk_trie(const void* logits, int64_t ld_prompt, int64_t ld_beam, int V, const int* special, int n_special,
                      const float* beam_score, float* cand_score, int* cand_tok, int* cand_parent, const int* prompt_ids,
                      int64_t ld_ids, const int* prompt_width, const int* hist, int G, const int* prompt_state, float penalty,
                      int ngram, int min_length, int min_new_tokens, int eos_id, const int* node_ptr, const int* child_tok,
                      const int* child_node, int n_nodes, int leaf_tok, int B, int K, void* stream);
/* nv_trie_score: the log-probability of every answer of a trie under each prompt.  logits bf16 [B * R, ld], R = 1 + N': row
 * b * R holds prompt b's next-token logits after its prompt, row b * R + 1 + j those after tree node j (DFS preorder).  The
 * log-prob of token c at a row is nv_beam_topk's: special ids -inf, fp32 max, fp64 sum, (x - m) - ls rounded once to bf16,
 * NaN -> -inf.  Answer a walks tree rows path_rows[path_off[a] .. path_off[a + 1]) from the root (tokens tok[row]), then EOS:
 * logprob[b, a] (fp32 [B, A]) is the fp32 left fold s = lp(row 0, t_1) + 0, s = lp(row of t_1, t_2) + s, ..., s = lp(row of
 * t_d, eos) + s.  stats (fp32 [B * R, 2]) is scratch for each row's max and log-sum.  tok and path_rows may be null when
 * R = 1 (a root without children: one empty answer).  Two kernels under PDL. */
int nv_trie_score(const void* logits, int64_t ld, int V, const int* special, int n_special, const int* tok, const int* path_off,
                  const int* path_rows, int eos, float* stats, float* logprob, int B, int R, int A, void* stream);
int nv_beam_select(const float* cand_score, const int* cand_tok, const int* cand_parent, float* beam_score, int* hist, int* src,
                   double* hyp_score, int* hyp_meta, int* hyp_tok, int* prompt_state, int* next_ids, int* lens, const double* norm,
                   int B, int K, int G, int eos_id, int pad_id, int early_stopping, void* stream);
int nv_decode_attn_rope_beam(const void* qkv, int64_t ld, const int* lens, const void* cos_t, const void* sin_t, const void* pk,
                             const void* pv, int Sp, const int* plens, void* kgen, void* vgen, const int* src, int G, void* out,
                             int64_t ldo, int R, int K, int H, int head_dim, float scale, void* stream);
int nv_decode_attn_rope_beam_fp8(const void* qkv, int64_t ld, const int* lens, const void* cos_t, const void* sin_t, const void* pkq,
                                 const void* pvq, const void* pkexp, const void* pvexp, int Sp, const int* plens, void* kq, void* vq,
                                 void* kexp, void* vexp, const int* src, int G, void* out, int64_t ldo, int R, int K, int H,
                                 int head_dim, float scale, void* stream);
/* Contrastive search = transformers 4.28 GenerationMixin.contrastive_search / _ranking_fast as generate(penalty_alpha > 0,
 * top_k > 1) reaches it through models/nav_model.py:388-396 -> lang_model.generate(**kwargs), for a model that returns HF's
 * hidden-state tuple (the reference's ModifiedLM returns one tensor, models/modified_lm.py:119,144).  K = top_k = 1..64
 * candidates per prompt, run as decode rows b * K + j; x^ = bf16(x / bf16(||x||)) of a final-norm hidden row.
 * nv_contrastive_topk: one CTA per prompt, p = bf16(softmax(logits)) (special ids -inf; computed in fp64 and rounded once, where
 * torch's bf16 softmax rounds an fp32 value: they can differ by one ulp next to a rounding midpoint) and the K largest p by
 * (p desc, token id asc) -> p [B, K] bf16, tok [B, K] int32.  V <= 51200.
 * nv_contrastive_context: ctx[b, i] = x^ of the packed final-norm prompt row hn[cu_seqlens[b] + i] ([T, D]), ctx_len[b] = its
 * length; ctx [B, Sc, D] bf16 is prompt b's context (left pads are not part of it).
 * nv_contrastive_rank: pen_j = max over the ctx_len[b] context rows of bf16(c^_i . h^_j) for the candidates' final-norm rows hn
 * [B * K, D], score_j = bf16(bf16(fp32(1 - alpha) p_j) - bf16(fp32(alpha) pen_j)), sel[b] = the first best j; next[b] = its
 * token, or pad_id once finished[b] (EOS sets finished[b] when stop_on_eos); x^ of its row is appended to ctx, the row itself
 * copied to hsel [B, D], plens[b] and lens[b * K .. b * K + K) advance by one.  pen_key uint32 [B * K] is zero before the call
 * and after it.  pen_out / score_out: optional fp32 [B, K].  Two launches: the context rows are split over 16 CTAs per prompt.
 * nv_contrastive_commit: per layer l, the K and V rows of candidate b * K + sel[b] in its one-slot cache ([B * K, 1, D]) go to
 * row plens[b] - 1 of prompt b's cache ([B, Sp, D]); table [L, 8] holds the layer's kc, vc, pk, pv pointers and, with fp8,
 * the four exponent arrays ([.., H] int8; the rows then hold D e4m3 bytes).  A byte copy: the bits are the candidate's. */
int nv_contrastive_topk(const void* logits, int64_t ld, int V, const int* special, int n_special, int K, void* p, int* tok, int B,
                        void* stream);
int nv_contrastive_context(const void* hn, const int* cu_seqlens, int B, int T, void* ctx, int* ctx_len, int Sc, int D, void* stream);
int nv_contrastive_rank(const void* hn, void* ctx, int* ctx_len, int Sc, int D, int K, unsigned* pen_key, const void* p,
                        const int* tok, double alpha, int* finished, int eos_id, int pad_id, int stop_on_eos, int* next, int* sel,
                        void* hsel, int* plens, int* lens, float* pen_out, float* score_out, int B, void* stream);
int nv_contrastive_commit(const unsigned long long* table, int L, const int* sel, const int* plens, int K, int Sp, int D, int H,
                          int fp8, int B, void* stream);
/* Prompt-lookup speculative decoding (greedy generate(prompt_lookup_num_tokens=K), K = 1..15, window W = K + 1 rows per prompt).
 * nv_decode_attn_rope_window[_fp8]: nv_decode_attn_rope[_fp8] for W consecutive new tokens per sequence, qkv row b * W + r
 * (pre-RoPE) at position lens[b] + r: the rotated k and the v of every row are stored (fp8: quantized) at rows lens[b] .. lens[b]
 * + W - 1, and query r attends over keys 0 .. lens[b] + r.  Query r's output and every cache byte equal those of W sequential
 * nv_decode_attn_rope[_fp8] calls at lens[b] + r.  A cached key is read once per 8 queries.  1 <= W <= 16; sizes and alignment as
 * nv_decode_attn_rope[_fp8], ldo % 8 == 0.
 * nv_lookup_draft: one CTA per row, HF's PromptLookupCandidateGenerator (max_matching_ngram_size = ngram) on the row's history
 * hist[b, 0 .. hist_len[b]) (int32, row stride ld_hist): the earliest earlier occurrence of its last n tokens, n = ngram down to
 * 1, proposes the up to K tokens after it, cut at the history's end and at the first special id or eos_id.  drafts [B, K] (-1
 * past the drafts) and win_ids [B, W] (the history's last token, the drafts, the last token again for a missing draft); a
 * finished row gets none.
 * nv_lookup_accept: one CTA per row; t_j = nv_argmax_masked's pick of logits row b * W + j, taken while drafts[b, j - 1] = t_{j-1}.
 * The row emits t_0 .. t_m (m accepted drafts), cut after EOS (stop_on_eos) and at max_new tokens, into out[b, n_out[b] ..]
 * (row stride ld_out >= max_new) and hist[b, hist_len[b] ..]; n_out, hist_len and lens[b] advance by the tokens emitted, n_acc by
 * the accepted drafts among them.  A row that emitted EOS or max_new tokens is finished and emits nothing more. */
int nv_decode_attn_rope_window(const void* qkv, int64_t ld, const int* lens, const void* cos_t, const void* sin_t, void* kcache,
                               void* vcache, void* out, int64_t ldo, int B, int W, int Smax, int H, int head_dim, float scale,
                               void* stream);
int nv_decode_attn_rope_window_fp8(const void* qkv, int64_t ld, const int* lens, const void* cos_t, const void* sin_t, void* kq,
                                   void* vq, void* kexp, void* vexp, void* out, int64_t ldo, int B, int W, int Smax, int H,
                                   int head_dim, float scale, void* stream);
int nv_lookup_draft(const int* hist, int ld_hist, const int* hist_len, const int* finished, const int* special, int n_special,
                    int eos_id, int K, int ngram, int* drafts, int* win_ids, int B, void* stream);
int nv_lookup_accept(const void* logits, int64_t ld, int V, const int* special, int n_special, const int* drafts, int K, int* finished,
                     int eos_id, int stop_on_eos, int max_new, int* out, int ld_out, int* hist, int ld_hist, int* hist_len, int* n_out,
                     int* lens, int* n_acc, int B, void* stream);
/* at most 64 special ids (n_special), here and in nv_sample_topk; longer lists return NV_ERR_BAD_ARG */
int nv_argmax_masked(const void* logits, int64_t ld, int V, const int* special, int n_special, int* finished, int eos_id,
                     int pad_id, int stop_on_eos, int* next, int B, void* stream);
int nv_add_int(int* x, int n, int delta, void* stream);
/* Sampled next token = HF GenerationMixin.sample as reached with do_sample=True (tasks/agents/llava.py:58-62 ->
 * models/nav_model.py:388-396): scores / temperature (bf16) -> top-k (transformers' generation default 50; ties at the k-th
 * value stay; top_k <= 0: off) -> softmax (bf16 output) -> inverse-CDF draw at u[b] in [0,1).  Special tokens masked,
 * finished / eos / pad handling as nv_argmax_masked.  probs_out: optional fp32 [B, V] copy of the distribution drawn from. */
int nv_sample_topk(const void* logits, int64_t ld, int V, const int* special, int n_special, int* finished, int eos_id, int pad_id,
                   int stop_on_eos, float temperature, int top_k, const float* u, int* next, float* probs_out, int B, void* stream);
/* nv_sample_topk with HF's TopPLogitsWarper between top-k and the softmax: the top-k survivors sorted by (score, token index)
 * ascending, their bf16 probabilities summed in that order (fp32, each partial rounded to bf16), and every position whose sum
 * is <= bf16(1 - top_p) removed, the largest always kept; then a fresh softmax over the rest.  top_p in [0, 1] (else
 * NV_ERR_BAD_ARG); top_p = 1 is nv_sample_topk, bit for bit.  Above 1024 survivors (top_k = 0) the sum is the exact prefix
 * sum rounded to bf16 instead (see csrc/decode.cu). */
int nv_sample(const void* logits, int64_t ld, int V, const int* special, int n_special, int* finished, int eos_id, int pad_id,
              int stop_on_eos, float temperature, int top_k, float top_p, const float* u, int* next, float* probs_out, int B,
              void* stream);
/* Trie-constrained decoding (TrieLogitsProcessor, models/modified_lm.py:10-30, reached from EQA validation,
 * tasks/agents/mp3d_agent.py:545-584), on the device.  The trie is flattened to CSR: node_ptr [n_nodes + 2], child_tok [E]
 * (ascending within a node, every id in [0, V)), child_node [E]; node 0 is the root, node n_nodes an extra childless dead node.
 * One CTA per row b: when last != NULL, state[b] advances by last[b] like tools/trie.py's get_next_node (a node without
 * children stays; a token that is not a child sets *miss = 1 and moves to the dead node).  Then out[b, 0:V) = -inf except
 * the allowed tokens - the node's children, or leaf_tok (the trie's eos) at a node without any - which carry their logit.
 * A row whose allowed non-special values are all -inf, or with an allowed NaN, sets *miss = 1 and gets 0.0 at its first
 * allowed non-special token (or its first non-special column), so a pick from out stays inside [0, V).  *miss is never
 * cleared here.  nv_argmax_masked / nv_sample_topk then pick from out.  ldo % 8 == 0, out 16-byte aligned,
 * n_special <= 64; launched with PDL like the rest of the decode chain. */
int nv_trie_mask(const void* logits, int64_t ld, void* out, int64_t ldo, int V, const int* node_ptr, const int* child_tok,
                 const int* child_node, int n_nodes, int leaf_tok, const int* special, int n_special, int* state, const int* last,
                 int* miss, int B, void* stream);
/* Per-step scores of generate(return_dict_in_generate=True, output_scores=True): HF GenerationMixin's `scores` (transformers
 * 4.28, the reference's pin; models/nav_model.py:388-399 reaches generate()).  The scores live in bf16 planes [G, rows,
 * ld_scores] (plane >= rows * ld_scores elements apart); a launch writes the plane its step pointer names on the device, so a
 * captured step writes a new plane at every replay.  Each entry below is the base entry's computation, unchanged, plus that
 * output; the base entries launch what they launched before.
 * nv_scores_store: rows r < R of src (ld) to plane step[0], row r, with the special ids -inf (greedy / trie / contrastive: the
 * values nv_argmax_masked, nv_trie_mask's output or nv_contrastive_topk read, as the reference's logits carry the mask).
 * nv_sample_scores: nv_sample, and row b of plane step[0] gets its warped scores: bf16(logit / T), -inf for the special ids and
 * outside the top-k / top-p set (4.28 next_token_scores after logits_warper).
 * nv_lookup_scores: after nv_lookup_accept, window row j of prompt b (logits row b * W + j) goes to plane n_prev[b] + j, row b,
 * for every j < n_out[b] - n_prev[b] (the tokens that step emitted), special ids -inf.
 * nv_beam_topk[_processed|_trie]_scores: beam k of prompt b writes its processed bf16 log-probs before the beam-score add
 * (4.28 next_token_scores_processed; special ids -inf) to plane prompt_state[b, 0], row b * K + k.
 * nv_beam_select_scores: nv_beam_select keeping 4.28's beam_indices: par_hist int32 [R, G] (each running beam's rows b * K +
 * parent so far) is gathered by parent like hist and gets this step's parent row at t; a hypothesis added at step t stores its
 * parent's rows and then that parent's row in hyp_par [B, K, G] (t + 1 entries); done_step[b] = t + 1 at the step prompt b
 * becomes done (the host zeroes it). */
int nv_scores_store(const void* src, int64_t ld, int V, const int* special, int n_special, void* scores, int64_t ld_scores,
                    int64_t plane, const int* step, int R, void* stream);
int nv_sample_scores(const void* logits, int64_t ld, int V, const int* special, int n_special, int* finished, int eos_id, int pad_id,
                     int stop_on_eos, float temperature, int top_k, float top_p, const float* u, int* next, float* probs_out,
                     void* scores, int64_t ld_scores, int64_t plane, const int* step, int B, void* stream);
int nv_lookup_scores(const void* logits, int64_t ld, int V, const int* special, int n_special, const int* n_prev, const int* n_out,
                     int W, void* scores, int64_t ld_scores, int64_t plane, int B, void* stream);
int nv_beam_topk_scores(const void* logits, int64_t ld_prompt, int64_t ld_beam, int V, const int* special, int n_special,
                        const float* beam_score, float* cand_score, int* cand_tok, int* cand_parent, const int* prompt_state,
                        void* scores, int64_t ld_scores, int64_t plane, int B, int K, void* stream);
int nv_beam_topk_processed_scores(const void* logits, int64_t ld_prompt, int64_t ld_beam, int V, const int* special, int n_special,
                                  const float* beam_score, float* cand_score, int* cand_tok, int* cand_parent, const int* prompt_ids,
                                  int64_t ld_ids, const int* prompt_width, const int* hist, int G, const int* prompt_state,
                                  float penalty, int ngram, int min_length, int min_new_tokens, int eos_id, void* scores,
                                  int64_t ld_scores, int64_t plane, int B, int K, void* stream);
int nv_beam_topk_trie_scores(const void* logits, int64_t ld_prompt, int64_t ld_beam, int V, const int* special, int n_special,
                             const float* beam_score, float* cand_score, int* cand_tok, int* cand_parent, const int* prompt_ids,
                             int64_t ld_ids, const int* prompt_width, const int* hist, int G, const int* prompt_state, float penalty,
                             int ngram, int min_length, int min_new_tokens, int eos_id, const int* node_ptr, const int* child_tok,
                             const int* child_node, int n_nodes, int leaf_tok, void* scores, int64_t ld_scores, int64_t plane, int B,
                             int K, void* stream);
int nv_beam_select_scores(const float* cand_score, const int* cand_tok, const int* cand_parent, float* beam_score, int* hist, int* src,
                          double* hyp_score, int* hyp_meta, int* hyp_tok, int* prompt_state, int* next_ids, int* lens,
                          const double* norm, int* par_hist, int* hyp_par, int* done_step, int B, int K, int G, int eos_id, int pad_id,
                          int early_stopping, void* stream);
/* Diverse (group) beam search: transformers 4.28's group_beam_search with num_beam_groups = n_groups and the
 * HammingDiversityLogitsProcessor.  The K beams of a prompt form n_groups groups of Kg = K / n_groups (K in 2..8, n_groups
 * dividing K); a step runs, for group = 0 .. n_groups - 1 in order, one top-k and one select launch.
 * nv_beam_topk_group[_processed][_scores]: nv_beam_topk[_processed][_scores] over beams group * Kg + [0, Kg) of each prompt
 * only, writing that group's 2Kg best to cand_* [B, 2Kg] (parents local to the group).  Before the processors, each bf16
 * log-prob of token c is lowered to bf16(lp - diversity_penalty * freq[c]) in fp32, freq[c] counting c among next_ids[b * K +
 * 0 .. group * Kg) (the earlier groups' tokens of this step, which their selects have written).  diversity_penalty > 0.
 * nv_beam_select_group[_scores]: nv_beam_select[_scores] over those candidates with group_size Kg against the prompt's one set
 * of K hypotheses; it reorders and writes only the group's rows (parents and beam_indices as global rows b * K + k), pads a
 * prompt that is already done (an earlier group of this step included), and only the last group advances prompt_state[b, 0]. */
int nv_beam_topk_group(const void* logits, int64_t ld_prompt, int64_t ld_beam, int V, const int* special, int n_special,
                       const float* beam_score, float* cand_score, int* cand_tok, int* cand_parent, const int* next_ids,
                       float diversity_penalty, int group, int n_groups, int B, int K, void* stream);
int nv_beam_topk_group_scores(const void* logits, int64_t ld_prompt, int64_t ld_beam, int V, const int* special, int n_special,
                              const float* beam_score, float* cand_score, int* cand_tok, int* cand_parent, const int* prompt_state,
                              void* scores, int64_t ld_scores, int64_t plane, const int* next_ids, float diversity_penalty, int group,
                              int n_groups, int B, int K, void* stream);
int nv_beam_topk_group_processed(const void* logits, int64_t ld_prompt, int64_t ld_beam, int V, const int* special, int n_special,
                                 const float* beam_score, float* cand_score, int* cand_tok, int* cand_parent, const int* prompt_ids,
                                 int64_t ld_ids, const int* prompt_width, const int* hist, int G, const int* prompt_state,
                                 float penalty, int ngram, int min_length, int min_new_tokens, int eos_id, const int* next_ids,
                                 float diversity_penalty, int group, int n_groups, int B, int K, void* stream);
int nv_beam_topk_group_processed_scores(const void* logits, int64_t ld_prompt, int64_t ld_beam, int V, const int* special,
                                        int n_special, const float* beam_score, float* cand_score, int* cand_tok, int* cand_parent,
                                        const int* prompt_ids, int64_t ld_ids, const int* prompt_width, const int* hist, int G,
                                        const int* prompt_state, float penalty, int ngram, int min_length, int min_new_tokens,
                                        int eos_id, void* scores, int64_t ld_scores, int64_t plane, const int* next_ids,
                                        float diversity_penalty, int group, int n_groups, int B, int K, void* stream);
int nv_beam_select_group(const float* cand_score, const int* cand_tok, const int* cand_parent, float* beam_score, int* hist, int* src,
                         double* hyp_score, int* hyp_meta, int* hyp_tok, int* prompt_state, int* next_ids, int* lens,
                         const double* norm, int group, int n_groups, int B, int K, int G, int eos_id, int pad_id, int early_stopping,
                         void* stream);
int nv_beam_select_group_scores(const float* cand_score, const int* cand_tok, const int* cand_parent, float* beam_score, int* hist,
                                int* src, double* hyp_score, int* hyp_meta, int* hyp_tok, int* prompt_state, int* next_ids, int* lens,
                                const double* norm, int* par_hist, int* hyp_par, int* done_step, int group, int n_groups, int B, int K,
                                int G, int eos_id, int pad_id, int early_stopping, void* stream);

/* ---- fused clip + AdamW over flat buffers (csrc/optim.cu) ------------------------------------------------------
 * torch.nn.utils.clip_grad_norm_(model.parameters(), 40.) + torch.optim.AdamW.step() of the reference
 * (train.py:86-89, tools/optims.py:43) as sum-of-squares partials -> device-side clip coefficient -> one update
 * pass per flat buffer.  clip_state: fp32 [2] = {grad norm, clip coefficient}. */
int nv_optim_partials(void);
int nv_grad_sumsq(const void* g, int64_t n, int is_bf16, float* partial, void* stream);
int nv_clip_coef(const float* partial, int n_partial, float max_norm, float* state, void* stream);
int nv_adamw_flat(void* p, void* g, void* m, void* v, int64_t n, int is_bf16, float lr, float beta1, float beta2, float eps,
                  float weight_decay, int step, const float* clip_state, int write_clipped_grad, void* stream);
/* Opt-in error-compensated form of the same optimizer.step() (tools/optims.py:43) for bf16 buffers: r is a bf16 residual
 * beside each weight, and the pair stands for the master value p + r.  Per element, in fp32: m and v advance exactly as in
 * nv_adamw_flat, x = p + r takes the AdamW update, then p = bf16_rn(x) and r = bf16_rn(x - p), rounded toward zero instead
 * where that keeps bf16_rn(p + r) == p.  With r == 0 on entry, p, m and v come out bit for bit as from nv_adamw_flat.  All operands bf16
 * and 16-byte aligned; 9 x 2 bytes of HBM traffic per element (10 with write_clipped_grad). */
int nv_adamw_flat_compensated(void* p, void* r, void* g, void* m, void* v, int64_t n, float lr, float beta1, float beta2,
                              float eps, float weight_decay, int step, const float* clip_state, int write_clipped_grad,
                              void* stream);
/* Opt-in block-wise 8-bit moments for the bf16 buffer (Dettmers et al., ICLR 2022).  Each 64-element block of m and of v
 * is one fp32 absmax and 64 uint8 codes, valued maps[code] * absmax; maps is fp32 [512]: the signed map of m, then the
 * unsigned map of v, both sorted (navillm_b200/optim.py builds them).  Per element, in fp32: m and v are dequantized, the
 * update of nv_adamw_flat (r null) or nv_adamw_flat_compensated runs on them, and each block is requantized to the nearest
 * code (a tie to the smaller magnitude) of x / absmax with its new absmax.  Codes [n] and absmax [ceil(n / 64)] per
 * moment; p, r and g 16-byte aligned, the codes 8-byte aligned.  10.25 bytes of HBM traffic per element, 14.25 with r. */
int nv_adamw_flat_8bit(void* p, void* r, void* g, void* m_code, float* m_absmax, void* v_code, float* v_absmax,
                       const float* maps, int64_t n, float lr, float beta1, float beta2, float eps, float weight_decay, int step,
                       const float* clip_state, int write_clipped_grad, void* stream);
/* One moment of n elements (bf16 or fp32) to the 8-bit form and back, in the blocks of nv_adamw_flat_8bit (is_signed: m's
 * map, else v's).  For optimizer state (de)serialisation. */
int nv_moments_quantize_8bit(const void* src, int is_bf16, void* code, float* absmax, int64_t n, int is_signed,
                             const float* maps, void* stream);
int nv_moments_dequantize_8bit(const void* code, const float* absmax, void* dst, int is_bf16, int64_t n, int is_signed,
                               const float* maps, void* stream);

/* ---- one decoder layer of the inference forward in ONE call (csrc/layer.cu) ----------------------------------------
 * transformers LlamaDecoderLayer (reached through models/modified_lm.py:112-116): RMSNorm -> fused qkv projection -> RoPE
 * -> causal attention over packed rows -> o_proj + residual -> RMSNorm -> gate|up -> SwiGLU -> down + residual, launched
 * in order on `stream` with every intermediate in the caller's workspace (nv_llama_layer_ws_bytes).  No activations are
 * kept: this is the forward of evaluation / prefill at small packed batches, where one ctypes call per kernel is the
 * bottleneck.  kv_mode 0: plain self-attention over the packed rows; 1: also store post-RoPE K/V of the rows in the caches
 * (prefill of generate); 2: the rows are suffixes of sequences whose prefixes are cached (cached / kv_start / kv_len as in
 * nv_kv_store_suffix / nv_attn_fwd_kv); 3: prefill of generate() into an fp8 cache (nv_kv_store_prefill_fp8: kcache / vcache
 * hold e4m3 bytes, kexp / vexp the row exponents; the layer's own attention reads the unrounded K, V); 4: kv_mode 2 over an
 * fp8 prefix cache (nv_kv_store_suffix_fp8 + nv_attn_fwd_kv_fp8: the new rows attend over their own rounded K', V' too).
 * out_rows (nullable, R rows): only these rows are produced (last layer). */
typedef struct nv_layer_args {
  const void* x;            /* [T, D] bf16 residual stream in */
  void* y;                  /* [R or T, D] bf16 residual stream out */
  const void* ln1; const void* wqkv; const void* wo; const void* ln2; const void* wgu; const void* wd;
  const int* pos; const void* cos_t; const void* sin_t; const int* cu_seqlens;
  void* kcache; void* vcache; const int* cached; const int* kv_start; const int* kv_len;
  const int* out_rows;
  void* ws; int64_t ws_bytes;
  int B, T, total_qblocks, Smax, Tkv, kv_mode, R, D, F, H;
  float eps, scale;
  /* optional fp8 copies of the four weights (e4m3 rows, int8 row exponents: nv_quantize_fp8_rows); a GEMM whose weight
   * pair is set and whose row count (T for qkv, R or T for the others) is <= fp8_max_rows runs nv_gemm_fp8w_bf16 */
  const void* wqkv_q; const void* wqkv_e; const void* wo_q; const void* wo_e;
  const void* wgu_q; const void* wgu_e; const void* wd_q; const void* wd_e;
  int fp8_max_rows;
  void* kexp; void* vexp;   /* kv_mode 3, 4: int8 row exponents [B, Smax, H] of the fp8 caches */
  /* 1: the four GEMMs run W8A8 at every row count (nv_quantize_act_fp8 of the GEMM input + nv_gemm_w8a8_bf16 on the fp8
   * weight pairs above, which must all be set; D and F multiples of 128); fp8_max_rows is then ignored */
  int act_fp8;
  /* optional int4 copies of the four weights (codes, bf16 scales, uint8 zero-points: nv_quantize_int4_groups); a GEMM
   * whose triple is set and whose row count is in 17..int4_max_rows runs nv_gemm_int4w_bf16 (at most 16 rows: bf16, as
   * without the copy).  Exclusive with the fp8 pairs and act_fp8. */
  const void* wqkv_c; const void* wqkv_s; const void* wqkv_z; const void* wo_c; const void* wo_s; const void* wo_z;
  const void* wgu_c; const void* wgu_s; const void* wgu_z; const void* wd_c; const void* wd_s; const void* wd_z;
  int int4_max_rows;
} nv_layer_args;
int nv_layer_args_size(void);                           /* sizeof(nv_layer_args): bindings check their mirror against it */
int64_t nv_llama_layer_ws_bytes(int T, int R, int D, int F);
int nv_llama_layer_infer(const nv_layer_args* a, void* stream);

/* ---- in-switch gradient all-reduce over NVLS multicast (csrc/nvls_allreduce.cu) ---------------------------------
 * The path's one exchange step (reference: DDP's NCCL all-reduce, tools/optims.py:52-54, fired from the last backward
 * outside no_sync, tasks/agents/mp3d_agent.py:661-667).  Elements [elem_off, elem_off + n) of a symmetric buffer whose
 * NVLS multicast address is mc_ptr are summed across the `world` replicas in the NVSwitch (multimem.ld_reduce, fp32
 * accumulation), scaled, and written back to every replica (multimem.st); rank r handles the r-th 1/world of the range.
 * Call on every rank, between two cross-rank barriers.  is_bf16: 1 = bf16, 0 = fp32 elements; range 16-byte aligned. */
int nv_multimem_allreduce(uint64_t mc_ptr, int64_t elem_off, int64_t n, int is_bf16, int rank, int world, float scale,
                          int ctas, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NAVILLM_B200_H_ */
