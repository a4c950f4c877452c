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
/* nv_gemm_fp8w_bf16 is nv_gemm_bf16 with K-major operands (a_mn = b_mn = 0) and the weight given as (Wq, exps) in the same
 * format, for the inference GEMMs above 16 rows (prefix-cached navigation suffixes, pruned last layers, decode batches
 * 17..256): C = bf16(bf16(A Wq'^T) + addend) with addend optional, bit for bit nv_gemm_bf16's result on W' at every M, N, K
 * and tile width.  block_n: 0 (auto), 32 or 128.  lda % 8 == 0, ldw (bytes) % 16 == 0. */
int nv_gemm_fp8w_bf16(const void* A, int64_t lda, const void* Wq, int64_t ldw, const void* exps, void* C, int64_t ldc,
                      const void* addend, int64_t ld_add, int M, int N, int K, int block_n, void* stream);
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

/* ---- fused clip + AdamW over flat buffers (csrc/optim.cu) ------------------------------------------------------
 * torch.nn.utils.clip_grad_norm_(model.parameters(), 40.) + torch.optim.AdamW.step() of the reference
 * (train.py:86-89, tools/optims.py:43) as sum-of-squares partials -> device-side clip coefficient -> one update
 * pass per flat buffer.  clip_state: fp32 [2] = {grad norm, clip coefficient}. */
int nv_optim_partials(void);
int nv_grad_sumsq(const void* g, int64_t n, int is_bf16, float* partial, void* stream);
int nv_clip_coef(const float* partial, int n_partial, float max_norm, float* state, void* stream);
int nv_adamw_flat(void* p, void* g, void* m, void* v, int64_t n, int is_bf16, float lr, float beta1, float beta2, float eps,
                  float weight_decay, int step, const float* clip_state, int write_clipped_grad, void* stream);

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
