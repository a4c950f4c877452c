// navillm_b200 — one decoder layer of the INFERENCE forward as a single C-ABI call.
//
// Host-side composite, no new kernels: nv_llama_layer_infer launches the ten kernels of a LLaMA decoder layer
// (reference: transformers LlamaDecoderLayer reached through models/modified_lm.py:112-116; SURVEY.md §2b K9) in order, on
// the caller's stream, with every intermediate in a caller-provided workspace.  Why it exists: small packed batches
// (one navigation step at batch 1, evaluation rollouts with cross-step prefix-KV reuse, SURVEY.md §8f n1) are HOST-bound
// when each kernel is its own ctypes call from Python (~20 us per call against a few microseconds of GPU work: 328 calls
// = 10 ms per forward at T = 192); one call per layer leaves the GPU as the limit.  Training-size batches do not
// need it (their step is GPU-bound) and keep the per-kernel path, which also saves the activations for the backward.
// act_fp8 (set_activation_dtype("fp8")): each of the four GEMMs is nv_quantize_act_fp8 of its input into the workspace
// followed by nv_gemm_w8a8_bf16 on the fp8 weight copy, at every row count.
#include <stdint.h>

#include "navillm_b200.h"
#include "nv_host.h"

namespace {

inline int64_t al(int64_t x) { return (x + 255) & ~int64_t(255); }

struct Carve {
  uint8_t* p;
  int64_t left;
  void* take(int64_t bytes) {
    bytes = al(bytes);
    if (bytes > left) return nullptr;
    void* r = p;
    p += bytes;
    left -= bytes;
    return r;
  }
};

}  // namespace

extern "C" int nv_layer_args_size(void) { return (int)sizeof(nv_layer_args); }

extern "C" int64_t nv_llama_layer_ws_bytes(int T, int R, int D, int F) {
  const int64_t Tm = R > 0 ? R : T;
  int64_t b = al((int64_t)T * D * 2) + al((int64_t)T * 4) + al((int64_t)T * 3 * D * 2) + al((int64_t)T * D * 2);
  if (R > 0) b += 2 * al((int64_t)R * D * 2);
  b += 2 * al(Tm * D * 2) + al(Tm * 4) + al(Tm * 2 * F * 2) + al(Tm * F * 2);
  // act_fp8: the e4m3 GEMM input (largest: T x D or Tm x F) and its exponents
  const int64_t qn = (int64_t)T * D > Tm * F ? (int64_t)T * D : Tm * F;
  b += al(qn) + al(qn / 128);
  return b + 256;
}

extern "C" int nv_llama_layer_infer(const nv_layer_args* a, void* stream) {
  using namespace nv;
  NV_REQUIRE(a && a->x && a->y && a->ws, "nv_llama_layer_infer: null argument");
  const int T = a->T, D = a->D, F = a->F, H = a->H, R = a->out_rows ? a->R : 0;
  NV_REQUIRE(T > 0 && D == H * 128 && F > 0, "nv_llama_layer_infer: needs head_dim 128 (D=%d H=%d)", D, H);
  NV_REQUIRE(a->ws_bytes >= nv_llama_layer_ws_bytes(T, R, D, F), "nv_llama_layer_infer: workspace too small");
  uintptr_t base = (reinterpret_cast<uintptr_t>(a->ws) + 255) & ~uintptr_t(255);
  Carve c{reinterpret_cast<uint8_t*>(base), a->ws_bytes - (int64_t)(base - reinterpret_cast<uintptr_t>(a->ws))};
  const int Tm = R > 0 ? R : T;
  void* xn = c.take((int64_t)T * D * 2);
  float* rstd = static_cast<float*>(c.take((int64_t)T * 4));
  uint8_t* qkv = static_cast<uint8_t*>(c.take((int64_t)T * 3 * D * 2));
  void* ao = c.take((int64_t)T * D * 2);
  void* aor = R > 0 ? c.take((int64_t)R * D * 2) : ao;
  void* xr = R > 0 ? c.take((int64_t)R * D * 2) : const_cast<void*>(a->x);
  void* xm = c.take((int64_t)Tm * D * 2);
  void* xn2 = c.take((int64_t)Tm * D * 2);
  float* rstd2 = static_cast<float*>(c.take((int64_t)Tm * 4));
  void* gu = c.take((int64_t)Tm * 2 * F * 2);
  void* h = c.take((int64_t)Tm * F * 2);
  const int64_t qn = (int64_t)T * D > (int64_t)Tm * F ? (int64_t)T * D : (int64_t)Tm * F;
  void* aq = c.take(qn);
  void* ae = c.take(qn / 128);
  NV_REQUIRE(ae != nullptr, "nv_llama_layer_infer: workspace carve failed");
  if (a->act_fp8) {
    NV_REQUIRE(a->wqkv_q && a->wqkv_e && a->wo_q && a->wo_e && a->wgu_q && a->wgu_e && a->wd_q && a->wd_e,
               "nv_llama_layer_infer: act_fp8 needs the fp8 copies of all four weights");
    NV_REQUIRE(D % 128 == 0 && F % 128 == 0, "nv_llama_layer_infer: act_fp8 needs D and F multiples of 128 (D=%d F=%d)", D, F);
  }
  int rc;
  // y[rows, N] = x[rows, K] W^T (+ addend): W8A8 on the fp8 copy of W in act_fp8 mode; else the fp8 copy of W when it is
  // given and the GEMM has at most fp8_max_rows rows
  auto linear = [&](const void* x, const void* w, const void* wq, const void* we, void* y, const void* addend, int rows, int N,
                    int K) {
    if (a->act_fp8) {
      const int qrc = nv_quantize_act_fp8(x, K, aq, K, ae, K / 128, rows, K, stream);
      if (qrc != NV_OK) return qrc;
      return nv_gemm_w8a8_bf16(aq, K, ae, K / 128, wq, K, we, y, N, addend, D, rows, N, K, stream);
    }
    if (wq && we && rows <= a->fp8_max_rows)
      return nv_gemm_fp8w_bf16(x, K, wq, K, we, y, N, addend, D, rows, N, K, 0, stream);
    return nv_gemm_bf16(x, K, 0, w, K, 0, y, N, addend, addend ? D : 0, rows, N, K, addend ? 1u : 0u, 0, stream);
  };
#define STEP(call) do { rc = (call); if (rc != NV_OK) return rc; } while (0)
  // ---- attention block:  xm = x + o_proj(attn(rope(qkv(rmsnorm1(x))))) ----
  STEP(nv_rmsnorm_fwd(a->x, D, a->ln1, xn, D, rstd, T, D, a->eps, stream));
  STEP(linear(xn, a->wqkv, a->wqkv_q, a->wqkv_e, qkv, nullptr, T, 3 * D, D));
  STEP(nv_rope_inplace(qkv, 3 * (int64_t)D, a->pos, a->cos_t, a->sin_t, T, 2 * H, 128, 0, stream));
  if (a->kv_mode == 2) {            // new rows appended to a cache that already holds a prefix; attention over the cache
    STEP(nv_kv_store_suffix(qkv, 3 * (int64_t)D, a->cu_seqlens, a->cached, a->kcache, a->vcache, a->B, T, a->Smax, D, stream));
    STEP(nv_attn_fwd_kv(qkv, 3 * (int64_t)D, a->kcache, D, a->vcache, D, ao, D, nullptr, a->cu_seqlens, a->kv_start, a->kv_len, a->B,
                        T, a->Tkv, H, 128, a->total_qblocks, a->scale, stream));
  } else if (a->kv_mode == 4) {     // ... over an fp8 cache: the new rows are quantized as they are stored, then read back
    STEP(nv_kv_store_suffix_fp8(qkv, 3 * (int64_t)D, a->cu_seqlens, a->cached, a->kcache, a->vcache, a->kexp, a->vexp, a->B, T, a->Smax,
                                H, stream));
    STEP(nv_attn_fwd_kv_fp8(qkv, 3 * (int64_t)D, a->kcache, a->vcache, a->kexp, a->vexp, ao, D, nullptr, a->cu_seqlens, a->kv_start,
                            a->kv_len, a->B, T, a->Tkv, H, 128, a->total_qblocks, a->scale, stream));
  } else {
    if (a->kv_mode == 1)            // prefill of generate(): post-RoPE K, V also go to the cache
      STEP(nv_kv_store_prefill(qkv, 3 * (int64_t)D, a->cu_seqlens, a->kcache, a->vcache, a->B, T, a->Smax, D, stream));
    else if (a->kv_mode == 3)       // ... into an fp8 cache
      STEP(nv_kv_store_prefill_fp8(qkv, 3 * (int64_t)D, a->cu_seqlens, a->kcache, a->vcache, a->kexp, a->vexp, a->B, T, a->Smax, H,
                                   stream));
    STEP(nv_attn_fwd(qkv, 3 * (int64_t)D, qkv + (int64_t)D * 2, 3 * (int64_t)D, qkv + (int64_t)D * 4, 3 * (int64_t)D, ao, D, nullptr,
                     a->cu_seqlens, a->B, T, H, 128, a->total_qblocks, a->scale, stream));
  }
  if (R > 0) {                      // last layer: only the requested rows continue (their K, V came from all rows)
    STEP(nv_gather_rows(ao, D, a->out_rows, aor, D, R, D, stream));
    STEP(nv_gather_rows(a->x, D, a->out_rows, xr, D, R, D, stream));
  }
  STEP(linear(aor, a->wo, a->wo_q, a->wo_e, xm, xr, Tm, D, D));
  // ---- MLP:  y = xm + down(silu(gate(xn2)) * up(xn2)) ----
  STEP(nv_rmsnorm_fwd(xm, D, a->ln2, xn2, D, rstd2, Tm, D, a->eps, stream));
  STEP(linear(xn2, a->wgu, a->wgu_q, a->wgu_e, gu, nullptr, Tm, 2 * F, D));
  STEP(nv_swiglu_fwd(gu, 2 * (int64_t)F, h, F, Tm, F, stream));
  STEP(linear(h, a->wd, a->wd_q, a->wd_e, a->y, xm, Tm, D, F));
#undef STEP
  return NV_OK;
}
