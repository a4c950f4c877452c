"""Python-side launchers for the sm_90a kernels (thin: argument checking + C-ABI call).

Every function here writes into caller-provided or freshly ``torch.empty``-allocated CUDA tensors and
launches on the current stream.  Nothing falls back to torch math.
"""
from __future__ import annotations

import ctypes
import os

import torch

from . import _lib
from ._lib import check, f32, i32, i64, ptr, stream_ptr, u32

bf16 = torch.bfloat16

gemm_timer = None   # set to a list by bench.py to collect (start_event, end_event, flops) per GEMM launch


def _rowmajor(t: torch.Tensor, name: str) -> None:
    if t.dim() != 2 or t.stride(1) != 1:
        raise ValueError(f"{name}: expected a 2-D tensor with unit inner stride, got shape {tuple(t.shape)} strides {t.stride()}")
    if not t.is_cuda:
        raise _lib.NvError(f"{name}: navillm_b200 kernels need CUDA tensors (no CPU fallback)")


def gemm(a: torch.Tensor, b: torch.Tensor, *, a_mn: bool = False, b_mn: bool = False, out: torch.Tensor | None = None,
         addend: torch.Tensor | None = None, out_f32: bool = False, block_n: int = 0) -> torch.Tensor:
    """C[M,N] = A·B (+ addend) on wgmma (csrc/gemm_bf16.cu).

    a: [M,K] (a_mn=False) or [K,M] (a_mn=True);  b: [N,K] (b_mn=False) or [K,N] (b_mn=True); bf16.
    """
    _rowmajor(a, "a"); _rowmajor(b, "b")
    assert a.dtype == bf16 and b.dtype == bf16
    M, K = (a.shape[1], a.shape[0]) if a_mn else (a.shape[0], a.shape[1])
    N, Kb = (b.shape[1], b.shape[0]) if b_mn else (b.shape[0], b.shape[1])
    if K != Kb:
        raise ValueError(f"gemm: contraction mismatch {K} vs {Kb}")
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32 if out_f32 else bf16, device=a.device)
    _rowmajor(out, "out")
    assert out.shape == (M, N) and out.dtype == (torch.float32 if out_f32 else bf16)
    flags = 0
    if addend is not None:
        _rowmajor(addend, "addend")
        assert addend.shape == (M, N) and addend.dtype == bf16
        flags |= _lib.GEMM_ADD
    if out_f32:
        flags |= _lib.GEMM_OUT_F32
    lib = _lib.load()
    timer = gemm_timer
    if timer is not None:       # bench.py: CUDA events on the launching stream around every GEMM launch
        st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        st.record()
    check(lib.nv_gemm_bf16(ptr(a), i64(a.stride(0)), i32(a_mn), ptr(b), i64(b.stride(0)), i32(b_mn), ptr(out),
                           i64(out.stride(0)), ptr(addend), i64(addend.stride(0) if addend is not None else 0),
                           i32(M), i32(N), i32(K), u32(flags), i32(block_n), stream_ptr()), "nv_gemm_bf16")
    if timer is not None:
        en.record()
        timer.append((st, en, 2.0 * M * N * K, 2.0 * (M * K + N * K + M * N * (2 if addend is not None else 1))))
    return out


WGRAD_SEG_MAX = 64          # NV_WGRAD_SEG_MAX of include/navillm_b200.h


def gemm_wgrad_seg(segs, out: torch.Tensor, *, addend: torch.Tensor | None = None) -> torch.Tensor:
    """out[M,N] = bf16(bf16(sum_s a_s^T b_s) (+ addend)) in one launch (nv_gemm_wgrad_seg_bf16): segs is a list of 1 ..
    WGRAD_SEG_MAX pairs (a_s [rows_s, M], b_s [rows_s, N]) of bf16 CUDA tensors on out's device, rounded to bf16 once.  Bit for bit
    ``gemm(a, b, a_mn=True, b_mn=True, addend=addend)`` over the row-concatenation of the segments, each zero-padded to a
    multiple of 64 rows.  ``addend`` may be ``out``."""
    if not 1 <= len(segs) <= WGRAD_SEG_MAX:
        raise ValueError(f"gemm_wgrad_seg: {len(segs)} segments (1..{WGRAD_SEG_MAX})")
    _rowmajor(out, "out")
    M, N = out.shape
    assert out.dtype == bf16
    n = len(segs)
    A, B = (ctypes.c_void_p * n)(), (ctypes.c_void_p * n)()
    lda, ldb, rows = (ctypes.c_int64 * n)(), (ctypes.c_int64 * n)(), (ctypes.c_int * n)()
    for s, (a, b) in enumerate(segs):
        _rowmajor(a, "a"); _rowmajor(b, "b")
        if a.device != out.device or b.device != out.device:
            raise ValueError(f"gemm_wgrad_seg: segment {s} on {a.device} / {b.device}, out on {out.device}")
        if a.dtype != bf16 or b.dtype != bf16 or a.shape[1] != M or b.shape[1] != N or a.shape[0] != b.shape[0]:
            raise ValueError(f"gemm_wgrad_seg: segment {s}: a {tuple(a.shape)} {a.dtype}, b {tuple(b.shape)} {b.dtype} for an "
                             f"output [{M}, {N}] (bf16 [rows, M] and [rows, N] expected)")
        A[s], B[s] = a.data_ptr(), b.data_ptr()
        lda[s], ldb[s], rows[s] = a.stride(0), b.stride(0), a.shape[0]
    if addend is not None:
        _rowmajor(addend, "addend")
        if addend.shape != (M, N) or addend.dtype != bf16 or addend.device != out.device:
            raise ValueError(f"gemm_wgrad_seg: addend bf16 [{M}, {N}] on {out.device} expected (got {addend.dtype} "
                             f"{tuple(addend.shape)} on {addend.device})")
    check(_lib.load().nv_gemm_wgrad_seg_bf16(A, lda, B, ldb, rows, i32(n), ptr(out), i64(out.stride(0)), ptr(addend),
                                             i64(addend.stride(0) if addend is not None else 0), i32(M), i32(N), stream_ptr()),
          "nv_gemm_wgrad_seg_bf16")
    return out


def _qblocks(seqlens) -> int:
    return int(sum((int(l) + 127) // 128 for l in seqlens))


def attn_fwd(qkv: torch.Tensor, cu_seqlens: torch.Tensor, seqlens, n_heads: int, *, out: torch.Tensor | None = None,
             lse: torch.Tensor | None = None, scale: float | None = None):
    """Causal self-attention over packed sequences (csrc/attn_fwd.cu).

    qkv: [T, 3*H*128] bf16 (q | k | v column blocks, RoPE already applied); cu_seqlens: int32 [B+1] on the
    device; seqlens: host list of the B lengths.  Returns (o [T, H*128] bf16, lse [H, T] fp32).
    """
    _rowmajor(qkv, "qkv")
    T, W = qkv.shape
    hd = 128
    assert W == 3 * n_heads * hd and qkv.dtype == bf16
    B = len(seqlens)
    assert cu_seqlens.dtype == torch.int32 and cu_seqlens.numel() == B + 1 and cu_seqlens.is_cuda
    if out is None:
        out = torch.empty((T, n_heads * hd), dtype=bf16, device=qkv.device)
    if lse is None:
        lse = torch.empty((n_heads, T), dtype=torch.float32, device=qkv.device)
    if scale is None:
        scale = hd ** -0.5
    q, k, v = qkv[:, : n_heads * hd], qkv[:, n_heads * hd: 2 * n_heads * hd], qkv[:, 2 * n_heads * hd:]
    lib = _lib.load()
    check(lib.nv_attn_fwd(ptr(q), i64(qkv.stride(0)), ptr(k), i64(qkv.stride(0)), ptr(v), i64(qkv.stride(0)), ptr(out),
                          i64(out.stride(0)), ptr(lse), ptr(cu_seqlens), i32(B), i32(T), i32(n_heads), i32(hd),
                          i32(_qblocks(seqlens)), f32(scale), stream_ptr()), "nv_attn_fwd")
    return out, lse


def attn_fwd_kv(q: torch.Tensor, kcache: torch.Tensor, vcache: torch.Tensor, cu_q: torch.Tensor, q_lens, kv_start: torch.Tensor,
                kv_len: torch.Tensor, n_heads: int, *, out: torch.Tensor | None = None, scale: float | None = None,
                lse: torch.Tensor | None = None):
    """Suffix attention over a KV cache (nv_attn_fwd_kv): q [Tq, >=H*128] bf16 view of the packed new rows (RoPE
    applied), caches [B, Smax, H*128] bf16 (already holding the new rows' K/V, zero-initialised), kv_start / kv_len
    int32 [B] on the device.  Query i of sequence b sees keys <= kv_len[b] - q_lens[b] + i.  Returns o [Tq, H*128].
    ``lse`` (fp32 [H, Tq], optional) receives the log-sum-exp of the scaled scores, as ``attn_fwd`` returns it (the
    input of ``attn_bwd_kv``)."""
    _rowmajor(q, "q")
    hd = 128
    Tq = q.shape[0]
    B = len(q_lens)
    assert q.dtype == bf16 and kcache.dtype == bf16 and vcache.dtype == bf16 and kcache.is_contiguous() and vcache.is_contiguous()
    assert kcache.dim() == 3 and kcache.shape[2] == n_heads * hd and kcache.shape == vcache.shape
    for t in (cu_q, kv_start, kv_len):
        assert t.dtype == torch.int32 and t.is_cuda
    if out is None:
        out = torch.empty((Tq, n_heads * hd), dtype=bf16, device=q.device)
    if lse is not None and (lse.dtype != torch.float32 or not lse.is_contiguous() or tuple(lse.shape) != (n_heads, Tq)):
        raise ValueError(f"attn_fwd_kv: lse fp32 [{n_heads}, {Tq}] contiguous expected (got {lse.dtype} {tuple(lse.shape)})")
    if scale is None:
        scale = hd ** -0.5
    Tkv = kcache.shape[0] * kcache.shape[1]
    ldk = kcache.shape[2]
    check(_lib.load().nv_attn_fwd_kv(ptr(q), i64(q.stride(0)), ptr(kcache), i64(ldk), ptr(vcache), i64(ldk), ptr(out),
                                     i64(out.stride(0)), ptr(lse), ptr(cu_q), ptr(kv_start), ptr(kv_len), i32(B), i32(Tq),
                                     i32(Tkv), i32(n_heads), i32(hd), i32(_qblocks(q_lens)), f32(scale), stream_ptr()),
          "nv_attn_fwd_kv")
    return out


def _tree_args(name, q_lens, tree_end):
    """Every sequence of a tree-masked attention holds the q_len rows of one tree: tree_end int32 [q_len] on the device."""
    n = {int(l) for l in q_lens}
    if len(n) != 1 or tree_end.dtype != torch.int32 or tree_end.dim() != 1 or not tree_end.is_contiguous() \
            or not tree_end.is_cuda or tree_end.numel() != next(iter(n)):
        raise ValueError(f"{name}: every sequence needs the same number of query rows and tree_end int32 [rows] contiguous on "
                         f"the device (got q_lens {sorted(n)}, tree_end {tree_end.dtype} {tuple(tree_end.shape)})")


def attn_fwd_tree(q: torch.Tensor, kcache: torch.Tensor, vcache: torch.Tensor, cu_q: torch.Tensor, q_lens, kv_start: torch.Tensor,
                  kv_len: torch.Tensor, tree_end: torch.Tensor, n_heads: int, *, out: torch.Tensor | None = None,
                  scale: float | None = None):
    """``attn_fwd_kv`` with the tree mask (nv_attn_fwd_tree): the q_len rows of every sequence are the nodes of one tree in DFS
    preorder, and query i sees the kv_len - q_len >= 1 cached keys and tree key j only when j <= i < tree_end[j] (its ancestors
    and itself; ``trie.tree_rows``).  Returns o [Tq, H*128]."""
    _rowmajor(q, "q")
    hd = 128
    Tq = q.shape[0]
    B = len(q_lens)
    assert q.dtype == bf16 and kcache.dtype == bf16 and vcache.dtype == bf16 and kcache.is_contiguous() and vcache.is_contiguous()
    assert kcache.dim() == 3 and kcache.shape[2] == n_heads * hd and kcache.shape == vcache.shape
    for t in (cu_q, kv_start, kv_len):
        assert t.dtype == torch.int32 and t.is_cuda
    _tree_args("attn_fwd_tree", q_lens, tree_end)
    if out is None:
        out = torch.empty((Tq, n_heads * hd), dtype=bf16, device=q.device)
    if scale is None:
        scale = hd ** -0.5
    Tkv = kcache.shape[0] * kcache.shape[1]
    ldk = kcache.shape[2]
    check(_lib.load().nv_attn_fwd_tree(ptr(q), i64(q.stride(0)), ptr(kcache), i64(ldk), ptr(vcache), i64(ldk), ptr(out),
                                       i64(out.stride(0)), ptr(None), ptr(cu_q), ptr(kv_start), ptr(kv_len), ptr(tree_end), i32(B),
                                       i32(Tq), i32(Tkv), i32(n_heads), i32(hd), i32(_qblocks(q_lens)), f32(scale), stream_ptr()),
          "nv_attn_fwd_tree")
    return out


# ---------------------------------------------------------------------------------------------------
# row-wise LM kernels (csrc/lm_ops.cu)
# ---------------------------------------------------------------------------------------------------
def rmsnorm_fwd(x, w, eps, *, out=None, rstd=None):
    _rowmajor(x, "x")
    T, D = x.shape
    if out is None:
        out = torch.empty((T, D), dtype=bf16, device=x.device)
    if rstd is None:
        rstd = torch.empty((T,), dtype=torch.float32, device=x.device)
    check(_lib.load().nv_rmsnorm_fwd(ptr(x), i64(x.stride(0)), ptr(w), ptr(out), i64(out.stride(0)), ptr(rstd), i32(T),
                                     i32(D), f32(eps), stream_ptr()), "nv_rmsnorm_fwd")
    return out, rstd


_ws_cache: dict = {}


def _workspace(dev, nfloat: int) -> torch.Tensor:
    key = (dev.index, "f32")
    ws = _ws_cache.get(key)
    if ws is None or ws.numel() < nfloat:
        ws = torch.empty((max(nfloat, 1 << 20),), dtype=torch.float32, device=dev)
        _ws_cache[key] = ws
    return ws


def rmsnorm_bwd(x, w, rstd, dy, *, dres=None, dx=None, dw=None, accumulate_dw=True):
    """dx = rmsnorm'(dy) (+ dres); dw (bf16 [D]) is accumulated in place when given."""
    _rowmajor(x, "x"); _rowmajor(dy, "dy")
    T, D = x.shape
    lib = _lib.load()
    if dx is None:
        dx = torch.empty((T, D), dtype=bf16, device=x.device)
    ws = _workspace(x.device, lib.nv_rmsnorm_bwd_partials() * D)
    check(lib.nv_rmsnorm_bwd(ptr(x), i64(x.stride(0)), ptr(w), ptr(rstd), ptr(dy), i64(dy.stride(0)), ptr(dres),
                             i64(dres.stride(0) if dres is not None else 0), ptr(dx), i64(dx.stride(0)), ptr(dw),
                             i32(1 if accumulate_dw else 0), ptr(ws), i32(T), i32(D), stream_ptr()), "nv_rmsnorm_bwd")
    return dx


def rope_(x, pos, cos_t, sin_t, n_heads, head_dim=128, backward=False):
    """In-place rotate-half RoPE on the first n_heads*head_dim columns of x ([T, ld] bf16)."""
    _rowmajor(x, "x")
    assert pos.dtype == torch.int32
    check(_lib.load().nv_rope_inplace(ptr(x), i64(x.stride(0)), ptr(pos), ptr(cos_t), ptr(sin_t), i32(x.shape[0]),
                                      i32(n_heads), i32(head_dim), i32(1 if backward else 0), stream_ptr()),
          "nv_rope_inplace")
    return x


def swiglu_fwd(gu, *, out=None):
    _rowmajor(gu, "gu")
    T, F2 = gu.shape
    F = F2 // 2
    if out is None:
        out = torch.empty((T, F), dtype=bf16, device=gu.device)
    check(_lib.load().nv_swiglu_fwd(ptr(gu), i64(gu.stride(0)), ptr(out), i64(out.stride(0)), i32(T), i32(F),
                                    stream_ptr()), "nv_swiglu_fwd")
    return out


def swiglu_bwd(gu, dh, *, out=None):
    T, F2 = gu.shape
    if out is None:
        out = torch.empty((T, F2), dtype=bf16, device=gu.device)
    check(_lib.load().nv_swiglu_bwd(ptr(gu), i64(gu.stride(0)), ptr(dh), i64(dh.stride(0)), ptr(out),
                                    i64(out.stride(0)), i32(T), i32(F2 // 2), stream_ptr()), "nv_swiglu_bwd")
    return out


def scale_(x: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """x[rows, cols] (bf16, unit inner stride, even row stride) *= scale (a one-element fp32 CUDA tensor), in place."""
    _rowmajor(x, "x")
    assert x.dtype == bf16 and scale.dtype == torch.float32 and scale.numel() == 1 and scale.is_cuda
    check(_lib.load().nv_scale_bf16(ptr(x), i64(x.stride(0)), i32(x.shape[0]), i32(x.shape[1]), ptr(scale), stream_ptr()), "nv_scale_bf16")
    return x


def embed_fwd(ids, E, vis_src=None, vis=None, *, out=None):
    T = ids.numel()
    V, D = E.shape
    assert ids.dtype == torch.int32
    if out is None:
        out = torch.empty((T, D), dtype=bf16, device=E.device)
    if vis is not None:
        assert vis.dtype == torch.float32 and vis.is_contiguous() and vis_src.dtype == torch.int32
    check(_lib.load().nv_embed_fwd(ptr(ids), ptr(E), i32(V), ptr(vis_src if vis is not None else None), ptr(vis),
                                   ptr(out), i32(T), i32(D), stream_ptr()), "nv_embed_fwd")
    return out


def embed_bwd_vis(dx, vis_src, n_vis):
    T, D = dx.shape
    dvis = torch.zeros((n_vis, D), dtype=torch.float32, device=dx.device)
    check(_lib.load().nv_embed_bwd_vis(ptr(dx), ptr(vis_src), ptr(dvis), i32(T), i32(D), stream_ptr()),
          "nv_embed_bwd_vis")
    return dvis


def embed_bwd_weight_(dx, ids, dE, *, order=None, sorted_ids=None):
    """dE[ids[t]] += dx[t] (deterministic: tokens are sorted by id, one owner per distinct id).  ``order`` / ``sorted_ids``:
    the stable argsort of ``ids`` and the sorted ids as int32 device tensors when the caller has them (PackedPrompt sorts
    on the host, where the ids come from); otherwise they are computed here."""
    T, D = dx.shape
    if order is None or sorted_ids is None:
        sorted_ids, order = torch.sort(ids.to(torch.int64), stable=True)
    # keep the int32 copies referenced until after the launch: a temporary freed inside the argument
    # list would hand its block back to the caching allocator before the kernel reads it
    order32, sorted32 = order.to(torch.int32), sorted_ids.to(torch.int32)
    assert order32.numel() == T and sorted32.numel() == T
    check(_lib.load().nv_embed_bwd_weight(ptr(dx), ptr(order32), ptr(sorted32), ptr(dE), i32(T), i32(D), stream_ptr()),
          "nv_embed_bwd_weight")
    return dE


def gather_rows(src, rows, *, out=None):
    R, D = rows.numel(), src.shape[1]
    if out is None:
        out = torch.empty((R, D), dtype=bf16, device=src.device)
    check(_lib.load().nv_gather_rows(ptr(src), i64(src.stride(0)), ptr(rows), ptr(out), i64(out.stride(0)), i32(R),
                                     i32(D), stream_ptr()), "nv_gather_rows")
    return out


def scatter_rows_(src, rows, dst):
    R, D = rows.numel(), src.shape[1]
    check(_lib.load().nv_scatter_rows(ptr(src), i64(src.stride(0)), ptr(rows), ptr(dst), i64(dst.stride(0)), i32(R),
                                      i32(D), stream_ptr()), "nv_scatter_rows")
    return dst


def head_fwd(x, W, bias):
    R, D = x.shape
    O = W.shape[0]
    out = torch.empty((R, O), dtype=bf16, device=x.device)
    check(_lib.load().nv_head_fwd(ptr(x), i64(x.stride(0)), ptr(W), ptr(bias), ptr(out), i32(R), i32(O), i32(D),
                                  stream_ptr()), "nv_head_fwd")
    return out


def head_bwd(dy, x, W, *, dW=None, db=None, need_dx=True):
    R, D = x.shape
    O = W.shape[0]
    dx = torch.empty((R, D), dtype=bf16, device=x.device) if need_dx else None
    check(_lib.load().nv_head_bwd(ptr(dy), ptr(x), i64(x.stride(0)), ptr(W), ptr(dx), i64(dx.stride(0) if need_dx else 0),
                                  ptr(dW), ptr(db), i32(R), i32(O), i32(D), stream_ptr()), "nv_head_bwd")
    return dx


def ce_fwd_bwd(logits, labels, special_ids, *, grad_scale=None):
    """Per-row masked CE on bf16 logits; returns (row_loss fp32 [N], dlogits bf16 [N,V] or None)."""
    N, V = logits.shape
    row_loss = torch.empty((N,), dtype=torch.float32, device=logits.device)
    # rows padded to a multiple of 64 elements so dlogits can feed the wgmma GEMMs (16-byte aligned rows)
    dlogits = torch.empty((N, (V + 63) // 64 * 64), dtype=bf16, device=logits.device)[:, :V] if grad_scale is not None else None
    check(_lib.load().nv_ce_fwd_bwd(ptr(logits), i64(logits.stride(0)), ptr(labels), ptr(special_ids),
                                    i32(special_ids.numel()), ptr(row_loss), ptr(dlogits),
                                    i64(dlogits.stride(0) if dlogits is not None else 0), i32(N), i32(V),
                                    f32(grad_scale if grad_scale is not None else 0.0), stream_ptr()), "nv_ce_fwd_bwd")
    return row_loss, dlogits


def attn_bwd(qkv: torch.Tensor, o: torch.Tensor, do: torch.Tensor, lse: torch.Tensor, cu_seqlens: torch.Tensor, seqlens,
             n_heads: int, *, dqkv: torch.Tensor | None = None, scale: float | None = None, rope=None,
             dvec: torch.Tensor | None = None) -> torch.Tensor:
    """Backward of attn_fwd (csrc/attn_bwd.cu): returns dqkv [T, 3*H*128] bf16 (dq | dk | dv).
    rope = (pos int32 [T], cos_t, sin_t): also undo the rotary embedding in the epilogue (gradients w.r.t. pre-RoPE q/k).
    dvec: fp32 [H*T] already holding D[h,t] = sum_d do·o (from gemm_attnd) -> the row-sum kernel is skipped."""
    T, W = qkv.shape
    hd = 128
    HD = n_heads * hd
    if dqkv is None:
        dqkv = torch.empty((T, W), dtype=bf16, device=qkv.device)
    if scale is None:
        scale = hd ** -0.5
    have_d = dvec is not None
    if not have_d:
        dvec = _workspace(qkv.device, n_heads * T + 16)
    q, k, v = qkv[:, :HD], qkv[:, HD:2 * HD], qkv[:, 2 * HD:]
    dq, dk, dv = dqkv[:, :HD], dqkv[:, HD:2 * HD], dqkv[:, 2 * HD:]
    ld = qkv.stride(0)
    check(_lib.load().nv_attn_bwd(ptr(q), i64(ld), ptr(k), i64(ld), ptr(v), i64(ld), ptr(None if have_d else o), i64(o.stride(0)), ptr(do),
                                  i64(do.stride(0)), ptr(lse), ptr(dvec), ptr(dq), i64(dqkv.stride(0)), ptr(dk),
                                  i64(dqkv.stride(0)), ptr(dv), i64(dqkv.stride(0)), ptr(cu_seqlens), i32(len(seqlens)),
                                  i32(T), i32(n_heads), i32(hd), i32(_qblocks(seqlens)), f32(scale),
                                  ptr(rope[0] if rope else None), ptr(rope[1] if rope else None), ptr(rope[2] if rope else None),
                                  stream_ptr()),
          "nv_attn_bwd")
    if have_d:
        _lib.launch_count -= 1          # the row-sum kernel was not launched
    return dqkv


def attn_bwd_kv(q: torch.Tensor, o: torch.Tensor, do: torch.Tensor, lse: torch.Tensor, kcache: torch.Tensor, vcache: torch.Tensor,
                acc: torch.Tensor, cu_q: torch.Tensor, q_lens, kv_start: torch.Tensor, kv_len: torch.Tensor, kv_lens, n_heads: int, *,
                dqkv: torch.Tensor | None = None, scale: float | None = None, rope=None, dvec: torch.Tensor | None = None) -> torch.Tensor:
    """Backward of ``attn_fwd_kv`` (nv_attn_bwd_kv): returns dqkv [Tq, 3*H*128] bf16 (dq | dk | dv of the packed suffix rows).

    q [Tq, >=H*128] (post-RoPE), o / do [Tq, H*128] bf16, lse fp32 [H, Tq] from ``attn_fwd_kv(lse=...)``; caches bf16
    [B, Smax, H*128] as the forward read them; acc fp32 [B, Smax, 2*H*128] (dK | dV columns) accumulator over the cache
    rows.  ``q_lens`` / ``kv_lens``: host lengths (``kv_len`` / ``kv_start`` int32 [B] on the device).  Rows j < kv_len - q_len
    of sequence b accumulate their dK / dV into acc; the suffix rows get dK + acc, dV + acc.  rope / dvec: as ``attn_bwd``."""
    hd = 128
    HD = n_heads * hd
    B = len(q_lens)
    Tq = int(sum(int(l) for l in q_lens))
    for name, t in (("q", q), ("o", o), ("do", do)):
        if t.dtype != bf16 or t.dim() != 2 or t.stride(1) != 1 or t.shape[0] != Tq or t.shape[1] < HD or not t.is_cuda:
            raise ValueError(f"attn_bwd_kv: {name} bf16 [{Tq}, >= {HD}] CUDA rows expected (got {t.dtype} {tuple(t.shape)})")
    if kcache.dtype != bf16 or vcache.dtype != bf16 or kcache.dim() != 3 or kcache.shape != vcache.shape or kcache.shape[2] != HD \
            or not kcache.is_contiguous() or not vcache.is_contiguous():
        raise ValueError(f"attn_bwd_kv: bf16 [B, Smax, {HD}] contiguous caches expected (got {kcache.dtype} {tuple(kcache.shape)}, "
                         f"{vcache.dtype} {tuple(vcache.shape)})")
    Bc, Smax = kcache.shape[:2]
    if acc.dtype != torch.float32 or tuple(acc.shape) != (Bc, Smax, 2 * HD) or not acc.is_contiguous() or acc.device != kcache.device:
        raise ValueError(f"attn_bwd_kv: accumulator fp32 [{Bc}, {Smax}, {2 * HD}] contiguous expected "
                         f"(got {acc.dtype} {tuple(acc.shape)})")
    if lse.dtype != torch.float32 or tuple(lse.shape) != (n_heads, Tq) or not lse.is_contiguous():
        raise ValueError(f"attn_bwd_kv: lse fp32 [{n_heads}, {Tq}] expected (got {lse.dtype} {tuple(lse.shape)})")
    for name, t, n in (("cu_q", cu_q, B + 1), ("kv_start", kv_start, B), ("kv_len", kv_len, B)):
        if t.dtype != torch.int32 or t.numel() != n or not t.is_cuda:
            raise ValueError(f"attn_bwd_kv: {name} int32 [{n}] on the device expected (got {t.dtype} {tuple(t.shape)})")
    if len(kv_lens) != B or any(int(k) < int(l) or int(k) > Smax for k, l in zip(kv_lens, q_lens)):
        raise ValueError(f"attn_bwd_kv: kv_lens {list(kv_lens)} must satisfy q_len <= kv_len <= {Smax}")
    if dqkv is None:
        dqkv = torch.empty((Tq, 3 * HD), dtype=bf16, device=q.device)
    if dqkv.dtype != bf16 or dqkv.stride(1) != 1 or tuple(dqkv.shape) != (Tq, 3 * HD):
        raise ValueError(f"attn_bwd_kv: dqkv bf16 [{Tq}, {3 * HD}] expected (got {dqkv.dtype} {tuple(dqkv.shape)})")
    if scale is None:
        scale = hd ** -0.5
    have_d = dvec is not None
    if not have_d:
        dvec = _workspace(q.device, n_heads * Tq + 16)
    dq, dk, dv = dqkv[:, :HD], dqkv[:, HD:2 * HD], dqkv[:, 2 * HD:]
    acc2 = acc.view(Bc * Smax, 2 * HD)
    n_kblocks = int(sum((int(k) + 127) // 128 for k in kv_lens))
    check(_lib.load().nv_attn_bwd_kv(ptr(q), i64(q.stride(0)), ptr(kcache), ptr(vcache), i64(HD), ptr(None if have_d else o),
                                     i64(o.stride(0)), ptr(do), i64(do.stride(0)), ptr(lse), ptr(dvec), ptr(dq), i64(dqkv.stride(0)),
                                     ptr(dk), i64(dqkv.stride(0)), ptr(dv), i64(dqkv.stride(0)), ptr(acc2[:, :HD]), ptr(acc2[:, HD:]),
                                     i64(2 * HD), ptr(cu_q), ptr(kv_start), ptr(kv_len), i32(B), i32(Tq), i32(Bc * Smax),
                                     i32(n_heads), i32(hd), i32(_qblocks(q_lens)), i32(n_kblocks), f32(scale),
                                     ptr(rope[0] if rope else None), ptr(rope[1] if rope else None), ptr(rope[2] if rope else None),
                                     stream_ptr()),
          "nv_attn_bwd_kv")
    if have_d:
        _lib.launch_count -= 1          # the row-sum kernel was not launched
    return dqkv


# ---------------------------------------------------------------------------------------------------
# fp32 panorama-encoder / fusion kernels (csrc/pano_ops.cu)
# ---------------------------------------------------------------------------------------------------
f32_t = torch.float32


def _f32_2d(t: torch.Tensor, name: str) -> None:
    if t.dtype != f32_t or t.dim() != 2 or t.stride(1) != 1 or not t.is_cuda:
        raise ValueError(f"{name}: expected a 2-D fp32 CUDA tensor with unit inner stride, got {t.dtype} {tuple(t.shape)} {t.stride()}")


# Numerical mode of the fp32 panorama-encoder GEMMs: "tf32" = wgmma tf32 (what the reference's pinned
# torch 1.10 did by default on Ampere+: torch.backends.cuda.matmul.allow_tf32 = True), "fp32" = exact CUDA-core sgemm.
_PANO_PRECISION = os.environ.get("NAVILLM_PANO_PRECISION", "tf32")


def set_pano_precision(mode: str) -> str:
    """Select "tf32" (default) or "fp32" for ops.sgemm; returns the previous mode."""
    global _PANO_PRECISION
    if mode not in ("tf32", "fp32"):
        raise ValueError(f"pano precision must be 'tf32' or 'fp32', got {mode!r}")
    prev, _PANO_PRECISION = _PANO_PRECISION, mode
    return prev


def sgemm(a, b, *, ta=False, tb=False, bias=None, out=None, accumulate=False):
    """C = op(A)·op(B) (+bias).  a: [M,K] (ta=False) / [K,M];  b: [N,K] (tb=False, nn.Linear weight) / [K,N]."""
    _f32_2d(a, "a"); _f32_2d(b, "b")
    M, K = (a.shape[1], a.shape[0]) if ta else a.shape
    N, Kb = (b.shape[1], b.shape[0]) if tb else b.shape
    assert K == Kb, f"sgemm contraction mismatch {K} vs {Kb}"
    if out is None:
        assert not accumulate
        out = torch.empty((M, N), dtype=f32_t, device=a.device)
    _f32_2d(out, "out")
    # tensor-core path when TMA can address the operands (16-byte bases, row strides % 4) and the problem is not tiny
    tc = (_PANO_PRECISION == "tf32" and K >= 32 and a.stride(0) % 4 == 0 and b.stride(0) % 4 == 0
          and a.data_ptr() % 16 == 0 and b.data_ptr() % 16 == 0)
    fn, name = (_lib.load().nv_gemm_tf32, "nv_gemm_tf32") if tc else (_lib.load().nv_sgemm, "nv_sgemm")
    check(fn(ptr(a), i64(a.stride(0)), i32(ta), ptr(b), i64(b.stride(0)), i32(tb), ptr(out),
             i64(out.stride(0)), ptr(bias), i32(M), i32(N), i32(K), i32(accumulate), stream_ptr()), name)
    return out


def layernorm_fwd(x, gamma, beta, eps, *, addend=None, out=None, save_stats=True):
    _f32_2d(x, "x")
    R, D = x.shape
    if out is None:
        out = torch.empty((R, D), dtype=f32_t, device=x.device)
    mean = torch.empty((R,), dtype=f32_t, device=x.device) if save_stats else None
    rstd = torch.empty((R,), dtype=f32_t, device=x.device) if save_stats else None
    check(_lib.load().nv_layernorm_fwd(ptr(x), i64(x.stride(0)), ptr(gamma), ptr(beta), ptr(addend),
                                       i64(addend.stride(0) if addend is not None else 0), ptr(out), i64(out.stride(0)),
                                       ptr(mean), ptr(rstd), i32(R), i32(D), f32(eps), stream_ptr()), "nv_layernorm_fwd")
    return out, mean, rstd


def layernorm_bwd(x, gamma, mean, rstd, dy, *, dx=None, accumulate_dx=False, dgamma=None, dbeta=None):
    _f32_2d(x, "x"); _f32_2d(dy, "dy")
    R, D = x.shape
    lib = _lib.load()
    if dx is None:
        assert not accumulate_dx
        dx = torch.empty((R, D), dtype=f32_t, device=x.device)
    ws = _workspace(x.device, lib.nv_layernorm_bwd_partials() * 2 * D)
    check(lib.nv_layernorm_bwd(ptr(x), i64(x.stride(0)), ptr(gamma), ptr(mean), ptr(rstd), ptr(dy), i64(dy.stride(0)),
                               ptr(dx), i64(dx.stride(0)), i32(accumulate_dx), ptr(dgamma), ptr(dbeta), ptr(ws), i32(R),
                               i32(D), stream_ptr()), "nv_layernorm_bwd")
    return dx


def colsum_(src, dst, accumulate=True):
    _f32_2d(src, "src")
    check(_lib.load().nv_colsum_f32(ptr(src), i64(src.stride(0)), i32(src.shape[0]), i32(src.shape[1]), ptr(dst),
                                    i32(accumulate), stream_ptr()), "nv_colsum_f32")
    return dst


def gelu_fwd(z):
    a = torch.empty_like(z)
    check(_lib.load().nv_gelu_fwd(ptr(z), ptr(a), i64(z.numel()), stream_ptr()), "nv_gelu_fwd")
    return a


def gelu_bwd(z, da):
    dz = torch.empty_like(z)
    check(_lib.load().nv_gelu_bwd(ptr(z), ptr(da), ptr(dz), i64(z.numel()), stream_ptr()), "nv_gelu_bwd")
    return dz


def mha_fwd(qkv, lens, n_heads, *, save_probs=True):
    """qkv: [B, N, 3E] fp32 contiguous; lens: int32 [B].  Returns (out [B,N,E], P [B,H,N,N] or None)."""
    B, N, E3 = qkv.shape
    E = E3 // 3
    assert qkv.is_contiguous() and qkv.dtype == f32_t and lens.dtype == torch.int32
    out = torch.empty((B, N, E), dtype=f32_t, device=qkv.device)
    P = torch.empty((B, n_heads, N, N), dtype=f32_t, device=qkv.device) if save_probs else None
    check(_lib.load().nv_mha_fwd(ptr(qkv), ptr(lens), ptr(out), ptr(P), i32(B), i32(N), i32(n_heads), i32(E // n_heads),
                                 stream_ptr()), "nv_mha_fwd")
    return out, P


def dropout(x: torch.Tensor, p: float, seed: int, *, out: torch.Tensor | None = None) -> torch.Tensor:
    """out = keep ? x / (1 - p) : 0 with keep(i) = hash(seed, i) >= p * 2^32 (fp32, contiguous).  Applying it with the same
    seed to the upstream gradient is the backward."""
    assert x.dtype == f32_t and x.is_contiguous() and x.is_cuda
    if out is None:
        out = torch.empty_like(x)
    check(_lib.load().nv_dropout(ptr(x), ptr(out), i64(x.numel()), f32(p), ctypes.c_uint64(seed & (2 ** 64 - 1)), stream_ptr()),
          "nv_dropout")
    return out


def mha_fwd_dropout(qkv, lens, n_heads, p: float, seed: int):
    """Train-mode attention with probability dropout: returns (out, P, Pd)."""
    B, N, E3 = qkv.shape
    E = E3 // 3
    assert qkv.is_contiguous() and qkv.dtype == f32_t and lens.dtype == torch.int32
    out = torch.empty((B, N, E), dtype=f32_t, device=qkv.device)
    P = torch.empty((B, n_heads, N, N), dtype=f32_t, device=qkv.device)
    Pd = torch.empty_like(P)
    check(_lib.load().nv_mha_fwd_dropout(ptr(qkv), ptr(lens), ptr(out), ptr(P), ptr(Pd), i32(B), i32(N), i32(n_heads),
                                         i32(E // n_heads), f32(p), ctypes.c_uint64(seed & (2 ** 64 - 1)), stream_ptr()),
          "nv_mha_fwd_dropout")
    return out, P, Pd


def mha_bwd_dropout(qkv, dout, P, Pd, lens, n_heads):
    B, N, E3 = qkv.shape
    E = E3 // 3
    assert dout.is_contiguous() and P.is_contiguous() and Pd.is_contiguous()
    dqkv = torch.empty_like(qkv)
    dS = torch.empty_like(P)
    check(_lib.load().nv_mha_bwd_dropout(ptr(qkv), ptr(dout), ptr(P), ptr(Pd), ptr(dS), ptr(dqkv), ptr(lens), i32(B), i32(N),
                                         i32(n_heads), i32(E // n_heads), stream_ptr()), "nv_mha_bwd_dropout")
    return dqkv


def mha_bwd(qkv, dout, P, lens, n_heads):
    B, N, E3 = qkv.shape
    E = E3 // 3
    assert dout.is_contiguous() and P.is_contiguous()
    dqkv = torch.empty_like(qkv)
    dS = torch.empty_like(P)
    check(_lib.load().nv_mha_bwd(ptr(qkv), ptr(dout), ptr(P), ptr(dS), ptr(dqkv), ptr(lens), i32(B), i32(N), i32(n_heads),
                                 i32(E // n_heads), stream_ptr()), "nv_mha_bwd")
    return dqkv


def rows_combine(out, a=None, ia=None, alpha=1.0, b=None, ib=None, beta=1.0, accumulate=False):
    """out[r] = (accumulate ? out[r] : 0) + alpha*a[ia[r]] + beta*b[ib[r]]  (index < 0 -> nothing; ia None -> r)."""
    _f32_2d(out, "out")
    R, D = out.shape
    check(_lib.load().nv_rows_combine(ptr(out), i64(out.stride(0)), ptr(a), i64(a.stride(0) if a is not None else 0), ptr(ia),
                                      f32(alpha), ptr(b), i64(b.stride(0) if b is not None else 0), ptr(ib), f32(beta),
                                      i32(R), i32(D), i32(accumulate), stream_ptr()), "nv_rows_combine")
    return out


def rows_scatter_add_(dst, idx, src, alpha=1.0):
    _f32_2d(dst, "dst"); _f32_2d(src, "src")
    check(_lib.load().nv_rows_scatter_add(ptr(dst), i64(dst.stride(0)), ptr(idx), ptr(src), i64(src.stride(0)), f32(alpha),
                                          i32(src.shape[0]), i32(src.shape[1]), stream_ptr()), "nv_rows_scatter_add")
    return dst


def logit_scatter_fwd(pred, slot, B, G):
    out = torch.empty((B, G), dtype=bf16, device=pred.device)
    check(_lib.load().nv_logit_scatter_fwd(ptr(pred), i32(pred.shape[1]), ptr(slot), ptr(out), i32(B), i32(G), stream_ptr()),
          "nv_logit_scatter_fwd")
    return out


def logit_scatter_bwd(dout, slot, O):
    B, G = dout.shape
    dpred = torch.zeros((B, O), dtype=bf16, device=dout.device)
    check(_lib.load().nv_logit_scatter_bwd(ptr(dout), ptr(slot), ptr(dpred), i32(O), i32(B), i32(G), stream_ptr()),
          "nv_logit_scatter_bwd")
    return dpred


# ---------------------------------------------------------------------------------------------------
# decode-phase kernels (csrc/decode.cu)
# ---------------------------------------------------------------------------------------------------
def kv_store_prefill(qkv, cu, kc, vc, B, T):
    Smax, HD = kc.shape[1], kc.shape[2]
    check(_lib.load().nv_kv_store_prefill(ptr(qkv), i64(qkv.stride(0)), ptr(cu), ptr(kc), ptr(vc), i32(B), i32(T), i32(Smax),
                                          i32(HD), stream_ptr()), "nv_kv_store_prefill")


def kv_store_suffix(qkv, cu, cached, kc, vc, B, T):
    """Store the K/V column blocks of the packed new rows after the `cached[b]` rows the cache holds for sequence b."""
    Smax, HD = kc.shape[1], kc.shape[2]
    check(_lib.load().nv_kv_store_suffix(ptr(qkv), i64(qkv.stride(0)), ptr(cu), ptr(cached), ptr(kc), ptr(vc), i32(B), i32(T),
                                         i32(Smax), i32(HD), stream_ptr()), "nv_kv_store_suffix")


def kv_append(qkv, lens, kc, vc):
    B, Smax, HD = kc.shape
    check(_lib.load().nv_kv_append(ptr(qkv), i64(qkv.stride(0)), ptr(lens), ptr(kc), ptr(vc), i32(B), i32(Smax), i32(HD),
                                   stream_ptr()), "nv_kv_append")


def decode_attn(q, kc, vc, lens, n_heads, *, out=None, scale=None):
    """q: [B, >=H*128] bf16 view (first H*128 columns used); caches [B, Smax, H*128]; lens: int32 [B] = index of the
    new token (already appended).  Returns [B, H*128] bf16."""
    B, Smax, HD = kc.shape
    if out is None:
        out = torch.empty((B, HD), dtype=bf16, device=q.device)
    if scale is None:
        scale = 128 ** -0.5
    check(_lib.load().nv_decode_attn(ptr(q), i64(q.stride(0)), ptr(kc), ptr(vc), ptr(lens), ptr(out), i64(out.stride(0)),
                                     i32(B), i32(Smax), i32(n_heads), i32(128), f32(scale), stream_ptr()), "nv_decode_attn")
    return out


def decode_attn_rope(qkv, lens, cos_t, sin_t, kc, vc, n_heads, *, out=None, scale=None):
    """decode_rope_kv_ + decode_attn in ONE launch: qkv [B, 3*H*128] bf16 PRE-RoPE (not modified), lens int32 [B] = position of
    the new token; the rotated k and the v are appended to the caches at row lens[b].  Returns [B, H*128] bf16."""
    B, Smax, HD = kc.shape
    if out is None:
        out = torch.empty((B, HD), dtype=bf16, device=qkv.device)
    if scale is None:
        scale = 128 ** -0.5
    check(_lib.load().nv_decode_attn_rope(ptr(qkv), i64(qkv.stride(0)), ptr(lens), ptr(cos_t), ptr(sin_t), ptr(kc), ptr(vc), ptr(out),
                                          i64(out.stride(0)), i32(B), i32(Smax), i32(n_heads), i32(128), f32(scale), stream_ptr()),
          "nv_decode_attn_rope")
    return out


def _fp8_cache(kq, ke, name):
    """kq: float8_e4m3fn [B, Smax, H*128] contiguous, ke: int8 [B, Smax, H] contiguous (the fp8 KV cache of one layer)."""
    if kq.dtype != torch.float8_e4m3fn or ke.dtype != torch.int8 or kq.dim() != 3 or not kq.is_contiguous() \
            or not ke.is_contiguous() or kq.shape[2] % 128 or tuple(ke.shape) != (kq.shape[0], kq.shape[1], kq.shape[2] // 128):
        raise ValueError(f"{name}: float8_e4m3fn [B, Smax, H*128] cache with int8 [B, Smax, H] exponents expected "
                         f"(got {kq.dtype} {tuple(kq.shape)}, {ke.dtype} {tuple(ke.shape)})")


def _fp8_kv(kq, vq, ke, ve, name):
    _fp8_cache(kq, ke, name)
    _fp8_cache(vq, ve, name)
    if kq.shape != vq.shape:
        raise ValueError(f"{name}: K cache {tuple(kq.shape)} and V cache {tuple(vq.shape)} differ")
    return kq.shape


def kv_store_prefill_fp8(qkv, cu, kq, vq, ke, ve, B, T):
    """``kv_store_prefill`` into an fp8 cache (include/navillm_b200.h): every stored (token, head) row of K and V is rounded
    to e4m3 with its own power-of-two exponent, the bytes ``quantize_fp8_`` writes for that row."""
    _, Smax, HD = _fp8_kv(kq, vq, ke, ve, "kv_store_prefill_fp8")
    if qkv.dtype != bf16 or qkv.stride(1) != 1 or qkv.shape[1] < 3 * HD:
        raise ValueError(f"kv_store_prefill_fp8: qkv bf16 [T, >= {3 * HD}] rows expected (got {qkv.dtype} {tuple(qkv.shape)})")
    check(_lib.load().nv_kv_store_prefill_fp8(ptr(qkv), i64(qkv.stride(0)), ptr(cu), ptr(kq), ptr(vq), ptr(ke), ptr(ve), i32(B), i32(T),
                                              i32(Smax), i32(HD // 128), stream_ptr()), "nv_kv_store_prefill_fp8")


def kv_store_suffix_fp8(qkv, cu, cached, kq, vq, ke, ve, B, T):
    """``kv_store_suffix`` into an fp8 cache: the new rows of sequence b go after its ``cached[b]`` rows, each (token, head)
    row of K and V rounded to e4m3 with its own power-of-two exponent, the bytes ``quantize_fp8_`` writes for that row."""
    _, Smax, HD = _fp8_kv(kq, vq, ke, ve, "kv_store_suffix_fp8")
    if qkv.dtype != bf16 or qkv.stride(1) != 1 or qkv.shape[1] < 3 * HD:
        raise ValueError(f"kv_store_suffix_fp8: qkv bf16 [T, >= {3 * HD}] rows expected (got {qkv.dtype} {tuple(qkv.shape)})")
    for name, t, n in (("cu_seqlens", cu, B + 1), ("cached", cached, B)):
        if t.dtype != torch.int32 or t.numel() != n or not t.is_cuda:
            raise ValueError(f"kv_store_suffix_fp8: {name} int32 [{n}] on the device expected (got {t.dtype} {tuple(t.shape)})")
    check(_lib.load().nv_kv_store_suffix_fp8(ptr(qkv), i64(qkv.stride(0)), ptr(cu), ptr(cached), ptr(kq), ptr(vq), ptr(ke), ptr(ve),
                                             i32(B), i32(T), i32(Smax), i32(HD // 128), stream_ptr()), "nv_kv_store_suffix_fp8")


def attn_fwd_kv_fp8(q: torch.Tensor, kq, vq, ke, ve, cu_q: torch.Tensor, q_lens, kv_start: torch.Tensor, kv_len: torch.Tensor,
                    n_heads: int, *, out: torch.Tensor | None = None, scale: float | None = None):
    """``attn_fwd_kv`` over an fp8 cache (kq / vq float8_e4m3fn [B, Smax, H*128], ke / ve int8 [B, Smax, H]): bit for bit
    ``attn_fwd_kv`` on bf16 caches holding the rounded rows K' / V'.  Rows past kv_len must widen to finite values (a zeroed
    cache, or rows a store wrote).  Returns o [Tq, H*128] bf16."""
    Bc, Smax, HD = _fp8_kv(kq, vq, ke, ve, "attn_fwd_kv_fp8")
    B = len(q_lens)
    Tq = int(sum(int(l) for l in q_lens))
    if HD != n_heads * 128 or q.dtype != bf16 or q.dim() != 2 or q.stride(1) != 1 or q.shape[1] < HD or q.shape[0] != Tq:
        raise ValueError(f"attn_fwd_kv_fp8: q bf16 [{Tq}, >= {HD}] and {HD // 128} heads expected "
                         f"(got {q.dtype} {tuple(q.shape)}, {n_heads} heads)")
    for name, t, n in (("cu_q", cu_q, B + 1), ("kv_start", kv_start, B), ("kv_len", kv_len, B)):
        if t.dtype != torch.int32 or t.numel() != n or not t.is_cuda:
            raise ValueError(f"attn_fwd_kv_fp8: {name} int32 [{n}] on the device expected (got {t.dtype} {tuple(t.shape)})")
    if out is None:
        out = torch.empty((Tq, HD), dtype=bf16, device=q.device)
    if out.dtype != bf16 or out.stride(1) != 1 or tuple(out.shape) != (Tq, HD):
        raise ValueError(f"attn_fwd_kv_fp8: out bf16 [{Tq}, {HD}] expected (got {out.dtype} {tuple(out.shape)})")
    if scale is None:
        scale = 128 ** -0.5
    check(_lib.load().nv_attn_fwd_kv_fp8(ptr(q), i64(q.stride(0)), ptr(kq), ptr(vq), ptr(ke), ptr(ve), ptr(out), i64(out.stride(0)),
                                         ptr(None), ptr(cu_q), ptr(kv_start), ptr(kv_len), i32(B), i32(Tq), i32(Bc * Smax),
                                         i32(n_heads), i32(128), i32(_qblocks(q_lens)), f32(scale), stream_ptr()),
          "nv_attn_fwd_kv_fp8")
    return out


def attn_fwd_tree_fp8(q: torch.Tensor, kq, vq, ke, ve, cu_q: torch.Tensor, q_lens, kv_start: torch.Tensor, kv_len: torch.Tensor,
                      tree_end: torch.Tensor, n_heads: int, *, out: torch.Tensor | None = None, scale: float | None = None):
    """``attn_fwd_tree`` over an fp8 cache (the layout of ``attn_fwd_kv_fp8``): bit for bit ``attn_fwd_tree`` on bf16 caches
    holding the rounded rows K' / V'.  Returns o [Tq, H*128] bf16."""
    Bc, Smax, HD = _fp8_kv(kq, vq, ke, ve, "attn_fwd_tree_fp8")
    B = len(q_lens)
    Tq = int(sum(int(l) for l in q_lens))
    if HD != n_heads * 128 or q.dtype != bf16 or q.dim() != 2 or q.stride(1) != 1 or q.shape[1] < HD or q.shape[0] != Tq:
        raise ValueError(f"attn_fwd_tree_fp8: q bf16 [{Tq}, >= {HD}] and {HD // 128} heads expected "
                         f"(got {q.dtype} {tuple(q.shape)}, {n_heads} heads)")
    for name, t, n in (("cu_q", cu_q, B + 1), ("kv_start", kv_start, B), ("kv_len", kv_len, B)):
        if t.dtype != torch.int32 or t.numel() != n or not t.is_cuda:
            raise ValueError(f"attn_fwd_tree_fp8: {name} int32 [{n}] on the device expected (got {t.dtype} {tuple(t.shape)})")
    _tree_args("attn_fwd_tree_fp8", q_lens, tree_end)
    if out is None:
        out = torch.empty((Tq, HD), dtype=bf16, device=q.device)
    if out.dtype != bf16 or out.stride(1) != 1 or tuple(out.shape) != (Tq, HD):
        raise ValueError(f"attn_fwd_tree_fp8: out bf16 [{Tq}, {HD}] expected (got {out.dtype} {tuple(out.shape)})")
    if scale is None:
        scale = 128 ** -0.5
    check(_lib.load().nv_attn_fwd_tree_fp8(ptr(q), i64(q.stride(0)), ptr(kq), ptr(vq), ptr(ke), ptr(ve), ptr(out), i64(out.stride(0)),
                                           ptr(None), ptr(cu_q), ptr(kv_start), ptr(kv_len), ptr(tree_end), i32(B), i32(Tq),
                                           i32(Bc * Smax), i32(n_heads), i32(128), i32(_qblocks(q_lens)), f32(scale), stream_ptr()),
          "nv_attn_fwd_tree_fp8")
    return out


def decode_attn_rope_fp8(qkv, lens, cos_t, sin_t, kq, vq, ke, ve, n_heads, *, out=None, scale=None):
    """``decode_attn_rope`` over an fp8 cache: the rotated k and the v of the new token are rounded to e4m3 (one exponent per
    head row) as they are appended at row lens[b]; the output equals ``decode_attn_rope`` on a bf16 cache holding the rounded
    rows K' / V', bit for bit.  Returns [B, H*128] bf16."""
    B, Smax, HD = _fp8_kv(kq, vq, ke, ve, "decode_attn_rope_fp8")
    if HD != n_heads * 128 or qkv.dtype != bf16 or qkv.stride(1) != 1 or tuple(qkv.shape) != (B, 3 * HD):
        raise ValueError(f"decode_attn_rope_fp8: qkv bf16 [{B}, {3 * HD}] and {HD // 128} heads expected "
                         f"(got {qkv.dtype} {tuple(qkv.shape)}, {n_heads} heads)")
    if lens.dtype != torch.int32 or lens.numel() != B:
        raise ValueError(f"decode_attn_rope_fp8: lens int32 [{B}] expected (got {lens.dtype} {tuple(lens.shape)})")
    if out is None:
        out = torch.empty((B, HD), dtype=bf16, device=qkv.device)
    if out.dtype != bf16 or out.stride(1) != 1 or tuple(out.shape) != (B, HD):
        raise ValueError(f"decode_attn_rope_fp8: out bf16 [{B}, {HD}] expected (got {out.dtype} {tuple(out.shape)})")
    if scale is None:
        scale = 128 ** -0.5
    check(_lib.load().nv_decode_attn_rope_fp8(ptr(qkv), i64(qkv.stride(0)), ptr(lens), ptr(cos_t), ptr(sin_t), ptr(kq), ptr(vq), ptr(ke),
                                              ptr(ve), ptr(out), i64(out.stride(0)), i32(B), i32(Smax), i32(n_heads), i32(128), f32(scale),
                                              stream_ptr()), "nv_decode_attn_rope_fp8")
    return out


def _window_args(name, qkv, lens, B, W, HD, n_heads, out):
    if not 1 <= W <= LOOKUP_WMAX:
        raise ValueError(f"{name}: window of {W} rows (1 .. {LOOKUP_WMAX} expected)")
    if HD != n_heads * 128 or qkv.dtype != bf16 or qkv.stride(1) != 1 or tuple(qkv.shape) != (B * W, 3 * HD):
        raise ValueError(f"{name}: qkv bf16 [{B * W}, {3 * HD}] and {HD // 128} heads expected (got {qkv.dtype} {tuple(qkv.shape)}, "
                         f"{n_heads} heads)")
    if lens.dtype != torch.int32 or lens.numel() != B or not lens.is_cuda:
        raise ValueError(f"{name}: lens int32 [{B}] on the device expected (got {lens.dtype} {tuple(lens.shape)})")
    if out is None:
        out = torch.empty((B * W, HD), dtype=bf16, device=qkv.device)
    if out.dtype != bf16 or out.stride(1) != 1 or tuple(out.shape) != (B * W, HD):
        raise ValueError(f"{name}: out bf16 [{B * W}, {HD}] expected (got {out.dtype} {tuple(out.shape)})")
    return out


def decode_attn_rope_window(qkv, lens, cos_t, sin_t, kc, vc, n_heads, W, *, out=None, scale=None):
    """``decode_attn_rope`` for W consecutive new tokens per sequence (nv_decode_attn_rope_window): qkv [B * W, 3*H*128] bf16
    PRE-RoPE, row b * W + r at position lens[b] + r; the rotated k and the v of every row go to cache rows lens[b] + r, and query
    r attends over keys 0 .. lens[b] + r.  Bit for bit W sequential ``decode_attn_rope`` calls.  Returns [B * W, H*128] bf16."""
    B, Smax, HD = kc.shape
    if kc.dtype != bf16 or vc.shape != kc.shape or vc.dtype != bf16:
        raise ValueError(f"decode_attn_rope_window: bf16 caches [B, Smax, {HD}] expected")
    out = _window_args("decode_attn_rope_window", qkv, lens, B, W, HD, n_heads, out)
    check(_lib.load().nv_decode_attn_rope_window(ptr(qkv), i64(qkv.stride(0)), ptr(lens), ptr(cos_t), ptr(sin_t), ptr(kc), ptr(vc),
                                                 ptr(out), i64(out.stride(0)), i32(B), i32(W), i32(Smax), i32(n_heads), i32(128),
                                                 f32(128 ** -0.5 if scale is None else scale), stream_ptr()),
          "nv_decode_attn_rope_window")
    return out


def decode_attn_rope_window_fp8(qkv, lens, cos_t, sin_t, kq, vq, ke, ve, n_heads, W, *, out=None, scale=None):
    """``decode_attn_rope_window`` over an fp8 cache: bit for bit W sequential ``decode_attn_rope_fp8`` calls."""
    B, Smax, HD = _fp8_kv(kq, vq, ke, ve, "decode_attn_rope_window_fp8")
    out = _window_args("decode_attn_rope_window_fp8", qkv, lens, B, W, HD, n_heads, out)
    check(_lib.load().nv_decode_attn_rope_window_fp8(ptr(qkv), i64(qkv.stride(0)), ptr(lens), ptr(cos_t), ptr(sin_t), ptr(kq), ptr(vq),
                                                     ptr(ke), ptr(ve), ptr(out), i64(out.stride(0)), i32(B), i32(W), i32(Smax),
                                                     i32(n_heads), i32(128), f32(128 ** -0.5 if scale is None else scale),
                                                     stream_ptr()), "nv_decode_attn_rope_window_fp8")
    return out


def _beam_io(name, B, K, G, **ts):
    """Dtype / shape / device checks of the beam-search state (include/navillm_b200.h, nv_beam_*)."""
    want = {"cand_score": (torch.float32, (B, 2 * K)), "cand_tok": (torch.int32, (B, 2 * K)), "cand_parent": (torch.int32, (B, 2 * K)),
            "beam_score": (torch.float32, (B * K,)), "hist": (torch.int32, (B * K, G)), "src": (torch.int32, (B * K, G)),
            "hyp_score": (torch.float64, (B, K + 1)), "hyp_meta": (torch.int32, (B, K, 2)), "hyp_tok": (torch.int32, (B, K, G)),
            "prompt_state": (torch.int32, (B, 5)), "next_ids": (torch.int32, (B * K,)), "lens": (torch.int32, (B * K,)),
            "norm": (torch.float64, (G,)),
            "plens": (torch.int32, (B,))}
    for k, t in ts.items():
        dt, shape = want[k]
        if t.dtype != dt or tuple(t.shape) != shape or not t.is_cuda or not t.is_contiguous():
            raise ValueError(f"{name}: {k} {dt} {list(shape)} contiguous on the device expected (got {t.dtype} {tuple(t.shape)})")


def _scores_io(name, scores, rows: int, V: int, step=None, step_numel: int = 1):
    """(ptr, ld, plane) of a per-step scores buffer: bf16 [G, >= rows, V] planes with unit inner stride (``scores_buffer``)."""
    if scores.dtype != bf16 or scores.dim() != 3 or scores.shape[1] < rows or scores.shape[2] != V or scores.stride(2) != 1 or \
            not scores.is_cuda:
        raise ValueError(f"{name}: scores bf16 [G, >= {rows}, {V}] with unit inner stride expected (got {scores.dtype} "
                         f"{tuple(scores.shape)})")
    if step is not None and (step.dtype != torch.int32 or step.numel() < step_numel or not step.is_cuda):
        raise ValueError(f"{name}: step int32 [>= {step_numel}] on the device expected")
    return ptr(scores), i64(scores.stride(1)), i64(scores.stride(0))


def scores_buffer(planes: int, rows: int, V: int, device) -> torch.Tensor:
    """Uninitialised bf16 [planes, rows, V] per-step scores whose rows start 16-byte aligned (``logits_buffer``'s stride)."""
    return torch.empty((planes, rows, (V + 63) // 64 * 64), dtype=bf16, device=device)[:, :, :V]


def scores_store(src, special, scores, step):
    """Rows of bf16 ``src`` [R, V] to plane ``step[0]`` (int32 on the device, read at run time) of ``scores`` [G, >= R, V], the
    special ids -inf (nv_scores_store)."""
    R, V = src.shape
    if src.dtype != bf16 or src.stride(1) != 1:
        raise ValueError(f"scores_store: bf16 src with unit inner stride expected (got {src.dtype})")
    args = _scores_io("scores_store", scores, R, V, step)
    check(_lib.load().nv_scores_store(ptr(src), i64(src.stride(0)), i32(V), ptr(special), i32(special.numel()), *args, ptr(step),
                                      i32(R), stream_ptr()), "nv_scores_store")


def lookup_scores(logits, special, n_prev, n_out, W, scores):
    """After ``lookup_accept``: logits row b * W + j of each token prompt b emitted in the step goes to plane n_prev[b] + j,
    row b of ``scores`` [G, >= B, V], special ids -inf (nv_lookup_scores)."""
    B = n_out.numel()
    V = logits.shape[1]
    for name, t in (("n_prev", n_prev), ("n_out", n_out)):
        if t.dtype != torch.int32 or t.numel() != B or not t.is_cuda:
            raise ValueError(f"lookup_scores: {name} int32 [{B}] on the device expected")
    args = _scores_io("lookup_scores", scores, B, V)
    check(_lib.load().nv_lookup_scores(ptr(logits), i64(logits.stride(0)), i32(V), ptr(special), i32(special.numel()), ptr(n_prev),
                                       ptr(n_out), i32(W), *args, i32(B), stream_ptr()), "nv_lookup_scores")


def beam_topk(logits, special, beam_score, K, cand_score, cand_tok, cand_parent, *, first_step=False, scores=None,
              prompt_state=None):
    """The 2K best next-token candidates of each prompt (nv_beam_topk): logits bf16 [B * K, V] (beam k of prompt b in row
    b * K + k), or with ``first_step`` [>= B, V] holding one prefill row per prompt that all K beams read.  beam_score fp32
    [B * K].  Writes cand_score fp32, cand_tok and cand_parent int32 [B, 2K], best first.  With ``scores`` (bf16 [G, B * K, V])
    each beam's bf16 log-probs also go to plane prompt_state[b, 0] (nv_beam_topk_scores)."""
    B = cand_score.shape[0]
    V = logits.shape[1]
    if logits.dtype != bf16 or logits.stride(1) != 1 or logits.shape[0] < (B if first_step else B * K):
        raise ValueError(f"beam_topk: bf16 logits with {B if first_step else B * K} rows expected (got {logits.dtype} {tuple(logits.shape)})")
    _beam_io("beam_topk", B, K, 1, cand_score=cand_score, cand_tok=cand_tok, cand_parent=cand_parent, beam_score=beam_score)
    ld = logits.stride(0)
    if scores is not None:
        check(_lib.load().nv_beam_topk_scores(ptr(logits), i64(ld if first_step else K * ld), i64(0 if first_step else ld), i32(V),
                                              ptr(special), i32(special.numel()), ptr(beam_score), ptr(cand_score), ptr(cand_tok),
                                              ptr(cand_parent), ptr(prompt_state),
                                              *_beam_scores_io("beam_topk", scores, prompt_state, B, K, V), i32(B), i32(K),
                                              stream_ptr()), "nv_beam_topk_scores")
        return
    check(_lib.load().nv_beam_topk(ptr(logits), i64(ld if first_step else K * ld), i64(0 if first_step else ld), i32(V), ptr(special),
                                   i32(special.numel()), ptr(beam_score), ptr(cand_score), ptr(cand_tok), ptr(cand_parent), i32(B),
                                   i32(K), stream_ptr()), "nv_beam_topk")


def _beam_scores_io(name, scores, prompt_state, B, K, V):
    if prompt_state is None:
        raise ValueError(f"{name}: scores= needs prompt_state (the plane of beam b is prompt_state[b, 0])")
    _beam_io(name, B, K, 1, prompt_state=prompt_state)
    return _scores_io(name, scores, B * K, V)


def _proc_io(name, V, prompt_ids, prompt_width, hist, proc):
    penalty, ngram, min_length, min_new, eos = proc
    if prompt_ids.dtype != torch.int32 or prompt_ids.dim() != 2 or prompt_ids.stride(1) != 1 or not prompt_ids.is_cuda:
        raise ValueError(f"{name}: prompt_ids int32 [P, >= S] with unit inner stride on the device expected")
    if prompt_width.dtype != torch.int32 or prompt_width.numel() != 1 or not prompt_width.is_cuda:
        raise ValueError(f"{name}: prompt_width int32 [1] on the device expected")
    if hist.dtype != torch.int32 or hist.dim() != 2 or not hist.is_contiguous() or not hist.is_cuda:
        raise ValueError(f"{name}: hist int32 [rows, G] contiguous on the device expected")
    return f32(penalty), i32(ngram), i32(min_length), i32(min_new), i32(eos)


def logits_process_(logits, prompt_ids, prompt_width, hist, hist_len, append, proc, *, rows_per_prompt=1):
    """HF's repetition-penalty / no-repeat-n-gram / min-length / min-new-tokens processors in place on bf16 logits [R, V]
    (nv_logits_process).  proc = (penalty, ngram, min_length, min_new_tokens, eos_id); prompt_ids int32 [P, >= S] (row r reads
    prompt r // rows_per_prompt), prompt_width int32 [1] = S, hist int32 [R, G] and hist_len int32 [R] the generated history;
    ``append`` (int32 [R] or None) is appended to it first."""
    R, V = logits.shape
    if logits.dtype != bf16 or logits.stride(1) != 1:
        raise ValueError(f"logits_process_: bf16 logits with unit inner stride expected (got {logits.dtype})")
    if hist.shape[0] != R or hist_len.dtype != torch.int32 or hist_len.numel() != R or \
            (append is not None and (append.dtype != torch.int32 or append.numel() != R)):
        raise ValueError(f"logits_process_: hist [{R}, G], hist_len / append int32 [{R}] expected")
    args = _proc_io("logits_process_", V, prompt_ids, prompt_width, hist, proc)
    check(_lib.load().nv_logits_process(ptr(logits), i64(logits.stride(0)), i32(V), ptr(prompt_ids), i64(prompt_ids.stride(0)),
                                        ptr(prompt_width), i32(rows_per_prompt), ptr(hist), i32(hist.shape[1]), ptr(hist_len),
                                        ptr(append), *args, i32(R), stream_ptr()), "nv_logits_process")
    return logits


def beam_topk_processed(logits, special, beam_score, K, cand_score, cand_tok, cand_parent, prompt_ids, prompt_width, hist,
                        prompt_state, proc, *, first_step=False, scores=None):
    """``beam_topk`` with the processors of ``logits_process_`` applied to each bf16 log-prob before the beam-score add
    (nv_beam_topk_processed); beam k of prompt b has the history prompt_ids[b, :S] ++ hist[b * K + k, :prompt_state[b, 0]].
    ``scores``: as in ``beam_topk`` (nv_beam_topk_processed_scores)."""
    B = cand_score.shape[0]
    V = logits.shape[1]
    if logits.dtype != bf16 or logits.stride(1) != 1 or logits.shape[0] < (B if first_step else B * K):
        raise ValueError(f"beam_topk_processed: bf16 logits with {B if first_step else B * K} rows expected "
                         f"(got {logits.dtype} {tuple(logits.shape)})")
    _beam_io("beam_topk_processed", B, K, hist.shape[1], cand_score=cand_score, cand_tok=cand_tok, cand_parent=cand_parent,
             beam_score=beam_score, hist=hist, prompt_state=prompt_state)
    args = _proc_io("beam_topk_processed", V, prompt_ids, prompt_width, hist, proc)
    ld = logits.stride(0)
    if scores is not None:
        check(_lib.load().nv_beam_topk_processed_scores(ptr(logits), i64(ld if first_step else K * ld), i64(0 if first_step else ld),
                                                        i32(V), ptr(special), i32(special.numel()), ptr(beam_score), ptr(cand_score),
                                                        ptr(cand_tok), ptr(cand_parent), ptr(prompt_ids), i64(prompt_ids.stride(0)),
                                                        ptr(prompt_width), ptr(hist), i32(hist.shape[1]), ptr(prompt_state), *args,
                                                        *_beam_scores_io("beam_topk_processed", scores, prompt_state, B, K, V), i32(B),
                                                        i32(K), stream_ptr()), "nv_beam_topk_processed_scores")
        return
    check(_lib.load().nv_beam_topk_processed(ptr(logits), i64(ld if first_step else K * ld), i64(0 if first_step else ld), i32(V),
                                             ptr(special), i32(special.numel()), ptr(beam_score), ptr(cand_score), ptr(cand_tok),
                                             ptr(cand_parent), ptr(prompt_ids), i64(prompt_ids.stride(0)), ptr(prompt_width),
                                             ptr(hist), i32(hist.shape[1]), ptr(prompt_state), *args, i32(B), i32(K), stream_ptr()),
          "nv_beam_topk_processed")


PROC_OFF = (1.0, 0, 0, 0, -1)  # the processors' off values: beam_topk_trie without processors


def beam_topk_trie(logits, special, beam_score, K, cand_score, cand_tok, cand_parent, prompt_ids, prompt_width, hist, prompt_state,
                   proc, node_ptr, child_tok, child_node, n_nodes, leaf_tok, *, first_step=False, scores=None):
    """``beam_topk_processed`` followed by the trie mask (nv_beam_topk_trie): every log-prob the trie does not allow at the beam's
    node becomes -inf.  Beam k of prompt b walks its generated tokens hist[b * K + k, :prompt_state[b, 0]] from the root;
    node_ptr / child_tok / child_node: the CSR trie of ``trie_mask`` with n_nodes real nodes plus the dead node n_nodes, leaf_tok
    the token a childless node allows.  ``proc`` = None (or ``PROC_OFF``) runs the trie mask alone.  ``scores``: as in
    ``beam_topk`` (nv_beam_topk_trie_scores)."""
    B = cand_score.shape[0]
    V = logits.shape[1]
    if logits.dtype != bf16 or logits.stride(1) != 1 or logits.shape[0] < (B if first_step else B * K):
        raise ValueError(f"beam_topk_trie: bf16 logits with {B if first_step else B * K} rows expected "
                         f"(got {logits.dtype} {tuple(logits.shape)})")
    _beam_io("beam_topk_trie", B, K, hist.shape[1], cand_score=cand_score, cand_tok=cand_tok, cand_parent=cand_parent,
             beam_score=beam_score, hist=hist, prompt_state=prompt_state)
    args = _proc_io("beam_topk_trie", V, prompt_ids, prompt_width, hist, PROC_OFF if proc is None else proc)
    n_nodes = int(n_nodes)
    for name, t, n in (("node_ptr", node_ptr, n_nodes + 2), ("child_tok", child_tok, None), ("child_node", child_node, None)):
        if t.dtype != torch.int32 or t.dim() != 1 or not t.is_contiguous() or not t.is_cuda or (n is not None and t.numel() < n):
            raise ValueError(f"beam_topk_trie: {name} int32 [{n if n is not None else 'E'}] contiguous on the device expected "
                             f"(got {t.dtype} {tuple(t.shape)})")
    if child_tok.numel() != child_node.numel():
        raise ValueError(f"beam_topk_trie: child_tok [{child_tok.numel()}] and child_node [{child_node.numel()}] differ in length")
    ld = logits.stride(0)
    if scores is not None:
        check(_lib.load().nv_beam_topk_trie_scores(ptr(logits), i64(ld if first_step else K * ld), i64(0 if first_step else ld), i32(V),
                                                   ptr(special), i32(special.numel()), ptr(beam_score), ptr(cand_score), ptr(cand_tok),
                                                   ptr(cand_parent), ptr(prompt_ids), i64(prompt_ids.stride(0)), ptr(prompt_width),
                                                   ptr(hist), i32(hist.shape[1]), ptr(prompt_state), *args, ptr(node_ptr),
                                                   ptr(child_tok), ptr(child_node), i32(n_nodes), i32(leaf_tok),
                                                   *_beam_scores_io("beam_topk_trie", scores, prompt_state, B, K, V), i32(B), i32(K),
                                                   stream_ptr()), "nv_beam_topk_trie_scores")
        return
    check(_lib.load().nv_beam_topk_trie(ptr(logits), i64(ld if first_step else K * ld), i64(0 if first_step else ld), i32(V),
                                        ptr(special), i32(special.numel()), ptr(beam_score), ptr(cand_score), ptr(cand_tok),
                                        ptr(cand_parent), ptr(prompt_ids), i64(prompt_ids.stride(0)), ptr(prompt_width), ptr(hist),
                                        i32(hist.shape[1]), ptr(prompt_state), *args, ptr(node_ptr), ptr(child_tok), ptr(child_node),
                                        i32(n_nodes), i32(leaf_tok), i32(B), i32(K), stream_ptr()), "nv_beam_topk_trie")


def beam_select(cand_score, cand_tok, cand_parent, beam_score, hist, src, hyp_score, hyp_meta, hyp_tok, prompt_state, next_ids, lens,
                norm, eos_id, pad_id, early_stopping, *, trace=None):
    """One BeamSearchScorer.process step on the device (nv_beam_select); norm fp64 [G]: (S + t) ** length_penalty for S padded
    prompt columns (``beam_norm``).  ``trace`` = (par_hist int32 [B * K, G], hyp_par int32 [B, K, G], done_step int32 [B]) also
    keeps 4.28's beam_indices (nv_beam_select_scores)."""
    B, K2 = cand_score.shape
    K, G = K2 // 2, hist.shape[1]
    _beam_io("beam_select", B, K, G, cand_score=cand_score, cand_tok=cand_tok, cand_parent=cand_parent, beam_score=beam_score,
             hist=hist, src=src, hyp_score=hyp_score, hyp_meta=hyp_meta, hyp_tok=hyp_tok, prompt_state=prompt_state,
             next_ids=next_ids, lens=lens, norm=norm)
    if trace is not None:
        par_hist, hyp_par, done_step = trace
        _beam_io("beam_select", B, K, G, hist=par_hist, hyp_tok=hyp_par, plens=done_step)
        check(_lib.load().nv_beam_select_scores(ptr(cand_score), ptr(cand_tok), ptr(cand_parent), ptr(beam_score), ptr(hist), ptr(src),
                                                ptr(hyp_score), ptr(hyp_meta), ptr(hyp_tok), ptr(prompt_state), ptr(next_ids),
                                                ptr(lens), ptr(norm), ptr(par_hist), ptr(hyp_par), ptr(done_step), i32(B), i32(K),
                                                i32(G), i32(eos_id), i32(pad_id), i32(1 if early_stopping else 0), stream_ptr()),
              "nv_beam_select_scores")
        return
    check(_lib.load().nv_beam_select(ptr(cand_score), ptr(cand_tok), ptr(cand_parent), ptr(beam_score), ptr(hist), ptr(src),
                                     ptr(hyp_score), ptr(hyp_meta), ptr(hyp_tok), ptr(prompt_state), ptr(next_ids), ptr(lens), ptr(norm),
                                     i32(B), i32(K), i32(G), i32(eos_id), i32(pad_id), i32(1 if early_stopping else 0), stream_ptr()),
          "nv_beam_select")


def beam_topk_group(logits, special, beam_score, K, groups, group, cand_score, cand_tok, cand_parent, next_ids, diversity_penalty, *,
                    first_step=False, proc=None, prompt_ids=None, prompt_width=None, hist=None, prompt_state=None, scores=None):
    """Diverse beam search's top-k for group ``group`` of ``groups`` (nv_beam_topk_group[_processed][_scores]): ``beam_topk`` over
    the Kg = K / groups beams group * Kg + [0, Kg) of each prompt, each bf16 log-prob first lowered by diversity_penalty times the
    count of its token among next_ids[b * K + 0 .. group * Kg) (4.28's Hamming diversity).  cand_* [B, 2Kg], parents local to the
    group.  ``proc``: the processors of ``beam_topk_processed`` (prompt_ids, prompt_width, hist, prompt_state); ``scores``: the
    group's rows of plane prompt_state[b, 0], as in ``beam_topk``."""
    B = cand_score.shape[0]
    V = logits.shape[1]
    if not (isinstance(groups, int) and 2 <= groups <= K and K % groups == 0 and 0 <= group < groups):
        raise ValueError(f"beam_topk_group: {K} beams in {groups} groups (group {group}) not supported")
    Kg = K // groups
    if logits.dtype != bf16 or logits.stride(1) != 1 or logits.shape[0] < (B if first_step else B * K):
        raise ValueError(f"beam_topk_group: bf16 logits with {B if first_step else B * K} rows expected "
                         f"(got {logits.dtype} {tuple(logits.shape)})")
    _beam_io("beam_topk_group", B, Kg, 1, cand_score=cand_score, cand_tok=cand_tok, cand_parent=cand_parent)
    _beam_io("beam_topk_group", B, K, 1, beam_score=beam_score, next_ids=next_ids)
    ld = logits.stride(0)
    head = (ptr(logits), i64(ld if first_step else K * ld), i64(0 if first_step else ld), i32(V), ptr(special), i32(special.numel()),
            ptr(beam_score), ptr(cand_score), ptr(cand_tok), ptr(cand_parent))
    tail = (ptr(next_ids), f32(diversity_penalty), i32(group), i32(groups), i32(B), i32(K), stream_ptr())
    sc = () if scores is None else _beam_scores_io("beam_topk_group", scores, prompt_state, B, K, V)
    lib = _lib.load()
    if proc is not None:
        _beam_io("beam_topk_group", B, K, hist.shape[1], hist=hist, prompt_state=prompt_state)
        args = _proc_io("beam_topk_group", V, prompt_ids, prompt_width, hist, proc)
        pa = (ptr(prompt_ids), i64(prompt_ids.stride(0)), ptr(prompt_width), ptr(hist), i32(hist.shape[1]), ptr(prompt_state), *args)
        if scores is not None:
            check(lib.nv_beam_topk_group_processed_scores(*head, *pa, *sc, *tail), "nv_beam_topk_group_processed_scores")
        else:
            check(lib.nv_beam_topk_group_processed(*head, *pa, *tail), "nv_beam_topk_group_processed")
    elif scores is not None:
        check(lib.nv_beam_topk_group_scores(*head, ptr(prompt_state), *sc, *tail), "nv_beam_topk_group_scores")
    else:
        check(lib.nv_beam_topk_group(*head, *tail), "nv_beam_topk_group")


def beam_select_group(cand_score, cand_tok, cand_parent, beam_score, hist, src, hyp_score, hyp_meta, hyp_tok, prompt_state, next_ids,
                      lens, norm, eos_id, pad_id, early_stopping, groups, group, *, trace=None):
    """``beam_select`` over group ``group``'s candidates [B, 2Kg] of ``beam_topk_group`` (nv_beam_select_group[_scores]): process
    with group_size Kg against the prompt's K hypotheses; only the group's rows are reordered and written, and only the last
    group advances prompt_state[:, 0].  ``trace``: as in ``beam_select``, with global rows."""
    B, K = hyp_score.shape[0], hyp_score.shape[1] - 1
    G = hist.shape[1]
    if not (isinstance(groups, int) and 2 <= groups <= K and K % groups == 0 and 0 <= group < groups):
        raise ValueError(f"beam_select_group: {K} beams in {groups} groups (group {group}) not supported")
    _beam_io("beam_select_group", B, K // groups, G, cand_score=cand_score, cand_tok=cand_tok, cand_parent=cand_parent)
    _beam_io("beam_select_group", B, K, G, beam_score=beam_score, hist=hist, src=src, hyp_score=hyp_score, hyp_meta=hyp_meta,
             hyp_tok=hyp_tok, prompt_state=prompt_state, next_ids=next_ids, lens=lens, norm=norm)
    head = (ptr(cand_score), ptr(cand_tok), ptr(cand_parent), ptr(beam_score), ptr(hist), ptr(src), ptr(hyp_score), ptr(hyp_meta),
            ptr(hyp_tok), ptr(prompt_state), ptr(next_ids), ptr(lens), ptr(norm))
    tail = (i32(group), i32(groups), i32(B), i32(K), i32(G), i32(eos_id), i32(pad_id), i32(1 if early_stopping else 0), stream_ptr())
    if trace is not None:
        par_hist, hyp_par, done_step = trace
        _beam_io("beam_select_group", B, K, G, hist=par_hist, hyp_tok=hyp_par, plens=done_step)
        check(_lib.load().nv_beam_select_group_scores(*head, ptr(par_hist), ptr(hyp_par), ptr(done_step), *tail),
              "nv_beam_select_group_scores")
        return
    check(_lib.load().nv_beam_select_group(*head, *tail), "nv_beam_select_group")


def beam_norm(S: int, G: int, length_penalty: float) -> torch.Tensor:
    """The hypothesis normalisers (S + t) ** length_penalty, t < G, in the Python float arithmetic of transformers 4.28's
    BeamHypotheses.add (host fp64 [G]; copy it to the device for ``beam_select``)."""
    return torch.tensor([(S + t) ** length_penalty for t in range(G)], dtype=torch.float64)


def trie_score(logits, special, tok, path_off, path_rows, eos, B, *, logprob=None, stats=None):
    """The log-probability of every answer of a trie under each of B prompts (nv_trie_score).  logits bf16 [B * R, V] (unit inner
    stride): row b * R the prompt's next-token logits, row b * R + 1 + j those after tree row j (``trie.tree_rows``).  tok int32
    [R - 1] the rows' tokens; path_off int32 [A + 1] / path_rows int32 the answers' rows, root to leaf; eos ends every answer.
    Each log-prob is ``beam_topk``'s bf16 one, folded along the path in fp32.  Returns logprob fp32 [B, A]."""
    V = logits.shape[1]
    if logits.dtype != bf16 or logits.dim() != 2 or logits.stride(1) != 1 or not logits.is_cuda or B < 1 or logits.shape[0] % B:
        raise ValueError(f"trie_score: bf16 logits [B * R, V] with unit inner stride on the device expected for B = {B} "
                         f"(got {logits.dtype} {tuple(logits.shape)})")
    R = logits.shape[0] // B
    A = path_off.numel() - 1
    for name, t, n in (("tok", tok, R - 1), ("path_off", path_off, None), ("path_rows", path_rows, None)):
        if t.dtype != torch.int32 or t.dim() != 1 or not t.is_contiguous() or not t.is_cuda or (n is not None and t.numel() != n):
            raise ValueError(f"trie_score: {name} int32 [{n if n is not None else 'n'}] contiguous on the device expected "
                             f"(got {t.dtype} {tuple(t.shape)})")
    if A < 1 or not 0 <= int(eos) < V:
        raise ValueError(f"trie_score: {A} answers (>= 1) and eos {eos} in [0, {V}) expected")
    if special.dtype != torch.int32 or not special.is_cuda:
        raise ValueError("trie_score: special int32 on the device expected")
    if logprob is None:
        logprob = torch.empty((B, A), dtype=torch.float32, device=logits.device)
    if logprob.dtype != torch.float32 or tuple(logprob.shape) != (B, A) or not logprob.is_contiguous():
        raise ValueError(f"trie_score: logprob fp32 [{B}, {A}] contiguous expected (got {logprob.dtype} {tuple(logprob.shape)})")
    if stats is None:
        stats = torch.empty((B * R, 2), dtype=torch.float32, device=logits.device)
    check(_lib.load().nv_trie_score(ptr(logits), i64(logits.stride(0)), i32(V), ptr(special), i32(special.numel()), ptr(tok),
                                    ptr(path_off), ptr(path_rows), i32(eos), ptr(stats), ptr(logprob), i32(B), i32(R), i32(A),
                                    stream_ptr()), "nv_trie_score")
    return logprob


def _beam_attn_args(name, qkv, lens, plens, src, R, K, HD, n_heads, out):
    if HD != n_heads * 128 or qkv.dtype != bf16 or qkv.stride(1) != 1 or tuple(qkv.shape) != (R, 3 * HD):
        raise ValueError(f"{name}: qkv bf16 [{R}, {3 * HD}] and {HD // 128} heads expected (got {qkv.dtype} {tuple(qkv.shape)}, "
                         f"{n_heads} heads)")
    if R % K:
        raise ValueError(f"{name}: {R} beam rows is not a multiple of {K} beams")
    _beam_io(name, R // K, K, src.shape[1], lens=lens, plens=plens, src=src)
    if out is None:
        out = torch.empty((R, HD), dtype=bf16, device=qkv.device)
    if out.dtype != bf16 or out.stride(1) != 1 or tuple(out.shape) != (R, HD):
        raise ValueError(f"{name}: out bf16 [{R}, {HD}] expected (got {out.dtype} {tuple(out.shape)})")
    return out


def decode_attn_rope_beam(qkv, lens, cos_t, sin_t, pk, pv, plens, kc, vc, src, K, n_heads, *, out=None, scale=None):
    """``decode_attn_rope`` for R = B * K beam rows (nv_decode_attn_rope_beam): keys [0, plens[b]) from the prompt cache pk / pv
    [B, Sp, H*128] shared by the K beams of prompt b, generated key i of row r from kc / vc [R, G, H*128] at row (src[r, i], i).
    The new k / v are written at (r, lens[r] - plens[r // K]).  Returns [R, H*128] bf16."""
    R, G, HD = kc.shape
    if pk.shape[2] != HD or vc.shape != kc.shape or pv.shape != pk.shape or pk.dtype != bf16 or kc.dtype != bf16:
        raise ValueError(f"decode_attn_rope_beam: bf16 caches [B, Sp, {HD}] / [R, G, {HD}] expected")
    out = _beam_attn_args("decode_attn_rope_beam", qkv, lens, plens, src, R, K, HD, n_heads, out)
    check(_lib.load().nv_decode_attn_rope_beam(ptr(qkv), i64(qkv.stride(0)), ptr(lens), ptr(cos_t), ptr(sin_t), ptr(pk), ptr(pv),
                                               i32(pk.shape[1]), ptr(plens), ptr(kc), ptr(vc), ptr(src), i32(G), ptr(out),
                                               i64(out.stride(0)), i32(R), i32(K), i32(n_heads), i32(128),
                                               f32(128 ** -0.5 if scale is None else scale), stream_ptr()), "nv_decode_attn_rope_beam")
    return out


def decode_attn_rope_beam_fp8(qkv, lens, cos_t, sin_t, pk, pv, pke, pve, plens, kq, vq, ke, ve, src, K, n_heads, *, out=None,
                              scale=None):
    """``decode_attn_rope_beam`` over fp8 caches (the format of ``decode_attn_rope_fp8``): bit for bit the bf16 beam kernel on
    caches holding the rounded rows K' / V'."""
    _fp8_kv(pk, pv, pke, pve, "decode_attn_rope_beam_fp8")
    R, G, HD = _fp8_kv(kq, vq, ke, ve, "decode_attn_rope_beam_fp8")
    if pk.shape[2] != HD:
        raise ValueError(f"decode_attn_rope_beam_fp8: prompt cache width {pk.shape[2]} != {HD}")
    out = _beam_attn_args("decode_attn_rope_beam_fp8", qkv, lens, plens, src, R, K, HD, n_heads, out)
    check(_lib.load().nv_decode_attn_rope_beam_fp8(ptr(qkv), i64(qkv.stride(0)), ptr(lens), ptr(cos_t), ptr(sin_t), ptr(pk), ptr(pv),
                                                   ptr(pke), ptr(pve), i32(pk.shape[1]), ptr(plens), ptr(kq), ptr(vq), ptr(ke), ptr(ve),
                                                   ptr(src), i32(G), ptr(out), i64(out.stride(0)), i32(R), i32(K), i32(n_heads), i32(128),
                                                   f32(128 ** -0.5 if scale is None else scale), stream_ptr()),
          "nv_decode_attn_rope_beam_fp8")
    return out


def argmax_masked(logits, special, finished, eos_id, pad_id, stop_on_eos, next_ids):
    B, V = logits.shape
    check(_lib.load().nv_argmax_masked(ptr(logits), i64(logits.stride(0)), i32(V), ptr(special), i32(special.numel()),
                                       ptr(finished), i32(eos_id), i32(pad_id), i32(1 if stop_on_eos else 0), ptr(next_ids),
                                       i32(B), stream_ptr()), "nv_argmax_masked")
    return next_ids


def sample_topk(logits, special, finished, eos_id, pad_id, stop_on_eos, temperature, top_k, u, next_ids, probs_out=None):
    """One sampled token per row (nv_sample_topk): logits [B, V] bf16, u [B] fp32 uniform in [0, 1)."""
    B, V = logits.shape
    assert logits.dtype == bf16 and logits.stride(1) == 1 and u.dtype == torch.float32 and u.numel() == B
    assert next_ids.dtype == torch.int32 and finished.dtype == torch.int32
    if probs_out is not None:
        assert probs_out.dtype == torch.float32 and probs_out.shape == (B, V) and probs_out.is_contiguous()
    check(_lib.load().nv_sample_topk(ptr(logits), i64(logits.stride(0)), i32(V), ptr(special), i32(special.numel()), ptr(finished),
                                     i32(eos_id), i32(pad_id), i32(1 if stop_on_eos else 0), f32(temperature), i32(top_k), ptr(u),
                                     ptr(next_ids), ptr(probs_out), i32(B), stream_ptr()), "nv_sample_topk")
    return next_ids


def sample(logits, special, finished, eos_id, pad_id, stop_on_eos, temperature, top_k, top_p, u, next_ids, probs_out=None, *,
           scores=None, step=None):
    """``sample_topk`` with top-p filtering after top-k (nv_sample); ``top_p`` in [0, 1], 1 is off.  With ``scores`` (bf16
    [G, >= B, V]) the warped bf16 scores (-inf outside the kept set) also go to plane ``step[0]`` (nv_sample_scores)."""
    B, V = logits.shape
    assert logits.dtype == bf16 and logits.stride(1) == 1 and u.dtype == torch.float32 and u.numel() == B
    assert next_ids.dtype == torch.int32 and finished.dtype == torch.int32
    if probs_out is not None:
        assert probs_out.dtype == torch.float32 and probs_out.shape == (B, V) and probs_out.is_contiguous()
    if scores is not None:
        args = _scores_io("sample", scores, B, V, step)
        check(_lib.load().nv_sample_scores(ptr(logits), i64(logits.stride(0)), i32(V), ptr(special), i32(special.numel()),
                                           ptr(finished), i32(eos_id), i32(pad_id), i32(1 if stop_on_eos else 0), f32(temperature),
                                           i32(top_k), f32(top_p), ptr(u), ptr(next_ids), ptr(probs_out), *args, ptr(step), i32(B),
                                           stream_ptr()), "nv_sample_scores")
        return next_ids
    check(_lib.load().nv_sample(ptr(logits), i64(logits.stride(0)), i32(V), ptr(special), i32(special.numel()), ptr(finished),
                                i32(eos_id), i32(pad_id), i32(1 if stop_on_eos else 0), f32(temperature), i32(top_k), f32(top_p),
                                ptr(u), ptr(next_ids), ptr(probs_out), i32(B), stream_ptr()), "nv_sample")
    return next_ids


def trie_mask(logits, out, node_ptr, child_tok, child_node, n_nodes, leaf_tok, special, state, last, miss):
    """out = logits masked to the tokens the trie allows per row (nv_trie_mask); advances ``state`` by ``last`` first
    unless ``last`` is None.  logits / out [B, V] bf16, state / last int32 [B], miss int32 [1] (set on a miss, never
    cleared); node_ptr / child_tok / child_node: the CSR trie with n_nodes real nodes plus the dead node n_nodes."""
    B, V = logits.shape
    assert out.shape == (B, V) and out.dtype == bf16 and logits.dtype == bf16 and logits.stride(1) == 1 and out.stride(1) == 1
    assert state.dtype == torch.int32 and miss.dtype == torch.int32 and (last is None or last.dtype == torch.int32)
    check(_lib.load().nv_trie_mask(ptr(logits), i64(logits.stride(0)), ptr(out), i64(out.stride(0)), i32(V), ptr(node_ptr),
                                   ptr(child_tok), ptr(child_node), i32(n_nodes), i32(leaf_tok), ptr(special),
                                   i32(0 if special is None else special.numel()), ptr(state), ptr(last), ptr(miss), i32(B),
                                   stream_ptr()), "nv_trie_mask")
    return out


CONTRASTIVE_KMAX = 64          # candidates per prompt the contrastive-search kernels are built for


def _dev_t(t, dtype, shape, name, what):
    if t.dtype != dtype or tuple(t.shape) != tuple(shape) or not t.is_cuda or not t.is_contiguous():
        raise ValueError(f"{name}: {what} {dtype} {list(shape)} contiguous on the device expected (got {t.dtype} {tuple(t.shape)})")


def contrastive_topk(logits, special, K, p, tok):
    """The K most probable tokens per row (nv_contrastive_topk): p = bf16(softmax(logits)) with the special ids at -inf, largest p
    first, equal p by lower token id.  logits bf16 [B, V] (unit inner stride); writes p bf16 and tok int32 [B, K]."""
    B, V = logits.shape
    if logits.dtype != bf16 or logits.stride(1) != 1 or not logits.is_cuda:
        raise ValueError(f"contrastive_topk: bf16 logits with unit inner stride on the device expected (got {logits.dtype})")
    _dev_t(p, bf16, (B, K), "contrastive_topk", "p")
    _dev_t(tok, torch.int32, (B, K), "contrastive_topk", "tok")
    check(_lib.load().nv_contrastive_topk(ptr(logits), i64(logits.stride(0)), i32(V), ptr(special), i32(special.numel()), i32(K),
                                          ptr(p), ptr(tok), i32(B), stream_ptr()), "nv_contrastive_topk")


def contrastive_context(hn, cu, ctx, ctx_len):
    """ctx[b, :len_b] = bf16(x / bf16(||x||)) of the packed final-norm prompt rows hn [T, D] (cu_seqlens ``cu`` int32 [B + 1]),
    ctx_len[b] = len_b (nv_contrastive_context).  ctx bf16 [B, Sc, D]."""
    T, D = hn.shape
    B, Sc = ctx.shape[0], ctx.shape[1]
    _dev_t(hn, bf16, (T, D), "contrastive_context", "hn")
    _dev_t(ctx, bf16, (B, Sc, D), "contrastive_context", "ctx")
    _dev_t(ctx_len, torch.int32, (B,), "contrastive_context", "ctx_len")
    _dev_t(cu, torch.int32, (B + 1,), "contrastive_context", "cu")
    check(_lib.load().nv_contrastive_context(ptr(hn), ptr(cu), i32(B), i32(T), ptr(ctx), ptr(ctx_len), i32(Sc), i32(D), stream_ptr()),
          "nv_contrastive_context")


def contrastive_rank(hn, ctx, ctx_len, pen_key, p, tok, alpha, finished, eos_id, pad_id, stop_on_eos, next_ids, sel, hsel, plens, lens,
                     pen_out=None, score_out=None):
    """One contrastive-search selection (nv_contrastive_rank): the candidates' final-norm rows hn bf16 [B * K, D] against the
    context ctx bf16 [B, Sc, D] (ctx_len int32 [B] rows each), their p bf16 / tok int32 [B, K] from ``contrastive_topk`` ->
    next_ids, sel int32 [B], finished updated, the selected row's x^ appended to ctx, the row copied to hsel bf16 [B, D], plens
    int32 [B] and lens int32 [B * K] advanced.  pen_key int32 [B * K] zero before and after; pen_out / score_out fp32 [B, K]."""
    B, K = p.shape
    Sc, D = ctx.shape[1], ctx.shape[2]
    name = "contrastive_rank"
    _dev_t(hn, bf16, (B * K, D), name, "hn")
    _dev_t(ctx, bf16, (B, Sc, D), name, "ctx")
    _dev_t(hsel, bf16, (B, D), name, "hsel")
    _dev_t(p, bf16, (B, K), name, "p")
    for what, t, n in (("ctx_len", ctx_len, B), ("pen_key", pen_key, B * K), ("finished", finished, B), ("next_ids", next_ids, B),
                       ("sel", sel, B), ("plens", plens, B), ("lens", lens, B * K)):
        _dev_t(t, torch.int32, (n,), name, what)
    _dev_t(tok, torch.int32, (B, K), name, "tok")
    for what, t in (("pen_out", pen_out), ("score_out", score_out)):
        if t is not None:
            _dev_t(t, torch.float32, (B, K), name, what)
    check(_lib.load().nv_contrastive_rank(ptr(hn), ptr(ctx), ptr(ctx_len), i32(Sc), i32(D), i32(K), ptr(pen_key), ptr(p), ptr(tok),
                                          ctypes.c_double(alpha), ptr(finished), i32(eos_id), i32(pad_id), i32(1 if stop_on_eos else 0),
                                          ptr(next_ids), ptr(sel), ptr(hsel), ptr(plens), ptr(lens), ptr(pen_out), ptr(score_out), i32(B),
                                          stream_ptr()), "nv_contrastive_rank")


def contrastive_commit_table(kc, vc, pk, pv) -> torch.Tensor:
    """The per-layer pointer table of ``contrastive_commit`` for the candidate caches kc / vc [B * K, 1, D] and the prompt caches
    pk / pv [B, Sp, D] (bf16 tensors, or ``(e4m3, exponents)`` pairs per layer): int64 [L, 8] on the device."""
    rows = []
    for layer in zip(kc, vc, pk, pv):
        if isinstance(layer[0], tuple):
            rows.append([c[0].data_ptr() for c in layer] + [c[1].data_ptr() for c in layer])
        else:
            rows.append([c.data_ptr() for c in layer] + [0] * 4)
    dev = (kc[0][0] if isinstance(kc[0], tuple) else kc[0]).device
    return torch.tensor(rows, dtype=torch.int64).to(dev)


def contrastive_commit(table, sel, plens, K, Sp, n_heads, fp8):
    """The selected candidate's K / V rows of every layer into row plens[b] - 1 of the prompt caches (nv_contrastive_commit);
    ``table`` from ``contrastive_commit_table`` (the tensors behind it must outlive the call)."""
    B = sel.numel()
    _dev_t(sel, torch.int32, (B,), "contrastive_commit", "sel")
    _dev_t(plens, torch.int32, (B,), "contrastive_commit", "plens")
    if table.dtype != torch.int64 or table.dim() != 2 or table.shape[1] != 8 or not table.is_cuda:
        raise ValueError("contrastive_commit: an int64 [L, 8] pointer table on the device expected")
    check(_lib.load().nv_contrastive_commit(ptr(table), i32(table.shape[0]), ptr(sel), ptr(plens), i32(K), i32(Sp), i32(n_heads * 128),
                                            i32(n_heads), i32(1 if fp8 else 0), i32(B), stream_ptr()), "nv_contrastive_commit")


class LayerRunner:
    """Inference forward of decoder layers through nv_llama_layer_infer (csrc/layer.cu): ONE C-ABI call per layer instead of
    ten.  Holds the argument block and a workspace for a given packing; ``run`` fills in what changes per layer."""

    def __init__(self, T: int, D: int, F: int, H: int, eps: float, pos, cos_t, sin_t, cu, B: int, total_qblocks: int, *, R: int = 0,
                 device=None, scale: float | None = None):
        lib = _lib.load()
        lib.nv_llama_layer_ws_bytes.restype = ctypes.c_int64
        self.T, self.D, self.R = T, D, R
        nbytes = max(int(lib.nv_llama_layer_ws_bytes(i32(T), i32(R), i32(D), i32(F))), int(lib.nv_llama_layer_ws_bytes(i32(T), i32(0), i32(D), i32(F))))
        self.ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
        a = _lib.LayerArgs()
        a.pos, a.cos_t, a.sin_t, a.cu_seqlens = pos.data_ptr(), cos_t.data_ptr(), sin_t.data_ptr(), cu.data_ptr()
        a.ws, a.ws_bytes = self.ws.data_ptr(), nbytes
        a.B, a.T, a.total_qblocks, a.D, a.F, a.H = B, T, total_qblocks, D, F, H
        a.eps, a.scale = eps, (128 ** -0.5 if scale is None else scale)
        a.kv_mode = 0
        self.args = a
        self._keep = (pos, cos_t, sin_t, cu)

    def set_cache_mode(self, mode: int, Smax: int, Tkv: int = 0, cached=None, kv_start=None, kv_len=None):
        a = self.args
        a.kv_mode, a.Smax, a.Tkv = mode, Smax, Tkv
        a.cached = cached.data_ptr() if cached is not None else None
        a.kv_start = kv_start.data_ptr() if kv_start is not None else None
        a.kv_len = kv_len.data_ptr() if kv_len is not None else None
        self._keep += (cached, kv_start, kv_len)

    def run(self, x, y, ln1, wqkv, wo, ln2, wgu, wd, *, kc=None, vc=None, out_rows=None, fp8=None, fp8_max_rows=0, ke=None, ve=None,
            act_fp8=False, int4=None, int4_max_rows=0):
        """``fp8``: None, or the (e4m3, exponents) pairs of wqkv, wo, wgu, wd (``Fp8Weights.view``); each GEMM with at most
        ``fp8_max_rows`` rows then streams its pair through nv_gemm_fp8w_bf16 (same bits as the bf16 weights W').
        ``int4``: None, or the (codes, scales, zeros) triples of wqkv, wo, wgu, wd (``Int4Weights.view``; a triple may be
        None); each GEMM with 17..``int4_max_rows`` rows then streams its triple through nv_gemm_int4w_bf16 (same bits as
        W').  Exclusive with ``fp8``.
        ``act_fp8``: every GEMM runs W8A8 on the four pairs of ``fp8`` (all required) at every row count.
        ``ke`` / ``ve``: the row exponents of an fp8 cache (cache modes 3 and 4, kc / vc then hold its e4m3 bytes)."""
        a = self.args
        pairs = fp8 if fp8 is not None else ((None, None),) * 4
        (a.wqkv_q, a.wqkv_e), (a.wo_q, a.wo_e), (a.wgu_q, a.wgu_e), (a.wd_q, a.wd_e) = \
            [(q.data_ptr(), e.data_ptr()) if q is not None else (None, None) for q, e in pairs]
        a.fp8_max_rows = fp8_max_rows if fp8 is not None else 0
        a.act_fp8 = 1 if act_fp8 else 0
        triples = int4 if int4 is not None else (None,) * 4
        for name, tr in zip(("wqkv", "wo", "wgu", "wd"), triples):
            c, sc, z = (t.data_ptr() for t in tr) if tr is not None else (None, None, None)
            setattr(a, name + "_c", c); setattr(a, name + "_s", sc); setattr(a, name + "_z", z)
        a.int4_max_rows = int4_max_rows if int4 is not None else 0
        a.x, a.y = x.data_ptr(), y.data_ptr()
        a.ln1, a.wqkv, a.wo, a.ln2, a.wgu, a.wd = ln1.data_ptr(), wqkv.data_ptr(), wo.data_ptr(), ln2.data_ptr(), wgu.data_ptr(), wd.data_ptr()
        a.kcache = kc.data_ptr() if kc is not None else None
        a.vcache = vc.data_ptr() if vc is not None else None
        if a.kv_mode in (3, 4):
            _fp8_kv(kc, vc, ke, ve, "LayerRunner.run")
        a.kexp = ke.data_ptr() if ke is not None else None
        a.vexp = ve.data_ptr() if ve is not None else None
        if out_rows is not None:
            a.out_rows, a.R = out_rows.data_ptr(), out_rows.numel()
        else:
            a.out_rows, a.R = None, 0
        check(_lib.load().nv_llama_layer_infer(ctypes.byref(a), stream_ptr()), "nv_llama_layer_infer")
        return y


class fixed_splits:
    """Context: the panorama encoder GEMMs (``sgemm``) split K by K alone (nv_set_fixed_splits), so that a row's bits do not
    depend on the batch; used by ``NavModel`` in batch-invariant mode."""

    def __init__(self, on: bool = True):
        self.on = on

    def __enter__(self):
        self.prev = _lib.load().nv_set_fixed_splits(i32(1 if self.on else 0))
        return self

    def __exit__(self, *a):
        _lib.load().nv_set_fixed_splits(i32(self.prev))


class pdl:
    """Context: launch the decode-chain kernels with programmatic dependent launch (nv_set_pdl)."""

    def __init__(self, on: bool = True):
        self.on = on

    def __enter__(self):
        self.prev = _lib.load().nv_set_pdl(i32(1 if self.on else 0))
        return self

    def __exit__(self, *a):
        _lib.load().nv_set_pdl(i32(self.prev))


LOOKUP_WMAX = 16               # verify-window rows per prompt the window kernel is built for (k drafts + 1)


def lookup_draft(hist, hist_len, finished, special, eos_id, ngram, drafts, win_ids):
    """Prompt-lookup drafts (nv_lookup_draft): for each row of the history hist int32 [B, G] (hist_len [B] tokens: the row's
    non-pad prompt ids, then its generated tokens), HF's PromptLookupCandidateGenerator with ``max_matching_ngram_size`` =
    ngram.  Writes drafts int32 [B, k] (-1 past the drafts) and the verify window's ids win_ids int32 [B, k + 1]."""
    B, k = drafts.shape
    _dev_t(hist_len, torch.int32, (B,), "lookup_draft", "hist_len")
    _dev_t(finished, torch.int32, (B,), "lookup_draft", "finished")
    _dev_t(win_ids, torch.int32, (B, k + 1), "lookup_draft", "win_ids")
    _dev_t(drafts, torch.int32, (B, k), "lookup_draft", "drafts")
    if hist.dtype != torch.int32 or hist.dim() != 2 or hist.shape[0] != B or hist.stride(1) != 1 or not hist.is_cuda:
        raise ValueError(f"lookup_draft: hist int32 [{B}, G] on the device expected (got {hist.dtype} {tuple(hist.shape)})")
    check(_lib.load().nv_lookup_draft(ptr(hist), i32(hist.stride(0)), ptr(hist_len), ptr(finished), ptr(special), i32(special.numel()),
                                      i32(eos_id), i32(k), i32(ngram), ptr(drafts), ptr(win_ids), i32(B), stream_ptr()),
          "nv_lookup_draft")


def lookup_accept(logits, special, drafts, finished, eos_id, stop_on_eos, max_new, out, hist, hist_len, n_out, lens, n_acc):
    """Verify a window (nv_lookup_accept): logits bf16 [B * (k + 1), V], row b * (k + 1) + j the prediction after window token j.
    Each unfinished row emits the masked argmax t_0 .. t_m of its rows while drafts[b, j] = t_j, cut after EOS (stop_on_eos) and
    at max_new tokens, into out int32 [B, >= max_new] at n_out[b] and into hist at hist_len[b]; lens advances by the tokens
    emitted, n_acc by the accepted drafts, and finished is set once a row is done."""
    B, k = drafts.shape
    V = logits.shape[1]
    if logits.dtype != bf16 or logits.stride(1) != 1 or logits.shape[0] != B * (k + 1):
        raise ValueError(f"lookup_accept: bf16 logits [{B * (k + 1)}, V] expected (got {logits.dtype} {tuple(logits.shape)})")
    for name, t in (("finished", finished), ("hist_len", hist_len), ("n_out", n_out), ("lens", lens), ("n_acc", n_acc)):
        _dev_t(t, torch.int32, (B,), "lookup_accept", name)
    _dev_t(drafts, torch.int32, (B, k), "lookup_accept", "drafts")
    for name, t in (("out", out), ("hist", hist)):
        if t.dtype != torch.int32 or t.dim() != 2 or t.shape[0] != B or t.stride(1) != 1 or not t.is_cuda:
            raise ValueError(f"lookup_accept: {name} int32 [{B}, n] on the device expected (got {t.dtype} {tuple(t.shape)})")
    check(_lib.load().nv_lookup_accept(ptr(logits), i64(logits.stride(0)), i32(V), ptr(special), i32(special.numel()), ptr(drafts),
                                       i32(k), ptr(finished), i32(eos_id), i32(1 if stop_on_eos else 0), i32(max_new), ptr(out),
                                       i32(out.shape[1]), ptr(hist), i32(hist.stride(0)), ptr(hist_len), ptr(n_out), ptr(lens),
                                       ptr(n_acc), i32(B), stream_ptr()), "nv_lookup_accept")


def add_int_(x, delta):
    check(_lib.load().nv_add_int(ptr(x), i32(x.numel()), i32(delta), stream_ptr()), "nv_add_int")
    return x


# ---------------------------------------------------------------------------------------------------
# fused-epilogue GEMMs on the 128 x 256 tile (csrc/gemm_bf16.cu)
# ---------------------------------------------------------------------------------------------------
def _timed(fn, flops, nbytes):
    timer = gemm_timer
    if timer is None:
        return fn()
    st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    st.record()
    r = fn()
    en.record()
    timer.append((st, en, flops, nbytes))
    return r


def gemm_skinny(x: torch.Tensor, w: torch.Tensor, *, addend: torch.Tensor | None = None,
                out: torch.Tensor | None = None) -> torch.Tensor:
    """Decode-step linear: x [M<=16, K] bf16, w [N, K] bf16 (nn.Linear weight) -> bf16 [M, N] (+ addend)."""
    _rowmajor(x, "x"); _rowmajor(w, "w")
    assert x.dtype == bf16 and w.dtype == bf16
    M, K = x.shape
    N = w.shape[0]
    if w.shape[1] != K or M > 16:
        raise ValueError(f"gemm_skinny: x {tuple(x.shape)} w {tuple(w.shape)} (needs M <= 16 and matching K)")
    if out is None:
        out = torch.empty((M, N), dtype=bf16, device=x.device)
    _rowmajor(out, "out")
    if addend is not None:
        _rowmajor(addend, "addend")
        assert addend.shape == (M, N) and addend.dtype == bf16
    check(_lib.load().nv_gemm_skinny_bf16(ptr(x), i64(x.stride(0)), ptr(w), i64(w.stride(0)), ptr(out), i64(out.stride(0)),
                                          ptr(addend), i64(addend.stride(0) if addend is not None else 0),
                                          i32(M), i32(N), i32(K), stream_ptr()), "nv_gemm_skinny_bf16")
    return out


def gemm_skinny_swiglu(x: torch.Tensor, wgu: torch.Tensor, *, out: torch.Tensor | None = None) -> torch.Tensor:
    """Decode-step gate/up projection + SwiGLU: x [M<=16, K], wgu [2F, K] -> h [M, F] bf16 (gate|up never materialised)."""
    _rowmajor(x, "x"); _rowmajor(wgu, "wgu")
    M, K = x.shape
    F = wgu.shape[0] // 2
    if wgu.shape[1] != K or M > 16 or F % 64:
        raise ValueError(f"gemm_skinny_swiglu: x {tuple(x.shape)} wgu {tuple(wgu.shape)} (needs M <= 16, F % 64 == 0)")
    if out is None:
        out = torch.empty((M, F), dtype=bf16, device=x.device)
    check(_lib.load().nv_gemm_skinny_swiglu_bf16(ptr(x), i64(x.stride(0)), ptr(wgu), i64(wgu.stride(0)), ptr(out), i64(out.stride(0)),
                                                 i32(M), i32(F), i32(K), stream_ptr()), "nv_gemm_skinny_swiglu_bf16")
    return out


BI_MAX_ROWS = 128           # batch-invariant linears: the weight-streaming kernel up to here, nv_gemm_bf16 above


def gemm_bi(x: torch.Tensor, w: torch.Tensor, *, addend: torch.Tensor | None = None,
            out: torch.Tensor | None = None) -> torch.Tensor:
    """Batch-invariant linear: x [M, K] bf16, w [N, K] bf16 (nn.Linear weight) -> bf16 [M, N] (+ addend), each row's bits a
    function of that row alone.  Up to ``BI_MAX_ROWS`` rows the weight-streaming kernel nv_gemm_bi_bf16 (csrc/gemm_bi.cu),
    above it ``gemm``: the same accumulation chain per element (include/navillm_b200.h)."""
    _rowmajor(x, "x"); _rowmajor(w, "w")
    M, K = x.shape
    N = w.shape[0]
    if x.dtype != bf16 or w.dtype != bf16 or w.shape[1] != K or M == 0:
        raise ValueError(f"gemm_bi: x {x.dtype} {tuple(x.shape)} w {w.dtype} {tuple(w.shape)} (bf16, M > 0, matching K)")
    if M > BI_MAX_ROWS:
        return gemm(x, w, addend=addend, out=out)
    if out is None:
        out = torch.empty((M, N), dtype=bf16, device=x.device)
    _rowmajor(out, "out")
    if out.shape != (M, N) or out.dtype != bf16:
        raise ValueError(f"gemm_bi: out bf16 [{M}, {N}] expected (got {out.dtype} {tuple(out.shape)})")
    if addend is not None:
        _rowmajor(addend, "addend")
        if addend.shape != (M, N) or addend.dtype != bf16:
            raise ValueError(f"gemm_bi: addend bf16 [{M}, {N}] expected (got {addend.dtype} {tuple(addend.shape)})")
    check(_lib.load().nv_gemm_bi_bf16(ptr(x), i64(x.stride(0)), ptr(w), i64(w.stride(0)), ptr(out), i64(out.stride(0)),
                                      ptr(addend), i64(addend.stride(0) if addend is not None else 0),
                                      i32(M), i32(N), i32(K), stream_ptr()), "nv_gemm_bi_bf16")
    return out


def gemm_bi_swiglu(x: torch.Tensor, wgu: torch.Tensor) -> torch.Tensor:
    """Batch-invariant gate|up projection + SwiGLU: x [M, K], wgu [2F, K] -> h [M, F] bf16, bit for bit
    ``swiglu_fwd(gemm_bi(x, wgu))``.  Up to ``BI_MAX_ROWS`` rows with F % 16 == 0 one kernel (gate|up never materialised)."""
    _rowmajor(x, "x"); _rowmajor(wgu, "wgu")
    M, K = x.shape
    F = wgu.shape[0] // 2
    if x.dtype != bf16 or wgu.dtype != bf16 or wgu.shape[1] != K or wgu.shape[0] % 2 or M == 0:
        raise ValueError(f"gemm_bi_swiglu: x {x.dtype} {tuple(x.shape)} wgu {wgu.dtype} {tuple(wgu.shape)}")
    if M > BI_MAX_ROWS or F % 16:
        return swiglu_fwd(gemm_bi(x, wgu))
    out = torch.empty((M, F), dtype=bf16, device=x.device)
    check(_lib.load().nv_gemm_bi_swiglu_bf16(ptr(x), i64(x.stride(0)), ptr(wgu), i64(wgu.stride(0)), ptr(out), i64(out.stride(0)),
                                             i32(M), i32(F), i32(K), stream_ptr()), "nv_gemm_bi_swiglu_bf16")
    return out


fp8 = torch.float8_e4m3fn


def quantize_fp8_(w: torch.Tensor, q: torch.Tensor, exps: torch.Tensor) -> torch.Tensor:
    """Round the bf16 weight w [N, K] in place to W' = e4m3(w / 2^e_n) * 2^e_n with one power-of-two exponent per row
    (csrc/quant.cu, format in include/navillm_b200.h): q [N, K] float8_e4m3fn receives the e4m3 values, exps [N] int8 the
    exponents.  Returns w."""
    _rowmajor(w, "w"); _rowmajor(q, "q")
    if w.dtype != bf16 or q.dtype != fp8 or exps.dtype != torch.int8:
        raise ValueError(f"quantize_fp8_: w bf16, q float8_e4m3fn, exps int8 expected (got {w.dtype}, {q.dtype}, {exps.dtype})")
    N, K = w.shape
    if tuple(q.shape) != (N, K) or exps.shape != (N,) or not exps.is_contiguous():
        raise ValueError(f"quantize_fp8_: w {tuple(w.shape)} q {tuple(q.shape)} exps {tuple(exps.shape)}")
    check(_lib.load().nv_quantize_fp8_rows(ptr(w), i64(w.stride(0)), ptr(q), i64(q.stride(0)), ptr(exps), i32(N), i32(K),
                                           stream_ptr()), "nv_quantize_fp8_rows")
    return w


def _fp8_weight(wq: torch.Tensor, exps: torch.Tensor, name: str) -> None:
    _rowmajor(wq, name)
    if wq.dtype != fp8 or exps.dtype != torch.int8 or exps.shape != (wq.shape[0],) or not exps.is_contiguous():
        raise ValueError(f"{name}: float8_e4m3fn [N, K] weight with int8 [N] row exponents expected "
                         f"(got {wq.dtype} {tuple(wq.shape)}, {exps.dtype} {tuple(exps.shape)})")


def gemm_skinny_fp8(x: torch.Tensor, wq: torch.Tensor, exps: torch.Tensor, *, addend: torch.Tensor | None = None,
                    out: torch.Tensor | None = None) -> torch.Tensor:
    """``gemm_skinny`` with the weight in the fp8 format of ``quantize_fp8_`` (wq e4m3 [N, K], exps int8 [N]): bit for
    bit ``gemm_skinny(x, W')`` while reading half the weight bytes."""
    _rowmajor(x, "x"); _fp8_weight(wq, exps, "wq")
    assert x.dtype == bf16
    M, K = x.shape
    N = wq.shape[0]
    if wq.shape[1] != K or M > 16:
        raise ValueError(f"gemm_skinny_fp8: x {tuple(x.shape)} wq {tuple(wq.shape)} (needs M <= 16 and matching K)")
    if out is None:
        out = torch.empty((M, N), dtype=bf16, device=x.device)
    _rowmajor(out, "out")
    assert out.shape == (M, N) and out.dtype == bf16
    if addend is not None:
        _rowmajor(addend, "addend")
        assert addend.shape == (M, N) and addend.dtype == bf16
    check(_lib.load().nv_gemm_skinny_fp8(ptr(x), i64(x.stride(0)), ptr(wq), i64(wq.stride(0)), ptr(exps), ptr(out),
                                         i64(out.stride(0)), ptr(addend), i64(addend.stride(0) if addend is not None else 0),
                                         i32(M), i32(N), i32(K), stream_ptr()), "nv_gemm_skinny_fp8")
    return out


def gemm_skinny_swiglu_fp8(x: torch.Tensor, wgu_q: torch.Tensor, exps: torch.Tensor, *,
                           out: torch.Tensor | None = None) -> torch.Tensor:
    """``gemm_skinny_swiglu`` with the fused gate|up weight in fp8 (wgu_q e4m3 [2F, K], exps int8 [2F])."""
    _rowmajor(x, "x"); _fp8_weight(wgu_q, exps, "wgu_q")
    assert x.dtype == bf16
    M, K = x.shape
    F = wgu_q.shape[0] // 2
    if wgu_q.shape[1] != K or M > 16 or F % 64 or wgu_q.shape[0] != 2 * F:
        raise ValueError(f"gemm_skinny_swiglu_fp8: x {tuple(x.shape)} wgu_q {tuple(wgu_q.shape)} (needs M <= 16, F % 64 == 0)")
    if out is None:
        out = torch.empty((M, F), dtype=bf16, device=x.device)
    _rowmajor(out, "out")
    assert out.shape == (M, F) and out.dtype == bf16
    check(_lib.load().nv_gemm_skinny_swiglu_fp8(ptr(x), i64(x.stride(0)), ptr(wgu_q), i64(wgu_q.stride(0)), ptr(exps), ptr(out),
                                                i64(out.stride(0)), i32(M), i32(F), i32(K), stream_ptr()),
          "nv_gemm_skinny_swiglu_fp8")
    return out


INT4_GROUP = 128


def int4_codes_shape(n: int, k: int) -> tuple:
    """Shape of the uint8 code buffer ``quantize_int4_`` fills for a weight [n, k]: rows padded to a multiple of 64, two
    codes per byte (in a layout private to csrc/quant.cu and csrc/gemm_skinny.cu)."""
    return ((n + 63) // 64 * 64, k // 2)


def _int4_weight(codes: torch.Tensor, scales: torch.Tensor, zeros: torch.Tensor, n: int, k: int, name: str) -> None:
    if not (codes.is_cuda and scales.is_cuda and zeros.is_cuda):
        raise _lib.NvError(f"{name}: navillm_b200 kernels need CUDA tensors (no CPU fallback)")
    if k % INT4_GROUP:
        raise ValueError(f"{name}: K must be a multiple of {INT4_GROUP} (got {k})")
    if codes.dtype != torch.uint8 or tuple(codes.shape) != int4_codes_shape(n, k) or not codes.is_contiguous():
        raise ValueError(f"{name}: contiguous uint8 codes {int4_codes_shape(n, k)} expected "
                         f"(got {codes.dtype} {tuple(codes.shape)})")
    g = k // INT4_GROUP
    for t, dt, what in ((scales, bf16, "scales"), (zeros, torch.uint8, "zeros")):
        if t.dtype != dt or tuple(t.shape) != (n, g) or not t.is_contiguous():
            raise ValueError(f"{name}: contiguous {dt} {what} [{n}, {g}] expected (got {t.dtype} {tuple(t.shape)})")
    if codes.data_ptr() % 16:
        raise ValueError(f"{name}: codes must be 16-byte aligned")


def quantize_int4_(w: torch.Tensor, codes: torch.Tensor, scales: torch.Tensor, zeros: torch.Tensor) -> torch.Tensor:
    """Round the bf16 weight w [N, K] (K % 128 == 0) in place to W' = bf16((q - z) * s) in groups of one row and 128
    columns (csrc/quant.cu, rule in include/navillm_b200.h): codes (``int4_codes_shape``) receives the 4-bit q, scales
    [N, K / 128] bf16 the s and zeros [N, K / 128] uint8 the z.  Returns w."""
    _rowmajor(w, "w")
    if w.dtype != bf16:
        raise ValueError(f"quantize_int4_: bf16 w expected (got {w.dtype})")
    N, K = w.shape
    _int4_weight(codes, scales, zeros, N, K, "quantize_int4_")
    if w.stride(0) % 8 or w.data_ptr() % 16:
        raise ValueError("quantize_int4_: w must be 16-byte aligned with a row stride that is a multiple of 8")
    check(_lib.load().nv_quantize_int4_groups(ptr(w), i64(w.stride(0)), ptr(codes), ptr(scales), ptr(zeros), i32(N), i32(K),
                                              stream_ptr()), "nv_quantize_int4_groups")
    return w


class CholeskyError(RuntimeError):
    pass


def _gptq_cholesky(h: torch.Tensor, damp: float, what: str) -> torch.Tensor:
    """fp64 lower Cholesky factor of the dampened H: a column no recorded row touched (H_ii = 0) gets H_ii = 1, then
    H += damp * mean(diag H) * I."""
    if h.dim() != 2 or h.shape[0] != h.shape[1] or h.dtype != f32_t or not h.is_cuda:
        raise ValueError(f"gptq_factor: fp32 CUDA H [K, K] expected (got {h.dtype} {tuple(h.shape)} on {h.device})")
    if not damp >= 0.0:
        raise ValueError(f"gptq_factor: damp must be >= 0 (got {damp})")
    H = h.double()
    d = H.diagonal()
    d[d == 0] = 1.0
    d += damp * d.mean()
    L, info = torch.linalg.cholesky_ex(H)
    if int(info) != 0:
        raise CholeskyError(f"GPTQ: the Cholesky factorisation of {what} failed (not positive definite at column "
                            f"{int(info) - 1} with damp={damp}); quantize again with a larger damp")
    return L


def gptq_factor(h: torch.Tensor, damp: float = 0.01, what: str = "the Hessian", check_only: bool = False):
    """U, the upper Cholesky factor of H^-1 (H^-1 = U^T U), fp32 [K, K] on h's device, for ``gptq_int4_``.  In fp64 with
    torch.linalg (a one-off O(K^3) factorisation per linear input): a column no recorded row touched (H_ii = 0) gets
    H_ii = 1, then H += damp * mean(diag H) * I.  Raises ``CholeskyError`` naming ``what`` when H is not positive definite.
    ``check_only``: only the factorisation of H, which is where that shows; returns None."""
    L = _gptq_cholesky(h, damp, what)
    if check_only:
        return None
    U, info = torch.linalg.cholesky_ex(torch.cholesky_inverse(L), upper=True)
    if int(info) != 0:
        raise CholeskyError(f"GPTQ: the Cholesky factorisation of the inverse of {what} failed (column {int(info) - 1} with "
                            f"damp={damp}); quantize again with a larger damp")
    return U.float().contiguous()                # torch returns the upper factor column-major


def gptq_int4_(w: torch.Tensor, h_or_u: torch.Tensor, codes: torch.Tensor, scales: torch.Tensor, zeros: torch.Tensor,
               damp: float | None = 0.01) -> torch.Tensor:
    """``quantize_int4_`` calibrated by GPTQ: the same format and outputs, with each column's rounding error fed forward onto
    the columns not yet rounded so that ||X (W - W')^T|| is what gets minimised (include/navillm_b200.h).  ``h_or_u``: the
    fp32 Hessian H = X^T X [K, K] of the linear's inputs, factored here by ``gptq_factor(h, damp)``, or with ``damp=None``
    the factor U that ``gptq_factor`` returned.  Per 128-column group: one nv_gptq_int4_block launch, then the exact fp32
    CUDA-core nv_sgemm adds -E U[group rows, later columns] to the later columns of an fp32 working copy of w.  w [N, K]
    bf16 with N % 64 == 0 and K % 128 == 0 is overwritten with W'.  Returns w."""
    _rowmajor(w, "w")
    if w.dtype != bf16:
        raise ValueError(f"gptq_int4_: bf16 w expected (got {w.dtype})")
    N, K = w.shape
    if N % 64:
        raise ValueError(f"gptq_int4_: N must be a multiple of 64 (got {N})")
    _int4_weight(codes, scales, zeros, N, K, "gptq_int4_")
    if h_or_u.dtype != f32_t or tuple(h_or_u.shape) != (K, K) or not h_or_u.is_contiguous() or h_or_u.device != w.device:
        raise ValueError(f"gptq_int4_: contiguous fp32 [{K}, {K}] H or U on {w.device} expected (got {h_or_u.dtype} "
                         f"{tuple(h_or_u.shape)} on {h_or_u.device})")
    u = h_or_u if damp is None else gptq_factor(h_or_u, damp)
    wf = w.float()
    ne = torch.empty((N, INT4_GROUP), dtype=f32_t, device=w.device)
    lib, st, G = _lib.load(), stream_ptr(), K // INT4_GROUP
    for g in range(G):
        c0 = g * INT4_GROUP
        check(lib.nv_gptq_int4_block(ptr(wf), i64(K), ptr(u[c0:, c0:]), i64(K), i32(g), ptr(w), i64(w.stride(0)), ptr(codes),
                                     ptr(scales), ptr(zeros), ptr(ne), i64(INT4_GROUP), i32(N), i32(K), st), "nv_gptq_int4_block")
        c1 = c0 + INT4_GROUP
        if c1 < K:
            check(lib.nv_sgemm(ptr(ne), i64(INT4_GROUP), i32(0), ptr(u[c0:, c1:]), i64(K), i32(1), ptr(wf[:, c1:]), i64(K),
                               ptr(None), i32(N), i32(K - c1), i32(INT4_GROUP), i32(1), st), "nv_sgemm")
    return w


def _skinny_x(x: torch.Tensor, k: int, name: str) -> int:
    _rowmajor(x, "x")
    if x.dtype != bf16 or x.dim() != 2 or x.shape[1] != k or not 1 <= x.shape[0] <= 16:
        raise ValueError(f"{name}: x bf16 [M <= 16, {k}] expected (got {x.dtype} {tuple(x.shape)})")
    return x.shape[0]


def gemm_skinny_int4(x: torch.Tensor, codes: torch.Tensor, scales: torch.Tensor, zeros: torch.Tensor, *,
                     addend: torch.Tensor | None = None, out: torch.Tensor | None = None) -> torch.Tensor:
    """``gemm_skinny`` with the weight in the 4-bit format of ``quantize_int4_`` (codes, scales [N, K / 128], zeros
    [N, K / 128]): bit for bit ``gemm_skinny(x, W')`` while reading about a quarter of the weight bytes."""
    if scales.dim() != 2:
        raise ValueError(f"gemm_skinny_int4: scales [N, K / 128] expected (got {tuple(scales.shape)})")
    N, G = scales.shape
    K = G * INT4_GROUP
    _int4_weight(codes, scales, zeros, N, K, "gemm_skinny_int4")
    M = _skinny_x(x, K, "gemm_skinny_int4")
    if out is None:
        out = torch.empty((M, N), dtype=bf16, device=x.device)
    _rowmajor(out, "out")
    if out.shape != (M, N) or out.dtype != bf16:
        raise ValueError(f"gemm_skinny_int4: out bf16 [{M}, {N}] expected (got {out.dtype} {tuple(out.shape)})")
    if addend is not None:
        _rowmajor(addend, "addend")
        if addend.shape != (M, N) or addend.dtype != bf16:
            raise ValueError(f"gemm_skinny_int4: addend bf16 [{M}, {N}] expected (got {addend.dtype} {tuple(addend.shape)})")
    check(_lib.load().nv_gemm_skinny_int4(ptr(x), i64(x.stride(0)), ptr(codes), ptr(scales), ptr(zeros), ptr(out),
                                          i64(out.stride(0)), ptr(addend), i64(addend.stride(0) if addend is not None else 0),
                                          i32(M), i32(N), i32(K), stream_ptr()), "nv_gemm_skinny_int4")
    return out


def gemm_skinny_swiglu_int4(x: torch.Tensor, codes: torch.Tensor, scales: torch.Tensor, zeros: torch.Tensor, *,
                            out: torch.Tensor | None = None) -> torch.Tensor:
    """``gemm_skinny_swiglu`` with the fused gate|up weight [2F, K] in the 4-bit format (F % 64 == 0)."""
    if scales.dim() != 2:
        raise ValueError(f"gemm_skinny_swiglu_int4: scales [2F, K / 128] expected (got {tuple(scales.shape)})")
    N2, G = scales.shape
    K, F = G * INT4_GROUP, N2 // 2
    if N2 != 2 * F or F % 64:
        raise ValueError(f"gemm_skinny_swiglu_int4: gate|up [2F, K] with F % 64 == 0 expected (got {N2} rows)")
    _int4_weight(codes, scales, zeros, N2, K, "gemm_skinny_swiglu_int4")
    M = _skinny_x(x, K, "gemm_skinny_swiglu_int4")
    if out is None:
        out = torch.empty((M, F), dtype=bf16, device=x.device)
    _rowmajor(out, "out")
    if out.shape != (M, F) or out.dtype != bf16:
        raise ValueError(f"gemm_skinny_swiglu_int4: out bf16 [{M}, {F}] expected (got {out.dtype} {tuple(out.shape)})")
    check(_lib.load().nv_gemm_skinny_swiglu_int4(ptr(x), i64(x.stride(0)), ptr(codes), ptr(scales), ptr(zeros), ptr(out),
                                                 i64(out.stride(0)), i32(M), i32(F), i32(K), stream_ptr()),
          "nv_gemm_skinny_swiglu_int4")
    return out


def gemm_fp8w(a: torch.Tensor, q: torch.Tensor, e: torch.Tensor, *, addend: torch.Tensor | None = None,
              out: torch.Tensor | None = None, block_n: int = 0) -> torch.Tensor:
    """``gemm(a, W', addend=addend, block_n=block_n)`` with the weight in the fp8 format of ``quantize_fp8_`` (q e4m3 [N, K],
    e int8 [N]; W' = q * 2^e): bit for bit the same result at any M while reading half the weight bytes (csrc/gemm_bf16.cu).
    block_n: 0 (auto), 32 or 128."""
    _rowmajor(a, "a"); _fp8_weight(q, e, "q")
    assert a.dtype == bf16
    M, K = a.shape
    N = q.shape[0]
    if q.shape[1] != K:
        raise ValueError(f"gemm_fp8w: contraction mismatch a {tuple(a.shape)} q {tuple(q.shape)}")
    if out is None:
        out = torch.empty((M, N), dtype=bf16, device=a.device)
    _rowmajor(out, "out")
    assert out.shape == (M, N) and out.dtype == bf16
    if addend is not None:
        _rowmajor(addend, "addend")
        assert addend.shape == (M, N) and addend.dtype == bf16
    check(_lib.load().nv_gemm_fp8w_bf16(ptr(a), i64(a.stride(0)), ptr(q), i64(q.stride(0)), ptr(e), ptr(out), i64(out.stride(0)),
                                        ptr(addend), i64(addend.stride(0) if addend is not None else 0), i32(M), i32(N), i32(K),
                                        i32(block_n), stream_ptr()), "nv_gemm_fp8w_bf16")
    return out


def gemm_int4w(a: torch.Tensor, codes: torch.Tensor, scales: torch.Tensor, zeros: torch.Tensor, *,
               addend: torch.Tensor | None = None, out: torch.Tensor | None = None, block_n: int = 0) -> torch.Tensor:
    """``gemm(a, W', addend=addend, block_n=block_n)`` with the weight in the 4-bit format of ``quantize_int4_`` (codes,
    scales [N, K / 128], zeros [N, K / 128]): bit for bit the same result at any M while reading about a quarter of the
    weight bytes (csrc/gemm_bf16.cu).  N % 64 == 0.  block_n: 0 (auto), 32 or 128."""
    if scales.dim() != 2:
        raise ValueError(f"gemm_int4w: scales [N, K / 128] expected (got {tuple(scales.shape)})")
    N, G = scales.shape
    K = G * INT4_GROUP
    if N % 64:
        raise ValueError(f"gemm_int4w: N must be a multiple of 64 (got {N})")
    _int4_weight(codes, scales, zeros, N, K, "gemm_int4w")
    _rowmajor(a, "a")
    if a.dtype != bf16 or a.dim() != 2 or a.shape[1] != K or a.shape[0] < 1:
        raise ValueError(f"gemm_int4w: a bf16 [M, {K}] expected (got {a.dtype} {tuple(a.shape)})")
    if a.stride(0) % 8 or a.data_ptr() % 16:
        raise ValueError("gemm_int4w: a must be 16-byte aligned with a row stride that is a multiple of 8")
    if block_n not in (0, 32, 128):
        raise ValueError(f"gemm_int4w: block_n must be 0, 32 or 128 (got {block_n})")
    M = a.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=bf16, device=a.device)
    _rowmajor(out, "out")
    if out.shape != (M, N) or out.dtype != bf16 or out.data_ptr() % 16:
        raise ValueError(f"gemm_int4w: 16-byte aligned out bf16 [{M}, {N}] expected (got {out.dtype} {tuple(out.shape)})")
    if addend is not None:
        _rowmajor(addend, "addend")
        if addend.shape != (M, N) or addend.dtype != bf16 or addend.data_ptr() % 16:
            raise ValueError(f"gemm_int4w: 16-byte aligned addend bf16 [{M}, {N}] expected "
                             f"(got {addend.dtype} {tuple(addend.shape)})")
    check(_lib.load().nv_gemm_int4w_bf16(ptr(a), i64(a.stride(0)), ptr(codes), ptr(scales), ptr(zeros), ptr(out),
                                         i64(out.stride(0)), ptr(addend), i64(addend.stride(0) if addend is not None else 0),
                                         i32(M), i32(N), i32(K), i32(block_n), stream_ptr()), "nv_gemm_int4w_bf16")
    return out


def quantize_act_fp8(x: torch.Tensor, *, q: torch.Tensor | None = None, e: torch.Tensor | None = None):
    """Quantize the bf16 activation x [M, K] (any row stride, K % 128 == 0) per (row, 128-column block) with the rule of
    ``quantize_fp8_`` (csrc/gemm_fp8.cu): returns (q float8_e4m3fn [M, K], e int8 [M, K / 128]) with
    x ~ q * 2^e[:, k // 128].  x is not modified."""
    _rowmajor(x, "x")
    if x.dtype != bf16:
        raise ValueError(f"quantize_act_fp8: bf16 input expected (got {x.dtype})")
    M, K = x.shape
    if K % 128:
        raise ValueError(f"quantize_act_fp8: K must be a multiple of 128 (got {K})")
    if q is None:
        q = torch.empty((M, K), dtype=fp8, device=x.device)
    if e is None:
        e = torch.empty((M, K // 128), dtype=torch.int8, device=x.device)
    _rowmajor(q, "q"); _rowmajor(e, "e")
    if q.dtype != fp8 or e.dtype != torch.int8 or tuple(q.shape) != (M, K) or tuple(e.shape) != (M, K // 128):
        raise ValueError(f"quantize_act_fp8: q float8_e4m3fn [M, K] and e int8 [M, K/128] expected "
                         f"(got {q.dtype} {tuple(q.shape)}, {e.dtype} {tuple(e.shape)})")
    check(_lib.load().nv_quantize_act_fp8(ptr(x), i64(x.stride(0)), ptr(q), i64(q.stride(0)), ptr(e), i64(e.stride(0)), i32(M),
                                          i32(K), stream_ptr()), "nv_quantize_act_fp8")
    return q, e


def gemm_w8a8(aq: torch.Tensor, ae: torch.Tensor, wq: torch.Tensor, we: torch.Tensor, *, addend: torch.Tensor | None = None,
              out: torch.Tensor | None = None) -> torch.Tensor:
    """C [M, N] = A' · W'^T (+ addend) on the e4m3 tensor cores (csrc/gemm_fp8.cu): A' = (aq, ae) from ``quantize_act_fp8``,
    W' = (wq, we) in the weight format of ``quantize_fp8_``; bf16 output, C = bf16(bf16(acc) + addend).  A row's output does
    not depend on M or on the other rows."""
    _fp8_weight(wq, we, "wq"); _rowmajor(aq, "aq"); _rowmajor(ae, "ae")
    M, K = aq.shape
    N = wq.shape[0]
    if aq.dtype != fp8 or ae.dtype != torch.int8 or tuple(ae.shape) != (M, K // 128) or K % 128:
        raise ValueError(f"gemm_w8a8: aq float8_e4m3fn [M, K] (K % 128 == 0) with int8 [M, K/128] exponents expected "
                         f"(got {aq.dtype} {tuple(aq.shape)}, {ae.dtype} {tuple(ae.shape)})")
    if wq.shape[1] != K:
        raise ValueError(f"gemm_w8a8: contraction mismatch aq {tuple(aq.shape)} wq {tuple(wq.shape)}")
    if out is None:
        out = torch.empty((M, N), dtype=bf16, device=aq.device)
    _rowmajor(out, "out")
    assert out.shape == (M, N) and out.dtype == bf16
    if addend is not None:
        _rowmajor(addend, "addend")
        assert addend.shape == (M, N) and addend.dtype == bf16
    lib = _lib.load()
    _timed(lambda: check(lib.nv_gemm_w8a8_bf16(ptr(aq), i64(aq.stride(0)), ptr(ae), i64(ae.stride(0)), ptr(wq), i64(wq.stride(0)),
                                                ptr(we), ptr(out), i64(out.stride(0)), ptr(addend),
                                                i64(addend.stride(0) if addend is not None else 0), i32(M), i32(N), i32(K),
                                                stream_ptr()), "nv_gemm_w8a8_bf16"),
           2.0 * M * N * K, M * K + N * K + 2.0 * M * N * (2 if addend is not None else 1))
    return out


def decode_rope_kv_(qkv, lens, cos_t, sin_t, kc, vc, n_heads):
    """In-place RoPE of the new token's q,k at position lens[b] + append of the rotated K and V to the caches."""
    B, Smax, HD = kc.shape
    check(_lib.load().nv_decode_rope_kv(ptr(qkv), i64(qkv.stride(0)), ptr(lens), ptr(cos_t), ptr(sin_t), ptr(kc), ptr(vc), i32(B),
                                        i32(Smax), i32(n_heads), i32(HD // n_heads), stream_ptr()), "nv_decode_rope_kv")
    return qkv


def gemm_swiglu(x, wgu, *, gu=None, h=None, keep_gu=True):
    """gu = x·Wgu^T ([T,2F]: gate | up) and h = silu(gate)*up ([T,F]) in ONE kernel (SwiGLU epilogue)."""
    _rowmajor(x, "x"); _rowmajor(wgu, "wgu")
    T, K = x.shape
    F = wgu.shape[0] // 2
    if gu is None:
        gu = torch.empty((T, 2 * F), dtype=bf16, device=x.device)
    if h is None:
        h = torch.empty((T, F), dtype=bf16, device=x.device)
    lib = _lib.load()
    _timed(lambda: check(lib.nv_gemm_swiglu_bf16(ptr(x), i64(x.stride(0)), ptr(wgu), i64(wgu.stride(0)), ptr(gu), i64(gu.stride(0)),
                                                  ptr(h), i64(h.stride(0)), i32(T), i32(F), i32(K), i32(1 if keep_gu else 0),
                                                  stream_ptr()), "nv_gemm_swiglu_bf16"),
           2.0 * T * 2 * F * K, 2.0 * (T * K + 2 * F * K + 3 * T * F))
    return gu, h


def gemm_dswiglu(dx, wd, gu, *, dgu=None):
    """dgu = swiglu'(gu) ∘ (dx·Wd)  ([T,2F]) in ONE kernel: down-projection dgrad with the SwiGLU backward epilogue."""
    _rowmajor(dx, "dx"); _rowmajor(wd, "wd"); _rowmajor(gu, "gu")
    T, D = dx.shape
    F = wd.shape[1]
    if dgu is None:
        dgu = torch.empty((T, 2 * F), dtype=bf16, device=dx.device)
    lib = _lib.load()
    _timed(lambda: check(lib.nv_gemm_dswiglu_bf16(ptr(dx), i64(dx.stride(0)), ptr(wd), i64(wd.stride(0)), ptr(gu), i64(gu.stride(0)),
                                                   ptr(dgu), i64(dgu.stride(0)), i32(T), i32(F), i32(D), stream_ptr()),
                         "nv_gemm_dswiglu_bf16"),
           2.0 * T * F * D, 2.0 * (T * D + F * D + 4 * T * F))
    return dgu


def gemm_attnd(dy, wo, o, *, dout=None, dvec=None):
    """o_proj dgrad dO = dy·Wo ([T,D]) with the attention backward's D[h,t] = sum_d dO·O computed in the epilogue.
    Returns (dO bf16 [T,D], dvec fp32 [H*T]); pass dvec to attn_bwd(..., dvec=dvec) to skip its row-sum kernel."""
    _rowmajor(dy, "dy"); _rowmajor(wo, "wo"); _rowmajor(o, "o")
    T, Dout = dy.shape
    D = wo.shape[1]
    assert wo.shape[0] == Dout and o.shape == (T, D) and D % 128 == 0
    if dout is None:
        dout = torch.empty((T, D), dtype=bf16, device=dy.device)
    if dvec is None:
        dvec = torch.empty(((D // 128) * T,), dtype=torch.float32, device=dy.device)
    lib = _lib.load()
    _timed(lambda: check(lib.nv_gemm_attnd_bf16(ptr(dy), i64(dy.stride(0)), ptr(wo), i64(wo.stride(0)), ptr(o), i64(o.stride(0)),
                                                 ptr(dout), i64(dout.stride(0)), ptr(dvec), i32(T), i32(D), i32(Dout), stream_ptr()),
                         "nv_gemm_attnd_bf16"),
           2.0 * T * D * Dout, 2.0 * (T * Dout + D * Dout + 2 * T * D))
    return dout, dvec


def gemm_rope(x, w, pos, cos_t, sin_t, rope_cols, *, out=None):
    """out = x·W^T with rotate-half RoPE applied to the first ``rope_cols`` columns in the epilogue."""
    _rowmajor(x, "x"); _rowmajor(w, "w")
    T, K = x.shape
    N = w.shape[0]
    if out is None:
        out = torch.empty((T, N), dtype=bf16, device=x.device)
    lib = _lib.load()
    _timed(lambda: check(lib.nv_gemm_rope_bf16(ptr(x), i64(x.stride(0)), ptr(w), i64(w.stride(0)), ptr(out), i64(out.stride(0)),
                                                ptr(pos), ptr(cos_t), ptr(sin_t), i32(T), i32(N), i32(K), i32(rope_cols),
                                                stream_ptr()), "nv_gemm_rope_bf16"),
           2.0 * T * N * K, 2.0 * (T * K + N * K + T * N))
    return out
