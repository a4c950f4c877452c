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
            act_fp8=False):
        """``fp8``: None, or the (e4m3, exponents) pairs of wqkv, wo, wgu, wd (``Fp8Weights.view``); each GEMM with at most
        ``fp8_max_rows`` rows then streams its pair through nv_gemm_fp8w_bf16 (same bits as the bf16 weights W').
        ``act_fp8``: every GEMM runs W8A8 on the four pairs of ``fp8`` (all required) at every row count.
        ``ke`` / ``ve``: the row exponents of an fp8 cache (cache modes 3 and 4, kc / vc then hold its e4m3 bytes)."""
        a = self.args
        pairs = fp8 if fp8 is not None else ((None, None),) * 4
        (a.wqkv_q, a.wqkv_e), (a.wo_q, a.wo_e), (a.wgu_q, a.wgu_e), (a.wd_q, a.wd_e) = \
            [(q.data_ptr(), e.data_ptr()) if q is not None else (None, None) for q, e in pairs]
        a.fp8_max_rows = fp8_max_rows if fp8 is not None else 0
        a.act_fp8 = 1 if act_fp8 else 0
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


class pdl:
    """Context: launch the decode-chain kernels with programmatic dependent launch (nv_set_pdl)."""

    def __init__(self, on: bool = True):
        self.on = on

    def __enter__(self):
        self.prev = _lib.load().nv_set_pdl(i32(1 if self.on else 0))
        return self

    def __exit__(self, *a):
        _lib.load().nv_set_pdl(i32(self.prev))


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
