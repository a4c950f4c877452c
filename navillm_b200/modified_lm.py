"""Modified LLaMA causal LM on the sm_90a kernels -- host mirror of the reference's
``ModifiedLlamaForCausalLM`` (models/modified_lm.py:33-146,176-199).

Same surface: ``init_tokenizer``, ``tokenize``, ``forward(input_ids, attention_mask, labels, cand_vis, hist_vis,
obj_vis)`` returning an object with ``loss / logits / hidden_states``, ``generate`` (greedy / sampling),
attributes ``tokenizer, cls_token, cand_token_id, hist_token_id, obj_token_id, cls_token_id, special_token_ids,
hidden_size, model_type`` and HF parameter names ``model.embed_tokens / model.layers.N.* / model.norm / lm_head``.

What differs is the execution (see llama.py): prompts are packed (pad tokens are never computed), the visual
scatter-add is fused with the embedding gather, ``lm_head`` runs only on rows whose logits are consumed
(reference computes [B,S,V] logits + a [B,S,V] bool mask in every mode: SURVEY.md Appendix A.10), and the
backward is hand-written.  ``hidden_states`` / ``logits`` at pad positions are zeros / absent here, where the
reference holds values computed from pad embeddings that nothing reads.
"""
from __future__ import annotations

import collections
import os
import time
import weakref
from types import SimpleNamespace
from typing import List, Optional

import numpy as np
import torch
import torch.nn as nn

from . import llama as llama_mod
from . import ops
from . import trie as trie_mod
from .llama import FlatParams, Fp8Weights, LlamaCore, LlamaDims, LlamaModelParams, _Linear
from .parallel import GradSync
from .tokenizer import HFTokenizerAdapter, SyntheticTokenizer

bf16 = torch.bfloat16


class LMOutput(SimpleNamespace):
    """Stand-in for transformers.CausalLMOutputWithPast (attribute and item access)."""

    def __getitem__(self, k):
        return getattr(self, k)


class PackedPrompt:
    """Host-side packing of a left-padded [B,S] prompt batch: everything the kernels need, built with numpy
    on the tokenizer's CPU tensors and shipped to the device in ONE int32 copy."""

    def __init__(self, input_ids: torch.Tensor, attention_mask: torch.Tensor, lm: "ModifiedLlamaForCausalLM",
                 device: torch.device, labels: Optional[torch.Tensor] = None, generate_positions: bool = False):
        ids = input_ids.detach().cpu().numpy().astype(np.int64)
        msk = attention_mask.detach().cpu().numpy().astype(bool)
        B, S = ids.shape
        self.B, self.S = B, S
        self.seqlens = msk.sum(1).astype(np.int64).tolist()
        flat_rows = np.flatnonzero(msk.reshape(-1))                       # packed order == row-major order
        self.T = int(flat_rows.size)
        tok = ids.reshape(-1)[flat_rows]
        if generate_positions:                                            # HF generate: cumsum(mask) - 1
            pos = (np.cumsum(msk, axis=1) - 1).reshape(-1)[flat_rows]
        else:                                                             # plain forward: arange(S), pads included
            pos = np.tile(np.arange(S), B)[flat_rows]
        cu = np.concatenate([[0], np.cumsum(self.seqlens)])
        # visual scatter map: row-major order of each token kind (models/modified_lm.py:100-110); the vis tensor
        # handed to the kernel is cat([cand_vis, hist_vis, obj_vis])
        is_c, is_h, is_o = tok == lm.cand_token_id[0], tok == lm.hist_token_id[0], tok == lm.obj_token_id[0]
        self.n_cand, self.n_hist, self.n_obj = int(is_c.sum()), int(is_h.sum()), int(is_o.sum())
        vis_src = np.full(self.T, -1, dtype=np.int64)
        vis_src[is_c] = np.arange(self.n_cand)
        vis_src[is_h] = self.n_cand + np.arange(self.n_hist)
        vis_src[is_o] = self.n_cand + self.n_hist + np.arange(self.n_obj)
        # <cls_1> rows (one per sequence is assumed by the reference: nav_model.py:237)
        cls_rows = np.flatnonzero(tok == lm.cls_token_id[0])
        # last real token of every sequence (decode)
        last_rows = cu[1:] - 1
        # LM-loss rows: position p predicts token p+1 (shifted CE, modified_lm.py:126-137)
        if labels is not None:
            lab = labels.detach().cpu().numpy().astype(np.int64)
            nxt = np.full((B, S), -100, dtype=np.int64)
            nxt[:, :-1] = lab[:, 1:]
            nxt_packed = nxt.reshape(-1)[flat_rows]
            loss_rows = np.flatnonzero(nxt_packed != -100)
            loss_tgt = nxt_packed[loss_rows]
        else:
            loss_rows = np.zeros(0, dtype=np.int64)
            loss_tgt = np.zeros(0, dtype=np.int64)
        self.n_cls, self.n_loss = int(cls_rows.size), int(loss_rows.size)
        # token order of the deterministic embedding-gradient kernel (one owner per distinct id): sorted on the host, where
        # the ids already are, instead of a device radix sort per backward
        if torch.is_grad_enabled():
            tok_order = np.argsort(tok, kind="stable")
            tok_sorted = tok[tok_order]
        else:
            tok_order = tok_sorted = np.zeros(0, dtype=np.int64)
        parts = [tok, pos, cu, vis_src, cls_rows, last_rows, loss_rows, loss_tgt, tok_order, tok_sorted]
        host = np.concatenate([p.astype(np.int32) for p in parts])
        buf = torch.from_numpy(host).pin_memory() if torch.cuda.is_available() else torch.from_numpy(host)
        dev = buf.to(device, non_blocking=True)
        self.h2d_bytes = host.nbytes
        o = 0
        views = []
        for p in parts:
            views.append(dev[o:o + p.size])
            o += p.size
        (self.ids, self.pos, self.cu, self.vis_src, self.cls_rows, self.last_rows, self.loss_rows, self.loss_tgt,
         self.tok_order, self.tok_sorted) = views
        self.flat_rows = flat_rows                                        # host copy (unpacking to [B,S])


class PrefixKVCache:
    """Per-rollout KV cache for cross-step prompt-prefix reuse (SURVEY.md §8f n1; not in the reference).

    In a navigation rollout the prompt of step t+1 repeats the prompt of step t up to the end of the history
    (tasks/agents/r2r.py:16-31: instruction | (0) <hist> ... (t-1) <hist> | candidates | output hint), yet the
    reference re-encodes it from scratch every step (tasks/agents/mp3d_agent.py:660-726).  With frozen weights
    (evaluation / inference) the K/V of that prefix can be kept: each step encodes only the tokens after the longest
    common token prefix with what the cache holds for the row.

    Positions: the reference gives token j of a left-padded row the rotary position pad_b + j, and pad_b changes
    from step to step.  Rotary attention depends on position DIFFERENCES only, so a row keeps the offset of its first
    step for the whole rollout (``off``); results differ from a from-scratch forward only through bf16 rounding of
    the cos/sin tables at different absolute positions (tests/test_prefix_reuse_gpu.py states the tolerance).

    Contract: rows are identified by batch index; the <hist> vectors of a row are append-only across steps (the
    reference's hist_vis lists are); call ``reset()`` when a new episode starts in a row.

    ``kv_dtype="fp8"`` (opt-in; default ``"bf16"``) stores the cache in the fp8 format of ``set_kv_cache_dtype("fp8")``
    (include/navillm_b200.h): per layer, e4m3 bytes [B, max_len, D] plus one int8 power-of-two exponent per (row, position,
    head), half the memory of the bf16 cache plus 1/256 (``nbytes``), which lets a rollout run a larger batch at the same
    ``max_len``.  Every suffix step attends over the cache, so the step's new rows read their own K / V rounded to e4m3 as
    well (K' / V'); generate()'s prefill, by contrast, attends over the unrounded K / V of the prompt.  The format is the
    caller's choice: it does not follow the model's ``kv_cache_dtype``.  Works with and without ``quantize_weights_fp8()``.

    ``train=True`` (opt-in, bf16 only) lets the cache serve a training rollout: ``model('navigation', batch, prefix_cache=...)``
    under grad mode, one ``backward()`` per step, weights fixed until the rollout's gradients are complete.  The gradient of
    a step's loss then has two parts.  (a) Through the step's own suffix rows: its ``backward()`` runs the stack over the
    suffix with the cache form of the attention backward, which also produces dK / dV of the cached rows the step attended
    to; those are ADDED to a per-layer fp32 accumulator over the cache rows (``acc``, [B, max_len, 2 D]: dK | dV), not
    propagated.  (b) Through the cached rows: linear in the accumulated dK / dV, so ONE backward per rollout covers every
    step -- ``flush_grads()`` re-runs the forward of each row's reused prefix (its token ids, the ``<hist>`` vectors it was
    given, rotary positions ``off + j``) with a tape and back-propagates the accumulator through it, the accumulated dK / dV
    entering each layer as the gradient of that layer's K / V.  Memory: the accumulator, no activations across steps; cost:
    one extra forward of the prefix per rollout.  A row whose reusable prefix shrinks (left truncation of a long prompt)
    runs its part (b) first, before its cache rows are overwritten.  Part (b) attends over the cached K/V (the rows the steps' dK / dV
    refer to; the flush writes no cache row) with the other prefix activations recomputed, which equal the steps' up to
    bf16 rounding (different GEMM shapes).  ``flush_grads()`` must run before the optimizer step:
    the data-parallel exchange of an armed pass does it itself; ``reset()`` of a row with pending gradient, ``zero_grad()``
    of the model, and any step or flush after the weights changed raise."""

    def __init__(self, lm: "ModifiedLlamaForCausalLM", batch_size: int, max_len: int = 2048, kv_dtype: str = "bf16",
                 train: bool = False):
        if kv_dtype not in ("bf16", "fp8"):
            raise ValueError(f"PrefixKVCache: kv_dtype must be 'bf16' or 'fp8' (got {kv_dtype!r})")
        if train and kv_dtype != "bf16":
            raise ValueError("PrefixKVCache: train=True needs the bf16 cache (the fp8 store is inference-only)")
        lm._ensure()
        dev, d = lm._device(), lm.dims
        self.B, self.max_len, self.kv_dtype = batch_size, max_len, kv_dtype
        # zero-initialised: rows past a sequence's length are masked in the attention kernel but must stay finite
        if kv_dtype == "fp8":
            if d.head_dim != 128:
                raise ValueError(f"PrefixKVCache: the fp8 cache needs head_dim 128 (got {d.head_dim})")

            def layer():
                return (torch.zeros((batch_size, max_len, d.hidden), dtype=torch.float8_e4m3fn, device=dev),
                        torch.zeros((batch_size, max_len, d.n_heads), dtype=torch.int8, device=dev))
        else:
            def layer():
                return torch.zeros((batch_size, max_len, d.hidden), dtype=bf16, device=dev)
        self.kc = [layer() for _ in range(d.n_layers)]
        self.vc = [layer() for _ in range(d.n_layers)]
        self.ids: List[np.ndarray] = [np.zeros(0, dtype=np.int64) for _ in range(batch_size)]
        self.off: List[Optional[int]] = [None] * batch_size
        self.stats = {"steps": 0, "tokens": 0, "tokens_encoded": 0}
        self.train = train
        self.acc = [torch.zeros((batch_size, max_len, 2 * d.hidden), dtype=torch.float32, device=dev)
                    for _ in range(d.n_layers)] if train else None
        self.hist: List[Optional[torch.Tensor]] = [None] * batch_size   # <hist> rows each row was last given (references)
        self.reused = [0] * batch_size        # R[b]: cached rows [0, R) whose part (b) has not run yet
        self._pending_rows = set()            # rows whose accumulator a step's backward has written since their last flush
        self.writes = 0                       # steps that wrote the cache: a step's tape is valid only until the next one
        self._lm = weakref.ref(lm)
        if train:
            self._weights = self._weight_state()
            lm._prefix_caches.add(self)

    @property
    def nbytes(self) -> int:
        """Device bytes of the K and V caches of all layers (exponents included) and, with ``train=True``, the gradient
        accumulator."""
        return sum(t.nbytes for c in self.kc + self.vc for t in (c if isinstance(c, tuple) else (c,))) + \
            sum(a.nbytes for a in (self.acc or []))

    @property
    def pending(self) -> bool:
        """True while part (b) of some row's gradient is outstanding (``flush_grads()`` has work to do)."""
        return bool(self._pending_rows)

    def reset(self, rows=None) -> None:
        rows = list(range(self.B) if rows is None else rows)
        lost = sorted(b for b in rows if b in self._pending_rows)
        if lost:
            raise RuntimeError(f"PrefixKVCache.reset: rows {lost} have pending gradient through their cached prefix; call "
                               f"flush_grads() first")
        for b in rows:
            self.ids[b] = np.zeros(0, dtype=np.int64)
            self.off[b] = None
            self.hist[b] = None
            self.reused[b] = 0
        if self.train and all(i.size == 0 for i in self.ids):
            self._weights = self._weight_state()         # nothing cached: the cache may be refilled under new weights

    # ---- training ----------------------------------------------------------------------------------------------
    def _weight_state(self):
        flat = self._lm().flat
        return flat.flat.data_ptr(), flat.flat._version, flat.generation, sum(p._version for p in flat.params)

    def check_weights(self) -> None:
        if self._weight_state() != self._weights:
            raise RuntimeError("PrefixKVCache: the weights changed since the cache was filled (optimizer step, load or "
                               "another write); its K/V and pending gradient belong to the old weights -- run flush_grads() "
                               "before the optimizer step, and reset() the cache (or build a new one) for the next rollout")

    def flush_grads(self) -> None:
        """Part (b) of the gradient for every row with pending gradient: one forward of the rows' reused prefixes with a tape
        and one backward that injects the accumulated dK / dV, accumulated into the model's gradients; then the accumulator
        of those rows is zero.  A no-op when nothing is pending."""
        self._flush_rows(sorted(self._pending_rows))

    def _flush_shrinking(self, ids: np.ndarray, msk: np.ndarray, cand_id: int) -> None:
        """Before a step overwrites the cache: flush the rows whose reusable prefix is shorter than what they reused so far."""
        rows = [b for b in range(self.B) if self.reused[b] > 0 and _reusable_prefix(self.ids[b], ids[b][msk[b]], cand_id) < self.reused[b]]
        self._flush_rows(rows)
        for b in rows:
            self.reused[b] = 0

    def _flush_rows(self, rows) -> None:
        rows = [b for b in rows if b in self._pending_rows]
        if not rows:
            return
        self.check_weights()
        lm = self._lm()
        lm._ensure()
        core, d, dev = lm.core, lm.dims, lm._device()
        hist_id = lm.hist_token_id[0]
        toks, pos, vsrc, hist, lens = [], [], [], [], []
        nh = 0
        for b in rows:
            R = self.reused[b]
            t = self.ids[b][:R]
            is_h = t == hist_id
            h = int(is_h.sum())
            vs = np.full(R, -1, dtype=np.int64)
            vs[is_h] = nh + np.arange(h)
            nh += h
            if h:
                hist.append(self.hist[b][:h])
            toks.append(t); pos.append(self.off[b] + np.arange(R)); vsrc.append(vs); lens.append(R)
        tok = np.concatenate(toks)
        order = np.argsort(tok, kind="stable")
        cu = np.concatenate([[0], np.cumsum(lens)])
        parts = [tok, np.concatenate(pos), cu, np.concatenate(vsrc), np.zeros(len(rows)), np.asarray(rows) * self.max_len,
                 np.asarray(lens), order, tok[order]]
        views = _to_device(parts, dev)
        tok_d, pos_d, cu_d, vs_d, zero_d, kvs_d, kvl_d, ord_d, srt_d = views
        vis = torch.cat(hist, 0).to(torch.float32).contiguous() if hist else None
        E = lm.model.embed_tokens.weight
        with torch.no_grad():
            x = ops.embed_fwd(tok_d, E.data, vs_d if vis is not None else None, vis)
            # the cache rows [0, R) of each flushed row already hold the K/V its steps attended over (and that the accumulated
            # dK / dV refer to): attend over them, and leave every slot of the cache as it is
            g, tape = core.forward_suffix(x, pos_d, cu_d, lens, self.kc, self.vc, zero_d, kvs_d, kvl_d, save=True, acc=self.acc,
                                          kv_lens=lens, store=False)
            lm._settle_lazy_zero()                     # part (b) adds to the gradients the steps' backwards left
            dx = core.backward(torch.zeros_like(g), tape)
            ops.embed_bwd_weight_(dx, tok_d, E.grad, order=ord_d, sorted_ids=srt_d)
            idx = torch.tensor(rows, dtype=torch.int64, device=dev)
            for a in self.acc:
                a[:, :max(lens)].index_fill_(0, idx, 0.0)
        self.writes += 1
        for b in rows:
            self.reused[b] = 0
            self._pending_rows.discard(b)


    def _mark_pending(self, cached) -> None:
        """A step's backward added the dK / dV of rows [0, cached[b]) to the accumulator."""
        for b, c in enumerate(cached):
            if c > 0:
                self._pending_rows.add(b)


def _to_device(parts, dev):
    """int32 device views of host integer arrays, shipped in ONE pinned copy."""
    host = np.concatenate([np.asarray(p).astype(np.int32).reshape(-1) for p in parts])
    buf = torch.from_numpy(host).pin_memory().to(dev, non_blocking=True)
    views, o = [], 0
    for p in parts:
        n = np.asarray(p).size
        views.append(buf[o:o + n]); o += n
    return views


def _reusable_prefix(old: np.ndarray, toks: np.ndarray, cand_id: int) -> int:
    """Rows of a row's new prompt ``toks`` whose K/V the cache holds: the longest common token prefix with ``old``, cut
    before the first <cand> token (candidates change every step) and at most L - 1 (the last token is always encoded)."""
    m = min(old.size, int(toks.size) - 1)
    neq = np.flatnonzero(old[:m] != toks[:m])
    n = int(neq[0]) if neq.size else m
    cpos = np.flatnonzero(toks == cand_id)
    if cpos.size:
        n = min(n, int(cpos[0]))
    return n


def plan_prefix_reuse(ids: np.ndarray, msk: np.ndarray, cache: "PrefixKVCache", hist_counts, n_cand_total: int, cand_id: int,
                      hist_id: int, cls_id: int):
    """Host-side plan of one cached navigation step (pure numpy; updates ``cache.ids`` / ``cache.off``).

    For every left-padded row: the reusable prefix = longest common token prefix with what the cache holds for the row, cut
    before the first <cand> token (candidates change every step) and at most L - 1 (the last token is always encoded).
    Returns per-row lists (new token ids, rotary positions, visual-source indices into cat([cand_vis, hist_vis]),
    number of new rows, cached rows, total context length) and the packed row index of each row's <cls_1> token."""
    B, S = ids.shape
    if B != cache.B:
        raise ValueError(f"prefix cache was built for batch {cache.B}, got {B} prompts")
    hist_base = np.concatenate([[0], np.cumsum(np.asarray(hist_counts, dtype=np.int64))])
    tok_new, pos_new, vis_new, q_lens, cached, kv_len, cls_rows = [], [], [], [], [], [], []
    n_cand_seen, t0 = 0, 0
    for b in range(B):
        toks = ids[b][msk[b]]
        L = int(toks.size)
        if L == 0 or not msk[b, S - L:].all():
            raise ValueError("prefix reuse needs left-padded prompts with at least one token")
        if L > cache.max_len:
            raise ValueError(f"prompt of {L} tokens exceeds the prefix cache length {cache.max_len}")
        if cache.off[b] is None:
            cache.off[b] = S - L                               # the row keeps this rotary offset for the rollout
        n = _reusable_prefix(cache.ids[b], toks, cand_id)
        new = toks[n:]
        is_h, is_c = new == hist_id, new == cand_id
        h_before = int((toks[:n] == hist_id).sum())
        vs = np.full(new.size, -1, dtype=np.int64)
        vs[is_c] = n_cand_seen + np.arange(int(is_c.sum()))
        vs[is_h] = n_cand_total + hist_base[b] + h_before + np.arange(int(is_h.sum()))
        if h_before + int(is_h.sum()) != int(hist_counts[b]):
            raise RuntimeError(f"row {b}: {h_before + int(is_h.sum())} <hist> tokens but {int(hist_counts[b])} hist_vis rows")
        n_cand_seen += int(is_c.sum())
        c = np.flatnonzero(new == cls_id)
        if c.size != 1:
            raise RuntimeError(f"expected one <cls_1> token after the reusable prefix of row {b}, found {c.size}")
        cls_rows.append(t0 + int(c[0]))
        tok_new.append(new); vis_new.append(vs)
        pos_new.append(cache.off[b] + n + np.arange(new.size))
        q_lens.append(int(new.size)); cached.append(n); kv_len.append(L)
        t0 += int(new.size)
        cache.ids[b] = toks.copy()
    if n_cand_seen != n_cand_total:
        raise RuntimeError(f"{n_cand_seen} <cand> tokens in the prompts but {n_cand_total} cand_vis rows")
    return tok_new, pos_new, vis_new, q_lens, cached, kv_len, cls_rows


class _LMFn(torch.autograd.Function):
    """Differentiable boundary of the language model for a packed prompt.

    inputs : vis [Nv, D] fp32 (cat of cand/hist/obj visual rows; may require grad)
    outputs: mode 'rows' -> final-RMSNorm'ed hidden states at ``rows`` ([R, D] bf16)
             mode 'loss' -> mean shifted-CE loss over ``pp.loss_rows`` (fp32 scalar)
    backward accumulates all LM weight gradients in place and returns d vis.
    """

    @staticmethod
    def forward(ctx, lm: "ModifiedLlamaForCausalLM", pp: PackedPrompt, vis: Optional[torch.Tensor], mode: str,
                rows: Optional[torch.Tensor], train: bool, anchor):
        # NB: grad mode is always off inside Function.forward, so `train` is decided by the caller
        core, d = lm.core, lm.dims
        E = lm.model.embed_tokens.weight.data
        x = ops.embed_fwd(pp.ids, E, pp.vis_src if vis is not None else None, vis)
        if mode == "loss":
            rows = pp.loss_rows
        # the stack returns only the requested rows (last layer pruned to them)
        kv = getattr(pp, "kv", None)
        if kv is not None:             # training step over a PrefixKVCache: the suffix rows only (hidden_rows_cached)
            c = kv.cache
            g, ctx.tape = core.forward_suffix(x, pp.pos, pp.cu, pp.seqlens, c.kc, c.vc, kv.cached, kv.kv_start, kv.kv_len,
                                              out_rows=rows, save=True, acc=c.acc, kv_lens=kv.kv_lens)
        else:
            g, ctx.tape = core.forward(x, pp.pos, pp.cu, pp.seqlens, save=train, out_rows=rows)
        ctx.lm, ctx.pp, ctx.mode, ctx.has_vis = lm, pp, mode, vis is not None
        ctx.n_vis = 0 if vis is None else vis.shape[0]
        hn, rstd = ops.rmsnorm_fwd(g, lm.model.norm.weight.data, d.rms_eps)
        if mode == "rows":
            ctx.saved = (g, rstd)
            return hn
        # ---- LM loss on the label rows only ----
        V = lm.lm_head.weight.shape[0]
        logits = torch.empty((g.shape[0], (V + 63) // 64 * 64), dtype=bf16, device=g.device)[:, :V]   # 16-byte aligned rows
        ops.gemm(hn, lm.lm_head.weight.data, out=logits)                 # [Nl, V] bf16
        row_loss, dlogits = ops.ce_fwd_bwd(logits, pp.loss_tgt, lm.special_ids_dev,
                                           grad_scale=(1.0 / max(pp.n_loss, 1)) if train else None)
        loss = row_loss.sum() / max(pp.n_loss, 1)
        ctx.saved = (g, rstd, hn, dlogits)
        return loss.to(bf16) if lm.model_type == bf16 else loss           # reference: CE on bf16 logits -> bf16 loss

    @staticmethod
    def backward(ctx, dout):
        lm, pp = ctx.lm, ctx.pp
        core, d = lm.core, lm.dims
        normw = lm.model.norm.weight
        lm.grad_sync.backward_begins()               # first custom node of the pass in the LM-loss modes (no-op if queued)
        if ctx.mode == "rows":
            g, rstd = ctx.saved
            dy = dout.contiguous().to(bf16)
        else:
            g, rstd, hn, dlogits = ctx.saved
            lm._lm_head_grad_clean = False
            # dlogits was produced with scale 1/N; fold the incoming scalar gradient in on the device (no sync)
            ops.scale_(dlogits, dout.detach().to(torch.float32).reshape(1))   # in place: keeps the 16-byte-aligned row stride
            dy = ops.gemm(dlogits, lm.lm_head.weight.data, b_mn=True)                    # [Nl, D]
            ops.gemm(dlogits, hn, a_mn=True, b_mn=True, out=lm.lm_head.weight.grad, addend=lm.lm_head.weight.grad)
        kv = getattr(pp, "kv", None)
        if kv is not None and kv.cache.writes != kv.write_id:
            raise RuntimeError("PrefixKVCache: a later step or flush rewrote the cache before this step's backward ran "
                               "(call backward() after every step, as the rollout does)")
        dg = ops.rmsnorm_bwd(g, normw.data, rstd, dy, dw=normw.grad)                     # [R, D]: gradient at the requested rows
        lm.grad_sync.short_backward = pp.T < lm.SHORT_BACKWARD_TOKENS
        # a pass that leaves prefix-cache gradient pending is not final per layer until the flush (before the exchange):
        # no overlapped per-layer reductions
        overlap = kv is None and not lm.prefix_grads_pending()
        dx = core.backward(dg, ctx.tape, layer_done=lm._grad_sync_hook() if overlap else None)
        if kv is not None:
            kv.cache._mark_pending(kv.cached_host)
        ops.embed_bwd_weight_(dx, pp.ids, lm.model.embed_tokens.weight.grad,
                              order=pp.tok_order if pp.tok_order.numel() == pp.T else None, sorted_ids=pp.tok_sorted)
        dvis = ops.embed_bwd_vis(dx, pp.vis_src, ctx.n_vis) if ctx.has_vis else None
        ctx.saved = ctx.tape = None
        return None, None, dvis, None, None, None, None


class ModifiedLlamaForCausalLM(nn.Module):
    def __init__(self, config, extra_config=None, tokenizer=None):
        """config: object with hidden_size, intermediate_size, num_hidden_layers, num_attention_heads, vocab_size,
        rms_norm_eps (a transformers LlamaConfig works).  extra_config.precision as in the reference."""
        super().__init__()
        precision = getattr(extra_config, "precision", "amp_bf16") if extra_config is not None else "amp_bf16"
        if not ("bf16" in precision or "bfloat16" in precision):
            raise NotImplementedError(f"navillm_b200 computes the LM in bf16 (reference 'amp_bf16'); got precision={precision!r}")
        self.model_type = bf16
        self.config = config
        self.hidden_size = config.hidden_size
        self.dims = LlamaDims(hidden=config.hidden_size, n_layers=config.num_hidden_layers, n_heads=config.num_attention_heads,
                              inter=config.intermediate_size, vocab=config.vocab_size,
                              rms_eps=getattr(config, "rms_norm_eps", 1e-6), rope_theta=getattr(config, "rope_theta", 10000.0))
        if self.dims.head_dim != 128:
            raise NotImplementedError("attention kernels are built for head_dim = 128 (Vicuna-7B)")
        self.model = LlamaModelParams(self.dims)
        self.lm_head = _Linear(self.dims.vocab, self.dims.hidden)
        self.core: Optional[LlamaCore] = None
        self.training_enabled = True
        self.register_buffer("_anchor", torch.zeros((), dtype=torch.float32), persistent=False)
        self.grad_sync = GradSync()                  # replaced by NavModel's shared state when owned by a NavModel
        self.grad_sync.flats = self._own_flats
        self.grad_sync.before_exchange = self.flush_prefix_caches
        self._prefix_caches = weakref.WeakSet()      # PrefixKVCache(train=True) instances built on this model
        if tokenizer is not None:
            self._set_tokenizer(tokenizer)

    # ---- tokenizer front-end (models/modified_lm.py:56-87) ----
    def init_tokenizer(self, pretrained_model_name_or_path: Optional[str], allow_synthetic: bool = False):
        """The reference's tokenizer construction (models/modified_lm.py:56-75) from a LOCAL tokenizer directory.  Without
        usable tokenizer files this raises: pretrained / resumed Vicuna weights on hash-derived token ids would run
        silently on garbage.  ``allow_synthetic=True`` (from-scratch runs, tests, benches) falls back to the deterministic
        ``SyntheticTokenizer`` and says so."""
        try:
            tok = HFTokenizerAdapter(pretrained_model_name_or_path)
        except Exception as e:
            if not allow_synthetic:
                raise RuntimeError(f"no usable LLaMA tokenizer under {pretrained_model_name_or_path!r} ({type(e).__name__}: {e}); "
                                   f"pass a local tokenizer directory, or model_config.tokenizer / --from_scratch for the "
                                   f"synthetic stand-in") from e
            import warnings
            warnings.warn(f"navillm_b200: no tokenizer files under {pretrained_model_name_or_path!r}; using SyntheticTokenizer "
                          f"(word-hash ids) -- only meaningful with randomly initialised weights")
            tok = SyntheticTokenizer(base_vocab=self.dims.vocab if self.dims.vocab < 32000 else 32000)
        self._set_tokenizer(tok)

    def _set_tokenizer(self, tok):
        self.tokenizer = tok
        self.cand_token, self.hist_token, self.obj_token = ["<cand>"], ["<hist>"], ["<obj>"]
        self.cls_token = ["<cls_1>", "<cls_2>"]
        self.cand_token_id = [tok.special["<cand>"]]
        self.hist_token_id = [tok.special["<hist>"]]
        self.obj_token_id = [tok.special["<obj>"]]
        self.cls_token_id = [tok.special["<cls_1>"], tok.special["<cls_2>"]]
        self.special_token_ids = self.cand_token_id + self.hist_token_id + self.obj_token_id + self.cls_token_id
        self.resize_token_embeddings(len(tok))

    def resize_token_embeddings(self, n: int):
        old = self.model.embed_tokens.weight
        if old.shape[0] == n:
            return
        assert self.core is None, "resize_token_embeddings after materialisation"
        D = old.shape[1]
        for holder in (self.model.embed_tokens, self.lm_head):
            w = holder.weight.data
            new = torch.empty(n, D, dtype=w.dtype)
            k = min(n, w.shape[0])
            new[:k] = w[:k]
            if n > k:
                new[k:] = (torch.randn(n - k, D) * 0.02).to(w.dtype)
            holder.weight = nn.Parameter(new)
        self.dims.vocab = n
        self.config.vocab_size = n

    def tokenize(self, text, add_special_tokens: bool = True):
        return self.tokenizer(text, max_length=1024, padding=True, truncation=True, return_tensors="pt",
                              add_special_tokens=add_special_tokens, return_token_type_ids=True)

    # ---- device materialisation ----
    def lm_parameters(self) -> List[nn.Parameter]:
        return self.model.flat_order() + [self.lm_head.weight]

    def materialize(self, device: torch.device, extra_params: Optional[List[nn.Parameter]] = None) -> FlatParams:
        """Move the LM parameters into one flat bf16 buffer on ``device`` (+ ``extra_params``: the bf16 heads of
        NavModel) and build the fused-view driver.  Idempotent while the views are intact."""
        if self.core is not None and self.flat.intact():
            return self.flat
        if extra_params is not None:
            self._extra_params = list(extra_params)
        params = self.lm_parameters() + list(getattr(self, "_extra_params", []))
        self.__dict__.pop("_decode_states", None)     # captured decode graphs hold pointers into the old buffers
        self.flat = FlatParams(params, device)
        self.flat.clean_segments = self._clean_grad_segments
        self.flat.on_zeroed = self.mark_grads_zeroed
        self._lm_head_grad_clean = False             # unknown until the next zero_grad
        self.core = LlamaCore(self.dims, self.model, self.flat)
        self.core.act_fp8 = self.activation_dtype == "fp8"
        self.special_ids_dev = torch.tensor(self.special_token_ids, dtype=torch.int32, device=device)
        return self.flat

    def _device(self) -> torch.device:
        return self.model.norm.weight.device

    # ---- data-parallel gradient exchange (navillm_b200/parallel.py; SURVEY.md §8e) ----
    def _grad_sync_hook(self):
        """Per-layer callback for LlamaCore.backward that all-reduces (AVG) the flat-gradient slice of every finished
        group of decoder layers asynchronously, so NCCL runs while the remaining layers' backward GEMMs execute.  Only
        an ARMED pass gets one (a forward outside ``no_sync()`` through the DDP wrapper, see ``GradSync``): a backward
        inside ``no_sync`` issues no collective, whatever the other ranks are doing."""
        flat, layers = self.flat, self.model.layers
        starts = [flat.offset_of(l.self_attn.q_proj.weight) for l in layers] + [flat.offset_of(self.model.embed_tokens.weight)]
        return self.grad_sync.layer_hook(flat, starts, self.dims.n_layers)

    SHORT_BACKWARD_TOKENS = 4096     # below this many packed rows a backward is shorter than the exchange of its gradients

    def _clean_grad_segments(self):
        """Flat-gradient ranges known to be all-zero (see GradSync.exchange): lm_head after a zero_grad when no LM-loss
        backward has run since (navigation / grounding steps never touch it)."""
        if not getattr(self, "_lm_head_grad_clean", False):
            return []
        o = self.flat.offset_of(self.lm_head.weight)
        return [(o, o + self.lm_head.weight.numel())]

    def mark_grads_zeroed(self) -> None:
        self._lm_head_grad_clean = True

    def _settle_lazy_zero(self) -> None:
        """``zero_grad(lazy=True)`` promised that the next LM backward overwrites the per-layer gradients; a backward that
        must ADD to them (or an exchange / optimizer step with no backward in between) first makes the promise true."""
        if self.core is not None and getattr(self.flat, "overwrite_layer_grads", False):
            self.flat.flat_grad[:self.flat.offset_of(self.model.embed_tokens.weight)].zero_()
            self.flat.overwrite_layer_grads = False

    # ---- training prefix caches (PrefixKVCache(train=True)) ----
    def prefix_grads_pending(self) -> bool:
        return any(c.pending for c in list(self._prefix_caches))

    def flush_prefix_caches(self) -> None:
        """``flush_grads()`` of every training prefix cache of this model (the armed pass runs it before the exchange)."""
        for c in list(self._prefix_caches):
            c.flush_grads()

    def _own_flats(self):
        return [(self.flat, self.flat.offset_of(self.model.embed_tokens.weight))] if self.core is not None else []

    def _ensure(self):
        dev = self._device()
        if dev.type != "cuda":
            raise RuntimeError("navillm_b200 has no CPU path: move the model to a CUDA device first")
        if self.core is None:
            self.materialize(dev)
            return
        p0 = self.flat.params[0]
        if p0.data_ptr() != self.flat._ptr0:              # parameters were moved/replaced (.to(), load): re-home
            self.core = None
            self.materialize(dev)
        elif p0.grad is None or p0.grad.data_ptr() != self.flat.flat_grad.data_ptr():
            self.flat.reattach_grads()                    # optimizer.zero_grad(set_to_none=True)

    # ---- packed entry points used by NavModel ----
    def hidden_rows(self, pp: PackedPrompt, vis: Optional[torch.Tensor], rows: torch.Tensor) -> torch.Tensor:
        self._ensure()
        train = torch.is_grad_enabled() and self.training_enabled
        anchor = self._anchor.detach().requires_grad_(train)
        return _LMFn.apply(self, pp, vis, "rows", rows, train, anchor)

    def hidden_rows_cached(self, input_ids: torch.Tensor, attention_mask: torch.Tensor, cand_vis: Optional[torch.Tensor],
                           hist_vis: Optional[torch.Tensor], hist_counts, cache: PrefixKVCache) -> torch.Tensor:
        """Twin of ``hidden_rows(pp, vis, pp.cls_rows)`` that encodes only the tokens after each row's
        longest common prefix with ``cache`` (see PrefixKVCache).  cand_vis: [sum cand, D] in row-major token order;
        hist_vis: [sum_b hist_counts[b], D] flattened sample-major (NavModel._flatten_hist).  Returns the final-
        RMSNorm'ed hidden states at the <cls_1> tokens, [B, D] bf16.  Inference (no grad) with any cache; under grad mode
        with a ``train=True`` cache, differentiable w.r.t. cand_vis and the weights (see PrefixKVCache for the gradient)."""
        self._ensure()
        train = torch.is_grad_enabled() and self.training_enabled
        if train and not cache.train:
            raise RuntimeError("prefix_cache: this cache is inference-only: call under torch.no_grad(), or build it with "
                               "PrefixKVCache(..., train=True) for a training rollout")
        if cache.train:
            cache.check_weights()
            if hist_vis is not None and hist_vis.requires_grad:
                raise RuntimeError("prefix_cache(train=True): hist_vis must be detached (the rollout's <hist> vectors are "
                                   "fuse_embeds.detach()); the cache keeps them for the prefix backward")
        dev, d = self._device(), self.dims
        ids = input_ids.detach().cpu().numpy().astype(np.int64)
        msk = attention_mask.detach().cpu().numpy().astype(bool)
        B = ids.shape[0]
        n_cand_total = 0 if cand_vis is None else cand_vis.shape[0]
        if cache.train:
            cache._flush_shrinking(ids, msk, self.cand_token_id[0])
        plan = plan_prefix_reuse(ids, msk, cache, hist_counts, n_cand_total, self.cand_token_id[0], self.hist_token_id[0],
                                 self.cls_token_id[0])
        tok_new, pos_new, vis_new, q_lens, cached, kv_len, cls_rows = plan
        cu = np.concatenate([[0], np.cumsum(q_lens)])
        kv_start = np.arange(B, dtype=np.int64) * cache.max_len
        tok = np.concatenate(tok_new)
        parts = [tok, np.concatenate(pos_new), cu, np.concatenate(vis_new), np.asarray(cls_rows),
                 np.asarray(cached), kv_start, np.asarray(kv_len)]
        if train:
            order = np.argsort(tok, kind="stable")           # token order of the deterministic embedding gradient
            parts += [order, tok[order]]
        views = _to_device(parts, dev)
        tok_d, pos_d, cu_d, vis_d, cls_d, cached_d, kvs_d, kvl_d = views[:8]
        cache.stats["steps"] += 1
        cache.stats["tokens"] += int(sum(kv_len))
        cache.stats["tokens_encoded"] += int(sum(q_lens))
        cache.writes += 1
        if cache.train:
            base = np.concatenate([[0], np.cumsum(np.asarray(hist_counts, dtype=np.int64))])
            for b in range(B):
                cache.hist[b] = None if hist_vis is None else hist_vis[base[b]:base[b + 1]].detach()
        vis_parts = [v.to(torch.float32) for v in (cand_vis, hist_vis) if v is not None and v.shape[0] > 0]
        vis = None if not vis_parts else (vis_parts[0].contiguous() if len(vis_parts) == 1 else torch.cat(vis_parts, 0))
        if train:
            for b in range(B):
                cache.reused[b] = max(cache.reused[b], int(cached[b]))
            kv = SimpleNamespace(cache=cache, cached=cached_d, kv_start=kvs_d, kv_len=kvl_d, kv_lens=list(kv_len),
                                 cached_host=list(cached), write_id=cache.writes)
            sp = SimpleNamespace(ids=tok_d, pos=pos_d, cu=cu_d, seqlens=list(q_lens), T=int(tok.size), vis_src=vis_d,
                                 tok_order=views[8], tok_sorted=views[9], n_loss=0, kv=kv)
            anchor = self._anchor.detach().requires_grad_(True)
            return _LMFn.apply(self, sp, vis, "rows", cls_d, True, anchor)
        with torch.no_grad():
            x = ops.embed_fwd(tok_d, self.model.embed_tokens.weight.data, vis_d if vis is not None else None, vis)
            g = self.core.forward_suffix(x, pos_d, cu_d, q_lens, cache.kc, cache.vc, cached_d, kvs_d, kvl_d, out_rows=cls_d)
            hn, _ = ops.rmsnorm_fwd(g, self.model.norm.weight.data, d.rms_eps)
        return hn

    def lm_loss(self, pp: PackedPrompt, vis: Optional[torch.Tensor]) -> torch.Tensor:
        self._ensure()
        train = torch.is_grad_enabled() and self.training_enabled
        anchor = self._anchor.detach().requires_grad_(train)
        return _LMFn.apply(self, pp, vis, "loss", None, train, anchor)

    @staticmethod
    def cat_vis(cand_vis, hist_vis, obj_vis, pp: PackedPrompt) -> Optional[torch.Tensor]:
        parts = []
        for name, v, n in (("cand", cand_vis, pp.n_cand), ("hist", hist_vis, pp.n_hist), ("obj", obj_vis, pp.n_obj)):
            if n == 0:
                continue
            if v is None or v.shape[0] != n:
                raise RuntimeError(f"{n} <{name}> tokens in the prompts but {0 if v is None else v.shape[0]} {name}_vis rows "
                                   f"(models/modified_lm.py:105-110 requires equal counts)")
            parts.append(v.to(torch.float32))
        if not parts:
            return None
        return parts[0].contiguous() if len(parts) == 1 else torch.cat(parts, dim=0)

    # ---- reference-compatible forward (models/modified_lm.py:89-146) ----
    def forward(self, input_ids, attention_mask, labels=None, cand_vis=None, hist_vis=None, obj_vis=None,
                return_logits: bool = False, **kwargs):
        """One full-prompt pass.  ``hidden_states`` is the reference's [B, S, D] tensor (zeros at pad positions, which the
        reference fills with values nothing reads); ``logits`` ([B, S, V] with the special tokens at -inf) only on request
        (``return_logits=True``): every caller on the path reads ``loss`` or ``hidden_states`` (SURVEY.md Appendix A.10).
        Incremental decoding arguments are not accepted here -- the KV-cache loop lives in ``generate``."""
        for k in ("past_key_values", "position_ids", "inputs_embeds"):
            if kwargs.get(k) is not None:
                raise NotImplementedError(f"ModifiedLlamaForCausalLM.forward({k}=...) is not supported: use .generate() for "
                                          f"incremental decoding (HF's generate loop is replaced by a native KV-cache loop)")
        self._ensure()
        dev = self._device()
        pp = PackedPrompt(input_ids, attention_mask, self, dev, labels=labels)
        vis = self.cat_vis(cand_vis, hist_vis, obj_vis, pp)
        loss = self.lm_loss(pp, vis) if labels is not None else None
        hidden = logits = None
        if labels is None or return_logits:
            all_rows = torch.arange(pp.T, device=dev, dtype=torch.int32)
            hn = self.hidden_rows(pp, vis, all_rows)
            flat = torch.from_numpy(pp.flat_rows).to(dev)
            hidden = torch.zeros((pp.B * pp.S, self.dims.hidden), dtype=bf16, device=dev).index_copy(0, flat, hn)
            hidden = hidden.view(pp.B, pp.S, -1)
            if return_logits:
                lg = ops.gemm(hn.detach().contiguous(), self.lm_head.weight.data)
                lg[:, self.special_token_ids] = float("-inf")
                logits = torch.zeros((pp.B * pp.S, lg.shape[1]), dtype=bf16, device=dev).index_copy(0, flat, lg).view(pp.B, pp.S, -1)
        return LMOutput(loss=loss, logits=logits, past_key_values=None, hidden_states=hidden, attentions=None)


    # ---- opt-in fp8 (e4m3) weight streaming in the decode step ----
    def fp8_linear_weights(self) -> List[nn.Parameter]:
        """The weights ``quantize_weights_fp8`` rounds: q/k/v/o and gate/up/down of every layer, and lm_head."""
        ps: List[nn.Parameter] = []
        for lyr in self.model.layers:
            a, m = lyr.self_attn, lyr.mlp
            ps += [a.q_proj.weight, a.k_proj.weight, a.v_proj.weight, a.o_proj.weight, m.gate_proj.weight, m.up_proj.weight,
                   m.down_proj.weight]
        return ps + [self.lm_head.weight]

    @torch.no_grad()
    def quantize_weights_fp8(self) -> int:
        """Round every LM linear weight IN PLACE to W' = e4m3(W / 2^e_n) * 2^e_n (one power-of-two exponent per output row,
        include/navillm_b200.h) and keep an fp8 copy of them (about 6.6 GB at Vicuna-7B).  W' is exact in bf16, so the
        model afterwards IS the model with weights W': prefill, navigation, training and ``state_dict()`` all see W'.
        The inference GEMMs then stream the fp8 copy (half the bytes; the same bits as the bf16 kernels on W'): every
        decode-step GEMM of ``generate`` and its lm_head at batches up to ``llama.FP8_MAX_ROWS``, and the GEMMs of at most
        that many rows in no-grad forwards (navigation and grounding steps, prefix-cached suffixes, prefills, the pruned
        last layer).  Training forwards and the LM-loss lm_head keep the bf16 weights.  Irreversible: reload the checkpoint
        to get W back.  Any later write to the weights (an optimizer step, ``load_state_dict``) makes ``generate`` raise
        until this is called again (or ``drop_fp8_weights``); the no-grad forwards then run bf16 on the current weights.
        Returns the size of the copy in bytes."""
        self._ensure()
        self.drop_fp8_weights()
        self._fp8 = Fp8Weights(self.flat, self.fp8_linear_weights())
        self.core.set_fp8(self._fp8)
        return self._fp8.nbytes

    def drop_fp8_weights(self) -> None:
        """Free the fp8 copy; ``generate`` goes back to the bf16 kernels (on the weights as they are, W' if quantized)."""
        self._fp8 = None
        if self.core is not None:
            self.core.set_fp8(None)
        self.__dict__.pop("_decode_states", None)     # captured decode graphs hold the pointers of the other kernels

    @property
    def fp8_weights(self) -> Optional[Fp8Weights]:
        return self.__dict__.get("_fp8")

    def _check_fp8_fresh(self) -> None:
        fp8 = self.fp8_weights
        if fp8 is None:
            return
        why = fp8.stale_reason(self.flat)
        if why is not None:
            raise RuntimeError(f"generate(): the fp8 copy of the weights is stale ({why} after quantize_weights_fp8()); call "
                               f"quantize_weights_fp8() again to re-quantize the current weights, or drop_fp8_weights() to "
                               f"decode with them in bf16")
        if self.core.fp8 is None:                    # the decoder stack was rebuilt around the same buffer
            self.core.set_fp8(fp8)

    # ---- opt-in fp8 (e4m3) activations (W8A8) in the no-grad prompt forwards ----
    activation_dtype = "bf16"

    def set_activation_dtype(self, dtype: str) -> str:
        """Number format of the decoder-layer GEMM inputs in the no-grad prompt forwards: ``"bf16"`` (default) or ``"fp8"``.
        Returns the previous format.

        ``"fp8"`` needs ``quantize_weights_fp8()``.  The four decoder-layer linears (q|k|v, o_proj, gate|up, down) then run on
        the e4m3 tensor cores (W8A8) in every no-grad forward at every row count: navigation and grounding evaluation, no-grad
        LM forwards, the prefill of ``generate()``, and ``PrefixKVCache`` suffix steps with the bf16 or the fp8 store.  Each
        GEMM input (the RMSNorm, attention or SwiGLU output) is quantized per (row, 128-column block) with the weight rule
        (include/navillm_b200.h), so a prompt's outputs do not depend on the batch it came in.  Decode steps, lm_head, the
        heads, the panorama encoder and every grad-enabled forward are unchanged.  A forward raises, naming the remedy, when
        the fp8 weight copy is missing or stale or when the hidden or intermediate size is not a multiple of 128; it never
        falls back to bf16.  Its effect on task metrics has not been measured."""
        if dtype not in ("bf16", "fp8"):
            raise ValueError(f"set_activation_dtype: 'bf16' or 'fp8' expected, got {dtype!r}")
        prev, self.activation_dtype = self.activation_dtype, dtype
        if self.core is not None:
            self.core.act_fp8 = dtype == "fp8"
        return prev

    # ---- opt-in fp8 (e4m3) KV cache in generate() ----
    kv_cache_dtype = "bf16"

    def set_kv_cache_dtype(self, dtype: str) -> str:
        """Storage format of ``generate()``'s KV cache: ``"bf16"`` (default) or ``"fp8"``.  Returns the previous format.

        ``"fp8"`` stores every cached (sequence, position, head) row of K and V as e4m3 with one power-of-two exponent per
        row (include/navillm_b200.h): half the cache memory, and half the bytes each decode step's attention reads.  The
        prefill's attention over the prompt reads the unrounded K/V, so the first generated token is the bf16 one; every
        later step attends over the rounded K'/V' (exactly, as bf16 attention over K'/V' would).  This covers greedy,
        sampled and trie-constrained decoding, graphed or eager, with or without ``quantize_weights_fp8()``, at any batch
        size.  The choice is always the caller's: a rule that depended on the batch size would make one prompt's tokens
        depend on the batch it came in.  Its effect on task metrics has not been measured."""
        if dtype not in ("bf16", "fp8"):
            raise ValueError(f"set_kv_cache_dtype: 'bf16' or 'fp8' expected, got {dtype!r}")
        prev, self.kv_cache_dtype = self.kv_cache_dtype, dtype
        return prev

    # ---- generation (models/nav_model.py:324-338,388-399; HF GenerationMixin greedy / sampling) ----
    decode_pdl = os.environ.get("NAVILLM_DECODE_PDL", "1") != "0"   # developer knob: 0 = plain stream-ordered launches
    max_decode_states = 2        # cached (KV buffers + captured decode graph) sets, least recently used evicted

    def _decode_state(self, B: int, Smax: int, key_extra: tuple, want_graph: bool):
        """Persistent per-shape decode state: the contiguous KV cache [B, Smax, D] per layer (in ``kv_cache_dtype``; the caller
        puts that format in ``key_extra``, so a graph is never replayed over the other one), the step's I/O buffers and --
        once captured -- the CUDA graph of ONE decode step.  Capturing and instantiating the ~260-node graph costs more than
        the 127 replays of a C3 generation save, so it is done once per (batch, cache length, stop rule, decoding mode and
        the scalars the step bakes in) and reused by every later ``generate`` call (evaluation loops call generate with the
        same shapes over and over).  The trie-constrained modes keep their flattened trie in ``trie_buf`` (see
        ``_load_trie``), sampled modes their uniform numbers in ``u``."""
        states = self.__dict__.setdefault("_decode_states", collections.OrderedDict())
        key = (B, Smax) + key_extra
        st = states.get(key) if want_graph else None
        if st is not None:
            states.move_to_end(key)
            return st
        dev, d = self._device(), self.dims
        V = self.lm_head.weight.shape[0]
        if self.kv_cache_dtype == "fp8":                          # (e4m3 bytes, int8 row exponents) per layer
            cache = lambda: [(torch.empty((B, Smax, d.hidden), dtype=ops.fp8, device=dev),
                              torch.empty((B, Smax, d.n_heads), dtype=torch.int8, device=dev)) for _ in range(d.n_layers)]
        else:
            cache = lambda: [torch.empty((B, Smax, d.hidden), dtype=bf16, device=dev) for _ in range(d.n_layers)]
        st = SimpleNamespace(
            kc=cache(), vc=cache(),
            logits=torch.empty((B, (V + 63) // 64 * 64), dtype=bf16, device=dev)[:, :V],
            next_ids=torch.empty((B,), dtype=torch.int32, device=dev),
            finished=torch.zeros((B,), dtype=torch.int32, device=dev),
            lens=torch.zeros((B,), dtype=torch.int32, device=dev), graph=None,
            u=None, masked=None, node=None, miss=None, trie_buf=None, trie_cap=(0, 0))
        if want_graph:
            states[key] = st
            while len(states) > self.max_decode_states:
                states.popitem(last=False)
        return st

    @staticmethod
    def _load_trie(st, table) -> tuple:
        """Copy a flattened trie into the state's persistent device buffers (a captured graph keeps their pointers) in one
        host-to-device copy.  Capacities grow in powers of two; growing drops the state's graph.  Returns the kernel's
        (node_ptr, child_tok, child_node, n_nodes) views."""
        ncap, ecap = st.trie_cap
        if table.n_nodes > ncap or table.n_edges > ecap:
            pow2 = lambda n: 1 << max(0, int(n) - 1).bit_length()
            ncap, ecap = max(ncap, pow2(table.n_nodes)), max(ecap, pow2(max(table.n_edges, 1)))
            st.trie_buf = torch.empty(ncap + 2 + 2 * ecap, dtype=torch.int32, device=st.next_ids.device)
            st.trie_cap = (ncap, ecap)
            st.graph = None
        st.trie_buf.copy_(torch.from_numpy(table.pack(ncap, ecap)))
        o = ncap + 2
        return st.trie_buf[:o], st.trie_buf[o:o + ecap], st.trie_buf[o + ecap:], ncap

    @torch.no_grad()
    def generate(self, input_ids, attention_mask, cand_vis=None, hist_vis=None, obj_vis=None, max_new_tokens: int = 20,
                 do_sample: bool = False, temperature: float = 1.0, eos_token_id: Optional[int] = None,
                 pad_token_id: Optional[int] = None, bos_token_id: Optional[int] = None, logits_processor=None, trie=None,
                 stop_on_eos: bool = True, use_cuda_graph: bool = True, stats: Optional[dict] = None, top_k: int = 50,
                 top_p: float = 1.0, **unused) -> torch.Tensor:
        """Prefill on the packed kernels (positions = cumsum(mask)-1 like HF generate; visual tokens injected only
        here, as in models/modified_lm.py:195-197), then one token per step over a pre-allocated KV cache.  The
        decode step of the greedy, sampled and trie-constrained modes has static shapes and is replayed as a CUDA graph
        (captured once per shape and mode, see ``_decode_state``); generic ``logits_processor=`` calls run eagerly.
        Returns [B, S0 + n_new] int64 ids (prompt part copied from the input; finished rows continue with pad_token_id
        like HF greedy search).

        ``do_sample=True`` follows HF ``sample`` as the reference reaches it (tasks/agents/llava.py:58-62): logits
        processors, then temperature and top-k (``top_k=50`` is transformers' generation default, which the reference
        never overrides), bf16 softmax, one multinomial draw per row - all in ``nv_sample_topk``; the uniform numbers
        are one [B] draw per token from the default CUDA generator, so ``torch.manual_seed`` makes a run reproducible,
        and the graph replays draw the same numbers as ``use_cuda_graph=False``.

        ``trie=`` (TrieLogitsProcessor, models/modified_lm.py:10-30) walks the trie on the device (``nv_trie_mask``
        between the lm_head and the pick) and replays as a CUDA graph too; the stop check stays per token, as on the host.
        A trie ``navillm_b200.trie.flatten_trie`` cannot represent faithfully, ``trie=`` together with
        ``logits_processor=``, and a call whose device walk reports a miss (a picked token outside the allowed set, which
        only a degenerate row can produce) run the host ``TrieLogitsProcessor`` instead - the miss case reruns the whole
        call, with the CUDA RNG state restored, and discards the device result."""
        if top_p is not None and top_p < 1.0:
            raise NotImplementedError("generate(top_p < 1) is not built: the reference never sets it (HF default 1.0)")
        if do_sample and not temperature > 0:
            raise ValueError("generate(do_sample=True) needs temperature > 0")
        self._ensure()
        self._check_fp8_fresh()
        dev = self._device()
        eos = self.tokenizer.eos_token_id if eos_token_id is None else eos_token_id
        pad = self.tokenizer.unk_token_id if pad_token_id is None else pad_token_id
        procs = list(logits_processor or [])
        args = (input_ids, attention_mask, cand_vis, hist_vis, obj_vis, max_new_tokens, do_sample, temperature, eos, pad,
                stop_on_eos, use_cuda_graph, stats, top_k)
        table, path = None, None
        if trie is not None and not procs:
            t0 = time.perf_counter()
            table = trie_mod.flatten_trie(trie, self.lm_head.weight.shape[0])
            flatten_ms = 1e3 * (time.perf_counter() - t0)
        if table is not None:
            rng = torch.cuda.get_rng_state(dev) if do_sample else None
            out = self._generate(*args, procs=[], table=table)
            path = "device" if out is not None else "device_miss_host"
            if out is None:
                if rng is not None:
                    torch.cuda.set_rng_state(rng, dev)
                out = self._generate(*args, procs=[trie_mod.TrieLogitsProcessor(trie)], table=None)
        else:
            if trie is not None:
                procs = [trie_mod.TrieLogitsProcessor(trie)] + procs
                path = "host"
            out = self._generate(*args, procs=procs, table=None)
        if stats is not None and trie is not None:
            stats.update({"trie_path": path, "trie_flatten_ms": flatten_ms if table is not None else None})
        return out

    def _generate(self, input_ids, attention_mask, cand_vis, hist_vis, obj_vis, max_new_tokens, do_sample, temperature, eos, pad,
                  stop_on_eos, use_cuda_graph, stats, top_k, *, procs, table):
        """``generate`` with the host processors ``procs`` (the host path when not empty) or the flattened trie ``table``
        walked on the device; returns None when the device walk reported a miss."""
        dev = self._device()
        core, d = self.core, self.dims
        ev = None
        if stats is not None:                                     # bench.py: device-side phase times (forces one sync at the end)
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            ev[0].record()
        pp = PackedPrompt(input_ids, attention_mask, self, dev, generate_positions=True)
        vis = self.cat_vis(cand_vis, hist_vis, obj_vis, pp)
        B = pp.B
        need_host = bool(procs)                                   # processors walk the generated ids on the host
        graphed = use_cuda_graph and not need_host
        mode = ("trie+sample" if do_sample else "trie") if table is not None else ("sample" if do_sample else "greedy")
        Smax = (max(pp.seqlens) + max_new_tokens + 127) // 128 * 128          # bucketed: more reuse of the cached state
        key = (int(eos), int(pad), bool(stop_on_eos), mode, float(temperature) if do_sample else None,
               int(top_k) if do_sample else None, table.eos if table is not None else None, self.kv_cache_dtype)
        st = self._decode_state(B, Smax, key, graphed)
        kc, vc, logits, next_ids, finished, lens = st.kc, st.vc, st.logits, st.next_ids, st.finished, st.lens
        if do_sample and not need_host and st.u is None:
            st.u = torch.empty((B,), dtype=torch.float32, device=dev)
        if table is not None:
            if st.masked is None:
                V = logits.shape[1]
                st.masked = torch.empty((B, (V + 63) // 64 * 64), dtype=bf16, device=dev)[:, :V]
                st.node = torch.zeros((B,), dtype=torch.int32, device=dev)
                st.miss = torch.zeros((1,), dtype=torch.int32, device=dev)
            trie_csr = self._load_trie(st, table)
        finished.zero_()
        lens.copy_(torch.tensor(pp.seqlens, dtype=torch.int32), non_blocking=True)

        E = self.model.embed_tokens.weight.data
        x = ops.embed_fwd(pp.ids, E, pp.vis_src if vis is not None else None, vis)
        hid_last, _ = core.forward(x, pp.pos, pp.cu, pp.seqlens, save=False, kv_store=(kc, vc), out_rows=pp.last_rows)
        special = self.special_ids_dev

        fp8_head = None
        if core.fp8 is not None:
            fp8_head = self._fp8.view([self.lm_head.weight], tuple(self.lm_head.weight.shape))

        def head(h_rows):
            hn, _ = ops.rmsnorm_fwd(h_rows, self.model.norm.weight.data, d.rms_eps)
            if B <= 16 and llama_mod.DECODE_BLOCK_N == 0 and fp8_head is not None:
                ops.gemm_skinny_fp8(hn, *fp8_head, out=logits)
            elif B <= llama_mod.FP8_MAX_ROWS and llama_mod.DECODE_BLOCK_N == 0 and fp8_head is not None:
                ops.gemm_fp8w(hn, *fp8_head, out=logits)
            elif B <= 16 and llama_mod.DECODE_BLOCK_N == 0:
                ops.gemm_skinny(hn, self.lm_head.weight.data, out=logits)
            else:
                ops.gemm(hn, self.lm_head.weight.data, out=logits, block_n=llama_mod.DECODE_BLOCK_N)

        def pick_host(all_ids_host):
            """next token from `logits` -> next_ids (device), through the host processors."""
            lg = logits.float()
            lg[:, self.special_token_ids] = float("-inf")
            for proc in procs:
                lg = proc(torch.tensor(all_ids_host, device=dev), lg)
            if do_sample:
                ops.sample_topk(lg.to(torch.bfloat16), special, finished, eos, pad, stop_on_eos, temperature, top_k,
                                torch.rand(B, device=dev, dtype=torch.float32), next_ids)
                return
            nxt = lg.argmax(dim=-1)
            fin = finished.bool()
            nxt = torch.where(fin, torch.full_like(nxt, pad), nxt)
            if stop_on_eos:
                finished.copy_((fin | (nxt == eos)).to(torch.int32))
            next_ids.copy_(nxt.to(torch.int32))

        def pick(advance):
            """next token from `logits` -> next_ids (device) without host work; with a trie, the row's node first advances by
            the token in next_ids (``advance``) and the pick reads the trie-masked copy of the logits."""
            src = logits
            if table is not None:
                ops.trie_mask(logits, st.masked, *trie_csr, table.eos, special, st.node, next_ids if advance else None, st.miss)
                src = st.masked
            if do_sample:
                st.u.uniform_()                                   # = torch.rand(B): the same numbers, into a static buffer
                ops.sample_topk(src, special, finished, eos, pad, stop_on_eos, temperature, top_k, st.u, next_ids)
            else:
                ops.argmax_masked(src, special, finished, eos, pad, stop_on_eos, next_ids)

        head(hid_last)
        host_ids = [row.tolist() for row in input_ids.cpu()] if need_host else None
        if need_host:
            pick_host(host_ids)
        else:
            if table is not None:                                 # every row starts at the root, in stream order
                st.node.zero_()
                st.miss.zero_()
            pick(advance=False)
        out_tokens = [next_ids.clone()]
        if ev is not None:
            ev[1].record()

        def step():
            with ops.pdl(self.decode_pdl):          # programmatic dependent launch along the whole decode chain
                xt = ops.embed_fwd(next_ids, E)
                h = core.decode_step(xt, lens, kc, vc)
                head(h)
                ops.add_int_(lens, 1)
                if not need_host:
                    pick(advance=True)

        # HF stops when every sequence has finished.  Asking the device after EVERY token would serialise host and device
        # (one blocking read per token); finished rows only emit pad tokens, so the greedy and sampled loops look every
        # `check_every` tokens and the surplus pad columns are trimmed below -- same ids as a per-token check.  Trie-constrained
        # answers are a handful of tokens: there the check stays per token, as on the host path.
        check_every = 1 if need_host or table is not None else 8
        replays = 0
        for it in range(1, max_new_tokens):
            if stop_on_eos and it % check_every == 0 and bool(finished.all()):
                break
            if need_host:
                for bn, t in enumerate(out_tokens[-1].tolist()):
                    host_ids[bn].append(t)
            if graphed:
                if st.graph is None:                              # first generation with this shape: eager step, then capture
                    step()
                    out_tokens.append(next_ids.clone())
                    g = torch.cuda.CUDAGraph()
                    torch.cuda.synchronize()
                    with torch.cuda.graph(g):
                        step()
                    st.graph = g
                    continue
                st.graph.replay()
                replays += 1
            else:
                step()
                if need_host:
                    pick_host(host_ids)
            out_tokens.append(next_ids.clone())
        miss = False
        if table is not None:
            # one more advance, outside the graph: a token picked at the last step that is not a child is a miss as well
            ops.trie_mask(logits, st.masked, *trie_csr, table.eos, special, st.node, next_ids, st.miss)
            miss = bool(st.miss.item())
        if ev is not None:
            ev[2].record()
            torch.cuda.synchronize()
            n_dec = len(out_tokens) - 1
            stats.update({"prefill_ms": ev[0].elapsed_time(ev[1]), "decode_ms": ev[1].elapsed_time(ev[2]) if n_dec else None,
                          "decode_steps": n_dec, "graph_replays": replays, "kv_rows": Smax, "prompt_lens": list(pp.seqlens)})
        if miss:
            return None
        new = torch.stack(out_tokens, dim=1).to(torch.int64)
        if stop_on_eos and check_every > 1 and new.shape[1] > 1:
            # trim the columns generated after the step at which the last row emitted EOS (see check_every above)
            is_eos = (new == eos)
            if bool(is_eos.any(dim=1).all()):
                last = int(is_eos.float().argmax(dim=1).max())        # first EOS per row; the slowest row decides
                new = new[:, :last + 1]
        return torch.cat([input_ids.to(dev), new], dim=1)
