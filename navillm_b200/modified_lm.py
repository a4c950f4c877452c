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

import contextlib
import dataclasses
import math
import numbers
import os
import time
import weakref
from types import SimpleNamespace
from typing import List, Optional

import numpy as np
import torch
import torch.nn as nn

from . import generation
from . import ops
from . import trie as trie_mod
from .llama import FlatParams, Fp8Weights, Int4Calibration, Int4Weights, LlamaCore, LlamaDims, LlamaModelParams, WgradStash, _Linear, kv_cache
from .parallel import GradSync
from .tokenizer import HFTokenizerAdapter, SyntheticTokenizer

bf16 = torch.bfloat16


class LMOutput(SimpleNamespace):
    """Stand-in for transformers.CausalLMOutputWithPast (attribute and item access)."""

    def __getitem__(self, k):
        return getattr(self, k)


class _GenerateOutput(LMOutput):
    """Stand-in for transformers 4.28's generate() output classes: the fields in 4.28's order, attribute access, item access by
    name, and by position over the fields that are not None (ModelOutput.to_tuple)."""
    FIELDS: tuple = ()

    def __init__(self, **kw):
        super().__init__(**{f: kw.get(f) for f in self.FIELDS})

    def to_tuple(self) -> tuple:
        return tuple(getattr(self, f) for f in self.FIELDS if getattr(self, f) is not None)

    def __getitem__(self, k):
        return self.to_tuple()[k] if isinstance(k, int) else getattr(self, k)


class GreedySearchDecoderOnlyOutput(_GenerateOutput):
    FIELDS = ("sequences", "scores", "attentions", "hidden_states")


class SampleDecoderOnlyOutput(_GenerateOutput):
    FIELDS = ("sequences", "scores", "attentions", "hidden_states")


class ContrastiveSearchDecoderOnlyOutput(_GenerateOutput):
    FIELDS = ("sequences", "scores", "attentions", "hidden_states")


class BeamSearchDecoderOnlyOutput(_GenerateOutput):
    FIELDS = ("sequences", "sequences_scores", "scores", "beam_indices", "attentions", "hidden_states")


def compute_transition_scores(sequences: torch.Tensor, scores, beam_indices: Optional[torch.Tensor] = None,
                              normalize_logits: bool = False) -> torch.Tensor:
    """transformers 4.28's GenerationMixin.compute_transition_scores: the score of each generated token, fp32 [rows, n] (the
    scores are cast to fp32 first, so ``normalize_logits`` log-softmaxes in fp32).  Without ``beam_indices`` row r reads
    scores[t][r] (greedy / sampled / contrastive); with them, step t of hypothesis i reads row beam_indices[i, t], a -1 reads
    row 0 and is zeroed, and the columns stop at the longest hypothesis."""
    if beam_indices is None:
        beam_indices = torch.arange(scores[0].shape[0]).view(-1, 1).to(sequences.device)
        beam_indices = beam_indices.expand(-1, len(scores))
    V = scores[0].shape[-1]
    sc = torch.stack(scores).float().reshape(len(scores), -1).transpose(0, 1)          # [rows * V, steps]
    if normalize_logits:
        sc = torch.nn.functional.log_softmax(sc.reshape(-1, V, sc.shape[-1]), dim=1).reshape(-1, sc.shape[-1])
    mask = beam_indices < 0
    max_len = int((1 - mask.long()).sum(-1).max())
    beam_indices = beam_indices.clone()[:, :max_len]
    mask = mask[:, :max_len]
    beam_indices[mask] = 0
    indices = sequences[:, sequences.shape[-1] - max_len:] + beam_indices * V
    out = sc.gather(0, indices)
    out[mask] = 0
    return out


def _lookup_k(k, ngram) -> tuple:
    """``generate(prompt_lookup_num_tokens=k, max_matching_ngram_size=ngram)`` as (drafts per step, ngram): k = 0 for None or 0
    (plain greedy decoding), else an int in 1 .. 15 (the window kernel's 16 rows); ngram None is HF's 2.  Any other k, or an
    ngram below 1, is a ``ValueError``."""
    if k is None or (not isinstance(k, bool) and isinstance(k, int) and k == 0):
        return 0, 0
    ngram = 2 if ngram is None else ngram
    if isinstance(k, bool) or not isinstance(k, int) or not 1 <= k <= ops.LOOKUP_WMAX - 1:
        raise ValueError(f"generate(prompt_lookup_num_tokens={k!r}): an int in 1 .. {ops.LOOKUP_WMAX - 1} expected (0 or None: off)")
    if isinstance(ngram, bool) or not isinstance(ngram, int) or ngram < 1:
        raise ValueError(f"generate(max_matching_ngram_size={ngram!r}): a positive int expected")
    return k, ngram


def _beam_groups(num_beams, num_beam_groups, diversity_penalty, do_sample: bool, other_processors: bool) -> int:
    """``generate(num_beam_groups=G, diversity_penalty=d)`` validated as transformers 4.28 does (``ValueError``), before any
    device work; returns G (1: no groups).  Groups without a penalty (None or 0), with sampling, or with ``trie=`` /
    ``logits_processor=`` are not built (``NotImplementedError`` naming "group").  ``d`` without groups is ignored."""
    if num_beam_groups is None or num_beam_groups <= 1:                  # as before: no groups (1, 1.0, np.int64(1), ...)
        return 1
    if isinstance(num_beam_groups, bool) or not isinstance(num_beam_groups, numbers.Integral):
        raise ValueError(f"generate(num_beam_groups={num_beam_groups!r}): `num_beam_groups` has to be an integer")
    groups = int(num_beam_groups)
    if groups > num_beams:
        raise ValueError(f"generate(num_beam_groups={groups}, num_beams={num_beams}): `num_beam_groups` has to be smaller or "
                         "equal to `num_beams`")
    if num_beams % groups:
        raise ValueError(f"generate(num_beam_groups={groups}, num_beams={num_beams}): `num_beams` has to be divisible by "
                         "`num_beam_groups`")
    if do_sample:
        raise NotImplementedError("generate(num_beam_groups > 1, do_sample=True): group (diverse) beam sampling is not built")
    if diversity_penalty is None or (not isinstance(diversity_penalty, bool) and diversity_penalty == 0):
        raise NotImplementedError("generate(num_beam_groups > 1) without diversity_penalty > 0: group beam search without a "
                                  "penalty is G copies of one search and is not built")
    if isinstance(diversity_penalty, bool) or not isinstance(diversity_penalty, float) or not diversity_penalty > 0:
        raise ValueError(f"generate(diversity_penalty={diversity_penalty!r}): `diversity_penalty` should be a float strictly "
                         "larger than 0")
    if other_processors:
        raise NotImplementedError("generate(num_beam_groups > 1) with trie= / logits_processor=: group (diverse) beam search "
                                  "runs the device processors only")
    return groups


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
        # batch-invariant no-grad forwards take generate's positions too: arange(S) would move a left-padded prompt's rotary
        # positions with the batch's longest prompt (the same attention up to the rounding of the cos/sin tables)
        invariant = callable(getattr(lm, "invariant_inference", None)) and lm.invariant_inference()
        if generate_positions or invariant:                               # HF generate: cumsum(mask) - 1
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
        self.kc = kv_cache(d, batch_size, max_len, kv_dtype, dev, zero=True)
        self.vc = kv_cache(d, batch_size, max_len, kv_dtype, dev, zero=True)
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
        return self._lm().flat.weight_state()

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
                      hist_id: int, cls_id: int, invariant: bool = False):
    """Host-side plan of one cached navigation step (pure numpy; updates ``cache.ids`` / ``cache.off``).  ``invariant``
    (batch-invariant mode): a new row's rotary offset is 0 instead of its left padding.

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
        if cache.off[b] is None:                               # the row keeps this rotary offset for the rollout; in
            # batch-invariant mode 0 (generate's positions), else the reference's S - L, which follows the longest prompt
            cache.off[b] = 0 if invariant else S - L
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
        logits = generation.logits_buffer(g.shape[0], V, g.device)
        head = ops.gemm_bi if lm.invariant_inference() else ops.gemm
        head(hn, lm.lm_head.weight.data, out=logits)                     # [Nl, V] bf16
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
        # (nor does a deferred weight gradient, final only at its flush)
        overlap = kv is None and not lm.prefix_grads_pending() and lm._wgrad_stash is None
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
        self.grad_sync.before_exchange = self.complete_pending_grads
        self._prefix_caches = weakref.WeakSet()      # PrefixKVCache(train=True) instances built on this model
        self._decode_states = generation.DecodeStates()  # generate()'s KV caches and captured decode graphs
        self.batch_invariant = os.environ.get("NAVILLM_BATCH_INVARIANT", "") == "1"   # set_batch_invariant
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
        self._decode_states.clear()                  # captured decode graphs hold pointers into the old buffers
        self.flat = FlatParams(params, device)
        self.flat.clean_segments = self._clean_grad_segments
        self.flat.on_zeroed = self.mark_grads_zeroed
        self._lm_head_grad_clean = False             # unknown until the next zero_grad
        self.core = LlamaCore(self.dims, self.model, self.flat)
        self.core.act_fp8 = self.activation_dtype == "fp8"
        self.core.batch_invariant = self.batch_invariant
        if self._wgrad_stash is not None:
            self._wgrad_stash.core = self.core
            self.core.wgrad_stash = self._wgrad_stash
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
                                 self.cls_token_id[0], invariant=self.invariant_inference())
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
                head = ops.gemm_bi if self.invariant_inference() else ops.gemm
                lg = head(hn.detach().contiguous(), self.lm_head.weight.data)
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
        Returns the size of the copy in bytes.  Drops the int4 copy (``quantize_weights_int4``) if there is one; quantizing
        after that rounds its W' further."""
        self._refuse_in_batch_invariant("quantize_weights_fp8()")
        self._ensure()
        self.drop_int4_weights()
        self.drop_fp8_weights()
        self._fp8 = Fp8Weights(self.flat, self.fp8_linear_weights())
        self.core.set_fp8(self._fp8)
        return self._fp8.nbytes

    def drop_fp8_weights(self) -> None:
        """Free the fp8 copy; ``generate`` goes back to the bf16 kernels (on the weights as they are, W' if quantized)."""
        self._fp8 = None
        if self.core is not None:
            self.core.set_fp8(None)
        self._decode_states.clear()                  # captured decode graphs hold the pointers of the other kernels

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

    # ---- opt-in 4-bit group-wise weight streaming (W4A16) in the decode step ----
    def int4_linear_weights(self) -> List[nn.Parameter]:
        """The weights ``quantize_weights_int4`` rounds: q/k/v/o and gate/up/down of every layer (lm_head stays bf16)."""
        return self.fp8_linear_weights()[:-1]

    @contextlib.contextmanager
    def int4_calibration(self):
        """Record the Hessians GPTQ needs from the forwards run inside the block; yields an ``Int4Calibration``::

            with model.int4_calibration() as cal:
                with torch.no_grad():
                    model('navigation', batch)          # any LM forward: prompts, prefix-cached suffixes, prefills
            model.quantize_weights_int4(calibration=cal)
            del cal                                     # frees the Hessians

        Every forward through the decoder stack adds its rows (the decode steps of ``generate()`` do not); its outputs are
        bit for bit those of the per-kernel path, which the forwards take while the block is open.  All Hessians come
        from the unquantized model in one pass (no sequential re-recording through already-quantized layers).  The
        Hessians take ``cal.nbytes`` of device memory (21.95 GB at Vicuna-7B widths).  One calibration at a time."""
        self._ensure()
        if self.core.calibration is not None:
            raise RuntimeError("int4_calibration(): a calibration is already open on this model; leave its `with` block "
                               "first")
        cal = Int4Calibration(self.core)
        core = self.core
        core.calibration = cal
        try:
            yield cal
        finally:
            cal.open = False
            if core.calibration is cal:
                core.calibration = None

    @torch.no_grad()
    def quantize_weights_int4(self, calibration: Optional[Int4Calibration] = None, damp: float = 0.01) -> int:
        """Round every decoder-layer linear weight IN PLACE to W' = bf16((q - z) * s): 4-bit codes q with one bf16 scale s
        and one 4-bit zero-point z per row and 128 columns (round to nearest; rule in include/navillm_b200.h), and keep a
        4-bit copy of them (about 3.4 GB at Vicuna-7B).

        ``calibration`` (from ``int4_calibration()``, closed, taken on the current weights): the codes come from GPTQ
        instead, which feeds each column's rounding error forward onto the columns not yet rounded so that the layer's
        output error on the recorded inputs, not the weight error, is minimised.  ``damp`` adds damp * mean(diag H) to
        H's diagonal before the factorisation; raise it if a factorisation fails.  The format, the copy and everything
        below are the same either way.  The model afterwards IS the
        model with weights W': prefill, navigation, training and ``state_dict()`` all see W'.  The decode-step GEMMs of
        ``generate`` with at most 16 rows (q|k|v, o_proj, gate|up with SwiGLU, down_proj) then stream the copy, a quarter of
        the bf16 bytes, with the same bits as the bf16 kernels on W'; so do the q|k|v projections of 17..``llama.INT4_MAX_ROWS``
        rows, in the decode step (larger batches, beams, several samples per prompt) and in the no-grad forwards while the
        copy is fresh.  The other GEMMs above 16 rows run the bf16 kernels on W'.  lm_head is neither rounded nor streamed in
        4 bits, and training keeps the bf16 kernels.  Needs hidden and intermediate sizes that are multiples of 128.
        Irreversible: reload the checkpoint to get W back.  Any later write to the weights makes ``generate`` raise until
        this is called again (or ``drop_int4_weights``); the no-grad forwards then run bf16 on the current weights.

        The fp8 and int4 copies exclude each other: this drops the fp8 copy (``quantize_weights_fp8``), and quantizing to
        fp8 drops this one.  The roundings compose: after ``quantize_weights_fp8()`` the weights are the fp8 W', and this
        rounds that W' to 4 bits (and the other way round).  Returns the size of the copy in bytes."""
        self._refuse_in_batch_invariant("quantize_weights_int4()")
        self._ensure()
        if calibration is not None:
            calibration.check(self.flat, damp)
        self.drop_fp8_weights()
        self.drop_int4_weights()
        self._int4 = Int4Weights(self.flat, self.int4_linear_weights(), calibration=calibration, damp=damp)
        self.core.set_int4(self._int4)
        return self._int4.nbytes

    def drop_int4_weights(self) -> None:
        """Free the int4 copy; ``generate`` goes back to the bf16 kernels (on the weights as they are, W' if quantized)."""
        self._int4 = None
        if self.core is not None:
            self.core.set_int4(None)
        self._decode_states.clear()                  # captured decode graphs hold the pointers of the other kernels

    @property
    def int4_weights(self) -> Optional[Int4Weights]:
        return self.__dict__.get("_int4")

    def _check_int4_fresh(self) -> None:
        int4 = self.int4_weights
        if int4 is None:
            return
        why = int4.stale_reason(self.flat)
        if why is not None:
            raise RuntimeError(f"generate(): the int4 copy of the weights is stale ({why} after quantize_weights_int4()); call "
                               f"quantize_weights_int4() again to re-quantize the current weights, or drop_int4_weights() to "
                               f"decode with them in bf16")
        if self.core.int4 is None:                   # the decoder stack was rebuilt around the same buffer
            self.core.set_int4(int4)

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
        if dtype == "fp8" and self.batch_invariant:
            raise ValueError("set_activation_dtype('fp8'): batch-invariant mode is on, and W8A8 is not part of its "
                             "arithmetic; call set_batch_invariant(False) first")
        prev, self.activation_dtype = self.activation_dtype, dtype
        if self.core is not None:
            self.core.act_fp8 = dtype == "fp8"
        return prev

    # ---- opt-in batch-invariant inference ----
    def set_batch_invariant(self, on: bool) -> bool:
        """Batch-invariant inference: while on, a prompt's no-grad LM outputs -- hidden states and logits, ``generate()`` ids
        and scores in the greedy, beam, group-beam, contrastive and prompt-lookup modes, ``score_answers`` -- are bitwise a
        function of that prompt alone, not of the batch size, the other prompts, its position among them or padding.
        Sampled modes keep HF's one RNG stream for the whole batch, so only their logits and scores are covered; a beam's
        ``sequences_scores`` keep HF's normalisation by the padded length (exact at ``length_penalty=0``).  No-grad forwards
        take generate's rotary positions (cumsum(mask) - 1) instead of arange(S), which moved with the longest prompt.
        Every inference GEMM then accumulates each element in one fp32 chain over 64-deep k-blocks, in order, without split-K
        (include/navillm_b200.h): decode steps and lm_head stream the weights through nv_gemm_bi_bf16 at every batch size,
        and the no-grad forwards run the plain GEMM with the RoPE / SwiGLU row kernels at every row count.  Training is
        unchanged.  Prefill need not equal decode, nor eager a graph replay.  The fp8 and int4 weight copies and fp8
        activations are refused while it is on.  Returns the previous value; ``NAVILLM_BATCH_INVARIANT=1`` in the
        environment makes it the default."""
        on = bool(on)
        if on and (self.fp8_weights is not None or self.int4_weights is not None or self.activation_dtype == "fp8"):
            what = ("the fp8 weight copy (drop_fp8_weights())" if self.fp8_weights is not None else
                    "the int4 weight copy (drop_int4_weights())" if self.int4_weights is not None else
                    "fp8 activations (set_activation_dtype('bf16'))")
            raise ValueError(f"set_batch_invariant(True): batch-invariant mode does not combine with {what}")
        prev, self.batch_invariant = self.batch_invariant, on
        if self.core is not None:
            self.core.batch_invariant = on
        return prev

    def invariant_inference(self) -> bool:
        """Whether batch-invariant mode governs the call being made: the mode is on and the call does not train (the
        forwards' ``train = torch.is_grad_enabled() and self.training_enabled``).  The one predicate for the positions, the
        heads, the prefix cache's offsets and the encoder's splits; inside the decoder stack the same decision arrives as
        ``save`` (a forward saves its activations exactly when it trains)."""
        return self.batch_invariant and not (torch.is_grad_enabled() and self.training_enabled)

    def _refuse_in_batch_invariant(self, what: str) -> None:
        if self.batch_invariant:
            raise ValueError(f"{what}: batch-invariant mode is on, and the quantized weight copies are not part of its "
                             f"arithmetic; call set_batch_invariant(False) first")

    # ---- opt-in deferred weight gradients of the decoder linears (WgradStash) ----
    _wgrad_stash: Optional[WgradStash] = None

    def defer_weight_grads(self, max_rows: Optional[int] = 2048) -> Optional[int]:
        """Defer the weight gradients of the decoder linears (q|k|v, o_proj, gate|up, down of every layer) across backwards:
        each backward records its wgrad operands (references to activations it computed anyway) and
        ``flush_weight_grads()`` adds them with ONE segmented-contraction GEMM per weight (``ops.gemm_wgrad_seg``).  For
        small-batch rollouts (one backward of a few hundred rows per step) this replaces a read-modify-write of the whole bf16
        gradient buffer per backward with one per flush.  A deferred gradient is the same sum as the per-backward one,
        rounded to bf16 once instead of once per backward.  RMSNorm weights, lm_head, embeddings, the heads and the panorama
        encoder keep their immediate gradients.

        ``max_rows`` bounds the stash in backward rows: a backward that would exceed it flushes first, and a backward of more
        than ``max_rows / 2`` rows (which could not share a flush with another of its size) runs its weight gradients at once.  The stash keeps (8 hidden + 3 intermediate) bf16 values per
        row and layer alive (4.2 MB a row at Vicuna-7B; ``weight_grad_stash_bytes()``).  ``None`` or 0 turns deferral off
        (flushing first).  Returns the previous setting.

        The flush runs in ``FlatAdamW.step()``, ``NavModel.allreduce_grads()`` and the data-parallel exchange of an armed pass
        (after the training prefix caches' ``flush_grads()``); anything else that reads the linears' ``.grad`` must call
        ``flush_weight_grads()`` first.  ``zero_grad()`` while rows are stashed raises, and so does a flush after the weights
        changed."""
        prev = None if self._wgrad_stash is None else self._wgrad_stash.max_rows
        if max_rows is not None and int(max_rows) < 0:
            raise ValueError(f"defer_weight_grads: max_rows must be >= 0 or None (got {max_rows})")
        self.flush_weight_grads()
        self._wgrad_stash = WgradStash(self.core, int(max_rows)) if max_rows else None
        if self.core is not None:
            self.core.wgrad_stash = self._wgrad_stash
        return prev

    def flush_weight_grads(self) -> None:
        """Add the stashed weight gradients of ``defer_weight_grads`` into ``.grad``; a no-op when nothing is stashed."""
        if self._wgrad_stash is not None:
            self._wgrad_stash.flush()

    def weight_grad_stash_bytes(self) -> int:
        """Device bytes the deferred weight gradients keep alive (0 when nothing is stashed)."""
        return 0 if self._wgrad_stash is None else self._wgrad_stash.nbytes

    def weight_grads_pending(self) -> bool:
        return self._wgrad_stash is not None and self._wgrad_stash.pending

    def complete_pending_grads(self) -> None:
        """Before a gradient exchange: part (b) of the training prefix caches, then the deferred weight gradients."""
        self.flush_prefix_caches()
        self.flush_weight_grads()

    def zero_grad(self, set_to_none: bool = True) -> None:
        if self.weight_grads_pending():
            raise RuntimeError("zero_grad(): deferred weight gradients are stashed; call flush_weight_grads() before "
                               "optimizer.step() / zero_grad()")
        super().zero_grad(set_to_none=set_to_none)

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

    # ---- generation (models/nav_model.py:324-338,388-399; HF GenerationMixin; navillm_b200/generation.py) ----
    @torch.no_grad()
    def generate(self, input_ids, attention_mask, cand_vis=None, hist_vis=None, obj_vis=None, max_new_tokens: int = 20,
                 do_sample: bool = False, temperature: float = 1.0, eos_token_id: Optional[int] = None,
                 pad_token_id: Optional[int] = None, bos_token_id: Optional[int] = None, logits_processor=None, trie=None,
                 stop_on_eos: bool = True, use_cuda_graph: bool = True, stats: Optional[dict] = None, top_k: int = 50,
                 top_p: float = 1.0, num_beams: int = 1, length_penalty: float = 1.0, early_stopping: bool = False,
                 num_return_sequences: int = 1, num_beam_groups: int = 1, repetition_penalty: Optional[float] = None,
                 no_repeat_ngram_size: Optional[int] = None, min_length: Optional[int] = None,
                 min_new_tokens: Optional[int] = None, penalty_alpha: Optional[float] = None,
                 prompt_lookup_num_tokens: Optional[int] = None, max_matching_ngram_size: Optional[int] = 2,
                 return_dict_in_generate: bool = False, output_scores: bool = False,
                 diversity_penalty: Optional[float] = None, **unused):
        """Prefill on the packed kernels (positions = cumsum(mask)-1 like HF generate; visual tokens injected only
        here, as in models/modified_lm.py:195-197), then one token per step over a pre-allocated KV cache.  The
        decode step of the greedy, sampled and trie-constrained modes has static shapes and is replayed as a CUDA graph
        (captured once per shape and mode, see ``generation.DecodeStates``); generic ``logits_processor=`` calls run eagerly.
        Returns [B, S0 + n_new] int64 ids (prompt part copied from the input; finished rows continue with pad_token_id
        like HF greedy search).

        ``do_sample=True`` follows HF ``sample`` as the reference reaches it (tasks/agents/llava.py:58-62): logits
        processors, then temperature and top-k (``top_k=50`` is transformers' generation default, which the reference
        never overrides), bf16 softmax, one multinomial draw per row - all in ``nv_sample``; the uniform numbers
        are one [B] draw per token from the default CUDA generator, so ``torch.manual_seed`` makes a run reproducible,
        and the graph replays draw the same numbers as ``use_cuda_graph=False``.

        ``trie=`` (TrieLogitsProcessor, models/modified_lm.py:10-30) walks the trie on the device (``nv_trie_mask``
        between the lm_head and the pick) and replays as a CUDA graph too; the stop check stays per token, as on the host.
        A trie ``navillm_b200.trie.flatten_trie`` cannot represent faithfully, ``trie=`` together with
        ``logits_processor=``, and a call whose device walk reports a miss (a picked token outside the allowed set, which
        only a degenerate row can produce) run the host ``TrieLogitsProcessor`` instead - the miss case reruns the whole
        call, with the CUDA RNG state restored, and discards the device result.

        ``top_p < 1`` adds HF's TopPLogitsWarper after top-k in every sampled mode (``nv_sample``); greedy and beam calls
        ignore it, as HF does.

        ``num_beams > 1`` is HF beam search as transformers 4.28 (the reference's pin) runs it, ``length_penalty``,
        ``early_stopping`` and ``num_return_sequences`` included; see ``generation.beam_search``.  Returns [B * num_return_sequences,
        L] ids.  Beam sampling, ``logits_processor=`` with beams and more return sequences than beams raise
        ``NotImplementedError``.

        ``num_beam_groups=G > 1`` with ``diversity_penalty > 0`` is 4.28's diverse (group) beam search: the K beams of a prompt
        form G groups of K / G that take their steps in order, and each group's log-probs are lowered by ``diversity_penalty``
        times the number of times the earlier groups chose the token in the same step (HammingDiversityLogitsProcessor, before
        the device processors).  All groups share the prompt's K hypotheses, as in 4.28.  It runs on the device in the captured
        step (``nv_beam_topk_group`` / ``nv_beam_select_group``, see ``generation.beam_search``); ``length_penalty``,
        ``early_stopping``, ``num_return_sequences``, the device processors, per-step scores (``beam_indices`` hold global rows
        b * K + k), the fp8 / int4 weight copies and the fp8 KV cache all apply.  ``num_beam_groups`` above ``num_beams`` or not
        dividing it, and a ``diversity_penalty`` that is not a float > 0, raise ``ValueError``; groups without a penalty (None or
        0: G identical copies of one search), with ``do_sample``, ``trie=`` or ``logits_processor=`` raise
        ``NotImplementedError``.  ``diversity_penalty`` without groups is ignored.

        ``trie=`` with ``num_beams > 1`` is 4.28's beam search with a PrefixConstrainedLogitsProcessor whose allowed tokens come
        from walking the trie: each beam walks its own generated tokens from ``trie.root`` (a node without children stays; a token
        that is not a child leads to a childless node), and at its node every log-prob but the node's children (``[trie.eos]`` at a
        childless node) becomes -inf, after the device processors and before the beam-score add.  A beam's score is therefore its
        log-probability under the full vocabulary, and ``num_return_sequences=n`` returns the n best answers of the trie, best
        first.  The walk runs inside the beam top-k on the device (``nv_beam_topk_trie``) and is graph-replayed; ``length_penalty``,
        ``early_stopping``, the device processors, the fp8 / int4 weight copies and the fp8 KV cache all apply.  The caller's trie
        is never modified.  A trie ``flatten_trie`` cannot represent raises ``NotImplementedError``, as the host processor's
        per-row state cannot follow reordered beams; ``stats`` gets ``trie_path = "device"`` and ``trie_flatten_ms``.

        ``do_sample=True, num_return_sequences=N`` draws N samples per prompt: [B * N, L] ids, row b * N + j a sample of
        prompt b (HF's order).  Each prompt is prefilled once and its N rows share its KV cache (``generation.decode``); the tokens
        are those of the same call on the prompts repeated N times.  With ``trie=`` / ``logits_processor=``, and without
        ``do_sample``, N > 1 raises ``NotImplementedError``.

        ``repetition_penalty``, ``no_repeat_ngram_size``, ``min_length`` and ``min_new_tokens`` are HF's logits processors as
        transformers 4.28 applies them, in every mode above: after the special-token mask and before ``trie=`` /
        ``logits_processor=``, on the bf16 next-token logits (greedy, sampled: before the warpers) or on the bf16 log-probs
        before the beam-score add (beams).  Their history is HF's ``input_ids``: the padded prompt row as passed, left pads
        included, then the row's (beam's, sample's) generated tokens.  They run on the device (``nv_logits_process``,
        ``nv_beam_topk_processed``) inside the captured step; values are checked as HF checks them (``ValueError``), and the
        defaults (1.0 / None or 0) leave the call on the processor-free path.

        ``penalty_alpha > 0`` with ``top_k > 1`` (the default 50 included), ``do_sample=False`` and ``num_beams=1`` is 4.28's
        contrastive search: each step the ``top_k`` most probable tokens run as candidate rows over the prompt's cache, and the
        one with the best (1 - penalty_alpha) * p - penalty_alpha * (its largest cosine similarity to the hidden states so far)
        is kept (``generation.contrastive_search``; the context starts at the prompt's non-pad positions).  Returns [B, S0 +
        n_new] ids like greedy decoding.  ``num_return_sequences > 1`` and a non-finite ``penalty_alpha`` raise ``ValueError``;
        ``trie=`` / ``logits_processor=`` and ``top_k`` above ``ops.CONTRASTIVE_KMAX`` raise ``NotImplementedError``.  Every
        other ``penalty_alpha`` (None, 0, or with ``top_k <= 1``, sampling or beams) is ignored, as in HF.

        ``prompt_lookup_num_tokens=k`` (1 .. 15; HF's name) is greedy decoding that verifies k drafted tokens per step
        (``generation.lookup_decode``): the drafts are the tokens that followed the latest n-gram (n = ``max_matching_ngram_size``
        down to 1) at its earliest earlier occurrence in the prompt or the generated text, and one step of k + 1 decode rows keeps
        those that equal greedy's own argmax, plus one more token.  The ids are greedy decoding's, with ``decode``'s width and
        pads; they can differ from a plain greedy call only at a near tie, because the step's GEMMs run over more rows.  bf16,
        fp8 or int4 weights, bf16 or fp8 KV cache, graphed or eager.  Sampling, beams, contrastive search, ``trie=``,
        ``logits_processor=``, the device processors and ``num_return_sequences > 1`` raise ``NotImplementedError``; a k
        outside 0 .. 15 or ``max_matching_ngram_size < 1`` raises ``ValueError``.  0 or None is plain greedy decoding.

        ``return_dict_in_generate=True`` returns transformers 4.28's output object instead of the ids (``GreedySearchDecoderOnlyOutput``
        for greedy, trie and prompt-lookup calls, ``SampleDecoderOnlyOutput``, ``BeamSearchDecoderOnlyOutput``,
        ``ContrastiveSearchDecoderOnlyOutput``); ``sequences`` is the ids tensor the same call returns without it, and beam calls set
        ``sequences_scores`` fp32 [B * n].  Adding ``output_scores=True`` fills ``scores``: one bf16 [rows, V] tensor per generated
        column (per step 4.28 runs, for beams) holding what that step's pick read -- the processed logits (greedy, trie, prompt
        lookup: the verify row that picked the column; contrastive search: the logits whose top-k formed the candidates), the
        warped scores (sampling) or the processed log-probs before the beam-score add (beams), special ids -inf -- and, for beams,
        ``beam_indices`` int64 [B * n, L] (-1 padded).  The kernels store them inside the captured step; see DESIGN §2.
        ``output_scores`` alone changes nothing, as in 4.28.  ``compute_transition_scores`` turns them into per-token scores."""
        lookup, ngram = _lookup_k(prompt_lookup_num_tokens, max_matching_ngram_size)
        if lookup:
            excluded = [("do_sample=True", do_sample), ("num_beams > 1", num_beams > 1),
                        ("penalty_alpha > 0 (contrastive search)", penalty_alpha is not None and penalty_alpha > 0),
                        ("trie=", trie is not None), ("logits_processor=", bool(logits_processor)),
                        ("repetition_penalty", repetition_penalty not in (None, 1.0)),
                        ("no_repeat_ngram_size", bool(no_repeat_ngram_size)), ("min_length", bool(min_length)),
                        ("min_new_tokens", bool(min_new_tokens)), ("num_return_sequences > 1", num_return_sequences > 1)]
            for name, on in excluded:
                if on:
                    raise NotImplementedError(f"generate(prompt_lookup_num_tokens={lookup}) with {name}: prompt-lookup decoding "
                                              "is built for plain greedy decoding only")
        contrastive = (penalty_alpha is not None and not (penalty_alpha <= 0) and top_k is not None and top_k > 1 and not do_sample
                       and num_beams == 1 and (num_beam_groups is None or num_beam_groups <= 1))
        if contrastive:
            if not math.isfinite(penalty_alpha):
                raise ValueError(f"generate(penalty_alpha={penalty_alpha!r}): has to be a finite number")
            if num_return_sequences > 1:
                raise ValueError(f"generate(num_return_sequences={num_return_sequences}): contrastive search returns one sequence "
                                 "per prompt")
            if trie is not None or logits_processor:
                raise NotImplementedError("generate(penalty_alpha > 0) with trie= / logits_processor=: contrastive search runs "
                                          "the device processors only")
            if top_k > ops.CONTRASTIVE_KMAX:
                raise NotImplementedError(f"generate(penalty_alpha > 0, top_k={top_k}): at most {ops.CONTRASTIVE_KMAX} candidates "
                                          "per prompt are built")
        groups = _beam_groups(num_beams, num_beam_groups, diversity_penalty, do_sample, trie is not None or bool(logits_processor))
        top_p = 1.0 if top_p is None else float(top_p)
        if not 0.0 <= top_p <= 1.0:
            raise ValueError(f"generate(top_p={top_p}): top_p must lie in [0, 1]")
        n_seq = int(num_return_sequences)
        if num_beams > 1:
            if num_return_sequences > num_beams:
                raise NotImplementedError(f"generate(num_return_sequences={num_return_sequences}) needs as many beams "
                                          f"(num_beams={num_beams})")
            if do_sample:
                raise NotImplementedError("generate(num_beams > 1, do_sample=True): beam sampling is not built")
            if logits_processor:
                raise NotImplementedError("generate(num_beams > 1) with logits_processor=: the processors keep per-row state that "
                                          "reordering the beams would scramble")
        elif n_seq > 1:
            if not do_sample:
                raise NotImplementedError(f"generate(num_return_sequences={n_seq}) without beams needs do_sample=True: greedy "
                                          "search returns one sequence per prompt")
            if trie is not None or logits_processor:
                raise NotImplementedError(f"generate(num_return_sequences={n_seq}, do_sample=True) with trie= / "
                                          "logits_processor=: the host processors have no per-sample expansion")
        if do_sample and not temperature > 0:
            raise ValueError("generate(do_sample=True) needs temperature > 0")
        self._ensure()
        self._check_fp8_fresh()
        self._check_int4_fresh()
        dev = self._device()
        eos = self.tokenizer.eos_token_id if eos_token_id is None else eos_token_id
        pad = self.tokenizer.unk_token_id if pad_token_id is None else pad_token_id
        proc = generation.processors(repetition_penalty, no_repeat_ngram_size, min_length, min_new_tokens, eos)
        call = (self, input_ids, attention_mask, (cand_vis, hist_vis, obj_vis), max_new_tokens, use_cuda_graph, stats)
        rd = bool(return_dict_in_generate)
        scores = rd and bool(output_scores)                  # the only combination that stores anything on the device
        fields = {} if rd else None

        def result(cls, ids):
            return ids if not rd else cls(sequences=ids, **fields)
        if lookup:
            dec = generation.Decoding(int(eos), int(pad), bool(stop_on_eos), "lookup", self.kv_cache_dtype,
                                      batch_invariant=self.batch_invariant, lookup_k=lookup,
                                      lookup_ngram=ngram, scores=scores)
            return result(GreedySearchDecoderOnlyOutput, generation.lookup_decode(*call, dec, out_fields=fields))
        if contrastive:
            dec = generation.Decoding(int(eos), int(pad), bool(stop_on_eos), "contrastive", self.kv_cache_dtype,
                                      batch_invariant=self.batch_invariant, top_k=int(top_k), n=int(top_k), proc=proc, penalty_alpha=float(penalty_alpha), scores=scores)
            return result(ContrastiveSearchDecoderOnlyOutput, generation.contrastive_search(*call, dec, out_fields=fields))
        if num_beams > 1:
            table = None
            if trie is not None:
                t0 = time.perf_counter()
                table = trie_mod.flatten_trie(trie, self.lm_head.weight.shape[0])
                flatten_ms = 1e3 * (time.perf_counter() - t0)
                if table is None:
                    raise NotImplementedError("generate(num_beams > 1) with a trie= that flatten_trie cannot represent: the host "
                                              "processors keep per-row state that reordering the beams would scramble")
            dec = generation.Decoding(int(eos), int(pad), None, "beam", self.kv_cache_dtype,
                                      batch_invariant=self.batch_invariant, n=int(num_beams), n_return=n_seq,
                                      length_penalty=float(length_penalty), early_stopping=bool(early_stopping), proc=proc,
                                      trie_eos=None if table is None else table.eos, scores=scores, groups=groups,
                                      diversity_penalty=float(diversity_penalty) if groups > 1 else None)
            out = generation.beam_search(*call, dec, table=table, out_fields=fields)
            if stats is not None and table is not None:
                stats.update({"trie_path": "device", "trie_flatten_ms": flatten_ms})
            return result(BeamSearchDecoderOnlyOutput, out)
        procs = list(logits_processor or [])
        table = None
        if trie is not None and not procs:
            t0 = time.perf_counter()
            table = trie_mod.flatten_trie(trie, self.lm_head.weight.shape[0])
            flatten_ms = 1e3 * (time.perf_counter() - t0)
        sampling = dict(temperature=float(temperature), top_k=int(top_k), top_p=top_p) if do_sample else {}
        dec = generation.Decoding(int(eos), int(pad), bool(stop_on_eos), "sample" if do_sample else "greedy", self.kv_cache_dtype,
                                  batch_invariant=self.batch_invariant, n=max(1, n_seq), proc=proc, scores=scores, **sampling)
        if table is not None:
            rng = torch.cuda.get_rng_state(dev) if do_sample else None
            trie_dec = dataclasses.replace(dec, mode="trie+sample" if do_sample else "trie", trie_eos=table.eos)
            out = generation.decode(*call, trie_dec, table=table, out_fields=fields)
            path = "device" if out is not None else "device_miss_host"
            if out is None:
                if rng is not None:
                    torch.cuda.set_rng_state(rng, dev)
                out = generation.decode(*call, dec, procs=[trie_mod.TrieLogitsProcessor(trie)], out_fields=fields)
        else:
            if trie is not None:
                procs = [trie_mod.TrieLogitsProcessor(trie)] + procs
                path = "host"
            out = generation.decode(*call, dec, procs=procs, out_fields=fields)
        if stats is not None and trie is not None:
            stats.update({"trie_path": path, "trie_flatten_ms": flatten_ms if table is not None else None})
        return result(SampleDecoderOnlyOutput if do_sample else GreedySearchDecoderOnlyOutput, out)

    @staticmethod
    def compute_transition_scores(sequences, scores, beam_indices=None, normalize_logits: bool = False) -> torch.Tensor:
        """transformers 4.28's ``compute_transition_scores`` on ``generate(return_dict_in_generate=True, output_scores=True)``'s
        output: fp32 [rows, n] scores of the generated tokens (see the module-level ``compute_transition_scores``)."""
        return compute_transition_scores(sequences, scores, beam_indices, normalize_logits)

    @torch.no_grad()
    def score_answers(self, input_ids, attention_mask, trie, cand_vis=None, hist_vis=None, obj_vis=None,
                      length_penalty: float = 1.0, stats: Optional[dict] = None) -> dict:
        """Score every answer of ``trie`` under each prompt exactly: the ranking ``generate(trie=...)`` can only approximate
        (greedy commits to the likeliest first token; trie beams see at most 8 answers).  An answer is a path from
        ``trie.root`` to a childless node, tokens (t_1 .. t_d), followed by ``trie.eos``; answers are listed in DFS preorder
        with children by ascending token id (``trie.tree_rows``).  A path that ends at a node with children is a prefix of
        longer answers, not an answer (every trie mode allows EOS only at a childless node); a root without children gives
        one empty answer.  ``trie`` is read as ``generate`` reads it and never modified.

        ``logprob[b, a]`` (fp32) folds, in fp32 and root to leaf, the bf16 log-probs of t_1 .. t_d and EOS as beam search
        computes them (special ids -inf, the log-softmax over the full vocabulary rounded once to bf16): the score a beam
        following that path would carry.  ``score[b, a]`` (fp64) is logprob / (S + d) ** length_penalty, S the padded prompt
        width, the value 4.28's beam search gives that hypothesis; ``best[b]`` its argmax, the lowest index on ties.  With
        ``length_penalty=0``, a trie of A <= K answers without EOS edges and enough ``max_new_tokens``, ``generate(trie=trie,
        num_beams=K, num_return_sequences=n)`` returns the n best answers by this score.

        One prefill per prompt (visual tokens injected there, as in ``generate``), then every trie node of every prompt as
        one row of a tree-masked suffix forward over the prompt cache (``generation.score_answers``).  bf16 / fp8 / int4
        weights and the bf16 / fp8 KV cache (``set_kv_cache_dtype``) apply as in ``generate``.  Returns dict(answers: token
        lists, logprob [B, A], score [B, A], best [B]) on the host.  A trie ``flatten_trie`` cannot represent, one whose
        nodes are shared between parents, or one with more than ``generation.TREE_MAX_ROWS`` nodes raises
        ``NotImplementedError``.  ``stats`` gets prefill_ms, tree_ms, score_ms, tree_rows and chunks."""
        lp = float(length_penalty)
        if not math.isfinite(lp):
            raise ValueError(f"score_answers(length_penalty={length_penalty!r}): has to be a finite number")
        self._ensure()
        self._check_fp8_fresh()
        self._check_int4_fresh()
        table = trie_mod.flatten_trie(trie, self.lm_head.weight.shape[0])
        if table is None:
            raise NotImplementedError("score_answers: a trie= that flatten_trie cannot represent")
        rows = trie_mod.tree_rows(table)
        if rows is None:
            raise NotImplementedError("score_answers: the trie shares a node between two parents; answer scoring needs a tree")
        eos = self.tokenizer.eos_token_id
        dec = generation.Decoding(int(eos), int(self.tokenizer.unk_token_id), True, "trie_score", self.kv_cache_dtype,
                                  batch_invariant=self.batch_invariant, trie_eos=table.eos)
        return generation.score_answers(self, input_ids, attention_mask, (cand_vis, hist_vis, obj_vis), rows, lp, stats, dec)
