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
from types import SimpleNamespace
from typing import List, Optional

import numpy as np
import torch
import torch.nn as nn

from . import llama as llama_mod
from . import ops
from .llama import FlatParams, LlamaCore, LlamaDims, LlamaModelParams, _Linear
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
    reference's hist_vis lists are); call ``reset()`` when a new episode starts in a row."""

    def __init__(self, lm: "ModifiedLlamaForCausalLM", batch_size: int, max_len: int = 2048):
        lm._ensure()
        dev, d = lm._device(), lm.dims
        self.B, self.max_len = batch_size, max_len
        # zero-initialised: rows past a sequence's length are masked in the attention kernel but must stay finite
        self.kc = [torch.zeros((batch_size, max_len, d.hidden), dtype=bf16, device=dev) for _ in range(d.n_layers)]
        self.vc = [torch.zeros((batch_size, max_len, d.hidden), dtype=bf16, device=dev) for _ in range(d.n_layers)]
        self.ids: List[np.ndarray] = [np.zeros(0, dtype=np.int64) for _ in range(batch_size)]
        self.off: List[Optional[int]] = [None] * batch_size
        self.stats = {"steps": 0, "tokens": 0, "tokens_encoded": 0}

    def reset(self, rows=None) -> None:
        for b in (range(self.B) if rows is None else rows):
            self.ids[b] = np.zeros(0, dtype=np.int64)
            self.off[b] = None


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
        old = cache.ids[b]
        m = min(old.size, L - 1)                               # at least the last token is encoded
        neq = np.flatnonzero(old[:m] != toks[:m])
        n = int(neq[0]) if neq.size else m
        cpos = np.flatnonzero(toks == cand_id)                 # candidates change every step: never reused
        if cpos.size:
            n = min(n, int(cpos[0]))
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
        dg = ops.rmsnorm_bwd(g, normw.data, rstd, dy, dw=normw.grad)                     # [R, D]: gradient at the requested rows
        lm.grad_sync.short_backward = pp.T < lm.SHORT_BACKWARD_TOKENS
        dx = core.backward(dg, ctx.tape, layer_done=lm._grad_sync_hook())
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

    @torch.no_grad()
    def hidden_rows_cached(self, input_ids: torch.Tensor, attention_mask: torch.Tensor, cand_vis: Optional[torch.Tensor],
                           hist_vis: Optional[torch.Tensor], hist_counts, cache: PrefixKVCache) -> torch.Tensor:
        """Inference twin of ``hidden_rows(pp, vis, pp.cls_rows)`` that encodes only the tokens after each row's
        longest common prefix with ``cache`` (see PrefixKVCache).  cand_vis: [sum cand, D] in row-major token order;
        hist_vis: [sum_b hist_counts[b], D] flattened sample-major (NavModel._flatten_hist).  Returns the final-
        RMSNorm'ed hidden states at the <cls_1> tokens, [B, D] bf16."""
        self._ensure()
        dev, d = self._device(), self.dims
        ids = input_ids.detach().cpu().numpy().astype(np.int64)
        msk = attention_mask.detach().cpu().numpy().astype(bool)
        B = ids.shape[0]
        n_cand_total = 0 if cand_vis is None else cand_vis.shape[0]
        plan = plan_prefix_reuse(ids, msk, cache, hist_counts, n_cand_total, self.cand_token_id[0], self.hist_token_id[0],
                                 self.cls_token_id[0])
        tok_new, pos_new, vis_new, q_lens, cached, kv_len, cls_rows = plan
        cu = np.concatenate([[0], np.cumsum(q_lens)])
        kv_start = np.arange(B, dtype=np.int64) * cache.max_len
        parts = [np.concatenate(tok_new), np.concatenate(pos_new), cu, np.concatenate(vis_new), np.asarray(cls_rows),
                 np.asarray(cached), kv_start, np.asarray(kv_len)]
        host = np.concatenate([p.astype(np.int32) for p in parts])
        dev_buf = torch.from_numpy(host).pin_memory().to(dev, non_blocking=True)
        views, o = [], 0
        for p in parts:
            views.append(dev_buf[o:o + p.size]); o += p.size
        tok_d, pos_d, cu_d, vis_d, cls_d, cached_d, kvs_d, kvl_d = views
        vis_parts = [v.to(torch.float32) for v in (cand_vis, hist_vis) if v is not None and v.shape[0] > 0]
        vis = None if not vis_parts else (vis_parts[0].contiguous() if len(vis_parts) == 1 else torch.cat(vis_parts, 0))
        x = ops.embed_fwd(tok_d, self.model.embed_tokens.weight.data, vis_d if vis is not None else None, vis)
        g = self.core.forward_suffix(x, pos_d, cu_d, q_lens, cache.kc, cache.vc, cached_d, kvs_d, kvl_d, out_rows=cls_d)
        hn, _ = ops.rmsnorm_fwd(g, self.model.norm.weight.data, d.rms_eps)
        cache.stats["steps"] += 1
        cache.stats["tokens"] += int(sum(kv_len))
        cache.stats["tokens_encoded"] += int(sum(q_lens))
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


    # ---- generation (models/nav_model.py:324-338,388-399; HF GenerationMixin greedy / sampling) ----
    decode_pdl = os.environ.get("NAVILLM_DECODE_PDL", "1") != "0"   # developer knob: 0 = plain stream-ordered launches
    max_decode_states = 2        # cached (KV buffers + captured decode graph) sets, least recently used evicted

    def _decode_state(self, B: int, Smax: int, key_extra: tuple, want_graph: bool):
        """Persistent per-shape decode state: the contiguous KV cache [B, Smax, D] per layer, the step's I/O buffers and --
        once captured -- the CUDA graph of ONE greedy decode step.  Capturing and instantiating the ~260-node graph costs
        more than the 127 replays of a C3 generation save, so it is done once per (batch, cache length, stop rule) and
        reused by every later ``generate`` call (evaluation loops call generate with the same shapes over and over)."""
        states = self.__dict__.setdefault("_decode_states", collections.OrderedDict())
        key = (B, Smax) + key_extra
        st = states.get(key) if want_graph else None
        if st is not None:
            states.move_to_end(key)
            return st
        dev, d = self._device(), self.dims
        V = self.lm_head.weight.shape[0]
        st = SimpleNamespace(
            kc=[torch.empty((B, Smax, d.hidden), dtype=bf16, device=dev) for _ in range(d.n_layers)],
            vc=[torch.empty((B, Smax, d.hidden), dtype=bf16, device=dev) for _ in range(d.n_layers)],
            logits=torch.empty((B, (V + 63) // 64 * 64), dtype=bf16, device=dev)[:, :V],
            next_ids=torch.empty((B,), dtype=torch.int32, device=dev),
            finished=torch.zeros((B,), dtype=torch.int32, device=dev),
            lens=torch.zeros((B,), dtype=torch.int32, device=dev), graph=None)
        if want_graph:
            states[key] = st
            while len(states) > self.max_decode_states:
                states.popitem(last=False)
        return st

    @torch.no_grad()
    def generate(self, input_ids, attention_mask, cand_vis=None, hist_vis=None, obj_vis=None, max_new_tokens: int = 20,
                 do_sample: bool = False, temperature: float = 1.0, eos_token_id: Optional[int] = None,
                 pad_token_id: Optional[int] = None, bos_token_id: Optional[int] = None, logits_processor=None, trie=None,
                 stop_on_eos: bool = True, use_cuda_graph: bool = True, stats: Optional[dict] = None, top_k: int = 50,
                 top_p: float = 1.0, **unused) -> torch.Tensor:
        """Prefill on the packed kernels (positions = cumsum(mask)-1 like HF generate; visual tokens injected only
        here, as in models/modified_lm.py:195-197), then one token per step over a pre-allocated KV cache.  The
        greedy step has static shapes and is replayed as a CUDA graph (captured once per shape, see ``_decode_state``).
        Returns [B, S0 + n_new] int64 ids (prompt part copied from the input; finished rows continue with pad_token_id
        like HF greedy search).

        ``do_sample=True`` follows HF ``sample`` as the reference reaches it (tasks/agents/llava.py:58-62): logits
        processors, then temperature and top-k (``top_k=50`` is transformers' generation default, which the reference
        never overrides), bf16 softmax, one multinomial draw per row - all in ``nv_sample_topk``; the uniform numbers
        come from ``torch.rand`` on the device, so ``torch.manual_seed`` makes a run reproducible."""
        if top_p is not None and top_p < 1.0:
            raise NotImplementedError("generate(top_p < 1) is not built: the reference never sets it (HF default 1.0)")
        if do_sample and not temperature > 0:
            raise ValueError("generate(do_sample=True) needs temperature > 0")
        self._ensure()
        dev = self._device()
        core, d = self.core, self.dims
        eos = self.tokenizer.eos_token_id if eos_token_id is None else eos_token_id
        pad = self.tokenizer.unk_token_id if pad_token_id is None else pad_token_id
        ev = None
        if stats is not None:                                     # bench.py: device-side phase times (forces one sync at the end)
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            ev[0].record()
        pp = PackedPrompt(input_ids, attention_mask, self, dev, generate_positions=True)
        vis = self.cat_vis(cand_vis, hist_vis, obj_vis, pp)
        B = pp.B
        greedy = (not do_sample) and trie is None and not logits_processor
        need_host = trie is not None or bool(logits_processor)    # processors walk the generated ids on the host
        graphed = greedy and use_cuda_graph
        Smax = (max(pp.seqlens) + max_new_tokens + 127) // 128 * 128          # bucketed: more reuse of the cached state
        st = self._decode_state(B, Smax, (int(eos), int(pad), bool(stop_on_eos)), graphed)
        kc, vc, logits, next_ids, finished, lens = st.kc, st.vc, st.logits, st.next_ids, st.finished, st.lens
        finished.zero_()
        lens.copy_(torch.tensor(pp.seqlens, dtype=torch.int32), non_blocking=True)

        E = self.model.embed_tokens.weight.data
        x = ops.embed_fwd(pp.ids, E, pp.vis_src if vis is not None else None, vis)
        hid_last, _ = core.forward(x, pp.pos, pp.cu, pp.seqlens, save=False, kv_store=(kc, vc), out_rows=pp.last_rows)
        special = self.special_ids_dev

        def head(h_rows):
            hn, _ = ops.rmsnorm_fwd(h_rows, self.model.norm.weight.data, d.rms_eps)
            if B <= 16 and llama_mod.DECODE_BLOCK_N == 0:
                ops.gemm_skinny(hn, self.lm_head.weight.data, out=logits)
            else:
                ops.gemm(hn, self.lm_head.weight.data, out=logits, block_n=llama_mod.DECODE_BLOCK_N)

        trie_state = [None]

        def pick(all_ids_host):
            """next token from `logits` -> next_ids (device)."""
            if greedy:
                ops.argmax_masked(logits, special, finished, eos, pad, stop_on_eos, next_ids)
                return
            if not need_host:                                     # plain sampling: straight from the bf16 logits
                ops.sample_topk(logits, special, finished, eos, pad, stop_on_eos, temperature, top_k,
                                torch.rand(B, device=dev, dtype=torch.float32), next_ids)
                return
            lg = logits.float()
            lg[:, self.special_token_ids] = float("-inf")
            if trie is not None:                                  # TrieLogitsProcessor (models/modified_lm.py:10-30)
                if trie_state[0] is None:
                    trie_state[0] = [trie.root for _ in range(B)]
                else:
                    for bn in range(B):
                        trie_state[0][bn] = trie.get_next_node(trie_state[0][bn], int(all_ids_host[bn][-1]))
                allow = torch.zeros_like(lg, dtype=torch.bool)
                for bn in range(B):
                    allow[bn, trie.get_child_index(trie_state[0][bn])] = True
                lg = lg.masked_fill(~allow, float("-inf"))
            for proc in (logits_processor or []):
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

        head(hid_last)
        host_ids = [row.tolist() for row in input_ids.cpu()] if need_host else None
        pick(host_ids)
        out_tokens = [next_ids.clone()]
        if ev is not None:
            ev[1].record()

        def step():
            with ops.pdl(self.decode_pdl):          # programmatic dependent launch along the whole decode chain
                xt = ops.embed_fwd(next_ids, E)
                h = core.decode_step(xt, lens, kc, vc)
                head(h)
                ops.add_int_(lens, 1)
                if greedy:
                    ops.argmax_masked(logits, special, finished, eos, pad, stop_on_eos, next_ids)

        # HF stops when every sequence has finished.  Asking the device after EVERY token would serialise host and device
        # (one blocking read per token); finished rows only emit pad tokens, so the greedy loop looks every `check_every`
        # tokens and the surplus pad columns are trimmed below -- same ids as a per-token check.
        check_every = 1 if need_host else 8
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
                if not greedy:
                    pick(host_ids)
            out_tokens.append(next_ids.clone())
        if ev is not None:
            ev[2].record()
            torch.cuda.synchronize()
            n_dec = len(out_tokens) - 1
            stats.update({"prefill_ms": ev[0].elapsed_time(ev[1]), "decode_ms": ev[1].elapsed_time(ev[2]) if n_dec else None,
                          "decode_steps": n_dec, "graph_replays": replays, "kv_rows": Smax, "prompt_lens": list(pp.seqlens)})
        new = torch.stack(out_tokens, dim=1).to(torch.int64)
        if stop_on_eos and not need_host and new.shape[1] > 1:
            # trim the columns generated after the step at which the last row emitted EOS (see check_every above)
            is_eos = (new == eos)
            if bool(is_eos.any(dim=1).all()):
                last = int(is_eos.float().argmax(dim=1).max())        # first EOS per row; the slowest row decides
                new = new[:, :last + 1]
        return torch.cat([input_ids.to(dev), new], dim=1)
