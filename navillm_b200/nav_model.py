"""``NavModel`` -- the drop-in boundary of the reference (models/nav_model.py:32-451) on sm_90a kernels.

Same constructor ``NavModel(args, logger, model_config)``, same ``forward(mode, batch, **kwargs)`` modes and
return keys, same child-module / parameter names (``lang_model, img_embeddings, token_type_embeddings,
gmap_pos_embeddings, gmap_step_embeddings, vp_pos_embeddings, obj_pos_embeddings, og_head, out_head``), so
``tasks/agents/*`` and ``train.py`` call it unchanged and reference checkpoints load (INTEGRATION.md).

Execution differs from the reference as documented in DESIGN.md: host-side index building replaces the
per-sample Python/string loops on device tensors; fusion, heads and the LM run in the C-ABI kernels; gradient
accumulation is native (``p.grad`` are views of flat buffers; see ``allreduce_grads``).  No CPU path.
"""
from __future__ import annotations

import collections
import contextlib
import json
import os
from types import SimpleNamespace
from typing import Any, Dict, List, Optional

import numpy as np
import torch
import torch.nn as nn

from . import ops
from .image_embedding import ImageEmbeddings, _grad, _lin_bwd, _lin_fwd, _ln_bwd, _ln_fwd
from .llama import FlatParams
from .modified_lm import LMOutput, ModifiedLlamaForCausalLM, PackedPrompt
from .parallel import GradSync

bf16 = torch.bfloat16
f32 = torch.float32

VICUNA_7B = dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=32, num_attention_heads=32, vocab_size=32000,
                 rms_norm_eps=1e-6, max_position_embeddings=2048)
BERT_LARGE = dict(hidden_size=1024, num_attention_heads=16, intermediate_size=4096, hidden_act="gelu", hidden_dropout_prob=0.1)


def init_vis_config(args, config):
    """models/nav_model.py:17-29.  'bert-large-uncased' only contributes five numbers; they are embedded here
    (no network), overridable through ``model_config.vis_config`` for reduced-size tests."""
    base = dict(BERT_LARGE)
    base.update(getattr(config, "vis_config", None) or {})
    vis = SimpleNamespace(**base)
    vis.num_pano_layers = config.num_pano_layers
    vis.precision = args.precision
    vis.pretrained_model_name_or_path = args.pretrained_model_name_or_path
    vis.max_action_steps = 100
    vis.image_feat_size = args.image_feat_size
    vis.angle_feat_size = args.angle_feat_size
    vis.obj_feat_size = args.obj_feat_size
    vis.obj_loc_size = 3
    vis.type_vocab_size = 3
    return vis


def _llama_config(args, model_config) -> SimpleNamespace:
    cfg = dict(VICUNA_7B)
    path = getattr(args, "pretrained_model_name_or_path", None)
    if path and os.path.isfile(os.path.join(str(path), "config.json")):
        with open(os.path.join(str(path), "config.json")) as f:
            disk = json.load(f)
        cfg.update({k: disk[k] for k in cfg if k in disk})
    cfg.update(getattr(model_config, "llama_config", None) or {})
    return SimpleNamespace(**cfg)


# =======================================================================================================
# differentiable pieces (autograd.Function boundaries; parameter gradients are accumulated natively)
# =======================================================================================================
class _PosEmbedFn(torch.autograd.Function):
    """y = LayerNorm(Linear(x)) for the Sequential(Linear, LayerNorm(eps=1e-12)) position embeddings
    (models/nav_model.py:60-75) on the fp32 kernels; x carries no gradient."""

    @staticmethod
    def forward(ctx, seq: nn.Sequential, x2d, anchor):
        z = _lin_fwd(x2d, seq[0])
        y, mean, rstd = _ln_fwd(z, seq[1])
        ctx.seq, ctx.saved = seq, (x2d, z, mean, rstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        x2d, z, mean, rstd = ctx.saved
        dz = _ln_bwd(dy.contiguous().to(f32), z, ctx.seq[1], mean, rstd)
        _lin_bwd(dz, x2d, ctx.seq[0], need_dx=False)
        return None, None, None


class _RowsFn(torch.autograd.Function):
    """out[r] = alpha * A[ia[r]] (+ beta * B[ib[r]]) with index < 0 -> 0; gradients flow back to A and B
    by scatter-add (fp32 atomics; the tables here have <= a few thousand rows)."""

    @staticmethod
    def forward(ctx, A, ia, B, ib, R):
        D = A.shape[1]
        out = torch.empty((R, D), dtype=f32, device=A.device)
        ops.rows_combine(out, a=A, ia=ia, b=B, ib=ib)
        ctx.saved = (ia, ib, A.shape, None if B is None else B.shape)
        return out

    @staticmethod
    def backward(ctx, dout):
        ia, ib, sa, sb = ctx.saved
        dout = dout.contiguous().to(f32)
        dA = dB = None
        if ctx.needs_input_grad[0]:
            dA = torch.zeros(sa, dtype=f32, device=dout.device)
            ops.rows_scatter_add_(dA, ia, dout)
        if sb is not None and ctx.needs_input_grad[2]:
            dB = torch.zeros(sb, dtype=f32, device=dout.device)
            ops.rows_scatter_add_(dB, ib, dout)
        return dA, None, dB, None, None


class _EmbedRowsFn(torch.autograd.Function):
    """rows of a small nn.Embedding table gathered by index (< 0 -> zero row); the table gradient is
    accumulated natively (gmap_step_embeddings, token_type_embeddings)."""

    @staticmethod
    def forward(ctx, emb: nn.Embedding, idx32, anchor):
        out = torch.empty((idx32.numel(), emb.weight.shape[1]), dtype=f32, device=emb.weight.device)
        ops.rows_combine(out, a=emb.weight.data, ia=idx32)
        ctx.emb, ctx.idx = emb, idx32
        return out

    @staticmethod
    def backward(ctx, dout):
        ops.rows_scatter_add_(_grad(ctx.emb.weight), ctx.idx, dout.contiguous().to(f32))
        return None, None, None


class _HeadFn(torch.autograd.Function):
    """predictions = out_head(hidden at <cls_1>)  (models/nav_model.py:237), then either the [B,G] action-logit
    scatter with -inf elsewhere (:239-242) when ``slot`` is given, or the raw [B,100] predictions."""

    @staticmethod
    def forward(ctx, lin: nn.Linear, h, slot, B, G, sync=None):
        pred = ops.head_fwd(h.contiguous(), lin.weight.data, lin.bias.data)
        ctx.lin, ctx.saved, ctx.sync = lin, (h, slot, pred.shape[1]), sync
        return ops.logit_scatter_fwd(pred, slot, B, G) if slot is not None else pred

    @staticmethod
    def backward(ctx, dout):
        h, slot, O = ctx.saved
        lin = ctx.lin
        if ctx.sync is not None:
            ctx.sync.backward_begins()               # first custom node of a navigation / grounding backward pass
        dout = dout.contiguous().to(bf16)
        dpred = ops.logit_scatter_bwd(dout, slot, O) if slot is not None else dout
        dh = ops.head_bwd(dpred, h.contiguous(), lin.weight.data, dW=lin.weight.grad, db=lin.bias.grad)
        return None, dh, None, None, None, None


class NavModel(nn.Module):
    def __init__(self, args, logger, model_config):
        super().__init__()
        self.args = args
        config = init_vis_config(args, model_config)
        self.config = config

        # Large Language Model (models/nav_model.py:39-49)
        if "opt" in str(config.pretrained_model_name_or_path).lower().split("/")[-1]:
            raise NotImplementedError("the OPT variant is out of scope (north star names LLaMA/Vicuna only)")
        if logger is not None:
            logger.info("Initialize the model from config.")
        lcfg = _llama_config(args, model_config)
        init_device = getattr(args, "device", None)
        with (torch.device(init_device) if init_device is not None else contextlib.nullcontext()):
            self.lang_model = ModifiedLlamaForCausalLM(lcfg, config)
        _init_lm(self.lang_model, seed=getattr(args, "seed", 0))
        if not (args.resume_from_checkpoint is not None or args.from_scratch):
            _load_pretrained_lm(self.lang_model, config.pretrained_model_name_or_path, logger)
        tok = getattr(model_config, "tokenizer", None)
        if tok is not None:
            self.lang_model._set_tokenizer(tok)
        else:
            self.lang_model.init_tokenizer(config.pretrained_model_name_or_path, allow_synthetic=bool(args.from_scratch))

        self.hidden_size = self.lang_model.hidden_size
        self.model_type = self.lang_model.model_type

        with (torch.device(init_device) if init_device is not None else contextlib.nullcontext()):
            # Panorama Encoding
            config.output_size = self.hidden_size
            self.img_embeddings = ImageEmbeddings(config, use_obj=args.enable_og, fuse_obj=args.fuse_obj)
            self.token_type_embeddings = nn.Embedding(config.type_vocab_size, self.hidden_size)
            # global encoding
            self.gmap_pos_embeddings = nn.Sequential(nn.Linear(config.angle_feat_size + 3, self.hidden_size),
                                                     nn.LayerNorm(self.hidden_size, eps=1e-12))
            self.gmap_step_embeddings = nn.Embedding(config.max_action_steps, self.hidden_size)
            # local encoding
            self.vp_pos_embeddings = nn.Sequential(nn.Linear(config.angle_feat_size * 2 + 6, self.hidden_size),
                                                   nn.LayerNorm(self.hidden_size, eps=1e-12))
            self.obj_pos_embeddings = nn.Sequential(nn.Linear(config.angle_feat_size + 3, self.hidden_size),
                                                    nn.LayerNorm(self.hidden_size, eps=1e-12))
            if self.config.obj_feat_size > 0:
                self.og_head = nn.Sequential(nn.Linear(self.hidden_size, 100)).to(self.model_type)
            # Classification from candidates
            self.out_head = nn.Sequential(nn.Linear(self.hidden_size, 100)).to(self.model_type)
            self.drop_env = nn.Dropout(p=args.feat_dropout)
            self.register_buffer("_anchor", torch.zeros((), dtype=f32), persistent=False)

        self.instruction = None
        self.history = None
        self.hist_vis = None
        self._flat32: Optional[FlatParams] = None
        # data-parallel gradient exchange: ONE state shared with the language model (navillm_b200/parallel.py)
        self.grad_sync = GradSync()
        self.grad_sync.flats = self._sync_flats
        self.grad_sync.before_exchange = self.lang_model.flush_prefix_caches
        self.lang_model.grad_sync = self.grad_sync
        if logger is not None:
            logger.info("model type: {}".format(self.model_type))

    # ---------------------------------------------------------------------------------------------------
    # device residency / gradient buffers
    # ---------------------------------------------------------------------------------------------------
    def _device(self) -> torch.device:
        return self.out_head[0].weight.device

    def _heads_bf16(self) -> List[nn.Parameter]:
        ps = [self.out_head[0].weight, self.out_head[0].bias]
        if hasattr(self, "og_head"):
            ps += [self.og_head[0].weight, self.og_head[0].bias]
        return ps

    def _params_f32(self) -> List[nn.Parameter]:
        lm_ids = {id(p) for p in self.lang_model.parameters()} | {id(p) for p in self._heads_bf16()}
        return [p for p in self.parameters() if id(p) not in lm_ids]

    def _ensure(self):
        dev = self._device()
        if dev.type != "cuda":
            raise RuntimeError("navillm_b200.NavModel has no CPU path: call .cuda() / .to('cuda') first")
        lm = self.lang_model
        if lm.core is None:
            lm.materialize(dev, extra_params=self._heads_bf16())
        else:
            lm._ensure()
        f = self._flat32
        if f is None or f.params[0].data_ptr() != f._ptr0:
            self._flat32 = FlatParams(self._params_f32(), dev)
        elif f.params[0].grad is None or f.params[0].grad.data_ptr() != f.flat_grad.data_ptr():
            f.reattach_grads()

    def quantize_weights_fp8(self) -> int:
        """Opt-in fp8 (e4m3) weight streaming for inference: ``ModifiedLlamaForCausalLM.quantize_weights_fp8`` on the
        language model.  Rounds its linear weights (and lm_head) in place; the embeddings, norms, ``out_head`` / ``og_head``
        and the fp32 panorama encoder are not touched.  Returns the size of the fp8 copy in bytes."""
        self._ensure()
        return self.lang_model.quantize_weights_fp8()

    def drop_fp8_weights(self) -> None:
        self.lang_model.drop_fp8_weights()

    def set_kv_cache_dtype(self, dtype: str) -> str:
        """KV-cache format of the language model's ``generate()`` (the 3dqa, summarization and embodied_qa modes): ``"bf16"``
        (default) or ``"fp8"``; see ``ModifiedLlamaForCausalLM.set_kv_cache_dtype``.  Returns the previous format."""
        return self.lang_model.set_kv_cache_dtype(dtype)

    def set_activation_dtype(self, dtype: str) -> str:
        """Number format of the language model's decoder-layer GEMM inputs in no-grad forwards: ``"bf16"`` (default) or
        ``"fp8"`` (W8A8 after ``quantize_weights_fp8()``); see ``ModifiedLlamaForCausalLM.set_activation_dtype``.  Returns the
        previous format."""
        return self.lang_model.set_activation_dtype(dtype)

    def _flat_buffers_ready(self) -> bool:
        return self.lang_model.core is not None and self._flat32 is not None

    def _sync_flats(self):
        """[(flat buffer, offset where the part NOT covered by the overlapped LM layer reductions starts)]."""
        if not self._flat_buffers_ready():
            return []
        self._settle_lazy_zero()
        lm = self.lang_model
        return [(lm.flat, lm.flat.offset_of(lm.model.embed_tokens.weight)), (self._flat32, None)]

    def adopt_symmetric_grads(self, reducer):
        """Move both flat gradient buffers into symmetric (NVLS multicast) allocations for the in-switch exchange of
        navillm_b200.parallel.NvlsReducer.  Collective: every rank calls it (the DDP wrapper does)."""
        self._ensure()
        lm = self.lang_model

        def rebind_lm(buf):
            lm.flat.rebind_grads(buf)
            lm.core.refresh_grad_views()
        reducer.adopt(lm.flat, rebind_lm)
        reducer.adopt(self._flat32, self._flat32.rebind_grads)
        return reducer

    def _settle_lazy_zero(self) -> None:
        """``zero_grad(lazy=True)`` promised that the next LM backward overwrites the per-layer gradients.  If an
        exchange or an optimizer step arrives with no LM backward in between (a skipped / guarded iteration), the stale
        values must not be applied: make the promise true by zero-filling now."""
        self.lang_model._settle_lazy_zero()

    @contextlib.contextmanager
    def no_sync(self):
        """Bare (unwrapped) use only: marks passes whose gradients stay local.  A bare NavModel never exchanges gradients
        on its own -- call ``allreduce_grads()`` after the last backward, or wrap the model in
        ``navillm_b200.parallel.DistributedDataParallel`` for the reference's DDP behaviour (tools/optims.py:52-54)."""
        yield

    def allreduce_grads(self, average: bool = True):
        """Explicit exchange for bare use: ONE all-reduce (average) per flat gradient buffer (SURVEY.md §8e).  No-op
        without an initialised multi-rank process group.  Returns the number of collectives issued."""
        return self.grad_sync.exchange()

    def zero_grad(self, set_to_none: bool = False, lazy: bool = False):
        """Gradients live in two flat buffers, so zeroing is two fills instead of one per parameter.  With
        ``lazy=True`` the per-layer LM gradients are not zeroed at all: the next backward OVERWRITES them
        (beta = 0 wgrad epilogue) -- identical result, 27 GB less HBM traffic per step; until that backward runs
        their ``.grad`` views hold stale values.  Raises while a training ``PrefixKVCache`` of the model has pending
        gradient: it would be added after the zeroing (call ``flush_grads()`` before the optimizer step)."""
        if self.lang_model.prefix_grads_pending():
            raise RuntimeError("zero_grad(): a PrefixKVCache(train=True) of this model has pending gradient; call "
                               "cache.flush_grads() before optimizer.step() / zero_grad()")
        if self.lang_model.core is None or self._flat32 is None:
            return super().zero_grad(set_to_none=set_to_none)
        self._ensure()
        lm = self.lang_model
        self._flat32.flat_grad.zero_()
        if lazy:
            lm.flat.flat_grad[lm.flat.offset_of(lm.model.embed_tokens.weight):].zero_()
            lm.flat.overwrite_layer_grads = True
        else:
            lm.flat.flat_grad.zero_()
        lm.mark_grads_zeroed()

    def _anchor_t(self):
        return self._anchor.detach().requires_grad_(torch.is_grad_enabled())

    # ---------------------------------------------------------------------------------------------------
    def forward(self, mode: str, batch: Dict[str, Any], **kwargs) -> Dict[str, Any]:
        self._ensure()
        batch = collections.defaultdict(lambda: None, batch)
        if mode == "panorama":                       # models/nav_model.py:99-111
            batch["view_img_fts"] = self.drop_env(batch["view_img_fts"])
            if "obj_img_fts" in batch and batch["obj_img_fts"] is not None:
                batch["obj_img_fts"] = self.drop_env(batch["obj_img_fts"])
            return self.img_embeddings.forward_panorama_per_step(
                batch["view_img_fts"], batch["view_lens"], batch["loc_fts"], batch["nav_types"], batch["obj_img_fts"],
                batch["obj_lens"], batch["obj_loc_fts"])
        elif mode == "navigation":
            return self.forward_navigation(mode, batch, **kwargs)
        elif mode == "summarization" or mode == "embodied_qa":
            return self.forward_summarization(mode, batch, **kwargs)
        elif mode == "3dqa":
            return self.forward_3dqa(mode, batch, **kwargs)
        elif mode == "object_grounding":
            return self.forward_object_grounding(mode, batch, **kwargs)
        else:
            raise NotImplementedError("wrong mode: %s" % mode)

    # ---------------------------------------------------------------------------------------------------
    @staticmethod
    def _flatten_hist(hist_vis, device):
        flat = [v for vis in (hist_vis or []) for v in vis]
        return torch.stack(flat, dim=0).to(device=device, dtype=f32) if flat else None

    def _idx(self, arr) -> torch.Tensor:
        a = np.ascontiguousarray(np.asarray(arr, dtype=np.int32).reshape(-1))
        return torch.from_numpy(a).to(self._device(), non_blocking=True)

    def forward_navigation(self, mode, batch: Dict[str, Any], training: bool = True, **kwargs) -> Dict[str, Any]:
        """models/nav_model.py:129-247.  The per-sample loops over string viewpoint ids run on the HOST over the
        host-side lists/masks and produce int32 index maps; all tensor work is in kernels."""
        dev = self._device()
        vp_img_embeds = batch["vp_img_embeds"]
        B, NV1, D = vp_img_embeds.shape
        gmap_img_embeds = batch["gmap_img_embeds"].to(device=dev, dtype=f32)
        G = gmap_img_embeds.shape[1]
        gmap_vpids, vp_cand_vpids = batch["gmap_vpids"], batch["vp_cand_vpids"]
        gmap_masks_h = batch["gmap_masks"].cpu().numpy().astype(bool)
        visited_h = batch["gmap_visited_masks"].cpu().numpy().astype(bool)
        pano_masks_h = batch["pano_masks"].cpu().numpy().astype(bool)
        step_h = batch["gmap_step_ids"].cpu().numpy().astype(np.int64)

        keep = gmap_masks_h & ~visited_h                                     # rows that survive both masked_fills
        keep_idx = np.where(keep.reshape(-1), np.arange(B * G), -1)
        step_idx = np.where(keep, step_h, -1).reshape(-1)
        type_idx = np.full((B, G), -1, dtype=np.int64)
        match_idx = np.full((B, G), -1, dtype=np.int64)
        for i in range(B):                                                   # :174-190 on host ids
            visited = set(vp for vp, m in zip(gmap_vpids[i], visited_h[i]) if m)
            tmp = {}
            for j, cv in enumerate(vp_cand_vpids[i]):
                if j > 0 and cv not in visited:
                    tmp[cv] = j
            for j, vp in enumerate(gmap_vpids[i]):
                if not keep[i, j]:
                    continue
                type_idx[i, j] = 0
                if j > 0 and vp not in visited:
                    if vp in tmp:
                        if pano_masks_h[i, tmp[vp]]:                         # local_vp_embeds zeroed where ~pano_masks
                            match_idx[i, j] = i * NV1 + tmp[vp]
                    else:
                        type_idx[i, j] = 1
        cand_nums = keep.sum(1)
        # candidate gather with the reference's RNG consumption (:214-224): one CPU randperm per sample
        sel, slot = [], np.full((B, G), -1, dtype=np.int64)
        for bn in range(B):
            cols = np.flatnonzero(keep[bn])
            rest = cols[1:]
            perm = torch.randperm(len(rest)).numpy()
            sel.extend((bn * G + rest[perm]).tolist())
            # fuse_logits[bn][cand_masks] = cat(pred[0:1], pred[1:cand_num][inv_perm]); inv_perm[perm[k]] = k
            inv = np.empty_like(perm)
            inv[perm] = np.arange(len(perm))
            slot[bn, cols[0]] = 0
            slot[bn, rest] = 1 + inv
        a = self._anchor_t()
        gm2 = gmap_img_embeds.reshape(B * G, D).contiguous()
        vp2 = vp_img_embeds.to(device=dev, dtype=f32).reshape(B * NV1, D)
        pg = _PosEmbedFn.apply(self.gmap_pos_embeddings, batch["gmap_pos_fts"].to(device=dev, dtype=f32).reshape(B * G, -1).contiguous(), a)
        pv = _PosEmbedFn.apply(self.vp_pos_embeddings, batch["vp_pos_fts"].to(device=dev, dtype=f32).reshape(B * NV1, -1).contiguous(), a)
        keep_t, match_t = self._idx(keep_idx), self._idx(match_idx)
        fuse = _RowsFn.apply(gm2, keep_t, pg, keep_t, B * G) \
            + _EmbedRowsFn.apply(self.gmap_step_embeddings, self._idx(step_idx), a) \
            + _EmbedRowsFn.apply(self.token_type_embeddings, self._idx(type_idx), a) \
            + _RowsFn.apply(vp2.contiguous(), match_t, pv, match_t, B * G)
        cand_embeds = _RowsFn.apply(fuse, self._idx(sel), None, None, len(sel))
        hist_vis_input = self._flatten_hist(batch["hist_vis"], dev)

        # `text_input` (optional, not in the reference): an already tokenised TokenBatch for callers that keep
        # the prompt ids resident; otherwise tokenise on the host exactly like models/nav_model.py:211
        text = batch["text_input"] if batch["text_input"] is not None else self.lang_model.tokenize(batch["prompts"])
        prefix_cache = kwargs.get("prefix_cache")
        if prefix_cache is not None:
            # rollouts (not in the reference): encode only what follows each row's cached prompt prefix; training needs a
            # PrefixKVCache(train=True), whose flush_grads() adds the gradient through the cached rows
            if torch.is_grad_enabled() and not prefix_cache.train:
                raise RuntimeError("prefix_cache is an inference feature: call under torch.no_grad() (weights must not change), "
                                   "or build the cache with PrefixKVCache(..., train=True) for a training rollout")
            hist_counts = [len(v) for v in (batch["hist_vis"] or [[] for _ in range(B)])]
            h_cls = self.lang_model.hidden_rows_cached(text["input_ids"], text["attention_mask"], cand_embeds, hist_vis_input,
                                                       hist_counts, prefix_cache)
        else:
            pp = PackedPrompt(text["input_ids"], text["attention_mask"], self.lang_model, dev)
            vis = self.lang_model.cat_vis(cand_embeds, hist_vis_input, None, pp)
            if pp.n_cls != B:
                raise RuntimeError(f"expected one <cls_1> token per prompt, found {pp.n_cls} in {B} prompts")
            h_cls = self.lang_model.hidden_rows(pp, vis, pp.cls_rows)
        fuse_logits = _HeadFn.apply(self.out_head[0], h_cls, self._idx(slot), B, G, self.grad_sync)
        return {"fuse_embeds": fuse.detach().view(B, G, D), "fuse_logits": fuse_logits}

    # ---------------------------------------------------------------------------------------------------
    def _const_vp_embed(self) -> torch.Tensor:
        """vp_pos_embeddings(0) + token_type_embeddings(0): one [1, D] row added to every view token in the
        summarization / 3dqa modes (models/nav_model.py:270-273, 371-374)."""
        a = self._anchor_t()
        dev = self._device()
        z = torch.zeros((1, self.config.angle_feat_size * 2 + 6), dtype=f32, device=dev)
        return _PosEmbedFn.apply(self.vp_pos_embeddings, z, a) \
            + _EmbedRowsFn.apply(self.token_type_embeddings, torch.zeros(1, dtype=torch.int32, device=dev), a)

    def _masked_rows_plus_const(self, x2d: torch.Tensor, mask_h: np.ndarray) -> torch.Tensor:
        rows = np.flatnonzero(mask_h.reshape(-1))
        const = self._const_vp_embed()
        return _RowsFn.apply(x2d.contiguous(), self._idx(rows), const, torch.zeros(len(rows), dtype=torch.int32, device=x2d.device),
                             len(rows))

    def _lm_labels(self, text):
        labels = text["input_ids"].clone()
        labels[text["token_type_ids"][:, -labels.shape[-1]:] == 0] = -100        # models/nav_model.py:306-308
        return labels

    def forward_summarization(self, mode, batch: Dict[str, Any], training: bool = True, **kwargs) -> Dict[str, Any]:
        """models/nav_model.py:251-343."""
        dev = self._device()
        vp_img_embeds = batch["vp_img_embeds"][:, 1:, :]                         # remove `stop`
        nav_masks_h = batch["vp_nav_masks"][:, 1:].cpu().numpy().astype(bool)
        B, NV, D = vp_img_embeds.shape
        cand_vis = self._masked_rows_plus_const(vp_img_embeds.to(device=dev, dtype=f32).reshape(B * NV, D), nav_masks_h)
        hist_vis_input = self._flatten_hist(batch["hist_vis"], dev)
        data_type, labels = batch["data_type"], batch["answer"]
        eos = self.lang_model.tokenizer.eos_token
        all_text = []
        for bn in range(B):
            prompt = batch["prompts"][bn]
            label = (labels[bn] if data_type[0] in ("eqa", "fgr2r") else batch["instruction"][bn]) + f"{eos}"
            all_text.append([prompt, label] if training else prompt)
        text = self.lang_model.tokenize(all_text)
        if training:
            pp = PackedPrompt(text["input_ids"], text["attention_mask"], self.lang_model, dev, labels=self._lm_labels(text))
            vis = self.lang_model.cat_vis(cand_vis, hist_vis_input, None, pp)
            return {"loss": self.lang_model.lm_loss(pp, vis)}
        trie = kwargs.get("trie", None)
        ids = self.lang_model.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand_vis,
                                       hist_vis=hist_vis_input, eos_token_id=self.lang_model.tokenizer.eos_token_id,
                                       pad_token_id=self.lang_model.tokenizer.unk_token_id, max_new_tokens=50, do_sample=False,
                                       trie=trie).tolist()
        ids = [s[text["input_ids"].shape[1]:] for s in ids]
        return {"generated_sentences": self.lang_model.tokenizer.batch_decode(ids, skip_special_tokens=True,
                                                                              clean_up_tokenization_spaces=False)}

    def forward_3dqa(self, mode, batch: Dict[str, Any], training: bool = True, **kwargs):
        """models/nav_model.py:346-404."""
        dev = self._device()
        B = len(batch["question"])
        eos = self.lang_model.tokenizer.eos_token
        all_text = []
        for bn in range(B):
            prompt = batch["prompts"][bn]
            all_text.append([prompt, batch["answers"][bn][0] + f"{eos}"] if training else prompt)
        feats = [batch["features"][bn] for bn in range(B)]
        lens = [int(f.shape[0]) for f in feats]
        mx = max(lens)
        view = torch.zeros((B, mx, feats[0].shape[1]), dtype=f32, device=dev)     # pad_tensors_wgrad (ops.py:44-66)
        for bn, f in enumerate(feats):
            view[bn, :lens[bn]] = f.to(device=dev, dtype=f32)
        pano = self.img_embeddings.forward_panorama_per_step(view_img_fts=view, view_lens=torch.tensor(lens, device=dev))
        pe = pano["pano_embeds"]
        mask_h = np.arange(mx)[None, :] < np.asarray(lens)[:, None]
        cand_vis = self._masked_rows_plus_const(pe.reshape(B * mx, -1), mask_h)
        text = self.lang_model.tokenize(all_text)
        if training:
            pp = PackedPrompt(text["input_ids"], text["attention_mask"], self.lang_model, dev, labels=self._lm_labels(text))
            vis = self.lang_model.cat_vis(cand_vis, None, None, pp)
            loss = self.lang_model.lm_loss(pp, vis)
            return LMOutput(loss=loss, logits=None, past_key_values=None, hidden_states=None, attentions=None)
        ids = self.lang_model.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand_vis,
                                       eos_token_id=self.lang_model.tokenizer.eos_token_id,
                                       pad_token_id=self.lang_model.tokenizer.unk_token_id, **kwargs).tolist()
        ids = [s[text["input_ids"].shape[1]:] for s in ids]
        return {"generated_sentences": self.lang_model.tokenizer.batch_decode(ids, skip_special_tokens=True,
                                                                              clean_up_tokenization_spaces=False)}

    def forward_object_grounding(self, mode, batch: Dict[str, Any], training: bool = True, **kwargs) -> Dict[str, Any]:
        """models/nav_model.py:407-451."""
        dev = self._device()
        obj_embeds, obj_loc_fts = batch["obj_embeds"], batch["obj_loc_fts"]
        obj_masks_h = batch["obj_masks"].cpu().numpy().astype(bool)
        B, O, D = obj_embeds.shape
        a = self._anchor_t()
        pos = _PosEmbedFn.apply(self.obj_pos_embeddings, obj_loc_fts.to(device=dev, dtype=f32).reshape(B * O, -1).contiguous(), a)
        rows = self._idx(np.flatnonzero(obj_masks_h.reshape(-1)))
        cand_vis = _RowsFn.apply(obj_embeds.to(device=dev, dtype=f32).reshape(B * O, D).contiguous(), rows, pos, rows, rows.numel())
        cand_nums = obj_masks_h.sum(1) + 1                                        # add not exist
        hist_vis_input = self._flatten_hist(batch["hist_vis"], dev)
        text = self.lang_model.tokenize(batch["prompts"])
        pp = PackedPrompt(text["input_ids"], text["attention_mask"], self.lang_model, dev)
        vis = self.lang_model.cat_vis(cand_vis, hist_vis_input, None, pp)
        h_cls = self.lang_model.hidden_rows(pp, vis, pp.cls_rows)
        n_out = self.out_head[0].weight.shape[0]
        slot = np.where(np.arange(n_out)[None, :] < cand_nums[:, None], np.arange(n_out)[None, :], -1)   # [i, cand_nums:] = -inf
        preds = _HeadFn.apply(self.out_head[0], h_cls, self._idx(slot), B, n_out, self.grad_sync)
        return {"obj_logits": preds}


# =======================================================================================================
def _init_lm(lm: ModifiedLlamaForCausalLM, seed: int = 0):
    """HF default init (normal(0, 0.02), RMSNorm weights 1) in place on whatever device the holders live on."""
    dev = lm.model.norm.weight.device
    g = torch.Generator(device=dev).manual_seed(seed)
    with torch.no_grad():
        for p in list(lm.model.parameters()) + list(lm.lm_head.parameters()):
            if p.dim() == 1:
                p.fill_(1.0)
            else:
                p.normal_(0.0, 0.02, generator=g)


def _load_pretrained_lm(lm: ModifiedLlamaForCausalLM, path, logger):
    """``from_pretrained`` for a LOCAL HF checkpoint directory (pytorch_model*.bin shards); there is no network."""
    import glob
    files = sorted(glob.glob(os.path.join(str(path), "pytorch_model*.bin")))
    if not files:
        raise FileNotFoundError(f"no local LLaMA weights under {path!r} (no network access): pass --from_scratch, or "
                                f"--resume_from_checkpoint with a NaviLLM checkpoint")
    sd = {}
    for f in files:
        sd.update(torch.load(f, map_location="cpu"))
    own = lm.state_dict()
    sd = {k: v for k, v in sd.items() if k in own and own[k].shape == v.shape}
    lm.load_state_dict(sd, strict=False)
    if logger is not None:
        logger.info(f"loaded {len(sd)} tensors from {path}")
