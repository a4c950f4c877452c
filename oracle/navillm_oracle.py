"""CPU ORACLE for the NaviLLM per-step hot path.  *** TEST INFRASTRUCTURE ONLY ***

A plain-PyTorch (CPU, eager) restatement of the reference algorithm behind
``NavModel.forward(mode, batch)`` -- panorama encoder, modified LLaMA forward, action/object heads, LM
loss and greedy decode -- written as pure functions over a reference-format ``state_dict``.  Only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl reference`` leg may import
this file, and only as the checker / CPU baseline.  The product (navillm_b200/) never imports it and has
no CPU path at all.

Pinning (SURVEY.md §8c): the reference ships NO tests or golden vectors for this path ("parity
unpinned" at the source).  The oracle is therefore pinned against outputs of the reference code itself,
imported unmodified from a checkout of the reference with three stubs (bert-large
config, AutoConfig, tokenizer): ``tests/golden/make_golden.py`` generates the fixtures in
``tests/golden/*.pt`` and ``tests/test_oracle_golden.py`` checks every function below against them
(forward outputs, loss and gradients).  The LLaMA block arithmetic is not in the reference tree: it is
``transformers.models.llama`` (pinned 4.28.0 by the reference's requirements.txt:20; 5.5.0 is what is
installed here and what the golden vectors were produced with, attn_implementation="eager").  The
greedy-decode loop restates HF GenerationMixin greedy search; it is pinned against token ids produced by the
reference's own generation branch run with a keyword-argument adapter for prepare_inputs_for_generation
(tests/golden/make_generate_golden.py -> generate_*.pt; the positional call of models/modified_lm.py:187-194 is the
only thing that does not run under transformers 5.x, SURVEY.md §8c).

Each function cites the reference file:line it follows (paths relative to the reference repository root).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional

import torch
import torch.nn.functional as F


@dataclass
class OracleConfig:
    # language model (Vicuna-7B defaults; SURVEY.md §2b)
    hidden: int = 4096
    n_layers: int = 32
    n_heads: int = 32
    inter: int = 11008
    vocab: int = 32006
    rms_eps: float = 1e-6
    rope_theta: float = 10000.0
    # panorama encoder (bert-large-uncased config via models/nav_model.py:17-29)
    image_feat_size: int = 1024
    angle_feat_size: int = 4
    obj_feat_size: int = 768
    pano_hidden: int = 1024
    pano_heads: int = 16
    pano_inter: int = 4096
    num_pano_layers: int = 2
    enable_og: bool = True
    # special token ids (models/modified_lm.py:59-73)
    cand_id: int = 32000
    hist_id: int = 32001
    obj_id: int = 32002
    cls_ids: tuple = (32003, 32004)
    precision: str = "amp_bf16"

    @property
    def special_token_ids(self) -> List[int]:
        return [self.cand_id, self.hist_id, self.obj_id, *self.cls_ids]

    @property
    def lm_dtype(self) -> torch.dtype:
        # models/modified_lm.py:40-48
        if self.precision == "fp16":
            return torch.float16
        if "bf16" in self.precision or "bfloat16" in self.precision:
            return torch.bfloat16
        return torch.float32


SD = Dict[str, torch.Tensor]


# =====================================================================================================
# Panorama encoder  (models/image_embedding.py:51-121, models/detr_transformer.py:62-89,170-182,
#                    models/ops.py:6-18,33-41)
# =====================================================================================================
def gen_seq_masks(seq_lens: torch.Tensor, max_len: Optional[int] = None) -> torch.Tensor:
    """models/ops.py:33-41."""
    if max_len is None:
        max_len = int(max(seq_lens))
    return torch.arange(max_len).unsqueeze(0).repeat(len(seq_lens), 1) < seq_lens.unsqueeze(1)


def _ln(x, sd, prefix, eps):
    return F.layer_norm(x, (x.shape[-1],), sd[prefix + ".weight"], sd[prefix + ".bias"], eps)


def _lin(x, sd, prefix):
    return F.linear(x, sd[prefix + ".weight"], sd.get(prefix + ".bias"))


def _mha(x, key_padding_mask, sd, prefix, n_heads):
    """torch.nn.MultiheadAttention self-attention in eval mode (seq-first semantics folded to batch-first).
    x: [B, N, E]; key_padding_mask: [B, N] True = ignore (models/detr_transformer.py:175-177)."""
    B, N, E = x.shape
    hd = E // n_heads
    qkv = F.linear(x, sd[prefix + ".in_proj_weight"], sd[prefix + ".in_proj_bias"])
    q, k, v = qkv.split(E, dim=-1)
    q = q.view(B, N, n_heads, hd).transpose(1, 2)
    k = k.view(B, N, n_heads, hd).transpose(1, 2)
    v = v.view(B, N, n_heads, hd).transpose(1, 2)
    scores = (q * (hd ** -0.5)) @ k.transpose(-1, -2)
    scores = scores.masked_fill(key_padding_mask[:, None, None, :], float("-inf"))
    attn = torch.softmax(scores, dim=-1)
    out = (attn @ v).transpose(1, 2).reshape(B, N, E)
    return F.linear(out, sd[prefix + ".out_proj.weight"], sd[prefix + ".out_proj.bias"])


def pano_encoder_layers(x, key_padding_mask, sd, cfg: OracleConfig, prefix="img_embeddings.pano_encoder"):
    """TransformerEncoder.forward / TransformerEncoderLayer.forward_pre (detr_transformer.py:62-89,170-182),
    eval mode (all dropouts off)."""
    for l in range(cfg.num_pano_layers):
        p = f"{prefix}.layers.{l}"
        h = _ln(x, sd, p + ".norm1", 1e-5)
        x = x + _mha(h, key_padding_mask, sd, p + ".self_attn", cfg.pano_heads)
        h = _ln(x, sd, p + ".norm2", 1e-5)
        h = _lin(F.gelu(_lin(h, sd, p + ".linear1")), sd, p + ".linear2")
        x = x + h
    return _ln(x, sd, prefix + ".norm", 1e-12)          # models/ops.py:14-16 (norm=True, eps 1e-12)


def forward_panorama(sd: SD, cfg: OracleConfig, view_img_fts, view_lens, loc_fts=None, nav_types=None,
                     obj_img_fts=None, obj_lens=None, obj_loc_fts=None, fuse_obj: bool = False) -> Dict[str, torch.Tensor]:
    """ImageEmbeddings.forward_panorama_per_step (models/image_embedding.py:51-121), eval mode.  ``fuse_obj`` is the
    constructor flag of the reference (``--fuse_obj``, tools/parser.py:95): object tokens join the views in the encoder
    (:78-94); pinned by tests/golden/pano_fuse_obj.pt."""
    P = "img_embeddings."
    x = _ln(_lin(view_img_fts, sd, P + "img_linear"), sd, P + "img_layer_norm", 1e-12)
    if loc_fts is None:
        loc_fts = torch.zeros(x.shape[:2] + (7,), dtype=torch.float)
    x = x + _ln(_lin(loc_fts, sd, P + "loc_linear"), sd, P + "loc_layer_norm", 1e-12)
    if nav_types is None:
        nav_types = torch.ones(x.shape[:2], dtype=torch.int)
    x = x + F.embedding(nav_types.long(), sd[P + "nav_type_embedding.weight"])
    x = _ln(x, sd, P + "layer_norm", 1e-12)
    pano_masks = gen_seq_masks(view_lens)
    if cfg.num_pano_layers > 0 and fuse_obj:
        # :79-94  obj tokens = obj_linear (Linear + LN) + the SHARED loc LN(Linear) + nav-type 2; NOT through layer_norm/dropout;
        # per row [views[:view_len] ; objs[:obj_len]], zero-padded, encoded with the joint mask; the view rows are taken back
        o = _ln(_lin(obj_img_fts, sd, P + "obj_linear.0"), sd, P + "obj_linear.1", 1e-12)
        o = o + _ln(_lin(obj_loc_fts, sd, P + "loc_linear"), sd, P + "loc_layer_norm", 1e-12)
        o = o + sd[P + "nav_type_embedding.weight"][2]
        B = x.shape[0]
        vl, ol = [int(v) for v in view_lens], [int(v) for v in obj_lens]
        Lf = max(v + w for v, w in zip(vl, ol))
        fused = x.new_zeros(B, Lf, x.shape[-1])
        for b in range(B):
            fused[b, :vl[b]] = x[b, :vl[b]]
            fused[b, vl[b]:vl[b] + ol[b]] = o[b, :ol[b]]
        fmask = gen_seq_masks(torch.tensor([v + w for v, w in zip(vl, ol)]))
        fused = pano_encoder_layers(fused, fmask.logical_not(), sd, cfg)
        x = x.new_zeros(B, max(vl), x.shape[-1])
        for b in range(B):
            x[b, :vl[b]] = fused[b, :vl[b]]
    elif cfg.num_pano_layers > 0:
        x = pano_encoder_layers(x, pano_masks.logical_not(), sd, cfg)
    x = _lin(x, sd, P + "mapper")
    x = x.masked_fill(pano_masks.logical_not().unsqueeze(-1), 0)
    ret = {"pano_embeds": x, "pano_masks": pano_masks}
    if obj_img_fts is not None and obj_img_fts.shape[1] > 0:
        o = _ln(_lin(obj_img_fts, sd, P + "obj_projector.0"), sd, P + "obj_projector.1", 1e-12)
        ret.update({"obj_embeds": o, "obj_loc_fts": obj_loc_fts, "obj_masks": gen_seq_masks(obj_lens)})
    return ret


# =====================================================================================================
# LLaMA decoder stack (transformers.models.llama, eager attention; call site models/modified_lm.py:112-116)
# =====================================================================================================
def _rmsnorm(x, w, eps):
    dt = x.dtype
    xf = x.float()
    xf = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)
    return w * xf.to(dt)


def rope_tables(cfg: OracleConfig, position_ids: torch.Tensor, dtype) -> tuple:
    hd = cfg.hidden // cfg.n_heads
    inv_freq = 1.0 / (cfg.rope_theta ** (torch.arange(0, hd, 2, dtype=torch.int64).float() / hd))
    freqs = position_ids[..., None].float() * inv_freq          # [B,S,hd/2]
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.cos().to(dtype), emb.sin().to(dtype)


def _rotate_half(x):
    h = x.shape[-1] // 2
    return torch.cat((-x[..., h:], x[..., :h]), dim=-1)


def llama_model(sd: SD, cfg: OracleConfig, inputs_embeds, attention_mask, position_ids=None,
                past_kv: Optional[list] = None, prefix="lang_model.model"):
    """LlamaModel.forward -> final RMSNorm'ed hidden states.  attention_mask: [B, S_total] (1 = real token).
    With ``past_kv`` (list of (k,v) per layer, [B,H,S_past,hd]) the new keys/values are appended in place."""
    B, S, D = inputs_embeds.shape
    H, hd = cfg.n_heads, D // cfg.n_heads
    dt = inputs_embeds.dtype
    S_past = past_kv[0][0].shape[2] if (past_kv and past_kv[0] is not None) else 0
    S_tot = S_past + S
    if position_ids is None:                                    # plain forward: arange, padding ignored
        position_ids = torch.arange(S_past, S_tot).unsqueeze(0).expand(B, S)
    cos, sin = rope_tables(cfg, position_ids, dt)
    cos, sin = cos.unsqueeze(1), sin.unsqueeze(1)
    minv = torch.finfo(dt).min
    causal = torch.ones(S, S_tot, dtype=torch.bool).tril(diagonal=S_past)
    allowed = causal[None, None] & attention_mask[:, None, None, :S_tot].bool()
    add_mask = torch.zeros(B, 1, S, S_tot, dtype=dt).masked_fill(~allowed, minv)
    x = inputs_embeds
    for l in range(cfg.n_layers):
        p = f"{prefix}.layers.{l}"
        h = _rmsnorm(x, sd[p + ".input_layernorm.weight"], cfg.rms_eps)
        q = F.linear(h, sd[p + ".self_attn.q_proj.weight"]).view(B, S, H, hd).transpose(1, 2)
        k = F.linear(h, sd[p + ".self_attn.k_proj.weight"]).view(B, S, H, hd).transpose(1, 2)
        v = F.linear(h, sd[p + ".self_attn.v_proj.weight"]).view(B, S, H, hd).transpose(1, 2)
        q = (q * cos) + (_rotate_half(q) * sin)
        k = (k * cos) + (_rotate_half(k) * sin)
        if past_kv is not None:
            if past_kv[l] is not None:
                k = torch.cat([past_kv[l][0], k], dim=2)
                v = torch.cat([past_kv[l][1], v], dim=2)
            past_kv[l] = (k, v)
        w = torch.matmul(q, k.transpose(2, 3)) * (hd ** -0.5)
        w = w + add_mask
        w = torch.softmax(w, dim=-1, dtype=torch.float32).to(dt)
        a = torch.matmul(w, v).transpose(1, 2).reshape(B, S, D)
        x = x + F.linear(a, sd[p + ".self_attn.o_proj.weight"])
        h = _rmsnorm(x, sd[p + ".post_attention_layernorm.weight"], cfg.rms_eps)
        h = F.linear(F.silu(F.linear(h, sd[p + ".mlp.gate_proj.weight"])) * F.linear(h, sd[p + ".mlp.up_proj.weight"]),
                     sd[p + ".mlp.down_proj.weight"])
        x = x + h
    return _rmsnorm(x, sd[prefix + ".norm.weight"], cfg.rms_eps)


def modified_lm_forward(sd: SD, cfg: OracleConfig, input_ids, attention_mask, labels=None, cand_vis=None, hist_vis=None,
                        obj_vis=None, position_ids=None, past_kv=None) -> Dict[str, Any]:
    """ModifiedLM.forward (models/modified_lm.py:89-146)."""
    hist_loc = input_ids == cfg.hist_id
    cand_loc = input_ids == cfg.cand_id
    obj_loc = input_ids == cfg.obj_id
    emb = F.embedding(input_ids, sd["lang_model.model.embed_tokens.weight"]).clone()
    if cand_loc.sum() != 0:
        emb[cand_loc] = (emb[cand_loc] + cand_vis).to(emb.dtype)     # bf16 += fp32 -> add in fp32, round
    if hist_loc.sum() != 0:
        emb[hist_loc] = (emb[hist_loc] + hist_vis).to(emb.dtype)
    if obj_loc.sum() != 0:
        emb[obj_loc] = (emb[obj_loc] + obj_vis).to(emb.dtype)
    hidden = llama_model(sd, cfg, emb, attention_mask, position_ids, past_kv)
    logits = F.linear(hidden, sd["lang_model.lm_head.weight"])
    mask = torch.zeros(logits.shape[-1], dtype=torch.bool)
    mask[cfg.special_token_ids] = True
    logits = logits.masked_fill(mask, float("-inf"))
    loss = None
    if labels is not None:
        sl = logits[..., :-1, :].contiguous().view(-1, logits.shape[-1])
        tl = labels[..., 1:].contiguous().view(-1)
        loss = F.cross_entropy(sl, tl)
    return {"loss": loss, "logits": logits, "hidden_states": hidden}


# =====================================================================================================
# NavModel modes (models/nav_model.py)
# =====================================================================================================
def _pos_embed(x, sd, name):
    """nn.Sequential(Linear, LayerNorm(eps=1e-12))  (models/nav_model.py:60-75)."""
    return _ln(_lin(x, sd, name + ".0"), sd, name + ".1", 1e-12)


def _flatten_hist(hist_vis):
    flat = [v for vis in hist_vis for v in vis]
    return torch.stack(flat, dim=0) if flat else None


def forward_navigation(sd: SD, cfg: OracleConfig, batch: Dict[str, Any], tokenize) -> Dict[str, torch.Tensor]:
    """NavModel.forward_navigation (models/nav_model.py:129-247).  Consumes the global CPU RNG exactly like
    the reference (one torch.randperm per sample, :219)."""
    vp_img_embeds = batch["vp_img_embeds"]
    B = vp_img_embeds.size(0)
    gmap_masks, gmap_visited = batch["gmap_masks"], batch["gmap_visited_masks"]
    gmap_vpids, vp_cand_vpids = batch["gmap_vpids"], batch["vp_cand_vpids"]
    gmap_embeds = batch["gmap_img_embeds"] + F.embedding(batch["gmap_step_ids"], sd["gmap_step_embeddings.weight"]) \
        + _pos_embed(batch["gmap_pos_fts"], sd, "gmap_pos_embeddings")                       # :146-150
    vp_embeds = vp_img_embeds + _pos_embed(batch["vp_pos_fts"], sd, "vp_pos_embeddings")      # :159-162
    gmap_embeds = gmap_embeds.masked_fill(gmap_visited.unsqueeze(-1), 0.)                    # :165-166
    gmap_embeds = gmap_embeds.masked_fill(gmap_masks.logical_not().unsqueeze(-1), 0.)
    type_ids = torch.zeros(gmap_embeds.shape[:2], dtype=torch.long)
    local = vp_embeds.masked_fill(batch["pano_masks"].logical_not().unsqueeze(-1), 0.)        # :169-170
    fuse = gmap_embeds.clone()
    for i in range(B):                                                                        # :174-190
        visited = set(vp for vp, m in zip(gmap_vpids[i], gmap_visited[i]) if m)
        tmp = {}
        for j, cv in enumerate(vp_cand_vpids[i]):
            if j > 0 and cv not in visited:
                tmp[cv] = local[i, j]
        add = {}
        for j, vp in enumerate(gmap_vpids[i]):
            if j > 0 and vp not in visited:
                if vp in tmp:
                    add[j] = tmp[vp]
                else:
                    type_ids[i, j] = 1
        if add:
            idx = torch.tensor(sorted(add))
            upd = torch.zeros_like(fuse[i])
            upd[idx] = torch.stack([add[int(j)] for j in idx])
            fuse = torch.cat([fuse[:i], (fuse[i] + upd).unsqueeze(0), fuse[i + 1:]], dim=0)
    fuse = fuse + F.embedding(type_ids, sd["token_type_embeddings.weight"])                   # :192-194
    fuse = fuse.masked_fill(gmap_visited.unsqueeze(-1), 0.)
    fuse = fuse.masked_fill(gmap_masks.logical_not().unsqueeze(-1), 0.)
    cand_masks = gmap_masks & gmap_visited.logical_not()                                      # :196-197
    cand_nums = cand_masks.sum(dim=-1)
    hist_vis_input = _flatten_hist(batch["hist_vis"])
    text = tokenize(batch["prompts"])
    cand_embeds, inv_perms = [], []
    for bn in range(B):                                                                       # :214-224
        ce = fuse[bn][cand_masks[bn]][1:]
        perm = torch.randperm(ce.shape[0])
        inv = torch.arange(ce.shape[0])
        inv[perm] = torch.arange(ce.shape[0])
        inv_perms.append(inv)
        cand_embeds.append(ce[perm])
    cand_embeds = torch.cat(cand_embeds, dim=0)
    out = modified_lm_forward(sd, cfg, text["input_ids"], text["attention_mask"], cand_vis=cand_embeds,
                              hist_vis=hist_vis_input)
    hidden = out["hidden_states"]
    preds = F.linear(hidden[text["input_ids"] == cfg.cls_ids[0]], sd["out_head.0.weight"], sd["out_head.0.bias"])  # :237
    rows = []
    for i in range(B):                                                                        # :239-242
        vals = torch.cat([preds[i, 0:1], preds[i, 1:cand_nums[i]][inv_perms[i]]], dim=0)
        row = torch.full((fuse.shape[1],), float("-inf"), dtype=preds.dtype)
        row = row.masked_scatter(cand_masks[i], vals)
        rows.append(row)
    fuse_logits = torch.stack(rows, 0)
    return {"fuse_embeds": fuse.detach(), "fuse_logits": fuse_logits, "hidden_states": hidden,
            "input_ids": text["input_ids"], "attention_mask": text["attention_mask"]}


def _lm_labels(text):
    """labels = ids with the prompt part (token_type_ids == 0) set to -100 (models/nav_model.py:306-308,377-379)."""
    labels = text["input_ids"].clone()
    labels[text["token_type_ids"][:, -labels.shape[-1]:] == 0] = -100
    return labels


def forward_summarization(sd: SD, cfg: OracleConfig, batch, tokenize, eos_token: str, training=True, max_new_tokens=50,
                          trie=None, eos_token_id=2, pad_token_id=0, return_logits=False):
    """NavModel.forward_summarization (models/nav_model.py:251-343), training branch and greedy branch."""
    vp = batch["vp_img_embeds"][:, 1:, :]                                                      # remove stop :267-268
    nav_masks = batch["vp_nav_masks"][:, 1:]
    zeros14 = torch.zeros(vp.shape[:2] + (14,), dtype=torch.float)
    vp = vp + _pos_embed(zeros14, sd, "vp_pos_embeddings")                                     # :270-273
    vp = vp + F.embedding(torch.zeros(vp.shape[:2], dtype=torch.long), sd["token_type_embeddings.weight"])
    hist_vis_input = _flatten_hist(batch["hist_vis"])
    dt = batch["data_type"]
    all_text = []
    for bn in range(vp.size(0)):
        prompt = batch["prompts"][bn]
        label = (batch["answer"][bn] if dt[0] in ("eqa", "fgr2r") else batch["instruction"][bn]) + eos_token
        all_text.append([prompt, label] if training else prompt)
    text = tokenize(all_text)
    if training:
        out = modified_lm_forward(sd, cfg, text["input_ids"], text["attention_mask"], labels=_lm_labels(text),
                                  cand_vis=vp[nav_masks], hist_vis=hist_vis_input)
        return {"loss": out["loss"]}
    procs = [TrieLogitsProcessor(trie)] if trie is not None else []              # models/nav_model.py:321-322
    ids = greedy_generate(sd, cfg, text["input_ids"], text["attention_mask"], cand_vis=vp[nav_masks],
                          hist_vis=hist_vis_input, max_new_tokens=max_new_tokens, eos_token_id=eos_token_id,
                          pad_token_id=pad_token_id, logits_processor=procs, return_logits=return_logits)
    step_logits = None
    if return_logits:
        ids, step_logits = ids
    return {"generated_ids": ids[:, text["input_ids"].shape[1]:], "step_logits": step_logits}


def forward_3dqa(sd: SD, cfg: OracleConfig, batch, tokenize, eos_token: str, training=True, max_new_tokens=20):
    """NavModel.forward_3dqa (models/nav_model.py:346-404)."""
    B = len(batch["question"])
    all_text = []
    for bn in range(B):
        prompt = batch["prompts"][bn]
        all_text.append([prompt, batch["answers"][bn][0] + eos_token] if training else prompt)
    feats = batch["features"]
    lens = [f.shape[0] for f in feats]
    mx = max(lens)
    view = torch.stack([torch.cat([f, f.new_zeros(mx - f.shape[0], f.shape[1])], 0) for f in feats], 0)  # ops.py:44-66
    pano = forward_panorama(sd, cfg, view, torch.tensor(lens))
    pe, pm = pano["pano_embeds"], pano["pano_masks"]
    pe = pe + _pos_embed(torch.zeros(pe.shape[:2] + (14,), dtype=torch.float), sd, "vp_pos_embeddings")
    pe = pe + F.embedding(torch.zeros(pe.shape[:2], dtype=torch.long), sd["token_type_embeddings.weight"])
    text = tokenize(all_text)
    if training:
        return modified_lm_forward(sd, cfg, text["input_ids"], text["attention_mask"], labels=_lm_labels(text),
                                   cand_vis=pe[pm])
    ids = greedy_generate(sd, cfg, text["input_ids"], text["attention_mask"], cand_vis=pe[pm],
                          max_new_tokens=max_new_tokens)
    return {"generated_ids": ids[:, text["input_ids"].shape[1]:]}


def forward_object_grounding(sd: SD, cfg: OracleConfig, batch, tokenize):
    """NavModel.forward_object_grounding (models/nav_model.py:407-451)."""
    obj_embeds = batch["obj_embeds"] + _pos_embed(batch["obj_loc_fts"], sd, "obj_pos_embeddings")
    obj_masks = batch["obj_masks"]
    cand_nums = obj_masks.sum(dim=1) + 1
    text = tokenize(batch["prompts"])
    out = modified_lm_forward(sd, cfg, text["input_ids"], text["attention_mask"], cand_vis=obj_embeds[obj_masks],
                              hist_vis=_flatten_hist(batch["hist_vis"]))
    preds = F.linear(out["hidden_states"][text["input_ids"] == cfg.cls_ids[0]], sd["out_head.0.weight"],
                     sd["out_head.0.bias"])
    cols = torch.arange(preds.shape[1])[None, :]
    preds = preds.masked_fill(cols >= cand_nums[:, None], float("-inf"))
    return {"obj_logits": preds}


# =====================================================================================================
# Greedy decode (HF GenerationMixin greedy search semantics; models/modified_lm.py:184-199,
# models/nav_model.py:324-338,388-399).  Restated: see module docstring.
# =====================================================================================================
class TrieLogitsProcessor:
    """models/modified_lm.py:10-30: per-row walk of a Trie (tools/trie.py interface: root, get_next_node,
    get_child_index); every token that is not a child of the row's current node is masked to -inf."""

    def __init__(self, trie):
        self.node_states, self.trie = None, trie

    def __call__(self, input_ids, scores):
        B = input_ids.shape[0]
        if self.node_states is None:
            self.node_states = [self.trie.root for _ in range(B)]
        else:
            for bn in range(B):
                self.node_states[bn] = self.trie.get_next_node(self.node_states[bn], int(input_ids[bn, -1]))
        masks = torch.zeros_like(scores, dtype=torch.bool)
        for bn in range(B):
            masks[bn][self.trie.get_child_index(self.node_states[bn])] = True
        return scores.masked_fill(~masks, float("-inf"))


def greedy_generate(sd: SD, cfg: OracleConfig, input_ids, attention_mask, cand_vis=None, hist_vis=None, obj_vis=None,
                    max_new_tokens=20, eos_token_id=2, pad_token_id=0, stop_on_eos=True, return_logits=False,
                    logits_processor=None):
    B = input_ids.shape[0]
    ids = input_ids.clone()
    mask = attention_mask.clone()
    past: list = [None] * cfg.n_layers
    unfinished = torch.ones(B, dtype=torch.bool)
    step_logits = []
    for step in range(max_new_tokens):
        pos = (mask.long().cumsum(-1) - 1).masked_fill(mask == 0, 1)
        if step == 0:          # full prompt + visual tensors only when there is no past (modified_lm.py:195-197)
            out = modified_lm_forward(sd, cfg, ids, mask, cand_vis=cand_vis, hist_vis=hist_vis, obj_vis=obj_vis,
                                      position_ids=pos, past_kv=past)
        else:
            out = modified_lm_forward(sd, cfg, ids[:, -1:], mask, position_ids=pos[:, -1:], past_kv=past)
        logits = out["logits"][:, -1, :].float()
        for proc in (logits_processor or []):            # HF applies the processors to the next-token scores
            logits = proc(ids, logits)
        if return_logits:
            step_logits.append(logits)
        nxt = logits.argmax(dim=-1)
        nxt = torch.where(unfinished, nxt, torch.full_like(nxt, pad_token_id))
        ids = torch.cat([ids, nxt[:, None]], dim=1)
        mask = torch.cat([mask, mask.new_ones(B, 1)], dim=1)
        if stop_on_eos:
            unfinished = unfinished & (nxt != eos_token_id)
            if not bool(unfinished.any()):
                break
    return (ids, step_logits) if return_logits else ids


def sampling_probs(scores: torch.Tensor, temperature: float = 1.0, top_k: int = 50) -> torch.Tensor:
    """The distribution HF ``GenerationMixin.sample`` draws the next token from when the reference generates with
    ``do_sample=True`` (tasks/agents/llava.py:58-62 -> models/nav_model.py:388-396 -> lang_model.generate(**kwargs)):
    the logits warpers of transformers' generation utilities in their order - TemperatureLogitsWarper
    (``scores / temperature``, only when != 1) then TopKLogitsWarper (``top_k = 50`` is the generation default the
    reference never overrides; ``scores < topk(scores, k)[0][..., -1, None]`` -> -inf, so ties at the k-th value stay)
    - followed by ``softmax(dim=-1)`` IN THE SCORES' DTYPE (bf16 next-token logits in the reference) and
    ``torch.multinomial(probs, 1)``.  ``scores`` are the next-token logits after the logits processors (special tokens
    already -inf, models/modified_lm.py:122-124).  Pinned against the installed transformers' warper classes in
    tests/test_sampling_cpu.py."""
    s = scores
    if temperature != 1.0:
        s = s / temperature
    if top_k is not None and top_k > 0:
        k = min(int(top_k), s.shape[-1])
        kth = torch.topk(s, k)[0][..., -1, None]
        s = s.masked_fill(s < kth, float("-inf"))
    return F.softmax(s, dim=-1)


# =====================================================================================================
# Random initialisation in the reference's parameter naming (for tests / CPU baseline; HF default init)
# =====================================================================================================
def init_state_dict(cfg: OracleConfig, seed: int = 0) -> SD:
    g = torch.Generator().manual_seed(seed)
    dt = cfg.lm_dtype
    sd: SD = {}

    def n(*shape, std=0.02, dtype=torch.float32):
        return (torch.randn(*shape, generator=g) * std).to(dtype)

    D, Fi, V = cfg.hidden, cfg.inter, cfg.vocab
    sd["lang_model.model.embed_tokens.weight"] = n(V, D, dtype=dt)
    for l in range(cfg.n_layers):
        p = f"lang_model.model.layers.{l}"
        for nm in ("q_proj", "k_proj", "v_proj", "o_proj"):
            sd[f"{p}.self_attn.{nm}.weight"] = n(D, D, dtype=dt)
        sd[f"{p}.mlp.gate_proj.weight"] = n(Fi, D, dtype=dt)
        sd[f"{p}.mlp.up_proj.weight"] = n(Fi, D, dtype=dt)
        sd[f"{p}.mlp.down_proj.weight"] = n(D, Fi, dtype=dt)
        sd[f"{p}.input_layernorm.weight"] = torch.ones(D, dtype=dt)
        sd[f"{p}.post_attention_layernorm.weight"] = torch.ones(D, dtype=dt)
    sd["lang_model.model.norm.weight"] = torch.ones(D, dtype=dt)
    sd["lang_model.lm_head.weight"] = n(V, D, dtype=dt)
    Hp, Fp = cfg.pano_hidden, cfg.pano_inter
    P = "img_embeddings."

    def lin(name, out_f, in_f, dtype=torch.float32):
        sd[name + ".weight"] = n(out_f, in_f, std=in_f ** -0.5, dtype=dtype)
        sd[name + ".bias"] = n(out_f, std=0.02, dtype=dtype)

    def lnorm(name, dim):
        sd[name + ".weight"] = 1 + n(dim, std=0.05)
        sd[name + ".bias"] = n(dim, std=0.05)

    lin(P + "img_linear", Hp, cfg.image_feat_size); lnorm(P + "img_layer_norm", Hp)
    lin(P + "loc_linear", Hp, cfg.angle_feat_size + 3); lnorm(P + "loc_layer_norm", Hp)
    if cfg.enable_og:
        lin(P + "obj_projector.0", D, cfg.obj_feat_size); lnorm(P + "obj_projector.1", D)
    sd[P + "nav_type_embedding.weight"] = n(3, Hp, std=1.0)
    lnorm(P + "layer_norm", Hp)
    for l in range(cfg.num_pano_layers):
        p = f"{P}pano_encoder.layers.{l}"
        sd[p + ".self_attn.in_proj_weight"] = n(3 * Hp, Hp, std=Hp ** -0.5)
        sd[p + ".self_attn.in_proj_bias"] = n(3 * Hp, std=0.02)
        lin(p + ".self_attn.out_proj", Hp, Hp)
        lin(p + ".linear1", Fp, Hp); lin(p + ".linear2", Hp, Fp)
        lnorm(p + ".norm1", Hp); lnorm(p + ".norm2", Hp)
    lnorm(P + "pano_encoder.norm", Hp)
    lin(P + "mapper", D, Hp)
    sd["token_type_embeddings.weight"] = n(3, D, std=1.0)
    lin("gmap_pos_embeddings.0", D, cfg.angle_feat_size + 3); lnorm("gmap_pos_embeddings.1", D)
    sd["gmap_step_embeddings.weight"] = n(100, D, std=1.0)
    lin("vp_pos_embeddings.0", D, cfg.angle_feat_size * 2 + 6); lnorm("vp_pos_embeddings.1", D)
    lin("obj_pos_embeddings.0", D, cfg.angle_feat_size + 3); lnorm("obj_pos_embeddings.1", D)
    if cfg.obj_feat_size > 0:
        lin("og_head.0", 100, D, dtype=dt)
    lin("out_head.0", 100, D, dtype=dt)
    return sd
