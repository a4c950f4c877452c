"""Panorama scene encoder on the fp32 sm_90a kernels (csrc/pano_ops.cu), forward + hand-written backward.

Mirror of the reference's ``ImageEmbeddings`` (models/image_embedding.py:11-121) with the DETR pre-LN encoder
(models/detr_transformer.py:62-89,170-182; built by models/ops.py:6-18): same constructor arguments, same
parameter names/shapes (``img_linear``, ``img_layer_norm``, ``loc_linear``, ``loc_layer_norm``,
``obj_projector.{0,1}``, ``nav_type_embedding``, ``layer_norm``, ``pano_encoder.layers.N.{self_attn.in_proj_weight,
in_proj_bias,self_attn.out_proj,linear1,linear2,norm1,norm2}``, ``pano_encoder.norm``, ``mapper``) so reference
checkpoints load.  The torch.nn modules below are parameter holders (and give the reference's default
initialisation); their ``forward`` is never called -- all arithmetic runs in the C-ABI kernels.

Dropout (``train()`` only, like the reference): ``nn.Dropout(hidden_dropout_prob)`` after the embedding LayerNorm
(models/image_embedding.py:72) and, per encoder layer, the attention-probability dropout of nn.MultiheadAttention plus
``dropout1`` / ``dropout`` / ``dropout2`` (models/detr_transformer.py:136-146,170-182, p = 0.1).  Masks come from a
counter-based RNG keyed by (torch.cuda.initial_seed(), call counter, site): the backward regenerates them, the CPU RNG
stream (which the reference consumes in ``forward_navigation``) is untouched, and a run is reproducible after
``torch.manual_seed``.  The random STREAM differs from torch's Philox, so train-mode outputs match the reference in
distribution, not element-wise; element-wise parity is defined in ``eval()`` (SURVEY.md §8c).
``fuse_obj`` (``--fuse_obj``, tools/parser.py:95; off in the released configs) is the reference's branch
models/image_embedding.py:78-94: object tokens join the views in the encoder input; built on the same kernels through
row-index maps (``_fuse_maps``), forward and backward, and checked against the reference's own module
(tests/golden/pano_fuse_obj.pt).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import ops

f32 = torch.float32


class _EncoderLayer(nn.Module):
    def __init__(self, d_model, nhead, dim_ff):
        super().__init__()
        self.self_attn = nn.MultiheadAttention(d_model, nhead, dropout=0.1)
        self.linear1 = nn.Linear(d_model, dim_ff)
        self.linear2 = nn.Linear(dim_ff, d_model)
        self.norm1 = nn.LayerNorm(d_model)
        self.norm2 = nn.LayerNorm(d_model)


class _Encoder(nn.Module):
    def __init__(self, d_model, nhead, dim_ff, num_layers):
        super().__init__()
        self.layers = nn.ModuleList([_EncoderLayer(d_model, nhead, dim_ff) for _ in range(num_layers)])
        self.norm = nn.LayerNorm(d_model, eps=1e-12)


_DROPOUT_CALLS = [0]


def _dropout_seed() -> int:
    """Base seed of one forward call; site k of the call uses base + k."""
    _DROPOUT_CALLS[0] += 1
    return (int(torch.cuda.initial_seed()) * 0x9E3779B1 + _DROPOUT_CALLS[0] * 0x1000003) & (2 ** 63 - 1)


def _grad(p: torch.Tensor) -> torch.Tensor:
    if p.grad is None:
        p.grad = torch.zeros_like(p)
    return p.grad


def _lin_fwd(x, lin: nn.Linear, out=None, accumulate=False):
    return ops.sgemm(x, lin.weight.data, bias=lin.bias.data if lin.bias is not None else None, out=out,
                     accumulate=accumulate)


def _lin_bwd(dy, x, lin: nn.Linear, need_dx=True):
    """dW += dy^T x ; db += colsum(dy) ; returns dx = dy W."""
    ops.sgemm(dy, x, ta=True, tb=True, out=_grad(lin.weight), accumulate=True)
    if lin.bias is not None:
        ops.colsum_(dy, _grad(lin.bias), accumulate=True)
    return ops.sgemm(dy, lin.weight.data, tb=True) if need_dx else None


def _ln_fwd(x, ln: nn.LayerNorm, addend=None):
    return ops.layernorm_fwd(x, ln.weight.data, ln.bias.data, ln.eps, addend=addend)


def _ln_bwd(dy, x, ln: nn.LayerNorm, mean, rstd, dx=None, accumulate_dx=False):
    return ops.layernorm_bwd(x, ln.weight.data, mean, rstd, dy, dx=dx, accumulate_dx=accumulate_dx,
                             dgamma=_grad(ln.weight), dbeta=_grad(ln.bias))


class _PanoFn(torch.autograd.Function):
    """Differentiable boundary of the encoder: the outputs carry grad_fn so the caller's loss.backward()
    reaches ``backward`` below, which accumulates every parameter gradient natively."""

    @staticmethod
    def forward(ctx, mod: "ImageEmbeddings", view, lens32, loc, types32, keep_idx, anchor, fuse=None):
        B, N, Dv = view.shape
        R = B * N
        v2 = view.reshape(R, Dv)
        t = {}
        t["v2"] = v2
        t["ximg"] = _lin_fwd(v2, mod.img_linear)
        a, t["m_img"], t["r_img"] = _ln_fwd(t["ximg"], mod.img_layer_norm)
        t["loc2"] = loc.reshape(R, loc.shape[-1])
        t["xloc"] = _lin_fwd(t["loc2"], mod.loc_linear)
        c, t["m_loc"], t["r_loc"] = _ln_fwd(t["xloc"], mod.loc_layer_norm, addend=a)
        ops.rows_combine(c, b=mod.nav_type_embedding.weight.data, ib=types32, accumulate=True)
        t["c"] = c
        x, t["m_ln"], t["r_ln"] = _ln_fwd(c, mod.layer_norm)
        # train-mode dropout: p of the embedding dropout, p_l of the encoder layers (nn.MultiheadAttention(dropout=0.1)
        # and the three nn.Dropout(0.1) of TransformerEncoderLayer); seeds = base + site index
        p_emb = float(mod.dropout.p) if mod.training else 0.0
        p_l = float(mod.encoder_dropout) if mod.training else 0.0
        seed = _dropout_seed() if (p_emb > 0 or p_l > 0) else 0
        t["p_emb"], t["p_l"], t["seed"] = p_emb, p_l, seed
        if p_emb > 0:
            x = ops.dropout(x, p_emb, seed)
        layers = []
        enc = mod.pano_encoder
        Ne, lens_e = N, lens32                         # the encoder's view of the batch (fuse_obj: views + objects per row)
        if enc is not None and fuse is not None:
            # `--fuse_obj` (models/image_embedding.py:78-94): object tokens = obj_linear (Linear + LN) + the SHARED
            # LN(loc_linear(obj_loc_fts)) + nav-type 2 - not through layer_norm / dropout - appended to each row's views
            obj, obj_loc = fuse["obj"], fuse["obj_loc"]
            O_ = obj.shape[1]
            t["o2"] = obj.reshape(B * O_, obj.shape[-1])
            t["ox"] = _lin_fwd(t["o2"], mod.obj_linear[0])
            oa, t["m_o"], t["r_o"] = _ln_fwd(t["ox"], mod.obj_linear[1])
            t["oloc2"] = obj_loc.reshape(B * O_, obj_loc.shape[-1])
            t["oxloc"] = _lin_fwd(t["oloc2"], mod.loc_linear)
            oe, t["m_oloc"], t["r_oloc"] = _ln_fwd(t["oxloc"], mod.loc_layer_norm, addend=oa)
            ops.rows_combine(oe, b=mod.nav_type_embedding.weight.data, ib=fuse["twos"], accumulate=True)
            Ne, lens_e = fuse["Nf"], fuse["lens_f"]
            xf = torch.empty((B * Ne, x.shape[1]), dtype=f32, device=x.device)
            ops.rows_combine(xf, a=x, ia=fuse["view_src"], b=oe, ib=fuse["obj_src"])       # pad rows: zeros (pad_tensors_wgrad)
            x = xf
        if enc is not None:
            N, lens32, R = Ne, lens_e, B * Ne
            for li, lyr in enumerate(enc.layers):
                s = {"x": x}
                sd = seed + 16 * (li + 1)
                s["h"], s["m1"], s["r1"] = _ln_fwd(x, lyr.norm1)
                s["qkv"] = ops.sgemm(s["h"], lyr.self_attn.in_proj_weight.data, bias=lyr.self_attn.in_proj_bias.data)
                if p_l > 0:
                    att, s["P"], s["Pd"] = ops.mha_fwd_dropout(s["qkv"].view(B, N, -1), lens32, mod.num_heads, p_l, sd)
                else:
                    att, s["P"] = ops.mha_fwd(s["qkv"].view(B, N, -1), lens32, mod.num_heads)
                s["att"] = att.view(R, -1)
                if p_l > 0:
                    x1 = x + ops.dropout(_lin_fwd(s["att"], lyr.self_attn.out_proj), p_l, sd + 1)      # dropout1
                else:
                    x1 = x.clone()
                    _lin_fwd(s["att"], lyr.self_attn.out_proj, out=x1, accumulate=True)
                s["x1"] = x1
                s["h2"], s["m2"], s["r2"] = _ln_fwd(x1, lyr.norm2)
                s["z"] = _lin_fwd(s["h2"], lyr.linear1)
                s["a1"] = ops.gelu_fwd(s["z"])
                if p_l > 0:
                    s["a1"] = ops.dropout(s["a1"], p_l, sd + 2)                                         # dropout (FFN)
                    x = x1 + ops.dropout(_lin_fwd(s["a1"], lyr.linear2), p_l, sd + 3)                   # dropout2
                else:
                    x2 = x1.clone()
                    _lin_fwd(s["a1"], lyr.linear2, out=x2, accumulate=True)
                    x = x2
                layers.append(s)
            if fuse is not None:                       # the view rows come back (:92-93); the final LayerNorm is row-wise
                N, R = view.shape[1], B * view.shape[1]
                xv = torch.empty((R, x.shape[1]), dtype=f32, device=x.device)
                ops.rows_combine(xv, a=x, ia=fuse["view_back"])
                x = xv
            t["xe"] = x
            x, t["m_f"], t["r_f"] = _ln_fwd(x, enc.norm)
        t["y"] = x
        m = _lin_fwd(x, mod.mapper)
        out = torch.empty_like(m)
        ops.rows_combine(out, a=m, ia=keep_idx)       # zero the padded rows (image_embedding.py:103)
        ctx.mod, ctx.t, ctx.layers = mod, t, layers
        ctx.dims = (B, N)
        ctx.enc_dims = (Ne, lens_e)
        ctx.fuse = fuse
        ctx.types32, ctx.keep_idx = types32, keep_idx
        return out.view(B, N, -1)

    @staticmethod
    def backward(ctx, dout):
        mod, t, layers = ctx.mod, ctx.t, ctx.layers
        B, N = ctx.dims
        R = B * N
        dout = dout.contiguous().view(R, -1).to(f32)
        dm = torch.empty_like(dout)
        ops.rows_combine(dm, a=dout, ia=ctx.keep_idx)               # padded rows carry no gradient
        dx = _lin_bwd(dm, t["y"], mod.mapper)
        enc = mod.pano_encoder
        fuse = ctx.fuse
        if enc is not None:
            dx = _ln_bwd(dx, t["xe"], enc.norm, t["m_f"], t["r_f"])
            if fuse is not None:                       # gradient of the view rows into the fused layout; object / pad rows: 0
                N, lens_e = ctx.enc_dims
                R = B * N
                dxf = torch.empty((R, dx.shape[1]), dtype=f32, device=dx.device)
                ops.rows_combine(dxf, a=dx, ia=fuse["view_src"])
                dx = dxf
            lens32 = ctx.enc_dims[1]
            p_l, seed = t["p_l"], t["seed"]
            n_l = len(layers)
            for li, (lyr, s) in enumerate(zip(reversed(list(enc.layers)), reversed(layers))):
                sd = seed + 16 * (n_l - li)
                dy2 = ops.dropout(dx, p_l, sd + 3) if p_l > 0 else dx                 # dropout2
                da1 = _lin_bwd(dy2, s["a1"], lyr.linear2)                             # s["a1"] = dropped activation
                if p_l > 0:
                    da1 = ops.dropout(da1, p_l, sd + 2)
                dz = ops.gelu_bwd(s["z"], da1)
                dh2 = _lin_bwd(dz, s["h2"], lyr.linear1)
                dx1 = dx.clone()
                _ln_bwd(dh2, s["x1"], lyr.norm2, s["m2"], s["r2"], dx=dx1, accumulate_dx=True)
                dy1 = ops.dropout(dx1, p_l, sd + 1) if p_l > 0 else dx1               # dropout1
                datt = _lin_bwd(dy1, s["att"], lyr.self_attn.out_proj)
                if p_l > 0:
                    dqkv = ops.mha_bwd_dropout(s["qkv"].view(B, N, -1), datt.view(B, N, -1), s["P"], s["Pd"], lens32,
                                               mod.num_heads).view(R, -1)
                else:
                    dqkv = ops.mha_bwd(s["qkv"].view(B, N, -1), datt.view(B, N, -1), s["P"], lens32, mod.num_heads).view(R, -1)
                sa = lyr.self_attn
                ops.sgemm(dqkv, s["h"], ta=True, tb=True, out=_grad(sa.in_proj_weight), accumulate=True)
                ops.colsum_(dqkv, _grad(sa.in_proj_bias), accumulate=True)
                dh = ops.sgemm(dqkv, sa.in_proj_weight.data, tb=True)
                dx = dx1
                _ln_bwd(dh, s["x"], lyr.norm1, s["m1"], s["r1"], dx=dx, accumulate_dx=True)
        if enc is not None and fuse is not None:
            # split the fused gradient: object rows -> obj_linear / shared loc branch / nav-type row 2; view rows go on
            O_ = t["o2"].shape[0] // B
            d_oe = torch.empty((B * O_, dx.shape[1]), dtype=f32, device=dx.device)
            ops.rows_combine(d_oe, a=dx, ia=fuse["obj_back"])
            ops.rows_scatter_add_(_grad(mod.nav_type_embedding.weight), fuse["twos"], d_oe)
            d_oxloc = _ln_bwd(d_oe, t["oxloc"], mod.loc_layer_norm, t["m_oloc"], t["r_oloc"])
            _lin_bwd(d_oxloc, t["oloc2"], mod.loc_linear, need_dx=False)
            d_ox = _ln_bwd(d_oe, t["ox"], mod.obj_linear[1], t["m_o"], t["r_o"])
            _lin_bwd(d_ox, t["o2"], mod.obj_linear[0], need_dx=False)
            N = ctx.dims[1]
            R = B * N
            dxv = torch.empty((R, dx.shape[1]), dtype=f32, device=dx.device)
            ops.rows_combine(dxv, a=dx, ia=fuse["view_back"])
            dx = dxv
        if t["p_emb"] > 0:
            dx = ops.dropout(dx.contiguous(), t["p_emb"], t["seed"])
        dc = _ln_bwd(dx, t["c"], mod.layer_norm, t["m_ln"], t["r_ln"])
        ops.rows_scatter_add_(_grad(mod.nav_type_embedding.weight), ctx.types32, dc)
        dxloc = _ln_bwd(dc, t["xloc"], mod.loc_layer_norm, t["m_loc"], t["r_loc"])
        _lin_bwd(dxloc, t["loc2"], mod.loc_linear, need_dx=False)
        dximg = _ln_bwd(dc, t["ximg"], mod.img_layer_norm, t["m_img"], t["r_img"])
        _lin_bwd(dximg, t["v2"], mod.img_linear, need_dx=False)
        ctx.t = ctx.layers = None
        return None, None, None, None, None, None, None, None


class _ObjFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mod: "ImageEmbeddings", obj, anchor):
        B, O, Do = obj.shape
        o2 = obj.reshape(B * O, Do)
        x = _lin_fwd(o2, mod.obj_projector[0])
        y, mean, rstd = _ln_fwd(x, mod.obj_projector[1])
        ctx.mod, ctx.saved = mod, (o2, x, mean, rstd)
        return y.view(B, O, -1)

    @staticmethod
    def backward(ctx, dy):
        mod = ctx.mod
        o2, x, mean, rstd = ctx.saved
        dy = dy.contiguous().view(x.shape[0], -1).to(f32)
        dx = _ln_bwd(dy, x, mod.obj_projector[1], mean, rstd)
        _lin_bwd(dx, o2, mod.obj_projector[0], need_dx=False)
        return None, None, None


def gen_seq_masks(seq_lens: torch.Tensor, max_len=None) -> torch.Tensor:
    """models/ops.py:33-41 (max over lens is a host value: lens arrive from the host in the agent)."""
    if max_len is None:
        max_len = int(seq_lens.max())
    return torch.arange(max_len, device=seq_lens.device).unsqueeze(0) < seq_lens.unsqueeze(1)


class ImageEmbeddings(nn.Module):
    def __init__(self, config, use_obj: bool = False, fuse_obj: bool = False):
        super().__init__()
        H = config.hidden_size
        self.num_heads = config.num_attention_heads
        self.img_linear = nn.Linear(config.image_feat_size, H)
        self.img_layer_norm = nn.LayerNorm(H, eps=1e-12)
        self.loc_linear = nn.Linear(config.angle_feat_size + 3, H)
        self.loc_layer_norm = nn.LayerNorm(H, eps=1e-12)
        self.fuse_obj = fuse_obj
        if use_obj:
            if fuse_obj:                                # registered before obj_projector, like the reference (:21-30)
                self.obj_linear = nn.Sequential(nn.Linear(config.obj_feat_size, H), nn.LayerNorm(H, eps=1e-12))
            self.obj_projector = nn.Sequential(nn.Linear(config.obj_feat_size, config.output_size),
                                               nn.LayerNorm(config.output_size, eps=1e-12))
        else:
            self.obj_projector = None
            self.obj_linear = None
        self.nav_type_embedding = nn.Embedding(3, H)
        self.layer_norm = nn.LayerNorm(H, eps=1e-12)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)
        self.encoder_dropout = config.hidden_dropout_prob   # models/ops.py:6-12: TransformerEncoderLayer(dropout=hidden_dropout_prob)
        if config.num_pano_layers > 0:
            self.pano_encoder = _Encoder(H, config.num_attention_heads, config.intermediate_size, config.num_pano_layers)
        else:
            self.pano_encoder = None
        self.mapper = nn.Linear(H, config.output_size)
        # autograd anchor: a 0-d tensor that requires grad so the Function's outputs get a grad_fn even
        # though no *input tensor* of the encoder needs a gradient (parameters are updated natively)
        self.register_buffer("_anchor", torch.zeros((), dtype=f32), persistent=False)

    def _fuse_maps(self, view_lens, obj_img_fts, obj_lens, obj_loc_fts, B, N, dev):
        """Index maps of the `fuse_obj` layout (models/image_embedding.py:81-93): row b of the encoder input is
        [views[b, :view_lens[b]] ; objs[b, :obj_lens[b]]] zero-padded to max_b(view_lens + obj_lens).  The lengths are
        host values in the agent (the reference reads them on the host too: `:view_lens[bn]` slices, gen_seq_masks max)."""
        if getattr(self, "obj_linear", None) is None:
            raise RuntimeError("fuse_obj=True needs a model built with enable_og=True (obj_linear is only created then, "
                               "models/image_embedding.py:21-26)")
        if obj_img_fts is None or obj_lens is None or obj_loc_fts is None:
            raise ValueError("fuse_obj=True: obj_img_fts, obj_lens and obj_loc_fts are required (models/image_embedding.py:79-80)")
        vl = [int(v) for v in view_lens.tolist()]
        ol = [int(v) for v in obj_lens.tolist()]
        O_ = obj_img_fts.shape[1]
        Nf = max(v + w for v, w in zip(vl, ol))
        view_src, obj_src = [-1] * (B * Nf), [-1] * (B * Nf)
        view_back, obj_back = [-1] * (B * N), [-1] * (B * O_)
        for b in range(B):
            for j in range(vl[b]):
                view_src[b * Nf + j] = b * N + j
                view_back[b * N + j] = b * Nf + j
            for j in range(ol[b]):
                obj_src[b * Nf + vl[b] + j] = b * O_ + j
                obj_back[b * O_ + j] = b * Nf + vl[b] + j
        maps = torch.tensor(view_src + obj_src + view_back + obj_back + [v + w for v, w in zip(vl, ol)] + [2] * (B * O_),
                            dtype=torch.int32).to(dev, non_blocking=True)                    # one upload
        o = [0, B * Nf, 2 * B * Nf, 2 * B * Nf + B * N, 2 * B * Nf + B * N + B * O_, 2 * B * Nf + B * N + B * O_ + B]
        return {"Nf": Nf, "view_src": maps[o[0]:o[1]], "obj_src": maps[o[1]:o[2]], "view_back": maps[o[2]:o[3]],
                "obj_back": maps[o[3]:o[4]], "lens_f": maps[o[4]:o[5]].contiguous(), "twos": maps[o[5]:],
                "obj": obj_img_fts.to(f32).contiguous(), "obj_loc": obj_loc_fts.to(f32).contiguous()}

    def forward_panorama_per_step(self, view_img_fts, view_lens, loc_fts=None, nav_types=None, obj_img_fts=None,
                                  obj_lens=None, obj_loc_fts=None):
        """Same contract as the reference (models/image_embedding.py:51-121)."""
        if not view_img_fts.is_cuda:
            raise RuntimeError("navillm_b200 has no CPU path: inputs must be CUDA tensors")
        dev = view_img_fts.device
        B, N = view_img_fts.shape[:2]
        view = view_img_fts.to(f32).contiguous()
        if loc_fts is None:
            loc_fts = torch.zeros((B, N, 7), dtype=f32, device=dev)
        if nav_types is None:
            nav_types = torch.ones((B, N), dtype=torch.int32, device=dev)
        lens32 = view_lens.to(device=dev, dtype=torch.int32)
        pano_masks = gen_seq_masks(view_lens.to(dev), N)
        rows = torch.arange(B * N, device=dev, dtype=torch.int32)
        keep_idx = torch.where(pano_masks.reshape(-1), rows, torch.full_like(rows, -1))
        anchor = self._anchor.detach().requires_grad_(torch.is_grad_enabled())
        fuse = None
        if self.fuse_obj and self.pano_encoder is not None:
            fuse = self._fuse_maps(view_lens, obj_img_fts, obj_lens, obj_loc_fts, B, N, dev)
        pano = _PanoFn.apply(self, view, lens32, loc_fts.to(f32).contiguous(), nav_types.to(torch.int32).reshape(-1).contiguous(),
                             keep_idx, anchor, fuse)
        ret = {"pano_embeds": pano, "pano_masks": pano_masks}
        if obj_img_fts is not None and obj_img_fts.shape[1] > 0:
            assert self.obj_projector is not None, "object features given but the model was built with enable_og=False"
            obj = _ObjFn.apply(self, obj_img_fts.to(f32).contiguous(), anchor)
            obj_masks = gen_seq_masks(obj_lens.to(dev), obj_img_fts.shape[1])
            assert obj.shape[:2] == obj_loc_fts.shape[:2], \
                f"shape of obj_embeds {obj.shape[:2]} must equal to shape of obj_loc_fts {obj_loc_fts.shape[:2]}"
            ret.update({"obj_embeds": obj, "obj_loc_fts": obj_loc_fts, "obj_masks": obj_masks})
        return ret
