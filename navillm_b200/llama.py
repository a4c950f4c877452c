"""Packed LLaMA decoder stack over the sm_90a kernels: hand-written forward AND backward.

Host-side mirror of what the reference reaches through ``ModifiedLlamaForCausalLM`` ->
``transformers.models.llama.LlamaModel`` (reference call site models/modified_lm.py:112-116; HF names kept
so released checkpoints load: SURVEY.md §5 "checkpoint / resume").  Differences in *how*, not *what*:

* rows are PACKED: only real tokens are computed (the reference pads to the longest prompt and computes the
  pads); the reference's ``position_ids`` convention is reproduced by explicit per-token positions;
* q/k/v and gate/up projections run as one GEMM each on fused weight views ([3D,D], [2F,D]);
* attention never materialises [B,H,S,S];
* backward is explicit (no autograd graph inside the stack): activations are saved per layer, weight
  gradients are accumulated in place into a flat bf16 gradient buffer by the wgrad GEMM epilogue.

PyTorch is used for device memory only.  There is no CPU path.
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import List, Optional

import torch
import torch.nn as nn

from . import ops

# decode GEMMs: 0 (default) = swap-AB skinny kernel for batches <= 16 (csrc/gemm_skinny.cu), nv_gemm_bf16's measured tile
# table above that; 128 / 32 = force that column-tile width of the general kernel (A/B measurements)
DECODE_BLOCK_N = int(os.environ.get("NAVILLM_DECODE_BLOCK_N", "0"))
# weight-gradient GEMMs on a side stream (see LlamaCore.backward)
WGRAD_STREAM = os.environ.get("NAVILLM_WGRAD_STREAM", "0") != "0"

bf16 = torch.bfloat16


@dataclass
class LlamaDims:
    hidden: int = 4096
    n_layers: int = 32
    n_heads: int = 32
    inter: int = 11008
    vocab: int = 32006
    rms_eps: float = 1e-6
    rope_theta: float = 10000.0
    max_pos: int = 4096

    @property
    def head_dim(self) -> int:
        return self.hidden // self.n_heads


class _Linear(nn.Module):
    """Parameter holder with HF naming (``<name>.weight``); the math lives in the C-ABI kernels."""

    def __init__(self, out_f: int, in_f: int, bias: bool = False, dtype=bf16):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(out_f, in_f, dtype=dtype))
        self.bias = nn.Parameter(torch.empty(out_f, dtype=dtype)) if bias else None


class _Norm(nn.Module):
    def __init__(self, dim: int, dtype=bf16):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(dim, dtype=dtype))


class _Attn(nn.Module):
    def __init__(self, d: LlamaDims, dtype):
        super().__init__()
        self.q_proj = _Linear(d.hidden, d.hidden, dtype=dtype)
        self.k_proj = _Linear(d.hidden, d.hidden, dtype=dtype)
        self.v_proj = _Linear(d.hidden, d.hidden, dtype=dtype)
        self.o_proj = _Linear(d.hidden, d.hidden, dtype=dtype)


class _MLP(nn.Module):
    def __init__(self, d: LlamaDims, dtype):
        super().__init__()
        # registration order of transformers==4.28.0's LlamaMLP (gate, down, up): torch.optim state indices of reference
        # checkpoints follow model.parameters() order (tools/optims.py:43,69-71).  The fused gate|up weight view depends
        # only on the flat-buffer order (ModifiedLlamaForCausalLM.lm_parameters), not on this one.
        self.gate_proj = _Linear(d.inter, d.hidden, dtype=dtype)
        self.down_proj = _Linear(d.hidden, d.inter, dtype=dtype)
        self.up_proj = _Linear(d.inter, d.hidden, dtype=dtype)


class _Layer(nn.Module):
    def __init__(self, d: LlamaDims, dtype):
        super().__init__()
        self.self_attn = _Attn(d, dtype)
        self.mlp = _MLP(d, dtype)
        self.input_layernorm = _Norm(d.hidden, dtype)
        self.post_attention_layernorm = _Norm(d.hidden, dtype)


class _Embedding(nn.Module):
    def __init__(self, n: int, dim: int, dtype):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(n, dim, dtype=dtype))


class LlamaModelParams(nn.Module):
    """``model.*`` sub-tree: embed_tokens, layers.N.{self_attn,mlp,input_layernorm,post_attention_layernorm}, norm."""

    def __init__(self, d: LlamaDims, dtype=bf16):
        super().__init__()
        self.embed_tokens = _Embedding(d.vocab, d.hidden, dtype)
        self.layers = nn.ModuleList([_Layer(d, dtype) for _ in range(d.n_layers)])
        self.norm = _Norm(d.hidden, dtype)

    def flat_order(self) -> List[nn.Parameter]:
        """Parameter order of the flat buffer: q|k|v and gate|up of a layer adjacent (fused [3D,D] / [2F,D] views).  NOT
        ``parameters()`` order, which follows the reference's registration order (see ``_MLP``)."""
        ps: List[nn.Parameter] = []
        for lyr in self.layers:
            a, m = lyr.self_attn, lyr.mlp
            ps += [a.q_proj.weight, a.k_proj.weight, a.v_proj.weight, a.o_proj.weight, m.gate_proj.weight, m.up_proj.weight,
                   m.down_proj.weight, lyr.input_layernorm.weight, lyr.post_attention_layernorm.weight]
        return ps + [self.embed_tokens.weight, self.norm.weight]


def init_llama_params_(model: LlamaModelParams, lm_head: _Linear, std: float = 0.02, seed: int = 0) -> None:
    """HF default init (normal(0, 0.02) for linears/embeddings, ones for RMSNorm), generated on the host."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in list(model.parameters()) + list(lm_head.parameters()):
            if p.dim() == 1:
                p.fill_(1.0)
            else:
                # chunked so a 7B init never holds more than one fp32 matrix on the host
                p.copy_((torch.randn(p.shape, generator=g) * std).to(p.dtype))


class FlatParams:
    """Re-homes a list of same-dtype parameters into ONE contiguous buffer (and one gradient buffer).

    q/k/v and gate/up of a layer become adjacent row blocks, so the fused [3D,D] / [2F,D] weights are plain
    views; ``p.grad`` of every parameter is a view of the flat gradient buffer, so data-parallel reduction is a
    single NCCL all-reduce over ``flat_grad`` (SURVEY.md §8e) and the optimizer sees ordinary ``.grad``s.
    """

    def __init__(self, params: List[nn.Parameter], device: torch.device):
        assert params and all(p.dtype == params[0].dtype for p in params)
        self.params = params
        self.dtype = params[0].dtype
        align = 64  # elements; keeps every view 128-byte aligned for TMA / vector access
        offs, total = [], 0
        for p in params:
            offs.append(total)
            total += (p.numel() + align - 1) // align * align
        self.offsets = offs
        self.flat = torch.empty(total, dtype=self.dtype, device=device)
        self.flat_grad = torch.zeros(total, dtype=self.dtype, device=device)
        with torch.no_grad():
            for p, o in zip(params, offs):
                view = self.flat[o:o + p.numel()].view(p.shape)
                view.copy_(p.data.to(device))
                p.data = view
                p.grad = self.flat_grad[o:o + p.numel()].view(p.shape)
        self._ptr0 = params[0].data_ptr()

    def intact(self) -> bool:
        return self.params[0].data_ptr() == self._ptr0 and self.params[0].grad is not None and \
            self.params[0].grad.data_ptr() == self.flat_grad.data_ptr()

    def offset_of(self, p: nn.Parameter) -> int:
        return self.offsets[next(k for k, q in enumerate(self.params) if q is p)]

    def rebind_grads(self, new_flat_grad: torch.Tensor) -> None:
        """Move the gradient buffer (e.g. into a symmetric NVLS allocation): same layout, ``p.grad`` re-viewed."""
        assert new_flat_grad.numel() == self.flat_grad.numel() and new_flat_grad.dtype == self.flat_grad.dtype
        self.flat_grad = new_flat_grad
        for p, o in zip(self.params, self.offsets):
            p.grad = self.flat_grad[o:o + p.numel()].view(p.shape)

    def reattach_grads(self) -> None:
        """After ``optimizer.zero_grad(set_to_none=True)``: zero the buffer and hand the views back."""
        self.flat_grad.zero_()
        for p, o in zip(self.params, self.offsets):
            p.grad = self.flat_grad[o:o + p.numel()].view(p.shape)
        if getattr(self, "on_zeroed", None) is not None:
            self.on_zeroed()

    def _fused_span(self, members, shape):
        """Offset / size of the fused view over ``members`` (parameters that must sit back to back, in this order, in the
        flat buffer -- identity-checked: a look-alike neighbour of the same size must not pass)."""
        i = next(k for k, p in enumerate(self.params) if p is members[0])
        o = self.offsets[i]
        numel = 1
        for s in shape:
            numel *= s
        end = o
        for j, m in enumerate(members):
            if i + j >= len(self.params) or self.params[i + j] is not m or self.offsets[i + j] != end:
                raise RuntimeError("fused weight view: the members are not adjacent, in order and unpadded in the flat buffer "
                                   "(build FlatParams from LlamaModelParams.flat_order())")
            end += m.numel()
        if end - o != numel:
            raise RuntimeError(f"fused weight view: members hold {end - o} elements, shape {tuple(shape)} needs {numel}")
        return o, numel

    def view(self, members, shape) -> torch.Tensor:
        o, numel = self._fused_span(members, shape)
        return self.flat[o:o + numel].view(shape)

    def grad_view(self, members, shape) -> torch.Tensor:
        o, numel = self._fused_span(members, shape)
        return self.flat_grad[o:o + numel].view(shape)


def allreduce_flat_grads(flats, average: bool = True) -> int:
    """Data-parallel gradient exchange of the path (SURVEY.md §8e): ONE all-reduce per flat gradient buffer
    (bf16 LM+heads, fp32 encoder/embeddings) instead of DDP's per-bucket reductions (tools/optims.py:52-54).
    Returns the number of collectives issued (0 without an initialised multi-rank process group)."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return 0
    ws = dist.get_world_size()
    n = 0
    for flat in flats:
        if flat is None:
            continue
        dist.all_reduce(flat.flat_grad)
        if average:
            flat.flat_grad.div_(ws)
        n += 1
    return n


def rope_tables(d: LlamaDims, device) -> tuple:
    """cos/sin [max_pos, head_dim] in bf16, built exactly like HF LlamaRotaryEmbedding (fp32 cos/sin of
    pos * inv_freq, concatenated halves, cast to the model dtype)."""
    hd = d.head_dim
    inv = 1.0 / (d.rope_theta ** (torch.arange(0, hd, 2, dtype=torch.int64).float() / hd))
    fr = torch.arange(d.max_pos, dtype=torch.float32)[:, None] * inv[None, :]
    emb = torch.cat([fr, fr], dim=-1)
    return emb.cos().to(bf16).to(device).contiguous(), emb.sin().to(bf16).to(device).contiguous()


class _Saved:
    __slots__ = ("x", "rstd1", "xn", "qkv", "ao", "lse", "xm", "rstd2", "xn2", "gu", "h", "rows", "ao_r")


class LlamaCore:
    """Forward/backward driver of the decoder stack on packed rows.  Not an nn.Module: parameters live in
    ``LlamaModelParams`` (HF-named) and are accessed through fused views of a ``FlatParams`` buffer."""

    def __init__(self, dims: LlamaDims, model: LlamaModelParams, flat: FlatParams):
        self.d = dims
        self.model = model
        self.flat = flat
        D, F = dims.hidden, dims.inter
        self.wqkv, self.gqkv, self.wo, self.go, self.wgu, self.ggu, self.wd, self.gd = [], [], [], [], [], [], [], []
        for lyr in model.layers:
            a, m = lyr.self_attn, lyr.mlp
            qkv = [a.q_proj.weight, a.k_proj.weight, a.v_proj.weight]
            self.wqkv.append(flat.view(qkv, (3 * D, D)))
            self.gqkv.append(flat.grad_view(qkv, (3 * D, D)))
            self.wo.append(a.o_proj.weight.data)
            self.go.append(a.o_proj.weight.grad)
            gu = [m.gate_proj.weight, m.up_proj.weight]
            self.wgu.append(flat.view(gu, (2 * F, D)))
            self.ggu.append(flat.grad_view(gu, (2 * F, D)))
            self.wd.append(m.down_proj.weight.data)
            self.gd.append(m.down_proj.weight.grad)
        self.cos, self.sin = rope_tables(dims, flat.flat.device)
        self.fused_epilogues = True

    def refresh_grad_views(self) -> None:
        """Re-derive the fused gradient views after ``FlatParams.rebind_grads``."""
        D, F = self.d.hidden, self.d.inter
        flat = self.flat
        for l, lyr in enumerate(self.model.layers):
            a, m = lyr.self_attn, lyr.mlp
            self.gqkv[l] = flat.grad_view([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], (3 * D, D))
            self.go[l] = a.o_proj.weight.grad
            self.ggu[l] = flat.grad_view([m.gate_proj.weight, m.up_proj.weight], (2 * F, D))
            self.gd[l] = m.down_proj.weight.grad

    # -------------------------------------------------------------------------------------------------
    # packed batches below this many rows run the inference forward through ONE C-ABI call per layer (csrc/layer.cu):
    # they are host-bound when every kernel is its own call from Python
    LAYER_CALL = os.environ.get("NAVILLM_LAYER_CALL", "1") != "0"

    def _forward_layer_calls(self, x, pos, cu, seqlens, kv_store, out_rows):
        d = self.d
        T = x.shape[0]
        R = 0 if out_rows is None else out_rows.numel()
        run = ops.LayerRunner(T, d.hidden, d.inter, d.n_heads, d.rms_eps, pos, self.cos, self.sin, cu, len(seqlens), ops._qblocks(seqlens),
                              R=R, device=x.device)
        if kv_store is not None:
            run.set_cache_mode(1, kv_store[0][0].shape[1])
        bufs = [torch.empty_like(x), torch.empty_like(x)]
        last = d.n_layers - 1
        for l, lyr in enumerate(self.model.layers):
            pruned = out_rows is not None and l == last
            y = torch.empty((R, d.hidden), dtype=bf16, device=x.device) if pruned else bufs[l & 1]
            run.run(x, y, lyr.input_layernorm.weight.data, self.wqkv[l], self.wo[l], lyr.post_attention_layernorm.weight.data, self.wgu[l],
                    self.wd[l], kc=kv_store[0][l] if kv_store is not None else None, vc=kv_store[1][l] if kv_store is not None else None,
                    out_rows=out_rows if pruned else None)
            x = y
        return x

    def forward(self, x: torch.Tensor, pos: torch.Tensor, cu: torch.Tensor, seqlens, save: bool = True, kv_sink=None,
                out_rows: Optional[torch.Tensor] = None, kv_store=None):
        """x: [T, D] bf16 input embeddings (packed); pos: int32 [T]; cu: int32 [B+1] (device); seqlens: host
        lengths.  Returns (residual stream after the last layer BEFORE the final RMSNorm, tape) where ``tape``
        holds the per-layer activations for ``backward`` (None when save=False).  The tape travels with the
        caller (autograd ctx), so several forwards may be in flight before their backwards run.

        ``out_rows`` (int32 [R], device): only these rows of the output are needed (the <cls_1> rows in the
        navigation / grounding modes, the label rows in the LM-loss modes, the last rows in prefill).  The last
        layer then runs o_proj / MLP on R rows instead of T (its K,V still come from all rows) and the return
        value is [R, D].  The reference computes all positions and reads only these (SURVEY.md Appendix A.10)."""
        d = self.d
        H = d.n_heads
        saved: List[_Saved] = []
        last = d.n_layers - 1
        # fused-epilogue kernels (128 x 256-tile GEMM) need head_dim 128, F % 128 == 0 and at least one wave of tiles
        fused = self.fused_epilogues and x.shape[0] >= 1024 and d.inter % 128 == 0 and d.hidden % 256 == 0
        if kv_store is not None and kv_sink is None:                  # (kc list, vc list): post-RoPE K, V of every layer go to the caches
            B_, T_ = len(seqlens), x.shape[0]
            kv_sink = lambda l, qkv: ops.kv_store_prefill(qkv, cu, kv_store[0][l], kv_store[1][l], B_, T_)
        if self.LAYER_CALL and not save and not fused and d.head_dim == 128 and (kv_store is not None or kv_sink is None):
            return self._forward_layer_calls(x, pos, cu, seqlens, kv_store, out_rows), None
        for l, lyr in enumerate(self.model.layers):
            s = _Saved()
            s.x = x
            s.xn, s.rstd1 = ops.rmsnorm_fwd(x, lyr.input_layernorm.weight.data, d.rms_eps)
            if fused:
                s.qkv = ops.gemm_rope(s.xn, self.wqkv[l], pos, self.cos, self.sin, 2 * d.hidden)   # RoPE in the epilogue
            else:
                s.qkv = ops.gemm(s.xn, self.wqkv[l])
                ops.rope_(s.qkv, pos, self.cos, self.sin, 2 * H, d.head_dim)
            if kv_sink is not None:
                kv_sink(l, s.qkv)                      # prefill of generate(): post-RoPE K,V go to the cache
            s.ao, s.lse = ops.attn_fwd(s.qkv, cu, seqlens, H)
            s.rows = None
            ao, xin = s.ao, x
            if out_rows is not None and l == last:
                s.rows = out_rows
                ao = s.ao_r = ops.gather_rows(s.ao, out_rows)
                xin = ops.gather_rows(x, out_rows)
            s.xm = ops.gemm(ao, self.wo[l], addend=xin)
            s.xn2, s.rstd2 = ops.rmsnorm_fwd(s.xm, lyr.post_attention_layernorm.weight.data, d.rms_eps)
            if fused and s.rows is None:
                s.gu, s.h = ops.gemm_swiglu(s.xn2, self.wgu[l])                                    # SwiGLU in the epilogue
            else:
                s.gu = ops.gemm(s.xn2, self.wgu[l])
                s.h = ops.swiglu_fwd(s.gu)
            x = ops.gemm(s.h, self.wd[l], addend=s.xm)
            if save:
                saved.append(s)
        return x, ((saved, (pos, cu, list(seqlens))) if save else None)

    # -------------------------------------------------------------------------------------------------
    def forward_suffix(self, x: torch.Tensor, pos: torch.Tensor, cu: torch.Tensor, q_lens, kc: List[torch.Tensor],
                       vc: List[torch.Tensor], cached: torch.Tensor, kv_start: torch.Tensor, kv_len: torch.Tensor,
                       out_rows: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Inference-only forward of NEW rows on top of a per-layer KV cache that already holds an encoded prefix of
        every sequence (cross-step prefix reuse, SURVEY.md §8f n1).  x: [Tn, D] packed embeddings of the new tokens,
        pos: their rotary positions, cu / q_lens: packing of the new rows, caches [B, Smax, D] (zero-initialised),
        cached / kv_start / kv_len: int32 [B] on the device (rows already cached, first cache row of the sequence,
        cached + new).  The new rows' K/V are appended to the cache; returns the residual stream ([Tn, D], or
        [R, D] with ``out_rows``) before the final RMSNorm."""
        d = self.d
        H, D = d.n_heads, d.hidden
        B, T = len(q_lens), x.shape[0]
        last = d.n_layers - 1
        fused = self.fused_epilogues and T >= 1024 and d.inter % 128 == 0 and d.hidden % 256 == 0
        if self.LAYER_CALL and not fused and d.head_dim == 128:
            R = 0 if out_rows is None else out_rows.numel()
            run = ops.LayerRunner(T, D, d.inter, H, d.rms_eps, pos, self.cos, self.sin, cu, B, ops._qblocks(q_lens), R=R, device=x.device)
            run.set_cache_mode(2, kc[0].shape[1], kc[0].shape[0] * kc[0].shape[1], cached, kv_start, kv_len)
            bufs = [torch.empty_like(x), torch.empty_like(x)]
            for l, lyr in enumerate(self.model.layers):
                pruned = out_rows is not None and l == last
                y = torch.empty((R, D), dtype=bf16, device=x.device) if pruned else bufs[l & 1]
                run.run(x, y, lyr.input_layernorm.weight.data, self.wqkv[l], self.wo[l], lyr.post_attention_layernorm.weight.data,
                        self.wgu[l], self.wd[l], kc=kc[l], vc=vc[l], out_rows=out_rows if pruned else None)
                x = y
            return x
        for l, lyr in enumerate(self.model.layers):
            xn, _ = ops.rmsnorm_fwd(x, lyr.input_layernorm.weight.data, d.rms_eps)
            if fused:
                qkv = ops.gemm_rope(xn, self.wqkv[l], pos, self.cos, self.sin, 2 * D)
            else:
                qkv = ops.gemm(xn, self.wqkv[l])
                ops.rope_(qkv, pos, self.cos, self.sin, 2 * H, d.head_dim)
            ops.kv_store_suffix(qkv, cu, cached, kc[l], vc[l], B, T)
            ao = ops.attn_fwd_kv(qkv[:, :D], kc[l], vc[l], cu, q_lens, kv_start, kv_len, H)
            xin = x
            if out_rows is not None and l == last:
                ao = ops.gather_rows(ao, out_rows)
                xin = ops.gather_rows(x, out_rows)
            xm = ops.gemm(ao, self.wo[l], addend=xin)
            xn2, _ = ops.rmsnorm_fwd(xm, lyr.post_attention_layernorm.weight.data, d.rms_eps)
            if fused and xm.shape[0] >= 1024:
                _, h = ops.gemm_swiglu(xn2, self.wgu[l], keep_gu=False)
            else:
                h = ops.swiglu_fwd(ops.gemm(xn2, self.wgu[l]))
            x = ops.gemm(h, self.wd[l], addend=xm)
        return x

    # -------------------------------------------------------------------------------------------------
    def backward(self, dx: torch.Tensor, tape, layer_done=None) -> torch.Tensor:
        """dx: [T, D] bf16 gradient w.r.t. the forward's hidden output; ``tape`` from that forward (consumed).
        Accumulates every weight gradient in place (or OVERWRITES it when ``flat.overwrite_layer_grads`` is set
        by a lazy zero_grad: beta = 0 instead of zero-fill + read-modify-write) and returns the gradient w.r.t.
        the input embeddings.  ``layer_done(l)`` is called after layer l's gradients have been enqueued (used to
        overlap the data-parallel all-reduce with the rest of the backward)."""
        if tape is None:
            raise RuntimeError("LlamaCore.backward: the forward ran without saving activations (no_grad / eval-only)")
        saved, (pos, cu, seqlens) = tape
        d = self.d
        H = d.n_heads
        acc = not getattr(self.flat, "overwrite_layer_grads", False)

        def add(g):
            return g if acc else None

        # Weight-gradient GEMMs on a SIDE stream (NAVILLM_WGRAD_STREAM=1): nothing downstream in the backward reads a weight
        # gradient, so they can trail the dgrad chain: when one GEMM's last, partially filled wave of tiles leaves SMs idle, the
        # other stream's kernel takes them.
        side = WGRAD_STREAM and dx.shape[0] >= 1024
        main = torch.cuda.current_stream() if side else None
        ws = self._wgrad_stream() if side else None

        def wgrad(a, b, out, *, keep=()):
            if not side:
                ops.gemm(a, b, a_mn=True, b_mn=True, out=out, addend=add(out))
                return
            ev = torch.cuda.Event()
            ev.record(main)
            ws.wait_event(ev)
            for t in (a, b) + tuple(keep):
                t.record_stream(ws)                      # the caching allocator must not recycle them under the side stream
            with torch.cuda.stream(ws):
                ops.gemm(a, b, a_mn=True, b_mn=True, out=out, addend=add(out))

        for l in range(d.n_layers - 1, -1, -1):
            lyr, s = self.model.layers[l], saved[l]
            # ---- MLP:  x_out = xm + down(swiglu(gate_up(rmsnorm2(xm)))) ----
            if self.fused_epilogues and dx.shape[0] >= 1024 and d.inter % 32 == 0:
                dgu = ops.gemm_dswiglu(dx, self.wd[l], s.gu)                           # dgrad + SwiGLU' in the epilogue
            else:
                dh = ops.gemm(dx, self.wd[l], b_mn=True)                               # [T,F]  dgrad
                dgu = ops.swiglu_bwd(s.gu, dh)
                del dh
            wgrad(dx, s.h, self.gd[l])                                                 # dWd += dx^T h
            dxn2 = ops.gemm(dgu, self.wgu[l], b_mn=True)                               # [T,D]
            wgrad(dgu, s.xn2, self.ggu[l])
            del dgu
            dxm = ops.rmsnorm_bwd(s.xm, lyr.post_attention_layernorm.weight.data, s.rstd2, dxn2, dres=dx,
                                  dw=lyr.post_attention_layernorm.weight.grad, accumulate_dw=acc)
            del dxn2
            # ---- attention:  xm = x + o_proj(attn(rope(qkv(rmsnorm1(x))))) ----
            dvec = None
            if s.rows is None and self.fused_epilogues and dxm.shape[0] >= 1024 and d.head_dim == 128:
                dao, dvec = ops.gemm_attnd(dxm, self.wo[l], s.ao)      # dgrad + the attention backward's D in the epilogue
            else:
                dao = ops.gemm(dxm, self.wo[l], b_mn=True)
            if s.rows is None:
                wgrad(dxm, s.ao, self.go[l])
            else:
                # pruned last layer: everything above ran on the R requested rows; scatter back to [T, D]
                wgrad(dxm, s.ao_r, self.go[l])
                full = torch.zeros_like(s.ao)
                ops.scatter_rows_(dao, s.rows, full)
                dao = full
                full = torch.zeros_like(s.x)
                ops.scatter_rows_(dxm, s.rows, full)
                dxm = full
            # attention backward with the inverse rotary embedding of dq/dk fused into its epilogue
            dqkv = ops.attn_bwd(s.qkv, s.ao, dao, s.lse, cu, seqlens, H, rope=(pos, self.cos, self.sin), dvec=dvec)
            del dao
            dxn = ops.gemm(dqkv, self.wqkv[l], b_mn=True)
            wgrad(dqkv, s.xn, self.gqkv[l])
            del dqkv
            dx = ops.rmsnorm_bwd(s.x, lyr.input_layernorm.weight.data, s.rstd1, dxn, dres=dxm,
                                 dw=lyr.input_layernorm.weight.grad, accumulate_dw=acc)
            del dxn, dxm
            saved[l] = None
            if layer_done is not None:
                if side:                                   # the layer's gradients are complete only when the side stream is
                    ev = torch.cuda.Event()
                    ev.record(ws)
                    main.wait_event(ev)
                layer_done(l)
        if side:
            ev = torch.cuda.Event()
            ev.record(ws)
            main.wait_event(ev)                            # whoever reads the gradients next is ordered after the wgrads
        self.flat.overwrite_layer_grads = False
        return dx

    def _wgrad_stream(self):
        if getattr(self, "_ws", None) is None:
            self._ws = torch.cuda.Stream()
        return self._ws


    # -------------------------------------------------------------------------------------------------
    def decode_step(self, x: torch.Tensor, lens: torch.Tensor, kc: List[torch.Tensor], vc: List[torch.Tensor]) -> torch.Tensor:
        """One new token per sequence.  x: [B, D] bf16 embeddings of the new tokens; lens: int32 [B] (device) =
        number of cached tokens = position of the new token; caches [B, Smax, D] per layer.  Static shapes and
        device-resident lengths: the whole step can be captured in a CUDA graph.  Returns the residual stream
        [B, D] before the final RMSNorm."""
        d = self.d
        H, D = d.n_heads, d.hidden
        # The step is HBM-bound weight streaming.  Batches <= 16 use the swap-AB cluster-split-K kernel with the SwiGLU fused
        # (gemm_skinny.cu); larger batches go through nv_gemm_bf16's auto dispatch, which picks the tile variant per (M, N)
        # from a measured table (32-column tiles for the 4096-wide projections, 256 for gate|up: tools/midm_bench.py).
        bn = DECODE_BLOCK_N
        skinny = bn == 0 and x.shape[0] <= 16
        fuse_mlp = skinny and d.inter % 64 == 0
        if skinny:
            lin = lambda a, w, addend=None: ops.gemm_skinny(a, w, addend=addend)
        else:
            lin = lambda a, w, addend=None: ops.gemm(a, w, addend=addend, block_n=bn)
        for l, lyr in enumerate(self.model.layers):
            xn, _ = ops.rmsnorm_fwd(x, lyr.input_layernorm.weight.data, d.rms_eps)
            qkv = lin(xn, self.wqkv[l])
            if d.head_dim == 128:
                ao = ops.decode_attn_rope(qkv, lens, self.cos, self.sin, kc[l], vc[l], H)   # RoPE + cache append + attention
            else:
                ops.rope_(qkv, lens, self.cos, self.sin, 2 * H, d.head_dim)
                ops.kv_append(qkv, lens, kc[l], vc[l])
                ao = ops.decode_attn(qkv, kc[l], vc[l], lens, H)
            xm = lin(ao, self.wo[l], x)
            xn2, _ = ops.rmsnorm_fwd(xm, lyr.post_attention_layernorm.weight.data, d.rms_eps)
            if fuse_mlp:
                h = ops.gemm_skinny_swiglu(xn2, self.wgu[l])                            # gate|up projection + SwiGLU
            else:
                h = ops.swiglu_fwd(lin(xn2, self.wgu[l]))
            x = lin(h, self.wd[l], xm)
        return x
