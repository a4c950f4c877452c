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
from types import SimpleNamespace
from typing import List, Optional

import torch
import torch.nn as nn

from . import ops

# decode GEMMs: 0 (default) = swap-AB skinny kernel for batches <= 16 (csrc/gemm_skinny.cu), nv_gemm_bf16's measured tile
# table above that; 128 / 32 = force that column-tile width of the general kernel (A/B measurements)
DECODE_BLOCK_N = int(os.environ.get("NAVILLM_DECODE_BLOCK_N", "0"))
# Largest GEMM row count at which an inference GEMM above 16 rows streams the fp8 copy of its weight (Fp8Weights,
# nv_gemm_fp8w_bf16) instead of the bf16 weights.  Measured (tools/midm_bench.py --fp8, H100 80GB HBM3 at 700 W, fp8 vs bf16):
# qkv 1.04-1.10x and down 1.10x at M = 17..64, o_proj 0.95-1.03x; from M = 96 qkv is slower (0.96x), from M = 128 down (0.90x),
# and at M >= 192 every shape is (0.64-0.94x).  The fused gate|up weight (N = 2F) is slower at every M (0.90-0.95x up to 128),
# so it keeps its bf16 weight above 16 rows (_fp8_layer).  lm_head: 0.94x at 17, 0.99x at 32, 1.06x at 64.
FP8_MAX_ROWS = 64
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
        # bumped by writers that bypass torch's version counters (the fused AdamW of optim.py writes through raw pointers)
        self.generation = 0

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


class Fp8Weights:
    """e4m3 copy of linear weights of a ``FlatParams`` buffer for the inference GEMMs: the decode-step skinny GEMMs
    (csrc/gemm_skinny.cu) and, up to ``FP8_MAX_ROWS`` rows, nv_gemm_fp8w_bf16 (csrc/gemm_bf16.cu).

    Building it rounds every listed weight IN PLACE to W' = e4m3(W / 2^e_n) * 2^e_n (one power-of-two exponent per output
    row, csrc/quant.cu), so the bf16 buffer and the fp8 copy describe the same model.  The copy keeps the flat buffer's
    parameter order and 64-element alignment (non-listed parameters are skipped), so members that are adjacent there --
    q|k|v, gate|up -- are adjacent here too and the fused weights are plain views.  ``stale_reason`` reports any write to
    the weights since: a torch in-place op on a parameter or on the buffer (version counters), or a bump of
    ``FlatParams.generation`` by a raw-pointer writer."""

    def __init__(self, flat: FlatParams, params: List[nn.Parameter]):
        want = {id(p) for p in params}
        align = 64
        self.flat = flat
        self.params = [p for p in flat.params if id(p) in want]
        if len(self.params) != len(want):
            raise RuntimeError("Fp8Weights: every weight must live in the flat buffer")
        self._off, self._row, total, rows = {}, {}, 0, 0
        for p in self.params:
            if p.dim() != 2:
                raise RuntimeError(f"Fp8Weights: 2-D weights only, got {tuple(p.shape)}")
            self._off[id(p)], self._row[id(p)] = total, rows
            total += (p.numel() + align - 1) // align * align
            rows += p.shape[0]
        dev = flat.flat.device
        self.q = torch.empty(total, dtype=ops.fp8, device=dev)
        self.exps = torch.empty(rows, dtype=torch.int8, device=dev)
        for p in self.params:
            q, e = self.view([p], tuple(p.shape))
            ops.quantize_fp8_(p.data, q, e)
        self._versions = self._version_state()
        self._generation = flat.generation

    @property
    def nbytes(self) -> int:
        return self.q.numel() + self.exps.numel()

    def view(self, members, shape):
        """(e4m3 [N, K], int8 exponents [N]) of the weight formed by ``members`` stacked in order (``FlatParams.view``)."""
        o, r = self._off[id(members[0])], self._row[id(members[0])]
        end_o, end_r = o, r
        for m in members:
            if self._off.get(id(m)) != end_o or self._row[id(m)] != end_r:
                raise RuntimeError("Fp8Weights.view: the members are not adjacent, in order and unpadded")
            end_o += m.numel()
            end_r += m.shape[0]
        if end_o - o != shape[0] * shape[1] or end_r - r != shape[0]:
            raise RuntimeError(f"Fp8Weights.view: members hold {end_o - o} elements, shape {tuple(shape)} needs {shape[0] * shape[1]}")
        return self.q[o:end_o].view(shape), self.exps[r:end_r]

    def _version_state(self):
        return self.flat.flat._version, sum(p._version for p in self.params)

    def stale_reason(self, flat: FlatParams) -> Optional[str]:
        if flat is not self.flat or flat.params[0].data_ptr() != flat._ptr0:
            return "the weights were moved to new storage"
        if flat.generation != self._generation:
            return "an optimizer step updated the weights"
        if self._version_state() != self._versions:
            return "the weights were modified in place (optimizer step, load_state_dict or another write)"
        return None


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


def is_fp8_kv(caches) -> bool:
    """True for the per-layer list of an fp8 KV cache: ``(e4m3 [B, Smax, H*128], int8 exponents [B, Smax, H])`` pairs
    (include/navillm_b200.h); False for bf16 tensors [B, Smax, H*128]."""
    return isinstance(caches[0], tuple)


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
        self.fp8 = None
        self.fp8_src = None
        self.act_fp8 = False          # W8A8 in the no-grad forwards (ModifiedLlamaForCausalLM.set_activation_dtype)

    def set_fp8(self, fp8: Optional[Fp8Weights]) -> None:
        """Stream ``fp8``'s copy of the linear weights in the inference GEMMs (None: the bf16 weights): the decode step, and
        the no-grad forwards while the copy is fresh (``fp8_for_inference``)."""
        self.fp8 = None
        self.fp8_src = fp8
        if fp8 is None:
            return
        D, F = self.d.hidden, self.d.inter
        w = SimpleNamespace(wqkv=[], wo=[], wgu=[], wd=[])
        for lyr in self.model.layers:
            a, m = lyr.self_attn, lyr.mlp
            w.wqkv.append(fp8.view([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], (3 * D, D)))
            w.wo.append(fp8.view([a.o_proj.weight], (D, D)))
            w.wgu.append(fp8.view([m.gate_proj.weight, m.up_proj.weight], (2 * F, D)))
            w.wd.append(fp8.view([m.down_proj.weight], (D, F)))
        self.fp8 = w

    def fp8_for_inference(self):
        """The per-layer fp8 weight pairs when the copy still describes the current weights, else None.  The inference
        forwards (navigation, grounding, prefix-cached steps, prefill) then run bf16 on the current weights: a weight write
        after ``quantize_weights_fp8`` must not change what they compute, and must not make them fail either."""
        if self.fp8 is None or self.fp8_src.stale_reason(self.flat) is not None:
            return None
        return self.fp8

    def act_fp8_weights(self):
        """The per-layer fp8 weight pairs of the W8A8 GEMMs when ``act_fp8`` is on, None when it is off.  Raises rather than
        run bf16: one evaluation must not mix two numerics."""
        if not self.act_fp8:
            return None
        D, F = self.d.hidden, self.d.inter
        if D % 128 or F % 128:
            raise RuntimeError(f"activation dtype 'fp8': the W8A8 GEMMs need hidden and intermediate sizes that are multiples "
                               f"of 128 (got {D}, {F}); call set_activation_dtype('bf16')")
        if self.fp8 is None:
            raise RuntimeError("activation dtype 'fp8' needs the fp8 copy of the weights: call quantize_weights_fp8() first, "
                               "or set_activation_dtype('bf16')")
        why = self.fp8_src.stale_reason(self.flat)
        if why is not None:
            raise RuntimeError(f"activation dtype 'fp8': the fp8 copy of the weights is stale ({why} after "
                               f"quantize_weights_fp8()); call quantize_weights_fp8() again, or set_activation_dtype('bf16')")
        return self.fp8

    @staticmethod
    def _linear(a, w, wq, addend=None, w8a8=False):
        """a · w^T (+ addend): W8A8 on the fp8 pair ``wq`` when ``w8a8``; else from ``wq`` when it is given and a has at most
        FP8_MAX_ROWS rows."""
        if w8a8:
            return ops.gemm_w8a8(*ops.quantize_act_fp8(a), *wq, addend=addend)
        if wq[0] is not None and a.shape[0] <= FP8_MAX_ROWS:
            return ops.gemm_fp8w(a, *wq, addend=addend)
        return ops.gemm(a, w, addend=addend)

    def _fp8_layer(self, f8, l):
        """(qkv, o, gate|up, down) fp8 pairs of layer l for the GEMMs above 16 rows: gate|up stays bf16 (see FP8_MAX_ROWS)."""
        return None if f8 is None else (f8.wqkv[l], f8.wo[l], (None, None), f8.wd[l])

    @staticmethod
    def _w8a8_layer(a8, l):
        """(qkv, o, gate|up, down) fp8 pairs of layer l for the W8A8 GEMMs."""
        return a8.wqkv[l], a8.wo[l], a8.wgu[l], a8.wd[l]

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

    def _forward_layer_calls(self, x, pos, cu, seqlens, kv_store, out_rows, a8=None):
        d = self.d
        T = x.shape[0]
        R = 0 if out_rows is None else out_rows.numel()
        run = ops.LayerRunner(T, d.hidden, d.inter, d.n_heads, d.rms_eps, pos, self.cos, self.sin, cu, len(seqlens), ops._qblocks(seqlens),
                              R=R, device=x.device)
        fp8_kv = kv_store is not None and is_fp8_kv(kv_store[0])
        if kv_store is not None:
            run.set_cache_mode(3 if fp8_kv else 1, kv_store[0][0][0].shape[1] if fp8_kv else kv_store[0][0].shape[1])
        bufs = [torch.empty_like(x), torch.empty_like(x)]
        last = d.n_layers - 1
        f8 = self.fp8_for_inference()
        for l, lyr in enumerate(self.model.layers):
            pruned = out_rows is not None and l == last
            y = torch.empty((R, d.hidden), dtype=bf16, device=x.device) if pruned else bufs[l & 1]
            kc = vc = ke = ve = None
            if fp8_kv:
                (kc, ke), (vc, ve) = kv_store[0][l], kv_store[1][l]
            elif kv_store is not None:
                kc, vc = kv_store[0][l], kv_store[1][l]
            run.run(x, y, lyr.input_layernorm.weight.data, self.wqkv[l], self.wo[l], lyr.post_attention_layernorm.weight.data, self.wgu[l],
                    self.wd[l], kc=kc, vc=vc, ke=ke, ve=ve, out_rows=out_rows if pruned else None,
                    fp8=self._w8a8_layer(a8, l) if a8 is not None else self._fp8_layer(f8, l), fp8_max_rows=FP8_MAX_ROWS,
                    act_fp8=a8 is not None)
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
        value is [R, D].  The reference computes all positions and reads only these (SURVEY.md Appendix A.10).

        ``kv_store`` (prefill of generate): (kc, vc) per-layer caches, bf16 [B, Smax, D] or fp8 ``(e4m3 [B, Smax, D], int8
        exponents [B, Smax, H])`` pairs (``is_fp8_kv``); the prompt's own attention reads the unrounded K, V either way."""
        d = self.d
        H = d.n_heads
        saved: List[_Saved] = []
        last = d.n_layers - 1
        a8 = None if save else self.act_fp8_weights()       # W8A8 (set_activation_dtype("fp8")): no-grad forwards only
        # fused-epilogue kernels (128 x 256-tile GEMM) need head_dim 128, F % 128 == 0 and at least one wave of tiles; W8A8
        # runs the plain GEMM and the RoPE / SwiGLU row kernels instead
        fused = a8 is None and self.fused_epilogues and x.shape[0] >= 1024 and d.inter % 128 == 0 and d.hidden % 256 == 0
        if kv_store is not None and kv_sink is None:                  # (kc list, vc list): post-RoPE K, V of every layer go to the caches
            B_, T_ = len(seqlens), x.shape[0]
            if is_fp8_kv(kv_store[0]):                                # fp8 cache: (e4m3 bytes, exponents) per layer
                kv_sink = lambda l, qkv: ops.kv_store_prefill_fp8(qkv, cu, kv_store[0][l][0], kv_store[1][l][0], kv_store[0][l][1],
                                                                  kv_store[1][l][1], B_, T_)
            else:
                kv_sink = lambda l, qkv: ops.kv_store_prefill(qkv, cu, kv_store[0][l], kv_store[1][l], B_, T_)
        if self.LAYER_CALL and not save and not fused and d.head_dim == 128 and (kv_store is not None or kv_sink is None):
            return self._forward_layer_calls(x, pos, cu, seqlens, kv_store, out_rows, a8), None
        f8 = None if save else self.fp8_for_inference()     # training forwards never read the fp8 copy
        q8 = a8 is not None
        for l, lyr in enumerate(self.model.layers):
            w8 = self._w8a8_layer(a8, l) if q8 else (self._fp8_layer(f8, l) or ((None, None),) * 4)
            s = _Saved()
            s.x = x
            s.xn, s.rstd1 = ops.rmsnorm_fwd(x, lyr.input_layernorm.weight.data, d.rms_eps)
            if fused:
                s.qkv = ops.gemm_rope(s.xn, self.wqkv[l], pos, self.cos, self.sin, 2 * d.hidden)   # RoPE in the epilogue
            else:
                s.qkv = self._linear(s.xn, self.wqkv[l], w8[0], w8a8=q8)
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
            s.xm = self._linear(ao, self.wo[l], w8[1], addend=xin, w8a8=q8)
            s.xn2, s.rstd2 = ops.rmsnorm_fwd(s.xm, lyr.post_attention_layernorm.weight.data, d.rms_eps)
            if fused and s.rows is None:
                s.gu, s.h = ops.gemm_swiglu(s.xn2, self.wgu[l])                                    # SwiGLU in the epilogue
            else:
                s.gu = self._linear(s.xn2, self.wgu[l], w8[2], w8a8=q8)
                s.h = ops.swiglu_fwd(s.gu)
            x = self._linear(s.h, self.wd[l], w8[3], addend=s.xm, w8a8=q8)
            if save:
                saved.append(s)
        return x, ((saved, (pos, cu, list(seqlens))) if save else None)

    # -------------------------------------------------------------------------------------------------
    def forward_suffix(self, x: torch.Tensor, pos: torch.Tensor, cu: torch.Tensor, q_lens, kc: List[torch.Tensor],
                       vc: List[torch.Tensor], cached: torch.Tensor, kv_start: torch.Tensor, kv_len: torch.Tensor,
                       out_rows: Optional[torch.Tensor] = None, save: bool = False, acc: Optional[List[torch.Tensor]] = None,
                       kv_lens=None, store: bool = True):
        """Forward of NEW rows on top of a per-layer KV cache that already holds an encoded prefix of
        every sequence (cross-step prefix reuse, SURVEY.md §8f n1).  x: [Tn, D] packed embeddings of the new tokens,
        pos: their rotary positions, cu / q_lens: packing of the new rows, caches [B, Smax, D] (zero-initialised),
        cached / kv_start / kv_len: int32 [B] on the device (rows already cached, first cache row of the sequence,
        cached + new).  The new rows' K/V are appended to the cache; returns the residual stream ([Tn, D], or
        [R, D] with ``out_rows``) before the final RMSNorm.

        The caches may also be fp8 ``(e4m3 [B, Smax, D], int8 exponents [B, Smax, H])`` pairs per layer (``is_fp8_kv``): the
        new rows are rounded as they are stored and the attention reads the rounded rows, theirs included.

        ``save=True`` (training; bf16 caches only): returns ``(residual, tape)``; the tape makes ``backward`` run the cache
        form of the attention backward (``ops.attn_bwd_kv``), which adds the cached rows' dK / dV into ``acc`` (per layer,
        fp32 [B, Smax, 2 D]) and hands the suffix rows theirs.  ``kv_lens``: host copy of ``kv_len``.  Runs the per-kernel
        path on the bf16 weights (never the fp8 copy); the caches must still hold these K/V when ``backward`` runs.
        ``store=False`` (the prefix flush of ``PrefixKVCache``, which recomputes rows the cache already holds): the rows' own K/V
        are not written; the attention reads the cached ones.  The store writes packed sequence i to cache slot i, so only a
        batch covering the slots 0..B-1 in order may store."""
        d = self.d
        H, D = d.n_heads, d.hidden
        B, T = len(q_lens), x.shape[0]
        last = d.n_layers - 1
        a8 = None if save else self.act_fp8_weights()       # W8A8 (set_activation_dtype("fp8")): no-grad forwards only
        q8 = a8 is not None
        fused = not q8 and self.fused_epilogues and T >= 1024 and d.inter % 128 == 0 and d.hidden % 256 == 0
        f8 = None if save else self.fp8_for_inference()     # training forwards never read the fp8 copy
        fp8_kv = is_fp8_kv(kc)
        if save and (fp8_kv or acc is None or kv_lens is None):
            raise ValueError("forward_suffix(save=True) needs bf16 caches, the gradient accumulators and the host kv_lens")
        Bc, Smax = (kc[0][0] if fp8_kv else kc[0]).shape[:2]
        if self.LAYER_CALL and not fused and d.head_dim == 128 and not save:
            R = 0 if out_rows is None else out_rows.numel()
            run = ops.LayerRunner(T, D, d.inter, H, d.rms_eps, pos, self.cos, self.sin, cu, B, ops._qblocks(q_lens), R=R, device=x.device)
            run.set_cache_mode(4 if fp8_kv else 2, Smax, Bc * Smax, cached, kv_start, kv_len)
            bufs = [torch.empty_like(x), torch.empty_like(x)]
            for l, lyr in enumerate(self.model.layers):
                pruned = out_rows is not None and l == last
                y = torch.empty((R, D), dtype=bf16, device=x.device) if pruned else bufs[l & 1]
                (kl, ke), (vl, ve) = (kc[l], vc[l]) if fp8_kv else ((kc[l], None), (vc[l], None))
                run.run(x, y, lyr.input_layernorm.weight.data, self.wqkv[l], self.wo[l], lyr.post_attention_layernorm.weight.data,
                        self.wgu[l], self.wd[l], kc=kl, vc=vl, ke=ke, ve=ve, out_rows=out_rows if pruned else None,
                        fp8=self._w8a8_layer(a8, l) if q8 else self._fp8_layer(f8, l), fp8_max_rows=FP8_MAX_ROWS, act_fp8=q8)
                x = y
            return x
        saved: List[_Saved] = []
        for l, lyr in enumerate(self.model.layers):
            w8 = self._w8a8_layer(a8, l) if q8 else (self._fp8_layer(f8, l) or ((None, None),) * 4)
            s = _Saved()
            s.x = x
            xn, s.rstd1 = ops.rmsnorm_fwd(x, lyr.input_layernorm.weight.data, d.rms_eps)
            if fused:
                qkv = ops.gemm_rope(xn, self.wqkv[l], pos, self.cos, self.sin, 2 * D)
            else:
                qkv = self._linear(xn, self.wqkv[l], w8[0], w8a8=q8)
                ops.rope_(qkv, pos, self.cos, self.sin, 2 * H, d.head_dim)
            s.lse = torch.empty((H, T), dtype=torch.float32, device=x.device) if save else None
            if fp8_kv:
                (kq, ke), (vq, ve) = kc[l], vc[l]
                ops.kv_store_suffix_fp8(qkv, cu, cached, kq, vq, ke, ve, B, T)
                ao = ops.attn_fwd_kv_fp8(qkv[:, :D], kq, vq, ke, ve, cu, q_lens, kv_start, kv_len, H)
            else:
                if store:
                    ops.kv_store_suffix(qkv, cu, cached, kc[l], vc[l], B, T)
                ao = ops.attn_fwd_kv(qkv[:, :D], kc[l], vc[l], cu, q_lens, kv_start, kv_len, H, lse=s.lse)
            s.xn, s.qkv, s.ao, s.rows = xn, qkv, ao, None
            xin = x
            if out_rows is not None and l == last:
                s.rows = out_rows
                ao = s.ao_r = ops.gather_rows(ao, out_rows)
                xin = ops.gather_rows(x, out_rows)
            s.xm = xm = self._linear(ao, self.wo[l], w8[1], addend=xin, w8a8=q8)
            s.xn2, s.rstd2 = xn2, _ = ops.rmsnorm_fwd(xm, lyr.post_attention_layernorm.weight.data, d.rms_eps)
            if fused and xm.shape[0] >= 1024:
                s.gu, s.h = ops.gemm_swiglu(xn2, self.wgu[l], keep_gu=save)
            else:
                s.gu = self._linear(xn2, self.wgu[l], w8[2], w8a8=q8)
                s.h = ops.swiglu_fwd(s.gu)
            x = self._linear(s.h, self.wd[l], w8[3], addend=xm, w8a8=q8)
            if save:
                saved.append(s)
        if not save:
            return x
        kv = SimpleNamespace(kc=kc, vc=vc, acc=acc, kv_start=kv_start, kv_len=kv_len, kv_lens=list(kv_lens))
        return x, (saved, (pos, cu, list(q_lens)), kv)

    # -------------------------------------------------------------------------------------------------
    def backward(self, dx: torch.Tensor, tape, layer_done=None) -> torch.Tensor:
        """dx: [T, D] bf16 gradient w.r.t. the forward's hidden output; ``tape`` from that forward (consumed).
        Accumulates every weight gradient in place (or OVERWRITES it when ``flat.overwrite_layer_grads`` is set
        by a lazy zero_grad: beta = 0 instead of zero-fill + read-modify-write) and returns the gradient w.r.t.
        the input embeddings.  ``layer_done(l)`` is called after layer l's gradients have been enqueued (used to
        overlap the data-parallel all-reduce with the rest of the backward)."""
        if tape is None:
            raise RuntimeError("LlamaCore.backward: the forward ran without saving activations (no_grad / eval-only)")
        saved, (pos, cu, seqlens) = tape[:2]
        kv = tape[2] if len(tape) > 2 else None          # forward_suffix tape: attention over a KV cache
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
            if kv is None:
                dqkv = ops.attn_bwd(s.qkv, s.ao, dao, s.lse, cu, seqlens, H, rope=(pos, self.cos, self.sin), dvec=dvec)
            else:
                dqkv = ops.attn_bwd_kv(s.qkv, s.ao, dao, s.lse, kv.kc[l], kv.vc[l], kv.acc[l], cu, seqlens, kv.kv_start,
                                       kv.kv_len, kv.kv_lens, H, rope=(pos, self.cos, self.sin), dvec=dvec)
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
        number of cached tokens = position of the new token; caches [B, Smax, D] bf16 per layer, or fp8 ``(e4m3, exponents)``
        pairs per layer (``is_fp8_kv``; the new rows are rounded as they are appended).  Static shapes and
        device-resident lengths: the whole step can be captured in a CUDA graph.  Returns the residual stream
        [B, D] before the final RMSNorm."""
        d = self.d
        H, D = d.n_heads, d.hidden
        # The step is HBM-bound weight streaming.  Batches <= 16 use the swap-AB cluster-split-K kernel with the SwiGLU fused
        # (gemm_skinny.cu); larger batches go through nv_gemm_bf16's auto dispatch, which picks the tile variant per (M, N)
        # from a measured table (32-column tiles for the 4096-wide projections, 256 for gate|up: tools/midm_bench.py).
        # With an fp8 copy of the weights (set_fp8), the skinny GEMMs and, up to FP8_MAX_ROWS rows, nv_gemm_fp8w_bf16 stream
        # it instead: same bits as bf16 on W'.  generate() refuses a stale copy before it gets here.
        bn = DECODE_BLOCK_N
        skinny = bn == 0 and x.shape[0] <= 16
        fuse_mlp = skinny and d.inter % 64 == 0
        f8 = self.fp8 if bn == 0 and x.shape[0] <= FP8_MAX_ROWS else None
        if f8 is not None:
            if skinny:
                lin = lambda a, w, addend=None: ops.gemm_skinny_fp8(a, *w, addend=addend)
            else:
                lin = lambda a, w, addend=None: ops.gemm_fp8w(a, *w, addend=addend) if w[0] is not None else ops.gemm(a, w[1], addend=addend)
            wqkv, wo, wd = f8.wqkv, f8.wo, f8.wd
            wgu = f8.wgu if skinny else [(None, w) for w in self.wgu]        # gate|up: bf16 above 16 rows (FP8_MAX_ROWS)
        else:
            wqkv, wo, wgu, wd = self.wqkv, self.wo, self.wgu, self.wd
            if skinny:
                lin = lambda a, w, addend=None: ops.gemm_skinny(a, w, addend=addend)
            else:
                lin = lambda a, w, addend=None: ops.gemm(a, w, addend=addend, block_n=bn)
        fp8_kv = is_fp8_kv(kc)
        if fp8_kv and d.head_dim != 128:
            raise NotImplementedError("the fp8 KV cache is built for head_dim = 128")
        for l, lyr in enumerate(self.model.layers):
            xn, _ = ops.rmsnorm_fwd(x, lyr.input_layernorm.weight.data, d.rms_eps)
            qkv = lin(xn, wqkv[l])
            if fp8_kv:                                                                   # same, quantizing the appended rows
                ao = ops.decode_attn_rope_fp8(qkv, lens, self.cos, self.sin, kc[l][0], vc[l][0], kc[l][1], vc[l][1], H)
            elif d.head_dim == 128:
                ao = ops.decode_attn_rope(qkv, lens, self.cos, self.sin, kc[l], vc[l], H)   # RoPE + cache append + attention
            else:
                ops.rope_(qkv, lens, self.cos, self.sin, 2 * H, d.head_dim)
                ops.kv_append(qkv, lens, kc[l], vc[l])
                ao = ops.decode_attn(qkv, kc[l], vc[l], lens, H)
            xm = lin(ao, wo[l], x)
            xn2, _ = ops.rmsnorm_fwd(xm, lyr.post_attention_layernorm.weight.data, d.rms_eps)
            if fuse_mlp and f8 is not None:
                h = ops.gemm_skinny_swiglu_fp8(xn2, *wgu[l])
            elif fuse_mlp:
                h = ops.gemm_skinny_swiglu(xn2, wgu[l])                                 # gate|up projection + SwiGLU
            else:
                h = ops.swiglu_fwd(lin(xn2, wgu[l]))
            x = lin(h, wd[l], xm)
        return x
