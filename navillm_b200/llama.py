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

from dataclasses import dataclass
from types import SimpleNamespace
from typing import List, Optional

import torch
import torch.nn as nn

from . import ops

# Largest GEMM row count at which an inference GEMM above 16 rows streams the fp8 copy of its weight (Fp8Weights,
# nv_gemm_fp8w_bf16) instead of the bf16 weights.  Measured (tools/midm_bench.py --fp8, H100 80GB HBM3 at 700 W, fp8 vs bf16):
# qkv 1.04-1.10x and down 1.10x at M = 17..64, o_proj 0.95-1.03x; from M = 96 qkv is slower (0.96x), from M = 128 down (0.90x),
# and at M >= 192 every shape is (0.64-0.94x).  The fused gate|up weight (N = 2F) is slower at every M (0.90-0.95x up to 128),
# so it keeps its bf16 weight above 16 rows (_fp8_layer).  lm_head: 0.94x at 17, 0.99x at 32, 1.06x at 64.
FP8_MAX_ROWS = 64

# Largest GEMM row count at which the fused q|k|v projection of an inference GEMM of 17 or more rows streams the int4 copy
# of its weight (Int4Weights, nv_gemm_int4w_bf16) instead of the bf16 weights; at most 16 rows the decode step's skinny
# int4 kernels read all four.  Measured (tools/midm_bench.py --int4, H100 80GB HBM3 at 700 W, int4 at its best tile width
# vs bf16 on W', auto tiles): q|k|v 1.15x / 1.21x / 1.20x / 1.15x / 1.11x at M = 17 / 24 / 32 / 48 / 64 and 1.00x at 96 and
# 128.  The other three stay bf16 above 16 rows (_int4_layer): o_proj 0.79-0.98x and down_proj 0.71-0.91x at every M,
# gate|up 0.93-1.02x (1.02x at 17, 1.00x at 24-48, 0.98x at 64).  The expansion of the 4-bit tile, not HBM, limits the
# kernel: it reaches 0.2-0.65 TB/s on its bytes.
INT4_MAX_ROWS = 64

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

    def weight_state(self):
        """Changes with every write to the weights: new storage, a torch in-place op on the buffer or a parameter (version
        counters), or a raw-pointer writer's ``generation`` bump."""
        return self.flat.data_ptr(), self.flat._version, self.generation, sum(p._version for p in self.params)

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


class _WeightStamp:
    """Something derived from weights ``params`` of ``flat`` (a quantized copy, a calibration): ``stale_reason`` reports any
    write to the weights since ``_stamp``: new storage, a torch in-place op on a parameter or on the buffer (version
    counters), or a bump of ``FlatParams.generation`` by a raw-pointer writer."""

    def _stamp(self) -> None:
        self._versions = self._version_state()
        self._generation = self.flat.generation

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


class _WeightCopy(_WeightStamp):
    """Quantized copy of linear weights of a ``FlatParams`` buffer (``Fp8Weights``, ``Int4Weights``).

    Building it rounds every listed weight IN PLACE to the W' the copy encodes (``_quantize``), so the bf16 buffer and the
    copy describe the same model.  Each storage of the copy (``_sizes``: elements per weight) keeps the flat buffer's
    parameter order, non-listed parameters skipped, so members that are adjacent there -- q|k|v, gate|up -- are adjacent
    here too and the fused weights are plain views.  ``stale_reason`` reports any write to the weights since: a torch
    in-place op on a parameter or on the buffer (version counters), or a bump of ``FlatParams.generation`` by a raw-pointer
    writer."""
    _align = (1,)                                # per storage: element alignment of each weight's start

    def __init__(self, flat: FlatParams, params: List[nn.Parameter]):
        name = type(self).__name__
        want = {id(p) for p in params}
        self.flat = flat
        self.params = [p for p in flat.params if id(p) in want]
        if len(self.params) != len(want):
            raise RuntimeError(f"{name}: every weight must live in the flat buffer")
        self._off, totals = {}, [0] * len(self._align)
        for p in self.params:
            if p.dim() != 2:
                raise RuntimeError(f"{name}: 2-D weights only, got {tuple(p.shape)}")
            self._check(p)
            self._off[id(p)] = tuple(totals)
            totals = [t + (n + a - 1) // a * a for t, n, a in zip(totals, self._sizes(tuple(p.shape)), self._align)]
        self._storage = self._allocate(totals, flat.flat.device)
        flat.generation += 1                     # the rounding below writes the weights through raw pointers
        for p in self.params:
            self._quantize(p.data, self.view([p], tuple(p.shape)))
        self._stamp()

    def _check(self, p: nn.Parameter) -> None:
        pass

    @property
    def nbytes(self) -> int:
        return sum(t.numel() * t.element_size() for t in self._storage)

    def view(self, members, shape):
        """The copy's tensors of the weight formed by ``members`` stacked in order (``FlatParams.view``)."""
        name = type(self).__name__
        start = self._off[id(members[0])]
        end = list(start)
        for m in members:
            if self._off.get(id(m)) != tuple(end):
                raise RuntimeError(f"{name}.view: the members are not adjacent, in order and unpadded")
            end = [e + n for e, n in zip(end, self._sizes(tuple(m.shape)))]
        if [e - o for e, o in zip(end, start)] != list(self._sizes(tuple(shape))):
            raise RuntimeError(f"{name}.view: members hold {end[0] - start[0]} elements, shape {tuple(shape)} needs "
                               f"{self._sizes(tuple(shape))[0]}")
        return self._views([t[o:e] for t, o, e in zip(self._storage, start, end)], shape)


class Fp8Weights(_WeightCopy):
    """e4m3 copy of linear weights for the inference GEMMs: the decode-step skinny GEMMs (csrc/gemm_skinny.cu) and, up to
    ``FP8_MAX_ROWS`` rows, nv_gemm_fp8w_bf16 (csrc/gemm_bf16.cu).  W' = e4m3(W / 2^e_n) * 2^e_n with one power-of-two
    exponent per output row (csrc/quant.cu); ``view`` gives (e4m3 [N, K], int8 exponents [N])."""
    _align = (64, 1)

    @staticmethod
    def _sizes(shape):
        return shape[0] * shape[1], shape[0]

    @staticmethod
    def _allocate(totals, dev):
        return torch.empty(totals[0], dtype=ops.fp8, device=dev), torch.empty(totals[1], dtype=torch.int8, device=dev)

    @property
    def q(self) -> torch.Tensor:
        return self._storage[0]

    @property
    def exps(self) -> torch.Tensor:
        return self._storage[1]

    @staticmethod
    def _views(parts, shape):
        return parts[0].view(shape), parts[1]

    @staticmethod
    def _quantize(w, v):
        ops.quantize_fp8_(w, *v)


class Int4Weights(_WeightCopy):
    """4-bit group-wise copy (W4A16) of the decoder-layer linear weights for the decode-step skinny GEMMs
    (csrc/gemm_skinny.cu, at most 16 rows).  W' = bf16((q - z) * s) with one bf16 scale s and one 4-bit zero-point z per
    row and 128 columns (csrc/quant.cu, rule in include/navillm_b200.h); ``view`` gives (codes, scales [N, K / 128] bf16,
    zeros [N, K / 128] uint8) in the form ``ops.gemm_skinny_int4`` takes.  Every weight needs K % 128 == 0 and, so that the
    packed codes of q|k|v and gate|up concatenate, N % 64 == 0.

    ``calibration`` (an ``Int4Calibration`` of these weights, closed and fresh): the codes come from GPTQ
    (``ops.gptq_int4_``) instead of round to nearest, with the factor U of each (layer, input) computed once (``damp``) and
    reused by the weights that share the input (q, k, v; gate, up).  The copy is the same kind of object either way."""
    _align = (16, 1, 1)

    def __init__(self, flat: FlatParams, params: List[nn.Parameter], calibration: Optional["Int4Calibration"] = None,
                 damp: float = 0.01):
        self._cal, self._damp, self._u = calibration, damp, None
        try:
            super().__init__(flat, params)
        finally:
            self._cal = self._u = None           # keeps neither the Hessians nor a factor alive

    def _quantize(self, w, v):
        if self._cal is None:
            ops.quantize_int4_(w, *v)
            return
        key = self._cal.input_of(w)
        if self._u is None or self._u[0] != key:
            self._u = None
            self._u = (key, self._cal.factor(*key, damp=self._damp))
        ops.gptq_int4_(w, self._u[1], *v, damp=None)

    def _check(self, p):
        if p.shape[0] % 64 or p.shape[1] % ops.INT4_GROUP:
            raise RuntimeError(f"Int4Weights: weights [N, K] with N % 64 == 0 and K % {ops.INT4_GROUP} == 0 only, "
                               f"got {tuple(p.shape)}")

    @staticmethod
    def _sizes(shape):
        g = shape[0] * shape[1] // ops.INT4_GROUP
        return shape[0] * shape[1] // 2, g, g

    @staticmethod
    def _allocate(totals, dev):
        return (torch.zeros(totals[0], dtype=torch.uint8, device=dev), torch.empty(totals[1], dtype=bf16, device=dev),
                torch.empty(totals[2], dtype=torch.uint8, device=dev))

    @staticmethod
    def _views(parts, shape):
        n, k = shape
        return parts[0].view(n, k // 2), parts[1].view(n, k // ops.INT4_GROUP), parts[2].view(n, k // ops.INT4_GROUP)


class Int4Calibration(_WeightStamp):
    """Second-order statistics of the decoder-layer linear inputs for GPTQ (``ModifiedLlamaForCausalLM.int4_calibration``):
    per layer one fp32 H = X^T X per distinct input, ``INPUTS``: the q|k|v input (the first RMSNorm's output), the o_proj
    input (the attention output; in a pruned last layer its gathered rows), the gate|up input (the second RMSNorm's
    output) and the down_proj input (the SwiGLU output).  ``h[(layer, input)]`` and ``rows[(layer, input)]`` (rows added
    so far) are keyed by layer index and input name.

    While it is open (``LlamaCore.calibration``), every forward through ``LlamaCore.forward`` or ``forward_suffix`` adds
    its rows: prompt forwards, prefix-cached suffixes, the prefill of ``generate()``, training forwards.  The decode steps
    of ``generate()`` add nothing.  Packed rows are real tokens only, so padding never enters H.  Each product is the
    wgmma bf16 GEMM in its weight-gradient form with fp32 output (bf16 products are exact in fp32, the sums are fp32),
    added to H.  At Vicuna-7B widths H takes 32 x (3 x 4096^2 + 11008^2) x 4 B = 21.95 GB (``nbytes``)."""
    INPUTS = ("qkv", "o_proj", "gate_up", "down_proj")

    def __init__(self, core: "LlamaCore"):
        d, dev = core.d, core.flat.flat.device
        self.flat = core.flat
        self.params, self._input = [], {}
        for l, lyr in enumerate(core.model.layers):
            a, m = lyr.self_attn, lyr.mlp
            for i, ps in enumerate(((a.q_proj, a.k_proj, a.v_proj), (a.o_proj,), (m.gate_proj, m.up_proj), (m.down_proj,))):
                for p in ps:
                    self.params.append(p.weight)
                    self._input[p.weight.data_ptr()] = (l, self.INPUTS[i])
        width = dict(qkv=d.hidden, o_proj=d.hidden, gate_up=d.hidden, down_proj=d.inter)
        self.h = {(l, n): torch.zeros((width[n], width[n]), dtype=torch.float32, device=dev)
                  for l in range(d.n_layers) for n in self.INPUTS}
        self.rows = {k: 0 for k in self.h}
        self.open = True
        self._stamp()

    @property
    def nbytes(self) -> int:
        return sum(h.numel() * h.element_size() for h in self.h.values())

    def record(self, layer: int, name: str, x: torch.Tensor) -> None:
        """H[(layer, name)] += x^T x for the bf16 rows x [T, K]."""
        if x.shape[0] == 0:
            return
        self.h[(layer, name)].add_(ops.gemm(x, x, a_mn=True, b_mn=True, out_f32=True))
        self.rows[(layer, name)] += x.shape[0]

    def check(self, flat: FlatParams, damp: float = 0.01) -> None:
        """Raises unless the calibration can quantize the weights of ``flat`` as they are now, before any weight is written:
        a failing factorisation (``ops.CholeskyError``) leaves the weights and the calibration usable with a larger damp."""
        if self.open:
            raise RuntimeError("int4 calibration: the calibration is still open; leave its `with model.int4_calibration()` "
                               "block before quantize_weights_int4(calibration=...)")
        empty = [k for k, n in self.rows.items() if n == 0]
        if empty:
            raise RuntimeError(f"int4 calibration: no rows were recorded for layer {empty[0][0]}'s {empty[0][1]} input "
                               f"({len(empty)} of {len(self.rows)} inputs empty); run LM forwards (model(mode, batch)) "
                               f"inside the calibration block")
        why = self.stale_reason(flat)
        if why is not None:
            raise RuntimeError(f"int4 calibration: the calibration is stale ({why} after it was opened); open a new "
                               f"calibration on the current weights")
        for (l, name), h in self.h.items():
            ops.gptq_factor(h, damp, what=f"layer {l}'s {name} input Hessian", check_only=True)

    def input_of(self, w: torch.Tensor):
        """(layer, input name) of a decoder-layer linear weight."""
        return self._input[w.data_ptr()]

    def factor(self, layer: int, name: str, damp: float = 0.01) -> torch.Tensor:
        """``ops.gptq_factor`` of H[(layer, name)]."""
        return ops.gptq_factor(self.h[(layer, name)], damp, what=f"layer {layer}'s {name} input Hessian")


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


class WgradStash:
    """Deferred weight gradients of the decoder linears (q|k|v, o_proj, gate|up, down of every layer).

    While a ``LlamaCore`` holds one (``wgrad_stash``), its ``backward`` records the operand pair (dY, X) of each of those
    wgrad GEMMs instead of launching it -- references to the tape and gradient tensors, no copies -- and ``flush`` runs
    ONE segmented-contraction GEMM per weight (``ops.gemm_wgrad_seg``) with the current gradient as addend: the same sum
    as the per-backward path, rounded to bf16 once instead of once per backward, and one read-modify-write of the
    gradient buffer instead of one per backward.

    ``max_rows`` bounds the stash in backward rows (the tensors it keeps alive, ``nbytes``): a backward that would take it
    past the bound, or past ``ops.WGRAD_SEG_MAX`` backwards, flushes it first; a backward of more than ``max_rows / 2`` rows
    (one that could not share a flush with another of its size) runs its weight gradients at once.  A backward under a
    lazy zero (``flat.overwrite_layer_grads``) records that the linears' gradients are logically zero, so that their flush
    overwrites the stale values instead of adding to them.  A backward's pairs enter the stash only when it completes
    (``commit``): one that raises leaves the stash as it was.  The flush raises when the weights changed after the first
    recorded backward (the gradient belongs to the old weights)."""

    def __init__(self, core: "LlamaCore", max_rows: int):
        self.core = core
        self.max_rows = int(max_rows)
        self._staged = None            # (rows, acc, weight state, [(key, a, b)]) of the running backward
        self._clear()

    def _clear(self) -> None:
        self.pairs = {}                # (gradient attribute, layer) -> [(a, b), ...], one pair per recorded backward
        self.rows = 0                  # backward rows recorded since the last flush
        self.backwards = 0
        self.zero = False              # the linears' gradients are logically zero: the flush overwrites them
        self._weights = None

    @property
    def pending(self) -> bool:
        return self.backwards > 0

    @property
    def nbytes(self) -> int:
        """Device bytes of the distinct tensors the stash keeps alive."""
        seen = {}
        for prs in self.pairs.values():
            for a, b in prs:
                for t in (a, b):
                    st = t.untyped_storage()
                    seen[st.data_ptr()] = st.nbytes()
        return sum(seen.values())

    def begin(self, rows: int, acc: bool) -> bool:
        """A backward of ``rows`` rows starts (``acc``: it would add to the gradients).  Returns True when it defers."""
        self._staged = None                              # the pairs of a backward that raised are dropped here
        if rows > self.max_rows // 2:
            self.flush()
            return False
        if self.rows + rows > self.max_rows or self.backwards >= ops.WGRAD_SEG_MAX:
            self.flush()
        if self.backwards > 0 and not acc:
            raise RuntimeError("deferred weight gradients: a zero_grad() ran while backward rows were stashed")
        self._staged = (rows, acc, self.core.flat.weight_state(), [])
        return True

    def record(self, grad: str, layer: int, a: torch.Tensor, b: torch.Tensor) -> None:
        self._staged[3].append(((grad, layer), a, b))

    def commit(self) -> None:
        """The backward that ``begin`` deferred completed: its pairs join the stash."""
        rows, acc, weights, recs = self._staged
        self._staged = None
        if self.backwards == 0:
            self._weights, self.zero = weights, not acc
        for key, a, b in recs:
            self.pairs.setdefault(key, []).append((a, b))
        self.rows += rows
        self.backwards += 1

    def flush(self) -> None:
        """One segmented wgrad GEMM per stashed weight into its gradient; then the stash is empty.  A no-op when empty."""
        if not self.pending:
            return
        if self.core.flat.weight_state() != self._weights:
            raise RuntimeError("deferred weight gradients: the weights changed while backward rows were stashed (optimizer "
                               "step, load or another write); flush_weight_grads() must run before the weights change")
        for (grad, l), prs in self.pairs.items():
            g = getattr(self.core, grad)[l]
            ops.gemm_wgrad_seg(prs, g, addend=None if self.zero else g)
        self._clear()


class _Saved:
    __slots__ = ("x", "rstd1", "xn", "qkv", "ao", "lse", "xm", "rstd2", "xn2", "gu", "h", "rows", "ao_r")


def is_fp8_kv(caches) -> bool:
    """True for the per-layer list of an fp8 KV cache: ``(e4m3 [B, Smax, H*128], int8 exponents [B, Smax, H])`` pairs
    (include/navillm_b200.h); False for bf16 tensors [B, Smax, H*128]."""
    return isinstance(caches[0], tuple)


def kv_cache(d: LlamaDims, rows: int, length: int, dtype: str, device, zero: bool = False) -> list:
    """A per-layer KV cache of ``rows`` sequences of ``length`` positions: bf16 [rows, length, D] tensors, or for ``dtype``
    "fp8" the ``is_fp8_kv`` pairs.  ``zero``: zero-initialised, else uninitialised."""
    new = torch.zeros if zero else torch.empty
    if dtype == "fp8":
        return [(new((rows, length, d.hidden), dtype=ops.fp8, device=device),
                 new((rows, length, d.n_heads), dtype=torch.int8, device=device)) for _ in range(d.n_layers)]
    return [new((rows, length, d.hidden), dtype=bf16, device=device) for _ in range(d.n_layers)]


class LlamaCore:
    """Forward/backward driver of the decoder stack on packed rows.  Not an nn.Module: parameters live in
    ``LlamaModelParams`` (HF-named) and are accessed through fused views of a ``FlatParams`` buffer."""

    def __init__(self, dims: LlamaDims, model: LlamaModelParams, flat: FlatParams):
        if dims.head_dim != 128:
            raise ValueError(f"LlamaCore: the attention kernels are built for head_dim 128 (got {dims.head_dim})")
        self.d = dims
        self.model = model
        self.flat = flat
        D, F = dims.hidden, dims.inter
        self.wqkv, self.wo, self.wgu, self.wd = [], [], [], []
        for lyr in model.layers:
            a, m = lyr.self_attn, lyr.mlp
            self.wqkv.append(flat.view([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], (3 * D, D)))
            self.wo.append(a.o_proj.weight.data)
            self.wgu.append(flat.view([m.gate_proj.weight, m.up_proj.weight], (2 * F, D)))
            self.wd.append(m.down_proj.weight.data)
        self.refresh_grad_views()
        self.cos, self.sin = rope_tables(dims, flat.flat.device)
        self.fp8 = None
        self.fp8_src = None
        self.int4 = None              # per-layer int4 weight triples (set_int4)
        self.int4_src = None
        self.act_fp8 = False          # W8A8 in the no-grad forwards (ModifiedLlamaForCausalLM.set_activation_dtype)
        self.batch_invariant = False  # ModifiedLlamaForCausalLM.set_batch_invariant
        self.wgrad_stash: Optional[WgradStash] = None   # deferred linear weight gradients (defer_weight_grads)
        self.calibration: Optional[Int4Calibration] = None   # open GPTQ calibration: the forwards record their linear inputs

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

    def set_int4(self, int4: Optional[Int4Weights]) -> None:
        """Stream ``int4``'s copy of the decoder-layer linear weights in the inference GEMMs (None: the bf16 weights): the
        decode step's GEMMs of at most 16 rows, and the q|k|v projections of 17..``INT4_MAX_ROWS`` rows in the decode step
        and, while the copy is fresh (``int4_for_inference``), in the no-grad forwards.  lm_head and training run bf16 on
        W'."""
        self.int4 = None
        self.int4_src = int4
        if int4 is None:
            return
        D, F = self.d.hidden, self.d.inter
        w = SimpleNamespace(wqkv=[], wo=[], wgu=[], wd=[])
        for lyr in self.model.layers:
            a, m = lyr.self_attn, lyr.mlp
            w.wqkv.append(int4.view([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], (3 * D, D)))
            w.wo.append(int4.view([a.o_proj.weight], (D, D)))
            w.wgu.append(int4.view([m.gate_proj.weight, m.up_proj.weight], (2 * F, D)))
            w.wd.append(int4.view([m.down_proj.weight], (D, F)))
        self.int4 = w

    def fp8_for_inference(self):
        """The per-layer fp8 weight pairs when the copy still describes the current weights, else None.  The inference
        forwards (navigation, grounding, prefix-cached steps, prefill) then run bf16 on the current weights: a weight write
        after ``quantize_weights_fp8`` must not change what they compute, and must not make them fail either."""
        if self.fp8 is None or self.fp8_src.stale_reason(self.flat) is not None:
            return None
        return self.fp8

    def int4_for_inference(self):
        """The per-layer int4 weight triples when the copy still describes the current weights, else None: as
        ``fp8_for_inference``, the no-grad forwards then run bf16 on the current weights."""
        if self.int4 is None or self.int4_src.stale_reason(self.flat) is not None:
            return None
        return self.int4

    @staticmethod
    def _int4_layer(q4, l):
        """(qkv, o, gate|up, down) int4 triples of layer l for the GEMMs of 17..INT4_MAX_ROWS rows: only q|k|v streams the
        copy (see INT4_MAX_ROWS)."""
        return None if q4 is None else (q4.wqkv[l], None, None, None)

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
    def _linear(a, w, wq, addend=None, w8a8=False, w4=None):
        """a · w^T (+ addend): W8A8 on the fp8 pair ``wq`` when ``w8a8``; else from ``wq`` when it is given and a has at most
        FP8_MAX_ROWS rows; else from the int4 triple ``w4`` when it is given and a has 17..INT4_MAX_ROWS rows."""
        if w8a8:
            return ops.gemm_w8a8(*ops.quantize_act_fp8(a), *wq, addend=addend)
        if wq[0] is not None and a.shape[0] <= FP8_MAX_ROWS:
            return ops.gemm_fp8w(a, *wq, addend=addend)
        if w4 is not None and 16 < a.shape[0] <= INT4_MAX_ROWS:
            return ops.gemm_int4w(a, *w4, addend=addend)
        return ops.gemm(a, w, addend=addend)

    def _fp8_layer(self, f8, l):
        """(qkv, o, gate|up, down) fp8 pairs of layer l for the GEMMs above 16 rows: gate|up stays bf16 (see FP8_MAX_ROWS)."""
        return None if f8 is None else (f8.wqkv[l], f8.wo[l], (None, None), f8.wd[l])

    @staticmethod
    def _w8a8_layer(a8, l):
        """(qkv, o, gate|up, down) fp8 pairs of layer l for the W8A8 GEMMs."""
        return a8.wqkv[l], a8.wo[l], a8.wgu[l], a8.wd[l]

    def refresh_grad_views(self) -> None:
        """(Re-)derive the fused gradient views, e.g. after ``FlatParams.rebind_grads``."""
        D, F = self.d.hidden, self.d.inter
        flat = self.flat
        self.gqkv, self.go, self.ggu, self.gd = [], [], [], []
        for lyr in self.model.layers:
            a, m = lyr.self_attn, lyr.mlp
            self.gqkv.append(flat.grad_view([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], (3 * D, D)))
            self.go.append(a.o_proj.weight.grad)
            self.ggu.append(flat.grad_view([m.gate_proj.weight, m.up_proj.weight], (2 * F, D)))
            self.gd.append(m.down_proj.weight.grad)

    # -------------------------------------------------------------------------------------------------
    # Inference forwards that do not run the fused-epilogue GEMMs go through ONE C-ABI call per layer (csrc/layer.cu): they
    # are host-bound when every kernel is its own call from Python.  Tests turn this off to run the per-kernel path as the
    # reference.  An open calibration also takes the per-kernel path: the layer call keeps the linear inputs it records in
    # its workspace.
    LAYER_CALL = True

    def _fused(self, T: int, a8, save: bool = True) -> bool:
        """Whether a forward of T rows runs the fused-epilogue kernels (RoPE / SwiGLU in the 128 x 256-tile GEMM's epilogue).
        They need F % 128 == 0, D % 256 == 0 and at least one wave of tiles; W8A8 runs the plain GEMM and the RoPE / SwiGLU
        row kernels instead.  So does a no-grad forward (``save`` False) in batch-invariant mode, at every T: one form of
        the layer whatever the batch."""
        d = self.d
        if self.batch_invariant and not save:
            return False
        return a8 is None and T >= 1024 and d.inter % 128 == 0 and d.hidden % 256 == 0

    def _layer_calls(self, x, pos, cu, seqlens, out_rows, a8, kc, vc, mode, Smax, Tkv=0, cached=None, kv_start=None,
                     kv_len=None):
        """The inference forward of every layer through ``ops.LayerRunner``.  ``mode`` .. ``kv_len``: the cache mode of
        ``LayerRunner.set_cache_mode`` (0: no cache, 1 / 3: prompt store, 2 / 4: suffix over the cache; 3 / 4 fp8) with the
        per-layer caches ``kc`` / ``vc``."""
        d = self.d
        R = 0 if out_rows is None else out_rows.numel()
        run = ops.LayerRunner(x.shape[0], d.hidden, d.inter, d.n_heads, d.rms_eps, pos, self.cos, self.sin, cu, len(seqlens),
                              ops._qblocks(seqlens), R=R, device=x.device)
        run.set_cache_mode(mode, Smax, Tkv, cached, kv_start, kv_len)
        bufs = [torch.empty_like(x), torch.empty_like(x)]
        last = d.n_layers - 1
        f8 = self.fp8_for_inference()
        q4 = self.int4_for_inference()
        for l, lyr in enumerate(self.model.layers):
            pruned = out_rows is not None and l == last
            y = torch.empty((R, d.hidden), dtype=bf16, device=x.device) if pruned else bufs[l & 1]
            k = v = ke = ve = None
            if mode in (3, 4):
                (k, ke), (v, ve) = kc[l], vc[l]
            elif mode:
                k, v = kc[l], vc[l]
            run.run(x, y, lyr.input_layernorm.weight.data, self.wqkv[l], self.wo[l], lyr.post_attention_layernorm.weight.data,
                    self.wgu[l], self.wd[l], kc=k, vc=v, ke=ke, ve=ve, out_rows=out_rows if pruned else None,
                    fp8=self._w8a8_layer(a8, l) if a8 is not None else self._fp8_layer(f8, l), fp8_max_rows=FP8_MAX_ROWS,
                    act_fp8=a8 is not None, int4=self._int4_layer(q4, l), int4_max_rows=INT4_MAX_ROWS)
            x = y
        return x

    def _layers(self, x, pos, out_rows, save, a8, fused, attend):
        """The per-kernel forward of every layer.  ``attend(l, qkv, s)`` is the attention step, the one part the prompt and
        the suffix forwards do differently: it returns the attention output of layer l and sets ``s.lse`` when saving.
        Returns the residual stream and the per-layer activations (empty unless ``save``).  With an open ``calibration``,
        each layer's four linear inputs are added to its Hessians."""
        d = self.d
        cal = self.calibration
        saved: List[_Saved] = []
        last = d.n_layers - 1
        f8 = None if save else self.fp8_for_inference()     # training forwards never read the fp8 or int4 copy
        q4 = None if save else self.int4_for_inference()
        q8 = a8 is not None
        for l, lyr in enumerate(self.model.layers):
            w8 = self._w8a8_layer(a8, l) if q8 else (self._fp8_layer(f8, l) or ((None, None),) * 4)
            w4 = self._int4_layer(q4, l) or (None,) * 4
            s = _Saved()
            s.x = x
            s.xn, s.rstd1 = ops.rmsnorm_fwd(x, lyr.input_layernorm.weight.data, d.rms_eps)
            if fused:
                s.qkv = ops.gemm_rope(s.xn, self.wqkv[l], pos, self.cos, self.sin, 2 * d.hidden)   # RoPE in the epilogue
            else:
                s.qkv = self._linear(s.xn, self.wqkv[l], w8[0], w8a8=q8, w4=w4[0])
                ops.rope_(s.qkv, pos, self.cos, self.sin, 2 * d.n_heads, d.head_dim)
            s.ao = attend(l, s.qkv, s)
            s.rows = None
            ao, xin = s.ao, x
            if out_rows is not None and l == last:
                s.rows = out_rows
                ao = s.ao_r = ops.gather_rows(s.ao, out_rows)
                xin = ops.gather_rows(x, out_rows)
            s.xm = self._linear(ao, self.wo[l], w8[1], addend=xin, w8a8=q8, w4=w4[1])
            s.xn2, s.rstd2 = ops.rmsnorm_fwd(s.xm, lyr.post_attention_layernorm.weight.data, d.rms_eps)
            if fused and s.rows is None:
                s.gu, s.h = ops.gemm_swiglu(s.xn2, self.wgu[l], keep_gu=save)                      # SwiGLU in the epilogue
            else:
                s.gu = self._linear(s.xn2, self.wgu[l], w8[2], w8a8=q8, w4=w4[2])
                s.h = ops.swiglu_fwd(s.gu)
            if cal is not None:
                for name, inp in zip(cal.INPUTS, (s.xn, ao, s.xn2, s.h)):
                    cal.record(l, name, inp)
            x = self._linear(s.h, self.wd[l], w8[3], addend=s.xm, w8a8=q8, w4=w4[3])
            if save:
                saved.append(s)
        return x, saved

    def forward(self, x: torch.Tensor, pos: torch.Tensor, cu: torch.Tensor, seqlens, save: bool = True,
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
        B, T, H = len(seqlens), x.shape[0], self.d.n_heads
        a8 = None if save else self.act_fp8_weights()       # W8A8 (set_activation_dtype("fp8")): no-grad forwards only
        fused = self._fused(T, a8, save)
        kc, vc = kv_store if kv_store is not None else (None, None)
        fp8_kv = kc is not None and is_fp8_kv(kc)
        if self.LAYER_CALL and not save and not fused and self.calibration is None:
            mode = 0 if kc is None else 3 if fp8_kv else 1
            Smax = 0 if kc is None else (kc[0][0] if fp8_kv else kc[0]).shape[1]
            return self._layer_calls(x, pos, cu, seqlens, out_rows, a8, kc, vc, mode, Smax), None

        def attend(l, qkv, s):
            if fp8_kv:                                       # prefill of generate(): post-RoPE K, V go to the cache
                ops.kv_store_prefill_fp8(qkv, cu, kc[l][0], vc[l][0], kc[l][1], vc[l][1], B, T)
            elif kc is not None:
                ops.kv_store_prefill(qkv, cu, kc[l], vc[l], B, T)
            ao, s.lse = ops.attn_fwd(qkv, cu, seqlens, H)
            return ao
        x, saved = self._layers(x, pos, out_rows, save, a8, fused, attend)
        return x, ((saved, (pos, cu, list(seqlens)), None) if save else None)

    # -------------------------------------------------------------------------------------------------
    def forward_suffix(self, x: torch.Tensor, pos: torch.Tensor, cu: torch.Tensor, q_lens, kc: List[torch.Tensor],
                       vc: List[torch.Tensor], cached: torch.Tensor, kv_start: torch.Tensor, kv_len: torch.Tensor,
                       out_rows: Optional[torch.Tensor] = None, save: bool = False, acc: Optional[List[torch.Tensor]] = None,
                       kv_lens=None, store: bool = True, tree_end: Optional[torch.Tensor] = None):
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
        batch covering the slots 0..B-1 in order may store.

        ``tree_end`` (int32 [q_len] on the device, answer scoring): the q_len new rows of every sequence are the nodes of one
        tree in DFS preorder (``trie.tree_rows``), and a row attends to the cached rows and to its ancestors and itself only
        (``ops.attn_fwd_tree`` / ``ops.attn_fwd_tree_fp8``).  The rows' K/V are stored as without it; the call runs the
        per-kernel path (inference only)."""
        d = self.d
        H, D = d.n_heads, d.hidden
        B, T = len(q_lens), x.shape[0]
        a8 = None if save else self.act_fp8_weights()       # W8A8 (set_activation_dtype("fp8")): no-grad forwards only
        fused = self._fused(T, a8, save)
        fp8_kv = is_fp8_kv(kc)
        if save and (fp8_kv or acc is None or kv_lens is None):
            raise ValueError("forward_suffix(save=True) needs bf16 caches, the gradient accumulators and the host kv_lens")
        tree = tree_end is not None
        if tree and (save or not store):
            raise ValueError("forward_suffix(tree_end=...) is an inference forward that stores its rows (save=False, store=True)")
        if self.LAYER_CALL and not save and not fused and self.calibration is None and not tree:
            Bc, Smax = (kc[0][0] if fp8_kv else kc[0]).shape[:2]
            return self._layer_calls(x, pos, cu, q_lens, out_rows, a8, kc, vc, 4 if fp8_kv else 2, Smax, Bc * Smax, cached,
                                     kv_start, kv_len)

        def attend(l, qkv, s):
            if fp8_kv:
                (kq, ke), (vq, ve) = kc[l], vc[l]
                ops.kv_store_suffix_fp8(qkv, cu, cached, kq, vq, ke, ve, B, T)
                if tree:
                    return ops.attn_fwd_tree_fp8(qkv[:, :D], kq, vq, ke, ve, cu, q_lens, kv_start, kv_len, tree_end, H)
                return ops.attn_fwd_kv_fp8(qkv[:, :D], kq, vq, ke, ve, cu, q_lens, kv_start, kv_len, H)
            if store:
                ops.kv_store_suffix(qkv, cu, cached, kc[l], vc[l], B, T)
            if tree:
                s.lse = None
                return ops.attn_fwd_tree(qkv[:, :D], kc[l], vc[l], cu, q_lens, kv_start, kv_len, tree_end, H)
            s.lse = torch.empty((H, T), dtype=torch.float32, device=x.device) if save else None
            return ops.attn_fwd_kv(qkv[:, :D], kc[l], vc[l], cu, q_lens, kv_start, kv_len, H, lse=s.lse)
        x, saved = self._layers(x, pos, out_rows, save, a8, fused, attend)
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
        saved, (pos, cu, seqlens), kv = tape          # kv: the cache of a forward_suffix tape, None for a prompt forward
        d = self.d
        H = d.n_heads
        acc = not getattr(self.flat, "overwrite_layer_grads", False)
        # deferred weight gradients (WgradStash): the four linears' wgrad operands are recorded, not launched
        defer = self.wgrad_stash is not None and self.wgrad_stash.begin(saved[0].x.shape[0], acc)   # the backward's rows

        def wgrad(a, b, grad, l):
            out = getattr(self, grad)[l]
            if defer:
                self.wgrad_stash.record(grad, l, a, b)
            else:
                ops.gemm(a, b, a_mn=True, b_mn=True, out=out, addend=out if acc else None)

        for l in range(d.n_layers - 1, -1, -1):
            lyr, s = self.model.layers[l], saved[l]
            # ---- MLP:  x_out = xm + down(swiglu(gate_up(rmsnorm2(xm)))) ----
            if dx.shape[0] >= 1024 and d.inter % 32 == 0:
                dgu = ops.gemm_dswiglu(dx, self.wd[l], s.gu)                           # dgrad + SwiGLU' in the epilogue
            else:
                dh = ops.gemm(dx, self.wd[l], b_mn=True)                               # [T,F]  dgrad
                dgu = ops.swiglu_bwd(s.gu, dh)
                del dh
            wgrad(dx, s.h, "gd", l)                                                 # dWd += dx^T h
            dxn2 = ops.gemm(dgu, self.wgu[l], b_mn=True)                               # [T,D]
            wgrad(dgu, s.xn2, "ggu", l)
            del dgu
            dxm = ops.rmsnorm_bwd(s.xm, lyr.post_attention_layernorm.weight.data, s.rstd2, dxn2, dres=dx,
                                  dw=lyr.post_attention_layernorm.weight.grad, accumulate_dw=acc)
            del dxn2
            # ---- attention:  xm = x + o_proj(attn(rope(qkv(rmsnorm1(x))))) ----
            dvec = None
            if s.rows is None and dxm.shape[0] >= 1024:
                dao, dvec = ops.gemm_attnd(dxm, self.wo[l], s.ao)      # dgrad + the attention backward's D in the epilogue
            else:
                dao = ops.gemm(dxm, self.wo[l], b_mn=True)
            if s.rows is None:
                wgrad(dxm, s.ao, "go", l)
            else:
                # pruned last layer: everything above ran on the R requested rows; scatter back to [T, D]
                wgrad(dxm, s.ao_r, "go", l)
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
            wgrad(dqkv, s.xn, "gqkv", l)
            del dqkv
            dx = ops.rmsnorm_bwd(s.x, lyr.input_layernorm.weight.data, s.rstd1, dxn, dres=dxm,
                                 dw=lyr.input_layernorm.weight.grad, accumulate_dw=acc)
            del dxn, dxm
            saved[l] = None
            if layer_done is not None:
                layer_done(l)
        if defer:
            self.wgrad_stash.commit()
        self.flat.overwrite_layer_grads = False
        return dx

    # -------------------------------------------------------------------------------------------------
    def decode_step(self, x: torch.Tensor, lens: torch.Tensor, kc: List[torch.Tensor], vc: List[torch.Tensor], beam=None,
                    window: int = 1) -> torch.Tensor:
        """One new token per sequence.  x: [B, D] bf16 embeddings of the new tokens; lens: int32 [B] (device) =
        number of cached tokens = position of the new token; caches [B, Smax, D] bf16 per layer, or fp8 ``(e4m3, exponents)``
        pairs per layer (``is_fp8_kv``; the new rows are rounded as they are appended).  Static shapes and
        device-resident lengths: the whole step can be captured in a CUDA graph.  Returns the residual stream
        [B, D] before the final RMSNorm.

        ``beam`` (beam search): the B rows are beams, ``beam.K`` per prompt; kc / vc hold only the generated keys [B, G, D]
        (addressed through ``beam.src``) and ``beam.pk`` / ``beam.pv`` the per-layer prompt caches [B / K, Sp, D] with
        ``beam.plens`` keys per prompt (``ops.decode_attn_rope_beam``).

        ``window`` = w > 1 (the verify step of prompt-lookup decoding): x holds w consecutive tokens per sequence, row b * w + r
        at position lens[b] + r (lens stays [B]); the attention is ``ops.decode_attn_rope_window``, everything else the same
        loop over B * w rows."""
        d = self.d
        H, D = d.n_heads, d.hidden
        # The step is HBM-bound weight streaming.  Batches <= 16 use the swap-AB cluster-split-K kernel with the SwiGLU fused
        # (gemm_skinny.cu); larger batches go through nv_gemm_bf16's auto dispatch, which picks the tile variant per (M, N)
        # from a measured table (32-column tiles for the 4096-wide projections, 256 for gate|up: tools/midm_bench.py).
        # With an fp8 copy of the weights (set_fp8), the skinny GEMMs and, up to FP8_MAX_ROWS rows, nv_gemm_fp8w_bf16 stream
        # it instead: same bits as bf16 on W'.  With an int4 copy (set_int4), the skinny GEMMs stream it, and up to
        # INT4_MAX_ROWS rows nv_gemm_int4w_bf16 does for q|k|v; again the same bits.  generate() refuses a stale copy before it gets here.
        # Batch-invariant mode (set_batch_invariant) streams every weight through nv_gemm_bi_bf16 at every batch size: one
        # accumulation chain per element, no split-K, the SwiGLU fused (gemm_bi.cu).
        inv = self.batch_invariant
        skinny = x.shape[0] <= 16 and not inv
        fuse_mlp = skinny and d.inter % 64 == 0
        f8 = self.fp8 if x.shape[0] <= FP8_MAX_ROWS and not inv else None
        q4 = self.int4 if x.shape[0] <= INT4_MAX_ROWS and not inv else None
        if inv:
            wqkv, wo, wgu, wd = self.wqkv, self.wo, self.wgu, self.wd
            lin = lambda a, w, addend=None: ops.gemm_bi(a, w, addend=addend)
        elif q4 is not None and skinny:
            lin = lambda a, w, addend=None: ops.gemm_skinny_int4(a, *w, addend=addend)
            wqkv, wo, wgu, wd = q4.wqkv, q4.wo, q4.wgu, q4.wd
        elif q4 is not None:                                  # q|k|v from the int4 copy, the others bf16 (INT4_MAX_ROWS)
            lin = lambda a, w, addend=None: ops.gemm(a, w, addend=addend) if torch.is_tensor(w) else ops.gemm_int4w(a, *w, addend=addend)
            wqkv, wo, wgu, wd = q4.wqkv, self.wo, self.wgu, self.wd
        elif f8 is not None:
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
                lin = lambda a, w, addend=None: ops.gemm(a, w, addend=addend)
        fp8_kv = is_fp8_kv(kc)
        for l, lyr in enumerate(self.model.layers):
            xn, _ = ops.rmsnorm_fwd(x, lyr.input_layernorm.weight.data, d.rms_eps)
            qkv = lin(xn, wqkv[l])
            if beam is not None and fp8_kv:
                ao = ops.decode_attn_rope_beam_fp8(qkv, lens, self.cos, self.sin, beam.pk[l][0], beam.pv[l][0], beam.pk[l][1],
                                                   beam.pv[l][1], beam.plens, kc[l][0], vc[l][0], kc[l][1], vc[l][1], beam.src, beam.K, H)
            elif beam is not None:
                ao = ops.decode_attn_rope_beam(qkv, lens, self.cos, self.sin, beam.pk[l], beam.pv[l], beam.plens, kc[l], vc[l],
                                               beam.src, beam.K, H)
            elif window > 1 and fp8_kv:
                ao = ops.decode_attn_rope_window_fp8(qkv, lens, self.cos, self.sin, kc[l][0], vc[l][0], kc[l][1], vc[l][1], H, window)
            elif window > 1:
                ao = ops.decode_attn_rope_window(qkv, lens, self.cos, self.sin, kc[l], vc[l], H, window)
            elif fp8_kv:                                                                 # same, quantizing the appended rows
                ao = ops.decode_attn_rope_fp8(qkv, lens, self.cos, self.sin, kc[l][0], vc[l][0], kc[l][1], vc[l][1], H)
            else:
                ao = ops.decode_attn_rope(qkv, lens, self.cos, self.sin, kc[l], vc[l], H)   # RoPE + cache append + attention
            xm = lin(ao, wo[l], x)
            xn2, _ = ops.rmsnorm_fwd(xm, lyr.post_attention_layernorm.weight.data, d.rms_eps)
            if inv:
                h = ops.gemm_bi_swiglu(xn2, wgu[l])
            elif q4 is not None and skinny:                                              # Int4Weights: F % 64 == 0
                h = ops.gemm_skinny_swiglu_int4(xn2, *wgu[l])
            elif fuse_mlp and f8 is not None:
                h = ops.gemm_skinny_swiglu_fp8(xn2, *wgu[l])
            elif fuse_mlp:
                h = ops.gemm_skinny_swiglu(xn2, wgu[l])                                 # gate|up projection + SwiGLU
            else:
                h = ops.swiglu_fwd(lin(xn2, wgu[l]))
            x = lin(h, wd[l], xm)
        return x
