"""Fused clip + AdamW over NavModel's flat buffers (SURVEY.md §8f n3; reference train.py:86-89,
tools/optims.py:43: ``clip_grad_norm_(40.)`` + ``torch.optim.AdamW(lr)`` with torch defaults).

    opt = FlatAdamW(model, lr=1e-5)          # instead of torch.optim.AdamW(model.parameters(), lr)
    ...backward(s)...; model.allreduce_grads()
    opt.step(max_grad_norm=40.0)             # clip + update: 2 + 1 + 2 launches, no host sync
    model.zero_grad(lazy=True)

``state_dict`` / ``load_state_dict`` use torch.optim's per-parameter layout (``exp_avg``, ``exp_avg_sq``, ``step``)
so checkpoints written by the reference (tools/optims.py:65-78) interoperate.

``compensated=True`` (opt-in; it changes results) keeps a bf16 residual r beside the language model's bf16 weights p: the
pair stands for the master value p + r, so AdamW updates far below half a bf16 ulp of p (most of them at the reference's
lr 3e-5) accumulate instead of being rounded away.  It costs 2 bytes per LM parameter (13.5 GB at Vicuna-7B), read and
written once per step.  The fp32 encoder buffer keeps the plain update.  The residual belongs to the
weights it was computed with: a write to them from anywhere else (``load_state_dict``, ``quantize_weights_fp8()``, an
in-place op) zeroes it before the next step.  It is saved as ``weight_residual`` next to each bf16 parameter's moments.

``moments="8bit"`` (opt-in; it changes results) stores the LM buffer's m and v block-wise in 8 bits (Dettmers et al.,
"8-bit Optimizers via Block-wise Quantization", ICLR 2022): per 64 consecutive elements one fp32 absmax and 64 uint8
codes, valued ``map[code] * absmax``.  2.125 bytes per LM parameter for m and v together instead of 4 (14.3 GB instead of
27.0 GB at Vicuna-7B); it combines with ``compensated=True``.  The update dequantizes to fp32, runs the same AdamW
arithmetic and requantizes each block to the nearest code under its new absmax.  This module owns the format: ``code_maps``
builds the two maps the kernels read.  The fp32 encoder buffer keeps fp32 moments.  ``state_dict`` writes each LM
parameter's moments dequantized into its dtype (``exp_avg`` / ``exp_avg_sq``, host tensors) and, for a bit-exact resume, its
codes and absmax (``exp_avg_code`` / ``exp_avg_absmax``, ``exp_avg_sq_code`` / ``exp_avg_sq_absmax``), which makes a
checkpoint 2.125 bytes per LM parameter larger (14.3 GB at Vicuna-7B).
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from ._lib import check, f32, i32, i64, ptr, stream_ptr


QBLOCK = 64          # elements per block of an 8-bit moment (FlatParams aligns every parameter to 64 elements)
M_ZERO = 128         # the signed map's code of 0; code 127 duplicates 0 and is never produced
V_ZERO = 0           # the unsigned map's code of 0


def tree_magnitudes(bits: int) -> np.ndarray:
    """Dynamic-tree magnitudes with ``bits`` bits after the sign, ascending (float64): exponent e = 0 .. bits-1 contributes
    10^-e times the midpoints of adjacent entries of linspace(0.1, 1, 2^(bits-1-e) + 1)."""
    out = []
    for e in range(bits):
        lin = np.linspace(0.1, 1.0, 2 ** (bits - 1 - e) + 1)
        out.append(10.0 ** -e * (lin[:-1] + lin[1:]) / 2)
    return np.sort(np.concatenate(out))


def code_maps() -> tuple[np.ndarray, np.ndarray]:
    """The two sorted fp32 code maps of 256 entries.  Signed (m): 0, +-1 and the 126 largest 7-bit tree magnitudes of each
    sign, with a spare second 0 at code 127, so that map[127 - k] == -map[128 + k].  Unsigned (v): 0, 1 and the 254 largest
    8-bit tree magnitudes."""
    m = tree_magnitudes(7)[-126:]
    signed = np.concatenate([[-1.0], -m[::-1], [0.0, 0.0], m, [1.0]]).astype(np.float32)
    unsigned = np.concatenate([[0.0], tree_magnitudes(8)[-254:], [1.0]]).astype(np.float32)
    return signed, unsigned


_MAPS: dict = {}


def device_maps(dev) -> torch.Tensor:
    """fp32 [512] on ``dev``: the signed map, then the unsigned one (2 KB, the layout the 8-bit kernels read)."""
    dev = torch.device(dev)
    if dev not in _MAPS:
        _MAPS[dev] = torch.from_numpy(np.concatenate(code_maps())).to(dev)
    return _MAPS[dev]


def quantize_moment(src: torch.Tensor, code: torch.Tensor, absmax: torch.Tensor, signed: bool) -> None:
    """``src`` (bf16 or fp32, n elements, on the device) into ``code`` (uint8 [n]) and ``absmax`` (fp32 [ceil(n / 64)])."""
    n = src.numel()
    assert src.is_contiguous() and src.dtype in (torch.bfloat16, torch.float32)
    assert code.numel() == n and code.dtype == torch.uint8 and absmax.numel() == -(-n // QBLOCK) and absmax.dtype == torch.float32
    check(_lib.load().nv_moments_quantize_8bit(ptr(src), i32(src.dtype == torch.bfloat16), ptr(code), ptr(absmax), i64(n),
                                               i32(signed), ptr(device_maps(src.device)), stream_ptr()),
          "nv_moments_quantize_8bit")


def dequantize_moment(code: torch.Tensor, absmax: torch.Tensor, dtype: torch.dtype, signed: bool) -> torch.Tensor:
    """The values ``map[code] * absmax`` of an 8-bit moment, rounded to ``dtype`` (bf16 or fp32), on the device."""
    n = code.numel()
    assert code.is_contiguous() and absmax.is_contiguous() and absmax.numel() == -(-n // QBLOCK)
    out = torch.empty(code.shape, dtype=dtype, device=code.device)
    check(_lib.load().nv_moments_dequantize_8bit(ptr(code), ptr(absmax), ptr(out), i32(dtype == torch.bfloat16), i64(n),
                                                 i32(signed), ptr(device_maps(code.device)), stream_ptr()),
          "nv_moments_dequantize_8bit")
    return out


class FlatAdamW:
    def __init__(self, model, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 1e-2,
                 compensated: bool = False, moments: str = "bf16"):
        if moments not in ("bf16", "8bit"):
            raise ValueError(f"moments must be 'bf16' or '8bit', got {moments!r}")
        model._ensure()
        self.model = model
        self.flats = [model.lang_model.flat, model._flat32]
        self.lr, self.betas, self.eps, self.weight_decay = lr, betas, eps, weight_decay
        self.step_count = 0
        self.moments = moments
        if moments == "8bit":
            lm = self.flats[0]
            assert lm.dtype == torch.bfloat16 and all(o % QBLOCK == 0 for o in lm.offsets), \
                "8-bit moments need the LM flat buffer in bf16 with every parameter aligned to 64 elements"
            n, dev = lm.flat.numel(), lm.flat.device
            nb = -(-n // QBLOCK)
            self.m_code = torch.zeros(n, dtype=torch.uint8, device=dev)      # code 0 under absmax 0: an all-zero block
            self.v_code = torch.zeros(n, dtype=torch.uint8, device=dev)
            self.m_absmax = torch.zeros(nb, dtype=torch.float32, device=dev)
            self.v_absmax = torch.zeros(nb, dtype=torch.float32, device=dev)
            self.maps = device_maps(dev)
            self.m = [None] + [torch.zeros_like(f.flat) for f in self.flats[1:]]
            self.v = [None] + [torch.zeros_like(f.flat) for f in self.flats[1:]]
        else:
            self.m = [torch.zeros_like(f.flat) for f in self.flats]
            self.v = [torch.zeros_like(f.flat) for f in self.flats]
        lib = _lib.load()
        self.n_part = lib.nv_optim_partials()
        dev = self.flats[0].flat.device
        self.partials = torch.zeros(self.n_part * len(self.flats), dtype=torch.float32, device=dev)
        self.clip_state = torch.zeros(2, dtype=torch.float32, device=dev)      # [grad norm, clip coefficient]
        self.param_groups = [{"lr": lr, "betas": betas, "eps": eps, "weight_decay": weight_decay}]   # lr schedulers poke here
        self.residual = torch.zeros_like(self.flats[0].flat) if compensated else None
        self._weights = self.flats[0].weight_state()           # the weights the residual was computed with

    @torch.no_grad()
    def step(self, max_grad_norm: float | None = None, write_clipped_grad: bool = False):
        lib = _lib.load()
        self.model.flush_weight_grads()              # deferred weight gradients (defer_weight_grads) enter .grad first
        self.model._settle_lazy_zero()               # a lazy zero_grad with no backward since: gradients are zero, not stale
        self.step_count += 1
        lr = self.param_groups[0]["lr"]
        state = None
        if max_grad_norm is not None:
            for k, f in enumerate(self.flats):
                check(lib.nv_grad_sumsq(ptr(f.flat_grad), i64(f.flat_grad.numel()), i32(f.dtype == torch.bfloat16),
                                        ptr(self.partials[k * self.n_part:]), stream_ptr()), "nv_grad_sumsq")
            check(lib.nv_clip_coef(ptr(self.partials), i32(self.partials.numel()), f32(max_grad_norm), ptr(self.clip_state),
                                   stream_ptr()), "nv_clip_coef")
            state = self.clip_state
        if self.residual is not None and self.flats[0].weight_state() != self._weights:
            self.residual.zero_()                      # written elsewhere since the last step: the residual is not theirs
        for k, f in enumerate(self.flats):
            if k == 0 and self.moments == "8bit":
                check(lib.nv_adamw_flat_8bit(ptr(f.flat), ptr(self.residual), ptr(f.flat_grad), ptr(self.m_code),
                                             ptr(self.m_absmax), ptr(self.v_code), ptr(self.v_absmax), ptr(self.maps),
                                             i64(f.flat.numel()), f32(lr), f32(self.betas[0]), f32(self.betas[1]),
                                             f32(self.eps), f32(self.weight_decay), i32(self.step_count), ptr(state),
                                             i32(write_clipped_grad), stream_ptr()), "nv_adamw_flat_8bit")
            elif k == 0 and self.residual is not None:
                check(lib.nv_adamw_flat_compensated(ptr(f.flat), ptr(self.residual), ptr(f.flat_grad), ptr(self.m[k]),
                                                    ptr(self.v[k]), i64(f.flat.numel()), f32(lr), f32(self.betas[0]),
                                                    f32(self.betas[1]), f32(self.eps), f32(self.weight_decay),
                                                    i32(self.step_count), ptr(state), i32(write_clipped_grad), stream_ptr()),
                      "nv_adamw_flat_compensated")
            else:
                check(lib.nv_adamw_flat(ptr(f.flat), ptr(f.flat_grad), ptr(self.m[k]), ptr(self.v[k]), i64(f.flat.numel()),
                                        i32(f.dtype == torch.bfloat16), f32(lr), f32(self.betas[0]), f32(self.betas[1]),
                                        f32(self.eps), f32(self.weight_decay), i32(self.step_count), ptr(state),
                                        i32(write_clipped_grad), stream_ptr()), "nv_adamw_flat")
            f.generation += 1                          # raw-pointer write: invalidates an fp8 copy of the weights
        if self.residual is not None:
            self._weights = self.flats[0].weight_state()

    def state_bytes(self) -> int:
        """Device bytes of the optimizer state: the moments of both flat buffers (codes and absmax for 8-bit ones) and the
        residual."""
        ts = [t for t in self.m + self.v if t is not None] + ([self.residual] if self.residual is not None else [])
        if self.moments == "8bit":
            ts += [self.m_code, self.m_absmax, self.v_code, self.v_absmax]
        return sum(t.numel() * t.element_size() for t in ts)

    def grad_norm(self) -> torch.Tensor:
        """Total gradient norm measured by the last ``step(max_grad_norm=...)`` (device scalar, no sync)."""
        return self.clip_state[0]

    def zero_grad(self, set_to_none: bool = False):
        self.model.zero_grad(lazy=True)

    # ---- torch.optim-compatible (de)serialisation ----
    def _named_views(self, bufs):
        """Per-parameter views of the flat moment buffers (None for a None buffer), in ``model.parameters()`` order (the order
        torch.optim.AdamW([p for n, p in model.named_parameters() if p.requires_grad]) indexes its state by)."""
        where = {}
        for f, buf in zip(self.flats, bufs):
            for p, o in zip(f.params, f.offsets):
                where[id(p)] = None if buf is None else buf[o:o + p.numel()].view(p.shape)
        return [where[id(p)] for p in self.model.parameters() if p.requires_grad and id(p) in where]

    def _code_views(self, p, o):
        """(code, absmax) views of m and of v for the LM parameter ``p`` at flat offset ``o`` (8-bit moments)."""
        n, b0, nb = p.numel(), o // QBLOCK, -(-p.numel() // QBLOCK)
        return ((self.m_code[o:o + n].view(p.shape), self.m_absmax[b0:b0 + nb]),
                (self.v_code[o:o + n].view(p.shape), self.v_absmax[b0:b0 + nb]))

    def _lm_slots(self):
        """(parameter, flat offset) of each trainable parameter in state-dict order, None where it is not in the LM buffer."""
        lm = self.flats[0]
        where = {id(p): (p, o) for p, o in zip(lm.params, lm.offsets)}
        rest = {id(p) for f in self.flats[1:] for p in f.params}
        return [where.get(id(p)) for p in self.model.parameters() if p.requires_grad and (id(p) in where or id(p) in rest)]

    def state_dict(self):
        ms, vs, rs = self._named_views(self.m), self._named_views(self.v), self._named_views([self.residual, None])
        slots = self._lm_slots() if self.moments == "8bit" else [None] * len(ms)
        step = torch.tensor(float(self.step_count))
        state = {}
        for i, (m, v, r) in enumerate(zip(ms, vs, rs)):
            if slots[i] is not None:                   # 8-bit LM moments: dequantized host copies, and the codes themselves
                p, o = slots[i]
                (mc, ma), (vc, va) = self._code_views(p, o)
                m = dequantize_moment(mc, ma, p.dtype, True).cpu()
                v = dequantize_moment(vc, va, p.dtype, False).cpu()
                state[i] = {"step": step, "exp_avg": m, "exp_avg_sq": v, "exp_avg_code": mc, "exp_avg_absmax": ma,
                            "exp_avg_sq_code": vc, "exp_avg_sq_absmax": va}
            else:
                state[i] = {"step": step, "exp_avg": m, "exp_avg_sq": v}
            if r is not None:
                state[i]["weight_residual"] = r
        return {"state": state, "param_groups": [dict(self.param_groups[0], params=list(range(len(ms))))]}

    def _load_8bit(self, i, name, st, p, o):
        """One LM parameter's 8-bit moments: its codes when the state has them with fp32 absmax (an 8-bit FlatAdamW's),
        else its ``exp_avg`` / ``exp_avg_sq`` quantized (a torch or bf16 state)."""
        views = self._code_views(p, o)
        keys = (("exp_avg", True), ("exp_avg_sq", False))
        exact = all(k + "_code" in st and k + "_absmax" in st and st[k + "_absmax"].dtype == torch.float32 for k, _ in keys)
        for key, _ in keys:
            want = [(key + "_code", views[0][0] if key == "exp_avg" else views[1][0]),
                    (key + "_absmax", views[0][1] if key == "exp_avg" else views[1][1])] if exact else [(key, p)]
            for k, dst in want:
                if tuple(st[k].shape) != tuple(dst.shape):
                    raise ValueError(f"optimizer state {i} ({name}): {k} has shape {tuple(st[k].shape)}, the parameter needs "
                                     f"{tuple(dst.shape)} -- was the checkpoint written for a different parameter order?")
        for (key, signed), (code, absmax) in zip(keys, views):
            if exact:
                code.copy_(st[key + "_code"])
                absmax.copy_(st[key + "_absmax"])
            else:
                src = st[key]
                src = src.to(device=code.device, dtype=src.dtype if src.dtype in (torch.bfloat16, torch.float32)
                             else torch.float32).contiguous()
                quantize_moment(src, code.view(-1), absmax, signed)

    def load_state_dict(self, sd):
        """torch.optim layout.  A compensated optimizer takes each bf16 parameter's ``weight_residual`` when present and
        zero otherwise (a torch or plain-FlatAdamW state), and from then on pairs it with the weights as they are now; a
        plain one ignores the key.  With 8-bit moments each LM parameter takes its codes when present with fp32 absmax,
        else its quantized ``exp_avg`` / ``exp_avg_sq``."""
        ms, vs, rs = self._named_views(self.m), self._named_views(self.v), self._named_views([self.residual, None])
        slots = self._lm_slots() if self.moments == "8bit" else [None] * len(ms)
        names = [n for n, p in self.model.named_parameters() if p.requires_grad]
        idx = sd["param_groups"][0].get("params")
        if idx is not None and len(idx) != len(ms):
            raise ValueError(f"optimizer state covers {len(idx)} parameters, this model has {len(ms)} trainable parameters")
        if self.residual is not None:
            self.residual.zero_()
        if self.moments == "8bit":                     # every element the state does not cover (padding included) is 0
            self.m_code.fill_(M_ZERO)
            self.v_code.fill_(V_ZERO)
            self.m_absmax.zero_()
            self.v_absmax.zero_()
        for i, st in sd["state"].items():
            i = int(i)
            if not 0 <= i < len(ms):
                raise ValueError(f"optimizer state index {i} out of range (model has {len(ms)} trainable parameters)")
            pairs = [] if slots[i] is not None else [("exp_avg", ms[i]), ("exp_avg_sq", vs[i])]
            if rs[i] is not None and "weight_residual" in st:
                pairs.append(("weight_residual", rs[i]))
            for key, dst in pairs:
                if tuple(st[key].shape) != tuple(dst.shape):
                    raise ValueError(f"optimizer state {i} ({names[i]}): {key} has shape {tuple(st[key].shape)}, the parameter "
                                     f"has {tuple(dst.shape)} -- was the checkpoint written for a different parameter order?")
            if slots[i] is not None:
                self._load_8bit(i, names[i], st, *slots[i])
            for key, dst in pairs:
                dst.copy_(st[key])
            self.step_count = int(st["step"])
        if self.residual is not None:
            self._weights = self.flats[0].weight_state()
        self.param_groups[0].update({k: v for k, v in sd["param_groups"][0].items() if k != "params"})
