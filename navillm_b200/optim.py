"""Fused clip + AdamW over NavModel's flat buffers (SURVEY.md §8f n3; reference train.py:86-89,
tools/optims.py:43: ``clip_grad_norm_(40.)`` + ``torch.optim.AdamW(lr)`` with torch defaults).

    opt = FlatAdamW(model, lr=1e-5)          # instead of torch.optim.AdamW(model.parameters(), lr)
    ...backward(s)...; model.allreduce_grads()
    opt.step(max_grad_norm=40.0)             # clip + update: 2 + 1 + 2 launches, no host sync
    model.zero_grad(lazy=True)

``state_dict`` / ``load_state_dict`` use torch.optim's per-parameter layout (``exp_avg``, ``exp_avg_sq``, ``step``)
so checkpoints written by the reference (tools/optims.py:65-78) interoperate.
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import check, f32, i32, i64, ptr, stream_ptr


class FlatAdamW:
    def __init__(self, model, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 1e-2):
        model._ensure()
        self.model = model
        self.flats = [model.lang_model.flat, model._flat32]
        self.lr, self.betas, self.eps, self.weight_decay = lr, betas, eps, weight_decay
        self.step_count = 0
        self.m = [torch.zeros_like(f.flat) for f in self.flats]
        self.v = [torch.zeros_like(f.flat) for f in self.flats]
        lib = _lib.load()
        self.n_part = lib.nv_optim_partials()
        dev = self.flats[0].flat.device
        self.partials = torch.zeros(self.n_part * len(self.flats), dtype=torch.float32, device=dev)
        self.clip_state = torch.zeros(2, dtype=torch.float32, device=dev)      # [grad norm, clip coefficient]
        self.param_groups = [{"lr": lr, "betas": betas, "eps": eps, "weight_decay": weight_decay}]   # lr schedulers poke here

    @torch.no_grad()
    def step(self, max_grad_norm: float | None = None, write_clipped_grad: bool = False):
        lib = _lib.load()
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
        for k, f in enumerate(self.flats):
            check(lib.nv_adamw_flat(ptr(f.flat), ptr(f.flat_grad), ptr(self.m[k]), ptr(self.v[k]), i64(f.flat.numel()),
                                    i32(f.dtype == torch.bfloat16), f32(lr), f32(self.betas[0]), f32(self.betas[1]), f32(self.eps),
                                    f32(self.weight_decay), i32(self.step_count), ptr(state), i32(write_clipped_grad),
                                    stream_ptr()), "nv_adamw_flat")
            f.generation += 1                          # raw-pointer write: invalidates an fp8 copy of the weights

    def grad_norm(self) -> torch.Tensor:
        """Total gradient norm measured by the last ``step(max_grad_norm=...)`` (device scalar, no sync)."""
        return self.clip_state[0]

    def zero_grad(self, set_to_none: bool = False):
        self.model.zero_grad(lazy=True)

    # ---- torch.optim-compatible (de)serialisation ----
    def _named_views(self, bufs):
        """Per-parameter views of the flat moment buffers, in ``model.parameters()`` order (the order
        torch.optim.AdamW([p for n, p in model.named_parameters() if p.requires_grad]) indexes its state by)."""
        where = {}
        for f, buf in zip(self.flats, bufs):
            for p, o in zip(f.params, f.offsets):
                where[id(p)] = buf[o:o + p.numel()].view(p.shape)
        return [where[id(p)] for p in self.model.parameters() if p.requires_grad and id(p) in where]

    def state_dict(self):
        ms, vs = self._named_views(self.m), self._named_views(self.v)
        step = torch.tensor(float(self.step_count))
        return {"state": {i: {"step": step, "exp_avg": m, "exp_avg_sq": v} for i, (m, v) in enumerate(zip(ms, vs))},
                "param_groups": [dict(self.param_groups[0], params=list(range(len(ms))))]}

    def load_state_dict(self, sd):
        ms, vs = self._named_views(self.m), self._named_views(self.v)
        names = [n for n, p in self.model.named_parameters() if p.requires_grad]
        idx = sd["param_groups"][0].get("params")
        if idx is not None and len(idx) != len(ms):
            raise ValueError(f"optimizer state covers {len(idx)} parameters, this model has {len(ms)} trainable parameters")
        for i, st in sd["state"].items():
            i = int(i)
            if not 0 <= i < len(ms):
                raise ValueError(f"optimizer state index {i} out of range (model has {len(ms)} trainable parameters)")
            for key, dst in (("exp_avg", ms[i]), ("exp_avg_sq", vs[i])):
                if tuple(st[key].shape) != tuple(dst.shape):
                    raise ValueError(f"optimizer state {i} ({names[i]}): {key} has shape {tuple(st[key].shape)}, the parameter "
                                     f"has {tuple(dst.shape)} -- was the checkpoint written for a different parameter order?")
            ms[i].copy_(st["exp_avg"]); vs[i].copy_(st["exp_avg_sq"])
            self.step_count = int(st["step"])
        self.param_groups[0].update({k: v for k, v in sd["param_groups"][0].items() if k != "params"})
