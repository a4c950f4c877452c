"""Data-parallel wrapper of the path: the one-line replacement for the reference's DDP wrap (tools/optims.py:52-54).

    # from torch.nn.parallel import DistributedDataParallel as DDP
    from navillm_b200.parallel import DistributedDataParallel as DDP
    model = DDP(model, device_ids=[device_id], find_unused_parameters=True)

Everything else of the reference stays as it is: ``isinstance(model, torch.nn.parallel.DistributedDataParallel)`` and
``model.no_sync`` in the rollout loop (tasks/agents/mp3d_agent.py:661-667), ``model.module.lang_model.cls_token`` (:817),
``save_checkpoint`` unwrapping ``model.module`` (tools/optims.py:66-67), ``clip_grad_norm_(model.parameters())`` and the
optimizer step with NO explicit reduce in train.py:86-89.

What is different from torch's DDP is the mechanism.  NavModel keeps its gradients in two flat buffers (bf16 LM + heads,
fp32 encoder / embeddings) that its hand-written backward accumulates into natively, so there are no per-parameter
autograd hooks and no buckets to rebuild.  ``GradSync`` reproduces DDP's *semantics* on top of that:

* a forward outside ``no_sync()`` with grad enabled ARMS the exchange, a forward inside ``no_sync()`` disarms it
  (DDP decides at forward time, from the last forward before the backward);
* the first custom backward node of an armed pass queues an end-of-backward callback on the autograd engine
  (``Variable._execution_engine.queue_callback`` -- the hook DDP itself finalises with): when the whole backward of
  the pass (head -> LM -> fusion glue -> panorama encoder) has run, every flat buffer is all-reduced (AVG) exactly once;
* while the LM backward is running, the gradient slice of each finished group of decoder layers is all-reduced
  asynchronously so NCCL overlaps the remaining wgrad GEMMs; the end-of-backward callback waits for those handles and
  reduces only what they did not cover;
* an unarmed backward (inside ``no_sync``) issues NO collective, so ranks whose rollouts have different lengths issue
  the same number of collectives as under the reference's DDP: one exchange per armed pass.

The class derives from ``torch.nn.parallel.DistributedDataParallel`` only so that the reference's ``isinstance`` test
holds; torch's reducer is never constructed.
"""
from __future__ import annotations

import contextlib
import os
from typing import Callable, List, Optional

import torch
import torch.nn as nn


def _dist():
    import torch.distributed as dist
    return dist if (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1) else None


class NvlsReducer:
    """In-switch all-reduce of flat gradient buffers over NVLS multicast (csrc/nvls_allreduce.cu) on a side stream.

    ``adopt(flat)`` moves a FlatParams gradient buffer into a SYMMETRIC allocation (torch.distributed._symmetric_memory:
    same size on every rank, bound to one multicast object) -- a collective call.  ``all_reduce(flat, a, b)`` then enqueues,
    on the side stream and ordered after everything the current stream has done so far:
        barrier (all replicas of the range are complete)  ->  nv_multimem_allreduce  ->  barrier (all parts are stored)
    and returns a CUDA event the consumer waits for.  Rank r reduces the r-th 1/W of the range: multimem.ld_reduce pulls
    the sum of the W replicas out of the switch, multimem.st pushes the average back into all of them."""

    def __init__(self, ctas: int = 0):
        self.stream = torch.cuda.Stream()
        self.handles = {}
        # CTAs issuing the multimem operations: few while the reduction hides behind the backward (they share SMs with the
        # persistent GEMMs; 8 vs 32 CTAs: 366.7 vs 368.9 ms/step at 8 GPUs), many when it is exposed anyway (the tail after the
        # backward, or a backward too short to hide 13.5 GB behind: 8 CTAs move 214 GB/s per rank pair)
        self.ctas = ctas or int(os.environ.get("NAVILLM_NVLS_CTAS", "8"))
        self.ctas_exposed = max(self.ctas, int(os.environ.get("NAVILLM_NVLS_CTAS_EXPOSED", "32")))
        self.n_reduced = 0

    @staticmethod
    def wanted() -> bool:
        dist = _dist()
        return dist is not None and dist.get_backend() == "nccl" and os.environ.get("NAVILLM_NVLS", "1") != "0"

    def adopt(self, flat, rebind) -> None:
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm
        buf = symm.empty(flat.flat_grad.numel(), dtype=flat.dtype, device=flat.flat.device)
        hdl = symm.rendezvous(buf, dist.group.WORLD)
        if not getattr(hdl, "multicast_ptr", 0):
            raise RuntimeError("symmetric memory has no NVLS multicast mapping on this system")
        buf.copy_(flat.flat_grad)
        rebind(buf)                                   # p.grad views (and the fused grad views) now live in `buf`
        self.handles[id(flat)] = (hdl, buf)

    def has(self, flat) -> bool:
        return id(flat) in self.handles

    def all_reduce(self, flat, a: int, b: int, scale: float, exposed: bool = False):
        from . import _lib
        hdl, buf = self.handles[id(flat)]
        if flat.flat_grad.data_ptr() != buf.data_ptr():
            raise RuntimeError("the symmetric gradient buffer was replaced (re-materialised model?): re-wrap the model")
        cur = torch.cuda.current_stream()
        ready = torch.cuda.Event()
        ready.record(cur)
        self.stream.wait_event(ready)
        with torch.cuda.stream(self.stream):
            hdl.barrier(channel=0)
            _lib.check(_lib.load().nv_multimem_allreduce(_lib.ctypes.c_uint64(int(hdl.multicast_ptr)), _lib.i64(a), _lib.i64(b - a),
                                                         _lib.i32(1 if flat.dtype == torch.bfloat16 else 0), _lib.i32(hdl.rank),
                                                         _lib.i32(hdl.world_size), _lib.f32(scale), _lib.i32(self.ctas_exposed if exposed else self.ctas),
                                                         _lib.ctypes.c_void_p(self.stream.cuda_stream)), "nv_multimem_allreduce")
            hdl.barrier(channel=0)
            done = torch.cuda.Event()
            done.record(self.stream)
        self.n_reduced += 1
        return done


class GradSync:
    """State machine of the gradient exchange of ONE model replica (shared by NavModel and its language model)."""

    def __init__(self):
        self.armed = False            # the last grad-enabled forward ran outside no_sync()
        self.queued = False           # the end-of-backward callback of the running pass is queued
        self.overlap = True           # reduce finished layer groups while the backward is still running
        self.chunk_layers = int(os.environ.get("NAVILLM_SYNC_CHUNK", "2"))   # decoder layers per overlapped reduction
        self.flats: Callable[[], list] = lambda: []          # -> [(FlatParams, tail_offset or None), ...]
        self.before_exchange: Callable[[], None] = lambda: None   # end of an armed pass: complete pending gradients first
        self._pending: List[tuple] = []
        self._lm_layers_reduced = False
        self.reducer: Optional[NvlsReducer] = None            # set by the DDP wrapper when NVLS multicast is available
        self.short_backward = False   # set per pass by the LM: too few tokens to hide the exchange behind (see NvlsReducer)
        self.stats = {"collectives": 0, "exchanges": 0, "async_slices": 0}

    # ---- forward side -------------------------------------------------------------------------------------------
    def on_forward(self, sync: bool) -> None:
        if torch.is_grad_enabled():
            self.armed = bool(sync) and _dist() is not None

    # ---- backward side ------------------------------------------------------------------------------------------
    def backward_begins(self) -> None:
        """Called by the first custom backward node of a pass (action head, or the LM in the loss modes)."""
        if self.armed and not self.queued:
            self.queued = True
            torch.autograd.Variable._execution_engine.queue_callback(self._end_of_backward)

    def layer_hook(self, flat, starts: List[int], n_layers: int) -> Optional[Callable[[int], None]]:
        """Per-layer callback for LlamaCore.backward (layers finish from n_layers-1 down to 0): all-reduces the flat
        gradient slice [starts[l], starts[l + chunk]) of a finished group asynchronously.  None unless this pass is armed."""
        dist = _dist()
        if not (self.armed and self.queued and self.overlap and dist is not None):
            return None
        chunk = max(1, self.chunk_layers)
        avg = dist.ReduceOp.AVG if dist.get_backend() == "nccl" else dist.ReduceOp.SUM
        ws = dist.get_world_size()
        self._lm_layers_reduced = True
        # group boundaries: every `chunk` layers, and the LAST group (layers chunk-1 .. 0, finished when the backward is
        # almost over, so its reduction is mostly exposed) is cut into single layers
        ends = {l: min(l + chunk, n_layers) for l in range(0, n_layers, chunk)}
        for l in range(1, min(chunk, n_layers)):
            ends[l] = l + 1
        if chunk > 1 and n_layers > 0:
            ends[0] = 1

        nvls = self.reducer if (self.reducer is not None and self.reducer.has(flat)) else None

        def done(l: int) -> None:
            if l not in ends:
                return
            if nvls is not None:                                  # in-switch reduction on the side stream
                self._pending.append((nvls.all_reduce(flat, starts[l], starts[ends[l]], 1.0 / ws, exposed=self.short_backward), None, ws))
            else:
                sl = flat.flat_grad[starts[l]:starts[ends[l]]]
                h = dist.all_reduce(sl, op=avg, async_op=True)
                self._pending.append((h, sl if avg == dist.ReduceOp.SUM else None, ws))
            self.stats["collectives"] += 1
            self.stats["async_slices"] += 1
        return done

    def _drain(self) -> None:
        for h, sl, ws in self._pending:
            if isinstance(h, torch.cuda.Event):
                torch.cuda.current_stream().wait_event(h)
                continue
            h.wait()
            if sl is not None:
                sl.div_(ws)
        self._pending = []

    def _end_of_backward(self) -> None:
        try:
            self.before_exchange()            # training prefix caches: part (b) of the gradient (PrefixKVCache.flush_grads)
            self.exchange(covered_lm_layers=self._lm_layers_reduced)
        finally:
            self.armed = self.queued = False
            self._lm_layers_reduced = False

    # ---- the exchange itself ------------------------------------------------------------------------------------
    def exchange(self, covered_lm_layers: bool = False) -> int:
        """All-reduce (average) every flat gradient buffer: ONE collective per buffer (SURVEY.md §8e), minus the LM layer
        slices the overlapped reductions of this pass already covered.  Returns the number of collectives issued here."""
        dist = _dist()
        self._drain()
        if dist is None:
            return 0
        avg = dist.ReduceOp.AVG if dist.get_backend() == "nccl" else dist.ReduceOp.SUM
        ws, n = dist.get_world_size(), 0
        for flat, tail in self.flats():
            if flat is None:
                continue
            lo = tail if (covered_lm_layers and tail is not None) else 0
            hi = flat.flat_grad.numel()
            # segments that no backward has written since they were zeroed are zero on EVERY rank (the decision is taken
            # from the call sequence, which the reference keeps identical on all ranks: tasks/loaders.py:179 broadcasts the
            # task): their average is zero, nothing to exchange.  In the navigation / grounding modes that is lm_head
            # (262 MB, half of what the overlapped layer reductions leave for the end of the backward).
            ranges, cur = [], lo
            for a, b in sorted(getattr(flat, "clean_segments", lambda: [])()):
                a, b = max(a, lo), min(b, hi)
                if a >= b:
                    continue
                if a > cur:
                    ranges.append((cur, a))
                cur = max(cur, b)
            if cur < hi:
                ranges.append((cur, hi))
            for a, b in ranges:
                if self.reducer is not None and self.reducer.has(flat):
                    self._pending.append((self.reducer.all_reduce(flat, a, b, 1.0 / ws, exposed=True), None, ws))
                else:
                    buf = flat.flat_grad[a:b]
                    dist.all_reduce(buf, op=avg)
                    if avg == dist.ReduceOp.SUM:
                        buf.div_(ws)
                n += 1
        self._drain()
        self.stats["collectives"] += n
        self.stats["exchanges"] += 1
        return n


class DistributedDataParallel(torch.nn.parallel.DistributedDataParallel):
    """Drop-in for ``torch.nn.parallel.DistributedDataParallel(model, device_ids=[...], find_unused_parameters=True)``
    around a ``navillm_b200.nav_model.NavModel`` (see the module docstring).  Replicas must start from identical
    parameters (same seed / same checkpoint), as the reference's do; ``broadcast_parameters()`` enforces it explicitly."""

    def __init__(self, module: nn.Module, device_ids=None, output_device=None, find_unused_parameters: bool = False,
                 broadcast_parameters: bool = True, **unused):
        nn.Module.__init__(self)                      # deliberately NOT torch DDP's __init__: no reducer, no buckets
        if not hasattr(module, "grad_sync"):
            raise TypeError("navillm_b200.parallel.DistributedDataParallel wraps a navillm_b200 NavModel "
                            f"(an object with a .grad_sync state), got {type(module).__name__}")
        self.module = module
        self.device_ids = list(device_ids) if device_ids is not None else None
        self.output_device = output_device
        self.find_unused_parameters = find_unused_parameters
        self.require_backward_grad_sync = True
        if broadcast_parameters:
            self.broadcast_parameters()
        self.nvls = False
        if NvlsReducer.wanted() and hasattr(module, "adopt_symmetric_grads"):
            try:
                module.grad_sync.reducer = module.adopt_symmetric_grads(NvlsReducer())
                self.nvls = module.grad_sync.reducer is not None
            except Exception as e:                    # no multicast support / symmetric memory unavailable: NCCL path
                import warnings
                warnings.warn(f"navillm_b200: NVLS gradient exchange unavailable ({type(e).__name__}: {e}); using NCCL all-reduce")
                module.grad_sync.reducer = None
            # every rank must take the same transport: one rank on NCCL and another in the switch would never meet
            dist = _dist()
            if dist is not None:
                ok = torch.tensor([1 if module.grad_sync.reducer is not None else 0], dtype=torch.int32,
                                  device=next(module.parameters()).device)
                dist.all_reduce(ok, op=dist.ReduceOp.MIN)
                if int(ok.item()) == 0 and module.grad_sync.reducer is not None:
                    import warnings
                    warnings.warn("navillm_b200: another rank could not set up the NVLS exchange; all ranks use NCCL")
                    module.grad_sync.reducer = None       # the symmetric buffers stay in use as ordinary gradient buffers
                self.nvls = module.grad_sync.reducer is not None

    def broadcast_parameters(self, src: int = 0) -> None:
        """DDP's construction-time parameter broadcast: one broadcast per flat weight buffer once they exist
        (``NavModel._ensure``), else per parameter."""
        dist = _dist()
        if dist is None:
            return
        flats = [f for f, _ in self.module.grad_sync.flats() if f is not None] if hasattr(self.module, "_flat_buffers_ready") \
            and self.module._flat_buffers_ready() else []
        if flats:
            for f in flats:
                dist.broadcast(f.flat, src=src)
        else:
            with torch.no_grad():
                for p in self.module.parameters():
                    dist.broadcast(p.data, src=src)

    def forward(self, *args, **kwargs):
        self.module.grad_sync.on_forward(self.require_backward_grad_sync)
        return self.module(*args, **kwargs)

    @contextlib.contextmanager
    def no_sync(self):
        """torch DDP's context (used by tasks/agents/mp3d_agent.py:661-667): backwards of forwards that ran inside
        accumulate locally; the first pass outside exchanges the accumulated gradients."""
        old = self.require_backward_grad_sync
        self.require_backward_grad_sync = False
        try:
            yield
        finally:
            self.require_backward_grad_sync = old

    # nn.Module plumbing that torch DDP overrides with reducer-dependent code
    def train(self, mode: bool = True):
        nn.Module.train(self, mode)
        return self

    def __getstate__(self):
        return self.__dict__

    def __setstate__(self, state):
        self.__dict__.update(state)
