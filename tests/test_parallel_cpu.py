"""navillm_b200.parallel on CPU (gloo, world_size 2): the reference's DDP usage replayed WITHOUT touching the callers.

* tools/optims.py:52-54          -> ``DDP(model, device_ids=[...], find_unused_parameters=True)`` (our class under that name)
* tasks/agents/mp3d_agent.py:661-667 -> ``isinstance(model, torch.nn.parallel.DistributedDataParallel)``, ``model.no_sync`` around
  every rollout step but the last, rollouts of DIFFERENT length per rank, two backwards in the synced step
  (``cnt_loss.backward()`` then ``obj_loss.backward()``, :750-757,823-825)
* train.py:86-89                 -> clip + optimizer step with no explicit reduce

The product has no CPU kernels, so the wrapped module here is a stub that speaks the same protocol as NavModel: gradients
live in FlatParams buffers written natively by a custom backward node that calls ``grad_sync.backward_begins()`` and the
per-layer overlap hook exactly like ``_LMFn.backward`` / ``LlamaCore.backward`` do.  (tests/test_ddp_nccl_gpu.py runs
the real NavModel over NCCL when two GPUs are present.)
"""
import os
import socket
import sys
from contextlib import nullcontext
from pathlib import Path

import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

N_LAYERS = 8


class _StubFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, model, x, anchor):
        ctx.model, ctx.x = model, x
        return (x * model.scale()).sum()

    @staticmethod
    def backward(ctx, dout):
        m = ctx.model
        m.grad_sync.backward_begins()
        starts = [m.flat.offset_of(p) for p in m.layers] + [m.flat.offset_of(m.tail)]
        hook = m.grad_sync.layer_hook(m.flat, starts, N_LAYERS)
        for l in range(N_LAYERS - 1, -1, -1):                       # native accumulation, layer by layer, last layer first
            m.layers[l].grad.add_(float(dout) * ctx.x.mean() * (l + 1))
            if hook is not None:
                hook(l)
        m.tail.grad.add_(float(dout) * ctx.x.sum())
        m.small.grad.add_(float(dout) * ctx.x.min())
        return None, None, None


class StubNav(nn.Module):
    """Same protocol as NavModel: .grad_sync (GradSync), two FlatParams buffers, lang_model.cls_token attribute."""

    def __init__(self):
        super().__init__()
        from navillm_b200.llama import FlatParams
        from navillm_b200.parallel import GradSync
        self.layers = nn.ParameterList([nn.Parameter(torch.full((64,), float(i))) for i in range(N_LAYERS)])
        self.tail = nn.Parameter(torch.ones(128))
        self.small = nn.Parameter(torch.ones(64))
        self.flat = FlatParams(list(self.layers) + [self.tail], torch.device("cpu"))
        self.flat32 = FlatParams([self.small], torch.device("cpu"))
        self.grad_sync = GradSync()
        self.grad_sync.chunk_layers = 2
        self.grad_sync.flats = lambda: [(self.flat, self.flat.offset_of(self.tail)), (self.flat32, None)]
        self.lang_model = type("LM", (), {"cls_token": ["<cls_1>", "<cls_2>"]})()
        self.register_buffer("_anchor", torch.zeros(()), persistent=False)

    def scale(self):
        return 1.0

    def forward(self, mode, batch):
        return {"loss": _StubFn.apply(self, batch["x"], self._anchor.detach().requires_grad_(True))}


def _agent_rollout(model, n_steps, gen, with_object_grounding):
    """tasks/agents/mp3d_agent.py:660-757,823-825, reduced to its synchronisation skeleton (callers unchanged)."""
    for t in range(n_steps):
        if isinstance(model, torch.nn.parallel.DistributedDataParallel):
            context = nullcontext if t == n_steps - 1 else model.no_sync
        else:
            context = nullcontext
        with context():
            out = model("navigation", {"x": torch.randn(64, generator=gen)})
            out["loss"].backward()
            if t == n_steps - 1 and with_object_grounding:
                cls = model.module.lang_model.cls_token[0] if hasattr(model, "module") else model.lang_model.cls_token[0]
                assert cls == "<cls_1>"
                obj = model("object_grounding", {"x": torch.randn(64, generator=gen)})
                obj["loss"].backward()


def _worker(rank, world, port, q, overlap):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from navillm_b200.parallel import DistributedDataParallel as DDP
    torch.manual_seed(0)
    ref_model = StubNav()                                             # local accumulation only (bare: never exchanges)
    model = StubNav()
    model.grad_sync.overlap = overlap
    model = DDP(model, device_ids=[0], find_unused_parameters=True)   # tools/optims.py:54, unchanged call
    assert isinstance(model, torch.nn.parallel.DistributedDataParallel) and hasattr(model, "module")
    n_steps = 3 + 2 * rank                                            # rollouts end at different steps on different ranks
    for it in range(2):                                               # two optimizer steps (train.py:67-89)
        _agent_rollout(model, n_steps, torch.Generator().manual_seed(100 * it + rank), with_object_grounding=True)
        _agent_rollout(ref_model, n_steps, torch.Generator().manual_seed(100 * it + rank), with_object_grounding=True)
        # expected: DDP semantics.  sync #1 averages everything accumulated so far, the object-grounding pass then adds its
        # local gradient and averages again => mean over ranks of the local sums.
        for name, f, rf in (("bf", model.module.flat, ref_model.flat), ("f32", model.module.flat32, ref_model.flat32)):
            gathered = [None] * world
            dist.all_gather_object(gathered, rf.flat_grad.clone().numpy())
            mean = sum(torch.from_numpy(g) for g in gathered) / world
            assert torch.allclose(f.flat_grad, mean, rtol=1e-5, atol=1e-5), f"rank {rank} it {it} buffer {name}: not the rank mean"
        torch.nn.utils.clip_grad_norm_(model.parameters(), 40.)       # train.py:87 on the views
        for m in (model, ref_model):
            for p in m.parameters():
                p.grad.zero_()
    st = model.module.grad_sync.stats
    counts = [None] * world
    dist.all_gather_object(counts, dict(st))
    assert counts[0] == counts[1], f"ranks issued different collectives: {counts}"   # equal although rollout lengths differ
    assert st["exchanges"] == 4                                       # 2 iterations x (navigation + object grounding)
    if overlap:
        # groups of 2 layers, the last group cut into single layers: 8 layers -> slices at l = 6, 4, 2, 1, 0
        assert st["async_slices"] == 4 * (N_LAYERS // 2 + 1) and st["collectives"] == 4 * (N_LAYERS // 2 + 1 + 2)
    else:
        assert st["async_slices"] == 0 and st["collectives"] == 4 * 2          # ONE collective per flat buffer per exchange
    # a validate-style forward with no backward, then a no_sync pass: must not exchange (DDP decides at the LAST forward)
    model("navigation", {"x": torch.randn(64)})
    with model.no_sync():
        model("navigation", {"x": torch.randn(64)})["loss"].backward()
    assert model.module.grad_sync.stats["exchanges"] == 4
    q.put((rank, "ok"))
    dist.destroy_process_group()


def _run(overlap):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q, overlap)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=180)
        assert p.exitcode == 0, f"rank failed with exit code {p.exitcode}"
    assert sorted(q.get(timeout=5) for _ in range(2)) == [(0, "ok"), (1, "ok")]


def test_ddp_wrapper_replays_agent_no_sync_pattern_overlapped():
    _run(overlap=True)


def test_ddp_wrapper_replays_agent_no_sync_pattern_end_of_backward_only():
    _run(overlap=False)


def test_bare_model_and_single_process_never_exchange():
    from navillm_b200.parallel import DistributedDataParallel as DDP
    m = StubNav()
    m("navigation", {"x": torch.randn(64)})["loss"].backward()
    assert m.grad_sync.stats["exchanges"] == 0 and m.grad_sync.exchange() == 0
    w = DDP(StubNav())                                                # no process group: wrapper is transparent
    w("navigation", {"x": torch.randn(64)})["loss"].backward()
    assert w.module.grad_sync.stats["collectives"] == 0 and not w.module.grad_sync.armed
    assert list(w.state_dict().keys())[0].startswith("module.")      # same key prefix as torch DDP (tools/optims.py:66 unwraps)


def test_parameter_order_matches_reference_optimizer_indexing():
    """torch.optim state indices of reference checkpoints follow model.named_parameters() order with transformers==4.28.0
    (LlamaMLP registers gate_proj, down_proj, up_proj): FlatAdamW.state_dict / load_state_dict index the same way."""
    from navillm_b200.llama import LlamaDims, LlamaModelParams
    names = [n for n, _ in LlamaModelParams(LlamaDims(hidden=128, n_layers=1, n_heads=1, inter=256, vocab=16)).named_parameters()]
    assert names == ["embed_tokens.weight", "layers.0.self_attn.q_proj.weight", "layers.0.self_attn.k_proj.weight",
                     "layers.0.self_attn.v_proj.weight", "layers.0.self_attn.o_proj.weight", "layers.0.mlp.gate_proj.weight",
                     "layers.0.mlp.down_proj.weight", "layers.0.mlp.up_proj.weight", "layers.0.input_layernorm.weight",
                     "layers.0.post_attention_layernorm.weight", "norm.weight"]


def test_fused_views_are_identity_checked():
    """The fused q|k|v / gate|up weight views must come from the flat-buffer order, not from parameters() order (where
    down_proj sits between gate_proj and up_proj and has the same size as up_proj)."""
    import pytest
    from navillm_b200.llama import FlatParams, LlamaDims, LlamaModelParams
    d = LlamaDims(hidden=128, n_layers=1, n_heads=1, inter=256, vocab=16)
    m = LlamaModelParams(d)
    mlp = m.layers[0].mlp
    good = FlatParams(m.flat_order(), torch.device("cpu"))
    v = good.view([mlp.gate_proj.weight, mlp.up_proj.weight], (2 * d.inter, d.hidden))
    assert v.data_ptr() == mlp.gate_proj.weight.data_ptr() and v[d.inter:].data_ptr() == mlp.up_proj.weight.data_ptr()
    m2 = LlamaModelParams(d)
    bad = FlatParams(list(m2.parameters()), torch.device("cpu"))
    with pytest.raises(RuntimeError):
        bad.view([m2.layers[0].mlp.gate_proj.weight, m2.layers[0].mlp.up_proj.weight], (2 * d.inter, d.hidden))


def test_decoder_stack_needs_head_dim_128():
    """The attention kernels are built for head_dim 128: a LlamaCore of any other head size is refused when it is built."""
    import pytest
    from navillm_b200.llama import FlatParams, LlamaCore, LlamaDims, LlamaModelParams
    d = LlamaDims(hidden=128, n_layers=1, n_heads=2, inter=256, vocab=16)
    m = LlamaModelParams(d)
    with pytest.raises(ValueError, match="head_dim 128"):
        LlamaCore(d, m, FlatParams(m.flat_order(), torch.device("cpu")))
