"""The real NavModel under navillm_b200.parallel.DistributedDataParallel over NCCL (2 GPUs): the rollout pattern of
tasks/agents/mp3d_agent.py:661-667 (no_sync around all steps but the last, different rollout lengths per rank, a second
backward in the synced step) must leave every rank with the rank-MEAN of the locally accumulated gradients -- with the
overlapped layer-slice reductions and without.  Skipped on a machine with one GPU; run it on two or more with
`python -m pytest tests/test_ddp_nccl_gpu.py -m gpu -q`."""
import os
import socket
import sys
from contextlib import nullcontext
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
GOLD = Path(__file__).resolve().parent / "golden"


def _rollout(model, g, dev, n_steps, B=2):
    from tests.test_navmodel_gpu import to_dev
    for t in range(n_steps):
        ddp = isinstance(model, torch.nn.parallel.DistributedDataParallel)
        context = model.no_sync if (ddp and t != n_steps - 1) else nullcontext
        with context():
            pano = model("panorama", to_dev(dict(g["pano_in"]), dev))
            nav_in = to_dev(dict(g["nav_in"]), dev)
            nav_in["vp_img_embeds"] = torch.cat([torch.zeros_like(pano["pano_embeds"][:, :1]), pano["pano_embeds"]], 1)
            nav_in["pano_masks"] = torch.cat([torch.ones(B, 1, dtype=torch.bool, device=dev), pano["pano_masks"]], 1)
            torch.manual_seed(1234 + t)
            nav = model("navigation", nav_in)
            loss = F.cross_entropy(nav["fuse_logits"].float(), g["targets"].to(dev), reduction="sum", ignore_index=-100) / B
            loss.backward()
            if t == n_steps - 1:                                       # second backward of the synced step (:823-825)
                og = model("object_grounding", to_dev(dict(g["og_in"]), dev))
                (og["obj_logits"].float().logsumexp(-1).sum() * 0.1).backward()


def _nvls_unit(rank, world, dev):
    """nv_multimem_allreduce on random data against the arithmetic it promises: fp32 sum of the replicas' bf16 values,
    times 1/world, rounded once to bf16 -- to one bf16 ulp: the switch rounds its fp32 accumulator to bf16 in its own way
    (measured: 1-ulp differences against round-to-nearest-even of the fp32 NCCL sum)."""
    import torch.distributed as dist
    import torch.distributed._symmetric_memory as symm
    from navillm_b200 import _lib
    n = 1 << 20
    results = {}
    for dtype in (torch.bfloat16, torch.float32):
        buf = symm.empty(n, dtype=dtype, device=dev)
        hdl = symm.rendezvous(buf, dist.group.WORLD)
        assert hdl.multicast_ptr, "no NVLS multicast mapping"
        g = torch.Generator(device=dev).manual_seed(100 + rank)
        buf.copy_(torch.randn(n, generator=g, device=dev).to(dtype))
        mine = buf.float().clone()
        ref = mine.clone()
        dist.all_reduce(ref)                                   # fp32 NCCL sum of the same values
        ref = (ref / world).to(dtype)
        off, cnt = 1024, n - 4096                              # an interior, 16-byte aligned range
        torch.cuda.synchronize()
        hdl.barrier(channel=0)
        _lib.check(_lib.load().nv_multimem_allreduce(_lib.ctypes.c_uint64(int(hdl.multicast_ptr)), _lib.i64(off), _lib.i64(cnt),
                                                     _lib.i32(1 if dtype == torch.bfloat16 else 0), _lib.i32(rank), _lib.i32(world),
                                                     _lib.f32(1.0 / world), _lib.i32(16), _lib.stream_ptr()), "nv_multimem_allreduce")
        hdl.barrier(channel=0)
        torch.cuda.synchronize()
        got = buf.clone()
        inside = slice(off, off + cnt)
        err = (got[inside].float() - ref[inside].float()).abs().max().item()
        lim = (2.0 ** -7 if dtype == torch.bfloat16 else 1e-6) * ref.float().abs().max().item()
        assert err <= lim, f"rank {rank} {dtype}: multimem all-reduce differs from the NCCL fp32 reference by {err}"
        # outside the range nothing was touched
        assert torch.equal(got[:off].float(), mine[:off]) and torch.equal(got[off + cnt:].float(), mine[off + cnt:])
        results[str(dtype)] = err
    return results


def _worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from navillm_b200.parallel import DistributedDataParallel as DDP
    from tests.test_navmodel_gpu import build_model
    g = torch.load(GOLD / "nav_amp_bf16.pt", weights_only=False)
    n_steps = 2 + rank                                                  # different rollout lengths per rank
    bare, _ = build_model(g, dev)
    bare.train(False)
    _rollout(bare, g, dev, n_steps)                                     # local accumulation only
    torch.cuda.synchronize()
    local = {n: p.grad.detach().float().clone() for n, p in bare.named_parameters() if p.grad is not None}
    nvls_ok = True
    try:
        _nvls_unit(rank, world, dev)
    except Exception as e:                                    # no multicast support on this box: the NCCL path is still tested
        nvls_ok = False
        if rank == 0:
            print(f"[nvls unit] unavailable: {type(e).__name__}: {e}")
    flags = [None] * world
    dist.all_gather_object(flags, nvls_ok)
    nvls_ok = all(flags)
    for overlap, nvls in ((True, False), (False, False), (True, True), (False, True)):
        if nvls and not nvls_ok:
            continue
        os.environ["NAVILLM_NVLS"] = "1" if nvls else "0"
        m, _ = build_model(g, dev)
        m.train(False)
        m.grad_sync.overlap, m.grad_sync.chunk_layers = overlap, 1
        model = DDP(m, device_ids=[rank], find_unused_parameters=True)   # tools/optims.py:54
        assert model.nvls == nvls, (model.nvls, nvls)
        _rollout(model, g, dev, n_steps)
        torch.cuda.synchronize()
        st = dict(m.grad_sync.stats)
        assert st["exchanges"] == 2 and (st["async_slices"] > 0) == overlap, st
        if rank == 0:
            print(f"[ddp overlap={overlap} nvls={nvls}] {st}")
        named = dict(m.named_parameters())
        worst = 0.0
        for n, gl in local.items():
            mean = gl.clone()
            dist.all_reduce(mean)
            mean /= world
            got = named[n].grad.float()
            scale = mean.abs().max().item() + 1e-6
            err = (got - mean).abs().max().item() / scale
            # two bf16 averaging rounds + a different accumulation order (avg-then-add vs add-then-avg)
            assert err <= (2e-2 if named[n].dtype == torch.bfloat16 else 1e-4), f"rank {rank} overlap={overlap} {n}: rel err {err:.3g}"
            worst = max(worst, err)
        counts = [None] * world
        dist.all_gather_object(counts, st)
        assert counts[0] == counts[1], counts
    q.put((rank, "ok"))
    dist.destroy_process_group()


def test_navmodel_ddp_two_ranks_nccl():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs; the gloo twin tests/test_parallel_cpu.py covers the logic on CPU")
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=600)
        assert p.exitcode == 0, f"rank failed with exit code {p.exitcode}"
    assert sorted(q.get(timeout=5) for _ in range(2)) == [(0, "ok"), (1, "ok")]
