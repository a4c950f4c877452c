"""Deferred weight gradients of the decoder linears (defer_weight_grads / flush_weight_grads) and their kernel,
nv_gemm_wgrad_seg_bf16 (the segmented-contraction wgrad GEMM).

Bounds, stated (u = 2^-8, the unit roundoff of bf16):
  * Kernel: bit for bit ops.gemm(a_mn=True, b_mn=True) over the row-concatenation of the segments, each zero-padded to a
    multiple of 64 rows (the same k-block partition).  Against an fp64 reference R = sum_s A_s^T B_s (+ addend), per
    element |C - R| <= u (|acc| + |R|) + 2^-22 K S, with S = sum_s |A_s|^T |B_s| and K the padded row count: one bf16
    rounding of the accumulator, one of the sum with the addend, and fp32 accumulation over K products.
  * Rollouts: deferral changes no forward, dgrad or other gradient, so both arms see the same operand pairs and every
    gradient outside the four decoder linears is bit-identical.  A linear's per-backward gradient is rounded twice per
    backward, the deferred one twice in all, so per element |deferred - per-backward| <= (2 n + 4) u S over the n recorded
    backwards.  Against the fp64 sum of the recorded pairs, the deferred gradient's max and RMS error per weight are no
    larger than the per-backward path's (max within 1 %).
"""
import sys
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
GOLD = Path(__file__).resolve().parent / "golden"
U = 2.0 ** -8

# (M, N) of the four wgrad GEMMs of a Vicuna-7B decoder layer: q|k|v, o_proj, gate|up, down
SHAPES = [(3 * 4096, 4096), (4096, 4096), (2 * 11008, 4096), (4096, 11008)]
RAGGED = [1, 63, 64, 65, 115, 1000]
SEG_LISTS = {"one": [115], "ragged": RAGGED, "rollout15": [115] * 15, "cap": [RAGGED[i % 5] for i in range(64)]}


def _segments(M, N, rows, seed):
    """Segments with their own row strides: odd segments are views into wider buffers (lda > M, ldb > N)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    segs = []
    for s, r in enumerate(rows):
        pad = 64 if s % 2 else 0
        a = torch.randn(r, M + pad, device="cuda", generator=g).to(torch.bfloat16)[:, :M]
        b = torch.randn(r, N + 8 * (s % 3), device="cuda", generator=g).to(torch.bfloat16)[:, :N]
        segs.append((a, b))
    return segs


def _padded_cat(segs, col):
    out = []
    for pair in segs:
        t = pair[col]
        r = t.shape[0]
        p = torch.zeros((r + 63) // 64 * 64, t.shape[1], dtype=t.dtype, device=t.device)
        p[:r] = t
        out.append(p)
    return torch.cat(out)


@pytest.mark.parametrize("addend", [False, True], ids=["overwrite", "addend"])
@pytest.mark.parametrize("segs_name", sorted(SEG_LISTS))
@pytest.mark.parametrize("shape", SHAPES, ids=["qkv", "o", "gate_up", "down"])
def test_wgrad_seg_matches_concatenated_gemm_and_fp64(cuda_dev, shape, segs_name, addend):
    from navillm_b200 import ops
    M, N = shape
    rows = SEG_LISTS[segs_name]
    segs = _segments(M, N, rows, seed=M + N + len(rows))
    add = (torch.randn(M, N, device=cuda_dev) * 4).to(torch.bfloat16) if addend else None
    got = torch.empty(M, N, dtype=torch.bfloat16, device=cuda_dev)
    if add is not None:
        got.copy_(add)
    ops.gemm_wgrad_seg(segs, got, addend=got if add is not None else None)          # in place, as the flush runs it
    A, B = _padded_cat(segs, 0), _padded_cat(segs, 1)
    want = ops.gemm(A, B, a_mn=True, b_mn=True, addend=add)
    torch.cuda.synchronize()
    assert torch.equal(got, want), (got.float() - want.float()).abs().max().item()
    acc = A.double().t() @ B.double()
    ref = acc + (add.double() if add is not None else 0)
    mag = A.double().abs().t() @ B.double().abs()
    bound = U * (acc.abs() + ref.abs()) + 2.0 ** -22 * A.shape[0] * mag
    err = (got.double() - ref).abs()
    assert bool((err <= bound).all()), (err - bound).max().item()


def test_wgrad_seg_rejects_mismatched_segments(cuda_dev):
    from navillm_b200 import ops
    a = torch.zeros(5, 256, dtype=torch.bfloat16, device=cuda_dev)
    b = torch.zeros(5, 128, dtype=torch.bfloat16, device=cuda_dev)
    out = torch.empty(256, 128, dtype=torch.bfloat16, device=cuda_dev)
    with pytest.raises(ValueError, match="segments"):
        ops.gemm_wgrad_seg([(a, b)] * (ops.WGRAD_SEG_MAX + 1), out)
    with pytest.raises(ValueError, match="segment 1"):
        ops.gemm_wgrad_seg([(a, b), (a[:4], b)], out)
    with pytest.raises(ValueError, match="segment 0"):
        ops.gemm_wgrad_seg([(b, a)], out)


# ------------------------------------------------------------------------------------------------------------------
# rollouts at the tiny test widths
# ------------------------------------------------------------------------------------------------------------------
def _golden():
    return torch.load(GOLD / "nav_amp_bf16.pt", weights_only=False)


def _golden_model(g, dev):
    from tests.test_navmodel_gpu import build_model
    return build_model(g, dev)[0]


def _nav_loss(model, g, dev, t, B=2):
    from tests.test_navmodel_gpu import to_dev
    pano = model("panorama", to_dev(dict(g["pano_in"]), dev))
    nav_in = to_dev(dict(g["nav_in"]), dev)
    nav_in["vp_img_embeds"] = torch.cat([torch.zeros_like(pano["pano_embeds"][:, :1]), pano["pano_embeds"]], 1)
    nav_in["pano_masks"] = torch.cat([torch.ones(B, 1, dtype=torch.bool, device=dev), pano["pano_masks"]], 1)
    torch.manual_seed(1234 + t)
    nav = model("navigation", nav_in)
    return F.cross_entropy(nav["fuse_logits"].float(), g["targets"].to(dev), reduction="sum", ignore_index=-100) / B


def _og_rollout(model, g, dev, steps=3, B=2):
    """Teacher-forced steps of the agent (tasks/agents/mp3d_agent.py:660-757,823-825): panorama, navigation backward and an
    object-grounding backward in every step -- two LM backwards per step."""
    from tests.test_navmodel_gpu import to_dev
    for t in range(steps):
        _nav_loss(model, g, dev, t, B).backward()
        og = model("object_grounding", to_dev(dict(g["og_in"]), dev))
        (og["obj_logits"].float().logsumexp(-1).sum() * (0.1 + 0.05 * t)).backward()


def _cache_rollout(model, d, dev, steps=4):
    """The teacher-forced rollout of tests/test_prefix_train_gpu.py over a PrefixKVCache(train=True), flush_grads() at the end."""
    from navillm_b200.modified_lm import PrefixKVCache
    from tests.test_prefix_train_gpu import INSTR, _batches
    cache = PrefixKVCache(model.lang_model, batch_size=2, max_len=256, train=True)
    for step, batch in enumerate(_batches(d, steps, INSTR)):
        batch = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in batch.items()}
        batch["hist_vis"] = [[v.to(dev) for v in vs] for vs in batch["hist_vis"]]
        torch.manual_seed(100 + step)
        out = model("navigation", batch, prefix_cache=cache)
        F.cross_entropy(out["fuse_logits"].float(), torch.zeros(2, dtype=torch.long, device=dev)).backward()
    cache.flush_grads()


def _grads(model):
    torch.cuda.synchronize()
    return {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}


def _linear_names(model):
    """(gradient attribute, layer) -> parameter names whose .grad views make up that fused gradient."""
    out = {}
    for l in range(len(model.lang_model.model.layers)):
        p = f"lang_model.model.layers.{l}."
        out[("gqkv", l)] = [p + f"self_attn.{x}_proj.weight" for x in "qkv"]
        out[("go", l)] = [p + "self_attn.o_proj.weight"]
        out[("ggu", l)] = [p + "mlp.gate_proj.weight", p + "mlp.up_proj.weight"]
        out[("gd", l)] = [p + "mlp.down_proj.weight"]
    return out


def _stash_reference(lm):
    """fp64 sum and sum of magnitudes of the recorded operand pairs of every stashed weight, and the number of backwards."""
    ref = {}
    for key, prs in lm._wgrad_stash.pairs.items():
        s = sum(a.double().t() @ b.double() for a, b in prs)
        m = sum(a.double().abs().t() @ b.double().abs() for a, b in prs)
        ref[key] = (s, m, len(prs))
    ref["rows"] = [a.shape[0] for a, _ in lm._wgrad_stash.pairs[("gqkv", 0)]]
    return ref


def _fused(grads, names):
    return torch.cat([grads[n].reshape(-1, grads[n].shape[-1]) for n in names])


def _compare_arms(model, step, deferred, ref, min_backwards=2):
    """Every non-linear gradient bit-identical; the linears within the stated bound of each other and no further from fp64."""
    lin = _linear_names(model)
    lin_names = {n for ns in lin.values() for n in ns}
    assert step.keys() == deferred.keys()
    for n in step:
        if n not in lin_names:
            assert torch.equal(step[n], deferred[n]), n
    assert set(ref) - {"rows"} == set(lin), set(ref) ^ set(lin)
    worst = 0.0
    for key, names in lin.items():
        s, m, nb = ref[key]
        assert nb >= min_backwards, (key, nb)
        gs, gd = _fused(step, names).double(), _fused(deferred, names).double()
        diff = (gs - gd).abs()
        bound = (2 * nb + 4) * U * m + 1e-30
        assert bool((diff <= bound).all()), (key, (diff - bound).max().item())
        es, ed = (gs - s).abs(), (gd - s).abs()
        assert ed.max().item() <= 1.01 * es.max().item() + 1e-30, (key, ed.max().item(), es.max().item())
        assert ed.pow(2).mean().sqrt().item() <= es.pow(2).mean().sqrt().item() + 1e-30, key
        worst = max(worst, diff.max().item() / max(s.abs().max().item(), 1e-30))
    return worst


def _deferred_run(model, run, max_rows=1 << 20):
    """``run`` with deferral on; returns (gradients after the flush, the fp64 reference of the stash before it)."""
    lm = model.lang_model
    assert model.defer_weight_grads(max_rows) is None
    run()
    assert lm.weight_grads_pending() and model.weight_grad_stash_bytes() > 0
    ref = _stash_reference(lm)
    model.flush_weight_grads()
    assert not lm.weight_grads_pending() and model.weight_grad_stash_bytes() == 0
    out = _grads(model)
    assert model.defer_weight_grads(None) == max_rows
    return out, ref


def test_og_rollout_deferred_matches_per_step(cuda_dev, monkeypatch):
    from navillm_b200 import ops
    g = _golden()
    model = _golden_model(g, cuda_dev)
    calls = []
    orig = ops.gemm_wgrad_seg
    monkeypatch.setattr(ops, "gemm_wgrad_seg", lambda *a, **k: (calls.append(len(a[0])), orig(*a, **k))[1])
    model.zero_grad()
    _og_rollout(model, g, cuda_dev)
    step = _grads(model)
    assert calls == []                                          # deferral off: no segmented launch
    model.zero_grad()
    deferred, ref = _deferred_run(model, lambda: _og_rollout(model, g, cuda_dev))
    n_lin = 4 * len(model.lang_model.model.layers)
    assert calls == [6] * n_lin, calls                          # one launch per weight, 3 steps x 2 backwards
    print("max |deferred - per-step| / max|grad|:", _compare_arms(model, step, deferred, ref, min_backwards=6))


def test_cache_rollout_deferred_matches_per_step(cuda_dev):
    from tests.test_prefix_reuse_gpu import _build
    model, d = _build(cuda_dev)
    model.zero_grad()
    _cache_rollout(model, d, cuda_dev)
    step = _grads(model)
    model.zero_grad()
    deferred, ref = _deferred_run(model, lambda: _cache_rollout(model, d, cuda_dev))
    print("max |deferred - per-step| / max|grad|:", _compare_arms(model, step, deferred, ref, min_backwards=5))


def test_max_rows_flushes_mid_rollout(cuda_dev, monkeypatch):
    """A stash bound below the rollout flushes in batches (same bounds); one below a single backward runs every backward's
    weight gradients at once: the per-step path, bit for bit."""
    from navillm_b200 import ops
    g = _golden()
    model = _golden_model(g, cuda_dev)
    model.zero_grad()
    _og_rollout(model, g, cuda_dev)
    step = _grads(model)
    model.zero_grad()
    _, ref = _deferred_run(model, lambda: _og_rollout(model, g, cuda_dev))
    rows = ref["rows"]                                          # per backward: navigation, grounding, ...
    cap = max(rows[0] + rows[1] + rows[2], rows[3] + rows[4] + rows[5])
    calls = []
    orig = ops.gemm_wgrad_seg
    monkeypatch.setattr(ops, "gemm_wgrad_seg", lambda *a, **k: (calls.append(len(a[0])), orig(*a, **k))[1])
    model.zero_grad()
    model.defer_weight_grads(cap)
    _og_rollout(model, g, cuda_dev)
    model.flush_weight_grads()
    model.defer_weight_grads(None)
    capped = _grads(model)
    n_lin = 4 * len(model.lang_model.model.layers)
    assert len(calls) > n_lin and sum(calls) == 6 * n_lin, calls     # flushed mid-rollout, every backward exactly once
    _compare_arms(model, step, capped, ref, min_backwards=6)
    model.zero_grad()
    calls.clear()
    model.defer_weight_grads(1)
    _og_rollout(model, g, cuda_dev)
    assert not model.lang_model.weight_grads_pending()
    model.defer_weight_grads(None)
    once = _grads(model)
    assert calls == []
    for n in step:
        assert torch.equal(once[n], step[n]), n
    # a backward of more than max_rows / 2 rows could not share a flush with another of its size: it runs at once, the
    # smaller ones are deferred
    big, small = max(rows), min(rows)
    assert big > small, rows
    seg_rows = []
    monkeypatch.setattr(ops, "gemm_wgrad_seg", lambda *a, **k: (seg_rows.extend(x.shape[0] for x, _ in a[0]), orig(*a, **k))[1])
    model.zero_grad()
    model.defer_weight_grads(2 * big - 1)
    _og_rollout(model, g, cuda_dev)
    model.flush_weight_grads()
    model.defer_weight_grads(None)
    mixed = _grads(model)
    n_small = sum(r <= big - 1 for r in rows)
    assert 0 < n_small < 6, rows
    assert max(seg_rows) <= big - 1 and len(seg_rows) >= n_small * n_lin, seg_rows
    _compare_arms(model, step, mixed, ref, min_backwards=6)


def test_failed_backward_leaves_the_stash_as_it_was(cuda_dev, monkeypatch):
    from navillm_b200 import ops
    g = _golden()
    model = _golden_model(g, cuda_dev)
    lm = model.lang_model
    model.zero_grad()
    model.defer_weight_grads()
    _og_rollout(model, g, cuda_dev, steps=1)
    st = lm._wgrad_stash
    before = (st.backwards, st.rows, {k: len(v) for k, v in st.pairs.items()})
    calls = []
    orig = ops.attn_bwd

    def fail_second(*a, **k):                 # layer n-1 has recorded its pairs when layer n-2's attention backward fails
        calls.append(1)
        if len(calls) == 2:
            raise RuntimeError("injected failure")
        return orig(*a, **k)
    monkeypatch.setattr(ops, "attn_bwd", fail_second)
    with pytest.raises(RuntimeError, match="injected"):
        _nav_loss(model, g, cuda_dev, 1).backward()
    assert (st.backwards, st.rows, {k: len(v) for k, v in st.pairs.items()}) == before
    monkeypatch.setattr(ops, "attn_bwd", orig)
    _nav_loss(model, g, cuda_dev, 1).backward()                  # the next backward is recorded as usual
    assert st.backwards == before[0] + 1
    model.flush_weight_grads()
    model.defer_weight_grads(None)


def test_flush_twice_equals_once_and_lazy_zero(cuda_dev):
    g = _golden()
    model = _golden_model(g, cuda_dev)
    # eager zero, deferred rollout
    model.zero_grad()
    model.defer_weight_grads()
    _og_rollout(model, g, cuda_dev, steps=2)
    model.flush_weight_grads()
    eager = _grads(model)
    model.flush_weight_grads()                                  # nothing stashed: a no-op
    assert all(torch.equal(v, eager[n]) for n, v in _grads(model).items())
    # stale gradients, lazy zero, deferred rollout: the first backward records that the linears are logically zero
    _og_rollout(model, g, cuda_dev, steps=1)
    model.flush_weight_grads()
    model.zero_grad(lazy=True)
    _og_rollout(model, g, cuda_dev, steps=2)
    assert model.lang_model._wgrad_stash.zero
    model.flush_weight_grads()
    lazy = _grads(model)
    model.defer_weight_grads(None)
    for n in eager:
        assert torch.equal(lazy[n], eager[n]), n


def test_optimizer_step_flushes_first(cuda_dev):
    from navillm_b200.optim import FlatAdamW
    g = _golden()
    params = []
    for flush_by_hand in (False, True):
        model = _golden_model(g, cuda_dev)
        opt = FlatAdamW(model, lr=1e-3)
        model.zero_grad()
        model.defer_weight_grads()
        _og_rollout(model, g, cuda_dev, steps=2)
        if flush_by_hand:
            model.flush_weight_grads()
        assert model.lang_model.weight_grads_pending() != flush_by_hand
        opt.step(max_grad_norm=40.0)
        assert not model.lang_model.weight_grads_pending()
        torch.cuda.synchronize()
        params.append({n: p.detach().clone() for n, p in model.named_parameters()})
    for n in params[0]:
        assert torch.equal(params[0][n], params[1][n]), n


def test_guards(cuda_dev):
    from navillm_b200.optim import FlatAdamW
    g = _golden()
    model = _golden_model(g, cuda_dev)
    lm = model.lang_model
    opt = FlatAdamW(model, lr=1e-3)
    model.zero_grad()
    with pytest.raises(ValueError, match="max_rows"):
        model.defer_weight_grads(-1)
    model.defer_weight_grads()
    _og_rollout(model, g, cuda_dev, steps=1)
    assert lm.weight_grads_pending()
    for zero in (lambda: model.zero_grad(), lambda: model.zero_grad(lazy=True), lambda: lm.zero_grad(), opt.zero_grad):
        with pytest.raises(RuntimeError, match="flush_weight_grads"):
            zero()
    # a weight write while rows are stashed: the next flush refuses
    with torch.no_grad():
        lm.model.layers[0].mlp.down_proj.weight.mul_(1.0)
    with pytest.raises(RuntimeError, match="weights changed"):
        model.flush_weight_grads()
    lm._wgrad_stash._clear()
    _og_rollout(model, g, cuda_dev, steps=1)
    lm.flat.generation += 1                                     # what a raw-pointer optimizer write does
    with pytest.raises(RuntimeError, match="weights changed"):
        model.flush_weight_grads()
    lm._wgrad_stash._clear()
    model.defer_weight_grads(None)


def test_armed_pass_flushes_before_exchange_and_skips_overlap(cuda_dev, monkeypatch):
    from navillm_b200 import parallel
    g = _golden()
    model = _golden_model(g, cuda_dev)
    lm = model.lang_model
    model.zero_grad()
    model.defer_weight_grads()
    _og_rollout(model, g, cuda_dev, steps=1)
    events = []
    orig_flush = lm.flush_weight_grads
    monkeypatch.setattr(lm, "flush_weight_grads", lambda: (events.append(("flush", lm.weight_grads_pending())), orig_flush())[1])
    monkeypatch.setattr(parallel.GradSync, "exchange", lambda self, covered_lm_layers=False: events.append(("exchange", covered_lm_layers)))
    orig_hook = lm._grad_sync_hook
    monkeypatch.setattr(lm, "_grad_sync_hook", lambda: (events.append("hook"), orig_hook())[1])
    loss = _nav_loss(model, g, cuda_dev, 1)
    model.grad_sync.armed = True
    loss.backward()
    assert events == [("flush", True), ("exchange", False)], events
    assert not lm.weight_grads_pending()
    model.defer_weight_grads(None)


# ------------------------------------------------------------------------------------------------------------------
# Vicuna-7B width: two decoder layers, B = 1, three steps over a PrefixKVCache(train=True)
# ------------------------------------------------------------------------------------------------------------------
def test_fullwidth_b1_rollout_deferred_matches_per_step(cuda_dev):
    import numpy as np
    from navillm_b200.modified_lm import PrefixKVCache
    from tests.test_fullwidth_parity_gpu import _full_navmodel
    sys.path.insert(0, str(ROOT / "tools"))
    from prefix_reuse_bench import make_step
    B, steps, D, G = 1, 3, 4096, 64
    model, _ = _full_navmodel(cuda_dev, base_vocab=4096)
    rng = np.random.RandomState(3)
    words = [f"w{i}" for i in range(3000)]
    instr = [" ".join(words[i] for i in rng.randint(0, 3000, size=80))]
    gh = torch.Generator().manual_seed(4)
    hist = [[torch.randn(D, generator=gh).to(cuda_dev) for _ in range(steps)]]
    target = torch.zeros(B, dtype=torch.long, device=cuda_dev)

    def run():
        r, gg = np.random.RandomState(5), torch.Generator().manual_seed(6)
        cache = PrefixKVCache(model.lang_model, batch_size=B, max_len=512, train=True)
        for t in range(steps):
            b = {k: (v.to(cuda_dev) if torch.is_tensor(v) else v) for k, v in make_step(r, gg, B, t, instr, 12, D, G).items()}
            b["hist_vis"] = [h[:t] for h in hist]
            torch.manual_seed(100 + t)
            out = model("navigation", b, prefix_cache=cache)
            F.cross_entropy(out["fuse_logits"].float(), target).backward()
        cache.flush_grads()

    model.zero_grad()
    run()
    step = _grads(model)
    model.zero_grad()
    deferred, ref = _deferred_run(model, run)
    print("max |deferred - per-step| / max|grad|:", _compare_arms(model, step, deferred, ref, min_backwards=4))
