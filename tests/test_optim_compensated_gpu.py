"""The error-compensated AdamW step (``FlatAdamW(model, compensated=True)``, ``nv_adamw_flat_compensated``).

Kernel bound, stated.  The fp64 reference takes the kernel's inputs, its fp32 hyper-parameters and its fp32 clipped
gradient gi = fl(g * coef), and computes m', v', u = lr / bc1 * m' / (sqrt(v') / bc2s + eps) and x64 = (p + r)(1 - lr wd) - u
in fp64.  The kernel's pair (p', r') may differ from x64 by
  * one bf16 ulp of r': r' is x' - p' rounded to bf16 (to nearest, toward zero where the pair would otherwise round away
    from p'), so it keeps at most 8 of the difference's bits;
  * 2^-22 (|x| + |u|): the fp32 decay factor and product and the final fp32 rounding of x' (each 2^-24 relative);
  * 2^-18 |u|: the fp32 bias corrections (1 - beta2^step loses ~20 ulp to cancellation at step 50), the approximate
    sqrt and reciprocals of --use_fast_math (a few ulp each) and the fp32 roundings of v';
  * 2^-20 lr / bc1 (|m| + |gi|) / denom: the fp32 roundings of the m' lerp, absolute because m' may cancel to near zero.
The bound is dominated by ulp(r') ~ 2^-16 |p|; at lr 1e-3 the update is ~2^6 times larger than that.

Trajectory: 4 M bf16 weights, 300 steps at lr 3e-5 and weight decay 0.01 (the reference's training settings) against
torch.optim.AdamW on an fp32 copy.  The moments stay bf16 in both arms, as in the plain kernel.  drift = final - initial weight; drift ratio = sum |drift| / sum |drift_fp32|, relative
drift error = ||drift - drift_fp32||_2 / ||drift_fp32||_2.
"""
import copy
import types

import pytest
import torch
import torch.nn.functional as F

from tests.test_navmodel_gpu import GOLD, build_model, to_dev

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16


def adamw(p, g, m, v, step, lr, wd, r=None, clip=None, write_clipped_grad=False, b1=0.9, b2=0.999, eps=1e-8):
    """One nv_adamw_flat (r None) or nv_adamw_flat_compensated step over bf16 vectors, in place."""
    from navillm_b200 import _lib
    from navillm_b200._lib import check, f32, i32, i64, ptr, stream_ptr
    lib = _lib.load()
    tail = (f32(lr), f32(b1), f32(b2), f32(eps), f32(wd), i32(step), ptr(clip), i32(write_clipped_grad), stream_ptr())
    if r is None:
        check(lib.nv_adamw_flat(ptr(p), ptr(g), ptr(m), ptr(v), i64(p.numel()), i32(1), *tail), "nv_adamw_flat")
    else:
        check(lib.nv_adamw_flat_compensated(ptr(p), ptr(r), ptr(g), ptr(m), ptr(v), i64(p.numel()), *tail),
              "nv_adamw_flat_compensated")


def bf16_ulp(t):
    """bf16 ulp of each element of a float tensor (0 for zeros)."""
    _, e = torch.frexp(t.float())
    return torch.where(t == 0, torch.zeros_like(t.float()), torch.ldexp(torch.ones_like(t.float()), e - 8))


def _inputs(step, n=(1 << 20) + 5, seed=0):
    """p ~ N(0, 0.02) with an eighth near 1.0, r within +-half an ulp of p, and g, m, v as at `step`.  Signed zeros and a
    subnormal with zero gradient and moments sit in the vectorised body and in the scalar tail (n % 8 = 5)."""
    gen = torch.Generator().manual_seed(seed + step)
    p = torch.randn(n, generator=gen) * 0.02
    p[: n // 8] = 1.0 + torch.randn(n // 8, generator=gen) * 0.01
    p = p.to(BF16)
    r = ((torch.rand(n, generator=gen) * 2 - 1) * 0.99 * bf16_ulp(p) / 2).to(BF16)
    g = (torch.randn(n, generator=gen) * 1e-3).to(BF16)
    if step == 1:
        m, v = torch.zeros(n, dtype=BF16), torch.zeros(n, dtype=BF16)
    else:
        m = (torch.randn(n, generator=gen) * 5e-4).to(BF16)
        v = ((torch.rand(n, generator=gen) * 1.5 + 0.5) * 1e-6).to(BF16)
    for idx in (n // 2, n - 3):
        p[idx:idx + 3] = torch.tensor([-0.0, 0.0, 1e-39]).to(BF16)
        for t in (r, g, m, v):
            t[idx:idx + 3] = 0
    return p, r, g, m, v


def _run(inputs, dev, step, lr, wd, compensated, clip=None, write_clipped_grad=False):
    p, r, g, m, v = (t.to(dev) for t in inputs)
    state = None if clip is None else torch.tensor([1.0, clip], dtype=torch.float32, device=dev)
    adamw(p, g, m, v, step, lr, wd, r=r if compensated else None, clip=state, write_clipped_grad=write_clipped_grad)
    torch.cuda.synchronize()
    return p.cpu(), r.cpu(), g.cpu(), m.cpu(), v.cpu()


@pytest.mark.parametrize("step", [1, 50])
@pytest.mark.parametrize("lr", [1e-3, 3e-5])
def test_kernel_against_fp64(cuda_dev, step, lr):
    wd, coef = 0.01, 0.37
    inputs = _inputs(step)
    pc, rc, _, mc, vc = _run(inputs, cuda_dev, step, lr, wd, True, clip=coef)
    _, _, _, mp, vp = _run(inputs, cuda_dev, step, lr, wd, False, clip=coef)
    assert torch.equal(mc.view(torch.int16), mp.view(torch.int16)) and torch.equal(vc.view(torch.int16), vp.view(torch.int16))
    # the pair is canonical: p' is the bf16 rounding of the master value p' + r' (the fp32 sum is exact; -0 + 0 = +0 counts
    # as p' = -0)
    assert torch.equal((pc.float() + rc.float()).to(BF16).float(), pc.float())

    p, r, g, m, v = (t.double() for t in inputs)
    h = lambda a: torch.tensor(a, dtype=torch.float32).double()          # the kernel's fp32 hyper-parameters
    b1, b2, eps, lr_, wd_ = h(0.9), h(0.999), h(1e-8), h(lr), h(wd)
    gi = (inputs[2].float() * torch.tensor(coef, dtype=torch.float32)).double()
    m2 = m + (1 - b1) * (gi - m)
    v2 = b2 * v + (1 - b2) * gi * gi
    bc1, bc2s = 1 - b1 ** step, torch.sqrt(1 - b2 ** step)
    denom = v2.sqrt() / bc2s + eps
    u = lr_ / bc1 * m2 / denom
    x = p + r
    x64 = x * (1 - lr_ * wd_) - u
    bound = (bf16_ulp(rc).double() + 2.0 ** -22 * (x.abs() + u.abs()) + 2.0 ** -18 * u.abs()
             + 2.0 ** -20 * lr_ / bc1 * (m.abs() + gi.abs()) / denom + 1e-30)
    err = (pc.double() + rc.double() - x64).abs()
    worst = int(torch.argmax(err / bound))
    assert bool((err <= bound).all()), (worst, float(err[worst]), float(bound[worst]), float(x64[worst]))
    # and the pair resolves the update far below bf16: the plain kernel's error is ~2^8 larger
    pp = _run(inputs, cuda_dev, step, lr, wd, False, clip=coef)[0]
    assert float(err.max()) * 16 < float((pp.double() - x64).abs().max())


@pytest.mark.parametrize("step", [1, 50])
@pytest.mark.parametrize("clip,write_clipped_grad", [(None, False), (0.37, False), (0.37, True)])
def test_zero_residual_is_the_plain_step(cuda_dev, step, clip, write_clipped_grad):
    p, r, g, m, v = _inputs(step)
    r.zero_()
    inputs = (p, r, g, m, v)
    pc, rc, gc, mc, vc = _run(inputs, cuda_dev, step, 1e-3, 0.01, True, clip, write_clipped_grad)
    pp, _, gp, mp, vp = _run(inputs, cuda_dev, step, 1e-3, 0.01, False, clip, write_clipped_grad)
    for a, b in ((pc, pp), (gc, gp), (mc, mp), (vc, vp)):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    assert torch.equal((pc.float() + rc.float()).to(BF16).float(), pc.float())


def test_misaligned_operands_are_rejected(cuda_dev):
    from navillm_b200._lib import NvError
    p, r, g, m, v = (t.to(cuda_dev) for t in _inputs(1, n=64))
    with pytest.raises(NvError, match="16-byte aligned"):
        adamw(p[1:], g[1:], m[1:], v[1:], 1, 1e-3, 0.01, r=r[1:])


def trajectory(dev, n=1 << 22, steps=300, lr=3e-5, wd=0.01, seed=0):
    """Plain and compensated bf16 AdamW against torch.optim.AdamW on an fp32 copy, from the same bf16 start and the same
    bf16 gradients: N(0, 0.02) weights with the last 1/256 at 1.0 (RMSNorm-like; they are 0.004 % of Vicuna-7B), gradients
    with a constant per-element bias under fresh noise, scaled down 10x halfway.  Returns, per arm, the drift ratio and
    relative drift error over all weights and over the 1.0 block alone, and whether the plain arm left that block
    bit-identical."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    n_one = n // 256
    w0 = torch.randn(n, generator=gen, device=dev) * 0.02
    w0[-n_one:] = 1.0
    w0 = w0.to(BF16)
    bias = torch.randn(n, generator=gen, device=dev) * 0.3
    w32 = torch.nn.Parameter(w0.float())
    ref = torch.optim.AdamW([w32], lr=lr, weight_decay=wd)
    zeros = lambda: torch.zeros(n, dtype=BF16, device=dev)
    arms = {"plain": [w0.clone(), None, zeros(), zeros()], "compensated": [w0.clone(), zeros(), zeros(), zeros()]}
    for t in range(1, steps + 1):
        scale = 1e-3 if t <= steps // 2 else 1e-4
        g = ((bias + torch.randn(n, generator=gen, device=dev)) * scale).to(BF16)
        for p, r, m, v in arms.values():
            adamw(p, g, m, v, t, lr, wd, r=r)
        w32.grad = g.float()
        ref.step()
    torch.cuda.synchronize()
    d_ref = w32.detach().double() - w0.double()
    out = {}
    for name, (p, r, _, _) in arms.items():
        d = p.double() + (0 if r is None else r.double()) - w0.double()
        stats = {}
        for part, sl in (("", slice(0, n)), ("ones_", slice(n - n_one, n))):
            stats[part + "drift_ratio"] = float(d[sl].abs().sum() / d_ref[sl].abs().sum())
            stats[part + "rel_err"] = float((d[sl] - d_ref[sl]).norm() / d_ref[sl].norm())
        out[name] = stats
    out["plain_ones_unchanged"] = torch.equal(arms["plain"][0][-n_one:], w0[-n_one:])
    return out


def test_trajectory_against_fp32_adamw(cuda_dev):
    res = trajectory(cuda_dev)
    c, p = res["compensated"], res["plain"]
    assert 0.98 <= c["drift_ratio"] <= 1.02 and c["rel_err"] <= 0.02, res
    assert p["rel_err"] >= 0.5 and res["plain_ones_unchanged"], res      # the defect the mode removes is visible here
    # near 1.0 the pair holds ~16 bits (2^-17 resolution against steps of ~1e-5), so these weights move, but ~8 % short
    assert c["ones_drift_ratio"] >= 0.85, res


# ---- model level ------------------------------------------------------------------------------------------------------

def _golden():
    return torch.load(GOLD / "nav_amp_bf16.pt", weights_only=False)


def _nav_train(model, g, dev, opt, iters=5):
    """Navigation forward + action CE + backward + clipped step, `iters` times (tests/test_navmodel_gpu.py's inputs)."""
    B = g["targets"].shape[0]
    for it in range(iters):
        model.zero_grad()
        pano = model("panorama", to_dev(dict(g["pano_in"]), dev))
        nav_in = to_dev(dict(g["nav_in"]), dev)
        nav_in["vp_img_embeds"] = torch.cat([torch.zeros_like(pano["pano_embeds"][:, :1]), pano["pano_embeds"]], 1)
        nav_in["pano_masks"] = torch.cat([torch.ones(B, 1, dtype=torch.bool, device=dev), pano["pano_masks"]], 1)
        torch.manual_seed(1234 + it)
        nav = model("navigation", nav_in)
        loss = F.cross_entropy(nav["fuse_logits"].float(), g["targets"].to(dev), reduction="sum", ignore_index=-100) / B
        loss.backward()
        opt.step(max_grad_norm=40.0)
    torch.cuda.synchronize()


def _residuals(opt):
    """The residual's per-parameter views (the flat buffer's alignment padding holds no parameter and is not compared)."""
    return [st["weight_residual"] for st in opt.state_dict()["state"].values() if "weight_residual" in st]


def test_model_training_is_deterministic(cuda_dev):
    from navillm_b200.optim import FlatAdamW
    g = _golden()
    runs = []
    for _ in range(2):
        model, _ = build_model(g, cuda_dev)
        opt = FlatAdamW(model, lr=3e-5, compensated=True)
        _nav_train(model, g, cuda_dev, opt)
        runs.append(([p.detach().cpu().clone() for p in model.parameters()], [r.cpu().clone() for r in _residuals(opt)]))
    (pa, ra), (pb, rb) = runs
    assert any(bool(r.any()) for r in ra)
    for a, b in zip(pa + ra, pb + rb):
        assert torch.equal(a.view(torch.int16) if a.dtype == BF16 else a, b.view(torch.int16) if b.dtype == BF16 else b)


@pytest.mark.parametrize("compensated", [False, True])
def test_step_invalidates_fp8_copy_and_training_cache(cuda_dev, compensated):
    from navillm_b200.modified_lm import PrefixKVCache
    from navillm_b200.optim import FlatAdamW
    from tests.test_prefix_reuse_gpu import _build
    from tests.test_prefix_train_gpu import _rollout
    model, d = _build(cuda_dev)
    lm = model.lang_model
    opt = FlatAdamW(model, lr=3e-5, compensated=compensated)
    model.quantize_weights_fp8()
    assert lm.fp8_weights.stale_reason(lm.flat) is None
    opt.step()
    assert lm.fp8_weights.stale_reason(lm.flat) is not None
    model.drop_fp8_weights()
    cache = PrefixKVCache(lm, batch_size=2, max_len=256, train=True)
    _rollout(model, d, cuda_dev, cache, steps=2, flush=False)
    opt.step()
    with pytest.raises(RuntimeError, match="weights changed"):
        cache.flush_grads()


def _set_grads(model, seed):
    gen = torch.Generator().manual_seed(seed)
    for p in model.parameters():
        p.grad.copy_((torch.randn(p.shape, generator=gen) * 1e-2).to(p.dtype))


def _steps(model, opt, seeds):
    for s in seeds:
        _set_grads(model, s)
        opt.step(max_grad_norm=40.0)
    torch.cuda.synchronize()


def _snapshot(opt, drop_residual=False):
    sd = opt.state_dict()
    return {"state": {i: {k: t.clone() for k, t in st.items() if not (drop_residual and k == "weight_residual")}
                      for i, st in sd["state"].items()},
            "param_groups": copy.deepcopy(sd["param_groups"])}


def _same(model_a, opt_a, model_b, opt_b):
    for a, b in zip(model_a.parameters(), model_b.parameters()):
        assert torch.equal(a.detach(), b.detach())
    for a, b in zip(_residuals(opt_a), _residuals(opt_b)):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))


@pytest.mark.parametrize("writer", ["load_state_dict", "quantize_weights_fp8"])
def test_foreign_write_resets_the_residual(cuda_dev, writer):
    """After a write the optimizer did not make, the next step is that of a compensated optimizer with a zero residual."""
    from navillm_b200.optim import FlatAdamW
    g = _golden()
    model, _ = build_model(g, cuda_dev)
    opt = FlatAdamW(model, lr=3e-5, compensated=True)
    _steps(model, opt, [1, 2])
    assert any(bool(r.any()) for r in _residuals(opt))
    if writer == "load_state_dict":
        model.load_state_dict({k: t.clone() for k, t in model.state_dict().items()})
    else:
        model.quantize_weights_fp8()
    weights, sd = {k: t.clone() for k, t in model.state_dict().items()}, _snapshot(opt, drop_residual=True)
    _steps(model, opt, [3])

    fresh, _ = build_model(g, cuda_dev)
    fresh.load_state_dict(weights)
    opt2 = FlatAdamW(fresh, lr=3e-5, compensated=True)
    opt2.load_state_dict(sd)
    assert not bool(opt2.residual.any())
    _steps(fresh, opt2, [3])
    _same(model, opt, fresh, opt2)


def test_checkpoint_resume_and_state_interop(cuda_dev, tmp_path):
    from navillm_b200.checkpoint import check_checkpoint, save_checkpoint
    from navillm_b200.optim import FlatAdamW
    g = _golden()
    model, _ = build_model(g, cuda_dev)
    opt = FlatAdamW(model, lr=3e-5, compensated=True)
    _steps(model, opt, [1, 2])
    path = tmp_path / "ckpt.pt"
    save_checkpoint(model, path, opt, epoch=0, save_states=True)
    sd = _snapshot(opt)
    _steps(model, opt, [3])

    # save -> resume into a fresh model and optimizer: the next step is bit for bit the uninterrupted one
    fresh, _ = build_model(g, cuda_dev)
    opt2 = FlatAdamW(fresh, lr=3e-5, compensated=True)
    assert check_checkpoint(types.SimpleNamespace(resume_from_checkpoint=str(path)), fresh, opt2) == 1
    _steps(fresh, opt2, [3])
    _same(model, opt, fresh, opt2)

    params = [p for p in fresh.parameters() if p.requires_grad]
    names = [n for n, p in fresh.named_parameters() if p.requires_grad]
    bf16_idx = next(i for i, p in enumerate(params) if p.dtype == BF16)
    f32_idx = next(i for i, p in enumerate(params) if p.dtype == torch.float32)
    assert "weight_residual" in sd["state"][bf16_idx] and "weight_residual" not in sd["state"][f32_idx], names[f32_idx]

    # a plain FlatAdamW takes the moments and ignores the residual
    plain = FlatAdamW(fresh, lr=3e-5)
    plain.load_state_dict(sd)
    assert plain.residual is None and "weight_residual" not in plain.state_dict()["state"][bf16_idx]
    assert torch.equal(plain.state_dict()["state"][bf16_idx]["exp_avg"], sd["state"][bf16_idx]["exp_avg"])

    # torch.optim.AdamW loads the compensated state and steps
    topt = torch.optim.AdamW(params, lr=3e-5)
    topt.load_state_dict(_snapshot(opt2))
    _set_grads(fresh, 4)
    topt.step()
    torch.cuda.synchronize()

    # a torch AdamW state loads into a compensated FlatAdamW with a zero residual
    tsd = topt.state_dict()
    tsd = {"state": {i: {k: t for k, t in st.items() if k != "weight_residual"} for i, st in tsd["state"].items()},
           "param_groups": tsd["param_groups"]}
    assert any(bool(r.any()) for r in _residuals(opt2))
    opt2.load_state_dict(tsd)
    assert not bool(opt2.residual.any())
    assert torch.equal(opt2.state_dict()["state"][bf16_idx]["exp_avg"], tsd["state"][bf16_idx]["exp_avg"])
