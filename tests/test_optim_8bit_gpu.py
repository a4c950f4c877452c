"""Block-wise 8-bit AdamW moments (``FlatAdamW(model, moments="8bit")``, ``nv_adamw_flat_8bit``).

Kernel bound.  The fp64 restatement takes the kernel's inputs with m and v dequantized (map[code] * absmax, exact in
fp32), its fp32 hyper-parameters and its fp32 clipped gradient, and computes p' (and r') as tests/
test_optim_compensated_gpu.py does; the bound is that file's, with half a bf16 ulp of p' in place of an ulp of r' for the
plain update.  The codes are checked against a numpy nearest-code restatement on the fp64 moments: equal, except one code
off where the fp32 moment and the fp64 one fall on either side of a decision boundary (the fp64 value within 2^-20 of
it, relative), which must be rare.

Trajectory: tests/test_optim_compensated_gpu.py's (4 M weights, 300 steps at lr 3e-5, against torch's fp32 AdamW) with
8-bit moments.  Moment tracking: 1 M elements, 2000 steps of stationary noisy gradients (N(0, 0.3) bias + N(0, 1)) 1e-3,
beta2 = 0.999; update = m_hat / (sqrt(v_hat) + eps) of each arm against fp32 moments on the same gradient stream.
"""
import types

import numpy as np
import pytest
import torch

from tests.test_navmodel_gpu import build_model
from tests.test_optim_compensated_gpu import (_golden, _inputs, _nav_train, _residuals, _set_grads, _snapshot, _steps, adamw,
                                             bf16_ulp)

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16


def adamw8(p, g, mc, ma, vc, va, step, lr, wd, r=None, clip=None, write_clipped_grad=False, b1=0.9, b2=0.999, eps=1e-8):
    """One nv_adamw_flat_8bit step (r None: plain update), in place."""
    from navillm_b200 import _lib
    from navillm_b200._lib import check, f32, i32, i64, ptr, stream_ptr
    from navillm_b200.optim import device_maps
    check(_lib.load().nv_adamw_flat_8bit(ptr(p), ptr(r), ptr(g), ptr(mc), ptr(ma), ptr(vc), ptr(va), ptr(device_maps(p.device)),
                                         i64(p.numel()), f32(lr), f32(b1), f32(b2), f32(eps), f32(wd), i32(step), ptr(clip),
                                         i32(write_clipped_grad), stream_ptr()), "nv_adamw_flat_8bit")


def quantized(x, signed):
    """(code, absmax) of a device moment."""
    from navillm_b200.optim import QBLOCK, quantize_moment
    code = torch.empty(x.numel(), dtype=torch.uint8, device=x.device)
    absmax = torch.empty(-(-x.numel() // QBLOCK), dtype=torch.float32, device=x.device)
    quantize_moment(x.contiguous(), code, absmax, signed)
    return code, absmax


def dequantized(code, absmax, signed):
    from navillm_b200.optim import dequantize_moment
    return dequantize_moment(code, absmax, torch.float32, signed)


def np_codes(x, signed):
    """Nearest code of x / absmax per 64-element block (fp64 x), a tie to the smaller magnitude; an all-zero block: code 0.
    Returns (codes, absmax)."""
    from navillm_b200.optim import M_ZERO, code_maps
    smap, umap = (m.astype(np.float64) for m in code_maps())
    n = x.size
    nb = -(-n // 64)
    xp = np.zeros(nb * 64)
    xp[:n] = x
    blocks = xp.reshape(nb, 64)
    amax = np.abs(blocks).max(1)
    y = np.divide(blocks, amax[:, None], out=np.zeros_like(blocks), where=amax[:, None] > 0)
    tab = smap[M_ZERO:] if signed else umap
    a = np.abs(y)
    i = np.clip(np.searchsorted(tab, a, side="right") - 1, 0, len(tab) - 1)
    up = np.minimum(i + 1, len(tab) - 1)
    k = np.where((up > i) & (tab[up] - a < a - tab[i]), up, i)
    code = np.where((y < 0) & (k > 0), M_ZERO - 1 - k, M_ZERO + k) if signed else k
    code[amax == 0] = 0
    return code.reshape(-1)[:n].astype(np.int64), amax


def ordinal(code, signed):
    """Position among the codes the quantizer produces (the signed map's spare code 127 is skipped)."""
    code = code.astype(np.int64)
    return np.where(code > 127, code - 1, code) if signed else code


def _inputs8(step, dev, n=(1 << 20) + 37):
    """_inputs' p, r, g with m and v in 8-bit form; block 3 is all zero (gradient and moments), n % 64 = 37."""
    p, r, g, m, v = _inputs(step, n=n)
    g[192:256] = 0
    m[192:256] = 0
    v[192:256] = 0
    mc, ma = quantized(m.to(dev), True)
    vc, va = quantized(v.to(dev), False)
    return p.to(dev), r.to(dev), g.to(dev), mc, ma, vc, va


def _run8(inputs, step, lr, wd, compensated, clip=None, write_clipped_grad=False):
    p, r, g, mc, ma, vc, va = (t.clone() for t in inputs)
    state = None if clip is None else torch.tensor([1.0, clip], dtype=torch.float32, device=p.device)
    adamw8(p, g, mc, ma, vc, va, step, lr, wd, r=r if compensated else None, clip=state, write_clipped_grad=write_clipped_grad)
    torch.cuda.synchronize()
    return p, r, g, mc, ma, vc, va


@pytest.mark.parametrize("step", [1, 50])
@pytest.mark.parametrize("compensated", [False, True])
@pytest.mark.parametrize("clip,write_clipped_grad", [(None, False), (0.37, False), (0.37, True)])
def test_kernel_against_fp64(cuda_dev, step, compensated, clip, write_clipped_grad):
    from navillm_b200.optim import code_maps
    lr, wd = 1e-3, 0.01
    inputs = _inputs8(step, cuda_dev)
    p0, r0, g0, mc0, ma0, vc0, va0 = inputs
    m0, v0 = dequantized(mc0, ma0, True).double().cpu(), dequantized(vc0, va0, False).double().cpu()
    pk, rk, gk, mck, mak, vck, vak = (t.cpu() for t in _run8(inputs, step, lr, wd, compensated, clip, write_clipped_grad))

    h = lambda a: torch.tensor(a, dtype=torch.float32).double()          # the kernel's fp32 hyper-parameters
    b1, b2, eps, lr_, wd_ = h(0.9), h(0.999), h(1e-8), h(lr), h(wd)
    g32 = g0.float().cpu() * (torch.tensor(clip, dtype=torch.float32) if clip is not None else 1.0)
    gi = g32.double()
    m2 = m0 + (1 - b1) * (gi - m0)
    v2 = b2 * v0 + (1 - b2) * gi * gi
    bc1, bc2s = 1 - b1 ** step, torch.sqrt(1 - b2 ** step)
    denom = v2.sqrt() / bc2s + eps
    u = lr_ / bc1 * m2 / denom
    x = p0.double().cpu() + (r0.double().cpu() if compensated else 0)
    x64 = x * (1 - lr_ * wd_) - u
    fp32_terms = 2.0 ** -22 * (x.abs() + u.abs()) + 2.0 ** -18 * u.abs() + 2.0 ** -20 * lr_ / bc1 * (m0.abs() + gi.abs()) / denom
    if compensated:
        err, bound = (pk.double() + rk.double() - x64).abs(), bf16_ulp(rk).double() + fp32_terms + 1e-30
        assert torch.equal((pk.float() + rk.float()).to(BF16).float(), pk.float())
    else:
        err, bound = (pk.double() - x64).abs(), bf16_ulp(pk).double() / 2 + fp32_terms + 1e-30
        assert torch.equal(rk.view(torch.int16), r0.cpu().view(torch.int16))
    worst = int(torch.argmax(err / bound))
    assert bool((err <= bound).all()), (worst, float(err[worst]), float(bound[worst]), float(x64[worst]))

    # the clipped gradient is left behind only when asked
    assert torch.equal(gk.view(torch.int16), (g32.to(BF16) if write_clipped_grad else g0.cpu()).view(torch.int16))

    # codes and absmax against the nearest-code restatement of the fp64 moments
    for name, new, code, amax, signed in (("m", m2, mck, mak, True), ("v", v2, vck, vak, False)):
        want, want_amax = np_codes(new.numpy(), signed)
        got = code.numpy().astype(np.int64)
        assert np.allclose(amax.double().numpy(), want_amax, rtol=2 ** -20, atol=0), name
        diff = np.abs(ordinal(got, signed) - ordinal(want, signed))
        off = np.nonzero(diff)[0]
        print(f"{name}: {off.size} of {got.size} codes one off the fp64 restatement")
        assert diff.max() <= 1 and off.size <= got.size * 2e-3, (name, off.size, int(diff.max()))
        # each of them: the fp64 y lies on the boundary between the two codes to within the fp32 error of the kernel's y
        # (step 1 makes exact ties: y = g / max|g| over bf16 gradients often is a midpoint of the map)
        mp = code_maps()[0 if signed else 1].astype(np.float64)
        y = new.numpy()[off] / want_amax[off // 64]
        mid = (mp[got[off]] + mp[want[off]]) / 2
        assert np.all(np.abs(y - mid) <= 2.0 ** -20 * np.abs(y)), (name, off[np.argmax(np.abs(y - mid) / np.abs(y))])
        if signed:
            assert not np.any(got == 127), "the spare code was produced"
        assert amax[3] == 0 and not np.any(got[192:256]), name          # the all-zero block: absmax 0, code 0
        assert (amax > 0).sum() == amax.numel() - 1, name


@pytest.mark.parametrize("compensated", [False, True])
@pytest.mark.parametrize("clip,write_clipped_grad", [(None, False), (0.37, True)])
def test_first_step_equals_the_bf16_moment_step(cuda_dev, compensated, clip, write_clipped_grad):
    """From zero moments both kernels compute p' from the same fp32 m' and v': p (and r) bit for bit."""
    p, r, g, _, _ = (t.to(cuda_dev) for t in _inputs(1))
    n = p.numel()
    state = None if clip is None else torch.tensor([1.0, clip], dtype=torch.float32, device=cuda_dev)
    zeros8 = lambda: (torch.zeros(n, dtype=torch.uint8, device=cuda_dev), torch.zeros(-(-n // 64), device=cuda_dev))
    p8, r8, g8 = p.clone(), r.clone(), g.clone()
    (mc, ma), (vc, va) = zeros8(), zeros8()
    adamw8(p8, g8, mc, ma, vc, va, 1, 1e-3, 0.01, r=r8 if compensated else None, clip=state,
           write_clipped_grad=write_clipped_grad)
    pb, rb, gb = p.clone(), r.clone(), g.clone()
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    adamw(pb, gb, m, v, 1, 1e-3, 0.01, r=rb if compensated else None, clip=state, write_clipped_grad=write_clipped_grad)
    torch.cuda.synchronize()
    for a, b in ((p8, pb), (r8, rb), (g8, gb)):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def test_quantize_round_trip(cuda_dev):
    """quantize -> dequantize -> quantize is the identity on the codes; a block's absmax element is exact."""
    gen = torch.Generator(device=cuda_dev).manual_seed(3)
    for signed in (True, False):
        x = torch.randn(64 * 1000 + 11, generator=gen, device=cuda_dev) * 1e-3
        x = x if signed else x * x
        code, amax = quantized(x, signed)
        y = dequantized(code, amax, signed)
        code2, amax2 = quantized(y, signed)
        assert torch.equal(code, code2) and torch.equal(amax, amax2)
        blk = torch.nn.functional.pad(x.abs(), (0, 64 - x.numel() % 64)).view(-1, 64)
        assert torch.equal(amax, blk.max(1).values)
        assert float((y - x).abs().max()) <= float(amax.max()) * 0.02


def trajectory8(dev, n=1 << 22, steps=300, lr=3e-5, wd=0.01, seed=0):
    """tests/test_optim_compensated_gpu.py::trajectory's setup with 8-bit moments: the compensated and plain updates
    against torch.optim.AdamW on an fp32 copy.  Drift ratio and relative drift error per arm."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    n_one = n // 256
    w0 = torch.randn(n, generator=gen, device=dev) * 0.02
    w0[-n_one:] = 1.0
    w0 = w0.to(BF16)
    bias = torch.randn(n, generator=gen, device=dev) * 0.3
    w32 = torch.nn.Parameter(w0.float())
    ref = torch.optim.AdamW([w32], lr=lr, weight_decay=wd)
    zeros = lambda: torch.zeros(n, dtype=BF16, device=dev)
    codes = lambda: [torch.zeros(n, dtype=torch.uint8, device=dev), torch.zeros(n // 64, device=dev),
                     torch.zeros(n, dtype=torch.uint8, device=dev), torch.zeros(n // 64, device=dev)]
    arms = {"compensated_8bit": [w0.clone(), zeros(), *codes()], "plain_8bit": [w0.clone(), None, *codes()]}
    for t in range(1, steps + 1):
        scale = 1e-3 if t <= steps // 2 else 1e-4
        g = ((bias + torch.randn(n, generator=gen, device=dev)) * scale).to(BF16)
        for p, r, mc, ma, vc, va in arms.values():
            adamw8(p, g, mc, ma, vc, va, t, lr, wd, r=r)
        w32.grad = g.float()
        ref.step()
    torch.cuda.synchronize()
    d_ref = w32.detach().double() - w0.double()
    out = {}
    for name, (p, r, *_) in arms.items():
        d = p.double() + (0 if r is None else r.double()) - w0.double()
        out[name] = {"drift_ratio": float(d.abs().sum() / d_ref.abs().sum()),
                     "rel_err": float((d - d_ref).norm() / d_ref.norm())}
    return out


def test_trajectory_against_fp32_adamw(cuda_dev):
    res = trajectory8(cuda_dev)
    print(res)
    c = res["compensated_8bit"]
    assert 0.95 <= c["drift_ratio"] <= 1.05 and c["rel_err"] <= 0.05, res


def moment_tracking(dev, n=1 << 20, steps=2000, seed=0, b1=0.9, b2=0.999, eps=1e-8):
    """bf16 and 8-bit moments against fp32 ones on one stream of stationary noisy gradients (lr 0, so only the moments
    move).  Per arm: relative L2 error of the update m_hat / (sqrt(v_hat) + eps) and median |v / v32 - 1|."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    bias = torch.randn(n, generator=gen, device=dev) * 0.3
    m32, v32 = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    p = torch.zeros(n, dtype=BF16, device=dev)
    mb, vb = torch.zeros(n, dtype=BF16, device=dev), torch.zeros(n, dtype=BF16, device=dev)
    mc, vc = torch.zeros(n, dtype=torch.uint8, device=dev), torch.zeros(n, dtype=torch.uint8, device=dev)
    ma, va = torch.zeros(n // 64, device=dev), torch.zeros(n // 64, device=dev)
    for t in range(1, steps + 1):
        g = ((bias + torch.randn(n, generator=gen, device=dev)) * 1e-3).to(BF16)
        gf = g.float()
        m32.lerp_(gf, 1 - b1)
        v32.mul_(b2).addcmul_(gf, gf, value=1 - b2)
        adamw(p, g.clone(), mb, vb, t, 0.0, 0.0)
        adamw8(p, g.clone(), mc, ma, vc, va, t, 0.0, 0.0)
    torch.cuda.synchronize()
    bc1, bc2 = 1 - b1 ** steps, 1 - b2 ** steps
    upd = lambda m, v: (m.double() / bc1) / ((v.double() / bc2).sqrt() + eps)
    u32 = upd(m32, v32)
    out = {}
    for name, (m, v) in {"bf16": (mb.float(), vb.float()),
                         "8bit": (dequantized(mc, ma, True), dequantized(vc, va, False))}.items():
        out[name] = {"update_rel_err": float((upd(m, v) - u32).norm() / u32.norm()),
                     "v_median_rel_err": float((v.double() / v32.double() - 1).abs().median())}
    return out


def test_moment_tracking_against_fp32_moments(cuda_dev):
    res = moment_tracking(cuda_dev)
    print(res)
    assert res["8bit"]["update_rel_err"] < res["bf16"]["update_rel_err"], res


# ---- model level ------------------------------------------------------------------------------------------------------

def _codes(opt):
    return [t.cpu().clone() for t in (opt.m_code, opt.m_absmax, opt.v_code, opt.v_absmax)]


def test_model_training_is_deterministic(cuda_dev):
    from navillm_b200.optim import FlatAdamW
    g = _golden()
    runs = []
    for _ in range(2):
        model, _ = build_model(g, cuda_dev)
        opt = FlatAdamW(model, lr=3e-5, compensated=True, moments="8bit")
        _nav_train(model, g, cuda_dev, opt)
        # the residual's per-parameter views: the flat buffer's alignment padding holds no parameter and is not compared
        runs.append([p.detach().cpu().clone() for p in model.parameters()] + [r.cpu().clone() for r in _residuals(opt)]
                    + _codes(opt))
    assert bool(runs[0][-4].any()) and bool(runs[0][-3].any())
    for a, b in zip(*runs):
        assert torch.equal(a.view(torch.int16) if a.dtype == BF16 else a, b.view(torch.int16) if b.dtype == BF16 else b)


@pytest.mark.parametrize("compensated", [False, True])
def test_checkpoint_resume_and_state_interop(cuda_dev, tmp_path, compensated):
    from navillm_b200.checkpoint import check_checkpoint, save_checkpoint
    from navillm_b200.optim import FlatAdamW
    g = _golden()
    model, _ = build_model(g, cuda_dev)
    opt = FlatAdamW(model, lr=3e-5, compensated=compensated, moments="8bit")
    _steps(model, opt, [1, 2])
    path = tmp_path / "ckpt.pt"
    save_checkpoint(model, path, opt, epoch=0, save_states=True)
    sd = _snapshot(opt)
    _steps(model, opt, [3])

    # save -> resume into a fresh model and optimizer: the next step is bit for bit the uninterrupted one
    fresh, _ = build_model(g, cuda_dev)
    opt2 = FlatAdamW(fresh, lr=3e-5, compensated=compensated, moments="8bit")
    assert check_checkpoint(types.SimpleNamespace(resume_from_checkpoint=str(path)), fresh, opt2) == 1
    _steps(fresh, opt2, [3])
    for a, b in zip(model.parameters(), fresh.parameters()):
        assert torch.equal(a.detach(), b.detach())
    for a, b in zip(_codes(opt), _codes(opt2)):
        assert torch.equal(a, b)
    for a, b in zip(_residuals(opt), _residuals(opt2)):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))

    params = [p for p in fresh.parameters() if p.requires_grad]
    bf16_idx = next(i for i, p in enumerate(params) if p.dtype == BF16)
    f32_idx = next(i for i, p in enumerate(params) if p.dtype == torch.float32)
    st = sd["state"][bf16_idx]
    assert st["exp_avg"].device.type == "cpu" and st["exp_avg"].dtype == BF16 and st["exp_avg"].shape == params[bf16_idx].shape
    assert st["exp_avg_code"].dtype == torch.uint8 and st["exp_avg_absmax"].dtype == torch.float32
    assert "exp_avg_code" not in sd["state"][f32_idx] and sd["state"][f32_idx]["exp_avg"].dtype == torch.float32

    # a bf16 FlatAdamW takes the dequantized moments and steps
    plain = FlatAdamW(fresh, lr=3e-5)
    plain.load_state_dict(sd)
    assert torch.equal(plain.state_dict()["state"][bf16_idx]["exp_avg"].cpu(), st["exp_avg"])
    _set_grads(fresh, 4)
    plain.step(max_grad_norm=40.0)

    # torch.optim.AdamW loads the 8-bit state and steps
    topt = torch.optim.AdamW(params, lr=3e-5)
    topt.load_state_dict(_snapshot(opt2))
    _set_grads(fresh, 5)
    topt.step()
    torch.cuda.synchronize()

    # a torch state (its copies of the absmax were cast to bf16) and a bf16 FlatAdamW state load into an 8-bit optimizer by
    # quantizing exp_avg / exp_avg_sq: their dequantized moments are those moments to within the code spacing
    for src in (topt.state_dict(), plain.state_dict()):
        opt3 = FlatAdamW(fresh, lr=3e-5, compensated=compensated, moments="8bit")
        opt3.load_state_dict(src)
        back = opt3.state_dict()["state"][bf16_idx]
        for key in ("exp_avg", "exp_avg_sq"):
            want = src["state"][bf16_idx][key].float().cpu()
            tol = 0.05 * want.abs().max() + 1e-30
            assert float((back[key].float() - want).abs().max()) <= float(tol), key
        _set_grads(fresh, 6)
        opt3.step(max_grad_norm=40.0)
    torch.cuda.synchronize()


def test_memory(cuda_dev):
    from navillm_b200.optim import FlatAdamW
    g = _golden()
    model, _ = build_model(g, cuda_dev)
    model._ensure()
    n16 = model.lang_model.flat.flat.numel()
    for compensated in (False, True):
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        opt = FlatAdamW(model, lr=3e-5, compensated=compensated, moments="8bit")
        torch.cuda.synchronize()
        grown = torch.cuda.memory_allocated() - before
        sb = opt.state_bytes()
        # the rest: clip partials and state, the 2 KB maps (first use on the device), allocator rounding
        assert sb <= grown <= sb + (1 << 20), (grown, sb)
        lm_bytes = sb - sum(t.numel() * t.element_size() for t in opt.m + opt.v if t is not None)
        if compensated:
            lm_bytes -= 2 * n16
        assert lm_bytes <= 2.13 * n16, (lm_bytes, n16)
        del opt
