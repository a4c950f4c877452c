"""The attention bounds of tests/test_train_kernels_gpu.py §1 at a key offset have teeth: on the CPU, at H = 2 and a few
hundred rows, an fp32 emulation of the KV-cache kernels' rounding points passes them and each of five plausible kernel
mistakes fails them.

The emulation follows nv_attn_fwd_kv / nv_attn_bwd_kv: fp32 scores, p = exp2(S·s·log2e - m) against the row maximum, the row
sum over the fp32 p, P rounded to bf16 before P·V, O normalised and rounded once; lse = m·ln 2 + ln l in fp32; the backward
recomputes p from lse, forms dS = p·(dP - D)·s in fp32, rounds P and dS to bf16 before the products, adds cached rows' dK /
dV to the fp32 accumulator and hands the suffix rows bf16(dK + acc0).  Every contraction is evaluated in fp64 and rounded
to fp32, so only the rounding points differ from the fp64 reference.
"""
import math

import pytest
import torch

from tests.test_train_kernels_gpu import _attn_seq_check

bf16 = torch.bfloat16
H, HD, LQ, LK = 2, 128, 200, 330          # dk = 130: the cached / suffix split falls inside key block 1
SCALE = HD ** -0.5
# mutant -> the first quantity it corrupts (the checks run o, lse, then per gradient dv, dk, dq; cached rows first)
MUTANTS = {
    "mask_off_by_one": "o",               # every query also sees key dk + i + 1
    "subblock_visible": "dq",             # the dq pass treats one masked 64-key sub-block of query rows 0..63 as visible
    "acc_bf16": "acc dv",                 # the accumulator is rounded to bf16 after the add
    "suffix_without_acc0": "dv",          # the suffix rows get bf16(dK), bf16(dV) instead of bf16(dK + acc0), ...
    "lse_wrong_dk": "lse",                # lse over the keys <= dk + 1 + i
}


def _inputs():
    g = torch.Generator().manual_seed(0)
    bfr = lambda *s: torch.randn(*s, generator=g).to(bf16).double()
    q, k, v, dO = bfr(H, LQ, HD), bfr(H, LK, HD), bfr(H, LK, HD), bfr(H, LQ, HD)
    acc0 = (torch.randn(H, LK, HD, generator=g).double(), torch.randn(H, LK, HD, generator=g).double())   # fp32 values
    return q, k, v, dO, tuple(a.float().double() for a in acc0)


def _emulate(q, k, v, dO, acc0, mutant=None):
    """(o, lse, (dq, dk, dv)) as the kernels round them; dk / dv over the LK key rows: rows j < dk the accumulator after the
    call, rows j >= dk the bf16 gradients.  fp64 tensors holding fp32 / bf16 values."""
    f32 = lambda x: x.float()
    rb = lambda x: x.to(bf16).float()
    dk = LK - LQ
    i = torch.arange(LQ)[:, None]
    j = torch.arange(LK)[None, :]
    vis = j <= dk + i + (1 if mutant == "mask_off_by_one" else 0)
    sl2 = f32(torch.tensor(SCALE * math.log2(math.e)))
    S = f32(q @ k.transpose(1, 2))

    def lse_of(vmask):
        Sv = S.masked_fill(~vmask, float("-inf"))
        m = Sv.amax(-1, keepdim=True) * sl2
        p = torch.exp2(Sv * sl2 - m)
        return m, p, f32(p.double().sum(-1, keepdim=True))

    m, p, l = lse_of(vis)
    o = rb(f32(rb(p).double() @ v) / l)
    if mutant == "lse_wrong_dk":
        m, _, l = lse_of(j <= dk + 1 + i)
    lse = m * f32(torch.tensor(math.log(2.0))) + torch.log(l)

    p_all = torch.exp2(S * sl2 - lse * f32(torch.tensor(math.log2(math.e))))
    D = f32((dO * o.double()).sum(-1, keepdim=True))
    dP = f32(dO @ v.transpose(1, 2))
    dS_of = lambda vmask: p_all.masked_fill(~vmask, 0.0) * ((dP - D) * f32(torch.tensor(SCALE)))
    P, dS = p_all.masked_fill(~vis, 0.0), dS_of(vis)
    dV = f32(rb(P).double().transpose(1, 2) @ dO)
    dK = f32(rb(dS).double().transpose(1, 2) @ q)
    if mutant == "subblock_visible":
        n = dk // 64 + 1                  # keys 64n .. 64n + 63 > dk: masked for query row 0 and the rows after it
        vis_q = vis.clone()
        vis_q[:64, 64 * n:64 * n + 64] = True
        dS = dS_of(vis_q)
    dQ = rb(f32(rb(dS).double() @ k))
    out = []
    for g, a0 in ((dK, acc0[0]), (dV, acc0[1])):
        a0 = f32(a0)
        cached = g[:, :dk] + a0[:, :dk]                                   # fp32 add
        if mutant == "acc_bf16":
            cached = rb(cached)
        suffix = rb(g[:, dk:] + (0 if mutant == "suffix_without_acc0" else a0[:, dk:]))
        out.append(torch.cat([cached, suffix], 1))
    return o.double(), lse.double().squeeze(-1), (dQ.double(), out[0].double(), out[1].double())


def test_emulated_kernel_is_within_bounds():
    q, k, v, dO, acc0 = _inputs()
    o, lse, grads = _emulate(q, k, v, dO, acc0)
    worst = _attn_seq_check(q, k, v, dO, o, lse, {"emulated": grads}, SCALE, "emulation", acc0=acc0)
    assert set(worst) == {"o", "lse", "dq", "dk", "dv", "acc dk", "acc dv"}, worst
    print("worst err/tol:", {n: round(r, 3) for n, r in worst.items()})


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_mutant_is_out_of_bounds(mutant):
    """Each mistake is reported, and by the quantity it corrupts first (the checks run o, lse, dv, dk, dq)."""
    q, k, v, dO, acc0 = _inputs()
    o, lse, grads = _emulate(q, k, v, dO, acc0, mutant)
    with pytest.raises(AssertionError, match=rf"^{MUTANTS[mutant]} .*out of bound"):
        _attn_seq_check(q, k, v, dO, o, lse, {"mutant": grads}, SCALE, mutant, acc0=acc0)
