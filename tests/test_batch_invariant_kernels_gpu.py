"""The batch-invariant linears (``ops.gemm_bi`` / ``ops.gemm_bi_swiglu``) at every Vicuna-7B inference GEMM shape.

A fixed set of probe rows is computed inside batches of M in ``MS`` rows, with random companion rows and the probes at
random positions: every probe row must come out with the same bits at every M and every position.  The batches span the
weight-streaming kernel nv_gemm_bi_bf16 (M <= 128) and the tile kernels of nv_gemm_bf16 (M > 128, 32 / 128 / 256-wide
tiles), so this also checks that they share one accumulation chain per element.  Each probe result is then bounded
against an fp64 reference on the same bf16 operands (the bounds of test_gemm_kernels_gpu.py, section B):
    bf16 out:       |C - C64| <= b |C64| + (1 + b) tc S,    S = |x| |W|^T,  tc = 8u ceil(K / 16)
    with addend:    |C - R| <= b |R| + F7 (b |C64| + tc S + 2u |R|),    R = C64 + add
    SwiGLU:         h against silu(g64) u64 with the row-kernel bound of that file's section D, widened by the rounding
                    of g and u to bf16.
A first check pins the premise every claim rests on: wgmma gives an element the same bits whatever the instruction's N
(32 / 128 / 256 tiles) and the element's row and column inside the tile.
"""
import pytest
import torch

from navillm_b200 import ops

pytestmark = pytest.mark.gpu

bf16 = torch.bfloat16
D, F, V = 4096, 11008, 32006
MS = (1, 2, 8, 16, 17, 33, 64, 65, 128, 129, 512, 1024, 4096)
P = 4                                   # probe rows
U, B8 = 2.0 ** -24, 2.0 ** -8
F7 = 1 + 2.0 ** -7

SHAPES = {                              # name: (N, K, form)
    "qkv": (3 * D, D, "plain"),
    "o_proj": (D, D, "addend"),
    "gate_up": (2 * F, D, "swiglu"),
    "down_proj": (D, F, "addend"),
    "lm_head": (V, D, "plain"),
}


def _bits(t):
    return t.contiguous().view(torch.int16)


def _weights(N, K, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return (torch.randn((N, K), generator=g, device=dev) * 0.02).to(bf16)


def _run(form, x, w, add):
    if form == "swiglu":
        return ops.gemm_bi_swiglu(x, w)
    return ops.gemm_bi(x, w, addend=add if form == "addend" else None)


@pytest.mark.parametrize("name", list(SHAPES))
def test_rows_identical_across_batches(cuda_dev, name):
    N, K, form = SHAPES[name]
    dev = cuda_dev
    w = _weights(N, K, dev, 1 + len(name))
    g = torch.Generator(device=dev).manual_seed(7)
    probes = torch.randn((P, K), generator=g, device=dev).to(bf16)
    n_out = N // 2 if form == "swiglu" else N
    probe_add = (torch.randn((P, n_out), generator=g, device=dev) * 0.5).to(bf16)
    ref = [None] * P
    gen = torch.Generator().manual_seed(11)
    for M in MS:
        x = torch.randn((M, K), generator=g, device=dev).to(bf16)
        add = (torch.randn((M, n_out), generator=g, device=dev) * 0.5).to(bf16)
        rows = torch.randperm(M, generator=gen)[:min(P, M)].tolist()
        for p, r in enumerate(rows):
            x[r] = probes[p]
            add[r] = probe_add[p]
        out = _run(form, x, w, add)
        torch.cuda.synchronize()
        for p, r in enumerate(rows):
            if ref[p] is None:
                ref[p] = (M, out[r].clone())
            else:
                m0, r0 = ref[p]
                assert torch.equal(_bits(out[r]), _bits(r0)), \
                    f"{name}: probe {p} differs between M = {m0} and M = {M} (row {r})"
        del x, add, out

    # fp64 bounds on the probe rows
    got = torch.stack([ref[p][1] for p in range(P)]).double()
    xd, wd = probes.double(), w.double()
    tc = 8 * U * ((K + 15) // 16)
    if form == "swiglu":
        c64 = xd @ wd.t()
        s = xd.abs() @ wd.abs().t()
        gg, uu = c64[:, :n_out], c64[:, n_out:]
        sg, su = s[:, :n_out], s[:, n_out:]
        silu = gg * torch.sigmoid(gg)
        r = silu * uu
        eps = 2 * U * (2 + 1.173 * gg.abs()) + 5 * U
        # g and u carry the GEMM error eg / eu and one bf16 rounding; silu' is bounded by 1.1
        eg = B8 * gg.abs() + (1 + B8) * tc * sg
        eu = B8 * uu.abs() + (1 + B8) * tc * su
        bound = (B8 + F7 * (B8 + eps + U)) * r.abs() + F7 * (1.1 * eg * (uu.abs() + eu) + silu.abs() * eu) + 1e-30
    else:
        c64 = xd @ wd.t()
        s = xd.abs() @ wd.abs().t()
        if form == "addend":
            rr = c64 + probe_add.double()
            bound = B8 * rr.abs() + F7 * (B8 * c64.abs() + tc * s + 2 * U * rr.abs())
            r = rr
        else:
            r = c64
            bound = B8 * c64.abs() + (1 + B8) * tc * s
    err = (got - r).abs()
    assert torch.isfinite(got).all()
    worst = (err / bound).max().item()
    assert worst <= 1.0, f"{name}: error {worst:.3g} x the fp64 bound"


def test_wgmma_element_bits_independent_of_tile(cuda_dev):
    """nv_gemm_bf16's 32-, 128- and 256-wide tiles and the 32-wide weight-streaming kernel give every element the same
    bits, at every row of the tile (the rows of one batch, shifted by one row, land on other tile rows and columns)."""
    dev = cuda_dev
    g = torch.Generator(device=dev).manual_seed(3)
    M, N, K = 1024, 4096, 4096
    x = torch.randn((M, K), generator=g, device=dev).to(bf16)
    w = _weights(N, K, dev, 5)
    base = ops.gemm(x, w, block_n=128)
    for bn in (32, 256):
        assert torch.equal(_bits(ops.gemm(x, w, block_n=bn)), _bits(base)), f"block_n {bn} vs 128"
    shifted = ops.gemm(torch.cat([x[1:], x[:1]]), w, block_n=128)
    assert torch.equal(_bits(shifted[:-1]), _bits(base[1:]))
    for m in (1, 7, 64, 128):
        assert torch.equal(_bits(ops.gemm_bi(x[:m], w)), _bits(base[:m])), f"gemm_bi at M = {m}"
    wp = torch.cat([w[1:], w[:1]])                     # weight rows at other tile columns
    assert torch.equal(_bits(ops.gemm(x, wp, block_n=128)[:, :-1]), _bits(base[:, 1:]))
