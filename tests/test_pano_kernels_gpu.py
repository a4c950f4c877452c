"""fp32 panorama-encoder and fusion kernels (csrc/pano_ops.cu, plus the action-logit scatter) one by one, against fp64
references or in-order fp32 references computed with torch on the device.

Bounds are stated per element from the kernels' rounding points, with u = 2^-24 the fp32 unit roundoff:
  - mha_fwd: a score is a <= 128-term dot product (per-lane sums of <= 4 products, then 5 shuffle levels), softmax is
    fp32 with the fast exp (a few ulp) and P·V sums <= 256 terms in order.  The worst case of the P·V sum, 256·u·max|v|,
    is about 1.5e-5·max|v|; its typical size and every other term are well under 1e-6 of the head's largest output, so
    outputs and P are held to 1e-5 of the head's maximum.
  - mha_bwd: dS = P·(dP - D) cancels, and dq / dk are sums of <= 256 such terms: 1e-4 of the head's maximum gradient.
  - sgemm (exact fp32 mode): a fused multiply-add chain over each split's k range plus one add per split is within
    2K·u·(|A|·|B|)_ij of the exact product; each added bias or accumulate term adds one fp32 ulp of the magnitude of the
    terms.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
f64 = torch.float64
U = 2.0 ** -24


def _assert_within(got, ref, tol, what):
    err = (got.double() - ref).abs()
    bad = err > tol
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} of {bad.numel()} out of bound, worst err/tol {(err / tol).max().item():.3g}"


@pytest.fixture
def exact_fp32():
    from navillm_b200 import ops
    prev = ops.set_pano_precision("fp32")
    yield
    ops.set_pano_precision(prev)


# ---------------------------------------------------------------------------------------------------------------------
# masked multi-head attention
# ---------------------------------------------------------------------------------------------------------------------
MHA_CASES = [
    (16, 64, 256, [256, 255, 200, 129, 128, 65, 1, 0]),   # C3: 256 features per row, 16 heads of 64
    (4, 32, 33, [33, 32, 0]),
    (3, 48, 33, [33, 17]),
    (2, 128, 33, [1, 33, 20]),
    (2, 128, 1, [1, 0]),
    (2, 48, 1, [1]),
]


@pytest.mark.parametrize("H,hd,N,lens_h", MHA_CASES)
def test_mha_fwd_bwd_match_fp64_masked_attention(cuda_dev, H, hd, N, lens_h):
    from navillm_b200 import ops
    B, E = len(lens_h), H * hd
    g = torch.Generator(device=cuda_dev).manual_seed(H * 1000 + hd * 10 + N)
    qkv = torch.randn(B, N, 3 * E, generator=g, device=cuda_dev)
    dout = torch.randn(B, N, E, generator=g, device=cuda_dev)               # padded rows too: the backward must ignore them
    lens = torch.tensor(lens_h, dtype=torch.int32, device=cuda_dev)
    out, P = ops.mha_fwd(qkv, lens, H)
    dqkv = ops.mha_bwd(qkv, dout, P, lens, H)
    torch.cuda.synchronize()

    x = qkv.double().requires_grad_(True)
    q, k, v = [t.view(B, N, H, hd).transpose(1, 2) for t in x.split(E, dim=-1)]
    valid = torch.arange(N, device=cuda_dev)[None, :] < lens[:, None]      # [B, N]
    s = (q @ k.transpose(-1, -2)) * hd ** -0.5
    s = s.masked_fill(~valid[:, None, None, :], float("-inf")).masked_fill(~valid[:, None, :, None], 0.0)
    p = torch.softmax(s, dim=-1) * valid[:, None, :, None]
    ref = (p @ v).transpose(1, 2)                                           # [B, N, H, hd]
    ref.backward(dout.double().view(B, N, H, hd))
    p, ref = p.detach(), ref.detach()

    pad_rows = ~valid
    assert bool((out[pad_rows] == 0).all()) and bool((dqkv[pad_rows] == 0).all())
    pair = valid[:, None, :, None] & valid[:, None, None, :]
    assert bool((P.masked_select(~pair.expand(B, H, N, N)) == 0).all())
    rows = P.double().sum(-1)
    assert bool(((rows - 1).abs()[valid[:, None, :].expand(B, H, N)] <= 4e-6).all()), "P rows do not sum to 1"

    head_max = lambda t: t.abs().amax(dim=(1, 3), keepdim=True)             # [B, N, H, hd] -> per (b, h)
    _assert_within(out.view(B, N, H, hd), ref, 1e-5 * head_max(ref), "out")
    _assert_within(P, p, 1e-5 * p.amax(dim=(2, 3), keepdim=True), "P")
    for i, name in enumerate(("dq", "dk", "dv")):
        r = x.grad[..., i * E:(i + 1) * E].reshape(B, N, H, hd)
        _assert_within(dqkv[..., i * E:(i + 1) * E].reshape(B, N, H, hd), r, 1e-4 * head_max(r), name)


def test_mha_rejects_more_than_256_keys(cuda_dev):
    from navillm_b200 import _lib, ops
    qkv = torch.zeros(1, 257, 3 * 64, device=cuda_dev)
    lens = torch.tensor([257], dtype=torch.int32, device=cuda_dev)
    with pytest.raises(_lib.NvError, match="N=257"):
        ops.mha_fwd(qkv, lens, 1)
    with pytest.raises(_lib.NvError, match="N=257"):
        ops.mha_bwd(qkv, torch.zeros(1, 257, 64, device=cuda_dev), torch.zeros(1, 1, 257, 257, device=cuda_dev), lens, 1)


# ---------------------------------------------------------------------------------------------------------------------
# exact fp32 GEMM (nv_sgemm)
# ---------------------------------------------------------------------------------------------------------------------
def _sgemm_splits(M, N, K, sms):
    """K-split count of nv_sgemm's host rule (csrc/pano_ops.cu)."""
    tiles = -(-N // 64) * -(-M // 64)
    s = 1
    while s < 8 and tiles * s < 3 * sms and K // (s * 2) >= 256:
        s *= 2
    return s


def _run_sgemm(dev, M, N, K, ta, tb, bias, accumulate, seed):
    from navillm_b200 import ops
    g = torch.Generator(device=dev).manual_seed(seed)
    a = torch.randn((K, M) if ta else (M, K), generator=g, device=dev)
    b = torch.randn((K, N) if tb else (N, K), generator=g, device=dev)
    bvec = torch.randn(N, generator=g, device=dev) if bias else None
    c0 = torch.randn(M, N, generator=g, device=dev)
    runs = []
    for _ in range(2):
        out = c0.clone() if accumulate else None
        runs.append(ops.sgemm(a, b, ta=ta, tb=tb, bias=bvec, out=out, accumulate=accumulate))
    torch.cuda.synchronize()
    assert torch.equal(runs[0], runs[1]), "two runs differ"
    A = a.double().t() if ta else a.double()
    Bm = b.double() if tb else b.double().t()
    ref, mag = A @ Bm, A.abs() @ Bm.abs()
    extra = torch.zeros_like(ref)
    if bias:
        ref, extra = ref + bvec.double(), extra + bvec.double().abs()
    if accumulate:
        ref, extra = ref + c0.double(), extra + c0.double().abs()
    tol = 2 * K * U * mag + (int(bias) + int(accumulate)) * 2 * U * (mag + extra)
    _assert_within(runs[0], ref, tol, f"sgemm {M}x{N}x{K} ta={ta} tb={tb}")


@pytest.mark.parametrize("epilogue", ["plain", "bias", "accumulate", "bias+accumulate"])
@pytest.mark.parametrize("ta,tb", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("splits,M,N,K", [(1, 300, 130, 200), (2, 100, 70, 777), (4, 130, 200, 1500), (8, 256, 1024, 4096)])
def test_sgemm_matches_fp64_at_every_split_count(cuda_dev, exact_fp32, splits, M, N, K, ta, tb, epilogue):
    """Each shape takes the split count it is listed with (M, N not multiples of 64, K not a multiple of 16 in the first
    three): 2..8 splits add their partial tiles in rank order over DSMEM, and the result must not depend on the run."""
    sms = torch.cuda.get_device_properties(cuda_dev).multi_processor_count
    assert _sgemm_splits(M, N, K, sms) == splits
    _run_sgemm(cuda_dev, M, N, K, ta, tb, "bias" in epilogue, "accumulate" in epilogue, seed=M + N + K)


@pytest.mark.parametrize("M,N,K", [(2048, 1024, 1408), (576, 4096, 1024), (576, 1024, 4096)])
def test_sgemm_full_width_encoder_shapes(cuda_dev, exact_fp32, M, N, K):
    _run_sgemm(cuda_dev, M, N, K, False, False, True, False, seed=M ^ N ^ K)


# ---------------------------------------------------------------------------------------------------------------------
# row and elementwise kernels
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [128, 1024])
def test_layernorm_fwd_with_addend(cuda_dev, D):
    """mean / rstd: <= 13 rounding steps of a per-thread + shuffle sum, rsqrt.approx within 2 ulp.  y: the normalised
    value carries those relative errors plus |mean error|·rstd, then three roundings (scale, shift, addend)."""
    from navillm_b200 import ops
    R, eps = 300, 1e-12
    g = torch.Generator(device=cuda_dev).manual_seed(D)
    x = torch.randn(R, D, generator=g, device=cuda_dev) * 3 + 0.5
    gamma = torch.randn(D, generator=g, device=cuda_dev)
    beta = torch.randn(D, generator=g, device=cuda_dev)
    add = torch.randn(R, D + 8, generator=g, device=cuda_dev)[:, :D]
    y, mean, rstd = ops.layernorm_fwd(x, gamma, beta, eps, addend=add)
    torch.cuda.synchronize()
    x64 = x.double()
    mu = x64.mean(-1, keepdim=True)
    rs = torch.rsqrt(((x64 - mu) ** 2).mean(-1, keepdim=True) + eps)
    xhat = (x64 - mu) * rs
    ref = xhat * gamma.double() + beta.double() + add.double()
    absmean = x64.abs().mean(-1, keepdim=True)
    _assert_within(mean, mu[:, 0], 16 * U * absmean[:, 0], "mean")
    _assert_within(rstd, rs[:, 0], 32 * U * rs[:, 0], "rstd")
    tol = 32 * U * ((xhat * gamma.double()).abs() + beta.double().abs() + add.double().abs()) + 16 * U * gamma.double().abs() * rs * absmean
    _assert_within(y, ref, tol, "y")


@pytest.mark.parametrize("R", [1, 131, 2048])
def test_layernorm_bwd_accumulates(cuda_dev, R):
    """R = 1: one CTA; 131: fewer rows than SMs; 2048: several rows per persistent CTA.  dx is added onto a nonzero dx and
    dgamma / dbeta onto nonzero values.  The reference uses the kernel's mean / rstd."""
    from navillm_b200 import ops
    D = 1024
    g = torch.Generator(device=cuda_dev).manual_seed(R)
    x = torch.randn(R, D, generator=g, device=cuda_dev) * 2 - 0.3
    gamma = torch.randn(D, generator=g, device=cuda_dev)
    dy = torch.randn(R, D, generator=g, device=cuda_dev)
    _, mean, rstd = ops.layernorm_fwd(x, gamma, torch.zeros(D, device=cuda_dev), 1e-12)
    dx0, dg0, db0 = [torch.randn(*s, generator=g, device=cuda_dev) for s in ((R, D), (D,), (D,))]
    dx, dgamma, dbeta = dx0.clone(), dg0.clone(), db0.clone()
    ops.layernorm_bwd(x, gamma, mean, rstd, dy, dx=dx, accumulate_dx=True, dgamma=dgamma, dbeta=dbeta)
    torch.cuda.synchronize()
    rs = rstd.double()[:, None]
    xhat = (x.double() - mean.double()[:, None]) * rs
    gg = dy.double() * gamma.double()
    m1, m2 = gg.mean(-1, keepdim=True), (gg * xhat).mean(-1, keepdim=True)
    o = rs * (gg - m1 - xhat * m2)
    tol = 32 * U * rs * (gg.abs() + gg.abs().mean(-1, keepdim=True) + xhat.abs() * (gg * xhat).abs().mean(-1, keepdim=True))
    _assert_within(dx, dx0.double() + o, tol + 2 * U * (dx0.double().abs() + o.abs()), "dx")
    sms = torch.cuda.get_device_properties(cuda_dev).multi_processor_count
    P = min(sms, R)
    depth = -(-R // P) + -(-P // 8) + 16             # rows per CTA, then the column sum over the CTA partials
    for got, init, terms, name in ((dgamma, dg0, dy.double() * xhat, "dgamma"), (dbeta, db0, dy.double(), "dbeta")):
        ref = init.double() + terms.sum(0)
        _assert_within(got, ref, depth * U * terms.abs().sum(0) + 2 * U * (init.double().abs() + ref.abs()), name)


def test_gelu_fwd_bwd_erf_form(cuda_dev):
    """erff within 2 ulp; 1 + erf(z/sqrt 2) cancels for z << 0 (absolute error ~ ulp(1)·|z|/2); the backward's exp is the
    fast form: the rounded argument -z^2/2 and its scaling by log2(e) each cost |z^2/2| ulp of relative error."""
    from navillm_b200 import ops
    z = torch.cat([torch.linspace(-10, 10, (1 << 20) + 3, device=cuda_dev), torch.tensor([0.0, -0.0], device=cuda_dev)])
    da = torch.randn(z.numel(), generator=torch.Generator(device=cuda_dev).manual_seed(4), device=cuda_dev)
    a = ops.gelu_fwd(z)
    dz = ops.gelu_bwd(z, da)
    torch.cuda.synchronize()
    z64 = z.double()
    cdf = 0.5 * (1 + torch.erf(z64 / 2 ** 0.5))
    pdf = torch.exp(-0.5 * z64 * z64) / (2 * torch.pi) ** 0.5
    _assert_within(a, z64 * cdf, 8 * U * (z64 * cdf).abs() + z64.abs() * 2 ** -23, "gelu")
    ref_b = da.double() * (cdf + z64 * pdf)
    tol_b = da.double().abs() * (8 * U * (cdf + (z64 * pdf).abs()) + 2 ** -23 + (z64 * pdf).abs() * (z64 * z64 + 8) * U)
    _assert_within(dz, ref_b, tol_b, "gelu backward")
    assert a[-2].item() == 0.0 and a[-1].item() == 0.0 and dz[-2].item() == 0.5 * da[-2].item()


@pytest.mark.parametrize("accumulate", [False, True])
def test_colsum(cuda_dev, accumulate):
    from navillm_b200 import ops
    P, D = 1000, 300
    g = torch.Generator(device=cuda_dev).manual_seed(5)
    src = torch.randn(P, D + 4, generator=g, device=cuda_dev)[:, :D]
    dst0 = torch.randn(D, generator=g, device=cuda_dev)
    dst = dst0.clone()
    ops.colsum_(src, dst, accumulate=accumulate)
    torch.cuda.synchronize()
    ref = src.double().sum(0) + (dst0.double() if accumulate else 0)
    tol = (P // 8 + 10) * U * src.double().abs().sum(0) + 2 * U * (dst0.double().abs() * accumulate + ref.abs())
    _assert_within(dst, ref, tol, "colsum")


@pytest.mark.parametrize("case", ["ia_only", "identity_a_ib", "ia_identity_b_acc", "both_indexed_acc"])
def test_rows_combine(cuda_dev, case):
    """out[r] = (accumulate ? out[r] : 0) + alpha·A[ia[r]] + beta·B[ib[r]]; index -1 adds nothing, None is the identity."""
    from navillm_b200 import ops
    R, D = 50, 300
    g = torch.Generator(device=cuda_dev).manual_seed(6)
    A = torch.randn(R, D + 4, generator=g, device=cuda_dev)[:, :D]
    Bm = torch.randn(R + 10, D, generator=g, device=cuda_dev)
    out0 = torch.randn(R, D, generator=g, device=cuda_dev)
    idx = lambda n: torch.where(torch.rand(R, generator=g, device=cuda_dev) < 0.25, -1,
                                torch.randint(0, n, (R,), generator=g, device=cuda_dev)).to(torch.int32)
    a, ia, alpha, b, ib, beta, acc = {
        "ia_only": (A, idx(R), 1.0, None, None, 1.0, False),
        "identity_a_ib": (A, None, 0.5, Bm, idx(R + 10), -1.25, False),
        "ia_identity_b_acc": (A, idx(R), 2.0, Bm, None, 0.75, True),
        "both_indexed_acc": (A, idx(R), -0.3, Bm, idx(R + 10), 1.0, True),
    }[case]
    out = out0.clone()
    ops.rows_combine(out, a, ia, alpha, b, ib, beta, accumulate=acc)
    torch.cuda.synchronize()

    def term(m, i, s):
        if m is None:
            return torch.zeros(R, D, dtype=f64, device=cuda_dev)
        i = torch.arange(R, device=cuda_dev) if i is None else i.long()
        return torch.where((i >= 0)[:, None], s * m.double()[i.clamp(min=0)], 0.0)

    ta, tb = term(a, ia, alpha), term(b, ib, beta)
    t0 = out0.double() if acc else torch.zeros_like(ta)
    ref = t0 + ta + tb
    if ia is not None:
        assert bool((ia < 0).any())
    _assert_within(out, ref, 4 * U * (t0.abs() + ta.abs() + tb.abs()), case)


def test_rows_scatter_add_is_an_in_order_sum(cuda_dev):
    """Duplicate destinations and -1 indices: at alpha = 1 bit for bit the sequential fp32 sum in source-row order, at
    alpha != 1 within the fp64 bound, and the same bits on every run."""
    from navillm_b200 import ops
    R, Rd, D = 200, 20, 300
    g = torch.Generator(device=cuda_dev).manual_seed(7)
    src = torch.randn(R, D + 4, generator=g, device=cuda_dev)[:, :D] * 100
    dst0 = torch.randn(Rd, D, generator=g, device=cuda_dev)
    idx_h = torch.randint(-1, Rd, (R,), generator=torch.Generator().manual_seed(7)).tolist()
    idx = torch.tensor(idx_h, dtype=torch.int32, device=cuda_dev)
    # sequential reference in waves: wave k adds the k-th source row of every destination (distinct destinations per wave)
    seen, waves = {}, []
    for r, d in enumerate(idx_h):
        if d >= 0:
            k = seen.get(d, 0)
            seen[d] = k + 1
            if k == len(waves):
                waves.append([])
            waves[k].append(r)
    assert len(waves) > 3 and -1 in idx_h
    ref = dst0.clone()
    for rows in waves:
        dsts = [idx_h[r] for r in rows]
        ref[dsts] = ref[dsts] + src[rows]
    got = [ops.rows_scatter_add_(dst0.clone(), idx, src) for _ in range(2)]
    torch.cuda.synchronize()
    assert torch.equal(got[0], ref) and torch.equal(got[1], ref)

    alpha = 0.37
    got = [ops.rows_scatter_add_(dst0.clone(), idx, src, alpha=alpha) for _ in range(2)]
    torch.cuda.synchronize()
    assert torch.equal(got[0], got[1])
    ref64, mag = dst0.double().clone(), dst0.double().abs()
    cnt = torch.zeros(Rd, 1, dtype=f64, device=cuda_dev)
    keep = idx >= 0
    ref64.index_add_(0, idx[keep].long(), alpha * src[keep].double())
    mag = mag.index_add(0, idx[keep].long(), alpha * src[keep].double().abs())
    cnt.index_add_(0, idx[keep].long(), torch.ones(int(keep.sum()), 1, dtype=f64, device=cuda_dev))
    _assert_within(got[0], ref64, 2 * (cnt + 1) * U * mag, "scatter alpha")


def test_logit_scatter_fwd_bwd(cuda_dev):
    """out[b, g] = pred[b, slot[b, g]] (slot -1: -inf) and its transpose for the gradient, bit for bit."""
    from navillm_b200 import ops
    B, O, G = 5, 40, 12
    gen = torch.Generator().manual_seed(8)
    pred = torch.randn(B, O, generator=gen).to(torch.bfloat16).to(cuda_dev)
    slot = torch.stack([torch.where(torch.rand(G, generator=gen) < 0.3, -1, torch.randperm(O, generator=gen)[:G])
                        for _ in range(B)]).to(torch.int32)
    dout = torch.randn(B, G, generator=gen).to(torch.bfloat16)
    out = ops.logit_scatter_fwd(pred, slot.to(cuda_dev), B, G)
    dpred = ops.logit_scatter_bwd(dout.to(cuda_dev), slot.to(cuda_dev), O)
    torch.cuda.synchronize()
    want = torch.full((B, G), float("-inf"), dtype=torch.bfloat16)
    want_d = torch.zeros(B, O, dtype=torch.bfloat16)
    for b in range(B):
        for gi in range(G):
            s = int(slot[b, gi])
            if s >= 0:
                want[b, gi] = pred[b, s].cpu()
                want_d[b, s] = dout[b, gi]
    assert bool((slot < 0).any())
    assert torch.equal(out.cpu(), want) and torch.equal(dpred.cpu(), want_d)
