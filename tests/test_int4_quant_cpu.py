"""The 4-bit group-wise weight rule (W4A16, include/navillm_b200.h) restated in torch, pinned on hand-built groups.

One group is a weight row and 128 consecutive columns.  In fp32 from the bf16 values, with IEEE division and
round-half-even rint: lo = min(0, min w), hi = max(0, max w), s = max(bf16((hi - lo) / 15), 2^-126),
z = clamp(rint(-lo / s), 0, 15), q = clamp(rint(w / s) + z, 0, 15), W' = bf16((q - z) * s).  The GPU quantizer is checked
against ``ref_int4`` bit for bit in tests/test_int4_weights_gpu.py."""
import torch

bf16 = torch.bfloat16
GROUP = 128
TINY = 2.0 ** -126


def ref_int4(W: torch.Tensor):
    """(q uint8 [N, K], s bf16 [N, K/128], z uint8 [N, K/128], W' bf16 [N, K]) of a bf16 weight W [N, K]."""
    N, K = W.shape
    w = W.float().view(N, K // GROUP, GROUP)
    lo = torch.clamp(w.amin(-1), max=0.0)
    hi = torch.clamp(w.amax(-1), min=0.0)
    s = ((hi - lo) / 15).to(bf16).float().clamp(min=TINY)
    z = torch.round(-lo / s).clamp(0, 15)
    q = (torch.round(w / s[..., None]) + z[..., None]).clamp(0, 15)
    wq = ((q - z[..., None]) * s[..., None]).to(bf16)
    return q.to(torch.uint8).view(N, K), s.to(bf16), z.to(torch.uint8), wq.view(N, K)


def _group(vals, fill=0.0):
    g = torch.full((GROUP,), fill)
    g[:len(vals)] = torch.tensor(vals, dtype=torch.float32)
    return g


def edge_groups():
    """{name: one group of 128 bf16 values} exercising each branch of the rule."""
    gen = torch.Generator().manual_seed(11)
    return {
        "zero": torch.zeros(GROUP),
        "negative_zero": torch.full((GROUP,), -0.0),
        "positive": torch.rand(GROUP, generator=gen) * 0.05 + 0.001,                 # lo = 0: z = 0
        "negative": -(torch.rand(GROUP, generator=gen) * 0.05 + 0.001),              # hi = 0: z = 15
        # s = 30 / 15 = 2 and -lo / s = 7.5: z = 8 (tie to even); w / s = 0.5, 1.5, -2.5, 6.5 are ties too
        "ties": _group([15.0, -15.0, 1.0, 3.0, -5.0, 13.0]),
        # hi - lo = 15.03125 rounds to s = 1, z = rint(7.5) = 8 and rint(7.53125) + 8 = 16: the code clamps to 15
        "clamped": _group([7.53125, -7.5, 7.5, 2.0]),
        # all bf16 subnormals: s clamps to 2^-126, z = rint(0.75) = 1, and w / s is 0.75, 0.5, -0.75, 0.25
        "subnormal": _group([3 * 2.0 ** -128, 2.0 ** -127, -3 * 2.0 ** -128, 2.0 ** -128, 5 * 2.0 ** -133]),
        # one normal value with subnormals: s = bf16(2^-120 / 15) is normal, the subnormals' w / s are fractions
        "mixed_subnormal": _group([2.0 ** -120, 3 * 2.0 ** -127, -5 * 2.0 ** -128, 2.0 ** -126, -(2.0 ** -124)]),
        "random": torch.randn(GROUP, generator=gen) * 0.02,
    }


def _one(vals):
    return ref_int4(vals.to(bf16)[None])


def test_all_zero_groups():
    for name in ("zero", "negative_zero"):
        q, s, z, wq = _one(edge_groups()[name])
        assert s.float().item() == TINY and int(z) == 0
        assert int(q.max()) == 0
        assert torch.equal(wq.view(torch.int16), torch.zeros_like(wq).view(torch.int16))   # -0 becomes +0


def test_one_signed_groups_pin_the_zero_point():
    q, s, z, wq = _one(edge_groups()["positive"])
    assert int(z) == 0 and int(q.min()) >= 0
    q, s, z, wq = _one(edge_groups()["negative"])
    assert int(z) == 15 and int(q.max()) <= 15


def test_exact_ties_round_to_even():
    q, s, z, wq = _one(edge_groups()["ties"])
    assert s.float().item() == 2.0 and int(z) == 8
    assert q[0, :6].tolist() == [15, 0, 8, 10, 6, 14]          # rint(7.5), rint(-7.5), rint(0.5), rint(1.5), rint(-2.5), rint(6.5)
    assert wq[0, :6].float().tolist() == [14.0, -16.0, 0.0, 4.0, -4.0, 12.0]


def test_clamped_code():
    q, s, z, wq = _one(edge_groups()["clamped"])
    assert s.float().item() == 1.0 and int(z) == 8
    assert q[0, :4].tolist() == [15, 0, 15, 10]
    assert wq[0, 0].item() == 7.0                               # 7.53125 clamps to 15 - 8 = 7


def test_subnormal_groups():
    q, s, z, wq = _one(edge_groups()["subnormal"])
    assert s.float().item() == TINY and int(z) == 1
    assert q[0, :5].tolist() == [2, 1, 0, 1, 1]
    assert wq[0, :5].float().tolist() == [TINY, 0.0, -TINY, 0.0, 0.0]
    q, s, z, wq = _one(edge_groups()["mixed_subnormal"])
    sv = s.float().item()
    assert sv == float(torch.tensor(2.0 ** -120 / 15 + 2.0 ** -124 / 15).to(bf16)) and sv > TINY
    assert q[0, 1].item() - int(z) == round(3 * 2.0 ** -127 / sv)          # a subnormal's code is not flushed to z


def test_error_bound_on_unclamped_elements():
    gen = torch.Generator().manual_seed(5)
    W = torch.cat([(torch.randn(48, 1024, generator=gen) * 0.02),
                   torch.stack([edge_groups()[k] for k in sorted(edge_groups())]).repeat(1, 8)]).to(bf16)
    q, s, z, wq = ref_int4(W)
    N, K = W.shape
    sf = s.float().repeat_interleave(GROUP, 1)
    zf = z.float().repeat_interleave(GROUP, 1)
    unclamped = (torch.round(W.float() / sf) + zf).le(15) & (torch.round(W.float() / sf) + zf).ge(0)
    # the grid point (q - z) * s (exact in fp32) is within s / 2 of W; W' is that point rounded once to bf16, which adds at
    # most half a bf16 ulp of W' (so |W - W'| <= s / 2 alone does not hold: 0.0228271 -> 3 * 0.0065308 = 0.0195923 -> 0.0195313)
    grid = (q.float() - zf) * sf
    assert bool((((W.float() - grid).abs() <= sf / 2) | ~unclamped).all())
    half_ulp = torch.ldexp(torch.ones_like(grid), torch.frexp(wq.float())[1] - 9)
    assert bool((((W.float() - wq.float()).abs() <= sf / 2 + half_ulp) | ~unclamped).all())
    assert bool(unclamped.float().mean() > 0.99)
    # W' is (q - z) * s exactly, and q and z are 4-bit
    assert torch.equal(wq.float(), ((q.float() - zf) * sf).to(bf16).float())
    assert int(q.max()) <= 15 and int(z.max()) <= 15
