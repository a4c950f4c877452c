"""Training-step kernels against fp64 references at the C2 and C5 shapes, with per-element error bounds.

Every reference runs in fp64 on the GPU from the same bf16 (or fp32) inputs the kernel reads.  A bound is per element: half a
bf16 ulp of the result at each point where the kernel rounds to bf16, applied to the reference's absolute-value contraction
(the same sum computed with |.| operands), plus an fp32 term.  Notation: u = 2^-24 (fp32 unit roundoff), b = 2^-8 (bf16 unit
roundoff: round-to-nearest moves a value by at most b·|value|), ulp(y) <= 2u·|y|.  Rounding a value x whose own error against
the reference r is e gives |bf16(x) - r| <= b·|r| + (1 + b)·e; products of two small error factors are absorbed by writing
(1 + 2^-7) for (1 + b)(1 + ...).  An fp32 sum of n terms evaluated with nesting depth d has error <= d·u·(sum of |terms|).  The
tensor cores' fp32 accumulation is not IEEE round-to-nearest; it is budgeted at 4 ulp = 8u of the |.| contraction per
wgmma k-step of 16.  The library is built with --use_fast_math: exp2f is ex2.approx (2 ulp), __expf has at most
2 + floor(1.173·|x|) ulp, __logf at most 2^-21.41 absolute on [0.5, 2] and 3 ulp elsewhere, rsqrtf and 1/x 2 ulp.

1. Causal attention, packed (nv_attn_fwd, nv_attn_bwd) and over a KV cache (nv_attn_fwd_kv, nv_attn_bwd_kv), head_dim 128,
   scale s = 128^-0.5.  A sequence has q_len query rows and kv_len keys; query i sits at key position dk + i with
   dk = kv_len - q_len (the packed form is dk = 0, kv_len = q_len) and sees the keys j <= dk + i.
   Per row i and visible key j: scores S = s·q·k, P = softmax(S), A_i = max_j s·sum_d |q_d||k_d|, Z_i = max_j |S_ij|·log2(e)
   (both maxima over the visible keys), n_i = dk + i + 1 visible keys, and nb_i = (dk + min(q0 + 128, q_len) + 127) // 128
   key blocks: the count the CTA of row i's 128-row query block (first row q0) walks (i // 128 + 1 when dk = 0).  With
   dk > 0 the last of them may be fully masked for row i: its p are exactly 0 and it rescales by alpha = exp2(0) = 1
   exactly, so it is only counted.
   Forward.  The kernel rounds P (unnormalised, against the running maximum) to bf16 before P·V and O once at the end.
     fp32 error of one unnormalised p_j:  eps_i = u·(4 + 3·Z_i + 64·A_i)
       (4u ex2.approx; <= 4u·Z_i of argument rounding in log2 units — fma, s·log2e and s itself rounded to fp32 — times ln 2;
       64u·A_i: the score's 8 k-steps at 8u each, times s).  Errors of the running maximum cancel between O and l.
     O: |o - o_ref| <= b·|o_ref| + (1 + 2^-7)·(b + F_i)·sum_j P_ij·|v_j|,
       F_i = 2·eps_i + u·(39 + 71·nb_i): 2·eps (numerator against denominator), row sum l at depth 32 + 2·nb + 2, P·V at
       8 k-steps of 8u plus the rescale by alpha (exp2 4u + product u) per key block, 1/l and the product 5u.
     lse: |lse - lse_ref| <= 2^-21 + 6u·ln(n_i) + 2u·|lse_ref| + 2u·Z_i + eps_i + u·(34 + 2·nb_i)
       (__logf: 2^-21.41 absolute or 3 ulp of ln l; the m·ln 2 product and its constant; the relative error of l).
   Backward.  The kernel recomputes p = exp2(S·log2e - lse·log2e) from the forward's fp32 lse, rounds P to bf16 for dV, forms
   dS = p·(dP - D)·s in fp32 with dP = dO·v on the tensor cores and D = sum_d dO·O from the forward's bf16 O, and rounds dS to
   bf16 for dK and dQ.  Relative error of p: rho_i = |lse_i - lse_ref,i| + u·(4 + 3·(Z_i + |lse_i|·log2 e) + 64·A_i); R = max_i rho_i.
   Error of D: dD_i = |sum_d dO_id·(o_id - o_ref,id)| (the rounded O the kernel reads, measured) + 12u·sum_d |dO_id||o_id|.
   E_ij = s·P_ij·(64u·sum_d |dO_id||v_jd| + dD_i) is the resulting absolute error of dS_ij; tc = 8u·ceil(n/16) the accumulation
   over the <= n partners: n = kv_len keys for dQ, n = q_len queries for dK and dV.  Under --use_fast_math a p or dS below 2^-126 may be flushed to 0 (keys no query attends to in the
   heads with scores of std 8 have p ~ e^-120): each such term moves a product by at most 2^-126·|partner|·(1 + s·max|dP - D|),
   and a result below 2^-126 may itself flush.  With fz = 1 + s·max_ij |dP_ij - D_i|, sums over the sequence's rows:
     dV: |dv - dv_ref| <= b·|dv_ref| + (1 + 2^-7)·(b + R + tc)·(|P|^T |dO|) + 2^-126·(1 + sum_i |dO_i|)
     dK: |dk - dk_ref| <= b·|dk_ref| + (1 + 2^-7)·((b + R + tc + 3u)·(|dS|^T |Q|) + E^T |Q|) + 2^-126·(1 + fz·sum_i |q_i|)
     dQ: |dq - dq_ref| <= b·|dq_ref| + (1 + 2^-7)·((b + R + tc + 3u)·(|dS| |K|) + E |K|) + 2^-126·(1 + fz·sum_j |k_j|)
   Over a KV cache the key rows' gradients meet an fp32 accumulator acc (dK | dV columns, acc0 before the call).  Write G
   for everything but the leading b·|ref| in the dK (dV) bound: the error of the fp32 gradient before it is stored.
     Cached rows j < dk: acc_j += dK_j in fp32, never rounded to bf16, so acc - acc0 (exact in fp64) is checked without the
       b·|ref| term; the bf16 P and dS inside G stay, and the fp32 add costs u·|acc0 + dK| <= u·(|acc0| + |dk_ref|) (to first
       order):  |(acc - acc0) - dk_ref| <= G + u·(|acc0| + |dk_ref|), the same for dV.
     Suffix rows j >= dk: bf16(dK_j + acc0_j) from the fp32 sum, so the reference is ref = dk_ref + acc0 and the add's
       rounding is carried through the bf16 rounding:  |dk - ref| <= b·|ref| + G + (1 + 2^-7)·u·|ref|, the same for dV.
   The same bounds hold with dvec = D handed over by nv_gemm_attnd_bf16 (fp32 row sums of dO·O, the same budget).
   Masked probabilities are exactly 0, so a sequence's o, lse and gradients do not depend on its neighbours: they are
   checked bit for bit across packings and against a second run.

2. RMSNorm (nv_rmsnorm_fwd / nv_rmsnorm_bwd), D <= 4096 (larger D is refused).
   rstd: the sum of squares has depth <= 32 + 5 + 5 (all terms positive: relative error 42u), /D and +eps 2u, rsqrtf 4u:
     |rstd - rstd_ref| <= 28u·rstd_ref (1/2·44u + 4u, rounded up).
   y = bf16(w·bf16(x·rstd)) is checked bit for bit against those rounding points evaluated with the kernel's rstd.
   dx, with the kernel's rstd r, xh = x·r, g = dy·w (exact in fp32), dot = sum_j g·xh / D:
     fp32 error of dot: 43u·a + u·|dot| with a = sum_j |g·xh| / D (depth 42 plus the rounding of xh); the element adds at most
     5 roundings.  So |dx - dx_ref| <= b·|dx_ref| + (1 + b)·64u·(|r·xh|·(a + |dot|) + |r·g| + |dres|).
   dw: each of the P' = min(P, T) CTAs sums its ceil(T/P') rows in fp32 (plus the rounding of xh), then 8 threads per column
     sum ceil(P'/8) partials each, 7 more adds combine them, one more adds dw0 (accumulate_dw):
     n = ceil(T/P') + ceil(P'/8) + 9,  |dw - dw_ref| <= b·|dw_ref| + (1 + 2^-7)·n·u·(|dw0|·[accumulate] + sum_t |dy·xh|).

3. Token embedding (nv_embed_fwd, nv_embed_bwd_weight, nv_embed_bwd_vis).
   dE: the owner of id v adds its c_v rows one by one into an fp32 copy of dE0[v] and rounds once:
     |dE - dE_ref| <= b·|dE_ref| + (1 + 2^-7)·c_v·u·(|dE0| + sum |dx|); rows no token touches stay bit-identical.
   The forward is a copy, or bf16(E[id] + vis) from the fp32 sum (the reference's bf16 + fp32 add): bit for bit.  d vis is the
   bf16 gradient widened to fp32: bit for bit.

4. LM cross-entropy (nv_ce_fwd_bwd), special columns masked.  x_c = l_c - max, se = sum_c exp(x_c), depth 126 + 5 + 5:
     relative error of se: eta = u·(136 + sum_c (4 + 3.35·|x_c|)·exp(x_c) / se)  (__expf plus the rounding of its argument);
     |lse - lse_ref| <= dl = eta + 2^-21 + 6u·|ln se| + u·|lse_ref|;
     row_loss: <= dl + 2u·|loss_ref|;  dlogits, ref = g·(p_c - [c = label]) with g the fp32 grad_scale:
     <= b·|ref| + (1 + 2^-7)·g·(p_c·(dl + u·(6 + 3.35·|l_c - lse|)) + 2u) + 2^-125·g  (flush-to-zero of tiny exponentials).
   Ignored rows and special columns are exactly 0.  (A label naming a special column is outside the contract.)

5. Navigation head (nv_head_fwd / nv_head_bwd), D = 4096, O = 100.
     out: depth 128 + 5 + 1 (bias):   <= b·|ref| + (1 + b)·135u·(|x| |W|^T + |bias|)
     dx:  depth O:                     <= b·|ref| + (1 + b)·(O + 1)u·(|dy| |W|)
     dW, db accumulate into their existing values, depth R + 1:  <= b·|ref| + (1 + b)·(R + 1)u·(|dW0| + |dy|^T |x|), same for db.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
U = 2.0 ** -24
B8 = 2.0 ** -8
F7 = 1.0 + 2.0 ** -7
TINY = 2.0 ** -126      # flush-to-zero: an fp32 / bf16 value below it may become 0
LOG2E = 1.4426950408889634
HD = 128


def _check(name, got, ref, tol):
    """Asserts |got - ref| <= tol per element; returns the worst err/tol."""
    got = got.double()
    assert bool(torch.isfinite(got).all()), f"{name}: non-finite values"
    err = (got - ref).abs()
    bad = err > tol
    assert not bool(bad.any()), (f"{name}: {int(bad.sum())} of {bad.numel()} elements out of bound, worst err/tol "
                                 f"{(err / tol).max().item():.3g}, first at {tuple(bad.nonzero()[0].tolist())}")
    return (err / tol).max().item() if err.numel() else 0.0


def _cu(lens, dev):
    return torch.tensor([0] + np.cumsum(lens).tolist(), dtype=torch.int32, device=dev)


# ---------------------------------------------------------------------------------------------------------------------
# 1. attention
# ---------------------------------------------------------------------------------------------------------------------
BOUNDARY = [1, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 257]   # both sides of the 64- and 128-row blocks
ATTN_CASES = {
    "c2": lambda: np.random.RandomState(0).randint(256, 1025, 16).tolist(),
    "c5": lambda: [2048] * 4,
    "boundary": lambda: BOUNDARY,
    "boundary_reversed": lambda: BOUNDARY[::-1],
}


def _attn_inputs(lens, H, seed, dev, stress):
    """qkv [T, 3*H*128] bf16.  stress: per-head score scales from std 0.5 to 8; on odd heads every query also has a large
    component along dims 0 and 1, key 0 of each sequence is a sink (score about 10x the head's scale) and key 300, in key
    block 2, exceeds it (about 14x), so the running maximum jumps late for every row past it."""
    T = sum(lens)
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(T, 3, H, HD, generator=g, device=dev)
    if stress:
        odd = torch.arange(H, device=dev) % 2 == 1
        x[:, 0, odd, 0:2] = 4.0
        s0 = 0
        for L in lens:
            x[s0, 1, odd, 0] = 28.0
            if L > 300:
                x[s0 + 300, 1, odd, 1] = 40.0
            s0 += L
        x[:, 0] *= torch.logspace(math.log10(0.5), math.log10(8.0), H, device=dev)[None, :, None]
    return x.reshape(T, 3 * H * HD).to(bf16)


def _attn_seq_check(q, k, v, dO, o, lse, grads, scale, where, acc0=None):
    """One sequence (a few of its heads) against fp64 autograd of its masked softmax, with the bounds of §1.  fp64 tensors
    [heads, rows, 128] of the values the kernel read or wrote: q, dO and the kernel's o over the q_len query rows, k and v
    over the kv_len keys (dk = kv_len - q_len); lse [heads, q_len] the kernel's.  grads: {tag: (dq, dk, dv)} with dk / dv
    over the kv_len key rows: rows j >= dk the kernel's bf16 gradients, rows j < dk its accumulator after the call.  acc0:
    None in the packed form (no accumulator, kv_len = q_len), else the (dK, dV) accumulator columns before the call.
    Returns {quantity: worst err/tol}."""
    Lq, Lk = q.shape[1], k.shape[1]
    dk = Lk - Lq
    assert dk >= 0 and (acc0 is not None or dk == 0), (Lq, Lk)
    dev = q.device
    i = torch.arange(Lq, device=dev, dtype=torch.float64)
    mask = torch.arange(Lk, device=dev)[None, :] <= dk + torch.arange(Lq, device=dev)[:, None]
    q0 = torch.div(i, 128, rounding_mode="floor") * 128
    nb = torch.div(dk + torch.clamp(q0 + 128, max=Lq) + 127, 128, rounding_mode="floor")
    tc_q = 8 * U * math.ceil(Lk / 16)          # dQ contracts over the keys
    tc_k = 8 * U * math.ceil(Lq / 16)          # dK and dV over the queries
    worst = {}

    def chk(name, tag, got, ref, tol):
        r = _check(" ".join(s for s in (name, tag, where) if s), got, ref, tol)
        worst[name] = max(worst.get(name, 0.0), r)

    qa, ka, va = (t.clone().requires_grad_(True) for t in (q, k, v))
    with torch.enable_grad():
        sc = (qa @ ka.transpose(1, 2) * scale).masked_fill(~mask, float("-inf"))
        p = torch.softmax(sc, dim=-1)
        oref = p @ va
        dq, dkr, dvr = torch.autograd.grad(oref, (qa, ka, va), dO)
    sc, p, oref = sc.detach(), p.detach(), oref.detach()
    del qa, ka, va
    lref = torch.logsumexp(sc, dim=-1)
    A = (q.abs() @ k.abs().transpose(1, 2) * scale).masked_fill(~mask, 0).amax(-1)
    Z = sc.abs().masked_fill(~mask, 0).amax(-1) * LOG2E
    del sc
    eps = U * (4 + 3 * Z + 64 * A)
    F = 2 * eps + U * (39 + 71 * nb)
    chk("o", "", o, oref, B8 * oref.abs() + F7 * (B8 + F)[..., None] * (p @ v.abs()))
    chk("lse", "", lse, lref, 2.0 ** -21 + U * (6 * torch.log(dk + i + 1) + 2 * lref.abs() + 2 * Z + 34 + 2 * nb) + eps)

    D = (dO * oref).sum(-1)
    dD = (dO * (o - oref)).sum(-1).abs() + 12 * U * (dO.abs() * o.abs()).sum(-1)
    R = ((lse - lref).abs() + U * (4 + 3 * (Z + lse.abs() * LOG2E) + 64 * A)).amax(-1)[:, None, None]
    dPD = (dO @ v.transpose(1, 2) - D[..., None]).masked_fill(~mask, 0)
    dS = (p * dPD * scale).abs()
    E = scale * p * (64 * U * (dO.abs() @ v.abs().transpose(1, 2)) + dD[..., None])
    fz = 1 + scale * dPD.abs().amax(dim=(1, 2))[:, None, None]
    # G of §1: the error of the fp32 gradient before it is rounded to bf16 or added to the accumulator
    g_dv = F7 * (B8 + R + tc_k) * (p.transpose(1, 2) @ dO.abs()) + TINY * (1 + dO.abs().sum(1, keepdim=True))
    g_dk = (F7 * ((B8 + R + tc_k + 3 * U) * (dS.transpose(1, 2) @ q.abs()) + E.transpose(1, 2) @ q.abs())
            + TINY * (1 + fz * q.abs().sum(1, keepdim=True)))
    tol_dq = (B8 * dq.abs() + F7 * ((B8 + R + tc_q + 3 * U) * (dS @ k.abs()) + E @ k.abs())
              + TINY * (1 + fz * k.abs().sum(1, keepdim=True)))
    del dPD, p, dS, E

    def key_rows(name, tag, got, ref, g, a0):
        if a0 is None:
            chk(name, tag, got, ref, B8 * ref.abs() + g)
            return
        if dk:
            c0, c = a0[:, :dk], ref[:, :dk]
            chk("acc " + name, tag, got[:, :dk] - c0, c, g[:, :dk] + U * (c0.abs() + c.abs()))
        r = ref[:, dk:] + a0[:, dk:]
        chk(name, tag, got[:, dk:], r, B8 * r.abs() + g[:, dk:] + F7 * U * r.abs())

    for tag, (gq, gk, gv) in grads.items():
        key_rows("dv", tag, gv, dvr, g_dv, None if acc0 is None else acc0[1])
        key_rows("dk", tag, gk, dkr, g_dk, None if acc0 is None else acc0[0])
        chk("dq", tag, gq, dq, tol_dq)
    return worst


def _attn_ref_check(qkv, o, lse, dqkvs, do, lens, H, scale):
    """Checks o, lse and every dqkv in dqkvs of the packed form against fp64 autograd of the masked softmax, one sequence
    (and a few heads) at a time, with the bounds of the module docstring."""
    T = qkv.shape[0]
    s0 = 0
    for b, L in enumerate(lens):
        hc = max(1, min(H, (1 << 23) // (L * L)))
        for h0 in range(0, H, hc):
            hs = slice(h0, min(H, h0 + hc))
            heads = lambda t: t[s0:s0 + L].view(L, H, HD)[:, hs].double().transpose(0, 1)
            split = lambda t: t[s0:s0 + L].view(L, 3, H, HD)[:, :, hs].double().permute(1, 2, 0, 3).unbind(0)
            q, k, v = split(qkv)
            _attn_seq_check(q, k, v, heads(do), heads(o), lse.view(H, T)[hs, s0:s0 + L].double(),
                            {tag: split(dqkv) for tag, dqkv in dqkvs.items()}, scale,
                            f"seq {b} (len {L}) heads {h0}..{min(H, h0 + hc) - 1}")
        s0 += L


@pytest.mark.parametrize("stress", [False, True], ids=["randn", "stress"])
@pytest.mark.parametrize("case", list(ATTN_CASES))
def test_attention_fwd_bwd_matches_fp64(cuda_dev, case, stress):
    """o, lse and dq / dk / dv at H = 32 against fp64 autograd, per element; the backward both computing D itself and with D
    handed over by the o_proj dgrad GEMM (gemm_attnd), as the training step runs it."""
    from navillm_b200 import ops
    lens = ATTN_CASES[case]()
    H = 32
    T = sum(lens)
    qkv = _attn_inputs(lens, H, 1000 + T, cuda_dev, stress)
    cu = _cu(lens, cuda_dev)
    g = torch.Generator(device=cuda_dev).manual_seed(T)
    dy = torch.randn(T, H * HD, generator=g, device=cuda_dev).to(bf16)
    wo = (torch.randn(H * HD, H * HD, generator=g, device=cuda_dev) * (H * HD) ** -0.5).to(bf16)
    o, lse = ops.attn_fwd(qkv, cu, lens, H)
    do, dvec = ops.gemm_attnd(dy, wo, o)
    del dy, wo
    own = ops.attn_bwd(qkv, o, do, lse, cu, lens, H)
    handed = ops.attn_bwd(qkv, o, do, lse, cu, lens, H, dvec=dvec)
    torch.cuda.synchronize()
    _attn_ref_check(qkv, o, lse, {"own D": own, "dvec": handed}, do, lens, H, HD ** -0.5)


def test_attention_is_packing_invariant_and_deterministic(cuda_dev):
    """A sequence's o, lse and dqkv are the same bits packed among neighbours whose rows are about 100x larger, packed in
    another order, and launched alone; a second identical run is bit-identical."""
    from navillm_b200 import ops
    H = 32
    own = [129, 300, 64, 1, 257]
    g = torch.Generator(device=cuda_dev).manual_seed(5)
    seq = [(torch.randn(L, 3 * H * HD, generator=g, device=cuda_dev).to(bf16),
            torch.randn(L, H * HD, generator=g, device=cuda_dev).to(bf16)) for L in own]
    nbr = [((torch.randn(L, 3 * H * HD, generator=g, device=cuda_dev) * 100).to(bf16),
            (torch.randn(L, H * HD, generator=g, device=cuda_dev) * 100).to(bf16)) for L in (77, 200, 31)]

    def run(items):
        """items: ("s", idx) or ("n", idx) -> {idx: (o, lse, dqkv) of own sequence idx}"""
        parts = [(seq if kind == "s" else nbr)[j] for kind, j in items]
        lens = [p[0].shape[0] for p in parts]
        qkv = torch.cat([p[0] for p in parts])
        do = torch.cat([p[1] for p in parts])
        cu = _cu(lens, cuda_dev)
        o, lse = ops.attn_fwd(qkv, cu, lens, H)
        dqkv = ops.attn_bwd(qkv, o, do, lse, cu, lens, H)
        torch.cuda.synchronize()
        out, s0 = {}, 0
        for (kind, j), L in zip(items, lens):
            if kind == "s":
                out[j] = (o[s0:s0 + L].clone(), lse[:, s0:s0 + L].clone(), dqkv[s0:s0 + L].clone())
            s0 += L
        return out, (o, lse, dqkv)

    order_a = [("n", 0), ("s", 0), ("n", 1), ("s", 1), ("s", 2), ("n", 2), ("s", 3), ("s", 4)]
    order_b = [("s", 4), ("s", 2), ("n", 1), ("s", 0), ("s", 3), ("n", 0), ("s", 1)]
    a, full_a = run(order_a)
    b, _ = run(order_b)
    for j in range(len(own)):
        alone, _ = run([("s", j)])
        for name, x, y, z in zip(("o", "lse", "dqkv"), a[j], b[j], alone[j]):
            assert bool(torch.isfinite(x.float()).all()), f"seq {j} {name}: non-finite"
            assert torch.equal(x, y), f"seq {j} {name}: differs between two packings"
            assert torch.equal(x, z), f"seq {j} {name}: differs between packed and alone"
    _, full_a2 = run(order_a)
    for name, x, y in zip(("o", "lse", "dqkv"), full_a, full_a2):
        assert torch.equal(x, y), f"{name}: two identical runs differ"


# ---------------------------------------------------------------------------------------------------------------------
# 2. RMSNorm
# ---------------------------------------------------------------------------------------------------------------------
def _rows(spec, P):
    return {"1": 1, "P-1": P - 1, "P": P, "P+1": P + 1, "2P+3": 2 * P + 3, "10425": 10425}[spec]


@pytest.mark.parametrize("accumulate", [True, False], ids=["acc", "overwrite"])
@pytest.mark.parametrize("with_dres", [False, True], ids=["no_dres", "dres"])
@pytest.mark.parametrize("D", [256, 4096])
@pytest.mark.parametrize("rows", ["1", "P-1", "P", "P+1", "2P+3", "10425"])
def test_rmsnorm_fwd_bwd_matches_fp64(cuda_dev, rows, D, with_dres, accumulate):
    """rstd and y of the forward; dx and dw (from a non-zero bf16 dw, accumulated or overwritten) of the persistent backward
    at row counts around the partial count P, so CTAs walk zero, one, two and ~26 rows with the next row prefetched.
    dy = x·c_t + noise has a large component along x, where a wrong mean(g·xh) shows."""
    from navillm_b200 import _lib, ops
    P = _lib.load().nv_rmsnorm_bwd_partials()
    T = _rows(rows, P)
    g = torch.Generator(device=cuda_dev).manual_seed(T * 7 + D)
    x = (torch.randn(T, D, generator=g, device=cuda_dev) * 1.7).to(bf16)
    w = (1 + 0.1 * torch.randn(D, generator=g, device=cuda_dev)).to(bf16)
    eps = 1e-6
    y, rstd = ops.rmsnorm_fwd(x, w, eps)
    c = 0.5 + 1.5 * torch.rand(T, 1, generator=g, device=cuda_dev)
    dy = (x.float() * c + 0.05 * torch.randn(T, D, generator=g, device=cuda_dev)).to(bf16)
    dres = torch.randn(T, D, generator=g, device=cuda_dev).to(bf16) if with_dres else None
    dw0 = (0.5 * torch.randn(D, generator=g, device=cuda_dev)).to(bf16)
    dw = dw0.clone()
    dx = ops.rmsnorm_bwd(x, w, rstd, dy, dres=dres, dw=dw, accumulate_dw=accumulate)
    torch.cuda.synchronize()

    xd, wd, dyd = x.double(), w.double(), dy.double()
    rref = torch.rsqrt(xd.pow(2).mean(-1) + eps)
    _check("rstd", rstd, rref, 28 * U * rref)
    assert torch.equal(y, (w.float() * (x.float() * rstd[:, None]).to(bf16).float()).to(bf16)), "y: rounding points differ"

    r = rstd.double()[:, None]
    xh = xd * r
    gg = dyd * wd
    dot = (gg * xh).mean(-1, keepdim=True)
    a = (gg * xh).abs().mean(-1, keepdim=True)
    ref = r * (gg - xh * dot) + (dres.double() if with_dres else 0)
    cabs = (r * xh).abs() * (a + dot.abs()) + (r * gg).abs() + (dres.double().abs() if with_dres else 0)
    _check("dx", dx, ref, B8 * ref.abs() + (1 + B8) * 64 * U * cabs)

    Pe = min(P, T)
    n = math.ceil(T / Pe) + math.ceil(Pe / 8) + 9
    dwref = (dyd * xh).sum(0) + (dw0.double() if accumulate else 0)
    dwabs = (dyd * xh).abs().sum(0) + (dw0.double().abs() if accumulate else 0)
    _check("dw", dw, dwref, B8 * dwref.abs() + F7 * n * U * dwabs)


def test_rmsnorm_refuses_rows_wider_than_4096(cuda_dev):
    from navillm_b200 import _lib, ops
    x = torch.randn(4, 4104, device=cuda_dev).to(bf16)
    w = torch.ones(4104, device=cuda_dev, dtype=bf16)
    with pytest.raises(_lib.NvError, match="bad"):
        ops.rmsnorm_fwd(x, w, 1e-6)
    rstd = torch.ones(4, device=cuda_dev)
    dw = torch.zeros(4104, device=cuda_dev, dtype=bf16)
    with pytest.raises(_lib.NvError, match="bad"):
        ops.rmsnorm_bwd(x, w, rstd, x, dw=dw)
    torch.cuda.synchronize()
    assert bool((dw == 0).all())


# ---------------------------------------------------------------------------------------------------------------------
# 3. token embedding
# ---------------------------------------------------------------------------------------------------------------------
V_TOK, T_TOK = 32006, 10425


def _prompt_ids(seed):
    """T_TOK ids over V_TOK: Zipf-distributed ranks through a fixed permutation, three template ids repeated 1200 times each,
    and the first and last ids of the vocabulary."""
    rs = np.random.RandomState(seed)
    perm = rs.permutation(V_TOK)
    ids = perm[np.minimum(rs.zipf(1.3, T_TOK) - 1, V_TOK - 1)]
    pos = rs.permutation(T_TOK)
    for n, tid in enumerate((13, 29871, 2)):
        ids[pos[n * 1200:(n + 1) * 1200]] = tid
    ids[pos[3600]], ids[pos[3601]] = 0, V_TOK - 1
    return ids.astype(np.int32)


def test_embed_bwd_weight_accumulates_like_fp64(cuda_dev):
    """dE = dE0 + index_add(dx) from a non-zero dE0 at C2's token count, with three ids repeated 1200 times; untouched rows
    keep dE0's bits; the host-sorted order PackedPrompt passes gives the bits of the internal sort."""
    from navillm_b200 import ops
    D = 4096
    ids_np = _prompt_ids(0)
    ids = torch.from_numpy(ids_np).to(cuda_dev)
    g = torch.Generator(device=cuda_dev).manual_seed(11)
    dx = torch.randn(T_TOK, D, generator=g, device=cuda_dev).to(bf16)
    dE0 = (0.3 * torch.randn(V_TOK, D, generator=g, device=cuda_dev)).to(bf16)
    dE = dE0.clone()
    ops.embed_bwd_weight_(dx, ids, dE)
    order = np.argsort(ids_np, kind="stable")
    dE_host = dE0.clone()
    ops.embed_bwd_weight_(dx, ids, dE_host, order=torch.from_numpy(order.astype(np.int32)).to(cuda_dev),
                          sorted_ids=torch.from_numpy(ids_np[order]).to(cuda_dev))
    torch.cuda.synchronize()
    assert torch.equal(dE.view(torch.int16), dE_host.view(torch.int16)), "host-sorted order differs from the internal sort"

    uniq, inv = torch.unique(ids.long(), return_inverse=True)
    counts = torch.bincount(inv).double()[:, None]
    assert int(counts.max()) > 1000
    ref = dE0[uniq].double().index_add_(0, inv, dx.double())
    cabs = dE0[uniq].double().abs().index_add_(0, inv, dx.double().abs())
    _check("dE (touched rows)", dE[uniq], ref, B8 * ref.abs() + F7 * counts * U * cabs)
    untouched = torch.ones(V_TOK, dtype=torch.bool, device=cuda_dev)
    untouched[uniq] = False
    assert torch.equal(dE[untouched].view(torch.int16), dE0[untouched].view(torch.int16)), "an untouched row changed"


def test_embed_fwd_with_visual_rows_and_vis_grad_are_exact(cuda_dev):
    """out[t] = E[id] or bf16(E[id] + vis[src]) from the fp32 sum, at D = 4096; d vis = the widened bf16 gradient rows."""
    from navillm_b200 import ops
    D, n_vis = 4096, 700
    ids = torch.from_numpy(_prompt_ids(1)).to(cuda_dev)
    g = torch.Generator(device=cuda_dev).manual_seed(12)
    E = (0.02 * torch.randn(V_TOK, D, generator=g, device=cuda_dev)).to(bf16)
    rows = torch.randperm(T_TOK, generator=g, device=cuda_dev)[:n_vis]
    vis_src = torch.full((T_TOK,), -1, dtype=torch.int32, device=cuda_dev)
    vis_src[rows] = torch.arange(n_vis, dtype=torch.int32, device=cuda_dev)
    vis = torch.randn(n_vis, D, generator=g, device=cuda_dev)
    out = ops.embed_fwd(ids, E, vis_src, vis)
    dx = torch.randn(T_TOK, D, generator=g, device=cuda_dev).to(bf16)
    dvis = ops.embed_bwd_vis(dx, vis_src, n_vis)
    torch.cuda.synchronize()
    ref = E[ids.long()].clone()
    ref[rows] = (E[ids[rows].long()].float() + vis).to(bf16)
    assert torch.equal(out.view(torch.int16), ref.view(torch.int16))
    assert torch.equal(dvis, dx[rows].float())


# ---------------------------------------------------------------------------------------------------------------------
# 4. LM cross-entropy
# ---------------------------------------------------------------------------------------------------------------------
SPECIAL = [32000, 32001, 32002, 32003, 32004]


def _ce_check(ops, logits, labels, special, gs):
    row_loss, dl = ops.ce_fwd_bwd(logits, labels, special, grad_scale=gs)
    torch.cuda.synchronize()
    V = logits.shape[1]
    gs = float(np.float32(gs))
    lg = logits.double().clone()
    lg[:, special.long()] = float("-inf")
    act = (labels >= 0) & (labels < V)
    mx = lg.amax(-1, keepdim=True)
    xs = lg - mx
    e = torch.exp(xs)
    se = e.sum(-1, keepdim=True)
    lse = mx + torch.log(se)
    p = torch.exp(lg - lse)
    lab = labels.clamp(0, V - 1).long()[:, None]
    xl = logits.double().gather(1, lab)
    eta = U * (136 + ((4 + 3.35 * xs.abs()) * e).nan_to_num(0.0).sum(-1, keepdim=True) / se)
    dlse = eta + 2.0 ** -21 + 6 * U * torch.log(se).abs() + U * lse.abs()
    loss_ref = torch.where(act[:, None], lse - xl, torch.zeros_like(lse))
    _check("row_loss", row_loss[:, None], loss_ref, torch.where(act[:, None], dlse + 2 * U * loss_ref.abs(), torch.zeros_like(lse)))
    onehot = torch.zeros_like(p).scatter_(1, lab, 1.0)
    ref = torch.where(act[:, None], gs * (p - onehot), torch.zeros_like(p))
    ref[:, special.long()] = 0
    arg = (logits.double() - lse).abs()
    tol = B8 * ref.abs() + F7 * gs * (p * (dlse + U * (6 + 3.35 * arg)) + 2 * U) + 2.0 ** -125 * gs
    tol = torch.where(act[:, None], tol, torch.zeros_like(tol))
    tol[:, special.long()] = 0
    _check("dlogits", dl, ref, tol)


@pytest.mark.parametrize("N", [1, 37, 512])
def test_ce_matches_fp64(cuda_dev, N):
    """row_loss and dlogits against fp64 masked CE: logits ~ 2·randn with rows that peak at +60 (on or off the label) and flat
    rows; labels at 0, at V - 1 and -100."""
    from navillm_b200 import ops
    V = 32006
    g = torch.Generator(device=cuda_dev).manual_seed(N)
    logits = 2 * torch.randn(N, V, generator=g, device=cuda_dev)
    labels = torch.randint(0, 32000, (N,), generator=g, device=cuda_dev, dtype=torch.int32)
    labels[0] = 0
    if N > 1:
        labels[1] = V - 1
        labels[2::5] = -100
        logits[3::4] = 1.25                                                     # flat rows
        logits[5::7, 777] = 60.0                                                # peak off the label
    pk = torch.arange(0, N, 3, device=cuda_dev)
    logits[pk, labels[pk].clamp(min=0).long()] = 60.0                           # peak on the label
    special = torch.tensor(SPECIAL, dtype=torch.int32, device=cuda_dev)
    n_act = max(int((labels >= 0).sum()), 1)
    _ce_check(ops, logits.to(bf16), labels, special, 1.0 / n_act)


def test_ce_all_rows_ignored(cuda_dev):
    from navillm_b200 import ops
    N, V = 37, 32006
    logits = (2 * torch.randn(N, V, device=cuda_dev)).to(bf16)
    labels = torch.full((N,), -100, dtype=torch.int32, device=cuda_dev)
    special = torch.tensor(SPECIAL, dtype=torch.int32, device=cuda_dev)
    row_loss, dl = ops.ce_fwd_bwd(logits, labels, special, grad_scale=1.0)
    torch.cuda.synchronize()
    assert bool((row_loss == 0).all()) and bool((dl == 0).all())


# ---------------------------------------------------------------------------------------------------------------------
# 5. navigation head
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [1, 16, 64])
def test_head_fwd_bwd_matches_fp64(cuda_dev, R):
    """out = x W^T + b, dx = dy W, and dW / db accumulated into non-zero gradients (one backward per rollout step)."""
    from navillm_b200 import ops
    D, O = 4096, 100
    g = torch.Generator(device=cuda_dev).manual_seed(R)
    x = torch.randn(R, D, generator=g, device=cuda_dev).to(bf16)
    W = (0.02 * torch.randn(O, D, generator=g, device=cuda_dev)).to(bf16)
    bias = torch.randn(O, generator=g, device=cuda_dev).to(bf16)
    dy = torch.randn(R, O, generator=g, device=cuda_dev).to(bf16)
    dW0 = (0.5 * torch.randn(O, D, generator=g, device=cuda_dev)).to(bf16)
    db0 = torch.randn(O, generator=g, device=cuda_dev).to(bf16)
    dW, db = dW0.clone(), db0.clone()
    out = ops.head_fwd(x, W, bias)
    dx = ops.head_bwd(dy, x, W, dW=dW, db=db)
    torch.cuda.synchronize()
    xd, Wd, dyd = x.double(), W.double(), dy.double()
    ref = xd @ Wd.t() + bias.double()
    _check("out", out, ref, B8 * ref.abs() + (1 + B8) * 135 * U * (xd.abs() @ Wd.abs().t() + bias.double().abs()))
    ref = dyd @ Wd
    _check("dx", dx, ref, B8 * ref.abs() + (1 + B8) * (O + 1) * U * (dyd.abs() @ Wd.abs()))
    ref = dW0.double() + dyd.t() @ xd
    _check("dW", dW, ref, B8 * ref.abs() + (1 + B8) * (R + 1) * U * (dW0.double().abs() + dyd.abs().t() @ xd.abs()))
    ref = db0.double() + dyd.sum(0)
    _check("db", db, ref, B8 * ref.abs() + (1 + B8) * (R + 1) * U * (db0.double().abs() + dyd.abs().sum(0)))
