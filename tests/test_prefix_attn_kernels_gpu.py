"""Suffix attention over a KV cache (nv_attn_fwd_kv, nv_attn_bwd_kv) against fp64 references at PrefixKVCache's rollout and
flush shapes, with per-element bounds on o, lse, dq, dk, dv and the fp32 accumulator.

Sequence b holds kv_len keys in cache rows kv_start .. +kv_len and q_len query rows, the last q_len positions: query i sees
the keys j <= dk + i, dk = kv_len - q_len.  Key rows j < dk are cached: their dK / dV go into the fp32 accumulator acc.
Rows j >= dk are the suffix's own: the kernel hands them bf16(dK + acc0), and flush_grads() runs the kernel over a whole
prefix (kv_len = q_len) with a nonzero acc0.  The reference is fp64 autograd of the masked softmax, from the same bf16
inputs.  The bounds are those of tests/test_train_kernels_gpu.py §1, which derives every term; u = 2^-24, b = 2^-8.
  o:   b·|o_ref| + (1 + 2^-7)·(b + 2·eps_i + u·(39 + 71·nb_i))·sum_j P_ij·|v_j|       (bf16 P, the row sum, P·V, 1/l)
  lse: 2^-21 + 6u·ln(n_i) + 2u·|lse_ref| + 2u·Z_i + eps_i + u·(34 + 2·nb_i)            (__logf, m·ln 2, the error of l)
  with eps_i = u·(4 + 3·Z_i + 64·A_i) the fp32 error of one p, and these terms specific to the offset:
    n_i = dk + i + 1 visible keys; A_i, Z_i maxima over them;
    nb_i = (dk + min(q0 + 128, q_len) + 127) // 128 key blocks walked by the CTA of row i's query block (first row q0):
      the forward counts key blocks from dk + q0, and the last may be fully masked for row i (it rescales by exactly 1).
  dq:  b·|dq_ref| + (1 + 2^-7)·((b + R + tc_q + 3u)·(|dS| |K|) + E |K|) + 2^-126·(1 + fz·sum_j |k_j|),
       tc_q = 8u·ceil(kv_len / 16): the dq pass contracts over every key, cached ones included.
  dk, dv: G = the fp32 error of the gradient before it is stored, tc_k = 8u·ceil(q_len / 16) (the dk/dv pass contracts
       over the queries):
       G_dv = (1 + 2^-7)·(b + R + tc_k)·(|P|^T |dO|) + 2^-126·(1 + sum_i |dO_i|),
       G_dk = (1 + 2^-7)·((b + R + tc_k + 3u)·(|dS|^T |Q|) + E^T |Q|) + 2^-126·(1 + fz·sum_i |q_i|).
    cached rows j < dk, on acc - acc0 (exact in fp64): G + u·(|acc0| + |d_ref|).  No bf16 rounding happens here, so there
       is no b·|ref| term: an accumulator rounded to bf16 (b·|acc0|) fails it.  u·(...) is the fp32 add.
    suffix rows j >= dk, against ref = d_ref + acc0: b·|ref| + G + (1 + 2^-7)·u·|ref|  (the fp32 add, then the rounding).
  R, E, fz: the lse error carried into p, the error of dS, and the flush-to-zero factor, as in §1.
tests/test_prefix_attn_bounds_cpu.py shows on the CPU that an emulation of these rounding points passes the bounds and that
a mask off by one key, a masked 64-key sub-block taken as visible, a bf16 accumulator, suffix rows without acc0 and an lse
over the wrong offset each fail them.

Beside the bounds, bit for bit:
  - acc rows outside [0, dk) of each sequence's slot, and every row of the other slots, are untouched; a second run from
    the same acc0 gives the same bits;
  - a sequence's outputs do not depend on neighbours of 100x magnitude, on the packing order, on being launched alone or on
    its cache slot;
  - with nothing cached and acc0 = 0 the KV kernels equal nv_attn_fwd / nv_attn_bwd on the same rows (the same blocks,
    masks and order; only the tensor maps differ), except that the fp32 add of acc in the dk/dv epilogue, FADD.FTZ in the
    fast-math build, turns a dk or dv below 2^-126 into 0 where the packed kernel rounds it to bf16 (at most 2^-126);
  - the suffix rows' o, lse and dq equal the last q_len rows of nv_attn_fwd / nv_attn_bwd over the whole sequence: each row
    walks the same key blocks in the same order with the same arithmetic; the KV form may add key blocks that are fully
    masked for the row, which rescale by exactly 1 and add P = 0 through the wgmma;
  - nv_attn_fwd_kv_fp8 equals nv_attn_fwd_kv over bf16 caches holding its rounded rows K' / V'.
Every cache row past kv_len (the rest of a slot, the slots no sequence uses, rows a last key block reaches) holds finite
junk of about 100x the data's scale.
"""
import numpy as np
import pytest
import torch

from tests.test_fp8_kv_gpu import _round_rows
from tests.test_train_kernels_gpu import ATTN_CASES, HD, _attn_inputs, _attn_seq_check, _cu

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
JUNK = 100.0
SCALE = HD ** -0.5


def _rollout(B, seed):
    """A rollout step of PrefixKVCache (Smax 2048): 256..1024 cached prompt rows (C2), 1..300 new rows, sequences in a
    permutation of B + 1 slots so that one slot is unused."""
    rs = np.random.RandomState(seed)
    cached, q = rs.randint(256, 1025, B), rs.randint(1, 301, B)
    return dict(H=32, Smax=2048, q=q.tolist(), kv=(cached + q).tolist(), slots=rs.permutation(B + 1)[:B].tolist(), n_slots=B + 1)


BOUNDARY_DK = [0, 1, 63, 64, 65, 127, 128, 129, 191, 192]
BOUNDARY_Q = [128, 64, 129, 127, 65, 63, 192, 256, 191, 255]
CASES = {
    "rollout_b8": lambda: _rollout(8, 8),
    "rollout_b16": lambda: _rollout(16, 16),
    # the query sub-block partition across key-block edges in every way
    "boundary": lambda: dict(H=32, Smax=512, q=BOUNDARY_Q, kv=[d + q for d, q in zip(BOUNDARY_DK, BOUNDARY_Q)]),
    # flush_grads(): nothing cached, the whole prefix, acc0 != 0 (C5 lengths)
    "flush": lambda: dict(H=32, Smax=2048, q=[2048, 777, 1290], kv=[2048, 777, 1290]),
    # Smax % 128 != 0: sequence 0's last key block reads slot 1's rows; sequence 2 ends on the cache's last row, so its
    # last key block runs past Tkv
    "cache_end": lambda: dict(H=32, Smax=1000, q=[300, 37, 128], kv=[1000, 613, 1000]),
    # the cases the loose fp32 comparisons of test_prefix_reuse_gpu / test_prefix_train_gpu used
    "h2_mixed": lambda: dict(H=2, Smax=1024, q=[128, 70, 1, 300], kv=[128, 75, 130, 300]),
    "h2_long_prefix": lambda: dict(H=2, Smax=1024, q=[40, 257, 200], kv=[1000, 600, 333]),
    "h2_tiny": lambda: dict(H=2, Smax=1024, q=[5], kv=[5]),
    "h2_misaligned": lambda: dict(H=2, Smax=1024, q=[256, 129], kv=[511, 129 + 384]),
    "h32_straddle": lambda: dict(H=32, Smax=1024, q=[200, 77], kv=[200 + 190, 77 + 300]),
}


class _Setup:
    """The whole sequences (qkv of kv_len rows each, from _attn_inputs: with stress the sink is key 0, in the cached part,
    and the late maximum key 300, in key block 2), their K / V in the cache slots among junk, the suffix queries as a
    [Tq, H*128] view of ld 3*H*128 (as the layer passes them), and a random fp32 accumulator."""

    def __init__(self, case, stress, dev, seed=0):
        self.H, self.Smax, self.q_lens, self.kv_lens = case["H"], case["Smax"], case["q"], case["kv"]
        B = len(self.q_lens)
        self.slots = case.get("slots", list(range(B)))
        n_slots = case.get("n_slots", B)
        H, D = self.H, self.H * HD
        self.D = D
        seed += sum(self.kv_lens) + 3 * sum(self.q_lens) + H
        self.full = _attn_inputs(self.kv_lens, H, seed, dev, stress)
        self.cu_full = _cu(self.kv_lens, dev)
        g = torch.Generator(device=dev).manual_seed(seed + 1)
        self.kc = (JUNK * torch.randn(n_slots, self.Smax, D, generator=g, device=dev)).to(bf16)
        self.vc = (JUNK * torch.randn(n_slots, self.Smax, D, generator=g, device=dev)).to(bf16)
        rows, s0 = [], 0
        for b, (Lq, Lk) in enumerate(zip(self.q_lens, self.kv_lens)):
            self.kc[self.slots[b], :Lk] = self.full[s0:s0 + Lk, D:2 * D]
            self.vc[self.slots[b], :Lk] = self.full[s0:s0 + Lk, 2 * D:]
            rows.append(self.full[s0 + Lk - Lq:s0 + Lk])
            s0 += Lk
        self.q = torch.cat(rows)[:, :D]
        self.cu = _cu(self.q_lens, dev)
        self.kv_start = torch.tensor(self.slots, dtype=torch.int32, device=dev) * self.Smax
        self.kv_len = torch.tensor(self.kv_lens, dtype=torch.int32, device=dev)
        self.acc0 = torch.randn(n_slots, self.Smax, 2 * D, generator=g, device=dev)
        self.g = g

    def fwd(self):
        from navillm_b200 import ops
        lse = torch.empty(self.H, self.q.shape[0], dtype=torch.float32, device=self.q.device)
        o = ops.attn_fwd_kv(self.q, self.kc, self.vc, self.cu, self.q_lens, self.kv_start, self.kv_len, self.H, lse=lse)
        return o, lse

    def bwd(self, o, do, lse, dvec=None):
        from navillm_b200 import ops
        acc = self.acc0.clone()
        dqkv = ops.attn_bwd_kv(self.q, o, do, lse, self.kc, self.vc, acc, self.cu, self.q_lens, self.kv_start, self.kv_len,
                               self.kv_lens, self.H, dvec=dvec)
        return dqkv, acc

    def cached_rows(self):
        """bool [slots, Smax]: the rows [0, dk) of each sequence's slot, the only accumulator rows the backward may write."""
        m = torch.zeros(self.acc0.shape[:2], dtype=torch.bool, device=self.acc0.device)
        for s, Lq, Lk in zip(self.slots, self.q_lens, self.kv_lens):
            m[s, :Lk - Lq] = True
        return m


def _ref_check(st, o, lse, do, results):
    """Every sequence (a few heads at a time) of every backward result {tag: (dqkv, acc)} against the bounds; returns the
    worst err/tol per quantity."""
    H, D, worst, t0 = st.H, st.D, {}, 0
    for b, (Lq, Lk) in enumerate(zip(st.q_lens, st.kv_lens)):
        dk, s = Lk - Lq, st.slots[b]
        hc = max(1, min(H, (1 << 23) // (Lq * Lk)))
        for h0 in range(0, H, hc):
            hs = slice(h0, min(H, h0 + hc))
            heads = lambda t: t.reshape(t.shape[0], H, HD)[:, hs].double().transpose(0, 1)
            grads = {}
            for tag, (dqkv, acc) in results.items():
                rows = dqkv[t0:t0 + Lq]
                grads[tag] = (heads(rows[:, :D]), torch.cat([heads(acc[s, :dk, :D]), heads(rows[:, D:2 * D])], 1),
                              torch.cat([heads(acc[s, :dk, D:]), heads(rows[:, 2 * D:])], 1))
            w = _attn_seq_check(heads(st.q[t0:t0 + Lq]), heads(st.kc[s, :Lk]), heads(st.vc[s, :Lk]), heads(do[t0:t0 + Lq]),
                                heads(o[t0:t0 + Lq]), lse[hs, t0:t0 + Lq].double(), grads, SCALE,
                                f"seq {b} (q_len {Lq}, kv_len {Lk}) heads {h0}..{min(H, h0 + hc) - 1}",
                                acc0=(heads(st.acc0[s, :Lk, :D]), heads(st.acc0[s, :Lk, D:])))
            for n, r in w.items():
                worst[n] = max(worst.get(n, 0.0), r)
        t0 += Lq
    return worst


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


@pytest.mark.parametrize("stress", [False, True], ids=["randn", "stress"])
@pytest.mark.parametrize("case", list(CASES))
def test_prefix_attention_matches_fp64(cuda_dev, case, stress):
    """o, lse, dq, the suffix rows' dk / dv and the cached rows' accumulator against fp64 autograd, per element; the
    backward both computing D itself and with D handed over by gemm_attnd, as LlamaCore runs it from 1024 rows.  The
    accumulator rows the backward may not write keep their bits, and a second run gives the same bits."""
    from navillm_b200 import ops
    st = _Setup(CASES[case](), stress, cuda_dev)
    D, Tq = st.D, st.q.shape[0]
    o, lse = st.fwd()
    dy = torch.randn(Tq, D, generator=st.g, device=cuda_dev).to(bf16)
    wo = (torch.randn(D, D, generator=st.g, device=cuda_dev) * D ** -0.5).to(bf16)
    do, dvec = ops.gemm_attnd(dy, wo, o)
    del dy, wo
    own = st.bwd(o, do, lse)
    handed = st.bwd(o, do, lse, dvec=dvec)
    again = st.bwd(o, do, lse)
    torch.cuda.synchronize()
    assert torch.equal(_bits(own[0]), _bits(again[0])) and torch.equal(_bits(own[1]), _bits(again[1])), "two runs differ"
    keep = ~st.cached_rows()
    for tag, (_, acc) in (("own D", own), ("dvec", handed)):
        assert torch.equal(_bits(acc[keep]), _bits(st.acc0[keep])), f"{tag}: an accumulator row outside [0, dk) changed"
    del again
    worst = _ref_check(st, o, lse, do, {"own D": own, "dvec": handed})
    print(f"\n{case} {'stress' if stress else 'randn'} worst err/tol: " + ", ".join(f"{n} {r:.3g}" for n, r in worst.items()))


@pytest.mark.parametrize("stress", [False, True], ids=["randn", "stress"])
@pytest.mark.parametrize("case", ["rollout_b16", "boundary", "flush", "cache_end", "h2_long_prefix", "h32_straddle"])
def test_suffix_rows_are_the_full_sequence_rows(cuda_dev, case, stress):
    """o, lse and dq of the suffix rows are bit for bit the last q_len rows of nv_attn_fwd / nv_attn_bwd over the whole
    sequence: per row the same key blocks in the same order with the same arithmetic, plus possibly key blocks that are
    fully masked for the row (alpha = 1 exactly, P = 0 into the wgmma)."""
    from navillm_b200 import ops
    st = _Setup(CASES[case](), stress, cuda_dev)
    D, Tq = st.D, st.q.shape[0]
    o, lse = st.fwd()
    do = torch.randn(Tq, D, generator=st.g, device=cuda_dev).to(bf16)
    dq = st.bwd(o, do, lse)[0][:, :D]
    o_f, lse_f = ops.attn_fwd(st.full, st.cu_full, st.kv_lens, st.H)
    do_f = torch.randn(st.full.shape[0], D, generator=st.g, device=cuda_dev).to(bf16)
    t0, s0 = 0, 0
    for Lq, Lk in zip(st.q_lens, st.kv_lens):
        do_f[s0 + Lk - Lq:s0 + Lk] = do[t0:t0 + Lq]
        t0, s0 = t0 + Lq, s0 + Lk
    dq_f = ops.attn_bwd(st.full, o_f, do_f, lse_f, st.cu_full, st.kv_lens, st.H)[:, :D]
    torch.cuda.synchronize()
    t0, s0 = 0, 0
    for b, (Lq, Lk) in enumerate(zip(st.q_lens, st.kv_lens)):
        sfx = slice(s0 + Lk - Lq, s0 + Lk)
        for name, got, want in (("o", o[t0:t0 + Lq], o_f[sfx]), ("lse", lse[:, t0:t0 + Lq], lse_f[:, sfx]),
                                ("dq", dq[t0:t0 + Lq], dq_f[sfx])):
            diff = _bits(got) != _bits(want)
            assert not bool(diff.any()), (f"seq {b} (q_len {Lq}, kv_len {Lk}) {name}: {int(diff.sum())} elements differ from "
                                          f"the full sequence, first at {tuple(diff.nonzero()[0].tolist())}")
        t0, s0 = t0 + Lq, s0 + Lk


@pytest.mark.parametrize("stress", [False, True], ids=["randn", "stress"])
@pytest.mark.parametrize("lens", ["boundary", "c5"])
def test_nothing_cached_equals_packed_kernels(cuda_dev, lens, stress):
    """kv_len = q_len and acc0 = 0: attn_fwd_kv / attn_bwd_kv give the values of attn_fwd / attn_bwd on the same rows, and
    the accumulator stays 0.  o, lse and dq are the same bits.  dk and dv pass through the epilogue's fp32 add of acc, which
    the fast-math build compiles as FADD.FTZ: -0 + 0 is +0, and a gradient below 2^-126 (keys almost no query attends to, in
    the stressed heads) becomes 0 where the packed kernel rounds it to bf16: a subnormal, or 2^-126 itself when it rounds up.
    So they are compared as values, and where they differ the packed value must be at most 2^-126 and the KV value 0."""
    from navillm_b200 import ops
    lens = ATTN_CASES[lens]()
    H, B = 32, len(lens)
    D, T, Smax = H * HD, sum(lens), -(-max(lens) // 128) * 128
    qkv = _attn_inputs(lens, H, 77 + T, cuda_dev, stress)
    cu = _cu(lens, cuda_dev)
    g = torch.Generator(device=cuda_dev).manual_seed(T)
    do = torch.randn(T, D, generator=g, device=cuda_dev).to(bf16)
    o, lse = ops.attn_fwd(qkv, cu, lens, H)
    dqkv = ops.attn_bwd(qkv, o, do, lse, cu, lens, H)
    kc = (JUNK * torch.randn(B, Smax, D, generator=g, device=cuda_dev)).to(bf16)
    vc = (JUNK * torch.randn(B, Smax, D, generator=g, device=cuda_dev)).to(bf16)
    for b, (s0, L) in enumerate(zip(np.cumsum([0] + lens).tolist(), lens)):
        kc[b, :L] = qkv[s0:s0 + L, D:2 * D]
        vc[b, :L] = qkv[s0:s0 + L, 2 * D:]
    kv_start = torch.arange(B, dtype=torch.int32, device=cuda_dev) * Smax
    kv_len = torch.tensor(lens, dtype=torch.int32, device=cuda_dev)
    lse_k = torch.empty_like(lse)
    o_k = ops.attn_fwd_kv(qkv[:, :D], kc, vc, cu, lens, kv_start, kv_len, H, lse=lse_k)
    acc = torch.zeros(B, Smax, 2 * D, device=cuda_dev)
    dqkv_k = ops.attn_bwd_kv(qkv[:, :D], o_k, do, lse_k, kc, vc, acc, cu, lens, kv_start, kv_len, lens, H)
    torch.cuda.synchronize()
    assert torch.equal(_bits(o_k), _bits(o)) and torch.equal(_bits(lse_k), _bits(lse)), "forward differs from attn_fwd"
    assert torch.equal(_bits(dqkv_k[:, :D]), _bits(dqkv[:, :D])), "dq differs from attn_bwd"
    for name, c in (("dk", slice(D, 2 * D)), ("dv", slice(2 * D, 3 * D))):
        got, want = dqkv_k[:, c], dqkv[:, c]
        diff = got != want
        # an fp32 subnormal rounds to at most 2^-126 in bf16
        flushed = diff & (want.float().abs() <= 2.0 ** -126) & (got == 0)
        bad = (diff & ~flushed).nonzero()[:4].tolist()
        assert not bad, (f"{name}: {int((diff & ~flushed).sum())} elements differ from attn_bwd by more than a flushed "
                         f"subnormal: " + ", ".join(f"{tuple(ix)} {got[ix[0], ix[1]].item():.4g} vs {want[ix[0], ix[1]].item():.4g}"
                                                     for ix in bad))
        print(f"\n{name}: {int(flushed.sum())} subnormal gradients flushed to 0")
    assert not bool(_bits(acc).any()), "the accumulator changed"


def test_prefix_attention_is_packing_and_slot_invariant(cuda_dev):
    """A sequence's o, lse, dqkv and accumulator rows are the same bits packed among neighbours whose rows are about 100x
    larger, packed in another order, launched alone, and in another cache slot (Smax = 1000, so a slot's last key block
    reads the next slot's rows, which differ between the runs)."""
    from navillm_b200 import ops
    H, Smax = 32, 1000
    D = H * HD
    g = torch.Generator(device=cuda_dev).manual_seed(9)

    def seq(Lq, Lk, mag):
        r = lambda n, w: (mag * torch.randn(n, w, generator=g, device=cuda_dev))
        return dict(Lq=Lq, Lk=Lk, q=r(Lq, D).to(bf16), k=r(Lk, D).to(bf16), v=r(Lk, D).to(bf16), do=r(Lq, D).to(bf16),
                    acc0=r(Lk, 2 * D))

    own = [seq(129, 429, 1), seq(1, 700, 1), seq(64, 129, 1), seq(300, 491, 1), seq(37, 1000, 1)]
    nbr = [seq(77, 500, JUNK), seq(200, 200, JUNK), seq(31, 900, JUNK)]

    def run(items, slots, n_slots):
        """items: ("s", j) or ("n", j) in packing order, slots: their cache slots -> {j: outputs of own sequence j}"""
        parts = [(own if kind == "s" else nbr)[j] for kind, j in items]
        kc = (JUNK * torch.randn(n_slots, Smax, D, generator=g, device=cuda_dev)).to(bf16)
        vc = (JUNK * torch.randn(n_slots, Smax, D, generator=g, device=cuda_dev)).to(bf16)
        acc = JUNK * torch.randn(n_slots, Smax, 2 * D, generator=g, device=cuda_dev)
        for p, s in zip(parts, slots):
            kc[s, :p["Lk"]], vc[s, :p["Lk"]], acc[s, :p["Lk"]] = p["k"], p["v"], p["acc0"]
        q_lens, kv_lens = [p["Lq"] for p in parts], [p["Lk"] for p in parts]
        q, do = torch.cat([p["q"] for p in parts]), torch.cat([p["do"] for p in parts])
        cu = _cu(q_lens, cuda_dev)
        kv_start = torch.tensor(slots, dtype=torch.int32, device=cuda_dev) * Smax
        kv_len = torch.tensor(kv_lens, dtype=torch.int32, device=cuda_dev)
        lse = torch.empty(H, q.shape[0], dtype=torch.float32, device=cuda_dev)
        o = ops.attn_fwd_kv(q, kc, vc, cu, q_lens, kv_start, kv_len, H, lse=lse)
        dqkv = ops.attn_bwd_kv(q, o, do, lse, kc, vc, acc, cu, q_lens, kv_start, kv_len, kv_lens, H)
        torch.cuda.synchronize()
        out, t0 = {}, 0
        for (kind, j), p, s in zip(items, parts, slots):
            if kind == "s":
                out[j] = tuple(_bits(x.clone()) for x in (o[t0:t0 + p["Lq"]], lse[:, t0:t0 + p["Lq"]], dqkv[t0:t0 + p["Lq"]],
                                                          acc[s, :p["Lk"]]))
            t0 += p["Lq"]
        return out

    order_a = [("n", 0), ("s", 0), ("n", 1), ("s", 1), ("s", 2), ("n", 2), ("s", 3), ("s", 4)]
    order_b = [("s", 4), ("s", 2), ("n", 1), ("s", 0), ("s", 3), ("n", 0), ("s", 1)]
    a = run(order_a, list(range(8)), 8)
    b = run(order_b, [6, 0, 3, 5, 1, 4, 2], 8)
    for j in range(len(own)):
        alone = run([("s", j)], [(j + 2) % 4], 4)
        for name, x, y, z in zip(("o", "lse", "dqkv", "acc"), a[j], b[j], alone[j]):
            assert torch.equal(x, y), f"seq {j} {name}: differs between two packings"
            assert torch.equal(x, z), f"seq {j} {name}: differs between packed and alone"


@pytest.mark.parametrize("case", ["rollout_b16", "boundary", "flush", "cache_end"])
def test_attn_fwd_kv_fp8_matches_bf16_on_rounded_rows(cuda_dev, case):
    """nv_attn_fwd_kv_fp8 is bit for bit nv_attn_fwd_kv over bf16 caches holding its rounded rows K' / V', junk included."""
    from navillm_b200 import ops
    st = _Setup(CASES[case](), False, cuda_dev)
    kq, ke = _round_rows(st.kc)                          # st.kc, st.vc now hold K', V'
    vq, ve = _round_rows(st.vc)
    want, _ = st.fwd()
    got = ops.attn_fwd_kv_fp8(st.q, kq, vq, ke, ve, st.cu, st.q_lens, st.kv_start, st.kv_len, st.H)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(got.float()).all())
    assert torch.equal(_bits(got), _bits(want))
