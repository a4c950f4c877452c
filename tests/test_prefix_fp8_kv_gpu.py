"""Opt-in fp8 (e4m3) store of PrefixKVCache: csrc/decode.cu (nv_kv_store_suffix_fp8), csrc/attn_fwd.cu (nv_attn_fwd_kv_fp8),
the layer call's kv_mode 4, LlamaCore.forward_suffix and PrefixKVCache(kv_dtype="fp8").

Every cached (sequence, position, head) row of 128 elements is stored as ``quantize_fp8_`` would round it (K' / V'), and
e4m3 * 2^e is exact in bf16, so each oracle is an existing bf16 kernel on rounded rows, compared bit for bit:
  - store: the bytes and exponents of ``quantize_fp8_`` on the rows ``kv_store_suffix`` writes;
  - attention: ``attn_fwd_kv`` on bf16 caches holding K' / V';
  - forward_suffix and the rollout: the bf16 cache path, per kernel, with the cache rounded to K' / V' after every store.
"""
import numpy as np
import pytest
import torch

from tests.test_decode_ops_gpu import NAN16
from tests.test_fp8_kv_gpu import EXP_SENTINEL, NAN8, _fp8_sentinel, _plant_edge_rows, _round_rows, _u8
from tests.test_prefix_reuse_gpu import _build, _nav_batch

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


def _cu(lens, dev):
    return torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device=dev)


# ---------------------------------------------------------------------------------------------------------------------
# store
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [2, 32])
def test_kv_store_suffix_fp8_matches_quantizer(cuda_dev, H):
    """Bytes and exponents = quantize_fp8_ of the rows kv_store_suffix writes after the cached rows; nothing else written."""
    from navillm_b200 import ops
    Smax = 64
    HD = H * 128
    q_lens = [5, 17, 1, 0, 9]
    cached_h = [0, 13, 63, 40, 60]              # row 2 ends at Smax - 1; row 4 runs past Smax (rows >= Smax dropped)
    B, T = len(q_lens), sum(q_lens)
    cu = _cu(q_lens, cuda_dev)
    cached = torch.tensor(cached_h, dtype=torch.int32, device=cuda_dev)
    g = torch.Generator(device=cuda_dev).manual_seed(5 + H)
    qkv = (torch.randn(T, 3 * HD + 8, generator=g, device=cuda_dev) * 3).to(bf16)[:, :3 * HD]      # ld = 3*HD + 8
    _plant_edge_rows(qkv, HD, H)
    kc = torch.empty(B, Smax, HD, dtype=bf16, device=cuda_dev)
    kc.view(torch.int16).fill_(NAN16)
    vc = kc.clone()
    ops.kv_store_suffix(qkv, cu, cached, kc, vc, B, T)
    written = torch.zeros(B, Smax, dtype=torch.bool, device=cuda_dev)
    for b, (c, l) in enumerate(zip(cached_h, q_lens)):
        written[b, c:min(c + l, Smax)] = True
    kq_ref, ke_ref = _round_rows(kc)
    vq_ref, ve_ref = _round_rows(vc)
    kq, ke = _fp8_sentinel(B, Smax, H, cuda_dev)
    vq, ve = _fp8_sentinel(B, Smax, H, cuda_dev)
    ops.kv_store_suffix_fp8(qkv, cu, cached, kq, vq, ke, ve, B, T)
    torch.cuda.synchronize()
    assert int(written.sum()) == 5 + 17 + 1 + 0 + 4
    for got, ref in ((_u8(kq), _u8(kq_ref)), (_u8(vq), _u8(vq_ref)), (ke, ke_ref), (ve, ve_ref)):
        assert torch.equal(got[written], ref[written])
    assert bool((_u8(kq)[~written] == NAN8).all()) and bool((_u8(vq)[~written] == NAN8).all())
    assert bool((ke[~written] == EXP_SENTINEL).all()) and bool((ve[~written] == EXP_SENTINEL).all())
    # the edge rows of the first tokens (sequence 0, cached 0) kept their quantizer results
    assert int(ke[0, 0, 0]) == 0 and bool((_u8(kq)[0, 0, :128] == 0).all())
    assert int(ke[0, 1, 0]) == -117
    assert int(ke[0, 2, 0]) == -8 and _u8(kq)[0, 2, :3].tolist() == [0x7E, 0xFE, 0x7E]


# ---------------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------------
ATTN_CASES = [
    dict(H=2, Smax=1024, q=[128, 70, 1, 300], kv=[128, 75, 130, 300]),         # the cases of test_prefix_reuse_gpu
    dict(H=2, Smax=1024, q=[40, 257, 200], kv=[1000, 600, 333]),
    dict(H=2, Smax=1024, q=[5], kv=[5]),
    dict(H=2, Smax=1024, q=[256, 129], kv=[511, 129 + 384]),
    # full width; Smax not a multiple of 128: key blocks cross into the next row's cache and, for the last row, past the end
    dict(H=32, Smax=2000, q=[128, 37, 300], kv=[2000, 1061, 1990]),
]


@pytest.mark.parametrize("case", ATTN_CASES, ids=lambda c: f"H{c['H']}-q{'_'.join(map(str, c['q']))}")
def test_attn_fwd_kv_fp8_is_bf16_attention_on_rounded_rows(cuda_dev, case):
    """torch.equal with attn_fwd_kv over bf16 caches holding K' / V'; finite junk past kv_len (every cache row is random and
    rows past kv_len are large) does not matter, and neither does zeroing it."""
    from navillm_b200 import ops
    H, Smax, q_lens, kv_lens = case["H"], case["Smax"], case["q"], case["kv"]
    HD, B, Tq = H * 128, len(q_lens), sum(q_lens)
    g = torch.Generator(device=cuda_dev).manual_seed(Tq + sum(kv_lens) + H)
    q = (torch.randn(Tq, 3 * HD, generator=g, device=cuda_dev) * 2).to(bf16)          # q view with ld = 3*HD, as in the layer
    kc = (torch.randn(B, Smax, HD, generator=g, device=cuda_dev) * 2).to(bf16)
    vc = torch.randn(B, Smax, HD, generator=g, device=cuda_dev).to(bf16)
    for b in range(B):
        kc[b, kv_lens[b]:] *= 1000.0                                                      # junk that would dominate the scores
        vc[b, kv_lens[b]:] *= -3000.0
    kq, ke = _round_rows(kc)                                                              # kc, vc now hold K', V'
    vq, ve = _round_rows(vc)
    cu = _cu(q_lens, cuda_dev)
    kv_start = torch.arange(B, dtype=torch.int32, device=cuda_dev) * Smax
    kv_len = torch.tensor(kv_lens, dtype=torch.int32, device=cuda_dev)
    qv = q[:, :HD]
    want = ops.attn_fwd_kv(qv, kc, vc, cu, q_lens, kv_start, kv_len, H)
    got = ops.attn_fwd_kv_fp8(qv, kq, vq, ke, ve, cu, q_lens, kv_start, kv_len, H)
    torch.cuda.synchronize()
    assert torch.isfinite(got).all()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))
    past = torch.arange(Smax, device=cuda_dev)[None, :] >= kv_len[:, None]
    for t in (_u8(kq), _u8(vq), ke, ve):
        t[past] = 0
    again = ops.attn_fwd_kv_fp8(qv, kq, vq, ke, ve, cu, q_lens, kv_start, kv_len, H)
    torch.cuda.synchronize()
    assert torch.equal(again.view(torch.int16), want.view(torch.int16))


# ---------------------------------------------------------------------------------------------------------------------
# forward_suffix: layer call (kv_mode 4), per kernel, per kernel with fused epilogues
# ---------------------------------------------------------------------------------------------------------------------
class _Spy:
    """Counts the fp8 suffix kernels the model reaches: layer calls in cache mode 4, per-kernel stores and attentions."""

    def __init__(self, monkeypatch):
        from navillm_b200 import ops
        self.layer = self.store = self.attn = 0
        store, attn, run = ops.kv_store_suffix_fp8, ops.attn_fwd_kv_fp8, ops.LayerRunner.run

        def store_w(*a, **kw):
            self.store += 1
            return store(*a, **kw)

        def attn_w(*a, **kw):
            self.attn += 1
            return attn(*a, **kw)

        def run_w(obj, *a, **kw):
            self.layer += obj.args.kv_mode == 4
            return run(obj, *a, **kw)
        monkeypatch.setattr(ops, "kv_store_suffix_fp8", store_w)
        monkeypatch.setattr(ops, "attn_fwd_kv_fp8", attn_w)
        monkeypatch.setattr(ops.LayerRunner, "run", run_w)


def _rounding_store(m):
    """ops.kv_store_suffix followed by rounding of the whole cache to K' / V' (already rounded rows keep their values)."""
    from navillm_b200 import ops
    real = ops.kv_store_suffix

    def store(qkv, cu, cached, kc, vc, B, T):
        real(qkv, cu, cached, kc, vc, B, T)
        _round_rows(kc)
        _round_rows(vc)
    m.setattr(ops, "kv_store_suffix", store)


def _widen(pair):
    q, e = pair
    B, S, HD = q.shape
    return (q.float().view(B, S, HD // 128, 128) * torch.exp2(e.float())[..., None]).view(B, S, HD).to(bf16)


def _suffix_steps(core, steps, kc, vc, dev):
    """Run forward_suffix for each (q_lens, cached) step over the given caches; returns the outputs at every row."""
    D = core.d.hidden
    outs = []
    for i, (q_lens, cached_h) in enumerate(steps):
        g = torch.Generator(device=dev).manual_seed(40 + i)
        T = sum(q_lens)
        x = torch.randn(T, D, generator=g, device=dev).to(bf16)
        pos = torch.cat([torch.arange(c, c + l, dtype=torch.int32) for c, l in zip(cached_h, q_lens)]).to(dev)
        cu = _cu(q_lens, dev)
        B = len(q_lens)
        Smax = (kc[0][0] if isinstance(kc[0], tuple) else kc[0]).shape[1]
        cached = torch.tensor(cached_h, dtype=torch.int32, device=dev)
        kv_start = torch.arange(B, dtype=torch.int32, device=dev) * Smax
        kv_len = torch.tensor([c + l for c, l in zip(cached_h, q_lens)], dtype=torch.int32, device=dev)
        with torch.no_grad():
            outs.append(core.forward_suffix(x, pos, cu, q_lens, kc, vc, cached, kv_start, kv_len).clone())
    return outs


@pytest.mark.parametrize("fp8_weights", [False, True], ids=["bf16w", "fp8w"])
def test_suffix_paths_write_the_same_fp8_cache(cuda_dev, monkeypatch, fp8_weights):
    """The layer call (kv_mode 4), the per-kernel path and a >= 1024-row step (fused epilogues) write the same bytes and give
    the same rows as the bf16 per-kernel path over a cache rounded after every store."""
    from navillm_b200 import llama
    model, d = _build(cuda_dev)
    if fp8_weights:
        model.quantize_weights_fp8()
    lm = model.lang_model
    lm._ensure()
    core = lm.core
    L, H, D, B, Smax = d["n_layers"], d["n_heads"], d["hidden"], 3, 1024
    steps = [([60, 1, 33], [0, 0, 0]), ([7, 20, 1], [60, 1, 33]), ([400, 380, 300], [67, 21, 34])]   # the last: 1080 rows
    assert sum(steps[-1][0]) >= 1024 and sum(steps[1][0]) < 1024

    def fp8_cache():
        return ([(torch.zeros(B, Smax, D, dtype=torch.float8_e4m3fn, device=cuda_dev),
                  torch.zeros(B, Smax, H, dtype=torch.int8, device=cuda_dev)) for _ in range(L)],
                [(torch.zeros(B, Smax, D, dtype=torch.float8_e4m3fn, device=cuda_dev),
                  torch.zeros(B, Smax, H, dtype=torch.int8, device=cuda_dev)) for _ in range(L)])

    with monkeypatch.context() as m:
        m.setattr(llama.LlamaCore, "LAYER_CALL", False)
        _rounding_store(m)
        rk = [torch.zeros(B, Smax, D, dtype=bf16, device=cuda_dev) for _ in range(L)]
        rv = [torch.zeros(B, Smax, D, dtype=bf16, device=cuda_dev) for _ in range(L)]
        want = _suffix_steps(core, steps, rk, rv, cuda_dev)

    results = {}
    for layer_call in (True, False):
        with monkeypatch.context() as m:
            m.setattr(llama.LlamaCore, "LAYER_CALL", layer_call)
            spy = _Spy(m)
            kc, vc = fp8_cache()
            got = _suffix_steps(core, steps, kc, vc, cuda_dev)
            torch.cuda.synchronize()
            if layer_call:      # the two small steps through the layer call, the 1080-row step per kernel (fused epilogues)
                assert spy.layer == 2 * L and spy.store == L and spy.attn == L
            else:
                assert spy.layer == 0 and spy.store == 3 * L and spy.attn == 3 * L
        for i, (a, b) in enumerate(zip(got, want)):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), (layer_call, i)
        for pair, ref in zip(kc + vc, rk + rv):
            assert torch.equal(_widen(pair).view(torch.int16), ref.view(torch.int16)), layer_call
        results[layer_call] = kc + vc
    for (q1, e1), (q0, e0) in zip(results[True], results[False]):
        assert torch.equal(_u8(q1), _u8(q0)) and torch.equal(e1, e0)


# ---------------------------------------------------------------------------------------------------------------------
# rollout through NavModel
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fp8_weights", [False, True], ids=["bf16w", "fp8w"])
def test_rollout_with_fp8_prefix_cache_matches_rounded_bf16(cuda_dev, monkeypatch, fp8_weights):
    """5-step, 2-row rollout: fuse_logits and fuse_embeds with PrefixKVCache(kv_dtype="fp8") are bit for bit those of a bf16
    cache rounded to K' / V' after every store; the fp8 kernels ran; reset(rows=[0]) clears only row 0; nbytes halves."""
    from navillm_b200 import llama
    from navillm_b200.modified_lm import PrefixKVCache
    model, d = _build(cuda_dev)
    if fp8_weights:
        model.quantize_weights_fp8()
    lm = model.lang_model
    g = torch.Generator().manual_seed(11)
    instr = ["walk past the sofa and stop at the door of the kitchen", "leave the room"]
    hist = [[], []]
    cache = PrefixKVCache(lm, batch_size=2, max_len=256, kv_dtype="fp8")
    ref_cache = PrefixKVCache(lm, batch_size=2, max_len=256)
    assert cache.kv_dtype == "fp8" and ref_cache.kv_dtype == "bf16"
    assert cache.nbytes == ref_cache.nbytes // 2 + ref_cache.nbytes // 256
    to_dev = lambda b: {k: (v.to(cuda_dev) if torch.is_tensor(v) else v) for k, v in b.items()}
    spy = _Spy(monkeypatch)
    with torch.no_grad():
        for step in range(5):
            batch = _nav_batch(d, step, hist, g, instr)
            batch["hist_vis"] = [[v.to(cuda_dev) for v in vs] for vs in batch["hist_vis"]]
            with monkeypatch.context() as m:
                m.setattr(llama.LlamaCore, "LAYER_CALL", False)
                _rounding_store(m)
                torch.manual_seed(100 + step)
                ref = model("navigation", to_dev(dict(batch)), prefix_cache=ref_cache)
            n = spy.layer + spy.store
            torch.manual_seed(100 + step)
            got = model("navigation", to_dev(dict(batch)), prefix_cache=cache)
            assert spy.layer + spy.store == n + d["n_layers"], step
            assert torch.equal(got["fuse_logits"].cpu(), ref["fuse_logits"].cpu()), step
            assert torch.equal(got["fuse_embeds"].cpu(), ref["fuse_embeds"].cpu()), step
            for b in range(2):
                hist[b].append(ref["fuse_embeds"][b, 2].float().cpu())
    for pair, r in zip(cache.kc + cache.vc, ref_cache.kc + ref_cache.vc):
        assert torch.equal(_widen(pair).view(torch.int16), r.view(torch.int16))
    assert cache.stats == ref_cache.stats and cache.stats["tokens_encoded"] < cache.stats["tokens"]
    cache.reset(rows=[0])
    assert cache.ids[0].size == 0 and cache.ids[1].size > 0 and cache.off[0] is None and cache.off[1] is not None


# ---------------------------------------------------------------------------------------------------------------------
# bad arguments
# ---------------------------------------------------------------------------------------------------------------------
def test_fp8_suffix_wrappers_reject_bad_arguments(cuda_dev):
    from navillm_b200 import _lib, ops
    from navillm_b200.modified_lm import PrefixKVCache
    B, Smax, H = 2, 64, 2
    HD = H * 128
    qkv = torch.zeros(4, 3 * HD, dtype=bf16, device=cuda_dev)
    cu = torch.tensor([0, 1, 4], dtype=torch.int32, device=cuda_dev)
    cached = torch.zeros(B, dtype=torch.int32, device=cuda_dev)
    kv_start = torch.tensor([0, Smax], dtype=torch.int32, device=cuda_dev)
    kv_len = torch.tensor([1, 3], dtype=torch.int32, device=cuda_dev)
    kq, ke = _fp8_sentinel(B, Smax, H, cuda_dev)
    vq, ve = _fp8_sentinel(B, Smax, H, cuda_dev)
    before = [t.clone() for t in (_u8(kq), _u8(vq), ke, ve)]
    q = qkv[:, :HD]
    bad_store = [
        (qkv, cu, cached, kq.view(torch.uint8), vq, ke, ve),             # bytes not e4m3
        (qkv, cu, cached, kq, vq, ke.to(torch.int16), ve),               # exponents not int8
        (qkv, cu, cached, kq, vq, ke[:, :, :1], ve),                     # exponents of the wrong shape
        (qkv, cu, cached, kq, vq[:1], ke, ve[:1]),                       # K and V caches differ
        (qkv.float(), cu, cached, kq, vq, ke, ve),                       # qkv not bf16
        (qkv[:, :2 * HD], cu, cached, kq, vq, ke, ve),                   # qkv too narrow
        (qkv, cu, cached.long(), kq, vq, ke, ve),                        # cached not int32
    ]
    for args in bad_store:
        with pytest.raises(ValueError):
            ops.kv_store_suffix_fp8(*args, B, 4)
    bad_attn = [
        ((q, kq.view(torch.uint8), vq, ke, ve), H),
        ((q, kq, vq, ke, ve.to(torch.uint8)), H),
        ((q, kq, vq, ke, ve), H + 1),                                    # heads do not match the cache width
        ((q.float(), kq, vq, ke, ve), H),
        ((q[:3], kq, vq, ke, ve), H),                                    # rows do not match q_lens
    ]
    for args, heads in bad_attn:
        with pytest.raises(ValueError):
            ops.attn_fwd_kv_fp8(*args, cu, [1, 3], kv_start, kv_len, heads)
    with pytest.raises(ValueError):
        ops.attn_fwd_kv_fp8(q, kq, vq, ke, ve, cu, [1, 3], kv_start.long(), kv_len, H)
    L = _lib.load()
    s = _lib.stream_ptr()
    out = torch.zeros(4, HD, dtype=bf16, device=cuda_dev)
    P = _lib.ptr
    for head_dim, ke_p in ((64, P(ke)), (128, None)):                   # head_dim != 128, a null exponent pointer
        rc = L.nv_attn_fwd_kv_fp8(P(q), _lib.i64(3 * HD), P(kq), P(vq), ke_p, P(ve), P(out), _lib.i64(HD), None, P(cu), P(kv_start),
                                  P(kv_len), 2, 4, B * Smax, H, head_dim, 2, _lib.f32(1.0), s)
        assert rc == -1
    rc = L.nv_kv_store_suffix_fp8(P(qkv), _lib.i64(3 * HD + 4), P(cu), P(cached), P(kq), P(vq), P(ke), P(ve), 2, 4, Smax, H, s)
    assert rc == -1
    rc = L.nv_kv_store_suffix_fp8(P(qkv), _lib.i64(3 * HD), P(cu), None, P(kq), P(vq), P(ke), P(ve), 2, 4, Smax, H, s)
    assert rc == -1
    torch.cuda.synchronize()
    for t, t0 in zip((_u8(kq), _u8(vq), ke, ve), before):
        assert torch.equal(t, t0)
    model, _ = _build(cuda_dev)
    with pytest.raises(ValueError):
        PrefixKVCache(model.lang_model, batch_size=2, max_len=64, kv_dtype="fp16")
