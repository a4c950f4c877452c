"""Opt-in fp8 (e4m3) KV cache of generate(): csrc/decode.cu (nv_kv_store_prefill_fp8, nv_decode_attn_rope_fp8), the layer call's
kv_mode 3 and ModifiedLlamaForCausalLM.set_kv_cache_dtype.

Every (sequence, position, head) row of 128 elements is stored as ``quantize_fp8_`` would round it, so the oracle of each
kernel is an existing bf16 kernel plus ``quantize_fp8_`` on [rows, 128] views:
  - stores: the bytes and exponents of ``quantize_fp8_`` on the rows ``kv_store_prefill`` writes;
  - attention: ``rope_`` + ``kv_append`` + rounding of the appended rows + bf16 ``decode_attn``, bit for bit, and the fp64
    bound of tests/test_decode_ops_gpu.py against attention over the rounded rows K' / V';
  - generate(): a run on the bf16 kernels, eager, without layer calls, whose cache is rounded after the prefill and whose
    appended rows are rounded at every step.
"""
import copy

import pytest
import torch

from tests.test_decode_ops_gpu import ATTN_CASES, NAN16, _attn_ref, _check_attn, _lens, _rope_ref, _tables

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
NAN8 = 0x7F              # e4m3 NaN: cache bytes a call must neither read nor write
EXP_SENTINEL = 99


def _round_rows(x):
    """quantize_fp8_ on the [rows, 128] view of a bf16 tensor whose last dimension is a multiple of 128: x is rounded in place
    to K'; returns (e4m3 bytes with x's shape, int8 exponents with shape x.shape[:-1] + (heads,))."""
    from navillm_b200 import ops
    shp = x.shape
    rows = x.reshape(-1, 128)
    q = torch.empty(rows.shape, dtype=ops.fp8, device=x.device)
    e = torch.empty(rows.shape[0], dtype=torch.int8, device=x.device)
    ops.quantize_fp8_(rows, q, e)
    x.copy_(rows.view(shp))
    return q.view(shp), e.view(*shp[:-1], shp[-1] // 128)


def _u8(t):
    return t.view(torch.uint8)


def _fp8_sentinel(B, Smax, H, dev):
    q = torch.full((B, Smax, H * 128), NAN8, dtype=torch.uint8, device=dev).view(torch.float8_e4m3fn)
    e = torch.full((B, Smax, H), EXP_SENTINEL, dtype=torch.int8, device=dev)
    return q, e


# ---------------------------------------------------------------------------------------------------------------------
# stores
# ---------------------------------------------------------------------------------------------------------------------
def _plant_edge_rows(qkv, HD, H):
    """Edge rows in K and V of the first tokens: all zero, negative zero, a subnormal amax, values that round to +-448, and
    an amax one bf16 step above 448 * 2^-8 (the next exponent)."""
    k = qkv[:, HD:2 * HD].view(-1, H, 128)
    v = qkv[:, 2 * HD:].view(-1, H, 128)
    k[0, 0] = 0.0
    v[0, 0] = -0.0
    k[1, 0] = torch.linspace(-1, 1, 128, device=qkv.device) * 1e-39           # bf16 subnormals
    v[1, 0] = 0.0
    v[1, 0, 5] = 9.2e-41
    k[2, 0] = 0.0
    k[2, 0, 0], k[2, 0, 1], k[2, 0, 2] = 1.75, -1.74, 1.73                    # 1.75 = 448 * 2^-8: e = -8, the others round to 448
    v[2, 0] = 0.0
    v[2, 0, 7], v[2, 0, 9] = -1.7578125, 1.74                                  # amax just above: e = -7
    k[3, 0] = -0.0
    k[3, 0, 64] = -3.0e38                                                      # near the top of the bf16 range


@pytest.mark.parametrize("H", [2, 32])
def test_kv_store_prefill_fp8_matches_quantizer(cuda_dev, H):
    """Bytes and exponents = quantize_fp8_ of the rows kv_store_prefill writes; rows at p >= Smax dropped, nothing else written."""
    from navillm_b200 import ops
    Smax = 64
    HD = H * 128
    seqlens = [5, 70, 1, 64, 0, 33]                                            # ragged, one empty, one past Smax
    B, T = len(seqlens), sum(seqlens)
    cu_h = [0]
    for l in seqlens:
        cu_h.append(cu_h[-1] + l)
    cu = torch.tensor(cu_h, dtype=torch.int32, device=cuda_dev)
    g = torch.Generator(device=cuda_dev).manual_seed(21 + H)
    qkv = (torch.randn(T, 3 * HD + 8, generator=g, device=cuda_dev) * 3).to(bf16)[:, :3 * HD]      # ld = 3*HD + 8
    _plant_edge_rows(qkv, HD, H)
    kc = torch.empty(B, Smax, HD, dtype=bf16, device=cuda_dev)
    kc.view(torch.int16).fill_(NAN16)
    vc = kc.clone()
    ops.kv_store_prefill(qkv, cu, kc, vc, B, T)
    written = torch.zeros(B, Smax, dtype=torch.bool, device=cuda_dev)
    for b, l in enumerate(seqlens):
        written[b, :min(l, Smax)] = True
    kq_ref, ke_ref = _round_rows(kc)
    vq_ref, ve_ref = _round_rows(vc)
    kq, ke = _fp8_sentinel(B, Smax, H, cuda_dev)
    vq, ve = _fp8_sentinel(B, Smax, H, cuda_dev)
    ops.kv_store_prefill_fp8(qkv, cu, kq, vq, ke, ve, B, T)
    torch.cuda.synchronize()
    for got, ref in ((kq, kq_ref), (vq, vq_ref), (ke, ke_ref), (ve, ve_ref)):
        assert torch.equal(got.view(torch.uint8)[written] if got.dtype != torch.int8 else got[written],
                           ref.view(torch.uint8)[written] if ref.dtype != torch.int8 else ref[written])
    assert bool((_u8(kq)[~written] == NAN8).all()) and bool((_u8(vq)[~written] == NAN8).all())
    assert bool((ke[~written] == EXP_SENTINEL).all()) and bool((ve[~written] == EXP_SENTINEL).all())
    # the edge rows: zero rows keep exponent 0, negative zero stays 0x80, the 448 rows hit the top byte
    assert int(ke[0, 0, 0]) == 0 and bool((_u8(kq)[0, 0, :128] == 0).all())
    assert int(ve[0, 0, 0]) == 0 and bool((_u8(vq)[0, 0, :128] == 0x80).all())
    assert int(ke[0, 1, 0]) == -117                                             # subnormal amax: clamped exponent
    assert int(ke[0, 2, 0]) == -8 and _u8(kq)[0, 2, :3].tolist() == [0x7E, 0xFE, 0x7E]
    assert int(ve[0, 2, 0]) == -7


def test_layer_call_prefill_fills_the_same_fp8_cache(cuda_dev, monkeypatch):
    """kv_mode 3 of the layer call and the per-kernel prefill store write the same bytes and exponents."""
    from navillm_b200 import llama, ops
    from navillm_b200.modified_lm import PackedPrompt
    g, cfg, tok, model = _golden(cuda_dev)
    lm = model.lang_model
    ids, mask = _qa_ids(g, tok)
    lm._ensure()
    d = lm.dims
    pp = PackedPrompt(ids, mask, lm, cuda_dev, generate_positions=True)
    Smax = 256
    assert max(pp.seqlens) < Smax and pp.T < 1024
    x = ops.embed_fwd(pp.ids, lm.model.embed_tokens.weight.data)
    caches = {}
    spy = _Fp8Spy(monkeypatch)
    for layer_call in (True, False):
        monkeypatch.setattr(llama.LlamaCore, "LAYER_CALL", layer_call)
        kc = [_fp8_sentinel(pp.B, Smax, d.n_heads, cuda_dev) for _ in range(d.n_layers)]
        vc = [_fp8_sentinel(pp.B, Smax, d.n_heads, cuda_dev) for _ in range(d.n_layers)]
        with torch.no_grad():
            lm.core.forward(x, pp.pos, pp.cu, pp.seqlens, save=False, kv_store=(kc, vc), out_rows=pp.last_rows)
        caches[layer_call] = kc + vc
    assert spy.layer == d.n_layers and spy.store == d.n_layers
    n_written = 0
    for (q1, e1), (q0, e0) in zip(caches[True], caches[False]):
        assert torch.equal(_u8(q1), _u8(q0)) and torch.equal(e1, e0)
        n_written += int((e1 != EXP_SENTINEL).sum())
    assert n_written == 2 * d.n_layers * d.n_heads * sum(pp.seqlens)


# ---------------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("use_pdl", [False, True], ids=["plain", "pdl"])
@pytest.mark.parametrize("B,H,Smax,scale,c3", ATTN_CASES)
def test_decode_attn_rope_fp8_is_bf16_attention_on_rounded_rows(cuda_dev, B, H, Smax, scale, c3, use_pdl):
    from navillm_b200 import ops
    HD = H * 128
    g = torch.Generator(device=cuda_dev).manual_seed(B * 7919 + H * 31 + Smax)
    lens_h = _lens(B, Smax, c3)
    lens = torch.tensor(lens_h, dtype=torch.int32, device=cuda_dev)
    cos_t, sin_t = _tables(Smax, H, cuda_dev)
    qkv = torch.randn(B, 3 * HD, generator=g, device=cuda_dev).to(bf16)
    kc = (torch.randn(B, Smax, HD, generator=g, device=cuda_dev) * 2).to(bf16)
    vc = torch.randn(B, Smax, HD, generator=g, device=cuda_dev).to(bf16)
    past = torch.arange(Smax, device=cuda_dev)[None, :] >= lens[:, None]          # the row the call writes and all after it
    kq, ke = _round_rows(kc)                                                        # cached rows K' / V' and their bytes
    vq, ve = _round_rows(vc)
    kc.view(torch.int16)[past] = NAN16
    vc.view(torch.int16)[past] = NAN16
    _u8(kq)[past] = NAN8
    _u8(vq)[past] = NAN8
    ke[past] = EXP_SENTINEL
    ve[past] = EXP_SENTINEL
    kq0, vq0, ke0, ve0, qkv0 = kq.clone(), vq.clone(), ke.clone(), ve.clone(), qkv.clone()

    out_buf = torch.full((B, HD + 64), 7.0, dtype=bf16, device=cuda_dev)            # ldo > H*128; pad columns keep 7
    with ops.pdl(use_pdl):
        ops.decode_attn_rope_fp8(qkv, lens, cos_t, sin_t, kq, vq, ke, ve, H, out=out_buf[:, :HD], scale=scale)
    torch.cuda.synchronize()
    assert torch.equal(qkv, qkv0)
    assert bool((out_buf[:, HD:] == 7.0).all())
    got = out_buf[:, :HD]

    # reference: rope_ + kv_append + rounding of the appended rows + bf16 decode_attn
    q = qkv.clone()
    ops.rope_(q, lens, cos_t, sin_t, 2 * H, 128)
    ops.kv_append(q, lens, kc, vc)
    bi, li = torch.arange(B, device=cuda_dev), lens.long()
    krow, vrow = kc[bi, li].contiguous(), vc[bi, li].contiguous()
    kq_new, ke_new = _round_rows(krow)
    vq_new, ve_new = _round_rows(vrow)
    kc[bi, li], vc[bi, li] = krow, vrow
    with ops.pdl(use_pdl):
        want = ops.decode_attn(q, kc, vc, lens, H, scale=scale)
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))

    # the appended rows are the quantizer's bytes and exponents; every other row is untouched
    assert torch.equal(_u8(kq)[bi, li], _u8(kq_new)) and torch.equal(ke[bi, li], ke_new)
    assert torch.equal(_u8(vq)[bi, li], _u8(vq_new)) and torch.equal(ve[bi, li], ve_new)
    other = torch.ones(B, Smax, dtype=torch.bool, device=cuda_dev)
    other[bi, li] = False
    for a, b in ((_u8(kq), _u8(kq0)), (_u8(vq), _u8(vq0)), (ke, ke0), (ve, ve0)):
        assert torch.equal(a[other], b[other])

    # fp64 attention over K' / V'
    q_rot = _rope_ref(qkv[:, :HD].view(B, H, 128), lens, cos_t, sin_t)
    ref, vmax = _attn_ref(q_rot, kc, vc, lens_h, 128 ** -0.5 if scale is None else scale)
    _check_attn(got, ref, vmax)


def test_fp8_wrappers_reject_bad_arguments(cuda_dev):
    from navillm_b200 import _lib, ops
    B, Smax, H = 2, 64, 2
    HD = H * 128
    qkv = torch.zeros(B, 3 * HD, dtype=bf16, device=cuda_dev)
    lens = torch.zeros(B, dtype=torch.int32, device=cuda_dev)
    cos_t, sin_t = _tables(Smax, H, cuda_dev)
    kq, ke = _fp8_sentinel(B, Smax, H, cuda_dev)
    vq, ve = _fp8_sentinel(B, Smax, H, cuda_dev)
    with pytest.raises(ValueError):
        ops.decode_attn_rope_fp8(qkv, lens, cos_t, sin_t, kq.view(torch.uint8), vq, ke, ve, H)
    with pytest.raises(ValueError):
        ops.decode_attn_rope_fp8(qkv, lens, cos_t, sin_t, kq, vq, ke[:, :, :1], ve, H)
    with pytest.raises(ValueError):
        ops.decode_attn_rope_fp8(qkv, lens, cos_t, sin_t, kq, vq, ke, ve, H + 1)
    L = _lib.load()
    s = _lib.stream_ptr()
    rc = L.nv_decode_attn_rope_fp8(_lib.ptr(qkv), _lib.i64(3 * HD), _lib.ptr(lens), _lib.ptr(cos_t), _lib.ptr(sin_t), _lib.ptr(kq),
                                   _lib.ptr(vq), _lib.ptr(ke), _lib.ptr(ve), _lib.ptr(qkv), _lib.i64(HD), 2, Smax, H, 64,
                                   _lib.f32(1.0), s)
    assert rc == -1
    rc = L.nv_decode_attn_rope_fp8(_lib.ptr(qkv), _lib.i64(3 * HD), _lib.ptr(lens), _lib.ptr(cos_t), _lib.ptr(sin_t), _lib.ptr(kq),
                                   _lib.ptr(vq), None, _lib.ptr(ve), _lib.ptr(qkv), _lib.i64(HD), 2, Smax, H, 128, _lib.f32(1.0), s)
    assert rc == -1
    cu = torch.tensor([0, 1, 2], dtype=torch.int32, device=cuda_dev)
    rc = L.nv_kv_store_prefill_fp8(_lib.ptr(qkv), _lib.i64(3 * HD + 4), _lib.ptr(cu), _lib.ptr(kq), _lib.ptr(vq), _lib.ptr(ke),
                                   _lib.ptr(ve), 2, 2, Smax, H, s)
    assert rc == -1


# ---------------------------------------------------------------------------------------------------------------------
# generate() on the golden tiny model
# ---------------------------------------------------------------------------------------------------------------------
def _golden(dev):
    from tests.test_fp8_weights_gpu import _golden_model
    return _golden_model(dev)


def _qa_ids(g, tok):
    text = tok(g["qa_in"]["prompts"])
    ids = text["input_ids"].clone()
    ids[ids == tok.special["<cand>"]] = 7
    return ids, text["attention_mask"]


def _batch(ids, mask, B):
    rep = (B + ids.shape[0] - 1) // ids.shape[0]
    return ids.repeat(rep, 1)[:B], mask.repeat(rep, 1)[:B]


class _Fp8Spy:
    """Counts the fp8 cache kernels the model reaches: stores (per-kernel), layer calls in cache mode 3, decode attention."""

    def __init__(self, monkeypatch):
        from navillm_b200 import ops
        self.store = self.layer = self.attn = 0
        store, attn, run = ops.kv_store_prefill_fp8, ops.decode_attn_rope_fp8, ops.LayerRunner.run

        def store_w(*a, **kw):
            self.store += 1
            return store(*a, **kw)

        def attn_w(*a, **kw):
            self.attn += 1
            return attn(*a, **kw)

        def run_w(obj, *a, **kw):
            self.layer += obj.args.kv_mode == 3
            return run(obj, *a, **kw)
        monkeypatch.setattr(ops, "kv_store_prefill_fp8", store_w)
        monkeypatch.setattr(ops, "decode_attn_rope_fp8", attn_w)
        monkeypatch.setattr(ops.LayerRunner, "run", run_w)


def _reference(lm, monkeypatch, kw):
    """generate() on the bf16 kernels, eagerly and without layer calls, with the cache rounded to K' / V' after the prefill
    and every appended row rounded before the attention reads it."""
    from navillm_b200 import llama, ops
    with monkeypatch.context() as m:
        m.setattr(llama.LlamaCore, "LAYER_CALL", False)
        fwd, attn_rope = llama.LlamaCore.forward, ops.decode_attn_rope

        def forward(self, *a, kv_store=None, **k):
            r = fwd(self, *a, kv_store=kv_store, **k)
            if kv_store is not None:
                for c in kv_store[0] + kv_store[1]:
                    _round_rows(c)
            return r

        def decode_attn_rope(qkv, lens, cos_t, sin_t, kc, vc, n_heads, *, out=None, scale=None):
            q = qkv.clone()
            ops.rope_(q, lens, cos_t, sin_t, 2 * n_heads, 128)
            ops.kv_append(q, lens, kc, vc)
            bi, li = torch.arange(kc.shape[0], device=kc.device), lens.long()
            for c in (kc, vc):
                rows = c[bi, li].contiguous()
                _round_rows(rows)
                c[bi, li] = rows
            return ops.decode_attn(q, kc, vc, lens, n_heads, out=out, scale=scale)
        m.setattr(llama.LlamaCore, "forward", forward)
        m.setattr(ops, "decode_attn_rope", decode_attn_rope)
        prev = lm.set_kv_cache_dtype("bf16")
        try:
            torch.manual_seed(123)
            return lm.generate(**dict(kw, use_cuda_graph=False)).cpu()
        finally:
            lm.set_kv_cache_dtype(prev)


def _fp8_run(lm, kw, graph):
    prev = lm.set_kv_cache_dtype("fp8")
    try:
        torch.manual_seed(123)
        return lm.generate(**dict(kw, use_cuda_graph=graph)).cpu()
    finally:
        lm.set_kv_cache_dtype(prev)


@pytest.mark.parametrize("fp8_weights", [False, True], ids=["bf16w", "fp8w"])
@pytest.mark.parametrize("B", [1, 5, 16, 20, 40])
def test_generate_fp8_kv_matches_rounded_bf16_reference(cuda_dev, monkeypatch, B, fp8_weights):
    """Greedy (eager and graph), sampled and trie-constrained tokens equal the rounded bf16 reference; the fp8 kernels ran."""
    from tests.test_trie_decode_gpu import WORDS, _bos_words
    from tests.test_trie_table_cpu import make_trie
    g, cfg, tok, model = _golden(cuda_dev)
    lm = model.lang_model
    if fp8_weights:
        model.quantize_weights_fp8()
    ids, mask = _batch(*_qa_ids(g, tok), B)
    trie = make_trie(_bos_words(tok, WORDS), eos=tok.eos_token_id)
    base = dict(input_ids=ids, attention_mask=mask, eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id)
    cases = {"greedy": dict(max_new_tokens=12, stop_on_eos=False),
             "sample": dict(max_new_tokens=12, stop_on_eos=False, do_sample=True, temperature=0.8),
             "trie": dict(max_new_tokens=7, trie=trie)}
    for name, extra in cases.items():
        kw = dict(base, **extra)
        want = _reference(lm, monkeypatch, kw)
        spy = _Fp8Spy(monkeypatch)
        eager = _fp8_run(lm, kw, graph=False)
        assert spy.attn > 0 and spy.layer + spy.store > 0, name
        assert torch.equal(eager, want), (name, eager[:, ids.shape[1]:], want[:, ids.shape[1]:])
        for _ in range(2):                                            # the capturing call, then a replaying one
            stats = {}
            assert torch.equal(_fp8_run(lm, dict(kw, stats=stats), graph=True), want), name
        assert stats["graph_replays"] > 0 or stats["decode_steps"] <= 1, name
        if name == "trie":
            assert stats["trie_path"] == "device"
        monkeypatch.undo()


@pytest.mark.parametrize("fp8_weights", [False, True], ids=["bf16w", "fp8w"])
def test_generate_fp8_kv_long_prompts_take_the_per_kernel_prefill(cuda_dev, monkeypatch, fp8_weights):
    """T >= 1024 packed prompt rows: the prefill runs per kernel (fused epilogues) and stores through kv_store_prefill_fp8."""
    g, cfg, tok, model = _golden(cuda_dev)
    lm = model.lang_model
    if fp8_weights:
        model.quantize_weights_fp8()
    gen = torch.Generator().manual_seed(5)
    ids = torch.randint(3, 250, (4, 300), generator=gen)
    mask = torch.ones_like(ids)
    mask[1, :40] = 0                                                  # left padding in one row
    kw = dict(input_ids=ids, attention_mask=mask, max_new_tokens=10, stop_on_eos=False, eos_token_id=tok.eos_token_id,
              pad_token_id=tok.unk_token_id)
    want = _reference(lm, monkeypatch, kw)
    spy = _Fp8Spy(monkeypatch)
    assert torch.equal(_fp8_run(lm, kw, graph=False), want)
    assert spy.store == lm.dims.n_layers and spy.layer == 0 and spy.attn > 0
    assert torch.equal(_fp8_run(lm, kw, graph=True), want)


# ---------------------------------------------------------------------------------------------------------------------
# bookkeeping
# ---------------------------------------------------------------------------------------------------------------------
def test_switching_formats_keeps_graphs_apart(cuda_dev, monkeypatch):
    """bf16 -> fp8 -> bf16 -> fp8: bf16 tokens never change, fp8 tokens never change, each format captures its own graph
    once and the cache tensors have the stated sizes."""
    from navillm_b200 import ops
    g, cfg, tok, model = _golden(cuda_dev)
    lm = model.lang_model
    B = 6
    ids, mask = _batch(*_qa_ids(g, tok), B)
    kw = dict(input_ids=ids, attention_mask=mask, max_new_tokens=12, stop_on_eos=False, use_cuda_graph=True)
    captures = {"n": 0}
    real = torch.cuda.graph

    def graph(*a, **k):
        captures["n"] += 1
        return real(*a, **k)
    monkeypatch.setattr(torch.cuda, "graph", graph)
    assert lm.kv_cache_dtype == "bf16"
    bf = lm.generate(**kw).cpu()
    assert model.set_kv_cache_dtype("fp8") == "bf16"
    f8 = lm.generate(**kw).cpu()
    assert captures["n"] == 2
    st8 = [s for k, s in lm._decode_states.items() if k[-1] == "fp8"]
    assert len(st8) == 1
    d = lm.dims
    Smax = st8[0].kc[0][0].shape[1]
    for c in st8[0].kc + st8[0].vc:
        q, e = c
        assert q.dtype == ops.fp8 and tuple(q.shape) == (B, Smax, d.hidden) and q.is_contiguous()
        assert e.dtype == torch.int8 and tuple(e.shape) == (B, Smax, d.n_heads) and e.is_contiguous()
        assert q.nbytes + e.nbytes == B * Smax * d.hidden * 2 // 2 + B * Smax * d.hidden * 2 // 256
    for fmt, want in (("bf16", bf), ("fp8", f8), ("bf16", bf)):
        model.set_kv_cache_dtype(fmt)
        stats = {}
        assert torch.equal(lm.generate(stats=stats, **kw).cpu(), want), fmt
        assert stats["graph_replays"] > 0
    assert captures["n"] == 2
    with pytest.raises(ValueError):
        lm.set_kv_cache_dtype("fp16")
    model.set_kv_cache_dtype("bf16")


def test_host_trie_processor_runs_on_the_fp8_cache(cuda_dev, monkeypatch):
    """logits_processor= (the host TrieLogitsProcessor path) decodes over the fp8 cache too, with the device path's tokens;
    a device-walk miss falls back to that path with the fp8 cache as well."""
    from oracle import navillm_oracle as O
    from tests.test_trie_decode_gpu import WORDS, _bos_words
    from tests.test_trie_table_cpu import make_trie
    g, cfg, tok, model = _golden(cuda_dev)
    lm = model.lang_model
    ids, mask = _batch(*_qa_ids(g, tok), 8)
    common = dict(input_ids=ids, attention_mask=mask, eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id, max_new_tokens=7)
    trie = make_trie(_bos_words(tok, WORDS), eos=tok.eos_token_id)
    spy = _Fp8Spy(monkeypatch)
    lm.set_kv_cache_dtype("fp8")
    try:
        torch.manual_seed(123)
        host = lm.generate(logits_processor=[O.TrieLogitsProcessor(copy.deepcopy(trie))], **common).cpu()
        assert spy.attn > 0
        stats = {}
        torch.manual_seed(123)
        dev = lm.generate(trie=trie, stats=stats, **common).cpu()
        assert stats["trie_path"] == "device" and torch.equal(host, dev)
        special = tok.special["<cand>"]
        miss = make_trie([[special, 11], [special, 12, 13]], eos=tok.eos_token_id)
        n = spy.attn
        out = lm.generate(trie=miss, stats=stats, **common).cpu()
        assert stats["trie_path"] == "device_miss_host" and spy.attn > n
        host_miss = lm.generate(logits_processor=[O.TrieLogitsProcessor(make_trie([[special, 11], [special, 12, 13]],
                                                                                    eos=tok.eos_token_id))], **common).cpu()
        assert torch.equal(out, host_miss)
    finally:
        lm.set_kv_cache_dtype("bf16")
    assert torch.equal(_reference(lm, monkeypatch, dict(common, logits_processor=[O.TrieLogitsProcessor(copy.deepcopy(trie))])), host)
