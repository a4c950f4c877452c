"""Prompt-lookup speculative decoding on the device: the window attention bit for bit against sequential decode steps, the draft
and accept kernels against tests/lookup_oracle.py, and generate(prompt_lookup_num_tokens=k) end to end: the same ids whatever
the drafts, greedy semantics teacher-forced against the CPU oracle, widths and pads, graphs, cache formats and weight copies,
and the launches of every other call."""
import numpy as np
import pytest
import torch

from tests import lookup_oracle as LO
from tests.test_decode_ops_gpu import _tables
from tests.test_fp8_kv_gpu import _round_rows

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


# ---------------------------------------------------------------------------------------------------------------------
# window attention
# ---------------------------------------------------------------------------------------------------------------------
def _window_case(dev, B, H, Smax, lens, W, fp8, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    HD = H * 128
    qkv = torch.randn(B * W, 3 * HD, generator=g, device=dev).to(bf16)
    kc = (torch.randn(B, Smax, HD, generator=g, device=dev) * 0.5).to(bf16)
    vc = torch.randn(B, Smax, HD, generator=g, device=dev).to(bf16)
    lens_t = torch.tensor(lens, dtype=torch.int32, device=dev)
    if fp8:
        kq, ke = _round_rows(kc)
        vq, ve = _round_rows(vc)
        return qkv, lens_t, [kq, vq, ke, ve]
    return qkv, lens_t, [kc, vc]


WINDOW_CASES = [(4, 2, 512, [1, 60, 63, 200]), (3, 32, 2048, [1, 127, None]), (2, 32, 1000, [64, None])]


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
@pytest.mark.parametrize("W", [1, 2, 5, 8, 16])
@pytest.mark.parametrize("case", range(len(WINDOW_CASES)), ids=["H2", "H32", "H32_end"])
def test_window_equals_sequential_decode_steps(cuda_dev, fp8, W, case):
    """Every output element and every cache byte (exponents included) of decode_attn_rope_window[_fp8] equals W sequential
    decode_attn_rope[_fp8] calls; None in lens puts the window's last row on the cache's last row."""
    from navillm_b200 import ops
    B, H, Smax, lens = WINDOW_CASES[case]
    lens = [Smax - W if l is None else l for l in lens]
    qkv, lens_t, caches = _window_case(cuda_dev, B, H, Smax, lens, W, fp8, seed=W)
    cos_t, sin_t = _tables(Smax, H, cuda_dev)
    ref = [c.clone() for c in caches]
    HD = H * 128
    win = ops.decode_attn_rope_window_fp8 if fp8 else ops.decode_attn_rope_window
    one = ops.decode_attn_rope_fp8 if fp8 else ops.decode_attn_rope
    out = win(qkv, lens_t, cos_t, sin_t, *caches, H, W)
    want = torch.empty_like(out)
    rows = torch.arange(B, device=cuda_dev) * W
    for j in range(W):
        want[rows + j] = one(qkv[rows + j].contiguous(), lens_t + j, cos_t, sin_t, *ref, H)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), want.view(torch.int16)), (out.float() - want.float()).abs().max()
    for got, exp in zip(caches, ref):
        assert torch.equal(got.view(torch.uint8), exp.view(torch.uint8))
    assert out.shape == (B * W, HD)


def test_window_rejects_bad_arguments(cuda_dev):
    from navillm_b200 import ops
    qkv, lens_t, (kc, vc) = _window_case(cuda_dev, 2, 2, 256, [3, 4], 17, False)
    cos_t, sin_t = _tables(256, 2, cuda_dev)
    with pytest.raises(ValueError, match="window of 17"):
        ops.decode_attn_rope_window(qkv, lens_t, cos_t, sin_t, kc, vc, 2, 17)
    with pytest.raises(ValueError, match="qkv"):
        ops.decode_attn_rope_window(qkv, lens_t, cos_t, sin_t, kc, vc, 2, 4)


# ---------------------------------------------------------------------------------------------------------------------
# draft and accept kernels
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k,ngram", [(1, 2), (4, 1), (8, 3), (15, 2)])
def test_lookup_draft_matches_oracle(cuda_dev, k, ngram):
    from navillm_b200 import ops
    rng = np.random.RandomState(k)
    B, G, eos, special = 24, 300, 2, [40, 41]
    lens = rng.randint(1, G, size=B)
    lens[:3] = [1, 2, 3]
    hist = rng.randint(0, 45, size=(B, G)).astype(np.int32)
    hist[5:10] = rng.randint(3, 7, size=(5, G))                     # repetitive rows: long matches
    finished = np.zeros(B, dtype=np.int32)
    finished[10] = 1
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda_dev)
    drafts = torch.zeros(B, k, dtype=torch.int32, device=cuda_dev)
    win = torch.zeros(B, k + 1, dtype=torch.int32, device=cuda_dev)
    ops.lookup_draft(dev(hist), dev(lens.astype(np.int32)), dev(finished), dev(np.array(special, dtype=np.int32)), eos, ngram,
                     drafts, win)
    drafts, win = drafts.cpu(), win.cpu()
    for b in range(B):
        h = hist[b, :lens[b]].tolist()
        d = [] if finished[b] else LO.draft(h, k, ngram, special=special, eos=eos)
        want = d + [-1] * (k - len(d))
        assert drafts[b].tolist() == want, b
        assert win[b].tolist() == [h[-1]] + [x if x >= 0 else h[-1] for x in want], b


def test_lookup_accept_matches_oracle(cuda_dev):
    from navillm_b200 import ops
    rng = np.random.RandomState(3)
    B, k, V, eos, pad, max_new = 40, 5, 300, 2, 0, 12
    W = k + 1
    special = torch.tensor([7, 8], dtype=torch.int32, device=cuda_dev)
    logits = torch.randn(B * W, V, generator=torch.Generator().manual_seed(3)).to(bf16)
    logits[3, 100] = logits[3, 50] = 9.0                            # a tie goes to the lower id
    logits[4, 7] = 50.0                                             # a special id is never picked
    t = logits.float().clone()
    t[:, [7, 8]] = float("-inf")
    t = t.argmax(1).view(B, W).numpy()
    drafts = np.full((B, k), -1, dtype=np.int32)
    for b in range(B):                                              # accept a random number of drafts, then a wrong one
        m = rng.randint(0, k + 1)
        drafts[b, :m] = t[b, :m]
        if m < k and rng.rand() < 0.5:
            drafts[b, m] = (t[b, m] + 1) % V
    t[6, 1] = eos                                                   # EOS inside an accepted window
    logits[6 * W + 1, eos] = 60.0
    drafts[6, :3] = t[6, :3]
    n_out = rng.randint(1, max_new, size=B).astype(np.int32)
    n_out[7] = max_new - 2                                          # the limit in the middle of a window
    drafts[7, :] = t[7, :k]
    finished = np.zeros(B, dtype=np.int32)
    finished[8] = 1
    for stop in (True, False):
        i32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(cuda_dev)
        out = torch.full((B, max_new), pad, dtype=torch.int32, device=cuda_dev)
        hist = torch.zeros(B, 64, dtype=torch.int32, device=cuda_dev)
        hlen, lens, nacc = i32(n_out + 10), i32(n_out + 300), i32(np.zeros(B))
        fin, nout = i32(finished), i32(n_out)
        ops.lookup_accept(logits.to(cuda_dev), special, i32(drafts), fin, eos, stop, max_new, out, hist, hlen, nout, lens, nacc)
        out, hist, fin, nout, lens, nacc = (x.cpu() for x in (out, hist, fin, nout, lens, nacc))
        for b in range(B):
            if finished[b]:
                assert int(nout[b]) == n_out[b] and int(fin[b]) == 1 and int(nacc[b]) == 0
                continue
            em, acc, f = LO.accept(t[b], drafts[b], int(n_out[b]), max_new, stop, eos)
            assert out[b, n_out[b]:n_out[b] + len(em)].tolist() == em, (b, stop)
            assert hist[b, n_out[b] + 10:n_out[b] + 10 + len(em)].tolist() == em
            assert int(nout[b]) == n_out[b] + len(em) and int(lens[b]) == n_out[b] + 300 + len(em)
            assert int(nacc[b]) == acc and int(fin[b]) == int(f), (b, stop)
        assert 0 < int(nout[6]) - n_out[6] <= 2 or not stop


# ---------------------------------------------------------------------------------------------------------------------
# generate(prompt_lookup_num_tokens=k) end to end
# ---------------------------------------------------------------------------------------------------------------------
def _golden(cuda_dev):
    from tests.test_contrastive_gpu import _golden as g
    return g(cuda_dev)


def _call(text, cand, dev, tok, **kw):
    return dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(dev),
                eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id, **kw)


class DraftSource:
    """Replaces ops.lookup_draft: "wrong" drafts a special id (never accepted), "oracle" the given greedy continuation."""

    def __init__(self, monkeypatch, kind, dev, text=None, greedy=None, special_id=None):
        import navillm_b200.ops as ops_mod
        self.kind, self.special_id = kind, special_id
        if greedy is not None:                                       # on the device: the call is captured in a graph
            S = text["input_ids"].shape[1]
            self.gen = greedy[:, S:].to(torch.int32).contiguous().to(dev)
            self.plens = text["attention_mask"].sum(1).to(torch.int32).to(dev)
        monkeypatch.setattr(ops_mod, "lookup_draft", self)

    def __call__(self, hist, hist_len, finished, special, eos_id, ngram, drafts, win_ids):
        B, k = drafts.shape
        if self.kind == "wrong":
            drafts.fill_(self.special_id)
        else:
            gen = self.gen
            i = (hist_len - self.plens).long()[:, None] + torch.arange(k, device=drafts.device)[None]
            ok = i < gen.shape[1]
            drafts.copy_(torch.where(ok, gen.gather(1, i.clamp(max=gen.shape[1] - 1)), torch.full_like(drafts, -1)))
        last = hist.gather(1, (hist_len.long() - 1)[:, None])
        win_ids[:, :1].copy_(last)
        win_ids[:, 1:].copy_(torch.where(drafts < 0, last, drafts))


@pytest.mark.parametrize("rows,k", [([0], 1), ([0], 4), ([0], 15), (None, 2), (None, 8)], ids=["B1k1", "B1k4", "B1k15", "B3k2", "B3k8"])
def test_draft_invariance_and_greedy_semantics(cuda_dev, monkeypatch, rows, k):
    """The n-gram drafts, drafts that are always wrong and the greedy output itself as drafts give bit-identical ids; the
    accepted counts differ.  The ids are greedy decoding teacher-forced against the CPU oracle (every column the argmax of its
    prefix, or within the bf16 noise floor), and equal plain greedy's up to a near tie."""
    g, cfg, tok, model, _qa = _golden(cuda_dev)
    lm = model.lang_model
    text, cand = _qa(g, cfg, tok, rows)
    n_new = 24
    base = _call(text, cand, cuda_dev, tok, max_new_tokens=n_new, stop_on_eos=False)
    plain = lm.generate(**base).cpu()
    runs = {}
    for kind in ("ngram", "wrong", "oracle"):
        with monkeypatch.context() as mp:
            if kind != "ngram":
                DraftSource(mp, kind, cuda_dev, text, plain if kind == "oracle" else None, special_id=int(lm.special_ids_dev[0]))
            st = {}
            ids = lm.generate(prompt_lookup_num_tokens=k, stats=st, **base).cpu()
            lm._decode_states.clear()                               # the monkeypatched drafts are baked into a graph
        runs[kind] = (ids, st)
    ids = runs["ngram"][0]
    for kind in ("wrong", "oracle"):
        assert torch.equal(runs[kind][0], ids), kind
    assert runs["wrong"][1]["lookup_accepted"] == 0 and runs["wrong"][1]["lookup_steps"] == n_new - 1
    B = ids.shape[0]
    o = runs["oracle"][1]
    assert o["lookup_tokens"] == B * (n_new - 1) and o["lookup_accepted"] > 0
    if torch.equal(ids, plain):                                     # then every oracle draft is right until the limit
        from navillm_b200.generation import LOOKUP_CHECK_EVERY as E
        need = (n_new - 1 + k) // (k + 1)                           # then the loop runs on to its next done-check
        assert o["lookup_steps"] == min(n_new - 1, E * ((need + E) // E) - 1)
        assert o["lookup_accepted"] == B * (n_new - 1 - need)
    S = text["input_ids"].shape[1]
    exact, excused, outside = LO.greedy_follow_path(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], ids,
                                                    cand_vis=cand, eos_token_id=tok.eos_token_id, stop_on_eos=False)
    print(f"\n[lookup rows={rows} k={k}] teacher-forced exact {exact}, excused {excused}, outside {outside}; "
          f"bit-identical to plain greedy: {torch.equal(ids, plain)}; accepted (ngram/wrong/oracle) "
          f"{[runs[x][1]['lookup_accepted'] for x in ('ngram', 'wrong', 'oracle')]}")
    assert outside == 0 and exact >= 2 * excused
    if not torch.equal(ids, plain):                                  # a difference starts at a near tie of the plain run's path
        e2, x2, o2 = LO.greedy_follow_path(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], plain,
                                           cand_vis=cand, eos_token_id=tok.eos_token_id, stop_on_eos=False)
        assert o2 == 0
        first = int((ids[:, S:] != plain[:, S:]).any(0).float().argmax())
        assert x2 + excused > 0, f"ids differ from plain greedy at column {first} without a near tie"


@pytest.mark.parametrize("stop", [True, False])
def test_widths_pads_graphs_and_buckets(cuda_dev, stop):
    """Width and pad layout as plain greedy (EOS inside accepted windows, the limit inside a window), graph = eager, and two cache
    buckets with a reused graph.  EOS is chosen among tokens the rows emit, so every row stops early."""
    g, cfg, tok, model, _qa = _golden(cuda_dev)
    lm = model.lang_model
    text, cand = _qa(g, cfg, tok, [1, 0, 1])
    B, S = text["input_ids"].shape
    free = lm.generate(**_call(text, cand, cuda_dev, tok, max_new_tokens=20, stop_on_eos=False)).cpu()
    for eos in (int(free[0, S + 5]), int(free[1, S + 2]), tok.eos_token_id):
        for n_new in (7, 20, 140):
            kw = _call(text, cand, cuda_dev, tok, max_new_tokens=n_new, stop_on_eos=stop)
            kw["eos_token_id"] = eos
            plain = lm.generate(**kw).cpu()
            got = [lm.generate(prompt_lookup_num_tokens=k, use_cuda_graph=gr, **kw).cpu() for k in (3, 8) for gr in (False, True, True)]
            for x in got[:3]:
                assert torch.equal(x, got[0]), (eos, n_new)
            for x in got[3:]:
                assert torch.equal(x, got[3]), (eos, n_new)
            for x in (got[0], got[3], plain):                       # decode()'s width rule and pads after EOS
                new = x[:, S:]
                is_eos = new == eos
                done = bool(is_eos.any(1).all()) and stop and n_new > 1
                width = int(is_eos.float().argmax(1).max()) + 1 if done else n_new
                assert new.shape[1] == width, (eos, n_new, stop)
                if stop:
                    for b in range(B):
                        if bool(is_eos[b].any()):
                            assert bool((new[b, int(is_eos[b].float().argmax()) + 1:] == tok.unk_token_id).all())
            same = [torch.equal(x, plain) for x in (got[0], got[3])]
            print(f"\n[lookup widths stop={stop} eos={eos} n_new={n_new}] k=3 / k=8 equal to plain greedy: {same}")
            st = next(reversed(lm._decode_states.values()))
            longest = int(text["attention_mask"].sum(1).max())
            assert st.G == (longest + n_new + 8 + 127) // 128 * 128 and tuple(st.logits.shape) == (B * 9, lm.lm_head.weight.shape[0])


def test_cache_formats_and_weight_copies(cuda_dev):
    """fp8 KV, fp8 weights and int4 weights: the lookup path equals itself graphed and eager and, on the golden model, plain
    greedy on the same format (checked teacher-forced where they differ)."""
    g, cfg, tok, model, _qa = _golden(cuda_dev)
    lm = model.lang_model
    text, cand = _qa(g, cfg, tok, [1, 0, 1])
    kw = _call(text, cand, cuda_dev, tok, max_new_tokens=16)
    prev = lm.set_kv_cache_dtype("fp8")
    try:
        got = [lm.generate(prompt_lookup_num_tokens=4, use_cuda_graph=gr, **kw).cpu() for gr in (False, True)]
        plain = lm.generate(**kw).cpu()
        assert isinstance(next(reversed(lm._decode_states.values())).kc[0], tuple)
    finally:
        lm.set_kv_cache_dtype(prev)
    assert torch.equal(got[0], got[1])
    print(f"\n[lookup fp8 KV] equal to plain greedy with fp8 KV: {torch.equal(got[0], plain)}")
    if not torch.equal(got[0], plain):
        _, _, outside = LO.greedy_follow_path(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], got[0], cand_vis=cand,
                                              eos_token_id=tok.eos_token_id, ulps=8)
        assert outside == 0
    for quant, drop in (("quantize_weights_fp8", "drop_fp8_weights"), ("quantize_weights_int4", "drop_int4_weights")):
        getattr(model, quant)()
        try:
            got = [lm.generate(prompt_lookup_num_tokens=4, use_cuda_graph=gr, **kw).cpu() for gr in (False, True)]
            plain = lm.generate(**kw).cpu()
        finally:
            getattr(model, drop)()
        assert torch.equal(got[0], got[1]), quant
        print(f"[lookup {quant}] equal to plain greedy on the same copy: {torch.equal(got[0], plain)}")


def test_other_calls_launch_todays_kernels(cuda_dev, monkeypatch):
    """Without the kwarg, or with 0 / None, every mode makes the same launches and returns the same ids; k > 0 launches the new
    kernels; the 3dqa mode forwards the kwarg."""
    from navillm_b200 import _lib
    import navillm_b200.ops as ops_mod
    g, cfg, tok, model, _qa = _golden(cuda_dev)
    text, cand = _qa(g, cfg, tok)
    kw = _call(text, cand, cuda_dev, tok, max_new_tokens=6, use_cuda_graph=False, stop_on_eos=False)
    calls = []
    real = _lib.check

    def spy(status, what):
        calls.append(what)
        return real(status, what)
    monkeypatch.setattr(ops_mod, "check", spy)
    lm = model.lang_model
    for extra in (dict(), dict(do_sample=True), dict(num_beams=4), dict(penalty_alpha=0.6, top_k=4)):
        calls.clear()
        torch.manual_seed(5)
        a = lm.generate(**kw, **extra).cpu()
        first = list(calls)
        assert not any("lookup" in c or "window" in c for c in first)
        for k in (None, 0):
            calls.clear()
            torch.manual_seed(5)
            b = lm.generate(prompt_lookup_num_tokens=k, max_matching_ngram_size=3, **kw, **extra).cpu()
            assert calls == first and torch.equal(a, b), (extra, k)
    calls.clear()
    lm.generate(prompt_lookup_num_tokens=3, **kw)
    assert {"nv_lookup_draft", "nv_lookup_accept", "nv_decode_attn_rope_window"} <= set(calls)
    assert "nv_decode_attn_rope" not in calls[calls.index("nv_lookup_draft"):]
    qa = dict(g["qa_in"])
    calls.clear()
    with torch.no_grad():
        out = model("3dqa", qa, training=False, prompt_lookup_num_tokens=4, max_new_tokens=8)["generated_sentences"]
        ref = model("3dqa", qa, training=False, max_new_tokens=8)["generated_sentences"]
    assert "nv_lookup_accept" in calls and len(out) == len(ref) == len(qa["question"])
    print(f"\n[3dqa lookup] equal sentences to plain greedy: {out == ref}")
    with pytest.raises(NotImplementedError, match="do_sample"):
        lm.generate(prompt_lookup_num_tokens=2, do_sample=True, **kw)
