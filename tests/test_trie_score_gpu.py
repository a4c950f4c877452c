"""Answer scoring on the device (ModifiedLlamaForCausalLM.score_answers): the tree attention (csrc/attn_fwd.cu
nv_attn_fwd_tree[_fp8]) against fp64 with per-element bounds and bit for bit against nv_attn_fwd_kv on a chain, nv_trie_score
bit for bit against a torch restatement, score_answers against the CPU restatement (tests/trie_score_oracle.py) and against
trie beams, the KV / weight formats, chunking and the model modes."""
import copy
import random

import pytest
import torch

from tests import trie_score_oracle as TS
from tests.test_fp8_kv_gpu import _round_rows
from tests.test_trie_beam_gpu import GOLD_WORDS, SPECIAL, _tiny
from tests.test_trie_table_cpu import make_trie

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
HD = 128
U, BF = 2.0 ** -24, 2.0 ** -8


def _rows(trie, V=32006):
    from navillm_b200.trie import flatten_trie, tree_rows
    return tree_rows(flatten_trie(trie, V))


def _random_tree(rng, n_words, max_len, V=500):
    return make_trie([[rng.randrange(3, V) for _ in range(rng.randint(1, max_len))] for _ in range(n_words)])


# ---------------------------------------------------------------------------------------------------------------------
# nv_attn_fwd_tree
# ---------------------------------------------------------------------------------------------------------------------
class _TreeSetup:
    """B sequences of dk_b cached keys followed by the N tree rows of ``rows``, in slots of Smax rows with finite junk past
    kv_len; q [B * N, H * 128]."""

    def __init__(self, rows, dks, H, dev, seed=0):
        g = torch.Generator(device="cpu").manual_seed(seed)
        self.B, self.N, self.H, self.D = len(dks), rows.n, H, H * HD
        self.dks = list(dks)
        self.Smax = (max(dks) + rows.n + 127) // 128 * 128 + 128
        self.kc = (torch.randn(self.B, self.Smax, self.D, generator=g) * 100.0).to(bf16)       # junk everywhere first
        self.vc = (torch.randn(self.B, self.Smax, self.D, generator=g) * 100.0).to(bf16)
        for b, dk in enumerate(dks):
            self.kc[b, :dk + rows.n] = torch.randn(dk + rows.n, self.D, generator=g).to(bf16)
            self.vc[b, :dk + rows.n] = torch.randn(dk + rows.n, self.D, generator=g).to(bf16)
        self.q = torch.randn(self.B * self.N, self.D, generator=g).to(bf16)
        self.kc, self.vc, self.q = self.kc.to(dev), self.vc.to(dev), self.q.to(dev)
        i32 = lambda x: torch.tensor(x, dtype=torch.int32, device=dev)
        self.cu = i32([b * self.N for b in range(self.B + 1)])
        self.kv_start = i32([b * self.Smax for b in range(self.B)])
        self.kv_len = i32([dk + self.N for dk in dks])
        self.end = torch.from_numpy(rows.end).to(dev)
        self.rows = rows

    def tree(self):
        from navillm_b200 import ops
        return ops.attn_fwd_tree(self.q, self.kc, self.vc, self.cu, [self.N] * self.B, self.kv_start, self.kv_len, self.end,
                                 self.H)

    def visible(self, dk):
        """[N, dk + N] bool: query i sees the cached keys and its ancestors-or-self."""
        N, end = self.N, self.rows.end
        m = torch.zeros(N, dk + N, dtype=torch.bool)
        m[:, :dk] = True
        for j in range(N):
            m[j:int(end[j]), dk + j] = True
        return m


def _check_fp64(st, o):
    """o against the fp64 masked softmax with the forward's bound of tests/test_prefix_attn_kernels_gpu.py:
    b·|o_ref| + (1 + 2^-7)·(b + 2·eps + u·(39 + 71·nb))·sum_j P_ij |v_j|, eps = u·(4 + 3·Z + 64·A)."""
    worst = 0.0
    for b, dk in enumerate(st.dks):
        q = st.q[b * st.N:(b + 1) * st.N].double().cpu().view(st.N, st.H, HD).transpose(0, 1)
        k = st.kc[b, :dk + st.N].double().cpu().view(-1, st.H, HD).transpose(0, 1)
        v = st.vc[b, :dk + st.N].double().cpu().view(-1, st.H, HD).transpose(0, 1)
        s = (q @ k.transpose(1, 2)) * HD ** -0.5
        vis = st.visible(dk)
        s = s.masked_fill(~vis, float("-inf"))
        p = torch.softmax(s, dim=-1)
        ref = p @ v
        A = s.masked_fill(~vis, 0).abs().amax(dim=-1, keepdim=True) * 1.4426950408889634
        Z = (s.amax(dim=-1, keepdim=True) - s.masked_fill(~vis, float("inf"))).abs().masked_fill(~vis, 0).amax(-1, keepdim=True)
        nb = (dk + st.N + 127) // 128
        eps = U * (4 + 3 * Z + 64 * A)
        tol = BF * ref.abs() + (1 + 2 ** -7) * (BF + 2 * eps + U * (39 + 71 * nb)) * (p @ v.abs())
        got = o[b * st.N:(b + 1) * st.N].double().cpu().view(st.N, st.H, HD).transpose(0, 1)
        err = (got - ref).abs()
        assert bool((err <= tol).all()), f"seq {b}: max err/tol {float((err / tol).max()):.3g}"
        worst = max(worst, float((err / tol).max()))
    return worst


@pytest.mark.parametrize("seed", range(4))
def test_tree_attention_matches_fp64(cuda_dev, seed):
    rng = random.Random(seed)
    rows = _rows(_random_tree(rng, rng.choice([5, 40, 120]), rng.choice([3, 6])))
    dks = [rng.choice([1, 63, 64, 127, 128, 200, 300]) for _ in range(rng.choice([1, 3]))]
    st = _TreeSetup(rows, dks, H=2, dev=cuda_dev, seed=seed)
    o = st.tree()
    torch.cuda.synchronize()
    print(f"\n[tree attention seed {seed}] N={rows.n} dk={dks} worst err/tol {_check_fp64(st, o):.3g}")


@pytest.mark.parametrize("n", [1, 5, 130, 300])
def test_chain_is_the_causal_suffix_attention(cuda_dev, n):
    """A trie of one answer is a chain: every row sees every earlier row, so the tree kernel is nv_attn_fwd_kv bit for bit."""
    from navillm_b200 import ops
    rows = _rows(make_trie([[7 + i for i in range(n)]]))
    st = _TreeSetup(rows, [1, 129, 64], H=2, dev=cuda_dev)
    want = ops.attn_fwd_kv(st.q, st.kc, st.vc, st.cu, [st.N] * st.B, st.kv_start, st.kv_len, st.H)
    assert torch.equal(st.tree().view(torch.int16), want.view(torch.int16))


def test_tree_attention_fp8_is_bf16_on_rounded_rows(cuda_dev):
    from navillm_b200 import ops
    rng = random.Random(9)
    rows = _rows(_random_tree(rng, 60, 5))
    st = _TreeSetup(rows, [5, 140, 256], H=2, dev=cuda_dev, seed=3)
    kq, ke = _round_rows(st.kc)
    vq, ve = _round_rows(st.vc)
    want = st.tree()
    got = ops.attn_fwd_tree_fp8(st.q, kq, vq, ke, ve, st.cu, [st.N] * st.B, st.kv_start, st.kv_len, st.end, st.H)
    assert bool(torch.isfinite(got.float()).all())
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))


def test_tree_attention_rejects_bad_trees(cuda_dev):
    from navillm_b200 import ops
    rows = _rows(make_trie([[5, 6], [7]]))
    st = _TreeSetup(rows, [3, 3], H=2, dev=cuda_dev)
    with pytest.raises(ValueError):
        ops.attn_fwd_tree(st.q, st.kc, st.vc, st.cu, [st.N] * st.B, st.kv_start, st.kv_len, st.end[:-1], st.H)
    with pytest.raises(ValueError):
        ops.attn_fwd_tree(st.q, st.kc, st.vc, st.cu, [st.N - 1, st.N + 1], st.kv_start, st.kv_len, st.end, st.H)


# ---------------------------------------------------------------------------------------------------------------------
# nv_trie_score
# ---------------------------------------------------------------------------------------------------------------------
def _restated_score(logits, B, rows, eos):
    """The kernel's arithmetic: beam_topk's bf16 log-probs (fp32 max, fp64 sum), NaN -> -inf, the fp32 left fold."""
    x = logits.float().cpu()
    x[:, SPECIAL] = float("-inf")
    m = x.max(dim=1, keepdim=True).values
    ls = torch.log(torch.exp((x - m).double()).sum(dim=1, keepdim=True)).float()
    lp = ((x - m) - ls).to(bf16).float()
    lp = torch.where(torch.isnan(lp), torch.full_like(lp, float("-inf")), lp)
    R = rows.n + 1
    out = torch.empty((B, len(rows.paths)), dtype=torch.float32)
    for b in range(B):
        for a, path in enumerate(rows.paths):
            s, src = torch.zeros((), dtype=torch.float32), 0
            for r in path:
                s = lp[b * R + src, int(rows.tok[r])] + s
                src = r + 1
            out[b, a] = lp[b * R + src, eos] + s
    return out


def _score_args(rows, dev):
    import numpy as np
    i32 = lambda x: torch.tensor(np.asarray(x, dtype=np.int64), dtype=torch.int32, device=dev)
    off = [0]
    for p in rows.paths:
        off.append(off[-1] + len(p))
    flat = [r for p in rows.paths for r in p] or [0]
    return i32(list(rows.tok) or [0])[:rows.n], i32(off), i32(flat)


@pytest.mark.parametrize("B,n_words,special", [(1, 1, False), (3, 20, False), (8, 64, True)])
def test_trie_score_matches_restatement(cuda_dev, B, n_words, special):
    from navillm_b200 import ops
    rng = random.Random(B * 7 + n_words)
    V = 32006
    words = [[rng.randrange(3, 32000) for _ in range(rng.randint(1, 4))] for _ in range(n_words)]
    if special:
        words += [[SPECIAL[1]], [words[0][0], SPECIAL[3]]]               # answers through a special id: -inf
    trie = make_trie(words)
    rows = _rows(trie, V)
    R = rows.n + 1
    g = torch.Generator().manual_seed(B)
    logits = (torch.randn(B * R, V, generator=g) * 4).to(bf16)
    logits[0, 5] = 40.0                                                  # a dominant logit
    ld = (V + 63) // 64 * 64
    buf = torch.zeros(B * R, ld, dtype=bf16, device=cuda_dev)
    buf[:, :V] = logits.to(cuda_dev)
    special_dev = torch.tensor(SPECIAL, dtype=torch.int32, device=cuda_dev)
    tok, off, prow = _score_args(rows, cuda_dev)
    got = ops.trie_score(buf[:, :V], special_dev, tok, off, prow, 2, B).cpu()
    want = _restated_score(logits, B, rows, 2)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    if special:
        assert bool(torch.isneginf(got[:, rows.answers.index([SPECIAL[1]])]).all())


def test_trie_score_empty_root(cuda_dev):
    from navillm_b200 import ops
    rows = _rows(make_trie([]))
    logits = torch.randn(2, 32006).to(bf16)
    tok, off, prow = _score_args(rows, cuda_dev)
    got = ops.trie_score(logits.to(cuda_dev), torch.tensor(SPECIAL, dtype=torch.int32, device=cuda_dev), tok, off, prow, 2, 2)
    assert torch.equal(got.cpu(), _restated_score(logits, 2, rows, 2))


# ---------------------------------------------------------------------------------------------------------------------
# score_answers
# ---------------------------------------------------------------------------------------------------------------------
def _oracle_scores(g, cfg, text, cand, trie, length_penalty):
    """tests/trie_score_oracle.py on the oracle's modified_lm_forward: each answer prefix teacher-forced after the prompts."""
    from oracle import navillm_oracle as O
    ids, mask = text["input_ids"], text["attention_mask"]
    B, S = ids.shape
    memo = {}

    def logits_fn(b, toks):
        key = tuple(toks)
        if key not in memo:
            x = torch.cat([ids, torch.tensor([toks] * B, dtype=ids.dtype).view(B, len(toks))], 1)
            m = torch.cat([mask, torch.ones(B, len(toks), dtype=mask.dtype)], 1)
            pos = (m.long().cumsum(-1) - 1).masked_fill(m == 0, 1)
            memo[key] = O.modified_lm_forward(g["state_dict"], cfg, x, m, cand_vis=cand, position_ids=pos)["logits"][:, -1]
        return memo[key][b]
    return TS.score(logits_fn, B, S, trie, length_penalty)


def _close(got, want, what):
    fin = torch.isfinite(want)
    assert torch.equal(torch.isfinite(got), fin), what
    err = (got[fin].double() - want[fin].double()).abs()
    tol = 0.05 + 0.02 * want[fin].double().abs()
    assert bool((err <= tol).all()), f"{what}: max err {float(err.max()):.4g}"


@pytest.mark.parametrize("lp,rows", [(1.0, None), (0.0, [0, 1, 0]), (2.0, [1])])
def test_score_answers_match_oracle(cuda_dev, lp, rows):
    g, cfg, tok, model, text, cand, kw = _tiny(cuda_dev, rows)
    lm = model.lang_model
    trie = make_trie(GOLD_WORDS + [[tok.bos_token_id, 70 + i] for i in range(3)], eos=tok.eos_token_id)
    stats = {}
    r = lm.score_answers(text["input_ids"], text["attention_mask"], trie, cand_vis=cand.to(cuda_dev), length_penalty=lp,
                         stats=stats)
    ans, lpo, sco, best = _oracle_scores(g, cfg, text, cand, trie, lp)
    assert r["answers"] == ans
    assert r["logprob"].dtype == torch.float32 and r["score"].dtype == torch.float64
    _close(r["logprob"], lpo, "logprob")
    S = text["input_ids"].shape[1]
    norm = torch.tensor([(S + len(a)) ** lp for a in ans], dtype=torch.float64)
    assert torch.equal(r["score"], r["logprob"].double() / norm)
    for b in range(len(best)):                                            # the device's best is the oracle's, or a near tie
        assert float(sco[b, int(r["best"][b])]) >= float(sco[b].max()) - 0.1, b
    assert stats["chunks"] == 1 and stats["tree_rows"] == r["logprob"].shape[0] * _rows(trie).n
    assert all(stats[k] >= 0 for k in ("prefill_ms", "tree_ms", "score_ms"))


def test_score_answers_and_trie_beams_at_length_penalty_0(cuda_dev):
    """A <= K answers, length_penalty 0: trie beams return the top-n answers by score (near ties allowed), with their scores,
    and greedy under the trie returns an answer scored no higher than the best."""
    g, cfg, tok, model, text, cand, kw = _tiny(cuda_dev)
    lm = model.lang_model
    trie = make_trie(GOLD_WORDS, eos=tok.eos_token_id)
    r = lm.score_answers(text["input_ids"], text["attention_mask"], trie, cand_vis=cand.to(cuda_dev), length_penalty=0.0)
    S, n, A = text["input_ids"].shape[1], 3, len(r["answers"])
    ids = lm.generate(trie=trie, num_beams=8, num_return_sequences=n, length_penalty=0.0, max_new_tokens=6, **kw).cpu()
    greedy = lm.generate(trie=trie, max_new_tokens=6, **kw).cpu()
    eos = tok.eos_token_id
    cut = lambda row: row[:row.index(eos)] if eos in row else row
    for b in range(r["score"].shape[0]):
        top = sorted(r["score"][b].tolist(), reverse=True)
        for i in range(n):
            a = r["answers"].index(cut(ids[b * n + i, S:].tolist()))
            assert float(r["score"][b, a]) >= top[i] - 0.05, (b, i)
        ga = r["answers"].index(cut(greedy[b, S:].tolist()))
        assert float(r["score"][b, int(r["best"][b])]) >= float(r["score"][b, ga])
    assert A <= 8


def test_score_answers_formats_and_chunks(cuda_dev, monkeypatch):
    """fp8 KV cache, fp8 and int4 weights: scores close to bf16's; a call split into one prompt per chunk agrees with one
    chunk."""
    from navillm_b200 import generation
    g, cfg, tok, model, text, cand, kw = _tiny(cuda_dev, [1, 0, 1])
    lm = model.lang_model
    trie = make_trie(GOLD_WORDS, eos=tok.eos_token_id)
    call = lambda **k: lm.score_answers(text["input_ids"], text["attention_mask"], trie, cand_vis=cand.to(cuda_dev), **k)
    base = call()
    stats = {}
    monkeypatch.setattr(generation, "TREE_MAX_ROWS", _rows(trie).n)
    split = call(stats=stats)
    monkeypatch.undo()
    assert stats["chunks"] == 3
    _close(split["logprob"], base["logprob"], "chunks")
    prev = lm.set_kv_cache_dtype("fp8")
    try:
        _close(call()["logprob"], base["logprob"], "fp8 kv")
    finally:
        lm.set_kv_cache_dtype(prev)
    for quant, drop in (("quantize_weights_fp8", "drop_fp8_weights"), ("quantize_weights_int4", "drop_int4_weights")):
        getattr(model, quant)()
        try:
            _close(call()["logprob"], base["logprob"], quant)
        finally:
            getattr(model, drop)()


def test_score_answers_rejects_shared_nodes(cuda_dev):
    g, cfg, tok, model, text, cand, kw = _tiny(cuda_dev)
    trie = make_trie(GOLD_WORDS, eos=tok.eos_token_id)
    trie.root.child[99] = trie.root.child[21]
    with pytest.raises(NotImplementedError):
        model.lang_model.score_answers(text["input_ids"], text["attention_mask"], trie, cand_vis=cand.to(cuda_dev))


def test_modes_rank_answers_and_launches(cuda_dev, monkeypatch):
    """3dqa / embodied_qa with rank_answers=True return the three keys; error cases raise; the modes without rank_answers
    launch none of the new kernels."""
    import navillm_b200.ops as ops_mod
    from navillm_b200 import _lib
    from tests.test_navmodel_gpu import build_model, to_dev
    from tests.test_oracle_golden import load
    g, cfg, tok = load("amp_bf16")
    model, _ = build_model(g, cuda_dev)
    words = [[tok.bos_token_id] + w for w in GOLD_WORDS]
    trie = make_trie(words, eos=tok.eos_token_id)
    answers = tok.batch_decode(words, skip_special_tokens=True, clean_up_tokenization_spaces=False)
    calls = []
    real = _lib.check

    def spy(status, what):
        calls.append(what)
        return real(status, what)
    monkeypatch.setattr(ops_mod, "check", spy)
    new = {"nv_attn_fwd_tree", "nv_attn_fwd_tree_fp8", "nv_trie_score"}
    with torch.no_grad():
        for mode, inp in (("3dqa", "qa_in"), ("embodied_qa", "sum_in")):
            out = model(mode, to_dev(dict(g[inp]), cuda_dev), training=False, trie=trie, rank_answers=True, length_penalty=0.5)
            B = len(out["generated_sentences"])
            assert set(out["generated_sentences"]) <= set(answers) and out["answers"] == answers
            assert tuple(out["answer_scores"].shape) == (B, len(answers))
            best = out["answer_scores"].argmax(dim=1)
            assert out["generated_sentences"] == [answers[int(i)] for i in best]
            assert new & set(calls) == {"nv_attn_fwd_tree", "nv_trie_score"}
            with pytest.raises(ValueError, match="num_beams"):
                model(mode, to_dev(dict(g[inp]), cuda_dev), training=False, trie=trie, rank_answers=True, num_beams=4)
            with pytest.raises(ValueError, match="trie"):
                model(mode, to_dev(dict(g[inp]), cuda_dev), training=False, rank_answers=True)
            calls.clear()
            model(mode, to_dev(dict(g[inp]), cuda_dev), training=False, trie=trie, max_new_tokens=6)
            model(mode, to_dev(dict(g[inp]), cuda_dev), training=False, trie=trie, num_beams=4, max_new_tokens=6)
            assert not new & set(calls), calls
            calls.clear()


def test_score_answers_fullwidth_two_layers(cuda_dev):
    """Two layers at Vicuna-7B widths, vocabulary 32006, 12 answers of 1-3 tokens after BOS, B = 2: against the oracle."""
    from oracle import navillm_oracle as O
    from tests.test_fullwidth_parity_gpu import _full_navmodel, _oracle_cfg
    model, tok = _full_navmodel(cuda_dev, 32000)
    lm = model.lang_model
    sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items() if k.startswith("lang_model.")}
    text = lm.tokenize(["Question : what color is the sofa in the living room ? Answer :", "Question : how many chairs ? Answer :"])
    rng = random.Random(0)
    words = [[tok.bos_token_id] + [rng.randrange(100, 31000) for _ in range(rng.randint(1, 3))] for _ in range(12)]
    trie = make_trie(words, eos=tok.eos_token_id)
    r = lm.score_answers(text["input_ids"], text["attention_mask"], trie, length_penalty=1.0)
    g = {"state_dict": sd}
    ans, lpo, sco, best = _oracle_scores(g, _oracle_cfg(tok, "amp_bf16"), text, None, copy.deepcopy(trie), 1.0)
    assert r["answers"] == ans
    _close(r["logprob"], lpo, "full width")
    print(f"\n[full-width score_answers] max |logprob - oracle| {float((r['logprob'] - lpo).abs().max()):.4g}")
    for b in range(2):
        assert float(sco[b, int(r["best"][b])]) >= float(sco[b].max()) - 0.1
