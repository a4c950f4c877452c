"""generate(return_dict_in_generate=True, output_scores=True) on the device: the scores outputs of nv_sample_scores and
nv_beam_topk[_processed|_trie]_scores against torch restatements (tests/gen_scores_oracle.py), and every decoding mode end to end
on the golden tiny model: sequences bit for bit those of the plain call, graph = eager, the number of entries, each mode's
scores against what its pick read, beam_indices and sequences_scores against the hypotheses, the fp8 KV cache and the fp8 / int4
weight copies, and the 3dqa mode."""
import pytest
import torch

from tests import gen_scores_oracle as GO

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
SPECIAL = [32000, 32001, 32002, 32003, 32004]
NEG = float("-inf")


# ---------------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("top_k,top_p,T", [(50, 1.0, 1.0), (0, 1.0, 0.7), (50, 0.8, 1.3), (0, 0.9, 1.0)],
                         ids=["k50", "full", "k50p08", "p09"])
def test_sample_scores_are_the_warped_scores(cuda_dev, top_k, top_p, T):
    from navillm_b200 import ops
    B, V, G = 6, 32006, 4
    g = torch.Generator().manual_seed(top_k + int(10 * top_p))
    logits = (torch.randn(B, V, generator=g) * 2).to(bf16)
    logits[1, 200:260] = logits[1].max()                   # ties at the top
    lg = ops.scores_buffer(1, B, V, cuda_dev)[0]
    lg.copy_(logits)
    special = torch.tensor(SPECIAL, dtype=torch.int32, device=cuda_dev)
    u = torch.rand(B, generator=g).to(cuda_dev)
    runs = []
    for scored in (False, True):
        fin = torch.zeros(B, dtype=torch.int32, device=cuda_dev)
        fin[B - 1] = 1
        nxt = torch.zeros(B, dtype=torch.int32, device=cuda_dev)
        probs = torch.zeros(B, V, device=cuda_dev)
        kw = {}
        if scored:
            sc = ops.scores_buffer(G, B, V, cuda_dev)
            sc.fill_(1.0)
            step = torch.tensor([2], dtype=torch.int32, device=cuda_dev)
            kw = dict(scores=sc, step=step)
        ops.sample(lg, special, fin, 7, 0, True, T, top_k, top_p, u, nxt, probs, **kw)
        runs.append((nxt.cpu(), fin.cpu(), probs.cpu()))
    assert all(torch.equal(a, b) for a, b in zip(*runs))            # the pick is the plain kernel's
    got = sc[2].cpu()
    assert bool((sc[[0, 1, 3]].cpu() == 1.0).all())                 # only plane step[0] is written
    want = GO.warped_scores(logits, SPECIAL, T, top_k)
    probs = runs[1][2]
    if top_p == 1.0:
        assert torch.equal(got, want)
    else:                                                           # top-p keeps a subset of top-k, with the same values
        kept = torch.isfinite(got.float())
        assert bool((kept <= torch.isfinite(want.float())).all())
        assert torch.equal(got.float()[kept], want.float()[kept])
        assert bool((probs > 0).le(kept).all())
    nxt = runs[1][0]
    for b in range(B - 1):
        assert torch.isfinite(got[b, nxt[b]].float())               # the drawn token is inside the kept set


def _beam_case(dev, B, K, V, t):
    g = torch.Generator().manual_seed(B * 10 + K)
    logits = (torch.randn(B * K, V, generator=g) * 3).to(bf16)
    logits[0, 5] = 30.0
    bs = torch.randn(B * K, generator=g).float()
    return logits, bs


@pytest.mark.parametrize("variant", ["plain", "processed", "trie"])
@pytest.mark.parametrize("first_step", [False, True])
def test_beam_topk_scores_are_the_processed_logprobs(cuda_dev, variant, first_step):
    from navillm_b200 import ops
    from navillm_b200.trie import flatten_trie
    from tests.test_trie_table_cpu import make_trie
    B, K, V, G, t = 3, 4, 32006, 8, 0 if first_step else 3
    logits, bs = _beam_case(cuda_dev, B, K, V, t)
    lg = ops.scores_buffer(1, B * K, V, cuda_dev)[0]
    lg.copy_(logits)
    special = torch.tensor(SPECIAL, dtype=torch.int32, device=cuda_dev)
    pstate = torch.zeros(B, 5, dtype=torch.int32, device=cuda_dev)
    pstate[:, 0] = t
    S = 6
    prompt = torch.randint(0, 1000, (B, S), dtype=torch.int32, device=cuda_dev)
    width = torch.tensor([S], dtype=torch.int32, device=cuda_dev)
    hist = torch.randint(0, 1000, (B * K, G), dtype=torch.int32, device=cuda_dev)
    proc = (1.3, 2, 0, 0, 2)
    if variant == "processed":                                      # the last history token occurs earlier: a 2-gram ban
        prompt[:, 2] = prompt[:, S - 1]
        hist[:, :t] = prompt.repeat_interleave(K, 0)[:, :t]
    trie_csr = None
    if variant == "trie":
        table = flatten_trie(make_trie([[11, 12, 13], [11, 14], [20, 21, 22, 23, 24]], eos=2), V)
        tb = torch.from_numpy(table.pack(table.n_nodes, max(table.n_edges, 1))).to(cuda_dev)
        o, e = table.n_nodes + 2, max(table.n_edges, 1)
        trie_csr = (tb[:o], tb[o:o + e], tb[o + e:], table.n_nodes, table.eos)
        hist[:, :t] = torch.tensor([11, 14, 99][:t], dtype=torch.int32)
    outs = []
    for scored in (False, True):
        cand = (torch.zeros(B, 2 * K, device=cuda_dev), torch.zeros(B, 2 * K, dtype=torch.int32, device=cuda_dev),
                torch.zeros(B, 2 * K, dtype=torch.int32, device=cuda_dev))
        kw = {}
        if scored:
            sc = ops.scores_buffer(G, B * K, V, cuda_dev)
            sc.fill_(1.0)
            kw = dict(scores=sc)
        b = bs.to(cuda_dev)
        if variant == "plain":
            ops.beam_topk(lg, special, b, K, *cand, first_step=first_step, prompt_state=pstate if scored else None, **kw)
        elif variant == "processed":
            ops.beam_topk_processed(lg, special, b, K, *cand, prompt, width, hist, pstate, proc, first_step=first_step, **kw)
        else:
            ops.beam_topk_trie(lg, special, b, K, *cand, prompt, width, hist, pstate, None, *trie_csr, first_step=first_step, **kw)
        outs.append([c.cpu() for c in cand])
    assert all(torch.equal(a, b) for a, b in zip(*outs))            # the candidates are the plain kernel's
    got = sc[t].cpu()
    assert bool((sc[[i for i in range(G) if i != t]].cpu() == 1.0).all())
    rows = logits[:B].repeat_interleave(K, 0) if first_step else logits
    # 4.28's next_token_scores_processed restated on the CPU: log_softmax, then the processors on each beam's history, then the
    # trie mask on its generated tokens
    history = torch.cat([prompt.cpu().long().repeat_interleave(K, 0), hist.cpu().long()[:, :t]], 1)
    if variant == "plain":
        want = GO.beam_logprobs(rows, SPECIAL)
    elif variant == "processed":
        want = GO.processed_beam_logprobs(rows, SPECIAL, history, S, dict(repetition_penalty=1.3, no_repeat_ngram_size=2))
    else:
        want = GO.processed_beam_logprobs(rows, SPECIAL, history, S, trie=make_trie([[11, 12, 13], [11, 14], [20, 21, 22, 23, 24]],
                                                                                      eos=2))
    # the kernel's fp64 sum runs in another order: ls may differ by an fp32 ulp, which moves a bf16 rounding rarely; the -inf
    # pattern (special ids, n-gram bans, the trie) is exact
    n, equal, _, _ = GO.compare(got, want, 1)
    diff = (got.float() - want.float()).abs()[torch.isfinite(want.float())]
    assert n - equal <= 64 and float(diff.max()) <= 2 ** -5, (n, equal, float(diff.max()))
    if variant == "trie":
        kids = {0: {11, 20}, 3: {2}}[t]                             # t = 3: 11, 14 is a whole word (EOS), 99 stays at its leaf
        assert set(torch.isfinite(got.float()).any(0).nonzero().view(-1).tolist()) == kids
    if variant == "processed":                                      # the ban the history sets up is there
        banned = (prompt[:, 3] if t == 0 else prompt[:, t]).cpu().long().repeat_interleave(K, 0)
        assert bool((got.float().gather(1, banned[:, None]) == NEG).all())
    # every candidate is its parent row's stored log-prob plus that beam's score, in fp32
    cs, ct, cp = outs[1]
    for b in range(B):
        for r in range(2 * K):
            row = b * K + int(cp[b, r])
            lp = float(got[row, int(ct[b, r])])
            if lp != NEG:
                assert float(torch.tensor(lp) + bs[row]) == float(cs[b, r])


# ---------------------------------------------------------------------------------------------------------------------
# generate() on the golden tiny model
# ---------------------------------------------------------------------------------------------------------------------
def _golden(cuda_dev):
    from tests.test_contrastive_gpu import _golden as g
    return g(cuda_dev)


def _call(text, cand, dev, tok, **kw):
    return dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(dev),
                eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id, **kw)


def _trie(tok):
    from tests.test_trie_beam_gpu import GOLD_WORDS
    from tests.test_trie_table_cpu import make_trie
    return make_trie(GOLD_WORDS, eos=tok.eos_token_id)


MODES = {
    "greedy": dict(),
    "greedy_proc": dict(repetition_penalty=1.3, no_repeat_ngram_size=2),
    "sample": dict(do_sample=True, top_k=20, top_p=0.9),
    "sample_n4": dict(do_sample=True, num_return_sequences=4),
    "trie": "trie",
    "trie_host": "trie_host",
    "beam": dict(num_beams=4, num_return_sequences=2, length_penalty=1.0),
    "beam_proc": dict(num_beams=3, repetition_penalty=1.2, early_stopping=True),
    "trie_beam": "trie_beam",
    "contrastive": dict(penalty_alpha=0.6, top_k=4),
    "lookup": dict(prompt_lookup_num_tokens=4),
}


def _mode_kw(mode, tok):
    m = MODES[mode]
    if m == "trie":
        return dict(trie=_trie(tok))
    if m == "trie_host":
        return dict(trie=_trie(tok), logits_processor=[lambda ids, s: s])
    if m == "trie_beam":
        return dict(trie=_trie(tok), num_beams=4, num_return_sequences=2)
    return dict(m)


def _gen(lm, seed, **kw):
    torch.manual_seed(seed)
    return lm.generate(**kw)


@pytest.mark.parametrize("mode", list(MODES))
def test_generate_scores_every_mode(cuda_dev, mode):
    """sequences = the plain call's ids bit for bit (rd + os, rd alone, os alone); scores bit-equal graphed and eager; one
    entry per generated column (per 4.28 step for beams); and the mode's own check of what its pick read."""
    from navillm_b200.modified_lm import ModifiedLlamaForCausalLM
    g, cfg, tok, model, _qa = _golden(cuda_dev)
    lm = model.lang_model
    text, cand = _qa(g, cfg, tok, [1, 0, 1])
    S = text["input_ids"].shape[1]
    kw = dict(_call(text, cand, cuda_dev, tok, max_new_tokens=12), **_mode_kw(mode, tok))
    beam = "num_beams" in kw
    plain = _gen(lm, 3, **kw).cpu()
    assert torch.equal(_gen(lm, 3, output_scores=True, **kw).cpu(), plain)
    rd = _gen(lm, 3, return_dict_in_generate=True, **kw)
    assert torch.equal(rd.sequences.cpu(), plain) and rd.scores is None
    assert (getattr(rd, "sequences_scores", None) is not None) == beam
    outs = {}
    for graph in (False, True, True):
        o = _gen(lm, 3, return_dict_in_generate=True, output_scores=True, **dict(kw, use_cuda_graph=graph))
        assert torch.equal(o.sequences.cpu(), plain), graph
        outs.setdefault(graph, []).append(o)
    o = outs[True][0]
    for a in outs[False] + outs[True][1:]:
        assert len(a.scores) == len(o.scores)
        assert all(torch.equal(x, y) for x, y in zip(a.scores, o.scores))
    assert outs[True][1].scores[0].data_ptr() != o.scores[0].data_ptr()   # fresh tensors, never the state's buffer
    rows, V = o.scores[0].shape
    assert all(s.dtype == bf16 and s.shape == (rows, V) and s.is_cuda for s in o.scores)
    seq = o.sequences
    new = seq[:, S:]
    assert rows == (seq.shape[0] if not beam else text["input_ids"].shape[0] * kw["num_beams"])
    if not beam:
        assert len(o.scores) == seq.shape[1] - S
        sc = torch.stack(o.scores, 1).float()                       # [rows, n, V]
        tok_sc = sc.gather(2, new[:, :, None]).squeeze(2)
        # a row runs at column c until it emitted EOS before c
        eos_before = torch.cumsum((new == tok.eos_token_id).long(), 1) - (new == tok.eos_token_id).long()
        running = eos_before == 0
        assert bool(torch.isfinite(tok_sc[running]).all())
        assert bool((sc[:, :, lm.special_token_ids] == NEG).all())   # the model's own special ids (the tiny vocabulary's)
        if mode in ("greedy", "greedy_proc", "trie", "trie_host", "lookup"):
            assert torch.equal(sc.argmax(2)[running], new[running])
        if mode == "contrastive":
            top = sc.topk(4, dim=2).indices
            assert bool((top == new[:, :, None]).any(2)[running].all())
        if mode == "lookup":
            assert bool((sc[~running] == NEG).all())                # columns after a row's EOS: the row does not run there
        ts = ModifiedLlamaForCausalLM.compute_transition_scores(seq, o.scores, normalize_logits=True)
        assert ts.shape == new.shape and bool((ts[running] <= 0).all())
    else:
        B, n = text["input_ids"].shape[0], kw.get("num_return_sequences", 1)
        bi = o.beam_indices.cpu()
        assert bi.shape == seq.shape and o.sequences_scores.shape == (B * n,)
        assert torch.equal(o.sequences_scores, rd.sequences_scores)
        assert len(o.scores) <= kw["max_new_tokens"]
        assert len(o.scores) >= int((bi >= 0).sum(1).max())
        ts = ModifiedLlamaForCausalLM.compute_transition_scores(seq, o.scores, o.beam_indices)
        lp = kw.get("length_penalty", 1.0)
        for i in range(B * n):
            L = int((bi[i] >= 0).sum())
            idx = bi[i, :L]
            assert bool(((idx // kw["num_beams"]) == i // n).all())  # rows of the hypothesis' own prompt
            # a hypothesis that ended with EOS at step L - 1 has 4.28 length S + L - 1; a running beam finalised after L steps S + L
            hyp_len = S + L - 1 if int(seq[i, S + L - 1]) == tok.eos_token_id else S + L
            total = float(ts[i].double().sum())
            # fp32 fold order: the device adds L bf16 log-probs left to right in fp32, torch sums them in its own order
            bound = L * 2 ** -23 * float(ts[i].abs().double().sum()) + 1e-6
            assert abs(total / hyp_len ** lp - float(o.sequences_scores[i])) <= bound / hyp_len ** lp + 1e-6, (i, total)
        # the stored rows reproduce each hypothesis: its token at step j is finite in row bi[i, j] of plane j
        for i in range(B * n):
            for j in range(int((bi[i] >= 0).sum())):
                assert torch.isfinite(o.scores[j][int(bi[i, j]), int(seq[i, S + j])].float())


@pytest.mark.parametrize("case", ["eos_early", "max_new", "one_token"])
def test_number_of_entries(cuda_dev, case):
    g, cfg, tok, model, _qa = _golden(cuda_dev)
    lm = model.lang_model
    text, cand = _qa(g, cfg, tok, [1, 0, 1])
    S = text["input_ids"].shape[1]
    n_new = 1 if case == "one_token" else 20
    kw = _call(text, cand, cuda_dev, tok, max_new_tokens=n_new)
    if case == "eos_early":                                         # EOS = a token every row emits early
        first = lm.generate(**dict(kw, max_new_tokens=4, stop_on_eos=False)).cpu()
        kw["eos_token_id"] = int(first[0, S + 1])
    for extra in (dict(), dict(num_beams=2), dict(penalty_alpha=0.6, top_k=4), dict(prompt_lookup_num_tokens=3)):
        o = lm.generate(return_dict_in_generate=True, output_scores=True, **kw, **extra)
        if "num_beams" in extra:
            assert 1 <= len(o.scores) <= n_new
            if case == "one_token":
                assert len(o.scores) == 1
        else:
            assert len(o.scores) == o.sequences.shape[1] - S, extra
            if case == "max_new":
                assert len(o.scores) <= n_new
            if case == "one_token":
                assert len(o.scores) == 1


def test_greedy_device_scores_equal_the_host_path(cuda_dev):
    """The device store (nv_scores_store after the processors) and the host-processor path's eager scores agree bit for bit."""
    g, cfg, tok, model, _qa = _golden(cuda_dev)
    lm = model.lang_model
    text, cand = _qa(g, cfg, tok)
    kw = _call(text, cand, cuda_dev, tok, max_new_tokens=10, return_dict_in_generate=True, output_scores=True)
    dev = lm.generate(**kw)
    host = lm.generate(logits_processor=[lambda ids, s: s], **kw)
    assert torch.equal(dev.sequences, host.sequences)
    assert len(dev.scores) == len(host.scores) and all(torch.equal(a, b) for a, b in zip(dev.scores, host.scores))


def test_quantized_weights_and_fp8_kv(cuda_dev):
    g, cfg, tok, model, _qa = _golden(cuda_dev)
    lm = model.lang_model
    text, cand = _qa(g, cfg, tok, [1, 0, 1])
    kw = _call(text, cand, cuda_dev, tok, max_new_tokens=10)
    modes = (dict(), dict(num_beams=3, num_return_sequences=2), dict(do_sample=True), dict(prompt_lookup_num_tokens=3),
             dict(penalty_alpha=0.6, top_k=4))

    def check(tag):
        for extra in modes:
            plain = _gen(lm, 5, **kw, **extra)
            outs = [_gen(lm, 5, return_dict_in_generate=True, output_scores=True, use_cuda_graph=gr, **kw, **extra)
                    for gr in (False, True)]
            for o in outs:
                assert torch.equal(o.sequences, plain), (tag, extra)
            assert all(torch.equal(a, b) for a, b in zip(outs[0].scores, outs[1].scores)), (tag, extra)
    prev = lm.set_kv_cache_dtype("fp8")
    try:
        check("fp8 kv")
    finally:
        lm.set_kv_cache_dtype(prev)
    for quant, drop in (("quantize_weights_fp8", "drop_fp8_weights"), ("quantize_weights_int4", "drop_int4_weights")):
        getattr(model, quant)()
        try:
            check(quant)
        finally:
            getattr(model, drop)()


def test_default_calls_launch_todays_kernels(cuda_dev, monkeypatch):
    """Without rd + os every mode makes the same launches (none of the scores entries) and returns the same ids."""
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
    for extra in (dict(), dict(do_sample=True), dict(num_beams=4), dict(penalty_alpha=0.6, top_k=4),
                  dict(prompt_lookup_num_tokens=3)):
        calls.clear()
        a = _gen(lm, 5, **kw, **extra).cpu()
        first = list(calls)
        assert not any("scores" in c for c in first)
        for flags in (dict(output_scores=True), dict(return_dict_in_generate=False, output_scores=True)):
            calls.clear()
            b = _gen(lm, 5, **kw, **extra, **flags).cpu()
            assert calls == first and torch.equal(a, b), (extra, flags)
        calls.clear()
        o = _gen(lm, 5, return_dict_in_generate=True, output_scores=True, **kw, **extra)
        assert any("scores" in c for c in calls) and torch.equal(o.sequences.cpu(), a)


def test_3dqa_mode_transition_scores(cuda_dev):
    g, cfg, tok, model, _qa = _golden(cuda_dev)
    qa = dict(g["qa_in"])
    with torch.no_grad():
        ref = model("3dqa", qa, training=False, max_new_tokens=8)
        out = model("3dqa", qa, training=False, max_new_tokens=8, output_scores=True)
        beams = model("3dqa", qa, training=False, max_new_tokens=8, num_beams=3, output_scores=True)
    assert out["generated_sentences"] == ref["generated_sentences"]
    ts = out["transition_scores"]
    assert ts.dtype == torch.float32 and ts.shape[0] == len(qa["question"]) and bool((ts <= 0).all())
    assert "sequences_scores" not in out
    assert beams["sequences_scores"].shape == (len(qa["question"]),) and beams["transition_scores"].dtype == torch.float32
