"""Diverse (group) beam search on the device (csrc/decode.cu nv_beam_topk_group* / nv_beam_select_group*, and
generate(num_beams=K, num_beam_groups=G, diversity_penalty=d)): the kernels bit for bit against a torch restatement of one whole
group step, generate() against tests/group_beam_oracle.py under the near-tie rule, the fp8 KV cache, per-step scores and
transition scores, the model modes, and the launches of calls without groups."""
import numpy as np
import pytest
import torch

from tests import group_beam_oracle as GO
from tests import processors_oracle as PO
from tests.beam_oracle import BeamHypotheses, process, top_candidates
from tests.gen_scores_oracle import beam_logprobs, compare

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
SPECIAL = [32000, 32001, 32002, 32003, 32004]
KG = [(2, 2), (4, 2), (4, 4), (6, 3), (8, 2), (8, 4), (8, 8)]
EOS, PAD = 2, 0


# ---------------------------------------------------------------------------------------------------------------------
# one group step: nv_beam_topk_group + nv_beam_select_group for g = 0 .. G - 1 against a torch restatement
# ---------------------------------------------------------------------------------------------------------------------
def _step_case(B, K, V, t, Gc, S, seed, first_step):
    g = torch.Generator().manual_seed(seed)
    R = B * K
    logits = (torch.randn(B if first_step else R, V, generator=g) * 2).to(bf16)
    best = 1234
    logits[:, best] = logits.float().max(dim=1).values.to(bf16) + 1.0      # every group's unpenalised best token
    logits[:, 500:508] = logits[:, best:best + 1].float().sub(1.5).to(bf16)  # equal scores just below it
    logits[::2, EOS] = logits[::2, best].float().sub(0.25).to(bf16)        # EOS near the top: hypotheses
    prompt = torch.randint(3, 900, (B, S), generator=g)
    hist = torch.randint(3, 900, (R, Gc), generator=g)
    hist[:, 1] = best                                                     # a repeated token for the penalty and the n-gram ban
    src = torch.randint(0, R * Gc, (R, Gc), generator=g)
    par = torch.randint(0, R, (R, Gc), generator=g)
    if first_step:
        bs = torch.full((B, K), -1e9)
    else:
        bs = -torch.rand(B, K, generator=g) * 6
    return logits, prompt, hist, src, par, bs


def _pairs(hist_row, par_row, t, r):
    """A beam's history for the restatement's process(): (token, row) pairs and a sentinel carrying its own row."""
    return [(int(hist_row[i]), int(par_row[i])) for i in range(t)] + [("row", r)]


@pytest.mark.parametrize("K,G", KG)
@pytest.mark.parametrize("first_step", [True, False], ids=["first", "later"])
@pytest.mark.parametrize("proc", [None, dict(repetition_penalty=1.3, no_repeat_ngram_size=2, min_new_tokens=2)],
                         ids=["plain", "proc"])
def test_group_step_matches_restatement(cuda_dev, K, G, first_step, proc):
    from navillm_b200 import ops
    dev = cuda_dev
    B, V, S, Gc, d = 3, 32006, 7, 16, 0.75
    Kg = K // G
    t = 0 if first_step else 3
    lp_pen, early = 1.0, True
    logits, prompt, hist, src, par, bs = _step_case(B, K, V, t, Gc, S, 100 * K + 10 * G + first_step, first_step)
    if first_step:
        bs[:, ::Kg] = 0.0
    R = B * K
    # prompt 1 starts with K kept hypotheses: with early stopping group 0 ends it, and its later groups pad in the same step
    pre = {1: [(-50.0 - i, [(7, 1 * K)] * 2 + [("row", 1 * K + i)]) for i in range(K)]}
    i32 = lambda x: x.to(torch.int32).to(dev).contiguous()
    st = dict(beam_score=bs.view(-1).float().to(dev).contiguous(), cand_score=torch.zeros((B, 2 * Kg), device=dev),
              cand_tok=torch.zeros((B, 2 * Kg), dtype=torch.int32, device=dev),
              cand_par=torch.zeros((B, 2 * Kg), dtype=torch.int32, device=dev), hist=i32(hist), src=i32(src),
              hyp_score=torch.zeros((B, K + 1), dtype=torch.float64, device=dev),
              hyp_meta=torch.zeros((B, K, 2), dtype=torch.int32, device=dev), hyp_tok=torch.zeros((B, K, Gc), dtype=torch.int32, device=dev),
              pstate=torch.zeros((B, 5), dtype=torch.int32, device=dev), next_ids=torch.full((R,), 77, dtype=torch.int32, device=dev),
              lens=torch.zeros((R,), dtype=torch.int32, device=dev), par_hist=i32(par),
              hyp_par=torch.zeros((B, K, Gc), dtype=torch.int32, device=dev), done_step=torch.zeros((B,), dtype=torch.int32, device=dev))
    st["hyp_score"][:, K] = 1e9
    st["pstate"][:, 0] = t
    st["pstate"][:, 1] = torch.tensor([S - b for b in range(B)], dtype=torch.int32)
    for b, hs in pre.items():
        for i, (s, toks) in enumerate(hs):
            st["hyp_score"][b, i] = s
            st["hyp_meta"][b, i, 0], st["hyp_meta"][b, i, 1] = 2, i
            st["hyp_tok"][b, i, :2] = 7
            st["hyp_par"][b, i, :2] = b * K
            st["hyp_par"][b, i, 2] = b * K + i
        st["hyp_score"][b, K] = min(s for s, _ in hs)
        st["pstate"][b, 2] = st["pstate"][b, 3] = K
    norm = ops.beam_norm(S, Gc, lp_pen).to(dev)
    scores = ops.scores_buffer(Gc, R, V, dev)
    scores.fill_(float("nan"))
    special = torch.tensor(SPECIAL, dtype=torch.int32, device=dev)
    dlogits = logits.to(dev)
    proc_t = None if proc is None else (1.3, 2, 0, 2, EOS)
    pids, pw = i32(prompt), torch.tensor([S], dtype=torch.int32, device=dev)

    # the restatement's state
    hyps = [BeamHypotheses(K, lp_pen, early) for _ in range(B)]
    for b, hs in pre.items():
        hyps[b].beams = [(s, list(toks)) for s, toks in hs]
        hyps[b].worst_score = min(s for s, _ in hs)
    done = [False] * B
    rows_lp = beam_logprobs(logits.repeat_interleave(K, 0) if first_step else logits, SPECIAL)
    pairs = [_pairs(hist[r], par[r], t, r) for r in range(R)]
    current = [0] * R
    want_hist, want_src, want_par = hist.clone(), src.clone(), par.clone()
    want_next, want_lens, want_bs = torch.full((R,), 77), torch.zeros(R, dtype=torch.int64), bs.view(-1).clone()
    want_scores = torch.zeros(R, V, dtype=bf16)
    for g in range(G):
        ops.beam_topk_group(dlogits, special, st["beam_score"], K, G, g, st["cand_score"], st["cand_tok"], st["cand_par"],
                            st["next_ids"], d, first_step=first_step, proc=proc_t, prompt_ids=pids, prompt_width=pw, hist=st["hist"],
                            prompt_state=st["pstate"], scores=scores)
        rows = [b * K + g * Kg + j for b in range(B) for j in range(Kg)]
        lp = rows_lp[rows]
        lp = torch.cat([GO.hamming(lp[b * Kg:(b + 1) * Kg], current, b, K, g, Kg, d) for b in range(B)])
        if proc is not None:
            lp = PO.process(lp, torch.cat([prompt.repeat_interleave(K, 0)[rows], hist[rows, :t].long()], 1), S, eos_token_id=EOS,
                            **proc)
        want_scores[rows] = lp
        sc = (lp.float() + bs.view(-1)[rows][:, None]).view(B, -1)
        cs, ct, cp = top_candidates(sc, Kg)
        torch.cuda.synchronize()
        assert torch.equal(st["cand_score"].cpu(), cs) and torch.equal(st["cand_tok"].cpu().long(), ct) and \
            torch.equal(st["cand_par"].cpu().long(), cp), (K, G, g)
        ops.beam_select_group(st["cand_score"], st["cand_tok"], st["cand_par"], st["beam_score"], st["hist"], st["src"],
                              st["hyp_score"], st["hyp_meta"], st["hyp_tok"], st["pstate"], st["next_ids"], st["lens"], norm, EOS, PAD,
                              early, G, g, trace=(st["par_hist"], st["hyp_par"], st["done_step"]))
        was_done = list(done)
        nsc, ntok, npar = process(hyps, done, S, t, [pairs[r] for r in rows], cs, ct, cp, EOS, PAD)
        for b in range(B):
            for j in range(Kg):
                r, p = b * K + g * Kg + j, b * K + g * Kg + int(npar[b, j])
                want_hist[r, :t], want_hist[r, t] = hist[p, :t], int(ntok[b, j])
                want_src[r, :t], want_src[r, t] = src[p, :t], r
                want_par[r, :t], want_par[r, t] = par[p, :t], p
                want_next[r], want_lens[r], want_bs[r] = int(ntok[b, j]), S - b + t, nsc[b, j]
                current[r] = int(ntok[b, j])
        if g == 0:
            assert done[1] and not was_done[1]
    torch.cuda.synchronize()
    assert torch.equal(st["hist"].cpu()[:, :t + 1], want_hist[:, :t + 1].int())
    assert torch.equal(st["src"].cpu()[:, :t + 1], want_src[:, :t + 1].int())
    assert torch.equal(st["par_hist"].cpu()[:, :t + 1], want_par[:, :t + 1].int())
    assert torch.equal(st["next_ids"].cpu().long(), want_next) and torch.equal(st["lens"].cpu().long(), want_lens)
    assert torch.equal(st["beam_score"].cpu(), want_bs.float())
    assert torch.equal(scores[t].cpu(), want_scores)
    ps = st["pstate"].cpu()
    assert ps[:, 0].tolist() == [t + 1] * B and ps[:, 4].tolist() == [int(x) for x in done]
    assert st["done_step"].cpu().tolist() == [t + 1 if x else 0 for x in done]
    hs, hm, ht, hp = st["hyp_score"].cpu(), st["hyp_meta"].cpu(), st["hyp_tok"].cpu(), st["hyp_par"].cpu()
    for b in range(B):
        n = int(ps[b, 2])
        assert n == len(hyps[b])
        kept = sorted(range(n), key=lambda i: int(hm[b, i, 1]))
        got = [(float(hs[b, i]), ht[b, i, :int(hm[b, i, 0])].tolist(), hp[b, i, :int(hm[b, i, 0]) + 1].tolist()) for i in kept]
        want = [(s, [p[0] for p in toks[:-1]], [p[1] for p in toks[:-1]] + [toks[-1][1]]) for s, toks in hyps[b].beams]
        assert got == want, (b, got, want)


# ---------------------------------------------------------------------------------------------------------------------
# generate() end to end
# ---------------------------------------------------------------------------------------------------------------------
def group_near_tie_ok(ids, ref, steps, S, n_ret, tag=""):
    """test_beam_gpu.near_tie_ok's rule for group steps: per prompt the device rows equal the oracle's, unless a group's decision
    was inside the bf16 noise floor (``GO.group_tie``: two of one group's best 2Kg + 1 scores within 3 bf16 ulp) at a step at
    or before the first differing column, or at the last step.  Returns the matched generated columns per prompt."""
    matched = []
    for b in range(ids.shape[0] // n_ret):
        a, r = ids[b * n_ret:(b + 1) * n_ret], ref[b * n_ret:(b + 1) * n_ret]
        L = min(a.shape[1], r.shape[1])
        if a.shape == r.shape and torch.equal(a, r):
            matched.append(L - S)
            continue
        diff = (a[:, :L] != r[:, :L]).any(0).nonzero()
        first = (int(diff[0]) if len(diff) else L) - S
        matched.append(first)
        ok = any(GO.group_tie(steps, t, b) for t in range(min(first + 1, len(steps)))) or GO.group_tie(steps, len(steps) - 1, b)
        assert ok, (tag, b, first, a[:, S:].tolist(), r[:, S:].tolist())
    return matched


def _golden(cuda_dev, rows=None):
    from tests.test_beam_gpu import _qa
    from tests.test_navmodel_gpu import build_model
    from tests.test_oracle_golden import load
    g, cfg, tok = load("amp_bf16")
    model, _ = build_model(g, cuda_dev)
    text, cand = _qa(g, cfg, tok, rows)
    return g, cfg, tok, model, text, cand


@pytest.mark.parametrize("K,G,n_ret,lp,early", [(2, 2, 1, 1.0, False), (4, 2, 4, 0.0, False), (4, 4, 1, 2.0, True),
                                                (6, 3, 6, 1.0, False), (8, 2, 1, 1.0, True), (8, 4, 8, 0.0, False),
                                                (8, 8, 2, 1.0, False)])
def test_generate_group_beams_match_oracle(cuda_dev, K, G, n_ret, lp, early):
    g, cfg, tok, model, text, cand = _golden(cuda_dev)
    n_new = 12
    kw = dict(num_beams=K, num_beam_groups=G, diversity_penalty=0.5, max_new_tokens=n_new, eos_token_id=tok.eos_token_id,
              pad_token_id=tok.unk_token_id, length_penalty=lp, early_stopping=early, num_return_sequences=n_ret)
    ref, info = GO.group_beam_generate(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], cand_vis=cand,
                                       return_steps=True, **kw)
    S = text["input_ids"].shape[1]
    outs = {}
    for graph in (False, True, True):
        ids = model.lang_model.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev),
                                        use_cuda_graph=graph, **kw).cpu()
        assert ids.shape[0] == ref.shape[0] and torch.equal(ids[:, :S], ref[:, :S])
        group_near_tie_ok(ids, ref, info["steps"], S, n_ret, tag=f"K{K} G{G} graph={graph}")
        if graph in outs:
            assert torch.equal(outs[graph], ids)
        outs[graph] = ids
    assert torch.equal(outs[False], outs[True])


def test_generate_group_beams_with_processors_match_oracle(cuda_dev):
    g, cfg, tok, model, text, cand = _golden(cuda_dev)
    proc = dict(repetition_penalty=1.2, no_repeat_ngram_size=2, min_new_tokens=2)
    kw = dict(num_beams=4, num_beam_groups=2, diversity_penalty=1.0, max_new_tokens=10, eos_token_id=tok.eos_token_id,
              pad_token_id=tok.unk_token_id, num_return_sequences=2)
    ref, info = GO.group_beam_generate(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], cand_vis=cand,
                                       return_steps=True, **kw, **proc)
    S = text["input_ids"].shape[1]
    ids = model.lang_model.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev),
                                    **kw, **proc).cpu()
    group_near_tie_ok(ids, ref, info["steps"], S, 2, tag="proc")


def test_generate_group_beams_c3_shape_vs_oracle(cuda_dev):
    """2 Vicuna-width layers at C3's shape (B = 8, 256 <cand> tokens, vocab 32006), K = 4 in G = 2 groups: against the oracle
    per prompt under the near-tie rule; graph equal to eager."""
    from tests.test_fullwidth_parity_gpu import _full_navmodel, _oracle_cfg
    B, N_CAND, N_NEW, K, G = 8, 256, 16, 4, 2
    model, tok = _full_navmodel(cuda_dev, base_vocab=32000)
    lm = model.lang_model
    sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items() if k.startswith("lang_model.")}
    rng = np.random.RandomState(5)
    prompts = []
    for b in range(B):
        words = " ".join(f"w{i}" for i in rng.randint(0, 5000, size=int(rng.randint(30, 61))))
        prompts.append("Scene " + " ".join(["<cand>"] * N_CAND) + " Question " + words + " Answer")
    text = tok(prompts)
    cand = torch.randn(B * N_CAND, 4096, generator=torch.Generator().manual_seed(9))
    kw = dict(num_beams=K, num_beam_groups=G, diversity_penalty=0.5, max_new_tokens=N_NEW, eos_token_id=tok.eos_token_id,
              pad_token_id=tok.unk_token_id)
    ref, info = GO.group_beam_generate(sd, _oracle_cfg(tok, "amp_bf16"), text["input_ids"], text["attention_mask"], cand_vis=cand,
                                       return_steps=True, **kw)
    S = text["input_ids"].shape[1]
    outs = {}
    for graph in (False, True):
        ids = lm.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev),
                          use_cuda_graph=graph, **kw).cpu()
        matched = group_near_tie_ok(ids, ref, info["steps"], S, 1, tag=f"c3 graph={graph}")
        print(f"\n[c3 group beams, graph={graph}] matched generated columns per prompt {matched} of {N_NEW}")
        assert sum(matched) >= B * N_NEW // 4, matched
        outs[graph] = ids
    assert torch.equal(outs[False], outs[True])
    # per-step scores at full width, where near ties are rarer than on the golden model: more steps are comparable
    out = lm.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev),
                      return_dict_in_generate=True, output_scores=True, **kw)
    assert torch.equal(out.sequences.cpu(), outs[True])
    compared = _compare_scores([s.cpu() for s in out.scores], info, B, K, G, "c3")
    assert compared >= B, compared


def test_generate_group_beams_fp8_kv_is_the_bf16_path_over_rounded_kv(cuda_dev, monkeypatch):
    from tests.test_beam_gpu import _rounded_bf16_beams
    g, cfg, tok, model, text, cand = _golden(cuda_dev, [0, 1])
    lm = model.lang_model
    kw = dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev), num_beams=4,
              num_beam_groups=2, diversity_penalty=0.5, eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id,
              max_new_tokens=16, num_return_sequences=2)
    want = _rounded_bf16_beams(lm, monkeypatch, kw)
    prev = lm.set_kv_cache_dtype("fp8")
    try:
        for graph in (False, True, True):
            assert torch.equal(lm.generate(**dict(kw, use_cuda_graph=graph)).cpu(), want), graph
    finally:
        lm.set_kv_cache_dtype(prev)


def _compare_scores(sc, info, B, K, G, tag) -> int:
    """The device's per-step scores ``sc`` against the oracle's where its path is the device's.  Group g's rows of prompt b at
    step t depend on the decisions of every group at the steps before t and of groups 0 .. g - 1 at step t; they are
    compared (same -inf pattern, finite values within 8 bf16 ulp of the row's largest magnitude, test_gen_scores_gpu's bound)
    while none of those decisions was a near tie (GO.group_tie's rule on each group alone) and the prompt runs (a done
    prompt's rows follow other histories, DESIGN §2).  Group 0 at step 0 depends on the prefill only and is always compared.
    Returns the number of (prompt, step, group) blocks compared."""
    Kg = K // G
    compared, worst = 0, 0.0
    for b in range(B):
        for t in range(min(len(sc), len(info["scores"]))):
            if not info["running"][t][b]:
                break
            for g in range(G):
                rows = slice(b * K + g * Kg, b * K + (g + 1) * Kg)
                _, _, bad, mx = compare(sc[t][rows], info["scores"][t][rows], 8)
                assert bad == 0, (tag, b, t, g, mx)
                compared, worst = compared + 1, max(worst, mx)
                if GO.group_tie([info["steps"][t][g:g + 1]], 0, b):
                    break
            else:
                continue
            break
    print(f"\n[group scores {tag}] {compared} (prompt, step, group) blocks compared, worst {worst:.2f} row ulp")
    return compared


@pytest.mark.parametrize("K,G,lp", [(4, 2, 1.0), (8, 4, 2.0), (6, 3, 0.0)])
def test_group_beam_scores(cuda_dev, K, G, lp):
    """output_scores: the per-step scores against the oracle's processed log-probs (bound of test_gen_scores_gpu), beam_indices
    in global rows, and compute_transition_scores summed over a row's generated columns over the length normaliser equal to
    sequences_scores."""
    g, cfg, tok, model, text, cand = _golden(cuda_dev)
    lm = model.lang_model
    n_new = 10
    kw = dict(num_beams=K, num_beam_groups=G, diversity_penalty=0.5, max_new_tokens=n_new, eos_token_id=tok.eos_token_id,
              pad_token_id=tok.unk_token_id, length_penalty=lp, num_return_sequences=K)
    call = dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev), **kw)
    plain = lm.generate(**call).cpu()
    out = lm.generate(return_dict_in_generate=True, output_scores=True, **call)
    seq = out.sequences.cpu()
    assert torch.equal(seq, plain)
    ref, info = GO.group_beam_generate(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], cand_vis=cand,
                                       return_steps=True, **kw)
    B, S = text["input_ids"].shape
    group_near_tie_ok(seq, ref, info["steps"], S, K, tag="scores")
    sc = [s.cpu() for s in out.scores]
    assert all(s.shape == (B * K, lm.lm_head.weight.shape[0]) and s.dtype == bf16 for s in sc)
    compared = _compare_scores(sc, info, B, K, G, f"K={K} G={G}")
    assert compared >= B, compared
    bi = out.beam_indices.cpu()
    assert bi.shape == seq.shape and int(bi.max()) < B * K
    for i in range(bi.shape[0]):
        b = i // K
        used = bi[i][bi[i] >= 0]
        assert bool(((used >= b * K) & (used < (b + 1) * K)).all()), (i, used.tolist())
    ts = lm.compute_transition_scores(out.sequences, out.scores, out.beam_indices).cpu()
    ss = out.sequences_scores.cpu()
    n_steps = len(sc)
    for i in range(seq.shape[0]):
        gen = seq[i, S:]
        n_used = int((bi[i] >= 0).sum())
        is_eos = (gen[:n_used] == tok.eos_token_id).nonzero()
        length = S + (int(is_eos[0]) if len(is_eos) else n_steps)
        total = float(ts[i, :n_used].double().sum())
        want = total / (length ** lp)
        assert abs(want - float(ss[i])) <= 1e-5 * max(1.0, abs(want)), (i, want, float(ss[i]))


def test_group_beams_in_the_modes(cuda_dev):
    """3dqa and summarization with groups: B * n sentences, transition_scores / sequences_scores with output_scores; the
    summarization mode with num_beam_groups alone runs exactly as before."""
    from tests.test_navmodel_gpu import build_model, to_dev
    from tests.test_oracle_golden import load
    g, cfg, tok = load("amp_bf16")
    model, _ = build_model(g, cuda_dev)
    with torch.no_grad():
        qa = model("3dqa", to_dev(dict(g["qa_in"]), cuda_dev), training=False, num_beams=4, num_beam_groups=2,
                   diversity_penalty=0.5, num_return_sequences=4, max_new_tokens=8, output_scores=True)
        sm = model("summarization", to_dev(dict(g["sum_in"]), cuda_dev), training=False, num_beams=4, num_beam_groups=4,
                   diversity_penalty=1.0, num_return_sequences=3, output_scores=True)
        base = model("summarization", to_dev(dict(g["sum_in"]), cuda_dev), training=False)
        alone = model("summarization", to_dev(dict(g["sum_in"]), cuda_dev), training=False, num_beam_groups=2)
        beams = model("summarization", to_dev(dict(g["sum_in"]), cuda_dev), training=False, num_beams=4)
        beams_alone = model("summarization", to_dev(dict(g["sum_in"]), cuda_dev), training=False, num_beams=4, num_beam_groups=2)
    nq, ns = len(g["qa_in"]["question"]), len(g["sum_in"]["prompts"])
    assert len(qa["generated_sentences"]) == 4 * nq and qa["sequences_scores"].shape == (4 * nq,)
    assert qa["transition_scores"].dtype == torch.float32 and qa["transition_scores"].shape[0] == 4 * nq
    assert len(sm["generated_sentences"]) == 3 * ns and sm["sequences_scores"].shape == (3 * ns,)
    assert sm["transition_scores"].shape[0] == 3 * ns
    assert alone["generated_sentences"] == base["generated_sentences"]
    assert beams_alone["generated_sentences"] == beams["generated_sentences"]


def test_group_of_one_launches_the_plain_beam_kernels(cuda_dev, monkeypatch):
    """diversity_penalty > 0 with num_beam_groups=1 is the plain beam call: the same ids and the same launches."""
    from navillm_b200 import _lib
    import navillm_b200.ops as ops_mod
    g, cfg, tok, model, text, cand = _golden(cuda_dev)
    lm = model.lang_model
    kw = dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev), num_beams=4,
              max_new_tokens=6, eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id, use_cuda_graph=False)
    calls = []
    real = _lib.check

    def spy(status, what):
        calls.append(what)
        return real(status, what)
    monkeypatch.setattr(ops_mod, "check", spy)
    a = lm.generate(**kw).cpu()
    first = list(calls)
    calls.clear()
    b = lm.generate(diversity_penalty=0.7, num_beam_groups=1, **kw).cpu()
    assert torch.equal(a, b) and calls == first and not any("group" in c for c in first)
    calls.clear()
    lm.generate(diversity_penalty=0.7, num_beam_groups=2, **kw)
    assert "nv_beam_topk_group" in calls and "nv_beam_select_group" in calls and "nv_beam_topk" not in calls
