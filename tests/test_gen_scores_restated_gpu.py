"""generate()'s per-step scores against 4.28 restated on the CPU oracle, teacher-forced on the device's own tokens
(tests/gen_scores_oracle.py): greedy, processors, trie, prompt lookup, contrastive search and sampling on the golden tiny model;
the number of beam steps against tests/beam_oracle.py; a beam call that ends at max_new_tokens with its hypotheses full;
``nv_scores_store`` at V = 32006; two Vicuna-width layers (V = 32006) for greedy, prompt lookup and beams; and the modes with
return_dict_in_generate alone."""
import pytest
import torch

from tests import gen_scores_oracle as GO

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
NEG = float("-inf")
# the device's logits and the oracle's differ by the bf16 noise of a differently ordered forward; a value may differ by this
# many bf16 ulp of its row's largest magnitude, and the share of bit-equal values is printed
ULPS = 8


def _golden(cuda_dev):
    from tests.test_contrastive_gpu import _golden as g
    return g(cuda_dev)


def _call(text, cand, dev, tok, **kw):
    return dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(dev),
                eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id, **kw)


def _running(new, eos):
    """[rows, n]: the row has not emitted EOS before column c."""
    e = (new == eos).long()
    return (torch.cumsum(e, 1) - e) == 0


MODES = {"greedy": {}, "greedy_proc": dict(repetition_penalty=1.3, no_repeat_ngram_size=2, min_new_tokens=3),
         "trie": "trie", "lookup": dict(prompt_lookup_num_tokens=3), "contrastive": dict(penalty_alpha=0.6, top_k=4),
         "contrastive_proc": dict(penalty_alpha=0.6, top_k=4, repetition_penalty=1.2), "sample_k20": dict(do_sample=True, top_k=20),
         "sample_n3": dict(do_sample=True, num_return_sequences=3)}


@pytest.mark.parametrize("mode", list(MODES))
def test_scores_match_the_teacher_forced_restatement(cuda_dev, mode):
    """scores[t] against the oracle's logits after the device's own prefix, processed as 4.28 processes them: the same -inf
    pattern (a sampled top-k boundary may move only at a near tie of the k-th value) and finite values within ULPS."""
    from tests.test_trie_beam_gpu import GOLD_WORDS
    from tests.test_trie_table_cpu import make_trie
    g, cfg, tok, model, _qa = _golden(cuda_dev)
    lm = model.lang_model
    text, cand = _qa(g, cfg, tok, [1, 0, 1])
    S = text["input_ids"].shape[1]
    kw = MODES[mode]
    trie = None
    if kw == "trie":
        trie = make_trie(GOLD_WORDS, eos=tok.eos_token_id)
        kw = dict(trie=trie)
    torch.manual_seed(11)
    o = lm.generate(**_call(text, cand, cuda_dev, tok, max_new_tokens=10, return_dict_in_generate=True, output_scores=True, **kw))
    seq = o.sequences.cpu()
    n = seq.shape[0] // text["input_ids"].shape[0]
    ids, mask = text["input_ids"].repeat_interleave(n, 0), text["attention_mask"].repeat_interleave(n, 0)
    per = torch.isin(text["input_ids"], torch.tensor(lm.cand_token_id)).sum(1).tolist()     # <cand> vectors per prompt
    cand_rows = torch.cat([c for c in cand.split(per) for _ in range(n)])
    logits = GO.teacher_forced_logits(g["state_dict"], cfg, ids, mask, seq, cand_vis=cand_rows)
    assert len(logits) == len(o.scores) == seq.shape[1] - S
    run = _running(seq[:, S:], tok.eos_token_id)
    proc = {k: v for k, v in kw.items() if k in ("repetition_penalty", "no_repeat_ngram_size", "min_new_tokens")}
    tot = equal = excused = 0
    worst = 0.0
    for t, (lg, got) in enumerate(zip(logits, o.scores)):
        rows = run[:, t]
        got = got.cpu()[rows]
        want = GO.processed_scores(lg, lm.special_token_ids, seq[:, :S + t], S, proc or None, trie, tok.eos_token_id)[rows]
        if mode.startswith("sample"):
            k = kw.get("top_k", 50)
            w = want.float()
            kth = torch.topk(w, k, dim=1).values[:, -1:]
            near = (w - kth).abs() <= ULPS * GO.ulp_bf16(kth)
            kept_w = w >= kth
            kept_g = torch.isfinite(got.float())
            moved = kept_w != kept_g
            assert bool(near[moved].all()), f"step {t}: the top-k set moved away from a near tie"
            excused += int(moved.sum())
            both = kept_w & kept_g
            got = torch.where(both, got.float(), torch.full_like(w, NEG))
            want = torch.where(both, w, torch.full_like(w, NEG))
        nv, ne, out, mx = GO.compare(got, want, ULPS)
        assert out == 0, f"step {t}: {out} values beyond {ULPS} ulp (max {mx:.1f})"
        tot, equal, worst = tot + nv, equal + ne, max(worst, mx)
        if mode == "lookup":                                         # a row that emitted EOS does not run: -inf
            assert bool((o.scores[t].cpu()[~run[:, t]] == NEG).all())
    print(f"\n[{mode}] {tot} finite values, {equal / max(tot, 1):.3f} bit-equal to the oracle, max {worst:.2f} ulp; "
          f"top-k boundary moved at {excused} near ties")


@pytest.mark.parametrize("case", [dict(num_beams=2), dict(num_beams=4, num_return_sequences=2),
                                  dict(num_beams=3, early_stopping=True), dict(num_beams=4, length_penalty=0.0)],
                         ids=["K2", "K4n2", "K3early", "K4lp0"])
def test_beam_step_count_matches_428(cuda_dev, case):
    """len(scores) is the number of steps 4.28's loop runs (tests/beam_oracle.py), whenever the oracle picks the same ids."""
    from tests import beam_oracle as BO
    g, cfg, tok, model, _qa = _golden(cuda_dev)
    lm = model.lang_model
    text, cand = _qa(g, cfg, tok, [1, 0, 1])
    S = text["input_ids"].shape[1]
    first = lm.generate(**_call(text, cand, cuda_dev, tok, max_new_tokens=6, stop_on_eos=False)).cpu()
    counts = []
    for eos in (tok.eos_token_id, int(first[0, S + 1]), int(first[1, S + 2])):   # EOS at tokens the model emits: early stops
        kw = dict(_call(text, cand, cuda_dev, tok, max_new_tokens=12), **case)
        kw["eos_token_id"] = eos
        o = lm.generate(return_dict_in_generate=True, output_scores=True, **kw)
        ref, steps = BO.beam_generate(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], cand_vis=cand,
                                      max_new_tokens=12, eos_token_id=eos, pad_token_id=tok.unk_token_id, return_steps=True,
                                      **{k: v for k, v in case.items()})
        if torch.equal(o.sequences.cpu(), ref):
            assert len(o.scores) == len(steps), (eos, len(o.scores), len(steps))
            counts.append(len(steps))
        else:
            print(f"\n[beams {case} eos={eos}] ids differ from the oracle's at a near tie; step count not compared")
    print(f"\n[beams {case}] 4.28 step counts compared: {counts}")
    assert counts, "no call matched the oracle's ids"


def test_beam_call_ends_at_the_cap_with_full_hypotheses(cuda_dev, monkeypatch):
    """A prompt that is not done at max_new_tokens while it keeps K hypotheses: its running beams go through the eviction of
    4.28's BeamHypotheses.add, and the scores call returns the plain call's ids with consistent indices and scores."""
    from navillm_b200 import generation
    from navillm_b200.modified_lm import ModifiedLlamaForCausalLM
    g, cfg, tok, model, _qa = _golden(cuda_dev)
    lm = model.lang_model
    text, cand = _qa(g, cfg, tok, [1, 0, 1])
    S = text["input_ids"].shape[1]
    K = 2
    real = generation.beam_finalize
    hit = []

    def spy(hyps, worst, running, S_, T, K_, n_return, lp, entries=False):
        hit.extend(b for b in range(len(hyps)) if running[b] is not None and len(hyps[b]) == K_ and
                   any(r[0] / (S_ + T) ** lp > worst[b] for r in running[b]))      # a running beam evicts a kept hypothesis
        return real(hyps, worst, running, S_, T, K_, n_return, lp, entries=entries)
    monkeypatch.setattr(generation, "beam_finalize", spy)
    # (cap, EOS) pairs at length_penalty 10 where the CPU oracle's 4.28 beam search ends at the cap with K hypotheses kept and a
    # running beam that evicts one (found by searching the oracle over EOS ids, penalties and caps)
    reached, lp = 0, 10.0
    for cap, eos in ((3, 39), (4, 39), (6, 52), (6, 39), (8, 52), (12, 52)):
        kw = _call(text, cand, cuda_dev, tok, max_new_tokens=cap, num_beams=K, num_return_sequences=K, length_penalty=lp)
        kw["eos_token_id"] = eos
        hit.clear()
        plain = lm.generate(**kw).cpu()
        if not hit:                                                  # the device parted from the oracle at a near tie
            continue
        hit.clear()
        o = lm.generate(return_dict_in_generate=True, output_scores=True, **kw)
        assert hit and torch.equal(o.sequences.cpu(), plain)
        assert len(o.scores) == cap                                  # a prompt still runs: 4.28 runs to the cap
        ts = ModifiedLlamaForCausalLM.compute_transition_scores(o.sequences, o.scores, o.beam_indices)
        bi = o.beam_indices.cpu()
        for i in range(plain.shape[0]):
            L = int((bi[i] >= 0).sum())
            hyp_len = S + L - 1 if int(plain[i, S + L - 1]) == eos else S + L
            total = float(ts[i].double().sum())
            # fp32 fold order of L terms, and the fp32 rounding of the returned score, relative to the un-normalised sum
            bound = L * 2 ** -23 * float(ts[i].abs().double().sum()) + 2 ** -23 * abs(total)
            assert abs(total - float(o.sequences_scores[i]) * hyp_len ** lp) <= bound, (i, total)
        reached += 1
    print(f"\n[beams at the cap with K hypotheses kept] {reached} calls")
    assert reached, "no call ended at the cap with K hypotheses kept"


@pytest.mark.parametrize("aligned", [True, False])
def test_scores_store_kernel_full_vocabulary(cuda_dev, aligned):
    """nv_scores_store at V = 32006 (16 column chunks): plane step[0] = the rows, special ids -inf in any chunk, other planes
    untouched; a source whose rows are not 16-byte aligned takes the element path."""
    from navillm_b200 import ops
    R, V, G = 5, 32006, 3
    special_ids = [3, 2047, 2048, 16000, 32000, 32005]
    g = torch.Generator().manual_seed(1)
    x = torch.randn(R, V, generator=g).to(bf16)
    src = ops.scores_buffer(1, R, V, cuda_dev)[0] if aligned else torch.empty(R, V, dtype=bf16, device=cuda_dev)
    src.copy_(x)
    if not aligned:
        assert src.stride(0) * 2 % 16 != 0
    sc = ops.scores_buffer(G, R, V, cuda_dev)
    sc.fill_(1.0)
    step = torch.tensor([1], dtype=torch.int32, device=cuda_dev)
    ops.scores_store(src, torch.tensor(special_ids, dtype=torch.int32, device=cuda_dev), sc, step)
    want = x.clone()
    want[:, special_ids] = NEG
    assert torch.equal(sc[1].cpu(), want)
    assert bool((sc[[0, 2]].cpu() == 1.0).all())


# ---------------------------------------------------------------------------------------------------------------------
# two layers at Vicuna-7B widths, V = 32006
# ---------------------------------------------------------------------------------------------------------------------
def test_fullwidth_two_layers_greedy_lookup_beams(cuda_dev):
    from tests.test_fullwidth_parity_gpu import _full_navmodel, _oracle_cfg
    from navillm_b200.modified_lm import ModifiedLlamaForCausalLM
    model, tok = _full_navmodel(cuda_dev, 32000)
    lm = model.lang_model
    assert len(tok) == 32006
    sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items() if k.startswith("lang_model.")}
    text = lm.tokenize(["Question : what color is the sofa in the living room ? Answer :", "Question : how many chairs ? Answer :"])
    S, n_new = text["input_ids"].shape[1], 8
    base = dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"], max_new_tokens=n_new, stop_on_eos=False)
    for extra in (dict(), dict(prompt_lookup_num_tokens=3), dict(num_beams=4, num_return_sequences=2)):
        plain = lm.generate(**base, **extra).cpu()
        outs = [lm.generate(**base, **extra, return_dict_in_generate=True, output_scores=True, use_cuda_graph=gr) for gr in (False, True)]
        for o in outs:
            assert torch.equal(o.sequences.cpu(), plain), extra
            assert o.scores[0].shape[1] == 32006
        assert len(outs[0].scores) == len(outs[1].scores)
        assert all(torch.equal(a, b) for a, b in zip(outs[0].scores, outs[1].scores)), extra
        o = outs[1]
        if "num_beams" in extra:
            ts = ModifiedLlamaForCausalLM.compute_transition_scores(o.sequences, o.scores, o.beam_indices)
            bi = o.beam_indices.cpu()
            for i in range(plain.shape[0]):
                L = int((bi[i] >= 0).sum())
                hyp_len = S + L - 1 if int(plain[i, S + L - 1]) == tok.eos_token_id else S + L
                bound = L * 2 ** -23 * float(ts[i].abs().double().sum()) + 1e-6
                assert abs(float(ts[i].double().sum()) / hyp_len - float(o.sequences_scores[i])) <= bound / hyp_len + 1e-6
            continue
        # greedy and lookup: against the oracle's logits after the device's own tokens, and the argmax
        logits = GO.teacher_forced_logits(sd, _oracle_cfg(tok, "amp_bf16"), text["input_ids"], text["attention_mask"], o.sequences.cpu())
        tot = equal = 0
        worst = 0.0
        for t, (lg, got) in enumerate(zip(logits, o.scores)):
            got = got.cpu()
            assert torch.equal(got.float().argmax(1), o.sequences.cpu()[:, S + t])
            want = GO.processed_scores(lg, lm.special_token_ids, o.sequences.cpu()[:, :S + t], S)
            nv, ne, out, mx = GO.compare(got, want, ULPS)
            assert out == 0, f"{extra} step {t}: {out} values beyond {ULPS} ulp (max {mx:.1f})"
            tot, equal, worst = tot + nv, equal + ne, max(worst, mx)
        print(f"\n[full width {extra}] {tot} values, {equal / tot:.3f} bit-equal to the oracle, max {worst:.2f} ulp")


def test_modes_with_return_dict_alone_are_unchanged(cuda_dev):
    g, cfg, tok, model, _qa = _golden(cuda_dev)
    qa = dict(g["qa_in"])
    with torch.no_grad():
        ref = model("3dqa", qa, training=False, max_new_tokens=8)
        rd = model("3dqa", qa, training=False, max_new_tokens=8, return_dict_in_generate=True)
    assert rd == ref
