"""Prompt-lookup decoding on the CPU: the draft rule (tests/lookup_oracle.py) on hand-made histories and against a transcription
of transformers' PromptLookupCandidateGenerator, the accept and width rules over a toy greedy model with any drafts, and
generate()'s validation of the mode's arguments before any device work."""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from tests import lookup_oracle as LO  # noqa: E402


def test_draft_hand_made_histories():
    # last bigram (7, 8) first occurs at 1: drafts follow it
    assert LO.draft([5, 7, 8, 9, 10, 11, 7, 8], 3) == [9, 10, 11]
    # k caps the drafts; the history's end cuts them
    assert LO.draft([5, 7, 8, 9, 7, 8], 8) == [9, 7, 8]
    # the earliest occurrence wins over a later one
    assert LO.draft([1, 2, 3, 1, 2, 4, 1, 2], 2) == [3, 1]
    # no bigram match: fall back to the last token
    assert LO.draft([4, 6, 9, 3, 6], 3) == [9, 3, 6]
    # no match at all, and too short a history
    assert LO.draft([1, 2, 3], 4) == [] and LO.draft([1], 4) == []
    # cut at the first special id or EOS; the match decides even when its drafts come out empty
    assert LO.draft([7, 8, 9, 50, 3, 7, 8], 4, special=[50]) == [9]
    assert LO.draft([7, 8, 2, 9, 3, 8, 9, 7, 8], 4, eos=2) == []
    # max_matching_ngram_size 3: the trigram decides before the bigram
    assert LO.draft([1, 2, 3, 9, 5, 2, 3, 4, 1, 2, 3], 2, ngram=3) == [9, 5]
    assert LO.draft([1, 2, 3, 9, 5, 2, 3, 4, 1, 2, 3], 2, ngram=2) == [9, 5]
    assert LO.draft([6, 2, 3, 9, 5, 2, 3, 4, 1, 2, 3], 2, ngram=3) == [9, 5]
    assert LO.draft([6, 2, 3, 9, 5, 2, 3, 4, 1, 2, 3], 2, ngram=1) == [9, 5]


@pytest.mark.parametrize("ngram", [1, 2, 3])
def test_draft_matches_hf_prompt_lookup(ngram):
    rng = np.random.RandomState(ngram)
    for _ in range(300):
        L = int(rng.randint(1, 40))
        hist = rng.randint(0, int(rng.choice([3, 6, 20])), size=L).tolist()
        k = int(rng.randint(1, 16))
        assert LO.draft(hist, k, ngram, eos=2) == LO.draft_hf_literal(hist, k, ngram, eos=2), (hist, k)


def _toy_greedy(V=7, seed=0, eos=2):
    """A deterministic next-token function with repetitive output (so n-gram drafts are often right)."""
    rng = np.random.RandomState(seed)
    table = rng.randint(0, V, size=(V + 1, V + 1))                  # id V: a draft no row ever emits
    return lambda prefix: int(table[prefix[-2] if len(prefix) > 1 else 0, prefix[-1]])


def _plain_greedy(next_token, prompts, max_new, stop_on_eos, eos, pad):
    """decode()'s output rule: one token per step, pad after EOS, trimmed to the slowest row's EOS when every row has one."""
    n = max(max_new, 1)
    gen = []
    for p in prompts:
        h, g, fin = list(p), [], False
        for _ in range(n):
            t = pad if fin else next_token(h)
            g.append(t)
            h.append(t)
            fin = fin or (stop_on_eos and t == eos)
        gen.append(g)
    ids = torch.tensor(gen, dtype=torch.int64)
    if stop_on_eos and n > 1 and all(eos in g for g in gen):
        ids = ids[:, :max(g.index(eos) for g in gen) + 1]
    return ids


@pytest.mark.parametrize("k", [1, 2, 4, 15])
@pytest.mark.parametrize("stop", [True, False])
def test_lookup_equals_greedy_whatever_the_drafts(k, stop):
    eos, pad = 2, 0
    for seed in range(6):
        nt = _toy_greedy(seed=seed, eos=eos)
        rng = np.random.RandomState(seed)
        prompts = [rng.randint(3, 7, size=int(rng.randint(1, 9))).tolist() for _ in range(3)]
        for max_new in (1, 2, 7, 20):
            want = _plain_greedy(nt, prompts, max_new, stop, eos, pad)
            ngram_ids, _, _ = LO.lookup_generate(nt, prompts, k, max_new, stop, eos, pad)
            wrong_ids, wrong_acc, _ = LO.lookup_generate(nt, prompts, k, max_new, stop, eos, pad,
                                                          drafts_of=lambda b, h: [7] * k)    # 7 is never emitted
            full = _plain_greedy(nt, prompts, max_new + k + 1, False, eos, pad)

            def oracle(b, h):
                i = len(h) - len(prompts[b])
                return full[b, i:i + k].tolist()
            orc_ids, orc_acc, orc_steps = LO.lookup_generate(nt, prompts, k, max_new, stop, eos, pad, drafts_of=oracle)
            for got in (ngram_ids, wrong_ids, orc_ids):
                assert torch.equal(got, want), (seed, max_new, got, want)
            assert wrong_acc == [0, 0, 0]
            if not stop:                                            # every step of a row takes k + 1 tokens until the limit
                assert orc_steps == (max(max_new, 1) - 1 + k) // (k + 1)
                assert all(a == max(max_new, 1) - 1 - orc_steps for a in orc_acc)


def test_accept_rule_cuts():
    # two drafts accepted, one more token
    assert LO.accept([4, 5, 6, 9], [4, 5, 8], 1, 20, True, 2) == ([4, 5, 6], 2, False)
    # EOS inside the accepted window ends the row
    assert LO.accept([4, 2, 6, 9], [4, 2, 6], 1, 20, True, 2) == ([4, 2], 1, True)
    assert LO.accept([4, 2, 6, 9], [4, 2, 6], 1, 20, False, 2) == ([4, 2, 6, 9], 3, False)
    # max_new in the middle of a window
    assert LO.accept([4, 5, 6, 9], [4, 5, 6], 18, 20, True, 2) == ([4, 5], 1, True)
    # a missing draft (-1) stops the acceptance
    assert LO.accept([4, 5, 6, 9], [4, -1, 6], 1, 20, True, 2) == ([4, 5], 1, False)


def test_lookup_k_validation():
    from navillm_b200.modified_lm import _lookup_k
    assert _lookup_k(None, 2) == (0, 0) and _lookup_k(0, 2) == (0, 0) and _lookup_k(0, 0) == (0, 0)
    assert _lookup_k(1, 2) == (1, 2) and _lookup_k(15, 1) == (15, 1) and _lookup_k(4, None) == (4, 2)
    for bad in (16, -1, 2.0, True, "3"):
        with pytest.raises(ValueError, match="prompt_lookup_num_tokens"):
            _lookup_k(bad, 2)
    for bad in (0, -2, 1.5):
        with pytest.raises(ValueError, match="max_matching_ngram_size"):
            _lookup_k(3, bad)


def test_generate_validation_before_any_device_work():
    """Each excluded combination raises a NotImplementedError that names it, before generate() touches the model or a device."""
    from navillm_b200.modified_lm import ModifiedLlamaForCausalLM
    lm = object.__new__(ModifiedLlamaForCausalLM)
    ids, mask = torch.ones(1, 3, dtype=torch.long), torch.ones(1, 3, dtype=torch.long)
    gen = lambda **kw: ModifiedLlamaForCausalLM.generate(lm, ids, mask, prompt_lookup_num_tokens=3, **kw)
    cases = [(dict(do_sample=True), "do_sample"), (dict(num_beams=2), "num_beams"), (dict(penalty_alpha=0.6, top_k=4), "contrastive"),
             (dict(trie=object()), "trie"), (dict(logits_processor=[lambda i, s: s]), "logits_processor"),
             (dict(repetition_penalty=1.2), "repetition_penalty"), (dict(no_repeat_ngram_size=2), "no_repeat_ngram_size"),
             (dict(min_length=5), "min_length"), (dict(min_new_tokens=2), "min_new_tokens"),
             (dict(num_return_sequences=2), "num_return_sequences")]
    for kw, name in cases:
        with pytest.raises(NotImplementedError, match=name):
            gen(**kw)
    with pytest.raises(ValueError, match="prompt_lookup_num_tokens"):
        ModifiedLlamaForCausalLM.generate(lm, ids, mask, prompt_lookup_num_tokens=16)
    with pytest.raises(ValueError, match="max_matching_ngram_size"):
        ModifiedLlamaForCausalLM.generate(lm, ids, mask, prompt_lookup_num_tokens=2, max_matching_ngram_size=0)
