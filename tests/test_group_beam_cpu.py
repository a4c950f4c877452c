"""Diverse (group) beam search on the CPU: tests/group_beam_oracle.py against a literal transcription of transformers 4.28's
``group_beam_search`` loop, ``HammingDiversityLogitsProcessor`` and group ``BeamSearchScorer.process`` / ``finalize`` (the
installed transformers no longer ships this mode), on bf16 toy scorers and on the golden tiny model; a prompt finished by its
first group; the Hamming penalty's effect; and generate()'s validation, which runs before any device work."""
import random
import sys
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from tests import group_beam_oracle as GO  # noqa: E402
from tests import processors_oracle as PO  # noqa: E402
from tests.test_trie_beam_cpu import _Hyps  # noqa: E402  (4.28 BeamHypotheses, transcribed)

EOS, PAD = 2, 0
KG = [(2, 2), (4, 2), (4, 4), (6, 3), (8, 2), (8, 4), (8, 8)]


# ---- 4.28, transcribed: HammingDiversityLogitsProcessor, BeamSearchScorer (group_size) and group_beam_search ----
class _Hamming:
    def __init__(self, diversity_penalty, num_beams, num_beam_groups):
        if not isinstance(diversity_penalty, float) or (not diversity_penalty > 0.0):
            raise ValueError("`diversity_penalty` should be a float strictly larger than 0.")
        self._diversity_penalty = diversity_penalty
        self._num_beams = num_beams
        self._num_sub_beams = num_beams // num_beam_groups

    def __call__(self, input_ids, scores, current_tokens, beam_group_idx):
        batch_size = current_tokens.shape[0] // self._num_beams
        group_start_idx = beam_group_idx * self._num_sub_beams
        group_end_idx = min(group_start_idx + self._num_sub_beams, self._num_beams)
        group_size = group_end_idx - group_start_idx
        vocab_size = scores.shape[-1]
        if group_start_idx == 0:
            return scores
        for batch_idx in range(batch_size):
            previous_group_tokens = current_tokens[batch_idx * self._num_beams: batch_idx * self._num_beams + group_start_idx]
            token_frequency = torch.bincount(previous_group_tokens, minlength=vocab_size).to(scores.device)
            scores[batch_idx * group_size: (batch_idx + 1) * group_size] -= self._diversity_penalty * token_frequency
        return scores


class _Scorer:
    def __init__(self, batch_size, num_beams, length_penalty, do_early_stopping, num_beam_groups):
        self.num_beams, self.num_beam_groups = num_beams, num_beam_groups
        self.group_size = num_beams // num_beam_groups
        self._beam_hyps = [_Hyps(num_beams, length_penalty, do_early_stopping) for _ in range(batch_size)]
        self._done = torch.tensor([False for _ in range(batch_size)], dtype=torch.bool)

    @property
    def is_done(self):
        return self._done.all()

    def process(self, input_ids, next_scores, next_tokens, next_indices, pad_token_id, eos_token_id):
        cur_len = input_ids.shape[-1]
        batch_size = len(self._beam_hyps)
        next_beam_scores = torch.zeros((batch_size, self.group_size), dtype=next_scores.dtype)
        next_beam_tokens = torch.zeros((batch_size, self.group_size), dtype=next_tokens.dtype)
        next_beam_indices = torch.zeros((batch_size, self.group_size), dtype=next_indices.dtype)
        for batch_idx, beam_hyp in enumerate(self._beam_hyps):
            if self._done[batch_idx]:
                next_beam_scores[batch_idx, :] = 0
                next_beam_tokens[batch_idx, :] = pad_token_id
                next_beam_indices[batch_idx, :] = 0
                continue
            beam_idx = 0
            for beam_token_rank, (next_token, next_score, next_index) in enumerate(
                    zip(next_tokens[batch_idx], next_scores[batch_idx], next_indices[batch_idx])):
                batch_beam_idx = batch_idx * self.group_size + next_index
                if next_token.item() == eos_token_id:
                    is_beam_token_worse_than_top_num_beams = beam_token_rank >= self.group_size
                    if is_beam_token_worse_than_top_num_beams:
                        continue
                    beam_hyp.add(input_ids[batch_beam_idx].clone(), next_score.item())
                else:
                    next_beam_scores[batch_idx, beam_idx] = next_score
                    next_beam_tokens[batch_idx, beam_idx] = next_token
                    next_beam_indices[batch_idx, beam_idx] = batch_beam_idx
                    beam_idx += 1
                if beam_idx == self.group_size:
                    break
            self._done[batch_idx] = self._done[batch_idx] or beam_hyp.is_done(next_scores[batch_idx].max().item(), cur_len)
        return next_beam_scores.view(-1), next_beam_tokens.view(-1), next_beam_indices.view(-1)

    def finalize(self, input_ids, final_beam_scores, max_length, pad_token_id, eos_token_id, num_return_sequences):
        for batch_idx, beam_hyp in enumerate(self._beam_hyps):
            if self._done[batch_idx]:
                continue
            for beam_id in range(self.num_beams):
                batch_beam_idx = batch_idx * self.num_beams + beam_id
                beam_hyp.add(input_ids[batch_beam_idx], final_beam_scores[batch_beam_idx].item())
        sent_lengths, best = [], []
        for beam_hyp in self._beam_hyps:
            sorted_hyps = sorted(beam_hyp.beams, key=lambda x: x[0])
            for _ in range(num_return_sequences):
                best_hyp = sorted_hyps.pop()[1]
                sent_lengths.append(len(best_hyp))
                best.append(best_hyp)
        sent_max_len = min(max(sent_lengths) + 1, max_length)
        decoded = torch.full((len(best), sent_max_len), pad_token_id, dtype=torch.int64)
        for i, hypo in enumerate(best):
            decoded[i, :sent_lengths[i]] = hypo
            if sent_lengths[i] < sent_max_len:
                decoded[i, sent_lengths[i]] = eos_token_id
        return decoded


def hf_group_beam_search(scorer, input_ids, num_beams, num_beam_groups, diversity_penalty, max_new_tokens, length_penalty=1.0,
                         early_stopping=False, num_return_sequences=1, proc=None):
    """4.28 ``group_beam_search`` with a ``max_length`` criterion; ``scorer(reordering_indices, current_tokens)`` is the model
    with its cache (None, None at the first step).  A stable descending sort stands in for ``torch.topk``.  Also returns the
    number of steps and, per step, 4.28's ``processed_score``."""
    batch_size, S = input_ids.shape
    max_length = S + max_new_tokens
    input_ids = input_ids.repeat_interleave(num_beams, dim=0)
    beam_scorer = _Scorer(batch_size, num_beams, length_penalty, early_stopping, num_beam_groups)
    logits_processor = [_Hamming(diversity_penalty, num_beams, num_beam_groups)]
    if proc:
        logits_processor.append(lambda ids, s: PO.process(s, ids, S, eos_token_id=EOS, **proc))
    num_sub_beams = num_beams // num_beam_groups
    beam_scores = torch.full((batch_size, num_beams), -1e9, dtype=torch.float)
    beam_scores[:, ::num_sub_beams] = 0
    beam_scores = beam_scores.view((batch_size * num_beams,))
    cur_len = S
    reorder = current = None
    scores, n_steps = [], 0
    while True:
        logits = scorer(reorder, current)
        current_tokens = torch.zeros(batch_size * num_beams, dtype=input_ids.dtype)
        reordering_indices = torch.zeros(batch_size * num_beams, dtype=torch.long)
        processed_score = torch.zeros_like(logits)
        for beam_group_idx in range(num_beam_groups):
            group_start_idx = beam_group_idx * num_sub_beams
            group_end_idx = min(group_start_idx + num_sub_beams, num_beams)
            group_size = group_end_idx - group_start_idx
            batch_group_indices = []
            for batch_idx in range(batch_size):
                batch_group_indices.extend([batch_idx * num_beams + idx for idx in range(group_start_idx, group_end_idx)])
            group_input_ids = input_ids[batch_group_indices]
            next_token_logits = logits[batch_group_indices]
            # log_softmax in the logits' dtype as torch's CUDA kernel computes it (fp32 inside, rounded once; the CPU kernel
            # rounds in between)
            next_token_scores = F.log_softmax(next_token_logits.float(), dim=-1).to(next_token_logits.dtype)
            vocab_size = next_token_scores.shape[-1]
            next_token_scores_processed = logits_processor[0](group_input_ids, next_token_scores, current_tokens=current_tokens,
                                                              beam_group_idx=beam_group_idx)
            for p in logits_processor[1:]:
                next_token_scores_processed = p(group_input_ids, next_token_scores_processed)
            next_token_scores = next_token_scores_processed + beam_scores[batch_group_indices].unsqueeze(-1)
            next_token_scores = next_token_scores.expand_as(next_token_scores_processed)
            processed_score[batch_group_indices] = next_token_scores_processed.to(processed_score.dtype)
            next_token_scores = next_token_scores.view(batch_size, group_size * vocab_size)
            next_token_scores, next_tokens = torch.sort(next_token_scores, dim=1, descending=True, stable=True)
            next_token_scores, next_tokens = next_token_scores[:, :2 * group_size], next_tokens[:, :2 * group_size]
            next_indices = torch.div(next_tokens, vocab_size, rounding_mode="floor")
            next_tokens = next_tokens % vocab_size
            nbs, beam_next_tokens, beam_idx = beam_scorer.process(group_input_ids, next_token_scores, next_tokens, next_indices,
                                                                  pad_token_id=PAD, eos_token_id=EOS)
            beam_scores[batch_group_indices] = nbs
            input_ids[batch_group_indices] = group_input_ids[beam_idx]
            group_input_ids = torch.cat([group_input_ids[beam_idx, :], beam_next_tokens.unsqueeze(-1)], dim=-1)
            current_tokens[batch_group_indices] = group_input_ids[:, -1]
            reordering_indices[batch_group_indices] = (
                num_beams * torch.div(beam_idx, group_size, rounding_mode="floor") + group_start_idx + (beam_idx % group_size))
        scores.append(processed_score)
        n_steps += 1
        input_ids = torch.cat([input_ids, current_tokens.unsqueeze(-1)], dim=-1)
        reorder, current = reordering_indices, current_tokens
        cur_len = cur_len + 1
        if beam_scorer.is_done or cur_len >= max_length:
            break
    out = beam_scorer.finalize(input_ids, beam_scores, max_length, PAD, EOS, num_return_sequences)
    return out, n_steps, scores


# ---- scorers ----
class Toy:
    """bf16 next-token logits from the last token and the length (values on a coarse grid, so that scores tie), special ids
    -inf.  ``scorer(src, last)`` keeps each row's ids and follows ``src``."""

    def __init__(self, V, seed, special=(), scale=3.0, eos_bias=0.0):
        g = torch.Generator().manual_seed(seed)
        self.table = (torch.randn(V, V, generator=g) * scale).to(torch.bfloat16).float()
        self.table[:, EOS] += eos_bias
        self.pos = (torch.randn(5, V, generator=g) * 0.5).to(torch.bfloat16).float()
        self.special = list(special)

    def scorer(self, prompt_ids, K):
        state = {"ids": prompt_ids.repeat_interleave(K, 0)}

        def scorer(src, last):
            if src is not None:
                state["ids"] = torch.cat([state["ids"][src], last[:, None]], dim=1)
            ids = state["ids"]
            x = self.table[ids[:, -1]] + self.pos[ids.shape[1] % 5]
            x[:, self.special] = float("-inf")
            return x.to(torch.bfloat16)
        return scorer


def _compare(make_scorer, prompt, K, G, d, n_new, n_ret=1, lp=1.0, early=False, proc=None):
    S = prompt.shape[1]
    want, n_steps, want_scores = hf_group_beam_search(make_scorer(), prompt, K, G, d, n_new, length_penalty=lp, early_stopping=early,
                                                      num_return_sequences=n_ret, proc=proc)
    got, info = GO.search(make_scorer(), prompt, num_beams=K, num_beam_groups=G, diversity_penalty=d, max_new_tokens=n_new,
                          eos_token_id=EOS, pad_token_id=PAD, length_penalty=lp, early_stopping=early, num_return_sequences=n_ret,
                          return_steps=True, **(proc or {}))
    assert torch.equal(got, want), (K, G, got[:, S:].tolist(), want[:, S:].tolist())
    assert info["n_steps"] == n_steps
    # a done prompt's rows continue their own history here, 4.28's the history of row 0 (DESIGN §2): compare running prompts
    for a, b, run in zip(info["scores"], want_scores, info["running"]):
        rows = torch.tensor(run).repeat_interleave(K)
        assert torch.equal(a[rows], b[rows])
    return got, info


@pytest.mark.parametrize("K,G", KG)
@pytest.mark.parametrize("seed", range(3))
def test_oracle_matches_the_428_transcription(K, G, seed):
    rng = random.Random(seed * 100 + K * 10 + G)
    V = 24
    toy = Toy(V, seed * 7 + K, special=[V - 1], eos_bias=rng.choice([0.0, 2.0]))
    B, S = 3, 4
    prompt = torch.tensor([[rng.randrange(3, V - 1) for _ in range(S)] for _ in range(B)])
    for n_new in (1, 4, 9):
        for n_ret in sorted({1, K}):
            for lp in (0.0, 1.0, 2.0):
                _compare(lambda: toy.scorer(prompt, K), prompt, K, G, rng.choice([0.25, 0.5, 1.5, 3.0]), n_new, n_ret=n_ret, lp=lp,
                         early=rng.random() < 0.5)


@pytest.mark.parametrize("proc", [dict(repetition_penalty=1.3), dict(no_repeat_ngram_size=2), dict(min_new_tokens=2),
                                  dict(min_length=7, repetition_penalty=0.8)], ids=["rep", "ngram", "min_new", "min_len+rep"])
@pytest.mark.parametrize("early", [False, True])
def test_oracle_matches_the_428_transcription_with_processors(proc, early):
    rng = random.Random(5)
    V = 20
    toy = Toy(V, 11, eos_bias=1.0)
    prompt = torch.tensor([[rng.randrange(3, V) for _ in range(5)] for _ in range(2)])
    for K, G in KG:
        for n_new in (2, 6):
            _compare(lambda: toy.scorer(prompt, K), prompt, K, G, 0.7, n_new, n_ret=2 if K >= 2 else 1, lp=1.0, early=early, proc=proc)


@pytest.mark.parametrize("K,G", [(4, 2), (8, 4)])
def test_oracle_matches_the_428_transcription_on_the_golden_model(K, G):
    from tests.test_beam_cpu import _qa
    from tests.test_oracle_golden import load
    g, cfg, tok = load("amp_bf16")
    text, cand = _qa(g, cfg, tok)
    sd, ids, mask = g["state_dict"], text["input_ids"], text["attention_mask"]
    for lp, early in ((1.0, False), (0.0, True)):
        make = lambda: GO.model_scorer(sd, cfg, ids, mask, K, cand_vis=cand)
        _compare(make, ids, K, G, 0.5, 6, n_ret=2, lp=lp, early=early)


def test_prompt_done_at_group_0_pads_its_later_groups_in_the_same_step():
    """EOS dominates every row, K = G = 2 (one beam per group), early stopping: group 0 adds an EOS hypothesis at each step,
    and the step at which the set of K = 2 fills ends the prompt inside group 0, so group 1 pads in that same step.  The oracle
    equals 4.28's loop on this path, which ends within two steps."""
    V, K, G = 12, 2, 2
    toy = Toy(V, 3, eos_bias=0.0)
    toy.table[:, :] = -4.0
    toy.table[:, EOS] = 4.0                                # EOS first, then a spread of other tokens
    toy.table[:, 5] = 3.0
    toy.table[:, 6] = 2.5
    prompt = torch.tensor([[5, 6, 7], [7, 6, 5]])
    got, info = _compare(lambda: toy.scorer(prompt, K), prompt, K, G, 0.5, 6, n_ret=2, lp=0.0, early=True)
    assert info["n_steps"] <= 2


def test_done_at_group_0_pads_later_groups_of_the_step():
    """A hand-driven step: prompt 0 is done by group 0 (its hypotheses fill up), so group 1 of the same step pads."""
    from tests.beam_oracle import BeamHypotheses, process
    hyps = [BeamHypotheses(2, 1.0, True)]
    hyps[0].add(4, [9], -0.5)
    done = [False]
    # group 0 (Kg = 1): EOS at rank 0 completes the set of K = 2 -> done with early stopping
    cs, ct, cp = torch.tensor([[-0.1, -0.2]]), torch.tensor([[EOS, 5]]), torch.tensor([[0, 0]])
    nsc, ntok, npar = process(hyps, done, 4, 1, [[7]], cs, ct, cp, EOS, PAD)
    assert done == [True] and int(ntok[0, 0]) == 5
    # group 1 of the same step: the prompt pads with score 0, whatever its candidates
    cs, ct, cp = torch.tensor([[-0.05, -0.3]]), torch.tensor([[6, EOS]]), torch.tensor([[0, 0]])
    nsc, ntok, npar = process(hyps, done, 4, 1, [[8]], cs, ct, cp, EOS, PAD)
    assert int(ntok[0, 0]) == PAD and float(nsc[0, 0]) == 0.0 and len(hyps[0]) == 2


@pytest.mark.parametrize("K,G", [(4, 2), (4, 4), (8, 8)])
def test_large_penalty_keeps_groups_apart_within_a_step(K, G):
    """With a penalty far above the spread of the log-probs, no token a group chose at a step is chosen by a later group of the
    same prompt at that step (while the prompt runs and the vocabulary has room)."""
    V = 40
    toy = Toy(V, 9, scale=1.0)
    prompt = torch.tensor([[3, 4, 5, 6], [9, 8, 7, 6]])
    B, Kg = prompt.shape[0], K // G
    seen = []
    inner = toy.scorer(prompt, K)

    def scorer(src, last):
        if last is not None:
            seen.append(last.clone())
        return inner(src, last)
    GO.search(scorer, prompt, num_beams=K, num_beam_groups=G, diversity_penalty=1000.0, max_new_tokens=6, eos_token_id=EOS,
              pad_token_id=PAD, length_penalty=1.0)
    assert seen
    for cur in seen:
        for b in range(B):
            toks = cur[b * K:(b + 1) * K].view(G, Kg)
            if bool((toks == PAD).all()):
                continue
            for g in range(1, G):
                assert not set(toks[g].tolist()) & set(toks[:g].flatten().tolist()), (b, cur.tolist())


def _gen_kw(**kw):
    from navillm_b200.modified_lm import ModifiedLlamaForCausalLM
    lm = ModifiedLlamaForCausalLM.__new__(ModifiedLlamaForCausalLM)   # no weights, no device: validation only
    ids, mask = torch.ones((1, 3), dtype=torch.int64), torch.ones((1, 3), dtype=torch.int64)
    return lambda: ModifiedLlamaForCausalLM.generate(lm, ids, mask, **kw)


@pytest.mark.parametrize("kw,exc,match", [
    (dict(num_beams=2, num_beam_groups=4, diversity_penalty=0.5), ValueError, "smaller or equal"),
    (dict(num_beams=1, num_beam_groups=2, diversity_penalty=0.5), ValueError, "smaller or equal"),
    (dict(num_beams=6, num_beam_groups=4, diversity_penalty=0.5), ValueError, "divisible"),
    (dict(num_beams=4, num_beam_groups=2, diversity_penalty=1), ValueError, "float"),
    (dict(num_beams=4, num_beam_groups=2, diversity_penalty=-0.5), ValueError, "float"),
    (dict(num_beams=4, num_beam_groups=2, diversity_penalty=float("nan")), ValueError, "float"),
    (dict(num_beams=4, num_beam_groups=2), NotImplementedError, "group"),
    (dict(num_beams=4, num_beam_groups=2, diversity_penalty=0.0), NotImplementedError, "group"),
    (dict(num_beams=4, num_beam_groups=2, diversity_penalty=0.5, do_sample=True), NotImplementedError, "group"),
    (dict(num_beams=4, num_beam_groups=2, diversity_penalty=0.5, trie=object()), NotImplementedError, "trie="),
    (dict(num_beams=4, num_beam_groups=2, diversity_penalty=0.5, logits_processor=[lambda i, s: s]), NotImplementedError,
     "logits_processor="),
    (dict(num_beams=4, num_beam_groups=2, diversity_penalty=0.5, num_return_sequences=5), NotImplementedError,
     "num_return_sequences"),
], ids=["groups>beams", "one-beam", "not-divisible", "int-penalty", "negative", "nan", "no-penalty", "zero-penalty", "sample",
        "trie", "logits_processor", "n_return>K"])
def test_generate_validation_before_any_device_work(kw, exc, match):
    with pytest.raises(exc, match=match):
        _gen_kw(**kw)()


def test_decoding_key_holds_the_groups_before_the_kv_format():
    from navillm_b200.generation import Decoding
    a = Decoding(2, 0, None, "beam", "bf16", n=4, groups=2, diversity_penalty=0.5)
    b = Decoding(2, 0, None, "beam", "bf16", n=4)
    c = Decoding(2, 0, None, "beam", "bf16", n=4, groups=2, diversity_penalty=1.0)
    assert len({a.key(), b.key(), c.key()}) == 3 and a.key()[-1] == "bf16"


def test_group_entry_points_are_exported():
    from navillm_b200 import _lib
    lib = _lib.load()
    for name in ("nv_beam_topk_group", "nv_beam_topk_group_scores", "nv_beam_topk_group_processed",
                 "nv_beam_topk_group_processed_scores", "nv_beam_select_group", "nv_beam_select_group_scores"):
        assert hasattr(lib, name), name


def test_group_tie_looks_within_each_group_only():
    """The near-tie rule of the device tests: a tie counts inside one group's sorted scores, never across groups."""
    g0 = torch.tensor([[-1.0, -2.0, -3.0]])
    g1 = torch.tensor([[-1.5, -2.5, -3.5]])
    assert not GO.group_tie([[g0, g1]], 0, 0)
    assert not GO.group_tie([[g0, torch.tensor([[-1.0, -2.0, -3.0]])]], 0, 0)          # equal values in different groups
    assert GO.group_tie([[g0, torch.tensor([[-1.5, -1.5078125, -3.5]])]], 0, 0)        # one bf16 ulp apart inside group 1
    assert not GO.group_tie([[g0, torch.tensor([[-1.5, float("-inf"), float("-inf")]])]], 0, 0)


def test_num_beam_groups_of_one_in_any_number_type_means_no_groups():
    """Calls that passed num_beam_groups=1 as another number type ran plain beams before and still do; an integral numpy G > 1
    is accepted, a float G > 1 is 4.28's ValueError."""
    import numpy as np
    from navillm_b200.modified_lm import _beam_groups
    for g in (None, 0, 1, 1.0, np.int64(1), np.float32(1.0)):
        assert _beam_groups(4, g, None, False, False) == 1
        assert _beam_groups(4, g, 0.5, True, True) == 1
    assert _beam_groups(4, np.int64(2), 0.5, False, False) == 2
    with pytest.raises(ValueError, match="integer"):
        _beam_groups(4, 2.0, 0.5, False, False)
