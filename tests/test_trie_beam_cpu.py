"""tests/trie_beam_oracle.py against a literal transcription of transformers 4.28's ``beam_search`` loop with a
``PrefixConstrainedLogitsProcessor`` (and ``BeamSearchScorer`` / ``BeamHypotheses``), on toy scorers; the stateless walk
against the reference's stateful ``TrieLogitsProcessor``; the caller's trie left as it was."""
import copy
import random

import pytest
import torch
import torch.nn.functional as F

from navillm_b200.trie import TrieLogitsProcessor
from tests import processors_oracle as PO
from tests import trie_beam_oracle as TB
from tests.test_trie_table_cpu import make_trie, structure

EOS, PAD = 2, 0


# ---- 4.28, transcribed (BeamHypotheses, BeamSearchScorer.process / finalize, beam_search, PrefixConstrainedLogitsProcessor) ----
class _Hyps:
    def __init__(self, num_beams, length_penalty, early_stopping):
        self.length_penalty, self.early_stopping, self.num_beams = length_penalty, early_stopping, num_beams
        self.beams, self.worst_score = [], 1e9

    def __len__(self):
        return len(self.beams)

    def add(self, hyp, sum_logprobs):
        score = sum_logprobs / (hyp.shape[-1] ** self.length_penalty)
        if len(self) < self.num_beams or score > self.worst_score:
            self.beams.append((score, hyp))
            if len(self) > self.num_beams:
                sorted_next_scores = sorted([(s, idx) for idx, (s, _) in enumerate(self.beams)])
                del self.beams[sorted_next_scores[0][1]]
                self.worst_score = sorted_next_scores[1][0]
            else:
                self.worst_score = min(score, self.worst_score)

    def is_done(self, best_sum_logprobs, cur_len):
        if len(self) < self.num_beams:
            return False
        elif self.early_stopping:
            return True
        cur_score = best_sum_logprobs / cur_len ** self.length_penalty
        return self.worst_score >= cur_score


def _prefix_constrained(prefix_allowed_tokens_fn, num_beams):
    def proc(input_ids, scores):
        mask = torch.full_like(scores, float("-inf"))
        for batch_id, beam_sent in enumerate(input_ids.view(-1, num_beams, input_ids.shape[-1])):
            for beam_id, sent in enumerate(beam_sent):
                mask[batch_id * num_beams + beam_id, prefix_allowed_tokens_fn(batch_id, sent)] = 0
        return scores + mask
    return proc


def hf_beam_search(scorer, input_ids, num_beams, max_new_tokens, logits_processor, length_penalty=1.0, early_stopping=False,
                   num_return_sequences=1):
    """4.28 ``beam_search`` with a ``max_length`` stopping criterion.  ``torch.topk`` leaves equal scores unordered; a stable
    descending sort stands in for it (the tie rule of the restatement and the kernel).  Also returns, per step after the first,
    whether the beams were reordered (beam_idx != arange)."""
    batch_size, S = input_ids.shape
    max_length = S + max_new_tokens
    input_ids = input_ids.repeat_interleave(num_beams, dim=0)
    beam_hyps = [_Hyps(num_beams, length_penalty, early_stopping) for _ in range(batch_size)]
    done = [False] * batch_size
    beam_scores = torch.zeros((batch_size, num_beams), dtype=torch.float)
    beam_scores[:, 1:] = -1e9
    beam_scores = beam_scores.view((batch_size * num_beams,))
    reordered = []
    cur_len = S
    while True:
        next_token_logits = scorer(input_ids)
        next_token_scores = F.log_softmax(next_token_logits, dim=-1)
        next_token_scores_processed = next_token_scores
        for p in logits_processor:
            next_token_scores_processed = p(input_ids, next_token_scores_processed)
        next_token_scores = next_token_scores_processed + beam_scores[:, None].expand_as(next_token_scores)
        vocab_size = next_token_scores.shape[-1]
        next_token_scores = next_token_scores.view(batch_size, num_beams * vocab_size)
        next_token_scores, next_tokens = torch.sort(next_token_scores, dim=1, descending=True, stable=True)
        next_token_scores, next_tokens = next_token_scores[:, :2 * num_beams], next_tokens[:, :2 * num_beams]
        next_indices = torch.div(next_tokens, vocab_size, rounding_mode="floor")
        next_tokens = next_tokens % vocab_size
        # BeamSearchScorer.process
        next_beam_scores = torch.zeros((batch_size, num_beams), dtype=next_token_scores.dtype)
        next_beam_tokens = torch.zeros((batch_size, num_beams), dtype=next_tokens.dtype)
        next_beam_indices = torch.zeros((batch_size, num_beams), dtype=next_indices.dtype)
        for batch_idx, beam_hyp in enumerate(beam_hyps):
            if done[batch_idx]:
                next_beam_scores[batch_idx, :] = 0
                next_beam_tokens[batch_idx, :] = PAD
                next_beam_indices[batch_idx, :] = 0
                continue
            beam_idx = 0
            for beam_token_rank, (next_token, next_score, next_index) in enumerate(
                    zip(next_tokens[batch_idx], next_token_scores[batch_idx], next_indices[batch_idx])):
                batch_beam_idx = batch_idx * num_beams + next_index
                if next_token.item() == EOS:
                    if beam_token_rank >= num_beams:
                        continue
                    beam_hyp.add(input_ids[batch_beam_idx].clone(), next_score.item())
                else:
                    next_beam_scores[batch_idx, beam_idx] = next_score
                    next_beam_tokens[batch_idx, beam_idx] = next_token
                    next_beam_indices[batch_idx, beam_idx] = batch_beam_idx
                    beam_idx += 1
                if beam_idx == num_beams:
                    break
            done[batch_idx] = done[batch_idx] or beam_hyp.is_done(next_token_scores[batch_idx].max().item(), cur_len)
        beam_scores = next_beam_scores.view(-1)
        beam_next_tokens = next_beam_tokens.view(-1)
        beam_idx = next_beam_indices.view(-1)
        if cur_len > S:
            reordered.append(not torch.equal(beam_idx, torch.arange(batch_size * num_beams)))
        input_ids = torch.cat([input_ids[beam_idx, :], beam_next_tokens.unsqueeze(-1)], dim=-1)
        cur_len = cur_len + 1
        if all(done) or cur_len >= max_length:
            break
    # BeamSearchScorer.finalize
    for batch_idx, beam_hyp in enumerate(beam_hyps):
        if done[batch_idx]:
            continue
        for beam_id in range(num_beams):
            batch_beam_idx = batch_idx * num_beams + beam_id
            beam_hyp.add(input_ids[batch_beam_idx], beam_scores[batch_beam_idx].item())
    sent_lengths, best = [], []
    for beam_hyp in beam_hyps:
        sorted_hyps = sorted(beam_hyp.beams, key=lambda x: x[0])
        for _ in range(num_return_sequences):
            best_hyp = sorted_hyps.pop()[1]
            sent_lengths.append(len(best_hyp))
            best.append(best_hyp)
    sent_max_len = min(max(sent_lengths) + 1, max_length)
    decoded = torch.full((len(best), sent_max_len), PAD, dtype=torch.int64)
    for i, hypo in enumerate(best):
        decoded[i, :sent_lengths[i]] = hypo
        if sent_lengths[i] < sent_max_len:
            decoded[i, sent_lengths[i]] = EOS
    return decoded, reordered


def _trie_fn(trie, S):
    """prefix_allowed_tokens_fn: the reference trie's own get_next_node / get_child_index over the generated tokens, on a copy
    (the reference's defaultdict grows where a token is not a child)."""
    def fn(batch_id, sent):
        t = copy.deepcopy(trie)
        node = t.root
        for tok in sent[S:].tolist():
            node = t.get_next_node(node, tok)
        return t.get_child_index(node)
    return fn


# ---- toy scorers ----
class Toy:
    """Next-token logits from the last token and the length: table[last] + pos[len % 5], values on the bf16 grid (so that
    scores tie), special ids -inf."""

    def __init__(self, V, seed, special=(), scale=3.0):
        g = torch.Generator().manual_seed(seed)
        self.table = (torch.randn(V, V, generator=g) * scale).to(torch.bfloat16).float()
        self.pos = (torch.randn(5, V, generator=g) * 0.5).to(torch.bfloat16).float()
        self.special = list(special)

    def __call__(self, ids):
        x = self.table[ids[:, -1]] + self.pos[ids.shape[1] % 5]
        x[:, self.special] = float("-inf")
        return x

    def oracle_scorer(self, prompt_ids, K):
        state = {"ids": prompt_ids.repeat_interleave(K, 0)}

        def scorer(src, last):
            if src is not None:
                state["ids"] = torch.cat([state["ids"][src], last[:, None]], dim=1)
            return self(state["ids"])
        return scorer


def _procs(proc, S):
    if not proc:
        return []
    return [lambda ids, s: PO.process(s, ids, S, eos_token_id=EOS, **proc)]


def _compare(toy, prompt, trie, K, n_new, n_ret=1, lp=1.0, early=False, proc=None):
    S = prompt.shape[1]
    want, reordered = hf_beam_search(toy, prompt, K, n_new, _procs(proc, S) + [_prefix_constrained(_trie_fn(trie, S), K)],
                                     length_penalty=lp, early_stopping=early, num_return_sequences=n_ret)
    before = structure(trie.root)
    got = TB.search(toy.oracle_scorer(prompt, K), prompt, trie, num_beams=K, max_new_tokens=n_new, eos_token_id=EOS,
                    pad_token_id=PAD, length_penalty=lp, early_stopping=early, num_return_sequences=n_ret, **(proc or {}))
    assert structure(trie.root) == before, "the oracle modified the trie"
    assert torch.equal(got, want), (got[:, S:].tolist(), want[:, S:].tolist())
    return got, reordered


def _random_trie(rng, V, n_words, max_len, eos=EOS, avoid=()):
    words = []
    for _ in range(n_words):
        words.append([rng.choice([c for c in range(3, V) if c not in avoid]) for _ in range(rng.randint(1, max_len))])
    return make_trie(words, eos=eos)


@pytest.mark.parametrize("K", [1, 2, 4])
@pytest.mark.parametrize("seed", range(6))
def test_oracle_matches_the_428_transcription(K, seed):
    rng = random.Random(seed * 10 + K)
    V = 24
    toy = Toy(V, seed, special=[V - 1])
    B, S = 3, 4
    prompt = torch.tensor([[rng.randrange(3, V - 1) for _ in range(S)] for _ in range(B)])
    # wide (>= 2K answers), narrow (fewer than 2K continuations: -inf candidates, off-trie beams), an EOS edge
    tries = [_random_trie(rng, V - 1, 12, 4), _random_trie(rng, V - 1, 1, 3), _random_trie(rng, V - 1, 2, 2),
             make_trie([[5, EOS, 7], [5, 6], [9]], eos=EOS)]
    for trie in tries:
        for n_new in (1, 3, 8):
            for n_ret in sorted({1, K}):
                _compare(toy, prompt, trie, K, n_new, n_ret=n_ret, lp=rng.choice([0.0, 1.0, 2.0]), early=rng.random() < 0.3)


@pytest.mark.parametrize("proc", [dict(repetition_penalty=1.3), dict(no_repeat_ngram_size=2), dict(min_new_tokens=2),
                                  dict(min_length=7, repetition_penalty=0.8)], ids=["rep", "ngram", "min_new", "min_len+rep"])
def test_oracle_matches_the_428_transcription_with_processors(proc):
    rng = random.Random(5)
    V = 20
    toy = Toy(V, 11)
    prompt = torch.tensor([[rng.randrange(3, V) for _ in range(5)] for _ in range(2)])
    # repeated tokens along the answers make the penalty and the n-gram ban bite inside the trie
    trie = make_trie([[4, 4, 5], [4, 5, 4, 5], [6, 7, 6, 7, 6], [8], [4, 9]], eos=EOS)
    for K in (2, 4):
        for n_new in (2, 6):
            _compare(toy, prompt, trie, K, n_new, n_ret=2, proc=proc)


def test_narrow_trie_selects_inf_candidates_and_they_end_in_eos():
    """One answer of one token with K = 4: the other beams are -inf candidates, ordered by flat index; their walk reaches a
    childless node, which allows only EOS."""
    V = 16
    toy = Toy(V, 3)
    prompt = torch.tensor([[5, 6, 7]])
    trie = make_trie([[9]], eos=EOS)
    got, _ = _compare(toy, prompt, trie, 4, 4, n_ret=4)
    assert got[0, 3:5].tolist() == [9, EOS]
    scorer = toy.oracle_scorer(prompt, 4)
    ids, steps = TB.search(scorer, prompt, trie, num_beams=4, max_new_tokens=4, eos_token_id=EOS, pad_token_id=PAD,
                           return_steps=True)
    # first step: token 9 of each beam (beams 1..3 at -1e9), then -inf candidates
    assert torch.isfinite(steps[0][0, :4]).all() and torch.isinf(steps[0][0, 4:]).all()
    # second step: EOS of each beam at the leaf, then -inf candidates, which become the running beams
    assert torch.isfinite(steps[1][0, :4]).all() and torch.isinf(steps[1][0, 4:]).all()
    assert TB.allowed_tokens(trie, [0]) == [EOS] and TB.allowed_tokens(trie, [9]) == [EOS] and TB.allowed_tokens(trie, []) == [9]


def test_stateless_walk_agrees_with_the_reference_processor_while_beams_keep_their_rows():
    """Chains of single children: after the first step each beam keeps its row, and the reference's per-row processor walks
    exactly the nodes the per-beam walk reaches."""
    V = 16
    toy = Toy(V, 7)
    toy.table[:] = 0.0
    toy.table[7, 4], toy.table[7, 9] = 3.0, 1.0                       # the prompt ends in 7: answer 4.. first, 9.. second
    prompt = torch.tensor([[3, 7]])
    trie = make_trie([[4, 5, 6, 8], [9, 10, 11, 12]], eos=EOS)
    S, K, n_new = 2, 2, 4
    ref_trie = copy.deepcopy(trie)
    ref, reordered = hf_beam_search(toy, prompt, K, n_new, [TrieLogitsProcessor(ref_trie)], num_return_sequences=2)
    assert not any(reordered)
    got, _ = _compare(toy, prompt, trie, K, n_new, n_ret=2)
    assert torch.equal(got, ref)
    assert structure(ref_trie.root) == structure(trie.root)


def test_reordered_beams_scramble_the_reference_processor_but_not_the_walk():
    """Both beams of step 2 descend from beam 0 (answer "b"): the reference's row-1 node still belongs to answer "a", the
    defaultdict grows an empty child there, and row 1 may only emit EOS; the per-beam walk keeps both continuations of "b"."""
    V = 16
    a, b, w, y, z, p, q, r = 4, 5, 6, 7, 8, 9, 10, 11
    toy = Toy(V, 1)
    toy.table[:] = 0.0
    toy.table[3, b], toy.table[3, a] = 5.0, 4.0
    toy.table[b, y], toy.table[b, z], toy.table[a, w] = 5.0, 4.9, -3.0
    toy.table[y, p], toy.table[z, q], toy.table[w, r] = 2.0, 2.0, 2.0
    prompt = torch.tensor([[1, 3]])
    trie = make_trie([[b, y, p], [b, z, q], [a, w, r]], eos=EOS)
    K, n_new = 2, 4
    ref_trie = copy.deepcopy(trie)
    ref, reordered = hf_beam_search(toy, prompt, K, n_new, [TrieLogitsProcessor(ref_trie)], num_return_sequences=2)
    assert any(reordered)
    got, _ = _compare(toy, prompt, trie, K, n_new, n_ret=2)
    assert got[:, 2:5].tolist() == [[b, y, p], [b, z, q]]
    assert not torch.equal(got, ref), "the reference processor should have lost beam 1's node"
    assert structure(ref_trie.root) != structure(trie.root), "the reference's defaultdict grows on the scrambled node"


def test_walk_never_inserts_into_the_trie():
    trie = make_trie([[11, 12], [11, 13], [20]], eos=EOS)
    before = structure(trie.root)
    assert sorted(TB.allowed_tokens(trie, [])) == [11, 20]
    assert sorted(TB.allowed_tokens(trie, [11])) == [12, 13]
    assert TB.allowed_tokens(trie, [11, 12]) == [EOS]                 # a leaf
    assert TB.allowed_tokens(trie, [11, 12, 99, 5]) == [EOS]          # a leaf stays a leaf
    assert TB.allowed_tokens(trie, [30]) == [EOS]                     # off the trie: childless
    assert TB.allowed_tokens(trie, [11, 30, 12]) == [EOS]
    assert structure(trie.root) == before


def test_oracle_matches_the_reference_generation_branch():
    """tests/golden/generate_trie_beam_amp_bf16.pt (the reference's 3dqa branch with prefix_allowed_tokens_fn walking the trie,
    tests/golden/make_trie_beam_golden.py): per prompt equal, or a near tie decided the first difference.  The golden's
    columns after a row's EOS are normalised to pad (``golden_ids``)."""
    from pathlib import Path
    from tests.test_beam_cpu import _near_tie_before, _qa
    from tests.test_oracle_golden import load
    g, cfg, tok = load("amp_bf16")
    gen = torch.load(Path(__file__).resolve().parent / "golden" / "generate_trie_beam_amp_bf16.pt", weights_only=False)
    text, cand = _qa(g, cfg, tok)
    S = gen["prompt_len"]
    assert S == text["input_ids"].shape[1]
    exact = 0
    for run in gen["runs"]:
        K, n = run["num_beams"], run["num_return_sequences"]
        trie = make_trie(run["words"], eos=tok.eos_token_id)
        ids, steps = TB.trie_beam_generate(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], trie, cand_vis=cand,
                                           num_beams=K, max_new_tokens=gen["meta"]["max_new_tokens"], eos_token_id=tok.eos_token_id,
                                           pad_token_id=tok.unk_token_id, length_penalty=0.0, num_return_sequences=n,
                                           return_steps=True)
        ref = TB.golden_ids(run["ids"], S, tok.eos_token_id, tok.unk_token_id)
        for b in range(text["input_ids"].shape[0]):
            a, r = ids[b * n:(b + 1) * n], ref[b * n:(b + 1) * n]
            if a.shape == r.shape and torch.equal(a, r):
                exact += 1
                continue
            L = min(a.shape[1], r.shape[1])
            diff = (a[:, :L] != r[:, :L]).any(0).nonzero()
            first = (int(diff[0]) if len(diff) else L) - S
            assert _near_tie_before(steps, b, first), (run["trie"], K, n, b, a[:, S:].tolist(), r[:, S:].tolist())
    assert exact >= len(gen["runs"])
