"""generate()'s per-step scores on the CPU: ``compute_transition_scores`` against a literal transcription of transformers 4.28's on
hand-made tensors, the 4.28 stand-in output classes, the host beam finalisation that carries the beam indices, and the decoding
key that keeps graphs with and without the scores apart."""
import math

import pytest
import torch

from tests import gen_scores_oracle as GO


def _scores(steps, rows, V, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(steps):
        s = torch.randn(rows, V, generator=g) * 3
        s[:, V - 2:] = float("-inf")                             # special ids
        out.append(s.to(torch.bfloat16))
    return tuple(out)


@pytest.mark.parametrize("normalize", [False, True])
def test_transition_scores_without_beams_match_428(normalize):
    from navillm_b200.modified_lm import ModifiedLlamaForCausalLM
    rows, V, S, n = 3, 17, 4, 5
    sc = _scores(n, rows, V, 1)
    g = torch.Generator().manual_seed(2)
    seq = torch.cat([torch.randint(0, V - 2, (rows, S), generator=g), torch.stack([s.float().argmax(1) for s in sc], 1)], 1)
    got = ModifiedLlamaForCausalLM.compute_transition_scores(seq, sc, normalize_logits=normalize)
    want = GO.compute_transition_scores_428(seq, tuple(s.float() for s in sc), normalize_logits=normalize, vocab_size=V)
    assert got.dtype == torch.float32 and got.shape == (rows, n)
    assert torch.equal(got, want)
    if not normalize:                                            # the emitted tokens' own scores
        assert torch.equal(got, torch.stack([s.float().max(1).values for s in sc], 1))
    else:
        assert bool((got <= 0).all())


def test_transition_scores_with_beam_indices_match_428():
    """Two prompts, K = 2 beams, n = 2 hypotheses each of lengths 3, 1, 2 and 3 steps: -1 padding, rows of other beams, the cut
    at the longest hypothesis."""
    from navillm_b200.modified_lm import compute_transition_scores
    K, V, S, steps = 2, 11, 3, 4
    sc = _scores(steps, 2 * K, V, 3)
    bi = torch.tensor([[0, 1, 1, -1, -1, -1, -1], [1, -1, -1, -1, -1, -1, -1], [2, 3, -1, -1, -1, -1, -1], [3, 2, 3, -1, -1, -1, -1]])
    g = torch.Generator().manual_seed(4)
    seq = torch.randint(0, V - 2, (4, S + 4), generator=g)
    got = compute_transition_scores(seq, sc, bi)
    want = GO.compute_transition_scores_428(seq, tuple(s.float() for s in sc), bi, vocab_size=V)
    assert got.shape == (4, 3) and torch.equal(got, want)
    assert float(got[1, 1]) == 0.0 and float(got[1, 2]) == 0.0
    # the gathered value of hypothesis 3, step 1 is row 2's score of its token at column S + 1 (cut = L - 3)
    assert float(got[3, 1]) == float(sc[1][2, seq[3, seq.shape[1] - 3 + 1]])


def test_output_classes_access_like_model_output():
    from navillm_b200.modified_lm import (BeamSearchDecoderOnlyOutput, ContrastiveSearchDecoderOnlyOutput,
                                          GreedySearchDecoderOnlyOutput, SampleDecoderOnlyOutput)
    seq = torch.zeros(2, 5, dtype=torch.long)
    o = GreedySearchDecoderOnlyOutput(sequences=seq, scores=None)
    assert o.sequences is seq and o["sequences"] is seq and o[0] is seq and o.scores is None and o.attentions is None
    assert len(o.to_tuple()) == 1
    sc = (torch.zeros(2, 3),)
    b = BeamSearchDecoderOnlyOutput(sequences=seq, sequences_scores=torch.zeros(2), scores=sc, beam_indices=seq)
    assert b[2] is sc and b["beam_indices"] is seq and b.hidden_states is None
    for cls in (SampleDecoderOnlyOutput, ContrastiveSearchDecoderOnlyOutput):
        x = cls(sequences=seq, scores=sc)
        assert x.scores is sc and x[1] is sc and type(x).__name__.endswith("DecoderOnlyOutput")


def test_beam_finalize_entries_carry_indices_and_keep_the_order():
    """``entries=True`` returns the same hypotheses (and order) as the plain call, with their scores and beam rows."""
    from navillm_b200.generation import beam_finalize
    S, T, K, lp = 4, 3, 2, 1.0
    hyps = [[(-1.5, [5, 6], [0, 1, 1]), (-0.9, [7], [1, 0])], []]
    worst = [-1.5, 1e9]
    running = [None, [(-2.0, [1, 2, 3], [2, 3, 3]), (-2.0, [4, 5, 6], [3, 2, 2])]]
    plain = beam_finalize([[h[:2] for h in p] for p in hyps], worst, [None, [r[:2] for r in running[1]]], S, T, K, 2, lp)
    full = beam_finalize(hyps, worst, running, S, T, K, 2, lp, entries=True)
    assert [[e[1] for e in p] for p in full] == plain
    assert full[0][0] == (-0.9, [7], [1, 0])
    assert full[1][0][0] == -2.0 / (S + T) ** lp and full[1][0][2] == [3, 2, 2]          # of equal scores the later one wins
    assert math.isclose(full[1][1][0], -2.0 / 7)


def test_beam_finalize_entries_when_a_running_beam_evicts_a_kept_hypothesis():
    """A prompt that is not done at the length cap, with K hypotheses kept, whose running beam beats the worst of them: the
    eviction branch (len(beams) > K) with entries that carry beam rows gives the plain call's tokens, ranked the same."""
    from navillm_b200.generation import beam_finalize
    from tests import beam_oracle as BO
    hyps = [[(-1.0, [1], [0, 1]), (-1.2, [2], [0, 1])]]
    running = [[(-3.0, [3, 4], [0, 1]), (-30.0, [5, 6], [1, 0])]]
    S, T, K = 4, 2, 2
    plain = beam_finalize([[h[:2] for h in p] for p in hyps], [-1.2], [[r[:2] for r in running[0]]], S, T, K, 2, 1.0)
    full = beam_finalize(hyps, [-1.2], running, S, T, K, 2, 1.0, entries=True)
    assert plain == [[[3, 4], [1]]]
    assert [[e[1] for e in p] for p in full] == plain
    assert full[0][0] == (-3.0 / (S + T), [3, 4], [0, 1]) and full[0][1] == (-1.0, [1], [0, 1])
    # against the restated 4.28 BeamHypotheses: the same kept hypotheses, in the same order
    h = BO.BeamHypotheses(K, 1.0, False)
    for sc, toks, _ in hyps[0]:
        h.beams.append((sc, toks))
    h.worst_score = -1.2
    for sc, toks, _ in running[0]:
        h.add(S + T, toks, sc)
    ranked = sorted(h.beams, key=lambda x: x[0])
    assert [ranked.pop()[1] for _ in range(2)] == plain[0]


def test_decoding_key_keeps_scores_apart():
    from navillm_b200.generation import Decoding
    a = Decoding(2, 0, True, "greedy", "bf16")
    b = Decoding(2, 0, True, "greedy", "bf16", scores=True)
    assert a.key() != b.key() and a.key()[-1] == b.key()[-1] == "bf16"
    assert not a.scores


def test_generate_signature_names_hf_kwargs():
    import inspect
    from navillm_b200.modified_lm import ModifiedLlamaForCausalLM
    p = inspect.signature(ModifiedLlamaForCausalLM.generate).parameters
    assert p["return_dict_in_generate"].default is False and p["output_scores"].default is False
