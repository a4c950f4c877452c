"""Beam search semantics on the CPU: the restated transformers 4.28 beam search (tests/beam_oracle.py) against token ids of the
reference's 3dqa generation branch (tests/golden/make_beam_golden.py), the scorer on hand-built score tables, the host
finalisation of generate() against the restatement, and the C ABI of the device pieces."""
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from tests import beam_oracle as BO  # noqa: E402
from tests.test_oracle_golden import GOLD, load  # noqa: E402
from oracle import navillm_oracle as O  # noqa: E402

EOS, PAD = 2, 0


def _qa(g, cfg, tok):
    sd = g["state_dict"]
    qa = g["qa_in"]
    feats = qa["features"]
    lens = torch.tensor([f.shape[0] for f in feats])
    view = torch.stack([torch.cat([f, f.new_zeros(int(lens.max()) - f.shape[0], f.shape[1])], 0) for f in feats], 0)
    pano = O.forward_panorama(sd, cfg, view, lens)
    pe = pano["pano_embeds"] + O._pos_embed(torch.zeros(pano["pano_embeds"].shape[:2] + (14,)), sd, "vp_pos_embeddings")
    pe = pe + sd["token_type_embeddings.weight"][0]
    return tok(qa["prompts"]), pe[pano["pano_masks"]]


def _near_tie_before(steps, b, first):
    """A step at or before generated column ``first`` whose best 2K + 1 scores of prompt b hold two within 2 bf16 ulp."""
    for t in range(min(first + 1, len(steps))):
        sc = steps[t][b]
        fin = sc[torch.isfinite(sc)]
        if bool(((fin[:-1] - fin[1:]).abs() <= 2 * 2.0 ** -8 * fin[:-1].abs()).any()):
            return True
    return False


@pytest.mark.parametrize("precision", ["fp32", "amp_bf16"])
def test_beam_oracle_matches_reference_generation_branch(precision):
    g, cfg, tok = load(precision)
    gen = torch.load(GOLD / f"generate_beam_{precision}.pt", weights_only=False)
    text, cand = _qa(g, cfg, tok)
    S = gen["prompt_len"]
    assert S == text["input_ids"].shape[1]
    for run in gen["runs"]:
        K, n = run["num_beams"], run["num_return_sequences"]
        ids, steps = BO.beam_generate(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], cand_vis=cand, num_beams=K,
                                      max_new_tokens=gen["meta"]["max_new_tokens"], eos_token_id=tok.eos_token_id,
                                      pad_token_id=tok.unk_token_id, length_penalty=0.0, num_return_sequences=n, return_steps=True)
        ref = run["ids"]
        if precision == "fp32":
            assert torch.equal(ids, ref), (K, n, ids[:, S:].tolist(), ref[:, S:].tolist())
            continue
        for b in range(text["input_ids"].shape[0]):          # per prompt: equal, or a near-tie decided the first difference
            a, r = ids[b * n:(b + 1) * n], ref[b * n:(b + 1) * n]
            if a.shape == r.shape and torch.equal(a, r):
                continue
            L = min(a.shape[1], r.shape[1])
            diff = (a[:, :L] != r[:, :L]).any(0).nonzero()
            first = (int(diff[0]) if len(diff) else L) - S
            assert _near_tie_before(steps, b, first), (K, n, b, a[:, S:].tolist(), r[:, S:].tolist())


def test_reference_expansion_misassigns_the_visual_tokens():
    """The reference's HF expansion (repeat_interleave of the row-major cand_vis) hands prompt 0's visual vectors to prompt 1's
    beams and so on; the recorded unpatched run differs from the per-prompt expansion this project implements."""
    g, cfg, tok = load("fp32")
    gen = torch.load(GOLD / "generate_beam_fp32.pt", weights_only=False)
    text, cand = _qa(g, cfg, tok)
    K = gen["unpatched"]["num_beams"]
    counts = (text["input_ids"] == cfg.cand_id).sum(1).tolist()
    per_prompt = torch.cat([blk for blk in cand.split(counts, 0) for _ in range(K)], 0)
    hf = cand.repeat_interleave(K, dim=0)
    assert per_prompt.shape == hf.shape and not torch.equal(per_prompt, hf)
    assert torch.equal(per_prompt[:counts[0]], cand[:counts[0]]) and not torch.equal(hf[:counts[0]], cand[:counts[0]])
    patched = next(r for r in gen["runs"] if r["num_beams"] == K and r["num_return_sequences"] == 1)
    assert not torch.equal(gen["unpatched"]["ids"], patched["ids"])


# ---------------------------------------------------------------------------------------------------------------------
# the scorer on hand-built tables
# ---------------------------------------------------------------------------------------------------------------------
def _step(hyps, done, S, t, history, rows):
    """rows[b] = [(score, token, parent)] * 2K, best first."""
    sc = torch.tensor([[r[0] for r in rr] for rr in rows], dtype=torch.float32)
    tk = torch.tensor([[r[1] for r in rr] for rr in rows])
    pr = torch.tensor([[r[2] for r in rr] for rr in rows])
    return BO.process(hyps, done, S, t, history, sc, tk, pr, EOS, PAD)


def test_eos_of_rank_below_k_becomes_a_hypothesis_and_of_rank_k_or_more_is_skipped():
    K, S = 2, 5
    hyps, done = [BO.BeamHypotheses(K, 1.0, False)], [False]
    history = [[7, 8], [9, 10]]
    # rank 1: EOS < K -> hypothesis; rank 2: EOS >= K, reached before the K-th running beam -> skipped; rank 3 fills beam 1
    nsc, ntok, npar = _step(hyps, done, S, 2, history, [[(-1.0, 11, 0), (-2.0, EOS, 1), (-3.0, EOS, 0), (-4.0, 12, 1)]])
    assert ntok.tolist() == [[11, 12]] and npar.tolist() == [[0, 1]] and nsc.tolist() == [[-1.0, -4.0]]
    assert hyps[0].beams == [(-2.0 / 7, [9, 10])]                # scored over S + t = 7 columns; the rank-2 EOS is not kept
    assert not done[0]


def test_full_set_rejects_a_worse_hypothesis_and_replaces_the_worst():
    K, S = 2, 4
    h = BO.BeamHypotheses(K, 0.0, False)
    h.add(S + 1, [1], -1.0)
    h.add(S + 1, [2], -3.0)
    h.add(S + 2, [3, 3], -5.0)                                   # worse than the worst kept: rejected
    assert [b[1] for b in h.beams] == [[1], [2]] and h.worst_score == -3.0
    h.add(S + 2, [4, 4], -2.0)                                   # better: the worst (-3) drops out
    assert [b[1] for b in h.beams] == [[1], [4, 4]] and h.worst_score == -2.0


@pytest.mark.parametrize("early", [True, False])
def test_early_stopping(early):
    K, S = 2, 3
    hyps, done = [BO.BeamHypotheses(K, 1.0, early)], [False]
    history = [[5], [6]]
    # two EOS in the top K: the set is full
    _step(hyps, done, S, 1, history, [[(-0.5, EOS, 0), (-0.6, EOS, 1), (-0.7, 11, 0), (-0.8, 12, 1)]])
    assert len(hyps[0]) == 2
    # early_stopping=False: worst kept = -0.6 / 4 >= best candidate -0.5 / 4 is false -> not done
    assert done[0] is early


def test_done_prompt_next_to_a_running_one_emits_pad():
    K, S = 2, 3
    hyps = [BO.BeamHypotheses(K, 1.0, True), BO.BeamHypotheses(K, 1.0, True)]
    done = [True, False]
    history = [[1], [1], [2], [3]]
    nsc, ntok, npar = _step(hyps, done, S, 1, history, [[(-0.1, 20, 0), (-0.2, 21, 1), (-0.3, 22, 0), (-0.4, 23, 1)],
                                                       [(-0.1, 30, 1), (-0.2, 31, 0), (-0.3, 32, 0), (-0.4, 33, 1)]])
    assert ntok[0].tolist() == [PAD, PAD] and nsc[0].tolist() == [0.0, 0.0]
    assert ntok[1].tolist() == [30, 31] and npar[1].tolist() == [1, 0]


def test_finalisation_at_max_length_adds_the_running_beams():
    K, S, T = 2, 3, 2
    hyps, done = [BO.BeamHypotheses(K, 1.0, False)], [False]
    hyps[0].add(S + 1, [4], -3.0)                                # -0.75
    history = [[5, 6], [7, 8]]
    seqs = BO.finalize(hyps, done, S, T, history, torch.tensor([-1.0, -10.0]), 2)
    assert seqs == [[[5, 6], [4]]]                               # -1/5 beats -3/4; -10/5 = -2 loses to -0.75
    ids = BO.sequences(torch.tensor([[1, 1, 1]]), seqs, S + T, EOS, PAD)
    assert ids.tolist() == [[1, 1, 1, 5, 6], [1, 1, 1, 4, EOS]]   # L = min(longest + 1, max_length)


@pytest.mark.parametrize("lp", [0.0, 1.0, 2.0])
def test_length_penalty_normalises_by_the_prompt_inclusive_length(lp):
    """A = 2 generated tokens with sum -2.0, B = 6 tokens with sum -4.5, after an S = 20 prompt.  4.28 divides by the full
    length (22 vs 26) and keeps A at every lp; dividing by the generated length only (2 vs 6, transformers 5.x) would pick B
    at lp = 1 and 2.  At lp = 0 the two rules agree."""
    S = 20
    h = BO.BeamHypotheses(2, lp, False)
    h.add(S + 2, [5, 6], -2.0)
    h.add(S + 6, [1, 2, 3, 4, 5, 6], -4.5)
    assert sorted(h.beams, key=lambda x: x[0])[-1][1] == [5, 6]
    assert (-4.5 / 6 ** lp > -2.0 / 2 ** lp) == (lp > 0)             # the generated-only rule's winner


def test_host_finalisation_of_generate_matches_the_restatement():
    """ModifiedLlamaForCausalLM's host finalisation (beam_finalize / beam_output) against the restated finalize / sequences on
    random hypothesis sets, ties included."""
    from navillm_b200.generation import beam_finalize, beam_output
    gen = torch.Generator().manual_seed(0)
    for trial in range(200):
        B, K, S, T = 3, int(torch.randint(2, 6, (1,), generator=gen)), 7, int(torch.randint(1, 9, (1,), generator=gen))
        lp = [0.0, 1.0, 2.0][trial % 3]
        n = int(torch.randint(1, K + 1, (1,), generator=gen))
        hyps = [BO.BeamHypotheses(K, lp, False) for _ in range(B)]
        for b in range(B):
            for _ in range(int(torch.randint(0, 2 * K, (1,), generator=gen))):
                L = int(torch.randint(0, T, (1,), generator=gen))
                hyps[b].add(S + L, torch.randint(3, 50, (L,), generator=gen).tolist(), float(-torch.randint(1, 6, (1,), generator=gen)))
        done = [bool(torch.rand(1, generator=gen) < 0.3) and len(h) == K for h in hyps]
        history = [torch.randint(3, 50, (T,), generator=gen).tolist() for _ in range(B * K)]
        scores = -torch.randint(1, 6, (B * K,), generator=gen).float()
        mine = beam_finalize([list(h.beams) for h in hyps], [h.worst_score for h in hyps],
                             [None if done[b] else [(float(scores[b * K + k]), history[b * K + k]) for k in range(K)]
                              for b in range(B)], S, T, K, n, lp)
        ref = BO.finalize(hyps, done, S, T, history, scores, n)
        assert mine == ref, trial
        prompt = torch.randint(3, 50, (B, S), generator=gen)
        assert torch.equal(beam_output(prompt, mine, S, S + T, EOS, PAD), BO.sequences(prompt, ref, S + T, EOS, PAD))


def test_beam_entry_points_are_exported():
    from navillm_b200 import _lib
    lib = _lib.load()
    for name in ("nv_beam_topk", "nv_beam_select", "nv_decode_attn_rope_beam", "nv_decode_attn_rope_beam_fp8"):
        assert hasattr(lib, name), name
