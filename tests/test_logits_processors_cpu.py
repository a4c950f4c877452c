"""The processor restatement of tests/processors_oracle.py against the installed transformers' own processor classes, on bf16
(and fp32) scores, bit for bit; and generate()'s argument checks, which need no device."""
import pytest
import torch

from tests import processors_oracle as PO

bf16 = torch.bfloat16
V, EOS = 300, 2


def _case(R, S, t, seed, dtype=bf16, logprobs=False):
    g = torch.Generator().manual_seed(seed)
    scores = torch.randn(R, V, generator=g) * 4
    if logprobs:
        scores = torch.log_softmax(scores, dim=-1)
    scores[:, 5] = 0.0                                               # zero scores
    scores[:, 7] = float("-inf")                                     # -inf scores
    scores = scores.to(dtype)
    ids = torch.randint(0, 12, (R, S + t), generator=g)              # a small alphabet: many repeats and n-gram matches
    ids[:, :3] = 0                                                   # left pads (pad id 0 here)
    ids[0, :] = 9                                                    # a row where every history id repeats
    ids[1, S:] = 7                                                   # a -inf id in the history
    ids[2, -1] = 5                                                   # a zero score in the history
    return scores, ids


def _hf(scores, ids, S, penalty, n, min_length, min_new):
    from transformers.generation import logits_process as LP
    s = scores
    if penalty != 1.0:
        s = LP.RepetitionPenaltyLogitsProcessor(penalty)(ids, s)
    if n > 0:
        s = LP.NoRepeatNGramLogitsProcessor(n)(ids, s)
    if min_length > 0:
        s = LP.MinLengthLogitsProcessor(min_length, EOS)(ids, s)
    if min_new > 0:
        s = LP.MinNewTokensLengthLogitsProcessor(S, min_new, EOS)(ids, s)
    return s


@pytest.mark.parametrize("dtype", [bf16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("logprobs", [False, True], ids=["logits", "logprobs"])
@pytest.mark.parametrize("penalty", [1.0, 1.3, 0.7, 1.2])
@pytest.mark.parametrize("n", [0, 1, 2, 3, 4])
def test_processors_match_transformers(dtype, logprobs, penalty, n):
    for S, t in ((6, 0), (6, 3), (20, 9), (1, 0), (2, 1)):           # histories shorter than n included
        for min_length, min_new in ((0, 0), (S + t + 1, 0), (0, t + 1), (S + t, t), (3, 0)):
            scores, ids = _case(4, S, t, seed=S * 31 + t + n, dtype=dtype, logprobs=logprobs)
            want = _hf(scores, ids, S, penalty, n, min_length, min_new)
            got = PO.process(scores, ids, S, repetition_penalty=penalty, no_repeat_ngram_size=n, min_length=min_length,
                             min_new_tokens=min_new, eos_token_id=EOS)
            assert got.dtype == dtype
            assert torch.equal(got.view(torch.int16 if dtype == bf16 else torch.int32),
                               want.view(torch.int16 if dtype == bf16 else torch.int32)), (S, t, min_length, min_new)


def test_repetition_penalty_is_ieee_division_in_bf16():
    """bf16 / p is the fp32 IEEE quotient rounded once (what the kernel's __fdiv_rn gives); p = 1.2 tells it apart from a
    multiply by the reciprocal."""
    import numpy as np
    x = torch.arange(0, 65536, dtype=torch.int32).to(torch.int16).view(bf16)
    x = x[torch.isfinite(x.float()) & (x.float() > 0)]
    for p in (1.2, 1.3):
        want = torch.from_numpy(x.float().numpy() / np.float32(p)).to(bf16)
        got = PO.process(x[None], torch.arange(x.numel())[None], 1, repetition_penalty=p)[0]
        assert torch.equal(got.view(torch.int16), want.view(torch.int16))


def test_processor_arguments_are_checked_like_hf():
    from navillm_b200.generation import processors
    assert processors(None, None, None, None, 2) is None
    assert processors(1.0, 0, 0, 0, 2) is None
    assert processors(1, 0, None, 0, 2) is None                   # HF builds no processor for 1: no type check either
    assert processors(1.3, 3, 0, 4, 2) == (1.3, 3, 0, 4, 2)
    for bad in (dict(repetition_penalty=0.0), dict(repetition_penalty=-1.0), dict(repetition_penalty=2),
                dict(no_repeat_ngram_size=-1), dict(no_repeat_ngram_size=2.0), dict(min_length=-1), dict(min_new_tokens=-2),
                dict(min_new_tokens=True)):
        kw = dict(repetition_penalty=None, no_repeat_ngram_size=None, min_length=None, min_new_tokens=None)
        kw.update(bad)
        with pytest.raises(ValueError):
            processors(*kw.values(), 2)


@pytest.mark.parametrize("precision", ["fp32", "amp_bf16"])
def test_oracle_matches_reference_processor_goldens(precision):
    """The restated loops against the reference's 3dqa branch with processors (tests/golden/make_processors_golden.py): fp32
    exactly; amp_bf16 equal until a bf16 near-tie of the oracle (5.5 processes fp32 copies of the bf16 scores there)."""
    from pathlib import Path
    from tests.test_beam_gpu import _qa, near_tie_ok
    from tests.test_fullwidth_parity_gpu import compare_greedy_rows
    from tests.test_oracle_golden import load
    g, cfg, tok = load(precision)
    gold = torch.load(Path(__file__).resolve().parent / "golden" / f"generate_processors_{precision}.pt", weights_only=False)
    text, cand = _qa(g, cfg, tok)
    S, n_new = gold["prompt_len"], gold["meta"]["max_new_tokens"]
    ids_kw = dict(cand_vis=cand, max_new_tokens=n_new, eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id)
    for run in gold["runs"]:
        K, proc = run["num_beams"], run["proc"]
        if K == 1:
            ids, steps = PO.greedy_generate(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], return_logits=True,
                                            **ids_kw, **proc)
        else:
            ids, steps = PO.beam_generate(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], num_beams=K,
                                          length_penalty=0.0, return_steps=True, **ids_kw, **proc)
        if precision == "fp32":
            assert torch.equal(ids, run["ids"]), (K, proc)
        elif not torch.equal(ids, run["ids"]):
            if K == 1:
                L = min(ids.shape[1], run["ids"].shape[1])
                compare_greedy_rows(ids[:, :L], run["ids"][:, :L], steps, S, min(L - S, len(steps)), tag=str(proc))
            else:
                near_tie_ok(ids, run["ids"], steps, S, 1, tag=f"K={K} {proc}")
