"""Top-p sampling on the CPU: tests/sampling_oracle.py against the installed transformers' warper chain
(Temperature -> TopK -> TopP -> softmax) on bf16 score rows at the model's vocabulary, rows with ties at the cut included."""
import pytest
import torch

from tests import sampling_oracle as SO

V = 32006
SPECIAL = [32000, 32001, 32002, 32003, 32004, 32005]


def _hf_probs(scores, temperature, top_k, top_p):
    lp = pytest.importorskip("transformers.generation.logits_process")
    s = scores
    if temperature != 1.0:
        s = lp.TemperatureLogitsWarper(temperature)(None, s)
    if top_k:
        s = lp.TopKLogitsWarper(top_k=top_k, min_tokens_to_keep=1)(None, s)
    if top_p < 1.0:
        s = lp.TopPLogitsWarper(top_p=top_p, min_tokens_to_keep=1)(None, s)
    return torch.softmax(s, dim=-1)


def score_rows(B=8, seed=0):
    g = torch.Generator().manual_seed(seed)
    s = (torch.randn(B, V, generator=g) * 2.5).to(torch.bfloat16)
    s[1, 1000:1040] = 9.0                                  # 40 equal maxima: every cut falls inside the group
    s[2, 7000:7400] = s[2].float().topk(30)[0][-1]         # a long run of ties at the 30th value
    s[3] = (torch.randn(V, generator=g) * 0.3).to(torch.bfloat16)      # flat: many tokens carry mass
    s[4, :] = -3.0
    s[4, 5] = 4.0                                          # one dominant token
    s[:, SPECIAL] = float("-inf")
    return s


@pytest.mark.parametrize("top_p", [0.0, 0.3, 0.9, 0.999, 1.0])
@pytest.mark.parametrize("top_k", [0, 1, 50])
@pytest.mark.parametrize("temperature", [1.0, 0.7])
def test_top_p_oracle_equals_hf_warpers(temperature, top_k, top_p):
    scores = score_rows(seed=top_k)
    got = SO.sampling_probs(scores, temperature, top_k, top_p)
    ref = _hf_probs(scores.clone(), temperature, top_k, top_p)
    assert got.dtype == torch.bfloat16
    for b in range(scores.shape[0]):
        if torch.equal(got[b], ref[b]):
            continue
        # torch's unstable sort may drop other members of a tie group at the cut: the same values, and the same outside the
        # group of equal scores at the cut
        assert torch.equal(got[b].sort().values, ref[b].sort().values), b
        s = scores[b].float() / temperature
        cut = s[got[b] > 0].min()
        other = s.to(torch.bfloat16).float() != cut.to(torch.bfloat16).float()
        assert torch.equal(got[b][other], ref[b][other]), b
    assert bool((got[:, SPECIAL] == 0).all())
    kept = (got > 0).sum(-1)
    assert bool((kept >= 1).all())
    if top_p == 0.0:                                        # only the largest (or a tie of the largest) survives
        assert bool((kept[[0, 3, 4]] == 1).all())


def test_top_p_removes_lowest_indices_of_a_tie_first():
    s = torch.full((1, 64), -20.0, dtype=torch.bfloat16)
    s[0, 10:20] = 1.0                                      # ten equal tokens, 0.1 each
    p = SO.sampling_probs(s, 1.0, 0, 0.55)
    assert (p[0] > 0).nonzero().flatten().tolist() == list(range(14, 20))


def test_cpu_cumsum_of_bf16_is_an_fp32_running_sum():
    """The rule nv_sample follows: torch's CPU cumsum of a bf16 row adds in fp32 and rounds each partial to bf16."""
    import numpy as np
    g = torch.Generator().manual_seed(1)
    p = torch.softmax((torch.randn(3, 4000, generator=g) * 3).to(torch.bfloat16).sort(-1).values, -1)
    acc = np.cumsum(p.float().numpy(), axis=-1, dtype=np.float32)
    assert torch.equal(p.cumsum(-1), torch.from_numpy(acc).to(torch.bfloat16))


def test_nv_sample_is_exported():
    from navillm_b200 import _lib
    lib = _lib.load()
    for name in ("nv_sample", "nv_sample_topk"):
        assert hasattr(lib, name), name
