"""Contrastive search semantics on the CPU: ``_ranking_fast`` of the restatement (tests/contrastive_oracle.py) on hand-built
vectors, the restatement against a literal transcription of transformers 4.28's contrastive_search on prompts without pads, and
generate()'s validation of the mode's arguments."""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from tests import contrastive_oracle as CO  # noqa: E402
from tests.test_beam_cpu import _qa  # noqa: E402
from tests.test_oracle_golden import load  # noqa: E402
from oracle import navillm_oracle as O  # noqa: E402

bf16 = torch.bfloat16


def test_bf_rounds_once_to_nearest_even():
    x = torch.tensor([1.0, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, 1.0 + 2.0 ** -8 + 2.0 ** -30, -0.3, 1e-3], dtype=torch.float64)
    want = torch.tensor([1.0, 1.0, 1.0 + 2 * 2.0 ** -7, 1.0 + 2.0 ** -7, -0.3, 1e-3]).to(bf16).double()
    assert torch.equal(CO.bf(x), want)


def test_ranking_fast_hand_built():
    ctx = CO.normalize(torch.tensor([[1.0, 0.0, 0.0, 0.0], [0.0, 1.0, 0.0, 0.0]]))
    cand = CO.normalize(torch.tensor([[1.0, 0.0, 0.0, 0.0],           # repeats context row 0: pen 1
                                      [0.0, 0.0, 1.0, 0.0],           # orthogonal: pen 0
                                      [1.0, 1.0, 0.0, 0.0]]))         # pen = bf16(1 / sqrt(2))
    p = torch.tensor([0.5, 0.25, 0.125]).double()
    j, pen, score = CO.ranking_fast(ctx, cand, p, 0.6)
    h = CO.bf(torch.tensor(1.0, dtype=torch.float64) / CO.bf(torch.tensor(2.0, dtype=torch.float64).sqrt()))
    assert torch.equal(pen, torch.stack([torch.tensor(1.0).double(), torch.tensor(0.0).double(), h]))
    a1, a = float(np.float32(1.0 - 0.6)), float(np.float32(0.6))
    want = CO.bf(CO.bf(a1 * p) - CO.bf(a * pen))                  # no product here lies near a bf16 midpoint
    assert torch.equal(score, want) and j == int(torch.argmax(want)) == 1
    assert float(score[1]) == float(CO.bf(torch.tensor(a1 * 0.25, dtype=torch.float64)))
    # torch's fp32 opmath: 0.0598 * fp32(0.7) lies on a bf16 midpoint after the fp32 rounding
    p = torch.tensor([0.0598], dtype=bf16)
    assert float(CO.contrastive_score(p, torch.zeros(1, dtype=torch.float64), 0.3)) == float((p.float() * 0.7).to(bf16))


def test_ranking_fast_ties_go_to_the_lowest_index():
    ctx = CO.normalize(torch.tensor([[0.0, 0.0, 1.0]]))
    cand = CO.normalize(torch.tensor([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [1.0, 1.0, 0.0]]))   # all orthogonal to the context
    p = torch.tensor([0.25, 0.25, 0.25]).double()
    assert CO.ranking_fast(ctx, cand, p, 0.5)[0] == 0
    # scores equal only after the bf16 rounding: 0.2500 and 0.2505 give the same bf16 product
    p = CO.bf(torch.tensor([0.125, 0.2500, 0.2505])).double()
    j, _, score = CO.ranking_fast(ctx, cand, p, 0.5)
    assert float(score[1]) == float(score[2]) > float(score[0]) and j == 1


def _ranking_fast_428(context_hidden, next_hidden, next_top_k_probs, alpha, beam_width):
    """transformers 4.28 ``_ranking_fast``, verbatim."""
    norm_context_hidden = context_hidden / context_hidden.norm(dim=2, keepdim=True)
    norm_next_hidden = next_hidden / next_hidden.norm(dim=2, keepdim=True)
    cosine_matrix = torch.matmul(norm_context_hidden, norm_next_hidden.transpose(1, 2)).squeeze(-1)   # [B*K, S]
    degeneration_penalty, _ = torch.max(cosine_matrix, dim=-1)                                      # [B*K]
    next_top_k_probs = next_top_k_probs.view(-1)                                                     # [B*K]
    contrastive_score = (1.0 - alpha) * next_top_k_probs - alpha * degeneration_penalty
    contrastive_score = torch.stack(torch.split(contrastive_score, beam_width))                      # [B, K]
    _, selected_idx = contrastive_score.max(dim=-1)                                                  # [B]
    return selected_idx


def _contrastive_428(sd, cfg, input_ids, mask, cand_vis, alpha, top_k, max_new_tokens, eos, pad):
    """4.28 ``contrastive_search`` on the oracle model, literally: the whole context (pads included), bf16 tensor ops,
    ``torch.topk`` (no ties at the k-th probability arise on these inputs)."""
    B = input_ids.shape[0]
    past: list = [None] * cfg.n_layers
    pos = (mask.long().cumsum(-1) - 1).masked_fill(mask == 0, 1)
    out = O.modified_lm_forward(sd, cfg, input_ids, mask, cand_vis=cand_vis, position_ids=pos, past_kv=past)
    last_hidden_states = out["hidden_states"]
    logit_for_next_step = out["logits"][:, -1, :]
    unfinished = torch.ones(B, dtype=torch.long)
    ids = input_ids.clone()
    for _ in range(max_new_tokens):
        next_probs = torch.nn.functional.softmax(logit_for_next_step, dim=-1)
        top_k_probs, top_k_ids = torch.topk(next_probs, dim=-1, k=top_k)
        past_k = [(k.repeat_interleave(top_k, 0), v.repeat_interleave(top_k, 0)) for k, v in past]
        mask_k = torch.cat([mask, mask.new_ones(B, 1)], 1).repeat_interleave(top_k, 0)
        pos_k = (mask_k.long().cumsum(-1) - 1)[:, -1:]
        outputs = O.modified_lm_forward(sd, cfg, top_k_ids.view(-1, 1), mask_k, position_ids=pos_k, past_kv=past_k)
        logits = outputs["logits"][:, -1, :]
        next_hidden = outputs["hidden_states"]
        context_hidden = last_hidden_states.repeat_interleave(top_k, dim=0)
        selected_idx = _ranking_fast_428(context_hidden, next_hidden, top_k_probs, alpha, top_k)
        next_tokens = top_k_ids[range(len(top_k_ids)), selected_idx]
        next_hidden = torch.stack(torch.split(next_hidden.squeeze(dim=1), top_k))
        next_hidden = next_hidden[range(B), selected_idx, :]
        last_hidden_states = torch.cat([last_hidden_states, next_hidden.unsqueeze(1)], dim=1)
        rows = torch.arange(B) * top_k + selected_idx
        past = [(k[rows], v[rows]) for k, v in past_k]
        logit_for_next_step = torch.stack(torch.split(logits, top_k))[range(B), selected_idx, :]
        next_tokens = next_tokens * unfinished + pad * (1 - unfinished)
        ids = torch.cat([ids, next_tokens[:, None]], dim=-1)
        mask = torch.cat([mask, mask.new_ones(B, 1)], 1)
        unfinished = unfinished.mul((next_tokens != eos).long())
        if unfinished.max() == 0:
            break
    return ids


@pytest.mark.parametrize("rows,k,alpha", [([0], 4, 0.6), ([1], 2, 0.3), ([0, 0], 10, 0.6)], ids=["B1k4", "B1k2", "B2k10"])
def test_oracle_matches_literal_428_without_pads(rows, k, alpha):
    g, cfg, tok = load("amp_bf16")
    text, cand = _qa(g, cfg, tok)
    n_cand = (text["input_ids"] == cfg.cand_id).sum(1).tolist()
    starts = np.cumsum([0] + n_cand)
    ids, vis = [], []
    for r in rows:                                           # each prompt alone: no pads
        m = text["attention_mask"][r].bool()
        ids.append(text["input_ids"][r][m])
        vis.append(cand[starts[r]:starts[r + 1]])
    input_ids = torch.stack(ids)
    mask = torch.ones_like(input_ids)
    cand_vis = torch.cat(vis, 0)
    kw = dict(penalty_alpha=alpha, top_k=k, max_new_tokens=10, eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id)
    got, steps = CO.contrastive_generate(g["state_dict"], cfg, input_ids, mask, cand_vis=cand_vis, return_steps=True, **kw)
    want = _contrastive_428(g["state_dict"], cfg, input_ids, mask, cand_vis, alpha, k, 10, tok.eos_token_id, tok.unk_token_id)
    # equal, or 4.28's fp32-accumulated bf16 ops and the restatement's fp64 chain part at a near tie of the restatement
    matched = CO.near_tie_ok(got, want, steps, input_ids.shape[1])
    assert min(matched) >= 1


@pytest.mark.parametrize("k", [4, 50])
def test_follow_path_accepts_the_restatement_and_rejects_a_wrong_token(k):
    """The teacher-forced check passes the restatement's own path with every step exact, and fails a path with one token
    replaced by one that can never be chosen."""
    g, cfg, tok = load("amp_bf16")
    text, cand = _qa(g, cfg, tok)
    kw = dict(penalty_alpha=0.6, top_k=k, eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id, stop_on_eos=False)
    S = text["input_ids"].shape[1]
    path = CO.contrastive_generate(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], cand_vis=cand, max_new_tokens=6,
                                   **kw)
    assert CO.follow_path(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], path, cand_vis=cand, **kw) == (12, 0, 0)
    bad = path.clone()
    bad[1, S + 3] = cfg.special_token_ids[-1]                 # a special id: its logit is -inf, never a candidate
    with pytest.raises(AssertionError):
        CO.follow_path(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], bad, cand_vis=cand, **kw)
    assert CO.follow_path(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], bad, cand_vis=cand, strict=False,
                          **kw)[2] >= 1


def test_generate_validation_before_any_device_work():
    """The mode's argument errors are raised before generate() touches the model or a device."""
    from navillm_b200.modified_lm import ModifiedLlamaForCausalLM
    lm = object.__new__(ModifiedLlamaForCausalLM)
    ids, mask = torch.ones(1, 3, dtype=torch.long), torch.ones(1, 3, dtype=torch.long)
    gen = lambda **kw: ModifiedLlamaForCausalLM.generate(lm, ids, mask, **kw)
    with pytest.raises(ValueError, match="num_return_sequences"):
        gen(penalty_alpha=0.6, top_k=4, num_return_sequences=2)
    for a in (float("nan"), float("inf")):
        with pytest.raises(ValueError, match="finite"):
            gen(penalty_alpha=a, top_k=4)
    with pytest.raises(NotImplementedError, match="trie"):
        gen(penalty_alpha=0.6, top_k=4, trie=object())
    with pytest.raises(NotImplementedError, match="logits_processor"):
        gen(penalty_alpha=0.6, logits_processor=[lambda i, s: s])
    with pytest.raises(NotImplementedError, match="at most 64"):
        gen(penalty_alpha=0.6, top_k=65)
