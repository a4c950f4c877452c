"""CPU restatement of the HF logits processors that generate() honours -- ``RepetitionPenaltyLogitsProcessor``,
``NoRepeatNGramLogitsProcessor``, ``MinLengthLogitsProcessor`` and ``MinNewTokensLengthLogitsProcessor`` of transformers 4.28
(the reference's pin), in its ``_get_logits_processor`` order -- and the greedy, sampled and beam loops of the oracle with them.
*** TEST INFRASTRUCTURE ONLY *** (the product never imports it).

4.28 runs the processors on the scores in their own dtype: the bf16 next-token logits (greedy, sampling) or the bf16
``log_softmax`` output (beam search, before the fp32 beam-score add).  transformers 5.5, installed here and used to record the
goldens, casts the logits to fp32 first; on an fp32 model the two agree, on amp_bf16 they may differ by bf16 near-ties.

The history of a row is HF's ``input_ids``: the padded prompt row as passed (left pads included) and the generated tokens.
"""
from __future__ import annotations

import sys
from pathlib import Path

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from oracle import navillm_oracle as O  # noqa: E402
from tests import beam_oracle as BO  # noqa: E402


def process(scores: torch.Tensor, input_ids: torch.Tensor, S: int, repetition_penalty: float = 1.0, no_repeat_ngram_size: int = 0,
            min_length: int = 0, min_new_tokens: int = 0, eos_token_id: int = 2) -> torch.Tensor:
    """The four processors on ``scores`` [R, V] (any float dtype, kept) for histories ``input_ids`` [R, S + t] int64; a new
    tensor.  S: the padded prompt width (MinNewTokensLength's ``prompt_length_to_skip``)."""
    s = scores.clone()
    R, L = input_ids.shape
    if repetition_penalty != 1.0:                                    # gather before scatter: each id penalised once
        sc = torch.gather(s, 1, input_ids)
        sc = torch.where(sc < 0, sc * repetition_penalty, sc / repetition_penalty)
        s.scatter_(1, input_ids, sc)
    n = no_repeat_ngram_size
    if n > 0 and L + 1 >= n:                                         # _calc_banned_ngram_tokens
        for r in range(R):
            toks = input_ids[r].tolist()
            grams: dict = {}
            for ng in zip(*[toks[i:] for i in range(n)]):
                grams[tuple(ng[:-1])] = grams.get(tuple(ng[:-1]), []) + [ng[-1]]
            banned = grams.get(tuple(toks[L + 1 - n:L]), [])
            s[r, banned] = float("-inf")
    if min_length > 0 and L < min_length:
        s[:, eos_token_id] = float("-inf")
    if min_new_tokens > 0 and L - S < min_new_tokens:
        s[:, eos_token_id] = float("-inf")
    return s


def greedy_generate(sd, cfg, input_ids, attention_mask, cand_vis=None, hist_vis=None, obj_vis=None, max_new_tokens=20, eos_token_id=2,
                    pad_token_id=0, stop_on_eos=True, return_logits=False, **proc):
    """4.28 greedy search on ``modified_lm_forward`` with the processors on the next-token logits in their dtype (the oracle's
    ``greedy_generate`` loop, processed before the argmax).  ``return_logits``: the processed scores of every step (fp32)."""
    B, S = input_ids.shape
    ids, mask = input_ids.clone(), attention_mask.clone()
    past: list = [None] * cfg.n_layers
    unfinished = torch.ones(B, dtype=torch.bool)
    steps = []
    for step in range(max_new_tokens):
        pos = (mask.long().cumsum(-1) - 1).masked_fill(mask == 0, 1)
        if step == 0:
            out = O.modified_lm_forward(sd, cfg, ids, mask, cand_vis=cand_vis, hist_vis=hist_vis, obj_vis=obj_vis, position_ids=pos,
                                        past_kv=past)
        else:
            out = O.modified_lm_forward(sd, cfg, ids[:, -1:], mask, position_ids=pos[:, -1:], past_kv=past)
        scores = process(out["logits"][:, -1, :], ids, S, eos_token_id=eos_token_id, **proc).float()
        steps.append(scores)
        nxt = scores.argmax(dim=-1)
        nxt = torch.where(unfinished, nxt, torch.full_like(nxt, pad_token_id))
        ids = torch.cat([ids, nxt[:, None]], dim=1)
        mask = torch.cat([mask, mask.new_ones(B, 1)], dim=1)
        if stop_on_eos:
            unfinished = unfinished & (nxt != eos_token_id)
            if not bool(unfinished.any()):
                break
    return (ids, steps) if return_logits else ids


def sample_support(sd, cfg, input_ids, attention_mask, generated, cand_vis=None, top_k=50, temperature=1.0, **proc):
    """For a sampled run ``generated`` [B, n] (the tokens the device drew), teacher-forced: per step, the bool [B, V] support of
    the distribution 4.28 ``sample`` draws from (processors on the bf16 logits, then temperature and top-k)."""
    B, S = input_ids.shape
    ids, mask = input_ids.clone(), attention_mask.clone()
    past: list = [None] * cfg.n_layers
    out_support = []
    for step in range(generated.shape[1]):
        pos = (mask.long().cumsum(-1) - 1).masked_fill(mask == 0, 1)
        if step == 0:
            out = O.modified_lm_forward(sd, cfg, ids, mask, cand_vis=cand_vis, position_ids=pos, past_kv=past)
        else:
            out = O.modified_lm_forward(sd, cfg, ids[:, -1:], mask, position_ids=pos[:, -1:], past_kv=past)
        scores = process(out["logits"][:, -1, :], ids, S, **proc)
        out_support.append(O.sampling_probs(scores, temperature, top_k) > 0)
        ids = torch.cat([ids, generated[:, step:step + 1]], dim=1)
        mask = torch.cat([mask, mask.new_ones(B, 1)], dim=1)
    return out_support


def beam_generate(sd, cfg, input_ids, attention_mask, cand_vis=None, num_beams=4, max_new_tokens=20, eos_token_id=2, pad_token_id=0,
                  length_penalty=1.0, early_stopping=False, num_return_sequences=1, return_steps=False, **proc):
    """tests/beam_oracle.beam_generate with the processors on the bf16 log-probs of each beam before the beam-score add."""
    B, S = input_ids.shape
    K = num_beams
    mask = attention_mask.clone()
    past: list = [None] * cfg.n_layers
    pos = (mask.long().cumsum(-1) - 1).masked_fill(mask == 0, 1)
    out = O.modified_lm_forward(sd, cfg, input_ids, mask, cand_vis=cand_vis, position_ids=pos, past_kv=past)
    logits = out["logits"][:, -1].repeat_interleave(K, 0)
    past = [(k.repeat_interleave(K, 0), v.repeat_interleave(K, 0)) for k, v in past]
    mask = mask.repeat_interleave(K, 0)
    prompt = input_ids.repeat_interleave(K, 0)
    beam_scores = torch.zeros((B, K), dtype=torch.float32)
    beam_scores[:, 1:] = -1e9
    beam_scores = beam_scores.view(-1)
    hyps = [BO.BeamHypotheses(K, length_penalty, early_stopping) for _ in range(B)]
    done = [False] * B
    history = [[] for _ in range(B * K)]
    steps = []
    T = 0
    for t in range(max_new_tokens):
        if t > 0:
            pos = (mask.long().cumsum(-1) - 1).masked_fill(mask == 0, 1)
            last = torch.tensor([h[-1] for h in history], dtype=torch.int64)[:, None]
            out = O.modified_lm_forward(sd, cfg, last, mask, position_ids=pos[:, -1:], past_kv=past)
            logits = out["logits"][:, -1]
        lp = F.log_softmax(logits.float(), dim=-1).to(logits.dtype)
        hist_ids = torch.cat([prompt, torch.tensor(history, dtype=torch.int64).view(B * K, t)], dim=1)
        lp = process(lp, hist_ids, S, eos_token_id=eos_token_id, **proc)
        scores = (lp.float() + beam_scores[:, None]).view(B, -1)
        if return_steps:
            steps.append(torch.sort(scores, dim=1, descending=True, stable=True)[0][:, :2 * K + 1])
        cs, ct, cp = BO.top_candidates(scores, K)
        nsc, ntok, npar = BO.process(hyps, done, S, t, history, cs, ct, cp, eos_token_id, pad_token_id)
        src = (torch.arange(B)[:, None] * K + npar).view(-1)
        history = [history[int(r)] + [int(tk)] for r, tk in zip(src, ntok.view(-1))]
        past = [(k[src], v[src]) for k, v in past]
        mask = torch.cat([mask, mask.new_ones(B * K, 1)], dim=1)
        beam_scores = nsc.view(-1)
        T = t + 1
        if all(done):
            break
    seqs = BO.finalize(hyps, done, S, T, history, beam_scores, num_return_sequences)
    ids = BO.sequences(input_ids, seqs, S + max_new_tokens, eos_token_id, pad_token_id)
    return (ids, steps) if return_steps else ids
