"""CPU restatement of diverse (group) beam search as transformers 4.28 runs it: ``GenerationMixin.group_beam_search`` with
``BeamSearchScorer(num_beam_groups=G)`` and the ``HammingDiversityLogitsProcessor``, on the oracle's ``modified_lm_forward``.
*** TEST INFRASTRUCTURE ONLY *** (the product never imports it).

K beams per prompt form G groups of Kg = K / G; group g owns beams g * Kg + [0, Kg).  Only the first beam of each group starts
at score 0.  A step runs the groups in order; group g's next-token scores are the bf16 log-softmax of its rows, lowered by the
Hamming penalty (``lp = bf16(fp32(lp) - fp32(d) * freq)``, freq the bincount of the tokens groups 0 .. g - 1 chose for the
prompt in this step, pad included), then the processors of tests/processors_oracle.py on the group's own histories, then the
fp32 beam-score add.  The 2Kg best (equal scores by ascending flat index, the kernels' rule) go through
``tests/beam_oracle.process`` with group_size Kg against the prompt's one ``BeamHypotheses`` of capacity K (4.28's shared
hypotheses).  A done prompt (one an earlier group of the same step finished included) pads.  Finalisation adds the K running
beams in row order.  Two deviations of the device path are kept here too (DESIGN §2): a done prompt's rows continue their own
history, and the visual tokens of prompt b reach all K of its beams.
"""
from __future__ import annotations

import sys
from pathlib import Path

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from oracle import navillm_oracle as O  # noqa: E402
from tests import processors_oracle as PO  # noqa: E402
from tests.beam_oracle import BeamHypotheses, finalize, process, sequences, top_candidates  # noqa: E402


def hamming(lp: torch.Tensor, current, b: int, K: int, g: int, Kg: int, penalty: float) -> torch.Tensor:
    """HammingDiversityLogitsProcessor on prompt b's Kg rows ``lp`` [Kg, V] of group g: ``lp -= penalty * bincount`` of the
    tokens ``current[b * K : b * K + g * Kg]`` in torch's arithmetic (bf16 in place minus an fp32 tensor)."""
    if g == 0:
        return lp
    freq = torch.bincount(torch.as_tensor(current[b * K:b * K + g * Kg], dtype=torch.int64), minlength=lp.shape[-1])
    lp = lp.clone()
    lp -= penalty * freq
    return lp


def group_tie(steps, t: int, b: int) -> bool:
    """A near tie of prompt b at step t of ``search(return_steps=True)``'s ``steps``: two of one group's best 2Kg + 1 scores
    within 3 bf16 ulp of their magnitude (tests/test_beam_gpu.near_tie_ok's rule, applied to each group on its own)."""
    for s in steps[t]:
        fin = s[b][torch.isfinite(s[b])]
        if fin.numel() < 2:
            continue
        ulp = torch.exp2(torch.floor(torch.log2(fin[:-1].abs().clamp_min(1e-30))) - 7)
        if bool(((fin[:-1] - fin[1:]).abs() <= 3 * ulp).any()):
            return True
    return False


def search(scorer, prompt_ids, num_beams=4, num_beam_groups=2, diversity_penalty=0.5, max_new_tokens=20, eos_token_id=2,
           pad_token_id=0, length_penalty=1.0, early_stopping=False, num_return_sequences=1, return_steps=False, **proc):
    """4.28 group beam search.  ``scorer(src, last)`` returns the next-token logits [B * K, V] of the beam rows (special tokens
    -inf): at the first step ``src`` and ``last`` are None and row b * K + k holds prompt b's prefill row; later ``src`` [B * K]
    says which row each beam continues and ``last`` [B * K] is its new token.  Returns [B * n, L] ids; with ``return_steps``
    also a dict: ``steps`` per step a list over groups of the [B, 2Kg + 1] best scores (near-tie checks), ``scores`` per step
    the [B * K, V] processed log-probs (4.28's ``processed_score``), ``running`` per step the prompts not done when it began
    (the rows whose scores 4.28 computes on the same histories), ``n_steps``."""
    B, S = prompt_ids.shape
    K, G = num_beams, num_beam_groups
    Kg = K // G
    prompt = prompt_ids.repeat_interleave(K, 0)
    beam_scores = torch.full((B, K), -1e9, dtype=torch.float32)
    beam_scores[:, ::Kg] = 0
    beam_scores = beam_scores.view(-1)
    hyps = [BeamHypotheses(K, length_penalty, early_stopping) for _ in range(B)]
    done = [False] * B
    history = [[] for _ in range(B * K)]
    steps, scores, running = [], [], []
    T = 0
    src = last = None
    for t in range(max_new_tokens):
        logits = scorer(src, last)
        run0 = [not x for x in done]
        lp_all = F.log_softmax(logits.float(), dim=-1).to(logits.dtype)
        current = [0] * (B * K)
        new_src = list(range(B * K))
        new_scores = beam_scores.clone()
        new_history = list(history)
        processed = torch.zeros_like(lp_all)
        per_group = []
        for g in range(G):
            rows = [b * K + g * Kg + j for b in range(B) for j in range(Kg)]
            lp = lp_all[rows]
            lp = torch.cat([hamming(lp[b * Kg:(b + 1) * Kg], current, b, K, g, Kg, diversity_penalty) for b in range(B)])
            if proc:
                hist_ids = torch.cat([prompt[rows], torch.tensor([history[r] for r in rows], dtype=torch.int64).view(len(rows), t)],
                                     dim=1)
                lp = PO.process(lp, hist_ids, S, eos_token_id=eos_token_id, **proc)
            processed[rows] = lp
            sc = (lp.float() + beam_scores[rows][:, None]).view(B, -1)
            per_group.append(torch.sort(sc, dim=1, descending=True, stable=True)[0][:, :2 * Kg + 1])
            cs, ct, cp = top_candidates(sc, Kg)
            nsc, ntok, npar = process(hyps, done, S, t, [history[r] for r in rows], cs, ct, cp, eos_token_id, pad_token_id)
            for b in range(B):
                for j in range(Kg):
                    r, p = b * K + g * Kg + j, b * K + g * Kg + int(npar[b, j])
                    new_src[r], current[r], new_scores[r] = p, int(ntok[b, j]), nsc[b, j]
                    new_history[r] = history[p] + [int(ntok[b, j])]
        steps.append(per_group)
        scores.append(processed)
        running.append(run0)
        src, last = torch.tensor(new_src), torch.tensor(current)
        history, beam_scores = new_history, new_scores
        T = t + 1
        if all(done):
            break
    seqs = finalize(hyps, done, S, T, history, beam_scores, num_return_sequences)
    ids = sequences(prompt_ids, seqs, S + max_new_tokens, eos_token_id, pad_token_id)
    if return_steps:
        return ids, {"steps": steps, "scores": scores, "running": running, "n_steps": T}
    return ids


def model_scorer(sd, cfg, input_ids, attention_mask, K, cand_vis=None, hist_vis=None, obj_vis=None):
    """``scorer`` of ``search`` on the oracle's ``modified_lm_forward`` with a KV cache: prompt b's prefill and visual tokens
    reach its K beams, the cache rows follow ``src``."""
    state = {"mask": attention_mask.clone(), "past": [None] * cfg.n_layers}

    def scorer(src, last):
        mask, past = state["mask"], state["past"]
        if src is None:
            pos = (mask.long().cumsum(-1) - 1).masked_fill(mask == 0, 1)
            out = O.modified_lm_forward(sd, cfg, input_ids, mask, cand_vis=cand_vis, hist_vis=hist_vis, obj_vis=obj_vis,
                                        position_ids=pos, past_kv=past)
            state["past"] = [(k.repeat_interleave(K, 0), v.repeat_interleave(K, 0)) for k, v in past]
            state["mask"] = mask.repeat_interleave(K, 0)
            return out["logits"][:, -1].repeat_interleave(K, 0)
        past = [(k[src], v[src]) for k, v in past]
        mask = torch.cat([mask, mask.new_ones(mask.shape[0], 1)], dim=1)
        pos = (mask.long().cumsum(-1) - 1).masked_fill(mask == 0, 1)
        out = O.modified_lm_forward(sd, cfg, last[:, None], mask, position_ids=pos[:, -1:], past_kv=past)
        state["past"], state["mask"] = past, mask
        return out["logits"][:, -1]
    return scorer


def group_beam_generate(sd, cfg, input_ids, attention_mask, cand_vis=None, hist_vis=None, obj_vis=None, num_beams=4, **kw):
    """``search`` on the oracle model (``model_scorer``)."""
    scorer = model_scorer(sd, cfg, input_ids, attention_mask, num_beams, cand_vis, hist_vis, obj_vis)
    return search(scorer, input_ids, num_beams=num_beams, **kw)
