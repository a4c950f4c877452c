"""CPU restatement of beam search as the reference reaches it: HF ``GenerationMixin.beam_search`` with
``BeamSearchScorer`` / ``BeamHypotheses`` of transformers 4.28.0 (the version requirements.txt:20 pins), driven through
``models/nav_model.py:388-396`` -> ``lang_model.generate(**kwargs)``, on the oracle's ``modified_lm_forward``.
*** TEST INFRASTRUCTURE ONLY *** (the product never imports it).

Where transformers 4.28 and the installed 5.5 differ, this follows 4.28: a hypothesis is scored
``sum_logprobs / len ** length_penalty`` with ``len`` the FULL sequence length, the S prompt columns included
(4.28 ``hyp.shape[-1]``); 5.5 divides by the generated length only.  The two agree at ``length_penalty=0``, where the goldens
of tests/golden/make_beam_golden.py are recorded.  ``torch.topk`` leaves the order of equal scores unspecified; here equal
scores order by ascending flat index (beam-major, then token), the rule the CUDA kernel implements.

One deliberate deviation from the reference: the visual vectors of prompt b reach all K beams of prompt b.  HF expands
every tensor model kwarg with ``repeat_interleave(num_beams, dim=0)``; ``cand_vis`` is [N_cand, D] in row-major token order,
so the reference's expansion hands the vectors to the wrong ``<cand>`` slots (models/modified_lm.py:105-110).
"""
from __future__ import annotations

import sys
from pathlib import Path

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from oracle import navillm_oracle as O  # noqa: E402


class BeamHypotheses:
    """transformers 4.28 ``BeamHypotheses``: the best ``num_beams`` finished hypotheses of one prompt."""

    def __init__(self, num_beams: int, length_penalty: float, early_stopping: bool):
        self.num_beams, self.length_penalty, self.early_stopping = num_beams, length_penalty, early_stopping
        self.beams, self.worst_score = [], 1e9

    def __len__(self):
        return len(self.beams)

    def add(self, hyp_len: int, tokens: list, sum_logprobs: float):
        """``hyp_len`` = hyp.shape[-1]: prompt columns + generated tokens."""
        score = sum_logprobs / (hyp_len ** self.length_penalty)
        if len(self) < self.num_beams or score > self.worst_score:
            self.beams.append((score, tokens))
            if len(self) > self.num_beams:
                ranked = sorted([(s, idx) for idx, (s, _) in enumerate(self.beams)])
                del self.beams[ranked[0][1]]
                self.worst_score = ranked[1][0]
            else:
                self.worst_score = min(score, self.worst_score)

    def is_done(self, best_sum_logprobs: float, cur_len: int) -> bool:
        if len(self) < self.num_beams:
            return False
        if self.early_stopping:
            return True
        return self.worst_score >= best_sum_logprobs / cur_len ** self.length_penalty


def top_candidates(scores: torch.Tensor, K: int):
    """scores [B, K * V] fp32 -> the 2K best per prompt by (score desc, flat index asc): (scores, tokens, parents)."""
    V = scores.shape[1] // K
    vals, idx = torch.sort(scores, dim=1, descending=True, stable=True)
    vals, idx = vals[:, :2 * K], idx[:, :2 * K]
    return vals, idx % V, idx // V


def process(hyps, done, S: int, t: int, history, cand_scores, cand_tokens, cand_parents, eos: int, pad: int):
    """``BeamSearchScorer.process``: history[b * K + k] = generated tokens of running beam k of prompt b (t of them).
    Returns the next (scores, tokens, parents-within-prompt) [B, K] and updates ``hyps`` / ``done``.  A done prompt's beams
    get pad with score 0 (4.28 points them at global beam 0; any parent leaves the output unchanged, this keeps their own)."""
    B, K2 = cand_scores.shape
    K = K2 // 2
    nsc = torch.zeros((B, K), dtype=torch.float32)
    ntok = torch.zeros((B, K), dtype=torch.int64)
    npar = torch.zeros((B, K), dtype=torch.int64)
    for b in range(B):
        if done[b]:
            ntok[b] = pad
            npar[b] = torch.arange(K)
            continue
        j = 0
        for rank in range(K2):
            tok, sc, par = int(cand_tokens[b, rank]), cand_scores[b, rank], int(cand_parents[b, rank])
            if tok == eos:
                if rank >= K:
                    continue
                hyps[b].add(S + t, list(history[b * K + par]), sc.item())
            else:
                nsc[b, j], ntok[b, j], npar[b, j] = sc, tok, par
                j += 1
            if j == K:
                break
        done[b] = done[b] or hyps[b].is_done(cand_scores[b].max().item(), S + t)
    return nsc, ntok, npar


def finalize(hyps, done, S: int, T: int, history, beam_scores, n_return: int):
    """``BeamSearchScorer.finalize``: generated tokens of the ``n_return`` best hypotheses per prompt, best first."""
    K = hyps[0].num_beams
    out = []
    for b, h in enumerate(hyps):
        if not done[b]:
            for k in range(K):
                h.add(S + T, list(history[b * K + k]), beam_scores[b * K + k].item())
        ranked = sorted(h.beams, key=lambda x: x[0])
        out.append([ranked.pop()[1] for _ in range(n_return)])
    return out


def sequences(input_ids, seqs, max_length: int, eos: int, pad: int) -> torch.Tensor:
    """HF ``sequences``: [B * n, min(longest + 1, max_length)]; EOS after a shorter row, then pad."""
    S = input_ids.shape[1]
    rows = [(b, t) for b, per in enumerate(seqs) for t in per]
    L = min(max(S + len(t) for _, t in rows) + 1, max_length)
    out = torch.full((len(rows), L), pad, dtype=torch.int64)
    for i, (b, toks) in enumerate(rows):
        n = S + len(toks)
        out[i, :S] = input_ids[b]
        out[i, S:n] = torch.tensor(toks, dtype=torch.int64)
        if n < L:
            out[i, n] = eos
    return out


def beam_generate(sd, cfg, input_ids, attention_mask, cand_vis=None, hist_vis=None, obj_vis=None, num_beams=4, max_new_tokens=20,
                  eos_token_id=2, pad_token_id=0, length_penalty=1.0, early_stopping=False, num_return_sequences=1,
                  return_steps=False):
    """4.28 ``beam_search`` on ``modified_lm_forward`` with a KV cache.  Next-token scores: the forward's logits (special
    tokens -inf, models/modified_lm.py:122-124), ``log_softmax`` in their dtype (fp32 inside, rounded once), plus the fp32
    running beam score.  With ``return_steps``, also returns per step the [B, 2K + 1] best scores (near-tie checks)."""
    B, S = input_ids.shape
    K = num_beams
    mask = attention_mask.clone()
    past: list = [None] * cfg.n_layers
    pos = (mask.long().cumsum(-1) - 1).masked_fill(mask == 0, 1)
    out = O.modified_lm_forward(sd, cfg, input_ids, mask, cand_vis=cand_vis, hist_vis=hist_vis, obj_vis=obj_vis, position_ids=pos,
                                past_kv=past)
    logits = out["logits"][:, -1].repeat_interleave(K, 0)            # the K beams of a prompt: its prefill, its visual tokens
    past = [(k.repeat_interleave(K, 0), v.repeat_interleave(K, 0)) for k, v in past]
    mask = mask.repeat_interleave(K, 0)
    beam_scores = torch.zeros((B, K), dtype=torch.float32)
    beam_scores[:, 1:] = -1e9
    beam_scores = beam_scores.view(-1)
    hyps = [BeamHypotheses(K, length_penalty, early_stopping) for _ in range(B)]
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
        scores = (lp.float() + beam_scores[:, None]).view(B, -1)
        if return_steps:
            steps.append(torch.sort(scores, dim=1, descending=True, stable=True)[0][:, :2 * K + 1])
        cs, ct, cp = top_candidates(scores, K)
        nsc, ntok, npar = process(hyps, done, S, t, history, cs, ct, cp, eos_token_id, pad_token_id)
        src = (torch.arange(B)[:, None] * K + npar).view(-1)
        history = [history[int(r)] + [int(tk)] for r, tk in zip(src, ntok.view(-1))]
        past = [(k[src], v[src]) for k, v in past]
        mask = torch.cat([mask, mask.new_ones(B * K, 1)], dim=1)
        beam_scores = nsc.view(-1)
        T = t + 1
        if all(done):
            break
    seqs = finalize(hyps, done, S, T, history, beam_scores, num_return_sequences)
    ids = sequences(input_ids, seqs, S + max_new_tokens, eos_token_id, pad_token_id)
    return (ids, steps) if return_steps else ids
