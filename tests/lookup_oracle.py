"""Prompt-lookup speculative decoding restated in Python: HF's PromptLookupCandidateGenerator (the drafts of
``ops.lookup_draft``), the accept rule of ``ops.lookup_accept``, a whole lookup generation over any next-token function, and a
teacher-forced greedy check of a generated path against the CPU oracle."""
from __future__ import annotations

import numpy as np
import torch

from oracle import navillm_oracle as O


def draft(hist, k: int, ngram: int = 2, special=(), eos=None) -> list:
    """The up to k drafts for a row whose history (non-pad prompt ids, then generated tokens) is ``hist``: for n = min(ngram,
    len - 1) down to 1, the earliest i with hist[i:i + n] equal to the last n tokens and i + n < len decides; the drafts are the
    tokens from i + n on, at most k, cut at the history's end and at the first special id or EOS (possibly none)."""
    hist = [int(t) for t in hist]
    L, stop = len(hist), set(int(s) for s in special) | ({int(eos)} if eos is not None else set())
    for n in range(min(ngram, L - 1), 0, -1):
        tail = hist[L - n:]
        for i in range(0, L - n):
            if hist[i:i + n] == tail:
                out = []
                for t in hist[i + n:i + n + k]:
                    if t in stop:
                        break
                    out.append(t)
                return out
    return []


def draft_hf_literal(hist, k: int, ngram: int, eos: int) -> list:
    """transformers' PromptLookupCandidateGenerator.get_candidates (max_length unbounded), transcribed on a [1, L] tensor."""
    input_ids = torch.tensor([hist], dtype=torch.long)
    input_length = input_ids.size(1)
    chosen_ids = None
    match_found = False
    for ngram_size in range(min(ngram, input_length - 1), 0, -1):
        windows = input_ids.unfold(dimension=1, size=ngram_size, step=1)
        ngram_tensor = input_ids[0, -ngram_size:]
        matches = (windows == ngram_tensor).all(dim=2)
        match_indices = matches.nonzero(as_tuple=True)[1]
        for idx in match_indices:
            start_idx = idx + ngram_size
            end_idx = min(start_idx + k, input_length)
            if start_idx < end_idx:
                chosen_ids = input_ids[0, start_idx:end_idx]
                match_found = True
                mask = chosen_ids == eos
                hit = torch.nonzero(mask)
                if hit.numel() > 0:
                    chosen_ids = chosen_ids[:hit[0].item()]
                break
        if match_found:
            break
    return [] if chosen_ids is None else chosen_ids.tolist()


def accept(t, drafts, n_out: int, max_new: int, stop_on_eos: bool, eos: int) -> tuple:
    """One verify step of a row that has emitted n_out tokens: t [k + 1] the argmax after each window token, drafts [k] (-1 none).
    Returns (emitted tokens, accepted drafts among them, finished)."""
    m = 0
    while m < len(drafts) and int(drafts[m]) == int(t[m]):
        m += 1
    out = []
    for j in range(m + 1):
        if n_out + len(out) >= max_new:
            break
        out.append(int(t[j]))
        if stop_on_eos and int(t[j]) == eos:
            return out, len(out) - 1, True
    return out, max(len(out) - 1, 0), n_out + len(out) >= max_new


def lookup_generate(next_token, prompts, k: int, max_new: int, stop_on_eos: bool, eos: int, pad: int, drafts_of=None):
    """Lookup decoding of ``prompts`` (lists of non-pad ids) over a greedy ``next_token(prefix) -> id``, with the drafts of
    ``drafts_of(row, history)`` (default: ``draft``).  Returns (generated [B, width] with pad after EOS, accepted drafts per row,
    steps); the width rule is ``decode()``'s: the slowest row's first EOS + 1 when every row emitted EOS, else max_new."""
    drafts_of = drafts_of or (lambda b, h: draft(h, k, eos=eos))
    n = max(max_new, 1)
    hist = [list(p) + [next_token(list(p))] for p in prompts]
    gen = [[h[-1]] for h in hist]
    done = [(stop_on_eos and g[0] == eos) or n == 1 for g in gen]
    acc, steps = [0] * len(prompts), 0
    while not all(done):
        steps += 1
        for b, h in enumerate(hist):
            if done[b]:
                continue
            d = (list(drafts_of(b, h)) + [-1] * k)[:k]
            window = [h[-1]] + [x if x >= 0 else h[-1] for x in d]
            t, ctx = [], list(h)
            for j in range(k + 1):                                  # row j predicts after window token j
                if j:
                    ctx.append(window[j])
                t.append(next_token(ctx))
            out, a, fin = accept(t, d, len(gen[b]), n, stop_on_eos, eos)
            gen[b] += out
            h += out
            acc[b] += a
            done[b] = fin
    width = n
    if stop_on_eos and n > 1 and all(eos in g for g in gen):
        width = max(g.index(eos) for g in gen) + 1
    ids = torch.full((len(prompts), width), pad, dtype=torch.int64)
    for b, g in enumerate(gen):
        ids[b, :min(len(g), width)] = torch.tensor(g[:width])
    return ids, acc, steps


def greedy_follow_path(sd, cfg, input_ids, attention_mask, path, cand_vis=None, eos_token_id=2, stop_on_eos=True, ulps=3):
    """Teacher-forced greedy check of ``path`` [B, S + n]: each generated token must be the oracle's argmax from the path's own
    prefix, or have a logit within ``ulps`` bf16 ulp of the largest (the bf16 noise floor of a differently ordered forward).  Rows
    are not checked after their EOS.  Returns (exact, excused, outside) counts."""
    def ulp(x):
        return 2.0 ** (np.floor(np.log2(max(abs(x), 1e-30))) - 7)
    B, S = input_ids.shape
    n = path.shape[1] - S
    mask = attention_mask.clone()
    past: list = [None] * cfg.n_layers
    pos = (mask.long().cumsum(-1) - 1).masked_fill(mask == 0, 1)
    out = O.modified_lm_forward(sd, cfg, input_ids, mask, cand_vis=cand_vis, position_ids=pos, past_kv=past)
    live = [True] * B
    exact = excused = outside = 0
    for t in range(n):
        logits = out["logits"][:, -1].double()
        d = path[:, S + t]
        for b in range(B):
            if not live[b]:
                continue
            best = int(torch.argmax(logits[b]))
            if int(d[b]) == best:
                exact += 1
            elif float(logits[b, best]) - float(logits[b, int(d[b])]) <= ulps * ulp(float(logits[b, best])):
                excused += 1
            else:
                outside += 1
        mask = torch.cat([mask, mask.new_ones(B, 1)], dim=1)
        pos = (mask.long().cumsum(-1) - 1)[:, -1:]
        out = O.modified_lm_forward(sd, cfg, d[:, None], mask, position_ids=pos, past_kv=past)
        if stop_on_eos:
            live = [live[b] and int(d[b]) != eos_token_id for b in range(B)]
    return exact, excused, outside
