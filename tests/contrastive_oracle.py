"""CPU restatement of contrastive search as transformers 4.28 runs it (``GenerationMixin.contrastive_search`` and
``_ranking_fast``, Su et al. 2022) for a model that returns HF's hidden-state tuple, driven through
``models/nav_model.py:388-396`` -> ``lang_model.generate(penalty_alpha=..., top_k=...)``, on the oracle's ``modified_lm_forward``
with a KV cache.  *** TEST INFRASTRUCTURE ONLY *** (the product never imports it).

4.28's bf16 tensor ops are restated in fp64 and rounded to bf16 where 4.28 rounds: p = bf16(softmax(logits)), x^ = bf16(x /
bf16(||x||)), cos = bf16(c^ . h^); the score's three scalar ops are torch's own fp32 ops, each rounded to bf16.  The k candidates are the k
largest p with equal p ordered by lower token id (``torch.topk`` leaves that order unspecified), the selection is the first best
score.  Left-pad positions are not part of the context (4.28 would include their hidden states).
"""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from oracle import navillm_oracle as O  # noqa: E402
from tests import processors_oracle as PO  # noqa: E402


def bf(x: torch.Tensor) -> torch.Tensor:
    """fp64 values rounded once to the nearest bf16 (ties to even), kept in fp64."""
    m, e = np.frexp(x.detach().double().numpy())
    return torch.from_numpy(np.asarray(np.ldexp(np.rint(m * 256.0), e - 8)))


def normalize(x: torch.Tensor) -> torch.Tensor:
    """x^ = bf16(x / bf16(||x||)) of rows [.., D] holding bf16 values."""
    x = x.double()
    return bf(x / bf(x.pow(2).sum(-1, keepdim=True).sqrt()))


def ranking_fast(ctx_hat: torch.Tensor, cand_hat: torch.Tensor, p: torch.Tensor, alpha: float):
    """``_ranking_fast`` for one prompt: context rows ctx_hat [S, D], candidates cand_hat [k, D] (both normalised), their p [k].
    Returns (selected index, pen [k], score [k])."""
    pen = bf(cand_hat @ ctx_hat.T).max(dim=1).values
    return int(torch.argmax(score := contrastive_score(p, pen, alpha))), pen, score


def contrastive_score(p: torch.Tensor, pen: torch.Tensor, alpha: float) -> torch.Tensor:
    """(1 - alpha) * p - alpha * pen on bf16 tensors as torch computes it: each op in fp32 (the Python floats become fp32
    scalars), its result rounded to bf16."""
    a1, a = torch.tensor(1.0 - alpha, dtype=torch.float32), torch.tensor(alpha, dtype=torch.float32)
    x = (a1 * p.float()).to(torch.bfloat16).float()
    y = (a * pen.float()).to(torch.bfloat16).float()
    return (x - y).to(torch.bfloat16).double()


def topk(logits: torch.Tensor, k: int):
    """p = bf16(softmax(logits)) and the k largest p per row, equal p by lower token id: (p [B, V], top p [B, k + 1], ids [B, k + 1])."""
    p = bf(torch.softmax(logits.double(), dim=-1))
    vals, idx = torch.sort(p, dim=1, descending=True, stable=True)
    return p, vals[:, :k + 1], idx[:, :k + 1]


def contrastive_generate(sd, cfg, input_ids, attention_mask, cand_vis=None, hist_vis=None, obj_vis=None, penalty_alpha=0.6, top_k=4,
                         max_new_tokens=20, eos_token_id=2, pad_token_id=0, stop_on_eos=True, return_steps=False, **proc):
    """4.28 contrastive search.  ``proc``: the processors of tests/processors_oracle.py on the bf16 logits.  With ``return_steps``
    also returns per step a dict: ``score`` [B, k] sorted descending, ``pk`` / ``pk1`` [B] the k-th and (k+1)-th largest p,
    ``lk`` / ``lk1`` [B] their (processed) logits."""
    B, S = input_ids.shape
    k = top_k
    mask = attention_mask.clone()
    past: list = [None] * cfg.n_layers
    pos = (mask.long().cumsum(-1) - 1).masked_fill(mask == 0, 1)
    out = O.modified_lm_forward(sd, cfg, input_ids, mask, cand_vis=cand_vis, hist_vis=hist_vis, obj_vis=obj_vis, position_ids=pos,
                                past_kv=past)
    ctx = [normalize(out["hidden_states"][b][mask[b].bool()]) for b in range(B)]
    logits = out["logits"][:, -1]
    ids = input_ids.clone()
    unfinished = torch.ones(B, dtype=torch.bool)
    steps = []
    for _ in range(max_new_tokens):
        if proc:
            logits = PO.process(logits, ids, S, eos_token_id=eos_token_id, **proc)
        logits_in = logits
        _, vals, idx = topk(logits, k)
        cand_ids = idx[:, :k]
        past_k = [(kk.repeat_interleave(k, 0), vv.repeat_interleave(k, 0)) for kk, vv in past]
        mask_k = torch.cat([mask, mask.new_ones(B, 1)], dim=1).repeat_interleave(k, 0)
        pos_k = (mask_k.long().cumsum(-1) - 1)[:, -1:]
        co = O.modified_lm_forward(sd, cfg, cand_ids.reshape(-1, 1), mask_k, position_ids=pos_k, past_kv=past_k)
        h = co["hidden_states"][:, 0]
        sel, scores = [], []
        for b in range(B):
            cand_hat = normalize(h[b * k:(b + 1) * k])
            j, _, score = ranking_fast(ctx[b], cand_hat, vals[b, :k], penalty_alpha)
            ctx[b] = torch.cat([ctx[b], cand_hat[j:j + 1]], dim=0)
            sel.append(j)
            scores.append(torch.sort(score, descending=True).values)
        sel = torch.tensor(sel)
        rows = torch.arange(B) * k + sel
        tok = cand_ids[torch.arange(B), sel]
        tok = torch.where(unfinished, tok, torch.full_like(tok, pad_token_id))
        ids = torch.cat([ids, tok[:, None]], dim=1)
        past = [(kk[rows], vv[rows]) for kk, vv in past_k]
        mask = torch.cat([mask, mask.new_ones(B, 1)], dim=1)
        logits = co["logits"][rows, 0]
        lg = logits_in.double().gather(1, idx[:, k - 1:k + 1])
        steps.append({"score": torch.stack(scores), "pk": vals[:, k - 1], "pk1": vals[:, k], "lk": lg[:, 0], "lk1": lg[:, 1]})
        if stop_on_eos:
            unfinished = unfinished & (tok != eos_token_id)
            if not bool(unfinished.any()):
                break
    return (ids, steps) if return_steps else ids


def near_tie(step: dict, b: int, ulps: int = 1) -> bool:
    """Prompt b's decision at this step lies inside the bf16 noise floor: its two best scores within ``ulps`` bf16 ulp, or the
    k-th and (k+1)-th candidate (which tokens are candidates) within ``ulps`` ulp of their p or of their logits: a logit one
    ulp off moves p by several of its ulps."""
    def close(x, y):
        ulp = 2.0 ** (np.floor(np.log2(max(abs(x), abs(y), 1e-30))) - 7)
        return abs(x - y) <= ulps * ulp
    sc = step["score"][b].tolist()
    return ((len(sc) > 1 and close(sc[0], sc[1])) or close(float(step["pk"][b]), float(step["pk1"][b]))
            or close(float(step["lk"][b]), float(step["lk1"][b])))


def near_tie_ok(ids: torch.Tensor, ref: torch.Tensor, steps: list, S: int, tag: str = "", ulps: int = 1) -> list:
    """Per prompt: the rows are equal, or they first differ at generated column c and the oracle's decision at some step <= c was
    a near tie (``near_tie`` within ``ulps``).  Returns the matched generated columns per prompt."""
    matched = []
    for b in range(ids.shape[0]):
        L = min(ids.shape[1], ref.shape[1])
        diff = (ids[b, :L] != ref[b, :L]).nonzero()
        if ids.shape[1] == ref.shape[1] and not len(diff):
            matched.append(L - S)
            continue
        first = (int(diff[0]) if len(diff) else L) - S
        matched.append(first)
        assert any(near_tie(steps[t], b, ulps) for t in range(min(first + 1, len(steps)))), \
            (tag, b, first, ids[b, S:].tolist(), ref[b, S:].tolist(), {n: v[b].tolist() for n, v in steps[min(first, len(steps) - 1)].items()})
    return matched


def follow_path(sd, cfg, input_ids, attention_mask, path, cand_vis=None, hist_vis=None, obj_vis=None, penalty_alpha=0.6, top_k=4,
                eos_token_id=2, pad_token_id=0, stop_on_eos=True, ulps=3, strict=True, **proc):
    """Teacher-forced check of a generated ``path`` [B, S + n] (prompt ids, then n tokens): every step runs 4.28 contrastive
    search from the path's own prefix, and the path's token must be the restatement's choice or lie inside that step's bf16 noise
    floor.  The candidates the path's run surely had are the k best whose logit is not within ``ulps`` bf16 ulp of the k-th (a
    logit that close may have fallen on either side of the boundary).  An excused token is a candidate, or a token outside the k
    whose logit is within ``ulps`` ulp of the k-th (then run as one extra candidate), whose score is within ``ulps`` ulp of the
    best surely-present score or above it.  Rows are not checked after their EOS (they emit pad, and the device keeps its own
    candidate's state, which no output shows).  Returns (exact, excused, outside) counts over the checked steps; ``strict``
    asserts that no step is outside the rule, otherwise such steps are counted (the path's token is followed either way)."""
    def ulp(x):
        return 2.0 ** (np.floor(np.log2(max(abs(x), 1e-30))) - 7)
    B, S = input_ids.shape
    k, k1, n = top_k, top_k + 1, path.shape[1] - S
    mask = attention_mask.clone()
    past: list = [None] * cfg.n_layers
    pos = (mask.long().cumsum(-1) - 1).masked_fill(mask == 0, 1)
    out = O.modified_lm_forward(sd, cfg, input_ids, mask, cand_vis=cand_vis, hist_vis=hist_vis, obj_vis=obj_vis, position_ids=pos,
                                past_kv=past)
    ctx = [normalize(out["hidden_states"][b][mask[b].bool()]) for b in range(B)]
    logits = out["logits"][:, -1]
    ids = input_ids.clone()
    live = [True] * B
    exact = excused = outside_rule = 0
    for t in range(n):
        if proc:
            logits = PO.process(logits, ids, S, eos_token_id=eos_token_id, **proc)
        p, _, idx = topk(logits, k)
        d = path[:, S + t]
        outside = torch.tensor([live[b] and int(d[b]) not in idx[b, :k].tolist() for b in range(B)])
        cand = torch.cat([idx[:, :k], torch.where(outside, d, idx[:, k])[:, None]], dim=1)          # [B, k + 1]
        past_k = [(kk.repeat_interleave(k1, 0), vv.repeat_interleave(k1, 0)) for kk, vv in past]
        mask_k = torch.cat([mask, mask.new_ones(B, 1)], dim=1).repeat_interleave(k1, 0)
        pos_k = (mask_k.long().cumsum(-1) - 1)[:, -1:]
        co = O.modified_lm_forward(sd, cfg, cand.reshape(-1, 1), mask_k, position_ids=pos_k, past_kv=past_k)
        h = co["hidden_states"][:, 0]
        commit = []
        for b in range(B):
            cand_hat = normalize(h[b * k1:(b + 1) * k1])
            _, _, score = ranking_fast(ctx[b], cand_hat, p[b, cand[b]], penalty_alpha)
            best = int(torch.argmax(score[:k]))
            j = best
            if live[b]:
                lg = logits[b].double()
                lk = float(lg[idx[b, k - 1]])
                near = lambda tok: abs(float(lg[tok]) - lk) <= ulps * ulp(lk)
                j = k if bool(outside[b]) else cand[b, :k].tolist().index(int(d[b]))
                if j == best:
                    exact += 1
                else:
                    sure = [float(score[i]) for i in range(k) if not near(int(cand[b, i]))]
                    bar = max(sure) if sure else float("-inf")
                    ok = (j < k or near(int(d[b]))) and float(score[j]) >= bar - ulps * ulp(bar)
                    assert ok or not strict, (t, b, int(d[b]), cand[b].tolist(), score.tolist(), [float(lg[c]) for c in cand[b]])
                    excused += ok
                    outside_rule += not ok
            ctx[b] = torch.cat([ctx[b], cand_hat[j:j + 1]], dim=0)
            commit.append(b * k1 + j)
        rows = torch.tensor(commit)
        ids = torch.cat([ids, d[:, None]], dim=1)
        past = [(kk[rows], vv[rows]) for kk, vv in past_k]
        mask = torch.cat([mask, mask.new_ones(B, 1)], dim=1)
        logits = co["logits"][rows, 0]
        if stop_on_eos:
            live = [live[b] and int(d[b]) != eos_token_id for b in range(B)]
    return exact, excused, outside_rule
