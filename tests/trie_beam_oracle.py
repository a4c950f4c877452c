"""CPU restatement of trie-constrained beam search: transformers 4.28's ``beam_search`` / ``BeamSearchScorer`` as
tests/beam_oracle.py restates them, with one more processor, 4.28's ``PrefixConstrainedLogitsProcessor``, whose
``prefix_allowed_tokens_fn(b, ids)`` walks a trie statelessly.  *** TEST INFRASTRUCTURE ONLY *** (the product never imports it).

The walk (``walk``): start at ``trie.root`` and follow the beam's generated tokens (the prompt columns excluded) by the rule of
the reference's tools/trie.py ``get_next_node``: a node without children stays where it is; a token that is not a child of a
node with children leads to a childless node (``DEAD``).  The trie is read through ``child.get`` only, so the reference's
``defaultdict`` never grows.  The allowed set is ``get_child_index(node)``: the node's children, or ``[trie.eos]`` at a
childless node.  The processor adds 0 to the allowed scores and -inf to every other one (``scores + mask``), after the
special-token mask, the log-softmax and the processors of tests/processors_oracle.py, and before the fp32 beam-score add.

Two deviations from the reference, both recorded in DESIGN §2: the walk is per beam (the reference's ``TrieLogitsProcessor``
keeps one node per row index, and HF's beam reorder hands a row's node to another beam), and an off-trie token inserts nothing
into the caller's trie.  Equal scores (the -inf candidates of a narrow trie included) order by ascending flat index, the rule
of ``top_candidates``.
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


class _Dead:
    """The childless node an off-trie token leads to."""
    child: dict = {}


DEAD = _Dead()


def walk(trie, tokens):
    """The node a beam reaches from ``trie.root`` by its generated ``tokens``; the trie is not modified."""
    node = trie.root
    for tok in tokens:
        if len(node.child) == 0:
            break
        node = node.child.get(int(tok), DEAD)
    return node


def allowed_tokens(trie, tokens) -> list:
    """``get_child_index`` at the node ``tokens`` reach: its children, or [trie.eos] at a childless node."""
    node = walk(trie, tokens)
    return list(node.child.keys()) if len(node.child) else [trie.eos]


def trie_mask(scores: torch.Tensor, history, trie) -> torch.Tensor:
    """PrefixConstrainedLogitsProcessor: ``scores`` [R, V] (any dtype) + a mask that is 0 at the allowed tokens of row r's
    generated tokens ``history[r]`` and -inf elsewhere."""
    mask = torch.full_like(scores, float("-inf"))
    for r, toks in enumerate(history):
        mask[r, allowed_tokens(trie, toks)] = 0
    return scores + mask


def search(scorer, prompt_ids, trie, num_beams=4, max_new_tokens=20, eos_token_id=2, pad_token_id=0, length_penalty=1.0,
           early_stopping=False, num_return_sequences=1, return_steps=False, **proc):
    """4.28 beam search with the trie processor.  ``scorer(src, last)`` returns the next-token logits [B * K, V] of the beam rows
    (special tokens -inf): at the first step ``src`` and ``last`` are None and row b * K + k holds prompt b's prefill row; later
    ``src`` [B * K] says which row each beam continues and ``last`` [B * K] is its new token.  log_softmax in the logits' dtype
    (fp32 inside, rounded once), the processors of ``proc`` and then the trie mask in that dtype, the fp32 beam-score add.
    Returns [B * n, L] ids (and with ``return_steps`` the per-step [B, 2K + 1] best scores, for near-tie checks)."""
    B, S = prompt_ids.shape
    K = num_beams
    prompt = prompt_ids.repeat_interleave(K, 0)
    beam_scores = torch.zeros((B, K), dtype=torch.float32)
    beam_scores[:, 1:] = -1e9
    beam_scores = beam_scores.view(-1)
    hyps = [BeamHypotheses(K, length_penalty, early_stopping) for _ in range(B)]
    done = [False] * B
    history = [[] for _ in range(B * K)]
    steps = []
    T = 0
    src = last = None
    for t in range(max_new_tokens):
        logits = scorer(src, last)
        lp = F.log_softmax(logits.float(), dim=-1).to(logits.dtype)
        if proc:
            hist_ids = torch.cat([prompt, torch.tensor(history, dtype=torch.int64).view(B * K, t)], dim=1)
            lp = PO.process(lp, hist_ids, S, eos_token_id=eos_token_id, **proc)
        lp = trie_mask(lp, history, trie)
        scores = (lp.float() + beam_scores[:, None]).view(B, -1)
        if return_steps:
            steps.append(torch.sort(scores, dim=1, descending=True, stable=True)[0][:, :2 * K + 1])
        cs, ct, cp = top_candidates(scores, K)
        nsc, ntok, npar = process(hyps, done, S, t, history, cs, ct, cp, eos_token_id, pad_token_id)
        src = (torch.arange(B)[:, None] * K + npar).view(-1)
        last = ntok.view(-1)
        history = [history[int(r)] + [int(tk)] for r, tk in zip(src, last)]
        beam_scores = nsc.view(-1)
        T = t + 1
        if all(done):
            break
    seqs = finalize(hyps, done, S, T, history, beam_scores, num_return_sequences)
    ids = sequences(prompt_ids, seqs, S + max_new_tokens, eos_token_id, pad_token_id)
    return (ids, steps) if return_steps else ids


def trie_beam_generate(sd, cfg, input_ids, attention_mask, trie, cand_vis=None, hist_vis=None, obj_vis=None, num_beams=4, **kw):
    """``search`` on the oracle's ``modified_lm_forward`` with a KV cache: prompt b's prefill and visual tokens reach its K beams
    (the deviation of tests/beam_oracle.py), the cache rows follow ``src``."""
    K = num_beams
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

    return search(scorer, input_ids, trie, num_beams=K, **kw)


def golden_ids(ids: torch.Tensor, S: int, eos: int, pad: int) -> torch.Tensor:
    """Ids recorded under transformers 5.5 as 4.28 writes them: 5.5 fills the columns after a shorter row's EOS with
    ``pad_token_id or eos_token_id`` (EOS when the pad id is 0), 4.28 with the pad id."""
    out = ids.clone()
    for r in range(out.shape[0]):
        hit = (out[r, S:] == eos).nonzero()
        if len(hit):
            out[r, S + int(hit[0]) + 1:] = pad
    return out
