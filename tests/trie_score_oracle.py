"""CPU restatement of answer scoring (``ModifiedLlamaForCausalLM.score_answers``).  *** TEST INFRASTRUCTURE ONLY *** (the
product never imports it).

The answers are read off the trie itself (``child.items()``, never indexing, so the reference's ``defaultdict`` does not grow):
every path from ``trie.root`` to a childless node, in DFS preorder with children by ascending token id; a root without
children gives one empty answer.  Each answer is teacher-forced token by token: the log-probs come from the logits after the
prompt and each prefix of the answer, in the logits' dtype as ``tests/trie_beam_oracle.search`` computes them
(``log_softmax`` in fp32, rounded once to the logits' dtype; NaN becomes -inf), and are folded in fp32, s = lp + s, root to
leaf and then EOS: the running score a beam following that path carries.  ``score`` divides by (S + d) ** length_penalty in
Python floats, as ``BeamHypotheses.add`` does; ``best`` is the first maximum.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def answers(trie) -> list:
    """The answers' token lists in DFS preorder, children by ascending token id."""
    out = []

    def visit(node, path):
        kids = sorted(node.child.items(), key=lambda e: e[0])
        if not kids:
            out.append(list(path))
        for tok, ch in kids:
            visit(ch, path + [int(tok)])
    visit(trie.root, [])
    return out


def log_probs(logits: torch.Tensor) -> torch.Tensor:
    """[V] logits -> [V] log-probs in the logits' dtype (``trie_beam_oracle.search``'s rule), NaN -> -inf, as fp32."""
    lp = F.log_softmax(logits.float(), dim=-1).to(logits.dtype).float()
    return torch.where(torch.isnan(lp), torch.full_like(lp, float("-inf")), lp)


def score(logits_fn, B: int, S: int, trie, length_penalty: float = 1.0):
    """``logits_fn(b, toks)``: the [V] next-token logits of prompt b followed by the answer tokens ``toks`` (special ids -inf).
    Returns (answers, logprob fp32 [B, A], score fp64 [B, A], best int64 [B])."""
    ans = answers(trie)
    lp = torch.empty((B, len(ans)), dtype=torch.float32)
    for b in range(B):
        for a, toks in enumerate(ans):
            s = torch.zeros((), dtype=torch.float32)
            for i, t in enumerate(toks + [trie.eos]):
                s = log_probs(logits_fn(b, toks[:i]))[t] + s
            lp[b, a] = s
    norm = torch.tensor([(S + len(t)) ** length_penalty for t in ans], dtype=torch.float64)
    sc = lp.to(torch.float64) / norm
    return ans, lp, sc, sc.argmax(dim=1)
