"""Answer scoring on the CPU: ``trie.tree_rows`` against brute-force path enumeration, the CPU restatement
(tests/trie_score_oracle.py) against trie-constrained beam search (tests/trie_beam_oracle.py) on toy scorers, and the new
entry points in the built library."""
import random

import pytest
import torch

from navillm_b200.trie import flatten_trie, tree_rows
from tests import trie_beam_oracle as TB
from tests import trie_score_oracle as TS
from tests.test_trie_beam_cpu import EOS, PAD, Toy, _random_trie
from tests.test_trie_table_cpu import V, make_trie


def _nodes(trie):
    """Brute force: every non-root node as its token path, in DFS preorder with ascending children."""
    out = []

    def visit(node, path):
        for tok, ch in sorted(node.child.items(), key=lambda e: e[0]):
            out.append(path + [tok])
            visit(ch, path + [tok])
    visit(trie.root, [])
    return out


@pytest.mark.parametrize("seed", range(12))
def test_tree_rows_against_path_enumeration(seed):
    rng = random.Random(seed)
    words = [[rng.randrange(3, 40) for _ in range(rng.randint(1, 6))] for _ in range(rng.randint(1, 30))]
    trie = make_trie(words)
    r = tree_rows(flatten_trie(trie, V))
    nodes = _nodes(trie)
    assert r.n == len(nodes)
    assert [int(t) for t in r.tok] == [p[-1] for p in nodes]
    assert [int(d) for d in r.depth] == [len(p) for p in nodes]
    for i, p in enumerate(nodes):
        assert int(r.parent[i]) == (nodes.index(p[:-1]) if len(p) > 1 else -1)
        for j, q in enumerate(nodes):
            ancestor = p[:len(q)] == q
            assert ancestor == (j <= i < int(r.end[j])), (i, j)
    assert r.answers == TS.answers(trie)
    assert [[r.tok[k] for k in path] for path in r.paths] == r.answers
    assert r.leaves == [p[-1] for p in r.paths]
    assert all(int(r.end[l]) == l + 1 for l in r.leaves)                # a leaf's subtree is itself


def test_tree_rows_empty_root_and_prefix_answers():
    r = tree_rows(flatten_trie(make_trie([]), V))
    assert r.n == 0 and r.answers == [[]] and r.paths == [[]] and r.leaves == [-1]
    # [5] is a prefix of [5, 6]: no EOS edge after 5, so it is not an answer
    r = tree_rows(flatten_trie(make_trie([[5, 6], [5], [4]]), V))
    assert r.answers == [[4], [5, 6]]


def test_tree_rows_rejects_shared_nodes():
    trie = make_trie([[5, 6], [7]])
    trie.root.child[8] = trie.root.child[5]                             # one node under two parents
    table = flatten_trie(trie, V)
    assert table is not None and tree_rows(table) is None


@pytest.mark.parametrize("seed", range(8))
def test_oracle_gives_the_top_answers_of_trie_beams_at_length_penalty_0(seed, monkeypatch):
    rng = random.Random(100 + seed)
    Vt = 24
    toy = Toy(Vt, seed, special=[Vt - 1])
    B, S = 3, 4
    prompt = torch.tensor([[rng.randrange(3, Vt - 1) for _ in range(S)] for _ in range(B)])
    K = rng.choice([4, 8])
    trie = _random_trie(rng, Vt - 1, rng.randint(1, K), 4, avoid=(EOS,))
    A = len(TS.answers(trie))
    assert A <= K
    n = rng.randint(1, A)
    longest = max(len(a) for a in TS.answers(trie))

    def logits_fn(b, toks):
        return toy(torch.tensor([prompt[b].tolist() + toks]))[0]
    ans, lp, sc, best = TS.score(logits_fn, B, S, trie, length_penalty=0.0)
    kept = []
    real_finalize = TB.finalize

    def spy(hyps, *a, **k):
        kept.extend([list(h.beams) for h in hyps])
        return real_finalize(hyps, *a, **k)
    monkeypatch.setattr(TB, "finalize", spy)
    ids = TB.search(toy.oracle_scorer(prompt, K), prompt, trie, num_beams=K, max_new_tokens=longest + 1, eos_token_id=EOS,
                    pad_token_id=PAD, length_penalty=0.0, num_return_sequences=n)
    for b in range(B):
        want = sorted(sc[b].tolist(), reverse=True)[:n]
        got = []
        for r in range(n):
            toks = ids[b * n + r, S:].tolist()
            toks = toks[:toks.index(EOS)] if EOS in toks else toks
            got.append(float(sc[b, ans.index(toks)]))
        assert got == want, (b, got, want)
        # each kept hypothesis of a real answer carries the oracle's score, bit for bit (beams 1 .. K - 1 start at -1e9, and
        # their copies of an answer are not the answer's hypothesis)
        for s, toks in kept[b]:
            if toks in ans and s > -1e8:
                assert s == float(sc[b, ans.index(toks)]), (b, toks, s, float(sc[b, ans.index(toks)]))
        assert int(best[b]) == max(range(len(ans)), key=lambda a: (float(sc[b, a]), -a))


def test_oracle_special_ids_and_nan_are_minus_inf():
    trie = make_trie([[3], [4, 5]], eos=EOS)

    def logits_fn(b, toks):
        x = torch.zeros(8)
        x[5] = float("-inf")                                            # a special id inside an answer
        return x
    ans, lp, sc, best = TS.score(logits_fn, 1, 2, trie)
    assert ans == [[3], [4, 5]] and float(lp[0, 1]) == float("-inf") and torch.isfinite(lp[0, 0]) and int(best[0]) == 0


def test_trie_score_entry_points_are_exported():
    from navillm_b200 import _lib
    lib = _lib.load()
    for name in ("nv_attn_fwd_tree", "nv_attn_fwd_tree_fp8", "nv_trie_score"):
        assert hasattr(lib, name), name
