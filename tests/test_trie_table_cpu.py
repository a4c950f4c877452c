"""Host side of trie-constrained decoding (navillm_b200/trie.py): the CSR table the device walk reads, the checks that route a
trie to the host processor instead, and the host processor against the oracle's restatement of models/modified_lm.py:10-30.

``ref_trie_mask`` is a plain-Python restatement of ``nv_trie_mask`` on a packed table; tests/test_trie_decode_gpu.py holds the
kernel to it bit for bit.  Here it is checked against the trie's own walk, which pins the table and the restatement together."""
import copy
import random
from collections import defaultdict

import numpy as np
import pytest
import torch

from navillm_b200.trie import TrieLogitsProcessor, flatten_trie

V = 32006
BOS, EOS = 1, 2
SPECIAL = [32000, 32001, 32002, 32003, 32004]


class TreeNode:
    def __init__(self):
        self.child = defaultdict(TreeNode)


class Trie:
    """The interface of the reference's tools/trie.py."""

    def __init__(self, bos, eos):
        self.root, self.bos, self.eos = TreeNode(), bos, eos

    def insert(self, word):
        cur = self.root
        for c in word:
            cur = cur.child[c]

    def get_child_index(self, cur):
        return [self.eos] if len(cur.child) == 0 else list(cur.child.keys())

    def get_next_node(self, cur, w):
        return cur if len(cur.child) == 0 else cur.child[w]


def make_trie(words, eos=EOS):
    t = Trie(BOS, eos)
    for w in words:
        t.insert(w)
    return t


def structure(node, seen=None):
    """The trie below ``node`` as nested sorted tuples (read through items(): no insertion)."""
    return tuple(sorted((tok, structure(ch)) for tok, ch in node.child.items()))


def unpack(table, node_cap=None, edge_cap=None):
    """(node_ptr, child_tok, child_node, n_nodes) of the packed int32 array the device buffers hold."""
    node_cap = table.n_nodes if node_cap is None else node_cap
    edge_cap = max(table.n_edges, 1) if edge_cap is None else edge_cap
    host = table.pack(node_cap, edge_cap)
    o = node_cap + 2
    return host[:o].tolist(), host[o:o + edge_cap].tolist(), host[o + edge_cap:].tolist(), node_cap


def ref_trie_mask(logits, csr, leaf_tok, special, state, last):
    """nv_trie_mask restated: logits [B, V] bf16 (CPU); state: list of node ids, updated in place; last: list or None.
    Returns (out [B, V] bf16, miss)."""
    node_ptr, child_tok, child_node, n_nodes = csr
    B, Vr = logits.shape
    out = torch.full((B, Vr), float("-inf"), dtype=torch.bfloat16)
    miss = 0
    sp = set(special)
    for b in range(B):
        node = state[b]
        e0, e1 = node_ptr[node], node_ptr[node + 1]
        if last is not None and e1 > e0:
            hit = [e for e in range(e0, e1) if child_tok[e] == last[b]]
            if hit:
                node = child_node[hit[0]]
            else:
                node, miss = n_nodes, 1
            state[b] = node
        e0, e1 = node_ptr[node], node_ptr[node + 1]
        allowed = child_tok[e0:e1] or [leaf_tok]
        vals = logits[b, allowed]
        out[b, allowed] = vals
        f = vals.float()
        live = any(bool(v > float("-inf")) and a not in sp for a, v in zip(allowed, f))
        if bool(torch.isnan(f).any()) or not live:
            miss = 1
            c = next((a for a in allowed if a not in sp), None)
            if c is None:
                c = next((c for c in range(Vr) if c not in sp), Vr)
            if c < Vr:
                out[b, c] = 0.0
    return out, miss


def _tries():
    rng = random.Random(0)
    wide = [[BOS, t] for t in range(100, 100 + 4200)]                       # a node with > 4096 children
    return {
        "prefixes": [[11, 12, 13], [11, 12], [11, 12, 40, 41], [11], [60, 61, 62]],
        "single_token": [[5], [9], [31999], [0]],
        "bos_prefixed": [[BOS, 7, 8], [BOS, 7, 9, 10], [BOS, 3]],
        "wide": wide + [[BOS, 100, 5]],
        "eos_child": [[11, EOS], [11, 12, EOS], [20, EOS, 21]],
        "random": [[rng.randrange(V - 10) for _ in range(rng.randint(1, 4))] for _ in range(300)],
    }


def _walk_check(trie, table, rng, n_walks=50):
    """Random walks through allowed tokens: the CSR walk and the trie's own walk allow the same tokens at every step."""
    node_ptr, child_tok, child_node, _ = unpack(table)
    for _ in range(n_walks):
        node, idx = trie.root, 0
        for _ in range(6):
            allowed = trie.get_child_index(node)
            e0, e1 = node_ptr[idx], node_ptr[idx + 1]
            assert child_tok[e0:e1] == sorted(child_tok[e0:e1])
            assert sorted(child_tok[e0:e1] or [table.eos]) == sorted(allowed)
            tok = rng.choice(allowed)
            if e1 > e0:
                idx = child_node[e0 + child_tok[e0:e1].index(tok)]
            node = trie.get_next_node(node, tok)


@pytest.mark.parametrize("name", list(_tries()))
def test_flatten_matches_the_trie_and_leaves_it_unchanged(name):
    words = _tries()[name]
    trie = make_trie(words)
    before = structure(trie.root)
    table = flatten_trie(trie, V)
    assert table is not None
    assert structure(trie.root) == before
    assert table.n_edges == table.n_nodes - 1                                # a tree: one edge into every node but the root
    assert table.ptr[0] == 0 and table.ptr[-1] == table.n_edges and all(a <= b for a, b in zip(table.ptr, table.ptr[1:]))
    _walk_check(trie, table, random.Random(1))
    assert structure(trie.root) == before
    if name == "wide":
        assert max(b - a for a, b in zip(table.ptr, table.ptr[1:])) >= 4096


def test_pack_pads_to_the_capacities_with_childless_nodes():
    table = flatten_trie(make_trie([[11, 12], [13]]), V)
    node_ptr, child_tok, child_node, n = unpack(table, 8, 4)
    assert n == 8 and len(node_ptr) == 10 and len(child_tok) == 4 and len(child_node) == 4
    assert node_ptr[table.n_nodes:] == [table.n_edges] * (10 - table.n_nodes)  # unused nodes and the dead node 8: no children
    assert child_tok[:3] == [11, 13, 12]


class _OtherChildren(Trie):
    def get_child_index(self, cur):
        return [self.eos] if len(cur.child) == 0 else list(cur.child.keys())[:1]


class _OtherNext(Trie):
    def get_next_node(self, cur, w):
        return self.root


def test_validation_failures_route_to_the_host():
    words = [[11, 12], [11, 13], [14]]
    assert flatten_trie(make_trie(words), V) is not None
    for cls in (_OtherChildren, _OtherNext):
        t = cls(BOS, EOS)
        for w in words:
            t.insert(w)
        assert flatten_trie(t, V) is None, cls.__name__
    no_root = make_trie(words)
    del no_root.root
    assert flatten_trie(no_root, V) is None
    no_eos = make_trie(words)
    del no_eos.eos
    assert flatten_trie(no_eos, V) is None
    bad_node = make_trie(words)
    bad_node.root.child[11].child[12] = object()                            # a node without `child`
    assert flatten_trie(bad_node, V) is None
    assert flatten_trie(make_trie(words + [[11, V]]), V) is None              # token id >= V
    assert flatten_trie(make_trie(words + [[-1]]), V) is None
    assert flatten_trie(make_trie(words, eos=V), V) is None                  # eos outside the vocabulary


def _random_walk_ids(rng, trie, B, steps, p_off=0.1):
    """Token columns of a batch walking the trie; with probability p_off a token that is not allowed (a miss)."""
    nodes = [trie.root] * B
    cols = []
    for _ in range(steps):
        col = []
        for b in range(B):
            allowed = trie.get_child_index(nodes[b])
            tok = rng.randrange(V) if rng.random() < p_off else rng.choice(allowed)
            col.append(tok)
            nodes[b] = nodes[b] if len(nodes[b].child) == 0 else nodes[b].child.get(tok, nodes[b])
        cols.append(col)
    return cols


def test_host_processor_matches_the_oracle_on_random_walks():
    from oracle.navillm_oracle import TrieLogitsProcessor as OracleProc
    rng = random.Random(3)
    for words in (_tries()["prefixes"], _tries()["random"], _tries()["eos_child"]):
        t_mine, t_orc = make_trie(words), make_trie(words)
        mine, orc = TrieLogitsProcessor(t_mine), OracleProc(t_orc)
        B = 5
        ids = torch.randint(0, V, (B, 4))
        cols = _random_walk_ids(rng, make_trie(words), B, 8)
        for step in range(8):
            scores = torch.randn(B, V, generator=torch.Generator().manual_seed(step))
            a, b = mine(ids, scores.clone()), orc(ids, scores.clone())
            assert torch.equal(a, b)
            ids = torch.cat([ids, torch.tensor(cols[step])[:, None]], 1)
        assert structure(t_mine.root) == structure(t_orc.root)               # the same defaultdict insertions on misses


def test_restated_kernel_follows_the_host_processor():
    """ref_trie_mask on the packed table gives the processor's mask (specials left to the pick) while no miss occurs, and
    reports a miss exactly when a step leaves the trie."""
    rng = random.Random(5)
    words = _tries()["prefixes"] + _tries()["bos_prefixed"] + _tries()["eos_child"]
    trie = make_trie(words)
    table = flatten_trie(trie, V)
    csr = unpack(table, 64, 64)
    B = 6
    proc = TrieLogitsProcessor(copy.deepcopy(trie))
    cols = _random_walk_ids(rng, trie, B, 6, p_off=0.0)
    state, last = [0] * B, None
    ids = torch.zeros(B, 1, dtype=torch.long)
    for step in range(6):
        logits = torch.randn(B, V, generator=torch.Generator().manual_seed(10 + step)).to(torch.bfloat16)
        out, miss = ref_trie_mask(logits, csr, table.eos, SPECIAL, state, last)
        want = proc(ids, logits.float())
        assert miss == 0
        assert torch.equal(out.float(), want)
        last = cols[step]
        ids = torch.cat([ids, torch.tensor(last)[:, None]], 1)
    state2 = [0] * B
    ref_trie_mask(logits, csr, table.eos, SPECIAL, state2, None)
    _, miss = ref_trie_mask(logits, csr, table.eos, SPECIAL, state2, [31990] * B)  # not a child of the root
    assert miss == 1 and state2 == [64] * B
