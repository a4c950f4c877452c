"""Trie-constrained decoding: the host processor of the reference and the flattened (CSR) table of the device path.

The reference constrains EQA answers with a ``Trie`` (tools/trie.py: ``root``, nodes with a ``child`` defaultdict,
``eos``, ``get_child_index``, ``get_next_node``) walked by ``TrieLogitsProcessor`` (models/modified_lm.py:10-30) on every
token.  ``generate(trie=...)`` runs that walk on the device (``nv_trie_mask``) from the table ``flatten_trie`` builds; a
trie it cannot flatten faithfully, and every miss the kernel reports, go through ``TrieLogitsProcessor`` below instead.
"""
from __future__ import annotations

from typing import List, Optional

import numpy as np
import torch


class TrieLogitsProcessor:
    """models/modified_lm.py:10-30: per-row walk of a trie; every token that is not allowed at the row's node is masked to
    -inf.  Like the reference it steps through ``trie.get_next_node``, so a token that is not a child inserts an empty
    node into the reference's defaultdict (which changes what later rows are allowed)."""

    def __init__(self, trie):
        self.node_states = None
        self.trie = trie

    def __call__(self, input_ids: torch.Tensor, scores: torch.Tensor) -> torch.Tensor:
        batch_size = input_ids.shape[0]
        if self.node_states is None:
            self.node_states = [self.trie.root for _ in range(batch_size)]
        else:
            for bn in range(batch_size):
                self.node_states[bn] = self.trie.get_next_node(self.node_states[bn], input_ids[bn, -1].item())
        masks = torch.zeros_like(scores, dtype=torch.bool)
        for bn in range(batch_size):
            masks[bn][self.trie.get_child_index(self.node_states[bn])] = True
        return scores.masked_fill(~masks, float("-inf"))


class TrieTable:
    """A trie in CSR form: node i's children are edges ptr[i] .. ptr[i+1] (tokens ascending); node 0 is the root."""

    def __init__(self, ptr: List[int], toks: List[int], kids: List[int], eos: int):
        self.ptr, self.toks, self.kids, self.eos = ptr, toks, kids, eos
        self.n_nodes, self.n_edges = len(ptr) - 1, len(toks)

    def pack(self, node_cap: int, edge_cap: int) -> np.ndarray:
        """int32 [node_cap + 2 + 2 * edge_cap] = node_ptr | child_tok | child_node for a kernel call with n_nodes =
        node_cap: nodes n_nodes .. node_cap (the dead node included) have no children and are unreachable but for misses."""
        assert node_cap >= self.n_nodes and edge_cap >= self.n_edges
        host = np.zeros(node_cap + 2 + 2 * edge_cap, dtype=np.int32)
        host[:node_cap + 2] = self.n_edges
        host[:self.n_nodes + 1] = self.ptr
        o = node_cap + 2
        host[o:o + self.n_edges] = self.toks
        host[o + edge_cap:o + edge_cap + self.n_edges] = self.kids
        return host


def _token(t, V: int) -> Optional[int]:
    if isinstance(t, (bool, np.bool_)) or not isinstance(t, (int, np.integer)):
        return None
    t = int(t)
    return t if 0 <= t < V else None


def flatten_trie(trie, V: int) -> Optional[TrieTable]:
    """The CSR table of ``trie``, or None when the device walk could differ from the host processor's: the object lacks
    ``root`` / ``eos`` / a node's ``child`` mapping, a token id lies outside [0, V), or a node's ``get_child_index`` or an
    edge's ``get_next_node`` disagrees with its ``child`` mapping (a subclass with other rules).  Reads the trie through
    ``child.items()`` only (indexing the reference's defaultdict would insert nodes): the trie is not modified."""
    try:
        root, eos = trie.root, trie.eos
    except AttributeError:
        return None
    eos = _token(eos, V)
    if eos is None:
        return None
    index = {id(root): 0}
    nodes, ptr, toks, kids = [root], [0], [], []
    i = 0
    while i < len(nodes):
        node = nodes[i]
        i += 1
        try:
            items = list(node.child.items())
        except AttributeError:
            return None
        edges = []
        for t, ch in items:
            tok = _token(t, V)
            if tok is None:
                return None
            edges.append((tok, ch))
        edges.sort(key=lambda e: e[0])
        allowed = [tok for tok, _ in edges] or [eos]
        try:
            if set(trie.get_child_index(node)) != set(allowed):
                return None
            if any(trie.get_next_node(node, tok) is not ch for tok, ch in edges):
                return None
        except Exception:
            return None
        for tok, ch in edges:
            j = index.get(id(ch))
            if j is None:
                j = index[id(ch)] = len(nodes)
                nodes.append(ch)
            toks.append(tok)
            kids.append(j)
        ptr.append(len(toks))
    return TrieTable(ptr, toks, kids, eos)


class TreeRows:
    """The non-root nodes of a flattened trie as the rows of one tree-masked forward (``tree_rows``), in DFS preorder with
    children by ascending token id.  Row i holds ``tok[i]`` at ``depth[i]`` (1 for a child of the root) under ``parent[i]``
    (-1: the root), and ``end[i]`` is the first row after its subtree, so row j is an ancestor-or-self of row i iff
    j <= i < end[j].  An answer is a path from the root to a childless node: ``answers[a]`` its tokens, ``paths[a]`` its rows
    (root to leaf), ``leaves[a]`` its last row (-1 for the one empty answer of a root without children).  ``eos`` ends every
    answer.  Arrays are int32 numpy arrays of length ``n`` = N'."""

    def __init__(self, tok, depth, parent, end, paths, eos: int):
        self.tok, self.depth, self.parent, self.end = (np.asarray(a, dtype=np.int32) for a in (tok, depth, parent, end))
        self.n = len(self.tok)
        self.paths = paths
        self.leaves = [p[-1] if p else -1 for p in paths]
        self.answers = [[int(self.tok[r]) for r in p] for p in paths]
        self.eos = eos

    @property
    def max_depth(self) -> int:
        return int(self.depth.max()) if self.n else 0


def tree_rows(table: TrieTable) -> Optional[TreeRows]:
    """The tree rows of ``table`` (``TreeRows``), or None when a node is reachable from two parents (``flatten_trie`` keeps
    one node per child object, so a trie whose child objects are shared, or a cycle, is not a tree)."""
    seen = np.zeros(table.n_nodes, dtype=np.int64)
    for k in table.kids:
        seen[k] += 1
    if table.n_nodes and (seen[0] or (seen > 1).any()):
        return None
    tok, depth, parent, end, paths = [], [], [], [], []
    # iterative preorder: a frame is (node, its row, the next edge to visit)
    stack = [(0, -1, table.ptr[0])]
    path = []
    while stack:
        node, row, e = stack[-1]
        if e == table.ptr[node + 1]:
            stack.pop()
            if row >= 0:
                end[row] = len(tok)
                path.pop()
            continue
        stack[-1] = (node, row, e + 1)
        kid = table.kids[e]
        r = len(tok)
        tok.append(table.toks[e])
        depth.append(len(path) + 1)
        parent.append(row)
        end.append(0)
        path.append(r)
        if table.ptr[kid + 1] == table.ptr[kid]:
            paths.append(list(path))
        stack.append((kid, r, table.ptr[kid]))
    if not tok:
        paths = [[]]
    return TreeRows(tok, depth, parent, end, paths, table.eos)
