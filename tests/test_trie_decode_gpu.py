"""Trie-constrained and sampled generate() on the device.

``nv_trie_mask`` is held bit for bit (``out`` and ``state``; ``miss`` exactly) to the restatement in
tests/test_trie_table_cpu.py.  ``generate(trie=t)`` - device walk, eager and through the CUDA graph - must return exactly the
ids of the host path, ``generate(logits_processor=[oracle TrieLogitsProcessor(deepcopy(t))])``, and sampled generation through
the graph exactly the ids of the eager loop under the same seed."""
import copy
import random
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from tests.test_trie_table_cpu import SPECIAL, V, make_trie, ref_trie_mask, structure, unpack  # noqa: E402

bf16 = torch.bfloat16


def _csr_dev(csr, dev):
    node_ptr, child_tok, child_node, n = csr
    return [torch.tensor(x, dtype=torch.int32, device=dev) for x in (node_ptr, child_tok, child_node)] + [n]


def _run_kernel(dev, logits, csr, leaf, state, last, ldo=None):
    from navillm_b200 import ops
    B, Vr = logits.shape
    ldo = ldo or (Vr + 63) // 64 * 64
    out_full = torch.full((B, ldo), 7.0, dtype=bf16, device=dev)            # canary past V
    out = out_full[:, :Vr]
    st = torch.tensor(state, dtype=torch.int32, device=dev)
    miss = torch.zeros(1, dtype=torch.int32, device=dev)
    sp = torch.tensor(SPECIAL, dtype=torch.int32, device=dev)
    lt = None if last is None else torch.tensor(last, dtype=torch.int32, device=dev)
    ops.trie_mask(logits, out, *_csr_dev(csr, dev), leaf, sp, st, lt, miss)
    torch.cuda.synchronize()
    assert bool((out_full[:, Vr:] == 7.0).all()), "wrote past V"
    return out.cpu(), st.cpu().tolist(), int(miss.item())


@pytest.mark.parametrize("B", [1, 3, 8, 64])
def test_trie_mask_matches_restatement(cuda_dev, B):
    from tests.test_trie_table_cpu import flatten_trie
    rng = random.Random(B)
    words = [[rng.randrange(V) for _ in range(rng.randint(1, 4))] for _ in range(200)] + [[7, t] for t in range(1000, 6000)]
    words += [[SPECIAL[0]], [SPECIAL[1], 5]]
    trie = make_trie(words)
    table = flatten_trie(trie, V)
    csr = unpack(table, 1 << (table.n_nodes - 1).bit_length(), table.n_edges)
    n = csr[3]
    gen = torch.Generator().manual_seed(B)
    for ld in (V + 26, 32064):                                               # ld != ldo and ld == ldo
        base = torch.randn(B, ld, generator=gen).to(bf16)
        logits = base.to(cuda_dev)[:, :V]
        # rows at the root, inside, at leaves, at the dead node, with last = None / a child / a missing child
        state = [rng.choice([0, 0, n, rng.randrange(table.n_nodes)]) for _ in range(B)]
        for last in (None, "child", "miss"):
            if last is None:
                lt = None
            else:
                lt = []
                for b in range(B):
                    e0, e1 = csr[0][state[b]], csr[0][state[b] + 1]
                    if last == "child" and e1 > e0:
                        lt.append(csr[1][rng.randrange(e0, e1)])
                    else:
                        lt.append(rng.randrange(V) if last == "miss" else 3)
            want_state = list(state)
            want, want_miss = ref_trie_mask(base[:, :V], csr, table.eos, SPECIAL, want_state, lt)
            out, got_state, got_miss = _run_kernel(cuda_dev, logits, csr, table.eos, state, lt)
            assert torch.equal(out.view(torch.int16), want.view(torch.int16)), (ld, last)
            assert got_state == want_state and got_miss == want_miss, (ld, last)


def test_trie_mask_degenerate_rows(cuda_dev):
    """All allowed children special, all allowed -inf, and an allowed NaN: miss, and 0.0 where the pick stays in [0, V)."""
    from tests.test_trie_table_cpu import flatten_trie
    trie = make_trie([[SPECIAL[0]], [SPECIAL[1]], [11, 12], [11, 13], [20, 21]])
    table = flatten_trie(trie, V)
    csr = unpack(table)
    root_kids = dict(zip(csr[1][csr[0][0]:csr[0][1]], csr[2][csr[0][0]:csr[0][1]]))
    n11, n20 = root_kids[11], root_kids[20]
    base = torch.randn(4, V, generator=torch.Generator().manual_seed(0)).to(bf16)
    base[1, [12, 13]] = float("-inf")
    base[2, 13] = float("nan")
    for rows, state in (([0], [0]), ([1], [n11]), ([2], [n11]), ([3], [n20])):
        lg = base[rows]
        want_state = list(state)
        want, want_miss = ref_trie_mask(lg, csr, table.eos, SPECIAL, want_state, None)
        out, got_state, got_miss = _run_kernel(cuda_dev, lg.to(cuda_dev), csr, table.eos, state, None)
        assert torch.equal(out.view(torch.int16), want.view(torch.int16)) and got_miss == want_miss, rows
        assert got_miss == (1 if rows in ([1], [2]) else 0), rows             # the root has live children 11 and 20
    # a root whose only children are special: degenerate, 0.0 at the first non-special column
    only_special = flatten_trie(make_trie([[SPECIAL[0]], [SPECIAL[2]]]), V)
    out, _, miss = _run_kernel(cuda_dev, base[:1].to(cuda_dev), unpack(only_special), only_special.eos, [0], None)
    assert miss == 1 and float(out[0, 0]) == 0.0


def test_trie_mask_bad_arguments(cuda_dev):
    from navillm_b200 import _lib, ops
    from tests.test_trie_table_cpu import flatten_trie
    table = flatten_trie(make_trie([[11, 12]]), V)
    node_ptr, child_tok, child_node, n = _csr_dev(unpack(table), cuda_dev)
    logits = torch.zeros(2, 64, dtype=bf16, device=cuda_dev)
    out = torch.zeros(2, 64, dtype=bf16, device=cuda_dev)
    st = torch.zeros(2, dtype=torch.int32, device=cuda_dev)
    miss = torch.zeros(1, dtype=torch.int32, device=cuda_dev)
    sp = torch.arange(65, dtype=torch.int32, device=cuda_dev)
    ok = dict(logits=logits, out=out, n_nodes=n, leaf_tok=2, special=sp[:4])
    ops.trie_mask(ok["logits"], ok["out"], node_ptr, child_tok, child_node, n, 2, sp[:4], st, None, miss)
    bad = [dict(out=torch.zeros(2, 68, dtype=bf16, device=cuda_dev)[:, :60], logits=logits[:, :60]),   # ldo % 8 != 0
           dict(n_nodes=0), dict(leaf_tok=64), dict(special=sp), dict(out=out[:, :0], logits=logits[:, :0])]
    for kw in bad:
        a = {**ok, **kw}
        with pytest.raises(_lib.NvError):
            ops.trie_mask(a["logits"], a["out"], node_ptr, child_tok, child_node, a["n_nodes"], a["leaf_tok"], a["special"], st,
                          None, miss)


# ---- generate() ------------------------------------------------------------------------------------------------------------
WORDS = [[11, 12, 13], [11, 12, 40, 41], [11, 50], [60, 61, 62], [11], [70]]


def _golden(cuda_dev):
    from tests.test_navmodel_gpu import build_model
    from tests.test_oracle_golden import load
    g, cfg, tok = load("amp_bf16")
    model, _ = build_model(g, cuda_dev)
    text = tok(g["qa_in"]["prompts"])
    ids = text["input_ids"].clone()
    ids[ids == tok.special["<cand>"]] = 7
    return model, tok, ids, text["attention_mask"]


def _bos_words(tok, words):
    return words + [[tok.bos_token_id] + w for w in words[:3]]


def _tokens(node):
    return [t for t, ch in node.child.items()] + [t for ch in node.child.values() for t in _tokens(ch)]


def _pair(lm, tok, ids, mask, trie, **kw):
    from oracle import navillm_oracle as O
    assert max(_tokens(trie.root)) < lm.lm_head.weight.shape[0]              # the host path indexes its mask with these ids
    common = dict(input_ids=ids, attention_mask=mask, eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id, **kw)
    torch.manual_seed(123)
    host = lm.generate(logits_processor=[O.TrieLogitsProcessor(copy.deepcopy(trie))], **common).cpu()
    stats = {}
    torch.manual_seed(123)
    dev = lm.generate(trie=trie, stats=stats, **common).cpu()
    return host, dev, stats


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("B", [1, 3, 8, 20, 40])
def test_generate_trie_device_matches_host_path(cuda_dev, B, fp8):
    model, tok, ids, mask = _golden(cuda_dev)
    lm = model.lang_model
    if fp8:
        model.quantize_weights_fp8()
    rep = (B + ids.shape[0] - 1) // ids.shape[0]
    ids, mask = ids.repeat(rep, 1)[:B], mask.repeat(rep, 1)[:B]
    trie = make_trie(_bos_words(tok, WORDS), eos=tok.eos_token_id)
    before = structure(trie.root)
    for do_sample in (False, True):
        for stop in (True, False):
            for graph in (False, True):
                kw = dict(max_new_tokens=7, stop_on_eos=stop, use_cuda_graph=graph, do_sample=do_sample, temperature=0.8)
                for _ in range(2 if graph else 1):                       # graph: the capturing call, then a replaying one
                    host, dev, stats = _pair(lm, tok, ids, mask, trie, **kw)
                    assert stats["trie_path"] == "device", kw
                    assert host.shape == dev.shape and torch.equal(host, dev), (kw, host[:, ids.shape[1]:], dev[:, ids.shape[1]:])
                if graph:
                    assert stats["graph_replays"] > 0 or stats["decode_steps"] <= 1
    assert structure(trie.root) == before


def test_generate_trie_fullwidth_two_layers(cuda_dev):
    from tests.test_fullwidth_parity_gpu import _full_navmodel
    model, tok = _full_navmodel(cuda_dev, 32000)
    model = model.to(cuda_dev)
    lm = model.lang_model
    prompts = ["Question : what color is the sofa in the living room ? Answer :", "Question : how many chairs ? Answer :"] * 4
    text = lm.tokenize(prompts)
    rng = random.Random(0)
    words = [[tok.bos_token_id] + [rng.randrange(100, 31000) for _ in range(rng.randint(1, 3))] for _ in range(64)]
    trie = make_trie(words, eos=tok.eos_token_id)
    for do_sample in (False, True):
        host, dev, stats = _pair(lm, tok, text["input_ids"], text["attention_mask"], trie, max_new_tokens=6, do_sample=do_sample)
        host2, dev2, stats2 = _pair(lm, tok, text["input_ids"], text["attention_mask"], trie, max_new_tokens=6, do_sample=do_sample)
        assert stats2["trie_path"] == "device" and stats2["graph_replays"] > 0
        assert torch.equal(host, dev) and torch.equal(host2, dev2)


class _CaptureSpy:
    def __init__(self, monkeypatch):
        self.n = 0
        real = torch.cuda.graph

        def graph(*a, **kw):
            self.n += 1
            return real(*a, **kw)
        monkeypatch.setattr(torch.cuda, "graph", graph)


def test_trie_graph_reuse_and_growth(cuda_dev, monkeypatch):
    model, tok, ids, mask = _golden(cuda_dev)
    lm = model.lang_model
    spy = _CaptureSpy(monkeypatch)
    kw = dict(max_new_tokens=6, stop_on_eos=False)
    t1 = make_trie(WORDS, eos=tok.eos_token_id)
    host, dev, _ = _pair(lm, tok, ids, mask, t1, **kw)
    assert torch.equal(host, dev) and spy.n == 1
    t2 = make_trie([[11, 14, 15], [11, 14, 42, 43], [11, 51], [63, 64, 65], [12], [71]], eos=tok.eos_token_id)   # same shape
    host, dev, stats = _pair(lm, tok, ids, mask, t2, **kw)
    assert torch.equal(host, dev) and spy.n == 1 and stats["graph_replays"] > 0
    big = make_trie(WORDS + [[a, b] for a in range(80, 110) for b in (5, 6)], eos=tok.eos_token_id)        # outgrows the buffers
    host, dev, stats = _pair(lm, tok, ids, mask, big, **kw)
    assert torch.equal(host, dev) and spy.n == 2 and stats["graph_replays"] > 0


def test_forced_miss_falls_back_to_the_host_path(cuda_dev):
    """A special id as the only child of the root: every row is degenerate, the device result is discarded and the host path
    runs on the caller's trie, inserting into it exactly what the host path inserts into a deep copy."""
    model, tok, ids, mask = _golden(cuda_dev)
    lm = model.lang_model
    special = tok.special["<cand>"]
    for do_sample in (False, True):
        for graph in (False, True):
            trie = make_trie([[special, 11], [special, 12, 13]], eos=tok.eos_token_id)
            copy_for_host = copy.deepcopy(trie)
            host, dev, stats = _pair(lm, tok, ids, mask, trie, max_new_tokens=5, do_sample=do_sample, use_cuda_graph=graph,
                                     temperature=0.9)
            assert stats["trie_path"] == "device_miss_host"
            assert torch.equal(host, dev)
            from oracle import navillm_oracle as O
            torch.manual_seed(123)
            lm.generate(input_ids=ids, attention_mask=mask, eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id,
                        max_new_tokens=5, do_sample=do_sample, temperature=0.9, logits_processor=[O.TrieLogitsProcessor(copy_for_host)])
            assert structure(trie.root) == structure(copy_for_host.root)
            assert structure(trie.root) != structure(make_trie([[special, 11], [special, 12, 13]]).root)


@pytest.mark.parametrize("B", [8, 20])
def test_sampled_graph_matches_eager(cuda_dev, B):
    model, tok, ids, mask = _golden(cuda_dev)
    lm = model.lang_model
    rep = (B + ids.shape[0] - 1) // ids.shape[0]
    ids, mask = ids.repeat(rep, 1)[:B], mask.repeat(rep, 1)[:B]
    for top_k in (50, 0):
        for T in (1.0, 0.6):
            outs = {}
            for graph in (False, True, True):
                stats = {}
                torch.manual_seed(9)
                out = lm.generate(input_ids=ids, attention_mask=mask, max_new_tokens=12, stop_on_eos=False, do_sample=True,
                                  temperature=T, top_k=top_k, use_cuda_graph=graph, stats=stats).cpu()
                if graph:
                    assert stats["graph_replays"] > 0
                    assert torch.equal(out, outs[False]), (top_k, T)
                outs[graph] = out


def test_model_modes_take_the_device_path(cuda_dev, monkeypatch):
    from navillm_b200 import ops
    from tests.test_navmodel_gpu import build_model, to_dev
    g = torch.load(ROOT / "tests" / "golden" / "nav_amp_bf16.pt", weights_only=False)
    gen = torch.load(ROOT / "tests" / "golden" / "generate_amp_bf16.pt", weights_only=False)
    model, tok = build_model(g, cuda_dev)
    calls = {"trie_mask": 0, "replay": 0}
    real_mask, real_replay = ops.trie_mask, torch.cuda.CUDAGraph.replay

    def trie_mask(*a, **kw):
        calls["trie_mask"] += 1
        return real_mask(*a, **kw)

    def replay(self):
        calls["replay"] += 1
        return real_replay(self)
    monkeypatch.setattr(ops, "trie_mask", trie_mask)
    monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", replay)
    trie = make_trie(gen["trie_words"], eos=tok.eos_token_id)
    trie.bos = tok.bos_token_id
    out = model("summarization", to_dev(dict(g["sum_in"]), cuda_dev), training=False, trie=trie)["generated_sentences"]
    assert out == gen["trie_sentences"]
    assert calls["trie_mask"] > 0
    r0 = calls["replay"]
    model("3dqa", to_dev(dict(g["qa_in"]), cuda_dev), training=False, max_new_tokens=8, do_sample=True, temperature=0.7)
    assert calls["replay"] > r0
