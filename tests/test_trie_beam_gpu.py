"""Trie-constrained beam search on the device (csrc/decode.cu nv_beam_topk_trie, ModifiedLlamaForCausalLM.generate(trie=t,
num_beams=K)): the kernel bit for bit against a CPU restatement, and generate() against tests/trie_beam_oracle.py and the
reference's own generation branch (tests/golden/generate_trie_beam_amp_bf16.pt)."""
import copy
import random
from pathlib import Path

import pytest
import torch

from tests import beam_oracle as BO
from tests import processors_oracle as PO
from tests import trie_beam_oracle as TB
from tests.test_trie_table_cpu import make_trie, structure, unpack

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
SPECIAL = [32000, 32001, 32002, 32003, 32004]
GOLD = Path(__file__).resolve().parent / "golden"
EOS = 2


# ---------------------------------------------------------------------------------------------------------------------
# nv_beam_topk_trie
# ---------------------------------------------------------------------------------------------------------------------
def _csr(trie, V, dev, grow=False):
    from navillm_b200.trie import flatten_trie
    table = flatten_trie(trie, V)
    caps = (1 << (table.n_nodes - 1).bit_length(), 1 << (max(table.n_edges, 1) - 1).bit_length()) if grow else (None, None)
    node_ptr, child_tok, child_node, n = unpack(table, *caps)
    return [torch.tensor(x, dtype=torch.int32, device=dev) for x in (node_ptr, child_tok, child_node)] + [n, table.eos]


def _histories(rng, trie_words, K, t, V):
    """K generated rows of length t: on the trie (a word's prefix), past a leaf (a whole word, then anything), off the trie
    (a token that is no child), random."""
    rows = []
    for _ in range(K):
        w = rng.choice(trie_words)
        kind = rng.randrange(4)
        if kind == 0:
            row = w[:t]
        elif kind == 1:
            row = list(w)
        elif kind == 2:
            row = w[:rng.randrange(len(w) + 1)] + [V - 7]
        else:
            row = []
        row = (row + [rng.randrange(V - 10) for _ in range(t)])[:t]
        rows.append(row)
    return rows


def _restated(logits, bs, K, prompt, hist, t, trie, proc, first_step):
    """The kernel's arithmetic on the CPU: bf16 log-probs (fp64 sum), the processors, the trie mask, the fp32 add; the 2K best
    by (score desc, flat index asc)."""
    x = logits.float().cpu()
    x[:, SPECIAL] = float("-inf")
    m = x.max(dim=1, keepdim=True).values
    ls64 = torch.log(torch.exp((x - m).double()).sum(dim=1, keepdim=True))
    lp = ((x - m) - ls64.float()).to(bf16)
    if first_step:
        lp = lp.repeat_interleave(K, 0)
    B, S = prompt.shape
    out = []
    for b in range(B):
        rows = slice(b * K, (b + 1) * K)
        gen = [hist[r][:t[b]] for r in range(b * K, (b + 1) * K)]
        p = lp[rows]
        if proc:
            ids = torch.cat([prompt[b:b + 1].repeat(K, 1), torch.tensor(gen, dtype=torch.int64).view(K, t[b])], 1)
            p = PO.process(p, ids, S, eos_token_id=EOS, **proc)
        out.append(TB.trie_mask(p, gen, trie))
    scores = (torch.cat(out).float() + bs.cpu()[:, None]).view(B, K * lp.shape[1])
    return scores, BO.top_candidates(scores, K)


def _run_trie_topk(dev, logits, bs, K, prompt, hist, t, csr, proc, first_step, G=64):
    from navillm_b200 import ops
    B = prompt.shape[0]
    special = torch.tensor(SPECIAL, dtype=torch.int32, device=dev)
    h = torch.zeros(B * K, G, dtype=torch.int32, device=dev)
    for r, row in enumerate(hist):
        h[r, :len(row)] = torch.tensor(row, dtype=torch.int32)
    pstate = torch.zeros(B, 5, dtype=torch.int32, device=dev)
    pstate[:, 0] = torch.tensor(t, dtype=torch.int32)
    pids = prompt.int().to(dev).contiguous()
    width = torch.tensor([prompt.shape[1]], dtype=torch.int32, device=dev)
    c = (torch.empty((B, 2 * K), dtype=torch.float32, device=dev), torch.empty((B, 2 * K), dtype=torch.int32, device=dev),
         torch.empty((B, 2 * K), dtype=torch.int32, device=dev))
    ptuple = None if not proc else (float(proc.get("repetition_penalty", 1.0)), proc.get("no_repeat_ngram_size", 0),
                                    proc.get("min_length", 0), proc.get("min_new_tokens", 0), EOS)
    ops.beam_topk_trie(logits, special, bs, K, *c, pids, width, h, pstate, ptuple, *csr, first_step=first_step)
    torch.cuda.synchronize()
    return [x.cpu() for x in c], (special, pids, width, h, pstate, ptuple)


@pytest.mark.parametrize("B", [1, 3, 8])
@pytest.mark.parametrize("K", [1, 2, 4, 8])
def test_beam_topk_trie_matches_restatement(cuda_dev, B, K):
    V, S = 32006, 24
    rng = random.Random(B * 100 + K)
    wide = [[rng.randrange(V - 10) for _ in range(rng.randint(1, 4))] for _ in range(300)] + [[5, EOS], [5, 6, 7]]
    narrow = [[rng.randrange(V - 10), rng.randrange(V - 10)]]          # one answer: -inf candidates fill the 2K
    g = torch.Generator(device=cuda_dev).manual_seed(B * 10 + K)
    prompt = torch.randint(0, 60, (B, S), generator=torch.Generator().manual_seed(K))
    for words in (wide, narrow):
        trie = make_trie(words, eos=EOS)
        before = structure(trie.root)
        csr = _csr(trie, V, cuda_dev, grow=True)
        for first_step in (False, True):
            for proc in (None, dict(repetition_penalty=1.3, no_repeat_ngram_size=2), dict(min_new_tokens=3)):
                t = [0] * B if first_step else [rng.randrange(6) for _ in range(B)]
                hist = [r for b in range(B) for r in _histories(rng, words, K, t[b], V)]
                logits = (torch.randn(B if first_step else B * K, V, generator=g, device=cuda_dev) * 3).to(bf16)
                if first_step:
                    bs = torch.tensor(([0.0] + [-1e9] * (K - 1)) * B, device=cuda_dev)
                else:
                    bs = (torch.randn(B * K, generator=g, device=cuda_dev) * 4).float()
                got, _ = _run_trie_topk(cuda_dev, logits, bs, K, prompt, hist, t, csr, proc, first_step)
                scores, (ws, wt, wp) = _restated(logits, bs, K, prompt, hist, t, trie, proc, first_step)
                srt = torch.sort(scores, dim=1, descending=True, stable=True)[0]
                if words is narrow and not first_step:
                    assert bool(torch.isinf(srt[:, 2 * K - 1]).all()), "the narrow trie leaves -inf candidates in the 2K"
                for b in range(B):
                    if srt[b, 2 * K - 1] == srt[b, 2 * K] and torch.isfinite(srt[b, 2 * K]):
                        continue                                      # a finite tie straddles rank 2K: the set is not unique
                    tag = (len(words), first_step, proc, b)
                    assert torch.equal(got[0][b], ws[b]), tag
                    assert got[1][b].long().tolist() == wt[b].tolist() and got[2][b].long().tolist() == wp[b].tolist(), tag
        assert structure(trie.root) == before


@pytest.mark.parametrize("K", [2, 4, 8])
def test_always_allowing_trie_is_the_plain_beam_topk(cuda_dev, K):
    """A root whose children are every token: at the first generated column the trie instantiation equals nv_beam_topk and,
    with processors, nv_beam_topk_processed."""
    from navillm_b200 import ops
    V, B, S = 32006, 3, 16
    trie = make_trie([[c] for c in range(V)], eos=EOS)
    csr = _csr(trie, V, cuda_dev)
    g = torch.Generator(device=cuda_dev).manual_seed(K)
    prompt = torch.randint(0, 60, (B, S), generator=torch.Generator().manual_seed(1))
    logits = (torch.randn(B * K, V, generator=g, device=cuda_dev) * 3).to(bf16)
    bs = (torch.randn(B * K, generator=g, device=cuda_dev) * 4).float()
    for proc in (None, dict(repetition_penalty=1.2, no_repeat_ngram_size=1)):
        got, (special, pids, width, h, pstate, ptuple) = _run_trie_topk(cuda_dev, logits, bs, K, prompt, [[]] * (B * K), [0] * B,
                                                                         csr, proc, False)
        c = (torch.empty((B, 2 * K), dtype=torch.float32, device=cuda_dev), torch.empty((B, 2 * K), dtype=torch.int32, device=cuda_dev),
             torch.empty((B, 2 * K), dtype=torch.int32, device=cuda_dev))
        if proc is None:
            ops.beam_topk(logits, special, bs, K, *c)
        else:
            ops.beam_topk_processed(logits, special, bs, K, *c, pids, width, h, pstate, ptuple)
        assert all(torch.equal(x, y.cpu()) for x, y in zip(got, c)), proc


def test_beam_topk_trie_bad_arguments(cuda_dev):
    from navillm_b200 import _lib, ops
    V, B, K = 32006, 2, 2
    csr = _csr(make_trie([[11, 12]], eos=EOS), V, cuda_dev)
    logits = torch.zeros(B * K, V, dtype=bf16, device=cuda_dev)
    bs = torch.zeros(B * K, device=cuda_dev)
    args = lambda: [torch.empty((B, 2 * K), dtype=torch.float32, device=cuda_dev)] + \
        [torch.empty((B, 2 * K), dtype=torch.int32, device=cuda_dev) for _ in range(2)]
    special = torch.tensor(SPECIAL, dtype=torch.int32, device=cuda_dev)
    pids, width = torch.zeros(B, 4, dtype=torch.int32, device=cuda_dev), torch.tensor([4], dtype=torch.int32, device=cuda_dev)
    h, pstate = torch.zeros(B * K, 8, dtype=torch.int32, device=cuda_dev), torch.zeros(B, 5, dtype=torch.int32, device=cuda_dev)
    ops.beam_topk_trie(logits, special, bs, K, *args(), pids, width, h, pstate, None, *csr)
    with pytest.raises(_lib.NvError):                                  # leaf token outside [0, V)
        ops.beam_topk_trie(logits, special, bs, K, *args(), pids, width, h, pstate, None, *csr[:4], V)
    with pytest.raises(ValueError):                                    # node_ptr too short for n_nodes
        ops.beam_topk_trie(logits, special, bs, K, *args(), pids, width, h, pstate, None, csr[0][:2], *csr[1:])
    with pytest.raises(_lib.NvError):                                  # three V-bit bitmaps exceed 48 KB
        big = torch.zeros(B * K, 140000, dtype=bf16, device=cuda_dev)
        ops.beam_topk_trie(big, special, bs, K, *args(), pids, width, h, pstate, None, *csr)


# ---------------------------------------------------------------------------------------------------------------------
# generate(trie=t, num_beams=K)
# ---------------------------------------------------------------------------------------------------------------------
def _tiny(cuda_dev, rows=None):
    from tests.test_beam_gpu import _qa
    from tests.test_navmodel_gpu import build_model
    from tests.test_oracle_golden import load
    g, cfg, tok = load("amp_bf16")
    model, _ = build_model(g, cuda_dev)
    text, cand = _qa(g, cfg, tok, rows)
    kw = dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev),
              eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id)
    return g, cfg, tok, model, text, cand, kw


def _leaf_paths(node, prefix=()):
    if len(node.child) == 0:
        return [list(prefix)]
    return [p for t, ch in node.child.items() for p in _leaf_paths(ch, prefix + (t,))]


def assert_answers(ids, S, trie, eos, pad, n_new):
    """Every returned row: a root-to-leaf path of the trie, EOS, then pad -- or a prefix of such a path cut at n_new tokens."""
    paths = _leaf_paths(trie.root)
    for row in ids[:, S:].tolist():
        if eos in row:
            i = row.index(eos)
            assert row[:i] in paths and all(x == pad for x in row[i + 1:]), row
        else:
            assert len(row) == n_new and any(p[:n_new] == row for p in paths), row


GOLD_WORDS = [[21, 22, 23], [21, 22, 30, 31], [21, 40], [50, 51, 52], [60], [61, 62]]


@pytest.mark.parametrize("K,n_ret,lp,early,rows", [(2, 1, 0.0, False, None), (4, 4, 0.0, False, None), (4, 2, 1.0, False, None),
                                                   (4, 3, 2.0, True, [0]), (8, 8, 1.0, False, [0, 1, 0])],
                         ids=["K2", "K4n4", "K4n2lp1", "B1K4n3early", "B3K8n8"])
def test_generate_trie_beams_match_oracle(cuda_dev, K, n_ret, lp, early, rows):
    from tests.test_beam_gpu import near_tie_ok
    g, cfg, tok, model, text, cand, kw = _tiny(cuda_dev, rows)
    lm = model.lang_model
    trie = make_trie(GOLD_WORDS + [[tok.bos_token_id, 70 + i] for i in range(3)], eos=tok.eos_token_id)
    before = structure(trie.root)
    n_new = 7
    call = dict(num_beams=K, num_return_sequences=n_ret, length_penalty=lp, early_stopping=early, max_new_tokens=n_new)
    ref, steps = TB.trie_beam_generate(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], trie, cand_vis=cand,
                                       eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id, return_steps=True, **call)
    S = text["input_ids"].shape[1]
    outs = {}
    for graph in (False, True, True):
        stats = {}
        ids = lm.generate(trie=trie, use_cuda_graph=graph, stats=stats, **call, **kw).cpu()
        assert ids.shape[0] == ref.shape[0] and torch.equal(ids[:, :S], ref[:, :S])
        near_tie_ok(ids, ref, steps, S, n_ret, tag=f"graph={graph}")
        assert_answers(ids, S, trie, tok.eos_token_id, tok.unk_token_id, n_new)
        assert stats["trie_path"] == "device" and stats["trie_flatten_ms"] >= 0 and stats["beam_steps"] >= 1
        if graph and graph in outs:
            assert stats["graph_replays"] > 0 or stats["decode_steps"] <= 1
        outs[graph] = ids
    assert torch.equal(outs[False], outs[True])
    assert structure(trie.root) == before


def test_generate_trie_beams_match_the_reference_golden(cuda_dev):
    """The reference's 3dqa branch with prefix_allowed_tokens_fn walking the trie (tests/golden/make_trie_beam_golden.py), at
    length_penalty 0: the device ids equal the golden's per prompt, or a near tie of the oracle decided the first difference."""
    from tests.test_beam_gpu import near_tie_ok
    g, cfg, tok, model, text, cand, kw = _tiny(cuda_dev)
    lm = model.lang_model
    gen = torch.load(GOLD / "generate_trie_beam_amp_bf16.pt", weights_only=False)
    S, n_new = gen["prompt_len"], gen["meta"]["max_new_tokens"]
    assert S == text["input_ids"].shape[1]
    exact = 0
    for run in gen["runs"]:
        K, n = run["num_beams"], run["num_return_sequences"]
        trie = make_trie(run["words"], eos=tok.eos_token_id)
        call = dict(num_beams=K, num_return_sequences=n, length_penalty=0.0, max_new_tokens=n_new)
        _, steps = TB.trie_beam_generate(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], trie, cand_vis=cand,
                                         eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id, return_steps=True, **call)
        ids = lm.generate(trie=trie, **call, **kw).cpu()
        want = TB.golden_ids(run["ids"], S, tok.eos_token_id, tok.unk_token_id)
        exact += int(ids.shape == want.shape and torch.equal(ids, want))
        near_tie_ok(ids, want, steps, S, n, tag=f"golden {run['trie']} K={K} n={n}")
        assert_answers(ids, S, trie, tok.eos_token_id, tok.unk_token_id, n_new)
    print(f"\n[trie beams vs reference golden] {exact} of {len(gen['runs'])} runs bit-identical")


class _CaptureSpy:
    def __init__(self, monkeypatch):
        self.n = 0
        real = torch.cuda.graph

        def graph(*a, **kw):
            self.n += 1
            return real(*a, **kw)
        monkeypatch.setattr(torch.cuda, "graph", graph)


def test_trie_beams_graph_reuse_and_growth(cuda_dev, monkeypatch):
    """Graph equals eager; a second trie of the same size replays the captured step; a trie that outgrows the buffers
    recaptures once."""
    g, cfg, tok, model, text, cand, kw = _tiny(cuda_dev)
    lm = model.lang_model
    call = dict(num_beams=4, num_return_sequences=2, max_new_tokens=8, **kw)
    spy = _CaptureSpy(monkeypatch)
    t1 = make_trie(GOLD_WORDS, eos=tok.eos_token_id)
    t2 = make_trie([[21, 24, 25], [21, 24, 32, 33], [21, 41], [53, 54, 55], [63], [64, 65]], eos=tok.eos_token_id)
    big = make_trie(GOLD_WORDS + [[a, b] for a in range(80, 110) for b in (5, 6)], eos=tok.eos_token_id)
    want = {id(t): lm.generate(trie=t, use_cuda_graph=False, **call).cpu() for t in (t1, t2, big)}
    assert spy.n == 0
    for t, n_capt in ((t1, 1), (t2, 1), (big, 2)):
        stats = {}
        got = lm.generate(trie=t, use_cuda_graph=True, stats=stats, **call).cpu()
        assert torch.equal(got, want[id(t)]) and spy.n == n_capt, (n_capt, spy.n)
        assert stats["graph_replays"] > 0


def test_trie_beams_on_fp8_kv_and_quantized_weights(cuda_dev, monkeypatch):
    """The fp8 KV cache: the bf16 trie-beam path over the rounded K' / V'.  fp8 and int4 weight copies: trie beams on W'."""
    from tests.test_beam_gpu import _rounded_bf16_beams
    g, cfg, tok, model, text, cand, kw = _tiny(cuda_dev, [1, 0, 1])
    lm = model.lang_model
    trie = make_trie(GOLD_WORDS, eos=tok.eos_token_id)
    call = dict(kw, num_beams=4, num_return_sequences=2, max_new_tokens=8, trie=trie)
    want = _rounded_bf16_beams(lm, monkeypatch, call)
    prev = lm.set_kv_cache_dtype("fp8")
    try:
        for graph in (False, True, True):
            assert torch.equal(lm.generate(**dict(call, use_cuda_graph=graph)).cpu(), want), graph
    finally:
        lm.set_kv_cache_dtype(prev)
    for quant, drop in (("quantize_weights_fp8", "drop_fp8_weights"), ("quantize_weights_int4", "drop_int4_weights")):
        getattr(model, quant)()
        try:
            got = [lm.generate(**dict(call, use_cuda_graph=gr)).cpu() for gr in (False, True)]
        finally:
            getattr(model, drop)()
        on_w = lm.generate(**dict(call, use_cuda_graph=False)).cpu()
        assert torch.equal(got[0], on_w) and torch.equal(got[1], on_w), quant
        assert_answers(on_w, text["input_ids"].shape[1], trie, tok.eos_token_id, tok.unk_token_id, 8)


@pytest.mark.parametrize("proc", [dict(repetition_penalty=1.3), dict(no_repeat_ngram_size=2, min_new_tokens=2)],
                         ids=["rep", "ngram+min_new"])
def test_trie_beams_with_processors_match_oracle(cuda_dev, proc):
    from tests.test_beam_gpu import near_tie_ok
    g, cfg, tok, model, text, cand, kw = _tiny(cuda_dev)
    lm = model.lang_model
    trie = make_trie([[21, 21, 22], [21, 22, 21, 22], [30, 31, 30], [40], [41, 42]], eos=tok.eos_token_id)
    call = dict(num_beams=4, num_return_sequences=2, max_new_tokens=7)
    ref, steps = TB.trie_beam_generate(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], trie, cand_vis=cand,
                                       eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id, return_steps=True, **call,
                                       **proc)
    S = text["input_ids"].shape[1]
    for graph in (False, True):
        ids = lm.generate(trie=trie, use_cuda_graph=graph, **call, **proc, **kw).cpu()
        near_tie_ok(ids, ref, steps, S, 2, tag=f"{proc} graph={graph}")


def test_launches_of_other_modes(cuda_dev, monkeypatch):
    """Beams without a trie launch nv_beam_topk, a trie without beams nv_trie_mask, as before; trie beams launch
    nv_beam_topk_trie and never nv_trie_mask."""
    import navillm_b200.ops as ops_mod
    from navillm_b200 import _lib
    g, cfg, tok, model, text, cand, kw = _tiny(cuda_dev)
    lm = model.lang_model
    calls = []
    real = _lib.check

    def spy(status, what):
        calls.append(what)
        return real(status, what)
    monkeypatch.setattr(ops_mod, "check", spy)
    trie = make_trie(GOLD_WORDS, eos=tok.eos_token_id)
    runs = {"beams": dict(num_beams=4), "beams+proc": dict(num_beams=4, repetition_penalty=1.2), "trie": dict(trie=trie),
            "trie_beams": dict(trie=trie, num_beams=4), "trie_beams+proc": dict(trie=trie, num_beams=4, repetition_penalty=1.2)}
    seen = {}
    for name, extra in runs.items():
        calls.clear()
        lm.generate(max_new_tokens=6, use_cuda_graph=False, **extra, **kw)
        seen[name] = set(calls)
    assert "nv_beam_topk" in seen["beams"] and "nv_beam_topk_processed" in seen["beams+proc"]
    assert not any("trie" in c for c in seen["beams"] | seen["beams+proc"])
    assert "nv_trie_mask" in seen["trie"] and not any("beam" in c for c in seen["trie"])
    for name in ("trie_beams", "trie_beams+proc"):
        assert "nv_beam_topk_trie" in seen[name] and "nv_trie_mask" not in seen[name], name
        assert not {"nv_beam_topk", "nv_beam_topk_processed"} & seen[name], name
    assert seen["trie_beams"] == seen["beams"] - {"nv_beam_topk"} | {"nv_beam_topk_trie"}


def test_modes_with_trie_beams(cuda_dev):
    """3dqa and embodied_qa with trie= and num_beams=4, num_return_sequences=3: B * 3 sentences, each an answer of the set;
    summarization with trie= and no beam kwargs keeps the greedy golden."""
    from tests.test_navmodel_gpu import build_model, to_dev
    from tests.test_oracle_golden import load
    g, cfg, tok = load("amp_bf16")
    model, _ = build_model(g, cuda_dev)
    gen = torch.load(GOLD / "generate_amp_bf16.pt", weights_only=False)
    words = [[tok.bos_token_id] + w for w in GOLD_WORDS]
    trie = make_trie(words, eos=tok.eos_token_id)
    answers = set(tok.batch_decode(words, skip_special_tokens=True, clean_up_tokenization_spaces=False))
    before = structure(trie.root)
    with torch.no_grad():
        qa = model("3dqa", to_dev(dict(g["qa_in"]), cuda_dev), training=False, trie=trie, num_beams=4, num_return_sequences=3,
                   max_new_tokens=8)["generated_sentences"]
        eqa = model("embodied_qa", to_dev(dict(g["sum_in"]), cuda_dev), training=False, trie=trie, num_beams=4,
                    num_return_sequences=3)["generated_sentences"]
        t_sum = make_trie(gen["trie_words"], eos=tok.eos_token_id)
        t_sum.bos = tok.bos_token_id
        summ = model("summarization", to_dev(dict(g["sum_in"]), cuda_dev), training=False, trie=t_sum)["generated_sentences"]
    assert len(qa) == 3 * len(g["qa_in"]["question"]) and set(qa) <= answers, qa
    assert len(eqa) == 3 * len(g["sum_in"]["prompts"]) and set(eqa) <= answers, eqa
    assert summ == gen["trie_sentences"]
    assert structure(trie.root) == before


def test_generate_trie_beams_fullwidth_two_layers(cuda_dev):
    """Two layers at Vicuna-7B widths, vocabulary 32006, an EQA-shaped trie (64 answers of 1-3 tokens after BOS), B = 4, K = 4:
    against the oracle under the near-tie rule, graph equal to eager."""
    from tests.test_beam_gpu import near_tie_ok
    from tests.test_fullwidth_parity_gpu import _full_navmodel, _oracle_cfg
    model, tok = _full_navmodel(cuda_dev, 32000)
    lm = model.lang_model
    sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items() if k.startswith("lang_model.")}
    prompts = ["Question : what color is the sofa in the living room ? Answer :", "Question : how many chairs ? Answer :",
               "Question : where is the lamp ? Answer :", "Question : is the door open ? Answer :"]
    text = lm.tokenize(prompts)
    rng = random.Random(0)
    words = [[tok.bos_token_id] + [rng.randrange(100, 31000) for _ in range(rng.randint(1, 3))] for _ in range(64)]
    trie = make_trie(words, eos=tok.eos_token_id)
    call = dict(num_beams=4, num_return_sequences=2, max_new_tokens=6, eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id)
    ref, steps = TB.trie_beam_generate(sd, _oracle_cfg(tok, "amp_bf16"), text["input_ids"], text["attention_mask"],
                                       copy.deepcopy(trie), return_steps=True, **call)
    S = text["input_ids"].shape[1]
    outs = {}
    for graph in (False, True):
        ids = lm.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], trie=trie, use_cuda_graph=graph,
                          **call).cpu()
        matched = near_tie_ok(ids, ref, steps, S, 2, tag=f"fullwidth graph={graph}")
        print(f"\n[full-width trie beams, graph={graph}] matched generated columns per prompt {matched}")
        assert_answers(ids, S, trie, tok.eos_token_id, tok.unk_token_id, 6)
        outs[graph] = ids
    assert torch.equal(outs[False], outs[True])
