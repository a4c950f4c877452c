"""Trie-constrained (EQA-shaped) and sampled (C3-shaped) generate(): host path against the device paths, in one process.

    python tools/constrained_decode_bench.py [--layers 32] [--answers 64] [--calls 12] [--gens 3] [--out FILE.json]

Full-width Vicuna-7B with random init (bench.build_model).
(i)  EQA-shaped: B = 8, prompts of tasks/agents/eqa.py:get_embodied_qa_prompt with 8 <hist>, 16 <cand> and 24 question
     words (the long prompts get as many more as it takes to reach the next Smax bucket); a trie of --answers synthetic
     answers of 1-3 tokens, bos-prefixed as in tasks/agents/mp3d_agent.py:551-556;
     max_new_tokens = 50, stop_on_eos.  Three paths per call, in rotating order: the host TrieLogitsProcessor, the device walk
     eager and the device walk through the CUDA graph.  ms per generate call (host clock, ends in a device sync) over a
     sequence whose prompt lengths alternate between two Smax buckets, starting with no captured graph (capture cost and LRU
     included), then the steady state in one bucket; the trie flattening cost per call; token equality with the host path.
(ii) C3-shaped sampled: B = 8, S0 = 320, 128 new tokens, do_sample, T = 1, top_k = 50, no EOS stop; decode ms/token eager
     against graph (device events), alternated, and token equality under the same seed.
(iii) the GPU name and power limit, read in the same run.
"""
import argparse
import copy
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from navillm_b200.trie import TrieLogitsProcessor  # noqa: E402


class _Node:
    def __init__(self):
        from collections import defaultdict
        self.child = defaultdict(_Node)


class Trie:
    """The interface of the reference's tools/trie.py."""

    def __init__(self, bos, eos):
        self.root, self.bos, self.eos = _Node(), bos, eos

    def insert(self, word):
        cur = self.root
        for c in word:
            cur = cur.child[c]

    def get_child_index(self, cur):
        return [self.eos] if len(cur.child) == 0 else list(cur.child.keys())

    def get_next_node(self, cur, w):
        return cur if len(cur.child) == 0 else cur.child[w]


def eqa_prompt(question, hist_num=8, cand_num=16):
    """tasks/agents/eqa.py:get_embodied_qa_prompt."""
    p = "### Instruction: Answer the question according to the scene. \n"
    p += "Following is the History, which contains the visual information of your previous decisions.\n"
    p += "### History: {}\n".format(" ".join("({}) <hist>".format(i) for i in range(hist_num)))
    p += "Following is the Observation, which contains panoramic views at your current location.\n"
    p += "### Candidate: {}\n".format(" ".join("({}) <cand>".format(i) for i in range(cand_num)))
    p += "### Question: {}\n".format(question)
    p += "### Answer: "
    return p


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0), out


def eqa(model, dev, n_answers, n_calls, seed=0):
    lm = model.lang_model
    tok = lm.tokenizer
    B, D = 8, lm.dims.hidden
    rng = np.random.RandomState(seed)
    trie = Trie(tok.bos_token_id, tok.eos_token_id)
    for _ in range(n_answers):
        trie.insert([tok.bos_token_id] + rng.randint(100, 31000, size=rng.randint(1, 4)).tolist())
    words = [f"w{i}" for i in range(5000)]

    def batch(n_words):
        prompts = [eqa_prompt(" ".join(words[i] for i in rng.randint(0, 5000, size=n_words)) + " ?") for _ in range(B)]
        text = lm.tokenize(prompts)
        g = torch.Generator().manual_seed(int(rng.randint(1 << 30)))
        hist = (torch.randn(B * 8, D, generator=g) * 0.02).to(dev)
        cand = (torch.randn(B * 16, D, generator=g) * 0.02).to(dev)
        return dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand, hist_vis=hist)

    # two groups of prompt lengths that land in two Smax buckets (prompt + 50 new tokens, rounded up to 128)
    def shape(b):
        L = int(b["attention_mask"].sum(1).max())
        return {"S0": L, "Smax": (L + 50 + 127) // 128 * 128}

    short = batch(24)
    n_long, long_ = 36, batch(36)
    while shape(long_)["Smax"] == shape(short)["Smax"]:              # lengthen the question until the next bucket
        n_long += 4
        long_ = batch(n_long)
    lens = {"short": dict(shape(short), question_words=24), "long": dict(shape(long_), question_words=n_long)}
    common = dict(max_new_tokens=50, stop_on_eos=True, eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id)
    paths = {
        "host": lambda b, st: lm.generate(**b, **common, logits_processor=[TrieLogitsProcessor(copy.deepcopy(trie))], stats=st),
        "device_eager": lambda b, st: lm.generate(**b, **common, trie=trie, use_cuda_graph=False, stats=st),
        "device_graph": lambda b, st: lm.generate(**b, **common, trie=trie, use_cuda_graph=True, stats=st),
    }
    names = list(paths)

    def run(seq):
        ms = {k: [] for k in names}
        flat, equal, steps, misses = [], [], [], 0
        for i, b in enumerate(seq):
            outs = {}
            for k in names[i % 3:] + names[:i % 3]:                   # rotating order
                st = {}
                t, outs[k] = timed(lambda: paths[k](b, st))
                ms[k].append(t)
                if k != "host":
                    flat.append(st["trie_flatten_ms"])
                    misses += st["trie_path"] != "device"
                else:
                    steps.append(st["decode_steps"])
            equal.append(all(torch.equal(outs["host"], outs[k]) for k in names[1:]))
        return ms, flat, equal, steps, misses

    lm.__dict__.pop("_decode_states", None)                          # start without a captured graph
    seq = [short if i % 2 == 0 else long_ for i in range(n_calls)]
    ms, flat, equal, steps, misses = run(seq)
    res = {"B": B, "answers": n_answers, "trie_nodes_edges": None, "buckets": lens, "calls": n_calls,
           "mixed_ms_per_call_mean": {k: round(float(np.mean(v)), 2) for k, v in ms.items()},
           "mixed_ms_per_call_median": {k: round(float(np.median(v)), 2) for k, v in ms.items()},
           "mixed_tokens_equal_all_paths": all(equal), "decode_steps_per_call": steps, "device_misses": misses}
    ms, flat2, equal, steps, misses = run([short] * n_calls)          # steady state, one bucket (graph already captured)
    res.update({"steady_ms_per_call_median": {k: round(float(np.median(v)), 2) for k, v in ms.items()},
                "steady_tokens_equal_all_paths": all(equal), "steady_device_misses": misses,
                "flatten_ms_per_call_median": round(float(np.median(flat + flat2)), 4)})
    from navillm_b200.trie import flatten_trie
    t = flatten_trie(trie, lm.lm_head.weight.shape[0])
    res["trie_nodes_edges"] = [t.n_nodes, t.n_edges]
    sm = res["steady_ms_per_call_median"]
    res["steady_speedup_graph_vs_host"] = round(sm["host"] / sm["device_graph"], 3)
    res["steady_speedup_graph_vs_eager"] = round(sm["device_eager"] / sm["device_graph"], 3)
    return res


def c3_sampled(model, dev, gens):
    lm = model.lang_model
    wl = bench.WORKLOADS["c3"]
    B, NV, NT, NEW = wl["B"], wl["n_cand_tok"], wl["n_text"], wl["n_new"]
    rng = np.random.RandomState(1234)
    words = [f"w{i}" for i in range(5000)]
    prompts = ["Scene " + " ".join(["<cand>"] * NV) + " Question " + " ".join(words[i] for i in rng.randint(0, 5000, size=NT - 5))
               + " Answer" for _ in range(B)]
    text = lm.tokenize(prompts)
    S0 = int(text["attention_mask"].sum(1).max())
    g = torch.Generator().manual_seed(1234)
    with torch.no_grad():
        view = torch.stack([torch.randn(NV, bench.IMG_FEAT, generator=g) for _ in range(B)], 0).to(dev)
        pano = model.img_embeddings.forward_panorama_per_step(view_img_fts=view, view_lens=torch.full((B,), NV, device=dev))
        cand = model._masked_rows_plus_const(pano["pano_embeds"].reshape(B * NV, -1), np.ones((B, NV), dtype=bool)).detach()
    per_tok = {False: [], True: []}
    ids = {}
    for rep in range(gens + 1):                                       # rep 0 warms up and captures the graph
        for graph in ((False, True) if rep % 2 == 0 else (True, False)):
            st = {}
            torch.manual_seed(100 + rep)
            out = lm.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand, max_new_tokens=NEW,
                              stop_on_eos=False, do_sample=True, temperature=1.0, top_k=50, use_cuda_graph=graph, stats=st)
            ids[(rep, graph)] = out.cpu()
            if rep > 0:
                per_tok[graph].append(st["decode_ms"] / st["decode_steps"])
    equal = all(torch.equal(ids[(r, False)], ids[(r, True)]) for r in range(gens + 1))
    e, gph = float(np.median(per_tok[False])), float(np.median(per_tok[True]))
    return {"B": B, "S0": S0, "new_tokens": NEW, "temperature": 1.0, "top_k": 50, "decode_ms_per_token_eager": round(e, 4),
            "decode_ms_per_token_graph": round(gph, 4), "speedup_graph_vs_eager": round(e / gph, 3),
            "tokens_equal_graph_vs_eager": equal}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--answers", type=int, default=64)
    ap.add_argument("--calls", type=int, default=12)
    ap.add_argument("--gens", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the result as JSON here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("constrained_decode_bench: needs an H100 (no CPU path)")
    dev = torch.device("cuda:0")
    if a.layers != bench.N_LAYERS:
        import navillm_b200.nav_model as nm
        nm.VICUNA_7B["num_hidden_layers"] = a.layers
    res = {"gpu": bench.gpu_info(0), "layers": a.layers}
    print(json.dumps(res["gpu"]), flush=True)
    model = bench.build_model(dev, seed=0).eval()
    model._ensure()
    with torch.no_grad():
        res["eqa_trie"] = eqa(model, dev, a.answers, a.calls)
        print(json.dumps(res["eqa_trie"]), flush=True)
        res["c3_sampled"] = c3_sampled(model, dev, a.gens)
        print(json.dumps(res["c3_sampled"]), flush=True)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
