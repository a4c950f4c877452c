"""Trie-constrained beam search in generate() at Vicuna-7B widths (random init), against the greedy device trie path.

    python tools/trie_beam_bench.py [--layers 32] [--gens 3] [--out FILE.json]

(i)   EQA shape: B = 8 prompts of tasks/agents/eqa.py:get_embodied_qa_prompt (8 <hist>, 16 <cand>), the trie of 64 synthetic
      answers of 1-3 tokens after BOS (133 nodes), max_new_tokens = 50 with EOS stopping.  Arms: greedy decoding under the trie
      and trie beams at K = 2 / 4 / 8 (num_return_sequences = K).
(ii)  3dqa shape: the C3 prompt (256 <cand> + 64 text tokens), B = 8, K = 4, a trie of 300 ScanQA-like short answers (1-4
      tokens), max_new_tokens = 20.  Arms: greedy under the trie, trie beams, plain beams without the trie.
Per arm: ms per call (host clock around a synchronised call), prefill_ms, decode steps and peak memory, median over --gens
calls after the capturing one; the arms alternate call by call.
(iii) The kernel alone: nv_beam_topk_trie against nv_beam_topk and nv_beam_topk_processed (processors off) at B = 8, K = 4,
      V = 32006, beams 1 and 3 tokens deep in the EQA trie, CUDA events over 200 launches.
The GPU name and power limit are read in the same run.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import bench  # noqa: E402
from beam_bench import prompts  # noqa: E402
from constrained_decode_bench import Trie, eqa_prompt, timed  # noqa: E402


def make_trie(tok, n_answers, lo, hi, bos, seed):
    rng = np.random.RandomState(seed)
    trie = Trie(tok.bos_token_id, tok.eos_token_id)
    words = []
    for _ in range(n_answers):
        w = ([tok.bos_token_id] if bos else []) + rng.randint(100, 31000, size=rng.randint(lo, hi + 1)).tolist()
        trie.insert(w)
        words.append(w)
    return trie, words


def eqa_batch(lm, dev, B=8, seed=0):
    rng = np.random.RandomState(seed)
    words = [f"w{i}" for i in range(5000)]
    text = lm.tokenize([eqa_prompt(" ".join(words[i] for i in rng.randint(0, 5000, size=24)) + " ?") for _ in range(B)])
    g = torch.Generator().manual_seed(seed)
    D = lm.dims.hidden
    return dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"],
                cand_vis=(torch.randn(B * 16, D, generator=g) * 0.02).to(dev), hist_vis=(torch.randn(B * 8, D, generator=g) * 0.02).to(dev))


def arms_timed(lm, batch, arms, gens, new):
    """Each arm once to capture, then ``gens`` rounds alternating the arms."""
    res = {name: [] for name in arms}
    for i in range(gens + 1):
        for name, kw in arms.items():
            torch.cuda.reset_peak_memory_stats()
            st = {}
            ms, ids = timed(lambda: lm.generate(**batch, max_new_tokens=new, use_cuda_graph=True, stats=st, **kw))
            if i:
                res[name].append((ms, st["prefill_ms"], st.get("beam_steps", st["decode_steps"] + 1), st["graph_replays"],
                                  torch.cuda.max_memory_allocated() / 2 ** 30, st.get("trie_path")))
    out = {}
    for name, v in res.items():
        out[name] = {"ms_per_call": round(float(np.median([x[0] for x in v])), 3),
                     "ms_spread": round(float(max(x[0] for x in v) - min(x[0] for x in v)), 3),
                     "prefill_ms": round(float(np.median([x[1] for x in v])), 3), "steps": int(v[-1][2]),
                     "graph_replays": int(v[-1][3]), "peak_gib": round(max(x[4] for x in v), 2), "trie_path": v[-1][5]}
        print(json.dumps({name: out[name]}), flush=True)
    return out


def kernel_times(lm, trie_words, trie, dev, B=8, K=4, n=200):
    from contrastive_bench import event_ms
    from navillm_b200 import ops
    from navillm_b200.trie import flatten_trie
    V = lm.lm_head.weight.shape[0]
    table = flatten_trie(trie, V)
    host = table.pack(table.n_nodes, table.n_edges)
    buf = torch.from_numpy(host).to(dev)
    o = table.n_nodes + 2
    csr = (buf[:o], buf[o:o + table.n_edges], buf[o + table.n_edges:], table.n_nodes, table.eos)
    g = torch.Generator(device=dev).manual_seed(0)
    logits = (torch.randn(B * K, V, generator=g, device=dev) * 3).to(torch.bfloat16)
    bs = torch.randn(B * K, generator=g, device=dev)
    special = lm.special_ids_dev
    cand = (torch.empty((B, 2 * K), dtype=torch.float32, device=dev), torch.empty((B, 2 * K), dtype=torch.int32, device=dev),
            torch.empty((B, 2 * K), dtype=torch.int32, device=dev))
    S, G = 96, 128
    pids = torch.randint(0, V - 10, (B, S), dtype=torch.int32, device=dev)
    width = torch.tensor([S], dtype=torch.int32, device=dev)
    rows = []
    for depth in (1, 3):
        hist = torch.zeros(B * K, G, dtype=torch.int32, device=dev)
        long_words = [w for w in trie_words if len(w) >= depth] or trie_words
        for r in range(B * K):
            w = long_words[r % len(long_words)]
            hist[r, :depth] = torch.tensor((w + w)[:depth], dtype=torch.int32)
        pstate = torch.zeros(B, 5, dtype=torch.int32, device=dev)
        pstate[:, 0] = depth
        off = (1.0, 0, 0, 0, -1)
        rows.append({"B": B, "K": K, "V": V, "depth": depth, "launches": n,
                     "beam_topk_us": event_ms(lambda: ops.beam_topk(logits, special, bs, K, *cand), n),
                     "beam_topk_processed_off_us": event_ms(lambda: ops.beam_topk_processed(logits, special, bs, K, *cand, pids, width,
                                                                                            hist, pstate, off), n),
                     "beam_topk_trie_us": event_ms(lambda: ops.beam_topk_trie(logits, special, bs, K, *cand, pids, width, hist,
                                                                              pstate, None, *csr), n)})
        print(json.dumps(rows[-1]), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=bench.N_LAYERS)
    ap.add_argument("--gens", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("trie_beam_bench needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}), flush=True)
    if a.layers != bench.N_LAYERS:
        import navillm_b200.nav_model as nm
        nm.VICUNA_7B["num_hidden_layers"] = a.layers
    model = bench.build_model(dev, seed=0).eval()
    model._ensure()
    lm = model.lang_model
    lm._decode_states.max_states = 6                                     # one captured graph per arm
    tok = lm.tokenizer
    from navillm_b200.trie import flatten_trie
    V = lm.lm_head.weight.shape[0]
    eqa_trie, eqa_words = make_trie(tok, 64, 1, 3, True, 0)
    t = flatten_trie(eqa_trie, V)
    res = {"gpu": gpu, "layers": a.layers, "kernel": kernel_times(lm, eqa_words, eqa_trie, dev)}
    arms = {"greedy_trie": dict(trie=eqa_trie)}
    arms.update({f"trie_beams_K{K}": dict(trie=eqa_trie, num_beams=K, num_return_sequences=K) for K in (2, 4, 8)})
    res["eqa"] = {"B": 8, "trie_nodes_edges": [t.n_nodes, t.n_edges], "max_new_tokens": 50,
                  "arms": arms_timed(lm, eqa_batch(lm, dev), arms, a.gens, 50)}
    lm._decode_states.clear()
    torch.cuda.empty_cache()
    qa_trie, _ = make_trie(tok, 300, 1, 4, False, 1)
    t = flatten_trie(qa_trie, V)
    wl = bench.WORKLOADS["c3"]
    text, cand = prompts(model, 8, wl["n_cand_tok"], wl["n_text"], dev)
    batch = dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand)
    arms = {"greedy_trie": dict(trie=qa_trie), "trie_beams_K4": dict(trie=qa_trie, num_beams=4),
            "beams_K4_no_trie": dict(num_beams=4)}
    res["3dqa"] = {"B": 8, "S0": int(text["input_ids"].shape[1]), "trie_nodes_edges": [t.n_nodes, t.n_edges], "max_new_tokens": 20,
                   "arms": arms_timed(lm, batch, arms, a.gens, 20)}
    print(json.dumps(res))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
