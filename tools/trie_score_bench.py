"""Answer scoring (score_answers) at Vicuna-7B widths (random init), against greedy decoding under the trie and trie beams.

    python tools/trie_score_bench.py [--layers 32] [--gens 3] [--out FILE.json]

The shapes and tries of tools/trie_beam_bench.py:
(i)   EQA shape: B = 8 EQA prompts, the trie of 64 answers of 1-3 tokens after BOS (133 nodes).  Arms: score_answers, greedy
      under the trie (max_new_tokens 50), trie beams at K = 4 and 8.
(ii)  3dqa shape: the C3 prompt, B = 8, a trie of 300 answers of 1-4 tokens.  Arms: score_answers, greedy under the trie and
      trie beams at K = 4 (max_new_tokens 20).
Per arm: ms per call (host clock around a synchronised call), score_answers' prefill / tree / score split and peak memory,
medians over --gens calls after a warm-up call; the arms alternate call by call.
(iii) The tree attention alone: nv_attn_fwd_tree against nv_attn_fwd_kv (causal) on the same rows (B = 8 prompts of the EQA
      shape's length, its 132 tree rows each, 32 heads), CUDA events over 50 launches.
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
from constrained_decode_bench import timed  # noqa: E402
from trie_beam_bench import eqa_batch, make_trie  # noqa: E402


def arms_timed(lm, batch, arms, gens, new):
    res = {name: [] for name in arms}
    for i in range(gens + 1):
        for name, kw in arms.items():
            torch.cuda.reset_peak_memory_stats()
            st = {}
            if kw.get("score"):
                ms, _ = timed(lambda: lm.score_answers(batch["input_ids"], batch["attention_mask"], kw["trie"],
                                                       cand_vis=batch.get("cand_vis"), hist_vis=batch.get("hist_vis"), stats=st))
                split = (st["prefill_ms"], st["tree_ms"], st["score_ms"], st["tree_rows"], st["chunks"])
            else:
                ms, _ = timed(lambda: lm.generate(**batch, max_new_tokens=new, use_cuda_graph=True, stats=st,
                                                  **{k: v for k, v in kw.items() if k != "score"}))
                split = (st["prefill_ms"], None, None, None, None)
            if i:
                res[name].append((ms, *split, torch.cuda.max_memory_allocated() / 2 ** 30))
    out = {}
    med = lambda v, j: None if v[0][j] is None else round(float(np.median([x[j] for x in v])), 3)
    for name, v in res.items():
        out[name] = {"ms_per_call": med(v, 0), "ms_spread": round(float(max(x[0] for x in v) - min(x[0] for x in v)), 3),
                     "prefill_ms": med(v, 1), "tree_ms": med(v, 2), "score_ms": med(v, 3), "tree_rows": v[-1][4],
                     "chunks": v[-1][5], "peak_gib": round(max(x[6] for x in v), 2)}
        print(json.dumps({name: out[name]}), flush=True)
    return out


def attention_times(lm, rows, S, dev, B=8, n=50):
    """nv_attn_fwd_tree and nv_attn_fwd_kv on B prompts of S cached keys and the N tree rows each."""
    from contrastive_bench import event_ms
    from navillm_b200 import ops
    H, N = lm.dims.n_heads, rows.n
    Smax = (S + N + 127) // 128 * 128
    g = torch.Generator(device=dev).manual_seed(0)
    kc = torch.randn(B, Smax, H * 128, generator=g, device=dev).to(torch.bfloat16)
    vc = torch.randn(B, Smax, H * 128, generator=g, device=dev).to(torch.bfloat16)
    q = torch.randn(B * N, H * 128, generator=g, device=dev).to(torch.bfloat16)
    i32 = lambda x: torch.tensor(x, dtype=torch.int32, device=dev)
    cu, kv_start, kv_len = i32([b * N for b in range(B + 1)]), i32([b * Smax for b in range(B)]), i32([S + N] * B)
    end = torch.from_numpy(rows.end).to(dev)
    r = {"B": B, "cached": S, "tree_rows": N, "heads": H, "launches": n,
         "attn_fwd_tree_us": event_ms(lambda: ops.attn_fwd_tree(q, kc, vc, cu, [N] * B, kv_start, kv_len, end, H), n),
         "attn_fwd_kv_us": event_ms(lambda: ops.attn_fwd_kv(q, kc, vc, cu, [N] * B, kv_start, kv_len, H), n)}
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=bench.N_LAYERS)
    ap.add_argument("--gens", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("trie_score_bench needs a CUDA device (there is no CPU path)")
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
    lm._decode_states.max_states = 6
    tok = lm.tokenizer
    from navillm_b200.trie import flatten_trie, tree_rows
    V = lm.lm_head.weight.shape[0]
    eqa_trie, _ = make_trie(tok, 64, 1, 3, True, 0)
    t = flatten_trie(eqa_trie, V)
    rows = tree_rows(t)
    batch = eqa_batch(lm, dev)
    res = {"gpu": gpu, "layers": a.layers,
           "attention": attention_times(lm, rows, int(batch["attention_mask"].sum(1).max()), dev)}
    arms = {"score_answers": dict(score=True, trie=eqa_trie), "greedy_trie": dict(trie=eqa_trie),
            "trie_beams_K4": dict(trie=eqa_trie, num_beams=4, num_return_sequences=4),
            "trie_beams_K8": dict(trie=eqa_trie, num_beams=8, num_return_sequences=8)}
    res["eqa"] = {"B": 8, "trie_nodes": t.n_nodes, "answers": len(rows.paths), "arms": arms_timed(lm, batch, arms, a.gens, 50)}
    lm._decode_states.clear()
    torch.cuda.empty_cache()
    qa_trie, _ = make_trie(tok, 300, 1, 4, False, 1)
    t = flatten_trie(qa_trie, V)
    wl = bench.WORKLOADS["c3"]
    text, cand = prompts(model, 8, wl["n_cand_tok"], wl["n_text"], dev)
    batch = dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand)
    arms = {"score_answers": dict(score=True, trie=qa_trie), "greedy_trie": dict(trie=qa_trie),
            "trie_beams_K4": dict(trie=qa_trie, num_beams=4)}
    res["3dqa"] = {"B": 8, "S0": int(text["input_ids"].shape[1]), "trie_nodes": t.n_nodes,
                   "answers": len(tree_rows(t).paths), "arms": arms_timed(lm, batch, arms, a.gens, 20)}
    print(json.dumps(res))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
