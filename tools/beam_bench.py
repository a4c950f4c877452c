"""Beam search in generate() at Vicuna-7B widths (random init), against greedy decoding of the same prompts.

    python tools/beam_bench.py [--layers 32] [--gens 3] [--out FILE.json]

Shapes: C3 (B = 8, 256 <cand> + 64 text tokens, 128 new tokens) at K = 4, and a ScanQA-like answer length (20 new tokens) at
B = 4 with K in {1, 4}.  EOS stopping is off (random weights would stop at arbitrary steps), so every call runs all its steps.
For each: prefill ms, ms per beam step (median over the generations after the one that captures the CUDA graph), peak device
memory of the call, and greedy decoding at B rows and at B * K rows for comparison.  The GPU name and power limit are read in
the same run.
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
import bench  # noqa: E402


def prompts(model, B, NV, NT, dev):
    lm = model.lang_model
    rng = np.random.RandomState(1234)
    words = [f"w{i}" for i in range(5000)]
    text = lm.tokenize(["Scene " + " ".join(["<cand>"] * NV) + " Question " +
                        " ".join(words[i] for i in rng.randint(0, 5000, size=NT - 5)) + " Answer" for _ in range(B)])
    g = torch.Generator().manual_seed(1234)
    with torch.no_grad():
        view = torch.stack([torch.randn(NV, bench.IMG_FEAT, generator=g) for _ in range(B)], 0).to(dev)
        pano = model.img_embeddings.forward_panorama_per_step(view_img_fts=view, view_lens=torch.full((B,), NV, device=dev))
        cand = model._masked_rows_plus_const(pano["pano_embeds"].reshape(B * NV, -1), np.ones((B, NV), dtype=bool)).detach()
    return text, cand


def timed(lm, text, cand, new, gens, **kw):
    pre, step, peak = [], [], 0
    for i in range(gens + 1):                                            # the first call captures the CUDA graph
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        st = {}
        lm.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand, max_new_tokens=new,
                    stop_on_eos=False, use_cuda_graph=True, stats=st, **kw)
        torch.cuda.synchronize()
        peak = max(peak, torch.cuda.max_memory_allocated())
        if i:
            pre.append(st["prefill_ms"])
            step.append(st["decode_ms"] / st["decode_steps"])
    return {"prefill_ms": round(float(np.median(pre)), 3), "ms_per_step": round(float(np.median(step)), 4),
            "peak_GB": round(peak / 1e9, 2)}


def case(model, dev, B, K, new, gens, NV, NT):
    lm = model.lang_model
    text, cand = prompts(model, B, NV, NT, dev)
    r = {"B": B, "K": K, "new_tokens": new, "S0": int(text["attention_mask"].sum(1).max())}
    if K > 1:
        r["beam"] = timed(lm, text, cand, new, gens, num_beams=K, eos_token_id=-1)
    r["greedy_B"] = timed(lm, text, cand, new, gens)
    if K > 1:
        tb, cb = prompts(model, B * K, NV, NT, dev)
        r["greedy_BK"] = timed(lm, tb, cb, new, gens)
    lm._decode_states.clear()
    torch.cuda.empty_cache()
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=bench.N_LAYERS)
    ap.add_argument("--gens", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("beam_bench needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    if a.layers != bench.N_LAYERS:
        import navillm_b200.nav_model as nm
        nm.VICUNA_7B["num_hidden_layers"] = a.layers
    model = bench.build_model(dev, seed=0).eval()
    model._ensure()
    wl = bench.WORKLOADS["c3"]
    rows = [case(model, dev, wl["B"], 4, wl["n_new"], a.gens, wl["n_cand_tok"], wl["n_text"])]
    for K in (1, 4):
        rows.append(case(model, dev, 4, K, 20, a.gens, wl["n_cand_tok"], wl["n_text"]))
    res = {"gpu": gpu, "layers": a.layers, "rows": rows}
    print(json.dumps(res))
    if a.out:
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
