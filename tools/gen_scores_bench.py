"""The cost of generate(return_dict_in_generate=True, output_scores=True) at Vicuna-7B widths (random init).

    python tools/gen_scores_bench.py [--layers 32] [--gens 3] [--out FILE.json]

Shape: C3 (B = 8, 256 <cand> + 64 text tokens, 128 new tokens, EOS stopping off: random weights would stop at arbitrary steps).
Arms: greedy at B = 8, N = 4 samples per prompt, beams at K = 4 and contrastive search at k = 4, each with the scores off and
on, alternated generation by generation.  Per arm: prefill ms and ms per step (median over the generations after the one that
captures the CUDA graph), the end-of-call copy of the scores (the device time of copying the live [steps, rows, V] block once)
and the peak device memory of one call with no other arm's state held.  The GPU name and power limit are read in the same run.
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

ARMS = {"greedy": {}, "sample_n4": dict(do_sample=True, num_return_sequences=4), "beam_k4": dict(num_beams=4),
        "contrastive_k4": dict(penalty_alpha=0.6, top_k=4)}
SCORES = dict(return_dict_in_generate=True, output_scores=True)


def one(lm, text, cand, new, **kw):
    st = {}
    out = lm.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand, max_new_tokens=new,
                      stop_on_eos=False, use_cuda_graph=True, stats=st, **kw)
    torch.cuda.synchronize()
    steps = st.get("decode_steps") or 1
    return st["prefill_ms"], st["decode_ms"] / steps, out


def peak_gb(lm, text, cand, new, **kw):
    lm._decode_states.clear()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    out = one(lm, text, cand, new, **kw)
    del out
    peak = torch.cuda.max_memory_allocated()
    lm._decode_states.clear()
    torch.cuda.empty_cache()
    return round(peak / 1e9, 2)


def copy_ms(lm):
    """Device time of the end-of-call copy of the most recent state's scores (``generation.take_scores``), median of 5."""
    from navillm_b200 import generation
    st = next(reversed(lm._decode_states.values()))
    n = st.score_cap[0]
    ts = []
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = generation.take_scores(st, n)
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
        del out
    return round(float(np.median(ts)), 3), round(st.scores[:n].numel() * 2 / 1e6, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=bench.N_LAYERS)
    ap.add_argument("--gens", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gen_scores_bench needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    if a.layers != bench.N_LAYERS:
        import navillm_b200.nav_model as nm
        nm.VICUNA_7B["num_hidden_layers"] = a.layers
    model = bench.build_model(dev, seed=0).eval()
    model._ensure()
    lm = model.lang_model
    lm._decode_states.max_states = 2                                   # the off and on states of one arm
    wl = bench.WORKLOADS["c3"]
    B, new = wl["B"], wl["n_new"]
    text, cand = prompts(model, B, wl["n_cand_tok"], wl["n_text"], dev)
    rows = []
    for name, kw in ARMS.items():
        runs = {"off": [], "on": []}
        copy = None
        for _ in range(a.gens + 1):                                     # off and on alternate, generation by generation
            for arm in ("off", "on"):
                torch.manual_seed(0)
                p, s, out = one(lm, text, cand, new, **kw, **(SCORES if arm == "on" else {}))
                runs[arm].append((p, s))
                if arm == "on" and copy is None:
                    copy = copy_ms(lm)
                del out
        r = {"arm": name, "B": B, "new_tokens": new}
        for arm, v in runs.items():
            v = v[1:]                                                   # the first call captures the CUDA graph
            r[arm] = {"prefill_ms": round(float(np.median([x[0] for x in v])), 3),
                      "ms_per_step": round(float(np.median([x[1] for x in v])), 4)}
        r["step_overhead_us"] = round((r["on"]["ms_per_step"] - r["off"]["ms_per_step"]) * 1e3, 1)
        r["end_copy_ms"], r["scores_MB"] = copy
        lm._decode_states.clear()
        torch.cuda.empty_cache()
        for arm in ("off", "on"):
            torch.manual_seed(0)
            r[arm]["peak_GB"] = peak_gb(lm, text, cand, new, **kw, **(SCORES if arm == "on" else {}))
        print(json.dumps(r), flush=True)
        rows.append(r)
    res = {"gpu": gpu, "layers": a.layers, "rows": rows}
    print(json.dumps(res))
    if a.out:
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
