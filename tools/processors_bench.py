"""Cost of HF's logits processors in generate() at C3's shape (Vicuna-7B widths, random init): ms per decode step with the
processors off and on (repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=4), the two arms alternated call by call;
greedy at B = 8 / 32 / 64, beams at B = 8, K = 4, and N = 4 samples of B = 8 prompts.  Then the kernels alone: nv_logits_process
and nv_beam_topk_processed vs nv_beam_topk, µs per launch (CUDA events over many launches).

    python tools/processors_bench.py [--layers 32] [--gens 3] [--out FILE.json]

EOS stopping is off, so every call runs all its steps.  The GPU name and power limit are read in the same run.
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

PROC = dict(repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=4)


def alternated(lm, text, cand, new, gens, **kw):
    """Median ms per decode step of the off and on arms, alternated; the first call of each arm captures its graph."""
    ms = {"off": [], "on": []}
    for i in range(gens + 1):
        for arm in ("off", "on"):
            st = {}
            lm.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand, max_new_tokens=new,
                        stop_on_eos=False, use_cuda_graph=True, stats=st, eos_token_id=-1 if kw.get("num_beams", 1) > 1 else None,
                        **kw, **(PROC if arm == "on" else {}))
            torch.cuda.synchronize()
            if i:
                ms[arm].append(st["decode_ms"] / st["decode_steps"])
    off, on = float(np.median(ms["off"])), float(np.median(ms["on"]))
    return {"ms_per_step_off": round(off, 4), "ms_per_step_on": round(on, 4), "overhead_pct": round(100 * (on / off - 1), 2)}


def kernel_us(fn, n=200):
    for _ in range(10):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return round(1e3 * a.elapsed_time(b) / n, 2)


def kernels(dev, V=32006, S=320, t=64, G=128):
    from navillm_b200 import ops
    proc = (1.3, 3, 0, 4, 2)
    out = {}
    for R in (8, 32, 64):
        logits = torch.randn(R, V, device=dev).to(torch.bfloat16)
        pids = torch.randint(0, V, (R, S), device=dev, dtype=torch.int32)
        width = torch.tensor([S], dtype=torch.int32, device=dev)
        hist = torch.randint(0, V, (R, G), device=dev, dtype=torch.int32)
        hl = torch.full((R,), t, dtype=torch.int32, device=dev)
        out[f"logits_process_R{R}_us"] = kernel_us(lambda: ops.logits_process_(logits, pids, width, hist, hl, None, proc))
    B, K = 8, 4
    logits = torch.randn(B * K, V, device=dev).to(torch.bfloat16)
    special = torch.tensor([32000, 32001, 32002, 32003, 32004], dtype=torch.int32, device=dev)
    bs = torch.zeros(B * K, device=dev)
    cs, ct, cp = (torch.empty((B, 2 * K), dtype=dt, device=dev) for dt in (torch.float32, torch.int32, torch.int32))
    pids = torch.randint(0, V, (B, S), device=dev, dtype=torch.int32)
    hist = torch.randint(0, V, (B * K, G), device=dev, dtype=torch.int32)
    pstate = torch.zeros(B, 5, dtype=torch.int32, device=dev)
    pstate[:, 0] = t
    out["beam_topk_B8K4_us"] = kernel_us(lambda: ops.beam_topk(logits, special, bs, K, cs, ct, cp))
    out["beam_topk_processed_B8K4_us"] = kernel_us(lambda: ops.beam_topk_processed(logits, special, bs, K, cs, ct, cp, pids, width, hist,
                                                                                    pstate, proc))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=bench.N_LAYERS)
    ap.add_argument("--gens", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("processors_bench needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    if a.layers != bench.N_LAYERS:
        import navillm_b200.nav_model as nm
        nm.VICUNA_7B["num_hidden_layers"] = a.layers
    model = bench.build_model(dev, seed=0).eval()
    model._ensure()
    lm = model.lang_model
    wl = bench.WORKLOADS["c3"]
    rows = []
    for B, kw in ((8, {}), (32, {}), (64, {}), (8, dict(num_beams=4)), (8, dict(do_sample=True, num_return_sequences=4))):
        text, cand = prompts(model, B, wl["n_cand_tok"], wl["n_text"], dev)
        r = {"B": B, **{k: v for k, v in kw.items()}, "new_tokens": wl["n_new"]}
        r.update(alternated(lm, text, cand, wl["n_new"], a.gens, **kw))
        lm._decode_states.clear()
        torch.cuda.empty_cache()
        print(json.dumps(r), flush=True)
        rows.append(r)
    res = {"gpu": gpu, "layers": a.layers, "rows": rows, "kernels": kernels(dev)}
    print(json.dumps(res))
    if a.out:
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
