"""bf16 activations against fp8 activations (W8A8, set_activation_dtype("fp8")) in the no-grad prompt forwards.

(i)   GEMM table: nv_gemm_bf16 on W' against nv_quantize_act_fp8 + nv_gemm_w8a8_bf16 on the fp8 copy, the four Vicuna-7B
      decoder-layer shapes at M = 64 .. 10425, arms alternated; TFLOP/s of each arm (2 M N K over the arm's time, the quantize
      pass included for W8A8) and the quantize pass's share of that W8A8 arm (not of the layer time).
(ii)  Rollouts on Vicuna-7B random init (quantize_weights_fp8() first, so both arms use W'): the prefix-cached navigation
      rollout in ms/step at B = 8 and 32 over the bf16 PrefixKVCache and at B = 64 over the fp8 one, and a no-grad navigation
      step without a cache at B = 16.  One cache per arm, both arms in lock-step with the order alternated per step; the
      largest |d fuse_logits| / max|logit| between the arms is reported, not asserted.
(iii) The GPU name and power limit, read in the same run.
Not covered here: the C3 prefill time, generate() token agreement on Vicuna-7B and the quantize passes' share of the layer
time.

    python tools/fp8_act_bench.py [--gemm-only] [--steps 5]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import bench  # noqa: E402
from navillm_b200 import ops  # noqa: E402

SHAPES = [("qkv", 12288, 4096), ("o", 4096, 4096), ("gateup", 22016, 4096), ("down", 4096, 11008)]
MS = [64, 128, 256, 512, 1024, 2048, 4096, 10425]


def gpu_info() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def _time(fn, iters):
    st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    st.record()
    for _ in range(iters):
        fn()
    en.record()
    torch.cuda.synchronize()
    return st.elapsed_time(en) / iters


def gemm_table(dev, iters=20, rounds=3):
    g = torch.Generator(device=dev).manual_seed(0)
    rows = []
    for name, N, K in SHAPES:
        w = (torch.randn(N, K, generator=g, device=dev) * 0.02).to(torch.bfloat16)
        wq = torch.empty((N, K), dtype=ops.fp8, device=dev)
        we = torch.empty(N, dtype=torch.int8, device=dev)
        ops.quantize_fp8_(w, wq, we)
        for M in MS:
            x = torch.randn(M, K, generator=g, device=dev).to(torch.bfloat16)
            c16 = torch.empty((M, N), dtype=torch.bfloat16, device=dev)
            c8 = torch.empty_like(c16)
            aq = torch.empty((M, K), dtype=ops.fp8, device=dev)
            ae = torch.empty((M, K // 128), dtype=torch.int8, device=dev)
            arms = {"bf16": lambda: ops.gemm(x, w, out=c16),
                    "w8a8": lambda: ops.gemm_w8a8(*ops.quantize_act_fp8(x, q=aq, e=ae), wq, we, out=c8),
                    "quant": lambda: ops.quantize_act_fp8(x, q=aq, e=ae)}
            for f in arms.values():
                f()
            torch.cuda.synchronize()
            ms = {k: [] for k in arms}
            for r in range(rounds):
                for k in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
                    ms[k].append(_time(arms[k], iters))
            t = {k: float(np.median(v)) for k, v in ms.items()}
            flop = 2.0 * M * N * K
            rel = float((c8.float() - c16.float()).abs().max() / c16.float().abs().max())
            row = {"shape": name, "M": M, "N": N, "K": K, "bf16_ms": round(t["bf16"], 4), "w8a8_ms": round(t["w8a8"], 4),
                   "bf16_TFLOPs": round(flop / t["bf16"] / 1e9, 1), "w8a8_TFLOPs": round(flop / t["w8a8"] / 1e9, 1),
                   "speedup": round(t["bf16"] / t["w8a8"], 3), "quant_share_of_w8a8_gemm": round(t["quant"] / t["w8a8"], 3),
                   "max_rel_diff": rel}
            rows.append(row)
            print(json.dumps(row), flush=True)
    return rows


def rollout(model, dev, B, kv_dtype, steps, cache=True, max_len=1024):
    """Both activation modes in lock-step, one cache each, arm order alternated per step."""
    from navillm_b200.modified_lm import PrefixKVCache
    from tools.prefix_reuse_bench import make_step
    lm = model.lang_model
    rng = np.random.RandomState(0)
    g = torch.Generator().manual_seed(0)
    D, G, n_cand = 4096, 64, 12
    words = [f"w{i}" for i in range(5000)]
    instr = [" ".join(words[i] for i in rng.randint(0, 5000, size=rng.randint(60, 100))) for _ in range(B)]
    hist = [[] for _ in range(B)]
    caches = {m: (PrefixKVCache(lm, batch_size=B, max_len=max_len, kv_dtype=kv_dtype) if cache else None) for m in ("bf16", "fp8")}
    to_dev = lambda b: {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in b.items()}
    ev = lambda: torch.cuda.Event(enable_timing=True)
    rows, max_rel = [], 0.0
    with torch.no_grad():
        for t in range(steps):
            batch = to_dev(make_step(rng, g, B, t, instr, n_cand, D, G))
            batch["hist_vis"] = [list(h) for h in hist]
            out, ms = {}, {}
            for mode in (("fp8", "bf16") if t % 2 == 0 else ("bf16", "fp8")):
                model.set_activation_dtype(mode)
                e0, e1 = ev(), ev()
                torch.manual_seed(t); e0.record()
                kw = {"prefix_cache": caches[mode]} if cache else {}
                out[mode] = model("navigation", dict(batch), **kw)
                e1.record(); torch.cuda.synchronize()
                ms[mode] = e0.elapsed_time(e1)
            r, c = out["bf16"]["fuse_logits"].float(), out["fp8"]["fuse_logits"].float()
            fin = torch.isfinite(r)
            max_rel = max(max_rel, ((r[fin] - c[fin]).abs().max() / r[fin].abs().max()).item())
            rows.append(ms)
            for b in range(B):
                hist[b].append(out["bf16"]["fuse_embeds"][b, 1 + (t % 3)].float())
    model.set_activation_dtype("bf16")
    timed = rows[1:] or rows                                   # the first step encodes whole prompts (and warms up)
    res = {"B": B, "cache": kv_dtype if cache else None, "steps_timed": len(timed)}
    for m in ("bf16", "fp8"):
        res[f"{m}_act_ms_per_step"] = round(sum(r[m] for r in timed) / len(timed), 2)
    res["speedup"] = round(res["bf16_act_ms_per_step"] / res["fp8_act_ms_per_step"], 3)
    res["max_rel_fuse_logit_diff"] = max_rel
    print(json.dumps(res), flush=True)
    del caches
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gemm-only", action="store_true")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--json", type=str, default="")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    res = {"gpu": gpu_info(), "gemm": gemm_table(dev)}
    if not a.gemm_only:
        model = bench.build_model(dev).eval()
        model.quantize_weights_fp8()
        res["rollouts"] = [rollout(model, dev, 8, "bf16", a.steps), rollout(model, dev, 32, "bf16", a.steps),
                           rollout(model, dev, 64, "fp8", a.steps), rollout(model, dev, 16, "bf16", a.steps, cache=False)]
    res["gpu_after"] = gpu_info()
    print(json.dumps({"gpu": res["gpu"], "gpu_after": res["gpu_after"]}), flush=True)
    if a.json:
        Path(a.json).parent.mkdir(parents=True, exist_ok=True)
        Path(a.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
