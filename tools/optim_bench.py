"""FlatAdamW.step(max_grad_norm=40.0) at Vicuna-7B size, plain vs compensated, and the fidelity of both updates.

    python tools/optim_bench.py [--rounds 7] [--steps 10] [--skip-fidelity]

Builds bench.py's Vicuna-7B NavModel (bf16 LM flat of ~6.7 B parameters plus the fp32 encoder flat), gives it seeded
gradients, and makes one compensated FlatAdamW over it: W, G, m, v and r of the bf16 buffer take 5 x 2 bytes per LM
parameter (67.4 GB).  The plain arm is a shallow copy of that optimizer without the residual, so both arms step the same
buffers and no second set of moments is allocated.  Rounds alternate the arms; a round runs one untimed step per arm
(the compensated arm's first step after a plain one zeroes the residual, because the plain step wrote the weights) and then
`--steps` steps timed with CUDA events.  Reports the median ms per step, the bytes the update moves per step (sum of
squares 1 x, update 7 x or 9 x the bf16 buffer's bytes; 4 x and 7 x the fp32 buffer's), that over the time as GB/s, and
its share of the H100 SXM data sheet's 3.35 TB/s.  Then runs the trajectory of tests/test_optim_compensated_gpu.py
(4 M weights, 300 steps at lr 3e-5) and prints its drift ratio and relative drift error for both arms.  One JSON line.
"""
from __future__ import annotations

import argparse
import copy
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402

HBM_GBS = 3350.0        # H100 SXM data sheet, for a card allowed 700 W


def card_info() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
    if out:
        pw, clk = (s.strip() for s in out[0].split(","))
        info.update(power_limit_w=float(pw), max_sm_clock_mhz=float(clk))
    return info


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--skip-fidelity", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("optim_bench.py needs a GPU")
    from navillm_b200.optim import FlatAdamW
    dev = torch.device("cuda:0")
    res = {"gpu": card_info()}

    model = bench.build_model(dev, seed=0)
    model._ensure()
    lm, enc = model.lang_model.flat, model._flat32
    gen = torch.Generator(device=dev).manual_seed(0)
    for f in (lm, enc):
        f.flat_grad.normal_(0.0, 1e-3, generator=gen)
    comp = FlatAdamW(model, lr=3e-5, compensated=True)
    plain = copy.copy(comp)
    plain.residual = None
    n16, n32 = lm.flat.numel(), enc.flat.numel()
    res.update(lm_params=n16, encoder_params=n32, bf16_buffers_gb=5 * 2 * n16 / 1e9,
               peak_allocated_gb=torch.cuda.max_memory_allocated() / 1e9)

    def moved(compensated: bool) -> int:
        return 2 * n16 * (1 + (9 if compensated else 7)) + 4 * n32 * (1 + 7)

    times = {"plain": [], "compensated": []}
    arms = {"plain": plain, "compensated": comp}
    for _ in range(a.rounds):
        for name, opt in arms.items():
            opt.step(max_grad_norm=40.0)                           # untimed: residual reset after the other arm's write
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                opt.step(max_grad_norm=40.0)
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / a.steps)
    for name in arms:
        ms = statistics.median(times[name])
        gbs = moved(name == "compensated") / (ms / 1e3) / 1e9
        res[name] = {"ms_per_step": round(ms, 3), "ms_rounds": [round(t, 3) for t in times[name]],
                     "bytes_per_step": moved(name == "compensated"), "gb_per_s": round(gbs, 1),
                     "share_of_3350_gbs": round(gbs / HBM_GBS, 3)}
    res["compensated_over_plain"] = round(res["compensated"]["ms_per_step"] / res["plain"]["ms_per_step"], 3)
    del comp, plain, model
    torch.cuda.empty_cache()

    if not a.skip_fidelity:
        from tests.test_optim_compensated_gpu import trajectory
        res["fidelity"] = trajectory(dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
