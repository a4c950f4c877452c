"""FlatAdamW.step(max_grad_norm=40.0) at Vicuna-7B size with bf16 and 8-bit moments, plain and compensated, and the
fidelity of the 8-bit moments.

    python tools/optim8_bench.py [--rounds 5] [--steps 10] [--skip-fidelity]

Builds bench.py's Vicuna-7B NavModel (bf16 LM flat of ~6.7 B parameters plus the fp32 encoder flat) and gives it seeded
gradients.  The bf16-moment and 8-bit-moment optimizers do not fit on one 80 GB card together (W, G, r and both sets of
moments come to ~82 GB), so each round makes one compensated FlatAdamW per moment format in turn, times it and a shallow
copy of it without the residual (the plain arm: same buffers), then frees it.  A round runs the four arms one after the
other, each with one untimed step (the compensated arm's first step after a plain one zeroes the residual, because the
plain step wrote the weights) and `--steps` steps timed with CUDA events.  Reports the median ms per step, the state bytes,
the bytes a step moves (sum of squares 2 bytes per LM parameter; update 14 / 18 bytes with bf16 moments, 10.25 / 14.25
with 8-bit ones, plain / compensated; the fp32 buffer's 4 + 28 bytes), that over the time as GB/s and its share of the
H100 SXM data sheet's 3.35 TB/s.  Then the trajectory and moment-tracking runs of tests/test_optim_8bit_gpu.py.  One JSON
line.
"""
from __future__ import annotations

import argparse
import copy
import gc
import json
import statistics
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import bench  # noqa: E402
from optim_bench import HBM_GBS, card_info  # noqa: E402

ARMS = ("plain_bf16", "compensated_bf16", "plain_8bit", "compensated_8bit")


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--skip-fidelity", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("optim8_bench.py needs a GPU")
    from navillm_b200.optim import FlatAdamW
    dev = torch.device("cuda:0")
    res = {"gpu": card_info()}

    model = bench.build_model(dev, seed=0)
    model._ensure()
    lm, enc = model.lang_model.flat, model._flat32
    gen = torch.Generator(device=dev).manual_seed(0)
    for f in (lm, enc):
        f.flat_grad.normal_(0.0, 1e-3, generator=gen)
    n16, n32 = lm.flat.numel(), enc.flat.numel()
    res.update(lm_params=n16, encoder_params=n32)

    def moved(arm: str) -> float:
        upd = {"plain_bf16": 14, "compensated_bf16": 18, "plain_8bit": 10.25, "compensated_8bit": 14.25}[arm]
        return n16 * (2 + upd) + n32 * (4 + 28)

    times = {arm: [] for arm in ARMS}
    state_bytes, peak = {}, {}
    for _ in range(a.rounds):
        for moments in ("bf16", "8bit"):
            torch.cuda.reset_peak_memory_stats()
            comp = FlatAdamW(model, lr=3e-5, compensated=True, moments=moments)
            plain = copy.copy(comp)
            plain.residual = None
            state_bytes[f"plain_{moments}"] = comp.state_bytes() - 2 * n16
            state_bytes[f"compensated_{moments}"] = comp.state_bytes()
            for arm, opt in ((f"plain_{moments}", plain), (f"compensated_{moments}", comp)):
                opt.step(max_grad_norm=40.0)                       # untimed: residual reset after the other arm's write
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.steps):
                    opt.step(max_grad_norm=40.0)
                e1.record()
                torch.cuda.synchronize()
                times[arm].append(e0.elapsed_time(e1) / a.steps)
            peak[moments] = torch.cuda.max_memory_allocated() / 1e9
            del comp, plain, opt
            gc.collect()
            torch.cuda.empty_cache()
    for arm in ARMS:
        ms = statistics.median(times[arm])
        gbs = moved(arm) / (ms / 1e3) / 1e9
        res[arm] = {"ms_per_step": round(ms, 3), "ms_rounds": [round(t, 3) for t in times[arm]],
                    "state_gb": round(state_bytes[arm] / 1e9, 2), "bytes_per_step": int(moved(arm)),
                    "gb_per_s": round(gbs, 1), "share_of_3350_gbs": round(gbs / HBM_GBS, 3)}
    res["peak_allocated_gb"] = {k: round(v, 2) for k, v in peak.items()}
    res["plain_8bit_over_bf16"] = round(res["plain_8bit"]["ms_per_step"] / res["plain_bf16"]["ms_per_step"], 3)
    res["compensated_8bit_over_bf16"] = round(res["compensated_8bit"]["ms_per_step"] /
                                              res["compensated_bf16"]["ms_per_step"], 3)
    del model
    gc.collect()
    torch.cuda.empty_cache()

    if not a.skip_fidelity:
        from tests.test_optim_8bit_gpu import moment_tracking, trajectory8
        res["trajectory"] = trajectory8(dev)
        res["moment_tracking"] = moment_tracking(dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
