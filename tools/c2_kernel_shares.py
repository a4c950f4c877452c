"""Where the GPU time of a warm C2 training step goes, per kernel.

Builds bench.py's C2 model and workload, runs warm-up steps, then records --steps steps under torch.profiler (CUDA
activities only).  It writes the Chrome trace and a JSON summary under --out (by default a directory in the system's
temporary directory, so the source tree stays untouched) and prints each kernel's time per step and share of the summed
kernel time.  GEMM kernels keep their template arguments, which name the form: gemm_bf16_wide<A_MN, B_MN, EPI>
(EPI 0 plain, 1 SwiGLU, 2 dSwiGLU, 3 RoPE, 4 attention-backward D) and gemm_bf16_wgmma<BLOCK_N, STAGES, A_MN, B_MN>.
The card, its power limit and the SM clock read after the profiled steps are printed with the table.

    python tools/c2_kernel_shares.py [--out DIR] [--steps 2] [--warmup 2] [--workload c2]
"""
import argparse
import collections
import json
import re
import subprocess
import sys
import tempfile
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402


def smi(query):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        return out or None
    except (OSError, subprocess.SubprocessError):
        return None


def kernel_key(name: str) -> str:
    """The kernel's name with its template arguments, without the parameter list."""
    name = re.sub(r"^void ", "", name)
    depth = 0
    for i, ch in enumerate(name):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            return name[:i]
    return name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=str(Path(tempfile.gettempdir()) / "c2_kernel_shares"))
    ap.add_argument("--workload", default="c2", choices=["c2", "c5"])
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--top", type=int, default=40)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("c2_kernel_shares: needs a CUDA device")
    dev = torch.device("cuda:0")
    out = Path(a.out)
    out.mkdir(parents=True, exist_ok=True)

    wl = bench.WORKLOADS[a.workload]
    model = bench.build_model(dev, seed=0)
    model._ensure()
    host, meta = bench.make_workload(1234, **wl)
    d = {k: v.to(dev) for k, v in host.items()}
    d["target_cols"] = meta["target_cols"].to(dev)
    text = None
    if wl["max_length"] != 1024:
        text = model.lang_model.tokenizer(meta["prompts"], max_length=wl["max_length"], padding=True, truncation=True,
                                          return_tensors="pt", add_special_tokens=True, return_token_type_ids=True)
    text = text or model.lang_model.tokenize(meta["prompts"])

    def step():
        model.zero_grad(lazy=True)
        loss = bench.nav_step(model, d, meta, dev, text=text)
        loss.backward()

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            step()
        torch.cuda.synchronize()
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": smi("power.limit"), "sm_clock_mhz": smi("clocks.sm"),
            "workload": a.workload, "steps": a.steps}
    trace = out / f"{a.workload}_trace.json"
    prof.export_chrome_trace(str(trace))

    events = json.loads(trace.read_text())["traceEvents"]
    per = collections.defaultdict(lambda: [0.0, 0])
    for e in events:
        if e.get("cat") == "kernel":
            k = per[kernel_key(e["name"])]
            k[0] += e["dur"] / 1e3
            k[1] += 1
    total = sum(v[0] for v in per.values())
    gemm = sum(v[0] for k, v in per.items() if "gemm" in k)
    rows = sorted(per.items(), key=lambda kv: -kv[1][0])
    summary = {"card": card, "kernel_ms_per_step": total / a.steps, "gemm_share": gemm / total if total else None,
               "kernels": [{"kernel": k, "ms_per_step": v[0] / a.steps, "launches_per_step": v[1] / a.steps,
                            "share": v[0] / total} for k, v in rows]}
    (out / f"{a.workload}_kernel_shares.json").write_text(json.dumps(summary, indent=1))
    print(json.dumps(card))
    print(f"summed kernel time {total / a.steps:.1f} ms per step, GEMMs {100 * gemm / total:.1f} %")
    print(f"{'share':>7} {'ms/step':>9} {'launches':>8}  kernel")
    for k, v in rows[:a.top]:
        print(f"{100 * v[0] / total:6.2f}% {v[0] / a.steps:9.2f} {v[1] / a.steps:8.0f}  {k}")


if __name__ == "__main__":
    main()
