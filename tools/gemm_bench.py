"""Time the wgmma bf16 GEMM on the LLaMA-7B shapes of the path and print TFLOP/s next to cuBLAS
(torch.matmul; comparison bar only, never used by the product), plus the four fused-epilogue GEMMs of the training
step (gate|up + SwiGLU, q|k|v + RoPE, down dgrad + SwiGLU backward, o_proj dgrad + attention row sums).
--tokens defaults to the 10 425 real tokens of bench.py's C2 step.  Every row records the card, its power limit and
the SM clock read right after the timed loop, since the rates only mean something next to those.

    python tools/gemm_bench.py [--tokens 10425] [--json gemm_bench.json]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from navillm_b200 import ops  # noqa: E402


def timeit(fn, iters=10, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    st.record()
    for _ in range(iters):
        fn()
    en.record()
    torch.cuda.synchronize()
    return st.elapsed_time(en) / iters


def smi(query):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        return out or None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=10425)
    ap.add_argument("--json", type=str, default="")
    ap.add_argument("--no-cublas", action="store_true")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    T = a.tokens
    dev = torch.device("cuda:0")
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": smi("power.limit"), "sm_clock_max_mhz": smi("clocks.max.sm")}
    print(json.dumps(card), flush=True)
    d, F = 4096, 11008
    cases = [
        # name, M, N, K, a_mn, b_mn
        ("qkv_fwd", T, 3 * d, d, False, False),
        ("o_fwd", T, d, d, False, False),
        ("gateup_fwd", T, 2 * F, d, False, False),
        ("down_fwd", T, d, F, False, False),
        ("qkv_dgrad", T, d, 3 * d, False, True),
        ("o_dgrad", T, d, d, False, True),
        ("gateup_dgrad", T, d, 2 * F, False, True),
        ("down_dgrad", T, F, d, False, True),
        ("qkv_wgrad", 3 * d, d, T, True, True),
        ("gateup_wgrad", 2 * F, d, T, True, True),
        ("down_wgrad", d, F, T, True, True),
    ]
    rows = []
    for name, M, N, K, a_mn, b_mn in cases:
        A = torch.randn((K, M) if a_mn else (M, K), device=dev, dtype=torch.bfloat16)
        B = torch.randn((K, N) if b_mn else (N, K), device=dev, dtype=torch.bfloat16)
        C = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        flops = 2.0 * M * N * K
        res = {"name": name, "M": M, "N": N, "K": K}
        for bn in (128, 256):
            ms = timeit(lambda: ops.gemm(A, B, a_mn=a_mn, b_mn=b_mn, out=C, block_n=bn), iters=a.iters, warmup=a.warmup)
            res[f"nv_bn{bn}_ms"] = ms
            res[f"nv_bn{bn}_tflops"] = flops / ms / 1e9
            res[f"nv_bn{bn}_sm_clock_mhz"] = smi("clocks.sm")
        if not a.no_cublas:
            At = A.t() if a_mn else A
            Bt = B if b_mn else B.t()
            ms = timeit(lambda: torch.matmul(At, Bt, out=C))
            res["cublas_ms"] = ms
            res["cublas_tflops"] = flops / ms / 1e9
        rows.append(res)
        print(json.dumps(res), flush=True)
        del A, B, C

    # fused epilogues (128 x 256 tile only), each with its rate over its plain counterpart's 256-wide rate in this run
    from navillm_b200.llama import LlamaDims, rope_tables
    g = torch.Generator(device="cpu").manual_seed(0)
    x = (torch.randn(T, d, generator=g) * 0.5).to(dev, torch.bfloat16)
    wgu = (torch.randn(2 * F, d, generator=g) * 0.02).to(dev, torch.bfloat16)
    wqkv = (torch.randn(3 * d, d, generator=g) * 0.02).to(dev, torch.bfloat16)
    wd = (torch.randn(d, F, generator=g) * 0.02).to(dev, torch.bfloat16)
    wo = (torch.randn(d, d, generator=g) * 0.02).to(dev, torch.bfloat16)
    cos_t, sin_t = rope_tables(LlamaDims(), dev)
    pos = (torch.arange(T, device=dev, dtype=torch.int32) % 1024)
    gu = torch.empty(T, 2 * F, device=dev, dtype=torch.bfloat16)
    h = torch.empty(T, F, device=dev, dtype=torch.bfloat16)
    qkv = torch.empty(T, 3 * d, device=dev, dtype=torch.bfloat16)
    dgu = torch.empty(T, 2 * F, device=dev, dtype=torch.bfloat16)
    dout = torch.empty(T, d, device=dev, dtype=torch.bfloat16)
    dvec = torch.empty(32 * T, device=dev, dtype=torch.float32)
    ops.gemm_swiglu(x, wgu, gu=gu, h=h)
    fused = [
        ("gateup_fwd_swiglu", "gateup_fwd", T, 2 * F, d, lambda: ops.gemm_swiglu(x, wgu, gu=gu, h=h)),
        ("qkv_fwd_rope", "qkv_fwd", T, 3 * d, d, lambda: ops.gemm_rope(x, wqkv, pos, cos_t, sin_t, 2 * d, out=qkv)),
        ("down_dgrad_dswiglu", "down_dgrad", T, F, d, lambda: ops.gemm_dswiglu(x, wd, gu, dgu=dgu)),
        ("o_dgrad_attnd", "o_dgrad", T, d, d, lambda: ops.gemm_attnd(x, wo, x, dout=dout, dvec=dvec)),
    ]
    plain = {r["name"]: r["nv_bn256_tflops"] for r in rows}
    for name, plain_name, M, N, K, fn in fused:
        ms = timeit(fn, iters=a.iters, warmup=a.warmup)
        tflops = 2.0 * M * N * K / ms / 1e9
        res = {"name": name, "M": M, "N": N, "K": K, "nv_bn256_ms": ms, "nv_bn256_tflops": tflops,
               "nv_bn256_sm_clock_mhz": smi("clocks.sm"), "plain": plain_name,
               "ratio_to_plain": tflops / plain[plain_name] if plain_name in plain else None}
        rows.append(res)
        print(json.dumps(res), flush=True)
    if a.json:
        Path(a.json).parent.mkdir(parents=True, exist_ok=True)
        Path(a.json).write_text(json.dumps({"card": card, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
