"""Time the wgmma bf16 GEMM on the LLaMA-7B shapes of the path and print TFLOP/s next to cuBLAS
(torch.matmul; comparison bar only, never used by the product).  Run on the GPU box:

    python tools/gemm_bench.py [--tokens 16384] [--json gemm_bench.json]
"""
import argparse
import json
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=16384)
    ap.add_argument("--json", type=str, default="")
    ap.add_argument("--no-cublas", action="store_true")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    T = a.tokens
    dev = torch.device("cuda:0")
    d, F = 4096, 11008
    cases = [
        # name, M, N, K, a_mn, b_mn
        ("qkv_fwd", T, 3 * d, d, False, False),
        ("o_fwd", T, d, d, False, False),
        ("gateup_fwd", T, 2 * F, d, False, False),
        ("down_fwd", T, d, F, False, False),
        ("qkv_dgrad", T, d, 3 * d, False, True),
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
        if not a.no_cublas:
            At = A.t() if a_mn else A
            Bt = B if b_mn else B.t()
            ms = timeit(lambda: torch.matmul(At, Bt, out=C))
            res["cublas_ms"] = ms
            res["cublas_tflops"] = flops / ms / 1e9
        rows.append(res)
        print(json.dumps(res), flush=True)
        del A, B, C
    if a.json:
        Path(a.json).parent.mkdir(parents=True, exist_ok=True)
        Path(a.json).write_text(json.dumps(rows, indent=1))


if __name__ == "__main__":
    main()
