"""Time the mid-M GEMM shapes (16 < M < 1024 activation rows: C1, evaluation rollouts, prefix-reuse suffixes) of
Vicuna-7B for every tile variant of nv_gemm_bf16 and report the weight-streaming bandwidth.
Usage: python tools/midm_bench.py [M ...]"""
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from navillm_b200 import ops  # noqa: E402


def timeit(fn, iters=24, warmup=4):
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
    dev = torch.device("cuda:0")
    Ms = [int(a) for a in sys.argv[1:]] or [48, 128, 192, 256, 384, 640]
    variants = [("bn32", 32), ("bn128", 128), ("bn256", 256), ("auto", 0)]
    if hasattr(ops, "gemm_stream"):
        variants.append(("stream", -1))
    for name, N, K in (("qkv", 12288, 4096), ("o", 4096, 4096), ("gateup", 22016, 4096), ("down", 4096, 11008)):
        ws = [torch.randn(N, K, device=dev, dtype=torch.bfloat16) for _ in range(8)]   # rotate: weights come from HBM
        for M in Ms:
            x = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
            out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            ref = None
            line = []
            for tag, bn in variants:
                if bn == 32 and M > 128:
                    continue
                i = [0]

                def f():
                    if bn == -1:
                        ops.gemm_stream(x, ws[i[0] % 8], out=out)
                    else:
                        ops.gemm(x, ws[i[0] % 8], out=out, block_n=bn)
                    i[0] += 1
                try:
                    ms = timeit(f)
                except Exception as e:
                    line.append(f"{tag}: {type(e).__name__}")
                    continue
                i[0] = 0
                f()
                if ref is None:
                    ref = out.clone()
                    same = ""
                else:
                    same = "" if torch.equal(out, ref) else f" (maxdiff {float((out.float() - ref.float()).abs().max()):.3g})"
                line.append(f"{tag} {ms * 1e3:6.1f}us {N * K * 2 / ms / 1e9:5.2f}TB/s{same}")
            print(f"{name:6s} M={M:4d}: " + " | ".join(line), flush=True)
        del ws


if __name__ == "__main__":
    main()
