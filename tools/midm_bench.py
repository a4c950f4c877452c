"""Time the mid-M GEMM shapes (16 < M < 1024 activation rows: C1, evaluation rollouts, prefix-reuse suffixes) of
Vicuna-7B for every tile variant of nv_gemm_bf16 and report the weight-streaming bandwidth.
Usage: python tools/midm_bench.py [M ...]
       python tools/midm_bench.py --fp8 [M ...]   bf16 weights (nv_gemm_bf16) against their fp8 copy (nv_gemm_fp8w_bf16), auto
                                                  tiles, timed in alternation; also checks that both give the same bits"""
import statistics
import subprocess
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


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def fp8_table(Ms):
    """Per shape and M: bf16 and fp8 times (median of 7 alternating rounds) and the bytes each one moves per second
    (weights + activations in + out, the fp8 weight as e4m3 bytes plus one exponent per row)."""
    dev = torch.device("cuda:0")
    print(f"# {gpu_info()}", flush=True)
    for name, N, K, add in (("qkv", 12288, 4096, False), ("o", 4096, 4096, True), ("gateup", 22016, 4096, False),
                            ("down", 4096, 11008, True), ("lm_head", 32006, 4096, False)):
        nw = max(2, (2 << 30) // (N * K * 3))                            # rotate > L2 worth of weights: they come from HBM
        ws = [(torch.randn(N, K, device=dev) * 0.02).to(torch.bfloat16) for _ in range(nw)]
        qs = []
        for w in ws:
            q = torch.empty((N, K), dtype=ops.fp8, device=dev)
            e = torch.empty(N, dtype=torch.int8, device=dev)
            ops.quantize_fp8_(w, q, e)
            qs.append((q, e))
        for M in Ms:
            x = torch.randn(M, K, device=dev).to(torch.bfloat16)
            a = torch.randn(M, N, device=dev).to(torch.bfloat16) if add else None
            out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            i = [0]

            def f16():
                ops.gemm(x, ws[i[0] % nw], addend=a, out=out)
                i[0] += 1

            def f8():
                ops.gemm_fp8w(x, *qs[i[0] % nw], addend=a, out=out)
                i[0] += 1
            t16, t8 = [], []
            for _ in range(7):
                t16.append(timeit(f16))
                t8.append(timeit(f8))
            ms16, ms8 = statistics.median(t16), statistics.median(t8)
            ref = ops.gemm(x, ws[0], addend=a).clone()
            same = torch.equal(ops.gemm_fp8w(x, *qs[0], addend=a), ref)
            act = (M * K + M * N * (2 if add else 1)) * 2
            gb16, gb8 = (N * K * 2 + act) / ms16 / 1e6, (N * K + N + act) / ms8 / 1e6
            print(f"{name:7s} M={M:4d}: bf16 {ms16 * 1e3:7.1f}us {gb16:6.0f}GB/s | fp8 {ms8 * 1e3:7.1f}us {gb8:6.0f}GB/s | "
                  f"speedup {ms16 / ms8:4.2f}x | bitwise {'equal' if same else 'DIFFERENT'}", flush=True)
        del ws, qs


def main():
    if sys.argv[1:2] == ["--fp8"]:
        fp8_table([int(a) for a in sys.argv[2:]] or [17, 32, 64, 96, 128, 192, 256, 384, 512])
        return
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
