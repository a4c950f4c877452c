"""GPTQ-calibrated int4 weights (quantize_weights_int4(calibration=...)) at Vicuna-7B widths, random init, in one process.

    python tools/int4_gptq_bench.py [--layers 32] [--reps 3] [--quality-layers 0 15 31] [--out FILE.json]

(i)   Calibration: C3-shaped prompt forwards (B = 8, 256 <cand> + 64 text tokens, the prefill of generate() with one new
      token) and C2-shaped no-grad navigation batches (B = 16, seq U{256..1024}), each timed with and without an open
      calibration, the two alternated over ``reps`` rounds; the calibration's size and the peak device memory.
(ii)  Quantization: total wall time of quantize_weights_int4(calibration=...), split by CUDA events into the
      factorisation (ops.gptq_factor, including the positive-definiteness check before any weight is written), the block
      kernels (nv_gptq_int4_block) and the trailing updates (nv_sgemm); the block kernel's time per launch at each weight
      shape; the peak device memory.
(iii) Quality, on random-init weights (says nothing about task metrics): for the linears of ``quality-layers``, the loss
      tr(dW H dW^T) of GPTQ over that of round to nearest, with H recorded on held-out prompts and batches.
(iv)  The GPU's name, power limit and max SM clock, read in the same run.
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from navillm_b200 import _lib, ops  # noqa: E402


def max_sm_clock():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def c3_inputs(model, dev, seed):
    wl = bench.WORKLOADS["c3"]
    B, NV, NT = wl["B"], wl["n_cand_tok"], wl["n_text"]
    lm = model.lang_model
    rng = np.random.RandomState(seed)
    prompts = ["Scene " + " ".join(["<cand>"] * NV) + " Question " + " ".join(f"w{i}" for i in rng.randint(0, 5000, size=NT - 5))
               + " Answer" for _ in range(B)]
    text = lm.tokenize(prompts)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        view = torch.stack([torch.randn(NV, bench.IMG_FEAT, generator=g) for _ in range(B)], 0).to(dev)
        pano = model.img_embeddings.forward_panorama_per_step(view_img_fts=view, view_lens=torch.full((B,), NV, device=dev))
        cand = model._masked_rows_plus_const(pano["pano_embeds"].reshape(B * NV, -1), np.ones((B, NV), dtype=bool)).detach()
    return lambda: lm.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand,
                               max_new_tokens=1, stop_on_eos=False, use_cuda_graph=False)


def c2_inputs(model, dev, seed):
    host, meta = bench.make_workload(seed, **bench.WORKLOADS["c2"])
    dev_in = {k: v.to(dev) for k, v in host.items()}
    meta = dict(meta, targets=meta["targets"].to(dev))
    dev_in["target_cols"] = meta["target_cols"].to(dev)
    return lambda: bench.nav_step(model, dev_in, meta, dev)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.no_grad():
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


class _Events:
    """CUDA events around every call of the named C-ABI entry points: device ms per entry point."""

    def __init__(self, names):
        self.lib, self.ev = _lib.load(), {n: [] for n in names}
        self.orig = {n: getattr(self.lib, n) for n in names}
        for n in names:
            def call(*a, _n=n):
                st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                st.record()
                rc = self.orig[_n](*a)
                en.record()
                self.ev[_n].append((st, en))
                return rc
            setattr(self.lib, n, call)

    def close(self):
        torch.cuda.synchronize()
        for n, f in self.orig.items():
            setattr(self.lib, n, f)
        return {n: sum(s.elapsed_time(e) for s, e in evs) for n, evs in self.ev.items()}, {n: len(v) for n, v in self.ev.items()}


def block_kernel_table(dev, iters=20):
    lib, rows = _lib.load(), []
    for name, N, K in (("q/k/v/o", 4096, 4096), ("gate/up", 11008, 4096), ("down", 4096, 11008)):
        wf = torch.randn(N, K, device=dev) * 0.02
        u = torch.linalg.cholesky(torch.eye(128, device=dev, dtype=torch.float64) * 2 + 0.01).T.float().contiguous()
        w = wf.to(torch.bfloat16)
        codes, scales, zeros = (torch.zeros(ops.int4_codes_shape(N, K), dtype=torch.uint8, device=dev),
                                torch.empty((N, K // 128), dtype=torch.bfloat16, device=dev),
                                torch.empty((N, K // 128), dtype=torch.uint8, device=dev))
        ne = torch.empty((N, 128), device=dev)
        f = lambda g: ops.check(lib.nv_gptq_int4_block(ops.ptr(wf), ops.i64(K), ops.ptr(u), ops.i64(128), ops.i32(g), ops.ptr(w),
                                                       ops.i64(K), ops.ptr(codes), ops.ptr(scales), ops.ptr(zeros), ops.ptr(ne),
                                                       ops.i64(128), ops.i32(N), ops.i32(K), ops.stream_ptr()), "nv_gptq_int4_block")
        for g in range(3):
            f(g)
        st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        st.record()
        for i in range(iters):
            f(i % (K // 128))
        en.record()
        torch.cuda.synchronize()
        rows.append({"weight": name, "N": N, "K": K, "us_per_launch": st.elapsed_time(en) * 1e3 / iters})
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=bench.N_LAYERS)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--quality-layers", type=int, nargs="+", default=[0, 15, 31])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("int4_gptq_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {"gpu": dict(bench.gpu_info(0), max_sm_mhz=max_sm_clock()), "layers": a.layers}
    if a.layers != bench.N_LAYERS:
        import navillm_b200.nav_model as nm
        nm.VICUNA_7B["num_hidden_layers"] = a.layers
    model = bench.build_model(dev, seed=0).to(dev).eval()
    model._ensure()
    lm = model.lang_model
    qlayers = [l for l in a.quality_layers if l < a.layers]
    calib = {"c3": [c3_inputs(model, dev, s) for s in (1, 2)], "c2": [c2_inputs(model, dev, s) for s in (3, 4)]}
    held = {"c3": c3_inputs(model, dev, 5), "c2": c2_inputs(model, dev, 6)}
    for fns in calib.values():
        for f in fns:
            timed(f)                                                           # warm-up, outside any calibration

    # (iii) held-out Hessians of the quality layers, recorded first (from the same unquantized weights)
    with model.int4_calibration() as held_cal:
        for f in held.values():
            timed(f)
    held_h = {k: h for k, h in held_cal.h.items() if k[0] in qlayers}
    del held_cal
    W0 = {id(p): p.detach().clone() for l in qlayers for p in lm.int4_linear_weights()[7 * l:7 * l + 7]}

    # (i) calibration: the same forward with and without an open calibration, alternated
    torch.cuda.reset_peak_memory_stats()
    times = {k: {"uncalibrated_ms": [], "calibrated_ms": []} for k in calib}
    with model.int4_calibration() as cal:
        for rep in range(a.reps):
            for k, fns in calib.items():
                for f in fns:
                    arms = ("uncalibrated_ms", "calibrated_ms") if rep % 2 == 0 else ("calibrated_ms", "uncalibrated_ms")
                    for arm in arms:
                        if arm == "uncalibrated_ms":
                            lm.core.calibration = None
                            times[k][arm].append(timed(f))
                            lm.core.calibration = cal
                        else:
                            times[k][arm].append(timed(f))
    res["calibration"] = {
        k: {arm: float(np.median(v)) for arm, v in t.items()} for k, t in times.items()}
    for k, t in res["calibration"].items():
        t["ratio"] = t["calibrated_ms"] / t["uncalibrated_ms"]
    res["calibration"]["h_bytes"] = cal.nbytes
    res["calibration"]["rows_min"] = min(cal.rows.values())
    res["calibration"]["peak_gb"] = torch.cuda.max_memory_allocated() / 1e9

    # (ii) quantization
    torch.cuda.reset_peak_memory_stats()
    ev = _Events(["nv_gptq_int4_block", "nv_sgemm"])
    fac = []
    factor = ops.gptq_factor

    def timed_factor(*args, **kw):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = factor(*args, **kw)
        torch.cuda.synchronize()
        fac.append((time.perf_counter() - t0) * 1e3)
        return out
    ops.gptq_factor = timed_factor
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        nbytes = model.quantize_weights_int4(calibration=cal)
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
    finally:
        ops.gptq_factor = factor
        dev_ms, calls = ev.close()
    res["quantize"] = {"total_s": total, "factorisation_s": sum(fac) / 1e3, "factorisations": len(fac),
                       "block_kernels_s": dev_ms["nv_gptq_int4_block"] / 1e3, "block_launches": calls["nv_gptq_int4_block"],
                       "trailing_updates_s": dev_ms["nv_sgemm"] / 1e3, "trailing_launches": calls["nv_sgemm"],
                       "copy_bytes": nbytes, "peak_gb": torch.cuda.max_memory_allocated() / 1e9,
                       "block_kernel": block_kernel_table(dev)}
    del cal

    # (iii) quality on the held-out Hessians
    names = ["q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj"]
    keys = ["qkv", "qkv", "qkv", "o_proj", "gate_up", "gate_up", "down_proj"]
    quality = []
    for l in qlayers:
        for p, n, key in zip(lm.int4_linear_weights()[7 * l:7 * l + 7], names, keys):
            w0 = W0[id(p)]
            w_rtn = w0.clone()
            N, K = w0.shape
            ops.quantize_int4_(w_rtn, torch.zeros(ops.int4_codes_shape(N, K), dtype=torch.uint8, device=dev),
                               torch.empty((N, K // 128), dtype=torch.bfloat16, device=dev),
                               torch.empty((N, K // 128), dtype=torch.uint8, device=dev))
            H = held_h[(l, key)].double()
            loss = lambda wq: float((((w0.double() - wq.double()) @ H) * (w0.double() - wq.double())).sum())
            quality.append({"layer": l, "linear": n, "gptq_over_rtn": loss(p.data) / loss(w_rtn)})
    res["quality_heldout"] = quality
    res["gpu_after"] = bench.gpu_info(0)
    print(json.dumps(res, indent=1))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
