"""Cost of batch-invariant mode (set_batch_invariant) against the default path, in one process, the two arms alternated.

    python tools/batch_invariant_bench.py [--layers 32] [--batch 1 8 32 64] [--gens 3] [--rounds 2] [--iters 50]
                                          [--out FILE.json]

(i)   per-GEMM time at the decode shapes of Vicuna-7B and M = 1, 8, 16, 32, 64 (CUDA events, weights rotated over copies
      larger than L2): the default kernel (swap-AB split-K skinny up to 16 rows, nv_gemm_bf16 above), nv_gemm_bi_bf16 /
      nv_gemm_bi_swiglu_bf16 (the mode's kernel), and nv_gemm_bf16 pinned to its 32-wide tile with the SwiGLU row kernel
      (the other batch-invariant candidate), with the bytes each must move and the achieved GB/s;
(ii)  C3-shaped generate() decode ms/token (S0 = 320, 128 new tokens, EOS stop off, CUDA graphs) at each batch, mode off and
      on alternated over `rounds` rounds, medians over the generations after each capture, and the prefill ms at each batch;
(iii) a no-grad navigation step (panorama encoder + navigation forward) at B = 16 of bench.py's C2 workload, off and on
      alternated;
(iv)  the GPU name and power limit, read in the same run.
Vicuna-7B widths, random init (bench.build_model).  Needs a GPU; there is no CPU path.
"""
import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from navillm_b200 import ops  # noqa: E402

SHAPES = [("qkv", 12288, 4096, False), ("o", 4096, 4096, False), ("gate_up+swiglu", 11008, 4096, True),
          ("down", 4096, 11008, False), ("lm_head", 32006, 4096, False)]


def _time(fns, iters, reps=6):
    """Median ms per call of each named callable f(i), the callables alternated (order reversed every other round)."""
    t = {k: [] for k in fns}
    for i in range(5):
        for f in fns.values():
            f(i)
    torch.cuda.synchronize()
    names = list(fns)
    for rep in range(reps):
        for k in (names if rep % 2 == 0 else names[::-1]):
            st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            st.record()
            for i in range(iters):
                fns[k](i)
            en.record()
            torch.cuda.synchronize()
            t[k].append(st.elapsed_time(en) / iters)
    return {k: float(np.median(v)) for k, v in t.items()}


def gemm_table(dev, iters):
    rows = []
    g = torch.Generator(device=dev).manual_seed(0)
    for name, N, K, swiglu in SHAPES:
        wrows = 2 * N if swiglu else N
        ncopy = max(2, -(-160 * 2 ** 20 // (wrows * K * 2)))              # > 3 x the 50 MB L2 per rotation
        ws = [(torch.randn(wrows, K, device=dev, generator=g) * 0.02).to(torch.bfloat16) for _ in range(ncopy)]
        for M in (1, 8, 16, 32, 64):
            x = torch.randn(M, K, device=dev, generator=g).to(torch.bfloat16)
            w = lambda i: ws[i % ncopy]
            if swiglu:
                default = (lambda i: ops.gemm_skinny_swiglu(x, w(i))) if M <= 16 else (lambda i: ops.swiglu_fwd(ops.gemm(x, w(i))))
                bi = lambda i: ops.gemm_bi_swiglu(x, w(i))
                tile32 = lambda i: ops.swiglu_fwd(ops.gemm(x, w(i), block_n=32))
            else:
                default = (lambda i: ops.gemm_skinny(x, w(i))) if M <= 16 else (lambda i: ops.gemm(x, w(i)))
                bi = lambda i: ops.gemm_bi(x, w(i))
                tile32 = lambda i: ops.gemm(x, w(i), block_n=32)
            same = torch.equal(bi(0), tile32(0))
            ms = _time({"default": default, "bi": bi, "tile32": tile32}, iters)
            by = wrows * K * 2 + M * K * 2 + M * N * 2
            r = {"gemm": name, "M": M, "N": N, "K": K, "bytes": by, "bi_equals_tile32": same}
            for k, v in ms.items():
                r[f"{k}_us"] = round(1e3 * v, 2)
                r[f"{k}_GBps"] = round(by / (1e3 * v) / 1e3, 1)
            r["bi_vs_default"] = round(ms["default"] / ms["bi"], 3)
            rows.append(r)
            print(json.dumps(r), flush=True)
        del ws
        torch.cuda.empty_cache()
    return rows


def c3_inputs(model, dev, B):
    wl = bench.WORKLOADS["c3"]
    NV, NT = wl["n_cand_tok"], wl["n_text"]
    lm = model.lang_model
    rng = np.random.RandomState(1234)
    words = [f"w{i}" for i in range(5000)]
    prompts = ["Scene " + " ".join(["<cand>"] * NV) + " Question " + " ".join(words[i] for i in rng.randint(0, 5000, size=NT - 5))
               + " Answer" for _ in range(B)]
    text = lm.tokenize(prompts)
    g = torch.Generator().manual_seed(1234)
    with torch.no_grad():
        view = torch.stack([torch.randn(NV, bench.IMG_FEAT, generator=g) for _ in range(B)], 0).to(dev)
        pano = model.img_embeddings.forward_panorama_per_step(view_img_fts=view, view_lens=torch.full((B,), NV, device=dev))
        cand = model._masked_rows_plus_const(pano["pano_embeds"].reshape(B * NV, -1), np.ones((B, NV), dtype=bool)).detach()
    return text, cand


def c3_generate(model, dev, batches, gens, rounds):
    lm = model.lang_model
    NEW = bench.WORKLOADS["c3"]["n_new"]
    out = []
    for B in batches:
        text, cand = c3_inputs(model, dev, B)
        res = {False: {"decode": [], "prefill": []}, True: {"decode": [], "prefill": []}}
        for rnd in range(rounds):
            for on in ((False, True) if rnd % 2 == 0 else (True, False)):
                model.set_batch_invariant(on)
                for j in range(gens + 1):                                 # the first call captures the CUDA graph
                    st = {}
                    lm.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand,
                                max_new_tokens=NEW, stop_on_eos=False, use_cuda_graph=True, stats=st)
                    if j > 0:
                        res[on]["decode"].append(st["decode_ms"] / st["decode_steps"])
                        res[on]["prefill"].append(st["prefill_ms"])
        model.set_batch_invariant(False)
        r = {"B": B, "S0": int(text["attention_mask"].sum(1).max()), "new_tokens": NEW}
        for on, tag in ((False, "default"), (True, "invariant")):
            r[f"decode_ms_per_token_{tag}"] = round(float(np.median(res[on]["decode"])), 4)
            r[f"prefill_ms_{tag}"] = round(float(np.median(res[on]["prefill"])), 3)
        r["decode_overhead"] = round(r["decode_ms_per_token_invariant"] / r["decode_ms_per_token_default"] - 1, 4)
        r["prefill_overhead"] = round(r["prefill_ms_invariant"] / r["prefill_ms_default"] - 1, 4)
        out.append(r)
        print(json.dumps(r), flush=True)
    return out


def nav_step_cost(model, dev, reps, rounds):
    host, meta = bench.make_workload(7, B=16)
    dev_in = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in host.items()}
    dev_in["target_cols"] = meta["target_cols"].to(dev)
    t = {False: [], True: []}
    for rnd in range(rounds):
        for on in ((False, True) if rnd % 2 == 0 else (True, False)):
            model.set_batch_invariant(on)
            with torch.no_grad():
                bench.nav_step(model, dev_in, meta, dev)                   # warm-up
                torch.cuda.synchronize()
                for _ in range(reps):
                    t0 = time.perf_counter()
                    torch.manual_seed(0)
                    bench.nav_step(model, dev_in, meta, dev)
                    torch.cuda.synchronize()
                    t[on].append(1e3 * (time.perf_counter() - t0))
    model.set_batch_invariant(False)
    r = {"B": 16, "nav_step_ms_default": round(float(np.median(t[False])), 3),
         "nav_step_ms_invariant": round(float(np.median(t[True])), 3)}
    r["overhead"] = round(r["nav_step_ms_invariant"] / r["nav_step_ms_default"] - 1, 4)
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=bench.N_LAYERS)
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 8, 32, 64])
    ap.add_argument("--gens", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--nav_reps", type=int, default=5)
    ap.add_argument("--out", type=str, default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("batch_invariant_bench: needs a GPU (no CPU path)")
    dev = torch.device("cuda:0")
    res = {"gpu": bench.gpu_info(0), "gemms": gemm_table(dev, a.iters)}
    if a.layers != bench.N_LAYERS:
        import navillm_b200.nav_model as nm
        nm.VICUNA_7B["num_hidden_layers"] = a.layers
    model = bench.build_model(dev, seed=0).eval()
    model._ensure()
    res["layers"] = a.layers
    res["c3"] = c3_generate(model, dev, a.batch, a.gens, a.rounds)
    res["nav_step"] = nav_step_cost(model, dev, a.nav_reps, a.rounds)
    print(json.dumps({"gpu": res["gpu"]}), flush=True)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
