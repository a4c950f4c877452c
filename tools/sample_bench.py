"""Several samples per prompt in generate() at Vicuna-7B widths (random init), and the device sampler on its own.

    python tools/sample_bench.py [--layers 32] [--gens 3] [--out FILE.json]

End to end at the C3 shape (B = 8 prompts, 256 <cand> + 64 text tokens, N = 4 samples each, top_p = 0.9) for 20 and 128 new
tokens: generate(do_sample=True, num_return_sequences=4), which prefills each prompt once and decodes its 4 rows over the
shared prompt cache, against generate(do_sample=True) on the prompts repeated 4 times (HF's expansion).  The two arms alternate
in one process under the same seeds; per arm: prefill ms and ms per decode step (medians over the calls after the one that
captures the CUDA graphs), and whether the two arms gave the same tokens.  Peak device memory is measured per arm in a call
of its own, with the other arm's decode state dropped first, so neither arm counts the other's KV caches.  EOS stopping is
off, so every call runs all its steps.  Then nv_sample alone at 8 / 32 / 64 / 128 rows of a 32006 vocabulary, for top_k = 50, top_k = 50
with top_p = 0.9, and top_k = 0 with top_p = 0.9 (CUDA events over 200 launches).  The GPU name and power limit are read in the
same run.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from tools.beam_bench import prompts  # noqa: E402


def arm(lm, text, cand, new, seed, **kw):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    st = {}
    torch.manual_seed(seed)
    ids = lm.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand, max_new_tokens=new,
                      stop_on_eos=False, use_cuda_graph=True, stats=st, do_sample=True, top_p=0.9, **kw)
    torch.cuda.synchronize()
    return ids.cpu(), st["prefill_ms"], st["decode_ms"] / max(1, st["decode_steps"]), torch.cuda.max_memory_allocated()


def peak(lm, text, cand, new, **kw):
    """Peak device memory of one call with no other generate() state resident: the weights, this call's own KV caches and
    captured graph, and its transients."""
    lm._decode_states.clear()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return arm(lm, text, cand, new, seed=0, **kw)[3]


def e2e(model, dev, B, N, new, gens, NV, NT):
    lm = model.lang_model
    text, cand = prompts(model, B, NV, NT, dev)
    text_rep = {k: v.repeat_interleave(N, 0) for k, v in text.items()}
    cand_rep = cand.view(B, NV, -1).repeat_interleave(N, 0).reshape(B * N * NV, -1)
    res = {"shared": [], "repeated": []}
    equal = True
    for i in range(gens + 1):                                 # the first round captures the CUDA graphs
        a = arm(lm, text, cand, new, seed=i, num_return_sequences=N)
        b = arm(lm, text_rep, cand_rep, new, seed=i)
        equal &= bool(torch.equal(a[0], b[0]))
        if i:
            res["shared"].append(a[1:3])
            res["repeated"].append(b[1:3])
    out = {"B": B, "N": N, "new_tokens": new, "S0": int(text["attention_mask"].sum(1).max()), "timed_calls": gens,
           "tokens_equal": equal}
    for k, v in res.items():
        v = np.array(v)
        out[k] = {"prefill_ms": round(float(np.median(v[:, 0])), 3), "prefill_ms_each": [round(float(x), 2) for x in v[:, 0]],
                  "ms_per_step": round(float(np.median(v[:, 1])), 4)}
    out["shared"]["peak_GB"] = round(peak(lm, text, cand, new, num_return_sequences=N) / 1e9, 2)
    out["repeated"]["peak_GB"] = round(peak(lm, text_rep, cand_rep, new) / 1e9, 2)
    lm._decode_states.clear()
    torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)
    return out


def sampler(dev, iters=200):
    from navillm_b200 import ops
    V = 32006
    special = torch.arange(32000, V, dtype=torch.int32, device=dev)
    out = []
    for rows in (8, 32, 64, 128):
        g = torch.Generator(device=dev).manual_seed(rows)
        lg = (torch.randn(rows, V, generator=g, device=dev) * 2.5).to(torch.bfloat16)
        u = torch.rand(rows, generator=g, device=dev)
        fin = torch.zeros(rows, dtype=torch.int32, device=dev)
        nxt = torch.zeros(rows, dtype=torch.int32, device=dev)
        r = {"rows": rows}
        for name, k, p in (("top_k50", 50, 1.0), ("top_k50_top_p0.9", 50, 0.9), ("top_k0_top_p0.9", 0, 0.9)):
            for _ in range(10):
                ops.sample(lg, special, fin, 2, 0, False, 1.0, k, p, u, nxt)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                ops.sample(lg, special, fin, 2, 0, False, 1.0, k, p, u, nxt)
            e1.record()
            torch.cuda.synchronize()
            r[name + "_us"] = round(1e3 * e0.elapsed_time(e1) / iters, 2)
        print(json.dumps(r), flush=True)
        out.append(r)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=bench.N_LAYERS)
    ap.add_argument("--gens", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sample_bench needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "layers": a.layers, "sampler": sampler(dev)}
    if a.layers != bench.N_LAYERS:
        import navillm_b200.nav_model as nm
        nm.VICUNA_7B["num_hidden_layers"] = a.layers
    model = bench.build_model(dev, seed=0).eval()
    model._ensure()
    wl = bench.WORKLOADS["c3"]
    res["e2e"] = [e2e(model, dev, wl["B"], 4, new, a.gens, wl["n_cand_tok"], wl["n_text"]) for new in (20, wl["n_new"])]
    print(json.dumps(res))
    if a.out:
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
