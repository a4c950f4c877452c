"""Contrastive search in generate() at Vicuna-7B widths (random init), against greedy decoding of the same prompts.

    python tools/contrastive_bench.py [--layers 32] [--gens 2] [--ks 4,10,50] [--out FILE.json]

Shape: C3 (B = 8, 256 <cand> + 64 text tokens, 128 new tokens, EOS stopping off: random weights would stop at arbitrary steps)
at k in --ks, alpha = 0.6.  Per k: prefill ms (the prompt forward and the first lm_head / top-k; the first candidate step is a
decode step), ms per step (median over the generations after the one that captures the CUDA graph), and greedy decoding at B
and at B * k rows, the three arms alternated generation by generation.  Then the peak device memory of one call of each arm
with no other arm's state held, the three new kernels timed with CUDA events over 50 launches each at the step's shapes, and
the decode attention's share of the device time of the steps alone: two torch.profiler runs of eager calls, 13 and 1 new
tokens, subtracted, so the prefill cancels.  The GPU name and power limit are read in the same run.
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
sys.path.insert(0, str(ROOT / "tools"))
import bench  # noqa: E402
from beam_bench import prompts  # noqa: E402

ALPHA = 0.6


def one(lm, text, cand, new, **kw):
    st = {}
    lm.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand, max_new_tokens=new,
                stop_on_eos=False, use_cuda_graph=True, stats=st, **kw)
    torch.cuda.synchronize()
    return st["prefill_ms"], st["decode_ms"] / st["decode_steps"]


def peak_gb(lm, text, cand, new, **kw):
    """Peak device memory of one call (weights included) with no other call's decode state held."""
    lm._decode_states.clear()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    one(lm, text, cand, new, **kw)
    peak = torch.cuda.max_memory_allocated()
    lm._decode_states.clear()
    torch.cuda.empty_cache()
    return round(peak / 1e9, 2)


def summary(runs):
    runs = runs[1:]                                                      # the first call captures the CUDA graph
    return {"prefill_ms": round(float(np.median([r[0] for r in runs])), 3),
            "ms_per_step": round(float(np.median([r[1] for r in runs])), 4)}


def event_ms(fn, n=50):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return round(a.elapsed_time(b) / n * 1e3, 2)                       # us


def kernel_times(lm, B, k, S0, new, dev):
    """The three new kernels at the step's shapes, on standalone buffers: the context at S0 + new / 2 rows per prompt."""
    from navillm_b200 import llama, ops
    d = lm.dims
    D, V = d.hidden, lm.lm_head.weight.shape[0]
    Sp = (S0 + new + 127) // 128 * 128
    n_ctx = S0 + new // 2
    g = torch.Generator(device=dev).manual_seed(0)
    logits = torch.randn(B, V, generator=g, device=dev).to(torch.bfloat16)
    p = torch.empty(B, k, dtype=torch.bfloat16, device=dev)
    tok = torch.empty(B, k, dtype=torch.int32, device=dev)
    hn = torch.randn(B * k, D, generator=g, device=dev).to(torch.bfloat16)
    ctx = torch.randn(B, Sp, D, generator=g, device=dev).to(torch.bfloat16)
    i32 = lambda *s: torch.zeros(s, dtype=torch.int32, device=dev)
    ctx_len, pen_key, fin, nxt, sel, plens, lens = i32(B), i32(B * k), i32(B), i32(B), i32(B), i32(B), i32(B * k)
    hsel = torch.empty(B, D, dtype=torch.bfloat16, device=dev)
    special = lm.special_ids_dev
    ops.contrastive_topk(logits, special, k, p, tok)

    def rank():
        ctx_len.fill_(n_ctx)                   # the rank appends a row; keep every launch at the same context length
        ops.contrastive_rank(hn, ctx, ctx_len, pen_key, p, tok, ALPHA, fin, -1, 0, False, nxt, sel, hsel, plens, lens)
    fill = event_ms(lambda: ctx_len.fill_(n_ctx))
    kc, vc = llama.kv_cache(d, B * k, 1, "bf16", dev), llama.kv_cache(d, B * k, 1, "bf16", dev)
    pk, pv = llama.kv_cache(d, B, Sp, "bf16", dev), llama.kv_cache(d, B, Sp, "bf16", dev)
    table = ops.contrastive_commit_table(kc, vc, pk, pv)
    plens.fill_(S0 + 1)
    ctx_bytes = B * n_ctx * D * 2
    r = {"topk_us": event_ms(lambda: ops.contrastive_topk(logits, special, k, p, tok)),
         "rank_us": round(event_ms(rank) - fill, 2),
         "commit_us": event_ms(lambda: ops.contrastive_commit(table, sel, plens, k, Sp, d.n_heads, False)),
         "rank_context_MB": round(ctx_bytes / 1e6, 1)}
    r["rank_context_GBps"] = round(ctx_bytes / (r["rank_us"] * 1e-6) / 1e9, 1)
    del kc, vc, pk, pv, ctx
    return r


def attention_share(lm, text, cand, k, new=13):
    """Share of the decode attention (decode_attn_kernel) in the device time of ``new - 1`` eager contrastive steps: the kernel
    times of a call with ``new`` tokens minus those of a call with 1 token (same prompts, same prefill)."""
    from torch.profiler import ProfilerActivity, profile
    kw = dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand, stop_on_eos=False,
              use_cuda_graph=False, penalty_alpha=ALPHA, top_k=k)

    def device_us(n):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            lm.generate(max_new_tokens=n, **kw)
            torch.cuda.synchronize()
        tot = attn = 0.0
        for e in prof.key_averages():
            t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            if "decode_attn_kernel" in e.key:
                attn += t
            tot += t
        return attn, tot
    lm.generate(max_new_tokens=new, **kw)
    torch.cuda.synchronize()
    a1, t1 = device_us(1)
    an, tn = device_us(new)
    return {"share": round((an - a1) / (tn - t1), 3), "steps": new - 1,
            "step_device_ms": round((tn - t1) / 1e3 / (new - 1), 3), "attn_ms_per_step": round((an - a1) / 1e3 / (new - 1), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=bench.N_LAYERS)
    ap.add_argument("--gens", type=int, default=2)
    ap.add_argument("--ks", default="4,10,50")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("contrastive_bench needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    if a.layers != bench.N_LAYERS:
        import navillm_b200.nav_model as nm
        nm.VICUNA_7B["num_hidden_layers"] = a.layers
    model = bench.build_model(dev, seed=0).eval()
    model._ensure()
    lm = model.lang_model
    lm._decode_states.max_states = 3                                     # one captured graph per arm
    wl = bench.WORKLOADS["c3"]
    B, new = wl["B"], wl["n_new"]
    text, cand = prompts(model, B, wl["n_cand_tok"], wl["n_text"], dev)
    S0 = int(text["attention_mask"].sum(1).max())
    rows = []
    for k in [int(x) for x in a.ks.split(",")]:
        tbk, cbk = prompts(model, B * k, wl["n_cand_tok"], wl["n_text"], dev)
        arms = {"contrastive": (text, cand, dict(penalty_alpha=ALPHA, top_k=k)), "greedy_B": (text, cand, {}),
                "greedy_Bk": (tbk, cbk, {})}
        runs = {name: [] for name in arms}
        for _ in range(a.gens + 1):                                      # the arms alternate, generation by generation
            for name, (t, c, kw) in arms.items():
                if runs[name] is None:
                    continue
                try:
                    runs[name].append(one(lm, t, c, new, **kw))
                except torch.cuda.OutOfMemoryError:                      # greedy at B * k rows holds B * k full caches
                    runs[name] = None
                    lm._decode_states.clear()
                    torch.cuda.empty_cache()
        r = {"B": B, "k": k, "alpha": ALPHA, "new_tokens": new, "S0": S0,
             **{n: summary(v) if v else "not measured: out of device memory" for n, v in runs.items()}}
        lm._decode_states.clear()
        torch.cuda.empty_cache()
        for name, (t, c, kw) in arms.items():
            if runs[name]:
                r[name]["peak_GB"] = peak_gb(lm, t, c, new, **kw)
        del tbk, cbk, arms
        lm._decode_states.clear()
        torch.cuda.empty_cache()
        r["kernels"] = kernel_times(lm, B, k, S0, new, dev)
        r["decode_attn_eager_steps"] = attention_share(lm, text, cand, k)
        lm._decode_states.clear()
        torch.cuda.empty_cache()
        print(json.dumps(r), flush=True)
        rows.append(r)
    res = {"gpu": gpu, "layers": a.layers, "rows": rows}
    print(json.dumps(res))
    if a.out:
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
