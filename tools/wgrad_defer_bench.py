"""Training-rollout timing with and without deferred weight gradients (defer_weight_grads), Vicuna-7B random init.

Teacher-forced navigation rollouts (one loss.backward() per step, as tasks/agents/mp3d_agent.py:660-757 does) in the R2R
prompt order of tools/prefix_reuse_bench.py, for every --batches x --steps, without a prefix cache and with
PrefixKVCache(train=True) (flush_grads() at the end).  Two arms per shape: the per-backward weight gradients (the default)
and deferral with --max-rows (flush_weight_grads() at the end of the rollout, inside the timed region).  Per shape: one
warm-up rollout per arm, then the arms alternated (A B B A); ms per rollout, peak allocated GiB per arm, rows per backward,
segmented launches per rollout, and the largest gradient difference between the arms over the bf16 gradient buffer
relative to max|grad|.  One JSON line per shape, then the GPU name, power limit and SM clocks read in the same run.

    python tools/wgrad_defer_bench.py [--batches 1,2,4,8] [--steps 8,15] [--max-rows 2048]
"""
import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import bench  # noqa: E402
from prefix_reuse_bench import _max_abs_diff, gpu_clocks, make_step  # noqa: E402


def rollout(model, dev, B, steps, instr, hist, cache_len, defer_rows, seg_calls):
    """One training rollout; returns (ms, peak GiB, rows of the first backward, segmented launches, largest stash GiB at the
    end of a step -- a host-side walk over the stash, inside the timed region)."""
    from navillm_b200.modified_lm import PrefixKVCache
    rng, g = np.random.RandomState(1), torch.Generator().manual_seed(1)
    D, G, n_cand = 4096, 64, 12
    model.zero_grad()
    model.defer_weight_grads(defer_rows or None)
    n0 = len(seg_calls)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
    t0.record()
    cache = PrefixKVCache(model.lang_model, batch_size=B, max_len=cache_len, train=True) if cache_len else None
    target = torch.zeros(B, dtype=torch.long, device=dev)
    rows0, stash = None, 0
    for t in range(steps):
        batch = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in make_step(rng, g, B, t, instr, n_cand, D, G).items()}
        batch["hist_vis"] = [h[:t] for h in hist]
        batch["text_input"] = text = model.lang_model.tokenize(batch["prompts"])
        if rows0 is None:
            rows0 = int(text["attention_mask"].sum())
        torch.manual_seed(t)
        out = model("navigation", batch, **({"prefix_cache": cache} if cache is not None else {}))
        torch.nn.functional.cross_entropy(out["fuse_logits"].float(), target).backward()
        stash = max(stash, model.weight_grad_stash_bytes())
    if cache is not None:
        cache.flush_grads()
    model.flush_weight_grads()
    t1.record()
    torch.cuda.synchronize()
    model.defer_weight_grads(None)
    return t0.elapsed_time(t1), torch.cuda.max_memory_allocated() / 2 ** 30, rows0, len(seg_calls) - n0, stash / 2 ** 30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=str, default="1,2,4,8")
    ap.add_argument("--steps", type=str, default="8,15")
    ap.add_argument("--max-rows", type=int, default=2048)
    ap.add_argument("--json", type=str, default="")
    a = ap.parse_args()
    from navillm_b200 import ops
    dev = torch.device("cuda:0")
    seg_calls = []
    orig = ops.gemm_wgrad_seg
    ops.gemm_wgrad_seg = lambda *x, **k: (seg_calls.append(len(x[0])), orig(*x, **k))[1]
    model = bench.build_model(dev).eval()          # dropout off; gradients still flow
    lm = model.lang_model
    words = [f"w{i}" for i in range(5000)]
    results = []
    for B in [int(x) for x in a.batches.split(",")]:
        for steps in [int(x) for x in a.steps.split(",")]:
            rng = np.random.RandomState(80 + B)
            instr = [" ".join(words[i] for i in rng.randint(0, 5000, size=80)) for _ in range(B)]
            gh = torch.Generator().manual_seed(B)
            hist = [[torch.randn(4096, generator=gh).to(dev) for _ in range(steps)] for _ in range(B)]
            longest = max(int(lm.tokenize(make_step(np.random.RandomState(0), torch.Generator(), B, steps - 1, instr, 12, 16, 64)
                                          ["prompts"])["attention_mask"].sum(1).max()), 1)
            for cache_len in (0, (longest + 127) // 128 * 128):
                run = lambda d: rollout(model, dev, B, steps, instr, hist, cache_len, a.max_rows if d else 0, seg_calls)
                run(False); run(True)                               # warm-up of both arms at this shape
                res, rel, ref = {False: [], True: []}, None, None
                for d in (False, True, True, False):
                    res[d].append(run(d))
                    if not d and ref is None and rel is None:
                        ref = lm.flat.flat_grad.cpu()          # host: a device copy would count in the deferred peak
                    elif d and rel is None:
                        scale = _max_abs_diff(ref, torch.zeros((), dtype=ref.dtype, device=dev))
                        rel = _max_abs_diff(ref, lm.flat.flat_grad) / scale
                        ref = None
                per, dfr = [x[0] for x in res[False]], [x[0] for x in res[True]]
                r = dict(B=B, steps=steps, prefix_cache=bool(cache_len), max_rows=a.max_rows, rows_first_backward=res[False][0][2],
                         per_step_ms=[round(x, 1) for x in per], deferred_ms=[round(x, 1) for x in dfr],
                         speedup=round(sum(per) / sum(dfr), 3),
                         peak_gib_per_step=round(max(x[1] for x in res[False]), 2), peak_gib_deferred=round(max(x[1] for x in res[True]), 2),
                         stash_gib=round(res[True][0][4], 2), seg_launches_per_rollout=res[True][0][3], max_grad_diff_rel=rel)
                print(json.dumps(r), flush=True)
                results.append(r)
    gpu = gpu_clocks()
    print(json.dumps({"gpu": gpu}), flush=True)
    if a.json:
        Path(a.json).write_text(json.dumps({"gpu": gpu, "shapes": results}, indent=1))


if __name__ == "__main__":
    main()
