"""Evaluation-rollout timing with and without cross-step prefix-KV reuse (SURVEY.md §8f n1), Vicuna-7B random init.

A synthetic rollout in the reference's prompt order (tasks/agents/r2r.py:16-31): B episodes, `--steps` navigation steps,
step t has t <hist> tokens, 12 candidates, an ~80-word instruction.  Every step runs model('navigation', ...) under
no_grad twice - from scratch (what the reference does, tasks/agents/mp3d_agent.py:660-726) and with a PrefixKVCache -
and the two fuse_logits are compared.  Prints one JSON line.

    python tools/prefix_reuse_bench.py [--batch 8] [--steps 16] [--hist0 0]
"""
import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import bench  # noqa: E402


def make_step(rng, g, B, t, instr, n_cand, D, G):
    prompts = []
    for b in range(B):
        hist_text = " ".join(f"( {i} ) <hist>" for i in range(t))
        cand_text = " ".join("( 0 ) stop" if i == 0 else f"( {i} ) <cand>" for i in range(n_cand + 1))
        prompts.append("### Instruction : Navigate following the instruction . " + instr[b]
                       + " Following is the History , which contains the visual information of your previous decisions . ### History : "
                       + hist_text
                       + " Following is the Candidate , which contains several directions you can go to at the current position , candidate ( 0 ) is stop . ### Candidate : "
                       + cand_text
                       + " Compare the History and Instruction to infer your current progress , and then select the correct direction from the candidates to go to the target location . ### Output : <cls_1>")
    n_vis = min(t, G - 2 - n_cand)
    gm = [[None] + [f"v{j}" for j in range(n_vis)] + [f"c{j}" for j in range(G - 1 - n_vis)] for _ in range(B)]
    visited = torch.zeros(B, G, dtype=torch.bool)
    visited[:, 1:1 + n_vis] = True
    step_ids = torch.zeros(B, G, dtype=torch.long)
    step_ids[:, 1:1 + n_vis] = torch.arange(1, n_vis + 1)
    gmask = torch.zeros(B, G, dtype=torch.bool)
    gmask[:, :1 + n_vis + n_cand] = True                   # stop + visited + the current candidates (one <cand> token each)
    return {"data_type": ["r2r"] * B, "vp_img_embeds": torch.randn(B, 37, D, generator=g),
            "pano_masks": torch.ones(B, 37, dtype=torch.bool), "vp_pos_fts": torch.randn(B, 37, 14, generator=g),
            "vp_cand_vpids": [[None] + [f"c{j}" for j in range(n_cand)] for _ in range(B)],
            "gmap_img_embeds": torch.randn(B, G, D, generator=g), "gmap_step_ids": step_ids,
            "gmap_pos_fts": torch.randn(B, G, 7, generator=g), "gmap_masks": gmask,
            "gmap_pair_dists": None, "gmap_visited_masks": visited, "gmap_vpids": gm, "instruction": instr,
            "history": [["h"] * t] * B, "prompts": prompts}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=16)
    ap.add_argument("--hist0", type=int, default=0, help="history length at the first step (C5: 40 with --steps 1..)")
    ap.add_argument("--json", type=str, default="")
    ap.add_argument("--fp8", action="store_true", help="quantize the weights and time the prefix-cached rollout with the fp8 copy "
                                                       "against bf16 on the same weights (bitwise-equal fuse_logits required)")
    a = ap.parse_args()
    from navillm_b200.modified_lm import PrefixKVCache
    dev = torch.device("cuda:0")
    model = bench.build_model(dev).eval()
    if a.fp8:
        return fp8_rollout(model, a, dev)
    rng = np.random.RandomState(0)
    g = torch.Generator().manual_seed(0)
    B, D, G, n_cand = a.batch, 4096, 64, 12
    words = [f"w{i}" for i in range(5000)]
    instr = [" ".join(words[i] for i in rng.randint(0, 5000, size=rng.randint(60, 100))) for _ in range(B)]
    hist = [[torch.randn(D, generator=g).to(dev) for _ in range(a.hist0)] for _ in range(B)]
    cache = PrefixKVCache(model.lang_model, batch_size=B, max_len=2048)
    to_dev = lambda b: {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in b.items()}
    ev = lambda: torch.cuda.Event(enable_timing=True)
    rows, max_rel = [], 0.0
    with torch.no_grad():
        # warm-up (allocator, tensor maps, autotuned nothing): one from-scratch step
        b0 = to_dev(make_step(rng, g, B, a.hist0, instr, n_cand, D, G)); b0["hist_vis"] = [list(h) for h in hist]
        model("navigation", b0)
        torch.cuda.synchronize()
        for t in range(a.hist0, a.hist0 + a.steps):
            batch = to_dev(make_step(rng, g, B, t, instr, n_cand, D, G))
            batch["hist_vis"] = [list(h) for h in hist]
            text = model.lang_model.tokenize(batch["prompts"])
            batch["text_input"] = text
            s0, s1, s2 = ev(), ev(), ev()
            torch.manual_seed(t); s0.record()
            ref = model("navigation", dict(batch))
            s1.record(); torch.manual_seed(t)
            enc0 = cache.stats["tokens_encoded"]
            got = model("navigation", dict(batch), prefix_cache=cache)
            s2.record(); torch.cuda.synchronize()
            r, c = ref["fuse_logits"].float(), got["fuse_logits"].float()
            fin = torch.isfinite(r)
            max_rel = max(max_rel, ((r[fin] - c[fin]).abs().max() / r[fin].abs().max()).item())
            rows.append({"hist": t, "prompt_tokens": int(text["attention_mask"].sum()), "encoded_tokens": cache.stats["tokens_encoded"] - enc0,
                         "scratch_ms": s0.elapsed_time(s1), "reuse_ms": s1.elapsed_time(s2)})
            for b in range(B):
                hist[b].append(ref["fuse_embeds"][b, 1 + (t % 3)].float())
    tot_s = sum(r["scratch_ms"] for r in rows); tot_r = sum(r["reuse_ms"] for r in rows)
    out = {"config": f"eval rollout B={B}, hist {a.hist0}..{a.hist0 + a.steps - 1}, 12 candidates, Vicuna-7B random init, no_grad",
           "scratch_ms_per_step": tot_s / len(rows), "reuse_ms_per_step": tot_r / len(rows), "speedup": tot_s / tot_r,
           "steps_per_s_scratch": B * len(rows) / tot_s * 1e3, "steps_per_s_reuse": B * len(rows) / tot_r * 1e3,
           "max_rel_logit_diff": max_rel, "first": rows[0], "last": rows[-1]}
    print(json.dumps(out), flush=True)
    if a.json:
        Path(a.json).write_text(json.dumps({"summary": out, "steps": rows}, indent=1))


def fp8_rollout(model, a, dev):
    """The same rollout twice in lock-step, each with its own prefix cache: with the fp8 copy of the weights and with bf16 on
    the same (quantized) weights, alternating per step."""
    from navillm_b200.modified_lm import PrefixKVCache
    lm = model.lang_model
    model.quantize_weights_fp8()
    copy = lm.fp8_weights
    rng = np.random.RandomState(0)
    g = torch.Generator().manual_seed(0)
    B, D, G, n_cand = a.batch, 4096, 64, 12
    words = [f"w{i}" for i in range(5000)]
    instr = [" ".join(words[i] for i in rng.randint(0, 5000, size=rng.randint(60, 100))) for _ in range(B)]
    hist = [[torch.randn(D, generator=g).to(dev) for _ in range(a.hist0)] for _ in range(B)]
    caches = {"fp8": PrefixKVCache(lm, batch_size=B, max_len=2048), "bf16": PrefixKVCache(lm, batch_size=B, max_len=2048)}
    to_dev = lambda b: {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in b.items()}
    ev = lambda: torch.cuda.Event(enable_timing=True)
    rows, equal = [], True
    with torch.no_grad():
        for t in range(a.hist0, a.hist0 + a.steps):
            batch = to_dev(make_step(rng, g, B, t, instr, n_cand, D, G))
            batch["hist_vis"] = [list(h) for h in hist]
            out, ms, enc = {}, {}, 0
            for mode in (("fp8", "bf16") if t % 2 == 0 else ("bf16", "fp8")):
                lm.core.set_fp8(copy if mode == "fp8" else None)
                e0, e1 = ev(), ev()
                enc0 = caches[mode].stats["tokens_encoded"]
                torch.manual_seed(t); e0.record()
                out[mode] = model("navigation", dict(batch), prefix_cache=caches[mode])
                e1.record(); torch.cuda.synchronize()
                ms[mode], enc = e0.elapsed_time(e1), caches[mode].stats["tokens_encoded"] - enc0
            equal &= torch.equal(out["fp8"]["fuse_logits"], out["bf16"]["fuse_logits"])
            rows.append({"hist": t, "encoded_tokens": enc, "bf16_ms": ms["bf16"], "fp8_ms": ms["fp8"]})
            for b in range(B):
                hist[b].append(out["bf16"]["fuse_embeds"][b, 1 + (t % 3)].float())
    timed = rows[1:] or rows                                   # the first step encodes whole prompts (and warms up)
    n = len(timed)
    res = {"config": f"eval rollout with PrefixKVCache, B={B}, hist {a.hist0}..{a.hist0 + a.steps - 1}, 12 candidates, "
                     f"Vicuna-7B random init, quantized, no_grad", "gpu": bench.gpu_info(0),
           "encoded_tokens_per_step": sum(r["encoded_tokens"] for r in timed) / n,
           "bf16_ms_per_step": sum(r["bf16_ms"] for r in timed) / n, "fp8_ms_per_step": sum(r["fp8_ms"] for r in timed) / n,
           "fuse_logits_bitwise_equal": bool(equal)}
    res["speedup"] = res["bf16_ms_per_step"] / res["fp8_ms_per_step"]
    print(json.dumps(res), flush=True)
    if a.json:
        Path(a.json).write_text(json.dumps({"summary": res, "steps": rows}, indent=1))
    if not equal:
        raise SystemExit("prefix_reuse_bench --fp8: fuse_logits differ between the fp8 copy and bf16")


if __name__ == "__main__":
    main()
