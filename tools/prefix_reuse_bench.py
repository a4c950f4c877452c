"""Evaluation-rollout timing with and without cross-step prefix-KV reuse (SURVEY.md §8f n1), Vicuna-7B random init.

A synthetic rollout in the reference's prompt order (tasks/agents/r2r.py:16-31): B episodes, `--steps` navigation steps,
step t has t <hist> tokens, 12 candidates, an ~80-word instruction.  Every step runs model('navigation', ...) under
no_grad twice - from scratch (what the reference does, tasks/agents/mp3d_agent.py:660-726) and with a PrefixKVCache -
and the two fuse_logits are compared.  Prints one JSON line.

    python tools/prefix_reuse_bench.py [--batch 8] [--steps 16] [--hist0 0]

--kv fp8 compares the bf16 PrefixKVCache with PrefixKVCache(kv_dtype="fp8") instead (max_len 2048, bf16 weights):
(i) the suffix attention alone, nv_attn_fwd_kv against nv_attn_fwd_kv_fp8, H = 32, 128 new rows per sequence over
512 / 1024 / 2048 cached rows, caches rotated over copies larger than L2, arms alternated, outputs checked bit for bit;
(ii) the prefix-cached rollout in ms/step for each --kv-batches x --kv-hist0, both caches in lock-step with the arm order
alternated per step, and the cache GiB of each; a bf16 cache that cannot be allocated is reported as such; (iii) the GPU
name, power limit and SM clocks, read in the same run.

    python tools/prefix_reuse_bench.py --kv fp8 --steps 5 [--kv-batches 8,32,64] [--kv-hist0 0,40]

--train times teacher-forced TRAINING rollouts (one backward per step, as tasks/agents/mp3d_agent.py:660-757 does) without a
cache (the reference's pattern) and with PrefixKVCache(train=True) plus flush_grads() at the end, for every --train-batches x
--train-steps x instruction length (the ~80-word R2R one and a CVDN-like ~300-word one).  Per shape: one warm-up rollout per
arm, then the arms alternated (A B B A); ms per rollout, tokens encoded per rollout (steps, and the flush's prefix recompute),
peak allocated GiB per arm, and the largest gradient difference over all parameters relative to max|grad|.  One JSON line per
shape, then the GPU name and power limit read in the same run.

    python tools/prefix_reuse_bench.py --train [--train-batches 8,16] [--train-steps 8,15]
"""
import argparse
import json
import subprocess
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
    ap.add_argument("--kv", choices=["bf16", "fp8"], default="bf16",
                    help="fp8: time the bf16 prefix cache against PrefixKVCache(kv_dtype='fp8') (kernel and rollout)")
    ap.add_argument("--kv-batches", type=str, default="8,32,64")
    ap.add_argument("--kv-hist0", type=str, default="0,40")
    ap.add_argument("--train", action="store_true", help="training rollouts without / with PrefixKVCache(train=True)")
    ap.add_argument("--train-batches", type=str, default="8,16")
    ap.add_argument("--train-steps", type=str, default="8,15")
    a = ap.parse_args()
    from navillm_b200.modified_lm import PrefixKVCache
    dev = torch.device("cuda:0")
    if a.kv == "fp8":
        return kv_compare(a, dev)
    if a.train:
        return train_compare(a, dev)
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


def train_rollout(model, dev, B, steps, instr, hist, cache_len):
    """One teacher-forced training rollout (loss.backward() after every step; with cache_len, a PrefixKVCache(train=True) and
    flush_grads() at the end).  Returns (ms, tokens encoded by the steps, tokens recomputed by the flush, peak GiB)."""
    from navillm_b200.modified_lm import PrefixKVCache
    rng, g = np.random.RandomState(1), torch.Generator().manual_seed(1)
    D, G, n_cand = 4096, 64, 12
    model.zero_grad()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
    t0.record()
    cache = PrefixKVCache(model.lang_model, batch_size=B, max_len=cache_len, train=True) if cache_len else None
    enc, target = 0, torch.zeros(B, dtype=torch.long, device=dev)
    for t in range(steps):
        batch = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in make_step(rng, g, B, t, instr, n_cand, D, G).items()}
        batch["hist_vis"] = [h[:t] for h in hist]
        text = model.lang_model.tokenize(batch["prompts"])
        batch["text_input"] = text
        torch.manual_seed(t)
        out = model("navigation", batch, **({"prefix_cache": cache} if cache is not None else {}))
        torch.nn.functional.cross_entropy(out["fuse_logits"].float(), target).backward()
        enc += int(text["attention_mask"].sum()) if cache is None else 0
    flush_tok = 0
    if cache is not None:
        enc = cache.stats["tokens_encoded"]
        flush_tok = sum(cache.reused)
        cache.flush_grads()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1), enc, flush_tok, torch.cuda.max_memory_allocated() / 2 ** 30


def _max_abs_diff(x, y, chunk=1 << 26):
    """max |x - y| over a flat gradient buffer in fp32 chunks (y may be a 0-d tensor); a full fp32 copy would not fit."""
    dev = y.device
    return max((x[i:i + chunk].to(dev).float() - (y if y.dim() == 0 else y[i:i + chunk]).float()).abs().max().item()
               for i in range(0, x.numel(), chunk))


def train_compare(a, dev):
    model = bench.build_model(dev).eval()          # dropout off; gradients still flow
    lm = model.lang_model
    words = [f"w{i}" for i in range(5000)]
    results = []
    for n_words, kind in ((80, "r2r"), (300, "cvdn")):
        for B in [int(x) for x in a.train_batches.split(",")]:
            for steps in [int(x) for x in a.train_steps.split(",")]:
                rng = np.random.RandomState(n_words + B)
                instr = [" ".join(words[i] for i in rng.randint(0, 5000, size=n_words)) for _ in range(B)]
                gh = torch.Generator().manual_seed(B)
                hist = [[torch.randn(4096, generator=gh).to(dev) for _ in range(steps)] for _ in range(B)]
                longest = max(int(lm.tokenize(make_step(np.random.RandomState(0), torch.Generator(), B, steps - 1, instr, 12, 16, 64)
                                              ["prompts"])["attention_mask"].sum(1).max()), 1)
                cache_len = (longest + 127) // 128 * 128
                run = lambda c: train_rollout(model, dev, B, steps, instr, hist, cache_len if c else 0)
                run(False); run(True)                                       # warm-up of both arms at this shape
                ms, ref, rel = {False: [], True: []}, None, None
                for c in (False, True, True, False):
                    ms[c].append(run(c))
                    if not c and ref is None and rel is None:          # the first scratch run's gradients ...
                        ref = [lm.flat.flat_grad.cpu(), model._flat32.flat_grad.cpu()]   # host: the flush's tape needs the room
                    elif c and rel is None:                           # ... against the first cache run's
                        scale = max(_max_abs_diff(x, torch.zeros((), dtype=x.dtype, device=dev)) for x in ref)
                        rel = max(_max_abs_diff(x, y) for x, y in zip(ref, (lm.flat.flat_grad, model._flat32.flat_grad))) / scale
                        ref = None
                r = dict(instruction=kind, words=n_words, B=B, steps=steps, cache_max_len=cache_len,
                         scratch_ms=[round(x[0], 1) for x in ms[False]], cache_ms=[round(x[0], 1) for x in ms[True]],
                         tokens_scratch=ms[False][0][1], tokens_cache_steps=ms[True][0][1], tokens_cache_flush=ms[True][0][2],
                         peak_gib_scratch=round(max(x[3] for x in ms[False]), 2), peak_gib_cache=round(max(x[3] for x in ms[True]), 2),
                         max_grad_diff_rel=rel)
                print(json.dumps(r), flush=True)
                results.append(r)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"gpu": gpu}), flush=True)
    if a.json:
        Path(a.json).write_text(json.dumps({"gpu": gpu, "shapes": results}, indent=1))


def gpu_clocks() -> dict:
    """Card name, power limit and SM clocks (maximum and current) of GPU 0."""
    info = bench.gpu_info(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm,clocks.sm", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["sm_clock_max_mhz"], info["sm_clock_mhz"] = (float(x) for x in out.split(","))
    except Exception:
        pass
    return info


def suffix_attn_table(dev, iters=50, B=8, H=32, q=128, cached=(512, 1024, 2048)):
    """One layer's suffix attention: B sequences of q new rows over `cached` rows, bf16 cache (holding K' / V') against the
    fp8 cache, launched straight through the C ABI (arguments prepared once), caches rotated over copies larger than L2."""
    from navillm_b200 import _lib, ops
    lib = _lib.load()
    g = torch.Generator(device=dev).manual_seed(0)
    HD = H * 128
    rows = []
    for c in cached:
        Smax = c + q
        per_copy = 2 * B * Smax * HD * 2
        ncopy = max(2, -(-200 * 2 ** 20 // per_copy))
        qkv = torch.randn(B * q, 3 * HD, device=dev, generator=g).to(torch.bfloat16)
        cu = torch.arange(B + 1, dtype=torch.int32, device=dev) * q
        kv_start = torch.arange(B, dtype=torch.int32, device=dev) * Smax
        kv_len = torch.full((B,), c + q, dtype=torch.int32, device=dev)
        out16 = torch.empty(B * q, HD, dtype=torch.bfloat16, device=dev)
        out8 = torch.empty_like(out16)
        c16, c8 = [], []
        for _ in range(ncopy):
            kc = torch.randn(B, Smax, HD, device=dev, generator=g).to(torch.bfloat16)
            vc = torch.randn(B, Smax, HD, device=dev, generator=g).to(torch.bfloat16)
            kq, ke = _round_cache(kc)
            vq, ve = _round_cache(vc)
            c16.append((kc, vc))
            c8.append((kq, vq, ke, ve))
        ops.attn_fwd_kv(qkv[:, :HD], *c16[0], cu, [q] * B, kv_start, kv_len, H, out=out16)
        ops.attn_fwd_kv_fp8(qkv[:, :HD], *c8[0], cu, [q] * B, kv_start, kv_len, H, out=out8)
        torch.cuda.synchronize()
        bitwise = torch.equal(out16.view(torch.int16), out8.view(torch.int16))
        P, i64, i32 = _lib.ptr, _lib.i64, _lib.i32
        common = (P(out16), i64(HD), None, P(cu), P(kv_start), P(kv_len), i32(B), i32(B * q), i32(B * Smax), i32(H), i32(128),
                  i32(B), _lib.f32(128 ** -0.5))
        a16 = [(P(qkv), i64(3 * HD), P(k), i64(HD), P(v), i64(HD)) + common for k, v in c16]
        a8 = [(P(qkv), i64(3 * HD), P(kq), P(vq), P(ke), P(ve)) + common for kq, vq, ke, ve in c8]
        stream = _lib.stream_ptr()
        f16 = lambda i: lib.nv_attn_fwd_kv(*a16[i % ncopy], stream)
        f8 = lambda i: lib.nv_attn_fwd_kv_fp8(*a8[i % ncopy], stream)
        for i in range(5):
            f16(i); f8(i)
        torch.cuda.synchronize()
        t = {"bf16": [], "fp8": []}
        for rep in range(6):
            for kind, f in (("bf16", f16), ("fp8", f8)) if rep % 2 == 0 else (("fp8", f8), ("bf16", f16)):
                st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                st.record()
                for i in range(iters):
                    rc = f(i)
                en.record()
                torch.cuda.synchronize()
                assert rc == 0, kind
                t[kind].append(st.elapsed_time(en) / iters)
        keys = B * (c + q)
        io = B * q * HD * 2 * 2                                   # q in, o out
        r = {"B": B, "H": H, "q_rows": q, "cached_rows": c, "fp8_bitwise_bf16_on_rounded": bool(bitwise)}
        for kind, by in (("bf16", keys * HD * 2 * 2 + io), ("fp8", keys * HD * 2 + keys * H * 2 + io)):
            us = 1e3 * float(np.median(t[kind]))
            r[f"{kind}_us"] = round(us, 2)
            r[f"{kind}_GBps"] = round(by / us / 1e3, 1)
        r["speedup"] = round(r["bf16_us"] / r["fp8_us"], 3)
        rows.append(r)
        print(json.dumps(r), flush=True)
        del c16, c8
        torch.cuda.empty_cache()
    return rows


def _round_cache(c):
    """quantize_fp8_ on the [rows, 128] view of a bf16 cache: c becomes K' in place; returns (e4m3 bytes, exponents)."""
    from navillm_b200 import ops
    rows = c.view(-1, 128)
    q = torch.empty(rows.shape, dtype=ops.fp8, device=c.device)
    e = torch.empty(rows.shape[0], dtype=torch.int8, device=c.device)
    ops.quantize_fp8_(rows, q, e)
    return q.view(c.shape), e.view(*c.shape[:-1], c.shape[-1] // 128)


def kv_rollout(model, dev, B, hist0, steps):
    """The prefix-cached rollout with a bf16 and an fp8 PrefixKVCache in lock-step (arm order alternated per step)."""
    from navillm_b200.modified_lm import PrefixKVCache
    lm = model.lang_model
    rng = np.random.RandomState(0)
    g = torch.Generator().manual_seed(0)
    D, G, n_cand = 4096, 64, 12
    words = [f"w{i}" for i in range(5000)]
    instr = [" ".join(words[i] for i in rng.randint(0, 5000, size=rng.randint(60, 100))) for _ in range(B)]
    hist = [[torch.randn(D, generator=g).to(dev) for _ in range(hist0)] for _ in range(B)]
    caches, res = {"fp8": PrefixKVCache(lm, batch_size=B, max_len=2048, kv_dtype="fp8")}, {"B": B, "hist0": hist0}
    try:
        caches["bf16"] = PrefixKVCache(lm, batch_size=B, max_len=2048)
    except torch.cuda.OutOfMemoryError:
        res["bf16"] = "cache does not fit"
    torch.cuda.empty_cache()
    for k, c in caches.items():
        res[f"{k}_cache_GiB"] = round(c.nbytes / 2 ** 30, 3)
    to_dev = lambda b: {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in b.items()}
    ev = lambda: torch.cuda.Event(enable_timing=True)
    rows, max_rel = [], 0.0
    with torch.no_grad():
        for t in range(hist0, hist0 + steps):
            batch = to_dev(make_step(rng, g, B, t, instr, n_cand, D, G))
            batch["hist_vis"] = [list(h) for h in hist]
            out, ms, enc = {}, {}, 0
            order = [k for k in (("fp8", "bf16") if t % 2 == 0 else ("bf16", "fp8")) if k in caches]
            for mode in order:
                e0, e1 = ev(), ev()
                enc0 = caches[mode].stats["tokens_encoded"]
                torch.manual_seed(t); e0.record()
                out[mode] = model("navigation", dict(batch), prefix_cache=caches[mode])
                e1.record(); torch.cuda.synchronize()
                ms[mode], enc = e0.elapsed_time(e1), caches[mode].stats["tokens_encoded"] - enc0
            if "bf16" in out:
                r, c = out["bf16"]["fuse_logits"].float(), out["fp8"]["fuse_logits"].float()
                fin = torch.isfinite(r)
                max_rel = max(max_rel, ((r[fin] - c[fin]).abs().max() / r[fin].abs().max()).item())
            rows.append(dict({"hist": t, "encoded_tokens": enc}, **{f"{k}_ms": v for k, v in ms.items()}))
            src = out.get("bf16", out["fp8"])
            for b in range(B):
                hist[b].append(src["fuse_embeds"][b, 1 + (t % 3)].float())
    timed = rows[1:] or rows                                   # the first step encodes whole prompts (and warms up)
    n = len(timed)
    res["encoded_tokens_per_step"] = sum(r["encoded_tokens"] for r in timed) / n
    res["first_step_encoded_tokens"] = rows[0]["encoded_tokens"]
    for k in caches:
        res[f"{k}_ms_per_step"] = round(sum(r[f"{k}_ms"] for r in timed) / n, 2)
        res[f"{k}_first_step_ms"] = round(rows[0][f"{k}_ms"], 2)
    if "bf16" in caches:
        res["speedup"] = round(res["bf16_ms_per_step"] / res["fp8_ms_per_step"], 3)
        res["max_rel_logit_diff_fp8_vs_bf16_cache"] = max_rel
    res["peak_allocated_GiB"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
    print(json.dumps(res), flush=True)
    del caches
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    return res


def kv_compare(a, dev):
    res = {"gpu_before": gpu_clocks(), "suffix_attention": suffix_attn_table(dev)}
    model = bench.build_model(dev).eval()
    res["config"] = ("eval rollout with PrefixKVCache max_len 2048, 12 candidates, Vicuna-7B random init, bf16 weights, "
                     f"no_grad, {a.steps} steps, the first one (whole prompts) reported apart")
    res["weights_GiB"] = round(torch.cuda.memory_allocated() / 2 ** 30, 2)
    res["rollouts"] = [kv_rollout(model, dev, int(B), int(h), a.steps)
                       for h in a.kv_hist0.split(",") for B in a.kv_batches.split(",")]
    res["gpu_after"] = gpu_clocks()
    print(json.dumps(res), flush=True)
    if a.json:
        Path(a.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
