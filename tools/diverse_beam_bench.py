"""Diverse (group) beam search in generate() at Vicuna-7B widths (random init), against plain beam search.

    python tools/diverse_beam_bench.py [--layers 32] [--gens 3] [--out FILE.json]

(i)  C3 shape: B = 8 prompts of 256 <cand> + 64 text tokens (S0 = 319), 128 new tokens, stop_on_eos as generate() runs beams.
(ii) Summarization shape: B = 8 copies of the summarization mode's prompt at 7 history steps and 6 candidates, as recorded from
     the reference's R2R agent in tests/golden/summarization_prompts.json, max_new_tokens = 50 as the mode sets it; the prompt
     length is its tokenized length, measured here and reported.
Arms: plain beams at K = 4 and K = 8; groups (K, G) = (4, 2), (4, 4), (8, 2), (8, 4), (8, 8) with diversity_penalty = 0.5
(num_return_sequences = K).  Per arm: ms per call (host clock around a synchronised call), prefill_ms, ms per decode step
(decode_ms / decode steps) and steps, medians over --gens calls after the capturing one, the arms alternating call by call; then
each arm's peak memory from one more call with only its own decode state resident (the other arms' states dropped).  Random weights end beams at max_new_tokens or at a random EOS, so the step counts are reported with each arm.
(iii) The beam kernels alone at B = 8, V = 32006 (CUDA events over 200 launches): one step's G group top-k + select launches
against one nv_beam_topk + nv_beam_select at the same K.
The GPU name, power limit and max SM clock are read in the same run.
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
from constrained_decode_bench import timed  # noqa: E402
from contrastive_bench import event_ms  # noqa: E402

GROUPS = [(4, 2), (4, 4), (8, 2), (8, 4), (8, 8)]


def summarization_prompt(hist_num=7, cand_num=6):
    """The summarization mode's prompt with ``hist_num`` history steps and ``cand_num`` candidates, as recorded from the
    reference (tests/golden/make_summarization_prompt_golden.py)."""
    gold = json.loads((ROOT / "tests" / "golden" / "summarization_prompts.json").read_text())
    return next(p["prompt"] for p in gold["prompts"] if (p["hist_num"], p["cand_num"]) == (hist_num, cand_num))


def summarization_batch(lm, dev, B=8, hist_num=7, cand_num=6, seed=0):
    text = lm.tokenize([summarization_prompt(hist_num, cand_num) for _ in range(B)])
    g = torch.Generator().manual_seed(seed)
    D = lm.dims.hidden
    return dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"],
                cand_vis=(torch.randn(B * cand_num, D, generator=g) * 0.02).to(dev),
                hist_vis=(torch.randn(B * hist_num, D, generator=g) * 0.02).to(dev))


def arms():
    a = {f"beams_K{K}": dict(num_beams=K, num_return_sequences=K) for K in (4, 8)}
    a.update({f"groups_K{K}_G{G}": dict(num_beams=K, num_beam_groups=G, diversity_penalty=0.5, num_return_sequences=K)
              for K, G in GROUPS})
    return a


def arms_timed(lm, batch, arms, gens, new):
    """Each arm once to capture, then ``gens`` rounds alternating the arms; then one call per arm with only its own decode
    state resident for its peak memory."""
    res = {name: [] for name in arms}
    for i in range(gens + 1):
        for name, kw in arms.items():
            st = {}
            ms, _ = timed(lambda: lm.generate(**batch, max_new_tokens=new, use_cuda_graph=True, stats=st, **kw))
            if i:
                res[name].append((ms, st["prefill_ms"], st["decode_ms"] / max(st["decode_steps"], 1), st["beam_steps"]))
    peak = {}
    for name, kw in arms.items():
        lm._decode_states.clear()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        lm.generate(**batch, max_new_tokens=new, use_cuda_graph=True, **kw)
        torch.cuda.synchronize()
        peak[name] = torch.cuda.max_memory_allocated() / 2 ** 30
    lm._decode_states.clear()
    torch.cuda.empty_cache()
    out = {}
    for name, v in res.items():
        out[name] = {"ms_per_call": round(float(np.median([x[0] for x in v])), 2),
                     "ms_spread": round(float(max(x[0] for x in v) - min(x[0] for x in v)), 2),
                     "prefill_ms": round(float(np.median([x[1] for x in v])), 2),
                     "ms_per_step": round(float(np.median([x[2] for x in v])), 3), "steps": int(v[-1][3]),
                     "peak_gib": round(peak[name], 2)}
        print(json.dumps({name: out[name]}), flush=True)
    return out


def kernel_times(lm, dev, B=8, n=200, t=20):
    """One step's beam launches at B prompts: G x (group top-k + group select) against nv_beam_topk + nv_beam_select."""
    from navillm_b200 import ops
    V = lm.lm_head.weight.shape[0]
    special = lm.special_ids_dev
    rows = []
    Gc, S = 128, 96
    for K in (4, 8):
        g = torch.Generator(device=dev).manual_seed(K)
        logits = (torch.randn(B * K, V, generator=g, device=dev) * 3).to(torch.bfloat16)
        i32 = lambda *s: torch.zeros(s, dtype=torch.int32, device=dev)

        def state():
            st = dict(bs=torch.randn(B * K, generator=g, device=dev), hist=i32(B * K, Gc), src=i32(B * K, Gc),
                      hs=torch.zeros((B, K + 1), dtype=torch.float64, device=dev), hm=i32(B, K, 2), ht=i32(B, K, Gc),
                      ps=i32(B, 5), nx=i32(B * K), lens=i32(B * K), norm=ops.beam_norm(S, Gc, 1.0).to(dev))
            st["hs"][:, K] = 1e9
            return st

        def plain(st, cand):
            st["ps"][:, ::4] = reset                                   # step t, not done: every launch is the same step
            ops.beam_topk(logits, special, st["bs"], K, *cand)
            ops.beam_select(*cand, st["bs"], st["hist"], st["src"], st["hs"], st["hm"], st["ht"], st["ps"], st["nx"], st["lens"],
                            st["norm"], 2, 0, False)

        def grouped(st, cand, G):
            st["ps"][:, ::4] = reset
            for gi in range(G):
                ops.beam_topk_group(logits, special, st["bs"], K, G, gi, *cand, st["nx"], 0.5)
                ops.beam_select_group(*cand, st["bs"], st["hist"], st["src"], st["hs"], st["hm"], st["ht"], st["ps"], st["nx"],
                                      st["lens"], st["norm"], 2, 0, False, G, gi)

        def cands(c):
            return (torch.empty((B, c), dtype=torch.float32, device=dev), torch.empty((B, c), dtype=torch.int32, device=dev),
                    torch.empty((B, c), dtype=torch.int32, device=dev))
        reset = torch.tensor([t, 0], dtype=torch.int32, device=dev)
        st = state()
        reset_us = event_ms(lambda: st["ps"].__setitem__((slice(None), slice(None, None, 4)), reset), n)
        c = cands(2 * K)
        row = {"B": B, "K": K, "V": V, "launches": n, "reset_us": reset_us,
               "plain_step_us": round(event_ms(lambda: plain(st, c), n) - reset_us, 2)}
        for G in [G for k, G in GROUPS if k == K]:
            st = state()
            c = cands(2 * K // G)
            row[f"group_G{G}_step_us"] = round(event_ms(lambda: grouped(st, c, G), n) - reset_us, 2)
        rows.append(row)
        print(json.dumps(row), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=bench.N_LAYERS)
    ap.add_argument("--gens", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("diverse_beam_bench needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}), flush=True)
    if a.layers != bench.N_LAYERS:
        import navillm_b200.nav_model as nm
        nm.VICUNA_7B["num_hidden_layers"] = a.layers
    model = bench.build_model(dev, seed=0).eval()
    model._ensure()
    lm = model.lang_model
    lm._decode_states.max_states = 8                                     # one captured graph per arm
    res = {"gpu": gpu, "layers": a.layers, "kernel": kernel_times(lm, dev)}
    wl = bench.WORKLOADS["c3"]
    text, cand = prompts(model, 8, wl["n_cand_tok"], wl["n_text"], dev)
    batch = dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand)
    res["c3"] = {"B": 8, "S0": int(text["input_ids"].shape[1]), "max_new_tokens": 128,
                 "arms": arms_timed(lm, batch, arms(), a.gens, 128)}
    lm._decode_states.clear()
    torch.cuda.empty_cache()
    batch = summarization_batch(lm, dev)
    res["summarization"] = {"B": 8, "S0": int(batch["input_ids"].shape[1]), "hist_num": 7, "cand_num": 6, "max_new_tokens": 50,
                            "arms": arms_timed(lm, batch, arms(), a.gens, 50)}
    print(json.dumps(res))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
