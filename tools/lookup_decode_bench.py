"""Prompt-lookup speculative decoding in generate() at Vicuna-7B widths (random init), against plain greedy decoding.

    python tools/lookup_decode_bench.py [--layers 32] [--gens 2] [--Bs 1,8,16] [--ks 2,4,8,15] [--weights bf16,fp8,int4]
                                        [--out FILE.json]

Shape: C3 (256 <cand> + 64 text tokens, 128 new tokens, EOS stopping off) at each B and k.  Per (weights, B, k) four arms,
alternated generation by generation (the first generation of each captures its CUDA graph and is not counted):
  greedy    plain greedy decoding at B: ms per token;
  rejected  every draft wrong (a special id, which the argmax never picks): 1 token per step, the pure cost of the window;
  oracle    the drafts are the lookup path's own output: k + 1 tokens per step, the upper bound;
  ngram     the n-gram drafts themselves: information only, random weights say nothing about trained text.
For each: ms per verify step (decode_ms / decode_steps, the steps after the first token) and tokens per step per row.  The
break-even is the accepted drafts per step at which a verify step costs what greedy pays for its tokens: rejected ms per step /
greedy ms per token - 1.  Then the window kernel alone against W sequential decode_attn_rope calls (B = 8, H = 32, S = 320 and
2048 cached keys), timed with CUDA events over 50 launches.  The GPU name and power limit are read in the same run.
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
from contrastive_bench import event_ms  # noqa: E402


class Drafts:
    """ops.lookup_draft replaced: "rejected" drafts a special id, "oracle" the given greedy continuation."""

    def __init__(self, kind, special_id=None, gen=None, plens=None):
        self.kind, self.special_id, self.gen, self.plens = kind, special_id, gen, plens

    def __call__(self, hist, hist_len, finished, special, eos_id, ngram, drafts, win_ids):
        k = drafts.shape[1]
        if self.kind == "rejected":
            drafts.fill_(self.special_id)
        else:
            i = (hist_len - self.plens).long()[:, None] + torch.arange(k, device=drafts.device)[None]
            ok = i < self.gen.shape[1]
            drafts.copy_(torch.where(ok, self.gen.gather(1, i.clamp(max=self.gen.shape[1] - 1)), torch.full_like(drafts, -1)))
        last = hist.gather(1, (hist_len.long() - 1)[:, None])
        win_ids[:, :1].copy_(last)
        win_ids[:, 1:].copy_(torch.where(drafts < 0, last, drafts))


def run(lm, text, cand, new, drafts=None, **kw):
    from navillm_b200 import ops
    real = ops.lookup_draft
    if drafts is not None:
        ops.lookup_draft = drafts
    try:
        st = {}
        ids = lm.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand, max_new_tokens=new,
                          stop_on_eos=False, use_cuda_graph=True, stats=st, **kw)
        torch.cuda.synchronize()
    finally:
        ops.lookup_draft = real
    return ids, st


def window_kernel_times(dev):
    """decode_attn_rope_window against W sequential decode_attn_rope calls: B = 8, H = 32, Smax = 2048 + 16."""
    from navillm_b200 import ops
    from navillm_b200.llama import LlamaDims, rope_tables
    B, H, Smax = 8, 32, 2048 + 16
    HD = H * 128
    cos_t, sin_t = rope_tables(LlamaDims(hidden=HD, n_heads=H, max_pos=Smax), dev)
    kc = torch.randn(B, Smax, HD, device=dev).to(torch.bfloat16)
    vc = torch.randn(B, Smax, HD, device=dev).to(torch.bfloat16)
    rows = []
    for S in (320, 2048):
        lens = torch.full((B,), S, dtype=torch.int32, device=dev)
        for W in (2, 3, 5, 9, 16):
            qkv = torch.randn(B * W, 3 * HD, device=dev).to(torch.bfloat16)
            out = torch.empty(B * W, HD, dtype=torch.bfloat16, device=dev)
            qs = [qkv[j::W].contiguous() for j in range(W)]
            ls = [lens + j for j in range(W)]
            outs = [torch.empty(B, HD, dtype=torch.bfloat16, device=dev) for _ in range(W)]
            win = event_ms(lambda: ops.decode_attn_rope_window(qkv, lens, cos_t, sin_t, kc, vc, H, W, out=out))

            def seq():
                for j in range(W):
                    ops.decode_attn_rope(qs[j], ls[j], cos_t, sin_t, kc, vc, H, out=outs[j])
            rows.append({"S": S, "W": W, "window_us": win, "sequential_us": event_ms(seq),
                         "one_step_us": event_ms(lambda: ops.decode_attn_rope(qs[0], ls[0], cos_t, sin_t, kc, vc, H, out=outs[0]))})
            print(json.dumps(rows[-1]), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=bench.N_LAYERS)
    ap.add_argument("--gens", type=int, default=2)
    ap.add_argument("--Bs", default="1,8,16")
    ap.add_argument("--ks", default="2,4,8,15")
    ap.add_argument("--weights", default="bf16,fp8,int4")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lookup_decode_bench needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    if a.layers != bench.N_LAYERS:
        import navillm_b200.nav_model as nm
        nm.VICUNA_7B["num_hidden_layers"] = a.layers
    model = bench.build_model(dev, seed=0).eval()
    model._ensure()
    lm = model.lang_model
    lm._decode_states.max_states = 5                                     # one captured graph per arm
    wl = bench.WORKLOADS["c3"]
    new = wl["n_new"]
    special_id = int(lm.special_ids_dev[0])
    res = {"gpu": gpu, "layers": a.layers, "new_tokens": new, "kernel": window_kernel_times(dev), "rows": []}
    for weights in a.weights.split(","):
        if weights != "bf16":
            getattr(model, f"quantize_weights_{weights}")()
        for B in [int(x) for x in a.Bs.split(",")]:
            text, cand = prompts(model, B, wl["n_cand_tok"], wl["n_text"], dev)
            S = text["input_ids"].shape[1]
            greedy_ids, _ = run(lm, text, cand, new)
            plens = text["attention_mask"].sum(1).to(torch.int32).to(dev)
            for k in [int(x) for x in a.ks.split(",")]:
                # the oracle drafts are the lookup path's own tokens at this k (the rejected arm's: the same B * (k + 1)-row
                # GEMMs give every draft source the same ids); plain greedy's can part from them at a near tie, which random
                # weights make common
                rej = Drafts("rejected", special_id)
                lk_ids, _ = run(lm, text, cand, new, prompt_lookup_num_tokens=k, max_matching_ngram_size=101, drafts=rej)
                gen = lk_ids[:, S:].to(torch.int32).contiguous()
                # the replaced drafts are baked into a captured step: a max_matching_ngram_size of their own (unused by them)
                # gives each of those arms its own decode state and graph
                arms = {"greedy": {}, "rejected": dict(prompt_lookup_num_tokens=k, max_matching_ngram_size=101, drafts=rej),
                        "oracle": dict(prompt_lookup_num_tokens=k, max_matching_ngram_size=102,
                                       drafts=Drafts("oracle", gen=gen, plens=plens)),
                        "ngram": dict(prompt_lookup_num_tokens=k)}
                runs = {n: [] for n in arms}
                for _ in range(a.gens + 1):                              # the arms alternate, generation by generation
                    for name, kw in arms.items():
                        ids, st = run(lm, text, cand, new, **kw)
                        tok = st.get("lookup_tokens", B * (st["decode_steps"]))
                        runs[name].append((st["decode_ms"] / st["decode_steps"], tok / B / st["decode_steps"],
                                           bool(torch.equal(ids, greedy_ids)), bool(torch.equal(ids, lk_ids))))
                r = {"weights": weights, "B": B, "k": k, "S0": S}
                for name, v in runs.items():
                    v = v[1:]
                    r[name] = {"ms_per_step": round(float(np.median([x[0] for x in v])), 4),
                               "ms_spread": round(float(max(x[0] for x in v) - min(x[0] for x in v)), 4),
                               "tokens_per_step": round(float(np.median([x[1] for x in v])), 3),
                               "ids_equal_greedy": all(x[2] for x in v), "ids_equal_rejected_arm": all(x[3] for x in v)}
                    r[name]["ms_per_token"] = round(r[name]["ms_per_step"] / r[name]["tokens_per_step"], 4)
                r["break_even_accepted_per_step"] = round(r["rejected"]["ms_per_step"] / r["greedy"]["ms_per_token"] - 1, 3)
                print(json.dumps(r), flush=True)
                res["rows"].append(r)
                lm._decode_states.clear()
            del text, cand
            torch.cuda.empty_cache()
        if weights != "bf16":
            getattr(model, f"drop_{weights}_weights")()
    print(json.dumps(res))
    if a.out:
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
