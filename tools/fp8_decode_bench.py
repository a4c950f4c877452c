"""fp8 (e4m3) weight streaming vs bf16 in the decode step, in one process.

    python tools/fp8_decode_bench.py [--layers 32] [--iters 50] [--gens 3] [--out FILE.json]

(i)   per-GEMM time (CUDA events, bf16 skinny and fp8 skinny alternated, weights rotated over copies larger than L2) at the
      decode shapes of Vicuna-7B, with the bytes each kernel must move and the achieved GB/s;
(ii)  C3-shaped generate() (B = 8, S0 = 320, 128 new tokens, EOS stop off) on a random-init model at Vicuna-7B widths:
      decode ms/token in bf16 on the quantized weights W' and with the fp8 copy;
(iii) token agreement of those two runs (must be 100 %: the fp8 kernels are bit-identical to bf16 on W');
(iv)  for information, token agreement with the unquantized weights W;
(v)   the GPU name and power limit, read in the same run.

    python tools/fp8_decode_bench.py --kv [--batch 8 32 64] [--layers 32] [--gens 3] [--out FILE.json]

compares the KV-cache formats instead (set_kv_cache_dtype): (i) one layer's decode attention (RoPE + append + attention) over
a bf16 and over an fp8 cache at H = 32, Smax = 512 and C3's context lengths (CUDA events, the two kernels alternated, caches
rotated over copies larger than L2, bytes moved and GB/s); (ii) C3-shaped decode ms/token for {bf16 on W', fp8 weights} x
{bf16 KV, fp8 KV}, alternated, medians over the generations after each capture; (iii) for information, the token agreement
between the two KV formats (not required to be 100 %: fp8 KV attends over rounded keys and values).

    python tools/fp8_decode_bench.py --int4 [--batch 1 8 16] [--beams K | --samples N] [--layers 32] [--gens 3] [--rounds 2]
                                     [--out FILE.json]

adds the 4-bit group-wise weight copy (quantize_weights_int4): (i) per-GEMM time of the bf16, fp8 and int4 skinny kernels,
alternated, at M = 1, 8, 16 and the four decoder shapes, weights rotated, bytes moved and GB/s on each format's bytes
(int4: K/2 bytes of codes per row plus 3 bytes of scale and zero-point per 128 columns); (ii) C3-shaped decode ms/token at
each batch for bf16 on the int4 W', the fp8 copy and the int4 copy, the arms alternated over ``rounds`` rounds (each visit
restores W, quantizes, captures once and times ``gens`` generations); (iii) token agreement: int4 vs bf16 on its W' (must
be 100 %), and for information int4 vs fp8 and vs the unquantized W.
"""
import argparse
import gc
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from navillm_b200 import ops  # noqa: E402

SHAPES = [("qkv", 12288, 4096, False), ("o", 4096, 4096, False), ("gate_up+swiglu", 11008, 4096, True),
          ("down", 4096, 11008, False), ("lm_head", 32006, 4096, False)]


def gemm_table(dev, iters):
    rows = []
    g = torch.Generator(device=dev).manual_seed(0)
    for name, N, K, swiglu in SHAPES:
        wrows = 2 * N if swiglu else N
        ncopy = max(2, -(-160 * 2 ** 20 // (wrows * K)))                      # > 2 x the 50 MB L2 of bf16 weights per rotation
        w16 = [(torch.randn(wrows, K, device=dev, generator=g) * 0.02).to(torch.bfloat16) for _ in range(ncopy)]
        w8 = []
        for w in w16:
            q = torch.empty((wrows, K), dtype=ops.fp8, device=dev)
            e = torch.empty(wrows, dtype=torch.int8, device=dev)
            ops.quantize_fp8_(w, q, e)
            w8.append((q, e))
        for M in (1, 2, 8, 16):
            x = torch.randn(M, K, device=dev, generator=g).to(torch.bfloat16)
            if swiglu:
                f16 = lambda i: ops.gemm_skinny_swiglu(x, w16[i % ncopy])
                f8 = lambda i: ops.gemm_skinny_swiglu_fp8(x, *w8[i % ncopy])
            else:
                f16 = lambda i: ops.gemm_skinny(x, w16[i % ncopy])
                f8 = lambda i: ops.gemm_skinny_fp8(x, *w8[i % ncopy])
            same = torch.equal(f16(0), f8(0))
            t = {"bf16": [], "fp8": []}
            for i in range(5):                                                # warm-up
                f16(i); f8(i)
            torch.cuda.synchronize()
            for rep in range(4):                                              # alternate the two kernels
                for kind, f in (("bf16", f16), ("fp8", f8)) if rep % 2 == 0 else (("fp8", f8), ("bf16", f16)):
                    st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    st.record()
                    for i in range(iters):
                        f(i)
                    en.record()
                    torch.cuda.synchronize()
                    t[kind].append(st.elapsed_time(en) / iters)
            out_b = M * N * 2
            by16 = wrows * K * 2 + M * K * 2 + out_b
            by8 = wrows * K + wrows + M * K * 2 + out_b
            r = {"gemm": name, "M": M, "N": N, "K": K, "bit_identical": same}
            for kind, by in (("bf16", by16), ("fp8", by8)):
                us = 1e3 * float(np.median(t[kind]))
                r[f"{kind}_us"] = round(us, 2)
                r[f"{kind}_bytes"] = by
                r[f"{kind}_GBps"] = round(by / us / 1e3, 1)
            r["speedup"] = round(r["bf16_us"] / r["fp8_us"], 3)
            rows.append(r)
            print(json.dumps(r), flush=True)
        del w16, w8
        torch.cuda.empty_cache()
    return rows


def c3_generate(dev, layers, gens, batch=None):
    wl = bench.WORKLOADS["c3"]
    B, NV, NT, NEW = batch or wl["B"], wl["n_cand_tok"], wl["n_text"], wl["n_new"]
    if layers != bench.N_LAYERS:
        import navillm_b200.nav_model as nm
        nm.VICUNA_7B["num_hidden_layers"] = layers
    model = bench.build_model(dev, seed=0).eval()
    model._ensure()
    lm = model.lang_model
    rng = np.random.RandomState(1234)
    words = [f"w{i}" for i in range(5000)]
    prompts = ["Scene " + " ".join(["<cand>"] * NV) + " Question " + " ".join(words[i] for i in rng.randint(0, 5000, size=NT - 5))
               + " Answer" for _ in range(B)]
    text = lm.tokenize(prompts)
    S0 = int(text["attention_mask"].sum(1).max())
    g = torch.Generator().manual_seed(1234)
    with torch.no_grad():
        view = torch.stack([torch.randn(NV, bench.IMG_FEAT, generator=g) for _ in range(B)], 0).to(dev)
        pano = model.img_embeddings.forward_panorama_per_step(view_img_fts=view, view_lens=torch.full((B,), NV, device=dev))
        cand = model._masked_rows_plus_const(pano["pano_embeds"].reshape(B * NV, -1), np.ones((B, NV), dtype=bool)).detach()

    def run():
        per_tok, ids = [], None
        for _ in range(gens + 1):                                             # the first one captures the CUDA graph
            st = {}
            ids = lm.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand, max_new_tokens=NEW,
                              stop_on_eos=False, use_cuda_graph=True, stats=st)
            per_tok.append(st["decode_ms"] / st["decode_steps"])
        return float(np.median(per_tok[1:])), ids[:, text["input_ids"].shape[1]:].cpu()

    ms_w, ids_w = run()                                                       # bf16 on the original weights W
    nbytes = model.quantize_weights_fp8()
    ms8, ids8 = run()                                                         # fp8 copy
    lm.drop_fp8_weights()
    ms16, ids16 = run()                                                       # bf16 on W'
    agree = lambda a, b: float((a == b).float().mean())
    return {"B": B, "S0": S0, "new_tokens": NEW, "layers": layers, "fp8_copy_GB": round(nbytes / 1e9, 3),
            "decode_ms_per_token_bf16_W": round(ms_w, 4), "decode_ms_per_token_bf16_Wq": round(ms16, 4),
            "decode_ms_per_token_fp8": round(ms8, 4), "decode_speedup_fp8_vs_bf16_Wq": round(ms16 / ms8, 3),
            "token_agreement_fp8_vs_bf16_Wq": agree(ids8, ids16), "token_agreement_fp8_vs_bf16_W": agree(ids8, ids_w)}


def _round_cache(c):
    """Round a bf16 cache [B, Smax, H*128] in place to K' and return its fp8 form (e4m3 bytes, int8 [B, Smax, H] exponents)."""
    rows = c.view(-1, 128)
    q = torch.empty(rows.shape, dtype=ops.fp8, device=c.device)
    e = torch.empty(rows.shape[0], dtype=torch.int8, device=c.device)
    ops.quantize_fp8_(rows, q, e)
    return q.view(c.shape), e.view(c.shape[0], c.shape[1], c.shape[2] // 128)


def kv_attn_table(dev, iters, batches, H=32, Smax=512):
    """Decode attention (RoPE + append + attention, one layer) over a bf16 cache and over the fp8 cache, alternated, caches
    rotated over copies larger than L2; C3's context lengths 320..447 (mean 383.5)."""
    rows = []
    g = torch.Generator(device=dev).manual_seed(0)
    HD = H * 128
    cos_t, sin_t = bench_rope(dev, H, Smax)
    for B in batches:
        lens_h = [320 + (b * 37) % 128 for b in range(B)]
        lens = torch.tensor(lens_h, dtype=torch.int32, device=dev)
        per_copy = 2 * B * Smax * HD * 2
        ncopy = max(2, -(-200 * 2 ** 20 // per_copy))
        c16, c8 = [], []
        for _ in range(ncopy):
            kc = torch.randn(B, Smax, HD, device=dev, generator=g).to(torch.bfloat16)
            vc = torch.randn(B, Smax, HD, device=dev, generator=g).to(torch.bfloat16)
            kq, ke = _round_cache(kc)
            vq, ve = _round_cache(vc)
            c16.append((kc, vc))
            c8.append((kq, vq, ke, ve))
        qkv = torch.randn(B, 3 * HD, device=dev, generator=g).to(torch.bfloat16)
        out = torch.empty(B, HD, dtype=torch.bfloat16, device=dev)
        f16 = lambda i: ops.decode_attn_rope(qkv, lens, cos_t, sin_t, *c16[i % ncopy], H, out=out)
        f8 = lambda i: ops.decode_attn_rope_fp8(qkv, lens, cos_t, sin_t, *c8[i % ncopy], H, out=out)
        t = {"bf16": [], "fp8": []}
        for i in range(5):
            f16(i); f8(i)
        torch.cuda.synchronize()
        for rep in range(6):
            for kind, f in (("bf16", f16), ("fp8", f8)) if rep % 2 == 0 else (("fp8", f8), ("bf16", f16)):
                st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                st.record()
                for i in range(iters):
                    f(i)
                en.record()
                torch.cuda.synchronize()
                t[kind].append(st.elapsed_time(en) / iters)
        keys = sum(l + 1 for l in lens_h)
        io = B * 3 * HD * 2 + B * HD * 2
        by16 = keys * HD * 2 * 2 + io
        by8 = keys * HD * 2 + keys * H * 2 + io
        r = {"B": B, "H": H, "Smax": Smax, "mean_len": sum(lens_h) / B}
        for kind, by in (("bf16", by16), ("fp8", by8)):
            us = 1e3 * float(np.median(t[kind]))
            r[f"{kind}_us"] = round(us, 2)
            r[f"{kind}_bytes"] = by
            r[f"{kind}_GBps"] = round(by / us / 1e3, 1)
        r["speedup"] = round(r["bf16_us"] / r["fp8_us"], 3)
        rows.append(r)
        print(json.dumps(r), flush=True)
        del c16, c8
        torch.cuda.empty_cache()
    return rows


def bench_rope(dev, H, Smax):
    from navillm_b200.llama import LlamaDims, rope_tables
    return rope_tables(LlamaDims(hidden=H * 128, n_heads=H, max_pos=Smax), dev)


def c3_generate_kv(dev, layers, gens, batch, rounds=2):
    """C3-shaped decode ms/token for {bf16 on W', fp8 weights} x {bf16 KV, fp8 KV}: the weight arms alternate in blocks (the
    captured graphs are dropped between blocks), the KV arms alternate inside each block; every visit captures once and
    times ``gens`` generations after the capture.  Medians per arm; token agreement between the KV formats for information."""
    wl = bench.WORKLOADS["c3"]
    B, NV, NT, NEW = batch, wl["n_cand_tok"], wl["n_text"], wl["n_new"]
    if layers != bench.N_LAYERS:
        import navillm_b200.nav_model as nm
        nm.VICUNA_7B["num_hidden_layers"] = layers
    model = bench.build_model(dev, seed=0).eval()
    model._ensure()
    lm = model.lang_model
    rng = np.random.RandomState(1234)
    words = [f"w{i}" for i in range(5000)]
    prompts = ["Scene " + " ".join(["<cand>"] * NV) + " Question " + " ".join(words[i] for i in rng.randint(0, 5000, size=NT - 5))
               + " Answer" for _ in range(B)]
    text = lm.tokenize(prompts)
    S0 = int(text["attention_mask"].sum(1).max())
    g = torch.Generator().manual_seed(1234)
    with torch.no_grad():
        view = torch.stack([torch.randn(NV, bench.IMG_FEAT, generator=g) for _ in range(B)], 0).to(dev)
        pano = model.img_embeddings.forward_panorama_per_step(view_img_fts=view, view_lens=torch.full((B,), NV, device=dev))
        cand = model._masked_rows_plus_const(pano["pano_embeds"].reshape(B * NV, -1), np.ones((B, NV), dtype=bool)).detach()
    model.quantize_weights_fp8()
    fp8w = lm.fp8_weights
    times = {(w, kv): [] for w in ("bf16", "fp8") for kv in ("bf16", "fp8")}
    ids = {}
    for rnd in range(2 * rounds):
        w = ("bf16", "fp8")[rnd % 2]
        lm._decode_states.clear()                                           # graphs bake in the weight kernels
        lm._fp8 = fp8w if w == "fp8" else None
        lm.core.set_fp8(lm._fp8)
        for kv in (("bf16", "fp8") if rnd % 4 < 2 else ("fp8", "bf16")):
            lm.set_kv_cache_dtype(kv)
            for i in range(gens + 1):                                       # the first one captures the CUDA graph
                st = {}
                out = lm.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand,
                                  max_new_tokens=NEW, stop_on_eos=False, use_cuda_graph=True, stats=st)
                if i > 0:
                    times[(w, kv)].append(st["decode_ms"] / st["decode_steps"])
            ids[(w, kv)] = out[:, text["input_ids"].shape[1]:].cpu()
    lm.set_kv_cache_dtype("bf16")
    med = {k: float(np.median(v)) for k, v in times.items()}
    agree = lambda a, b: float((a == b).float().mean())
    r = {"B": B, "S0": S0, "new_tokens": NEW, "layers": layers, "generations_per_arm": len(times[("bf16", "bf16")])}
    for (w, kv), ms in med.items():
        r[f"decode_ms_per_token_w_{w}_kv_{kv}"] = round(ms, 4)
    for w in ("bf16", "fp8"):
        r[f"kv_speedup_fp8_vs_bf16_w_{w}"] = round(med[(w, "bf16")] / med[(w, "fp8")], 3)
        r[f"token_agreement_kv_fp8_vs_bf16_w_{w}"] = agree(ids[(w, "fp8")], ids[(w, "bf16")])
    return r


INT4_SHAPES = SHAPES[:4]


def gemm_table_int4(dev, iters):
    """bf16 / fp8 / int4 skinny GEMMs alternated at the four decoder shapes, M = 1, 8, 16."""
    rows = []
    g = torch.Generator(device=dev).manual_seed(0)
    for name, N, K, swiglu in INT4_SHAPES:
        wrows = 2 * N if swiglu else N
        ncopy = max(2, -(-160 * 2 ** 20 // (wrows * K)))
        w16, w8, w4 = [], [], []
        for _ in range(ncopy):
            w = (torch.randn(wrows, K, device=dev, generator=g) * 0.02).to(torch.bfloat16)
            q = torch.empty((wrows, K), dtype=ops.fp8, device=dev)
            e = torch.empty(wrows, dtype=torch.int8, device=dev)
            ops.quantize_fp8_(w.clone(), q, e)
            c = torch.empty(ops.int4_codes_shape(wrows, K), dtype=torch.uint8, device=dev)
            sc = torch.empty((wrows, K // 128), dtype=torch.bfloat16, device=dev)
            z = torch.empty((wrows, K // 128), dtype=torch.uint8, device=dev)
            ops.quantize_int4_(w, c, sc, z)                                   # w is now the int4 W'
            w16.append(w); w8.append((q, e)); w4.append((c, sc, z))
        for M in (1, 8, 16):
            x = torch.randn(M, K, device=dev, generator=g).to(torch.bfloat16)
            if swiglu:
                fs = {"bf16": lambda i: ops.gemm_skinny_swiglu(x, w16[i % ncopy]),
                      "fp8": lambda i: ops.gemm_skinny_swiglu_fp8(x, *w8[i % ncopy]),
                      "int4": lambda i: ops.gemm_skinny_swiglu_int4(x, *w4[i % ncopy])}
            else:
                fs = {"bf16": lambda i: ops.gemm_skinny(x, w16[i % ncopy]),
                      "fp8": lambda i: ops.gemm_skinny_fp8(x, *w8[i % ncopy]),
                      "int4": lambda i: ops.gemm_skinny_int4(x, *w4[i % ncopy])}
            same = torch.equal(fs["bf16"](0), fs["int4"](0))
            t = {k: [] for k in fs}
            for i in range(5):
                for f in fs.values():
                    f(i)
            torch.cuda.synchronize()
            order = list(fs)
            for rep in range(6):                                              # rotate the order of the three kernels
                for kind in order[rep % 3:] + order[:rep % 3]:
                    st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    st.record()
                    for i in range(iters):
                        fs[kind](i)
                    en.record()
                    torch.cuda.synchronize()
                    t[kind].append(st.elapsed_time(en) / iters)
            io = M * K * 2 + M * N * 2
            by = {"bf16": wrows * K * 2 + io, "fp8": wrows * K + wrows + io, "int4": wrows * K // 2 + wrows * (K // 128) * 3 + io}
            r = {"gemm": name, "M": M, "N": N, "K": K, "int4_bit_identical_to_bf16_on_Wq": same}
            for kind in fs:
                us = 1e3 * float(np.median(t[kind]))
                r[f"{kind}_us"] = round(us, 2)
                r[f"{kind}_bytes"] = by[kind]
                r[f"{kind}_GBps"] = round(by[kind] / us / 1e3, 1)
            r["int4_vs_fp8"] = round(r["fp8_us"] / r["int4_us"], 3)
            r["int4_vs_bf16"] = round(r["bf16_us"] / r["int4_us"], 3)
            rows.append(r)
            print(json.dumps(r), flush=True)
        del w16, w8, w4
        torch.cuda.empty_cache()
    return rows


def c3_model(dev, layers):
    if layers != bench.N_LAYERS:
        import navillm_b200.nav_model as nm
        nm.VICUNA_7B["num_hidden_layers"] = layers
    model = bench.build_model(dev, seed=0).eval()
    model._ensure()
    return model, model.lang_model.flat.flat.clone()


def c3_generate_int4(dev, model, W, layers, gens, batch, rounds, beams=1, samples=1):
    """C3-shaped decode ms/token for bf16 on the int4 W', the fp8 copy and the int4 copy, alternated: every visit restores
    the weights W, quantizes for its arm, captures once and times ``gens`` generations.  ``beams`` > 1: beam search with
    that many beams per prompt; ``samples`` > 1: that many sampled sequences per prompt (top-p 0.9, one seed per call)."""
    wl = bench.WORKLOADS["c3"]
    B, NV, NT, NEW = batch, wl["n_cand_tok"], wl["n_text"], wl["n_new"]
    lm = model.lang_model
    lm.drop_fp8_weights()
    lm.drop_int4_weights()
    with torch.no_grad():
        lm.flat.flat.copy_(W)
    rng = np.random.RandomState(1234)
    words = [f"w{i}" for i in range(5000)]
    prompts = ["Scene " + " ".join(["<cand>"] * NV) + " Question " + " ".join(words[i] for i in rng.randint(0, 5000, size=NT - 5))
               + " Answer" for _ in range(B)]
    text = lm.tokenize(prompts)
    S0 = int(text["attention_mask"].sum(1).max())
    g = torch.Generator().manual_seed(1234)
    with torch.no_grad():
        view = torch.stack([torch.randn(NV, bench.IMG_FEAT, generator=g) for _ in range(B)], 0).to(dev)
        pano = model.img_embeddings.forward_panorama_per_step(view_img_fts=view, view_lens=torch.full((B,), NV, device=dev))
        cand = model._masked_rows_plus_const(pano["pano_embeds"].reshape(B * NV, -1), np.ones((B, NV), dtype=bool)).detach()

    mode = dict(num_beams=beams) if beams > 1 else dict(do_sample=True, top_p=0.9, num_return_sequences=samples) if samples > 1 else {}

    def run(n):
        per_tok, out = [], None
        for i in range(n + 1):                                                # the first one captures the CUDA graph
            st = {}
            torch.manual_seed(0)
            out = lm.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand,
                              max_new_tokens=NEW, stop_on_eos=False, use_cuda_graph=True, stats=st, **mode)
            if i > 0:
                per_tok.append(st["decode_ms"] / st["decode_steps"])
        return per_tok, out[:, text["input_ids"].shape[1]:].cpu()

    _, ids_w = run(0)                                                         # bf16 on the unquantized W
    arms = ("int4", "fp8", "bf16_Wq4")
    times, ids, nbytes = {a: [] for a in arms}, {}, {}
    for rnd in range(rounds):
        for arm in arms[rnd % 3:] + arms[:rnd % 3]:
            lm.drop_fp8_weights()
            lm.drop_int4_weights()
            with torch.no_grad():
                lm.flat.flat.copy_(W)
            if arm == "fp8":
                nbytes["fp8"] = model.quantize_weights_fp8()
            else:
                nbytes["int4"] = model.quantize_weights_int4()
                if arm == "bf16_Wq4":
                    lm.drop_int4_weights()
            pt, ids[arm] = run(gens)
            times[arm] += pt
    lm.drop_fp8_weights()
    lm.drop_int4_weights()
    med = {a: float(np.median(v)) for a, v in times.items()}
    agree = lambda a, b: float((a == b).float().mean())
    return {"B": B, "beams": beams, "samples": samples, "decode_rows": B * beams * samples, "S0": S0, "new_tokens": NEW,
            "layers": layers, "generations_per_arm": len(times["int4"]),
            "int4_copy_GB": round(nbytes["int4"] / 1e9, 3), "fp8_copy_GB": round(nbytes["fp8"] / 1e9, 3),
            "decode_ms_per_token_bf16_Wq4": round(med["bf16_Wq4"], 4), "decode_ms_per_token_fp8": round(med["fp8"], 4),
            "decode_ms_per_token_int4": round(med["int4"], 4),
            "decode_ms_per_token_spread": {a: [round(min(v), 4), round(max(v), 4)] for a, v in times.items()},
            "int4_vs_fp8": round(med["fp8"] / med["int4"], 3), "int4_vs_bf16_Wq4": round(med["bf16_Wq4"] / med["int4"], 3),
            "token_agreement_int4_vs_bf16_Wq4": agree(ids["int4"], ids["bf16_Wq4"]),
            "token_agreement_int4_vs_fp8": agree(ids["int4"], ids["fp8"]), "token_agreement_int4_vs_bf16_W": agree(ids["int4"], ids_w)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--gens", type=int, default=3)
    ap.add_argument("--skip-gemm", action="store_true")
    ap.add_argument("--batch", type=int, nargs="*", default=[], help="decode batch sizes of the generate comparison (default: C3's)")
    ap.add_argument("--kv", action="store_true", help="compare the bf16 and the fp8 KV cache instead of the weight formats alone: "
                                                       "decode-attention kernel times, then generate() over weights x KV formats")
    ap.add_argument("--int4", action="store_true", help="add the int4 weight copy: bf16 / fp8 / int4 GEMMs, then generate() "
                                                         "for bf16 on the int4 W', fp8 and int4, alternated")
    ap.add_argument("--rounds", type=int, default=2, help="--int4: visits of each arm per batch size")
    ap.add_argument("--beams", type=int, default=1, help="--int4: beam search with this many beams per prompt")
    ap.add_argument("--samples", type=int, default=1, help="--int4: this many sampled sequences per prompt")
    ap.add_argument("--out", default=None, help="also write the result as JSON here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_decode_bench: needs an H100 (no CPU path)")
    dev = torch.device("cuda:0")
    res = {"gpu": bench.gpu_info(0)}
    print(json.dumps(res["gpu"]), flush=True)
    if a.int4:
        res["gemm_int4"] = [] if a.skip_gemm else gemm_table_int4(dev, a.iters)
        res["c3_generate_int4"] = []
        model, W = c3_model(dev, a.layers)
        for b in a.batch or [1, 8, 16]:
            res["c3_generate_int4"].append(c3_generate_int4(dev, model, W, a.layers, a.gens, b, a.rounds, a.beams, a.samples))
            print(json.dumps(res["c3_generate_int4"][-1]), flush=True)
            gc.collect()
            torch.cuda.empty_cache()
        res["gpu_after"] = bench.gpu_info(0)
        if a.out:
            Path(a.out).parent.mkdir(parents=True, exist_ok=True)
            Path(a.out).write_text(json.dumps(res, indent=1))
        return
    if a.kv:
        batches = a.batch or [8, 32, 64]
        res["kv_attention"] = kv_attn_table(dev, a.iters, batches)
        res["c3_generate_kv"] = []
        for b in batches:
            res["c3_generate_kv"].append(c3_generate_kv(dev, a.layers, a.gens, b))
            print(json.dumps(res["c3_generate_kv"][-1]), flush=True)
            gc.collect()
            torch.cuda.empty_cache()
        if a.out:
            Path(a.out).parent.mkdir(parents=True, exist_ok=True)
            Path(a.out).write_text(json.dumps(res, indent=1))
        return
    res["gemm"] = [] if a.skip_gemm else gemm_table(dev, a.iters)
    res["c3_generate"] = []
    for b in a.batch or [None]:
        res["c3_generate"].append(c3_generate(dev, a.layers, a.gens, b))
        print(json.dumps(res["c3_generate"][-1]), flush=True)
        gc.collect()                                                          # one 7B model (+ copy, + KV caches) at a time
        torch.cuda.empty_cache()
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
