"""bench.py — throughput of the NaviLLM per-step hot path on synthetic batches, Vicuna-7B, bf16, on N H100s (one process per GPU).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--workload c2|c5|c3]   # this repo (sm_90a kernels)
    python bench.py ... --dump-outputs DIR                                      # + what the last timed step computed
    python bench.py --impl reference [...]                                      # the reference path on the host cores

Workloads (BASELINE.json `configs`, SURVEY.md §8d):
  c2 (default; configs[1], the configuration the metric is quoted on): R2R-shaped training step, B=16 per GPU, 36 x 1408
     views, hist=8, 24 graph nodes, 15 candidates + stop, prompt lengths U{256..1024}.  One "step" = one batch of 16
     navigation steps: model('panorama') -> model('navigation') -> CE(fuse_logits, targets) -> backward.  nav-steps/s.
  c1 (configs[0], the reference's own CPU-runnable case): ONE navigation step, forward only, batch=1; `--impl reference`
     runs the FULL 32-layer oracle port on the host cores for it (no layer scaling).
  c5 (configs[4] per rank): CVDN long horizon, B=4 per GPU, hist=40, 64 graph nodes, 24 candidates, dense S=2048.
  c4 (configs[3] per rank): multi-task mixed batch, 8 samples per GPU as 4 micro-batches (R2R, CVDN, SOON + object grounding,
     ScanQA LM loss) accumulated under no_sync() with ONE gradient exchange per step; samples/s.
  c3 (configs[2]): ScanQA-shaped greedy generation, B=8 per GPU, 256 <cand> + 64 text tokens, 128 new tokens;
     tokens/s, prefill ms, ms/token and the HBM roofline of the CUDA-graph decode step.
`value` times the step with all inputs resident in HBM; `e2e` times the same call sequence through the public API from
HOST (pinned) buffers: per step the H2D copy of every input tensor, host tokenisation / index building and a D2H read of the
result.  Multi-GPU: weak scaling, one batch per rank; the model is wrapped in navillm_b200.parallel.DistributedDataParallel
(the one-line replacement of tools/optims.py:52-54) and exchanges its flat gradient buffers over NCCL every step, inside
the timed region.

The `--impl reference` arm and `cpu_baseline` time the CPU oracle port of the reference algorithm (oracle/navillm_oracle.py;
kind "port": the reference is Python and is not part of this repository) on the host cores over a BOUNDED
sample: full-width Vicuna-7B layers, B=1, one prompt of the workload's mean length, 2 of the 32 layers, at most 3 timed
passes and a hard wall-clock cap, whatever --steps says.

`--dump-outputs DIR` writes, after the timed steps, what the timed path computed in its last step as DIR/<name>.npy
(float32 / float64, finite): the loss and the navigation logits (training workloads; per micro-batch losses for c4) or the generated
token ids (c3), plus a fixed, seeded sample of every parameter gradient.  The inputs depend only on the arguments (seeded
synthetic batches, seeded initialisation) and every reduction of the path sums in a fixed order (no float atomics), so
two runs of one build write identical files and two builds can be compared output for output.

Progress goes to stderr, one line per phase, so a lost box is attributable; stdout carries exactly one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time
import types
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

D_MODEL, N_LAYERS, N_HEADS, D_FF, VOCAB = 4096, 32, 32, 11008, 32000
IMG_FEAT = 1408
N_VIEWS = 36
# C2 defaults (module-level so tools/ and tests/ can import the generator)
B_STEP, N_HIST, N_GMAP, N_CAND = 16, 8, 24, 16
LEN_LO, LEN_HI = 256, 1024

WORKLOADS = {
    "c2": dict(B=16, n_hist=8, n_gmap=24, n_cand=16, len_lo=256, len_hi=1024, max_length=1024,
               name="C2 R2R-shaped training step (panorama+navigation fwd+bwd), B=16/GPU, 36x1408 views, hist=8, 24 graph nodes, "
                    "15 candidates, seq U{256..1024} (packed: pad tokens not computed), Vicuna-7B random init"),
    "c5": dict(B=4, n_hist=40, n_gmap=64, n_cand=24, len_lo=2048, len_hi=2048, max_length=4096,
               name="C5 CVDN long-horizon training step (panorama+navigation fwd+bwd), B=4/GPU (32 on 8 GPUs), 36x1408 views, hist=40, "
                    "64 graph nodes, 23 candidates, dense seq=2048, Vicuna-7B random init"),
    "c1": dict(B=1, n_hist=0, n_gmap=4, n_cand=4, len_lo=192, len_hi=192, max_length=1024,
               name="C1 single navigation step FORWARD only (plumbing config): batch=1, 36x1408 views, 64-token instruction + prompt "
                    "boilerplate (S=192), 3 candidates + stop, Vicuna-7B random init"),
    "c4": dict(B=8, name="C4 multi-task mixed step (fwd+bwd, gradient accumulation over 4 micro-batches of 2 samples per GPU: R2R hist=8 "
                         "S<=512; CVDN hist=20 S<=1024; SOON hist=10 S<=768 + object grounding over 40 objects; ScanQA 36 <cand> + "
                         "16-token answer LM loss), 8 samples/GPU = global batch 64 on 8 GPUs, Vicuna-7B random init"),
    "c3": dict(B=8, n_cand_tok=256, n_text=64, n_new=128,
               name="C3 ScanQA-shaped greedy generate, B=8/GPU, 256 <cand> visual tokens + 64 text tokens (S0=320), 128 new tokens, "
                    "Vicuna-7B random init"),
}

C4_MEAN_LEN = 520           # mean prompt length of the four C4 micro-batch shapes (384, 768, 576, ~350)
T0 = time.time()


def log(msg: str) -> None:
    print(f"[bench +{time.time() - T0:6.1f}s rank{os.environ.get('RANK', '0')}] {msg}", file=sys.stderr, flush=True)


def peaks():
    p = ROOT / "MEASURED_PEAKS.json"
    if p.exists():
        j = json.loads(p.read_text())
        return {"bf16_tflops": j.get("bf16_tflops_sustained", j.get("bf16_tflops")), "hbm_gbs": j.get("hbm_gbs"), "src": "measured"}
    # NVIDIA H100 SXM data sheet (dense bf16, HBM3), for a card allowed 700 W: an upper bound, not a measured rate
    return {"bf16_tflops": 989.0, "hbm_gbs": 3350.0, "src": "H100 SXM data sheet"}


def gpu_info(index: int) -> dict:
    """Which card the numbers of this run were measured on, and its power limit."""
    info = {"name": torch.cuda.get_device_name(index), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(index)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except Exception:
        pass
    return info


DUMP_GRAD_SAMPLE = 4096      # gradient elements sampled per parameter tensor by --dump-outputs


def dump_outputs(out_dir, arrays: dict, model=None) -> None:
    """--dump-outputs: arrays (name -> tensor / ndarray) as DIR/<name>.npy in float32 (float64 stays float64), plus
    `grad_sample.npy`: DUMP_GRAD_SAMPLE elements of every parameter gradient at indices drawn from a generator seeded
    with the parameter's position (the same elements in every run), concatenated in parameter order.  Every file holds
    finite numbers: an array with non-finite entries (the -inf of masked navigation slots) is written with those entries
    set to 0, next to `<name>_finite.npy` (1 where the value was finite, 0 where not)."""
    d = Path(out_dir)
    d.mkdir(parents=True, exist_ok=True)
    total = 0
    if model is not None:
        parts = []
        for i, p in enumerate(model.parameters()):
            if p.grad is None:
                continue
            flat = p.grad.detach().reshape(-1)
            idx = torch.randint(flat.numel(), (min(DUMP_GRAD_SAMPLE, flat.numel()),), generator=torch.Generator().manual_seed(i))
            parts.append(flat[idx.to(flat.device)].float().cpu())
        if parts:
            arrays = dict(arrays, grad_sample=torch.cat(parts))
    for name, v in arrays.items():
        a = v.detach().cpu().numpy() if torch.is_tensor(v) and v.dtype != torch.bfloat16 else (
            v.detach().float().cpu().numpy() if torch.is_tensor(v) else np.asarray(v))
        a = a.astype(np.float64 if a.dtype == np.float64 else np.float32)
        fin = np.isfinite(a)
        if not fin.all():
            np.save(d / f"{name}_finite.npy", fin.astype(np.float32))
            total += fin.size * 4
            a = np.where(fin, a, 0).astype(a.dtype)
        total += a.nbytes
        np.save(d / f"{name}.npy", a)
    assert total <= 64 << 20, f"--dump-outputs wrote {total} bytes (> 64 MB)"
    log(f"outputs of the last timed step written to {d} ({total} bytes)")


# ---------------------------------------------------------------------------------------------------------
# synthetic workloads (SURVEY.md §8d)
# ---------------------------------------------------------------------------------------------------------
def make_workload(seed: int, B: int = None, n_hist: int = None, n_gmap: int = None, n_cand: int = None, len_lo: int = None,
                  len_hi: int = None, **unused):
    B = B_STEP if B is None else B
    n_hist = N_HIST if n_hist is None else n_hist
    n_gmap = N_GMAP if n_gmap is None else n_gmap
    n_cand = N_CAND if n_cand is None else n_cand
    len_lo = LEN_LO if len_lo is None else len_lo
    len_hi = LEN_HI if len_hi is None else len_hi
    assert n_gmap == 1 + n_hist + (n_cand - 1), "graph = stop + visited (history) + current candidates (one <cand> token each)"
    rng = np.random.RandomState(seed)
    g = torch.Generator().manual_seed(seed)
    lens = rng.randint(len_lo, len_hi + 1, size=B)
    words = [f"w{i}" for i in range(5000)]
    prompts = []
    n_c = n_cand - 1
    for b in range(B):
        n_words = int(lens[b]) - (1 + n_hist + n_c + 1 + 4)          # bos + hist + cand + cls + 4 section words
        instr = " ".join(words[i] for i in rng.randint(0, len(words), size=max(n_words, 1)))
        prompts.append("Instruction " + instr + " History " + " ".join(["<hist>"] * n_hist) + " Candidates stop "
                       + " ".join(["<cand>"] * n_c) + " Answer <cls_1>")
    heading = torch.rand(B, N_VIEWS, generator=g) * 6.2831853
    elev = (torch.randint(0, 3, (B, N_VIEWS), generator=g).float() - 1) * 0.5235988
    loc = torch.stack([heading.sin(), heading.cos(), elev.sin(), elev.cos()], -1)
    loc = torch.cat([loc, torch.ones(B, N_VIEWS, 3)], -1)
    nav_types = torch.zeros(B, N_VIEWS, dtype=torch.long)
    nav_types[:, :n_c] = 1
    # graph: slot 0 = stop, n_hist visited nodes, then unvisited; the first n_c unvisited are the current candidates
    gmap_vpids = [[None] + [f"v{j}" for j in range(n_hist)] + [f"c{j}" for j in range(n_gmap - 1 - n_hist)] for _ in range(B)]
    visited = torch.zeros(B, n_gmap, dtype=torch.bool)
    visited[:, 1:1 + n_hist] = True
    step_ids = torch.zeros(B, n_gmap, dtype=torch.long)
    step_ids[:, 1:1 + n_hist] = torch.arange(1, n_hist + 1)
    host = {
        "view_img_fts": torch.randn(B, N_VIEWS, IMG_FEAT, generator=g),
        "loc_fts": loc,
        "nav_types": nav_types,
        "vp_pos_fts": torch.randn(B, N_VIEWS + 1, 14, generator=g),
        "gmap_img_embeds": torch.randn(B, n_gmap, D_MODEL, generator=g),
        "gmap_pos_fts": torch.randn(B, n_gmap, 7, generator=g),
        "hist_vis": torch.randn(B, n_hist, D_MODEL, generator=g),
    }
    meta = {
        "view_lens": torch.full((B,), N_VIEWS, dtype=torch.long),
        "gmap_step_ids": step_ids, "gmap_masks": torch.ones(B, n_gmap, dtype=torch.bool), "gmap_visited_masks": visited,
        "gmap_vpids": gmap_vpids, "vp_cand_vpids": [[None] + [f"c{j}" for j in range(n_c)] for _ in range(B)],
        "prompts": prompts, "targets": torch.from_numpy(rng.randint(0, n_cand, size=B)).long(),
        "lens": lens, "n_hist": n_hist,
    }
    # candidate slot -> gmap column of the target (slot 0 = stop = column 0; candidate j = column 1+n_hist+j)
    meta["target_cols"] = torch.where(meta["targets"] == 0, torch.zeros_like(meta["targets"]), meta["targets"] + n_hist)
    return host, meta


def build_model(dev, seed=0):
    from navillm_b200.nav_model import NavModel
    from navillm_b200.tokenizer import SyntheticTokenizer
    args = types.SimpleNamespace(precision="amp_bf16", pretrained_model_name_or_path="vicuna-7b-synthetic", image_feat_size=IMG_FEAT,
                                 angle_feat_size=4, obj_feat_size=768, enable_og=True, fuse_obj=False, feat_dropout=0.4,
                                 resume_from_checkpoint=None, from_scratch=True, device=str(dev), seed=seed)
    mc = types.SimpleNamespace(num_pano_layers=2, tokenizer=SyntheticTokenizer(base_vocab=VOCAB))
    torch.manual_seed(seed)
    model = NavModel(args, None, mc)
    model.train()
    return model


def nav_step(model, dev_in, meta, dev, text=None, outputs=None):
    """One batch of navigation steps through the public API; returns the loss tensor (on device).  With `outputs` (a dict)
    the navigation logits are kept there as well."""
    B = dev_in["view_img_fts"].shape[0]
    n_hist = dev_in["hist_vis"].shape[1]
    pano = model("panorama", {"view_img_fts": dev_in["view_img_fts"], "view_lens": meta["view_lens"], "loc_fts": dev_in["loc_fts"],
                              "nav_types": dev_in["nav_types"]})
    pe = pano["pano_embeds"]
    batch = {"data_type": ["r2r"] * B,
             "vp_img_embeds": torch.cat([torch.zeros_like(pe[:, :1]), pe], 1),                    # mp3d_agent.py:268-270
             "pano_masks": torch.ones((B, N_VIEWS + 1), dtype=torch.bool),                         # host mask (all views valid)
             "vp_pos_fts": dev_in["vp_pos_fts"], "vp_cand_vpids": meta["vp_cand_vpids"],
             "gmap_img_embeds": dev_in["gmap_img_embeds"], "gmap_step_ids": meta["gmap_step_ids"],
             "gmap_pos_fts": dev_in["gmap_pos_fts"], "gmap_masks": meta["gmap_masks"], "gmap_pair_dists": None,
             "gmap_visited_masks": meta["gmap_visited_masks"], "gmap_vpids": meta["gmap_vpids"],
             "instruction": [""] * B, "history": [["h"] * n_hist] * B,
             "hist_vis": [list(dev_in["hist_vis"][b].unbind(0)) for b in range(B)], "prompts": meta["prompts"]}
    if text is not None:
        batch["text_input"] = text
    out = model("navigation", batch)
    loss = torch.nn.functional.cross_entropy(out["fuse_logits"].float(), dev_in["target_cols"], reduction="sum",
                                             ignore_index=-100) / B                               # mp3d_agent.py:750
    if outputs is not None:
        outputs["fuse_logits"] = out["fuse_logits"]
    return loss


class ClockSampler:
    """nvidia-smi clocks / throttle reasons DURING the timed region (profiling recipe)."""

    def __init__(self, index: int):
        self.rows, self.proc, self.index = [], None, index

    def __enter__(self):
        q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-lms", "200",
                                          "-i", str(self.index)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None
        return self

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([x.strip() for x in line.split(",")])

    def __exit__(self, *a):
        if self.proc is not None:
            self.proc.terminate()
            try:
                self.proc.wait(timeout=2)
            except Exception:
                self.proc.kill()

    def summary(self):
        sm, mx, reasons = [], 0.0, set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            try:
                sm.append(float(r[0])); mx = max(mx, float(r[1]))
                for n, v in zip(names, r[3:7]):
                    if v.lower().startswith("active"):
                        reasons.add(n)
            except Exception:
                continue
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": mx or None, "reasons": sorted(reasons),
                "samples": len(sm)}


# ---------------------------------------------------------------------------------------------------------
# CPU arm: oracle port of the reference on host cores (bounded sample)
# ---------------------------------------------------------------------------------------------------------
CPU_BUDGET_S = 60.0          # hard wall-clock cap of one cpu_reference_sample() call (both dtypes together)
CPU_MAX_TIMED = 3            # timed passes per dtype, whatever --steps says


def pick_cpu_threads() -> int:
    from oracle.hostcpu import pick_cpu_threads as _p
    return _p(D_MODEL)


def _oracle_layers(n_layers: int, dtype):
    g = torch.Generator().manual_seed(0)
    sd = {}
    for l in range(n_layers):
        p = f"lang_model.model.layers.{l}"
        for nm, shp in (("self_attn.q_proj", (D_MODEL, D_MODEL)), ("self_attn.k_proj", (D_MODEL, D_MODEL)),
                        ("self_attn.v_proj", (D_MODEL, D_MODEL)), ("self_attn.o_proj", (D_MODEL, D_MODEL)),
                        ("mlp.gate_proj", (D_FF, D_MODEL)), ("mlp.up_proj", (D_FF, D_MODEL)), ("mlp.down_proj", (D_MODEL, D_FF))):
            sd[f"{p}.{nm}.weight"] = torch.empty(shp, dtype=dtype).normal_(0, 0.02, generator=g).requires_grad_(True)
        sd[f"{p}.input_layernorm.weight"] = torch.ones(D_MODEL, dtype=dtype, requires_grad=True)
        sd[f"{p}.post_attention_layernorm.weight"] = torch.ones(D_MODEL, dtype=dtype, requires_grad=True)
    sd["lang_model.model.norm.weight"] = torch.ones(D_MODEL, dtype=dtype, requires_grad=True)
    return sd, g


def _cpu_train_sample(n_layers: int, seq: int, dtype, deadline: float):
    """fwd+bwd of `n_layers` full-width layers on one prompt of `seq` tokens; returns seconds per pass (median of the timed
    passes; the warm pass itself if the deadline allows nothing more)."""
    from oracle import navillm_oracle as O
    cfg = O.OracleConfig(hidden=D_MODEL, n_layers=n_layers, n_heads=N_HEADS, inter=D_FF, vocab=64,
                         precision="amp_bf16" if dtype == torch.bfloat16 else "fp32")
    sd, g = _oracle_layers(n_layers, dtype)
    emb = torch.randn(1, seq, D_MODEL, generator=g).to(dtype).requires_grad_(True)
    mask = torch.ones(1, seq, dtype=torch.long)
    times = []
    for i in range(1 + CPU_MAX_TIMED):                               # pass 0 = warm
        t0 = time.perf_counter()
        h = O.llama_model(sd, cfg, emb, mask)
        h[:, -1].float().sum().backward()
        dt = time.perf_counter() - t0
        times.append(dt)
        if time.time() + dt > deadline:                              # the next pass would cross the cap
            break
    timed = times[1:] or times
    return statistics.median(timed), len(times) - 1


def _cpu_generate_sample(n_layers: int, B: int, s0: int, dtype, deadline: float):
    """prefill of `n_layers` layers on [B, s0] + decode steps with a KV cache; returns (prefill s, s per decode step)."""
    from oracle import navillm_oracle as O
    cfg = O.OracleConfig(hidden=D_MODEL, n_layers=n_layers, n_heads=N_HEADS, inter=D_FF, vocab=64,
                         precision="amp_bf16" if dtype == torch.bfloat16 else "fp32")
    sd, g = _oracle_layers(n_layers, dtype)
    with torch.no_grad():
        emb = torch.randn(B, s0, D_MODEL, generator=g).to(dtype)
        mask = torch.ones(B, s0, dtype=torch.long)
        pos = torch.arange(s0).unsqueeze(0).expand(B, s0)
        best_pre, steps = None, []
        for i in range(2):
            past = [None] * n_layers
            t0 = time.perf_counter()
            O.llama_model(sd, cfg, emb, mask, pos, past)
            dt = time.perf_counter() - t0
            best_pre = dt if best_pre is None else min(best_pre, dt)
            if time.time() + dt > deadline:
                break
        x1 = torch.randn(B, 1, D_MODEL, generator=g).to(dtype)
        for i in range(1 + CPU_MAX_TIMED):
            mask = torch.cat([mask, mask.new_ones(B, 1)], 1)
            t0 = time.perf_counter()
            O.llama_model(sd, cfg, x1, mask, torch.full((B, 1), mask.shape[1] - 1), past)
            steps.append(time.perf_counter() - t0)
            if time.time() > deadline:
                break
    return best_pre, statistics.median(steps[1:] or steps)


def _cpu_c1_full(dtype, deadline):
    """C1 as BASELINE.json states it: the whole step (panorama + navigation forward) through the oracle port with ALL 32
    decoder layers on the host cores, batch 1.  The 32 layers alias one set of full-width matrices (values do not matter for
    a timing; 13.5 GB of distinct random weights would only add minutes of initialisation) - every layer still streams and
    multiplies its own 202 M parameters' worth of data per token."""
    from oracle import navillm_oracle as O
    from navillm_b200.tokenizer import SyntheticTokenizer
    tok = SyntheticTokenizer(base_vocab=VOCAB)
    prec = "amp_bf16" if dtype == torch.bfloat16 else "fp32"
    cfg1 = O.OracleConfig(hidden=D_MODEL, n_layers=1, n_heads=N_HEADS, inter=D_FF, vocab=len(tok), image_feat_size=IMG_FEAT, obj_feat_size=768,
                          cand_id=tok.special["<cand>"], hist_id=tok.special["<hist>"], obj_id=tok.special["<obj>"],
                          cls_ids=(tok.special["<cls_1>"], tok.special["<cls_2>"]), precision=prec)
    sd = O.init_state_dict(cfg1, seed=0)
    for k in list(sd):
        if k.startswith("lang_model.model.layers.0."):
            for l in range(1, N_LAYERS):
                sd[k.replace("layers.0.", f"layers.{l}.")] = sd[k]
    cfg = O.OracleConfig(**{**cfg1.__dict__, "n_layers": N_LAYERS})
    host, meta = make_workload(1234, **{k: v for k, v in WORKLOADS["c1"].items() if k not in ("name", "max_length")})
    times = []
    with torch.no_grad():
        for i in range(1 + CPU_MAX_TIMED):
            t0 = time.perf_counter()
            pano = O.forward_panorama(sd, cfg, host["view_img_fts"], meta["view_lens"], host["loc_fts"], host["nav_types"])
            pe = pano["pano_embeds"]
            nav = {"vp_img_embeds": torch.cat([torch.zeros_like(pe[:, :1]), pe], 1), "pano_masks": torch.ones((1, N_VIEWS + 1), dtype=torch.bool),
                   "vp_pos_fts": host["vp_pos_fts"], "vp_cand_vpids": meta["vp_cand_vpids"], "gmap_img_embeds": host["gmap_img_embeds"],
                   "gmap_step_ids": meta["gmap_step_ids"], "gmap_pos_fts": host["gmap_pos_fts"], "gmap_masks": meta["gmap_masks"],
                   "gmap_visited_masks": meta["gmap_visited_masks"], "gmap_vpids": meta["gmap_vpids"], "hist_vis": [[]], "prompts": meta["prompts"]}
            O.forward_navigation(sd, cfg, nav, tok)
            dt = time.perf_counter() - t0
            times.append(dt)
            if time.time() + dt > deadline:
                break
    timed_ = times[1:] or times
    return statistics.median(timed_), len(times) - 1


def cpu_reference_sample(workload: str, n_layers: int = 2, budget_s: float = CPU_BUDGET_S):
    """Times the oracle port in the reference's own precision ('amp_bf16' -> bf16 LM) AND in fp32 and reports the faster one:
    hosts without AMX / AVX512-BF16 run torch's bf16 CPU GEMMs far below their fp32 rate, and a user of the reference on
    such a CPU would pick fp32.  Bounded: <= 1 warm + 3 timed passes per dtype and `budget_s` of wall clock in total."""
    cores = pick_cpu_threads()
    wl = WORKLOADS[workload]
    t_start = time.time()
    res = {}
    for k, dtype in enumerate((torch.float32, torch.bfloat16)):
        deadline = t_start + budget_s * (0.5 if k == 0 else 1.0)
        if k == 1 and time.time() > t_start + 0.75 * budget_s:
            break                                                    # fp32 used the budget: report fp32 only
        name = "fp32" if dtype == torch.float32 else "bf16"
        if workload == "c1":
            t, n_timed = _cpu_c1_full(dtype, deadline)
            res[name] = {"value": 1.0 / t, "detail": f"{t:.2f} s per full 32-layer forward step (median of {max(n_timed, 1)})"}
        elif workload == "c3":
            pre, stp = _cpu_generate_sample(n_layers, wl["B"], wl["n_cand_tok"] + wl["n_text"], dtype, deadline)
            total = (pre + (wl["n_new"] - 1) * stp) * N_LAYERS / n_layers
            res[name] = {"value": wl["B"] * wl["n_new"] / total, "detail": f"prefill {pre:.2f} s + decode step {stp * 1e3:.0f} ms per {n_layers} layers"}
        else:
            seq = (wl["len_lo"] + wl["len_hi"]) // 2 if "len_lo" in wl else C4_MEAN_LEN
            t, n_timed = _cpu_train_sample(n_layers, seq, dtype, deadline)
            res[name] = {"value": 1.0 / (t * N_LAYERS / n_layers), "detail": f"{t:.2f} s per pass (median of {max(n_timed, 1)})"}
        log(f"cpu arm {name}: {res[name]['value']:.4g} ({res[name]['detail']})")
    best = max(res, key=lambda k: res[k]["value"])
    if workload == "c1":
        sample = (f"oracle port ({best}), the WHOLE C1 step on the host cores: panorama encoder + navigation forward with all {N_LAYERS} "
                  f"full-width Vicuna-7B layers, batch 1, S=192 (no scaling)")
    elif workload == "c3":
        sample = (f"oracle port ({best}), B={wl['B']}, S0={wl['n_cand_tok'] + wl['n_text']}, {n_layers} of {N_LAYERS} full-width Vicuna-7B "
                  f"layers: prefill + KV-cache decode steps timed, scaled x{N_LAYERS}/{n_layers} to {wl['n_new']} new tokens")
    else:
        sample = (f"oracle port ({best}), B=1, seq={(wl['len_lo'] + wl['len_hi']) // 2 if 'len_lo' in wl else C4_MEAN_LEN} (workload mean length), {n_layers} of {N_LAYERS} "
                  f"full-width Vicuna-7B layers fwd+bwd timed, scaled x{N_LAYERS}/{n_layers}")
    sample += " [" + ", ".join(f"{k}: {v['value']:.4g}/s, {v['detail']}" for k, v in res.items()) + "; faster one reported]"
    return {"value": res[best]["value"], "cores": cores, "sample": sample, "wall_s": time.time() - t_start}


def metric_of(workload: str):
    if workload == "c3":
        return ("generated_tokens_per_sec", "tokens/s")
    if workload == "c4":
        return ("mixed_samples_per_sec", "samples/s")
    return ("nav_steps_per_sec", "nav-steps/s")


def run_reference_arm(a, rank, world):
    if rank != 0:
        return
    log(f"reference arm (CPU oracle port), workload {a.workload}")
    r = cpu_reference_sample(a.workload, a.cpu_layers)
    v = r["value"]
    metric, unit = metric_of(a.workload)
    per_step = WORKLOADS[a.workload]["B"] * (WORKLOADS[a.workload].get("n_new", 1))   # units of the metric per bench step
    line = {"impl": "reference", "metric": metric, "value": v, "unit": unit, "n_gpus": a.gpus, "steps": a.steps,
            "warmup": a.warmup, "ms_per_step": 1000.0 * per_step / v, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "bf16", "data": "synthetic", "config": {"workload": WORKLOADS[a.workload]["name"]},
            "cpu_baseline": {"value": v, "unit": unit, "cores": r["cores"], "kind": "port", "sample": r["sample"]},
            "e2e": {"value": v, "unit": unit, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "gpu_launches": 0}
    print(json.dumps(line), flush=True)


# ---------------------------------------------------------------------------------------------------------
def timed(fn, k, world, dev):
    import torch.distributed as dist
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    st.record()
    for _ in range(k):
        fn()
    en.record()
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    ms = st.elapsed_time(en)
    if world > 1:
        t = torch.tensor([ms], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms = float(t)
    return ms


def run_train(a, rank, local_rank, world, dev):
    """c2 / c5: panorama + navigation forward, action CE, backward (+ gradient exchange for N > 1)."""
    import torch.distributed as dist
    from navillm_b200 import _lib, ops
    wl = WORKLOADS[a.workload]
    B = wl["B"]
    if a.layers != N_LAYERS:
        import navillm_b200.nav_model as nm
        nm.VICUNA_7B["num_hidden_layers"] = a.layers
    log(f"building the model ({a.layers} layers) on {dev}")
    core_model = build_model(dev, seed=0)
    core_model._ensure()
    model = core_model
    do_sync = world > 1 and a.grad_sync != "none"
    if world > 1:
        from navillm_b200.parallel import DistributedDataParallel as DDP
        core_model.grad_sync.overlap = a.grad_sync == "overlap"
        model = DDP(core_model, device_ids=[local_rank], find_unused_parameters=True)      # tools/optims.py:54
    host, meta = make_workload(1234 + rank, **wl)
    pinned = {k: v.pin_memory() for k, v in host.items()}
    tgt_pinned = meta["target_cols"].pin_memory()

    def upload():
        d = {k: v.to(dev, non_blocking=True) for k, v in pinned.items()}
        d["target_cols"] = tgt_pinned.to(dev, non_blocking=True)
        return d

    h2d_bytes = sum(v.numel() * v.element_size() for v in pinned.values()) + tgt_pinned.numel() * 8
    resident = upload()

    def tokenize():
        # the reference tokenises with max_length=1024 (models/modified_lm.py:80); C5's S = 2048 is BASELINE's synthetic
        # long-history size, so its prompts are tokenised without that truncation and handed over as `text_input`
        if wl["max_length"] == 1024:
            return None
        return core_model.lang_model.tokenizer(meta["prompts"], max_length=wl["max_length"], padding=True, truncation=True,
                                               return_tensors="pt", add_special_tokens=True, return_token_type_ids=True)

    text = tokenize() or core_model.lang_model.tokenize(meta["prompts"])
    tokens_real = int(text["attention_mask"].sum())
    import contextlib
    sync_ctx = (lambda: contextlib.nullcontext()) if (do_sync or world == 1) else model.no_sync

    fwd_only = a.workload == "c1"                          # the plumbing config: one forward step, no gradient
    if fwd_only:
        core_model.eval()

    last = {}                                              # outputs of the latest resident step (--dump-outputs)

    def step_resident():
        if fwd_only:
            with torch.no_grad():
                last["loss"] = nav_step(model, resident, meta, dev, text=text, outputs=last)
                return last["loss"]
        core_model.zero_grad(lazy=True)
        with sync_ctx():
            loss = nav_step(model, resident, meta, dev, text=text, outputs=last)
            loss.backward()                                # N > 1: the flat-gradient exchange fires from this backward
        last["loss"] = loss
        return loss

    def step_e2e():
        if fwd_only:
            with torch.no_grad():
                return float(nav_step(model, upload(), meta, dev, text=tokenize()))
        core_model.zero_grad(lazy=True)
        d = upload()
        with sync_ctx():
            loss = nav_step(model, d, meta, dev, text=tokenize())   # tokenises the prompt strings on the host, like the reference
            loss.backward()
        return float(loss.detach())                   # D2H read of the step's result

    log(f"warm-up: {a.warmup} steps ({tokens_real} real tokens per step)")
    for i in range(a.warmup):
        step_resident()
        if i == 0:
            torch.cuda.synchronize()
            log("first step done")
    torch.cuda.synchronize()
    launches0 = _lib.launch_count
    ops.gemm_timer = []
    log(f"timed region: {a.steps} steps")
    with ClockSampler(local_rank) as clk:
        ms = timed(step_resident, a.steps, world, dev)
    timer, ops.gemm_timer = ops.gemm_timer, None
    launches = (_lib.launch_count - launches0) // max(a.steps, 1)
    gemm_ms = sum(t[0].elapsed_time(t[1]) for t in timer)
    gemm_flops = sum(t[2] for t in timer)
    gemm_bytes = sum(t[3] for t in timer)
    n_gemm = len(timer)
    log(f"timed region done: {ms / a.steps:.1f} ms/step")
    if a.dump_outputs and rank == 0:
        dump_outputs(a.dump_outputs, {"loss": last["loss"].double(), "fuse_logits": last["fuse_logits"]},
                     None if fwd_only else core_model)

    if a.profile:
        if rank == 0:
            print(json.dumps({"profile_run": True, "ms_per_step": ms / a.steps, "launches": int(launches)}))
        return
    log("e2e region (host buffers, H2D + tokenisation + D2H inside)")
    step_e2e()                                       # warm the e2e path (pinned staging, tokenizer caches)
    ms_e2e = timed(step_e2e, a.steps, world, dev)
    log(f"e2e done: {ms_e2e / a.steps:.1f} ms/step")

    if rank == 0:
        pk = peaks()
        value = world * B * a.steps / (ms / 1e3)
        e2e = world * B * a.steps / (ms_e2e / 1e3)
        achieved = gemm_flops / (gemm_ms * 1e-3) / 1e12 if gemm_ms > 0 else None
        # algorithmic FLOPs of the whole step on REAL (non-pad) tokens (SURVEY.md §8d): 3 x (12.952 GF/token + attention)
        lens = np.asarray(text["attention_mask"].sum(1), dtype=np.float64)
        algo_step = (1.0 if fwd_only else 3.0) * (float((lens * 12.952e9 + 0.262144e6 * lens * lens).sum()) + 2.229e9 * B)
        st = core_model.grad_sync.stats
        line = {
            "metric": "nav_steps_per_sec", "value": value, "unit": "nav-steps/s", "n_gpus": world, "steps": a.steps, "warmup": a.warmup,
            "ms_per_step": ms / a.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16",
            "data": "synthetic",
            "config": {"workload": wl["name"], "layers": a.layers, "real_tokens_per_step": tokens_real,
                       "l2": "inputs_exceed_l2 (13.5 GB of weights streamed per pass)",
                       "grad_exchange": ({"overlap": "every step, fired from the backward by navillm_b200.parallel.DistributedDataParallel; LM layer slices overlapped with the backward", "end": "every step, at the end of the backward (debug)", "none": "DISABLED (debug, invalid)"}[a.grad_sync]
                                         + ("; transport: own in-switch all-reduce over NVLS multicast (multimem.ld_reduce / multimem.st, csrc/nvls_allreduce.cu) on a side stream"
                                            if getattr(model, "nvls", False) else "; transport: NCCL all-reduce")
                                         + f"; {st['collectives']} collectives in {st['exchanges']} exchanges so far") if world > 1 else "n/a",
                       "zero_grad": "lazy (first wgrad of a step overwrites: beta=0)", "optimizer_step": "outside the boundary (train.py:86-89), not timed"},
            "e2e": {"value": e2e, "unit": "nav-steps/s", "h2d_bytes_per_step": int(h2d_bytes), "d2h_bytes_per_step": 4,
                    "ms_per_step": ms_e2e / a.steps},
            "gpu_launches": int(launches), "gpu": gpu_info(local_rank),
            "roofline": {"bound": "tensor", "kernel": "gemm_bf16_wgmma (128 x 256 and 128 x 128 tiles)", "achieved": achieved, "peak": pk["bf16_tflops"], "unit": "TFLOP/s",
                         "frac": (achieved / pk["bf16_tflops"]) if achieved else None, "peak_src": pk["src"],
                         "launches_per_step": n_gemm // max(a.steps, 1), "share_of_step": gemm_ms / ms,
                         "traffic": None, "traffic_unit": "bytes/launch (DRAM read+write)", "traffic_src": "not measured",
                         "algorithmic_bytes_per_launch_mean": gemm_bytes / max(n_gemm, 1),
                         "step_algorithmic_tflop": algo_step / 1e12,
                         "step_frac_of_peak": algo_step / 1e12 / (ms / a.steps / 1e3) / pk["bf16_tflops"]},
            "clocks": clk.summary(),
        }
        if not a.no_cpu_baseline and world == 1:
            log("cpu_baseline (bounded sample of the oracle port on the host cores)")
            r = cpu_reference_sample(a.workload, a.cpu_layers)
            line["cpu_baseline"] = {"value": r["value"], "unit": "nav-steps/s", "cores": r["cores"], "kind": "port", "sample": r["sample"]}
        if a.layers != N_LAYERS:
            line["INVALID"] = f"debug run with {a.layers} layers"
        if world > 1 and a.grad_sync == "none":
            line["INVALID"] = "debug run without the gradient exchange"
        print(json.dumps(line), flush=True)
        log("done")


def run_mixed(a, rank, local_rank, world, dev):
    """c4: four micro-batches of different task shapes per step, accumulated under no_sync(), one exchange per step."""
    import contextlib
    import torch.distributed as dist
    from navillm_b200 import _lib
    wl = WORKLOADS["c4"]
    if a.layers != N_LAYERS:
        import navillm_b200.nav_model as nm
        nm.VICUNA_7B["num_hidden_layers"] = a.layers
    log(f"building the model ({a.layers} layers) on {dev}")
    core_model = build_model(dev, seed=0)
    core_model._ensure()
    model = core_model
    do_sync = world > 1 and a.grad_sync != "none"
    if world > 1:
        from navillm_b200.parallel import DistributedDataParallel as DDP
        core_model.grad_sync.overlap = a.grad_sync == "overlap"
        model = DDP(core_model, device_ids=[local_rank], find_unused_parameters=True)
    MB = 2
    shapes = [("r2r", dict(B=MB, n_hist=8, n_gmap=24, n_cand=16, len_lo=256, len_hi=512)),
              ("cvdn", dict(B=MB, n_hist=20, n_gmap=36, n_cand=16, len_lo=512, len_hi=1024)),
              ("soon", dict(B=MB, n_hist=10, n_gmap=26, n_cand=16, len_lo=384, len_hi=768))]
    navs = []
    for k, (name, kw) in enumerate(shapes):
        host, meta = make_workload(1234 + 10 * rank + k, **kw)
        navs.append((name, {k2: v.pin_memory() for k2, v in host.items()}, meta, meta["target_cols"].pin_memory()))
    g = torch.Generator().manual_seed(99 + rank)
    N_OBJ = 40
    og_host = {"obj_img_fts": torch.randn(MB, N_OBJ, 768, generator=g).pin_memory(), "obj_loc_fts": torch.randn(MB, N_OBJ, 7, generator=g).pin_memory(),
               "targets": torch.randint(0, N_OBJ, (MB,), generator=g).pin_memory()}
    rng = np.random.RandomState(77 + rank)
    qa_host = {"features": [torch.randn(N_VIEWS, IMG_FEAT, generator=g).pin_memory() for _ in range(MB)]}
    qa_prompts = ["Scene " + " ".join(["<cand>"] * N_VIEWS) + " Question " + " ".join(f"w{i}" for i in rng.randint(0, 5000, size=290)) + " Answer"
                  for _ in range(MB)]
    qa_answers = [[" ".join(f"w{i}" for i in rng.randint(0, 5000, size=15))] for _ in range(MB)]
    h2d_bytes = sum(v.numel() * v.element_size() for _, p, _, t in navs for v in list(p.values()) + [t]) \
        + sum(v.numel() * v.element_size() for v in og_host.values()) + sum(f.numel() * 4 for f in qa_host["features"])

    def micro_batches(up):
        """yields callables, one per micro-batch, each returning its loss"""
        for name, pinned, meta, tgt in navs:
            def nav(pinned=pinned, meta=meta, tgt=tgt, name=name):
                d = {k: up(v) for k, v in pinned.items()}
                d["target_cols"] = up(tgt)
                if name != "soon":
                    return nav_step(model, d, meta, dev)
                # SOON: the panorama call also projects the objects; the step ends with the object-grounding sub-task
                B = MB
                pano = model("panorama", {"view_img_fts": d["view_img_fts"], "view_lens": meta["view_lens"], "loc_fts": d["loc_fts"],
                                          "nav_types": d["nav_types"], "obj_img_fts": up(og_host["obj_img_fts"]),
                                          "obj_lens": torch.full((B,), N_OBJ, dtype=torch.long), "obj_loc_fts": up(og_host["obj_loc_fts"])})
                n_hist = d["hist_vis"].shape[1]
                og = model("object_grounding", {"data_type": ["soon"] * B, "obj_embeds": pano["obj_embeds"], "obj_masks": pano["obj_masks"],
                                                "obj_loc_fts": up(og_host["obj_loc_fts"]),
                                                "hist_vis": [list(d["hist_vis"][b].unbind(0)) for b in range(B)],
                                                "prompts": ["Find " + " ".join(["<hist>"] * n_hist) + " Objects " + " ".join(["<cand>"] * N_OBJ) + " <cls_1>"
                                                            for _ in range(B)]})
                og_loss = torch.nn.functional.cross_entropy(og["obj_logits"].float(), up(og_host["targets"]), reduction="sum") / B
                return nav_step(model, d, meta, dev) + og_loss
            yield nav

        def qa():
            out = model("3dqa", {"question": [""] * MB, "prompts": qa_prompts, "answers": qa_answers,
                                 "features": [up(f) for f in qa_host["features"]]}, training=True)
            return out.loss.float()
        yield qa

    losses = []                                         # micro-batch losses of the latest step (--dump-outputs)

    def step(up, read):
        core_model.zero_grad(lazy=True)
        mbs = list(micro_batches(up))
        total = 0.0
        losses.clear()
        for i, mb in enumerate(mbs):
            last = i == len(mbs) - 1
            ctx = contextlib.nullcontext() if ((last and do_sync) or world == 1) else model.no_sync()
            with ctx:                                   # tasks/agents/mp3d_agent.py:661-667: only the last backward exchanges
                loss = mb()
                loss.backward()
            losses.append(loss.detach())
            if read:
                total += float(loss.detach())
        return total

    resident_cache = {}

    def up_resident(v):
        k = id(v)
        if k not in resident_cache:
            resident_cache[k] = v.to(dev)
        return resident_cache[k]

    up_h2d = lambda v: v.to(dev, non_blocking=True)
    log(f"warm-up: {a.warmup} steps")
    for _ in range(a.warmup):
        step(up_resident, False)
    torch.cuda.synchronize()
    launches0 = _lib.launch_count
    log(f"timed region: {a.steps} steps")
    with ClockSampler(local_rank) as clk:
        ms = timed(lambda: step(up_resident, False), a.steps, world, dev)
    launches = (_lib.launch_count - launches0) // max(a.steps, 1)
    log(f"timed region done: {ms / a.steps:.1f} ms/step")
    if a.dump_outputs and rank == 0:
        dump_outputs(a.dump_outputs, {"micro_batch_losses": torch.stack([x.double() for x in losses])}, core_model)
    if a.profile:
        if rank == 0:
            print(json.dumps({"profile_run": True, "ms_per_step": ms / a.steps, "launches": int(launches)}))
        return
    step(up_h2d, True)
    ms_e2e = timed(lambda: step(up_h2d, True), a.steps, world, dev)
    log(f"e2e done: {ms_e2e / a.steps:.1f} ms/step")
    if rank == 0:
        pk = peaks()
        B = wl["B"]
        lens = np.concatenate([m["lens"] for _, _, m, _ in navs] + [np.asarray([1 + N_VIEWS + 290 + 4 + 16] * MB)]).astype(np.float64)
        lens = np.concatenate([lens, np.asarray([1 + 10 + N_OBJ + 3] * MB, dtype=np.float64)])      # + the object-grounding prompts
        algo_step = 3.0 * float((lens * 12.952e9 + 0.262144e6 * lens * lens).sum()) + 3.0 * 2.229e9 * (len(navs) * MB + MB)
        st = core_model.grad_sync.stats
        line = {"metric": "mixed_samples_per_sec", "value": world * B * a.steps / (ms / 1e3), "unit": "samples/s", "n_gpus": world, "steps": a.steps,
                "warmup": a.warmup, "ms_per_step": ms / a.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16",
                "data": "synthetic",
                "config": {"workload": wl["name"], "layers": a.layers, "l2": "inputs_exceed_l2 (13.5 GB of weights streamed per pass)",
                           "micro_batches": "r2r | cvdn | soon (+object grounding) | scanqa; no_sync() around all but the last backward",
                           "grad_exchange": (f"one exchange per step; {st['collectives']} collectives in {st['exchanges']} exchanges so far; "
                                             + ("NVLS in-switch all-reduce" if getattr(model, "nvls", False) else "NCCL")) if world > 1 else "n/a"},
                "e2e": {"value": world * B * a.steps / (ms_e2e / 1e3), "unit": "samples/s", "h2d_bytes_per_step": int(h2d_bytes),
                        "d2h_bytes_per_step": 4 * 4, "ms_per_step": ms_e2e / a.steps},
                "gpu_launches": int(launches), "gpu": gpu_info(local_rank),
                "roofline": {"bound": "tensor", "kernel": "whole step (algorithmic FLOPs of the four micro-batches on real tokens)",
                             "achieved": algo_step / 1e12 / (ms / a.steps / 1e3), "peak": pk["bf16_tflops"], "unit": "TFLOP/s",
                             "frac": algo_step / 1e12 / (ms / a.steps / 1e3) / pk["bf16_tflops"], "peak_src": pk["src"],
                             "step_algorithmic_tflop": algo_step / 1e12, "traffic": None},
                "clocks": clk.summary()}
        if not a.no_cpu_baseline and world == 1:
            r = cpu_reference_sample("c4", a.cpu_layers)
            line["cpu_baseline"] = {"value": r["value"], "unit": "samples/s", "cores": r["cores"], "kind": "port", "sample": r["sample"]}
        if a.layers != N_LAYERS:
            line["INVALID"] = f"debug run with {a.layers} layers"
        print(json.dumps(line), flush=True)
        log("done")


def run_generate(a, rank, local_rank, world, dev):
    """c3: ScanQA-shaped greedy generation through model('3dqa', training=False) (e2e) and lang_model.generate (resident)."""
    import torch.distributed as dist
    from navillm_b200 import _lib
    wl = WORKLOADS["c3"]
    B, NV, NT, NEW = wl["B"], wl["n_cand_tok"], wl["n_text"], wl["n_new"]
    if a.layers != N_LAYERS:
        import navillm_b200.nav_model as nm
        nm.VICUNA_7B["num_hidden_layers"] = a.layers
    log(f"building the model ({a.layers} layers) on {dev}")
    model = build_model(dev, seed=0).eval()
    model._ensure()
    lm = model.lang_model
    rng = np.random.RandomState(1234 + rank)
    words = [f"w{i}" for i in range(5000)]
    n_words = NT - 5                                                 # bos + 3 section words + trailing word
    prompts = ["Scene " + " ".join(["<cand>"] * NV) + " Question " + " ".join(words[i] for i in rng.randint(0, 5000, size=n_words))
               + " Answer" for _ in range(B)]
    g = torch.Generator().manual_seed(1234 + rank)
    feats_host = [torch.randn(NV, IMG_FEAT, generator=g).pin_memory() for _ in range(B)]
    batch_host = {"question": [""] * B, "prompts": prompts, "features": feats_host}
    text = lm.tokenize(prompts)
    S0 = int(text["attention_mask"].sum(1).max())
    with torch.no_grad():
        view = torch.stack([f.to(dev) for f in feats_host], 0)
        pano = model.img_embeddings.forward_panorama_per_step(view_img_fts=view, view_lens=torch.full((B,), NV, device=dev))
        cand = model._masked_rows_plus_const(pano["pano_embeds"].reshape(B * NV, -1), np.ones((B, NV), dtype=bool)).detach()
    stats = {}

    def step_resident(st=None):
        return lm.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand, max_new_tokens=NEW,
                           stop_on_eos=False, use_cuda_graph=True, stats=st)

    def step_e2e():
        b = dict(batch_host)
        b["features"] = [f.to(dev, non_blocking=True) for f in feats_host]
        out = model("3dqa", b, training=False, max_new_tokens=NEW, do_sample=False, stop_on_eos=False)
        return out["generated_sentences"]                          # decoded strings on the host = the D2H read

    log(f"warm-up: {a.warmup} generations (S0={S0}, {NEW} new tokens)")
    for _ in range(a.warmup):
        step_resident()
    torch.cuda.synchronize()
    launches0 = _lib.launch_count
    log(f"timed region: {a.steps} generations")
    per, last = [], {}
    with ClockSampler(local_rank) as clk:
        def one():
            s = {}
            last["out"] = step_resident(s)
            per.append(s)
        ms = timed(one, a.steps, world, dev)
    launches = (_lib.launch_count - launches0) // max(a.steps, 1)
    log(f"timed region done: {ms / a.steps:.1f} ms per generation")
    if a.dump_outputs and rank == 0:
        dump_outputs(a.dump_outputs, {"token_ids": last["out"].double()})      # [B, S0 + new] ids
    if a.profile:
        if rank == 0:
            print(json.dumps({"profile_run": True, "ms_per_step": ms / a.steps, "launches": int(launches)}))
        return
    step_e2e()
    ms_e2e = timed(step_e2e, a.steps, world, dev)
    log(f"e2e done: {ms_e2e / a.steps:.1f} ms per generation")
    if rank == 0:
        pk = peaks()
        value = world * B * NEW * a.steps / (ms / 1e3)
        e2e = world * B * NEW * a.steps / (ms_e2e / 1e3)
        dec = [s["decode_ms"] / s["decode_steps"] for s in per if s.get("decode_ms")]
        ms_tok = statistics.median(dec) if dec else None
        prefill = statistics.median(s["prefill_ms"] for s in per)
        # algorithmic bytes of one decode step (SURVEY.md §8d): all weights once + KV read (mean context of the replayed
        # steps) + KV write;  524 288 B per token and sequence
        mean_ctx = S0 + 1 + (NEW - 1) / 2.0
        bytes_tok = 2 * (6.476e9 * a.layers / N_LAYERS + 0.131e9) + B * mean_ctx * 524288 * a.layers / N_LAYERS + B * 524288 * a.layers / N_LAYERS
        achieved = bytes_tok / (ms_tok * 1e-3) / 1e9 if ms_tok else None
        h2d = sum(f.numel() * 4 for f in feats_host)
        line = {
            "metric": "generated_tokens_per_sec", "value": value, "unit": "tokens/s", "n_gpus": world, "steps": a.steps, "warmup": a.warmup,
            "ms_per_step": ms / a.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
            "config": {"workload": wl["name"], "layers": a.layers, "prompt_tokens": S0, "new_tokens": NEW,
                       "l2": "inputs_exceed_l2 (13.2 GB of weights streamed per token)", "prefill_ms": prefill, "ms_per_token": ms_tok,
                       "decode": "CUDA-graph replay per token (swap-AB skinny GEMMs, fused RoPE+KV append, split-KV attention)",
                       "step_includes": "prefill + first token + 127 CUDA-graph replays (graph captured once per shape, in the warm-up)"},
            "e2e": {"value": e2e, "unit": "tokens/s", "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": int(B * (S0 + NEW) * 8),
                    "ms_per_step": ms_e2e / a.steps, "path": "model('3dqa', batch, training=False): panorama encoder + tokenisation + generate + batch_decode"},
            "gpu_launches": int(launches), "gpu": gpu_info(local_rank),
            "roofline": {"bound": "hbm", "kernel": "decode step (CUDA graph: gemm_skinny_wgmma x4/layer + rmsnorm/rope-kv/decode_attn)", "achieved": achieved,
                         "peak": pk["hbm_gbs"], "unit": "GB/s", "frac": (achieved / pk["hbm_gbs"]) if achieved else None, "peak_src": pk["src"],
                         "algorithmic_bytes_per_token_step": bytes_tok, "traffic": None,
                         "traffic_unit": "bytes per decode step (DRAM read+write)", "traffic_src": "not measured"},
            "clocks": clk.summary(),
        }
        if not a.no_cpu_baseline and world == 1:
            log("cpu_baseline (bounded sample of the oracle port on the host cores)")
            r = cpu_reference_sample("c3", a.cpu_layers)
            line["cpu_baseline"] = {"value": r["value"], "unit": "tokens/s", "cores": r["cores"], "kind": "port", "sample": r["sample"]}
        if a.layers != N_LAYERS:
            line["INVALID"] = f"debug run with {a.layers} layers"
        print(json.dumps(line), flush=True)
        log("done")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="nv", choices=["nv", "reference"])
    ap.add_argument("--workload", default="c2", choices=sorted(WORKLOADS))
    ap.add_argument("--cpu-layers", type=int, default=2)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--layers", type=int, default=N_LAYERS, help="debug only: fewer layers => number is INVALID")
    ap.add_argument("--grad-sync", default="overlap", choices=["overlap", "end", "none"],
                    help="debug only (N>1): 'end' = exchange at the end of the backward only, 'none' = no exchange => number is INVALID")
    ap.add_argument("--profile", action="store_true", help="for runs under ncu: no e2e / cpu arms, any warm-up count; the printed number is not a bench value")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last one computed as DIR/<name>.npy (see the module docstring)")
    a = ap.parse_args()

    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if a.impl == "reference":
        run_reference_arm(a, rank, world)
        return
    assert a.warmup >= 3 or a.layers != N_LAYERS or a.profile, "timing rule: at least 3 warm-up steps"

    import torch.distributed as dist
    log(f"start: workload {a.workload}, world {world}, steps {a.steps}, warmup {a.warmup}")
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)
        log("process group up")
    try:
        if a.workload == "c3":
            run_generate(a, rank, local_rank, world, dev)
        elif a.workload == "c4":
            run_mixed(a, rank, local_rank, world, dev)
        else:
            run_train(a, rank, local_rank, world, dev)
    finally:
        if world > 1:
            dist.destroy_process_group()


if __name__ == "__main__":
    main()
