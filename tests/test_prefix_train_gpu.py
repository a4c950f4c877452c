"""Training over a PrefixKVCache (PrefixKVCache(train=True)): the cache form of the attention backward
(nv_attn_bwd_kv), the suffix-only training step and the deferred prefix backward (``flush_grads``).

Tolerances, stated:
  * nv_attn_bwd_kv vs autograd of the fp32 masked attention: the kernel rounds P and dS to bf16 before the products and the
    gradients to bf16 (as nv_attn_bwd): 3e-2 of the gradient's max, the bound of tests/test_attn_gpu.py.  Accumulated rows:
    the same bound on (acc_after - acc_before), and rows the kernel must not touch are compared bit for bit.
  * Rollout gradients with the cache vs the from-scratch CUDA path: the cached path computes the same sums, but a row keeps
    the rotary offset of its first step and part (b) runs on recomputed prefix activations, so only bf16 rounding
    differs; each parameter gradient must lie within 5e-2 of its max|grad| (the gradient floor of the boundary rule of
    tests/test_fullwidth_parity_gpu.py), fuse_logits within 3e-2 of max|logit| (tests/test_prefix_reuse_gpu.py).
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_prefix_reuse_gpu import _build, _nav_batch

pytestmark = pytest.mark.gpu

HD = 128

CASES = [
    dict(q=[128, 70, 1, 300], kv=[128, 75, 130, 300], H=2),            # cached 0, 5, 129, 0
    dict(q=[40, 257, 200], kv=[1000, 600, 333], H=2),                  # long cached prefixes, misaligned diagonals
    dict(q=[5], kv=[5], H=2),
    dict(q=[256, 129], kv=[511, 129 + 384], H=2),
    dict(q=[200, 77], kv=[200 + 190, 77 + 300], H=32),                 # key blocks straddle the cached count
]


def _setup(cuda_dev, case):
    H, Smax = case["H"], 1024
    q_lens, kv_lens = case["q"], case["kv"]
    B, Tq = len(q_lens), sum(q_lens)
    g = torch.Generator().manual_seed(sum(q_lens) + 7 * sum(kv_lens) + H)
    q = torch.randn(Tq, H * HD, generator=g).to(cuda_dev, torch.bfloat16)
    kc = torch.zeros(B, Smax, H * HD, dtype=torch.bfloat16, device=cuda_dev)
    vc = torch.zeros_like(kc)
    for b in range(B):
        kc[b, :kv_lens[b]] = torch.randn(kv_lens[b], H * HD, generator=g).to(cuda_dev, torch.bfloat16)
        vc[b, :kv_lens[b]] = torch.randn(kv_lens[b], H * HD, generator=g).to(cuda_dev, torch.bfloat16)
    do = torch.randn(Tq, H * HD, generator=g).to(cuda_dev, torch.bfloat16)
    acc0 = torch.randn(B, Smax, 2 * H * HD, generator=g).to(cuda_dev)
    cu = torch.tensor([0] + list(np.cumsum(q_lens)), dtype=torch.int32, device=cuda_dev)
    kv_start = torch.arange(B, dtype=torch.int32, device=cuda_dev) * Smax
    kv_len = torch.tensor(kv_lens, dtype=torch.int32, device=cuda_dev)
    return H, q, kc, vc, do, acc0, cu, kv_start, kv_len


def _reference(q, kc, vc, do, q_lens, kv_lens, H):
    """fp32 autograd of the masked attention per sequence: (o, lse, dq, dk, dv) with dk / dv over the kv_len rows."""
    scale = HD ** -0.5
    out, t0 = [], 0
    for b, (nq, nk) in enumerate(zip(q_lens, kv_lens)):
        dkc = nk - nq
        mask = torch.arange(nk, device=q.device)[None, :] <= dkc + torch.arange(nq, device=q.device)[:, None]
        qq = q[t0:t0 + nq].float().view(nq, H, HD).transpose(0, 1).requires_grad_(True)
        kk = kc[b, :nk].float().view(nk, H, HD).transpose(0, 1).requires_grad_(True)
        vv = vc[b, :nk].float().view(nk, H, HD).transpose(0, 1).requires_grad_(True)
        s = (qq @ kk.transpose(1, 2)) * scale
        s = s.masked_fill(~mask, float("-inf"))
        lse = torch.logsumexp(s, -1)
        o = torch.softmax(s, -1) @ vv
        o.backward(do[t0:t0 + nq].float().view(nq, H, HD).transpose(0, 1))
        flat = lambda t: t.transpose(0, 1).reshape(t.shape[1], H * HD)
        out.append((flat(o.detach()), lse.detach(), flat(qq.grad), flat(kk.grad), flat(vv.grad)))
        t0 += nq
    return out


def _close(name, got, ref, frac=3e-2):
    err = (got.float() - ref).abs().max().item()
    assert err <= frac * ref.abs().max().item() + 1e-6, f"{name}: err {err} vs max {ref.abs().max().item()}"


@pytest.mark.parametrize("case", CASES)
def test_attn_bwd_kv_matches_autograd(cuda_dev, case):
    from navillm_b200 import ops
    from navillm_b200.llama import LlamaDims, rope_tables
    H, q, kc, vc, do, acc0, cu, kv_start, kv_len = _setup(cuda_dev, case)
    q_lens, kv_lens = case["q"], case["kv"]
    Tq, D = q.shape[0], H * HD
    lse = torch.empty(H, Tq, dtype=torch.float32, device=cuda_dev)
    o = ops.attn_fwd_kv(q, kc, vc, cu, q_lens, kv_start, kv_len, H, lse=lse)
    acc = acc0.clone()
    dqkv = ops.attn_bwd_kv(q, o, do, lse, kc, vc, acc, cu, q_lens, kv_start, kv_len, kv_lens, H)
    # determinism: a second run from the same accumulator is bit-identical
    acc2 = acc0.clone()
    dqkv2 = ops.attn_bwd_kv(q, o, do, lse, kc, vc, acc2, cu, q_lens, kv_start, kv_len, kv_lens, H)
    # the inverse rotary embedding in the epilogue: bit for bit the plain output rotated back (as nv_attn_bwd)
    pos = torch.randint(0, 1024, (Tq,), generator=torch.Generator().manual_seed(5)).to(cuda_dev, torch.int32)
    cos_t, sin_t = rope_tables(LlamaDims(hidden=D, n_heads=H, max_pos=1024), cuda_dev)
    acc3 = acc0.clone()
    roped = ops.attn_bwd_kv(q, o, do, lse, kc, vc, acc3, cu, q_lens, kv_start, kv_len, kv_lens, H, rope=(pos, cos_t, sin_t))
    torch.cuda.synchronize()
    assert torch.equal(dqkv, dqkv2) and torch.equal(acc, acc2)
    plain = dqkv.clone()
    ops.rope_(plain, pos, cos_t, sin_t, 2 * H, backward=True)
    assert torch.equal(roped, plain) and torch.equal(acc3, acc)

    ref = _reference(q, kc, vc, do, q_lens, kv_lens, H)
    t0 = 0
    for b, (nq, nk) in enumerate(zip(q_lens, kv_lens)):
        o_r, lse_r, dq_r, dk_r, dv_r = ref[b]
        c = nk - nq
        assert torch.allclose(lse[:, t0:t0 + nq], lse_r, rtol=1e-3, atol=2e-3), (lse[:, t0:t0 + nq] - lse_r).abs().max().item()
        _close(f"dq[{b}]", dqkv[t0:t0 + nq, :D], dq_r)
        # suffix rows: dK + acc, dV + acc (acc read, not written)
        _close(f"dk[{b}]", dqkv[t0:t0 + nq, D:2 * D], dk_r[c:] + acc0[b, c:nk, :D])
        _close(f"dv[{b}]", dqkv[t0:t0 + nq, 2 * D:], dv_r[c:] + acc0[b, c:nk, D:])
        # cached rows accumulate; every other row of the sequence's slot (suffix rows, rows past kv_len) is untouched
        if c:
            _close(f"acc dk[{b}]", acc[b, :c, :D] - acc0[b, :c, :D], dk_r[:c])
            _close(f"acc dv[{b}]", acc[b, :c, D:] - acc0[b, :c, D:], dv_r[:c])
        assert torch.equal(acc[b, c:], acc0[b, c:]), b
        t0 += nq


def test_attn_bwd_kv_rejects_bad_accumulator(cuda_dev):
    from navillm_b200 import ops
    case = CASES[0]
    H, q, kc, vc, do, acc0, cu, kv_start, kv_len = _setup(cuda_dev, case)
    lse = torch.empty(H, q.shape[0], dtype=torch.float32, device=cuda_dev)
    o = ops.attn_fwd_kv(q, kc, vc, cu, case["q"], kv_start, kv_len, H, lse=lse)
    with pytest.raises(ValueError, match="accumulator"):
        ops.attn_bwd_kv(q, o, do, lse, kc, vc, acc0[:, :, :H * HD].contiguous(), cu, case["q"], kv_start, kv_len, case["kv"], H)
    with pytest.raises(ValueError, match="accumulator"):
        ops.attn_bwd_kv(q, o, do, lse, kc, vc, acc0.to(torch.bfloat16), cu, case["q"], kv_start, kv_len, case["kv"], H)


# ------------------------------------------------------------------------------------------------------------------
# rollouts on the tiny-width NavModel of tests/test_prefix_reuse_gpu.py
# ------------------------------------------------------------------------------------------------------------------
INSTR = ["walk past the sofa and stop at the door of the kitchen then turn left and wait by the stairs",
         "leave the room and go down the hall to the second door on the right"]


def _batches(d, steps, instr):
    """The CPU batches of a teacher-forced rollout: fixed detached <hist> vectors, identical in every arm."""
    g = torch.Generator().manual_seed(11)
    gh = torch.Generator().manual_seed(12)
    hist, out = [[] for _ in instr], []
    for step in range(steps):
        out.append(_nav_batch(d, step, hist, g, instr))
        for h in hist:
            h.append(torch.randn(d["hidden"], generator=gh))
    return out


def _rollout(model, d, cuda_dev, cache=None, steps=5, max_length=None, flush=True, instr=INSTR, ddp=None):
    """Teacher-forced rollout with one backward per step (the agent's pattern), the same seed before each step in every
    arm.  ``ddp``: the wrapped model, run in the agent's pattern (no_sync around every step but the last).  Returns
    (per-step fuse_logits, {name: grad})."""
    from contextlib import nullcontext
    if ddp is None:
        model.zero_grad()
    logits = []
    to_dev = lambda b: {k: (v.to(cuda_dev) if torch.is_tensor(v) else v) for k, v in b.items()}
    for step, batch in enumerate(_batches(d, steps, instr)):
        batch = to_dev(batch)
        batch["hist_vis"] = [[v.to(cuda_dev) for v in vs] for vs in batch["hist_vis"]]
        if max_length is not None:                   # left truncation (the tokenizer's truncation_side)
            batch["text_input"] = model.lang_model.tokenizer(batch["prompts"], max_length=max_length, padding=True,
                                                             truncation=True, return_tensors="pt")
        torch.manual_seed(100 + step)
        kw = {} if cache is None else {"prefix_cache": cache}
        ctx = ddp.no_sync if ddp is not None and step != steps - 1 else nullcontext
        with ctx():
            out = (ddp or model)("navigation", batch, **kw)
            F.cross_entropy(out["fuse_logits"].float(), torch.zeros(len(instr), dtype=torch.long, device=cuda_dev)).backward()
        logits.append(out["fuse_logits"].detach().float().cpu())
    if cache is not None and flush and ddp is None:
        cache.flush_grads()
    torch.cuda.synchronize()
    grads = {n: p.grad.detach().float().cpu().clone() for n, p in model.named_parameters() if p.grad is not None}
    return logits, grads


def _oracle_truth(model, d, steps=5, max_length=1024, instr=INSTR):
    """The fp32 CPU oracle on the model's (bf16-valued) weights: the rollout's per-step losses summed, one backward."""
    from oracle import navillm_oracle as O
    tok = model.lang_model.tokenizer
    cfg = O.OracleConfig(hidden=d["hidden"], n_layers=d["n_layers"], n_heads=d["n_heads"], inter=d["inter"], vocab=len(tok),
                         image_feat_size=d["image_feat_size"], obj_feat_size=d["obj_feat_size"], pano_hidden=d["pano_hidden"],
                         pano_heads=d["pano_heads"], pano_inter=d["pano_inter"], cand_id=tok.special["<cand>"],
                         hist_id=tok.special["<hist>"], obj_id=tok.special["<obj>"],
                         cls_ids=(tok.special["<cls_1>"], tok.special["<cls_2>"]), precision="fp32")
    sd = {k: (v.detach().cpu().float().requires_grad_(True) if v.is_floating_point() else v.detach().cpu())
          for k, v in model.state_dict().items()}
    tokenize = lambda p: tok(p, max_length=max_length, padding=True, truncation=True, return_tensors="pt")
    loss, logits = 0.0, []
    for step, batch in enumerate(_batches(d, steps, instr)):
        torch.manual_seed(100 + step)
        out = O.forward_navigation(sd, cfg, batch, tokenize)
        loss = loss + F.cross_entropy(out["fuse_logits"].float(), torch.zeros(len(instr), dtype=torch.long))
        logits.append(out["fuse_logits"].detach().float())
    loss.backward()
    return logits, {k: v.grad.float() for k, v in sd.items() if v.grad is not None}


def _boundary(name, mine, ref, truth, k=3.0, floor=5e-2):
    """The boundary rule of tests/test_fullwidth_parity_gpu.py: |mine - ref| <= k |ref - truth| + floor max|ref|."""
    fin = torch.isfinite(ref)
    assert torch.equal(torch.isfinite(mine), fin), f"{name}: -inf pattern differs"
    scale = ref[fin].abs().max().item()
    e_ref = (ref[fin] - truth[fin]).abs().max().item()
    e = (mine[fin] - ref[fin]).abs().max().item()
    assert e <= k * e_ref + floor * scale + 1e-12, f"{name}: |cache-ref|={e:.4g} > {k}*{e_ref:.4g} + {floor}*{scale:.3g}"
    return e / max(scale, 1e-30)


def _compare(ref, got, truth):
    """fuse_logits of every step within 3e-2 max|logit| of the from-scratch CUDA path; every parameter gradient by the
    boundary rule against that path (ref) and the fp32 oracle (truth)."""
    (lr, gr), (lg, gg), (lt, gt) = ref, got, truth
    for step, (a, r) in enumerate(zip(lg, lr)):
        fin = torch.isfinite(r)
        assert torch.equal(torch.isfinite(a), fin)
        assert (a[fin] - r[fin]).abs().max().item() <= 3e-2 * r[fin].abs().max().item() + 1e-3, step
    assert gr.keys() == gg.keys(), set(gr) ^ set(gg)
    for n in set(gr) - set(gt):           # parameters navigation does not reach (panorama encoder, og_head): untouched
        assert gr[n].abs().max().item() == 0 and gg[n].abs().max().item() == 0, n
    return max(_boundary("grad " + n, gg[n], gr[n], gt[n]) for n in gr if n in gt)


def test_training_rollout_with_cache_matches_from_scratch(cuda_dev):
    from navillm_b200.modified_lm import PrefixKVCache
    model, d = _build(cuda_dev)
    truth = _oracle_truth(model, d)
    ref = _rollout(model, d, cuda_dev)
    cache = PrefixKVCache(model.lang_model, batch_size=2, max_len=256, train=True)
    got = _rollout(model, d, cuda_dev, cache)
    print("max relative gradient difference:", _compare(ref, got, truth))
    st = cache.stats
    assert st["tokens_encoded"] < st["tokens"] and not cache.pending
    assert all(a.abs().max().item() == 0 for a in cache.acc)
    # bit-identical on a second identical rollout (no float atomics anywhere on the path)
    cache2 = PrefixKVCache(model.lang_model, batch_size=2, max_len=256, train=True)
    again = _rollout(model, d, cuda_dev, cache2)
    for n in got[1]:
        assert torch.equal(got[1][n], again[1][n]), n


def test_partial_flush_on_prefix_shrink(cuda_dev):
    """max_length below the prompt length: the tokenizer drops the start of row 1's long instruction once its history
    grows, so row 1's reusable prefix shrinks at step 3 and its pending part (b) runs alone, before its cache rows are
    overwritten.  Row 0 (short instruction, never truncated) keeps reusing its prefix through and after that flush: its
    cache slot must come out of row 1's flush untouched, which the later fuse_logits and the gradients check."""
    from navillm_b200.modified_lm import PrefixKVCache
    model, d = _build(cuda_dev)
    L = 60
    instr = ["go to the door",
             "walk past the sofa and stop at the door of the kitchen then turn left and wait by the stairs next to the big red chair"]
    truth = _oracle_truth(model, d, max_length=L, instr=instr)
    ref = _rollout(model, d, cuda_dev, max_length=L, instr=instr)
    cache = PrefixKVCache(model.lang_model, batch_size=2, max_len=256, train=True)
    events = []
    orig = cache._flush_rows
    cache._flush_rows = lambda rows: (events.append(([b for b in rows if b in cache._pending_rows], list(cache.reused))),
                                      orig(rows))[1]
    got = _rollout(model, d, cuda_dev, cache, max_length=L, instr=instr)
    # step 3: row 1 alone is flushed while row 0 holds reused rows; the final flush covers row 0
    partial = [(rows, reused) for rows, reused in events[:-1] if rows]
    assert partial and all(rows == [1] and reused[0] > 0 for rows, reused in partial), events
    assert events[-1][0] and 0 in events[-1][0], events
    _compare(ref, got, truth)


def test_flush_twice_equals_once(cuda_dev):
    from navillm_b200.modified_lm import PrefixKVCache
    model, d = _build(cuda_dev)
    cache = PrefixKVCache(model.lang_model, batch_size=2, max_len=256, train=True)
    _, once = _rollout(model, d, cuda_dev, cache, steps=3)
    cache.flush_grads()
    torch.cuda.synchronize()
    twice = {n: p.grad.detach().float().cpu() for n, p in model.named_parameters() if p.grad is not None}
    for n in once:
        assert torch.equal(once[n], twice[n]), n


def test_training_cache_guards(cuda_dev):
    from navillm_b200.modified_lm import PrefixKVCache
    model, d = _build(cuda_dev)
    lm = model.lang_model
    with pytest.raises(ValueError, match="train=True"):
        PrefixKVCache(lm, batch_size=2, max_len=128, kv_dtype="fp8", train=True)
    plain = PrefixKVCache(lm, batch_size=2, max_len=128)
    cache = PrefixKVCache(lm, batch_size=2, max_len=256, train=True)
    assert cache.nbytes == plain.nbytes * 2 + sum(a.nbytes for a in cache.acc)
    _rollout(model, d, cuda_dev, cache, steps=3, flush=False)
    assert cache.pending
    with pytest.raises(RuntimeError, match="pending"):
        cache.reset(rows=[0])
    with pytest.raises(RuntimeError, match="pending"):
        model.zero_grad()
    with pytest.raises(RuntimeError, match="pending"):
        model.zero_grad(lazy=True)
    # a weight write before the flush: the flush refuses (its K/V and gradient belong to the old weights)
    with torch.no_grad():
        lm.model.layers[0].mlp.down_proj.weight.mul_(1.0)
    with pytest.raises(RuntimeError, match="weights changed"):
        cache.flush_grads()
    # detached <hist> vectors only
    cache2 = PrefixKVCache(lm, batch_size=2, max_len=256, train=True)
    g = torch.Generator().manual_seed(1)
    batch = _nav_batch(d, 1, [[torch.randn(d["hidden"], requires_grad=True)] for _ in range(2)], g, INSTR)
    batch = {k: (v.to(cuda_dev) if torch.is_tensor(v) else v) for k, v in batch.items()}
    batch["hist_vis"] = [[v.to(cuda_dev) for v in vs] for vs in batch["hist_vis"]]
    with pytest.raises(RuntimeError, match="detached"):
        model("navigation", batch, prefix_cache=cache2)
    # the default cache still refuses grad mode
    with pytest.raises(RuntimeError, match="no_grad"):
        model("navigation", batch, prefix_cache=plain)


def test_weight_change_mid_rollout_raises(cuda_dev):
    from navillm_b200.modified_lm import PrefixKVCache
    model, d = _build(cuda_dev)
    cache = PrefixKVCache(model.lang_model, batch_size=2, max_len=256, train=True)
    _rollout(model, d, cuda_dev, cache, steps=2, flush=False)
    cache.flush_grads()
    model.lang_model.flat.generation += 1            # what the fused AdamW does after a step
    with pytest.raises(RuntimeError, match="weights changed"):
        _rollout(model, d, cuda_dev, cache, steps=1, flush=False)


def test_armed_pass_flushes_before_exchange_and_skips_overlap(cuda_dev, monkeypatch):
    """One process: arm the pass by hand (as the DDP wrapper does outside no_sync) and spy on the order of events."""
    from navillm_b200 import parallel
    from navillm_b200.modified_lm import PrefixKVCache
    model, d = _build(cuda_dev)
    lm = model.lang_model
    cache = PrefixKVCache(lm, batch_size=2, max_len=256, train=True)
    _rollout(model, d, cuda_dev, cache, steps=2, flush=False)
    assert cache.pending
    events = []
    orig_flush = cache.flush_grads
    monkeypatch.setattr(cache, "flush_grads", lambda: (events.append("flush"), orig_flush())[1])
    monkeypatch.setattr(parallel.GradSync, "exchange", lambda self, covered_lm_layers=False: events.append(("exchange", covered_lm_layers)))
    orig_hook = lm._grad_sync_hook
    monkeypatch.setattr(lm, "_grad_sync_hook", lambda: (events.append("hook"), orig_hook())[1])
    g = torch.Generator().manual_seed(3)
    hist = [[torch.randn(d["hidden"]) for _ in range(2)] for _ in range(2)]
    batch = _nav_batch(d, 2, hist, g, INSTR)
    batch = {k: (v.to(cuda_dev) if torch.is_tensor(v) else v) for k, v in batch.items()}
    batch["hist_vis"] = [[v.to(cuda_dev) for v in vs] for vs in batch["hist_vis"]]
    out = model("navigation", batch, prefix_cache=cache)
    model.grad_sync.armed = True
    F.cross_entropy(out["fuse_logits"].float(), torch.zeros(2, dtype=torch.long, device=cuda_dev)).backward()
    assert events == ["flush", ("exchange", False)], events
    assert not cache.pending


# ------------------------------------------------------------------------------------------------------------------
# Vicuna-7B width: two decoder layers, the fused (T >= 1024) branches of the training suffix path and of the flush
# ------------------------------------------------------------------------------------------------------------------
def test_fullwidth_training_rollout_vs_oracle(cuda_dev, monkeypatch):
    """B = 4, 3 steps of the R2R prompt template of tools/prefix_reuse_bench.py with 240-word instructions (378 tokens a row
    at step 0, 271 reused rows a row at the end), so the first step and the flush's prefix recompute both pack more than 1024 rows and take the fused-epilogue GEMMs, and
    gemm_attnd hands the attention backward its D vector).  The nine weight gradients of both layers and the embedding
    rows satisfy the boundary rule against the from-scratch CUDA path and the fp32 oracle; a call spy proves that
    attn_bwd_kv ran in every step's backward and in the flush."""
    from navillm_b200 import ops
    from navillm_b200.modified_lm import PrefixKVCache
    from oracle import navillm_oracle as O
    from tests.test_fullwidth_parity_gpu import LAYERS, _full_navmodel, _oracle_cfg
    sys_path = __import__("sys").path
    sys_path.insert(0, str(__import__("pathlib").Path(__file__).resolve().parents[1] / "tools"))
    from prefix_reuse_bench import make_step
    B, steps, D, G = 4, 3, 4096, 64
    model, tok = _full_navmodel(cuda_dev, base_vocab=4096)
    rng = np.random.RandomState(3)
    words = [f"w{i}" for i in range(3000)]
    instr = [" ".join(words[i] for i in rng.randint(0, 3000, size=240)) for _ in range(B)]
    gh = torch.Generator().manual_seed(4)
    hist = [[torch.randn(D, generator=gh) for _ in range(steps)] for _ in range(B)]

    def batches():
        r, g = np.random.RandomState(5), torch.Generator().manual_seed(6)
        for t in range(steps):
            b = make_step(r, g, B, t, instr, 12, D, G)
            b["hist_vis"] = [h[:t] for h in hist]
            yield b

    target = torch.zeros(B, dtype=torch.long)
    sd = {k: (v.detach().cpu().float().requires_grad_(True) if v.is_floating_point() else v.detach().cpu())
          for k, v in model.state_dict().items()}
    cfg = _oracle_cfg(tok, "fp32")
    loss = 0.0
    for t, b in enumerate(batches()):
        torch.manual_seed(100 + t)
        loss = loss + F.cross_entropy(O.forward_navigation(sd, cfg, b, tok)["fuse_logits"].float(), target)
    loss.backward()

    calls = []
    orig_bwd, orig_attnd = ops.attn_bwd_kv, ops.gemm_attnd
    monkeypatch.setattr(ops, "attn_bwd_kv", lambda *a, **k: (calls.append(("kv", a[0].shape[0], k.get("dvec") is not None)),
                                                             orig_bwd(*a, **k))[1])
    monkeypatch.setattr(ops, "gemm_attnd", lambda *a, **k: (calls.append(("attnd",)), orig_attnd(*a, **k))[1])

    def run(cache):
        model.zero_grad()
        phases = []
        for t, b in enumerate(batches()):
            b = {k: (v.to(cuda_dev) if torch.is_tensor(v) else v) for k, v in b.items()}
            b["hist_vis"] = [[v.to(cuda_dev) for v in vs] for vs in b["hist_vis"]]
            torch.manual_seed(100 + t)
            out = model("navigation", b, **({"prefix_cache": cache} if cache is not None else {}))
            n0 = len(calls)
            F.cross_entropy(out["fuse_logits"].float(), target.to(cuda_dev)).backward()
            phases.append(calls[n0:])
        if cache is not None:
            n0 = len(calls)
            cache.flush_grads()
            phases.append(calls[n0:])
        torch.cuda.synchronize()
        return phases, {n: p.grad.detach().float().cpu().clone() for n, p in model.named_parameters() if p.grad is not None}

    _, ref = run(None)
    cache = PrefixKVCache(model.lang_model, batch_size=B, max_len=512, train=True)
    phases, got = run(cache)
    kv = [[c for c in ph if c[0] == "kv"] for ph in phases]
    assert all(len(k) == LAYERS for k in kv), phases                       # every step's backward and the flush
    assert kv[0][0][1] >= 1024 and kv[-1][0][1] >= 1024, kv                # step 0 and the flush: more than 1024 rows
    assert any(c[2] for c in kv[0]) and any(c[2] for c in kv[-1]), kv       # D from the gemm_attnd epilogue
    named = dict(model.named_parameters())
    keys = [f"lang_model.model.layers.{l}.{nm}.weight" for l in range(LAYERS)
            for nm in ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj", "mlp.gate_proj",
                       "mlp.up_proj", "mlp.down_proj", "input_layernorm", "post_attention_layernorm")]
    keys.append("lang_model.model.embed_tokens.weight")
    truth = {k: sd[k].grad.float() for k in keys}
    for k in keys:
        assert named[k].grad is not None, k
        _boundary("grad " + k, got[k], ref[k], truth[k])


# ------------------------------------------------------------------------------------------------------------------
# two ranks: the agent's no_sync pattern, the armed last step flushes before the exchange
# ------------------------------------------------------------------------------------------------------------------
def _two_rank_worker(rank, world, port, q):
    import os
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"], os.environ["NAVILLM_NVLS"] = "127.0.0.1", str(port), "0"
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from navillm_b200.modified_lm import PrefixKVCache
    from navillm_b200.parallel import DistributedDataParallel as DDP
    bare, d = _build(dev)
    cache = PrefixKVCache(bare.lang_model, batch_size=2, max_len=256, train=True)
    _, single = _rollout(bare, d, dev, cache)                              # one process: flush_grads() by hand
    m, _ = _build(dev)
    ddp = DDP(m, device_ids=[rank], find_unused_parameters=True)
    cache = PrefixKVCache(m.lang_model, batch_size=2, max_len=256, train=True)
    _, synced = _rollout(m, d, dev, cache, ddp=ddp)                        # identical inputs on both ranks
    assert not cache.pending and m.grad_sync.stats["exchanges"] == 1, m.grad_sync.stats
    bad = [n for n in single if not torch.equal(single[n], synced[n])]
    q.put((rank, bad))
    dist.destroy_process_group()


def test_two_rank_no_sync_rollout_matches_single_process():
    """Both ranks run the same rollout, so the exchanged mean equals each rank's own gradient: the DDP result must be the
    single-process flush_grads() result bit for bit."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_two_rank_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=600)
        assert p.exitcode == 0, f"rank failed with exit code {p.exitcode}"
    assert sorted(q.get(timeout=5) for _ in range(2)) == [(0, []), (1, [])]
