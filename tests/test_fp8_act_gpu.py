"""Opt-in fp8 activations (W8A8) in the no-grad prompt forwards (set_activation_dtype("fp8")): the activation quantizer
(nv_quantize_act_fp8), the e4m3 GEMM (nv_gemm_w8a8_bf16) and their use in the decoder layers.

The quantizer is exact (bitwise against a torch reference of the rule).  The GEMM is checked against an fp64 product of
the dequantized operands with a per-element bound, and for batch independence bitwise.  The model paths are checked for
which kernels run, for bitwise agreement between the layer-call and the per-kernel paths, and for their distance from the
bf16 forward on the same W'."""
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

bf16, fp8 = torch.bfloat16, torch.float8_e4m3fn

# c of the bound |C - C64| <= 2^-8 |C64| (+ 2^-8 |A'W'^T| with an addend: the kernel rounds the product to bf16 before it
# adds; 2^-8 is bf16's unit roundoff) + c * sum_k |a_k w_k|: the e4m3 accumulation inside one 128-deep k-block.  The e4m3
# wgmma aligns the products of a k32 step to the largest and keeps fewer bits than fp32, so c is set by the largest
# product of a block.  The largest c measured over every shape and M below was 2^-10.7 (columns of the edge-case weight
# rows; H100 80GB HBM3, 700 W); above 2^-10 the promotion would be broken.
C_BOUND = 2.0 ** -10


def _bits(t):
    return t.contiguous().view(torch.int16)


def ref_quantize_act(x: torch.Tensor):
    """torch reference of the activation rule: (e4m3 [M, K], int8 exponents [M, K/128]) of a bf16 [M, K]."""
    M, K = x.shape
    xb = x.float().reshape(M, K // 128, 128)
    amax = xb.abs().amax(-1)
    m, ex = torch.frexp(amax)
    e = torch.where(m <= 0.875, ex - 9, ex - 8)
    e = torch.where(amax == 0, torch.zeros_like(e), e).clamp(min=-117)
    q = (xb / torch.exp2(e.float())[..., None]).to(fp8)
    return q.reshape(M, K), e.to(torch.int8)


def dequant_act(q, e):
    M, K = q.shape
    return (q.double().reshape(M, K // 128, 128) * torch.exp2(e.double())[..., None]).reshape(M, K)


# ---------------------------------------------------------------------------------------------------------------------
# quantizer
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [4096, 11008])
def test_quantize_act_bitwise_reference(cuda_dev, K):
    from navillm_b200 import ops
    from tests.test_fp8_weights_gpu import edge_rows
    g = torch.Generator(device=cuda_dev).manual_seed(K)
    x = (torch.randn(300, K, generator=g, device=cuda_dev) * 3).to(bf16)
    e_rows = edge_rows(K).to(cuda_dev).to(bf16)
    x[:e_rows.shape[0]] = e_rows
    x[20, 128:256] = 0                                            # a zero block inside a non-zero row
    x[21, :] = -0.0
    x[22, 256:384] *= 2.0 ** 40                                   # a block far above the rest of its row
    x[23, 384:512] *= 2.0 ** -60
    full = torch.randn(300, K + 136, generator=g, device=cuda_dev).to(bf16)
    full[:, 8:K + 8] = x
    for inp in (x, full[:, 8:K + 8]):                             # contiguous and strided (row stride K + 136)
        q, e = ops.quantize_act_fp8(inp)
        torch.cuda.synchronize()
        rq, re = ref_quantize_act(inp.cpu())
        assert torch.equal(e.cpu(), re)
        assert torch.equal(q.cpu().view(torch.uint8), rq.view(torch.uint8))
    # the input is not modified, and rows do not see each other
    q1, e1 = ops.quantize_act_fp8(x[5:6])
    assert torch.equal(q1.view(torch.uint8), q[5:6].view(torch.uint8)) and torch.equal(e1, e[5:6])


def test_quantize_act_rejects_bad_arguments(cuda_dev):
    from navillm_b200 import _lib, ops
    with pytest.raises(ValueError, match="multiple of 128"):
        ops.quantize_act_fp8(torch.zeros(4, 200, dtype=bf16, device=cuda_dev))
    x = torch.zeros(4, 4096 + 4, dtype=bf16, device=cuda_dev)[:, :4096]       # row stride 4100: not 16-byte aligned
    with pytest.raises(_lib.NvError, match="ldx"):
        ops.quantize_act_fp8(x)


# ---------------------------------------------------------------------------------------------------------------------
# GEMM against fp64 on the dequantized operands
# ---------------------------------------------------------------------------------------------------------------------
SHAPES = [("qkv", 12288, 4096, False), ("o", 4096, 4096, True), ("gateup", 22016, 4096, False), ("down", 4096, 11008, True)]
MS = [1, 8, 64, 65, 128, 129, 1000, 4096]


@pytest.fixture(scope="module")
def w8_weights(cuda_dev):
    from navillm_b200 import ops
    from tests.test_fp8_weights_gpu import edge_rows
    g = torch.Generator(device=cuda_dev).manual_seed(7)
    out = {}
    for name, N, K, _ in SHAPES:
        w = (torch.randn(N, K, generator=g, device=cuda_dev) * 0.02).to(bf16)
        er = edge_rows(K).to(cuda_dev)
        w[:er.shape[0]] = er
        q = torch.empty((N, K), dtype=fp8, device=cuda_dev)
        e = torch.empty(N, dtype=torch.int8, device=cuda_dev)
        ops.quantize_fp8_(w, q, e)
        out[name] = (q, e, (q.double() * torch.exp2(e.double())[:, None]))
    return out


def _check_bound(C, A64, W64, add, what):
    acc = A64 @ W64.T
    C64 = acc + add.double() if add is not None else acc
    S = A64.abs() @ W64.abs().T
    slack = (C.double() - C64).abs() - 2.0 ** -8 * C64.abs()
    if add is not None:
        slack = slack - 2.0 ** -8 * acc.abs()
    c = float((slack / S.clamp(min=1e-300)).max())
    print(f"[w8a8 bound] {what}: largest c = {c:.3e} (2^{torch.tensor(max(c, 1e-30)).log2().item():.2f})")
    assert torch.isfinite(C).all(), what
    assert bool((slack <= C_BOUND * S).all()), (what, c)
    return c


@pytest.mark.parametrize("M", MS)
def test_gemm_w8a8_fp64_bound(cuda_dev, w8_weights, M):
    from navillm_b200 import ops
    g = torch.Generator(device=cuda_dev).manual_seed(100 + M)
    for name, N, K, with_add in SHAPES:
        wq, we, W64 = w8_weights[name]
        x = torch.randn(M, K, generator=g, device=cuda_dev).to(bf16)
        add = torch.randn(M, N, generator=g, device=cuda_dev).to(bf16) if with_add else None
        aq, ae = ops.quantize_act_fp8(x)
        buf = torch.full((M + 8, N), 1234.0, dtype=bf16, device=cuda_dev)       # canary rows past M
        C = ops.gemm_w8a8(aq, ae, wq, we, addend=add, out=buf[:M])
        torch.cuda.synchronize()
        assert bool((buf[M:] == 1234.0).all()), (name, M, "wrote past row M")
        _check_bound(C, dequant_act(aq, ae), W64, add, f"{name} M={M}")


def test_gemm_w8a8_all_positive_deep_k(cuda_dev, w8_weights):
    """All-positive operands at K = 11008: no cancellation hides an accumulation error.  Here C64 = sum_k |a_k w_k|, so the
    bound enforced is |C - C64| <= (2^-8 + C_BOUND) C64: the bf16 output rounding dominates it, and it catches a lost,
    repeated or misscaled k-block (each is >= 1/86 of C64), not the promotion interval.  The interval shows in the
    mixed-sign cases above, where sum |a w| is about sqrt(K) times |C64|.  Measured: 2^-7.87 C64 (H100 80GB HBM3, 700 W),
    against 2^-7.71 allowed."""
    from navillm_b200 import ops
    g = torch.Generator(device=cuda_dev).manual_seed(9)
    M, N, K = 512, 4096, 11008
    w = (torch.rand(N, K, generator=g, device=cuda_dev) * 0.05).to(bf16)
    wq = torch.empty((N, K), dtype=fp8, device=cuda_dev)
    we = torch.empty(N, dtype=torch.int8, device=cuda_dev)
    ops.quantize_fp8_(w, wq, we)
    x = (torch.rand(M, K, generator=g, device=cuda_dev) * 4).to(bf16)
    aq, ae = ops.quantize_act_fp8(x)
    C = ops.gemm_w8a8(aq, ae, wq, we)
    torch.cuda.synchronize()
    C64 = dequant_act(aq, ae) @ (wq.double() * torch.exp2(we.double())[:, None]).T
    rel = float(((C.double() - C64).abs() / C64).max())
    print(f"[w8a8 bound] all-positive K=11008: max |C - C64| / C64 = {rel:.3e} (2^{torch.tensor(rel).log2().item():.2f})")
    assert torch.isfinite(C).all() and rel <= 2.0 ** -8 + C_BOUND, rel


def test_gemm_w8a8_rows_are_batch_independent(cuda_dev, w8_weights):
    """A row's output bits are the same alone, in any M and at any position of the packing."""
    from navillm_b200 import ops
    g = torch.Generator(device=cuda_dev).manual_seed(3)
    for name, N, K, with_add in SHAPES:
        wq, we, _ = w8_weights[name]
        M = 1000
        x = torch.randn(M, K, generator=g, device=cuda_dev).to(bf16)
        add = torch.randn(M, N, generator=g, device=cuda_dev).to(bf16) if with_add else None
        lin = lambda xs, ad: ops.gemm_w8a8(*ops.quantize_act_fp8(xs), wq, we, addend=ad)
        full = lin(x, add)
        perm = torch.randperm(M, generator=torch.Generator().manual_seed(1)).to(cuda_dev)
        shuffled = lin(x[perm], add[perm] if add is not None else None)
        assert torch.equal(_bits(shuffled), _bits(full[perm])), name
        for r in (0, 1, 127, 128, 500, 999):
            one = lin(x[r:r + 1], add[r:r + 1] if add is not None else None)
            assert torch.equal(_bits(one), _bits(full[r:r + 1])), (name, r)
        part = lin(x[:65], add[:65] if add is not None else None)
        assert torch.equal(_bits(part), _bits(full[:65])), name


def test_gemm_w8a8_rejects_bad_arguments(cuda_dev, w8_weights):
    from navillm_b200 import _lib, ops
    wq, we, _ = w8_weights["o"]
    aq, ae = ops.quantize_act_fp8(torch.randn(16, 4096, device=cuda_dev).to(bf16))
    with pytest.raises(ValueError, match="contraction"):
        ops.gemm_w8a8(aq[:, :2048], ae[:, :16], wq, we)
    q_pad = torch.zeros((4096, 4096 + 8), dtype=fp8, device=cuda_dev)[:, :4096]     # row stride 4104 bytes
    with pytest.raises(_lib.NvError, match="lda / ldw"):
        ops.gemm_w8a8(aq, ae, q_pad, we)


# ---------------------------------------------------------------------------------------------------------------------
# one decoder layer through nv_llama_layer_infer: a sequence's rows do not depend on the packing, in every kv_mode
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kv_mode", [0, 1, 2, 3, 4])
def test_layer_call_w8a8_packing_independent(cuda_dev, kv_mode):
    from navillm_b200 import llama, ops
    D, H, F, Smax = 1024, 8, 2816, 256
    lens = [70, 41, 23]
    B, T = len(lens), sum(lens)
    g = torch.Generator(device=cuda_dev).manual_seed(kv_mode)
    rnd = lambda *s, sc=0.02: (torch.randn(*s, generator=g, device=cuda_dev) * sc).to(bf16)
    ws, pairs = [], []
    for n, k in ((3 * D, D), (D, D), (2 * F, D), (D, F)):
        w = rnd(n, k)
        q = torch.empty((n, k), dtype=fp8, device=cuda_dev)
        e = torch.empty(n, dtype=torch.int8, device=cuda_dev)
        ops.quantize_fp8_(w, q, e)
        ws.append(w)
        pairs.append((q, e))
    ln1, ln2 = 1 + rnd(D, sc=0.1), 1 + rnd(D, sc=0.1)
    xs = [rnd(n, D, sc=1.0) for n in lens]
    cos, sin = llama.rope_tables(llama.LlamaDims(hidden=D, n_heads=H, inter=F), cuda_dev)
    cached = [30, 0, 12] if kv_mode in (2, 4) else [0] * B
    fp8_cache = kv_mode in (3, 4)
    prefix = rnd(B, Smax, D, sc=1.0)
    if fp8_cache:
        pk = torch.empty((B, Smax, D), dtype=fp8, device=cuda_dev)
        pe = torch.empty((B * Smax * H,), dtype=torch.int8, device=cuda_dev)
        ops.quantize_fp8_(prefix.clone().view(-1, 128), pk.view(-1, 128), pe)
        pe = pe.view(B, Smax, H)

    def run(order):
        ls = [lens[i] for i in order]
        cs = [cached[i] for i in order]
        x = torch.cat([xs[i] for i in order])
        pos = torch.cat([torch.arange(c, c + n, dtype=torch.int32) for c, n in zip(cs, ls)]).to(cuda_dev)
        cu = torch.tensor([0] + list(torch.tensor(ls).cumsum(0)), dtype=torch.int32, device=cuda_dev)
        run = ops.LayerRunner(T, D, F, H, 1e-6, pos, cos, sin, cu, B, ops._qblocks(ls), device=cuda_dev)
        o = torch.tensor(order, device=cuda_dev)
        ke = ve = None
        if fp8_cache:
            kc, vc, ke, ve = pk[o].clone(), pk[o].clone(), pe[o].clone(), pe[o].clone()
        else:
            kc, vc = prefix[o].clone(), prefix[o].clone() * 0.5
        if kv_mode in (1, 3):
            run.set_cache_mode(kv_mode, Smax)
        elif kv_mode in (2, 4):
            c = torch.tensor(cs, dtype=torch.int32, device=cuda_dev)
            start = torch.arange(B, dtype=torch.int32, device=cuda_dev) * Smax
            run.set_cache_mode(kv_mode, Smax, B * Smax, c, start, c + torch.tensor(ls, dtype=torch.int32, device=cuda_dev))
        y = torch.empty((T, D), dtype=bf16, device=cuda_dev)
        run.run(x, y, ln1, ws[0], ws[1], ln2, ws[2], ws[3], kc=kc if kv_mode else None, vc=vc if kv_mode else None,
                ke=ke, ve=ve, fp8=pairs, act_fp8=True)
        torch.cuda.synchronize()
        per_seq = dict(zip(order, torch.split(y, ls)))
        return [per_seq[i] for i in range(B)], kc, vc, o

    ya, kca, vca, _ = run([0, 1, 2])
    yb, kcb, vcb, ob = run([2, 0, 1])
    for a, b in zip(ya, yb):
        assert torch.equal(_bits(a), _bits(b))
    if kv_mode:
        view = (lambda t: t.view(torch.uint8)) if fp8_cache else _bits
        assert torch.equal(view(kcb), view(kca[ob])) and torch.equal(view(vcb), view(vca[ob]))
    assert all(torch.isfinite(t.float()).all() for t in ya)


# ---------------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------------
class _Spy:
    """Counts W8A8 work: ops.gemm_w8a8 calls and layer calls with act_fp8, and the decode-step GEMM launchers."""

    def __init__(self, monkeypatch):
        from navillm_b200 import ops
        self.gemms, self.layer_calls, self.decode = 0, 0, 0
        g8, run = ops.gemm_w8a8, ops.LayerRunner.run

        def gemm_w8a8(*a, **kw):
            self.gemms += 1
            return g8(*a, **kw)

        def layer_run(obj, *a, act_fp8=False, **kw):
            self.layer_calls += bool(act_fp8)
            return run(obj, *a, act_fp8=act_fp8, **kw)
        monkeypatch.setattr(ops, "gemm_w8a8", gemm_w8a8)
        monkeypatch.setattr(ops.LayerRunner, "run", layer_run)
        for name in ("gemm_skinny", "gemm_skinny_fp8", "gemm_skinny_swiglu", "gemm_skinny_swiglu_fp8", "gemm_fp8w"):
            f = getattr(ops, name)

            def wrap(*a, _f=f, **kw):
                self.decode += 1
                return _f(*a, **kw)
            monkeypatch.setattr(ops, name, wrap)

    @property
    def n(self):
        return self.gemms + self.layer_calls


def _rollout(model, d, dev, kv_dtype="bf16", cache=True, steps=3, B=2, seed=11):
    from navillm_b200.modified_lm import PrefixKVCache
    from tests.test_prefix_reuse_gpu import _nav_batch
    g = torch.Generator().manual_seed(seed)
    instr = ["walk past the sofa and stop at the door of the kitchen", "leave the room", "go up the stairs", "turn left"]
    hist = [[] for _ in range(B)]
    pc = PrefixKVCache(model.lang_model, batch_size=B, max_len=256, kv_dtype=kv_dtype) if cache else None
    outs = []
    with torch.no_grad():
        for step in range(steps):
            parts = [_nav_batch(d, step, hist[i:i + 2], g, instr[i:i + 2]) for i in range(0, B, 2)]
            batch = {k: (torch.cat([p[k] for p in parts]) if torch.is_tensor(parts[0][k])
                         else None if parts[0][k] is None else sum((p[k] for p in parts), [])) for k in parts[0]}
            batch = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in batch.items()}
            batch["hist_vis"] = [[v.to(dev) for v in vs] for vs in batch["hist_vis"]]
            torch.manual_seed(100 + step)
            got = model("navigation", batch, prefix_cache=pc) if cache else model("navigation", batch)
            outs.append(got["fuse_logits"].float().cpu())
            for b in range(B):
                hist[b].append(got["fuse_embeds"][b, 2].float().cpu())
    return outs


def _rel(a, b):
    m = torch.isfinite(b)
    return float((a[m] - b[m]).abs().max() / b[m].abs().max())


@pytest.mark.parametrize("per_kernel", [False, True])
def test_navigation_rollouts_run_w8a8(cuda_dev, monkeypatch, per_kernel):
    from navillm_b200 import llama
    from tests.test_prefix_reuse_gpu import _build
    model, d = _build(cuda_dev)
    model.quantize_weights_fp8()
    if per_kernel:
        monkeypatch.setattr(llama.LlamaCore, "LAYER_CALL", False)
    spy = _Spy(monkeypatch)
    runs = {}
    for mode in ("bf16", "fp8"):
        model.set_activation_dtype(mode)
        for kind in ("plain", "bf16_store", "fp8_store"):
            n = spy.n
            runs[mode, kind] = _rollout(model, d, cuda_dev, kv_dtype="fp8" if kind == "fp8_store" else "bf16", cache=kind != "plain")
            if mode == "bf16":
                assert spy.n == n, ("a W8A8 kernel ran in the default mode", kind)
            else:
                assert spy.n > n, ("W8A8 did not run", kind)
    assert model.set_activation_dtype("bf16") == "fp8"
    for kind in ("plain", "bf16_store", "fp8_store"):
        for a, b in zip(runs["fp8", kind], runs["bf16", kind]):
            r = _rel(a, b)
            print(f"[w8a8 nav] {kind} per_kernel={per_kernel}: max|d fuse_logits| / max|logit| = {r:.3e}")
            assert r < 0.1, (kind, r)


def test_generate_prefill_w8a8_decode_unchanged(cuda_dev, monkeypatch):
    from tests.test_fp8_weights_gpu import _golden_model
    g, cfg, tok, model = _golden_model(cuda_dev)
    lm = model.lang_model
    text = tok(g["qa_in"]["prompts"])
    ids, mask = text["input_ids"].clone(), text["attention_mask"]
    ids[ids == tok.special["<cand>"]] = 7
    model.quantize_weights_fp8()
    spy = _Spy(monkeypatch)
    kw = dict(input_ids=ids, attention_mask=mask, max_new_tokens=8, stop_on_eos=False, use_cuda_graph=False)
    base = lm.generate(**kw).cpu()
    n16, dec16 = spy.n, spy.decode
    assert n16 == 0
    assert model.set_activation_dtype("fp8") == "bf16"
    out = lm.generate(**kw).cpu()
    assert spy.layer_calls == lm.dims.n_layers, "the prefill runs one W8A8 layer call per layer"
    assert spy.gemms == 0, "no W8A8 GEMM outside the prefill"
    assert spy.decode - dec16 == dec16, "the decode steps launch the same GEMMs"
    agree = float((out == base).float().mean())
    print(f"[w8a8 generate] token agreement with bf16 activations: {agree:.3f}")
    assert out.shape == base.shape


def test_grad_forwards_unchanged_by_the_mode(cuda_dev, monkeypatch):
    from tests.test_fp8_midm_gpu import _train_step_grads
    from tests.test_fp8_weights_gpu import _golden_model
    g, cfg, tok, model = _golden_model(cuda_dev)
    model.quantize_weights_fp8()
    spy = _Spy(monkeypatch)
    grads16 = _train_step_grads(model, g, cuda_dev)
    model.set_activation_dtype("fp8")
    grads8 = _train_step_grads(model, g, cuda_dev)
    assert spy.n == 0, "a grad-enabled forward ran W8A8"
    assert grads8.keys() == grads16.keys() and len(grads8) > 0
    for k in grads8:
        assert torch.equal(_bits(grads8[k]), _bits(grads16[k])), k


def test_prefix_cache_training_unchanged_by_the_mode(cuda_dev, monkeypatch):
    """PrefixKVCache(train=True) suffix steps with one backward each, then flush_grads(): no W8A8 kernel runs with the mode
    on, and the logits and every gradient are bitwise those of the mode off."""
    from navillm_b200.modified_lm import PrefixKVCache
    from tests.test_prefix_reuse_gpu import _build
    from tests.test_prefix_train_gpu import _rollout as train_rollout
    model, d = _build(cuda_dev)
    model.quantize_weights_fp8()
    spy = _Spy(monkeypatch)
    runs = {}
    for mode in ("bf16", "fp8"):
        model.set_activation_dtype(mode)
        cache = PrefixKVCache(model.lang_model, batch_size=2, max_len=256, train=True)
        runs[mode] = train_rollout(model, d, cuda_dev, cache, steps=3)
        assert cache.stats["tokens_encoded"] < cache.stats["tokens"] and not cache.pending
    assert spy.n == 0, "a grad-enabled forward or the flush ran W8A8"
    (l16, g16), (l8, g8) = runs["bf16"], runs["fp8"]
    assert all(torch.equal(a, b) for a, b in zip(l8, l16))
    assert g8.keys() == g16.keys() and len(g8) > 0
    for k in g8:
        assert torch.equal(g8[k], g16[k]), k


def test_stale_dropped_and_missing_copy_raise(cuda_dev):
    from tests.test_fp8_midm_gpu import _nav_og
    from tests.test_fp8_weights_gpu import _golden_model
    g, cfg, tok, model = _golden_model(cuda_dev)
    with pytest.raises(ValueError):
        model.set_activation_dtype("fp16")
    model.set_activation_dtype("fp8")
    with pytest.raises(RuntimeError, match="quantize_weights_fp8"):          # never quantized
        _nav_og(model, g, cuda_dev)
    model.quantize_weights_fp8()
    _nav_og(model, g, cuda_dev)
    lm = model.lang_model
    torch.optim.SGD([p for p in lm.parameters() if p.requires_grad], lr=1e-2).step()
    with pytest.raises(RuntimeError, match="stale"):
        _nav_og(model, g, cuda_dev)
    model.quantize_weights_fp8()
    _nav_og(model, g, cuda_dev)
    model.drop_fp8_weights()
    with pytest.raises(RuntimeError, match="quantize_weights_fp8"):
        _nav_og(model, g, cuda_dev)
    model.set_activation_dtype("bf16")
    _nav_og(model, g, cuda_dev)


def test_bad_dims_raise(cuda_dev):
    from navillm_b200 import llama
    dims = llama.LlamaDims(hidden=256, n_layers=1, n_heads=2, inter=192, vocab=64)
    model = llama.LlamaModelParams(dims)
    llama.init_llama_params_(model, llama._Linear(64, 256))
    flat = llama.FlatParams(model.flat_order(), cuda_dev)
    core = llama.LlamaCore(dims, model, flat)
    core.act_fp8 = True
    x = torch.zeros((8, 256), dtype=bf16, device=cuda_dev)
    pos = torch.arange(8, dtype=torch.int32, device=cuda_dev)
    cu = torch.tensor([0, 8], dtype=torch.int32, device=cuda_dev)
    with pytest.raises(RuntimeError, match="multiples of 128"):
        core.forward(x, pos, cu, [8], save=False)


# ---------------------------------------------------------------------------------------------------------------------
# full width: Vicuna-7B layer widths, 2 layers, against an fp64 emulation of the quantized dataflow
# ---------------------------------------------------------------------------------------------------------------------
# The fp64 emulation is checked stage by stage: each kernel of a layer (RMSNorm, quantize + W8A8 GEMM, RoPE, attention,
# SwiGLU) runs on the bf16 tensor the previous kernel produced, and its output is within STAGE_BOUND * max|out| of the fp64
# emulation of that stage from the same input.  Measured on H100 80GB HBM3 at 700 W: at most 0.0055 of max|out| (about one
# bf16 ulp of the largest element; RMSNorm, RoPE and SwiGLU exact), for qkv, o, gate|up and down alike.  The same stages
# without the activation quantization are 0.027 of max|qkv| away, so the bound tells the two apart.  The layers of the
# forward (layer-call and per-kernel paths) must then equal that chain of kernels bit for bit: same weight pairs, same
# addends, same order.  The stages are not chained through the emulation itself: one bf16 ulp of difference in a GEMM input
# can move an element to the neighbouring e4m3 value (1/16 of it) or a whole block to the neighbouring exponent, so an
# emulation run from the first layer input drifts by a few % of max|y| per layer whatever the kernels do; that drift is
# printed, not bounded.
STAGE_BOUND = 2.0 ** -6


def _emulate_w8a8(core, x, lens):
    """fp64 emulation of the W8A8 inference forward, one layer per call: every GEMM input quantized by ref_quantize_act, the
    dequantized fp8 weight copy W', fp64 products; RMSNorm, RoPE, attention and SwiGLU in fp64 with bf16 rounding where the
    kernels round (RMSNorm bf16(w * bf16(x rstd)); RoPE bf16(bf16(x1 c) + bf16(-x2 s)); attention output; SwiGLU
    bf16(bf16(silu(g)) u); each GEMM output bf16(acc), then bf16(bf16(acc) + residual)).  Returns stage(name, l, *inputs)
    for the stage-wise check and layer(l, h) for the whole layer."""
    d = core.d
    D, F, H, T = d.hidden, d.inter, d.n_heads, x.shape[0]
    r = lambda t: t.to(bf16).double()
    pos = torch.cat([torch.arange(n) for n in lens]).to(x.device)
    c, s = core.cos.double()[pos][:, None], core.sin.double()[pos][:, None]        # [T, 1, 128]
    pairs = lambda l: {"qkv": core.fp8.wqkv[l], "o": core.fp8.wo[l], "gateup": core.fp8.wgu[l], "down": core.fp8.wd[l]}

    def lin(a, pair, addend=None, quant=True):
        a = a.double()
        if quant:
            a = dequant_act(*ref_quantize_act(a.to(bf16)))
        out = r(a @ (pair[0].double() * torch.exp2(pair[1].double())[:, None]).T)
        return out if addend is None else r(out + addend.double())

    def rms(h, w):
        h = h.double()
        rstd = 1.0 / torch.sqrt((h * h).mean(-1, keepdim=True) + d.rms_eps)
        return r(w.double() * r(h * rstd))

    def rope(qkv):
        qk = qkv[:, :2 * D].double().reshape(T, 2 * H, 128)
        x1, x2 = qk[..., :64], qk[..., 64:]
        return torch.cat([r(r(x1 * c[..., :64]) + r(-x2 * s[..., :64])), r(r(x2 * c[..., 64:]) + r(x1 * s[..., 64:]))], -1)

    def attn(qkv):
        qkv = qkv.double()
        q, k, v = (qkv[:, i * D:(i + 1) * D].reshape(T, H, 128) for i in range(3))
        ao = torch.empty((T, D), dtype=torch.float64, device=x.device)
        t0 = 0
        for n in lens:
            sc = torch.einsum("qhd,khd->hqk", q[t0:t0 + n], k[t0:t0 + n]) * 128 ** -0.5
            sc = sc.masked_fill(torch.ones(n, n, dtype=torch.bool, device=x.device).triu(1), float("-inf"))
            ao[t0:t0 + n] = r(torch.einsum("hqk,khd->qhd", sc.softmax(-1), v[t0:t0 + n]).reshape(n, D))
            t0 += n
        return ao

    def swiglu(gu):
        g, u = gu[:, :F].double(), gu[:, F:].double()
        return r(r(g / (1 + torch.exp(-g))) * u)

    def stage(name, l, *a, quant=True):
        lyr = core.model.layers[l]
        if name == "rms1":
            return rms(a[0], lyr.input_layernorm.weight)
        if name == "rms2":
            return rms(a[0], lyr.post_attention_layernorm.weight)
        if name in ("rope", "attn", "swiglu"):
            return {"rope": rope, "attn": attn, "swiglu": swiglu}[name](a[0])
        return lin(a[0], pairs(l)[name], a[1] if len(a) > 1 else None, quant=quant)

    def layer(l, h):
        xn = stage("rms1", l, h)
        qkv = stage("qkv", l, xn)
        qkv = torch.cat([rope(qkv).reshape(T, 2 * D), qkv[:, 2 * D:]], 1)
        xm = stage("o", l, attn(qkv), h)
        return stage("down", l, swiglu(stage("gateup", l, stage("rms2", l, xm))), xm)
    return stage, layer


def _kernel_chain(core, l, x, pos, cu, lens, stage):
    """Layer l of the W8A8 forward as its chain of kernels (ops calls), each stage checked against the emulation from the
    same input.  Returns (the layer output, {stage: max|out - emu| / max|emu|})."""
    from navillm_b200 import ops
    d = core.d
    lyr, f8 = core.model.layers[l], core.fp8
    err = {}

    def chk(name, out, *inp):
        emu = stage(name, l, *inp)
        if name == "rope":
            out = out[:, :2 * d.hidden].reshape(emu.shape)
        err[name] = float((out.double() - emu).abs().max() / emu.abs().max())
        return out

    w8 = lambda a, p, add=None: ops.gemm_w8a8(*ops.quantize_act_fp8(a), *p, addend=add)
    xn = chk("rms1", ops.rmsnorm_fwd(x, lyr.input_layernorm.weight.data, d.rms_eps)[0], x)
    qkv = chk("qkv", w8(xn, f8.wqkv[l]), xn)
    err["qkv without activation quantization"] = float((qkv.double() - stage("qkv", l, xn, quant=False)).abs().max() /
                                                       qkv.double().abs().max())
    pre = qkv.clone()
    ops.rope_(qkv, pos, core.cos, core.sin, 2 * d.n_heads, d.head_dim)
    chk("rope", qkv, pre)
    ao = chk("attn", ops.attn_fwd(qkv, cu, lens, d.n_heads)[0], qkv)
    xm = chk("o", w8(ao, f8.wo[l], x), ao, x)
    xn2 = chk("rms2", ops.rmsnorm_fwd(xm, lyr.post_attention_layernorm.weight.data, d.rms_eps)[0], xm)
    gu = chk("gateup", w8(xn2, f8.wgu[l]), xn2)
    h = chk("swiglu", ops.swiglu_fwd(gu), gu)
    y = chk("down", w8(h, f8.wd[l], xm), h, xm)
    return y, err


@pytest.mark.parametrize("lens", [[300, 213], [700, 500]])
def test_fullwidth_w8a8_forward(cuda_dev, monkeypatch, lens):
    """Every layer of both the layer-call path and the per-kernel path (at T >= 1024 the fused-epilogue GEMMs give way to
    W8A8 + the RoPE / SwiGLU row kernels) equals its chain of kernels, each kernel within STAGE_BOUND of the fp64 emulation;
    the two paths, and the pruned last layer's rows, bitwise equal."""
    from navillm_b200 import ops
    from navillm_b200 import llama
    from tests.test_fullwidth_parity_gpu import _full_navmodel
    model, tok = _full_navmodel(cuda_dev, base_vocab=32000)
    model = model.to(cuda_dev)
    lm = model.lang_model
    model.quantize_weights_fp8()
    core = lm.core
    T = sum(lens)
    gen = torch.Generator().manual_seed(4)
    x = (torch.randn(T, 4096, generator=gen) * 0.5).to(bf16).to(cuda_dev)
    pos = torch.cat([torch.arange(n, dtype=torch.int32) for n in lens]).to(cuda_dev)
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32, device=cuda_dev)
    rows = torch.tensor([lens[0] - 1, T - 1], dtype=torch.int32, device=cuda_dev)

    ln1 = {lyr.input_layernorm.weight.data_ptr() for lyr in core.model.layers}
    trace = []                                             # the input of every layer, in order

    def run_spy(obj, xin, *a, **kw):
        trace.append(xin.clone())
        return run(obj, xin, *a, **kw)

    def rms_spy(xin, w, *a, **kw):
        if w.data_ptr() in ln1:
            trace.append(xin.clone())
        return rms(xin, w, *a, **kw)

    def fwd(layer_call, out_rows=None):
        monkeypatch.setattr(llama.LlamaCore, "LAYER_CALL", layer_call)
        trace.clear()
        with torch.no_grad():
            h, _ = core.forward(x, pos, cu, lens, save=False, out_rows=out_rows)
        torch.cuda.synchronize()
        return h

    def layers(layer_call):
        """(input, output) of each layer of the last forward"""
        h = fwd(layer_call)
        assert len(trace) == core.d.n_layers
        return list(zip(trace, trace[1:] + [h]))

    spy = _Spy(monkeypatch)
    run, rms = ops.LayerRunner.run, ops.rmsnorm_fwd            # (the call spy's run)
    monkeypatch.setattr(ops.LayerRunner, "run", run_spy)
    monkeypatch.setattr(ops, "rmsnorm_fwd", rms_spy)
    io16 = layers(True)
    h16 = io16[-1][1]
    assert spy.n == 0
    model.set_activation_dtype("fp8")
    io_call, io_kern = layers(True), layers(False)
    h8_call, h8_kern = io_call[-1][1], io_kern[-1][1]
    assert spy.layer_calls == core.d.n_layers and spy.gemms == 4 * core.d.n_layers
    assert torch.equal(_bits(h8_call), _bits(h8_kern))
    p8_call, p8_kern = fwd(True, rows), fwd(False, rows)                 # pruned last layer: R rows
    assert torch.equal(_bits(p8_call), _bits(p8_kern))
    assert torch.equal(_bits(p8_call), _bits(h8_call[rows.long()]))
    stage, layer = _emulate_w8a8(core, x, lens)
    with torch.no_grad():
        for l in range(core.d.n_layers):
            xin = io_call[l][0]
            assert torch.equal(_bits(xin), _bits(io_kern[l][0]))
            y, err = _kernel_chain(core, l, xin, pos, cu, lens, stage)
            print(f"[w8a8 full width] T={T} layer {l}: stage error / max|out| " + ", ".join(f"{k} {v:.2e}" for k, v in err.items()))
            control = err.pop("qkv without activation quantization")
            assert max(err.values()) <= STAGE_BOUND, (l, err)
            assert control > STAGE_BOUND, ("the bound does not separate W8A8 from bf16 activations", l, control)
            assert torch.equal(_bits(y), _bits(io_call[l][1])) and torch.equal(_bits(y), _bits(io_kern[l][1])), l
            assert not torch.equal(_bits(y), _bits(io16[l][1]))
        drift = float((h8_call.double() - layer(1, layer(0, x.double()))).abs().max() / h8_call.double().abs().max())
    err16 = float((h8_call.float() - h16.float()).abs().max() / h16.float().abs().max())
    print(f"[w8a8 full width] T={T}: emulation chained from the input drifts by {drift:.3e} of max|h|; "
          f"max|h_w8a8 - h_bf16| / max|h_bf16| = {err16:.3e}")
