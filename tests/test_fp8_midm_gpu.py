"""fp8 weight streaming in the inference GEMMs above 16 rows (nv_gemm_fp8w_bf16): navigation and grounding steps,
prefix-cached suffixes, the pruned last layer and decode batches 17..FP8_MAX_ROWS.

The contract is exact: with the fp8 copy the result is bit for bit what the bf16 kernels return on W', so every check
here is bitwise, or a call spy that shows which kernel ran."""
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

bf16, fp8 = torch.bfloat16, torch.float8_e4m3fn


def _bits(t):
    return t.contiguous().view(torch.int16)


# ---------------------------------------------------------------------------------------------------------------------
# kernel: gemm_fp8w == gemm on W'
# ---------------------------------------------------------------------------------------------------------------------
# (name, N, K, with addend): the four Vicuna-7B layer GEMMs and lm_head (ragged N)
SHAPES = [("qkv", 12288, 4096, False), ("o", 4096, 4096, True), ("gateup", 22016, 4096, False), ("down", 4096, 11008, True),
          ("lm_head", 32006, 4096, False)]


@pytest.fixture(scope="module")
def quantized_weights(cuda_dev):
    from navillm_b200 import ops
    from tests.test_fp8_weights_gpu import edge_rows
    g = torch.Generator(device=cuda_dev).manual_seed(5)
    out = {}
    for name, N, K, _ in SHAPES:
        w = (torch.randn(N, K, generator=g, device=cuda_dev) * 0.02).to(bf16)
        e_rows = edge_rows(K).to(cuda_dev)
        w[:e_rows.shape[0]] = e_rows                               # first tile
        w[N - e_rows.shape[0]:] = e_rows                           # last (ragged) tile
        q = torch.empty((N, K), dtype=fp8, device=cuda_dev)
        e = torch.empty(N, dtype=torch.int8, device=cuda_dev)
        ops.quantize_fp8_(w, q, e)                                 # w becomes W'
        out[name] = (w, q, e)
    return out


@pytest.mark.parametrize("M", [17, 31, 64, 100, 128, 129, 200, 256, 300])
def test_gemm_fp8w_equals_bf16_gemm_on_quantized_weights(cuda_dev, quantized_weights, M):
    from navillm_b200 import ops
    g = torch.Generator(device=cuda_dev).manual_seed(M)
    for name, N, K, with_add in SHAPES:
        w, q, e = quantized_weights[name]
        x = torch.randn(M, K, generator=g, device=cuda_dev).to(bf16)
        add = torch.randn(M, N, generator=g, device=cuda_dev).to(bf16) if with_add else None
        ref = ops.gemm(x, w, addend=add)
        for bn in (0, 32, 128):
            buf = torch.full((M + 8, N), 1234.0, dtype=bf16, device=cuda_dev)    # canary rows past M
            out = ops.gemm_fp8w(x, q, e, addend=add, out=buf[:M], block_n=bn)
            torch.cuda.synchronize()
            assert torch.equal(_bits(out), _bits(ref)), (name, M, bn)
            assert bool((buf[M:] == 1234.0).all()), (name, M, bn, "wrote past row M")


def test_gemm_fp8w_rejects_bad_arguments(cuda_dev, quantized_weights):
    from navillm_b200 import _lib, ops
    w, q, e = quantized_weights["o"]
    x = torch.randn(20, 4096, device=cuda_dev).to(bf16)
    with pytest.raises(_lib.NvError, match="block_n"):
        ops.gemm_fp8w(x, q, e, block_n=256)
    q_pad = torch.zeros((4096, 4096 + 8), dtype=fp8, device=cuda_dev)[:, :4096]     # row stride 4104 bytes
    with pytest.raises(_lib.NvError, match="ldw"):
        ops.gemm_fp8w(x, q_pad, e)


# ---------------------------------------------------------------------------------------------------------------------
# one decoder layer through nv_llama_layer_infer, with and without the fp8 pairs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kv_mode", [0, 1, 2])
@pytest.mark.parametrize("pruned", [False, True])
def test_layer_call_with_fp8_pairs_is_bitwise_bf16(cuda_dev, kv_mode, pruned):
    from navillm_b200 import llama, ops
    D, H, F, Smax = 1024, 8, 2816, 256
    lens = [70, 41, 23]
    B, T = len(lens), sum(lens)
    g = torch.Generator(device=cuda_dev).manual_seed(kv_mode * 2 + pruned)
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
    x = rnd(T, D, sc=1.0)
    cos, sin = llama.rope_tables(llama.LlamaDims(hidden=D, n_heads=H, inter=F), cuda_dev)
    cached = [0] * B if kv_mode != 2 else [30, 0, 12]
    pos = torch.cat([torch.arange(c, c + n, dtype=torch.int32) for c, n in zip(cached, lens)]).to(cuda_dev)
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32, device=cuda_dev)
    out_rows = torch.tensor([69, 110, 133], dtype=torch.int32, device=cuda_dev) if pruned else None
    R = 0 if out_rows is None else out_rows.numel()
    prefix = rnd(B, Smax, D, sc=1.0)

    def run(fp8_pairs, max_rows=256):
        kc, vc = prefix.clone(), prefix.clone() * 0.5
        run = ops.LayerRunner(T, D, F, H, 1e-6, pos, cos, sin, cu, B, ops._qblocks(lens), R=R, device=cuda_dev)
        if kv_mode == 1:
            run.set_cache_mode(1, Smax)
        elif kv_mode == 2:
            c = torch.tensor(cached, dtype=torch.int32, device=cuda_dev)
            start = torch.arange(B, dtype=torch.int32, device=cuda_dev) * Smax
            run.set_cache_mode(2, Smax, B * Smax, c, start, c + torch.tensor(lens, dtype=torch.int32, device=cuda_dev))
        y = torch.empty((R or T, D), dtype=bf16, device=cuda_dev)
        run.run(x, y, ln1, ws[0], ws[1], ln2, ws[2], ws[3], kc=kc if kv_mode else None, vc=vc if kv_mode else None,
                out_rows=out_rows, fp8=fp8_pairs, fp8_max_rows=max_rows)
        torch.cuda.synchronize()
        return y, kc, vc

    y16, kc16, vc16 = run(None)
    y8, kc8, vc8 = run(pairs)
    assert torch.equal(_bits(y8), _bits(y16))
    assert torch.equal(_bits(kc8), _bits(kc16)) and torch.equal(_bits(vc8), _bits(vc16))
    # the pairs are really read: exponents one higher (the weights doubled) change the output
    y_wrong, _, _ = run([(q, e + 1) for q, e in pairs])
    assert not torch.equal(_bits(y_wrong), _bits(y16))
    # ... and only up to fp8_max_rows rows
    y_cut, _, _ = run([(q, e + 1) for q, e in pairs], max_rows=min(lens) - 1 if not pruned else R - 1)
    assert torch.equal(_bits(y_cut), _bits(y16))


# ---------------------------------------------------------------------------------------------------------------------
# the model: golden tiny model, quantized, with the fp8 copy vs after drop_fp8_weights()
# ---------------------------------------------------------------------------------------------------------------------
class _Spy:
    """Counts fp8 GEMMs of more than 16 rows: ops.gemm_fp8w calls (with their row counts) and layer calls given fp8 pairs."""

    def __init__(self, monkeypatch):
        from navillm_b200 import ops
        self.rows, self.layer_calls, self.bf16_rows = [], 0, []
        f, run, gemm = ops.gemm_fp8w, ops.LayerRunner.run, ops.gemm

        def gemm_fp8w(a, *args, **kw):
            self.rows.append(a.shape[0])
            return f(a, *args, **kw)

        def layer_run(obj, *args, fp8=None, **kw):
            self.layer_calls += fp8 is not None
            return run(obj, *args, fp8=fp8, **kw)

        def gemm_bf16(a, *args, **kw):
            self.bf16_rows.append(a.shape[0])
            return gemm(a, *args, **kw)
        monkeypatch.setattr(ops, "gemm_fp8w", gemm_fp8w)
        monkeypatch.setattr(ops.LayerRunner, "run", layer_run)
        monkeypatch.setattr(ops, "gemm", gemm_bf16)

    @property
    def n(self):
        return len(self.rows) + self.layer_calls


def _golden(dev):
    from tests.test_fp8_weights_gpu import _golden_model
    return _golden_model(dev)


def _nav_og(model, g, dev):
    from tests.test_navmodel_gpu import to_dev
    with torch.no_grad():
        pano = model("panorama", to_dev(dict(g["pano_in"]), dev))
        nav_in = to_dev(dict(g["nav_in"]), dev)
        B = pano["pano_embeds"].shape[0]
        nav_in["vp_img_embeds"] = torch.cat([torch.zeros_like(pano["pano_embeds"][:, :1]), pano["pano_embeds"]], 1)
        nav_in["pano_masks"] = torch.cat([torch.ones(B, 1, dtype=torch.bool, device=dev), pano["pano_masks"]], 1)
        torch.manual_seed(1234)
        nav = model("navigation", nav_in)
        og = model("object_grounding", to_dev(dict(g["og_in"]), dev))
    return [nav["fuse_logits"].float().cpu(), nav["fuse_embeds"].float().cpu(), og["obj_logits"].float().cpu()]


def test_navigation_and_grounding_fp8_equal_bf16_on_quantized_weights(cuda_dev, monkeypatch):
    g, cfg, tok, model = _golden(cuda_dev)
    model.quantize_weights_fp8()
    spy = _Spy(monkeypatch)
    with_fp8 = _nav_og(model, g, cuda_dev)
    assert spy.n > 0, "the fp8 copy was not used"
    model.drop_fp8_weights()
    n = spy.n
    without = _nav_og(model, g, cuda_dev)
    assert spy.n == n
    for a, b in zip(with_fp8, without):
        assert torch.equal(a, b)


def test_per_kernel_forward_selects_fp8_by_row_count(cuda_dev, monkeypatch):
    """The per-kernel inference forward (no layer calls) streams fp8 only in GEMMs of at most FP8_MAX_ROWS rows: here the
    full-prompt qkv projections stay bf16 and the <cls> rows of the pruned last layer take the copy."""
    from navillm_b200 import llama
    g, cfg, tok, model = _golden(cuda_dev)
    model.quantize_weights_fp8()
    monkeypatch.setattr(llama.LlamaCore, "LAYER_CALL", False)
    monkeypatch.setattr(llama, "FP8_MAX_ROWS", 16)
    spy = _Spy(monkeypatch)
    with_fp8 = _nav_og(model, g, cuda_dev)
    assert spy.rows and max(spy.rows) <= 16, spy.rows
    assert max(spy.bf16_rows) > 16, spy.bf16_rows
    model.drop_fp8_weights()
    n = spy.n
    without = _nav_og(model, g, cuda_dev)
    assert spy.n == n
    for a, b in zip(with_fp8, without):
        assert torch.equal(a, b)


def _rollout(model, d, dev, steps=4, B=2, seed=11):
    from navillm_b200.modified_lm import PrefixKVCache
    from tests.test_prefix_reuse_gpu import _nav_batch
    g = torch.Generator().manual_seed(seed)
    instr = ["walk past the sofa and stop at the door of the kitchen", "leave the room", "go up the stairs", "turn left"]
    hist = [[] for _ in range(B)]
    cache = PrefixKVCache(model.lang_model, batch_size=B, max_len=256)
    outs = []
    with torch.no_grad():
        for step in range(steps):
            parts = [_nav_batch(d, step, hist[i:i + 2], g, instr[i:i + 2]) for i in range(0, B, 2)]
            batch = {k: (torch.cat([p[k] for p in parts]) if torch.is_tensor(parts[0][k])
                         else None if parts[0][k] is None else sum((p[k] for p in parts), [])) for k in parts[0]}
            batch = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in batch.items()}
            batch["hist_vis"] = [[v.to(dev) for v in vs] for vs in batch["hist_vis"]]
            torch.manual_seed(100 + step)
            got = model("navigation", batch, prefix_cache=cache)
            outs.append((got["fuse_logits"].float().cpu(), got["fuse_embeds"].float().cpu()))
            for b in range(B):
                hist[b].append(got["fuse_embeds"][b, 2].float().cpu())
    assert cache.stats["tokens_encoded"] < cache.stats["tokens"]
    return outs


def test_prefix_cached_rollout_fp8_equals_bf16(cuda_dev, monkeypatch):
    from tests.test_prefix_reuse_gpu import _build
    model, d = _build(cuda_dev)
    model.quantize_weights_fp8()
    spy = _Spy(monkeypatch)
    with_fp8 = _rollout(model, d, cuda_dev)
    assert spy.n > 0
    model.drop_fp8_weights()
    without = _rollout(model, d, cuda_dev)
    for (a1, a2), (b1, b2) in zip(with_fp8, without):
        assert torch.equal(a1, b1) and torch.equal(a2, b2)


def test_generate_above_16_rows_fp8_equals_bf16(cuda_dev, monkeypatch):
    g, cfg, tok, model = _golden(cuda_dev)
    lm = model.lang_model
    text = tok(g["qa_in"]["prompts"])
    ids, mask = text["input_ids"].clone(), text["attention_mask"]
    ids[ids == tok.special["<cand>"]] = 7
    cases = {f"b{rep * 2}_{'graph' if graph else 'eager'}": dict(input_ids=ids.repeat(rep, 1), attention_mask=mask.repeat(rep, 1),
                                                                 max_new_tokens=8, stop_on_eos=False, use_cuda_graph=graph)
             for rep in (10, 20) for graph in (False, True)}
    model.quantize_weights_fp8()
    spy = _Spy(monkeypatch)
    with_fp8 = {}
    for k, kw in cases.items():
        n = len(spy.rows)
        with_fp8[k] = lm.generate(**kw).cpu()
        assert len(spy.rows) > n and min(spy.rows[n:]) > 16, k      # decode GEMMs and lm_head on nv_gemm_fp8w_bf16
    model.drop_fp8_weights()
    n = spy.n
    for k, kw in cases.items():
        assert torch.equal(lm.generate(**kw).cpu(), with_fp8[k]), k
    assert spy.n == n


# ---------------------------------------------------------------------------------------------------------------------
# boundaries: training and stale copies never read the fp8 copy
# ---------------------------------------------------------------------------------------------------------------------
def _train_step_grads(model, g, dev):
    import torch.nn.functional as F
    from tests.test_navmodel_gpu import to_dev
    model.zero_grad(set_to_none=False)
    pano = model("panorama", to_dev(dict(g["pano_in"]), dev))
    nav_in = to_dev(dict(g["nav_in"]), dev)
    B = pano["pano_embeds"].shape[0]
    nav_in["vp_img_embeds"] = torch.cat([torch.zeros_like(pano["pano_embeds"][:, :1]), pano["pano_embeds"]], 1)
    nav_in["pano_masks"] = torch.cat([torch.ones(B, 1, dtype=torch.bool, device=dev), pano["pano_masks"]], 1)
    torch.manual_seed(1234)
    nav = model("navigation", nav_in)
    loss = F.cross_entropy(nav["fuse_logits"].float(), g["targets"].to(dev), reduction="sum", ignore_index=-100) / B
    loss.backward()
    torch.cuda.synchronize()
    return {n: p.grad.detach().clone() for n, p in model.lang_model.named_parameters() if p.grad is not None}


def test_training_forward_and_stale_copy_run_bf16(cuda_dev, monkeypatch):
    g, cfg, tok, model = _golden(cuda_dev)
    model.quantize_weights_fp8()
    spy = _Spy(monkeypatch)
    grads8 = _train_step_grads(model, g, cuda_dev)
    assert spy.n == 0, "a training forward read the fp8 copy"
    model.drop_fp8_weights()
    grads16 = _train_step_grads(model, g, cuda_dev)
    assert grads8.keys() == grads16.keys() and len(grads8) > 0
    for k in grads8:
        assert torch.equal(_bits(grads8[k]), _bits(grads16[k])), k

    # an optimizer step after quantization: the no-grad forwards run bf16 on the new weights, without raising
    model.quantize_weights_fp8()
    lm = model.lang_model
    torch.optim.SGD([p for p in lm.parameters() if p.requires_grad], lr=1e-2).step()
    assert lm.fp8_weights.stale_reason(lm.flat) is not None
    n = spy.n
    stale = _nav_og(model, g, cuda_dev)
    assert spy.n == n, "a stale fp8 copy was read"
    model.drop_fp8_weights()
    fresh_bf16 = _nav_og(model, g, cuda_dev)
    for a, b in zip(stale, fresh_bf16):
        assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------------------
# full width: Vicuna-7B layer widths, 2 layers
# ---------------------------------------------------------------------------------------------------------------------
def test_fullwidth_prefix_step_and_b32_decode_fp8_equal_bf16(cuda_dev, monkeypatch):
    from tests.test_fullwidth_parity_gpu import _full_navmodel
    model, tok = _full_navmodel(cuda_dev, base_vocab=32000)
    model = model.to(cuda_dev)
    d = dict(hidden=4096)
    lm = model.lang_model
    model.quantize_weights_fp8()
    core = lm.core
    Smax, B = 64, 32
    gen = torch.Generator().manual_seed(2)
    x = (torch.randn(B, 4096, generator=gen) * 0.5).to(bf16).to(cuda_dev)
    lens = torch.randint(1, 40, (B,), generator=gen, dtype=torch.int32).to(cuda_dev)
    kv0 = [(torch.randn(B, Smax, 4096, generator=gen) * 0.5).to(bf16).to(cuda_dev) for _ in range(2 * core.d.n_layers)]

    def decode():
        kc, vc = [k.clone() for k in kv0[::2]], [v.clone() for v in kv0[1::2]]
        h = core.decode_step(x, lens, kc, vc)
        torch.cuda.synchronize()
        return h, kc, vc

    spy = _Spy(monkeypatch)
    h8, kc8, vc8 = decode()
    assert spy.rows and min(spy.rows) == B
    roll8 = _rollout(model, d, cuda_dev, steps=2, B=4, seed=5)
    assert spy.layer_calls > 0
    model.drop_fp8_weights()
    n = spy.n
    h16, kc16, vc16 = decode()
    roll16 = _rollout(model, d, cuda_dev, steps=2, B=4, seed=5)
    assert spy.n == n
    assert torch.equal(_bits(h8), _bits(h16))
    for a, b in zip(kc8 + vc8, kc16 + vc16):
        assert torch.equal(_bits(a), _bits(b))
    for (a1, a2), (b1, b2) in zip(roll8, roll16):
        assert torch.equal(a1, b1) and torch.equal(a2, b2)
