"""4-bit weight streaming in the inference GEMMs of 17 or more rows (nv_gemm_int4w_bf16): decode batches, beams and samples
of 17..INT4_MAX_ROWS rows, navigation and grounding steps, prefix-cached suffixes and the pruned last layer.

The contract is exact: with the int4 copy the result is bit for bit what the bf16 kernels return on W', so every check
here is bitwise, or a call spy that shows which kernel ran.  Int4Weights needs N % 64 and K % 128, so the model checks run
a 2-layer model at Vicuna-7B widths."""
import ctypes
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


def _int4_copy(w):
    """Quantize w in place to W' and return its (codes, scales, zeros)."""
    from navillm_b200 import ops
    N, K = w.shape
    c = (torch.zeros(ops.int4_codes_shape(N, K), dtype=torch.uint8, device=w.device),
         torch.empty((N, K // 128), dtype=bf16, device=w.device), torch.empty((N, K // 128), dtype=torch.uint8, device=w.device))
    ops.quantize_int4_(w, *c)
    return c


# ---------------------------------------------------------------------------------------------------------------------
# kernel: gemm_int4w == gemm on W'
# ---------------------------------------------------------------------------------------------------------------------
# (name, N, K): the four Vicuna-7B decoder-layer GEMMs
SHAPES = [("qkv", 12288, 4096), ("o", 4096, 4096), ("gateup", 22016, 4096), ("down", 4096, 11008)]


@pytest.fixture(scope="module")
def quantized_weights(cuda_dev):
    from tests.test_int4_weights_gpu import _edge_rows
    g = torch.Generator(device=cuda_dev).manual_seed(5)
    out = {}
    for name, N, K in SHAPES:
        w = (torch.randn(N, K, generator=g, device=cuda_dev) * 0.02).to(bf16)
        e_rows = _edge_rows(K).to(cuda_dev)                           # zero, one-signed, tie, clamped, subnormal groups
        w[:e_rows.shape[0]] = e_rows                                   # first tile
        w[N - e_rows.shape[0]:] = e_rows                               # last tile
        out[name] = (w, _int4_copy(w))                                 # w becomes W'
    return out


@pytest.mark.parametrize("M", [17, 31, 32, 33, 48, 63, 64, 65, 128, 300])
def test_gemm_int4w_equals_bf16_gemm_on_quantized_weights(cuda_dev, quantized_weights, M):
    from navillm_b200 import ops
    g = torch.Generator(device=cuda_dev).manual_seed(M)
    for name, N, K in SHAPES:
        w, c = quantized_weights[name]
        x = torch.randn(M, K, generator=g, device=cuda_dev).to(bf16)
        for add in (None, torch.randn(M, N, generator=g, device=cuda_dev).to(bf16)):
            ref = ops.gemm(x, w, addend=add)
            for bn in (0, 32, 128):
                buf = torch.full((M + 8, N), 1234.0, dtype=bf16, device=cuda_dev)    # canary rows past M
                out = ops.gemm_int4w(x, *c, addend=add, out=buf[:M], block_n=bn)
                torch.cuda.synchronize()
                assert torch.equal(_bits(out), _bits(ref)), (name, M, bn, add is not None)
                assert bool((buf[M:] == 1234.0).all()), (name, M, bn, "wrote past row M")


def test_gemm_int4w_refuses_bad_arguments_and_leaves_buffers(cuda_dev, quantized_weights):
    from navillm_b200 import _lib, ops
    w, (codes, scales, zeros) = quantized_weights["o"]
    lib = _lib.load()
    M, N, K = 20, 4096, 4096
    x = torch.randn(M, K, device=cuda_dev).to(bf16)
    out = torch.full((M, N), 7.0, dtype=bf16, device=cuda_dev)
    before = [t.clone() for t in (x, codes, scales, zeros, out)]
    P = lambda t, off=0: ctypes.c_void_p(t.data_ptr() + off)
    null = ctypes.c_void_p(0)
    i32, i64 = ctypes.c_int, ctypes.c_int64

    def call(a=None, c=None, s=None, z=None, o=None, lda=K, ldc=N, m=M, n=N, k=K, bn=0):
        return lib.nv_gemm_int4w_bf16(P(x) if a is None else a, i64(lda), P(codes) if c is None else c,
                                      P(scales) if s is None else s, P(zeros) if z is None else z, P(out) if o is None else o,
                                      i64(ldc), null, i64(0), i32(m), i32(n), i32(k), i32(bn), _lib.stream_ptr())
    refusals = {
        "null A": call(a=null), "null codes": call(c=null), "null scales": call(s=null), "null zeros": call(z=null),
        "null C": call(o=null), "K % 128": call(k=K - 64, lda=K), "N % 64": call(n=N - 32), "lda % 8": call(lda=K + 4),
        "lda < K": call(lda=K - 8), "ldc < N": call(ldc=N - 8), "A alignment": call(a=P(x, 8)),
        "codes alignment": call(c=P(codes, 8)), "C alignment": call(o=P(out, 8)), "block_n 64": call(bn=64),
        "block_n 256": call(bn=256), "M 0": call(m=0),
    }
    torch.cuda.synchronize()
    for what, rc in refusals.items():
        assert rc != 0, what
    for a, b in zip(before, (x, codes, scales, zeros, out)):
        assert torch.equal(a, b)
    # the Python entry point checks before any launch
    with pytest.raises(ValueError, match="block_n"):
        ops.gemm_int4w(x, codes, scales, zeros, block_n=256)
    with pytest.raises(ValueError, match="multiple of 64"):
        ops.gemm_int4w(x, codes[:, :], scales[:32], zeros[:32])
    with pytest.raises(ValueError, match="codes"):
        ops.gemm_int4w(x, codes[:64], scales, zeros)
    with pytest.raises(ValueError, match=r"a bf16 \[M, 4096\]"):
        ops.gemm_int4w(x[:, :2048], codes, scales, zeros)
    with pytest.raises(ValueError, match="out"):
        ops.gemm_int4w(x, codes, scales, zeros, out=out[:, :2048])
    torch.cuda.synchronize()
    for a, b in zip(before, (x, codes, scales, zeros, out)):
        assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------------------
# one decoder layer through nv_llama_layer_infer, with and without the int4 triples
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kv_mode", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("pruned", [False, True])
def test_layer_call_with_int4_triples_is_bitwise_bf16(cuda_dev, kv_mode, pruned):
    from navillm_b200 import _lib, llama, ops
    D, H, F, Smax = 1024, 8, 2816, 256
    lens = [30, 21, 18]
    B, T = len(lens), sum(lens)
    g = torch.Generator(device=cuda_dev).manual_seed(kv_mode * 2 + pruned)
    rnd = lambda *s, sc=0.02: (torch.randn(*s, generator=g, device=cuda_dev) * sc).to(bf16)
    ws, triples = [], []
    for n, k in ((3 * D, D), (D, D), (2 * F, D), (D, F)):
        w = rnd(n, k)
        triples.append(_int4_copy(w))
        ws.append(w)
    ln1, ln2 = 1 + rnd(D, sc=0.1), 1 + rnd(D, sc=0.1)
    x = rnd(T, D, sc=1.0)
    cos, sin = llama.rope_tables(llama.LlamaDims(hidden=D, n_heads=H, inter=F), cuda_dev)
    suffix = kv_mode in (2, 4)
    cached = [30, 0, 12] if suffix else [0] * B
    pos = torch.cat([torch.arange(c, c + n, dtype=torch.int32) for c, n in zip(cached, lens)]).to(cuda_dev)
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32, device=cuda_dev)
    out_rows = torch.arange(0, T, 3, dtype=torch.int32, device=cuda_dev)[:23] if pruned else None    # 23 rows: > 16
    R = 0 if out_rows is None else out_rows.numel()
    fp8_kv = kv_mode in (3, 4)
    prefix = rnd(B, Smax, D, sc=1.0)

    def run(int4, max_rows=256):
        if fp8_kv:
            kc, vc = prefix.to(fp8), (prefix * 0.5).to(fp8)
            ke = torch.zeros((B, Smax, H), dtype=torch.int8, device=cuda_dev)
            ve = torch.ones((B, Smax, H), dtype=torch.int8, device=cuda_dev)
        else:
            kc, vc, ke, ve = prefix.clone(), prefix.clone() * 0.5, None, None
        run = ops.LayerRunner(T, D, F, H, 1e-6, pos, cos, sin, cu, B, ops._qblocks(lens), R=R, device=cuda_dev)
        if kv_mode in (1, 3):
            run.set_cache_mode(kv_mode, Smax)
        elif suffix:
            c = torch.tensor(cached, dtype=torch.int32, device=cuda_dev)
            start = torch.arange(B, dtype=torch.int32, device=cuda_dev) * Smax
            run.set_cache_mode(kv_mode, Smax, B * Smax, c, start, c + torch.tensor(lens, dtype=torch.int32, device=cuda_dev))
        y = torch.empty((R or T, D), dtype=bf16, device=cuda_dev)
        run.run(x, y, ln1, ws[0], ws[1], ln2, ws[2], ws[3], kc=kc if kv_mode else None, vc=vc if kv_mode else None,
                ke=ke, ve=ve, out_rows=out_rows, int4=int4, int4_max_rows=max_rows)
        torch.cuda.synchronize()
        return [y] + ([kc.view(torch.uint8), vc.view(torch.uint8), ke, ve] if fp8_kv else [kc, vc] if kv_mode else [])

    ref = run(None)
    got = run(triples)
    for a, b in zip(got, ref):
        assert torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))
    # the triples are really read: doubled scales change the output ...
    doubled = [(c, s * 2, z) for c, s, z in triples]
    assert not torch.equal(_bits(run(doubled)[0]), _bits(ref[0]))
    # ... and only at 17..int4_max_rows rows
    assert torch.equal(_bits(run(doubled, max_rows=16)[0]), _bits(ref[0]))
    # the int4 and the fp8 copies exclude each other
    q = torch.empty((3 * D, D), dtype=fp8, device=cuda_dev)
    e = torch.zeros(3 * D, dtype=torch.int8, device=cuda_dev)
    run_ = ops.LayerRunner(T, D, F, H, 1e-6, pos, cos, sin, cu, B, ops._qblocks(lens), R=R, device=cuda_dev)
    with pytest.raises(_lib.NvError, match="exclude each other"):
        run_.run(x, torch.empty((R or T, D), dtype=bf16, device=cuda_dev), ln1, ws[0], ws[1], ln2, ws[2], ws[3],
                 out_rows=out_rows, fp8=[(q, e), (None, None), (None, None), (None, None)], fp8_max_rows=64, int4=triples,
                 int4_max_rows=64)


# ---------------------------------------------------------------------------------------------------------------------
# the model: a 2-layer model at Vicuna-7B widths, with the int4 copy vs after drop_int4_weights()
# ---------------------------------------------------------------------------------------------------------------------
class _Spy:
    """Records the row count of every nv_gemm_int4w_bf16 call (ops.gemm_int4w) and counts layer calls given int4 triples
    with a GEMM of 17..int4_max_rows rows."""

    def __init__(self, monkeypatch):
        from navillm_b200 import ops
        self.rows, self.layer_calls = [], 0
        f, run = ops.gemm_int4w, ops.LayerRunner.run

        def gemm_int4w(a, *args, **kw):
            self.rows.append(a.shape[0])
            return f(a, *args, **kw)

        def layer_run(obj, *args, int4=None, int4_max_rows=0, out_rows=None, **kw):
            rows = [obj.T] + ([out_rows.numel()] if out_rows is not None else [])
            self.layer_calls += int4 is not None and any(16 < r <= int4_max_rows for r in rows)
            return run(obj, *args, int4=int4, int4_max_rows=int4_max_rows, out_rows=out_rows, **kw)
        monkeypatch.setattr(ops, "gemm_int4w", gemm_int4w)
        monkeypatch.setattr(ops.LayerRunner, "run", layer_run)

    @property
    def n(self):
        return len(self.rows) + self.layer_calls


@pytest.fixture(scope="module")
def fullwidth(cuda_dev):
    from tests.test_fullwidth_parity_gpu import _full_navmodel
    model, tok = _full_navmodel(cuda_dev, base_vocab=32000)
    model = model.to(cuda_dev)
    model._ensure()
    return model, tok


def test_generate_17_to_64_rows_int4_equals_bf16(cuda_dev, fullwidth, monkeypatch):
    from navillm_b200 import llama
    from tests.test_fullwidth_parity_gpu import HID
    from tests.test_generate_gpu import _Trie
    from tests.test_int4_weights_gpu import N_CAND, _prompts
    model, tok = fullwidth
    lm = model.lang_model
    cand = lambda B: torch.randn(B * N_CAND, HID, generator=torch.Generator().manual_seed(B)).to(cuda_dev)
    base = lambda B, seed: dict(input_ids=(t := _prompts(tok, B, seed=seed))["input_ids"], attention_mask=t["attention_mask"],
                                cand_vis=cand(B), stop_on_eos=False)
    eos = tok.eos_token_id
    trie = _Trie(tok.bos_token_id, eos)
    for w in ([11, 12, 13], [11, 12, 40, 41], [11, 50], [60, 61, 62]):
        trie.insert(w)
    cases = {
        "greedy_b20_eager": (dict(base(20, 1), max_new_tokens=6, use_cuda_graph=False), 20),
        "greedy_b20_graph": (dict(base(20, 1), max_new_tokens=6, use_cuda_graph=True), 20),
        "greedy_b40_eager": (dict(base(40, 2), max_new_tokens=6, use_cuda_graph=False), 40),
        "greedy_b40_graph": (dict(base(40, 2), max_new_tokens=6, use_cuda_graph=True), 40),
        "trie_b20": (dict(base(20, 3), max_new_tokens=6, trie=trie, eos_token_id=eos, pad_token_id=tok.unk_token_id), 20),
        "beams4_b8": (dict(base(8, 4), max_new_tokens=6, num_beams=4), 32),
        "samples4_b8": (dict(base(8, 5), max_new_tokens=6, do_sample=True, temperature=0.8, top_p=0.9, num_return_sequences=4), 32),
        "fp8_kv_greedy_b20": (dict(base(20, 1), max_new_tokens=6), 20),
        "fp8_kv_beams4_b8": (dict(base(8, 4), max_new_tokens=6, num_beams=4), 32),
    }
    assert llama.INT4_MAX_ROWS >= 40

    def run_all(spy=None):
        out = {}
        for k, (kw, rows) in cases.items():
            lm.set_kv_cache_dtype("fp8" if k.startswith("fp8_kv") else "bf16")
            n0 = len(spy.rows) if spy else 0
            torch.manual_seed(77)
            out[k] = lm.generate(**kw).cpu()
            if spy is not None:
                assert rows in spy.rows[n0:], (k, sorted(set(spy.rows[n0:])))     # the decode step streamed the copy
        lm.set_kv_cache_dtype("bf16")
        return out

    model.quantize_weights_int4()
    try:
        spy = _Spy(monkeypatch)
        with_int4 = run_all(spy)
    finally:
        model.drop_int4_weights()
    n = spy.n
    without = run_all()
    assert spy.n == n
    for k in with_int4:
        assert torch.equal(with_int4[k], without[k]), k


def _nav_og_rollout(model, dev, steps=4, B=4):
    """fuse_logits / fuse_embeds of one navigation step without a prefix cache, obj_logits of one grounding step, and a
    ``steps``-step prefix-cached rollout, at full width."""
    from tests.test_fp8_midm_gpu import _rollout
    from tests.test_oracle_golden import load
    from tests.test_prefix_reuse_gpu import _nav_batch
    D = 4096
    g = torch.Generator().manual_seed(3)
    instr = ["walk past the sofa and stop at the door of the kitchen", "leave the room"]
    batch = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in _nav_batch(dict(hidden=D), 1, [[torch.randn(D, generator=g)]] * 2,
                                                                                g, instr).items()}
    batch["hist_vis"] = [[v.to(dev) for v in vs] for vs in batch["hist_vis"]]
    og = dict(load("amp_bf16")[0]["og_in"])
    og["obj_embeds"] = torch.randn(2, 5, D, generator=g).to(dev)
    og["obj_masks"], og["obj_loc_fts"] = og["obj_masks"].to(dev), og["obj_loc_fts"].to(dev)
    og["hist_vis"] = [[torch.randn(D, generator=g).to(dev) for _ in vs] for vs in og["hist_vis"]]
    with torch.no_grad():
        torch.manual_seed(1234)
        nav = model("navigation", batch)
        obj = model("object_grounding", og)
    outs = [nav["fuse_logits"].float().cpu(), nav["fuse_embeds"].float().cpu(), obj["obj_logits"].float().cpu()]
    for a, b in _rollout(model, dict(hidden=D), dev, steps=steps, B=B, seed=5):
        outs += [a, b]
    return outs


@pytest.mark.parametrize("layer_call", [True, False])
def test_navigation_grounding_and_prefix_rollout_int4_equal_bf16(cuda_dev, fullwidth, monkeypatch, layer_call):
    """The no-grad forwards stream the copy in their GEMMs of 17..INT4_MAX_ROWS rows; here every GEMM of at least 17 rows
    takes it (INT4_MAX_ROWS raised), through the layer calls and through the per-kernel path."""
    from navillm_b200 import llama
    model, tok = fullwidth
    monkeypatch.setattr(llama.LlamaCore, "LAYER_CALL", layer_call)
    monkeypatch.setattr(llama, "INT4_MAX_ROWS", 1 << 20)
    model.quantize_weights_int4()
    try:
        spy = _Spy(monkeypatch)
        with_int4 = _nav_og_rollout(model, cuda_dev)
        assert spy.n > 0, "the int4 copy was not used"
        if not layer_call:
            assert min(spy.rows) > 16, spy.rows
    finally:
        model.drop_int4_weights()
    n = spy.n
    without = _nav_og_rollout(model, cuda_dev)
    assert spy.n == n
    for a, b in zip(with_int4, without):
        assert torch.equal(a, b)


def test_training_forward_and_stale_copy_run_bf16(cuda_dev, fullwidth, monkeypatch):
    from navillm_b200 import llama
    from tests.test_prefix_reuse_gpu import _nav_batch
    model, tok = fullwidth
    lm = model.lang_model
    monkeypatch.setattr(llama, "INT4_MAX_ROWS", 1 << 20)
    g = torch.Generator().manual_seed(9)
    batch = {k: (v.to(cuda_dev) if torch.is_tensor(v) else v)
             for k, v in _nav_batch(dict(hidden=4096), 0, [[], []], g, ["leave the room", "turn left"]).items()}

    def train_forward():
        torch.manual_seed(1)
        out = model("navigation", batch)["fuse_logits"]
        out.float().sum().backward()
        torch.cuda.synchronize()
        grads = [p.grad.detach().clone() for p in lm.int4_linear_weights() if p.grad is not None]
        assert grads
        model.zero_grad(set_to_none=False)
        return out.detach().float().cpu(), grads

    model.quantize_weights_int4()
    try:
        spy = _Spy(monkeypatch)
        y4, g4 = train_forward()
        assert spy.n == 0, "a training forward read the int4 copy"
        model.drop_int4_weights()
        y16, g16 = train_forward()
        assert torch.equal(y4, y16)
        for a, b in zip(g4, g16):
            assert torch.equal(_bits(a), _bits(b))

        # a weight write after quantization: the no-grad forwards run bf16 on the current weights, without raising
        model.quantize_weights_int4()
        with torch.no_grad():
            lm.model.layers[1].mlp.down_proj.weight.mul_(0.5)
        assert lm.int4_weights.stale_reason(lm.flat) is not None
        assert lm.core.int4_for_inference() is None
        n = spy.n
        stale = _nav_og_rollout(model, cuda_dev, steps=2, B=2)
        assert spy.n == n, "a stale int4 copy was read"
        with pytest.raises(RuntimeError, match="int4 copy of the weights is stale"):     # generate() keeps refusing it
            t = tok(["Question w1 w2 Answer"] * 20)
            lm.generate(input_ids=t["input_ids"], attention_mask=t["attention_mask"], max_new_tokens=2)
    finally:
        model.drop_int4_weights()
    fresh = _nav_og_rollout(model, cuda_dev, steps=2, B=2)
    for a, b in zip(stale, fresh):
        assert torch.equal(a, b)
