"""GPTQ-calibrated 4-bit weights: Hessians recorded from ordinary forwards (Int4Calibration), the error-feedback quantizer
on the device (ops.gptq_int4_, nv_gptq_int4_block) and the public switch quantize_weights_int4(calibration=...).

The copy has the format of the round-to-nearest one, so the decode kernels' bitwise contract (bf16 on W') is checked here
only as a spot check; the quantizer is checked against the fp64 restatement of tests/gptq_oracle.py."""
import ctypes
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from tests import gptq_oracle as O  # noqa: E402
from tests.test_int4_gptq_cpu import correlated_inputs  # noqa: E402

bf16 = torch.bfloat16


def _bits(t):
    return t.contiguous().view(torch.int16)


def _copy_bufs(N, K, dev):
    from navillm_b200 import ops
    return (torch.zeros(ops.int4_codes_shape(N, K), dtype=torch.uint8, device=dev),
            torch.empty((N, K // 128), dtype=bf16, device=dev), torch.empty((N, K // 128), dtype=torch.uint8, device=dev))


# ---------------------------------------------------------------------------------------------------------------------
# the quantizer
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,K", [(12288, 4096), (4096, 4096), (22016, 4096), (4096, 11008)])
def test_identity_hessian_is_bitwise_round_to_nearest(cuda_dev, N, K):
    """With H = I no error reaches another column, so GPTQ is the RTN rule: codes, scales, zeros and W' bit for bit."""
    from navillm_b200 import ops
    g = torch.Generator(device=cuda_dev).manual_seed(N + K)
    w = (torch.randn(N, K, generator=g, device=cuda_dev) * 0.02).to(bf16)
    w[5, :128] = 0.0                                                       # an all-zero group
    w[70, 128:256] = w[70, 128:256].abs()                                  # one-signed groups
    w[N - 1, -128:] = -w[N - 1, -128:].abs()
    w_rtn, w_gptq = w.clone(), w
    rtn, gptq = _copy_bufs(N, K, cuda_dev), _copy_bufs(N, K, cuda_dev)
    ops.quantize_int4_(w_rtn, *rtn)
    ops.gptq_int4_(w_gptq, torch.eye(K, device=cuda_dev), *gptq)
    torch.cuda.synchronize()
    assert torch.equal(_bits(w_gptq), _bits(w_rtn))
    for a, b in zip(gptq, rtn):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))


@pytest.mark.parametrize("N,K", [(256, 512), (192, 1024)])
def test_quantizer_against_fp64_oracle(cuda_dev, N, K):
    from navillm_b200 import ops
    gen = torch.Generator().manual_seed(N * K)
    W = (torch.randn(N, K, generator=gen) * 0.02).to(bf16)
    X = correlated_inputs(4096, K, seed=K)
    H32 = torch.from_numpy(X.T @ X).float()                                # the fp32 H both sides factor
    H = H32.double().numpy()
    q_ref, s_ref, z_ref, wq_ref = O.gptq(W.float().numpy(), O.factor(H))
    w = W.to(cuda_dev)
    codes, scales, zeros = _copy_bufs(N, K, cuda_dev)
    ops.gptq_int4_(w, H32.to(cuda_dev), codes, scales, zeros)
    s, z, wq = scales.float().cpu().numpy(), zeros.cpu().numpy().astype(np.float64), w.float().cpu().numpy()
    # group 0 starts from the unmodified weights: its (s, z) are exact
    assert np.array_equal(s[:, 0], s_ref[:, 0]) and np.array_equal(z[:, 0], z_ref[:, 0])
    # the codes: W' = bf16((q - z) s) with |q - z| <= 15 determines q
    q = np.rint(wq / np.repeat(s, 128, 1)) + np.repeat(z, 128, 1)
    assert np.array_equal(O.value(q, np.repeat(s, 128, 1), np.repeat(z, 128, 1)), wq.astype(np.float64)), "W' off grid"
    assert (q == q_ref).mean() >= 0.99, (q == q_ref).mean()
    # the packed codes describe the same W' (the skinny GEMM on them is bitwise the bf16 GEMM on W')
    x = torch.randn(7, K, generator=gen).to(bf16).to(cuda_dev)
    assert torch.equal(_bits(ops.gemm_skinny_int4(x, codes, scales, zeros)), _bits(ops.gemm_skinny(x, w)))
    l_gpu, l_ref = O.loss(W.float().numpy(), wq, H), O.loss(W.float().numpy(), wq_ref, H)
    w_rtn = W.to(cuda_dev)
    ops.quantize_int4_(w_rtn, *_copy_bufs(N, K, cuda_dev))
    l_rtn = O.loss(W.float().numpy(), w_rtn.float().cpu().numpy(), H)
    assert abs(l_gpu - l_ref) <= 0.01 * l_ref, (l_gpu, l_ref)
    assert l_gpu < l_rtn, (l_gpu, l_rtn)


def test_block_kernel_refuses_bad_arguments_and_leaves_buffers(cuda_dev):
    from navillm_b200 import _lib, ops
    N, K = 128, 256
    lib = _lib.load()
    wf = torch.randn(N, K, device=cuda_dev)
    u = torch.eye(K, device=cuda_dev)
    w = torch.randn(N, K, device=cuda_dev).to(bf16)
    codes, scales, zeros = _copy_bufs(N, K, cuda_dev)
    scales.fill_(1.0)
    zeros.fill_(3)
    ne = torch.full((N, 128), 5.0, device=cuda_dev)
    bufs = (wf, u, w, codes, scales, zeros, ne)
    before = [t.clone() for t in bufs]
    P = lambda t, off=0: ctypes.c_void_p(t.data_ptr() + off)
    null = ctypes.c_void_p(0)
    i32, i64 = ctypes.c_int, ctypes.c_int64

    def call(wf_=None, u_=None, w_=None, c=None, e=None, ldwf=K, ldu=K, ldw=K, lde=128, g=0, n=N, k=K):
        return lib.nv_gptq_int4_block(P(wf) if wf_ is None else wf_, i64(ldwf), P(u) if u_ is None else u_, i64(ldu), i32(g),
                                      P(w) if w_ is None else w_, i64(ldw), P(codes) if c is None else c, P(scales), P(zeros),
                                      P(ne) if e is None else e, i64(lde), i32(n), i32(k), _lib.stream_ptr())
    refusals = {
        "null Wf": call(wf_=null), "null U": call(u_=null), "null W": call(w_=null), "null codes": call(c=null),
        "null E": call(e=null), "N % 64": call(n=96), "N 0": call(n=0), "K % 128": call(k=192), "g < 0": call(g=-1),
        "g >= K / 128": call(g=2), "ldwf < K": call(ldwf=K - 1), "ldw < K": call(ldw=K - 8), "ldu < 128": call(ldu=64),
        "lde < 128": call(lde=64), "codes alignment": call(c=P(codes, 8)),
    }
    torch.cuda.synchronize()
    for what, rc in refusals.items():
        assert rc != 0, what
    for a, b in zip(before, bufs):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))
    # the Python entry point checks before any launch
    with pytest.raises(ValueError, match="multiple of 64"):
        ops.gptq_int4_(w[:96], u, *_copy_bufs(96, K, cuda_dev))
    with pytest.raises(ValueError, match="H or U"):
        ops.gptq_int4_(w, u[:128, :128], codes, scales, zeros)
    with pytest.raises(ValueError, match="H or U"):
        ops.gptq_int4_(w, u.double(), codes, scales, zeros)
    with pytest.raises(ValueError, match="codes"):
        ops.gptq_int4_(w, u, codes[:64], scales, zeros)
    torch.cuda.synchronize()
    for a, b in zip(before, bufs):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))


# ---------------------------------------------------------------------------------------------------------------------
# the Hessians: recorded from LlamaCore.forward / forward_suffix on a small model (widths multiples of 128)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def small(cuda_dev):
    from tests.test_prefix_reuse_gpu import _build
    model, d = _build(cuda_dev)
    model._ensure()
    return model, d


class _Inputs:
    """Records, independently of Int4Calibration, the operand every decoder-layer linear consumed, keyed like its H."""

    def __init__(self, monkeypatch, core):
        from navillm_b200 import llama, ops
        self.x = {}
        key = {}
        for l in range(core.d.n_layers):
            for name, w in zip(("qkv", "o_proj", "gate_up", "down_proj"), (core.wqkv[l], core.wo[l], core.wgu[l], core.wd[l])):
                key[w.data_ptr()] = (l, name)

        def keep(a, w):
            self.x.setdefault(key[w.data_ptr()], []).append(a.detach().clone())
        lin, rope, swiglu = llama.LlamaCore._linear, ops.gemm_rope, ops.gemm_swiglu

        def _linear(a, w, *args, **kw):
            keep(a, w)
            return lin(a, w, *args, **kw)

        def gemm_rope(a, w, *args, **kw):
            keep(a, w)
            return rope(a, w, *args, **kw)

        def gemm_swiglu(a, w, *args, **kw):
            keep(a, w)
            return swiglu(a, w, *args, **kw)
        monkeypatch.setattr(llama.LlamaCore, "_linear", staticmethod(_linear))
        monkeypatch.setattr(ops, "gemm_rope", gemm_rope)
        monkeypatch.setattr(ops, "gemm_swiglu", gemm_swiglu)


def _packed(seqlens, D, dev, seed, cached=None):
    g = torch.Generator().manual_seed(seed)
    cached = cached or [0] * len(seqlens)
    x = torch.randn(sum(seqlens), D, generator=g).to(bf16).to(dev)
    pos = torch.cat([torch.arange(c, c + n, dtype=torch.int32) for c, n in zip(cached, seqlens)]).to(dev)
    cu = torch.tensor([0] + np.cumsum(seqlens).tolist(), dtype=torch.int32, device=dev)
    return x, pos, cu


def test_hessians_equal_fp64_products_and_forwards_keep_their_bits(cuda_dev, small, monkeypatch):
    from navillm_b200 import llama
    model, d = small
    lm = model.lang_model
    core, D = lm.core, d["hidden"]
    B, Smax = 2, 768
    kc = [torch.zeros((B, Smax, D), dtype=bf16, device=cuda_dev) for _ in range(d["n_layers"])]
    vc = [torch.zeros_like(k) for k in kc]
    start = torch.arange(B, dtype=torch.int32, device=cuda_dev) * Smax

    def forwards():
        outs = []
        for seqlens, seed in (([37, 50], 1), ([300], 2), ([5, 7, 9], 3)):          # per-kernel path
            x, pos, cu = _packed(seqlens, D, cuda_dev, seed)
            outs.append(core.forward(x, pos, cu, seqlens, save=False)[0])
        x, pos, cu = _packed([600, 500], D, cuda_dev, 4)                           # T >= 1024: gemm_rope / gemm_swiglu
        assert core._fused(x.shape[0], None)
        outs.append(core.forward(x, pos, cu, [600, 500], save=False)[0])
        x, pos, cu = _packed([40, 33], D, cuda_dev, 5)                             # pruned last layer
        rows = torch.tensor([39, 72, 10], dtype=torch.int32, device=cuda_dev)
        outs.append(core.forward(x, pos, cu, [40, 33], save=False, out_rows=rows)[0])
        for k in kc + vc:
            k.zero_()
        for cached, new, seed in (([0, 0], [30, 20], 6), ([30, 20], [9, 14], 7)):  # PrefixKVCache-style suffix steps
            x, pos, cu = _packed(new, D, cuda_dev, seed, cached)
            c = torch.tensor(cached, dtype=torch.int32, device=cuda_dev)
            kvl = c + torch.tensor(new, dtype=torch.int32, device=cuda_dev)
            outs.append(core.forward_suffix(x, pos, cu, new, kc, vc, c, start, kvl,
                                            out_rows=torch.tensor([0, sum(new) - 1], dtype=torch.int32, device=cuda_dev)))
        torch.cuda.synchronize()
        return [o.clone() for o in outs]

    spy = _Inputs(monkeypatch, core)
    with lm.int4_calibration() as cal:
        assert core.calibration is cal
        with pytest.raises(RuntimeError, match="already open"):
            with lm.int4_calibration():
                pass
        got = forwards()
    assert core.calibration is None and not cal.open
    assert cal.nbytes == d["n_layers"] * (3 * D * D + d["inter"] ** 2) * 4
    for (l, name), xs in spy.x.items():
        X = torch.cat(xs).double()
        ref = X.T @ X
        bound = 1e-5 * (X.abs().T @ X.abs()) + 1e-30
        assert cal.rows[(l, name)] == X.shape[0], (l, name)
        assert bool(((cal.h[(l, name)].double() - ref).abs() <= bound).all()), (l, name)
    assert len(spy.x) == 4 * d["n_layers"]
    assert cal.rows[(d["n_layers"] - 1, "o_proj")] < cal.rows[(d["n_layers"] - 1, "qkv")]   # the pruned layer's rows
    monkeypatch.setattr(llama.LlamaCore, "LAYER_CALL", False)
    ref = forwards()
    for a, b in zip(got, ref):
        assert torch.equal(_bits(a), _bits(b))


# ---------------------------------------------------------------------------------------------------------------------
# end to end on the small model: calibrate, quantize, decode
# ---------------------------------------------------------------------------------------------------------------------
def _calibrate(model, d, dev, steps=3):
    from tests.test_prefix_reuse_gpu import _nav_batch
    g = torch.Generator().manual_seed(21)
    to_dev = lambda b: {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in b.items()}
    instr = ["walk past the sofa and stop at the door of the kitchen", "leave the room and turn left at the stairs"]
    hist = [[], []]
    with model.int4_calibration() as cal:
        with torch.no_grad():
            for step in range(steps):
                batch = _nav_batch(d, step, hist, g, instr)
                batch["hist_vis"] = [[v.to(dev) for v in vs] for vs in batch["hist_vis"]]
                model("navigation", to_dev(batch))
                for b in range(2):
                    hist[b].append(torch.randn(d["hidden"], generator=g))
            tok = model.lang_model.tokenizer
            t = tok([f"Question w{i} w{i + 1} w{i + 7} about the room Answer" for i in range(8)])
            model.lang_model.generate(input_ids=t["input_ids"], attention_mask=t["attention_mask"], max_new_tokens=2,
                                      stop_on_eos=False)
    return cal


def test_gptq_end_to_end_beats_rtn_and_decodes_like_bf16_on_its_weights(cuda_dev, small, monkeypatch):
    from navillm_b200 import ops
    from tests.test_int4_midm_gpu import _Spy as MidSpy
    from tests.test_int4_weights_gpu import _Spy as SkinnySpy
    model, d = small
    lm = model.lang_model
    linears = lm.int4_linear_weights()
    W0 = [p.detach().clone() for p in linears]
    cal = _calibrate(model, d, cuda_dev)
    assert all(n > 0 for n in cal.rows.values())
    rows_before = dict(cal.rows)
    nbytes = model.quantize_weights_int4(calibration=cal)
    assert lm.int4_weights is not None and nbytes == lm.int4_weights.nbytes
    assert cal.rows == rows_before
    for p, w0 in zip(linears, W0):
        key = cal.input_of(p.data)
        H = cal.h[key].double()
        w_rtn = w0.clone()
        ops.quantize_int4_(w_rtn, *_copy_bufs(*w0.shape, cuda_dev))
        loss = lambda wq: float((((w0.double() - wq.double()) @ H) * (w0.double() - wq.double())).sum())
        assert loss(p.data) < loss(w_rtn), (key, loss(p.data), loss(w_rtn))
    del cal

    tok = lm.tokenizer
    prompts = lambda B: tok([f"Question w{i} w{3 * i + 1} w{i + 5} Answer" for i in range(B)])
    cases = {"b8_eager": (8, False), "b8_graph": (8, True), "b20_eager": (20, False), "b20_graph": (20, True)}

    def run_all(skinny=None, mid=None):
        out = {}
        for k, (B, graph) in cases.items():
            t = prompts(B)
            n0, m0 = (len(skinny.rows), len(mid.rows)) if skinny else (0, 0)
            out[k] = lm.generate(input_ids=t["input_ids"], attention_mask=t["attention_mask"], max_new_tokens=8,
                                 stop_on_eos=False, use_cuda_graph=graph).cpu()
            if skinny is not None:
                ran = skinny.rows[n0:] if B <= 16 else mid.rows[m0:]
                assert ran and B in ran, (k, ran[:4])
        return out

    skinny, mid = SkinnySpy(monkeypatch, ops), MidSpy(monkeypatch)
    with_copy = run_all(skinny, mid)
    lm.drop_int4_weights()
    without = run_all()
    for k in cases:
        assert torch.equal(with_copy[k], without[k]), k


def test_calibration_refusals(cuda_dev, small):
    from navillm_b200 import ops
    model, d = small
    lm = model.lang_model
    flat_before = lm.flat.flat.clone()
    with model.int4_calibration() as cal:
        with pytest.raises(RuntimeError, match="still open"):
            model.quantize_weights_int4(calibration=cal)
    with pytest.raises(RuntimeError, match="no rows were recorded for layer 0's qkv input"):
        model.quantize_weights_int4(calibration=cal)
    cal = _calibrate(model, d, cuda_dev, steps=1)
    # a failing factorisation names its layer and input and writes no weight
    h = cal.h[(1, "o_proj")]
    saved = h.clone()
    h.copy_(-torch.eye(h.shape[0], device=cuda_dev))
    with pytest.raises(ops.CholeskyError, match="layer 1's o_proj input Hessian.*larger damp"):
        model.quantize_weights_int4(calibration=cal)
    assert torch.equal(lm.flat.flat.view(torch.int16), flat_before.view(torch.int16)) and lm.int4_weights is None
    h.copy_(saved)
    # weights written since the calibration was opened
    with torch.no_grad():
        lm.model.layers[0].mlp.down_proj.weight.mul_(1.0)
    with pytest.raises(RuntimeError, match="calibration is stale.*modified in place"):
        model.quantize_weights_int4(calibration=cal)
    cal = _calibrate(model, d, cuda_dev, steps=1)
    model.quantize_weights_int4(calibration=cal)
    with pytest.raises(RuntimeError, match="calibration is stale.*optimizer step"):       # the quantization wrote them
        model.quantize_weights_int4(calibration=cal)
    lm.drop_int4_weights()
