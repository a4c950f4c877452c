"""Opt-in 4-bit group-wise weight streaming (W4A16) of the decode step (ModifiedLlamaForCausalLM.quantize_weights_int4).

The contract is exact: the quantizer rounds W to W' = bf16((q - z) * s) by the rule of tests/test_int4_quant_cpu.py, and
the int4 skinny GEMMs return bit for bit what the bf16 skinny GEMMs return on W'.  So every check here is bitwise."""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from tests.test_int4_quant_cpu import edge_groups, ref_int4  # noqa: E402

bf16 = torch.bfloat16


def _quantize_dev(W_cpu, dev):
    from navillm_b200 import ops
    N, K = W_cpu.shape
    w = W_cpu.to(dev)
    codes = torch.zeros(ops.int4_codes_shape(N, K), dtype=torch.uint8, device=dev)
    scales = torch.empty((N, K // 128), dtype=bf16, device=dev)
    zeros = torch.empty((N, K // 128), dtype=torch.uint8, device=dev)
    ops.quantize_int4_(w, codes, scales, zeros)
    return w, codes, scales, zeros


def _edge_rows(K):
    """One row per edge group, the group repeated along K, plus a row cycling through all of them."""
    groups = edge_groups()
    rows = [v.repeat(K // 128) for v in groups.values()]
    names = list(groups)
    rows.append(torch.cat([groups[names[i % len(names)]] for i in range(K // 128)]))
    return torch.stack(rows)


@pytest.mark.parametrize("K", [4096, 11008])
def test_quantizer_matches_cpu_rule_bitwise(cuda_dev, K):
    g = torch.Generator().manual_seed(K)
    W = torch.cat([torch.randn(64, K, generator=g) * 0.02, _edge_rows(K)]).to(bf16)    # 74 rows: a partial 64-row block
    rq, rs, rz, rw = ref_int4(W)
    w, codes, scales, zeros = _quantize_dev(W, cuda_dev)
    torch.cuda.synchronize()
    assert torch.equal(w.cpu().view(torch.int16), rw.view(torch.int16))        # bits, so -0 vs +0 counts
    assert torch.equal(scales.cpu().view(torch.int16), rs.view(torch.int16))
    assert torch.equal(zeros.cpu(), rz)
    # the codes are private to the kernels: the GEMM on them must reproduce the bf16 GEMM on W' for these rows too
    from navillm_b200 import ops
    x = torch.randn(5, K, generator=g).to(bf16).to(cuda_dev)
    assert torch.equal(ops.gemm_skinny_int4(x, codes, scales, zeros).view(torch.int16), ops.gemm_skinny(x, w).view(torch.int16))


def _expected_splits(N_tiles, K, sm):
    splits, kb = 1, (K + 63) // 64
    while splits < 8 and N_tiles * splits * 2 <= 3 * sm and kb // (splits * 2) >= 8:
        splits *= 2
    return splits


# (N, K, kind) and the cluster split the device rule picks on a 132-SM H100: qkv 4, o_proj 8, gate|up 2, down 8,
# 32000 x 4096 1 (250 tiles), the tail shape 1000 x 384 1 (6 k-blocks; its last tile is partial)
SHAPES = [(12288, 4096, "plain"), (4096, 4096, "plain"), (11008, 4096, "swiglu"), (4096, 11008, "plain"),
          (32000, 4096, "plain"), (1000, 384, "plain")]


def test_int4_skinny_gemms_equal_bf16_on_quantized_weights(cuda_dev):
    from navillm_b200 import _lib, ops
    sm = _lib.load().nv_sm_count()
    g = torch.Generator().manual_seed(7)
    seen = set()
    for N, K, kind in SHAPES:
        rows = 2 * N if kind == "swiglu" else N
        W = (torch.randn(rows, K, generator=g) * 0.02).to(bf16)
        W[3, :128] = 0.0                                                  # an all-zero group
        w, codes, scales, zeros = _quantize_dev(W, cuda_dev)
        if kind == "swiglu":
            seen.add(_expected_splits((N + 63) // 64, K, sm))
        else:
            seen.add(_expected_splits((N + 127) // 128, K, sm))
        for M in range(1, 17):
            x = torch.randn(M, K, generator=g).to(bf16).to(cuda_dev)
            if kind == "swiglu":
                ref = ops.gemm_skinny_swiglu(x, w)
                out = ops.gemm_skinny_swiglu_int4(x, codes, scales, zeros)
                assert torch.equal(out.view(torch.int16), ref.view(torch.int16)), (M, N, K, kind)
                continue
            add = torch.randn(M, N, generator=g).to(bf16).to(cuda_dev)
            for addend in (None, add):
                ref = ops.gemm_skinny(x, w, addend=addend)
                out = ops.gemm_skinny_int4(x, codes, scales, zeros, addend=addend)
                assert torch.equal(out.view(torch.int16), ref.view(torch.int16)), (M, N, K, addend is not None)
        del w, codes, scales, zeros
    if sm == 132:
        assert seen == {1, 2, 4, 8}, seen


def test_bad_arguments_are_refused_before_a_launch(cuda_dev):
    from navillm_b200 import _lib, ops
    from navillm_b200._lib import i32, i64, ptr, stream_ptr
    g = torch.Generator().manual_seed(3)
    N, K = 256, 512
    W = (torch.randn(N, K, generator=g) * 0.02).to(bf16)
    w, codes, scales, zeros = _quantize_dev(W, cuda_dev)
    x = torch.randn(4, K, generator=g).to(bf16).to(cuda_dev)
    out = torch.full((4, N), 3.0, dtype=bf16, device=cuda_dev)
    snap = lambda: [t.clone() for t in (w, codes, scales, zeros, out)]
    before = snap()

    bad = [
        lambda: ops.gemm_skinny_int4(torch.randn(17, K, device=cuda_dev).to(bf16), codes, scales, zeros),     # M > 16
        lambda: ops.gemm_skinny_int4(x.half(), codes, scales, zeros, out=out),                                 # x dtype
        lambda: ops.gemm_skinny_int4(x, codes.view(torch.int8), scales, zeros, out=out),                       # codes dtype
        lambda: ops.gemm_skinny_int4(x, codes, scales.float(), zeros, out=out),                                # scales dtype
        lambda: ops.gemm_skinny_int4(x, codes, scales, zeros.view(torch.int8), out=out),                       # zeros dtype
        lambda: ops.gemm_skinny_int4(x[:, :384], codes, scales, zeros, out=out),                               # K mismatch
        lambda: ops.gemm_skinny_swiglu_int4(x, codes[:96], scales[:96], zeros[:96]),                           # F % 64
        lambda: ops.quantize_int4_(w[:, :192], codes, scales, zeros),                                          # K % 128
        lambda: ops.quantize_int4_(w.float(), codes, scales, zeros),                                           # w dtype
    ]
    for f in bad:
        with pytest.raises(ValueError):
            f()
    # the C ABI refuses K % 128 != 0 and M > 16 itself (status, no launch)
    lib = _lib.load()
    assert lib.nv_gemm_skinny_int4(ptr(x), i64(K), ptr(codes), ptr(scales), ptr(zeros), ptr(out), i64(N), ptr(None), i64(0),
                                   i32(4), i32(N), i32(320), stream_ptr()) != 0
    assert lib.nv_gemm_skinny_int4(ptr(x), i64(K), ptr(codes), ptr(scales), ptr(zeros), ptr(out), i64(N), ptr(None), i64(0),
                                   i32(17), i32(N), i32(K), stream_ptr()) != 0
    assert lib.nv_gemm_skinny_swiglu_int4(ptr(x), i64(K), ptr(codes), ptr(scales), ptr(zeros), ptr(out), i64(N), i32(4),
                                          i32(96), i32(K), stream_ptr()) != 0
    assert lib.nv_quantize_int4_groups(ptr(w), i64(K), ptr(codes), ptr(scales), ptr(zeros), i32(N), i32(200), stream_ptr()) != 0
    torch.cuda.synchronize()
    for a, b in zip(before, snap()):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))


# ---------------------------------------------------------------------------------------------------------------------
# end to end: a 2-layer model at Vicuna-7B widths, C3-shaped prompts
# ---------------------------------------------------------------------------------------------------------------------
N_CAND = 256


def _prompts(tok, B, seed=5):
    rng = np.random.RandomState(seed)
    prompts = []
    for _ in range(B):
        words = " ".join(f"w{i}" for i in rng.randint(0, 5000, size=int(rng.randint(30, 61))))
        prompts.append("Scene " + " ".join(["<cand>"] * N_CAND) + " Question " + words + " Answer")
    return tok(prompts)


class _Spy:
    """Records the row count of every int4 GEMM call."""

    def __init__(self, monkeypatch, ops):
        self.rows = []
        for name in ("gemm_skinny_int4", "gemm_skinny_swiglu_int4"):
            f = getattr(ops, name)

            def wrap(x, *a, _f=f, **kw):
                self.rows.append(x.shape[0])
                return _f(x, *a, **kw)
            monkeypatch.setattr(ops, name, wrap)


def test_generate_int4_is_bitwise_bf16_on_quantized_weights(cuda_dev, monkeypatch):
    from navillm_b200 import ops
    from tests.test_fullwidth_parity_gpu import HID, _full_navmodel
    model, tok = _full_navmodel(cuda_dev, base_vocab=32000)
    lm = model.lang_model
    model._ensure()
    text8, text4, text32 = _prompts(tok, 8), _prompts(tok, 4, seed=6), _prompts(tok, 32, seed=7)
    cand = lambda B: torch.randn(B * N_CAND, HID, generator=torch.Generator().manual_seed(B)).to(cuda_dev)
    base = lambda t, B: dict(input_ids=t["input_ids"], attention_mask=t["attention_mask"], cand_vis=cand(B), stop_on_eos=False)
    cases = {
        "greedy_eager": dict(base(text8, 8), max_new_tokens=16, use_cuda_graph=False),
        "greedy_graph": dict(base(text8, 8), max_new_tokens=16, use_cuda_graph=True),
        "sampled": dict(base(text8, 8), max_new_tokens=16, do_sample=True, temperature=0.8, top_p=0.9),
        "beams4_b4": dict(base(text4, 4), max_new_tokens=8, num_beams=4),
        "samples4_b4": dict(base(text4, 4), max_new_tokens=8, do_sample=True, temperature=0.8, num_return_sequences=4),
        "b32": dict(base(text32, 32), max_new_tokens=8),
    }

    def run_all(spy=None):
        out = {}
        for kv in ("bf16", "fp8"):
            lm.set_kv_cache_dtype(kv)
            for k, kw in cases.items():
                if kv == "fp8" and k not in ("greedy_graph", "beams4_b4"):
                    continue
                n0 = len(spy.rows) if spy else 0
                torch.manual_seed(77)
                out[(k, kv)] = lm.generate(**kw).cpu()
                if spy is not None:
                    ran = spy.rows[n0:]
                    if k == "b32":
                        assert not ran, "32 rows must stay on the bf16 kernels"
                    else:
                        assert ran and max(ran) <= 16, (k, ran[:4])
        lm.set_kv_cache_dtype("bf16")
        return out

    W = lm.model.layers[0].self_attn.q_proj.weight.detach().clone()
    head = lm.lm_head.weight.detach().clone()
    nbytes = model.quantize_weights_int4()
    assert lm.int4_weights is not None and lm.fp8_weights is None
    ws = lm.int4_linear_weights()
    n = sum(p.numel() for p in ws)
    assert nbytes == n // 2 + 3 * (n // 128)
    # state_dict() holds W' (the CPU rule applied to W), and lm_head is not rounded
    sd = lm.state_dict()
    assert torch.equal(sd["model.layers.0.self_attn.q_proj.weight"].cpu().view(torch.int16), ref_int4(W.cpu())[3].view(torch.int16))
    assert torch.equal(sd["lm_head.weight"], head)
    spy = _Spy(monkeypatch, ops)
    with_int4 = run_all(spy)
    # the decode step itself, bitwise on its hidden output with and without the int4 copy
    core, d = lm.core, lm.dims
    kc = [torch.zeros((3, 64, d.hidden), dtype=bf16, device=cuda_dev) for _ in range(d.n_layers)]
    vc = [torch.zeros_like(k) for k in kc]
    lens = torch.tensor([5, 9, 1], dtype=torch.int32, device=cuda_dev)
    x = (torch.randn(3, d.hidden, generator=torch.Generator().manual_seed(2)) * 0.5).to(bf16).to(cuda_dev)
    h4 = core.decode_step(x, lens, kc, vc)
    lm.drop_int4_weights()
    assert lm.int4_weights is None and core.int4 is None
    h16 = core.decode_step(x, lens, [k.clone() for k in kc], [v.clone() for v in vc])
    assert torch.equal(h4.view(torch.int16), h16.view(torch.int16))
    n0 = len(spy.rows)
    without = run_all()
    assert len(spy.rows) == n0
    for k in with_int4:
        assert torch.equal(with_int4[k], without[k]), k


def test_int4_lifecycle(cuda_dev):
    from navillm_b200.modified_lm import PrefixKVCache
    from tests.test_fullwidth_parity_gpu import _full_navmodel
    model, tok = _full_navmodel(cuda_dev, base_vocab=32000)
    lm = model.lang_model
    model._ensure()
    text = _prompts(tok, 2)
    ids = text["input_ids"].clone()
    ids[ids == tok.special["<cand>"]] = 7
    gen = lambda: lm.generate(input_ids=ids, attention_mask=text["attention_mask"], max_new_tokens=4, stop_on_eos=False)
    cache = PrefixKVCache(lm, batch_size=2, max_len=512, train=True)
    cache.check_weights()

    model.quantize_weights_int4()
    with pytest.raises(RuntimeError, match="weights changed"):        # filled under W, the weights are now W'
        cache.check_weights()
    gen()
    with torch.no_grad():
        lm.model.layers[1].mlp.down_proj.weight.mul_(1.0)              # any write makes the copy stale
    with pytest.raises(RuntimeError, match="int4 copy of the weights is stale.*quantize_weights_int4"):
        gen()
    model.quantize_weights_int4()
    gen()

    # each format's quantizer drops the other copy; W' composes
    model.quantize_weights_fp8()
    assert lm.fp8_weights is not None and lm.int4_weights is None and lm.core.int4 is None
    gen()
    lm.set_activation_dtype("fp8")
    model.quantize_weights_int4()
    assert lm.int4_weights is not None and lm.fp8_weights is None
    with pytest.raises(RuntimeError, match="needs the fp8 copy"):     # W8A8 keeps needing the fp8 copy
        lm.generate(input_ids=ids, attention_mask=text["attention_mask"], max_new_tokens=2, stop_on_eos=False)
    lm.set_activation_dtype("bf16")
    gen()
    lm.drop_int4_weights()
    gen()
