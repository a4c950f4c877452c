"""Opt-in fp8 (e4m3) weight streaming of the decode step (ModifiedLlamaForCausalLM.quantize_weights_fp8).

The contract is exact: the quantizer rounds W to W' = e4m3(W / 2^e_n) * 2^e_n (one power-of-two exponent per row), which
bf16 holds exactly, and the fp8 skinny GEMMs must return bit for bit what the bf16 skinny GEMMs return on W'.  So every
check here is bitwise, against a CPU reference quantizer or against the bf16 path on the same W'."""
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

bf16, fp8 = torch.bfloat16, torch.float8_e4m3fn


def ref_quantize(W: torch.Tensor):
    """CPU reference: (e4m3 values, int8 exponents, W') of a bf16 weight [N, K]."""
    Wf = W.float()
    amax = Wf.abs().amax(dim=1)
    m, x = torch.frexp(amax)
    e = torch.where(m <= 0.875, x - 9, x - 8)
    e = torch.where(amax == 0, torch.zeros_like(e), e).clamp(min=-117)
    s = torch.exp2(e.float())[:, None]
    q = (Wf / s).to(fp8)
    return q, e.to(torch.int8), (q.float() * s).to(bf16)


def edge_rows(K: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(3)
    rows = []
    rows.append(torch.zeros(K))                                            # all-zero row: e = 0
    r = torch.randn(K, generator=g) * 0.01
    r[5] = 448 * 2.0 ** -10                                                # amax exactly 448 * 2^k: scaled max is 448
    rows.append(r)
    r = torch.randn(K, generator=g) * 0.01
    r[7] = -448 * 2.0 ** -3
    rows.append(r)
    # amax 1.0 (e = -8, scale 256): flush to zero, e4m3 subnormals, exact ties, negative zeros
    r = torch.zeros(K)
    r[0] = 1.0
    vals = [2.0 ** -18, 3 * 2.0 ** -18, 2.0 ** -17, 5 * 2.0 ** -19, 2.0 ** -20, 7 * 2.0 ** -17,   # -> 0, 2^-8, subnormals
            1.0625 / 256, 1.1875 / 256, 2.5 / 256, 9.0 / 256, 17.0 / 256, 0.0 / 256]             # ties to even
    for i, v in enumerate(vals):
        r[1 + 2 * i], r[2 + 2 * i] = v, -v
    r[40:60] = -0.0
    rows.append(r)
    r = torch.full((K,), -0.0)                                             # all negative zeros
    rows.append(r)
    r = torch.randn(K, generator=g) * 0.02
    r[9] = 0.96875 * 2.0 ** -4                                             # mantissa above 0.875: e = x - 8
    rows.append(r)
    r = torch.randn(K, generator=g) * 0.02
    r[11] = 0.875 * 2.0 ** -4 + 2.0 ** -12                                 # just above 448 * 2^k
    rows.append(r)
    return torch.stack(rows).to(bf16)


def _quantize_dev(W_cpu, dev):
    from navillm_b200 import ops
    w = W_cpu.to(dev)
    q = torch.empty(W_cpu.shape, dtype=fp8, device=dev)
    e = torch.empty(W_cpu.shape[0], dtype=torch.int8, device=dev)
    ops.quantize_fp8_(w, q, e)
    return w, q, e


@pytest.mark.parametrize("K", [4096, 11008])
def test_quantizer_matches_cpu_reference_bitwise(cuda_dev, K):
    g = torch.Generator().manual_seed(K)
    W = torch.cat([(torch.randn(64, K, generator=g) * 0.02).to(bf16), edge_rows(K)])
    rq, re_, rw = ref_quantize(W)
    assert int(re_[64]) == 0 and int(re_[65]) == -10 and int(re_[67]) == -8  # the hand-built rows exercise what they claim
    w, q, e = _quantize_dev(W, cuda_dev)
    assert torch.equal(e.cpu(), re_)
    assert torch.equal(q.cpu().view(torch.uint8), rq.view(torch.uint8))
    assert torch.equal(w.cpu().view(torch.int16), rw.view(torch.int16))        # bits, so -0 vs +0 counts
    assert torch.equal(rw.float(), rq.float() * torch.exp2(re_.float())[:, None])   # W' is exactly e4m3 * 2^e


def _expected_splits(N_tiles, K, sm):
    splits, kb = 1, (K + 63) // 64
    while splits < 8 and N_tiles * splits * 2 <= 3 * sm and kb // (splits * 2) >= 8:
        splits *= 2
    return splits


# (N, K, kind): the decode shapes of a Vicuna-7B layer and lm_head; the cluster split each one takes on a 132-SM H100 is
# asserted below so that all four split sizes are covered
SHAPES = [(12288, 4096, "plain"), (4096, 4096, "addend"), (11008, 4096, "swiglu"), (4096, 11008, "addend"), (32006, 4096, "plain")]


@pytest.mark.parametrize("M", [1, 3, 8, 16])
def test_fp8_skinny_gemm_equals_bf16_on_quantized_weights(cuda_dev, M):
    from navillm_b200 import _lib, ops
    sm = _lib.load().nv_sm_count()
    g = torch.Generator().manual_seed(M)
    seen = set()
    for N, K, kind in SHAPES:
        rows = 2 * N if kind == "swiglu" else N
        W = (torch.randn(rows, K, generator=g) * 0.02).to(bf16)
        w, q, e = _quantize_dev(W, cuda_dev)
        x = (torch.randn(M, K, generator=g)).to(bf16).to(cuda_dev)
        if kind == "swiglu":
            seen.add(_expected_splits((N + 63) // 64, K, sm))
            ref = ops.gemm_skinny_swiglu(x, w)
            out = ops.gemm_skinny_swiglu_fp8(x, q, e)
        else:
            seen.add(_expected_splits((N + 127) // 128, K, sm))
            add = (torch.randn(M, N, generator=g)).to(bf16).to(cuda_dev) if kind == "addend" else None
            ref = ops.gemm_skinny(x, w, addend=add)
            out = ops.gemm_skinny_fp8(x, q, e, addend=add)
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int16), ref.view(torch.int16)), (M, N, K, kind)
    if sm == 132:
        assert seen == {1, 2, 4, 8}, seen


# ---------------------------------------------------------------------------------------------------------------------
# the model level: tiny golden model
# ---------------------------------------------------------------------------------------------------------------------
def _golden_model(dev):
    from tests.test_navmodel_gpu import build_model
    from tests.test_oracle_golden import load
    g, cfg, tok = load("amp_bf16")
    model, _ = build_model(g, dev)
    return g, cfg, tok, model


def _cand(g, cfg, O):
    qa = g["qa_in"]
    sd = g["state_dict"]
    feats = qa["features"]
    lens = torch.tensor([f.shape[0] for f in feats])
    view = torch.stack([torch.cat([f, f.new_zeros(int(lens.max()) - f.shape[0], f.shape[1])], 0) for f in feats], 0)
    pano = O.forward_panorama(sd, cfg, view, lens)
    pe = pano["pano_embeds"] + O._pos_embed(torch.zeros(pano["pano_embeds"].shape[:2] + (14,)), sd, "vp_pos_embeddings")
    pe = pe + sd["token_type_embeddings.weight"][0]
    return pe[pano["pano_masks"]]


class _Count:
    def __init__(self, monkeypatch, ops):
        self.n = 0
        for name in ("gemm_skinny_fp8", "gemm_skinny_swiglu_fp8"):
            f = getattr(ops, name)

            def wrap(*a, _f=f, **kw):
                self.n += 1
                return _f(*a, **kw)
            monkeypatch.setattr(ops, name, wrap)


def test_generate_fp8_is_bitwise_bf16_on_quantized_weights(cuda_dev, monkeypatch):
    from navillm_b200 import ops
    from tests.test_generate_gpu import _Trie
    g, cfg, tok, model = _golden_model(cuda_dev)
    lm = model.lang_model
    text = tok(g["qa_in"]["prompts"])
    ids_in, mask = text["input_ids"], text["attention_mask"]
    ids_plain = ids_in.clone()
    ids_plain[ids_plain == tok.special["<cand>"]] = 7
    trie = _Trie(tok.bos_token_id, tok.eos_token_id)
    for w in ([11, 12, 13], [11, 12, 40, 41], [11, 50], [60, 61, 62]):
        trie.insert(w)
    cases = {
        "greedy_eager": dict(input_ids=ids_plain, attention_mask=mask, max_new_tokens=12, stop_on_eos=False, use_cuda_graph=False),
        "greedy_graph": dict(input_ids=ids_plain, attention_mask=mask, max_new_tokens=12, stop_on_eos=False, use_cuda_graph=True),
        "sampled": dict(input_ids=ids_plain, attention_mask=mask, max_new_tokens=12, stop_on_eos=False, do_sample=True,
                        temperature=0.7),
        "trie": dict(input_ids=ids_plain, attention_mask=mask, max_new_tokens=6, trie=trie, eos_token_id=tok.eos_token_id,
                     pad_token_id=tok.unk_token_id),
        "b20": dict(input_ids=ids_plain.repeat(10, 1), attention_mask=mask.repeat(10, 1), max_new_tokens=8, stop_on_eos=False),
    }

    def run_all():
        out = {}
        for k, kw in cases.items():
            torch.manual_seed(77)
            out[k] = lm.generate(**kw).cpu()
        return out

    nbytes = model.quantize_weights_fp8()
    assert nbytes > 0 and lm.fp8_weights is not None
    cnt = _Count(monkeypatch, ops)
    with_fp8 = {}
    for k, kw in cases.items():
        n0 = cnt.n
        torch.manual_seed(77)
        with_fp8[k] = lm.generate(**kw).cpu()
        if k == "b20":
            assert cnt.n == n0, "B > 16 must stay on the bf16 kernels"
        else:
            assert cnt.n > n0, f"{k}: the fp8 kernels did not run"
    # also the decode step itself, bitwise on its hidden output (the logits' input) with and without the fp8 copy
    core, d = lm.core, lm.dims
    Smax = 64
    kc = [torch.zeros((3, Smax, d.hidden), dtype=bf16, device=cuda_dev) for _ in range(d.n_layers)]
    vc = [torch.zeros_like(k) for k in kc]
    lens = torch.tensor([5, 9, 1], dtype=torch.int32, device=cuda_dev)
    x = (torch.randn(3, d.hidden, generator=torch.Generator().manual_seed(2)) * 0.5).to(bf16).to(cuda_dev)
    h8 = core.decode_step(x, lens, kc, vc)
    fp8_copy = core.fp8
    lm.drop_fp8_weights()
    assert lm.fp8_weights is None and core.fp8 is None
    h16 = core.decode_step(x, lens, [k.clone() for k in kc], [v.clone() for v in vc])
    assert torch.equal(h8.view(torch.int16), h16.view(torch.int16))
    del fp8_copy
    n0 = cnt.n
    without = run_all()
    assert cnt.n == n0
    for k in cases:
        assert torch.equal(with_fp8[k], without[k]), k


def test_fp8_generate_vs_oracle_on_quantized_state_dict(cuda_dev):
    from oracle import navillm_oracle as O
    from tests.test_fullwidth_parity_gpu import compare_greedy_rows
    g, cfg, tok, model = _golden_model(cuda_dev)
    model.quantize_weights_fp8()
    sd = dict(g["state_dict"])
    sd.update({k: v.detach().cpu() for k, v in model.state_dict().items() if k.startswith("lang_model.")})
    changed = sum(not torch.equal(sd[k], g["state_dict"][k]) for k in sd if k.startswith("lang_model."))
    assert changed > 0                                                     # the state dict holds W', not W
    cand = _cand(g, cfg, O)
    text = tok(g["qa_in"]["prompts"])
    n_new = 12
    ref_ids, ref_logits = O.greedy_generate(sd, cfg, text["input_ids"], text["attention_mask"], cand_vis=cand,
                                            max_new_tokens=n_new, stop_on_eos=False, return_logits=True)
    S0 = text["input_ids"].shape[1]
    for graph in (False, True):
        ids = model.lang_model.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"],
                                        cand_vis=cand.to(cuda_dev), max_new_tokens=n_new, stop_on_eos=False,
                                        use_cuda_graph=graph).cpu()
        assert ids.shape == ref_ids.shape
        matched, cut = compare_greedy_rows(ids, ref_ids, ref_logits, S0, n_new, tag=f"fp8 graph={graph}")
        assert sum(matched) >= ids.shape[0] * n_new // 2, matched


def test_fp8_generate_c3_shape_fullwidth_vs_oracle(cuda_dev):
    import numpy as np
    from oracle import navillm_oracle as O
    from tests.test_fullwidth_parity_gpu import HID, _full_navmodel, _oracle_cfg, compare_greedy_rows
    B, N_CAND, N_NEW = 8, 256, 16
    model, tok = _full_navmodel(cuda_dev, base_vocab=32000)
    model.quantize_weights_fp8()
    sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items() if k.startswith("lang_model.")}
    rng = np.random.RandomState(5)
    prompts = []
    for b in range(B):
        words = " ".join(f"w{i}" for i in rng.randint(0, 5000, size=int(rng.randint(30, 61))))
        prompts.append("Scene " + " ".join(["<cand>"] * N_CAND) + " Question " + words + " Answer")
    text = tok(prompts)
    cand = torch.randn(B * N_CAND, HID, generator=torch.Generator().manual_seed(9))
    ref_ids, ref_logits = O.greedy_generate(sd, _oracle_cfg(tok, "amp_bf16"), text["input_ids"], text["attention_mask"],
                                            cand_vis=cand, max_new_tokens=N_NEW, stop_on_eos=False, return_logits=True)
    S0 = text["input_ids"].shape[1]
    ids = model.lang_model.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev),
                                    max_new_tokens=N_NEW, stop_on_eos=False).cpu()
    matched, cut = compare_greedy_rows(ids, ref_ids, ref_logits, S0, N_NEW, tag="fp8 c3")
    print(f"\n[fp8 c3 generate] matched tokens per row {matched} of {N_NEW}; near-tie cuts {cut}")
    assert sum(matched) >= B * N_NEW // 4, matched


def test_fp8_copy_goes_stale_after_weight_writes(cuda_dev):
    from navillm_b200.optim import FlatAdamW
    g, cfg, tok, model = _golden_model(cuda_dev)
    lm = model.lang_model
    text = tok(g["qa_in"]["prompts"])
    ids = text["input_ids"].clone()
    ids[ids == tok.special["<cand>"]] = 7
    gen = lambda: lm.generate(input_ids=ids, attention_mask=text["attention_mask"], max_new_tokens=4, stop_on_eos=False)
    model.quantize_weights_fp8()
    gen()
    saved = {k: v.clone() for k, v in lm.state_dict().items()}

    opt = torch.optim.AdamW([p for p in lm.parameters() if p.requires_grad], lr=1e-3)
    lm._ensure()
    opt.step()
    with pytest.raises(RuntimeError, match="stale"):
        gen()
    model.quantize_weights_fp8()
    gen()

    FlatAdamW(model, lr=1e-3).step()
    with pytest.raises(RuntimeError, match="stale"):
        gen()
    model.quantize_weights_fp8()
    gen()

    lm.load_state_dict(saved, strict=False)
    with pytest.raises(RuntimeError, match="stale"):
        gen()
    model.quantize_weights_fp8()
    gen()
    lm.drop_fp8_weights()
    gen()


def test_fp8_copy_size_and_release(cuda_dev):
    g, cfg, tok, model = _golden_model(cuda_dev)
    lm = model.lang_model
    model._ensure()                                                        # both flat buffers exist before the baseline
    ws = lm.fp8_linear_weights()
    n = sum(p.numel() for p in ws)
    rows = sum(p.shape[0] for p in ws)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    nbytes = model.quantize_weights_fp8()
    assert n + rows <= nbytes <= n + rows + 64 * len(ws)
    torch.cuda.synchronize()
    held = torch.cuda.memory_allocated() - before
    assert nbytes <= held <= nbytes + 4096
    lm.drop_fp8_weights()
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == before


def test_navigation_after_quantization_equals_a_model_loaded_with_quantized_weights(cuda_dev):
    from tests.test_navmodel_gpu import build_model, to_dev
    g, cfg, tok, model = _golden_model(cuda_dev)
    model.quantize_weights_fp8()
    other, _ = build_model(g, cuda_dev)
    other.load_state_dict({k: v.detach().clone() for k, v in model.state_dict().items()})
    outs = []
    with torch.no_grad():
        for m in (model, other):
            pano = m("panorama", to_dev(dict(g["pano_in"]), cuda_dev))
            nav_in = to_dev(dict(g["nav_in"]), cuda_dev)
            B = pano["pano_embeds"].shape[0]
            nav_in["vp_img_embeds"] = torch.cat([torch.zeros_like(pano["pano_embeds"][:, :1]), pano["pano_embeds"]], 1)
            nav_in["pano_masks"] = torch.cat([torch.ones(B, 1, dtype=torch.bool, device=cuda_dev), pano["pano_masks"]], 1)
            torch.manual_seed(1234)
            outs.append(m("navigation", nav_in)["fuse_logits"].float().cpu())
    assert torch.equal(outs[0], outs[1])
    untouched = [k for k in g["state_dict"] if not k.startswith("lang_model.") or "norm" in k or "embed_tokens" in k]
    sd = model.state_dict()
    for k in untouched:
        assert torch.equal(sd[k].cpu(), g["state_dict"][k]), f"{k} must not be quantized"
