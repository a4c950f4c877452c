"""Packed LLaMA stack (navillm_b200/llama.py: wgmma GEMMs + flash attention + row kernels, hand-written
backward) against the CPU oracle's restatement of HF LLaMA (oracle/navillm_oracle.py::llama_model).

"bf16 tolerance", stated: let `truth` be the oracle run in fp32 with the same (bf16-valued) weights.  The
reference itself, run in bf16 (oracle precision='amp_bf16'), deviates from truth by e_ref (pure bf16
rounding noise).  The CUDA path must satisfy  max|cuda - truth| <= 2 * e_ref + 1e-3 * max|truth|.
"""
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
bf16 = torch.bfloat16


def build(cuda_dev, hidden=256, heads=2, inter=256, layers=2, vocab=262):
    from oracle import navillm_oracle as O
    from navillm_b200 import llama
    cfg = O.OracleConfig(hidden=hidden, n_layers=layers, n_heads=heads, inter=inter, vocab=vocab, pano_hidden=64,
                         pano_heads=2, pano_inter=64, image_feat_size=32, obj_feat_size=32)
    sd = O.init_state_dict(cfg, seed=3)
    # non-trivial norm weights
    g = torch.Generator().manual_seed(5)
    for k in sd:
        if "layernorm" in k or k.endswith("model.norm.weight"):
            sd[k] = (1 + 0.1 * torch.randn(sd[k].shape, generator=g)).to(bf16)
    dims = llama.LlamaDims(hidden=hidden, n_layers=layers, n_heads=heads, inter=inter, vocab=vocab)
    model = llama.LlamaModelParams(dims)
    model.load_state_dict({k[len("lang_model.model."):]: v for k, v in sd.items() if k.startswith("lang_model.model.")})
    flat = llama.FlatParams(model.flat_order(), cuda_dev)
    core = llama.LlamaCore(dims, model, flat)
    return cfg, sd, dims, model, flat, core


def pack(emb, mask):
    B, S, D = emb.shape
    seqlens = mask.sum(1).tolist()
    rows = mask.flatten().nonzero().squeeze(1)
    pos = torch.arange(S).repeat(B, 1).flatten()[rows]          # plain forward: arange(S) incl. left padding
    cu = torch.tensor([0] + list(torch.tensor(seqlens).cumsum(0)), dtype=torch.int32)
    return rows, pos.to(torch.int32), cu, seqlens


def test_llama_stack_forward_backward(cuda_dev):
    from oracle import navillm_oracle as O
    from navillm_b200 import ops
    cfg, sd, dims, model, flat, core = build(cuda_dev)
    B, S, D = 3, 200, dims.hidden
    lens = [37, 200, 130]
    g = torch.Generator().manual_seed(11)
    emb = (torch.randn(B, S, D, generator=g) * 0.5).to(bf16)
    mask = torch.zeros(B, S, dtype=torch.long)
    for b, L in enumerate(lens):
        mask[b, S - L:] = 1                                     # left padding, like the reference tokenizer
    G = torch.randn(B, S, D, generator=g).to(bf16) * mask[..., None]

    def run_oracle(dtype):
        sdd = {k: v.to(dtype).requires_grad_(True) for k, v in sd.items() if k.startswith("lang_model.model.")}
        e = emb.to(dtype).requires_grad_(True)
        cfg2 = O.OracleConfig(**{**cfg.__dict__, "precision": "fp32" if dtype == torch.float32 else "amp_bf16"})
        h = O.llama_model(sdd, cfg2, e, mask)
        (h.float() * G.float()).sum().backward()
        return h.detach().float(), e.grad.float(), {k: v.grad.float() for k, v in sdd.items() if v.grad is not None}

    h_truth, de_truth, gw_truth = run_oracle(torch.float32)
    h_ref, de_ref, gw_ref = run_oracle(bf16)

    rows, pos, cu, seqlens = pack(emb, mask)
    x = emb.view(B * S, D)[rows].to(cuda_dev).contiguous()
    hid, tape = core.forward(x, pos.to(cuda_dev), cu.to(cuda_dev), seqlens)
    hn, rstd = ops.rmsnorm_fwd(hid, model.norm.weight.data, dims.rms_eps)
    dy = G.view(B * S, D)[rows].to(cuda_dev).contiguous()
    dhid = ops.rmsnorm_bwd(hid, model.norm.weight.data, rstd, dy, dw=model.norm.weight.grad)
    dx = core.backward(dhid, tape)
    torch.cuda.synchronize()

    def check(name, mine, truth, ref):
        e_ref = (ref - truth).abs().max().item()
        e_mine = (mine - truth).abs().max().item()
        lim = 2 * e_ref + 1e-3 * truth.abs().max().item()
        assert e_mine <= lim, f"{name}: cuda err {e_mine:.4g} > 2*ref err {e_ref:.4g} (+1e-3*{truth.abs().max().item():.3g})"

    m = mask.bool().flatten()
    check("hidden", hn.float().cpu(), h_truth.view(B * S, D)[m], h_ref.view(B * S, D)[m])
    check("d_embeds", dx.float().cpu(), de_truth.view(B * S, D)[m], de_ref.view(B * S, D)[m])
    named = dict(model.named_parameters())
    for k in ("layers.0.self_attn.q_proj.weight", "layers.0.self_attn.v_proj.weight", "layers.1.self_attn.o_proj.weight",
              "layers.0.mlp.gate_proj.weight", "layers.1.mlp.up_proj.weight", "layers.1.mlp.down_proj.weight",
              "layers.0.input_layernorm.weight", "layers.1.post_attention_layernorm.weight", "norm.weight"):
        check(k, named[k].grad.float().cpu(), gw_truth["lang_model.model." + k], gw_ref["lang_model.model." + k])


def test_layer_call_inference_forward_is_bit_identical(cuda_dev):
    """The one-call-per-layer inference forward (nv_llama_layer_infer, csrc/layer.cu) launches the same kernels as the
    per-kernel path: residual stream bit-identical, with and without last-layer row pruning and with the K/V store of a
    generate() prefill."""
    cfg, sd, dims, model, flat, core = build(cuda_dev)
    B, S, D = 3, 200, dims.hidden
    lens = [37, 200, 130]
    g = torch.Generator().manual_seed(12)
    emb = (torch.randn(B, S, D, generator=g) * 0.5).to(bf16)
    mask = torch.zeros(B, S, dtype=torch.long)
    for b, L in enumerate(lens):
        mask[b, S - L:] = 1
    rows, pos, cu, seqlens = pack(emb, mask)
    x = emb.view(B * S, D)[rows].to(cuda_dev).contiguous()
    pos, cu = pos.to(cuda_dev), cu.to(cuda_dev)
    out_rows = torch.tensor([36, 236, 366], dtype=torch.int32, device=cuda_dev)          # last row of every sequence
    Smax = 256
    results = {}
    for mode in (True, False):
        core.LAYER_CALL = mode
        kc = [torch.zeros((B, Smax, D), dtype=bf16, device=cuda_dev) for _ in range(dims.n_layers)]
        vc = [torch.zeros((B, Smax, D), dtype=bf16, device=cuda_dev) for _ in range(dims.n_layers)]
        full, tape = core.forward(x, pos, cu, seqlens, save=False)
        pruned, _ = core.forward(x, pos, cu, seqlens, save=False, out_rows=out_rows, kv_store=(kc, vc))
        torch.cuda.synchronize()
        assert tape is None
        results[mode] = (full.clone(), pruned.clone(), [k.clone() for k in kc], [v.clone() for v in vc])
    core.LAYER_CALL = type(core).LAYER_CALL
    a, b = results[True], results[False]
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert torch.equal(a[1], a[0][out_rows.long()])                    # pruning = row selection of the full forward
    for l in range(dims.n_layers):
        assert torch.equal(a[2][l], b[2][l]) and torch.equal(a[3][l], b[3][l])
