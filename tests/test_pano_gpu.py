"""Panorama encoder on the fp32 kernels (navillm_b200/image_embedding.py) vs the CPU oracle restatement of
the reference's ImageEmbeddings (oracle.forward_panorama), forward and parameter gradients.

Two numerical modes (ops.set_pano_precision):
  fp32  exact CUDA-core GEMMs: both sides fp32, only summation order differs -> 1e-4 (forward) / 2e-4 (gradients)
        relative to the tensor's max.
  tf32  wgmma tf32 GEMMs (the product default; what the reference's pinned torch 1.10 did on Ampere+ with its
        default allow_tf32 = True): operands carry a 10-bit mantissa (unit roundoff 2^-10 under truncation), errors
        accumulate over 2 encoder layers + projections -> 4e-3 (forward) / 1e-2 (gradients) relative to the max.
"""
import sys
import types
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def rel_err(a, b):
    return (a - b).abs().max().item() / (b.abs().max().item() + 1e-12)


@pytest.mark.parametrize("B,N,lens,with_obj", [(2, 12, [12, 9], True), (3, 36, [36, 36, 36], False), (2, 70, [70, 33], False)])
def test_pano_encoder_matches_oracle(cuda_dev, B, N, lens, with_obj, pano_precision):
    precision = pano_precision
    from oracle import navillm_oracle as O
    from navillm_b200.image_embedding import ImageEmbeddings
    tol_f, tol_g = (1e-4, 2e-4) if precision == "fp32" else (4e-3, 1e-2)
    cfg = O.OracleConfig(hidden=256, n_layers=1, n_heads=2, inter=256, vocab=70, image_feat_size=72, obj_feat_size=40,
                         pano_hidden=128, pano_heads=2, pano_inter=256, num_pano_layers=2)
    sd = O.init_state_dict(cfg, seed=1)
    vis_cfg = types.SimpleNamespace(hidden_size=128, num_attention_heads=2, intermediate_size=256, hidden_dropout_prob=0.1,
                                    image_feat_size=72, angle_feat_size=4, obj_feat_size=40, output_size=256, num_pano_layers=2)
    mod = ImageEmbeddings(vis_cfg, use_obj=True).eval()
    mod.load_state_dict({k[len("img_embeddings."):]: v for k, v in sd.items() if k.startswith("img_embeddings.")})
    mod = mod.to(cuda_dev)
    g = torch.Generator().manual_seed(B * 100 + N)
    view = torch.randn(B, N, 72, generator=g)
    loc = torch.randn(B, N, 7, generator=g)
    types_ = torch.randint(0, 2, (B, N), generator=g)
    lens_t = torch.tensor(lens)
    kw = {}
    if with_obj:
        kw = dict(obj_img_fts=torch.randn(B, 5, 40, generator=g), obj_lens=torch.tensor([5, 3][:B]),
                  obj_loc_fts=torch.randn(B, 5, 7, generator=g))
    # oracle with autograd
    sda = {k: v.clone().requires_grad_(True) for k, v in sd.items() if k.startswith("img_embeddings.")}
    ref = O.forward_panorama(sda, cfg, view, lens_t, loc, types_, **kw)
    Gp = torch.randn(ref["pano_embeds"].shape, generator=g)
    loss = (ref["pano_embeds"] * Gp).sum()
    if with_obj:
        Go = torch.randn(ref["obj_embeds"].shape, generator=g)
        loss = loss + (ref["obj_embeds"] * Go).sum()
    loss.backward()
    # CUDA
    out = mod.forward_panorama_per_step(view.to(cuda_dev), lens_t.to(cuda_dev), loc.to(cuda_dev), types_.to(cuda_dev),
                                        **{k: v.to(cuda_dev) for k, v in kw.items()})
    assert rel_err(out["pano_embeds"].detach().cpu(), ref["pano_embeds"].detach()) < tol_f
    assert torch.equal(out["pano_masks"].cpu(), ref["pano_masks"])
    l2 = (out["pano_embeds"] * Gp.to(cuda_dev)).sum()
    if with_obj:
        assert rel_err(out["obj_embeds"].detach().cpu(), ref["obj_embeds"].detach()) < tol_f
        l2 = l2 + (out["obj_embeds"] * Go.to(cuda_dev)).sum()
    l2.backward()
    torch.cuda.synchronize()
    for name, p in mod.named_parameters():
        r = sda["img_embeddings." + name].grad
        if r is None:
            continue
        assert p.grad is not None, name
        assert rel_err(p.grad.cpu(), r) < tol_g, f"{name}: {rel_err(p.grad.cpu(), r)}"


# ---------------------------------------------------------------------------------------------------------
# train-mode dropout (models/image_embedding.py:72, models/detr_transformer.py:136-146,170-182)
# ---------------------------------------------------------------------------------------------------------
def test_dropout_kernel_statistics_and_determinism(cuda_dev):
    from navillm_b200 import ops
    n, p = 1 << 20, 0.1
    x = torch.randn(n, device=cuda_dev)
    y = ops.dropout(x, p, seed=1234)
    keep = y != 0
    frac = keep.float().mean().item()
    assert abs(frac - (1 - p)) < 5 * (p * (1 - p) / n) ** 0.5 + 1e-4, frac          # binomial 5 sigma
    assert torch.allclose(y[keep], x[keep] / (1 - p), rtol=1e-6, atol=0)
    assert torch.equal(y, ops.dropout(x, p, seed=1234))                               # same seed -> same mask
    assert not torch.equal(keep, ops.dropout(x, p, seed=1235) != 0)
    g = ops.dropout(torch.ones_like(x), p, seed=1234)                                 # backward = same op on the gradient
    assert torch.equal(g != 0, keep)
    assert torch.equal(ops.dropout(x, 0.0, seed=7), x)


def test_mha_dropout_forward_backward_match_torch_with_the_same_mask(cuda_dev):
    from navillm_b200 import ops
    B, N, H, hd, p = 3, 36, 4, 32, 0.1
    E = H * hd
    g = torch.Generator().manual_seed(5)
    qkv = torch.randn(B, N, 3 * E, generator=g).to(cuda_dev)
    lens = torch.tensor([36, 20, 7], dtype=torch.int32, device=cuda_dev)
    out, P, Pd = ops.mha_fwd_dropout(qkv, lens, H, p, seed=99)
    valid = (torch.arange(N, device=cuda_dev)[None, :] < lens[:, None])               # [B, N]
    pair = (valid[:, None, :, None] & valid[:, None, None, :]).expand(B, H, N, N)
    mask = (Pd != 0)
    frac = mask[pair].float().mean().item()
    assert abs(frac - (1 - p)) < 0.02, frac
    assert torch.allclose(Pd, P * mask / (1 - p), rtol=1e-6, atol=1e-9)
    # torch reference with the extracted mask
    x = qkv.clone().requires_grad_(True)
    q, k, v = [t.view(B, N, H, hd).transpose(1, 2) for t in x.split(E, dim=-1)]
    s = (q @ k.transpose(-1, -2)) * hd ** -0.5
    s = s.masked_fill(~valid[:, None, None, :], float("-inf"))
    pr = torch.softmax(s, dim=-1) * mask / (1 - p)
    ref = (pr @ v).transpose(1, 2).reshape(B, N, E) * valid[:, :, None]
    assert torch.allclose(out, ref.detach(), rtol=1e-4, atol=1e-5)
    go = torch.randn(B, N, E, generator=g).to(cuda_dev) * valid[:, :, None]
    ref.backward(go)
    dqkv = ops.mha_bwd_dropout(qkv, go.contiguous(), P, Pd, lens, H)
    vr = valid[:, :, None].expand(B, N, 3 * E)
    assert torch.allclose(dqkv[vr], x.grad[vr], rtol=1e-3, atol=1e-4), (dqkv[vr] - x.grad[vr]).abs().max().item()


def test_train_mode_dropout_is_applied_and_its_backward_is_consistent(cuda_dev):
    """Fixed RNG state => the train-mode encoder is a deterministic function; its hand-written backward must agree with
    central differences along random parameter directions (fp32 GEMMs: 2e-2 relative)."""
    import navillm_b200.image_embedding as IE
    from navillm_b200 import ops
    prev = ops.set_pano_precision("fp32")
    try:
        vis_cfg = types.SimpleNamespace(hidden_size=128, num_attention_heads=2, intermediate_size=256, hidden_dropout_prob=0.1,
                                        image_feat_size=72, angle_feat_size=4, obj_feat_size=40, output_size=256, num_pano_layers=2)
        torch.manual_seed(0)
        mod = IE.ImageEmbeddings(vis_cfg, use_obj=False).to(cuda_dev)
        g = torch.Generator().manual_seed(3)
        view = torch.randn(2, 12, 72, generator=g).to(cuda_dev)
        loc = torch.randn(2, 12, 7, generator=g).to(cuda_dev)
        types_ = torch.randint(0, 2, (2, 12), generator=g).to(cuda_dev)
        lens = torch.tensor([12, 9], device=cuda_dev)
        G = torch.randn(2, 12, 256, generator=g).to(cuda_dev)

        def f(train=True):
            IE._DROPOUT_CALLS[0] = 41                               # same masks on every evaluation
            mod.train(train)
            return (mod.forward_panorama_per_step(view, lens, loc, types_)["pano_embeds"] * G).sum()

        with torch.no_grad():
            assert abs(f(True).item() - f(False).item()) > 1e-3      # dropout changes the output in train()
            assert f(True).item() == f(True).item()                  # and is reproducible for a fixed call counter
        mod.zero_grad()
        f(True).backward()
        torch.cuda.synchronize()
        for name in ("img_linear.weight", "pano_encoder.layers.0.linear1.weight", "pano_encoder.layers.1.self_attn.in_proj_weight",
                     "mapper.weight"):
            prm = dict(mod.named_parameters())[name]
            d = torch.randn(prm.shape, generator=g).to(cuda_dev)
            d = d / d.norm()
            eps = 2e-2
            with torch.no_grad():
                prm.add_(eps * d); fp = f(True).item()
                prm.sub_(2 * eps * d); fm = f(True).item()
                prm.add_(eps * d)
            num = (fp - fm) / (2 * eps)
            ana = (prm.grad * d).sum().item()
            assert abs(num - ana) <= 2e-2 * max(abs(num), abs(ana)) + 2e-2, (name, num, ana)
    finally:
        ops.set_pano_precision(prev)


# ---------------------------------------------------------------------------------------------------------
# `--fuse_obj` branch (models/image_embedding.py:78-94) against the reference's own module (golden fixture)
# ---------------------------------------------------------------------------------------------------------
def test_pano_fuse_obj_matches_reference_golden(cuda_dev, pano_precision):
    """Forward outputs and every parameter gradient of the object-fusing encoder vs tests/golden/pano_fuse_obj.pt (the
    UNMODIFIED reference ImageEmbeddings(use_obj=True, fuse_obj=True), CPU fp32, eval): ragged view / object counts, one
    row without objects.  Two backward passes check that gradients accumulate."""
    from navillm_b200.image_embedding import ImageEmbeddings
    tol_f, tol_g = (1e-4, 2e-4) if pano_precision == "fp32" else (4e-3, 1e-2)
    g = torch.load(Path(__file__).resolve().parent / "golden" / "pano_fuse_obj.pt", weights_only=False)
    d = g["dims"]
    vis_cfg = types.SimpleNamespace(hidden_size=d["pano_hidden"], num_attention_heads=d["pano_heads"], intermediate_size=d["pano_inter"],
                                    hidden_dropout_prob=0.1, image_feat_size=d["image_feat_size"], angle_feat_size=4,
                                    obj_feat_size=d["obj_feat_size"], output_size=d["output_size"], num_pano_layers=d["num_pano_layers"])
    mod = ImageEmbeddings(vis_cfg, use_obj=True, fuse_obj=True).eval()
    assert list(mod.state_dict().keys()) == list(g["state_dict"].keys()), "parameter names / order must equal the reference's"
    mod.load_state_dict(g["state_dict"])
    mod = mod.to(cuda_dev)
    inp = {k: v.to(cuda_dev) for k, v in g["inputs"].items()}
    for rep in (1, 2):
        out = mod.forward_panorama_per_step(**inp)
        assert rel_err(out["pano_embeds"].detach().cpu(), g["pano_embeds"]) < tol_f
        assert rel_err(out["obj_embeds"].detach().cpu(), g["obj_embeds"]) < tol_f
        assert torch.equal(out["pano_masks"].cpu(), g["pano_masks"]) and torch.equal(out["obj_masks"].cpu(), g["obj_masks"])
        loss = (out["pano_embeds"] * g["wp"].to(cuda_dev)).sum() + (out["obj_embeds"] * g["wo"].to(cuda_dev)).sum()
        loss.backward()
        torch.cuda.synchronize()
        for name, p in mod.named_parameters():
            assert p.grad is not None, name
            assert rel_err(p.grad.cpu() / rep, g["grads"][name]) < tol_g, f"{name} (pass {rep}): {rel_err(p.grad.cpu() / rep, g['grads'][name])}"
    # without the flag the same weights give the plain encoder (object tokens not attended to)
    plain = ImageEmbeddings(vis_cfg, use_obj=True, fuse_obj=False).eval()
    plain.load_state_dict({k: v for k, v in g["state_dict"].items() if not k.startswith("obj_linear.")})
    plain = plain.to(cuda_dev)
    p2 = plain.forward_panorama_per_step(**inp)["pano_embeds"]
    assert rel_err(p2.detach().cpu(), g["pano_embeds"]) > 10 * tol_f


def test_pano_fuse_obj_errors(cuda_dev):
    from navillm_b200.image_embedding import ImageEmbeddings
    vis_cfg = types.SimpleNamespace(hidden_size=128, num_attention_heads=2, intermediate_size=256, hidden_dropout_prob=0.1,
                                    image_feat_size=64, angle_feat_size=4, obj_feat_size=48, output_size=256, num_pano_layers=1)
    mod = ImageEmbeddings(vis_cfg, use_obj=True, fuse_obj=True).eval().to(cuda_dev)
    with pytest.raises(ValueError):
        mod.forward_panorama_per_step(torch.randn(1, 4, 64, device=cuda_dev), torch.tensor([4], device=cuda_dev))
