"""End-to-end parity of navillm_b200.NavModel (the drop-in boundary) on an H100 against
(a) golden vectors produced by the UNMODIFIED reference (tests/golden/nav_amp_bf16.pt) and
(b) the CPU oracle, forward outputs, losses and gradients, for every mode of NavModel.forward.

bf16 tolerance, stated: `truth` = golden fp32 run of the reference (nav_fp32.pt; same seeds, weights before
bf16 rounding); the reference's own bf16 run deviates from it by e_ref.  The CUDA path, loaded with the bf16
golden weights, must satisfy |cuda - ref_bf16| <= 3 * |ref_bf16 - truth|_max + 2e-2 * scale  for logits/losses
and gradient tensors (scale = max|ref|).  fp32 parts (pano encoder outputs, fuse_embeds) must agree to 1e-4 with the
exact-fp32 panorama GEMMs and to 4e-3 with the default wgmma tf32 GEMMs (10-bit-mantissa operands, the mode
the reference's pinned torch 1.10 used on Ampere+; see tests/test_pano_gpu.py).
"""
import sys
import types
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
GOLD = Path(__file__).resolve().parent / "golden"


def build_model(g, dev):
    from navillm_b200.nav_model import NavModel
    from navillm_b200.tokenizer import SyntheticTokenizer
    d = g["meta"]["dims"]
    tok = SyntheticTokenizer(base_vocab=d["base_vocab"])
    args = types.SimpleNamespace(precision="amp_bf16", pretrained_model_name_or_path="vicuna-tiny", image_feat_size=d["image_feat_size"],
                                 angle_feat_size=4, obj_feat_size=d["obj_feat_size"], enable_og=True, fuse_obj=False, feat_dropout=0.4,
                                 resume_from_checkpoint=None, from_scratch=True)
    mc = types.SimpleNamespace(num_pano_layers=2, tokenizer=tok,
                               llama_config=dict(hidden_size=d["hidden"], intermediate_size=d["inter"], num_hidden_layers=d["n_layers"],
                                                 num_attention_heads=d["n_heads"], vocab_size=d["base_vocab"]),
                               vis_config=dict(hidden_size=d["pano_hidden"], num_attention_heads=d["pano_heads"],
                                               intermediate_size=d["pano_inter"]))
    model = NavModel(args, None, mc)
    missing, unexpected = model.load_state_dict(g["state_dict"], strict=False)
    assert not unexpected and not missing, (missing, unexpected)          # reference checkpoint keys == our keys
    return model.to(dev).eval(), tok


def to_dev(x, dev):
    if torch.is_tensor(x):
        return x.to(dev)
    if isinstance(x, dict):
        return {k: to_dev(v, dev) for k, v in x.items()}
    if isinstance(x, list) and x and torch.is_tensor(x[0]):
        return [v.to(dev) for v in x]
    if isinstance(x, list) and x and isinstance(x[0], list) and x[0] and torch.is_tensor(x[0][0]):
        return [[v.to(dev) for v in y] for y in x]
    return x


def check(name, mine, ref, truth, k=3.0, floor=2e-2):
    mine, ref, truth = mine.float().cpu(), ref.float(), truth.float()
    fin = torch.isfinite(ref)
    assert torch.equal(torch.isfinite(mine), fin), f"{name}: -inf pattern differs"
    scale = ref[fin].abs().max().item() + 1e-12
    e_ref = (ref[fin] - truth[fin]).abs().max().item()
    e = (mine[fin] - ref[fin]).abs().max().item()
    assert e <= k * e_ref + floor * scale, f"{name}: |cuda-ref|={e:.4g} > {k}*{e_ref:.4g} + {floor}*{scale:.3g}"


def test_navmodel_all_modes_match_reference(cuda_dev, pano_precision):
    tol32 = 1e-4 if pano_precision == "fp32" else 4e-3
    g = torch.load(GOLD / "nav_amp_bf16.pt", weights_only=False)
    t = torch.load(GOLD / "nav_fp32.pt", weights_only=False)
    model, tok = build_model(g, cuda_dev)
    named = dict(model.named_parameters())

    # ---- panorama (fp32) ----
    pano = model("panorama", to_dev(dict(g["pano_in"]), cuda_dev))
    for k in ("pano_embeds", "obj_embeds"):
        ref = g["pano_out"][k]
        assert (pano[k].detach().cpu() - ref).abs().max().item() <= tol32 * ref.abs().max().item(), k
    assert torch.equal(pano["pano_masks"].cpu(), g["pano_out"]["pano_masks"])
    assert torch.equal(pano["obj_masks"].cpu(), g["pano_out"]["obj_masks"])

    # ---- navigation + action CE + backward (tasks/agents/mp3d_agent.py:683-757) ----
    B = 2
    nav_in = to_dev(dict(g["nav_in"]), cuda_dev)
    nav_in["vp_img_embeds"] = torch.cat([torch.zeros_like(pano["pano_embeds"][:, :1]), pano["pano_embeds"]], 1)
    nav_in["pano_masks"] = torch.cat([torch.ones(B, 1, dtype=torch.bool, device=cuda_dev), pano["pano_masks"]], 1)
    torch.manual_seed(1234)                                  # same CPU RNG state as the reference run
    nav = model("navigation", nav_in)
    check("fuse_logits", nav["fuse_logits"].detach(), g["nav_out"]["fuse_logits"], t["nav_out"]["fuse_logits"])
    ref_fe = g["nav_out"]["fuse_embeds"]
    assert (nav["fuse_embeds"].cpu() - ref_fe).abs().max().item() <= tol32 * ref_fe.abs().max().item()
    loss = F.cross_entropy(nav["fuse_logits"].float(), g["targets"].to(cuda_dev), reduction="sum", ignore_index=-100) / B
    check("nav loss", loss.detach(), g["nav_out"]["loss"], t["nav_out"]["loss"])
    loss.backward()
    torch.cuda.synchronize()
    for name, gr in g["nav_grads"].items():
        assert named[name].grad is not None, name
        check("grad " + name, named[name].grad, gr, t["nav_grads"][name], k=3.0, floor=5e-2)

    # ---- object grounding ----
    og = model("object_grounding", to_dev(dict(g["og_in"]), cuda_dev))
    check("obj_logits", og["obj_logits"].detach(), g["og_out"]["obj_logits"], t["og_out"]["obj_logits"])

    # ---- summarization (LM loss) ----
    model.zero_grad(set_to_none=False)
    s = model("summarization", to_dev(dict(g["sum_in"]), cuda_dev), training=True)
    check("sum loss", s["loss"].detach(), g["sum_out"]["loss"], t["sum_out"]["loss"])
    s["loss"].backward()
    for name, gr in g["sum_grads"].items():
        check("sum grad " + name, named[name].grad, gr, t["sum_grads"][name], k=3.0, floor=5e-2)

    # ---- 3dqa (pano encoder + LM loss; gradient reaches img_linear through the visual tokens) ----
    model.zero_grad(set_to_none=True)                        # exercises the grad re-attach path
    q = model("3dqa", to_dev(dict(g["qa_in"]), cuda_dev), training=True)
    check("qa loss", q.loss.detach(), g["qa_out"]["loss"], t["qa_out"]["loss"])
    q.loss.backward()
    for name, gr in g["qa_grads"].items():
        check("qa grad " + name, named[name].grad, gr, t["qa_grads"][name], k=3.0, floor=5e-2)


def test_lang_model_forward_direct(cuda_dev):
    """ModifiedLlamaForCausalLM.forward called the way a reference caller would (models/modified_lm.py:89-146): loss,
    [B,S,D] hidden states and (on request) [B,S,V] logits with the special tokens at -inf, against the oracle."""
    from oracle import navillm_oracle as O
    from tests.test_oracle_golden import load
    g, cfg, tok = load("amp_bf16")
    _, cfg32, _ = load("fp32")
    model, _ = build_model(g, cuda_dev)
    sd = g["state_dict"]
    sd32 = {k: v.float() for k, v in sd.items()}
    text = tok([["Question : what <cand> <cand> is <hist> this", "a red chair </s>"], ["Describe <cand> <hist> <hist>", "kitchen </s>"]])
    ids, mask = text["input_ids"], text["attention_mask"]
    labels = ids.clone()
    labels[text["token_type_ids"] == 0] = -100
    n_c, n_h = int((ids == tok.special["<cand>"]).sum()), int((ids == tok.special["<hist>"]).sum())
    gen = torch.Generator().manual_seed(3)
    cand, hist = torch.randn(n_c, cfg.hidden, generator=gen), torch.randn(n_h, cfg.hidden, generator=gen)
    ref = O.modified_lm_forward(sd, cfg, ids, mask, labels=labels, cand_vis=cand, hist_vis=hist)
    truth = O.modified_lm_forward(sd32, cfg32, ids, mask, labels=labels, cand_vis=cand, hist_vis=hist)
    out = model.lang_model(input_ids=ids, attention_mask=mask, labels=labels, cand_vis=cand.to(cuda_dev), hist_vis=hist.to(cuda_dev),
                           return_logits=True, use_cache=False, output_hidden_states=True)
    m = mask.bool()
    check("lm loss", out.loss.detach(), ref["loss"].detach(), truth["loss"].detach())
    check("hidden_states", out.hidden_states.detach()[m.to(cuda_dev)], ref["hidden_states"].detach()[m], truth["hidden_states"].detach()[m])
    check("logits", out["logits"].detach()[m.to(cuda_dev)], ref["logits"].detach()[m], truth["logits"].detach()[m])
    assert out.hidden_states.shape == ref["hidden_states"].shape and out.logits.shape == ref["logits"].shape
    assert float(out.hidden_states[~m.to(cuda_dev)].abs().sum()) == 0.0            # pad rows: documented zeros
    plain = model.lang_model(input_ids=ids, attention_mask=mask, cand_vis=cand.to(cuda_dev), hist_vis=hist.to(cuda_dev))
    assert plain.loss is None and plain.logits is None and plain.hidden_states.shape == ref["hidden_states"].shape
    with pytest.raises(NotImplementedError):
        model.lang_model(input_ids=ids[:, -1:], attention_mask=mask, past_key_values=[(None, None)])


def test_wrong_mode_and_cpu_fail_loudly(cuda_dev):
    g = torch.load(GOLD / "nav_amp_bf16.pt", weights_only=False)
    model, tok = build_model(g, cuda_dev)
    with pytest.raises(NotImplementedError):
        model("teleport", {})
    cpu_model, _ = build_model(g, torch.device("cpu"))
    with pytest.raises(RuntimeError):
        cpu_model("panorama", dict(g["pano_in"]))
