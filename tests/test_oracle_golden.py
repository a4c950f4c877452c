"""Pin the CPU oracle (oracle/navillm_oracle.py) against golden vectors produced by the UNMODIFIED
reference code (tests/golden/make_golden.py, run against a checkout of the reference).  CPU only: runs under `-m "not gpu"`.

Tolerances: the oracle restates the same torch arithmetic in the same dtypes, so fp32 results agree to
accumulation-order noise (1e-5 relative) and the bf16 LM path to 1 bf16 ulp on logits / hidden states.
"""
import sys
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from oracle import navillm_oracle as O  # noqa: E402
from navillm_b200.tokenizer import SyntheticTokenizer  # noqa: E402

GOLD = Path(__file__).resolve().parent / "golden"


def load(precision):
    g = torch.load(GOLD / f"nav_{precision}.pt", weights_only=False)
    d = g["meta"]["dims"]
    tok = SyntheticTokenizer(base_vocab=d["base_vocab"])
    cfg = O.OracleConfig(hidden=d["hidden"], n_layers=d["n_layers"], n_heads=d["n_heads"], inter=d["inter"],
                         vocab=len(tok), image_feat_size=d["image_feat_size"], obj_feat_size=d["obj_feat_size"],
                         pano_hidden=d["pano_hidden"], pano_heads=d["pano_heads"], pano_inter=d["pano_inter"],
                         cand_id=tok.special["<cand>"], hist_id=tok.special["<hist>"], obj_id=tok.special["<obj>"],
                         cls_ids=(tok.special["<cls_1>"], tok.special["<cls_2>"]), precision=precision)
    return g, cfg, tok


def tol(precision):
    return dict(rtol=2e-5, atol=2e-5) if precision == "fp32" else dict(rtol=1.6e-2, atol=1.6e-2)


def nav_batch(g, pano_embeds, pano_masks):
    B = pano_embeds.shape[0]
    b = dict(g["nav_in"])
    b["vp_img_embeds"] = torch.cat([torch.zeros_like(pano_embeds[:, :1]), pano_embeds], 1)
    b["pano_masks"] = torch.cat([torch.ones(B, 1, dtype=torch.bool), pano_masks], 1)
    return b


@pytest.mark.parametrize("precision", ["fp32", "amp_bf16"])
def test_panorama_matches_reference(precision):
    g, cfg, tok = load(precision)
    out = O.forward_panorama(g["state_dict"], cfg, **g["pano_in"])
    for k in ("pano_embeds", "obj_embeds"):
        assert torch.allclose(out[k], g["pano_out"][k], rtol=2e-5, atol=2e-5), k   # encoder is fp32 in both precisions
    assert torch.equal(out["pano_masks"], g["pano_out"]["pano_masks"])
    assert torch.equal(out["obj_masks"], g["pano_out"]["obj_masks"])


@pytest.mark.parametrize("precision", ["fp32", "amp_bf16"])
def test_navigation_forward_and_backward_match_reference(precision):
    g, cfg, tok = load(precision)
    sd = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in g["state_dict"].items()}
    pano = O.forward_panorama(sd, cfg, **g["pano_in"])
    batch = nav_batch(g, pano["pano_embeds"], pano["pano_masks"])
    torch.manual_seed(1234)                      # same RNG state as the reference run -> same candidate permutation
    nav = O.forward_navigation(sd, cfg, batch, tok)
    ref = g["nav_out"]
    assert torch.equal(torch.isinf(nav["fuse_logits"]), torch.isinf(ref["fuse_logits"]))
    fin = ~torch.isinf(ref["fuse_logits"])
    assert torch.allclose(nav["fuse_logits"][fin].float(), ref["fuse_logits"][fin].float(), **tol(precision))
    assert torch.allclose(nav["fuse_embeds"], ref["fuse_embeds"], rtol=2e-5, atol=2e-5)
    loss = F.cross_entropy(nav["fuse_logits"], g["targets"], reduction="sum", ignore_index=-100) / 2
    assert torch.allclose(loss.float(), ref["loss"].float(), **tol(precision))
    loss.backward()
    for name, gr in g["nav_grads"].items():
        mine = sd[name].grad
        assert mine is not None, name
        scale = gr.float().abs().max().item() + 1e-12
        err = (mine.float() - gr.float()).abs().max().item()
        lim = 1e-4 if precision == "fp32" else 4e-2
        assert err <= lim * scale, f"{name}: err {err} vs scale {scale}"


@pytest.mark.parametrize("precision", ["fp32", "amp_bf16"])
def test_object_grounding_matches_reference(precision):
    g, cfg, tok = load(precision)
    out = O.forward_object_grounding(g["state_dict"], cfg, g["og_in"], tok)["obj_logits"]
    ref = g["og_out"]["obj_logits"]
    assert torch.equal(torch.isinf(out), torch.isinf(ref))
    fin = ~torch.isinf(ref)
    assert torch.allclose(out[fin].float(), ref[fin].float(), **tol(precision))


@pytest.mark.parametrize("precision", ["fp32", "amp_bf16"])
def test_lm_loss_modes_match_reference(precision):
    g, cfg, tok = load(precision)
    sd = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in g["state_dict"].items()}
    s = O.forward_summarization(sd, cfg, g["sum_in"], tok, tok.eos_token, training=True)
    assert torch.allclose(s["loss"].float(), g["sum_out"]["loss"].float(), **tol(precision))
    s["loss"].backward()
    for name, gr in g["sum_grads"].items():
        err = (sd[name].grad.float() - gr.float()).abs().max().item()
        assert err <= (1e-4 if precision == "fp32" else 4e-2) * (gr.float().abs().max().item() + 1e-12), name
    sd = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in g["state_dict"].items()}
    q = O.forward_3dqa(sd, cfg, g["qa_in"], tok, tok.eos_token, training=True)
    assert torch.allclose(q["loss"].float(), g["qa_out"]["loss"].float(), **tol(precision))
    last = q["logits"][:, -1, :]
    ref = g["qa_out"]["logits_last"]
    fin = ~torch.isinf(ref)
    assert torch.equal(torch.isinf(last), torch.isinf(ref))
    assert torch.allclose(last[fin].float(), ref[fin].float(), **tol(precision))
    q["loss"].backward()
    for name, gr in g["qa_grads"].items():
        err = (sd[name].grad.float() - gr.float()).abs().max().item()
        assert err <= (1e-4 if precision == "fp32" else 4e-2) * (gr.float().abs().max().item() + 1e-12), name


def test_greedy_generate_is_consistent_with_full_forward():
    """The restated KV-cache greedy loop must produce the tokens a cache-free full re-forward produces
    (fp32: no near-tie ambiguity at these dims)."""
    g, cfg, tok = load("fp32")
    sd = g["state_dict"]
    qa = g["qa_in"]
    text = tok(qa["prompts"])
    feats = qa["features"]
    lens = torch.tensor([f.shape[0] for f in feats])
    view = torch.stack([torch.cat([f, f.new_zeros(int(lens.max()) - f.shape[0], f.shape[1])], 0) for f in feats], 0)
    pano = O.forward_panorama(sd, cfg, view, lens)
    pe = pano["pano_embeds"] + O._pos_embed(torch.zeros(pano["pano_embeds"].shape[:2] + (14,)), sd, "vp_pos_embeddings")
    pe = pe + sd["token_type_embeddings.weight"][0]
    cand = pe[pano["pano_masks"]]
    ids = O.greedy_generate(sd, cfg, text["input_ids"], text["attention_mask"], cand_vis=cand, max_new_tokens=4,
                            stop_on_eos=False)
    cur, mask = text["input_ids"].clone(), text["attention_mask"].clone()
    for _ in range(4):
        pos = (mask.cumsum(-1) - 1).masked_fill(mask == 0, 1)
        out = O.modified_lm_forward(sd, cfg, cur, mask, cand_vis=cand, position_ids=pos)
        nxt = out["logits"][:, -1].float().argmax(-1)
        cur = torch.cat([cur, nxt[:, None]], 1)
        mask = torch.cat([mask, mask.new_ones(2, 1)], 1)
    assert torch.equal(ids, cur)


@pytest.mark.parametrize("precision", ["fp32", "amp_bf16"])
def test_greedy_generate_matches_reference_generation_branch(precision):
    """The oracle's restated greedy loop against token ids produced by the reference's own generation branch
    (models/nav_model.py:386-402 driving HF generate; tests/golden/make_generate_golden.py, which documents the
    one-line signature adapter needed under transformers 5.x)."""
    g, cfg, tok = load(precision)
    gen = torch.load(GOLD / f"generate_{precision}.pt", weights_only=False)
    sd = g["state_dict"]
    qa = g["qa_in"]
    text = tok(qa["prompts"])
    feats = qa["features"]
    lens = torch.tensor([f.shape[0] for f in feats])
    view = torch.stack([torch.cat([f, f.new_zeros(int(lens.max()) - f.shape[0], f.shape[1])], 0) for f in feats], 0)
    pano = O.forward_panorama(sd, cfg, view, lens)
    pe = pano["pano_embeds"] + O._pos_embed(torch.zeros(pano["pano_embeds"].shape[:2] + (14,)), sd, "vp_pos_embeddings")
    pe = pe + sd["token_type_embeddings.weight"][0]
    cand = pe[pano["pano_masks"]]
    n_new = gen["meta"]["max_new_tokens"]
    ids, step_logits = O.greedy_generate(sd, cfg, text["input_ids"], text["attention_mask"], cand_vis=cand, max_new_tokens=n_new,
                                         eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id, return_logits=True)
    S0 = gen["prompt_len"]
    assert S0 == text["input_ids"].shape[1] and torch.equal(ids[:, :S0], gen["ids"][:, :S0])
    if precision == "fp32":
        assert torch.equal(ids, gen["ids"]), (ids[:, S0:].tolist(), gen["ids"][:, S0:].tolist())
        return
    # bf16: identical until a step whose top-2 logits are within the bf16 noise floor (2 ulp of the top logit); after
    # such a near-tie the two sequences may legitimately diverge
    for b in range(ids.shape[0]):
        for t in range(min(ids.shape[1], gen["ids"].shape[1]) - S0):
            if ids[b, S0 + t] == gen["ids"][b, S0 + t]:
                continue
            top2 = torch.topk(step_logits[t][b], 2).values
            assert (top2[0] - top2[1]).item() <= 2 * 2.0 ** -8 * top2[0].abs().item(), (b, t, top2.tolist())
            break
        else:
            continue
    assert torch.equal(ids[:, S0:S0 + 4], gen["ids"][:, S0:S0 + 4])          # the first tokens are far from ties


class _Node:
    def __init__(self):
        from collections import defaultdict
        self.child = defaultdict(_Node)


class _Trie:
    """tools/trie.py interface."""

    def __init__(self, bos, eos):
        self.root, self.bos, self.eos = _Node(), bos, eos

    def insert(self, word):
        cur = self.root
        for c in word:
            cur = cur.child[c]

    def get_child_index(self, cur):
        return [self.eos] if len(cur.child) == 0 else list(cur.child.keys())

    def get_next_node(self, cur, w):
        return cur if len(cur.child) == 0 else cur.child[w]


@pytest.mark.parametrize("precision", ["fp32", "amp_bf16"])
def test_summarization_generation_branch_matches_reference(precision):
    """Oracle vs the reference's summarization generation branch (models/nav_model.py:320-341): <hist> and <cand> visual
    tokens, 50 new tokens, free and Trie-constrained (TrieLogitsProcessor, models/modified_lm.py:10-30)."""
    g, cfg, tok = load(precision)
    gen = torch.load(GOLD / f"generate_{precision}.pt", weights_only=False)
    sd = g["state_dict"]
    S0 = gen["sum_prompt_len"]
    trie = _Trie(tok.bos_token_id, tok.eos_token_id)
    for w in gen["trie_words"]:
        trie.insert(w)
    out = O.forward_summarization(sd, cfg, g["sum_in"], tok, tok.eos_token, training=False, trie=trie,
                                  eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id)["generated_ids"]
    assert out.tolist() == gen["trie_ids"][:, S0:].tolist()
    free = O.forward_summarization(sd, cfg, g["sum_in"], tok, tok.eos_token, training=False,
                                   eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id)["generated_ids"]
    ref = gen["sum_ids"][:, S0:]
    n = min(free.shape[1], ref.shape[1])
    if precision == "fp32":
        assert free[:, :n].tolist() == ref[:, :n].tolist()
    else:
        assert free[:, :5].tolist() == ref[:, :5].tolist()                   # later steps may hit a bf16 near-tie


def load_fuse_obj():
    g = torch.load(GOLD / "pano_fuse_obj.pt", weights_only=False)
    d = g["dims"]
    cfg = O.OracleConfig(image_feat_size=d["image_feat_size"], obj_feat_size=d["obj_feat_size"], pano_hidden=d["pano_hidden"],
                         pano_heads=d["pano_heads"], pano_inter=d["pano_inter"], num_pano_layers=d["num_pano_layers"])
    return g, cfg


def test_panorama_fuse_obj_matches_reference():
    """`--fuse_obj` branch (models/image_embedding.py:78-94): forward outputs and every parameter gradient against the
    reference's own ImageEmbeddings (tests/golden/make_fuse_obj_golden.py)."""
    g, cfg = load_fuse_obj()
    sd = {"img_embeddings." + k: v.clone().requires_grad_(True) for k, v in g["state_dict"].items()}
    out = O.forward_panorama(sd, cfg, **g["inputs"], fuse_obj=True)
    assert torch.allclose(out["pano_embeds"], g["pano_embeds"], rtol=2e-5, atol=2e-5)
    assert torch.allclose(out["obj_embeds"], g["obj_embeds"], rtol=2e-5, atol=2e-5)
    assert torch.equal(out["pano_masks"], g["pano_masks"]) and torch.equal(out["obj_masks"], g["obj_masks"])
    loss = (out["pano_embeds"] * g["wp"]).sum() + (out["obj_embeds"] * g["wo"]).sum()
    assert torch.allclose(loss, g["loss"], rtol=1e-5, atol=1e-4)
    loss.backward()
    assert not g["no_grad"]
    for n, ref in g["grads"].items():
        got = sd["img_embeddings." + n].grad
        assert got is not None, n
        scale = float(ref.abs().max()) + 1e-6
        assert float((got - ref).abs().max()) <= 2e-5 * scale + 2e-5, n
    # the branch differs from the plain encoder (object tokens are attended to)
    plain = O.forward_panorama(sd, cfg, **g["inputs"], fuse_obj=False)["pano_embeds"]
    assert float((plain - g["pano_embeds"]).abs().max()) > 1e-3
