"""Cross-step prompt-prefix KV reuse (SURVEY.md §8f n1): the NavModel rollout API.  The suffix attention kernel itself
(nv_attn_fwd_kv) is checked against fp64 with per-element bounds in tests/test_prefix_attn_kernels_gpu.py.

Tolerances, stated:
  * fuse_logits with the cache vs the from-scratch forward of the same prompts: the math is identical except that a
    row keeps the rotary offset of its first step (rotary attention depends on position differences only), so only
    bf16 rounding differs (cos/sin table entries, accumulation order of the split softmax): 3e-2 of max|logit|.
"""
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _build(cuda_dev):
    from navillm_b200.nav_model import NavModel
    from navillm_b200.tokenizer import SyntheticTokenizer
    from oracle import navillm_oracle as O
    tok = SyntheticTokenizer(base_vocab=256)
    d = dict(hidden=256, n_layers=2, n_heads=2, inter=256, pano_hidden=128, pano_heads=2, pano_inter=256, image_feat_size=64,
             obj_feat_size=48)
    cfg = O.OracleConfig(hidden=d["hidden"], n_layers=d["n_layers"], n_heads=d["n_heads"], inter=d["inter"], vocab=len(tok),
                         image_feat_size=d["image_feat_size"], obj_feat_size=d["obj_feat_size"], pano_hidden=d["pano_hidden"],
                         pano_heads=d["pano_heads"], pano_inter=d["pano_inter"], cand_id=tok.special["<cand>"],
                         hist_id=tok.special["<hist>"], obj_id=tok.special["<obj>"],
                         cls_ids=(tok.special["<cls_1>"], tok.special["<cls_2>"]))
    sd = O.init_state_dict(cfg, seed=3)
    args = types.SimpleNamespace(precision="amp_bf16", pretrained_model_name_or_path="vicuna-tiny", image_feat_size=d["image_feat_size"],
                                 angle_feat_size=4, obj_feat_size=d["obj_feat_size"], enable_og=True, fuse_obj=False, feat_dropout=0.4,
                                 resume_from_checkpoint=None, from_scratch=True)
    mc = types.SimpleNamespace(num_pano_layers=2, tokenizer=tok,
                               llama_config=dict(hidden_size=d["hidden"], intermediate_size=d["inter"], num_hidden_layers=d["n_layers"],
                                                 num_attention_heads=d["n_heads"], vocab_size=256),
                               vis_config=dict(hidden_size=d["pano_hidden"], num_attention_heads=d["pano_heads"],
                                               intermediate_size=d["pano_inter"]))
    model = NavModel(args, None, mc)
    model.load_state_dict(sd, strict=True)
    return model.to(cuda_dev).eval(), d


def _nav_batch(d, step, hist, g, instr):
    """Step `step` of a synthetic 2-episode rollout: prompts in the reference's order (tasks/agents/r2r.py:16-31) with
    `step` history tokens; the numbers of candidates differ per row and per step."""
    B, G, D, NV1 = 2, 6, d["hidden"], 9
    n_cand = [2 + (step + b) % 3 for b in range(B)]
    vp_c = [[None] + [f"c{j}" for j in range(n)] for n in n_cand]
    gm = [[None, "s"] + [f"c{j}" for j in range(4)] for _ in range(B)]
    prompts = []
    for b in range(B):
        hist_text = " ".join(f"( {i} ) <hist>" for i in range(step))
        cand_text = " ".join("( 0 ) stop" if i == 0 else f"( {i} ) <cand>" for i in range(n_cand[b] + 1))
        prompts.append(f"Instruction : {instr[b]} History : {hist_text} Candidate : {cand_text} Output : <cls_1>")
    return {"data_type": ["r2r"] * B, "vp_img_embeds": torch.randn(B, NV1, D, generator=g),
            "pano_masks": torch.ones(B, NV1, dtype=torch.bool), "vp_pos_fts": torch.randn(B, NV1, 14, generator=g),
            "vp_cand_vpids": vp_c, "gmap_img_embeds": torch.randn(B, G, D, generator=g),
            "gmap_step_ids": torch.tensor([[0, 1, 0, 0, 0, 0]] * B), "gmap_pos_fts": torch.randn(B, G, 7, generator=g),
            "gmap_masks": torch.tensor([[True, True] + [j < n for j in range(4)] for n in n_cand]),
            "gmap_pair_dists": None, "gmap_visited_masks": torch.tensor([[0, 1, 0, 0, 0, 0]] * B, dtype=torch.bool),
            "gmap_vpids": gm, "instruction": instr, "history": [["h"] * step] * B,
            "hist_vis": [list(h) for h in hist], "prompts": prompts}


def test_rollout_with_prefix_cache_matches_from_scratch(cuda_dev):
    from navillm_b200.modified_lm import PrefixKVCache
    model, d = _build(cuda_dev)
    g = torch.Generator().manual_seed(11)
    instr = ["walk past the sofa and stop at the door of the kitchen", "leave the room"]
    hist = [[], []]
    cache = PrefixKVCache(model.lang_model, batch_size=2, max_len=256)
    to_dev = lambda b: {k: (v.to(cuda_dev) if torch.is_tensor(v) else v) for k, v in b.items()}
    encoded = []
    with torch.no_grad():
        for step in range(5):
            batch = _nav_batch(d, step, hist, g, instr)
            batch["hist_vis"] = [[v.to(cuda_dev) for v in vs] for vs in batch["hist_vis"]]
            torch.manual_seed(100 + step)
            ref = model("navigation", to_dev(dict(batch)))
            torch.manual_seed(100 + step)
            got = model("navigation", to_dev(dict(batch)), prefix_cache=cache)
            a, r = got["fuse_logits"].float().cpu(), ref["fuse_logits"].float().cpu()
            fin = torch.isfinite(r)
            assert torch.equal(torch.isfinite(a), fin)
            scale = r[fin].abs().max().item()
            assert (a[fin] - r[fin]).abs().max().item() <= 3e-2 * scale + 1e-3, (step, (a[fin] - r[fin]).abs().max().item(), scale)
            assert torch.equal(got["fuse_embeds"].cpu(), ref["fuse_embeds"].cpu())
            encoded.append(cache.stats["tokens_encoded"])
            # the chosen node's fused embedding becomes the next <hist> vector (mp3d_agent.py:774-778)
            for b in range(2):
                hist[b].append(ref["fuse_embeds"][b, 2].float().cpu())
    st = cache.stats
    assert st["steps"] == 5 and st["tokens_encoded"] < st["tokens"]
    # from step 1 on only the tail (new <hist> + candidates + output hint) is encoded: far fewer rows than the prompt
    per_step = np.diff([0] + encoded)
    assert per_step[1:].max() < per_step[0] + 8 * 5, per_step
    # a new episode in row 0 invalidates only that row
    cache.reset(rows=[0])
    assert cache.ids[0].size == 0 and cache.ids[1].size > 0


def test_prefix_cache_refuses_grad_mode(cuda_dev):
    from navillm_b200.modified_lm import PrefixKVCache
    model, d = _build(cuda_dev)
    g = torch.Generator().manual_seed(1)
    batch = _nav_batch(d, 0, [[], []], g, ["a b c", "d e"])
    cache = PrefixKVCache(model.lang_model, batch_size=2, max_len=128)
    with pytest.raises(RuntimeError, match="no_grad"):
        model("navigation", {k: (v.to(cuda_dev) if torch.is_tensor(v) else v) for k, v in batch.items()}, prefix_cache=cache)
