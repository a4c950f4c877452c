"""Generate golden vectors from the UNMODIFIED reference (zd11024/NaviLLM) at tiny dimensions.

Needs a checkout of the reference, named by the NAVILLM_REFERENCE environment variable (nothing under tests/ reads
it at test time).  The reference's model
code is imported as-is; three things it would fetch from the network are stubbed (SURVEY.md §8c):
  (i)   PretrainedConfig.from_pretrained('bert-large-uncased')   -> tiny pano-encoder config
  (ii)  AutoConfig.from_pretrained(vicuna)                        -> tiny LlamaConfig (eager attention)
  (iii) ModifiedLM.init_tokenizer / tokenize                      -> navillm_b200.tokenizer.SyntheticTokenizer
Everything else (NavModel, ImageEmbeddings, DETR encoder, ModifiedLM.forward, HF LLaMA) is the
reference's own code path, run on CPU in eval() mode with precision 'amp_bf16' (LM in bf16, encoder fp32)
and in 'fp32'.

    python tests/golden/make_golden.py          # writes tests/golden/nav_<precision>.pt

Recorded: transformers.__version__, torch.__version__, the state_dict, all inputs, forward outputs of
every mode, the action-CE / LM losses and a selection of gradients.
"""
import os
import sys
import types
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
REF = os.environ["NAVILLM_REFERENCE"]

DIMS = dict(hidden=256, n_layers=2, n_heads=2, inter=256, base_vocab=256,
            pano_hidden=128, pano_heads=2, pano_inter=256, image_feat_size=64, obj_feat_size=48)


def build_reference_model(precision: str):
    sys.path.insert(0, REF)
    import transformers
    from transformers import LlamaConfig
    import models.nav_model as nm
    import models.modified_lm as ml
    from navillm_b200.tokenizer import SyntheticTokenizer

    class _VisCfg(transformers.PretrainedConfig):
        pass

    def fake_vis_from_pretrained(name, *a, **k):
        return _VisCfg(hidden_size=DIMS["pano_hidden"], num_attention_heads=DIMS["pano_heads"],
                       intermediate_size=DIMS["pano_inter"], hidden_act="gelu", hidden_dropout_prob=0.1)

    def fake_auto_from_pretrained(name, *a, **k):
        return LlamaConfig(hidden_size=DIMS["hidden"], intermediate_size=DIMS["inter"], num_hidden_layers=DIMS["n_layers"],
                           num_attention_heads=DIMS["n_heads"], num_key_value_heads=DIMS["n_heads"],
                           vocab_size=DIMS["base_vocab"], max_position_embeddings=2048, rms_norm_eps=1e-6,
                           attn_implementation="eager")

    nm.PretrainedConfig.from_pretrained = staticmethod(fake_vis_from_pretrained)
    nm.AutoConfig.from_pretrained = staticmethod(fake_auto_from_pretrained)

    def init_tokenizer(self, path):
        tok = SyntheticTokenizer(base_vocab=DIMS["base_vocab"])
        self.tokenizer = tok
        self.cand_token, self.hist_token, self.obj_token = ["<cand>"], ["<hist>"], ["<obj>"]
        self.cls_token = ["<cls_1>", "<cls_2>"]
        self.cand_token_id = [tok.special["<cand>"]]
        self.hist_token_id = [tok.special["<hist>"]]
        self.obj_token_id = [tok.special["<obj>"]]
        self.cls_token_id = [tok.special["<cls_1>"], tok.special["<cls_2>"]]
        self.special_token_ids = self.cand_token_id + self.hist_token_id + self.obj_token_id + self.cls_token_id
        self.resize_token_embeddings(len(tok))

    def tokenize(self, text, add_special_tokens=True):
        return self.tokenizer(text, max_length=1024, padding=True, truncation=True, return_tensors="pt",
                              add_special_tokens=add_special_tokens, return_token_type_ids=True)

    ml.ModifiedLM.init_tokenizer = init_tokenizer
    ml.ModifiedLM.tokenize = tokenize

    args = types.SimpleNamespace(precision=precision, pretrained_model_name_or_path="vicuna-tiny", image_feat_size=DIMS["image_feat_size"],
                                 angle_feat_size=4, obj_feat_size=DIMS["obj_feat_size"], enable_og=True, fuse_obj=False,
                                 feat_dropout=0.4, resume_from_checkpoint=None, from_scratch=True)
    logger = types.SimpleNamespace(info=lambda *a, **k: None)
    torch.manual_seed(0)
    model = nm.NavModel(args, logger, types.SimpleNamespace(num_pano_layers=2))
    # non-trivial LayerNorm/RMSNorm affine parameters and head biases so parity exercises them
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if p.dim() == 1:
                p.add_((torch.randn(p.shape, generator=g) * 0.05).to(p.dtype))
    model.eval()
    return model, transformers.__version__


def make_inputs(seed=0):
    """Synthetic R2R-shaped step (SURVEY.md §8d) at tiny sizes: B=2, 12 views, ragged candidates/history."""
    g = torch.Generator().manual_seed(100 + seed)
    B, NV, Dv, Do = 2, 12, DIMS["image_feat_size"], DIMS["obj_feat_size"]
    D = DIMS["hidden"]
    view_lens = torch.tensor([12, 9])
    n_cand = [3, 2]                      # navigable views per sample (first k views)
    pano = {
        "view_img_fts": torch.randn(B, NV, Dv, generator=g),
        "view_lens": view_lens,
        "loc_fts": torch.cat([torch.randn(B, NV, 4, generator=g).clamp(-1, 1), torch.ones(B, NV, 3)], -1),
        "nav_types": torch.tensor([[1] * n_cand[b] + [0] * (NV - n_cand[b]) for b in range(B)]),
        "obj_img_fts": torch.randn(B, 5, Do, generator=g),
        "obj_lens": torch.tensor([5, 3]),
        "obj_loc_fts": torch.randn(B, 5, 7, generator=g),
    }
    G = 7
    hist = [2, 1]
    gmap_vpids = [[None, "v0", "v1", "c0", "c1", "c2", "f0"], [None, "v0", "c0", "c1", "f0", "f1", None]]
    gmap_visited = torch.tensor([[0, 1, 1, 0, 0, 0, 0], [0, 1, 0, 0, 0, 0, 0]], dtype=torch.bool)
    gmap_masks = torch.tensor([[1, 1, 1, 1, 1, 1, 1], [1, 1, 1, 1, 1, 1, 0]], dtype=torch.bool)
    vp_cand_vpids = [[None, "c0", "c1", "c2"], [None, "c0", "c1"]]
    nav = {
        "data_type": ["r2r", "r2r"],
        "vp_pos_fts": torch.randn(B, NV + 1, 14, generator=g),
        "vp_nav_masks": torch.tensor([[1] + [1] * n_cand[b] + [0] * (NV - n_cand[b]) for b in range(B)], dtype=torch.bool),
        "vp_cand_vpids": vp_cand_vpids,
        "gmap_img_embeds": torch.randn(B, G, D, generator=g),
        "gmap_step_ids": torch.tensor([[0, 1, 2, 0, 0, 0, 0], [0, 1, 0, 0, 0, 0, 0]]),
        "gmap_pos_fts": torch.randn(B, G, 7, generator=g),
        "gmap_masks": gmap_masks,
        "gmap_pair_dists": None,
        "gmap_visited_masks": gmap_visited,
        "gmap_vpids": gmap_vpids,
        "instruction": ["walk past the sofa and stop at the door", "go up the stairs"],
        "history": [["h"] * hist[0], ["h"] * hist[1]],
        "hist_vis": [[torch.randn(D, generator=g) for _ in range(hist[b])] for b in range(B)],
    }
    prompts = []
    for b in range(B):
        n_c = int((gmap_masks[b] & ~gmap_visited[b]).sum()) - 1
        prompts.append("Instruction : " + nav["instruction"][b] + " History : " + " ".join(["<hist>"] * hist[b])
                       + " Candidates : stop " + " ".join(["<cand>"] * n_c) + " Answer : <cls_1>")
    nav["prompts"] = prompts
    targets = torch.tensor([3, 0])
    return pano, nav, targets


def run(precision: str):
    model, tf_version = build_reference_model(precision)
    pano_in, nav_in, targets = make_inputs()
    out = {"meta": {"transformers": tf_version, "torch": torch.__version__, "precision": precision, "dims": DIMS,
                    "reference": "zd11024/NaviLLM (unmodified; 3 stubs, see make_golden.py)"},
           "state_dict": {k: v.detach().clone() for k, v in model.state_dict().items()},
           "pano_in": pano_in, "nav_in": nav_in, "targets": targets}
    model.zero_grad()
    # ---- panorama + navigation + action CE + backward (tasks/agents/mp3d_agent.py:683-757) ----
    pano = model("panorama", dict(pano_in))
    B = pano["pano_embeds"].shape[0]
    vp_img_embeds = torch.cat([torch.zeros_like(pano["pano_embeds"][:, :1]), pano["pano_embeds"]], 1)   # mp3d_agent.py:268-270
    pano_masks = torch.cat([torch.ones(B, 1, dtype=torch.bool), pano["pano_masks"]], 1)
    nav_batch = dict(nav_in)
    nav_batch.update(vp_img_embeds=vp_img_embeds, pano_masks=pano_masks)
    torch.manual_seed(1234)
    nav = model("navigation", nav_batch)
    loss = torch.nn.functional.cross_entropy(nav["fuse_logits"], targets, reduction="sum", ignore_index=-100) / B
    loss.backward()
    out["pano_out"] = {k: (v.detach().clone() if torch.is_tensor(v) else v) for k, v in pano.items()}
    out["nav_out"] = {"fuse_embeds": nav["fuse_embeds"].clone(), "fuse_logits": nav["fuse_logits"].detach().clone(),
                      "loss": loss.detach().clone()}
    grad_names = ["out_head.0.weight", "out_head.0.bias", "lang_model.model.layers.0.self_attn.q_proj.weight",
                  "lang_model.model.layers.1.mlp.down_proj.weight", "lang_model.model.layers.0.input_layernorm.weight",
                  "lang_model.model.norm.weight", "lang_model.model.embed_tokens.weight",
                  "img_embeddings.img_linear.weight", "img_embeddings.pano_encoder.layers.0.self_attn.in_proj_weight",
                  "img_embeddings.pano_encoder.layers.1.linear2.weight", "img_embeddings.mapper.weight",
                  "img_embeddings.layer_norm.weight", "vp_pos_embeddings.0.weight", "gmap_pos_embeddings.1.weight",
                  "gmap_step_embeddings.weight", "token_type_embeddings.weight"]
    named = dict(model.named_parameters())
    out["nav_grads"] = {n: named[n].grad.detach().clone() for n in grad_names if named[n].grad is not None}

    # ---- object grounding (mp3d_agent.py:788-825) ----
    og_batch = {"data_type": ["reverie"] * 2, "obj_embeds": pano["obj_embeds"].detach(), "obj_masks": pano["obj_masks"],
                "obj_loc_fts": pano_in["obj_loc_fts"], "instruction": nav_in["instruction"], "history": nav_in["history"],
                "hist_vis": nav_in["hist_vis"],
                "prompts": ["Find : " + nav_in["instruction"][b] + " " + " ".join(["<hist>"] * len(nav_in["history"][b]))
                            + " Objects : " + " ".join(["<cand>"] * int(pano_in["obj_lens"][b])) + " <cls_1>" for b in range(2)]}
    out["og_in"] = og_batch
    out["og_out"] = {"obj_logits": model("object_grounding", dict(og_batch))["obj_logits"].detach().clone()}

    # ---- summarization, training branch (mp3d_agent.py:880-904) ----
    model.zero_grad()
    sum_batch = dict(nav_in)
    sum_batch.update(vp_img_embeds=vp_img_embeds.detach().clone(), answer=["the door", "upstairs hall"], data_type=["fgr2r"] * 2,
                     prompts=["Summarize : " + " ".join(["<hist>"] * len(nav_in["history"][b])) + " Views : "
                              + " ".join(["<cand>"] * int(nav_in["vp_nav_masks"][b, 1:].sum())) + " Answer :" for b in range(2)])
    out["sum_in"] = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in sum_batch.items()}
    s = model("summarization", dict(sum_batch), training=True)
    s["loss"].backward()
    out["sum_out"] = {"loss": s["loss"].detach().clone()}
    out["sum_grads"] = {n: named[n].grad.detach().clone() for n in
                        ["lang_model.lm_head.weight", "lang_model.model.layers.1.mlp.gate_proj.weight", "vp_pos_embeddings.0.bias"]
                        if named[n].grad is not None}

    # ---- 3dqa, training branch (tasks/agents/llava.py:19-42) ----
    model.zero_grad()
    g = torch.Generator().manual_seed(7)
    qa_batch = {"question": ["what color is the chair", "where is the lamp"], "data_type": ["scanqa"] * 2,
                "answers": [["brown"], ["on the desk"]],
                "features": [torch.randn(5, DIMS["image_feat_size"], generator=g), torch.randn(3, DIMS["image_feat_size"], generator=g)],
                "prompts": ["Scene : " + " ".join(["<cand>"] * n) + " Question : " + q + " Answer :"
                            for n, q in ((5, "what color is the chair"), (3, "where is the lamp"))]}
    out["qa_in"] = qa_batch
    q = model("3dqa", dict(qa_batch), training=True)
    q.loss.backward()
    out["qa_out"] = {"loss": q.loss.detach().clone(), "logits_last": q.logits[:, -1, :].detach().clone()}
    out["qa_grads"] = {n: named[n].grad.detach().clone() for n in
                       ["img_embeddings.img_linear.weight", "lang_model.model.layers.0.mlp.up_proj.weight"]
                       if named[n].grad is not None}
    path = Path(__file__).resolve().parent / f"nav_{precision}.pt"
    torch.save(out, path)
    print("wrote", path, f"{path.stat().st_size / 1e6:.2f} MB")


if __name__ == "__main__":
    for prec in (sys.argv[1:] or ["amp_bf16", "fp32"]):
        # a fresh interpreter state per precision is not needed: the stubs are idempotent
        run(prec)
