"""Golden vectors for the `fuse_obj` branch of the panorama encoder (models/image_embedding.py:78-94; `--fuse_obj`,
tools/parser.py:95: "whether fuse object features for REVERIE and SOON"), from the UNMODIFIED reference's
ImageEmbeddings run on CPU in eval() mode at tiny dimensions.  Needs a checkout of the reference, named by the
NAVILLM_REFERENCE environment variable (nothing under tests/ reads it at test time).

    python tests/golden/make_fuse_obj_golden.py     # writes tests/golden/pano_fuse_obj.pt

Recorded: the module's state_dict, the inputs, `pano_embeds / pano_masks / obj_embeds / obj_masks`, and the gradients
of every parameter for the scalar  sum(pano_embeds * wp) + sum(obj_embeds * wo)  with recorded random weights."""
import os
import sys
import types
from pathlib import Path

import torch

REF = os.environ["NAVILLM_REFERENCE"]
OUT = Path(__file__).resolve().parent / "pano_fuse_obj.pt"
DIMS = dict(pano_hidden=128, pano_heads=2, pano_inter=256, image_feat_size=64, obj_feat_size=48, output_size=256, num_pano_layers=2)


def main():
    sys.path.insert(0, REF)
    from models.image_embedding import ImageEmbeddings
    cfg = types.SimpleNamespace(hidden_size=DIMS["pano_hidden"], num_attention_heads=DIMS["pano_heads"],
                                intermediate_size=DIMS["pano_inter"], hidden_act="gelu", hidden_dropout_prob=0.1,
                                image_feat_size=DIMS["image_feat_size"], angle_feat_size=4, obj_feat_size=DIMS["obj_feat_size"],
                                output_size=DIMS["output_size"], num_pano_layers=DIMS["num_pano_layers"])
    torch.manual_seed(0)
    mod = ImageEmbeddings(cfg, use_obj=True, fuse_obj=True).eval()
    g = torch.Generator().manual_seed(1)
    B, N, O = 4, 8, 6
    view_lens = torch.tensor([8, 5, 8, 3])
    obj_lens = torch.tensor([6, 2, 0, 4])
    inp = {
        "view_img_fts": torch.randn(B, N, DIMS["image_feat_size"], generator=g),
        "view_lens": view_lens,
        "loc_fts": torch.randn(B, N, 7, generator=g),
        "nav_types": torch.randint(0, 2, (B, N), generator=g),
        "obj_img_fts": torch.randn(B, O, DIMS["obj_feat_size"], generator=g),
        "obj_lens": obj_lens,
        "obj_loc_fts": torch.randn(B, O, 7, generator=g),
    }
    out = mod.forward_panorama_per_step(**{k: v.clone() for k, v in inp.items()})
    wp = torch.randn(out["pano_embeds"].shape, generator=g)
    wo = torch.randn(out["obj_embeds"].shape, generator=g)
    loss = (out["pano_embeds"] * wp).sum() + (out["obj_embeds"] * wo).sum()
    loss.backward()
    grads = {n: p.grad.clone() for n, p in mod.named_parameters() if p.grad is not None}
    no_grad = [n for n, p in mod.named_parameters() if p.grad is None]
    torch.save({"dims": DIMS, "state_dict": {k: v.clone() for k, v in mod.state_dict().items()}, "inputs": inp,
                "pano_embeds": out["pano_embeds"].detach(), "pano_masks": out["pano_masks"], "obj_embeds": out["obj_embeds"].detach(),
                "obj_masks": out["obj_masks"], "wp": wp, "wo": wo, "loss": loss.detach(), "grads": grads, "no_grad": no_grad,
                "torch": torch.__version__}, OUT)
    print("wrote", OUT, "loss", float(loss), "params without grad:", no_grad)


if __name__ == "__main__":
    main()
