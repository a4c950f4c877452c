"""Generate tests/golden/generate_processors_{fp32,amp_bf16}.pt: token ids of the REFERENCE's 3dqa generation branch
(models/nav_model.py:386-402 -> HF GenerationMixin.generate(**kwargs) -> models/modified_lm.py:89-146) on the golden 3dqa batch
with HF's logits processors on: repetition_penalty=1.3, no_repeat_ngram_size in {2, 3} and min_new_tokens=4, each alone and all
together, greedy and with beams K in {2, 4} at length_penalty=0.

    NAVILLM_REFERENCE=<reference checkout> python tests/golden/make_processors_golden.py

Runs under the installed transformers 5.5 with the adapters of make_generate_golden.py / make_beam_golden.py.  5.5 casts the
logits to fp32 before the processors, where 4.28 (the reference's pin) runs them on the bf16 scores: the fp32 goldens are 4.28's
tokens exactly; the amp_bf16 ones may differ from 4.28 at bf16 near-ties (tests/processors_oracle.py).
"""
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import make_golden as MG  # noqa: E402

N_NEW = 10
VIS = ("cand_vis", "hist_vis", "obj_vis")
SETTINGS = [dict(repetition_penalty=1.3), dict(no_repeat_ngram_size=2), dict(no_repeat_ngram_size=3), dict(min_new_tokens=4),
            dict(repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=4)]


def main():
    for precision in ("fp32", "amp_bf16"):
        model, tfv = MG.build_reference_model(precision)
        from transformers import GenerationMixin, LlamaForCausalLM
        import models.modified_lm as ml

        def prepare_inputs_for_generation(self, input_ids, past_key_values=None, attention_mask=None, inputs_embeds=None,
                                          cand_vis=None, hist_vis=None, obj_vis=None, **kwargs):
            model_inputs = LlamaForCausalLM.prepare_inputs_for_generation(
                self, input_ids, past_key_values=past_key_values, attention_mask=attention_mask, inputs_embeds=inputs_embeds, **kwargs)
            empty = past_key_values is None or (hasattr(past_key_values, "get_seq_length") and past_key_values.get_seq_length() == 0)
            if empty:
                model_inputs["cand_vis"], model_inputs["hist_vis"], model_inputs["obj_vis"] = cand_vis, hist_vis, obj_vis
            return model_inputs

        ml.ModifiedLlamaForCausalLM.prepare_inputs_for_generation = prepare_inputs_for_generation
        lm = model.lang_model
        ids_of = {"cand_vis": lm.cand_token_id[0], "hist_vis": lm.hist_token_id[0], "obj_vis": lm.obj_token_id[0]}
        orig_expand = GenerationMixin._expand_inputs_for_generation

        def expand(expand_size=1, is_encoder_decoder=False, input_ids=None, **model_kwargs):
            vis = {k: model_kwargs.pop(k) for k in VIS if k in model_kwargs}
            out_ids, kw = orig_expand(expand_size=expand_size, is_encoder_decoder=is_encoder_decoder, input_ids=input_ids,
                                      **model_kwargs)
            for k, v in vis.items():                     # prompt b's block of visual rows once per beam (make_beam_golden.py)
                if v is None or expand_size == 1:
                    kw[k] = v
                else:
                    counts = (input_ids == ids_of[k]).sum(1).tolist()
                    kw[k] = torch.cat([blk for blk in v.split(counts, 0) for _ in range(expand_size)], 0)
            return out_ids, kw

        GenerationMixin._expand_inputs_for_generation = staticmethod(expand)
        gold = torch.load(Path(__file__).resolve().parent / f"nav_{precision}.pt", weights_only=False)
        model.load_state_dict(gold["state_dict"], strict=True)
        model.eval()
        captured = {}
        orig = lm.generate

        def spy(*a, **k):
            ids = orig(*a, **k)
            captured["ids"] = ids.clone()
            captured["prompt_len"] = k["input_ids"].shape[1]
            return ids
        lm.generate = spy
        out = {"meta": {"transformers": tfv, "precision": precision, "max_new_tokens": N_NEW, "length_penalty": 0.0}, "runs": []}
        for K in (1, 2, 4):
            for proc in SETTINGS:
                extra = dict(num_beams=K, length_penalty=0.0) if K > 1 else {}
                with torch.no_grad():
                    model("3dqa", dict(gold["qa_in"]), training=False, max_new_tokens=N_NEW, do_sample=False, **extra, **proc)
                out["runs"].append({"num_beams": K, "proc": proc, "ids": captured["ids"]})
        out["prompt_len"] = captured["prompt_len"]
        GenerationMixin._expand_inputs_for_generation = staticmethod(orig_expand)
        path = Path(__file__).resolve().parent / f"generate_processors_{precision}.pt"
        torch.save(out, path)
        S = out["prompt_len"]
        print("wrote", path, [(r["num_beams"], r["proc"], r["ids"][:, S:].tolist()) for r in out["runs"][:5]])


if __name__ == "__main__":
    main()
