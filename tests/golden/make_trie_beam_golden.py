"""Generate tests/golden/generate_trie_beam_amp_bf16.pt: token ids of trie-constrained beam search through the REFERENCE's 3dqa
generation branch (models/nav_model.py:386-402 -> HF GenerationMixin.generate(num_beams=K, prefix_allowed_tokens_fn=...) ->
models/modified_lm.py:89-146) on the golden 3dqa batch.

    NAVILLM_REFERENCE=<reference checkout> python tests/golden/make_trie_beam_golden.py

Runs under the installed transformers 5.5 with the prepare_inputs_for_generation adapter and the per-prompt expansion of the
visual rows of make_beam_golden.py.  The trie is the reference's own tools/trie.py ``Trie``; ``prefix_allowed_tokens_fn`` walks a
beam's generated tokens from its root by ``get_next_node``'s rule (a node without children stays, a token that is not a child
leads to a childless node) without inserting into it, and allows ``get_child_index`` of the node reached, i.e. HF's
PrefixConstrainedLogitsProcessor on the log-probs, after the log-softmax.  Recorded at ``length_penalty=0.0``, where 4.28 and
5.5 normalise alike, for K in {2, 4} x num_return_sequences in {1, K}, with tries of at least K answers so that no returned
sequence depends on how ``torch.topk`` orders -inf candidates.
"""
import random
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import make_golden as MG  # noqa: E402

N_NEW = 10
VIS = ("cand_vis", "hist_vis", "obj_vis")


def tries(bos: int) -> dict:
    """Answer sets as token-id lists: short answers that share prefixes, and an EQA-shaped set (BOS, then 1-3 tokens)."""
    rng = random.Random(0)
    eqa = [[bos] + [rng.randrange(3, 250) for _ in range(rng.randint(1, 3))] for _ in range(8)]
    return {"shared_prefixes": [[21, 22, 23], [21, 22, 30, 31], [21, 40], [50, 51, 52], [60], [61, 62]], "eqa": eqa}


def main():
    precision = "amp_bf16"
    model, tfv = MG.build_reference_model(precision)
    from transformers import GenerationMixin, LlamaForCausalLM
    import models.modified_lm as ml
    from tools.trie import Trie

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
        out_ids, kw = orig_expand(expand_size=expand_size, is_encoder_decoder=is_encoder_decoder, input_ids=input_ids, **model_kwargs)
        for k, v in vis.items():                             # prompt b's block of visual rows once per beam
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
        captured["prompt_len"] = k["input_ids"].shape[1]
        ids = orig(*a, **k)
        captured["ids"] = ids.clone()
        return ids
    lm.generate = spy
    tok = lm.tokenizer

    def allowed_fn(trie):
        def fn(batch_id, sent):
            node = trie.root
            for t in sent[captured["prompt_len"]:].tolist():
                if len(node.child) == 0:
                    break
                node = node.child[t] if t in node.child else None
                if node is None:
                    return [trie.eos]
            return trie.get_child_index(node)
        return fn

    out = {"meta": {"transformers": tfv, "precision": precision, "max_new_tokens": N_NEW, "length_penalty": 0.0}, "runs": []}
    for name, words in tries(tok.bos_token_id).items():
        trie = Trie(tok.bos_token_id, tok.eos_token_id)
        for w in words:
            trie.insert(w)
        for K in (2, 4):
            for n in (1, K):
                with torch.no_grad():
                    sent = model("3dqa", dict(gold["qa_in"]), training=False, max_new_tokens=N_NEW, do_sample=False, num_beams=K,
                                 num_return_sequences=n, length_penalty=0.0,
                                 prefix_allowed_tokens_fn=allowed_fn(trie))["generated_sentences"]
                out["runs"].append({"trie": name, "words": words, "num_beams": K, "num_return_sequences": n,
                                    "ids": captured["ids"], "sentences": sent})
    out["prompt_len"] = captured["prompt_len"]
    GenerationMixin._expand_inputs_for_generation = staticmethod(orig_expand)
    path = Path(__file__).resolve().parent / f"generate_trie_beam_{precision}.pt"
    torch.save(out, path)
    S = out["prompt_len"]
    for r in out["runs"]:
        print(r["trie"], r["num_beams"], r["num_return_sequences"], r["ids"][:, S:].tolist())
    print("wrote", path)


if __name__ == "__main__":
    main()
