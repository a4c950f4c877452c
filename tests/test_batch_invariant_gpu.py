"""Batch-invariant mode end to end (``set_batch_invariant(True)``): a prompt's hidden states, generated ids and scores in every
decoding mode, and answer scores are bitwise the same when it runs alone and inside batches of
2 / 16 / 17 / 64 / 65 prompts with random companions at random positions (other lengths, so other padding).  The model is
the tiny golden NavModel of tests/golden; the kernels' own invariance at Vicuna-7B widths is
tests/test_batch_invariant_kernels_gpu.py."""
import random

import pytest
import torch

pytestmark = pytest.mark.gpu

BATCHES = (2, 16, 17, 64, 65)
N_NEW = 32


@pytest.fixture(scope="module")
def tiny(cuda_dev):
    from tests.test_navmodel_gpu import build_model
    from tests.test_oracle_golden import load
    g, cfg, tok = load("amp_bf16")
    model, _ = build_model(g, cuda_dev)
    lm = model.lang_model
    prev = model.set_batch_invariant(True)
    assert prev is False
    yield model, lm, tok
    model.set_batch_invariant(False)


def _prompts(tok, n, seed, lo=6, hi=40):
    """n random prompts of ordinary tokens (no special ids), random lengths."""
    rng = random.Random(seed)
    first = max(tok.special.values()) + 1 if getattr(tok, "special", None) else 16
    V = len(tok) if hasattr(tok, "__len__") else 256
    return [[tok.bos_token_id] + [rng.randrange(first, V) for _ in range(rng.randint(lo, hi))] for _ in range(n)]


def _pack(prompts, dev, pad):
    """Left-padded input_ids / attention_mask, as the tokenizer pads."""
    S = max(len(p) for p in prompts)
    ids = torch.full((len(prompts), S), pad, dtype=torch.long)
    mask = torch.zeros((len(prompts), S), dtype=torch.long)
    for i, p in enumerate(prompts):
        ids[i, S - len(p):] = torch.tensor(p)
        mask[i, S - len(p):] = 1
    return ids.to(dev), mask.to(dev)


def _batches(target, tok, seed):
    """(batch prompts, row of the target) for every size in BATCHES, companions random, the target at a random row."""
    rng = random.Random(seed)
    for B in BATCHES:
        comp = _prompts(tok, B - 1, seed * 1000 + B)
        r = rng.randrange(B)
        yield comp[:r] + [target] + comp[r:], r


def _bits(t):
    return t.contiguous().view(torch.int16) if t.dtype == torch.bfloat16 else t.contiguous().view(torch.int32)


def _gen(lm, tok, prompts, dev, **kw):
    ids, mask = _pack(prompts, dev, tok.unk_token_id)
    out = lm.generate(ids, mask, max_new_tokens=N_NEW, eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id,
                      stop_on_eos=False, return_dict_in_generate=True, output_scores=True, **kw)
    return out, ids.shape[1]


def test_hidden_states_and_logits(cuda_dev, tiny):
    """lang_model(...) hidden states and logits at every row of the prompt, with the batch below and above 1024 rows."""
    model, lm, tok = tiny
    for t, target in enumerate(_prompts(tok, 2, 5)):
        with torch.no_grad():
            ids, mask = _pack([target], cuda_dev, tok.unk_token_id)
            solo = lm(ids, mask, return_logits=True)
            h0, l0 = solo.hidden_states[0, -len(target):], solo.logits[0, -len(target):]
            rows = 0
            for prompts, r in _batches(target, tok, 17 + t):
                ids, mask = _pack(prompts, cuda_dev, tok.unk_token_id)
                rows = max(rows, int(mask.sum()))
                o = lm(ids, mask, return_logits=True)
                assert torch.equal(_bits(o.hidden_states[r, -len(target):]), _bits(h0)), (len(prompts), r)
                assert torch.equal(_bits(o.logits[r, -len(target):]), _bits(l0)), (len(prompts), r)
    assert rows > 1024


@pytest.mark.parametrize("mode", ["greedy", "beam", "contrastive", "lookup", "group_beam"])
def test_generate_ids_and_scores(cuda_dev, tiny, mode):
    model, lm, tok = tiny
    # beams at length_penalty 0: HF normalises a finished beam's score by the padded length of the batch's prompts
    kw = dict(greedy={}, beam=dict(num_beams=4, length_penalty=0.0), contrastive=dict(penalty_alpha=0.6, top_k=4),
              lookup=dict(prompt_lookup_num_tokens=4),
              group_beam=dict(num_beams=4, num_beam_groups=2, diversity_penalty=0.5, length_penalty=0.0))[mode]
    target = _prompts(tok, 1, 23)[0]
    solo, S1 = _gen(lm, tok, [target], cuda_dev, **kw)
    for prompts, r in _batches(target, tok, 29):
        out, S = _gen(lm, tok, prompts, cuda_dev, **kw)
        assert torch.equal(out.sequences[r, S:].cpu(), solo.sequences[0, S1:].cpu()), (mode, len(prompts), r)
        if mode in ("beam", "group_beam"):
            assert torch.equal(out.sequences_scores[r].cpu(), solo.sequences_scores[0].cpu())
            K = 4                                              # per-step scores: the prompt's K beam rows
            for a, b in zip(out.scores, solo.scores):
                assert torch.equal(_bits(a[r * K:(r + 1) * K]), _bits(b[:K]))
        else:
            for a, b in zip(out.scores, solo.scores):
                assert torch.equal(_bits(a[r]), _bits(b[0])), (mode, len(prompts), r)


def test_lookup_equals_greedy(cuda_dev, tiny):
    model, lm, tok = tiny
    prompts = _prompts(tok, 17, 31)
    greedy, _ = _gen(lm, tok, prompts, cuda_dev)
    look, _ = _gen(lm, tok, prompts, cuda_dev, prompt_lookup_num_tokens=4)
    assert torch.equal(greedy.sequences.cpu(), look.sequences.cpu())


def test_sampled_step0_scores_and_samples(cuda_dev, tiny):
    """A sampled call's step-0 scores of each row; N = 4 samples per prompt equal the prompts repeated 4 times."""
    model, lm, tok = tiny
    target = _prompts(tok, 1, 37)[0]
    torch.manual_seed(0)
    solo, _ = _gen(lm, tok, [target], cuda_dev, do_sample=True, top_k=20)
    for prompts, r in _batches(target, tok, 41):
        torch.manual_seed(0)
        out, _ = _gen(lm, tok, prompts, cuda_dev, do_sample=True, top_k=20)
        assert torch.equal(_bits(out.scores[0][r]), _bits(solo.scores[0][0])), (len(prompts), r)
    prompts = _prompts(tok, 5, 43)
    torch.manual_seed(1)
    many, _ = _gen(lm, tok, prompts, cuda_dev, do_sample=True, num_return_sequences=4)
    torch.manual_seed(1)
    rep, _ = _gen(lm, tok, [p for p in prompts for _ in range(4)], cuda_dev, do_sample=True)
    assert torch.equal(many.sequences.cpu(), rep.sequences.cpu())
    for a, b in zip(many.scores, rep.scores):
        assert torch.equal(_bits(a), _bits(b))


def test_score_answers(cuda_dev, tiny):
    from tests.test_trie_beam_gpu import GOLD_WORDS
    from tests.test_trie_table_cpu import make_trie
    model, lm, tok = tiny
    trie = make_trie(GOLD_WORDS, eos=tok.eos_token_id)
    target = _prompts(tok, 1, 47)[0]
    ids, mask = _pack([target], cuda_dev, tok.unk_token_id)
    solo = lm.score_answers(ids, mask, trie)
    for prompts, r in _batches(target, tok, 53):
        ids, mask = _pack(prompts, cuda_dev, tok.unk_token_id)
        got = lm.score_answers(ids, mask, trie)
        assert torch.equal(got["logprob"][r].cpu(), solo["logprob"][0].cpu()), (len(prompts), r)


# ---------------------------------------------------------------------------------------------------------------------
# panorama encoder, navigation, PrefixKVCache, object grounding
# ---------------------------------------------------------------------------------------------------------------------
def _pad1(t, L):
    """t [1, n, ...] zero-padded along dim 1 to L."""
    return torch.cat([t, t.new_zeros((1, L - t.shape[1]) + tuple(t.shape[2:]))], 1)


def _cat_eps(eps, L=None):
    """One batch from one-episode dicts: tensors with a second dimension padded to the longest (or L), lists joined."""
    out = {}
    for k in eps[0]:
        vs = [e[k] for e in eps]
        if torch.is_tensor(vs[0]):
            if vs[0].dim() >= 2:
                n = L if L is not None and k in ("view_img_fts", "loc_fts", "nav_types") else max(v.shape[1] for v in vs)
                vs = [_pad1(v, n) for v in vs]
            out[k] = torch.cat(vs, 0)
        elif isinstance(vs[0], list):
            out[k] = [x for v in vs for x in v]
        else:
            out[k] = vs[0]
    return out


def _placed(n, seed):
    """A batch order of n episodes and the row of episode 0 in it."""
    order = list(range(n))
    random.Random(seed).shuffle(order)
    return order, order.index(0)


def test_panorama_encoder(cuda_dev, tiny):
    """View and object embeddings of an episode alone (no padding) and inside 16 episodes padded to 12 views."""
    model, lm, tok = tiny
    g = torch.Generator().manual_seed(61)
    F, O = model.img_embeddings.img_linear.in_features, 48
    eps = []
    for i in range(16):
        n, m = 3 + (5 * i) % 10, 1 + i % 5
        eps.append(dict(view_img_fts=torch.randn(1, n, F, generator=g), view_lens=torch.tensor([n]),
                        loc_fts=torch.randn(1, n, 7, generator=g), nav_types=torch.randint(0, 2, (1, n), generator=g),
                        obj_img_fts=torch.randn(1, m, O, generator=g), obj_lens=torch.tensor([m]),
                        obj_loc_fts=torch.randn(1, m, 7, generator=g)))
    order, r = _placed(16, 67)
    run = lambda b: model("panorama", {k: v.to(cuda_dev) for k, v in b.items()})
    with torch.no_grad():
        alone = run(eps[0])
        both = run(_cat_eps([eps[i] for i in order], L=12))
    n, m = eps[0]["view_lens"].item(), eps[0]["obj_lens"].item()
    assert torch.equal(both["pano_embeds"][r, :n].view(torch.int32), alone["pano_embeds"][0, :n].view(torch.int32))
    assert torch.equal(both["obj_embeds"][r, :m].view(torch.int32), alone["obj_embeds"][0, :m].view(torch.int32))


def _nav_episodes(d, n_pairs, steps, seed):
    """[episode][step] one-episode navigation batches (two at a time from test_prefix_reuse_gpu._nav_batch)."""
    from tests.test_prefix_reuse_gpu import _nav_batch
    g = torch.Generator().manual_seed(seed)
    rng = random.Random(seed)
    words = "walk past the sofa and stop at the door of the kitchen leave room turn left right go up stairs".split()
    eps = []
    for _ in range(n_pairs):
        instr = [" ".join(rng.choice(words) for _ in range(rng.randint(3, 14))) for _ in range(2)]
        hist = [[], []]
        pair = [[], []]
        for step in range(steps):
            batch = _nav_batch(d, step, hist, g, instr)
            for b in range(2):
                e = {k: (v[b:b + 1] if torch.is_tensor(v) or isinstance(v, list) else v) for k, v in batch.items()}
                pair[b].append(e)
            hist = [h + [torch.randn(d["hidden"], generator=g)] for h in hist]
        eps += pair
    return eps


def test_navigation_step_and_prefix_cache(cuda_dev, monkeypatch):
    """fuse_logits of one episode alone and inside 16, from scratch and over a PrefixKVCache for two steps.  The candidate
    shuffle (one CPU randperm per episode, as in the reference) is held to the identity: it is input randomness drawn from
    one stream per batch, like a sampled token, not arithmetic."""
    from navillm_b200.modified_lm import PrefixKVCache
    from tests.test_prefix_reuse_gpu import _build
    monkeypatch.setattr(torch, "randperm", lambda n, *a, **k: torch.arange(n))
    model, d = _build(cuda_dev)
    model.set_batch_invariant(True)
    eps = _nav_episodes(d, 8, 2, 71)
    order, r = _placed(16, 73)

    def run(batch, cache=None):
        b = dict(batch)
        b["hist_vis"] = [[v.to(cuda_dev) for v in vs] for vs in b["hist_vis"]]
        b = {k: (v.to(cuda_dev) if torch.is_tensor(v) else v) for k, v in b.items()}
        with torch.no_grad():
            return model("navigation", b, training=False, **({} if cache is None else {"prefix_cache": cache}))["fuse_logits"]

    for step in range(2):
        alone = run(eps[0][step])
        both = run(_cat_eps([eps[i][step] for i in order]))
        assert torch.equal(both[r].view(torch.int16), alone[0].view(torch.int16)), step
    c1 = PrefixKVCache(model.lang_model, batch_size=1, max_len=256)
    c16 = PrefixKVCache(model.lang_model, batch_size=16, max_len=256)
    for step in range(2):
        alone = run(eps[0][step], c1)
        both = run(_cat_eps([eps[i][step] for i in order]), c16)
        assert torch.equal(both[r].view(torch.int16), alone[0].view(torch.int16)), ("cached", step)
    model.set_batch_invariant(False)


def test_object_grounding(cuda_dev, tiny):
    """obj_logits of an episode alone and inside 16 (the golden episodes at random rows, objects padded to 8)."""
    from tests.test_oracle_golden import load
    model, lm, tok = tiny
    og = load("amp_bf16")[0]["og_in"]
    eps = [{k: (v[b:b + 1] if torch.is_tensor(v) or isinstance(v, list) else v) for k, v in og.items()} for b in range(2)]
    pick = [0] + [random.Random(79 + i).randrange(2) for i in range(15)]
    order, r = _placed(16, 83)
    run = lambda b: model("object_grounding", {k: (v.to(cuda_dev) if torch.is_tensor(v) else v) for k, v in b.items()})
    with torch.no_grad():
        alone = run(eps[0])["obj_logits"]
        both = run(_cat_eps([eps[pick[i]] for i in order] + [dict(eps[0], obj_embeds=_pad1(eps[0]["obj_embeds"], 8),
                                                                  obj_masks=_pad1(eps[0]["obj_masks"], 8),
                                                                  obj_loc_fts=_pad1(eps[0]["obj_loc_fts"], 8))]))["obj_logits"]
    n = alone.shape[1]
    assert torch.equal(both[r, :n].view(torch.int16), alone[0].view(torch.int16))
    assert torch.isfinite(alone[0].float()).any()
