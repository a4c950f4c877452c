"""Top-p in the device sampler (nv_sample) and several samples per prompt from one shared prefill
(generate(do_sample=True, num_return_sequences=N)).

The sampler is checked against tests/sampling_oracle.py run by torch on the CPU, whose cumsum rule (fp32 running sum, bf16
partials) the kernel follows.  The multi-sample path is checked against the same call on the prompts repeated N times: both
draw [B * N] uniform numbers per token, the decode GEMMs see the same rows, and the beam attention kernel is bit for bit the
contiguous one, so the tokens must be equal in every row."""
import numpy as np
import pytest
import torch

from tests import sampling_oracle as SO
from tests.test_beam_gpu import _qa
from tests.test_top_p_cpu import SPECIAL, V, score_rows

pytestmark = pytest.mark.gpu


def _sample(lg, u, temperature, top_k, top_p, dev):
    from navillm_b200 import ops
    B = lg.shape[0]
    special = torch.tensor(SPECIAL, dtype=torch.int32, device=dev)
    fin = torch.zeros(B, dtype=torch.int32, device=dev)
    nxt = torch.full((B,), -1, dtype=torch.int32, device=dev)
    probs = torch.empty(B, V, dtype=torch.float32, device=dev)
    ops.sample(lg.to(dev), special, fin, 2, 0, True, temperature, top_k, top_p, u.to(dev), nxt, probs_out=probs)
    return nxt.cpu(), probs.cpu()


def _near_cut(scores, temperature, top_k, top_p):
    """Rows whose oracle running sum lies within one bf16 ulp of the threshold's rounding boundary at some position: there
    the kernel's softmax denominator (another fp32 summation order) may move a probability by one ulp and the cut by one."""
    s = scores.float() / temperature if temperature != 1.0 else scores.float()
    s = s.to(torch.bfloat16)
    if top_k:
        kth = torch.topk(s, top_k)[0][..., -1, None]
        s = s.masked_fill(s < kth, float("-inf"))
    p = torch.sort(s, dim=-1, stable=True).values.softmax(-1).float()
    run = torch.from_numpy(np.cumsum(p.numpy(), -1, dtype=np.float32))
    thr = float(torch.tensor(1 - top_p).to(torch.bfloat16))
    ulp = 2.0 ** (np.floor(np.log2(max(thr, 2 ** -30))) - 8)
    return ((run - (thr + ulp)).abs() <= 2 * ulp).any(-1)


def _rules_straddle(scores, temperature, top_k, top_p, dev):
    """Rows where torch's CPU cumsum (fp32 running sum, the rule nv_sample follows) and its CUDA cumsum (bf16 adds) of the
    sorted top-k softmax put some position on different sides of ``<= bf16(1 - top_p)``, both computed on the [B, V] batch."""
    s = scores / temperature if temperature != 1.0 else scores
    s = s.masked_fill(SO.O.sampling_probs(scores, temperature, top_k) == 0, float("-inf"))
    srt = torch.sort(s, dim=-1, stable=True).values
    thr = float(torch.tensor(1 - top_p).to(torch.bfloat16))
    cpu = srt.softmax(-1).cumsum(-1).float() <= thr
    gpu = srt.to(dev).softmax(-1).cumsum(-1).float().cpu() <= thr
    return (cpu != gpu)[:, :-1].any(-1)


@pytest.mark.parametrize("top_p", [0.0, 0.3, 0.9, 0.999])
@pytest.mark.parametrize("temperature,top_k", [(1.0, 50), (0.7, 50), (1.0, 8), (1.0, 0), (0.8, 0)])
def test_top_p_distribution_matches_oracle(cuda_dev, temperature, top_k, top_p):
    B = 24
    scores = torch.cat([score_rows(8, seed=1), score_rows(8, seed=2), score_rows(8, seed=3)])
    scores[8:16] = (scores[8:16].float() * 0.2).to(torch.bfloat16)          # flatter rows: top_k = 0 cuts deep in the tail
    u = torch.rand(B, generator=torch.Generator().manual_seed(4))
    nxt, probs = _sample(scores, u, temperature, top_k, top_p, cuda_dev)
    ref = SO.sampling_probs(scores, temperature, top_k, top_p).float()
    near = _near_cut(scores, temperature, top_k, top_p)
    same = (probs > 0).eq(ref > 0).all(-1)
    off = (~same).nonzero().flatten().tolist()
    print(f"\n[top_p={top_p} T={temperature} k={top_k}] support differs in rows {off}; rows near the cut {near.nonzero().flatten().tolist()}")
    assert all(bool(near[b]) for b in off), off
    assert len(off) <= 2, off
    ok = same.nonzero().flatten()
    r, p = ref[ok], probs[ok]
    ulp = torch.where(r > 0, 2.0 ** (torch.floor(torch.log2(r.clamp_min(1e-38))) - 7), torch.zeros_like(r))
    assert bool(((p - r).abs() <= ulp).all())
    for b in range(B):                                       # the draw lies in the kernel's support
        assert probs[b, int(nxt[b])] > 0
    # Against the oracle run by torch on CUDA, whose bf16 cumsum adds in bf16 in a batch-dependent order (DESIGN §2): a row may
    # differ only where that running sum and the CPU rule's fall on different sides of the threshold at some position, and
    # every other row has the same support.
    cuda_ref = SO.sampling_probs(scores.to(cuda_dev), temperature, top_k, top_p).float().cpu()
    differs = ~(probs > 0).eq(cuda_ref > 0).all(-1)
    straddle = _rules_straddle(scores, temperature, top_k, top_p, cuda_dev)
    print(f"[top_p={top_p} T={temperature} k={top_k}] rows whose support differs from torch on CUDA: "
          f"{differs.nonzero().flatten().tolist()}; rows where the two cumsum rules straddle the threshold: "
          f"{straddle.nonzero().flatten().tolist()}")
    assert not bool((differs & ~straddle).any()), (differs & ~straddle).nonzero().flatten().tolist()


def test_sample_topk_and_top_p_1_return_the_recorded_bits(cuda_dev):
    """nv_sample_topk, and nv_sample at top_p = 1, return the ids and the bit-exact distribution that nv_sample_topk returned
    before top-p was added (tests/golden/sample_topk.json, recorded by make_sample_topk_golden.py)."""
    import json
    from pathlib import Path
    from navillm_b200 import ops
    from tests.golden import make_sample_topk_golden as MG
    gold = json.loads((Path(__file__).parent / "golden" / "sample_topk.json").read_text())
    scores, u = MG.inputs()
    assert MG.sha(scores) == gold["scores_sha256"] and MG.sha(u) == gold["u_sha256"], "the recorded inputs changed"

    def topk(lg, special, fin, nxt, probs, ud, temperature, top_k):
        ops.sample_topk(lg, special, fin, 2, 0, True, temperature, top_k, ud, nxt, probs_out=probs)

    def top_p_1(lg, special, fin, nxt, probs, ud, temperature, top_k):
        ops.sample(lg, special, fin, 2, 0, True, temperature, top_k, 1.0, ud, nxt, probs_out=probs)

    for case in gold["cases"]:
        for fn in (topk, top_p_1):
            ids, h = MG.run(fn, scores, u, case["temperature"], case["top_k"], cuda_dev)
            assert ids == case["next"] and h == case["probs_sha256"], (fn.__name__, case)


@pytest.mark.parametrize("top_k", [50, 0])
def test_top_p_empirical_frequencies(cuda_dev, top_k):
    """20k draws of one row: frequencies of the kept tokens agree with the oracle's probabilities (chi-square)."""
    g = torch.Generator().manual_seed(3)
    row = (torch.randn(1, V, generator=g) * (1.0 if top_k else 0.2) + 0).to(torch.bfloat16)
    row[:, SPECIAL] = float("-inf")
    n = 20000
    ref = SO.sampling_probs(row, 0.9, top_k, 0.9).float()[0]
    ref = ref / ref.sum()
    u = torch.rand(n, generator=torch.Generator().manual_seed(0))
    nxt, _ = _sample(row.expand(n, V).contiguous(), u, 0.9, top_k, 0.9, cuda_dev)
    counts = torch.bincount(nxt.long(), minlength=V).float()
    assert float(counts[ref == 0].sum()) == 0
    kept = ref > 0
    exp = ref[kept] * n
    chi2 = float((((counts[kept] - exp) ** 2) / exp).sum())
    dof = int(kept.sum()) - 1
    assert chi2 < dof + 6 * (2 * dof) ** 0.5, (chi2, dof)


# ---------------------------------------------------------------------------------------------------------------------
# generate(do_sample=True, num_return_sequences=N)
# ---------------------------------------------------------------------------------------------------------------------
_MODEL = {}


def _tiny(dev):
    from tests.test_navmodel_gpu import build_model
    from tests.test_oracle_golden import load
    if "tiny" not in _MODEL:
        g, cfg, tok = load("amp_bf16")
        _MODEL["tiny"] = (build_model(g, dev)[0], g, cfg, tok)
    return _MODEL["tiny"]


def _both_arms(lm, text, cand, text_rep, cand_rep, N, seed=0, **kw):
    dev = lm._device()
    torch.manual_seed(seed)
    shared = lm.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(dev), do_sample=True,
                         num_return_sequences=N, **kw).cpu()
    torch.manual_seed(seed)
    rep = lm.generate(input_ids=text_rep["input_ids"], attention_mask=text_rep["attention_mask"], cand_vis=cand_rep.to(dev),
                      do_sample=True, **kw).cpu()
    return shared, rep


def _prompts(g, cfg, tok, B, N):
    n_gold = len(g["qa_in"]["prompts"])
    rows = [b % n_gold for b in range(B)]
    text, cand = _qa(g, cfg, tok, rows)
    text_rep, cand_rep = _qa(g, cfg, tok, [r for r in rows for _ in range(N)])
    return text, cand, text_rep, cand_rep


@pytest.mark.parametrize("N", [2, 4, 16])
@pytest.mark.parametrize("B", [1, 3, 8])
def test_multi_sample_equals_repeated_prompts(cuda_dev, B, N):
    model, g, cfg, tok = _tiny(cuda_dev)
    lm = model.lang_model
    text, cand, text_rep, cand_rep = _prompts(g, cfg, tok, B, N)
    kw = dict(max_new_tokens=12, top_p=0.9, temperature=1.2, eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id)
    a, b = _both_arms(lm, text, cand, text_rep, cand_rep, N, seed=B * 10 + N, **kw)
    S = text["input_ids"].shape[1]
    assert a.shape[0] == B * N and torch.equal(a[:, :S], text["input_ids"].repeat_interleave(N, 0))
    assert torch.equal(a, b)
    assert len({tuple(r) for r in a[:, S:].tolist()}) > 1 or B * N == 1


@pytest.mark.parametrize("variant", ["eager", "no_eos_stop", "one_token", "fp8_kv", "fp8_weights", "top_p_1", "top_k_0"])
def test_multi_sample_variants(cuda_dev, variant):
    model, g, cfg, tok = _tiny(cuda_dev)
    if variant == "fp8_weights":                                # quantize_weights_fp8() rounds in place: not the shared model
        from tests.test_navmodel_gpu import build_model
        model = build_model(g, cuda_dev)[0]
    lm = model.lang_model
    B, N = 3, 4
    text, cand, text_rep, cand_rep = _prompts(g, cfg, tok, B, N)
    kw = dict(max_new_tokens=16, top_p=0.8, eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id)
    if variant == "eager":
        kw["use_cuda_graph"] = False
    elif variant == "no_eos_stop":
        kw["stop_on_eos"] = False
    elif variant == "one_token":
        kw["max_new_tokens"] = 1
    elif variant == "top_p_1":
        kw["top_p"] = 1.0
    elif variant == "top_k_0":
        kw["top_k"] = 0
    prev = lm.set_kv_cache_dtype("fp8") if variant == "fp8_kv" else None
    if variant == "fp8_weights":
        lm.quantize_weights_fp8()
    try:
        for seed in (1, 2):                                     # the second call replays the captured graphs
            a, b = _both_arms(lm, text, cand, text_rep, cand_rep, N, seed=seed, **kw)
            assert torch.equal(a, b), (variant, seed)
        if variant == "no_eos_stop":
            assert a.shape[1] == text["input_ids"].shape[1] + 16
        if variant == "one_token":
            assert a.shape[1] == text["input_ids"].shape[1] + 1
    finally:
        if prev is not None:
            lm.set_kv_cache_dtype(prev)


def test_multi_sample_vicuna_width(cuda_dev):
    """2 Vicuna-width layers, vocab 32006, B = 4 prompts with 128 <cand> tokens, N = 4: 16 rows through the skinny decode
    GEMMs and the beam attention over a 256-row prompt cache."""
    from tests.test_fullwidth_parity_gpu import _full_navmodel
    B, N, N_CAND = 4, 4, 128
    model, tok = _full_navmodel(cuda_dev, base_vocab=32000)
    lm = model.lang_model
    rng = np.random.RandomState(3)
    prompts = []
    for b in range(B):
        words = " ".join(f"w{i}" for i in rng.randint(0, 5000, size=int(rng.randint(20, 41))))
        prompts.append("Scene " + " ".join(["<cand>"] * N_CAND) + " Question " + words + " Answer")
    cand = torch.randn(B * N_CAND, 4096, generator=torch.Generator().manual_seed(2))
    text = tok(prompts)
    text_rep = tok([p for p in prompts for _ in range(N)])
    cand_rep = torch.cat([cand[b * N_CAND:(b + 1) * N_CAND] for b in range(B) for _ in range(N)])
    kw = dict(max_new_tokens=24, top_p=0.95, eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id, stop_on_eos=False)
    a, b = _both_arms(lm, text, cand, text_rep, cand_rep, N, **kw)
    assert torch.equal(a, b)


def test_3dqa_returns_n_sentences_per_question_in_hf_order(cuda_dev):
    """3dqa with num_return_sequences = N gives the sentences of the 3dqa mode on each question repeated N times (same seed):
    sentence b * N + j is a sample of question b."""
    model, g, cfg, tok = _tiny(cuda_dev)
    qa = dict(g["qa_in"])
    n_q, N = len(qa["question"]), 3
    rep = {k: ([x for x in v for _ in range(N)] if isinstance(v, (list, tuple)) and len(v) == n_q else v) for k, v in qa.items()}
    kw = dict(training=False, do_sample=True, top_p=0.9, temperature=1.5, max_new_tokens=6)
    with torch.no_grad():
        torch.manual_seed(5)
        a = model("3dqa", qa, num_return_sequences=N, **kw)["generated_sentences"]
        torch.manual_seed(5)
        b = model("3dqa", rep, **kw)["generated_sentences"]
    assert len(a) == N * n_q and a == b
    assert len(set(a)) > n_q                                    # the samples of a question differ, so the order is pinned


def test_greedy_and_beams_ignore_top_p(cuda_dev):
    model, g, cfg, tok = _tiny(cuda_dev)
    lm = model.lang_model
    text, cand = _qa(g, cfg, tok)
    kw = dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev), max_new_tokens=8,
              eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id)
    assert torch.equal(lm.generate(**kw).cpu(), lm.generate(top_p=0.3, **kw).cpu())
    assert torch.equal(lm.generate(num_beams=4, num_return_sequences=2, **kw).cpu(),
                       lm.generate(num_beams=4, num_return_sequences=2, top_p=0.3, **kw).cpu())


def test_error_cases(cuda_dev):
    model, g, cfg, tok = _tiny(cuda_dev)
    lm = model.lang_model
    text, cand = _qa(g, cfg, tok)
    kw = dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev), max_new_tokens=4)
    for p in (-0.1, 1.5):
        with pytest.raises(ValueError, match="top_p"):
            lm.generate(do_sample=True, top_p=p, **kw)
    with pytest.raises(NotImplementedError, match="do_sample"):
        lm.generate(num_return_sequences=2, **kw)
    with pytest.raises(NotImplementedError, match="processors"):
        lm.generate(do_sample=True, num_return_sequences=2, trie=object(), **kw)
    with pytest.raises(NotImplementedError, match="processors"):
        lm.generate(do_sample=True, num_return_sequences=2, logits_processor=[lambda i, s: s], **kw)
    with pytest.raises(NotImplementedError, match="beam sampling"):
        lm.generate(num_beams=2, do_sample=True, num_return_sequences=2, **kw)
    with pytest.raises(NotImplementedError, match="group"):
        lm.generate(num_beams=4, num_beam_groups=2, do_sample=True, **kw)
