"""HF's repetition-penalty / no-repeat-n-gram / min-length processors on the device (csrc/decode.cu nv_logits_process and
nv_beam_topk_processed, ModifiedLlamaForCausalLM.generate(repetition_penalty=, no_repeat_ngram_size=, min_length=,
min_new_tokens=)) against the CPU restatement of transformers 4.28 (tests/processors_oracle.py)."""
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import beam_oracle as BO
from tests import processors_oracle as PO

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
SPECIAL = [32000, 32001, 32002, 32003, 32004]
GOLD = Path(__file__).resolve().parent / "golden"
PROC = dict(repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=4)


def _hist(R, S, t, V, seed, alphabet=None):
    """Prompt rows [R, S] with left pads (id 0), generated rows [R, t]; every history id of row 0 repeats; a small alphabet
    makes n-gram matches frequent."""
    g = torch.Generator().manual_seed(seed)
    hi = alphabet or V
    prompt = torch.randint(0, hi, (R, S), generator=g)
    for r in range(R):
        prompt[r, :int(torch.randint(0, max(1, S // 2), (1,), generator=g))] = 0
    gen = torch.randint(0, hi, (R, t), generator=g)
    prompt[0], gen[0] = 17 % V, 17 % V
    return prompt, gen


def _proc_tuple(kw, eos):
    return (float(kw.get("repetition_penalty", 1.0)), kw.get("no_repeat_ngram_size", 0), kw.get("min_length", 0),
            kw.get("min_new_tokens", 0), eos)


CASES = [dict(repetition_penalty=1.3), dict(repetition_penalty=0.8, no_repeat_ngram_size=1), dict(no_repeat_ngram_size=2),
         dict(no_repeat_ngram_size=4, min_length=2000), dict(repetition_penalty=1.2, no_repeat_ngram_size=3, min_new_tokens=200)]


@pytest.mark.parametrize("V,alphabet", [(32006, None), (32006, 40), (262, 20)], ids=["V32006", "V32006-small-alphabet", "tiny"])
@pytest.mark.parametrize("R,S,t", [(1, 5, 0), (8, 300, 17), (64, 1024, 128), (3, 2, 1)])
def test_logits_process_kernel_matches_oracle(cuda_dev, V, alphabet, R, S, t):
    from navillm_b200 import ops
    eos = 2
    prompt, gen = _hist(R, S, t, V, seed=R * 7 + S + t, alphabet=alphabet)
    G = 128 + 8
    for i, kw in enumerate(CASES):
        g = torch.Generator(device=cuda_dev).manual_seed(i)
        logits = (torch.randn(R, V, generator=g, device=cuda_dev) * 3).to(bf16)
        logits[:, 3] = float("-inf")
        logits[:, 4] = 0.0
        want = PO.process(logits.cpu(), torch.cat([prompt, gen], 1), S, eos_token_id=eos, **kw)
        pids = torch.zeros(R, S + 5, dtype=torch.int32, device=cuda_dev)       # a wider buffer: only S columns are read
        pids[:, :S] = prompt.int().to(cuda_dev)
        width = torch.tensor([S], dtype=torch.int32, device=cuda_dev)
        hist = torch.zeros(R, G, dtype=torch.int32, device=cuda_dev)
        hist[:, :t] = gen.int().to(cuda_dev)
        for append in (False, True):                                            # t already stored / the last one appended
            if append and t == 0:
                continue
            hl = torch.full((R,), t - 1 if append else t, dtype=torch.int32, device=cuda_dev)
            h = hist.clone()
            if append:
                h[:, t - 1] = -5
            got = logits.clone()
            ops.logits_process_(got, pids, width, h, hl, gen[:, t - 1].int().to(cuda_dev) if append else None, _proc_tuple(kw, eos))
            torch.cuda.synchronize()
            assert torch.equal(got.cpu().view(torch.int16), want.view(torch.int16)), (kw, append)
            assert hl.cpu().tolist() == [t] * R and torch.equal(h[:, :t], hist[:, :t])


@pytest.mark.parametrize("B,K", [(1, 2), (8, 4), (4, 8), (16, 8)])
def test_beam_topk_processed_matches_oracle(cuda_dev, B, K):
    from navillm_b200 import ops
    V, S, t, G, eos = 32006, 257, 33, 128, 2
    prompt, gen = _hist(B * K, S, t, V, seed=B * 10 + K, alphabet=60)
    prompt = prompt.view(B, K, S)[:, 0]
    g = torch.Generator(device=cuda_dev).manual_seed(B + K)
    logits = (torch.randn(B * K, V, generator=g, device=cuda_dev) * 3).to(bf16)
    bs = (torch.randn(B * K, generator=g, device=cuda_dev) * 4).float()
    special = torch.tensor(SPECIAL, dtype=torch.int32, device=cuda_dev)
    hist = torch.zeros(B * K, G, dtype=torch.int32, device=cuda_dev)
    hist[:, :t] = gen.int().to(cuda_dev)
    pstate = torch.zeros(B, 5, dtype=torch.int32, device=cuda_dev)
    pstate[:, 0] = t
    pids = prompt.int().to(cuda_dev).contiguous()
    width = torch.tensor([S], dtype=torch.int32, device=cuda_dev)
    out = lambda: (torch.empty((B, 2 * K), dtype=torch.float32, device=cuda_dev), torch.empty((B, 2 * K), dtype=torch.int32, device=cuda_dev),
                   torch.empty((B, 2 * K), dtype=torch.int32, device=cuda_dev))
    # all off: the processed instantiation is the plain one
    a, b_ = out(), out()
    ops.beam_topk(logits, special, bs, K, *a)
    ops.beam_topk_processed(logits, special, bs, K, *b_, pids, width, hist, pstate, (1.0, 0, 0, 0, eos))
    assert all(torch.equal(x, y) for x, y in zip(a, b_))
    x = logits.float().cpu()
    x[:, SPECIAL] = float("-inf")
    m = x.max(dim=1, keepdim=True).values
    ls64 = torch.log(torch.exp((x - m).double()).sum(dim=1, keepdim=True))
    lp = ((x - m) - ls64.float()).to(bf16)
    hist_ids = torch.cat([prompt.repeat_interleave(K, 0), gen], 1)
    for kw in CASES:
        c = out()
        ops.beam_topk_processed(logits, special, bs, K, *c, pids, width, hist, pstate, _proc_tuple(kw, eos))
        torch.cuda.synchronize()
        plp = PO.process(lp, hist_ids, S, eos_token_id=eos, **kw)
        scores = (plp.float() + bs.cpu()[:, None]).view(B, K * V)
        ws, wt, wp = BO.top_candidates(scores, K)
        srt = torch.sort(scores, dim=1, descending=True, stable=True)[0]
        for b in range(B):
            if srt[b, 2 * K - 1] == srt[b, 2 * K] and torch.isfinite(srt[b, 2 * K]):
                continue                                                        # a tie straddles rank 2K
            assert torch.equal(c[0][b].cpu(), ws[b]), (kw, b)
            assert c[1][b].cpu().long().tolist() == wt[b].tolist() and c[2][b].cpu().long().tolist() == wp[b].tolist(), (kw, b)


# ---------------------------------------------------------------------------------------------------------------------
# generate()
# ---------------------------------------------------------------------------------------------------------------------
def _tiny(cuda_dev, rows=None):
    from tests.test_beam_gpu import _qa
    from tests.test_navmodel_gpu import build_model
    from tests.test_oracle_golden import load
    g, cfg, tok = load("amp_bf16")
    model, _ = build_model(g, cuda_dev)
    text, cand = _qa(g, cfg, tok, rows)
    kw = dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev),
              eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id)
    return g, cfg, tok, model.lang_model, text, cand, kw


def test_generate_greedy_and_beams_match_oracle(cuda_dev):
    from tests.test_beam_gpu import near_tie_ok
    from tests.test_fullwidth_parity_gpu import compare_greedy_rows
    g, cfg, tok, lm, text, cand, kw = _tiny(cuda_dev)
    S, n_new = text["input_ids"].shape[1], 12
    for proc in (dict(repetition_penalty=1.3), dict(no_repeat_ngram_size=2), dict(min_new_tokens=4, min_length=S + 6), PROC):
        ref, steps = PO.greedy_generate(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], cand_vis=cand,
                                        max_new_tokens=n_new, eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id,
                                        stop_on_eos=False, return_logits=True, **proc)
        for graph in (False, True):
            ids = lm.generate(max_new_tokens=n_new, stop_on_eos=False, use_cuda_graph=graph, **proc, **kw).cpu()
            matched, _ = compare_greedy_rows(ids, ref, steps, S, n_new, tag=f"greedy {proc} graph={graph}")
            assert sum(matched) >= n_new, matched
        for K in (2, 4):
            bkw = dict(num_beams=K, max_new_tokens=n_new, length_penalty=0.0)
            ref, steps = PO.beam_generate(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], cand_vis=cand,
                                          eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id, return_steps=True, **bkw, **proc)
            outs = [lm.generate(use_cuda_graph=graph, **bkw, **proc, **kw).cpu() for graph in (False, True, True)]
            assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2]), (proc, K)
            near_tie_ok(outs[0], ref, steps, S, 1, tag=f"beams K={K} {proc}")


@pytest.mark.skipif(not (GOLD / "generate_processors_amp_bf16.pt").exists(), reason="processor goldens not recorded")
def test_generate_matches_reference_goldens(cuda_dev):
    """The reference's own 3dqa branch under transformers 5.5 (tests/golden/make_processors_golden.py; fp32 processing of
    bf16 logits there, bf16 here and in 4.28): equal tokens, or a divergence at a step where the oracle's decision is a bf16
    near-tie."""
    from tests.test_beam_gpu import near_tie_ok
    from tests.test_fullwidth_parity_gpu import compare_greedy_rows
    gold = torch.load(GOLD / "generate_processors_amp_bf16.pt", weights_only=False)
    g, cfg, tok, lm, text, cand, kw = _tiny(cuda_dev)
    S, n_new = gold["prompt_len"], gold["meta"]["max_new_tokens"]
    assert S == text["input_ids"].shape[1]
    for run in gold["runs"]:
        K, proc = run["num_beams"], run["proc"]
        extra = dict(num_beams=K, length_penalty=0.0) if K > 1 else {}
        ids = lm.generate(max_new_tokens=n_new, **extra, **proc, **kw).cpu()
        if torch.equal(ids, run["ids"]):
            continue
        if K == 1:
            _, steps = PO.greedy_generate(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], cand_vis=cand,
                                          max_new_tokens=n_new, eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id,
                                          return_logits=True, **proc)
            L = min(ids.shape[1], run["ids"].shape[1])
            compare_greedy_rows(ids[:, :L], run["ids"][:, :L], steps, S, min(L - S, len(steps)), tag=f"golden {proc}")
        else:
            _, steps = PO.beam_generate(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], cand_vis=cand, num_beams=K,
                                        max_new_tokens=n_new, eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id,
                                        length_penalty=0.0, return_steps=True, **proc)
            near_tie_ok(ids, run["ids"], steps, S, 1, tag=f"golden K={K} {proc}")


@pytest.mark.parametrize("kv", ["bf16", "fp8"])
def test_generate_mode_properties_with_processors(cuda_dev, kv):
    """Graph = eager; device trie = host trie; a user logits_processor= (host path) = the device path; N samples = the prompts
    repeated N times -- all with the processors on."""
    from oracle import navillm_oracle as O
    from tests.test_trie_decode_gpu import WORDS, _bos_words
    from tests.test_trie_table_cpu import make_trie
    g, cfg, tok, lm, text, cand, kw = _tiny(cuda_dev)
    prev = lm.set_kv_cache_dtype(kv)
    try:
        for do_sample in (False, True):
            base = dict(max_new_tokens=14, do_sample=do_sample, temperature=0.9, **kw)
            outs = []
            for graph in (False, True, True):
                torch.manual_seed(11)
                outs.append(lm.generate(use_cuda_graph=graph, **PROC, **base).cpu())
            assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2]), do_sample
            torch.manual_seed(11)
            host = lm.generate(logits_processor=[lambda ids, s: s], **PROC, **base).cpu()
            assert torch.equal(host, outs[0]), do_sample
            # min_new_tokens bans EOS, the only token a trie leaf allows: such a row is degenerate and the call takes the
            # miss-rerun host path; without it the device walk stands
            trie = make_trie(_bos_words(tok, WORDS), eos=tok.eos_token_id)
            for tproc, path in ((dict(repetition_penalty=1.3, no_repeat_ngram_size=2), "device"), (PROC, "device_miss_host")):
                tkw = dict(base, max_new_tokens=7, **tproc)
                torch.manual_seed(5)
                h = lm.generate(logits_processor=[O.TrieLogitsProcessor(trie)], **tkw).cpu()
                for graph in (False, True):
                    stats = {}
                    torch.manual_seed(5)
                    d = lm.generate(trie=trie, stats=stats, use_cuda_graph=graph, **tkw).cpu()
                    assert torch.equal(h, d), (do_sample, graph, tproc)
                    assert stats["trie_path"] == path, (do_sample, graph, tproc, stats["trie_path"])
        N = 3
        skw = dict(kw, input_ids=text["input_ids"], attention_mask=text["attention_mask"])
        for graph in (False, True):
            torch.manual_seed(3)
            many = lm.generate(max_new_tokens=10, do_sample=True, num_return_sequences=N, use_cuda_graph=graph, **PROC, **skw).cpu()
            rows = [b for b in range(text["input_ids"].shape[0]) for _ in range(N)]
            from tests.test_beam_gpu import _qa
            t2, c2 = _qa(g, cfg, tok, rows)
            torch.manual_seed(3)
            rep = lm.generate(max_new_tokens=10, do_sample=True, use_cuda_graph=graph, input_ids=t2["input_ids"],
                              attention_mask=t2["attention_mask"], cand_vis=c2.to(cuda_dev), eos_token_id=tok.eos_token_id,
                              pad_token_id=tok.unk_token_id, **PROC).cpu()
            assert torch.equal(many, rep), graph
        for K in (2, 4):
            b = [lm.generate(num_beams=K, max_new_tokens=10, use_cuda_graph=gr, **PROC, **kw).cpu() for gr in (False, True)]
            assert torch.equal(b[0], b[1]), K
    finally:
        lm.set_kv_cache_dtype(prev)


def test_generate_fp8_weights_with_processors(cuda_dev):
    """quantize_weights_fp8() with processors: the bf16 path on the rounded weights."""
    g, cfg, tok, lm, text, cand, kw = _tiny(cuda_dev)
    lm.quantize_weights_fp8()
    got = [lm.generate(max_new_tokens=10, use_cuda_graph=gr, **PROC, **kw).cpu() for gr in (False, True)]
    gotb = lm.generate(num_beams=4, max_new_tokens=10, **PROC, **kw).cpu()
    lm.drop_fp8_weights()
    assert torch.equal(got[0], lm.generate(max_new_tokens=10, use_cuda_graph=False, **PROC, **kw).cpu()) and torch.equal(got[0], got[1])
    assert torch.equal(gotb, lm.generate(num_beams=4, max_new_tokens=10, use_cuda_graph=False, **PROC, **kw).cpu())


def test_sampled_tokens_lie_in_the_oracle_support(cuda_dev):
    g, cfg, tok, lm, text, cand, kw = _tiny(cuda_dev)
    S = text["input_ids"].shape[1]
    proc = dict(repetition_penalty=1.5, no_repeat_ngram_size=2, min_new_tokens=6)
    torch.manual_seed(0)
    ids = lm.generate(max_new_tokens=12, do_sample=True, top_k=20, stop_on_eos=False, **proc, **kw).cpu()
    sup = PO.sample_support(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], ids[:, S:], cand_vis=cand, top_k=20,
                            eos_token_id=tok.eos_token_id, **proc)
    for t, s in enumerate(sup):
        assert bool(s[torch.arange(ids.shape[0]), ids[:, S + t]].all()), t
        if t < 6:
            assert not bool(s[:, tok.eos_token_id].any())


def test_defaults_launch_no_processor_and_bad_values_raise(cuda_dev, monkeypatch):
    import navillm_b200.ops as ops_mod
    from navillm_b200 import _lib
    g, cfg, tok, lm, text, cand, kw = _tiny(cuda_dev)
    calls = []
    real = _lib.check

    def spy(status, what):
        calls.append(what)
        return real(status, what)
    monkeypatch.setattr(ops_mod, "check", spy)
    off_kw = dict(repetition_penalty=1.0, no_repeat_ngram_size=0, min_length=0, min_new_tokens=None)
    for extra in (dict(), dict(num_beams=4)):
        base = lm.generate(max_new_tokens=8, use_cuda_graph=False, **extra, **kw).cpu()
        first = list(calls)
        calls.clear()
        off = lm.generate(max_new_tokens=8, use_cuda_graph=False, **off_kw, **extra, **kw).cpu()
        assert torch.equal(base, off) and calls == first                   # the same launches, eager
        lm.generate(max_new_tokens=8, **extra, **kw)
        keys = set(lm._decode_states)
        assert torch.equal(lm.generate(max_new_tokens=8, **off_kw, **extra, **kw).cpu(), base)
        assert set(lm._decode_states) == keys                              # the same graph-state key: no new state
        assert not any("logits_process" in c or "topk_processed" in c for c in first)
        calls.clear()
        lm.generate(max_new_tokens=8, **PROC, **extra, **kw)
        assert any("logits_process" in c or "topk_processed" in c for c in calls)
        calls.clear()
    for bad in (dict(repetition_penalty=0.0), dict(repetition_penalty=2), dict(no_repeat_ngram_size=-1), dict(min_length=-3),
                dict(min_new_tokens=-1)):
        with pytest.raises(ValueError):
            lm.generate(max_new_tokens=4, **bad, **kw)


def test_generate_c3_shape_with_processors_vs_oracle(cuda_dev):
    """2 Vicuna-width layers at C3's shape (B = 8, 256 <cand>, 32 new tokens, vocab 32006), repetition_penalty=1.3,
    no_repeat_ngram_size=3: greedy tokens row by row against the oracle under the near-tie rule of test_fullwidth_parity_gpu."""
    from tests.test_fullwidth_parity_gpu import _full_navmodel, _oracle_cfg, compare_greedy_rows
    B, N_CAND, N_NEW = 8, 256, 32
    proc = dict(repetition_penalty=1.3, no_repeat_ngram_size=3)
    model, tok = _full_navmodel(cuda_dev, base_vocab=32000)
    sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items() if k.startswith("lang_model.")}
    rng = np.random.RandomState(5)
    prompts = []
    for b in range(B):
        words = " ".join(f"w{i}" for i in rng.randint(0, 5000, size=int(rng.randint(30, 61))))
        prompts.append("Scene " + " ".join(["<cand>"] * N_CAND) + " Question " + words + " Answer")
    text = tok(prompts)
    cand = torch.randn(B * N_CAND, 4096, generator=torch.Generator().manual_seed(9))
    ref, steps = PO.greedy_generate(sd, _oracle_cfg(tok, "amp_bf16"), text["input_ids"], text["attention_mask"], cand_vis=cand,
                                    max_new_tokens=N_NEW, stop_on_eos=False, return_logits=True, eos_token_id=tok.eos_token_id, **proc)
    S0 = text["input_ids"].shape[1]
    outs = []
    for graph in (False, True):
        ids = model.lang_model.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev),
                                        max_new_tokens=N_NEW, stop_on_eos=False, use_cuda_graph=graph, eos_token_id=tok.eos_token_id,
                                        **proc).cpu()
        matched, cut = compare_greedy_rows(ids, ref, steps, S0, N_NEW, tag=f"c3 processors graph={graph}")
        print(f"\n[c3 processors, graph={graph}] matched tokens per row {matched} of {N_NEW}; near-tie cuts {cut}")
        assert sum(matched) >= B * N_NEW // 4, matched
        outs.append(ids)
    assert torch.equal(outs[0], outs[1])
