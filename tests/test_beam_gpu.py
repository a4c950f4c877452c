"""Beam search on the device (csrc/decode.cu nv_beam_topk / nv_beam_select / nv_decode_attn_rope_beam[_fp8], and
ModifiedLlamaForCausalLM.generate(num_beams=K)), piece by piece and end to end, against the CPU restatement of transformers
4.28's beam search (tests/beam_oracle.py)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import beam_oracle as BO
from tests.test_decode_ops_gpu import _tables

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
SPECIAL = [32000, 32001, 32002, 32003, 32004]


# ---------------------------------------------------------------------------------------------------------------------
# nv_beam_topk
# ---------------------------------------------------------------------------------------------------------------------
def _topk_run(logits, bs, K, first_step=False):
    from navillm_b200 import ops
    B = bs.numel() // K
    dev = logits.device
    cs = torch.empty((B, 2 * K), dtype=torch.float32, device=dev)
    ct = torch.empty((B, 2 * K), dtype=torch.int32, device=dev)
    cp = torch.empty((B, 2 * K), dtype=torch.int32, device=dev)
    special = torch.tensor(SPECIAL, dtype=torch.int32, device=dev)
    ops.beam_topk(logits, special, bs, K, cs, ct, cp, first_step=first_step)
    torch.cuda.synchronize()
    return cs.cpu(), ct.cpu().long(), cp.cpu().long()


@pytest.mark.parametrize("B", [1, 8, 64])
@pytest.mark.parametrize("K", [2, 4, 8])
def test_beam_topk_matches_torch(cuda_dev, B, K):
    V = 32006
    g = torch.Generator(device=cuda_dev).manual_seed(B * 100 + K)
    logits = (torch.randn(B * K, V, generator=g, device=cuda_dev) * 3).to(bf16)
    bs = (torch.randn(B * K, generator=g, device=cuda_dev) * 4).float()
    cs, ct, cp = _topk_run(logits, bs, K)
    # restatement: fp64 row sums, the fp32 subtraction order of the kernel, one rounding to bf16, the fp32 add
    x = logits.float().cpu()
    x[:, SPECIAL] = float("-inf")
    m = x.max(dim=1, keepdim=True).values
    ls64 = torch.log(torch.exp((x - m).double()).sum(dim=1, keepdim=True))
    lp = ((x - m) - ls64.float()).to(bf16).float()
    torch_lp = F.log_softmax(x, dim=-1).to(bf16).float()
    same = (lp == torch_lp) | torch.isinf(lp)
    assert same.float().mean().item() > 0.99, "log-probs off the fp32 log_softmax beyond its own rounding"
    scores = (lp + bs.cpu()[:, None]).view(B, K * V)
    ws, wt, wp = BO.top_candidates(scores, K)
    sorted_all = torch.sort(scores, dim=1, descending=True, stable=True)[0]
    for b in range(B):
        if sorted_all[b, 2 * K - 1] == sorted_all[b, 2 * K]:
            continue                                      # a tie straddles rank 2K: the set is not unique
        assert torch.equal(cs[b], ws[b]), (b, cs[b], ws[b])
        assert torch.equal(ct[b], wt[b]) and torch.equal(cp[b], wp[b]), b


def test_beam_topk_first_step_and_forced_ties(cuda_dev):
    """Equal scores order by flat index (beam-major, then token); at the first step every beam reads the prompt's prefill row
    and beams 1..K-1 carry -1e9, so only beam 0 expands."""
    V, K, B = 32006, 4, 3
    logits = torch.full((B * K, V), -5.0, dtype=bf16, device=cuda_dev)
    logits[:, 100:140] = 2.0                              # 40 equal maxima per row
    bs = torch.zeros(B * K, device=cuda_dev)
    cs, ct, cp = _topk_run(logits, bs, K)
    for b in range(B):
        assert cp[b].tolist() == [0] * 8 and ct[b].tolist() == list(range(100, 108))
        assert (cs[b] == cs[b, 0]).all()
    bs = torch.tensor([0.0, -1e9, -1e9, -1e9] * B, device=cuda_dev)
    g = torch.Generator(device=cuda_dev).manual_seed(3)
    pre = torch.randn(B, V, generator=g, device=cuda_dev).to(bf16)
    big = torch.empty((B * K, V), dtype=bf16, device=cuda_dev)
    big[:B] = pre
    cs, ct, cp = _topk_run(big, bs, K, first_step=True)
    # beam 0's scores as the kernel forms them (the restatement of test_beam_topk_matches_torch): near -11 a bf16 log-prob
    # step is 2^-4, so logits one bf16 step apart often share a score, and the tie goes to the lower token index
    x = pre.float().cpu()
    x[:, SPECIAL] = float("-inf")
    m = x.max(dim=1, keepdim=True).values
    lp = ((x - m) - torch.log(torch.exp((x - m).double()).sum(dim=1, keepdim=True)).float()).to(bf16).float()
    ws, wt = torch.sort(lp, dim=1, descending=True, stable=True)
    for b in range(B):
        assert (cp[b] == 0).all()
        assert torch.equal(ct[b], wt[b, :2 * K]) and torch.equal(cs[b], ws[b, :2 * K]), (b, ct[b], wt[b, :2 * K])


# ---------------------------------------------------------------------------------------------------------------------
# nv_beam_select
# ---------------------------------------------------------------------------------------------------------------------
def _select_state(B, K, G, plens, dev):
    st = dict(beam_score=torch.zeros(B * K, device=dev), hist=torch.zeros(B * K, G, dtype=torch.int32, device=dev),
              src=torch.zeros(B * K, G, dtype=torch.int32, device=dev),
              hyp_score=torch.zeros(B, K + 1, dtype=torch.float64, device=dev),
              hyp_meta=torch.zeros(B, K, 2, dtype=torch.int32, device=dev),
              hyp_tok=torch.zeros(B, K, G, dtype=torch.int32, device=dev),
              prompt_state=torch.zeros(B, 5, dtype=torch.int32, device=dev),
              next_ids=torch.zeros(B * K, dtype=torch.int32, device=dev), lens=torch.zeros(B * K, dtype=torch.int32, device=dev))
    st["hyp_score"][:, K] = 1e9
    st["prompt_state"][:, 1] = torch.tensor(plens, dtype=torch.int32)
    return st


@pytest.mark.parametrize("K,lp,early", [(2, 1.0, False), (4, 0.0, False), (4, 2.0, True), (8, 1.0, False)])
def test_beam_select_matches_cpu_scorer(cuda_dev, K, lp, early):
    from navillm_b200 import ops
    B, G, S, steps, eos, pad = 6, 64, 11, 60, 2, 0
    gen = torch.Generator().manual_seed(K * 10 + int(lp))
    plens = [S - b % 3 for b in range(B)]
    st = _select_state(B, K, G, plens, cuda_dev)
    norm = ops.beam_norm(S, G, lp).to(cuda_dev)
    hyps = [BO.BeamHypotheses(K, lp, early) for _ in range(B)]
    done = [False] * B
    history = [[] for _ in range(B * K)]
    src_ref = [[] for _ in range(B * K)]
    for t in range(steps):
        # a random candidate table: descending scores, distinct (token, parent) pairs, EOS injected at random ranks
        sc = torch.sort(-(torch.rand(B, 2 * K, generator=gen) * 3 + 0.5 * t), dim=1, descending=True)[0].float()
        tok = torch.randint(3, 500, (B, 2 * K), generator=gen)
        par = torch.randint(0, K, (B, 2 * K), generator=gen)
        eos_at = torch.rand(B, 2 * K, generator=gen) < (0.15 if t > 3 else 0.0)
        tok[eos_at] = eos
        for b in range(B):                                  # the (parent, token) pairs of one prompt are distinct
            e = (tok[b] == eos).nonzero().flatten()
            tok[b, e[K:]] = 700                             # at least K non-EOS candidates, as top-2K over a vocabulary gives
            seen = set()
            for r in range(2 * K):
                while (int(par[b, r]), int(tok[b, r])) in seen:
                    tok[b, r] = int(tok[b, r]) + 1 if int(tok[b, r]) != eos else 600 + r
                seen.add((int(par[b, r]), int(tok[b, r])))
        nsc, ntok, npar = BO.process(hyps, done, S, t, history, sc, tok, par, eos, pad)
        ops.beam_select(sc.to(cuda_dev), tok.int().to(cuda_dev), par.int().to(cuda_dev), st["beam_score"], st["hist"], st["src"],
                        st["hyp_score"], st["hyp_meta"], st["hyp_tok"], st["prompt_state"], st["next_ids"], st["lens"], norm, eos,
                        pad, early)
        rows = (torch.arange(B)[:, None] * K + npar).view(-1)
        history = [history[int(r)] + [int(x)] for r, x in zip(rows, ntok.view(-1))]
        src_ref = [src_ref[int(r)] + [i] for i, r in enumerate(rows)]
        torch.cuda.synchronize()
        ps = st["prompt_state"].cpu()
        assert ps[:, 4].tolist() == [int(d) for d in done], t
        assert st["next_ids"].cpu().tolist() == ntok.view(-1).tolist(), t
        assert torch.equal(st["beam_score"].cpu(), nsc.view(-1)), t
        live = [r for r in range(B * K) if not done[r // K]]
        hist = st["hist"].cpu()[:, :t + 1]
        src = st["src"].cpu()[:, :t + 1]
        for r in live:
            assert hist[r].tolist() == history[r], (t, r)
            assert src[r].tolist() == src_ref[r], (t, r)
        assert st["lens"].cpu().tolist() == [plens[r // K] + t for r in range(B * K)]
        hs, hm, ht = st["hyp_score"].cpu(), st["hyp_meta"].cpu(), st["hyp_tok"].cpu()
        for b in range(B):
            n = int(ps[b, 2])
            assert n == len(hyps[b]), (t, b)
            kept = sorted(range(n), key=lambda i: int(hm[b, i, 1]))
            got = [(float(hs[b, i]), ht[b, i, :int(hm[b, i, 0])].tolist()) for i in kept]
            assert got == hyps[b].beams, (t, b)
            assert float(hs[b, K]) == hyps[b].worst_score
    assert any(done) or K == 8


# ---------------------------------------------------------------------------------------------------------------------
# nv_decode_attn_rope_beam[_fp8]
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
@pytest.mark.parametrize("K", [1, 4, 8])
def test_beam_attention_is_contiguous_attention_through_src(cuda_dev, K, fp8):
    """Every step position 0..127 with ragged prompt lengths: the beam kernel equals nv_decode_attn_rope[_fp8] on a contiguous
    cache [prompt keys of r / K ; generated keys gathered through src] (the same bytes), bit for bit, and writes the new k / v
    at (r, i) as the contiguous kernel writes them at row lens[r]."""
    from navillm_b200 import ops
    from tests.test_fp8_kv_gpu import _round_rows
    H, B, G, Sp = 2, 3, 128, 128
    HD, R, Smax = H * 128, B * K, Sp + G
    plens = [37, 64, 5]
    cos_t, sin_t = _tables(Smax + 8, H, cuda_dev)
    g = torch.Generator(device=cuda_dev).manual_seed(K * 3 + int(fp8))
    u8 = lambda t: t.view(torch.uint8) if t.dtype == ops.fp8 else t
    pk = torch.randn(B, Sp, HD, generator=g, device=cuda_dev).to(bf16)
    pv = torch.randn(B, Sp, HD, generator=g, device=cuda_dev).to(bf16)
    kg = torch.zeros(R, G, HD, dtype=bf16, device=cuda_dev)
    vg = torch.zeros(R, G, HD, dtype=bf16, device=cuda_dev)
    if fp8:                                   # (bytes, exponents) per cache
        pk, pv, kg, vg = (_round_rows(t) for t in (pk, pv, kg, vg))
    caches = (pk, pv, kg, vg) if fp8 else ((pk,), (pv,), (kg,), (vg,))
    src = torch.zeros(R, G, dtype=torch.int32, device=cuda_dev)
    plens_d = torch.tensor(plens, dtype=torch.int32, device=cuda_dev)
    gen = torch.Generator().manual_seed(7)
    rr = torch.arange(R, device=cuda_dev)

    def contiguous(pc, gc, i):
        out = torch.zeros((R, Smax) + tuple(pc.shape[2:]), dtype=u8(pc).dtype, device=cuda_dev)
        for r in range(R):
            P = plens[r // K]
            out[r, :P] = u8(pc)[r // K, :P]
            if i:
                out[r, P:P + i] = u8(gc)[src[r, :i].long(), torch.arange(i, device=cuda_dev)]
        return out.view(pc.dtype)

    for i in range(G):
        # a beam reorder: each row takes a random parent's history of its prompt, then its own slot i
        par = (torch.randint(0, K, (R,), generator=gen) + (torch.arange(R) // K) * K).to(cuda_dev)
        src[:, :i] = src[par, :i].clone()
        src[:, i] = rr.int()
        lens = torch.tensor([plens[r // K] + i for r in range(R)], dtype=torch.int32, device=cuda_dev)
        qkv = torch.randn(R, 3 * HD, generator=g, device=cuda_dev).to(bf16)
        ref = [[contiguous(p, c, i) for p, c in zip(pc, gc)] for pc, gc in ((caches[0], caches[2]), (caches[1], caches[3]))]
        if fp8:
            out = ops.decode_attn_rope_beam_fp8(qkv, lens, cos_t, sin_t, pk[0], pv[0], pk[1], pv[1], plens_d, kg[0], vg[0], kg[1],
                                                vg[1], src, K, H)
            want = ops.decode_attn_rope_fp8(qkv, lens, cos_t, sin_t, ref[0][0], ref[1][0], ref[0][1], ref[1][1], H)
        else:
            out = ops.decode_attn_rope_beam(qkv, lens, cos_t, sin_t, pk, pv, plens_d, kg, vg, src, K, H)
            want = ops.decode_attn_rope(qkv, lens, cos_t, sin_t, ref[0][0], ref[1][0], H)
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int16), want.view(torch.int16)), (K, i)
        for gc, rc in zip(caches[2:], ref):                  # the new rows: what the contiguous kernel appended
            for a, w in zip(gc, rc):
                assert torch.equal(u8(a)[rr, i], u8(w)[rr, lens.long()]), i


# ---------------------------------------------------------------------------------------------------------------------
# generate(num_beams=K) end to end
# ---------------------------------------------------------------------------------------------------------------------
def _qa(g, cfg, tok, rows=None):
    """The golden 3dqa prompts (``rows`` picks and repeats them) and their <cand> vectors in row-major token order."""
    from oracle import navillm_oracle as O
    sd = g["state_dict"]
    qa = g["qa_in"]
    feats = qa["features"]
    lens = torch.tensor([f.shape[0] for f in feats])
    view = torch.stack([torch.cat([f, f.new_zeros(int(lens.max()) - f.shape[0], f.shape[1])], 0) for f in feats], 0)
    pano = O.forward_panorama(sd, cfg, view, lens)
    pe = pano["pano_embeds"] + O._pos_embed(torch.zeros(pano["pano_embeds"].shape[:2] + (14,)), sd, "vp_pos_embeddings")
    pe = pe + sd["token_type_embeddings.weight"][0]
    rows = list(range(len(qa["prompts"]))) if rows is None else rows
    return tok([qa["prompts"][i] for i in rows]), torch.cat([pe[i][pano["pano_masks"][i]] for i in rows], 0)


def near_tie_ok(ids, ref, steps, S, n_ret, tag=""):
    """Per prompt: the device rows equal the oracle's, unless the oracle's decision was inside the bf16 noise floor: two of its
    best 2K + 1 scores within 3 bf16 ulp of their magnitude (the rule of test_fullwidth_parity_gpu's greedy check) at a step
    at or before the first differing column, or at the last step (which ranks the final beams).  Returns the matched generated
    columns per prompt."""
    def tie(t, b):
        sc = steps[t][b]
        fin = sc[torch.isfinite(sc)]
        ulp = torch.exp2(torch.floor(torch.log2(fin[:-1].abs().clamp_min(1e-30))) - 7)
        return bool(((fin[:-1] - fin[1:]).abs() <= 3 * ulp).any())

    matched = []
    for b in range(ids.shape[0] // n_ret):
        a, r = ids[b * n_ret:(b + 1) * n_ret], ref[b * n_ret:(b + 1) * n_ret]
        L = min(a.shape[1], r.shape[1])
        if a.shape == r.shape and torch.equal(a, r):
            matched.append(L - S)
            continue
        diff = (a[:, :L] != r[:, :L]).any(0).nonzero()
        first = (int(diff[0]) if len(diff) else L) - S
        matched.append(first)
        ok = any(tie(t, b) for t in range(min(first + 1, len(steps)))) or tie(len(steps) - 1, b)
        assert ok, (tag, b, first, a[:, S:].tolist(), r[:, S:].tolist())
    return matched


@pytest.mark.parametrize("K,n_ret,lp,rows", [(2, 1, 1.0, None), (4, 4, 0.0, None), (4, 2, 2.0, None), (4, 1, 1.0, [0]),
                                             (2, 2, 1.0, [0, 1, 0])], ids=["K2", "K4n4", "K4n2lp2", "B1K4", "B3K2"])
def test_generate_beam_matches_oracle(cuda_dev, K, n_ret, lp, rows):
    from tests.test_navmodel_gpu import build_model
    from tests.test_oracle_golden import load
    g, cfg, tok = load("amp_bf16")
    model, _ = build_model(g, cuda_dev)
    text, cand = _qa(g, cfg, tok, rows)
    n_new = 12
    kw = dict(num_beams=K, max_new_tokens=n_new, eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id, length_penalty=lp,
              num_return_sequences=n_ret)
    ref, steps = BO.beam_generate(g["state_dict"], cfg, text["input_ids"], text["attention_mask"], cand_vis=cand, return_steps=True,
                                  **kw)
    S = text["input_ids"].shape[1]
    outs = {}
    for graph in (False, True):
        stats = {}
        ids = model.lang_model.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev),
                                        use_cuda_graph=graph, stats=stats, **kw).cpu()
        assert ids.shape[0] == ref.shape[0] == text["input_ids"].shape[0] * n_ret and torch.equal(ids[:, :S], ref[:, :S])
        near_tie_ok(ids, ref, steps, S, n_ret, tag=f"graph={graph}")
        assert stats["beam_steps"] >= 1 and stats["prefill_ms"] > 0
        outs[graph] = ids
    assert torch.equal(outs[False], outs[True])


def test_generate_beam_graph_reuse_and_buckets(cuda_dev):
    """Graph and eager give the same ids across two cache buckets and a graph reused by a second call."""
    from tests.test_navmodel_gpu import build_model
    from tests.test_oracle_golden import load
    g, cfg, tok = load("amp_bf16")
    model, _ = build_model(g, cuda_dev)
    lm = model.lang_model
    text, cand = _qa(g, cfg, tok)
    base = dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev), num_beams=4,
                eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id, length_penalty=1.0)
    for n_new in (20, 140):                                             # two generated-cache buckets
        e = lm.generate(max_new_tokens=n_new, use_cuda_graph=False, **base).cpu()
        g1 = lm.generate(max_new_tokens=n_new, use_cuda_graph=True, **base).cpu()
        g2 = lm.generate(max_new_tokens=n_new, use_cuda_graph=True, **base).cpu()     # the cached graph again
        assert torch.equal(e, g1) and torch.equal(e, g2), n_new


def _rounded_bf16_beams(lm, monkeypatch, kw):
    """generate(num_beams=K) on the bf16 kernels, eagerly and without layer calls, with the prompt cache rounded to K' / V'
    after the prefill and every appended generated row rounded before the attention reads it: the attention of a step is
    rope + append + rounding + nv_decode_attn over a contiguous cache gathered through src (nv_decode_attn_rope_beam is bit
    for bit the contiguous kernel over the same keys: test_beam_attention_is_contiguous_attention_through_src)."""
    from navillm_b200 import llama, ops
    from tests.test_fp8_kv_gpu import _round_rows
    with monkeypatch.context() as m:
        m.setattr(llama.LlamaCore, "LAYER_CALL", False)
        fwd = llama.LlamaCore.forward

        def forward(self, *a, kv_store=None, **k):
            r = fwd(self, *a, kv_store=kv_store, **k)
            if kv_store is not None:
                for c in kv_store[0] + kv_store[1]:
                    _round_rows(c)
            return r

        def attn_beam(qkv, lens, cos_t, sin_t, pk, pv, plens, kc, vc, src, K, n_heads, *, out=None, scale=None):
            R, G, HD = kc.shape
            Sp = pk.shape[1]
            q = qkv.clone()
            ops.rope_(q, lens, cos_t, sin_t, 2 * n_heads, 128)
            r = torch.arange(R, device=kc.device)
            P = plens.long()[r // K]
            i_new = lens.long() - P
            for c, col in ((kc, HD), (vc, 2 * HD)):
                rows = q[:, col:col + HD].contiguous()
                _round_rows(rows)
                c[r, i_new] = rows
            j = torch.arange(Sp + G, device=kc.device)
            i = j[None, :] - P[:, None]
            ii = i.clamp(0, G - 1)
            gen_rows = src.long().gather(1, ii)
            cont = []
            for pc, gc in ((pk, kc), (pv, vc)):
                prompt = torch.zeros((R, Sp + G, HD), dtype=pc.dtype, device=pc.device)
                prompt[:, :Sp] = pc[r // K]
                cont.append(torch.where((i >= 0)[..., None], gc[gen_rows, ii], prompt).contiguous())
            return ops.decode_attn(q, cont[0], cont[1], lens, n_heads, out=out, scale=scale)
        m.setattr(llama.LlamaCore, "forward", forward)
        m.setattr(ops, "decode_attn_rope_beam", attn_beam)
        prev = lm.set_kv_cache_dtype("bf16")
        try:
            return lm.generate(**dict(kw, use_cuda_graph=False)).cpu()
        finally:
            lm.set_kv_cache_dtype(prev)


@pytest.mark.parametrize("rows,K", [([0, 1], 4), ([0], 2), ([1, 0, 1], 4)], ids=["B2K4", "B1K2", "B3K4"])
def test_generate_beam_fp8_kv_is_the_bf16_beam_path_over_rounded_kv(cuda_dev, monkeypatch, rows, K):
    """set_kv_cache_dtype("fp8") with beams: the same ids as the bf16 beam path over K' / V', eager and graphed."""
    from tests.test_navmodel_gpu import build_model
    from tests.test_oracle_golden import load
    g, cfg, tok = load("amp_bf16")
    model, _ = build_model(g, cuda_dev)
    lm = model.lang_model
    text, cand = _qa(g, cfg, tok, rows)
    kw = dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev), num_beams=K,
              eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id, max_new_tokens=16, num_return_sequences=2)
    want = _rounded_bf16_beams(lm, monkeypatch, kw)
    prev = lm.set_kv_cache_dtype("fp8")
    try:
        for graph in (False, True, True):                              # eager, the capturing call, a replaying call
            assert torch.equal(lm.generate(**dict(kw, use_cuda_graph=graph)).cpu(), want), graph
    finally:
        lm.set_kv_cache_dtype(prev)


@pytest.mark.parametrize("rows,K", [([0, 1], 4), ([0], 4), ([1, 0, 1], 2)], ids=["B2K4", "B1K4", "B3K2"])
def test_generate_beam_fp8_weights_are_bf16_beams_on_rounded_weights(cuda_dev, rows, K):
    """quantize_weights_fp8() with beams: the same ids as bf16 beams on the rounded weights W' (drop_fp8_weights())."""
    from tests.test_navmodel_gpu import build_model
    from tests.test_oracle_golden import load
    g, cfg, tok = load("amp_bf16")
    model, _ = build_model(g, cuda_dev)
    lm = model.lang_model
    text, cand = _qa(g, cfg, tok, rows)
    kw = dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev), num_beams=K,
              eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id, max_new_tokens=16)
    lm.quantize_weights_fp8()
    got = [lm.generate(**dict(kw, use_cuda_graph=gr)).cpu() for gr in (False, True)]
    lm.drop_fp8_weights()
    want = lm.generate(**dict(kw, use_cuda_graph=False)).cpu()
    assert torch.equal(got[0], want) and torch.equal(got[1], want)


def test_generate_beam_c3_shape_vs_oracle(cuda_dev):
    """2 Vicuna-width layers at C3's shape (B = 8, 256 <cand> tokens, vocab 32006) with K = 4 beams: 32 beam rows take the
    mid-M decode GEMMs and lm_head, 1024 attention CTAs and the 384-row prompt bucket.  Against the CPU oracle per prompt, under
    the near-tie rule of test_fullwidth_parity_gpu's greedy check; then the fp8 weight copy gives bf16 beams on W'."""
    from tests.test_fullwidth_parity_gpu import _full_navmodel, _oracle_cfg
    B, N_CAND, N_NEW, K = 8, 256, 32, 4
    model, tok = _full_navmodel(cuda_dev, base_vocab=32000)
    assert len(tok) == 32006
    lm = model.lang_model
    sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items() if k.startswith("lang_model.")}
    rng = np.random.RandomState(5)
    prompts = []
    for b in range(B):
        words = " ".join(f"w{i}" for i in rng.randint(0, 5000, size=int(rng.randint(30, 61))))
        prompts.append("Scene " + " ".join(["<cand>"] * N_CAND) + " Question " + words + " Answer")
    text = tok(prompts)
    g = torch.Generator().manual_seed(9)
    cand = torch.randn(B * N_CAND, 4096, generator=g)
    kw = dict(num_beams=K, max_new_tokens=N_NEW, eos_token_id=tok.eos_token_id, pad_token_id=tok.unk_token_id)
    ref, steps = BO.beam_generate(sd, _oracle_cfg(tok, "amp_bf16"), text["input_ids"], text["attention_mask"], cand_vis=cand,
                                  return_steps=True, **kw)
    S = text["input_ids"].shape[1]
    outs = {}
    for graph in (False, True):
        stats = {}
        ids = lm.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev),
                          use_cuda_graph=graph, stats=stats, **kw).cpu()
        assert ids.shape[0] == B and torch.equal(ids[:, :S], text["input_ids"])
        assert stats["kv_rows"] == 384 + 128
        matched = near_tie_ok(ids, ref, steps, S, 1, tag=f"c3 graph={graph}")
        print(f"\n[c3 beams, graph={graph}] matched generated columns per prompt {matched} of {N_NEW}")
        assert sum(matched) >= B * N_NEW // 4, f"too few columns before near-ties: {matched}"
        outs[graph] = ids
    assert torch.equal(outs[False], outs[True])
    model.quantize_weights_fp8()
    got = lm.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev), **kw).cpu()
    lm.drop_fp8_weights()
    want = lm.generate(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev), **kw).cpu()
    assert torch.equal(got, want)


def test_3dqa_mode_with_beams_and_error_cases(cuda_dev):
    from tests.test_navmodel_gpu import build_model, to_dev
    from tests.test_oracle_golden import load
    g, cfg, tok = load("amp_bf16")
    model, _ = build_model(g, cuda_dev)
    qa = dict(g["qa_in"])
    with torch.no_grad():
        out = model("3dqa", qa, training=False, num_beams=4, max_new_tokens=8)["generated_sentences"]
    assert len(out) == len(qa["question"])
    text, cand = _qa(g, cfg, tok)
    kw = dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev), max_new_tokens=4)
    lm = model.lang_model
    with pytest.raises(NotImplementedError, match="beam sampling"):
        lm.generate(num_beams=2, do_sample=True, **kw)
    with pytest.raises(NotImplementedError, match="processors"):
        lm.generate(num_beams=2, trie=object(), **kw)
    with pytest.raises(NotImplementedError, match="processors"):
        lm.generate(num_beams=2, logits_processor=[lambda i, s: s], **kw)
    with pytest.raises(NotImplementedError, match="group"):
        lm.generate(num_beams=4, num_beam_groups=2, **kw)
    with pytest.raises(NotImplementedError, match="num_return_sequences"):
        lm.generate(num_beams=2, num_return_sequences=3, **kw)


def test_num_beams_1_launches_the_greedy_kernels(cuda_dev, monkeypatch):
    from navillm_b200 import _lib
    from tests.test_navmodel_gpu import build_model
    from tests.test_oracle_golden import load
    g, cfg, tok = load("amp_bf16")
    model, _ = build_model(g, cuda_dev)
    text, cand = _qa(g, cfg, tok)
    kw = dict(input_ids=text["input_ids"], attention_mask=text["attention_mask"], cand_vis=cand.to(cuda_dev), max_new_tokens=6,
              use_cuda_graph=False, stop_on_eos=False)
    calls = []
    real = _lib.check

    def spy(status, what):
        calls.append(what)
        return real(status, what)
    import navillm_b200.ops as ops_mod
    monkeypatch.setattr(ops_mod, "check", spy)
    a = model.lang_model.generate(**kw).cpu()
    first = list(calls)
    calls.clear()
    b = model.lang_model.generate(num_beams=1, **kw).cpu()
    assert calls == first and torch.equal(a, b)
    assert not any("beam" in c for c in first)
