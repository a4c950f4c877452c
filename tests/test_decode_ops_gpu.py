"""Decode-step kernels (csrc/decode.cu) against plain references of the same operations.

Attention: ``decode_attn_rope`` and ``decode_attn`` against softmax attention computed in fp64 from the same bf16 inputs.
The kernel takes the q·k dot products and the online softmax in fp32, never rounds P and rounds the output once to
bf16.  So every element must satisfy |got - ref| <= 2^-8·|ref| + 1e-5·max|v|:
  - 2^-8·|ref| bounds half a bf16 ulp (8 significant bits) of the result;
  - 1e-5·max|v| (max over the head's visible V rows) covers fp32 rounding in the scores and exp2, and the accumulation
    of p·v: one half-warp adds at most Smax/16 = 128 terms, each rounding by at most 2^-24 of a partial sum bounded by
    max|v| (<= 7.6e-6·max|v| in the worst case, far less in practice), and a result next to a rounding midpoint.
Cache rows the call must neither read nor write hold a NaN, so a stray read turns the output NaN.

KV stores are copies and are checked bit for bit against index-copy references; ``argmax_masked`` is checked against
``torch.argmax`` (first maximal index) on the same logits with the special columns at -inf.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
NAN16 = 0x7FA5          # bf16 NaN with a payload no kernel writes: marks cache rows a call must not read or write


def _tables(Smax, H, dev):
    from navillm_b200.llama import LlamaDims, rope_tables
    return rope_tables(LlamaDims(hidden=H * 128, n_heads=H, max_pos=Smax), dev)


def _rope_ref(x, pos, cos_t, sin_t):
    """x [B, H, 128] bf16 rotated at positions pos [B] with the eager bf16 arithmetic of HF apply_rotary_pos_emb
    (the rounding points of tests/test_lm_ops_gpu.py::test_rope)."""
    c, s = cos_t[pos.long()][:, None, :], sin_t[pos.long()][:, None, :]
    rot = torch.cat([-x[..., 64:], x[..., :64]], -1)
    return x * c + rot * s


def _attn_ref(q, kc, vc, lens, scale):
    """fp64 softmax attention of q [B, H, 128] over cache rows 0..lens[b] -> (o [B, H, 128], max|v| per head [B, H])."""
    B, _, HD = kc.shape
    H = HD // 128
    o = torch.empty(B, H, 128, dtype=torch.float64, device=q.device)
    vmax = torch.empty(B, H, dtype=torch.float64, device=q.device)
    for b, l in enumerate(lens):
        k = kc[b, :l + 1].double().view(l + 1, H, 128)
        v = vc[b, :l + 1].double().view(l + 1, H, 128)
        p = torch.softmax(torch.einsum("hd,nhd->hn", q[b].double(), k) * scale, dim=-1)
        o[b] = torch.einsum("hn,nhd->hd", p, v)
        vmax[b] = v.abs().amax(dim=(0, 2))
    return o, vmax


def _check_attn(got, ref, vmax):
    got = got.reshape(ref.shape).double()
    assert bool(torch.isfinite(got).all()), "non-finite attention output (a masked cache row was read)"
    err = (got - ref).abs()
    tol = 2.0 ** -8 * ref.abs() + 1e-5 * vmax[..., None]
    bad = err > tol
    assert not bool(bad.any()), f"{int(bad.sum())} of {bad.numel()} elements out of bound, worst err/tol {(err / tol).max().item():.3g}"


def _lens(B, Smax, c3):
    if c3:
        return [320, 447, 383, 384, 351, 415, 336, 400][:B]
    # 4 keys per half-warp, 8 per warp and 64 per CTA iteration: lengths on both sides of each boundary
    edges = sorted({l for l in (0, 1, 7, 8, 63, 64, 65, 127, 128, Smax - 1) if l < Smax})
    return [edges[(len(edges) - 1 - b) % len(edges)] for b in range(B)]


# (B, H, Smax, scale, C3 lengths): every B with both head counts, every Smax, and C3's decode (8 rows, 32 heads, 512 rows
# of cache, 320..447 tokens cached)
ATTN_CASES = [
    (1, 2, 128, 0.15, False), (1, 32, 2048, None, False), (8, 2, 2048, 0.15, False), (20, 32, 128, None, False),
    (20, 2, 512, 0.15, False), (64, 2, 2048, None, False), (64, 32, 512, 0.15, False), (8, 32, 512, None, True),
]


@pytest.mark.parametrize("use_pdl", [False, True], ids=["plain", "pdl"])
@pytest.mark.parametrize("B,H,Smax,scale,c3", ATTN_CASES)
def test_decode_attn_matches_fp64_attention(cuda_dev, B, H, Smax, scale, c3, use_pdl):
    """Fused RoPE + cache append + attention, then the unfused attention on the same caches: outputs within the bound,
    the appended rows bit-exact, every other cache row, the pad columns of ``out`` and ``qkv`` untouched."""
    from navillm_b200 import ops
    HD = H * 128
    g = torch.Generator(device=cuda_dev).manual_seed(B * 10007 + H * 101 + Smax)
    lens_h = _lens(B, Smax, c3)
    lens = torch.tensor(lens_h, dtype=torch.int32, device=cuda_dev)
    cos_t, sin_t = _tables(Smax, H, cuda_dev)
    qkv = torch.randn(B, 3 * HD, generator=g, device=cuda_dev).to(bf16)
    kc = torch.randn(B, Smax, HD, generator=g, device=cuda_dev).to(bf16)
    vc = torch.randn(B, Smax, HD, generator=g, device=cuda_dev).to(bf16)
    past = torch.arange(Smax, device=cuda_dev)[None, :] >= lens[:, None]        # the row the call writes and all after it
    kc.view(torch.int16)[past] = NAN16
    vc.view(torch.int16)[past] = NAN16
    kc0, vc0, qkv0 = kc.clone(), vc.clone(), qkv.clone()
    eff_scale = 128 ** -0.5 if scale is None else scale

    out_buf = torch.full((B, HD + 64), 7.0, dtype=bf16, device=cuda_dev)        # ldo > H*128; pad columns keep 7
    with ops.pdl(use_pdl):
        ops.decode_attn_rope(qkv, lens, cos_t, sin_t, kc, vc, H, out=out_buf[:, :HD], scale=scale)
    torch.cuda.synchronize()
    assert torch.equal(qkv, qkv0)
    assert bool((out_buf[:, HD:] == 7.0).all())
    q_rot = _rope_ref(qkv[:, :HD].view(B, H, 128), lens, cos_t, sin_t)
    k_rot = _rope_ref(qkv[:, HD:2 * HD].view(B, H, 128), lens, cos_t, sin_t).reshape(B, HD)
    bi, li = torch.arange(B, device=cuda_dev), lens.long()
    assert torch.equal(kc[bi, li].view(torch.int16), k_rot.view(torch.int16))
    assert torch.equal(vc[bi, li].view(torch.int16), qkv[:, 2 * HD:].view(torch.int16))
    other = torch.ones(B, Smax, dtype=torch.bool, device=cuda_dev)
    other[bi, li] = False
    assert torch.equal(kc.view(torch.int16)[other], kc0.view(torch.int16)[other])
    assert torch.equal(vc.view(torch.int16)[other], vc0.view(torch.int16)[other])
    ref, vmax = _attn_ref(q_rot, kc, vc, lens_h, eff_scale)
    _check_attn(out_buf[:, :HD], ref, vmax)

    # unfused attention: rotated q in a wider row whose extra columns are NaN; rows past lens[b] are still NaN
    q_buf = torch.full((B, HD + 128), float("nan"), dtype=bf16, device=cuda_dev)
    q_buf[:, :HD] = q_rot.reshape(B, HD)
    kc1, vc1 = kc.clone(), vc.clone()
    out2 = torch.empty(B, HD + 64, dtype=bf16, device=cuda_dev)[:, :HD]
    with ops.pdl(use_pdl):
        ops.decode_attn(q_buf, kc, vc, lens, H, out=out2, scale=scale)
    torch.cuda.synchronize()
    _check_attn(out2, ref, vmax)
    assert torch.equal(out2, out_buf[:, :HD])
    assert torch.equal(kc.view(torch.int16), kc1.view(torch.int16)) and torch.equal(vc.view(torch.int16), vc1.view(torch.int16))


# ---------------------------------------------------------------------------------------------------------------------
# KV stores
# ---------------------------------------------------------------------------------------------------------------------
def _sentinel_caches(B, Smax, HD, dev):
    kc = torch.empty(B, Smax, HD, dtype=bf16, device=dev)
    kc.view(torch.int16).fill_(NAN16)
    return kc, kc.clone()


@pytest.mark.parametrize("mode", ["prefill", "suffix"])
def test_kv_store_packed_rows_match_index_copy(cuda_dev, mode):
    """Packed rows of sequence b go to cache rows off[b] + i (off = 0 for prefill, cached[b] for suffix); rows at
    p >= Smax are dropped and nothing else is written."""
    from navillm_b200 import ops
    Smax, H = 64, 2
    HD = H * 128
    if mode == "prefill":
        seqlens, offs = [5, 70, 1, 64, 0, 33], [0] * 6            # 70 > Smax
    else:
        seqlens, offs = [3, 5, 4, 5, 0, 2], [0, 5, Smax - 3, Smax - 3, 5, 0]
    B, T = len(seqlens), sum(seqlens)
    cu_h = [0]
    for l in seqlens:
        cu_h.append(cu_h[-1] + l)
    cu = torch.tensor(cu_h, dtype=torch.int32, device=cuda_dev)
    g = torch.Generator(device=cuda_dev).manual_seed(11)
    qkv = torch.randn(T, 3 * HD + 8, generator=g, device=cuda_dev).to(bf16)[:, :3 * HD]      # ld = 3*HD + 8
    kc, vc = _sentinel_caches(B, Smax, HD, cuda_dev)
    kref, vref = kc.clone(), vc.clone()
    if mode == "prefill":
        ops.kv_store_prefill(qkv, cu, kc, vc, B, T)
    else:
        ops.kv_store_suffix(qkv, cu, torch.tensor(offs, dtype=torch.int32, device=cuda_dev), kc, vc, B, T)
    torch.cuda.synchronize()
    kept = [(cu_h[b] + i, b, offs[b] + i) for b, l in enumerate(seqlens) for i in range(l) if offs[b] + i < Smax]
    assert len(kept) < T                                          # some rows were dropped
    t_i, b_i, p_i = map(list, zip(*kept))
    kref[b_i, p_i] = qkv[t_i, HD:2 * HD]
    vref[b_i, p_i] = qkv[t_i, 2 * HD:]
    assert torch.equal(kc.view(torch.int16), kref.view(torch.int16))
    assert torch.equal(vc.view(torch.int16), vref.view(torch.int16))


def test_kv_append_matches_index_copy(cuda_dev):
    """Row b of qkv goes to cache row lens[b]; lens[b] == Smax drops it."""
    from navillm_b200 import ops
    Smax, H = 64, 2
    HD = H * 128
    lens_h = [0, Smax - 1, Smax, 17, Smax]
    B = len(lens_h)
    g = torch.Generator(device=cuda_dev).manual_seed(12)
    qkv = torch.randn(B, 3 * HD + 64, generator=g, device=cuda_dev).to(bf16)[:, :3 * HD]
    kc, vc = _sentinel_caches(B, Smax, HD, cuda_dev)
    kref, vref = kc.clone(), vc.clone()
    ops.kv_append(qkv, torch.tensor(lens_h, dtype=torch.int32, device=cuda_dev), kc, vc)
    torch.cuda.synchronize()
    keep = [b for b in range(B) if lens_h[b] < Smax]
    kref[keep, [lens_h[b] for b in keep]] = qkv[keep, HD:2 * HD]
    vref[keep, [lens_h[b] for b in keep]] = qkv[keep, 2 * HD:]
    assert torch.equal(kc.view(torch.int16), kref.view(torch.int16))
    assert torch.equal(vc.view(torch.int16), vref.view(torch.int16))


# ---------------------------------------------------------------------------------------------------------------------
# greedy pick
# ---------------------------------------------------------------------------------------------------------------------
V = 32006                    # V % 8 == 6: six columns past the last 8-vector
LD_PAD = 32064
SPECIAL = [0, 2, 1234, 31990, 32001]
EOS, PAD = 777, 3
TOP = 8.0                    # above every N(0, 1) logit


def _planted_logits(B, ld, dev):
    """N(0, 1) logits with planted maxima, one pattern per row (row b takes pattern b % 7; B = 1 takes the cross-thread
    tie).  Columns past V hold a larger value, so reading them would change the pick."""
    g = torch.Generator(device=dev).manual_seed(B + ld)
    buf = torch.full((B, ld), 100.0, device=dev)
    buf[:, :V] = torch.randn(B, V, generator=g, device=dev)
    patterns = [
        [(6402, TOP), (6405, TOP)],                        # tie inside one 8-vector
        [(8 * 900 + 3, TOP), (8 * (1024 + 5) + 1, TOP)],   # tie across threads and warps: the lower thread holds the larger index
        [(8 * 37 + 4, TOP), (8 * 37 + 4 + 8192, TOP)],     # tie in one thread, 8*1024 columns apart
        [(31999, TOP), (32003, TOP)],                      # tie between the vector body and the tail
        [(32004, TOP), (32005, TOP)],                      # maximum only in the tail
        [(1234, TOP + 4), (20000, TOP)],                   # a special id holds the global maximum
        [(EOS, TOP)],                                      # greedy pick is eos
    ]
    for b in range(B):
        for c, v in patterns[1 if B == 1 else b % 7]:
            buf[b, c] = v
    return buf.to(bf16)[:, :V] if ld != V else buf.to(bf16)


@pytest.mark.parametrize("stop_on_eos", [True, False])
@pytest.mark.parametrize("ld", [LD_PAD, V], ids=["vector", "scalar"])
@pytest.mark.parametrize("B", [1, 64])
def test_argmax_masked_matches_torch_argmax(cuda_dev, B, ld, stop_on_eos):
    from navillm_b200 import ops
    logits = _planted_logits(B, ld, cuda_dev)
    assert logits.stride(0) == ld
    special = torch.tensor(SPECIAL, dtype=torch.int32, device=cuda_dev)
    fin0 = torch.tensor([int(B > 1 and b % 5 == 4) for b in range(B)], dtype=torch.int32, device=cuda_dev)
    finished = fin0.clone()
    nxt = torch.full((B,), -7, dtype=torch.int32, device=cuda_dev)
    ops.argmax_masked(logits, special, finished, EOS, PAD, stop_on_eos, nxt)
    torch.cuda.synchronize()
    lg = logits.float()
    lg[:, SPECIAL] = float("-inf")
    pick = lg.argmax(dim=1).to(torch.int32)
    want = torch.where(fin0.bool(), torch.full_like(pick, PAD), pick)
    assert torch.equal(nxt, want), (nxt.tolist(), want.tolist())
    fin_want = fin0 | ((pick == EOS) & ~fin0.bool() & stop_on_eos).to(torch.int32)
    assert torch.equal(finished, fin_want)
    if B > 1:
        assert bool(((pick == EOS) & ~fin0.bool()).any()) and bool(fin0.bool().any())


def test_special_id_limit(cuda_dev):
    """64 special ids are all masked by argmax_masked and sample_topk; 65 are rejected, not silently truncated."""
    from navillm_b200 import _lib, ops
    B, Vs = 2, 1000
    g = torch.Generator(device=cuda_dev).manual_seed(13)
    ids = torch.arange(3, 3 + 64 * 7, 7, device=cuda_dev)
    logits = torch.randn(B, Vs, generator=g, device=cuda_dev)
    logits[:, ids] = 20.0 + torch.arange(64, device=cuda_dev, dtype=torch.float32) / 8     # every special id beats the rest
    logits = logits.to(bf16)
    special = ids.to(torch.int32)
    lg = logits.float()
    lg[:, ids] = float("-inf")
    want = lg.argmax(dim=1).to(torch.int32)

    def args():
        return torch.zeros(B, dtype=torch.int32, device=cuda_dev), torch.empty(B, dtype=torch.int32, device=cuda_dev)

    fin, nxt = args()
    ops.argmax_masked(logits, special, fin, -1, PAD, True, nxt)
    torch.cuda.synchronize()
    assert torch.equal(nxt, want)
    fin, nxt = args()
    probs = torch.empty(B, Vs, device=cuda_dev)
    u = torch.rand(B, generator=g, device=cuda_dev)
    ops.sample_topk(logits, special, fin, -1, PAD, True, 1.0, 0, u, nxt, probs_out=probs)
    torch.cuda.synchronize()
    assert bool((probs[:, ids] == 0).all()) and not bool(torch.isin(nxt, special).any())

    special65 = torch.cat([special, torch.tensor([Vs - 1], dtype=torch.int32, device=cuda_dev)])
    fin, nxt = args()
    with pytest.raises(_lib.NvError, match="n_special"):
        ops.argmax_masked(logits, special65, fin, -1, PAD, True, nxt)
    with pytest.raises(_lib.NvError, match="n_special"):
        ops.sample_topk(logits, special65, fin, -1, PAD, True, 1.0, 0, u, nxt)
