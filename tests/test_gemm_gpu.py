"""wgmma bf16 GEMM (csrc/gemm_bf16.cu) against a plain PyTorch fp32 reference of the same op.

Tolerance: inputs are bf16, accumulation fp32, output rounded once to bf16 -> the only admissible
difference from an fp32 reference rounded to bf16 is accumulation order: |diff| <= 2 bf16 ulp of the
result magnitude (rtol 1.6e-2 covers 2 ulp at 8 mantissa bits) plus a small atol for cancellation.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(a, b, a_mn, b_mn):
    A = a.float().t() if a_mn else a.float()
    B = b.float() if b_mn else b.float().t()
    return A @ B


SHAPES = [
    (128, 128, 64), (128, 256, 128), (256, 512, 4096), (384, 4096, 4096), (1000, 1032, 520),
    (77, 200, 72), (4096, 12288, 4096), (2048, 4096, 11008),
]


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gemm_matches_fp32_reference(cuda_dev, M, N, K, a_mn, b_mn):
    from navillm_b200 import ops
    # an MN-major operand is stored [K, MN]: its leading dimension (MN) must be a multiple of 8 elements
    if a_mn:
        M = (M + 7) // 8 * 8
    if b_mn:
        N = (N + 7) // 8 * 8
    g = torch.Generator(device="cpu").manual_seed(M * 7 + N * 3 + K)
    a = torch.randn((K, M) if a_mn else (M, K), generator=g).to(cuda_dev, torch.bfloat16)
    b = torch.randn((K, N) if b_mn else (N, K), generator=g).to(cuda_dev, torch.bfloat16)
    for bn in (128, 256):
        out = ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, block_n=bn)
        torch.cuda.synchronize()
        ref = _ref(a, b, a_mn, b_mn)
        err = (out.float() - ref).abs()
        tol = 1.6e-2 * ref.abs() + 2e-2 * (K ** 0.5) * 0.05
        assert bool((err <= tol).all()), f"bn={bn} max err {err.max().item()} (ref max {ref.abs().max().item()})"


def test_gemm_residual_add_and_strided(cuda_dev):
    from navillm_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(5)
    M, N, K = 300, 4096, 512
    big = torch.randn(M, 3 * K, generator=g).to(cuda_dev, torch.bfloat16)
    a = big[:, K:2 * K]                      # strided view: lda = 3K
    w = torch.randn(N, K, generator=g).to(cuda_dev, torch.bfloat16)
    res = torch.randn(M, N, generator=g).to(cuda_dev, torch.bfloat16)
    out = ops.gemm(a, w, addend=res)
    torch.cuda.synchronize()
    ref = ((a.float() @ w.float().t()).to(torch.bfloat16).float() + res.float()).to(torch.bfloat16)
    err = (out.float() - ref.float()).abs()
    assert bool((err <= 1.6e-2 * ref.float().abs() + 0.25).all()), err.max().item()
    # in-place accumulation (gradient accumulation form): C = bf16(acc) + C
    acc = res.clone()
    ops.gemm(a, w, out=acc, addend=acc)
    torch.cuda.synchronize()
    assert torch.equal(acc, out)


def test_gemm_fp32_out(cuda_dev):
    from navillm_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(9)
    M, N, K = 130, 1000, 256
    a = torch.randn(M, K, generator=g).to(cuda_dev, torch.bfloat16)
    w = torch.randn(N, K, generator=g).to(cuda_dev, torch.bfloat16)
    out = ops.gemm(a, w, out_f32=True)
    torch.cuda.synchronize()
    ref = a.float() @ w.float().t()
    assert torch.allclose(out, ref, rtol=1e-4, atol=1e-3), (out - ref).abs().max().item()


def test_gemm_skinny_m_weight_streaming(cuda_dev):
    """block_n = 32 variant used by the decode step and the pruned last layer (M <= 128)."""
    from navillm_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(3)
    for M, N, K in ((8, 4096, 4096), (16, 22016, 4096), (8, 32006, 4096), (1, 4096, 11008)):
        a = torch.randn(M, K, generator=g).to(cuda_dev, torch.bfloat16)
        w = torch.randn(N, K, generator=g).to(cuda_dev, torch.bfloat16)
        ld = (N + 63) // 64 * 64
        out = torch.empty(M, ld, device=cuda_dev, dtype=torch.bfloat16)[:, :N]
        ops.gemm(a, w, out=out, block_n=32)
        auto = ops.gemm(a, w)
        torch.cuda.synchronize()
        ref = a.float() @ w.float().t()
        tol = 1.6e-2 * ref.abs() + 0.2
        assert bool(((out.float() - ref).abs() <= tol).all()) and bool(((auto.float() - ref).abs() <= tol).all())


def test_fused_epilogues_are_bit_identical_to_unfused(cuda_dev):
    """SwiGLU / SwiGLU-backward / RoPE epilogues of the fused GEMM vs GEMM followed by the row kernels."""
    from navillm_b200 import ops
    from navillm_b200.llama import LlamaDims, rope_tables
    g = torch.Generator(device="cpu").manual_seed(21)
    T, D, F, H = 1500, 1024, 1408, 8                                  # ragged T, F % 128 == 0, 8 heads of 128
    x = torch.randn(T, D, generator=g).to(cuda_dev, torch.bfloat16)
    wgu = (torch.randn(2 * F, D, generator=g) * 0.05).to(cuda_dev, torch.bfloat16)
    gu_f, h_f = ops.gemm_swiglu(x, wgu)
    gu_u = ops.gemm(x, wgu)
    h_u = ops.swiglu_fwd(gu_u)
    assert torch.equal(gu_f, gu_u) and torch.equal(h_f, h_u)
    wd = (torch.randn(D, F, generator=g) * 0.05).to(cuda_dev, torch.bfloat16)
    dx = torch.randn(T, D, generator=g).to(cuda_dev, torch.bfloat16)
    dgu_f = ops.gemm_dswiglu(dx, wd, gu_u)
    dgu_u = ops.swiglu_bwd(gu_u, ops.gemm(dx, wd, b_mn=True))
    assert torch.equal(dgu_f, dgu_u)
    wqkv = (torch.randn(3 * D, D, generator=g) * 0.05).to(cuda_dev, torch.bfloat16)
    cos_t, sin_t = rope_tables(LlamaDims(hidden=D, n_heads=H, max_pos=2048), cuda_dev)
    pos = torch.randint(0, 2048, (T,), generator=g).to(cuda_dev, torch.int32)
    q_f = ops.gemm_rope(x, wqkv, pos, cos_t, sin_t, 2 * D)
    q_u = ops.gemm(x, wqkv)
    ops.rope_(q_u, pos, cos_t, sin_t, 2 * H)
    assert torch.equal(q_f, q_u)


@pytest.mark.parametrize("M", [1, 8, 16])
@pytest.mark.parametrize("N,K", [(4096, 4096), (12288, 4096), (22016, 4096), (4096, 11008), (32006, 4096), (200, 72), (136, 520)])
@pytest.mark.parametrize("with_add", [False, True])
def test_skinny_swap_ab_gemm(cuda_dev, M, N, K, with_add):
    """Decode-step kernel (csrc/gemm_skinny.cu): same contract and tolerance as the general GEMM; the K range is
    split over a cluster, so only the fp32 accumulation order differs."""
    from navillm_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(M * 11 + N + K)
    x = torch.randn(M, K, generator=g).to(cuda_dev, torch.bfloat16)
    w = (torch.randn(N, K, generator=g) * 0.05).to(cuda_dev, torch.bfloat16)
    add = torch.randn(M, N, generator=g).to(cuda_dev, torch.bfloat16) if with_add else None
    out = ops.gemm_skinny(x, w, addend=add)
    torch.cuda.synchronize()
    ref = (x.float() @ w.float().t()).to(torch.bfloat16).float()
    if with_add:
        ref = (ref + add.float()).to(torch.bfloat16).float()
    torch.testing.assert_close(out.float(), ref, rtol=1.6e-2, atol=2e-2)
    # and against the general kernel: identical up to accumulation order (<= 2 bf16 ulp: accumulator rounding, then the rounded sum with the addend)
    gen = ops.gemm(x, w, addend=add, block_n=128)
    torch.testing.assert_close(out.float(), gen.float(), rtol=1.6e-2, atol=2e-2)


@pytest.mark.parametrize("M", [1, 8, 16])
@pytest.mark.parametrize("F,K", [(11008, 4096), (256, 256), (192, 520)])
def test_skinny_swiglu_is_bit_identical_to_gemm_then_swiglu(cuda_dev, M, F, K):
    """Fused gate|up projection + SwiGLU of the decode step vs the two separate kernels (same tiles, same k-splits)."""
    from navillm_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(M + F + K)
    x = torch.randn(M, K, generator=g).to(cuda_dev, torch.bfloat16)
    wgu = (torch.randn(2 * F, K, generator=g) * 0.05).to(cuda_dev, torch.bfloat16)
    h = ops.gemm_skinny_swiglu(x, wgu)
    ref = ops.swiglu_fwd(ops.gemm_skinny(x, wgu))
    torch.cuda.synchronize()
    assert torch.equal(h, ref)
    gu = (x.float() @ wgu.float().t()).to(torch.bfloat16).float()
    want = (torch.nn.functional.silu(gu[:, :F]).to(torch.bfloat16).float() * gu[:, F:]).to(torch.bfloat16).float()
    torch.testing.assert_close(h.float(), want, rtol=3e-2, atol=3e-2)


def test_decode_rope_kv_matches_rope_then_append(cuda_dev):
    from navillm_b200 import ops
    from navillm_b200.llama import LlamaDims, rope_tables
    B, H, Smax = 5, 4, 64
    HD = H * 128
    g = torch.Generator(device="cpu").manual_seed(0)
    qkv = torch.randn(B, 3 * HD, generator=g).to(cuda_dev, torch.bfloat16)
    lens = torch.tensor([0, 3, 17, 63, 40], dtype=torch.int32, device=cuda_dev)
    cos, sin = rope_tables(LlamaDims(hidden=H * 128, n_layers=1, n_heads=H, inter=256, vocab=64), cuda_dev)
    kc = torch.zeros(B, Smax, HD, dtype=torch.bfloat16, device=cuda_dev)
    vc = torch.zeros_like(kc)
    a = qkv.clone()
    ops.decode_rope_kv_(a, lens, cos, sin, kc, vc, H)
    b = qkv.clone()
    kc2, vc2 = torch.zeros_like(kc), torch.zeros_like(vc)
    ops.rope_(b, lens, cos, sin, 2 * H, 128)
    ops.kv_append(b, lens, kc2, vc2)
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(kc, kc2) and torch.equal(vc, vc2)


def test_decode_attn_rope_fused_matches_two_kernels(cuda_dev):
    """nv_decode_attn_rope (RoPE + cache append + attention in one launch) is bit-identical to nv_decode_rope_kv followed by
    nv_decode_attn: outputs, appended cache rows, untouched cache rows; the input qkv is not modified."""
    from navillm_b200 import ops
    from navillm_b200.llama import LlamaDims, rope_tables
    B, H, Smax = 5, 4, 192
    HD = H * 128
    g = torch.Generator(device="cpu").manual_seed(1)
    qkv = torch.randn(B, 3 * HD, generator=g).to(cuda_dev, torch.bfloat16)
    lens = torch.tensor([0, 3, 17, 190, 100], dtype=torch.int32, device=cuda_dev)
    cos, sin = rope_tables(LlamaDims(hidden=HD, n_layers=1, n_heads=H, inter=256, vocab=64), cuda_dev)
    kc = (torch.randn(B, Smax, HD, generator=g) * 0.5).to(cuda_dev, torch.bfloat16)
    vc = (torch.randn(B, Smax, HD, generator=g) * 0.5).to(cuda_dev, torch.bfloat16)
    kc2, vc2, q2 = kc.clone(), vc.clone(), qkv.clone()
    ops.decode_rope_kv_(q2, lens, cos, sin, kc2, vc2, H)
    want = ops.decode_attn(q2, kc2, vc2, lens, H)
    q1 = qkv.clone()
    got = ops.decode_attn_rope(q1, lens, cos, sin, kc, vc, H)
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    assert torch.equal(kc, kc2) and torch.equal(vc, vc2) and torch.equal(q1, qkv)


@pytest.mark.parametrize("M", [17, 48, 128, 129, 192, 256, 257, 384, 511])
@pytest.mark.parametrize("N,K", [(4096, 4096), (12288, 4096), (22016, 4096), (4096, 11008)])
def test_mid_m_auto_dispatch_is_bit_identical_to_every_tile_variant(cuda_dev, M, N, K):
    """16 < M < 512 (one forward of a small batch, evaluation rollouts, prefix-reuse suffixes): nv_gemm_bf16's auto rule
    picks the tile variant per (M, N).  Every variant accumulates the k-blocks in
    the same order, so the choice must not change one output bit - with and without the residual add - and the result
    matches the fp32 reference."""
    from navillm_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    a = (torch.randn((M, K), generator=g) * 0.5).to(cuda_dev, torch.bfloat16)
    b = (torch.randn((N, K), generator=g) * 0.5).to(cuda_dev, torch.bfloat16)
    add = torch.randn((M, N), generator=g).to(cuda_dev, torch.bfloat16)
    for addend in (None, add):
        auto = ops.gemm(a, b, addend=addend)
        for bn in (32, 128, 256):
            if bn == 32 and M > 128:
                continue
            assert torch.equal(ops.gemm(a, b, addend=addend, block_n=bn), auto), (bn, addend is not None)
    ref = a.float() @ b.float().t()
    assert torch.allclose(ops.gemm(a, b).float(), ref, rtol=1.6e-2, atol=2e-2 * float(ref.abs().max()) / 8)
