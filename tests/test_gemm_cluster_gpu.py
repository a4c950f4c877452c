"""The plain 128 x 256 GEMM tile (2-CTA clusters sharing the B tile by TMA multicast, bf16 epilogue staging) against
the 128-wide kernel.  Both accumulate each output tile's k-blocks in one chain, in the same order, so every output bit
must agree; the shapes cover an odd m-block count (the cluster partner of the last tile lies past M), M <= 128, fewer
tile pairs than clusters, many tile pairs per cluster and K % 64 != 0, in all four operand forms and with the in-place
residual add of gradient accumulation.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

FORMS = [(False, False), (False, True), (True, True), (True, False)]
SHAPES = [
    (77, 200, 72),        # one m-block: the partner CTA computes zeros and stores nothing
    (128, 1032, 520),     # M = 128, ragged N and K
    (300, 512, 4096),     # 3 m-blocks x 2 n-blocks: 4 tile pairs, fewer than the clusters
    (600, 1000, 136),     # 5 m-blocks
    (3900, 8200, 520),    # 31 m-blocks x 33 n-blocks: several tile pairs per cluster
]


@pytest.mark.parametrize("a_mn,b_mn", FORMS)
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_wide_tile_is_bit_identical_to_128_wide(cuda_dev, M, N, K, a_mn, b_mn):
    from navillm_b200 import ops
    if a_mn:
        M = (M + 7) // 8 * 8
    if b_mn:
        N = (N + 7) // 8 * 8
    g = torch.Generator(device="cpu").manual_seed(M * 5 + N + K)
    a = torch.randn((K, M) if a_mn else (M, K), generator=g).to(cuda_dev, torch.bfloat16)
    b = (torch.randn((K, N) if b_mn else (N, K), generator=g) * 0.1).to(cuda_dev, torch.bfloat16)
    add = torch.randn(M, N, generator=g).to(cuda_dev, torch.bfloat16)
    for addend in (None, add):
        wide = ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, addend=addend, block_n=256)
        narrow = ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, addend=addend, block_n=128)
        torch.cuda.synchronize()
        assert torch.equal(wide, narrow), (addend is not None, (wide.float() - narrow.float()).abs().max().item())
    # in place: out is addend (the wgrad accumulation form)
    acc_w, acc_n = add.clone(), add.clone()
    ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out=acc_w, addend=acc_w, block_n=256)
    ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out=acc_n, addend=acc_n, block_n=128)
    torch.cuda.synchronize()
    assert torch.equal(acc_w, acc_n)
    ref = (a.float().t() if a_mn else a.float()) @ (b.float() if b_mn else b.float().t())
    assert torch.allclose(narrow.float(), (ref.to(torch.bfloat16).float() + add.float()), rtol=1.6e-2, atol=0.1)


@pytest.mark.parametrize("T", [77, 1401])
def test_wide_fused_epilogues_match_gemm_then_row_kernel(cuda_dev, T):
    """SwiGLU, SwiGLU backward, RoPE and the attention-backward row sums of the fused 256-wide GEMMs against the
    128-wide GEMM followed by the row kernel, at a single m-block and at an odd m-block count (11)."""
    from navillm_b200 import ops
    from navillm_b200.llama import LlamaDims, rope_tables
    g = torch.Generator(device="cpu").manual_seed(T)
    D, F, H = 1024, 1408, 8
    x = torch.randn(T, D, generator=g).to(cuda_dev, torch.bfloat16)
    wgu = (torch.randn(2 * F, D, generator=g) * 0.05).to(cuda_dev, torch.bfloat16)
    gu_f, h_f = ops.gemm_swiglu(x, wgu)
    gu_u = ops.gemm(x, wgu, block_n=128)
    assert torch.equal(gu_f, gu_u) and torch.equal(h_f, ops.swiglu_fwd(gu_u))

    wd = (torch.randn(D, F, generator=g) * 0.05).to(cuda_dev, torch.bfloat16)
    dx = torch.randn(T, D, generator=g).to(cuda_dev, torch.bfloat16)
    dgu_f = ops.gemm_dswiglu(dx, wd, gu_u)
    assert torch.equal(dgu_f, ops.swiglu_bwd(gu_u, ops.gemm(dx, wd, b_mn=True, block_n=128)))

    wqkv = (torch.randn(3 * D, D, generator=g) * 0.05).to(cuda_dev, torch.bfloat16)
    cos_t, sin_t = rope_tables(LlamaDims(hidden=D, n_heads=H, max_pos=2048), cuda_dev)
    pos = torch.randint(0, 2048, (T,), generator=g).to(cuda_dev, torch.int32)
    q_f = ops.gemm_rope(x, wqkv, pos, cos_t, sin_t, 2 * D)
    q_u = ops.gemm(x, wqkv, block_n=128)
    ops.rope_(q_u, pos, cos_t, sin_t, 2 * H)
    assert torch.equal(q_f, q_u)

    wo = (torch.randn(D, D, generator=g) * 0.03).to(cuda_dev, torch.bfloat16)
    o = torch.randn(T, D, generator=g).to(cuda_dev, torch.bfloat16)
    dout, dvec = ops.gemm_attnd(dx, wo, o)
    torch.cuda.synchronize()
    assert torch.equal(dout, ops.gemm(dx, wo, b_mn=True, block_n=128))
    want = (dout.float() * o.float()).view(T, H, 128).sum(-1).t().contiguous()
    assert (dvec.view(H, T) - want).abs().max().item() <= 1e-4 * want.abs().max().item() + 1e-5
