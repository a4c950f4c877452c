"""The fused-epilogue GEMMs on the 2-CTA cluster kernel (SwiGLU, SwiGLU backward, RoPE, attention-backward row sums),
at the cases the other GEMM tests do not reach: an odd head count, so that the last n-block is half a tile and its TMA
stores are clipped at N; the inference SwiGLU that does not keep g|u; and the real shapes of bench.py's C2 step.  Each
output is compared bit for bit with the 128-wide GEMM followed by the row kernel.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _dvec_close(dout, o, dvec, H):
    T = dout.shape[0]
    want = (dout.double() * o.double()).view(T, H, 128).sum(-1).t().contiguous()
    err = (dvec.view(H, T).double() - want).abs().max().item()
    assert err <= 1e-4 * want.abs().max().item() + 1e-5, err


@pytest.mark.parametrize("T", [77, 1401])
def test_rope_and_attnd_with_a_half_last_n_block(cuda_dev, T):
    from navillm_b200 import ops
    from navillm_b200.llama import LlamaDims, rope_tables
    H = 5                                   # D = 640 = 2.5 tiles of 256: the last n-block holds one head
    D = 128 * H
    g = torch.Generator(device="cpu").manual_seed(T + 5)
    x = torch.randn(T, D, generator=g).to(cuda_dev, torch.bfloat16)
    wqkv = (torch.randn(3 * D, D, generator=g) * 0.05).to(cuda_dev, torch.bfloat16)
    cos_t, sin_t = rope_tables(LlamaDims(hidden=D, n_heads=H, max_pos=2048), cuda_dev)
    pos = torch.randint(0, 2048, (T,), generator=g).to(cuda_dev, torch.int32)
    # a sentinel column block past N in a wider buffer: the clipped stores must not reach it
    buf = torch.full((T, 3 * D + 128), 7.0, device=cuda_dev, dtype=torch.bfloat16)
    q_f = ops.gemm_rope(x, wqkv, pos, cos_t, sin_t, 2 * D, out=buf[:, :3 * D])
    q_u = ops.gemm(x, wqkv, block_n=128)
    ops.rope_(q_u, pos, cos_t, sin_t, 2 * H)
    torch.cuda.synchronize()
    assert torch.equal(q_f, q_u)
    assert bool((buf[:, 3 * D:] == 7.0).all())

    wo = (torch.randn(D, D, generator=g) * 0.03).to(cuda_dev, torch.bfloat16)
    o = torch.randn(T, D, generator=g).to(cuda_dev, torch.bfloat16)
    dbuf = torch.full((T, D + 128), 7.0, device=cuda_dev, dtype=torch.bfloat16)
    dout, dvec = ops.gemm_attnd(x, wo, o, dout=dbuf[:, :D])
    torch.cuda.synchronize()
    assert torch.equal(dout, ops.gemm(x, wo, b_mn=True, block_n=128))
    assert bool((dbuf[:, D:] == 7.0).all())
    _dvec_close(dout, o, dvec, H)


@pytest.mark.parametrize("T", [77, 1401])
def test_swiglu_without_keeping_gu(cuda_dev, T):
    from navillm_b200 import ops
    D, F = 1024, 1408
    g = torch.Generator(device="cpu").manual_seed(T + 11)
    x = torch.randn(T, D, generator=g).to(cuda_dev, torch.bfloat16)
    wgu = (torch.randn(2 * F, D, generator=g) * 0.05).to(cuda_dev, torch.bfloat16)
    gu = torch.full((T, 2 * F), 7.0, device=cuda_dev, dtype=torch.bfloat16)
    _, h = ops.gemm_swiglu(x, wgu, gu=gu, keep_gu=False)
    torch.cuda.synchronize()
    assert bool((gu == 7.0).all()), "keep_gu=False must not write g|u"
    assert torch.equal(h, ops.swiglu_fwd(ops.gemm(x, wgu, block_n=128)))


def test_fused_forms_at_the_c2_shape(cuda_dev):
    """T = 10 425 tokens (C2), D = 4096, F = 11008, 32 heads: 82 m-blocks, and F is 43 n-blocks of the SwiGLU tile."""
    from navillm_b200 import ops
    from navillm_b200.llama import LlamaDims, rope_tables
    T, D, F, H = 10425, 4096, 11008, 32
    g = torch.Generator(device="cpu").manual_seed(2)
    x = (torch.randn(T, D, generator=g) * 0.5).to(cuda_dev, torch.bfloat16)

    wgu = (torch.randn(2 * F, D, generator=g) * 0.02).to(cuda_dev, torch.bfloat16)
    gu_f, h_f = ops.gemm_swiglu(x, wgu)
    gu_u = ops.gemm(x, wgu, block_n=128)
    assert torch.equal(gu_f, gu_u) and torch.equal(h_f, ops.swiglu_fwd(gu_u))
    del h_f, gu_f

    wd = (torch.randn(D, F, generator=g) * 0.02).to(cuda_dev, torch.bfloat16)
    dgu_f = ops.gemm_dswiglu(x, wd, gu_u)
    assert torch.equal(dgu_f, ops.swiglu_bwd(gu_u, ops.gemm(x, wd, b_mn=True, block_n=128)))
    del dgu_f, gu_u, wgu, wd

    wqkv = (torch.randn(3 * D, D, generator=g) * 0.02).to(cuda_dev, torch.bfloat16)
    cos_t, sin_t = rope_tables(LlamaDims(), cuda_dev)
    pos = (torch.arange(T, dtype=torch.int32) % 1024).to(cuda_dev)
    q_f = ops.gemm_rope(x, wqkv, pos, cos_t, sin_t, 2 * D)
    q_u = ops.gemm(x, wqkv, block_n=128)
    ops.rope_(q_u, pos, cos_t, sin_t, 2 * H)
    assert torch.equal(q_f, q_u)
    del q_f, q_u, wqkv

    wo = (torch.randn(D, D, generator=g) * 0.02).to(cuda_dev, torch.bfloat16)
    o = torch.randn(T, D, generator=g).to(cuda_dev, torch.bfloat16)
    dout, dvec = ops.gemm_attnd(x, wo, o)
    torch.cuda.synchronize()
    assert torch.equal(dout, ops.gemm(x, wo, b_mn=True, block_n=128))
    _dvec_close(dout, o, dvec, H)
