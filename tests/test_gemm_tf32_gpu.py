"""wgmma tf32 GEMM (csrc/gemm_tf32.cu) against PyTorch references of the same op.

Two checks, tolerances stated:
  * exactness of the TF32 model: the tensor core reads fp32 operands with a 10-bit mantissa.  Against an fp64 product
    of operands whose low 13 mantissa bits were cleared (truncation) the only admissible difference is fp32
    accumulation order: 2e-5 of max|ref| (K up to 4096).
  * distance from the exact fp32 product: unit roundoff 2^-10 per truncated operand and random-sign accumulation
    => well below 2e-3 of max|ref| for the shapes of the panorama encoder.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _trunc_tf32(x):
    return (x.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def _op(a, b, ta, tb, fn=lambda t: t):
    A = fn(a).double()
    B = fn(b).double()
    A = A.t() if ta else A
    B = B if tb else B.t()
    return A @ B


SHAPES = [(128, 128, 32), (576, 1024, 1408), (576, 3072, 1024), (576, 4096, 1024), (576, 1024, 4096), (77, 200, 72),
          (36, 128, 64), (1000, 520, 260), (2520, 1024, 1024)]


@pytest.mark.parametrize("ta,tb", [(False, False), (False, True), (True, True), (True, False)])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_tf32_gemm(cuda_dev, M, N, K, ta, tb):
    from navillm_b200 import ops
    if ta:
        M = (M + 3) // 4 * 4          # an MN-major operand is stored [K, MN]: leading dimension % 4 floats
    if tb:
        N = (N + 3) // 4 * 4
    g = torch.Generator().manual_seed(M * 5 + N * 3 + K)
    a = torch.randn((K, M) if ta else (M, K), generator=g).to(cuda_dev)
    b = torch.randn((K, N) if tb else (N, K), generator=g).to(cuda_dev)
    bias = torch.randn(N, generator=g).to(cuda_dev)
    prev = ops.set_pano_precision("tf32")
    try:
        out = ops.sgemm(a, b, ta=ta, tb=tb, bias=bias)
        acc = torch.full((M, N), 0.5, device=cuda_dev)
        ops.sgemm(a, b, ta=ta, tb=tb, out=acc, accumulate=True)
    finally:
        ops.set_pano_precision(prev)
    torch.cuda.synchronize()
    model = _op(a, b, ta, tb, _trunc_tf32)
    exact = _op(a, b, ta, tb)
    scale = exact.abs().max().item()
    assert (out.double() - bias.double() - model).abs().max().item() <= 2e-5 * scale
    assert (acc.double() - 0.5 - model).abs().max().item() <= 2e-5 * scale
    assert (out.double() - bias.double() - exact).abs().max().item() <= 2e-3 * scale


def test_tf32_falls_back_to_exact_kernel_for_unaligned_operands(cuda_dev):
    """K = 7 location features (row stride 7 floats) cannot be addressed by TMA: ops.sgemm must use the fp32 kernel."""
    from navillm_b200 import ops
    g = torch.Generator().manual_seed(3)
    a = torch.randn(72, 7, generator=g).to(cuda_dev)
    w = torch.randn(128, 7, generator=g).to(cuda_dev)
    out = ops.sgemm(a, w)
    ref = a.double() @ w.double().t()
    assert (out.double() - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()
