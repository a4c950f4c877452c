"""wgmma flash attention (csrc/attn_fwd.cu, attn_bwd.cu) against a plain PyTorch fp32 reference.

Tolerance (forward): q,k,v are bf16; the kernel keeps S and the running softmax in fp32 and rounds P to
bf16 before the PV product and O to bf16 at the end, like the reference's eager path (fp32 softmax cast
to bf16, bf16 matmul).  |o - o_ref| <= 2e-2 * max|o_ref| covers the bf16 rounding of P (2^-9 relative
per probability) and of O.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

HD = 128


def ref_attention(qkv, seqlens, H):
    T = qkv.shape[0]
    q, k, v = [x.float().view(T, H, HD) for x in qkv.split(H * HD, dim=1)]
    o = torch.zeros(T, H, HD, device=qkv.device)
    lse = torch.zeros(H, T, device=qkv.device)
    s0 = 0
    for L in seqlens:
        qs, ks, vs = q[s0:s0 + L].transpose(0, 1), k[s0:s0 + L].transpose(0, 1), v[s0:s0 + L].transpose(0, 1)
        sc = qs @ ks.transpose(1, 2) * HD ** -0.5
        mask = torch.ones(L, L, device=qkv.device, dtype=torch.bool).tril()
        sc = sc.masked_fill(~mask, float("-inf"))
        lse[:, s0:s0 + L] = torch.logsumexp(sc, dim=-1)
        o[s0:s0 + L] = (torch.softmax(sc, dim=-1) @ vs).transpose(0, 1)
        s0 += L
    return o.reshape(T, H * HD), lse


@pytest.mark.parametrize("seqlens,H", [([128], 1), ([256], 2), ([100], 2), ([1, 129, 300], 2), ([1024, 517, 640], 4),
                                       ([2048], 2)])
def test_attn_fwd(cuda_dev, seqlens, H):
    from navillm_b200 import ops
    T = sum(seqlens)
    g = torch.Generator(device="cpu").manual_seed(T + H)
    qkv = (torch.randn(T, 3 * H * HD, generator=g) * 1.5).to(cuda_dev, torch.bfloat16)
    cu = torch.tensor([0] + list(torch.tensor(seqlens).cumsum(0)), dtype=torch.int32, device=cuda_dev)
    o, lse = ops.attn_fwd(qkv, cu, seqlens, H)
    torch.cuda.synchronize()
    o_ref, lse_ref = ref_attention(qkv, seqlens, H)
    err = (o.float() - o_ref).abs().max().item()
    assert err <= 2e-2 * o_ref.abs().max().item(), f"o err {err}"
    assert torch.allclose(lse, lse_ref, rtol=1e-3, atol=2e-3), (lse - lse_ref).abs().max().item()


@pytest.mark.parametrize("seqlens,H", [([128], 1), ([256], 1), ([100], 2), ([1, 129, 300], 2), ([640, 517], 2)])
def test_attn_bwd(cuda_dev, seqlens, H):
    """Backward against autograd of the fp32 reference.  The kernel rounds P and dS to bf16 before the
    dV/dK/dQ products (2^-9 relative per element) and the gradients to bf16: 3e-2 of the gradient's max."""
    from navillm_b200 import ops
    T = sum(seqlens)
    g = torch.Generator(device="cpu").manual_seed(T * 3 + H)
    qkv = torch.randn(T, 3 * H * HD, generator=g).to(cuda_dev, torch.bfloat16)
    do = torch.randn(T, H * HD, generator=g).to(cuda_dev, torch.bfloat16)
    cu = torch.tensor([0] + list(torch.tensor(seqlens).cumsum(0)), dtype=torch.int32, device=cuda_dev)
    o, lse = ops.attn_fwd(qkv, cu, seqlens, H)
    dqkv = ops.attn_bwd(qkv, o, do, lse, cu, seqlens, H)
    torch.cuda.synchronize()
    qa = qkv.float().requires_grad_(True)
    o_ref, _ = ref_attention(qa, seqlens, H)
    o_ref.backward(do.float())
    for name, sl in (("dq", slice(0, H * HD)), ("dk", slice(H * HD, 2 * H * HD)), ("dv", slice(2 * H * HD, None))):
        a, b = dqkv[:, sl].float(), qa.grad[:, sl]
        err = (a - b).abs().max().item()
        assert err <= 3e-2 * b.abs().max().item(), f"{name} err {err} vs max {b.abs().max().item()}"


def test_attn_bwd_fused_inverse_rope_is_bit_identical(cuda_dev):
    from navillm_b200 import ops
    from navillm_b200.llama import LlamaDims, rope_tables
    seqlens, H = [300, 129, 640], 2
    T = sum(seqlens)
    g = torch.Generator(device="cpu").manual_seed(77)
    qkv = torch.randn(T, 3 * H * HD, generator=g).to(cuda_dev, torch.bfloat16)
    do = torch.randn(T, H * HD, generator=g).to(cuda_dev, torch.bfloat16)
    cu = torch.tensor([0] + list(torch.tensor(seqlens).cumsum(0)), dtype=torch.int32, device=cuda_dev)
    pos = torch.randint(0, 1024, (T,), generator=g).to(cuda_dev, torch.int32)
    cos_t, sin_t = rope_tables(LlamaDims(hidden=H * HD, n_heads=H, max_pos=1024), cuda_dev)
    o, lse = ops.attn_fwd(qkv, cu, seqlens, H)
    fused = ops.attn_bwd(qkv, o, do, lse, cu, seqlens, H, rope=(pos, cos_t, sin_t))
    plain = ops.attn_bwd(qkv, o, do, lse, cu, seqlens, H)
    ops.rope_(plain, pos, cos_t, sin_t, 2 * H, backward=True)
    torch.cuda.synchronize()
    assert torch.equal(fused, plain)


def test_o_proj_dgrad_with_fused_attention_D(cuda_dev):
    """nv_gemm_attnd_bf16: dO is bit-identical to the plain dgrad GEMM; D matches the fp32 row sums of dO * O; the
    attention backward fed with it agrees with the one that runs its own row-sum kernel."""
    import numpy as np
    from navillm_b200 import ops
    H, HD = 8, 128
    D = H * HD
    seqlens = [700, 324, 1024]
    T = sum(seqlens)
    g = torch.Generator().manual_seed(4)
    dy = torch.randn(T, D, generator=g).to(cuda_dev, torch.bfloat16)
    wo = (torch.randn(D, D, generator=g) * 0.03).to(cuda_dev, torch.bfloat16)
    qkv = torch.randn(T, 3 * D, generator=g).to(cuda_dev, torch.bfloat16)
    cu = torch.tensor([0] + list(np.cumsum(seqlens)), dtype=torch.int32, device=cuda_dev)
    o, lse = ops.attn_fwd(qkv, cu, seqlens, H)
    dout, dvec = ops.gemm_attnd(dy, wo, o)
    ref = ops.gemm(dy, wo, b_mn=True, block_n=256)
    torch.cuda.synchronize()
    assert torch.equal(dout, ref)
    want = (dout.float() * o.float()).view(T, H, HD).sum(-1).t().contiguous()          # [H, T]
    got = dvec.view(H, T)
    assert (got - want).abs().max().item() <= 1e-4 * want.abs().max().item() + 1e-5
    a = ops.attn_bwd(qkv, o, dout, lse, cu, seqlens, H)
    b = ops.attn_bwd(qkv, o, dout, lse, cu, seqlens, H, dvec=dvec)
    torch.cuda.synchronize()
    assert (a.float() - b.float()).abs().max().item() <= 2e-2 * a.float().abs().max().item()
    assert (a == b).float().mean().item() > 0.99                                        # identical except where D's rounding moved a bf16 ulp
