"""The fp64 GPTQ restatement (tests/gptq_oracle.py) the GPU quantizer is checked against: its reduction to the round-to-
nearest rule, its blocked form, its gain on correlated inputs, dead columns and dampening."""
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from tests import gptq_oracle as O  # noqa: E402
from tests.test_int4_quant_cpu import edge_groups, ref_int4  # noqa: E402

bf16 = torch.bfloat16


def _weights(N, K, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(N, K, generator=g) * 0.02).to(bf16)


def correlated_inputs(T, K, seed, outliers=4):
    """Rows with correlated channels (a random mixing of a few latent factors plus noise) and a few outlier channels."""
    rng = np.random.RandomState(seed)
    X = rng.randn(T, 16) @ rng.randn(16, K) + 0.3 * rng.randn(T, K)
    X[:, rng.choice(K, outliers, replace=False)] *= 20.0
    return X


def test_identity_hessian_is_the_round_to_nearest_rule():
    K = 512
    W = torch.cat([_weights(60, K, 1), torch.stack([v.repeat(K // 128) for v in edge_groups().values()])]).to(bf16)
    q, s, z, wq = O.gptq(W.float().numpy(), O.factor(np.eye(K)))
    rq, rs, rz, rw = ref_int4(W)
    assert np.array_equal(q, rq.numpy()) and np.array_equal(z, rz.numpy())
    assert np.array_equal(s, rs.float().numpy())
    assert np.array_equal(wq.astype(np.float32), rw.float().numpy())


def test_blocked_form_equals_column_by_column():
    K = 384
    W = _weights(64, K, 2).float().numpy()
    X = correlated_inputs(1024, K, 3)
    H = X.T @ X
    U = O.factor(H)
    a, b = O.gptq(W, U, lazy=True), O.gptq(W, U, lazy=False)
    assert (a[0] != b[0]).mean() < 1e-3                 # a code may only flip where a value sits on a rounding tie
    la, lb = O.loss(W, a[3], H), O.loss(W, b[3], H)
    assert abs(la - lb) <= 1e-9 * lb
    same = (a[0] == b[0]).all(1)
    assert same.sum() >= 60 and np.array_equal(a[3][same], b[3][same])


def test_gptq_beats_round_to_nearest_on_correlated_inputs():
    for N, K, seed in ((128, 512, 4), (64, 1024, 5)):
        W = _weights(N, K, seed)
        X = correlated_inputs(2048, K, seed)
        H = X.T @ X
        _, _, _, wq = O.gptq(W.float().numpy(), O.factor(H))
        rtn = ref_int4(W)[3].float().numpy()
        lg, lr = O.loss(W.float().numpy(), wq, H), O.loss(W.float().numpy(), rtn, H)
        assert lg < 0.7 * lr, (N, K, lg / lr)


def test_dead_columns_keep_their_weights_and_feed_nothing_forward():
    K = 256
    W = _weights(32, K, 6)
    X = correlated_inputs(512, K, 7)
    dead = [3, 50, 200]
    X[:, dead] = 0.0
    H = X.T @ X
    Hd = O.damped(H, 0.01)
    assert np.allclose(np.diag(Hd)[dead], 1.0 + 0.01 * np.mean(np.where(np.diag(H) == 0, 1.0, np.diag(H))))
    U = O.factor(H)
    for j in dead:
        assert np.all(U[j, j + 1:] == 0.0) and np.all(U[:j, j] == 0.0)
    _, _, _, wq = O.gptq(W.float().numpy(), U)
    rtn = ref_int4(W)[3].float().numpy()
    # group 0's (s, z) are RTN's and no error reaches a dead column: columns 3 and 50 are rounded exactly as RTN rounds them
    assert np.array_equal(wq[:, [3, 50]], rtn[:, [3, 50]])
    assert np.count_nonzero(wq[:, dead]) > 0                    # not zeroed


def test_dampening_is_relative_to_the_mean_diagonal():
    K = 128
    X = correlated_inputs(64, K, 8)                              # 64 rows: H has rank 64, singular without dampening
    H = X.T @ X
    for damp in (0.01, 0.1):
        U = O.factor(H, damp)
        assert np.allclose(np.triu(U), U)
        ref = np.linalg.inv(H + damp * np.mean(np.diag(H)) * np.eye(K))
        assert np.allclose(U.T @ U, ref, rtol=1e-6, atol=1e-9 * np.abs(ref).max())
