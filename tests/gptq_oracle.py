"""GPTQ (Frantar et al., 2022) for the 4-bit group format, restated in fp64 numpy.

The group rule is the one of include/navillm_b200.h (tests/test_int4_quant_cpu.py), evaluated in fp32 on the current
working values: lo = min(0, min w), hi = max(0, max w), s = max(bf16((hi - lo) / 15), 2^-126), z = clamp(rint(-lo / s), 0,
15), q = clamp(rint(w / s) + z, 0, 15), W' = bf16((q - z) s).  Everything else is fp64: the dampened Hessian, U (the upper
Cholesky factor of H^-1), the scaled errors e_j = (w_j - W'_j) / U_jj and their feedback onto the later columns.  A group's
(lo, hi, s, z) are taken when the group's first column is reached."""
import numpy as np

GROUP = 128
TINY = np.float32(2.0 ** -126)


def bf16(x) -> np.ndarray:
    """Round fp32 values to bf16 (nearest, ties to even); returned as fp32."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    b = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16) << 16
    return b.astype(np.uint32).view(np.float32)


def group_params(w: np.ndarray):
    """(s, z) fp32 / int of the rows of one group w [N, 128] (any float dtype; the rule runs in fp32)."""
    w32 = w.astype(np.float32)
    lo = np.minimum(w32.min(1), np.float32(0))
    hi = np.maximum(w32.max(1), np.float32(0))
    s = np.maximum(bf16((hi - lo) / np.float32(15)), TINY)
    z = np.clip(-np.rint(lo / s), 0, 15)
    return s, z


def code(w: np.ndarray, s: np.ndarray, z: np.ndarray) -> np.ndarray:
    return np.clip(np.rint(w.astype(np.float32) / s) + z, 0, 15)


def value(q: np.ndarray, s: np.ndarray, z: np.ndarray) -> np.ndarray:
    return bf16(((q - z) * s).astype(np.float32)).astype(np.float64)


def damped(H: np.ndarray, damp: float = 0.01) -> np.ndarray:
    """H with every zero diagonal entry (a column no row touched) set to 1, then damp * mean(diag) added to the diagonal."""
    H = np.array(H, dtype=np.float64)
    d = np.diag(H).copy()
    d[d == 0] = 1.0
    d += damp * d.mean()
    H[np.diag_indices_from(H)] = d
    return H


def factor(H: np.ndarray, damp: float = 0.01) -> np.ndarray:
    """U, upper triangular with H_damped^-1 = U^T U."""
    return np.linalg.cholesky(np.linalg.inv(damped(H, damp))).T


def gptq(W: np.ndarray, U: np.ndarray, lazy: bool = True):
    """(q [N, K], s [N, K / 128], z [N, K / 128], W' [N, K]) of W [N, K].  ``lazy``: the blocked form (a block is a group;
    inside it every column updates the block's later columns, and the block's errors reach the later blocks in one product
    at its end); otherwise every column updates all later columns at once."""
    W = np.array(W, dtype=np.float64)
    N, K = W.shape
    G = K // GROUP
    Q, Wq = np.zeros((N, K)), np.zeros((N, K))
    S, Z = np.zeros((N, G), dtype=np.float32), np.zeros((N, G))
    for g in range(G):
        c0, c1 = g * GROUP, (g + 1) * GROUP
        S[:, g], Z[:, g] = group_params(W[:, c0:c1])
        E = np.zeros((N, GROUP))
        for j in range(c0, c1):
            Q[:, j] = code(W[:, j], S[:, g], Z[:, g])
            Wq[:, j] = value(Q[:, j], S[:, g], Z[:, g])
            e = (W[:, j] - Wq[:, j]) / U[j, j]
            end = c1 if lazy else K
            W[:, j + 1:end] -= np.outer(e, U[j, j + 1:end])
            E[:, j - c0] = e
        if lazy:
            W[:, c1:] -= E @ U[c0:c1, c1:]
    return Q, S, Z, Wq


def loss(W: np.ndarray, Wq: np.ndarray, H: np.ndarray) -> float:
    """tr(dW H dW^T), dW = W - W': the summed squared output error on the rows H was recorded from."""
    dW = np.asarray(W, dtype=np.float64) - np.asarray(Wq, dtype=np.float64)
    return float(np.einsum("nk,kl,nl->", dW, np.asarray(H, dtype=np.float64), dW))
