"""Argument checks of nv_gemm_wgrad_seg_bf16 (the segmented-contraction weight gradient): malformed segment tables are
rejected with NV_ERR_BAD_ARG before the library touches a device, so they are checked here with placeholder pointers."""
import ctypes
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

M, N = 256, 128
BASE = 1 << 20                    # placeholder device addresses: 16-byte aligned, never dereferenced


def _table(n=2, rows=None, lda=None, ldb=None, a=None, b=None):
    rows = rows if rows is not None else [5 + 60 * s for s in range(n)]
    lda = lda if lda is not None else [M] * n
    ldb = ldb if ldb is not None else [N] * n
    a = a if a is not None else [BASE + 4096 * s for s in range(n)]
    b = b if b is not None else [2 * BASE + 4096 * s for s in range(n)]
    k = max(n, 1)
    A, B = (ctypes.c_void_p * k)(*a), (ctypes.c_void_p * k)(*b)
    LA, LB, R = (ctypes.c_int64 * k)(*lda), (ctypes.c_int64 * k)(*ldb), (ctypes.c_int * k)(*rows)
    return A, LA, B, LB, R


def _call(table, n=2, C=3 * BASE, ldc=N, addend=None, ld_add=0, m=M, nn=N):
    from navillm_b200 import _lib
    lib = _lib.load()
    A, LA, B, LB, R = table
    rc = lib.nv_gemm_wgrad_seg_bf16(A, LA, B, LB, R, ctypes.c_int(n), ctypes.c_void_p(C), ctypes.c_int64(ldc),
                                    ctypes.c_void_p(addend), ctypes.c_int64(ld_add), ctypes.c_int(m), ctypes.c_int(nn), None)
    return rc, lib.nv_last_error().decode()


MALFORMED = {
    "no segments": lambda: _call(_table(1), n=0),
    "above the cap": lambda: _call(_table(65), n=65),
    "zero rows": lambda: _call(_table(rows=[5, 0])),
    "negative rows": lambda: _call(_table(rows=[-3, 7])),
    "null operand": lambda: _call(_table(a=[BASE, 0])),
    "lda not a multiple of 8": lambda: _call(_table(lda=[M, M + 4])),
    "lda below M": lambda: _call(_table(lda=[M - 8, M])),
    "ldb below N": lambda: _call(_table(ldb=[N, N - 8])),
    "misaligned base": lambda: _call(_table(b=[2 * BASE, 2 * BASE + 8])),
    "ldc below N": lambda: _call(_table(), ldc=N - 8),
    "null C": lambda: _call(_table(), C=0),
    "misaligned addend": lambda: _call(_table(), addend=4 * BASE + 2, ld_add=N),
    "empty output": lambda: _call(_table(), m=0),
}


@pytest.mark.parametrize("case", sorted(MALFORMED))
def test_malformed_segment_table_is_rejected(case):
    rc, msg = MALFORMED[case]()
    assert rc == -1, (case, rc, msg)                     # NV_ERR_BAD_ARG
    assert "nv_gemm_wgrad_seg_bf16" in msg, msg


def test_cap_matches_header():
    from navillm_b200 import ops
    text = (ROOT / "include" / "navillm_b200.h").read_text()
    assert f"#define NV_WGRAD_SEG_MAX {ops.WGRAD_SEG_MAX}" in text
    with pytest.raises(ValueError, match="segments"):
        ops.gemm_wgrad_seg([], torch.zeros(8, 8, dtype=torch.bfloat16))


@pytest.mark.skipif(torch.cuda.is_available(), reason="exercises the no-GPU failure path")
def test_well_formed_table_fails_loudly_without_a_gpu():
    rc, _ = _call(_table(64), n=64)
    assert rc == -2                                      # NV_ERR_NO_DEVICE: past the checks, no device to run on
