"""The code maps of FlatAdamW's 8-bit moments (``navillm_b200.optim.code_maps``), checked without a GPU."""
import numpy as np

from navillm_b200.optim import M_ZERO, V_ZERO, code_maps


def _tree(bits):
    """The dynamic-tree magnitudes, restated: for e = 0 .. bits-1 the 2^(bits-1-e) midpoints of the linspace(0.1, 1)
    grid of 2^(bits-1-e) + 1 points, scaled by 10^-e."""
    vals = []
    for e in range(bits):
        k = 2 ** (bits - 1 - e)
        for j in range(k):
            lo, hi = 0.1 + 0.9 * j / k, 0.1 + 0.9 * (j + 1) / k
            vals.append((lo + hi) / 2 / 10 ** e)
    return sorted(vals)


def test_maps_are_sorted_256_entry_fp32():
    for mp in code_maps():
        assert mp.dtype == np.float32 and mp.shape == (256,)
        assert np.all(np.diff(mp) >= 0)


def test_signed_map():
    signed, _ = code_maps()
    assert signed[0] == -1.0 and signed[-1] == 1.0
    assert signed[M_ZERO] == 0.0 and signed[M_ZERO - 1] == 0.0            # the spare code duplicates 0
    assert len(np.unique(signed)) == 255
    assert np.array_equal(np.delete(signed, M_ZERO - 1), np.unique(signed))
    # symmetric about the zero code, so a magnitude search over map[128:] plus the sign finds the nearest code
    k = np.arange(128)
    assert np.array_equal(signed[M_ZERO - 1 - k[1:]], -signed[M_ZERO + k[1:]])
    mags = np.float32(_tree(7)[-126:])
    expect = np.concatenate([[-1.0], -mags[::-1], [0.0, 0.0], mags, [1.0]]).astype(np.float32)
    assert np.array_equal(signed, expect)
    assert len(_tree(7)) == 127                                          # the smallest magnitude is the one left out


def test_unsigned_map():
    _, unsigned = code_maps()
    assert unsigned[V_ZERO] == 0.0 and unsigned[-1] == 1.0
    assert len(np.unique(unsigned)) == 256
    mags = _tree(8)
    assert len(mags) == 255
    assert np.array_equal(unsigned, np.float32([0.0] + mags[-254:] + [1.0]))
    assert np.all(unsigned[1:] > 0) and np.all(unsigned < 1.0 + 1e-7)
