"""CPU-side checks of the drop-in boundary: the shared library builds for sm_90a, loads without a GPU,
exports every symbol include/navillm_b200.h declares, and fails loudly (never computes on the host) when no
device is present."""
import ctypes
import re
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


@pytest.fixture(scope="module")
def lib():
    from navillm_b200 import _lib
    return _lib.load()


def declared_symbols():
    text = (ROOT / "include" / "navillm_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(nv_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_are_exported(lib):
    syms = declared_symbols()
    assert len(syms) >= 30
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, f"declared in include/navillm_b200.h but not exported: {missing}"


def test_every_exported_entry_point_is_declared(lib):
    import subprocess
    out = subprocess.run(["nm", "-D", "--defined-only", str(ROOT / "navillm_b200" / "lib" / "libnavillm_b200.so")],
                         capture_output=True, text=True).stdout
    exported = sorted(set(re.findall(r"\bT (nv_[a-z0-9_]+)$", out, flags=re.M)))
    undeclared = [s for s in exported if s not in declared_symbols()]
    assert not undeclared, f"exported but missing from the header: {undeclared}"


def test_abi_version_and_error_string(lib):
    assert lib.nv_abi_version() == 1
    lib.nv_last_error.restype = ctypes.c_char_p
    assert isinstance(lib.nv_last_error(), bytes)


@pytest.mark.skipif(torch.cuda.is_available(), reason="exercises the no-GPU failure path")
def test_no_gpu_means_loud_failure_not_cpu_fallback(lib):
    assert lib.nv_device_check() != 0
    a = (ctypes.c_uint16 * (128 * 64))()
    c = (ctypes.c_uint16 * (128 * 128))()
    rc = lib.nv_gemm_bf16(ctypes.byref(a), ctypes.c_int64(64), 0, ctypes.byref(a), ctypes.c_int64(64), 0, ctypes.byref(c),
                          ctypes.c_int64(128), None, ctypes.c_int64(0), 128, 128, 64, 0, 0, None)
    assert rc != 0, "compute entry point succeeded without a GPU"
    from navillm_b200 import ops, _lib as L
    with pytest.raises((L.NvError, ValueError)):
        ops.gemm(torch.zeros(128, 64, dtype=torch.bfloat16), torch.zeros(128, 64, dtype=torch.bfloat16))


def test_sass_contains_hopper_tensor_and_tma_instructions():
    import shutil
    import subprocess
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    out = subprocess.run(["cuobjdump", "-sass", str(ROOT / "navillm_b200" / "lib" / "libnavillm_b200.so")],
                         capture_output=True, text=True).stdout
    assert "arch = sm_90a" in out
    assert "HGMMA" in out and "UTMALDG" in out          # warpgroup MMA and TMA loads
    assert "HMMA." not in out, "legacy mma.sync path found"


def test_layer_args_mirror_matches_the_c_struct():
    """ctypes mirror of nv_layer_args (navillm_b200/_lib.py) against sizeof in the library."""
    import ctypes
    from navillm_b200 import _lib
    assert _lib.load(build_if_missing=False).nv_layer_args_size() == ctypes.sizeof(_lib.LayerArgs)
