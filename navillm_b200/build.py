"""Build the navillm_b200 C-ABI shared library (sm_90a only) with nvcc, in-tree.

    python -m navillm_b200.build [--force] [--verbose]

Produces ``navillm_b200/lib/libnavillm_b200.so``.  The CUDA runtime is linked statically and the
driver API is resolved at run time, so the library can be ``dlopen``-ed (symbol-export test) on a
machine without a GPU or libcuda; every compute entry point then fails with NV_ERR_NO_DEVICE.
"""
from __future__ import annotations

import argparse
import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIBDIR = PKG / "lib"
OBJDIR = PKG / "lib" / "obj"
LIB = LIBDIR / "libnavillm_b200.so"

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    "-O3", "-std=c++17", "-lineinfo", "--use_fast_math", "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr", "-Xptxas", "-v", "-DNDEBUG",
]
# developer-only extra flags (e.g. NV_NVCC_EXTRA="-DNV_MBAR_TIMEOUT_CYCLES=1000000000")
NVCC_FLAGS += os.environ.get("NV_NVCC_EXTRA", "").split()


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found (needed to build navillm_b200 for sm_90a)")


def _sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu"))


def _digest(src: Path) -> str:
    h = hashlib.sha256()
    h.update(src.read_bytes())
    for hdr in sorted(list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")) + list((PKG.parent / "include").glob("*.h"))):
        h.update(hdr.read_bytes())
    h.update(" ".join(NVCC_FLAGS + ARCH).encode())
    return h.hexdigest()


def _compile_one(nvcc: str, src: Path, verbose: bool) -> tuple[Path, str]:
    obj = OBJDIR / (src.stem + ".o")
    stamp = OBJDIR / (src.stem + ".sha")
    dig = _digest(src)
    if obj.exists() and stamp.exists() and stamp.read_text() == dig:
        return obj, ""
    cmd = [nvcc, *ARCH, *NVCC_FLAGS, "-I", str(CSRC), "-I", str(PKG.parent / "include"), "-c", str(src), "-o", str(obj)]
    p = subprocess.run(cmd, capture_output=True, text=True)
    if p.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src.name}:\n{p.stdout}\n{p.stderr}")
    stamp.write_text(dig)
    log = p.stderr if verbose else ""
    (OBJDIR / (src.stem + ".ptxas.log")).write_text(p.stderr)
    return obj, log


def build(force: bool = False, verbose: bool = False) -> Path:
    srcs = _sources()
    if not srcs:
        raise RuntimeError(f"no CUDA sources under {CSRC}")
    nvcc = _nvcc()
    OBJDIR.mkdir(parents=True, exist_ok=True)
    if force:
        for f in OBJDIR.glob("*.sha"):
            f.unlink()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(lambda s: _compile_one(nvcc, s, verbose), srcs))
    objs = [str(o) for o, _ in results]
    for _, log in results:
        if log:
            print(log, file=sys.stderr)
    newest = max(Path(o).stat().st_mtime for o in objs)
    if force or not LIB.exists() or LIB.stat().st_mtime < newest:
        cmd = [nvcc, *ARCH, "-shared", "-cudart", "static", "-o", str(LIB), *objs]
        p = subprocess.run(cmd, capture_output=True, text=True)
        if p.returncode != 0:
            raise RuntimeError(f"link failed:\n{p.stdout}\n{p.stderr}")
    return LIB


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", action="store_true")
    a = ap.parse_args()
    print(build(a.force, a.verbose))


if __name__ == "__main__":
    main()
