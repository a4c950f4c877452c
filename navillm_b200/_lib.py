"""ctypes binding of the navillm_b200 C-ABI (include/navillm_b200.h).

PyTorch is used only for device memory and streams: every call passes raw device pointers
(``tensor.data_ptr()``), explicit sizes and the current CUDA stream handle.  A missing library or a
non-zero status raises -- there is no CPU / eager fallback on the product path.
"""
from __future__ import annotations

import ctypes
import os
from pathlib import Path

import torch

_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "lib" / "libnavillm_b200.so"

GEMM_ADD = 1
GEMM_OUT_F32 = 2


class NvError(RuntimeError):
    pass


_lib = None


def load(build_if_missing: bool = True) -> ctypes.CDLL:
    """dlopen the in-tree shared library (building it with nvcc first if it is absent)."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        if not build_if_missing or os.environ.get("NAVILLM_B200_NO_BUILD"):
            raise NvError(f"{LIB_PATH} is missing: run `python -m navillm_b200.build` (no CPU fallback exists)")
        from . import build as _build
        _build.build()
    _lib = ctypes.CDLL(str(LIB_PATH))
    _lib.nv_last_error.restype = ctypes.c_char_p
    return _lib


class LayerArgs(ctypes.Structure):
    """nv_layer_args of include/navillm_b200.h (field order and types must match)."""
    _fields_ = ([(n, ctypes.c_void_p) for n in ("x", "y", "ln1", "wqkv", "wo", "ln2", "wgu", "wd", "pos", "cos_t", "sin_t", "cu_seqlens",
                                                "kcache", "vcache", "cached", "kv_start", "kv_len", "out_rows", "ws")]
                + [("ws_bytes", ctypes.c_int64)]
                + [(n, ctypes.c_int) for n in ("B", "T", "total_qblocks", "Smax", "Tkv", "kv_mode", "R", "D", "F", "H")]
                + [("eps", ctypes.c_float), ("scale", ctypes.c_float)]
                + [(n, ctypes.c_void_p) for n in ("wqkv_q", "wqkv_e", "wo_q", "wo_e", "wgu_q", "wgu_e", "wd_q", "wd_e")]
                + [("fp8_max_rows", ctypes.c_int)]
                + [(n, ctypes.c_void_p) for n in ("kexp", "vexp")]
                + [("act_fp8", ctypes.c_int)]
                + [(n, ctypes.c_void_p) for n in ("wqkv_c", "wqkv_s", "wqkv_z", "wo_c", "wo_s", "wo_z",
                                                  "wgu_c", "wgu_s", "wgu_z", "wd_c", "wd_s", "wd_z")]
                + [("int4_max_rows", ctypes.c_int)])


launch_count = 0          # kernels launched through the C ABI since import (bench.py reports the per-step delta)

# entry points that launch more than one kernel per call
_MULTI = {"nv_rmsnorm_bwd": 2, "nv_attn_bwd": 3, "nv_attn_bwd_kv": 3, "nv_layernorm_bwd": 3, "nv_head_bwd": 2, "nv_mha_bwd": 2, "nv_llama_layer_infer": 10,
          "nv_contrastive_rank": 2}


def check(status: int, what: str) -> None:
    global launch_count
    launch_count += _MULTI.get(what, 1)
    if status != 0:
        msg = load().nv_last_error().decode(errors="replace")
        raise NvError(f"{what} failed with status {status}: {msg}")


def stream_ptr() -> ctypes.c_void_p:
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t) -> ctypes.c_void_p:
    if t is None:
        return ctypes.c_void_p(0)
    return ctypes.c_void_p(t.data_ptr())


def i64(v) -> ctypes.c_int64:
    return ctypes.c_int64(int(v))


def i32(v) -> ctypes.c_int:
    return ctypes.c_int(int(v))


def u32(v) -> ctypes.c_uint:
    return ctypes.c_uint(int(v))


def f32(v) -> ctypes.c_float:
    return ctypes.c_float(float(v))
