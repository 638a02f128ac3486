"""ctypes binding of libaniportrait_b200.so (the C ABI declared in include/aniportrait_b200.h).

There is deliberately no fallback: if the shared library is missing or a call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes
import os
import re
from ctypes import c_char_p, c_int, c_longlong, c_void_p, c_float, POINTER  # noqa: F401

_HERE = os.path.dirname(os.path.abspath(__file__))
# AP_LIB_PATH: load another build of the same library (A/B timing of kernel variants on one box)
LIB_PATH = os.environ.get("AP_LIB_PATH") or os.path.join(_HERE, "libaniportrait_b200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "aniportrait_b200.h")

_lib = None
_inited_devices = set()


class ApError(RuntimeError):
    pass


def declared_symbols():
    """Every function the public header declares (used by the CPU-side symbol-coverage test)."""
    text = open(HEADER_PATH).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(ap_[a-z0-9_]+)\s*\(", text)))


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ApError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(aniportrait_b200 has no CPU or PyTorch fallback)")
        _lib = ctypes.CDLL(LIB_PATH)
        _lib.ap_last_error.restype = c_char_p
        _lib.ap_version.restype = c_int
    return _lib


def check(rc: int, what: str):
    if rc != 0:
        msg = lib().ap_last_error().decode(errors="replace")
        raise ApError(f"{what} failed (rc={rc}): {msg}")


def init(device_index: int):
    if device_index not in _inited_devices:
        check(lib().ap_init(c_int(device_index)), "ap_init")
        _inited_devices.add(device_index)


def ptr(t):
    """Device pointer of a torch tensor (or None)."""
    if t is None:
        return c_void_p(0)
    return c_void_p(t.data_ptr())


def fptr(t):
    if t is None:
        return ctypes.cast(c_void_p(0), POINTER(c_float))
    return ctypes.cast(c_void_p(t.data_ptr()), POINTER(c_float))


def stream_ptr():
    import torch
    return c_void_p(torch.cuda.current_stream().cuda_stream)


I = c_int
LL = c_longlong


class EpilogueExt(ctypes.Structure):
    """ap_epilogue_ext of include/aniportrait_b200.h."""
    _fields_ = [("row_stat_out", c_void_p), ("row_stat_ld", c_longlong), ("col_stat_out", c_void_p),
                ("col_stat_ld", c_longlong), ("ln_rstd", c_void_p), ("bias_ld", c_longlong)]


class PoseDecoderParams(ctypes.Structure):
    """ap_pose_decoder_params of include/aniportrait_b200.h, taken by ap_pose_decoder_f16 and by its test hook
    ap_pose_decoder_trace_f16(params, T, kv_cache, out, trace, stream), which also writes every stage's input."""
    _fields_ = [("layers", c_int), ("out_dim", c_int), ("embed_dim", c_int), ("heads", c_int), ("ffn_dim", c_int),
                ("mask_len", c_int), ("pe_len", c_int), ("eps", c_float),
                ("w_qkv", c_void_p), ("w_out", c_void_p), ("w_ff1", c_void_p), ("w_ff2", c_void_p), ("vec", c_void_p),
                ("pose_map_w", c_void_p), ("pose_map_b", c_void_p), ("pose_map_r_w", c_void_p),
                ("pose_map_r_b", c_void_p), ("pe", c_void_p), ("id_row", c_void_p), ("mask", c_void_p),
                ("cross", c_void_p)]


class GridTile(ctypes.Structure):
    """ap_grid_tile of include/aniportrait_b200.h."""
    _fields_ = [("data", c_void_p), ("dtype", c_int), ("bgr", c_int), ("stride_t", c_longlong), ("stride_h", c_longlong),
                ("stride_w", c_longlong), ("stride_c", c_longlong)]


def ext_ptr(ext):
    """NULL or a pointer to an EpilogueExt (the struct is copied by the callee before it returns)."""
    if ext is None:
        return ctypes.cast(c_void_p(0), POINTER(EpilogueExt))
    return ctypes.byref(ext)
