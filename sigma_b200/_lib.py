"""ctypes binding of libsigma_b200.so (include/sigma_b200.h).  There is NO fallback: if the
library is missing or a call fails, a RuntimeError carrying sigma_last_error() is raised."""
import ctypes
import os
import re
from ctypes import c_char_p, c_double, c_float, c_int, c_int64, c_size_t, c_uint64, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsigma_b200.so")

F32, F16, BF16 = 0, 1, 2
DIRS_CROSS4, DIRS_SEQ2, DIRS_CROSS = 0, 1, 2


class ScanStrides(ctypes.Structure):
    _fields_ = [(n, c_int64) for n in (
        "u_batch", "u_dim", "delta_batch", "delta_dim", "A_dim", "A_dstate",
        "B_batch", "B_group", "B_dstate", "C_batch", "C_group", "C_dstate", "out_batch", "out_dim")]


HEADER = os.path.join(os.path.dirname(_HERE), "include", "sigma_b200.h")
_SCALARS = {"void": None, "int": c_int, "int64_t": c_int64, "uint64_t": c_uint64, "size_t": c_size_t, "float": c_float,
            "double": c_double}


def _ctype(decl):
    """ctypes type of one declarator of the header ("const float *A", "int64_t *out8_host", "size_t", ...).  Every pointer is
    passed as c_void_p except host int64 output arrays, the strides struct and the error string."""
    decl = decl.replace("const ", "").strip()
    if "*" not in decl:
        return _SCALARS[decl.split()[0]]
    base, name = (t.strip() for t in decl.split("*", 1))
    if base == "sigma_scan_strides":
        return ctypes.POINTER(ScanStrides)
    if base == "int64_t" and name.endswith("_host"):
        return ctypes.POINTER(c_int64)
    return c_char_p if base == "char" else c_void_p


def _signatures():
    """name -> (restype, argtypes) of every function include/sigma_b200.h declares."""
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    sigs = {}
    for ret, name, args in re.findall(r"^([A-Za-z_][\w ]*?\s*\**)\s*(sigma_\w+)\s*\(([^)]*)\)\s*;", src, flags=re.M):
        params = [a for a in args.split(",") if a.strip() not in ("", "void")]
        sigs[name] = (_ctype(ret), [_ctype(a) for a in params])
    return sigs


SIGNATURES = _signatures()

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -m sigma_b200.build` "
                "(sigma_b200 has no CPU or library fallback path)")
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


def check(rc, what):
    if rc != 0:
        raise RuntimeError(f"{what} failed (code {rc}): {lib().sigma_last_error().decode()}")


def launch_count():
    return int(lib().sigma_launch_count())


def ptr(t):
    """a tensor's device pointer as a `void *` / `float *` argument; None passes NULL"""
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def stream():
    """torch's current CUDA stream as the `void *stream` argument"""
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
