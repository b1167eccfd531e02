"""ctypes binding of libsigma_b200.so (include/sigma_b200.h).  There is NO fallback: if the
library is missing or a call fails, a RuntimeError carrying sigma_last_error() is raised."""
import ctypes
import os
from ctypes import c_char_p, c_double, c_float, c_int, c_int64, c_size_t, c_uint64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsigma_b200.so")

F32, F16, BF16 = 0, 1, 2
DIRS_CROSS4, DIRS_SEQ2, DIRS_CROSS = 0, 1, 2


class ScanStrides(ctypes.Structure):
    _fields_ = [(n, c_int64) for n in (
        "u_batch", "u_dim", "delta_batch", "delta_dim", "A_dim", "A_dstate",
        "B_batch", "B_group", "B_dstate", "C_batch", "C_group", "C_dstate", "out_batch", "out_dim")]


# name -> (restype, argtypes); mirrors include/sigma_b200.h declaration by declaration
SIGNATURES = {
    "sigma_abi_version": (c_int, []),
    "sigma_last_error": (c_char_p, []),
    "sigma_launch_count": (c_uint64, []),
    "sigma_scan_fwd_workspace_bytes": (c_size_t, [c_int] * 6),
    "sigma_scan_fwd": (c_int, [c_void_p] * 9 + [c_int] * 7 + [ctypes.POINTER(ScanStrides), c_void_p, c_size_t, c_void_p]),
    "sigma_scan_fwd_split": (c_int, [c_void_p] * 9 + [c_int] * 7 + [ctypes.POINTER(ScanStrides), c_void_p, c_size_t, c_int, c_void_p]),
    "sigma_test_scan_plan": (c_int, [c_int] * 8 + [c_size_t, ctypes.POINTER(c_int64)]),
    "sigma_scan_bwd_workspace_bytes": (c_size_t, [c_int] * 6),
    "sigma_scan_bwd": (c_int, [c_void_p] * 15 + [c_int] * 7 + [c_void_p, c_size_t, c_void_p]),
    "sigma_scan_bwd_split": (c_int, [c_void_p] * 15 + [c_int] * 7 + [c_void_p, c_size_t, c_int, c_void_p]),
    "sigma_ss2d_padded_cp": (c_int, [c_int, c_int]),
    "sigma_ss2d_scan_workspace_bytes": (c_size_t, [c_int] * 6),
    "sigma_ss2d_scan_fwd": (c_int, [c_int] + [c_void_p] * 7 + [c_int] * 7 + [c_void_p, c_size_t, c_void_p]),
    "sigma_ss2d_scan_fwd_split": (c_int, [c_int] + [c_void_p] * 7 + [c_int] * 7 + [c_void_p, c_size_t, c_int, c_void_p]),
    "sigma_ss2d_scan_bwd_workspace_bytes": (c_size_t, [c_int] * 6),
    "sigma_ss2d_scan_hs_bytes": (c_size_t, [c_int] * 6),
    "sigma_test_pick_segments": (c_int, [c_int64, c_int, c_int, c_int]),
    "sigma_test_pick_bn": (c_int, [c_int, c_int64]),
    "sigma_test_gemm_plan": (c_int, [c_int64, c_int, c_int, c_int, c_int, c_int, c_int, ctypes.POINTER(c_int64)]),
    "sigma_test_ss2d_bwd_plan": (c_int, [c_int] * 7 + [ctypes.POINTER(c_int64)]),
    "sigma_test_ss2d_fwd_plan": (c_int, [c_int] * 9 + [c_size_t, ctypes.POINTER(c_int64)]),
    "sigma_ss2d_scan_fwd_save": (c_int, [c_int] + [c_void_p] * 9 + [c_int] * 7 + [c_void_p, c_size_t, c_int, c_void_p]),
    "sigma_ss2d_scan_bwd_saved": (c_int, [c_int] + [c_void_p] * 15 + [c_int] * 7 + [c_void_p, c_size_t, c_int, c_void_p]),
    "sigma_ss2d_scan_bwd": (c_int, [c_int] + [c_void_p] * 14 + [c_int] * 7 + [c_void_p, c_size_t, c_void_p]),
    "sigma_ss2d_scan_bwd_split": (c_int, [c_int] + [c_void_p] * 14 + [c_int] * 7 + [c_void_p, c_size_t, c_int, c_void_p]),
    "sigma_layernorm_fwd": (c_int, [c_void_p] * 4 + [c_int64, c_int, c_float, c_void_p]),
    "sigma_layernorm_bwd": (c_int, [c_void_p] * 6 + [c_int64, c_int, c_float, c_void_p]),
    "sigma_dwconv3x3_silu_fwd": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_int64] + [c_int] * 4 + [c_void_p]),
    "sigma_merge_norm_gate_fwd": (c_int, [c_void_p, c_int, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_int64, c_void_p,
                                          c_void_p, c_int64, c_int64, c_int64, c_int64, c_int, c_float, c_void_p]),
    "sigma_upsample2x_norm_fwd": (c_int, [c_void_p] * 4 + [c_int] * 4 + [c_float, c_void_p]),
    "sigma_argmax_hist_fwd": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int64, c_void_p]),
    "sigma_patch_merge_norm_fwd": (c_int, [c_void_p] * 4 + [c_int] * 4 + [c_float, c_void_p]),
    "sigma_pixel_shuffle_norm_fwd": (c_int, [c_void_p] * 4 + [c_int] * 4 + [c_float, c_void_p]),
    "sigma_upsample2x_norm_head_fwd": (c_int, [c_void_p] * 4 + [c_int, c_void_p] + [c_int] * 4 + [c_float, c_void_p]),
    "sigma_pool_avgmax_partial_fwd": (c_int, [c_void_p, c_void_p, c_int, c_int64, c_int, c_int, c_void_p]),
    "sigma_scale_add_fwd": (c_int, [c_void_p] * 5 + [c_int64, c_int64, c_int, c_void_p]),
    "sigma_image_pre_fwd": (c_int, [c_void_p] * 4 + [c_int] * 4 + [c_double, c_double] + [c_int] * 7 + [c_void_p] * 4),
    "sigma_eval_exp_accumulate_fwd": (c_int, [c_void_p] * 3 + [c_int] * 11 + [c_void_p]),
    "sigma_eval_resize_add_fwd": (c_int, [c_void_p] + [c_int] * 7 + [c_void_p, c_int, c_int, c_void_p]),
    "sigma_eval_argmax_hist_fwd": (c_int, [c_void_p] * 5 + [c_int, c_int64, c_void_p]),
    "sigma_linear_tf32": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_void_p]),
    "sigma_linear_tf32x3": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_void_p]),
    "sigma_conv3x3_tf32": (c_int, [c_void_p] * 4 + [c_int, c_void_p] + [c_int] * 5 + [c_void_p]),
    "sigma_split_tf32_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_void_p]),
    "sigma_linear_bf16": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_int, c_int64, c_int, c_int, c_void_p]),
    "sigma_layernorm_fwd_bf16": (c_int, [c_void_p] * 4 + [c_int64, c_int, c_float, c_void_p]),
    "sigma_patch_merge_norm_fwd_bf16": (c_int, [c_void_p] * 4 + [c_int] * 4 + [c_float, c_void_p]),
    "sigma_merge_norm_gate_fwd_bf16": (c_int, [c_void_p, c_int, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_int64, c_void_p,
                                               c_void_p, c_int64, c_int64, c_int64, c_int64, c_int, c_float, c_void_p]),
    "sigma_dwconv3x3_silu_fwd_bf16": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_int64] + [c_int] * 4 + [c_void_p]),
    "sigma_ss2d_scan_fwd_bf16": (c_int, [c_int] + [c_void_p] * 7 + [c_int] * 7 + [c_void_p, c_size_t, c_void_p]),
    "sigma_scan_bwd_det_workspace_bytes": (c_size_t, [c_int] * 6),
    "sigma_scan_bwd_det": (c_int, [c_void_p] * 15 + [c_int] * 7 + [c_void_p, c_size_t, c_int, c_void_p]),
    "sigma_ss2d_scan_bwd_det_workspace_bytes": (c_size_t, [c_int] * 6),
    "sigma_ss2d_scan_bwd_det": (c_int, [c_int] + [c_void_p] * 14 + [c_int] * 7 + [c_void_p, c_size_t, c_int, c_void_p]),
    "sigma_ss2d_scan_bwd_saved_det": (c_int, [c_int] + [c_void_p] * 15 + [c_int] * 7 + [c_void_p, c_size_t, c_int, c_void_p]),
    "sigma_layernorm_bwd_det_workspace_bytes": (c_size_t, [c_int64, c_int]),
    "sigma_layernorm_bwd_det": (c_int, [c_void_p] * 6 + [c_int64, c_int, c_float, c_void_p, c_size_t, c_void_p]),
    "sigma_upsample_bilinear_bwd": (c_int, [c_void_p, c_void_p] + [c_int] * 6 + [c_float, c_float, c_int, c_void_p]),
}

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
