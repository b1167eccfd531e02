"""Host-side logic of the C-ABI that needs no GPU: layout helpers, workspace sizes, and argument validation (every
entry point rejects bad arguments with a negative code + message BEFORE touching the device, mirroring the
TORCH_CHECKs of the reference's binding, selective_scan.cpp:165-249)."""
import ctypes

import pytest

from sigma_b200 import _lib


def test_padded_cp_layout():
    L = _lib.lib()
    # x_dbl row = [B (N) | C (N) | dt_r padded to one of 4, 8, 12, 16, 24, 32, 48, 64]
    for N in (4, 8, 16):
        for R, pad in [(1, 4), (4, 4), (5, 8), (6, 8), (12, 12), (13, 16), (24, 24), (25, 32), (48, 48), (49, 64), (64, 64)]:
            assert L.sigma_ss2d_padded_cp(N, R) == 2 * N + pad
        assert L.sigma_ss2d_padded_cp(N, 65) == -1
    # every Sigma width: dt_rank = ceil(d_model / 16) (vmamba.py:1035)
    for d_model, R in [(96, 6), (192, 12), (384, 24), (768, 48), (128, 8), (256, 16), (512, 32), (1024, 64)]:
        assert L.sigma_ss2d_padded_cp(16, R) % 4 == 0 and L.sigma_ss2d_padded_cp(16, R) >= 32 + R


def test_workspace_sizes_are_sane():
    L = _lib.lib()
    L.sigma_ss2d_scan_workspace_bytes.restype = ctypes.c_size_t
    small = L.sigma_ss2d_scan_workspace_bytes(_lib.DIRS_CROSS4, 2, 120, 160, 192, 16)
    big = L.sigma_ss2d_scan_workspace_bytes(_lib.DIRS_CROSS4, 4, 120, 160, 192, 16)
    assert 0 < small < big <= 2 * small + 4096
    assert L.sigma_ss2d_scan_workspace_bytes(_lib.DIRS_CROSS, 2, 120, 160, 192, 4) < small


# The 16-bit and e4m3 row norms: (entry point, valid arguments, index of a pointer to NULL, (index, value) of a bad size, (index,
# address) of an element pointer aligned to 2 of the 4 elements the kernels move at once: 20 is 4- but not 8-byte aligned (16-bit),
# 18 is 2- but not 4-byte aligned (e4m3)).
_ROW_NORM_16_E4M3 = [
    ("sigma_layernorm_fwd_bf16", (16, 16, 16, 16, 4, 96, 1e-5, None), 0, (5, 98), (3, 20)),
    ("sigma_layernorm_fwd_fp16", (16, 16, 16, 16, 4, 96, 1e-5, None), 3, (4, -1), (3, 20)),
    ("sigma_layernorm_fwd_fp8", (16, 16, 16, 16, 16, 4, 96, 1e-5, None), 4, (6, 0), (3, 18)),
    ("sigma_layernorm_fwd_bf16io", (16, 16, 16, 16, 4, 96, 1e-5, None), 1, (5, 98), (0, 20)),
    ("sigma_layernorm_fwd_fp16io", (16, 16, 16, 16, 4, 96, 1e-5, None), 2, (5, 98), (3, 20)),
    ("sigma_layernorm_bwd_bf16", (16, 16, 16, 16, 16, 16, 4, 96, 1e-5, None), 5, (7, 94), (1, 20)),
    ("sigma_layernorm_bwd_fp16", (16, 16, 16, 16, 16, 16, 4, 96, 1e-5, None), 3, (6, -1), (3, 20)),
    ("sigma_patch_merge_norm_fwd_bf16", (16, 16, 16, 16, 1, 4, 4, 96, 1e-5, None), 3, (5, 0), (3, 20)),
    ("sigma_patch_merge_norm_fwd_fp16", (16, 16, 16, 16, 1, 4, 4, 96, 1e-5, None), 0, (7, 98), (3, 20)),
    ("sigma_patch_merge_norm_fwd_fp8", (16, 16, 16, 16, 16, 1, 4, 4, 96, 1e-5, None), 4, (8, 98), (3, 18)),
    ("sigma_merge_norm_gate_fwd_bf16", (16, 4, 96, 96, 16, 16, 16, 96, 16, 16, 96, 96, 4, 4, 96, 1e-5, None), 9, (1, 9), (6, 20)),
    ("sigma_merge_norm_gate_fwd_fp16", (16, 4, 96, 96, 16, 16, 16, 96, 16, 16, 96, 96, 4, 4, 96, 1e-5, None), 0, (14, 98), (9, 20)),
    ("sigma_merge_norm_gate_fwd_fp8", (16, 4, 96, 96, 16, 16, 16, 96, 16, 16, 16, 96, 96, 4, 4, 96, 1e-5, None), 10, (1, 2), (9, 18)),
]


def _with(args, i, v):
    return args[:i] + (v,) + args[i + 1:]


@pytest.mark.parametrize("call", [
    lambda L: L.sigma_layernorm_fwd(None, None, None, None, 4, 96, 1e-5, None),
    lambda L: L.sigma_layernorm_fwd(16, 16, 16, 16, 4, 98, 1e-5, None),                       # C % 4 != 0
    lambda L: L.sigma_layernorm_fwd(16, 16, 16, 20, 4, 96, 1e-5, None),                       # misaligned y
    lambda L: L.sigma_patch_merge_norm_fwd(16, 16, 16, 16, 0, 4, 4, 96, 1e-5, None),          # batch = 0
    lambda L: L.sigma_pixel_shuffle_norm_fwd(16, 16, 16, None, 1, 4, 4, 96, 1e-5, None),
    lambda L: L.sigma_dwconv3x3_silu_fwd(16, 96, 96 * 16, 16, None, 16, 96 * 16, 1, 4, 4, 98, None),
    lambda L: L.sigma_upsample2x_norm_fwd(16, 16, None, 16, 1, 4, 4, 96, 1e-5, None),         # w without b
    lambda L: L.sigma_argmax_hist_fwd(16, 16, 1, 16, 16, None, 1, 300, 16, None),             # > 255 classes
    lambda L: L.sigma_argmax_hist_fwd(16, None, 1, 16, 16, None, 1, 9, 16, None),
    lambda L: L.sigma_ss2d_scan_fwd(7, 16, 16, 16, 16, 16, 16, 16, 2, 4, 4, 64, 16, 4, 36, None, 0, None),    # unknown kind
    lambda L: L.sigma_ss2d_scan_fwd(0, 16, 16, 16, 16, 16, 16, 16, 2, 4, 4, 64, 5, 4, 14, None, 0, None),     # d_state 5
    lambda L: L.sigma_ss2d_scan_fwd(0, 16, 16, 16, 16, 16, 16, 16, 2, 4, 4, 64, 16, 4, 40, None, 0, None),    # wrong Cp
    lambda L: L.sigma_ss2d_scan_fwd(2, 16, 16, 16, 16, 16, 16, 16, 3, 4, 4, 64, 4, 4, 12, None, 0, None),     # CROSS, odd batch
] + [lambda L, fn=fn, a=a: getattr(L, fn)(*a) for fn, args, null, (si, sv), (ai, av) in _ROW_NORM_16_E4M3
     for a in (_with(args, null, None), _with(args, si, sv), _with(args, ai, av))])
def test_bad_arguments_are_rejected_before_the_device(call):
    L = _lib.lib()
    L.sigma_last_error.restype = ctypes.c_char_p
    rc = call(L)
    assert rc < 0, "bad arguments must not be accepted"
    msg = L.sigma_last_error().decode()
    assert msg and "sigma_" in msg, f"no diagnostic for rc={rc}: {msg!r}"
