"""CPU: the op-level scan backward at 16 < d_state <= 256 (scan_op_bwd_wide.cu), host side and SASS.
* sigma_test_scan_plan's backward sweeps plan every d_state 17..256 (one walk per CTA after a serial state sweep, 32 channels per
  CTA, 32-position tiles, forced L-segment counts ignored) and refuse 257; the workspace queries are non-zero and the
  deterministic one is no smaller than the default one.
* The kernel exists for every (element type, padded width), contains no float atomic or reduction, and adds no `_det` symbol:
  every entry point runs the same deterministic kernel."""
import re

import pytest
import torch

from helpers import scan_plan
from test_deterministic_sass_cpu import FLOAT_ATOMIC, sass  # noqa: F401  (module-scoped fixture: the library's SASS by function)

SHAPES = [(2, 1536, 4800, 4), (1, 36, 77, 3), (3, 96, 2100, 2), (1, 8192, 690, 4)]   # (batch, dim, L, groups)
WIDE = [f"_ZN5sigma23scan_op_bwd_wide_kernelI{t}Li{n}EEEvNS_17ScanBwdWideParamsE"
        for t in ("f", "6__half", "13__nv_bfloat16") for n in (32, 64, 128, 256)]


def test_plan_every_wide_state():
    for bt, dim, L, G in SHAPES:
        for N in range(17, 257):
            for sweep in ("bwd", "bwd_det"):
                dt = (torch.float32, torch.float16, torch.bfloat16)[N % 3]
                p = scan_plan(sweep, bt, dim, L, N, G, dt, nsplit=N % 5)
                what = (bt, dim, L, N, G, sweep, p)
                assert p["route"] == "generic" and p["nsplit"] == 1 and p["channels"] == 32, what
                assert p["ntiles"] == p["tiles_per_split"] == -(-L // 32), what
                assert p["state_nsplit"] == 1 and p["state_tiles_per_split"] == p["ntiles"], what
        for sweep in ("bwd", "bwd_det"):
            with pytest.raises(RuntimeError):
                scan_plan(sweep, bt, dim, L, 257, G, ws_bytes=1 << 40)


def test_plan_refuses_a_short_workspace():
    with pytest.raises(RuntimeError):
        scan_plan("bwd", 2, 1536, 4800, 32, 4, ws_bytes=1 << 20)


def test_workspace_queries():
    from sigma_b200 import _lib
    L_ = _lib.lib()
    for bt, dim, L, G in SHAPES:
        for N in (17, 32, 33, 64, 100, 128, 171, 256):
            for dt in (_lib.F32, _lib.F16, _lib.BF16):
                w = L_.sigma_scan_bwd_workspace_bytes(bt, dim, L, N, G, dt)
                wd = L_.sigma_scan_bwd_det_workspace_bytes(bt, dim, L, N, G, dt)
                assert w > 0 and wd >= w, (bt, dim, L, N, G, dt, w, wd)
                # at least the tile-start states of the state sweep and the dB / dC partials of every channel tile of a group
                npad = 1 << max(5, (N - 1).bit_length())
                tpg = -(-(dim // G) // 32)
                assert w >= 4 * (bt * dim * -(-L // 32) * npad + 2 * tpg * bt * G * N * L)
    assert L_.sigma_scan_bwd_det_workspace_bytes(2, 64, 100, 257, 1, _lib.F32) == 0


def test_every_wide_instance_exists(sass):  # noqa: F811
    missing = [n for n in WIDE if n not in sass]
    assert not missing, missing
    assert sorted(n for n in sass if "scan_op_bwd_wide_kernel" in n) == sorted(WIDE)


def test_wide_kernels_have_no_float_atomics(sass):  # noqa: F811
    bad = {n: [l.strip() for l in body if FLOAT_ATOMIC.search(l)][:3] for n, body in sass.items() if "scan_op_bwd_wide" in n}
    bad = {n: v for n, v in bad.items() if v}
    assert not bad, f"float atomics / reductions in the wide-state backward: {bad}"


def test_no_wide_det_symbol(sass):  # noqa: F811
    assert not [n for n in sass if "wide" in n and "_det" in n]
    assert not [n for n in sass if re.search(r"scan_op_bwd_wide\w*_det", n)]
