"""CPU: the FP8 inference mode's host pieces — the e4m3 emulation the GPU tests compare against, the e4m3 GEMM's launch plan, and
the symbols the library exports (every kernel the bf16 mode had keeps its name; the FP8 kernels are separate ones)."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import fp8_ref as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_e4m3_emulation_matches_torch_on_every_fp32_in_range():
    """Every non-negative fp32 bit pattern up to 448 (e4m3's largest finite value, where torch's cast stops saturating), and the
    same values negated in a strided sample: the emulation rounds exactly like torch.float8_e4m3fn (round to nearest even,
    subnormals from 2^-9)."""
    hi = int(np.float32(448.0).view(np.uint32))
    for start in range(0, hi + 1, 1 << 24):
        x = np.arange(start, min(start + (1 << 24), hi + 1), dtype=np.uint32).view(np.float32)
        ref = torch.from_numpy(x).to(torch.float8_e4m3fn).float().numpy()
        got = F.e4m3(x)
        assert np.array_equal(got, ref), f"first mismatch at {x[np.argmax(got != ref)]!r}"
        xn = -x[::97]
        assert np.array_equal(F.e4m3(xn), torch.from_numpy(xn).to(torch.float8_e4m3fn).float().numpy())


def test_e4m3_emulation_saturates_and_quantize_rows_rules():
    assert np.array_equal(F.e4m3(np.array([464.0, 1e30, -np.inf, np.inf], np.float32)), np.array([448, 448, -448, 448], np.float32))
    x = np.array([[0, 0, 0, 0], [1, -2, 3, 448], [1e-40, 0, -1e-40, 0]], np.float32)
    q, s = F.quantize_rows(x)
    assert s[0] == 1 and not q[0].any()                                   # zero row: s = 1, q = 0
    assert s[1] == np.float32(448) / np.float32(448) and q[1, 3] == 448   # the row's amax maps to 448
    assert np.isfinite(q).all() and np.isfinite(s).all()                  # a subnormal amax: 448 / amax clamped to FLT_MAX
    assert np.all(np.abs(q).max(axis=1)[1:] <= 448)


def _plan(M, N, K, mode):
    from sigma_b200 import _lib
    out = (ctypes.c_int64 * 6)()
    rc = _lib.lib().sigma_test_gemm_plan(M, N, K, mode, 0, 0, 0, out)
    return rc, list(out)


FP8_WIDTHS = {32, 64}


@pytest.mark.parametrize("N", [8, 40, 96, 136, 192, 264, 384, 768, 1536, 3072])
@pytest.mark.parametrize("M", [1, 1200, 19200, 76800, 307200])
def test_fp8_plan_picks_only_instantiated_widths(M, N, monkeypatch):
    monkeypatch.delenv("SIGMA_GEMM_BN", raising=False)
    rc, (bn, stages, grid, tiles, smem, ctas) = _plan(M, N, 128, 4)
    assert rc == 0
    assert bn in FP8_WIDTHS
    assert ctas == 2                                     # the two accumulator sets fit two CTAs per SM at these widths
    assert stages >= 2 and smem <= 227 * 1024 and grid <= 132 * ctas


def test_fp8_plan_rejects_forced_widths_beyond_64(monkeypatch):
    for bn in (32, 64):
        monkeypatch.setenv("SIGMA_GEMM_BN", str(bn))
        assert _plan(4096, 384, 96, 4)[1][0] == bn
    for bn in (96, 128, 256):
        monkeypatch.setenv("SIGMA_GEMM_BN", str(bn))
        assert _plan(4096, 384, 96, 4)[0] != 0
    assert _plan(4096, 384, 96, 2)[0] == 0               # the bf16 instance keeps its widths


def _kernels():
    from sigma_b200 import _lib
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True)
    if out.returncode != 0:
        pytest.skip("cuobjdump is not available")
    return set(re.findall(r"Function : (\S+)", out.stdout))


def test_fp8_kernels_are_separate_symbols_and_the_bf16_ones_stay():
    names = _kernels()
    for bn in (32, 64, 96, 128, 160, 192, 224, 256):
        assert f"_ZN5sigma16gemm_tf32_kernelILi{bn}ELb0ELb0ELb1EEEvNS_10GemmParamsE" in names     # bf16 instance, same name
        assert f"_ZN5sigma16gemm_tf32_kernelILi{bn}ELb1ELb0ELb0EEEvNS_10GemmParamsE" in names     # tf32x3
    for bn in sorted(FP8_WIDTHS):
        assert f"_ZN5sigma15gemm_fp8_kernelILi{bn}EEEvNS_10GemmParamsE" in names
    assert not any(re.match(r"_ZN5sigma15gemm_fp8_kernelILi(?!32E|64E)", n) for n in names)
    assert "_ZN5sigma25quantize_e4m3_rows_kernelIfEEvPKT_xPhxPfxi" in names
    assert "_ZN5sigma25quantize_e4m3_rows_kernelI13__nv_bfloat16EEvPKT_xPhxPfxi" in names
    e4m3_norms = [n for n in names if "row_norm" in n and "E4M3Rows" in n]
    assert e4m3_norms and all(n.startswith(("_ZN5sigma20row_norm_fast_kernel", "_ZN5sigma15row_norm_kernel")) for n in e4m3_norms)
    assert "_ZN5sigma20row_norm_fast_kernelILi32ELi6ELi1ELi0Ef13__nv_bfloat16EEvNS_13RowNormParamsE" in names   # the bf16 LN stays


def test_fp8_mode_selection_on_the_host():
    from sigma_b200 import fused
    with torch.no_grad():
        assert fused.precision() in ("tf32", "tf32x3")
        with fused.fp8_inference():
            assert fused.precision() == "fp8"
            with torch.enable_grad():
                assert fused.precision() in ("tf32", "tf32x3")   # autograd on: the mode does not exist
            with fused.fp8_inference(False):
                assert fused.precision() in ("tf32", "tf32x3")
        assert fused.precision() in ("tf32", "tf32x3")
