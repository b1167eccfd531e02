"""CPU: the fp16 inference mode's host pieces — mode selection, the symbols the library exports (the fp16 kernels are separate
instances; every bf16 one keeps its name), and the launch plans: the fp16 GEMM and the fp16 fused scan stage the same bytes as
their bf16 twins, so they must launch exactly the bf16 plans, and refuse exactly what the bf16 calls refuse."""
import ctypes
import re
import subprocess

import pytest
import torch

from test_launch_heuristics_cpu import FWD_SHAPES, GEMM_SHAPES


def _lib():
    from sigma_b200 import _lib as L
    return L


def test_fp16_mode_selection_on_the_host():
    from sigma_b200 import fused
    with torch.no_grad():
        assert fused.precision() in ("tf32", "tf32x3")
        with fused.fp16_inference():
            assert fused.precision() == "fp16"
            assert fused._interior_dtype() == torch.float16
            with torch.autocast("cuda", dtype=torch.bfloat16):
                assert fused.precision() == "fp16"                 # the context wins over autocast, as fp8's does
            with torch.enable_grad():
                assert fused.precision() in ("tf32", "tf32x3")   # autograd on: the mode does not exist
            with fused.fp16_inference(False):
                assert fused.precision() in ("tf32", "tf32x3")
            with fused.fp8_inference():
                with pytest.raises(ValueError):
                    fused.precision()
            assert fused.precision() == "fp16"
            assert fused.logits_bar(0.01) == pytest.approx(2 * 0.01 + fused.BF16_FLOOR)
            with pytest.raises(ValueError):
                fused.logits_bar()                                 # relative bar: the composed error is required
        assert fused.precision() in ("tf32", "tf32x3")
        with torch.autocast("cuda", dtype=torch.float16):
            assert fused.precision() in ("tf32", "tf32x3")       # fp16 autocast is still not a mode


def test_inference_pipeline_refuses_fp8_and_fp16_together():
    from sigma_b200.pipeline import InferencePipeline
    with pytest.raises(ValueError):
        InferencePipeline(None, 1, 64, 96, fp8=True, fp16=True)


def _kernels():
    from sigma_b200 import _lib as L
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-sass", L.LIB_PATH], capture_output=True, text=True)
    if out.returncode != 0:
        pytest.skip("cuobjdump is not available")
    return set(re.findall(r"Function : (\S+)", out.stdout))


WIDTHS = (32, 64, 96, 128, 160, 192, 224, 256)


def test_fp16_kernels_are_separate_symbols_and_the_bf16_ones_stay():
    names = _kernels()
    for bn in WIDTHS:
        assert f"_ZN5sigma16gemm_fp16_kernelILi{bn}EEEvNS_10GemmParamsE" in names
        assert f"_ZN5sigma16gemm_tf32_kernelILi{bn}ELb0ELb0ELb1EEEvNS_10GemmParamsE" in names     # bf16 instance, same name
    assert "_ZN5sigma25dwconv3x3_silu_tma_kernelI6__halfEEvNS_11DwTmaParamsE" in names
    assert "_ZN5sigma25dwconv3x3_silu_tma_kernelI13__nv_bfloat16EEvNS_11DwTmaParamsE" in names
    # the fused scan: every (d_state, padded dt_rank, pass) of the bf16 inference build, 3-CTA budget only
    for XT in ("6__half", "13__nv_bfloat16"):
        scans = {n for n in names if n.startswith("_ZN5sigma16ss2d_scan_kernel") and n.endswith(f"Lb0E{XT}EEvNS_10Ss2dParamsE")}
        want = {f"_ZN5sigma16ss2d_scan_kernelILi{n}ELi1ELi{rp}ELi{mode}ELi3ELb0E{XT}EEvNS_10Ss2dParamsE"
                for n in (4, 8, 16) for rp in (4, 8, 12, 16, 24, 32, 48, 64) for mode in (0, 1, 2)}
        assert scans == want, XT
    # row-wise: fp16-output LayerNorm / patch-merge LayerNorm and fp16-in / fp16-out merge + norm + gate, fast and generic
    assert "_ZN5sigma20row_norm_fast_kernelILi32ELi6ELi1ELi0Ef6__halfEEvNS_13RowNormParamsE" in names
    assert "_ZN5sigma20row_norm_fast_kernelILi32ELi6ELi1ELi1Ef6__halfEEvNS_13RowNormParamsE" in names
    assert any(re.match(r"_ZN5sigma20row_norm_fast_kernelILi\d+ELi\d+ELi4ELi0E6__halfS1_EEvNS_13RowNormParamsE", n) for n in names)
    assert any(re.match(r"_ZN5sigma15row_norm_kernelILi\d+E6__halfS1_EEvNS_13RowNormParamsE", n) for n in names)
    assert "_ZN5sigma20row_norm_fast_kernelILi32ELi6ELi1ELi0Ef13__nv_bfloat16EEvNS_13RowNormParamsE" in names   # the bf16 LN stays


def _gemm_plan(M, N, K, mode):
    out = (ctypes.c_int64 * 6)()
    rc = _lib().lib().sigma_test_gemm_plan(M, N, K, mode, 0, 0, 0, out)
    return rc, list(out)


@pytest.mark.parametrize("bn", [None, *WIDTHS])
@pytest.mark.parametrize("M,N,K", [(74 * 60 * 80, 768, 192), (128 * 300 + 1, 264, 104), (129, 8, 8)] + GEMM_SHAPES)
def test_fp16_gemm_plan_is_the_bf16_plan(M, N, K, bn, monkeypatch):
    if bn is None:
        monkeypatch.delenv("SIGMA_GEMM_BN", raising=False)
    else:
        monkeypatch.setenv("SIGMA_GEMM_BN", str(bn))
    rc16, p16 = _gemm_plan(M, N, K, 7)
    rcb, pb = _gemm_plan(M, N, K, 2)
    assert rc16 == rcb == 0
    assert p16 == pb
    if bn is not None:
        assert p16[0] == bn


def test_fp16_gemm_plan_rejects_what_the_bf16_plan_rejects(monkeypatch):
    monkeypatch.setenv("SIGMA_GEMM_BN", "48")
    assert _gemm_plan(1280, 768, 192, 7)[0] != 0
    monkeypatch.delenv("SIGMA_GEMM_BN")
    out = (ctypes.c_int64 * 6)()
    assert _lib().lib().sigma_test_gemm_plan(1280, 768, 192, 7, 2, 30, 40, out) != 0      # no conv instance
    assert _gemm_plan(1280, 768, 192, 6)[0] != 0 and _gemm_plan(1280, 768, 192, 8)[0] != 0   # not modes


def _scan_plan(kind, B, H, W, D, N, R, code, force=0, ws=None):
    from helpers import ss2d_kind
    L = _lib().lib()
    k = ss2d_kind(kind)
    if ws is None:
        ws = L.sigma_ss2d_scan_workspace_bytes(k, B, H, W, D, N)
    out = (ctypes.c_int64 * 8)()
    rc = L.sigma_test_ss2d_fwd_plan(k, B, H, W, D, N, R, code, force, ws, out)
    return rc, list(out)


@pytest.mark.parametrize("kind,H,W,D,N,R", FWD_SHAPES)
@pytest.mark.parametrize("images", [1, 2, 8, 74])
def test_fp16_scan_plan_is_the_bf16_plan(kind, H, W, D, N, R, images, monkeypatch):
    from test_launch_heuristics_cpu import SCAN_ENV
    for e in SCAN_ENV:
        monkeypatch.delenv(e, raising=False)
    B = 2 * images if kind == "cross" else images
    for force in (0, 1, 2, 7, 100):
        for ws in (None, 0):
            rc16, p16 = _scan_plan(kind, B, H, W, D, N, R, 3, force, ws)
            rcb, pb = _scan_plan(kind, B, H, W, D, N, R, 1, force, ws)
            assert rc16 == rcb and p16 == pb, (force, ws)
    assert _scan_plan(kind, B, H, W, D, N, R, 3)[1][6] == 3                     # the 3-CTA register budget, as bf16


@pytest.mark.parametrize("kind,B,H,W,D,N,R", [
    ("cross4", 2, 30, 40, 36, 16, 24),      # D % 8 != 0: not 16-byte TMA rows of a 16-bit xc
    ("cross4", 2, 30, 40, 768, 5, 24),      # d_state not in {4, 8, 16}
    ("seq2", 2, 30, 40, 768, 4, 65),        # dt_rank > 64
    ("cross", 3, 30, 40, 768, 4, 24),       # CROSS: batch = 2·images
])
def test_fp16_scan_plan_fails_where_the_bf16_plan_fails(kind, B, H, W, D, N, R):
    rc16, _ = _scan_plan(kind, B, H, W, D, N, R, 3)
    rcb, _ = _scan_plan(kind, B, H, W, D, N, R, 1)
    assert rc16 != 0 and rc16 == rcb
