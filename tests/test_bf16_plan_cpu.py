"""CPU: the launch plans of the bf16 GEMM instance (sigma_test_gemm_plan with x3 = 2) — every width fits shared memory with a
ring of >= 2 stages, the plan equals the tf32 one (a bf16 k-block is the same 128-byte swizzle row), and bad widths or modes are
rejected."""
import ctypes

import pytest

from helpers import gemm_plan


def _plan(M, N, K, mode, conv=(0, 0, 0)):
    from sigma_b200 import _lib
    out = (ctypes.c_int64 * 6)()
    rc = _lib.lib().sigma_test_gemm_plan(M, N, K, mode, *conv, out)
    return rc, dict(zip(("bn", "stages", "grid", "tiles", "smem", "ctas_per_sm"), (int(v) for v in out)))


@pytest.mark.parametrize("bn", [32, 64, 96, 128, 160, 192, 224, 256])
@pytest.mark.parametrize("M,N,K", [(74 * 60 * 80, 768, 192), (128 * 300 + 1, 264, 104), (129, 8, 8)])
def test_bf16_plan_fits_shared_memory(bn, M, N, K, monkeypatch):
    monkeypatch.setenv("SIGMA_GEMM_BN", str(bn))
    rc, pl = _plan(M, N, K, 2)
    assert rc == 0
    assert pl["bn"] == bn and pl["stages"] >= 2
    assert pl["smem"] * pl["ctas_per_sm"] <= 228 * 1024 and pl["smem"] <= 227 * 1024
    assert pl["tiles"] == -(-M // 128) * -(-N // bn) and 1 <= pl["grid"] <= min(pl["tiles"], 132 * pl["ctas_per_sm"])
    assert pl == gemm_plan(M, N, K, False)


@pytest.mark.parametrize("bad", ["0", "16", "48", "288", "x"])
def test_bf16_plan_rejects_bad_width(bad, monkeypatch):
    monkeypatch.setenv("SIGMA_GEMM_BN", bad)
    rc, _ = _plan(128 * 10, 768, 192, 2)
    assert rc != 0


@pytest.mark.parametrize("mode,conv", [(3, (0, 0, 0)), (-1, (0, 0, 0)), (2, (2, 30, 40))])
def test_bf16_plan_rejects_bad_mode(mode, conv, monkeypatch):
    monkeypatch.delenv("SIGMA_GEMM_BN", raising=False)
    rc, _ = _plan(128 * 10, 768, 192, mode, conv)
    assert rc != 0
