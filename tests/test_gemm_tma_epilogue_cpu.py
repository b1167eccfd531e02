"""CPU: the tf32x3 linear instance with TMA-stored output tiles (gemm_x3_tma_kernel, plan mode 5 of sigma_test_gemm_plan).
* its launch plan: the tile width is the register-stored instance's, the ring stages [A | W_hi | W_lo] after two 8 KB staging
  buffers per consumer warpgroup, and every plan fits the H100's shared memory with the CTAs per SM it counts on;
* the built instances keep accumulators, A fragments and the staged epilogue in registers: no local memory at any width."""
import ctypes
import re
import subprocess

import pytest

WIDTHS = list(range(32, 257, 32))
SMEM_PER_BLOCK = 227 * 1024
SMEM_PER_SM = 228 * 1024
STAGING = 2 * 2 * 64 * 32 * 4
GEMM_SHAPES = [(1, 16, 32), (77, 160, 192), (1000, 384, 96), (4096, 320, 1536), (38417, 768, 384), (102401, 4, 36),
               (355200, 768, 192), (2841600, 384, 96), (177600, 1536, 384), (177600, 384, 768), (700, 3072, 768)]


@pytest.fixture(scope="module")
def L():
    from sigma_b200 import _lib
    return _lib.lib()


def _plan(L, M, N, K, mode):
    from sigma_b200 import _lib
    out = (ctypes.c_int64 * 6)()
    _lib.check(L.sigma_test_gemm_plan(M, N, K, mode, 0, 0, 0, out), "sigma_test_gemm_plan")
    return dict(zip(("bn", "stages", "grid", "tiles", "smem", "ctas_per_sm"), (int(v) for v in out)))


def _w_bytes(bn):
    return -(-bn * 32 * 4 // 1024) * 1024


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_tma_epilogue_plan_is_launchable(L, M, N, K, monkeypatch):
    monkeypatch.delenv("SIGMA_GEMM_BN", raising=False)
    for bn in [None] + WIDTHS:
        if bn is not None:
            monkeypatch.setenv("SIGMA_GEMM_BN", str(bn))
        pl, reg = _plan(L, M, N, K, 5), _plan(L, M, N, K, 1)
        assert pl["bn"] == reg["bn"] == (bn or L.sigma_test_pick_bn(N, -(-M // 128)))
        assert pl["tiles"] == reg["tiles"]
        assert 2 <= pl["stages"] <= 8
        assert pl["smem"] == pl["stages"] * (128 * 32 * 4 + 2 * _w_bytes(pl["bn"])) + STAGING + 1024
        assert pl["smem"] <= SMEM_PER_BLOCK
        assert pl["ctas_per_sm"] * (pl["smem"] + 1024) <= SMEM_PER_SM
        assert 1 <= pl["grid"] <= min(pl["tiles"], 132 * pl["ctas_per_sm"])
        # the stage without the unwritten A_lo tile: never a shallower ring where one CTA runs per SM either way
        if pl["ctas_per_sm"] == 1 and reg["ctas_per_sm"] == 1:
            assert pl["stages"] >= reg["stages"]


def test_tma_epilogue_ring_depths(L, monkeypatch):
    """The widths the Sigma-tiny projections run at: 96 keeps two CTAs per SM, 160 and 192 get a third stage."""
    expect = {32: (3, 2), 64: (2, 2), 96: (2, 2), 128: (4, 1), 160: (3, 1), 192: (3, 1), 224: (2, 1), 256: (2, 1)}
    for bn, (stages, ctas) in expect.items():
        monkeypatch.setenv("SIGMA_GEMM_BN", str(bn))
        pl = _plan(L, 177600, 1536, 384, 5)
        assert (pl["stages"], pl["ctas_per_sm"]) == (stages, ctas), f"BN={bn}: {pl}"


def test_tma_epilogue_plan_has_no_conv(L):
    out = (ctypes.c_int64 * 6)()
    assert L.sigma_test_gemm_plan(0, 96, 96, 5, 2, 30, 40, out) == -1    # SIGMA_EINVAL
    assert L.sigma_test_gemm_plan(1000, 96, 96, 6, 0, 0, 0, out) == -1


def test_tma_epilogue_instances_do_not_spill():
    from sigma_b200 import build
    lib = build.build()
    out = subprocess.run(["cuobjdump", "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    seen = {}
    for name, usage in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out):
        m = re.fullmatch(r"_ZN5sigma18gemm_x3_tma_kernelILi(\d+)EEEvNS_10GemmParamsE", name)
        if m:
            seen[int(m.group(1))] = usage
    assert sorted(seen) == WIDTHS, f"instances found: {sorted(seen)}"
    for bn, usage in sorted(seen.items()):
        fields = dict(kv.split(":", 1) for kv in usage.split())
        assert fields["LOCAL"] == "0" and fields["STACK"] == "0", f"BN={bn}: {usage}"


def test_tf32x3_rejects_what_a_tensor_map_cannot_describe(L):
    """The TMA-stored epilogue needs C and the residual 16-byte aligned in base and row stride; sigma_linear_tf32x3 rejects
    anything else before it touches the device (the pointers here are never dereferenced)."""
    from sigma_b200 import _lib
    P = ctypes.c_void_p
    A, W, Wlo, C, R = P(1 << 20), P(2 << 20), P(3 << 20), P(4 << 20), P(5 << 20)
    ok = dict(A=A, lda=64, W=W, Wlo=Wlo, res=R, ldr=64, C=C, ldc=64)
    for bad in [dict(C=P((4 << 20) + 4)), dict(ldc=66), dict(res=P((5 << 20) + 8)), dict(ldr=66)]:
        a = {**ok, **bad}
        rc = L.sigma_linear_tf32x3(a["A"], a["lda"], a["W"], a["Wlo"], None, a["res"], a["ldr"], None, a["C"], a["ldc"], 1000, 64, 64, None)
        assert rc == -1, bad                                                        # SIGMA_EINVAL
        assert "sigma_linear_tf32x3" in _lib.lib().sigma_last_error().decode()
