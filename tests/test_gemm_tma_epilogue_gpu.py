"""GPU: sigma_linear_tf32x3 stores its output tiles through shared memory with TMA; sigma_test_linear_tf32x3_regs runs the same
call with the register-stored epilogue.  Both add bias and residual·rscale with the same operations in the same order, so C is
BIT-IDENTICAL: at every tile width, with and without bias, residual and rscale, with an M tail (a last row tile whose second
warpgroup has no rows, and one where it has some), a last column tile that overhangs N, C and the residual inside wider rows,
and several tiles per CTA so each staging buffer is reused across tiles.  Neither route writes past M rows or N columns."""
import ctypes

import pytest
import torch

import procedural as P

pytestmark = pytest.mark.gpu
S = 67
NAN_BITS = 0x7FC00000


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _plan(M, N, K, mode):
    from sigma_b200 import _lib
    out = (ctypes.c_int64 * 6)()
    _lib.check(_lib.lib().sigma_test_gemm_plan(M, N, K, mode, 0, 0, 0, out), "sigma_test_gemm_plan")
    return dict(zip(("bn", "stages", "grid", "tiles", "smem", "ctas_per_sm"), (int(v) for v in out)))


def _split(W):
    hi = (W.view(torch.int32) & -8192).view(torch.float32)       # the low 13 mantissa bits cleared
    return hi.contiguous(), (W - hi).contiguous()


def _linear(A, Whi, Wlo, bias, res, rs, C, regs=False):
    from sigma_b200 import _lib
    M, K = A.shape
    N = Whi.shape[0]
    fn = _lib.lib().sigma_test_linear_tf32x3_regs if regs else _lib.lib().sigma_linear_tf32x3
    rc = fn(_p(A), A.stride(0), _p(Whi), _p(Wlo), _p(bias), _p(res), res.stride(0) if res is not None else 0, _p(rs), _p(C), C.stride(0),
            M, N, K, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    _lib.check(rc, fn.__name__)


def _inputs(tag, M, N, K, extras, ldr):
    A = P.randn(S, tag + "/A", (M, K)).cuda()
    Whi, Wlo = _split(P.randn(S, tag + "/W", (N, K), K ** -0.5).cuda())
    bias = P.randn(S, tag + "/b", (N,)).cuda() if "b" in extras else None
    res = rs = None
    if "r" in extras:
        res = torch.full((M, ldr), float("nan"), device="cuda")[:, :N]
        res.copy_(P.randn(S, tag + "/r", (M, N)).cuda())
        rs = P.randn(S, tag + "/s", (N,), 0.2, 1.0).cuda() if "s" in extras else None
    return A, Whi, Wlo, bias, res, rs


def _untouched(t, what):
    bad = int((t.contiguous().view(torch.int32) != NAN_BITS).sum())
    assert bad == 0, f"{what}: {bad} guard elements were written"


def _compare(tag, M, N, K, extras, ldc=None, ldr=None):
    """C of the TMA route against C of the register route; C has ldc - N guard columns and 3 guard rows in both"""
    A, Whi, Wlo, bias, res, rs = _inputs(tag, M, N, K, extras, ldr or N)
    outs = []
    for regs in (False, True):
        cbuf = torch.full((M + 3, ldc or N), float("nan"), device="cuda")
        _linear(A, Whi, Wlo, bias, res, rs, cbuf[:M, :N], regs)
        torch.cuda.synchronize()
        route = "register" if regs else "TMA"
        _untouched(cbuf[:, N:], f"{tag} {route}: columns past N")
        _untouched(cbuf[M:], f"{tag} {route}: rows past M")
        outs.append(cbuf[:M, :N])
    got, ref = outs
    assert bool(torch.isfinite(got).all()), f"{tag}: non-finite output"
    neq = int((got.view(torch.int32) != ref.view(torch.int32)).sum())
    assert neq == 0, f"{tag}: {neq} of {M * N} elements differ between the TMA and the register epilogue"
    # and both are the fp32-grade product: max error over the largest |A|·|W|^T + |bias| + |residual·rscale| below the tf32x3
    # max-norm bar (the register route's own fp64 tests bound it element by element)
    W64 = Whi.double() + Wlo.double()
    r64, mag = A.double() @ W64.t(), A.double().abs() @ W64.abs().t()
    if bias is not None:
        r64 += bias.double()
        mag += bias.double().abs()
    if res is not None:
        rr = res.double() * (rs.double() if rs is not None else 1.0)
        r64 += rr
        mag += rr.abs()
    err = float((got.double() - r64).abs().max() / mag.max())
    assert err < 4e-6, f"{tag}: max-norm error {err:.2e}"


@pytest.mark.parametrize("extras", ["", "b", "r", "brs"])
@pytest.mark.parametrize("bn", [32, 64, 96, 128, 160, 192, 224, 256])
def test_tma_and_register_epilogues_are_bit_identical(bn, extras, monkeypatch):
    """N = 200: the last column tile overhangs N at every width but 32 (8 columns of its last chunk); M % 128 = 17 leaves the
    last tile's second warpgroup without rows."""
    monkeypatch.setenv("SIGMA_GEMM_BN", str(bn))
    M, N, K = 128 * 400 + 17, 200, 96
    pl = _plan(M, N, K, 5)
    assert pl["bn"] == bn and pl["tiles"] >= 3 * pl["grid"], pl      # premise: every CTA reuses its staging buffers
    _compare(f"tma-bn{bn}/{extras}", M, N, K, extras)


@pytest.mark.parametrize("bn", [96, 192])
def test_tma_epilogue_strided(bn, monkeypatch):
    """C and the residual inside wider rows (ldc, ldr > N), M % 128 = 100 (the last row tile's second warpgroup has 36 rows),
    K = 200 (a k-block that overhangs K)."""
    monkeypatch.setenv("SIGMA_GEMM_BN", str(bn))
    _compare(f"strided-bn{bn}", 128 * 300 + 100, 384, 200, "brs", ldc=384 + 12, ldr=384 + 20)


@pytest.mark.parametrize("name,N,K,extras", [("in_proj0", 384, 96, ""), ("out_proj0", 96, 192, "r"), ("out_proj2", 384, 768, "r")])
def test_tma_epilogue_sigma_shapes(name, N, K, extras, monkeypatch):
    """Sigma-tiny's stage-0 and stage-2 projections at their planned widths, on the rows of two 480 x 640 images (both
    modalities: 2 x 2 x 19200 stage-0 tokens, 2 x 2 x 1200 at stage 2)."""
    monkeypatch.delenv("SIGMA_GEMM_BN", raising=False)
    _compare(f"sigma/{name}", 4 * (19200 if name.endswith("0") else 1200), N, K, extras)
