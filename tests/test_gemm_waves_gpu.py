"""GPU: the wgmma GEMM (sigma_linear_tf32 / sigma_linear_tf32x3 through fused.linear), its implicit-GEMM 3x3 convolution
(sigma_conv3x3_tf32) and the depthwise conv (sigma_dwconv3x3_silu_fwd, and its bf16 instance at Sigma's widths in its three
production stride layouts) in the regime the model runs them in: persistent CTAs
that walk several tiles each — so the producer runs ahead across tile boundaries, the mbarrier ring carries its phase from tile to
tile and the accumulators restart per tile — at every tile width (SIGMA_GEMM_BN), with ragged M / N / K / channel counts and
every epilogue, against fp64 ELEMENT BY ELEMENT, with the memory around each output filled with NaN and checked untouched.
Each multi-wave case asserts its own premise through the library's launch planner (sigma_test_gemm_plan): >= 3 tiles per CTA.

Per-element error bounds.  u = 2^-24 (fp32 unit roundoff); mag = (|A|·|W|^T)_ij, or (|x| ⊛ |w|) for a convolution; K = the
number of products summed (9·Cin for the 3x3 conv).
  tf32    Each operand reaches the tensor core with 10 explicit mantissa bits (truncated or rounded, |a' - a| < 2^-10 |a|),
          so each product is off by less than ((1 + 2^-10)^2 - 1)|a||w| <= (2^-9 + 2^-20)|a||w|.  The fp32 accumulation adds
          at most 2u (one truncating addition) of a partial sum <= mag per product: K·2^-23·mag.
              gamma_tf32(K) = 2^-9 + 2^-20 + K·2^-23          (2.0e-3 at K = 384; < 2.5e-3, the max-norm bar, for K <= 4096)
  tf32x3  a = a_hi + a_lo exactly with |a_lo| < 2^-10 |a| (a_hi keeps 10 mantissa bits).  Lost per product: the dropped
          a_lo·w_lo (< 2^-20 |a||w|) and the tensor core's 10-bit view of a_lo and of w_lo (< 2^-10 of each, so < 2^-20 |a||w|
          each): 3·2^-20 |a||w|.  The accumulation of the 3K partial products: its worst case (3K·2u·mag) is far above what
          occurs — the partial sums of products of either sign stay far below mag — so it is allowed 2^-20·mag.
              gamma_x3 = 3·2^-20 + 2^-20 = 2^-18 = 3.8e-6     (< 4e-6, the max-norm bar)
  Both    The epilogue rounds (acc + bias) and (· + residual·rscale) once each: + 2u·(mag + |bias| + |residual·rscale|).
          GELU (|GELU'| <= 1.13, erff within 2 ulp) scales the pre-activation bound by 1.13 and adds 2^-21·|pre-activation|.
          + 1e-5 absolute, as in the max-norm tests; so at the largest element no bound here is looser than theirs.
A mag-relative bound per element (not one bound against max mag) catches a defect confined to a few tiles or columns.
Measured on an H100 SXM (700 W limit) with the seeded inputs below: tf32 uses up to 0.90 of its bound at K = 4 (few products,
so the 2^-9 operand term is nearly attained) and <= 0.5 elsewhere; tf32x3's error grows like sqrt(K)·u·mag: <= 0.42 of the
bound for the GEMMs (K <= 384), 0.96 for the 384 -> 128 convolution (K = 9·384), the largest K here."""
import ctypes

import pytest
import torch

import procedural as P
from helpers import gemm_plan, record

pytestmark = pytest.mark.gpu
S = 61
U = 2.0 ** -24
NAN_BITS = 0x7FC00000
ABS = 1e-5           # the max-norm tests' absolute term


def gamma(mode, K):
    return 2.0 ** -9 + 2.0 ** -20 + K * 2.0 ** -23 if mode == "tf32" else 2.0 ** -18


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _lib():
    from sigma_b200 import _lib as L
    return L


def _assert_nan_untouched(t, what):
    bits = t.contiguous().view(torch.int32)
    bad = int((bits != NAN_BITS).sum())
    assert bad == 0, f"{what}: {bad} guard elements were written"


def _ratio(tag, got, ref, mag, extra, gam):
    """max over elements of |got - ref| / bound (<= 1 passes); got fp32, the rest fp64, same shape."""
    assert bool(torch.isfinite(got).all()), f"{tag}: non-finite output"
    err = (got.double() - ref).abs()
    bound = gam * mag + 2 * U * extra + ABS
    r = err / bound
    worst = float(r.max())
    if worst > 1.0:
        idx = int(r.argmax())
        pos = tuple(int(i) for i in torch.unravel_index(torch.tensor(idx), r.shape))
        n_bad = int((r > 1).sum())
        raise AssertionError(f"{tag}: {n_bad}/{r.numel()} elements out of bound; worst at {pos}: err {float(err.flatten()[idx]):.3e} "
                             f"> bound {float(bound.flatten()[idx]):.3e} (mag {float(mag.flatten()[idx]):.3e})")
    return worst, float((err / (mag + 1e-30)).max())


def _check_linear(tag, got, A, W, bias, res, rs, mode, chunk=1 << 15):
    """got (M, N) against fp64 A·W^T (+bias) (+res·rs), in row chunks (the full fp64 product of a production shape is GBs)."""
    W64 = W.double()
    Wa = W64.abs()
    K = A.shape[1]
    worst = rel = 0.0
    for r0 in range(0, A.shape[0], chunk):
        a = A[r0:r0 + chunk].double()
        ref = a @ W64.t()
        mag = a.abs() @ Wa.t()
        extra = mag.clone()
        if bias is not None:
            ref += bias.double()
            extra += bias.double().abs()
        if res is not None:
            rr = res[r0:r0 + chunk].double() * (rs.double() if rs is not None else 1.0)
            ref += rr
            extra += rr.abs()
        w, e = _ratio(f"{tag} rows {r0}..", got[r0:r0 + chunk], ref, mag, extra, gamma(mode, K))
        worst, rel = max(worst, w), max(rel, e)
    record("gemm_waves", case=tag, mode=mode, K=K, bound_used=worst, max_err_over_mag=rel)
    return worst


def _multiwave(pl, need=3):
    assert pl["tiles"] >= need * pl["grid"], f"premise: {pl['tiles']} tiles over {pl['grid']} CTAs is < {need} per CTA"


def _run_linear(M, N, K, mode, monkeypatch, bn=None, extras="", lda=None, ldc=None, ldr=None, tag=None):
    from sigma_b200 import fused
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", mode == "tf32")
    assert fused.precision() == mode and fused.USE_OWN_GEMM
    if bn is not None:
        monkeypatch.setenv("SIGMA_GEMM_BN", str(bn))
    else:
        monkeypatch.delenv("SIGMA_GEMM_BN", raising=False)
    pl = gemm_plan(M, N, K, mode == "tf32x3")
    if bn is not None:
        assert pl["bn"] == bn
    _multiwave(pl)
    tag = tag or f"gemm/{M}/{N}/{K}/{extras}"
    dev = "cuda"
    lda, ldc, ldr = lda or K, ldc or N, ldr or N
    abuf = torch.full((M, lda), float("nan"), device=dev)          # columns past K must never be read
    A = P.randn(S, tag + "/A", (M, K)).to(dev)
    abuf[:, :K] = A
    Wt = P.randn(S, tag + "/W", (N, K), K ** -0.5).to(dev)
    bias = P.randn(S, tag + "/b", (N,)).to(dev) if "b" in extras else None
    res = rs = None
    if "r" in extras:
        rbuf = torch.full((M, ldr), float("nan"), device=dev)
        rbuf[:, :N] = P.randn(S, tag + "/r", (M, N)).to(dev)
        res = rbuf[:, :N]
        rs = P.randn(S, tag + "/s", (N,), 0.2, 1.0).to(dev) if "s" in extras else None
    cbuf = torch.full((M + 3, ldc), float("nan"), device=dev)      # rows past M and columns past N are guards
    out = cbuf[:M, :N]
    got = fused.linear(abuf[:, :K], Wt, bias, out=out, residual=res, rscale=rs)
    assert got.data_ptr() == out.data_ptr()
    torch.cuda.synchronize()
    _assert_nan_untouched(cbuf[:, N:], f"{tag}: columns past N")
    _assert_nan_untouched(cbuf[M:], f"{tag}: rows past M")
    _check_linear(f"{tag} {mode} bn={pl['bn']}", out, A, Wt, bias, res, rs, mode)


MODES = ["tf32", "tf32x3"]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("bn", [32, 64, 96, 128, 160, 192, 224, 256])
def test_gemm_every_tile_width_multiwave(bn, mode, monkeypatch):
    """Every wgmma instance (m64nBNk8), forced, on 301 row tiles (M % 128 = 17) x N = 768 — column tiles that overhang N at
    widths 160 and 224 — so every CTA walks >= 3 tiles.  bias + residual·rscale exercise the whole epilogue at each width."""
    _run_linear(128 * 300 + 17, 768, 384, mode, monkeypatch, bn=bn, extras="brs", tag=f"gemm-bn{bn}")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("M,N,K,bn", [
    (128 * 800 + 1, 4, 36, None), (128 * 800 + 127, 36, 4, None), (128 * 300 + 1, 260, 100, None),
    (128 * 300 + 127, 260, 36, 256), (128 * 800 + 1, 4, 100, 32), (128 * 800 + 127, 36, 100, 64), (128 * 400 + 1, 36, 4, 256),
])
def test_gemm_ragged_multiwave(M, N, K, bn, mode, monkeypatch):
    """Ragged edges inside multi-wave runs: K < 32 and K % 32 != 0 (TMA fills past K with zeros), a last column tile that
    overhangs N (N > 256 included), M % 128 in {1, 127}; the planner's width and forced ones."""
    _run_linear(M, N, K, mode, monkeypatch, bn=bn, extras="b")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("extras", ["b", "r", "rs", "brs"])
def test_gemm_epilogues_strided_multiwave(extras, mode, monkeypatch):
    """bias, residual, residual·rscale and all three, with A, C and the residual inside wider rows (lda, ldc, ldr > K, N)."""
    _run_linear(128 * 300 + 17, 768, 192, mode, monkeypatch, extras=extras, lda=192 + 36, ldc=768 + 12, ldr=768 + 20,
                tag=f"gemm-epi/{extras}")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name,N,K,extras", [("in_proj", 768, 192, "b"), ("x_proj", 4 * 44, 384, "")])
def test_gemm_production_shapes_b74(name, N, K, extras, mode, monkeypatch):
    """Sigma-tiny stage 1 (layers.1, 60 x 80 at 480 x 640) at the benchmark's 74 images: M = 355200 rows.  in_proj
    (192 -> 768, oracle/state_shapes.json) and the packed four-direction x_proj (384 -> 4 x Cp, Cp = 2·16 + 12 = 44); every row is
    compared, in chunks."""
    _run_linear(74 * 60 * 80, N, K, mode, monkeypatch, extras=extras, tag=f"prod/{name}")


# ---------------------------------------------------------------- weight-split caches (fused._SPLIT, fused._W9)
def _ref_linear(x, lin):
    return x.double() @ lin.weight.detach().double().t() + lin.bias.detach().double()


def _ref_conv(x, conv):
    return torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).double(), conv.weight.detach().double(), conv.bias.detach().double(),
                                      padding=1).permute(0, 2, 3, 1)


def _mag_conv(x, conv):
    return torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).double().abs(), conv.weight.detach().double().abs(),
                                      padding=1).permute(0, 2, 3, 1)


def _check_cached(what, x, lin, xc, conv, mode):
    from sigma_b200 import fused
    got = fused.linear(x, lin.weight, lin.bias)
    mag = x.double().abs() @ lin.weight.detach().double().abs().t()
    _ratio(f"linear {what} {mode}", got, _ref_linear(x, lin), mag, mag + lin.bias.detach().double().abs(), gamma(mode, x.shape[1]))
    gotc = fused.conv3x3(xc, conv)
    magc = _mag_conv(xc, conv)
    _ratio(f"conv3x3 {what} {mode}", gotc, _ref_conv(xc, conv), magc, magc + conv.bias.detach().double().abs(),
           gamma(mode, 9 * xc.shape[-1]))


@pytest.mark.parametrize("mode", MODES)
def test_weight_caches_follow_in_place_updates(mode, monkeypatch):
    """The tf32x3 weight split (fused._SPLIT) and the conv weight re-ordering (fused._W9) are cached per weight version:
    results must follow the new weights after an optimizer step, a torch.no_grad() in-place op and load_state_dict."""
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", mode == "tf32")
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", mode == "tf32")
    torch.manual_seed(0)
    lin = torch.nn.Linear(96, 160).cuda()
    conv = torch.nn.Conv2d(32, 64, 3, padding=1).cuda()
    x = P.randn(S, "cache/x", (1000, 96)).cuda()
    xc = P.randn(S, "cache/xc", (2, 20, 24, 32)).cuda()
    _check_cached("initial", x, lin, xc, conv, mode)
    params = [lin.weight, lin.bias, conv.weight, conv.bias]
    opt = torch.optim.AdamW(params, lr=1e-2)
    for i, prm in enumerate(params):
        prm.grad = P.randn(S, f"cache/g{i}", tuple(prm.shape)).cuda()
    opt.step()
    _check_cached("after AdamW.step()", x, lin, xc, conv, mode)
    with torch.no_grad():
        lin.weight.mul_(-0.5)
        conv.weight.add_(0.05)
    _check_cached("after a no_grad in-place op", x, lin, xc, conv, mode)
    lin.load_state_dict({"weight": P.randn(S, "cache/lw", (160, 96), 0.1), "bias": P.randn(S, "cache/lb", (160,))})
    conv.load_state_dict({"weight": P.randn(S, "cache/cw", (64, 32, 3, 3), 0.05), "bias": P.randn(S, "cache/cb", (64,))})
    _check_cached("after load_state_dict", x, lin, xc, conv, mode)


def test_writes_through_data_are_not_seen_by_the_weight_caches(monkeypatch):
    """A known limitation (documented in fused.linear and INTEGRATION.md): a write through `.data` does not bump the parameter's
    `_version`, so the cached split / re-ordered weight is used as it was.  A later tracked in-place op refreshes it."""
    from sigma_b200 import fused
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    lin = torch.nn.Linear(96, 160).cuda()
    conv = torch.nn.Conv2d(32, 64, 3, padding=1).cuda()
    x = P.randn(S, "data/x", (1000, 96)).cuda()
    xc = P.randn(S, "data/xc", (2, 20, 24, 32)).cuda()
    y0, c0 = fused.linear(x, lin.weight, lin.bias), fused.conv3x3(xc, conv)
    v0, v1 = lin.weight._version, conv.weight._version
    lin.weight.data.mul_(2.0)
    conv.weight.data.mul_(2.0)
    assert lin.weight._version == v0 and conv.weight._version == v1
    assert torch.equal(fused.linear(x, lin.weight, lin.bias), y0)          # stale: the old split
    assert torch.equal(fused.conv3x3(xc, conv), c0)                         # stale: the old re-ordered weight
    with torch.no_grad():
        lin.weight.mul_(1.0)
        conv.weight.mul_(1.0)
    _check_cached("after a tracked op", x, lin, xc, conv, "tf32x3")


# ---------------------------------------------------------------- implicit-GEMM 3x3 conv through the C-ABI
def _conv_abi(tag, x, w, bias, gelu, mode, B, H, W, Cin, Cout, guard=64):
    """sigma_conv3x3_tf32 on a y that sits inside a NaN-filled buffer; checks the guards and returns y (B, H, W, Cout)."""
    L = _lib()
    w9 = w.permute(2, 3, 0, 1).reshape(9 * Cout, Cin).contiguous()
    lo = None
    if mode == "tf32x3":
        hi, lo = torch.empty_like(w9), torch.empty_like(w9)
        L.check(L.lib().sigma_split_tf32_fwd(_p(w9), _p(hi), _p(lo), w9.numel(), _stream()), "split")
        w9 = hi
    n = B * H * W * Cout
    buf = torch.full((n + 2 * guard,), float("nan"), device="cuda")
    y = buf[guard:guard + n]
    L.check(L.lib().sigma_conv3x3_tf32(_p(x), _p(w9), _p(lo), _p(bias), 1 if gelu else 0, _p(y), B, H, W, Cin, Cout, _stream()), tag)
    torch.cuda.synchronize()
    _assert_nan_untouched(buf[:guard], f"{tag}: before y")
    _assert_nan_untouched(buf[guard + n:], f"{tag}: after y")
    return y.view(B, H, W, Cout)


def _conv_case(B, H, W, Cin, Cout, with_bias, runs, monkeypatch, tag):
    dev = "cuda"
    x = P.randn(S, tag + "/x", (B, H, W, Cin)).to(dev)
    w = P.randn(S, tag + "/w", (Cout, Cin, 3, 3), (9 * Cin) ** -0.5).to(dev)
    bias = P.randn(S, tag + "/b", (Cout,), 0.2).to(dev) if with_bias else None
    xn = x.permute(0, 3, 1, 2).double()
    pre = torch.nn.functional.conv2d(xn, w.double(), bias.double() if with_bias else None, padding=1).permute(0, 2, 3, 1)
    mag = torch.nn.functional.conv2d(xn.abs(), w.double().abs(), padding=1).permute(0, 2, 3, 1)
    extra = mag + (bias.double().abs() if with_bias else 0.0)
    del xn
    for mode, gelu, bn in runs:
        if bn is None:
            monkeypatch.delenv("SIGMA_GEMM_BN", raising=False)
        else:
            monkeypatch.setenv("SIGMA_GEMM_BN", str(bn))
        pl = gemm_plan(0, Cout, Cin, mode == "tf32x3", conv=(B, H, W))
        assert bn is None or pl["bn"] == bn
        _multiwave(pl)
        t = f"{tag} {mode} gelu={gelu} bn={pl['bn']}"
        y = _conv_abi(t, x, w, bias, gelu, mode, B, H, W, Cin, Cout)
        if gelu:   # 1.13 x the pre-activation bound, + 2^-21·|pre| (= 2u · 4|pre|) for the GELU evaluation
            worst, rel = _ratio(t, y, torch.nn.functional.gelu(pre), 1.13 * mag, 1.13 * extra + 4.0 * pre.abs(), gamma(mode, 9 * Cin))
        else:
            worst, rel = _ratio(t, y, pre, mag, extra, gamma(mode, 9 * Cin))
        record("conv_waves", case=t, bound_used=worst, max_err_over_mag=rel)


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(6, 120, 160, 96, 32), (6, 120, 160, 32, 96), (20, 60, 80, 192, 64), (66, 30, 40, 384, 128)])
def test_conv3x3_decoder_shapes_multiwave(B, H, W, Cin, Cout, monkeypatch):
    """The ChannelAttentionBlock's conv pair at the decoder's map sizes, batched so that every CTA walks >= 3 tiles; both
    precisions, with and without the GELU epilogue."""
    runs = [(m, g, None) for m in MODES for g in (False, True)]
    _conv_case(B, H, W, Cin, Cout, True, runs, monkeypatch, f"conv/{B}/{H}/{W}/{Cin}/{Cout}")


@pytest.mark.parametrize("Cin", [4, 36, 100])
@pytest.mark.parametrize("Cout", [36, 40])
def test_conv3x3_ragged_channels_multiwave(Cin, Cout, monkeypatch):
    """Cin < 32 or Cin % 32 != 0 (channels >= Cin zero-filled in the A box and the W box); Cout in {36, 40}, where the W box of
    tap t overhangs into tap t+1's rows, which the epilogue must mask; forced widths 32 / 64 / 256 on a ragged 57 x 75 map; no
    bias when Cin = 36."""
    runs = [(m, g, bn) for m in MODES for bn in (32, 64, 256) for g in ((False, True) if bn == 64 else (False,))]
    _conv_case(20, 57, 75, Cin, Cout, Cin != 36, runs, monkeypatch, f"conv-ragged/{Cin}/{Cout}")


# ---------------------------------------------------------------- depthwise 3x3 + SiLU with a wrapping ring
def _dwconv_grid(B, H, W, D):
    """The persistent grid of dwconv3x3_silu_tma_launch (dwconv_tma.cu): (channel blocks, spatial CTAs), 2 CTAs per SM."""
    cblocks = -(-D // 32)
    ntiles = B * -(-H // 8) * -(-W // 16)
    return cblocks, max(1, min(ntiles, (132 * 2) // cblocks)), ntiles


@pytest.mark.parametrize("B,H,W,D", [(4, 120, 160, 192), (8, 30, 40, 1536), (3, 123, 155, 132)])
def test_dwconv_silu_ring_wraps(B, H, W, D):
    """Every CTA walks >= 9 tiles (> 2 x the 4 ring slots), so the persistent refill and the phase flip run.  x is the strided
    x half of [x | z] rows; the output images sit DC apart with NaN gaps between them; fp64 reference element by element:
    9 FMAs + bias in fp32 (<= 9u·mag), then SiLU (|SiLU'| <= 1.1, ex2.approx / fast division within a few ulp)."""
    L = _lib()
    _, ny, ntiles = _dwconv_grid(B, H, W, D)
    assert ntiles // ny >= 9, f"premise: {ntiles} tiles over {ny} spatial CTAs"
    tag = f"dwring/{B}/{H}/{W}/{D}"
    dev = "cuda"
    xz = P.randn(S, tag + "/xz", (B, H, W, 2 * D)).to(dev)
    w = P.randn(S, tag + "/w", (D, 1, 3, 3), 0.4).to(dev)
    b = P.randn(S, tag + "/b", (D,), 0.2).to(dev)
    ybs = H * W * D + 16                                           # image stride: 16 NaN floats between images
    buf = torch.full((B * ybs + 64,), float("nan"), device=dev)
    rc = L.lib().sigma_dwconv3x3_silu_fwd(_p(xz), 2 * D, H * W * 2 * D, _p(w), _p(b), _p(buf), ybs, B, H, W, D, _stream())
    L.check(rc, tag)
    torch.cuda.synchronize()
    img = buf[:B * ybs].view(B, ybs)
    _assert_nan_untouched(img[:, H * W * D:], f"{tag}: gaps between images")
    _assert_nan_untouched(buf[B * ybs:], f"{tag}: after the last image")
    y = img[:, :H * W * D].reshape(B, H, W, D)
    ref, bound = _dwconv_ref(xz[..., :D], w, b)
    record("dwconv_ring", case=tag, max_err_over_bound=_dwconv_check(tag, y, ref, bound))


def _dwconv_ref(x, w, b):
    """fp64 conv + bias + SiLU of x (B, H, W, D) and the per-element bound of the fp32 kernel: 9 FMAs + bias (<= 10u·mag), then
    SiLU (|SiLU'| <= 1.1, ex2.approx / fast division within a few ulp)"""
    D = x.shape[-1]
    xn = x.permute(0, 3, 1, 2).double()
    pre = torch.nn.functional.conv2d(xn, w.double(), b.double(), padding=1, groups=D).permute(0, 2, 3, 1)
    mag = torch.nn.functional.conv2d(xn.abs(), w.double().abs(), b.double().abs(), padding=1, groups=D).permute(0, 2, 3, 1)
    ref = torch.nn.functional.silu(pre)
    return ref, 1.1 * 10 * U * mag + 2.0 ** -19 * ref.abs() + 1e-12


def _dwconv_check(tag, y, ref, bound):
    assert bool(torch.isfinite(y).all()), f"{tag}: non-finite output (not written?)"
    err = (y.double() - ref).abs()
    bad = err > bound
    assert not bool(bad.any()), (f"{tag}: {int(bad.sum())}/{bad.numel()} elements out of bound; max err {float(err.max()):.3e}, "
                                 f"worst err/bound {float((err / bound).max()):.2f}")
    return float((err / bound).max())


# (D, H, W): Sigma's d_inner at its 480 x 640 stages, Sigma-base's widest (2048 at 720 x 960), and D = 136: a partial 32-channel block
DW_BF16 = [(192, 120, 160), (384, 60, 80), (768, 30, 40), (1536, 15, 20), (2048, 23, 30), (136, 57, 75)]
NAN16 = 0x7FC0


@pytest.mark.parametrize("layout", ["ss2d", "cromb", "conmb"])
@pytest.mark.parametrize("D,H,W", DW_BF16)
def test_dwconv_silu_bf16(D, H, W, layout):
    """sigma_dwconv3x3_silu_fwd_bf16 (dwconv3x3_silu_tma_kernel<__nv_bfloat16>) with the strides of its production calls:
      ss2d   x the x half of in_proj's [x | z] rows (row stride 2D), out (B, L, D)                      (fused.ss2d)
      cromb  x (2, B·L, D) modality-major, one call over the 2B images, out (2B, L, D)                  (fused.cromb_ss2d)
      conmb  x (B·L, D), out the second half of seq (B, 2L, D): offset L·D, image stride 2L·D           (fused.conmb_ss2d)
    with enough images that every CTA walks >= 9 tiles.  x is bf16 and the reference runs on its exact values; the bound is the fp32
    one plus one bf16 store (rowwise_ref64.bf16_store_bound).  The first half of every conmb image (NaN gaps between the images)
    and the guards around the buffer stay NaN."""
    from oracle import rowwise_ref64 as RR
    L = _lib()
    step = 2 if layout == "cromb" else 1
    B = step
    while True:
        _, ny, ntiles = _dwconv_grid(B, H, W, D)
        if ntiles // ny >= 9:
            break
        B += step
    tag = f"dw16/{layout}/{B}/{H}/{W}/{D}"
    dev = "cuda"
    HW = H * W
    xin = P.randn(S, tag + "/x", (B, H, W, 2 * D if layout == "ss2d" else D)).to(dev).to(torch.bfloat16)
    w = P.randn(S, tag + "/w", (D, 1, 3, 3), 0.4).to(dev)
    b = P.randn(S, tag + "/b", (D,), 0.2).to(dev)
    xrs = 2 * D if layout == "ss2d" else D
    ybs, yoff = (2 * HW * D, HW * D) if layout == "conmb" else (HW * D, 0)
    g = 64
    buf = torch.full((B * ybs + 2 * g,), float("nan"), dtype=torch.bfloat16, device=dev)
    yp = ctypes.c_void_p(buf.data_ptr() + 2 * (g + yoff))
    L.check(L.lib().sigma_dwconv3x3_silu_fwd_bf16(_p(xin), xrs, HW * xrs, _p(w), _p(b), yp, ybs, B, H, W, D, _stream()), tag)
    torch.cuda.synchronize()
    bits = buf.view(torch.int16)
    gaps = [bits[:g], bits[g + B * ybs:]] + ([bits[g:g + B * ybs].view(B, ybs)[:, :HW * D]] if layout == "conmb" else [])
    bad = sum(int((t != NAN16).sum()) for t in gaps)
    assert bad == 0, f"{tag}: {bad} elements written outside the output"
    y = buf[g:g + B * ybs].view(B, ybs)[:, yoff:yoff + HW * D].reshape(B, H, W, D)
    ref, e = _dwconv_ref(xin[..., :D], w, b)
    worst = _dwconv_check(tag, y, ref, RR.bf16_store_bound(ref, e))
    record("dwconv_bf16", case=tag, tiles_per_cta=ntiles // ny, max_err_over_bound=worst)
