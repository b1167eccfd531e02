"""GPU: the FP8 inference mode (sigma_b200.fused.fp8_inference with autograd off) — its kernels against fp64 element by element,
the fused blocks and whole networks against the reference goldens, and the boundaries of the mode.

Quantization (include/sigma_b200.h): s = amax/448, q = e4m3(x·448/amax) round to nearest even.  A quantized producer's output
must satisfy |q·s - x64| <= 2^-4·|x64| (half an e4m3 step: 3 mantissa bits) + its own fp32 error + 2^-10·s (half the
subnormal step), and s must be amax64/448 to within that fp32 error.

GEMM bound.  Operands are exact e4m3 values built on the host, so the fp64 reference sees the kernel's inputs.  Each 128-wide
k-block accumulates in the tensor core (fewer bits than fp32; test_fp8_kblock_accumulation_precision measures it and holds it
to KB_ACC = 2^-8 of the k-block's sum of |products|: measured on an H100 SXM (700 W limit), 11.7 bits on random operands and
8.9 bits when one product is 2^12 times the others, whose low bits the accumulator drops) and is added to an fp32 accumulator (one rounding per k-block, 2^-24 of
the running sum); the epilogue multiplies by sa·sw and adds bias / residual·rscale (two roundings each).  Per element, with
mag = sum_k |a_k·w_k|:
    |C - C64| <= (KB_ACC + nkb·2^-23)·mag·sa·sw + 2^-22·(|C64| + |bias| + |residual·rscale|) + 1e-30
and a bf16 output adds 2^-8·|C64|.  Outputs sit inside NaN-filled buffers whose guard elements must stay intact.

End to end the bar is the bf16 mode's construction: 2 x the error of the composed path (the reference's op composition) under
bf16 autocast with the same per-row / per-channel e4m3 quantize-dequantize at exactly the GEMMs the mode quantizes, plus a floor
of 1e-3 of the output's scale; labels may flip only where the reference's top-2 margin is below 2.5x the bar (DESIGN §3)."""
import contextlib
import ctypes
import io
import math

import numpy as np
import pytest
import torch

import procedural as P
from helpers import SEED, cfg_tiny, golden, record
from oracle import fp8_ref as F

pytestmark = pytest.mark.gpu
S = 83
KB_ACC = 2.0 ** -8
BF = torch.bfloat16
E4 = torch.float8_e4m3fn


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _nan(shape, dtype):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def _guard_ok(t, what):
    """NaN guards: fp32 / bf16 NaN, or the e4m3 NaN byte 0x7f"""
    if t.numel() == 0:
        return
    t = t.contiguous()
    if t.dtype == E4:
        bad = int((t.view(torch.uint8) != 0x7F).sum())
    else:
        bad = int((~torch.isnan(t.float())).sum())
    assert bad == 0, f"{what}: {bad} guard elements were written"


def _lib():
    from sigma_b200 import _lib as L
    return L


def _check_quant(tag, q, s, x64, err64):
    """q (rows, C) e4m3, s (rows,) fp32 from the kernel; x64 (rows, C) the fp64 value; err64 the producer's own fp32 error bound"""
    q = q.float().double()
    s = s.double()
    am = x64.abs().amax(1)
    slack = err64.amax(1)
    want_s = torch.where(am == 0, torch.ones_like(am), am / 448.0)
    ds = (s - want_s).abs()
    assert bool((ds <= (slack + 2.0 ** -23 * am) / 448.0 + 1e-45).all()), f"{tag}: scale off by {float(ds.max()):.3e}"
    bound = 2.0 ** -4 * x64.abs() + err64 * (1 + 2.0 ** -4) + 2.0 ** -10 * s[:, None]
    err = (q * s[:, None] - x64).abs()
    r = float((err / bound).max())
    assert r <= 1.0, f"{tag}: |q·s - x| / bound = {r:.3f}"
    return r


# ---------------------------------------------------------------- quantizers
@pytest.mark.parametrize("dtype", ["f32", "bf16"])
def test_row_quantizer_bit_identical_to_the_oracle(dtype):
    """Weights (N, K) per output channel, ragged widths, a zero row, a row of tiny values, strided input, guarded output."""
    L = _lib()
    for rows, C in [(3072, 768), (96, 1536), (1537, 100), (7, 4)]:
        x = P.randn(S, f"q/{rows}/{C}", (rows, C), C ** -0.5)
        x[1] = 0
        x[min(2, rows - 1)] *= 1e-38
        td = BF if dtype == "bf16" else torch.float32
        xb = torch.zeros((rows, C + 12), dtype=td)
        xb[:, :C] = x.to(td)
        xg = xb.cuda()
        qbuf = _nan((rows + 2, C + 8), E4)
        sbuf = _nan((rows + 3,), torch.float32)
        L.check(L.lib().sigma_quantize_e4m3_rows(_p(xg), L.BF16 if dtype == "bf16" else L.F32, C + 12, _p(qbuf), C + 8, _p(sbuf),
                                                 rows, C, _stream()), "sigma_quantize_e4m3_rows")
        torch.cuda.synchronize()
        _guard_ok(qbuf[:rows, C:], "q columns past C")
        _guard_ok(qbuf[rows:], "q rows past the end")
        _guard_ok(sbuf[rows:], "scales past the end")
        qr, sr = F.quantize_rows(xb[:, :C].float().numpy())
        assert np.array_equal(sbuf[:rows].cpu().numpy(), sr), f"{rows}x{C}: scales differ"
        assert np.array_equal(qbuf[:rows, :C].float().cpu().numpy(), qr), f"{rows}x{C}: e4m3 rows differ"
        assert float(sbuf[1]) == 1.0 and not qbuf[1, :C].float().any()


def _ln_ref(x64, w, b, eps):
    mu = x64.mean(1, keepdim=True)
    var = ((x64 - mu) ** 2).mean(1, keepdim=True)
    xh = (x64 - mu) / torch.sqrt(var + eps)
    y = xh * w.double() + b.double()
    err = 2.0 ** -16 * (xh.abs() * w.double().abs() + b.double().abs()) + 1e-7
    return y, err


@pytest.mark.parametrize("C", [32, 96, 128, 192, 256, 384, 512, 768, 1024])
def test_layernorm_fp8_vs_fp64(C):
    """Every LayerNorm width in front of in_proj (Sigma tiny / small / base: 96..768 and 128..1024; 32 = the block tests'
    generic-kernel width), zero rows included (a constant row normalizes to beta: zero when beta is)."""
    L = _lib()
    rows = 132 * 8 * 3 + 5
    x = P.randn(S, f"ln/{C}/x", (rows, C), 2.0, 0.3).cuda()
    w = P.randn(S, f"ln/{C}/w", (C,), 0.5, 1.0).cuda()
    b = P.randn(S, f"ln/{C}/b", (C,), 0.1).cuda()
    b0 = torch.zeros_like(b)
    for tag, bb in (("beta", b), ("zero-beta", b0)):
        x[5] = 1.5                                       # constant row
        qbuf = _nan((rows + 1, C), E4)
        sbuf = _nan((rows + 1,), torch.float32)
        L.check(L.lib().sigma_layernorm_fwd_fp8(_p(x), _p(w), _p(bb), _p(qbuf), _p(sbuf), rows, C, 1e-5, _stream()), "ln fp8")
        torch.cuda.synchronize()
        _guard_ok(qbuf[rows:], "q past the end")
        _guard_ok(sbuf[rows:], "s past the end")
        y, err = _ln_ref(x.double(), w, bb, 1e-5)
        r = _check_quant(f"ln{C}/{tag}", qbuf[:rows], sbuf[:rows], y, err)
        if tag == "zero-beta":
            assert float(sbuf[5]) == 1.0 and not qbuf[5].float().any(), "a zero row: s = 1, q = 0"
        record("fp8_quant", case=f"layernorm/{C}/{tag}", bound_used=r)


@pytest.mark.parametrize("H,W,C", [(5, 7, 96), (15, 21, 192), (30, 40, 384), (29, 39, 128)])
def test_patch_merge_norm_fp8_vs_fp64(H, W, C):
    L = _lib()
    Bn = 3
    x = P.randn(S, f"pm/{H}/{W}/{C}", (Bn, H, W, C), 1.0, 0.2).cuda()
    w = P.randn(S, f"pm/{C}/w", (4 * C,), 0.5, 1.0).cuda()
    b = P.randn(S, f"pm/{C}/b", (4 * C,), 0.1).cuda()
    H2, W2 = (H + 1) // 2, (W + 1) // 2
    rows = Bn * H2 * W2
    qbuf = _nan((rows + 1, 4 * C), E4)
    sbuf = _nan((rows + 1,), torch.float32)
    L.check(L.lib().sigma_patch_merge_norm_fwd_fp8(_p(x), _p(w), _p(b), _p(qbuf), _p(sbuf), Bn, H, W, C, 1e-5, _stream()), "pm fp8")
    torch.cuda.synchronize()
    _guard_ok(qbuf[rows:], "q past the end")
    _guard_ok(sbuf[rows:], "s past the end")
    xp = torch.nn.functional.pad(x.double(), (0, 0, 0, 2 * W2 - W, 0, 2 * H2 - H))
    cat = torch.cat([xp[:, 0::2, 0::2], xp[:, 1::2, 0::2], xp[:, 0::2, 1::2], xp[:, 1::2, 1::2]], -1).reshape(rows, 4 * C)
    y, err = _ln_ref(cat, w, b, 1e-5)
    record("fp8_quant", case=f"patchmerge/{H}x{W}/{C}", bound_used=_check_quant(f"pm{H}x{W}", qbuf[:rows], sbuf[:rows], y, err))


@pytest.mark.parametrize("layout", ["ss2d", "cromb"])
@pytest.mark.parametrize("D", [64, 192, 384, 768, 1536])
def test_merge_norm_gate_fp8_vs_fp64(layout, D):
    """SS2D: sum of 4 bf16 direction slabs, out_norm, ·SiLU(z) (z a strided view of xz); CroMB: one slab per modality, the second
    call at row offset B·L (its scales at s[B·L:])."""
    from sigma_b200 import fused
    Bn, Lh = 2, 600
    rows = Bn * Lh
    K = 4 if layout == "ss2d" else 1
    y = P.randn(S, f"mg/{layout}/{D}/y", (K if K == 4 else 2, rows, D), 0.7).to(BF).cuda()
    ln = torch.nn.LayerNorm(D).cuda()
    with torch.no_grad():
        ln.weight.copy_(P.randn(S, f"mg/{D}/w", (D,), 0.5, 1.0))
        ln.bias.copy_(P.randn(S, f"mg/{D}/b", (D,), 0.1))
    if layout == "ss2d":
        xz = P.randn(S, f"mg/{D}/xz", (rows, 2 * D)).to(BF).cuda()
        out = fused.E4M3Rows(_nan((rows + 1, D), E4), _nan((rows + 1,), torch.float32))
        z = ctypes.c_void_p(xz.data_ptr() + 2 * D)
        fused.merge_norm_gate(y, 4, rows * D, 0, ln, z, 2 * D, None, out, 0, D, rows, rows, D)
        ysum = y.double().sum(0)
        zz = xz[:, D:].double()
        gate = zz / (1 + torch.exp(-zz))
        nrows = rows
    else:
        out = fused.E4M3Rows(_nan((2 * rows + 1, D), E4), _nan((2 * rows + 1,), torch.float32))
        fused.merge_norm_gate(y, 1, 0, 0, ln, None, 0, None, out, 0, D, rows, rows, D)
        fused.merge_norm_gate(y, 1, 0, 0, ln, None, 0, None, out, 0, D, rows, rows, D, y_offset=rows * D, out_offset=rows * D)
        ysum = y.double().reshape(2 * rows, D)
        gate = None
        nrows = 2 * rows
    torch.cuda.synchronize()
    _guard_ok(out.q[nrows:], "q past the end")
    _guard_ok(out.s[nrows:], "s past the end")
    ref, err = _ln_ref(ysum, ln.weight.detach(), ln.bias.detach(), ln.eps)
    if gate is not None:
        err = err * gate.abs() + 2.0 ** -20 * ref.abs() * gate.abs()
        ref = ref * gate
    r = _check_quant(f"merge/{layout}/{D}", out.q[:nrows], out.s[:nrows], ref, err + 1e-7)
    record("fp8_quant", case=f"merge/{layout}/{D}", bound_used=r)


# ---------------------------------------------------------------- GEMM
def _e4m3_operand(tag, rows, K, scale=1.0, zero_rows=()):
    """exact e4m3 rows (fp32 holding e4m3 values) and positive power-free fp32 scales"""
    x = P.randn(S, tag, (rows, K), scale)
    for r in zero_rows:
        x[r] = 0
    q, s = F.quantize_rows(x.numpy())
    return torch.from_numpy(q), torch.from_numpy(s)


def _run_fp8_gemm(M, N, K, out_dtype, monkeypatch, bn=None, extras="", lda=None, ldc=None, ldr=None, tag=None, need=0):
    L = _lib()
    if bn is not None:
        monkeypatch.setenv("SIGMA_GEMM_BN", str(bn))
    else:
        monkeypatch.delenv("SIGMA_GEMM_BN", raising=False)
    plan = (ctypes.c_int64 * 6)()
    assert L.lib().sigma_test_gemm_plan(M, N, K, 4, 0, 0, 0, plan) == 0
    pbn, grid, tiles = plan[0], plan[2], plan[3]
    if bn is not None:
        assert pbn == bn
    assert tiles >= need * grid, f"premise: {tiles} tiles over {grid} CTAs"
    tag = tag or f"fp8gemm/{M}/{N}/{K}/{extras}"
    lda, ldc, ldr = lda or K, ldc or N, ldr or N
    Aq, sa = _e4m3_operand(tag + "/A", M, K, 3.0, zero_rows=(0,))
    Wq, sw = _e4m3_operand(tag + "/W", N, K, K ** -0.5)
    abuf = torch.zeros((M, lda), dtype=E4, device="cuda")
    abuf[:, :K] = Aq.cuda().to(E4)
    wq = Wq.cuda().to(E4).contiguous()
    sa_g, sw_g = sa.cuda(), sw.cuda()
    bias = P.randn(S, tag + "/b", (N,)).cuda() if "b" in extras else None
    res = rs = None
    if "r" in extras:
        rbuf = _nan((M, ldr), torch.float32)
        rbuf[:, :N] = P.randn(S, tag + "/r", (M, N)).cuda()
        res = rbuf[:, :N]
        rs = P.randn(S, tag + "/s", (N,), 0.2, 1.0).cuda() if "s" in extras else None
    cbuf = _nan((M + 3, ldc), out_dtype)
    out = cbuf[:M, :N]
    c_dtype = L.BF16 if out_dtype == BF else L.F32
    L.check(L.lib().sigma_linear_fp8(_p(abuf), lda, _p(sa_g), _p(wq), _p(sw_g), _p(bias), _p(res), ldr, _p(rs), _p(out), ldc, c_dtype,
                                     M, N, K, _stream()), "sigma_linear_fp8")
    torch.cuda.synchronize()
    _guard_ok(cbuf[:, N:], f"{tag}: columns past N")
    _guard_ok(cbuf[M:], f"{tag}: rows past M")
    nkb = -(-K // 128)
    W64, Wa = Wq.double().cuda(), Wq.double().abs().cuda()
    s_w = sw.double().cuda()
    worst = 0.0
    for r0 in range(0, M, 1 << 15):
        a = Aq[r0:r0 + (1 << 15)].double().cuda()
        s_a = sa[r0:r0 + (1 << 15)].double().cuda()[:, None]
        ref = (a @ W64.t()) * s_a * s_w
        mag = (a.abs() @ Wa.t()) * s_a * s_w
        extra = ref.abs().clone()
        if bias is not None:
            ref += bias.double()
            extra += bias.double().abs()
        if res is not None:
            rr = res[r0:r0 + (1 << 15)].double() * (rs.double() if rs is not None else 1.0)
            ref += rr
            extra += rr.abs()
        bound = (KB_ACC + nkb * 2.0 ** -23) * mag + 2.0 ** -22 * extra + 1e-30
        if out_dtype == BF:
            bound = bound + 2.0 ** -8 * ref.abs()
        got = out[r0:r0 + (1 << 15)].double()
        assert bool(torch.isfinite(got).all()), f"{tag}: non-finite output"
        r = ((got - ref).abs() / bound)
        worst = max(worst, float(r.max()))
        assert worst <= 1.0, f"{tag}: {int((r > 1).sum())} elements out of bound (worst {worst:.3f})"
    record("fp8_gemm", case=tag, out=str(out_dtype), bn=pbn, bound_used=worst)


OUTS = [torch.float32, BF]


def test_fp8_kblock_accumulation_precision():
    """What the promotion interval rests on: the error of ONE k-block (four k32 MMAs, 128 products) accumulated inside the tensor
    core, against fp64, over random operands and an adversarial layout (one product about 2^12 times the others, then 127
    smaller ones whose low bits a truncating accumulator aligned to the large one drops).  Recorded as retained bits (-log2 of the worst error over the
    k-block's sum of |products|), and held to KB_ACC, the per-k-block term of the GEMM bound."""
    L = _lib()
    M, N, K = 128 * 64, 128, 128
    res = {}
    for case in ("random", "adversarial"):
        Aq, sa = _e4m3_operand(f"acc/{case}/A", M, K)
        Wq, sw = _e4m3_operand(f"acc/{case}/W", N, K)
        if case == "adversarial":
            Aq[:, 0] = 448.0
            Wq[:, 0] = 448.0 * torch.sign(Wq[:, 0] + 0.5)
            Aq[:, 1:] = torch.sign(Aq[:, 1:]) * 2.0 ** -4 * (1 + (torch.arange(K - 1) % 8) / 8.0)
        ag, wg = Aq.cuda().to(E4), Wq.cuda().to(E4).contiguous()          # kept alive until the kernel has run
        sa, sw = torch.ones(M, device="cuda"), torch.ones(N, device="cuda")
        out = torch.empty((M, N), device="cuda")
        L.check(L.lib().sigma_linear_fp8(_p(ag), K, _p(sa), _p(wg), _p(sw), None, None, 0, None, _p(out), N, L.F32, M, N, K, _stream()),
                "sigma_linear_fp8")
        torch.cuda.synchronize()
        a, w = Aq.double().cuda(), Wq.double().cuda()
        ref = a @ w.t()
        mag = a.abs() @ w.abs().t()
        rel = float(((out.double() - ref).abs() / mag.clamp_min(1e-300)).max())
        res[case] = rel
        record("fp8_accumulation", case=case, rel_err=rel, bits=(-math.log2(rel) if rel > 0 else 99.0))
        assert rel <= KB_ACC, f"{case}: one k-block's accumulation error {rel:.3e} of sum|products| > {KB_ACC:.3e}"


@pytest.mark.parametrize("out_dtype", OUTS, ids=["f32out", "bf16out"])
@pytest.mark.parametrize("bn", [32, 64])
def test_fp8_gemm_every_tile_width_multiwave(bn, out_dtype, monkeypatch):
    """Every m64nBNk32 e4m3 instance, forced, on 301 row tiles x N = 768 (>= 3 tiles per CTA), K = 384, the whole epilogue."""
    _run_fp8_gemm(128 * 300 + 17, 768, 384, out_dtype, monkeypatch, bn=bn, extras="brs", tag=f"fp8gemm-bn{bn}", need=3)


@pytest.mark.parametrize("out_dtype", OUTS, ids=["f32out", "bf16out"])
@pytest.mark.parametrize("M,N,K,bn", [
    (128 * 800 + 1, 8, 16, None), (128 * 300 + 127, 40, 48, None), (128 * 300 + 1, 264, 144, None),
    (128 * 300 + 127, 264, 208, 64), (128 * 400 + 1, 8, 112, 32), (128 * 300 + 127, 136, 1536, 64),
    (128 * 120 + 5, 768, 1536, None), (128 * 120 + 3, 3072, 768, None),
])
def test_fp8_gemm_ragged_multiwave(M, N, K, bn, out_dtype, monkeypatch):
    """K < 128 and K % 128 != 0 (TMA zero-fills past K), K up to 1536 (12 promotions), column tiles overhanging N, M % 128 in
    {1, 3, 5, 127}, Sigma-tiny's widest in_proj / out_proj shapes."""
    _run_fp8_gemm(M, N, K, out_dtype, monkeypatch, bn=bn, extras="b")


@pytest.mark.parametrize("out_dtype", OUTS, ids=["f32out", "bf16out"])
@pytest.mark.parametrize("extras", ["", "b", "r", "rs", "brs"])
def test_fp8_gemm_epilogues_strided_multiwave(extras, out_dtype, monkeypatch):
    _run_fp8_gemm(128 * 300 + 17, 768, 192, out_dtype, monkeypatch, extras=extras, lda=192 + 48, ldc=768 + 12, ldr=768 + 20,
                  tag=f"fp8gemm-epi/{extras}")


# ---------------------------------------------------------------- blocks and networks
def _qdq_rows_t(x):
    """the mode's per-row quantize-dequantize, in torch on the GPU (fp32), along the last dim"""
    xf = x.float()
    am = xf.abs().amax(-1, keepdim=True)
    zero = am == 0
    inv = torch.where(zero, torch.ones_like(am), torch.clamp(448.0 / am, max=3.4028234663852886e38))
    s = torch.where(zero, torch.ones_like(am), am / 448.0)
    q = torch.clamp(xf * inv, -448.0, 448.0).to(E4).float()
    return (q * s).to(x.dtype)


FP8_LINEARS = ("in_proj", "in_proj_modalx", "out_proj", "out_proj_rgb", "out_proj_e", "reduction")


@contextlib.contextmanager
def _fake_quant(model):
    """The composed path with the mode's e4m3 quantize-dequantize at exactly the GEMMs it quantizes: SS2D / ConMB / CroMB in_proj,
    in_proj_modalx, out_proj, out_proj_rgb, out_proj_e and PatchMerging2D.reduction (weights per output channel, inputs per row)."""
    from sigma_b200 import modules as M
    owners = (M.SS2D, M.ConMB_SS2D, M.CrossMambaFusion_SS2D_SSM, M.PatchMerging2D)
    lins = []
    for mod in model.modules():
        if isinstance(mod, owners):
            for n in FP8_LINEARS:
                lin = getattr(mod, n, None)
                if isinstance(lin, torch.nn.Linear):
                    lins.append(lin)
    saved = [lin.weight.data.clone() for lin in lins]
    hooks = [lin.register_forward_pre_hook(lambda _m, args: (_qdq_rows_t(args[0]),) + tuple(args[1:])) for lin in lins]
    with torch.no_grad():
        for lin in lins:
            lin.weight.data.copy_(_qdq_rows_t(lin.weight.data))
    try:
        yield
    finally:
        for h in hooks:
            h.remove()
        with torch.no_grad():
            for lin, w in zip(lins, saved):
                lin.weight.data.copy_(w)


def _composed_fq(model, *inputs):
    from sigma_b200 import modules as M
    with M.composed_path(), torch.autocast("cuda", dtype=BF), _fake_quant(model):
        return model(*inputs)


def _model(backbone, H, W, ncls, seed=SEED):
    from sigma_b200 import modules as M
    with contextlib.redirect_stdout(io.StringIO()):
        model = M.EncoderDecoder(cfg_tiny(H, W, num_classes=ncls, backbone=backbone), criterion=None)
    P.fill_state_dict(model, seed)
    return model.cuda().eval()


CASES = {
    "tiny": ("sigma_tiny_480x640", "sigma_tiny", 480, 640, 9),
    "small": ("sigma_small_480x640", "sigma_small", 480, 640, 40),
    "base": ("sigma_base_720x960", "sigma_base", 720, 960, 5),
}


@pytest.mark.parametrize("which", ["tiny", "small", "base"])
def test_fp8_logits_vs_reference_golden_fullsize(which):
    """Measured on an H100 SXM (700 W limit): the fused fp8 error is 1.07 (tiny), 1.00 (small) and 0.94 (base) of the composed
    path's with the same fake quantization under bf16 autocast (recorded per case in the parity log as ratio_to_composed)."""
    from sigma_b200 import fused
    tag, backbone, H, W, ncls = CASES[which]
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    g = golden(tag)
    model = _model(backbone, H, W, ncls)
    rgb = P.randn(SEED, tag + "/rgb", (1, 3, H, W)).cuda()
    mx = P.randn(SEED, tag + "/x", (1, 3, H, W)).cuda()
    scale = float(g["logits_absmax"])
    err = lambda t: float(np.abs(t[:, :, 3::8, 5::8].float().cpu().numpy() - g["logits_sub"]).max()) / scale
    with torch.no_grad():
        ec = err(_composed_fq(model, rgb, mx))
        with fused.fp8_inference():
            assert fused.precision() == "fp8"
            fl = model(rgb, mx).float()
            bar = fused.logits_bar(ec)
    ef = err(fl)
    record("fp8_fullsize", tag=tag, fused_err=ef, composed_err=ec, ratio_to_composed=ef / max(ec, 1e-12))
    assert ef <= bar, f"{tag}: fused fp8 logits error {ef:.2e} of scale > 2 x composed-with-fake-quant {ec:.2e} + floor"
    pred = fl.argmax(1).cpu().numpy().astype(np.uint8)
    diff = pred != g["argmax"]
    worst = float(g["margin"].astype(np.float32)[diff].max()) if diff.any() else 0.0
    assert worst <= 2.5 * bar * scale, f"{tag}: a label flipped where the reference's top-2 margin is {worst:.3e}"


@pytest.mark.parametrize("name", ["ss2d_n16", "ss2d_n4", "vssblock", "patchmerge_odd", "cromb", "conmb", "cvss_dec", "mamba_decoder",
                                  "rgbx_encoder_small"])
def test_fp8_blocks_vs_reference_goldens(name):
    from sigma_b200 import fused
    from test_bf16_gpu import _block_cases
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    ctor, inputs = _block_cases()[name]
    mod = ctor()
    P.fill_state_dict(mod, SEED)
    mod = mod.cuda().eval()
    g = golden(name)
    as_tuple = lambda o: tuple(o) if isinstance(o, (tuple, list)) else (o,)
    with torch.no_grad():
        co = as_tuple(_composed_fq(mod, *inputs))
        with fused.fp8_inference():
            assert fused.precision() == "fp8"
            fo = as_tuple(mod(*inputs))
            for i, (f, c) in enumerate(zip(fo, co)):
                ref = g[f"out{i}"]
                sc = float(np.abs(ref).max())
                ef = float(np.abs(f.float().cpu().numpy() - ref).max()) / sc
                ec = float(np.abs(c.float().cpu().numpy() - ref).max()) / sc
                bar = fused.logits_bar(ec)
                record("fp8_block", tag=name, out=i, fused_err=ef, composed_err=ec, ratio_to_composed=ef / max(ec, 1e-12))
                assert f.dtype == torch.float32, f"{name}[{i}]: the block output (residual stream) must stay fp32"
                assert ef <= bar, f"{name}[{i}]: fused fp8 error {ef:.2e} of scale > bar {bar:.2e} (composed with fake quant {ec:.2e})"


# ---------------------------------------------------------------- mode boundaries
@pytest.mark.parametrize("mode", ["tf32x3", "tf32", "bf16"])
def test_context_off_is_bit_identical_to_never_entering_it(mode):
    from sigma_b200 import fused
    torch.backends.cuda.matmul.allow_tf32 = mode == "tf32"
    try:
        model = _model("sigma_tiny", 64, 96, 9)
        rgb = P.randn(S, "fb/rgb", (2, 3, 64, 96)).cuda()
        mx = P.randn(S, "fb/x", (2, 3, 64, 96)).cuda()
        amp = torch.autocast("cuda", dtype=BF) if mode == "bf16" else contextlib.nullcontext()
        with torch.no_grad(), amp:
            assert fused.precision() == mode
            base = model(rgb, mx)
            with fused.fp8_inference():
                q = model(rgb, mx)
                with fused.fp8_inference(False):
                    assert fused.precision() == mode
                    off = model(rgb, mx)
            after = model(rgb, mx)
        assert torch.equal(base, off) and torch.equal(base, after)
        assert not torch.equal(base, q)                  # the mode did run in between
    finally:
        torch.backends.cuda.matmul.allow_tf32 = False


@pytest.mark.parametrize("which", ["vssblock", "conmb", "cromb", "cvss_dec"])
def test_grad_enabled_inside_the_context_keeps_the_training_path(which):
    from sigma_b200 import fused
    from test_bf16_gpu import _block_cases
    ctor, inputs = _block_cases()[which]

    def run(ctx):
        mod = ctor()
        P.fill_state_dict(mod, S)
        mod = mod.cuda().train()
        xs = [t.detach().clone().requires_grad_(True) for t in inputs]
        with ctx:
            assert fused.precision() != "fp8"
            out = mod(*xs)
            out = out if isinstance(out, (tuple, list)) else (out,)
            sum(o.float().sum() for o in out).backward()
        return [o.detach() for o in out], [x.grad for x in xs]

    y1, g1 = run(contextlib.nullcontext())
    y2, g2 = run(fused.fp8_inference())
    for a, b in zip(y1, y2):
        assert a.dtype == b.dtype and torch.equal(a, b)
    for a, b in zip(g1, g2):
        assert a is not None and torch.isfinite(a).all()
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)   # parameter-gradient atomics may reorder sums


def test_inference_pipeline_fp8_replays_eager_and_recaptures():
    from sigma_b200 import fused
    from sigma_b200.pipeline import InferencePipeline
    torch.backends.cuda.matmul.allow_tf32 = False
    B, H, W = 2, 64, 96
    model = _model("sigma_tiny", H, W, 9)
    pipe = InferencePipeline(model, B, H, W, fp8=True)
    h_rgb = P.randn(S, "pipe8/rgb", (B, 3, H, W)).pin_memory()
    h_x = P.randn(S, "pipe8/x", (B, 3, H, W)).pin_memory()
    out = torch.empty((B,) + pipe.out_shape[1:], dtype=pipe.out.dtype).pin_memory()

    def eager():
        with torch.no_grad(), fused.fp8_inference():
            return model(h_rgb.cuda(), h_x.cuda()).cpu()

    pipe.submit(h_rgb, h_x, out)
    pipe.drain()
    first = eager()
    assert torch.equal(out, first)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    P.fill_state_dict(model, S + 1)
    with torch.no_grad():
        for p_ in model.parameters():
            p_.mul_(1.0)                                  # in-place: bumps every version counter -> re-capture, re-quantized weights
    pipe.submit(h_rgb, h_x, out)
    pipe.drain()
    second = eager()
    assert torch.equal(out, second) and not torch.equal(first, second)
    model.load_state_dict(sd)
    pipe.submit(h_rgb, h_x, out)
    pipe.drain()
    assert torch.equal(out, eager()) and torch.equal(out, first)
