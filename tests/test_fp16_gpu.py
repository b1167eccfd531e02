"""GPU: the fp16 inference mode (sigma_b200.fused.fp16_inference with autograd off) — every new kernel against fp64 (or, for the
scan, against the fp32 kernel fed the same fp16 xc), the fused blocks and whole networks against the reference goldens, and the
boundaries of the mode.

Per-element bounds.  Inputs are fp16 values built on the host and the fp64 reference is computed from them, so operand rounding does
not enter.  u = 2^-24, HU = 2^-11 (fp16 unit roundoff: 11 significant bits, round to nearest even), and an fp16 store of a value
below the normal range (2^-14) rounds on the subnormal grid: at most 2^-25 absolute.  One fp16 store of a value the fp32 kernel
holds to ref within e is within e + HU·(|ref| + e) + 2^-25.
  GEMM   fp16 x fp16 products are exact in fp32; the fp32 accumulation and epilogue as the bf16 GEMM's (tests/test_bf16_gpu.py).
  Scan   the fp16 instance runs the fp32 recurrence on the same xc values and segment plan as the fp32 kernel; y is rounded once.
Outputs sit inside NaN-filled buffers whose guard elements must stay NaN.

End to end the bar is the bf16 mode's construction: 2 x the error of the composed path (the reference's op composition) under
torch.autocast(dtype=torch.float16), plus a floor of 1e-3 of the output's scale; a label may flip only where the reference's top-2
margin is below 2.5x the bar."""
import contextlib
import ctypes
import io

import numpy as np
import pytest
import torch

import procedural as P
from helpers import SEED, cfg_tiny, gemm_plan, golden, record

pytestmark = pytest.mark.gpu
S = 89
U = 2.0 ** -24
HU = 2.0 ** -11
SUB = 2.0 ** -25
H16 = torch.float16


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _lib():
    from sigma_b200 import _lib as L
    return L


def _nan(shape, dtype):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def _guard_ok(t, what):
    if t.numel() == 0:
        return
    bad = int((~torch.isnan(t.float())).sum())
    assert bad == 0, f"{what}: {bad} guard elements were written"


def _store(ref, e):
    """bound of one fp16 store of a value the fp32 kernel holds to ref within e"""
    return e + HU * (ref.abs() + e) + SUB


def _ratio(tag, got, ref, bound):
    assert bool(torch.isfinite(got).all()), f"{tag}: non-finite output"
    err = (got.double() - ref).abs()
    r = err / bound
    worst = float(r.max())
    if worst > 1.0:
        i = int(r.argmax())
        raise AssertionError(f"{tag}: {int((r > 1).sum())}/{r.numel()} elements out of bound; worst err {float(err.flatten()[i]):.3e} "
                             f"> {float(bound.flatten()[i]):.3e}")
    return worst


# ---------------------------------------------------------------- GEMM
def _run_gemm(M, N, K, out_dtype, monkeypatch, bn=None, extras="", lda=None, ldc=None, ldr=None, tag=None, need=3):
    from sigma_b200 import fused
    L = _lib()
    if bn is not None:
        monkeypatch.setenv("SIGMA_GEMM_BN", str(bn))
    else:
        monkeypatch.delenv("SIGMA_GEMM_BN", raising=False)
    pl = gemm_plan(M, N, K, False)
    if bn is not None:
        assert pl["bn"] == bn
    assert pl["tiles"] >= need * pl["grid"], f"premise: {pl['tiles']} tiles over {pl['grid']} CTAs"
    tag = tag or f"fp16gemm/{M}/{N}/{K}/{extras}"
    lda, ldc, ldr = lda or K, ldc or N, ldr or N
    abuf = _nan((M, lda), H16)
    A = P.randn(S, tag + "/A", (M, K)).to(H16).cuda()
    abuf[:, :K] = A
    Wt = P.randn(S, tag + "/W", (N, K), K ** -0.5).cuda()
    Wh = Wt.to(H16)
    bias = P.randn(S, tag + "/b", (N,)).cuda() if "b" in extras else None
    res = rs = None
    if "r" in extras:
        rbuf = _nan((M, ldr), torch.float32)
        rbuf[:, :N] = P.randn(S, tag + "/r", (M, N)).cuda()
        res = rbuf[:, :N]
        rs = P.randn(S, tag + "/s", (N,), 0.2, 1.0).cuda() if "s" in extras else None
    cbuf = _nan((M + 3, ldc), out_dtype)
    out = cbuf[:M, :N]
    c_dtype = L.F16 if out_dtype == H16 else L.F32
    L.check(L.lib().sigma_linear_fp16(_p(abuf), lda, _p(Wh), _p(bias), _p(res), ldr, _p(rs), _p(out), ldc, c_dtype, M, N, K,
                                      _stream()), "sigma_linear_fp16")
    via = fused.linear(abuf[:, :K], Wt, bias, out=torch.empty_like(out), residual=res, rscale=rs)   # fused.linear routes fp16 here
    torch.cuda.synchronize()
    assert torch.equal(via, out), f"{tag}: fused.linear differs from sigma_linear_fp16"
    _guard_ok(cbuf[:, N:], f"{tag}: columns past N")
    _guard_ok(cbuf[M:], f"{tag}: rows past M")
    W64, Wa = Wh.double(), Wh.double().abs()
    worst = 0.0
    for r0 in range(0, M, 1 << 15):
        a = A[r0:r0 + (1 << 15)].double()
        ref = a @ W64.t()
        mag = a.abs() @ Wa.t()
        extra = mag.clone()
        if bias is not None:
            ref += bias.double()
            extra += bias.double().abs()
        if res is not None:
            rr = res[r0:r0 + (1 << 15)].double() * (rs.double() if rs is not None else 1.0)
            ref += rr
            extra += rr.abs()
        bound = (2.0 ** -20 + K * 2.0 ** -23) * mag + 2 * U * extra + 1e-5
        if out_dtype == H16:
            bound = _store(ref, bound)
        worst = max(worst, _ratio(f"{tag} rows {r0}..", out[r0:r0 + (1 << 15)], ref, bound))
    record("fp16_gemm", case=tag, out=str(out_dtype), bn=pl["bn"], bound_used=worst)


OUTS = [torch.float32, H16]


@pytest.mark.parametrize("out_dtype", OUTS, ids=["f32out", "f16out"])
@pytest.mark.parametrize("bn", [32, 64, 96, 128, 160, 192, 224, 256])
def test_fp16_gemm_every_tile_width_multiwave(bn, out_dtype, monkeypatch):
    """Every m64nBNk16 fp16 instance, forced, on 301 row tiles x N = 768 (>= 3 tiles per CTA), with the whole epilogue."""
    _run_gemm(128 * 300 + 17, 768, 384, out_dtype, monkeypatch, bn=bn, extras="brs", tag=f"fp16gemm-bn{bn}")


@pytest.mark.parametrize("out_dtype", OUTS, ids=["f32out", "f16out"])
@pytest.mark.parametrize("M,N,K,bn", [
    (128 * 800 + 1, 8, 40, None), (128 * 800 + 127, 40, 8, None), (128 * 300 + 1, 264, 104, None),
    (128 * 300 + 127, 264, 40, 256), (128 * 800 + 1, 8, 104, 32), (128 * 800 + 127, 40, 104, 64),
])
def test_fp16_gemm_ragged_multiwave(M, N, K, bn, out_dtype, monkeypatch):
    """K < 64 and K % 64 != 0 (TMA zero-fills past K), column tiles overhanging N (N > 256 too), M % 128 in {1, 127}."""
    _run_gemm(M, N, K, out_dtype, monkeypatch, bn=bn, extras="b")


@pytest.mark.parametrize("out_dtype", OUTS, ids=["f32out", "f16out"])
@pytest.mark.parametrize("extras", ["b", "r", "rs", "brs"])
def test_fp16_gemm_epilogues_strided_multiwave(extras, out_dtype, monkeypatch):
    _run_gemm(128 * 300 + 17, 768, 192, out_dtype, monkeypatch, extras=extras, lda=192 + 40, ldc=768 + 12, ldr=768 + 20,
              tag=f"fp16gemm-epi/{extras}")


def test_fp16_store_past_65504_is_inf_like_torch_half():
    """The documented range limit: the GEMM's fp16 store and the fp16 LayerNorm round once, so a value past ±65504 (from 65520 on)
    is ±inf and one just below rounds to 65504, exactly as torch's .half() does."""
    L = _lib()
    vals = torch.tensor([70000.0, -70000.0, 65519.0, 65520.0, -65520.0, 65504.0, 1e30, 3e-8], device="cuda")
    M, N, K = 130, vals.numel(), 8
    A = torch.zeros((M, K), dtype=H16, device="cuda")
    W = torch.zeros((N, K), dtype=H16, device="cuda")
    C = _nan((M, N), H16)
    L.check(L.lib().sigma_linear_fp16(_p(A), K, _p(W), _p(vals), None, 0, None, _p(C), N, L.F16, M, N, K, _stream()), "sigma_linear_fp16")
    want = vals.half()
    assert torch.isinf(want[:2]).all() and want[2] == 65504 and torch.isinf(want[3])
    torch.cuda.synchronize()
    assert torch.equal(C, want.expand(M, N)), f"GEMM store: {C[0].tolist()} vs torch {want.tolist()}"
    # LayerNorm with gamma = 0: y = beta, stored once
    C2 = 8
    x = P.randn(S, "ovf/x", (64, C2)).cuda()
    w = torch.zeros(C2, device="cuda")
    y = _nan((64, C2), H16)
    L.check(L.lib().sigma_layernorm_fwd_fp16(_p(x), _p(w), _p(vals), _p(y), 64, C2, 1e-5, _stream()), "ln fp16")
    torch.cuda.synchronize()
    assert torch.equal(y, want.expand(64, C2)), f"LayerNorm store: {y[0].tolist()} vs torch {want.tolist()}"


# ---------------------------------------------------------------- row-wise and depthwise conv
def _ln_ref(x64, w, b, eps):
    mu = x64.mean(1, keepdim=True)
    var = ((x64 - mu) ** 2).mean(1, keepdim=True)
    xh = (x64 - mu) / torch.sqrt(var + eps)
    y = xh * w.double() + b.double()
    err = 2.0 ** -16 * (xh.abs() * w.double().abs() + b.double().abs()) + 1e-7
    return y, err


@pytest.mark.parametrize("C", [32, 96, 128, 192, 256, 384, 512, 768, 1024, 1100])
def test_layernorm_fp16_vs_fp64(C):
    """Every LayerNorm width in front of in_proj (fast widths; 32 and 1100 take the generic kernel)."""
    L = _lib()
    rows = 132 * 8 * 3 + 5
    x = P.randn(S, f"ln/{C}/x", (rows, C), 2.0, 0.3).cuda()
    w = P.randn(S, f"ln/{C}/w", (C,), 0.5, 1.0).cuda()
    b = P.randn(S, f"ln/{C}/b", (C,), 0.1).cuda()
    buf = _nan((rows + 1, C), H16)
    L.check(L.lib().sigma_layernorm_fwd_fp16(_p(x), _p(w), _p(b), _p(buf), rows, C, 1e-5, _stream()), "ln fp16")
    torch.cuda.synchronize()
    _guard_ok(buf[rows:], "past the end")
    y, err = _ln_ref(x.double(), w, b, 1e-5)
    record("fp16_rowwise", case=f"layernorm/{C}", bound_used=_ratio(f"ln{C}", buf[:rows], y, _store(y, err)))


@pytest.mark.parametrize("H,W,C", [(5, 7, 96), (15, 21, 192), (30, 40, 384), (29, 39, 128)])
def test_patch_merge_norm_fp16_vs_fp64(H, W, C):
    L = _lib()
    Bn = 3
    x = P.randn(S, f"pm/{H}/{W}/{C}", (Bn, H, W, C), 1.0, 0.2).cuda()
    w = P.randn(S, f"pm/{C}/w", (4 * C,), 0.5, 1.0).cuda()
    b = P.randn(S, f"pm/{C}/b", (4 * C,), 0.1).cuda()
    H2, W2 = (H + 1) // 2, (W + 1) // 2
    rows = Bn * H2 * W2
    buf = _nan((rows + 1, 4 * C), H16)
    L.check(L.lib().sigma_patch_merge_norm_fwd_fp16(_p(x), _p(w), _p(b), _p(buf), Bn, H, W, C, 1e-5, _stream()), "pm fp16")
    torch.cuda.synchronize()
    _guard_ok(buf[rows:], "past the end")
    xp = torch.nn.functional.pad(x.double(), (0, 0, 0, 2 * W2 - W, 0, 2 * H2 - H))
    cat = torch.cat([xp[:, 0::2, 0::2], xp[:, 1::2, 0::2], xp[:, 0::2, 1::2], xp[:, 1::2, 1::2]], -1).reshape(rows, 4 * C)
    y, err = _ln_ref(cat, w, b, 1e-5)
    record("fp16_rowwise", case=f"patchmerge/{H}x{W}/{C}", bound_used=_ratio(f"pm{H}x{W}", buf[:rows], y, _store(y, err)))


@pytest.mark.parametrize("layout", ["ss2d", "cromb", "conmb"])
@pytest.mark.parametrize("D", [64, 192, 384, 768, 1536, 1100])
def test_merge_norm_gate_fp16_vs_fp64(layout, D):
    """SS2D: 4 fp16 direction slabs, out_norm, ·SiLU(z) with z a strided view of xz; CroMB: one slab per modality at a row offset;
    ConMB: 2 slabs, an fp32 gate per image, written into half of each ycat row.  D = 1100 takes the generic kernel."""
    from sigma_b200 import fused
    Bn, Lh = 2, 600
    rows = Bn * Lh
    ln = torch.nn.LayerNorm(D).cuda()
    with torch.no_grad():
        ln.weight.copy_(P.randn(S, f"mg/{D}/w", (D,), 0.5, 1.0))
        ln.bias.copy_(P.randn(S, f"mg/{D}/b", (D,), 0.1))
    tag = f"merge/{layout}/{D}"
    if layout == "ss2d":
        y = P.randn(S, tag + "/y", (4, rows, D), 0.7).to(H16).cuda()
        xz = P.randn(S, tag + "/xz", (rows, 2 * D)).to(H16).cuda()
        out = _nan((rows + 1, D), H16)
        z = ctypes.c_void_p(xz.data_ptr() + 2 * D)
        fused.merge_norm_gate(y, 4, rows * D, 0, ln, z, 2 * D, None, out, 0, D, rows, rows, D)
        zz = xz[:, D:].double()
        ref, err = _ln_ref(y.double().sum(0), ln.weight.detach(), ln.bias.detach(), ln.eps)
        g = zz / (1 + torch.exp(-zz))
        ref, err = ref * g, err * g.abs() + 2.0 ** -20 * (ref * g).abs()
        got, guard = out[:rows], out[rows:]
    elif layout == "cromb":
        y = P.randn(S, tag + "/y", (2, rows, D), 0.7).to(H16).cuda()
        out = _nan((2 * rows + 1, D), H16)
        fused.merge_norm_gate(y, 1, 0, 0, ln, None, 0, None, out, 0, D, rows, rows, D)
        fused.merge_norm_gate(y, 1, 0, 0, ln, None, 0, None, out, 0, D, rows, rows, D, y_offset=rows * D, out_offset=rows * D)
        ref, err = _ln_ref(y.double().reshape(2 * rows, D), ln.weight.detach(), ln.bias.detach(), ln.eps)
        got, guard = out[:2 * rows], out[2 * rows:]
    else:
        y = P.randn(S, tag + "/y", (2, Bn, 2 * Lh, D), 0.7).to(H16).cuda()
        gate = P.randn(S, tag + "/g", (Bn, D), 0.5, 1.0).cuda()
        out = _nan((rows + 1, 2 * D), H16)
        fused.merge_norm_gate(y, 2, Bn * 2 * Lh * D, 2 * Lh * D, ln, None, 0, gate, out, Lh * 2 * D, 2 * D, rows, Lh, D)
        ys = y.double().sum(0)[:, :Lh].reshape(rows, D)
        ref, err = _ln_ref(ys, ln.weight.detach(), ln.bias.detach(), ln.eps)
        gg = gate.double().repeat_interleave(Lh, 0)
        ref, err = ref * gg, err * gg.abs() + 2.0 ** -22 * (ref * gg).abs()
        got, guard = out[:rows, :D], torch.cat([out[:rows, D:].flatten(), out[rows:].flatten()])
    torch.cuda.synchronize()
    _guard_ok(guard, "guards")
    record("fp16_rowwise", case=tag, bound_used=_ratio(tag, got, ref, _store(ref, err)))


@pytest.mark.parametrize("Bn,H,W,D,layout", [(7, 121, 161, 64, "xz"), (2, 120, 160, 192, "xz"), (2, 30, 40, 768, "plain"),
                                             (3, 57, 75, 136, "plain")])
def test_fp16_dwconv_vs_fp64(Bn, H, W, D, layout):
    """The 4-slot ring wraps (D = 64: every CTA walks >= 9 tiles), Sigma's widths, a partial 32-channel block (136), ragged H / W,
    x a strided view ([x | z] rows) or contiguous.  Against fp64 on the fp16 input's exact values, inside the fp32 kernel's bound
    plus one fp16 store."""
    L = _lib()
    from test_gemm_waves_gpu import _dwconv_check, _dwconv_ref
    C = 2 * D if layout == "xz" else D
    xz = P.randn(S, f"dw/{D}/x", (Bn, H, W, C)).to(H16).cuda()
    w = P.randn(S, f"dw/{D}/w", (D, 1, 3, 3), 0.3).cuda()
    b = P.randn(S, f"dw/{D}/b", (D,), 0.1).cuda()
    buf = _nan((Bn * H * W + 5, D), H16)
    L.check(L.lib().sigma_dwconv3x3_silu_fwd_fp16(_p(xz), C, H * W * C, _p(w), _p(b), _p(buf), H * W * D, Bn, H, W, D, _stream()), "dw")
    torch.cuda.synchronize()
    _guard_ok(buf[Bn * H * W:], "past the end")
    ref, e = _dwconv_ref(xz[..., :D], w, b)
    worst = _dwconv_check(f"dwconv fp16 {D}", buf[:Bn * H * W].view(Bn, H, W, D), ref, _store(ref, e))
    record("fp16_dwconv", case=f"{Bn}x{H}x{W}x{D}/{layout}", max_err_over_bound=worst)


# ---------------------------------------------------------------- scan
SCAN_SHAPES = {"stage0": (120, 160, 192, 6), "stage2": (30, 40, 768, 24), "stage3": (15, 20, 1536, 48)}


def _scan_inputs(kind, N, shape, images):
    from sigma_b200 import _lib as L
    H, W, D, R = SCAN_SHAPES[shape]
    batch = 2 * images if kind == "CROSS" else images
    K = {"CROSS4": 4, "SEQ2": 2, "CROSS": 1}[kind]
    Lseq = 2 * H * W if kind == "SEQ2" else H * W
    Cp = L.lib().sigma_ss2d_padded_cp(N, R)
    tag = f"scan/{kind}/{N}/{shape}/{images}"
    nw = 2 if kind == "CROSS" else K
    xc = P.randn(S, tag + "/xc", (batch, Lseq, D)).to(H16).cuda()
    xdbl = P.randn(S, tag + "/dbl", (batch, Lseq, K, Cp), 0.5).cuda()
    dtw = P.randn(S, tag + "/dtw", (nw * D, R), R ** -0.5).cuda()
    dt = torch.exp(P.rand(S, tag + "/dt", (nw * D,)) * (np.log(0.1) - np.log(1e-3)) + np.log(1e-3))
    dtb = (dt + torch.log(-torch.expm1(-dt))).cuda()
    A = (-torch.exp(P.randn(S, tag + "/A", (nw * D, N), 0.5))).cuda().contiguous()
    Ds = torch.ones(nw * D, device="cuda")
    return tag, (xc, xdbl, dtw, dtb, A, Ds, batch, H, W, D, N, R, Cp)


@pytest.mark.parametrize("plan", ["serial", "segments", "old-rule"])
@pytest.mark.parametrize("N", [4, 8, 16])
@pytest.mark.parametrize("kind", ["CROSS4", "SEQ2", "CROSS"])
def test_fp16_scan_matches_fp32_kernel_after_one_rounding(kind, N, plan, monkeypatch):
    """sigma_ss2d_scan_fwd_fp16 against the fp32 kernel fed the same xc values and forced to the same number of L-segments
    (sigma_ss2d_scan_fwd_split): serial (8 images at stage 2), the library's segmented plan (one image at Sigma's stage 3: 4 or 8
    segments) and the round-1 rule's count (SIGMA_SCAN_SPLIT_RULE=old, one image at stage 2: 6 to 22 segments).  y differs only by
    its one fp16 rounding."""
    from sigma_b200 import fused
    from helpers import ss2d_fwd_plan
    L = _lib()
    monkeypatch.delenv("SIGMA_SCAN_SPLIT_RULE", raising=False)
    shape, images = {"serial": ("stage2", 8), "segments": ("stage3", 1), "old-rule": ("stage2", 1)}[plan]
    if plan == "old-rule":
        monkeypatch.setenv("SIGMA_SCAN_SPLIT_RULE", "old")
    tag, (xc, xdbl, dtw, dtb, A, Ds, batch, H, W, D, N, R, Cp) = _scan_inputs(kind, N, shape, images)
    k = getattr(L, "DIRS_" + kind)
    out = (ctypes.c_int64 * 8)()
    L.check(L.lib().sigma_test_ss2d_fwd_plan(k, batch, H, W, D, N, R, 3, 0, L.lib().sigma_ss2d_scan_workspace_bytes(k, batch, H, W, D, N),
                                             out), "plan")
    nsplit = int(out[0])
    assert (nsplit == 1) == (plan == "serial"), nsplit
    assert nsplit == ss2d_fwd_plan(kind.lower(), batch, H, W, D, N, R, bf16=True)["nsplit"]
    y16 = fused.ss2d_scan(k, xc, xdbl, dtw, dtb, A, Ds, batch, H, W, D, N, R, Cp)
    monkeypatch.setattr(fused, "_FORCE_SPLIT", nsplit)
    y32 = fused.ss2d_scan(k, xc.float(), xdbl, dtw, dtb, A, Ds, batch, H, W, D, N, R, Cp)
    torch.cuda.synchronize()
    assert y16.dtype == H16 and y16.shape == y32.shape
    ref = y32.double()
    worst = _ratio(tag, y16, ref, HU * ref.abs() + SUB)
    record("fp16_scan", case=f"{tag}/{plan}", nsplit=nsplit, bound_used=worst, exact=bool(torch.equal(y16, y32.half())))


# ---------------------------------------------------------------- blocks and networks
CASES = {
    "tiny": ("sigma_tiny_480x640", "sigma_tiny", 480, 640, 9),
    "small": ("sigma_small_480x640", "sigma_small", 480, 640, 40),
    "base": ("sigma_base_720x960", "sigma_base", 720, 960, 5),
}


def _model(backbone, H, W, ncls, seed=SEED):
    from sigma_b200 import modules as M
    with contextlib.redirect_stdout(io.StringIO()):
        model = M.EncoderDecoder(cfg_tiny(H, W, num_classes=ncls, backbone=backbone), criterion=None)
    P.fill_state_dict(model, seed)
    return model.cuda().eval()


def _composed_fp16(model, *inputs):
    from sigma_b200 import modules as M
    with M.composed_path(), torch.autocast("cuda", dtype=H16):
        return model(*inputs)


@pytest.mark.parametrize("which", ["tiny", "small", "base"])
def test_fp16_logits_vs_reference_golden_fullsize(which):
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
        ec = err(_composed_fp16(model, rgb, mx))
        with fused.fp16_inference():
            assert fused.precision() == "fp16"
            fl = model(rgb, mx).float()
            bar = fused.logits_bar(ec)
    ef = err(fl)
    record("fp16_fullsize", tag=tag, fused_err=ef, composed_err=ec, ratio_to_composed=ef / max(ec, 1e-12))
    assert bool(torch.isfinite(fl).all()), f"{tag}: non-finite logits"
    assert ef <= bar, f"{tag}: fused fp16 logits error {ef:.2e} of scale > 2 x composed-under-fp16-autocast {ec:.2e} + floor"
    pred = fl.argmax(1).cpu().numpy().astype(np.uint8)
    diff = pred != g["argmax"]
    worst = float(g["margin"].astype(np.float32)[diff].max()) if diff.any() else 0.0
    assert worst <= 2.5 * bar * scale, f"{tag}: a label flipped where the reference's top-2 margin is {worst:.3e}"


@pytest.mark.parametrize("name", ["ss2d_n16", "ss2d_n4", "vssblock", "patchmerge_odd", "cromb", "conmb", "cvss_dec", "mamba_decoder",
                                  "rgbx_encoder_small"])
def test_fp16_blocks_vs_reference_goldens(name):
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
        co = as_tuple(_composed_fp16(mod, *inputs))
        with fused.fp16_inference():
            assert fused.precision() == "fp16"
            fo = as_tuple(mod(*inputs))
            for i, (f, c) in enumerate(zip(fo, co)):
                ref = g[f"out{i}"]
                sc = float(np.abs(ref).max())
                ef = float(np.abs(f.float().cpu().numpy() - ref).max()) / sc
                ec = float(np.abs(c.float().cpu().numpy() - ref).max()) / sc
                bar = fused.logits_bar(ec)
                record("fp16_block", tag=name, out=i, fused_err=ef, composed_err=ec, ratio_to_composed=ef / max(ec, 1e-12))
                assert f.dtype == torch.float32, f"{name}[{i}]: the block output (residual stream) must stay fp32"
                assert ef <= bar, f"{name}[{i}]: fused fp16 error {ef:.2e} of scale > bar {bar:.2e} (composed under fp16 autocast {ec:.2e})"


# ---------------------------------------------------------------- mode boundaries
@pytest.mark.parametrize("mode", ["tf32x3", "tf32", "bf16"])
def test_context_off_is_bit_identical_to_never_entering_it(mode):
    from sigma_b200 import fused
    torch.backends.cuda.matmul.allow_tf32 = mode == "tf32"
    try:
        model = _model("sigma_tiny", 64, 96, 9)
        rgb = P.randn(S, "fb/rgb", (2, 3, 64, 96)).cuda()
        mx = P.randn(S, "fb/x", (2, 3, 64, 96)).cuda()
        amp = torch.autocast("cuda", dtype=torch.bfloat16) if mode == "bf16" else contextlib.nullcontext()
        with torch.no_grad(), amp:
            assert fused.precision() == mode
            base = model(rgb, mx)
            with fused.fp16_inference():
                assert fused.precision() == "fp16"
                h = model(rgb, mx)
                with fused.fp16_inference(False):
                    assert fused.precision() == mode
                    off = model(rgb, mx)
            after = model(rgb, mx)
        assert torch.equal(base, off) and torch.equal(base, after)
        assert not torch.equal(base, h) and bool(torch.isfinite(h).all())   # the mode did run in between
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
            assert fused.precision() != "fp16"
            out = mod(*xs)
            out = out if isinstance(out, (tuple, list)) else (out,)
            sum(o.float().sum() for o in out).backward()
        return [o.detach() for o in out], [x.grad for x in xs]

    y1, g1 = run(contextlib.nullcontext())
    y2, g2 = run(fused.fp16_inference())
    for a, b in zip(y1, y2):
        assert a.dtype == b.dtype and torch.equal(a, b)
    for a, b in zip(g1, g2):
        assert a is not None and torch.isfinite(a).all()
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)   # parameter-gradient atomics may reorder sums


def test_inference_pipeline_fp16_replays_eager_and_recaptures():
    from sigma_b200 import fused
    from sigma_b200.pipeline import InferencePipeline
    torch.backends.cuda.matmul.allow_tf32 = False
    B, H, W = 2, 64, 96
    model = _model("sigma_tiny", H, W, 9)
    pipe = InferencePipeline(model, B, H, W, fp16=True)
    h_rgb = P.randn(S, "pipe16/rgb", (B, 3, H, W)).pin_memory()
    h_x = P.randn(S, "pipe16/x", (B, 3, H, W)).pin_memory()
    out = torch.empty((B,) + pipe.out_shape[1:], dtype=pipe.out.dtype).pin_memory()

    def eager():
        with torch.no_grad(), fused.fp16_inference():
            return model(h_rgb.cuda(), h_x.cuda()).cpu()

    pipe.submit(h_rgb, h_x, out)
    pipe.drain()
    first = eager()
    assert torch.equal(out, first)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    P.fill_state_dict(model, S + 1)
    with torch.no_grad():
        for p_ in model.parameters():
            p_.mul_(1.0)                                  # in-place: bumps every version counter -> re-capture, new fp16 weights
    pipe.submit(h_rgb, h_x, out)
    pipe.drain()
    second = eager()
    assert torch.equal(out, second) and not torch.equal(first, second)
    model.load_state_dict(sd)
    pipe.submit(h_rgb, h_x, out)
    pipe.drain()
    assert torch.equal(out, eager()) and torch.equal(out, first)
