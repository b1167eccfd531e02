"""GPU: the bf16 inference mode of the fused path (torch.autocast("cuda", dtype=torch.bfloat16) with autograd off) — every new
kernel against fp64 (or, for the scan, against the fp32 kernel fed the same bf16-rounded xc), the modules end to end against the
reference goldens, and the boundaries of the mode.

Per-element bounds.  Inputs are rounded to bf16 first and the fp64 reference is computed from those rounded values, so operand
rounding does not enter.  u = 2^-24; mag = (|A|·|W|^T)_ij or (|x| ⊛ |w|); K = products summed.
  GEMM     bf16 x bf16 products are exact in fp32; the fp32 accumulation adds at most K·2^-23·mag (one truncating addition per
           product of a partial sum <= mag), + 2^-20·mag of slack, and the epilogue rounds twice: 2u·(mag + |bias| + |res·rscale|).
           A bf16 output is then rounded once more: + 2^-8·|ref| (round to nearest even, 8 significand bits).
  Scan     the bf16 instance runs the same fp32 recurrence on the same (bf16-exact) xc values as the fp32 kernel; y is rounded once
           on its store, so |y_bf16 - y_fp32| <= 2^-8·|y_fp32| (+ 1e-6 for the sink of ties at tiny values).
Outputs sit inside NaN-filled buffers whose guard elements must stay bit-identical.

End to end, the bar calibrates itself against the reference's own semantics: under the same autocast the composed path (the
reference's op composition: nn.Linear / nn.Conv2d in bf16, the selective scan in fp32) is run on the same inputs, and the fused
bf16 logits must be within 2x its error against the fp32 golden, plus a floor of 1e-3 of the logit scale.  A flipped label is
accepted only where the reference's top-2 margin is below 2.5x that bar (DESIGN.md §3)."""
import contextlib
import ctypes
import io

import numpy as np
import pytest
import torch

import procedural as P
from helpers import SEED, cfg_tiny, gemm_plan, golden, record

pytestmark = pytest.mark.gpu
S = 67
U = 2.0 ** -24
BU = 2.0 ** -8       # bf16 unit roundoff: 8 significand bits, round to nearest even
NAN16 = 0x7FC0
NAN32 = 0x7FC00000
BF = torch.bfloat16


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _nan(shape, dtype):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def _guard_ok(t, what):
    if t.numel() == 0:
        return
    t = t.contiguous()
    bits = t.view(torch.int16) if t.dtype == BF else t.view(torch.int32)
    nan = NAN16 if t.dtype == BF else NAN32
    bad = int(((bits.to(torch.int32) & (0xFFFF if t.dtype == BF else -1)) != nan).sum())
    assert bad == 0, f"{what}: {bad} guard elements were written"


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
    if bn is not None:
        monkeypatch.setenv("SIGMA_GEMM_BN", str(bn))
    else:
        monkeypatch.delenv("SIGMA_GEMM_BN", raising=False)
    pl = gemm_plan(M, N, K, False)
    if bn is not None:
        assert pl["bn"] == bn
    assert pl["tiles"] >= need * pl["grid"], f"premise: {pl['tiles']} tiles over {pl['grid']} CTAs"
    tag = tag or f"bf16gemm/{M}/{N}/{K}/{extras}"
    lda, ldc, ldr = lda or K, ldc or N, ldr or N
    abuf = _nan((M, lda), BF)
    A = P.randn(S, tag + "/A", (M, K)).to(BF).cuda()
    abuf[:, :K] = A
    Wt = P.randn(S, tag + "/W", (N, K), K ** -0.5).cuda()
    Wb = Wt.to(BF)
    bias = P.randn(S, tag + "/b", (N,)).cuda() if "b" in extras else None
    res = rs = None
    if "r" in extras:
        rbuf = _nan((M, ldr), torch.float32)
        rbuf[:, :N] = P.randn(S, tag + "/r", (M, N)).cuda()
        res = rbuf[:, :N]
        rs = P.randn(S, tag + "/s", (N,), 0.2, 1.0).cuda() if "s" in extras else None
    cbuf = _nan((M + 3, ldc), out_dtype)
    out = cbuf[:M, :N]
    from sigma_b200 import _lib
    c_dtype = _lib.BF16 if out_dtype == BF else _lib.F32
    # the entry point itself (no torch.mm fallback can stand in for the wgmma instance)
    _lib.check(_lib.lib().sigma_linear_bf16(_p(abuf), lda, _p(Wb), _p(bias), _p(res), ldr, _p(rs), _p(out), ldc, c_dtype, M, N, K,
                                            _stream()), "sigma_linear_bf16")
    # and fused.linear routes a bf16 operand to it: the same bits
    via = fused.linear(abuf[:, :K], Wt, bias, out=torch.empty_like(out), residual=res, rscale=rs)
    torch.cuda.synchronize()
    assert torch.equal(via, out), f"{tag}: fused.linear differs from sigma_linear_bf16"
    got = out
    _guard_ok(cbuf[:, N:], f"{tag}: columns past N")
    _guard_ok(cbuf[M:], f"{tag}: rows past M")
    W64, Wa = Wb.double(), Wb.double().abs()
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
        if out_dtype == BF:
            bound = bound + BU * ref.abs()
        worst = max(worst, _ratio(f"{tag} rows {r0}..", got[r0:r0 + (1 << 15)], ref, bound))
    record("bf16_gemm", case=tag, out=str(out_dtype), bn=pl["bn"], bound_used=worst)


OUTS = [torch.float32, BF]


@pytest.mark.parametrize("out_dtype", OUTS, ids=["f32out", "bf16out"])
@pytest.mark.parametrize("bn", [32, 64, 96, 128, 160, 192, 224, 256])
def test_bf16_gemm_every_tile_width_multiwave(bn, out_dtype, monkeypatch):
    """Every m64nBNk16 bf16 instance, forced, on 301 row tiles x N = 768 (>= 3 tiles per CTA), with the whole epilogue."""
    _run_gemm(128 * 300 + 17, 768, 384, out_dtype, monkeypatch, bn=bn, extras="brs", tag=f"bf16gemm-bn{bn}")


@pytest.mark.parametrize("out_dtype", OUTS, ids=["f32out", "bf16out"])
@pytest.mark.parametrize("M,N,K,bn", [
    (128 * 800 + 1, 8, 40, None), (128 * 800 + 127, 40, 8, None), (128 * 300 + 1, 264, 104, None),
    (128 * 300 + 127, 264, 40, 256), (128 * 800 + 1, 8, 104, 32), (128 * 800 + 127, 40, 104, 64),
])
def test_bf16_gemm_ragged_multiwave(M, N, K, bn, out_dtype, monkeypatch):
    """K < 64 and K % 64 != 0 (TMA zero-fills past K), column tiles overhanging N (N > 256 too), M % 128 in {1, 127}."""
    _run_gemm(M, N, K, out_dtype, monkeypatch, bn=bn, extras="b")


@pytest.mark.parametrize("out_dtype", OUTS, ids=["f32out", "bf16out"])
@pytest.mark.parametrize("extras", ["b", "r", "rs", "brs"])
def test_bf16_gemm_epilogues_strided_multiwave(extras, out_dtype, monkeypatch):
    _run_gemm(128 * 300 + 17, 768, 192, out_dtype, monkeypatch, extras=extras, lda=192 + 40, ldc=768 + 12, ldr=768 + 20,
              tag=f"bf16gemm-epi/{extras}")


# The bf16 row-wise kernels (LayerNorm, patch-merge, merge + norm + gate) are compared with fp64 in tests/test_rowwise_fp64_gpu.py
# (io axis); the bf16 depthwise conv at Sigma's widths and production layouts in tests/test_gemm_waves_gpu.py (test_dwconv_silu_bf16).

# ---------------------------------------------------------------- depthwise conv
def test_bf16_dwconv_ring_wraps():
    """D = 64 (two 32-channel blocks): every CTA walks >= 9 tiles (the 4-slot ring wraps twice), ragged H / W, x a strided view
    ([x | z] rows).  Element by element against fp64 on the bf16 input's exact values, inside the fp32 kernel's per-element bound
    (test_gemm_waves_gpu._dwconv_ref) plus one bf16 store (rowwise_ref64.bf16_store_bound)."""
    from sigma_b200 import _lib
    from oracle import rowwise_ref64 as RR
    from test_gemm_waves_gpu import _dwconv_check, _dwconv_ref
    Bn, H, W, D = 7, 121, 161, 64
    tiles = Bn * -(-W // 16) * -(-H // 8)
    assert tiles >= 9 * (132 * 2 // (D // 32))
    xz = P.randn(S, "dw/x", (Bn, H, W, 2 * D)).to(BF).cuda()
    w = P.randn(S, "dw/w", (D, 1, 3, 3), 0.3).cuda()
    b = P.randn(S, "dw/b", (D,), 0.1).cuda()
    buf = _nan((Bn * H * W + 5, D), BF)
    _lib.check(_lib.lib().sigma_dwconv3x3_silu_fwd_bf16(_p(xz), 2 * D, H * W * 2 * D, _p(w), _p(b), _p(buf), H * W * D, Bn, H, W, D,
                                                        _stream()), "dw")
    torch.cuda.synchronize()
    _guard_ok(buf[Bn * H * W:], "past the end")
    ref, e = _dwconv_ref(xz[..., :D], w, b)
    worst = _dwconv_check("dwconv bf16", buf[:Bn * H * W].view(Bn, H, W, D), ref, RR.bf16_store_bound(ref, e))
    record("bf16_dwconv", case="ring", max_err_over_bound=worst)


# ---------------------------------------------------------------- scan
SCAN_SHAPES = {"stage0": (120, 160, 192, 6), "stage2": (30, 40, 768, 24)}   # stage 2: 4 CTAs per SM in fp32, 3 in bf16 (DESIGN §5.4)


@pytest.mark.parametrize("shape", ["stage0", "stage2"])
@pytest.mark.parametrize("N", [4, 16])
@pytest.mark.parametrize("kind", ["CROSS4", "SEQ2", "CROSS"])
def test_bf16_scan_matches_fp32_kernel_after_one_rounding(kind, N, shape):
    from sigma_b200 import _lib, fused
    H, W, D, R = SCAN_SHAPES[shape]
    k = getattr(_lib, "DIRS_" + kind)
    batch = 2
    K = {"CROSS4": 4, "SEQ2": 2, "CROSS": 1}[kind]
    Lseq = 2 * H * W if kind == "SEQ2" else H * W
    Cp = _lib.lib().sigma_ss2d_padded_cp(N, R)
    tag = f"scan/{kind}/{N}/{shape}"
    nw = 2 if kind == "CROSS" else K                     # weight sets: modalities or directions
    xc = P.randn(S, tag + "/xc", (batch, Lseq, D)).to(BF).cuda()
    xdbl = P.randn(S, tag + "/dbl", (batch, Lseq, K, Cp), 0.5).cuda()
    dtw = P.randn(S, tag + "/dtw", (nw * D, R), R ** -0.5).cuda()
    dt = torch.exp(P.rand(S, tag + "/dt", (nw * D,)) * (np.log(0.1) - np.log(1e-3)) + np.log(1e-3))
    dtb = (dt + torch.log(-torch.expm1(-dt))).cuda()
    A = (-torch.exp(P.randn(S, tag + "/A", (nw * D, N), 0.5))).cuda().contiguous()
    Ds = torch.ones(nw * D, device="cuda")
    y16 = fused.ss2d_scan(k, xc, xdbl, dtw, dtb, A, Ds, batch, H, W, D, N, R, Cp)
    y32 = fused.ss2d_scan(k, xc.float(), xdbl, dtw, dtb, A, Ds, batch, H, W, D, N, R, Cp)
    torch.cuda.synchronize()
    assert y16.dtype == BF and y16.shape == y32.shape
    ref = y32.double()
    worst = _ratio(tag, y16, ref, BU * ref.abs() + 1e-6)
    record("bf16_scan", case=tag, bound_used=worst, exact=bool(torch.equal(y16, y32.to(BF))))


# ---------------------------------------------------------------- modules end to end
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


def _bf16():
    return torch.autocast("cuda", dtype=torch.bfloat16)


@pytest.mark.parametrize("which", ["tiny", "small", "base"])
def test_bf16_logits_vs_reference_golden_fullsize(which):
    """Measured on an H100 SXM (700 W limit): the fused bf16 error is 0.46 (tiny), 0.77 (small) and 0.88 (base) of the composed path's
    under the same autocast (recorded per case
    in the parity log as ratio_to_composed)."""
    from sigma_b200 import fused, modules as M
    tag, backbone, H, W, ncls = CASES[which]
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    g = golden(tag)
    model = _model(backbone, H, W, ncls)
    rgb = P.randn(SEED, tag + "/rgb", (1, 3, H, W)).cuda()
    mx = P.randn(SEED, tag + "/x", (1, 3, H, W)).cuda()
    scale = float(g["logits_absmax"])
    err = lambda t: float(np.abs(t[:, :, 3::8, 5::8].float().cpu().numpy() - g["logits_sub"]).max()) / scale
    with torch.no_grad(), _bf16():
        assert fused.precision() == "bf16"
        fl = model(rgb, mx).float()
        with M.composed_path():
            ec = err(model(rgb, mx))
        bar = fused.logits_bar(ec)
    ef = err(fl)
    record("bf16_fullsize", tag=tag, fused_err=ef, composed_err=ec, ratio_to_composed=ef / max(ec, 1e-12))
    assert ef <= bar, f"{tag}: fused bf16 logits error {ef:.2e} of scale > 2 x composed-under-autocast {ec:.2e} + floor"
    pred = fl.argmax(1).cpu().numpy().astype(np.uint8)
    diff = pred != g["argmax"]
    worst = float(g["margin"].astype(np.float32)[diff].max()) if diff.any() else 0.0
    assert worst <= 2.5 * bar * scale, f"{tag}: a label flipped where the reference's top-2 margin is {worst:.3e}"


def _block_cases():
    import torch.nn as nn
    from sigma_b200 import modules as M
    xin = P.randn(SEED, "mod/x", (2, 6, 5, 32)).cuda()
    xin2 = P.randn(SEED, "mod/x2", (2, 6, 5, 32)).cuda()
    return {
        "ss2d_n16": (lambda: M.SS2D(d_model=32, d_state=16), (xin,)),
        "ss2d_n4": (lambda: M.SS2D(d_model=32, d_state=4), (xin,)),
        "vssblock": (lambda: M.VSSBlock(hidden_dim=32, norm_layer=nn.LayerNorm, mlp_ratio=0.0, d_state=16), (xin,)),
        "patchmerge_odd": (lambda: M.PatchMerging2D(32, 64), (P.randn(SEED, "mod/pm", (2, 5, 7, 32)).cuda(),)),
        "cromb": (lambda: M.CrossMambaFusionBlock(hidden_dim=32, mlp_ratio=0.0, d_state=4), (xin, xin2)),
        "conmb": (lambda: M.ConcatMambaFusionBlock(hidden_dim=32, mlp_ratio=0.0, d_state=4), (xin, xin2)),
        "cvss_dec": (lambda: M.CVSSDecoderBlock(hidden_dim=32, norm_layer=nn.LayerNorm, d_state=4, mlp_ratio=4.0), (xin,)),
        "mamba_decoder": (lambda: M.MambaDecoder(img_size=[64, 96], in_channels=[32, 64, 128, 256], num_classes=5, embed_dim=32),
                          ([P.randn(SEED, f"dec/f{i}", (1, 32 * 2 ** i, 16 // 2 ** i, 24 // 2 ** i)).cuda() for i in range(4)],)),
        "rgbx_encoder_small": (lambda: M.RGBXTransformer(depths=[1, 1, 2, 1], dims=32, pretrained=None, mlp_ratio=0.0,
                                                         downsample_version="v1", drop_path_rate=0.2),
                               (P.randn(SEED, "enc/rgb", (1, 3, 64, 96)).cuda(), P.randn(SEED, "enc/x", (1, 3, 64, 96)).cuda())),
    }


@pytest.mark.parametrize("name", ["ss2d_n16", "ss2d_n4", "vssblock", "patchmerge_odd", "cromb", "conmb", "cvss_dec", "mamba_decoder",
                                  "rgbx_encoder_small"])
def test_bf16_blocks_vs_reference_goldens(name):
    """Each module of the bf16 mode against the reference's golden (the same goldens tests/test_modules_gpu.py uses): SS2D at
    d_state 4 / 16, VSSBlock, PatchMerging2D at odd 5 x 7, CroMB (residual=True: the residual in the out_proj epilogue), ConMB
    (SE gates, SEQ2 scan), CVSSDecoderBlock (the rscale epilogue), the decoder and a small encoder.  Bar per output:
    fused.logits_bar(composed error) = 2 x the composed path's error under the same autocast + the floor, of the output's scale."""
    from sigma_b200 import fused, modules as M
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    ctor, inputs = _block_cases()[name]
    mod = ctor()
    P.fill_state_dict(mod, SEED)
    mod = mod.cuda().eval()
    g = golden(name)
    as_tuple = lambda o: tuple(o) if isinstance(o, (tuple, list)) else (o,)
    with torch.no_grad(), _bf16():
        assert fused.precision() == "bf16"
        fo = as_tuple(mod(*inputs))
        with M.composed_path():
            co = as_tuple(mod(*inputs))
        for i, (f, c) in enumerate(zip(fo, co)):
            ref = g[f"out{i}"]
            scale = float(np.abs(ref).max())
            ef = float(np.abs(f.float().cpu().numpy() - ref).max()) / scale
            ec = float(np.abs(c.float().cpu().numpy() - ref).max()) / scale
            bar = fused.logits_bar(ec)
            record("bf16_block", tag=name, out=i, fused_err=ef, composed_err=ec, ratio_to_composed=ef / max(ec, 1e-12))
            assert f.dtype == torch.float32, f"{name}[{i}]: the block output (residual stream) must stay fp32"
            assert ef <= bar, f"{name}[{i}]: fused bf16 error {ef:.2e} of scale > bar {bar:.2e} (composed under autocast {ec:.2e})"


# ---------------------------------------------------------------- mode boundaries
def test_autocast_off_and_fp16_are_the_fp32_path_bit_for_bit():
    from sigma_b200 import fused
    torch.backends.cuda.matmul.allow_tf32 = False
    model = _model("sigma_tiny", 64, 96, 9)
    rgb = P.randn(S, "mb/rgb", (2, 3, 64, 96)).cuda()
    mx = P.randn(S, "mb/x", (2, 3, 64, 96)).cuda()
    with torch.no_grad():
        assert fused.precision() == "tf32x3"
        base = model(rgb, mx)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=False):
            off = model(rgb, mx)
        with torch.autocast("cuda", dtype=torch.float16):
            assert fused.precision() == "tf32x3"
            h = model(rgb, mx)
    assert torch.equal(base, off) and torch.equal(base, h)
    assert base.dtype == torch.float32


@pytest.mark.parametrize("which", ["vssblock", "conmb", "cromb", "cvss_dec"])
def test_grad_enabled_under_bf16_autocast_keeps_the_training_path(which, monkeypatch):
    """With autograd on, the bf16 mode must not exist: a training forward + backward under bf16 autocast gives the same output
    (bit for bit) and the same input gradients as with the mode selection replaced by the dense-only rule it extends."""
    from sigma_b200 import fused
    ctor, inputs = _block_cases()[which]

    def run():
        mod = ctor()
        P.fill_state_dict(mod, S)
        mod = mod.cuda().train()
        xs = [t.detach().clone().requires_grad_(True) for t in inputs]
        with _bf16():
            assert fused.precision() != "bf16"
            out = mod(*xs)
        out = out if isinstance(out, (tuple, list)) else (out,)
        sum(o.float().sum() for o in out).backward()
        return [o.detach() for o in out], [x.grad for x in xs]

    y1, g1 = run()
    monkeypatch.setattr(fused, "precision", fused._dense_precision)
    y2, g2 = run()
    for a, b in zip(y1, y2):
        assert a.dtype == b.dtype and torch.equal(a, b)
    for a, b in zip(g1, g2):
        assert a is not None and torch.isfinite(a).all()
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)   # parameter-gradient atomics may reorder sums


def test_inference_pipeline_bf16_replays_eager_and_recaptures():
    from sigma_b200 import modules as M
    from sigma_b200.pipeline import InferencePipeline
    torch.backends.cuda.matmul.allow_tf32 = False
    B, H, W = 2, 64, 96
    model = _model("sigma_tiny", H, W, 9)
    pipe = InferencePipeline(model, B, H, W, amp_dtype=torch.bfloat16)
    h_rgb = P.randn(S, "pipe/rgb", (B, 3, H, W)).pin_memory()
    h_x = P.randn(S, "pipe/x", (B, 3, H, W)).pin_memory()
    out = torch.empty((B,) + pipe.out_shape[1:], dtype=pipe.out.dtype).pin_memory()

    def eager():
        with torch.no_grad(), _bf16():
            return model(h_rgb.cuda(), h_x.cuda()).cpu()

    pipe.submit(h_rgb, h_x, out)
    pipe.drain()
    assert torch.equal(out, eager())
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    P.fill_state_dict(model, S + 1)
    model.load_state_dict({k: v for k, v in model.state_dict().items()})
    with torch.no_grad():
        for p_ in model.parameters():
            p_.mul_(1.0)                                  # in-place: bumps every version counter -> re-capture
    pipe.submit(h_rgb, h_x, out)
    pipe.drain()
    assert torch.equal(out, eager())
    model.load_state_dict(sd)
    pipe.submit(h_rgb, h_x, out)
    pipe.drain()
    assert torch.equal(out, eager())
    assert isinstance(model, M.EncoderDecoder)
