"""GPU: the fp16 training mode of the fused core (sigma_ss2d_scan_fwd_save_fp16 + sigma_ss2d_scan_bwd_saved_fp16, LayerNormFn on fp16
activations) against fp64, and its range semantics under loss scaling.
* The C-ABI pair, element by element inside the per-element bounds of oracle/ss2d_ref64.py run on a given delta'.  Inputs are
  drawn, then xc and dy are rounded to fp16, so the reference sees the exact values (widened to fp32, which the oracle takes as
  exact).  The kernel's delta' is checked on its own against the fp64 softplus inside `fp32 bound + 2^-11·|delta'| + 2^-25` (the
  last term: a delta' below 2^-14 is stored subnormal); everything downstream is checked against the reference run on THAT delta'
  (`delta=`), so nothing is loosened.  y's bound adds its one fp16 rounding the same way.  Kinds cross4 / seq2 at d_state 4 and
  16, every padded dt_rank Sigma trains with, ragged maps, batch 1 / 2 / 3, L-segments 1, 2, 7, the library's choice, the cap,
  and a forward cut differently from its backward; outputs inside NaN-filled guards; the dt_r and padding columns of dxdbl 0.
* Kind cross (CroMB) the same way at CroMB's training shapes.
* FusedSS2DCore.apply under fp16 autocast with the switch on (fp16 output, fp16 saved xc and delta', the _fp16 entry points, all
  six gradients against the fp64 chain), off and under the deterministic switch (the fp32 and fp32 _det entry points).
* LayerNormFn with fp16 activations against fp64 at every width of ops._LN_WIDTHS.
* Range: an inf in dy reaches dxc and every parameter gradient; a finite dy whose fp32 dxc passes 65504 gives ±inf there, never a
  clamped value; a VSSBlock trained through TrainStep with a GradScaler skips an overflowing first step (as the switch-off run
  does at the same scale) and applies a later one."""
import math

import pytest
import torch
import torch.nn as nn

import procedural as P
from helpers import SEED, guard_ok as _guard_ok, guarded as _guarded, ptr as _p, record, ss2d_kind as _kid, ss2d_params, stream as _stream
from oracle import ss2d_ref64 as R64
from sigma_b200.ops import _LN_WIDTHS
from test_ss2d_bwd_fp64_gpu import CROSS_CASES

pytestmark = pytest.mark.gpu
S = 307
F16 = torch.float16
F16_RN = 2.0 ** -11          # relative error of rounding to fp16 (11 significand bits) to nearest
F16_SUB = 2.0 ** -25         # absolute error of rounding into fp16's subnormal range (spacing 2^-24)


def _round_bound(ref, bnd):
    """per-element bound of a value the kernel rounded once to fp16, from the fp64 value and its bound before the rounding"""
    return bnd + F16_RN * (ref.abs() + bnd) + F16_SUB


def _delta_ref(kind, xdbl, dtw, dtb, N):
    """fp64 softplus(dt_proj) slabs (K, B, Lseq, D) and the bound of a kernel delta' rounded to fp16"""
    ref, bnd = R64.delta_ref64(kind, xdbl, dtw, dtb, N)
    return ref, _round_bound(ref, bnd)


def _ref(kind, xc, xdbl, dtw, dtb, A, Ds, dy, H, W, delta):
    """ss2d_ref64 on the fp16 inputs' exact fp32 values and the kernel's delta'; y's bound gets its fp16 store"""
    ref, bnd = R64.ss2d_ref64(kind, xc.float(), xdbl, dtw, dtb, A, Ds, dy.float(), H, W, delta=delta.double())
    bnd["y"] = _round_bound(ref["y"], bnd["y"])
    return ref, bnd


def _check(tag, name, got, ref, bnd, worst):
    ok = ~ref.isnan()
    assert bool(torch.equal(got.isnan(), ~ok)), f"{tag} {name}: written where the kernel has nothing to write, or NaN"
    frac = R64.bound_fraction(got[ok], ref[ok], bnd[ok])
    worst[name] = max(worst.get(name, 0.0), frac)
    assert frac <= 1.0, f"{tag} {name}: {frac:.3f} of the per-element bound"


def _pair(kind, B, H, W, D, N, R, Cp, args16, fs, bs):
    """run the fp16 pair into guarded buffers; returns (buffers, outputs)"""
    from sigma_b200 import _lib
    L_ = _lib.lib()
    xc, xdbl, dtw, dtb, A, Ds, dy = args16
    K, Lseq = xdbl.shape[2], xc.shape[1]
    Kw = 2 if kind == "cross" else K
    T = L_.sigma_ss2d_scan_hs_bytes(_kid(kind), B, H, W, D, N) // (4 * K * B * D * N)
    bufs, outs = {}, {}
    for name, shape, dt in [("y", (K, B, Lseq, D), F16), ("delta", (K, B, Lseq, D), F16), ("hs", (K, B, T, D, N), torch.float32),
                            ("dxc", (B, Lseq, D), torch.float32), ("ddelta", (K, B, Lseq, D), torch.float32),
                            ("dxdbl", (B, Lseq, K, Cp), torch.float32), ("dA", (Kw * D, N), torch.float32), ("dDs", (Kw * D,), torch.float32),
                            ("ddtb", (Kw, D), torch.float32)]:
        bufs[name], outs[name] = _guarded(shape, dt)
    head = (_kid(kind), _p(xc), _p(xdbl), _p(dtw), _p(dtb), _p(A), _p(Ds))
    fwb = L_.sigma_ss2d_scan_workspace_bytes(_kid(kind), B, H, W, D, N)
    fws = torch.zeros(max(fwb, 4), dtype=torch.uint8, device="cuda")
    _lib.check(L_.sigma_ss2d_scan_fwd_save_fp16(*head, _p(outs["y"]), _p(outs["delta"]), _p(outs["hs"]), B, H, W, D, N, R, Cp, _p(fws), fwb,
                                                fs, _stream()), "sigma_ss2d_scan_fwd_save_fp16")
    wsb = L_.sigma_ss2d_scan_bwd_workspace_bytes(_kid(kind), B, H, W, D, N)
    ws = torch.full((wsb // 4,), float("nan"), device="cuda")
    tail = (_p(outs["dxc"]), _p(outs["ddelta"]), _p(outs["dxdbl"]), _p(outs["dA"]), _p(outs["dDs"]), _p(outs["ddtb"]), B, H, W, D, N, R, Cp,
            _p(ws), wsb)
    _lib.check(L_.sigma_ss2d_scan_bwd_saved_fp16(*head, _p(dy), _p(outs["delta"]), _p(outs["hs"]), *tail, bs, _stream()),
               "sigma_ss2d_scan_bwd_saved_fp16")
    torch.cuda.synchronize()
    return bufs, outs


def _args16(kind, B, H, W, D, N, R, tag):
    (xc, xdbl, dtw, dtb, A, Ds, dy), Cp = ss2d_params(S, kind, B, H, W, D, N, R, tag)
    return [xc.to(F16), xdbl, dtw, dtb, A, Ds, dy.to(F16)], Cp


def _check_outputs(t, N, outs, bufs, ref, bnd, worst):
    for name in ("y", "hs", "dxc", "ddelta", "dA", "dDs", "ddtb"):
        _check(t, name, outs[name], ref[name], bnd[name], worst)
    dx = outs["dxdbl"]
    _check(t, "dB", dx[..., :N], ref["dB"], bnd["dB"], worst)
    _check(t, "dC", dx[..., N:2 * N], ref["dC"], bnd["dC"], worst)
    assert bool((dx[..., 2 * N:] == 0).all()), f"{t}: the dt_r / padding columns of dxdbl must stay 0"
    for name, buf in bufs.items():
        _guard_ok(buf, f"{t} {name}")


SPLITS = [(0, 0), (1, 1), (2, 2), (7, 7), (100, 100), (3, 7), (1, 2)]

# kind, B, H, W, D, N, R
CASES = [
    ("cross4", 2, 120, 160, 192, 16, 6), ("cross4", 2, 60, 80, 384, 16, 12), ("cross4", 2, 30, 40, 768, 16, 24),
    ("cross4", 2, 15, 20, 1536, 16, 48), ("cross4", 2, 45, 60, 1024, 16, 32), ("cross4", 2, 23, 30, 2048, 16, 64),   # SS2D
    ("seq2", 2, 120, 160, 192, 4, 6), ("seq2", 2, 15, 20, 1536, 4, 48), ("seq2", 2, 23, 30, 2048, 4, 64),              # ConMB
    ("cross4", 2, 120, 160, 192, 4, 6), ("cross4", 2, 60, 80, 384, 4, 12), ("cross4", 2, 30, 40, 768, 4, 24),          # decoder SS2D
    ("cross4", 1, 30, 40, 768, 16, 24), ("cross4", 3, 30, 40, 768, 16, 24),
]


@pytest.mark.parametrize("kind,B,H,W,D,N,R", CASES)
def test_fp16_pair_matches_fp64(kind, B, H, W, D, N, R):
    tag = f"{kind}/{B}/{H}x{W}/D{D}/N{N}/R{R}"
    args16, Cp = _args16(kind, B, H, W, D, N, R, tag)
    xc, xdbl, dtw, dtb, A, Ds, dy = args16
    dref, dbnd = _delta_ref(kind, xdbl, dtw, dtb, N)
    worst, refs = {}, {}
    for fs, bs in SPLITS:
        t = f"{tag} fwd={fs} bwd={bs}"
        bufs, outs = _pair(kind, B, H, W, D, N, R, Cp, args16, fs, bs)
        _check(t, "delta", outs["delta"], dref, dbnd, worst)
        key = outs["delta"].view(torch.int16).clone()
        hit = [v for kk, v in refs.values() if torch.equal(kk, key)]       # delta' does not depend on the cut: one reference run
        if not hit:
            refs[fs] = (key, _ref(kind, xc, xdbl, dtw, dtb, A, Ds, dy, H, W, outs["delta"]))
            hit = [refs[fs][1]]
        ref, bnd = hit[0]
        _check_outputs(t, N, outs, bufs, ref, bnd, worst)
    assert len(refs) == 1, "delta' must not depend on the L-segment cut"
    record(f"ss2d fp16 train fp64 {tag}", **worst)


# Bt = 2·images, H, W, D, N, R: CroMB's training shapes at d_state 4 with 1-3 images, and two d_state 16 cases
CROSS = [(B, H, W, D, N, R) for _, B, H, W, D, N, R in CROSS_CASES] + [(2, 60, 80, 384, 16, 12), (4, 23, 30, 192, 16, 6)]


@pytest.mark.parametrize("B,H,W,D,N,R", CROSS)
def test_fp16_pair_cross(B, H, W, D, N, R):
    kind, tag = "cross", f"cross/{B}/{H}x{W}/D{D}/N{N}/R{R}"
    args16, Cp = _args16(kind, B, H, W, D, N, R, tag)
    xc, xdbl, dtw, dtb, A, Ds, dy = args16
    dref, dbnd = _delta_ref(kind, xdbl, dtw, dtb, N)
    worst, key, ref = {}, None, None
    for fs, bs in [(0, 0), (1, 1), (3, 7), (100, 100)]:
        t = f"{tag} fwd={fs} bwd={bs}"
        bufs, outs = _pair(kind, B, H, W, D, N, R, Cp, args16, fs, bs)
        _check(t, "delta", outs["delta"], dref, dbnd, worst)
        if key is None:
            key = outs["delta"].view(torch.int16).clone()
            ref, bnd = _ref(kind, xc, xdbl, dtw, dtb, A, Ds, dy, H, W, outs["delta"])
        assert torch.equal(outs["delta"].view(torch.int16), key), f"{t}: delta' depends on the L-segment cut"
        _check_outputs(t, N, outs, bufs, ref, bnd, worst)
    record(f"ss2d fp16 train fp64 {tag}", **worst)


def _h(t):
    return t.to(F16).float()


def _core_leaves(kind, B, H, W, D, N, R, tag, Ds_scale=1.0):
    K = {"cross4": 4, "seq2": 2, "cross": 1}[kind]
    Kw = 2 if kind == "cross" else K
    Lseq = H * W * (2 if kind == "seq2" else 1)
    xc0 = P.randn(S, tag + "/xc", (B, Lseq, D)).cuda().to(F16)
    xpw = _h(P.randn(S, tag + "/xpw", (Kw, R + 2 * N, D), D ** -0.5).cuda())           # exact in the fp16 x_proj GEMM
    dtw = P.rand(S, tag + "/dtw", (Kw, D, R), -R ** -0.5, R ** -0.5).cuda()
    dt = torch.exp(P.rand(S, tag + "/dt", (Kw, D), math.log(1e-3), math.log(0.1)))
    dtb = (dt + torch.log(-torch.expm1(-dt))).cuda()
    Al = (torch.log(torch.arange(1, N + 1, dtype=torch.float32)).repeat(Kw * D, 1) + P.rand(S, tag + "/A", (Kw * D, N), -0.2, 0.2)).cuda()
    Ds = P.randn(S, tag + "/Ds", (Kw * D,), 0.1, 1.0).cuda() * Ds_scale
    return [xc0, xpw, dtw, dtb, Al, Ds], K, Kw, Lseq


@pytest.mark.parametrize("kind,B,H,W,D,N,R", [("cross4", 2, 60, 80, 384, 16, 12), ("seq2", 2, 15, 20, 1536, 4, 48), ("cross4", 2, 30, 40, 768, 4, 24),
                                               ("cross", 4, 30, 40, 768, 4, 24)])
def test_fused_core_autograd_fp16_mode(kind, B, H, W, D, N, R, monkeypatch):
    from sigma_b200 import _lib, fused, ops
    from test_ss2d_bwd_fp64_gpu import core_chain64, core_xdbl
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    Cp = _lib.lib().sigma_ss2d_padded_cp(N, R)
    tag = f"ag16/{kind}/{B}/{H}x{W}/D{D}/N{N}/R{R}"
    leaves0, K, Kw, Lseq = _core_leaves(kind, B, H, W, D, N, R, tag)
    wgt = _h(P.randn(S, tag + "/w", (B, Lseq, D)).cuda())

    def run(on):
        leaves = [t.clone().requires_grad_(True) for t in leaves0]
        saved, calls = [], []
        s0, b0 = fused.ss2d_scan_save, ops._call_ss2d_bwd
        monkeypatch.setattr(fused, "ss2d_scan_save", lambda kd, xc, *a: (calls.append(("fwd", xc.dtype)), s0(kd, xc, *a))[1])
        monkeypatch.setattr(ops, "_call_ss2d_bwd", lambda args, sv=False, det=False: (calls.append(("bwd", sv, det)), b0(args, sv, det))[1])
        with torch.autograd.graph.saved_tensors_hooks(lambda t: (saved.append(t), t)[1], lambda t: t):
            with torch.autocast("cuda", dtype=F16):
                if on is None:
                    y = ops.FusedSS2DCore.apply(*leaves, _kid(kind), H, W)
                else:
                    with ops.fp16_training_core(on):
                        y = ops.FusedSS2DCore.apply(*leaves, _kid(kind), H, W)
        (y.float() * wgt).sum().backward()
        monkeypatch.setattr(fused, "ss2d_scan_save", s0)
        monkeypatch.setattr(ops, "_call_ss2d_bwd", b0)
        return y.detach(), [t.grad for t in leaves], saved, calls

    y0, g0, _, c0 = run(None)                     # the switch never touched
    y1, g1, saved, c1 = run(True)
    y2, g2, _, c2 = run(False)
    with torch.autocast("cuda", dtype=F16), ops.bf16_training_core():   # the bf16 switch does not apply under fp16 autocast
        y3 = ops.FusedSS2DCore.apply(*[t.clone().requires_grad_(True) for t in leaves0], _kid(kind), H, W)
    assert y3.dtype == torch.float32 and torch.equal(y3.detach(), y0)
    # off: the fp32 entry points, the same output bits, gradients the same up to the order of the backward's atomic sums
    assert c0 == c2 == [("fwd", torch.float32), ("bwd", True, False)] and y0.dtype == torch.float32 and torch.equal(y0, y2)
    for a, b in zip(g0, g2):          # (the fp16 leaf xc gets the fp32 dxc rounded by autograd: a last-bit difference there is one fp16 ulp)
        tol = 2.0 ** -10 if a.dtype == F16 else 1e-4
        assert a.dtype == b.dtype and float((a.float() - b.float()).abs().max()) <= tol * float(a.float().abs().max())
    # on: fp16 in, out and saved
    assert c1 == [("fwd", F16), ("bwd", ops._SAVED_FP16, False)] and y1.dtype == F16
    assert g1[0].dtype == F16 and all(g.dtype == torch.float32 for g in g1[1:])
    slabs = [t for t in saved if t.shape == (K, B, Lseq, D)]
    assert len(slabs) == 1 and slabs[0].dtype == F16 and [t.dtype for t in saved if t.shape == (B, Lseq, D)] == [F16]
    hs_bytes = _lib.lib().sigma_ss2d_scan_hs_bytes(_kid(kind), B, H, W, D, N)
    want = (B * Lseq * D * 2 + K * B * Lseq * D * 2 + B * Lseq * K * Cp * 4 + Kw * Cp * D * 4 + Kw * D * R * 4 + Kw * D * 4
            + Kw * D * N * 4 + Kw * D * 4 + hs_bytes)          # xc, delta' (fp16); x_dbl, xw, W_dt, bias, A, Ds, hs (fp32)
    assert sum(t.numel() * t.element_size() for t in saved) == want
    # the fp64 chain on the delta' the forward saved
    xc0, xpw, dtw, dtb, Al, Ds = leaves0
    with torch.no_grad():
        xdbl, xw = core_xdbl(kind, xc0, xpw, N, R, Cp)                # the forward's own x_proj GEMM calls
        A = -torch.exp(Al)
        ref, _ = R64.ss2d_ref64(kind, xc0.float(), xdbl, dtw, dtb, A, Ds, wgt, H, W, delta=slabs[0].double())
        want, _ = core_chain64(kind, ref, None, xc0, xdbl, xw, dtw, N, R, Cp)
        want[4] = want[4] * A.double()
        dxc = want[0]
        worst = {}
        # y: K directions each rounded to fp16, added in fp32, rounded once more; dxc: one rounding of the fp32 sum
        yr = ref["y"].sum(0)
        ey = float(((y1.double() - yr).abs() - F16_RN * (ref["y"].abs().sum(0) + yr.abs())).max()) / float(yr.abs().max())
        assert ey <= 1e-4, f"{tag} y: {ey:.2e} of scale beyond the roundings"
        edx = float(((g1[0].double() - dxc).abs() - F16_RN * dxc.abs()).max()) / float(dxc.abs().max())
        assert edx <= 1e-4, f"{tag} dxc: {edx:.2e} of scale beyond the rounding"
        for name, g, r in zip(["dx_proj_weight", "ddt_projs_weight", "ddt_projs_bias", "dA_logs", "dDs"], g1[1:], want[1:]):
            err = float((g.double() - r).abs().max()) / float(r.abs().max())
            worst[name] = err
            assert err <= 1e-3, f"{tag} {name}: {err:.2e} of its scale"
    record(f"ss2d fp16 autograd fp64 {tag}", y=ey, dxc=edx, **worst)


def test_deterministic_switch_keeps_the_fp32_det_path():
    from sigma_b200 import ops
    kind, B, H, W, D, N, R = "cross4", 2, 15, 20, 192, 16, 6
    leaves, *_ = _core_leaves(kind, B, H, W, D, N, R, "det16")
    leaves = [t.requires_grad_(True) for t in leaves]
    calls, b0 = [], ops._call_ss2d_bwd
    ops._call_ss2d_bwd = lambda args, sv=False, det=False: (calls.append((sv, det)), b0(args, sv, det))[1]
    torch.use_deterministic_algorithms(True)
    try:
        with torch.autocast("cuda", dtype=F16), ops.fp16_training_core():
            y = ops.FusedSS2DCore.apply(*leaves, _kid(kind), H, W)
        y.float().sum().backward()
    finally:
        torch.use_deterministic_algorithms(False)
        ops._call_ss2d_bwd = b0
    assert y.dtype == torch.float32 and calls == [(True, True)]
    assert all(t.grad is not None and bool(t.grad.isfinite().all()) for t in leaves)


@pytest.mark.parametrize("C", sorted(_LN_WIDTHS))
@pytest.mark.parametrize("rows", [2 * 120 * 160, 2 * 15 * 20, 7])
def test_layernorm_fp16_matches_fp64(C, rows):
    from sigma_b200 import ops
    if rows * C > 2 * 120 * 160 * 384:
        rows = 2 * 30 * 40                                   # Sigma's widths above 384 only occur from stage 2 on
    tag = f"ln16/{rows}x{C}"
    x = (P.randn(S, tag + "/x", (rows, C)) * 1.5 + 0.3).cuda().to(F16).requires_grad_(True)
    w = P.randn(S, tag + "/w", (C,), 0.2, 1.0).cuda().requires_grad_(True)
    b = P.randn(S, tag + "/b", (C,), 0.2).cuda().requires_grad_(True)
    dy = P.randn(S, tag + "/dy", (rows, C)).cuda().to(F16)
    norm = torch.nn.LayerNorm(C).cuda()
    with torch.no_grad():
        norm.weight.copy_(w); norm.bias.copy_(b)
    with torch.autocast("cuda", dtype=F16), ops.fp16_training_core():
        y = ops.layer_norm(norm, x)
    assert y.dtype == F16
    y.backward(dy)
    assert x.grad.dtype == F16 and norm.weight.grad.dtype == torch.float32
    xd = x.detach().double().requires_grad_(True)
    wd, bd = w.detach().double().requires_grad_(True), b.detach().double().requires_grad_(True)
    yr = torch.nn.functional.layer_norm(xd, (C,), wd, bd, norm.eps)
    yr.backward(dy.double())
    tol = lambda r: F16_RN * r.abs() + F16_SUB + 1e-5 * (1.0 + r.abs())
    assert bool(((y.double() - yr).abs() <= tol(yr.detach())).all())
    assert bool(((x.grad.double() - xd.grad).abs() <= tol(xd.grad) + 1e-5 * float(xd.grad.abs().max())).all())
    for got, ref in ((norm.weight.grad, wd.grad), (norm.bias.grad, bd.grad)):
        assert float((got.double() - ref).abs().max()) <= 1e-4 * float(ref.abs().max()) + 1e-4 * math.sqrt(rows)
    # with the switch off the same call widens: fp32 out, as before; the bf16 switch does not apply under fp16 autocast
    x2 = x.detach().clone().requires_grad_(True)
    with torch.autocast("cuda", dtype=F16):
        assert ops.layer_norm(norm, x2).dtype == torch.float32
    with torch.autocast("cuda", dtype=F16), ops.bf16_training_core():
        assert ops.layer_norm(norm, x2).dtype == torch.float32


# ---- range semantics: what a loss scaler relies on ----
def _core_grads(leaves0, kind, H, W, dy):
    from sigma_b200 import ops
    leaves = [t.clone().requires_grad_(True) for t in leaves0]
    with torch.autocast("cuda", dtype=F16), ops.fp16_training_core():
        y = ops.FusedSS2DCore.apply(*leaves, _kid(kind), H, W)
    assert y.dtype == F16
    y.backward(dy)
    return [t.grad for t in leaves]


def test_inf_in_dy_reaches_dxc_and_every_parameter_gradient():
    kind, B, H, W, D, N, R = "cross4", 2, 15, 20, 192, 16, 6
    leaves0, K, Kw, Lseq = _core_leaves(kind, B, H, W, D, N, R, "inf16")
    dy = P.randn(S, "inf16/dy", (B, Lseq, D)).cuda().to(F16)
    g = _core_grads(leaves0, kind, H, W, dy)
    assert all(bool(t.isfinite().all()) for t in g)
    dy[1, Lseq // 3, D // 2] = float("inf")
    g = _core_grads(leaves0, kind, H, W, dy)
    names = ["dxc", "dx_proj_weight", "ddt_projs_weight", "ddt_projs_bias", "dA_logs", "dDs"]
    assert not [n for n, t in zip(names, g) if bool(t.isfinite().all())], "an inf in dy must reach every gradient"
    assert g[0].dtype == F16 and not bool(g[0][1, Lseq // 3].isfinite().all())


def test_dxc_past_the_fp16_range_is_inf_not_clamped():
    """dxc is linear in dy: scaling dy by a power of two scales the fp32 dxc exactly (up to the order of the backward's atomic
    sums), so the elements whose scaled value passes 65504 must come back as ±inf with their sign, the others as the scaled value"""
    kind, B, H, W, D, N, R = "cross4", 2, 15, 20, 192, 16, 6
    leaves0, K, Kw, Lseq = _core_leaves(kind, B, H, W, D, N, R, "ovf16", Ds_scale=16.0)
    dy = P.randn(S, "ovf16/dy", (B, Lseq, D)).cuda().to(F16)
    g0 = _core_grads(leaves0, kind, H, W, dy)[0].float()
    big = float(g0.abs().max())
    s = 2.0 ** math.ceil(math.log2(4 * 65504 / big))                  # the largest elements land near 4 x 65504
    assert float(dy.float().abs().max()) * s < 65504, "dy itself must stay finite for this test"
    gs = _core_grads(leaves0, kind, H, W, (dy.float() * s).to(F16))[0].float()
    want = g0 * s
    over = want.abs() > 65520 * (1 + 2.0 ** -9)                       # past the fp16 range even after a one-ulp difference of g0
    under = want.abs() < 65504 * (1 - 2.0 ** -9)
    assert int(over.sum()) > 0 and int(under.sum()) > 0, (int(over.sum()), int(under.sum()), big, s)
    assert bool(torch.isinf(gs[over]).all()), f"a dxc past ±65504 must be ±inf: {gs[over][~torch.isinf(gs[over])][:8].tolist()}"
    assert bool((torch.sign(gs[over]) == torch.sign(want[over])).all())
    # one fp16 ulp, and the fp32 sums' order (2^-20 of the scale) where they cancel
    err = (gs[under] - want[under]).abs() - (2.0 ** -9 * want[under].abs() + F16_SUB * s + 2.0 ** -20 * big * s)
    assert float(err.max()) <= 0, f"below the range the scaled dxc must be the scaled value: {float(err.max())} beyond, scale {s}"
    record("fp16 train dxc overflow", scale=s, over=int(over.sum()), pos_inf=int((gs == float("inf")).sum()),
           neg_inf=int((gs == -float("inf")).sum()))


class _Wrap(nn.Module):
    """a block under TrainStep's (rgb, modal_x, label) call: label is the weight of the block's output in the loss"""

    def __init__(self, blk):
        super().__init__()
        self.blk = blk

    def forward(self, x, _unused, wgt):
        return (self.blk(x).float() * wgt).mean()


def test_gradscaler_skips_an_overflowing_step_and_applies_a_later_one():
    from sigma_b200 import modules as M, ops, train_util
    x = P.randn(SEED, "gs16/x", (2, 12, 10, 32)).cuda()
    wgt = P.randn(SEED, "gs16/w", (2, 12, 10, 32)).cuda()
    init = 2.0 ** 40                                                   # the scaled loss's gradient overflows fp16 at once
    res = {}
    for on in (False, True):
        torch.manual_seed(SEED)
        model = _Wrap(M.VSSBlock(hidden_dim=32, norm_layer=nn.LayerNorm, mlp_ratio=0.0, d_state=16)).cuda().train()
        opt = torch.optim.AdamW(model.parameters(), lr=1e-3)
        scaler = torch.amp.GradScaler("cuda", init_scale=init, backoff_factor=2.0 ** -24, growth_interval=1000)
        calls, b0 = [], ops._call_ss2d_bwd
        ops._call_ss2d_bwd = lambda args, sv=False, det=False: (calls.append(sv), b0(args, sv, det))[1]
        try:
            step = train_util.TrainStep(model, opt, amp_dtype=F16, fp16_core=on, scaler=scaler)
            before = [p.detach().clone() for p in model.parameters()]
            loss = step(x, None, wgt)
            assert torch.isfinite(loss) and abs(float(loss)) < 1e3         # the returned loss is unscaled
            assert all(torch.equal(a, p.detach()) for a, p in zip(before, model.parameters())), f"on={on}: step 1 must be skipped"
            assert scaler.get_scale() < init
            applied = None
            for i in range(2, 6):
                before = [p.detach().clone() for p in model.parameters()]
                scale = scaler.get_scale()
                step(x, None, wgt)
                if scaler.get_scale() >= scale:                        # no inf found: the step was taken
                    applied = i
                    assert all(p.grad is None or bool(p.grad.isfinite().all()) for p in model.parameters())
                    assert any(not torch.equal(a, p.detach()) for a, p in zip(before, model.parameters()))
                    break
            assert applied is not None, f"on={on}: no step applied after the scale backed off"
        finally:
            ops._call_ss2d_bwd = b0
        assert ops.FP16_TRAINING_CORE is False
        assert calls and all(c == (ops._SAVED_FP16 if on else True) for c in calls), calls
        res[on] = (applied, scaler.get_scale())
    record("fp16 train gradscaler", applied_off=res[False][0], applied_on=res[True][0], scale_off=res[False][1], scale_on=res[True][1])
