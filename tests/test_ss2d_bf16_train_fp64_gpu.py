"""GPU: the bf16 training mode of the fused core (sigma_ss2d_scan_fwd_save_bf16 + sigma_ss2d_scan_bwd_saved_bf16, LayerNormFn on bf16
activations) against fp64.
* The C-ABI pair, element by element inside the per-element bounds of oracle/ss2d_ref64.py run on a given delta'.  Inputs are
  drawn, then xc and dy are rounded to bf16, so the reference sees the exact values.  The kernel's delta' is checked on its own
  against the fp64 softplus inside `fp32 bound + 2^-8·|delta'|`; everything downstream is checked against the reference run on THAT delta' (`delta=`), so a
  rounding tie never turns into a false failure and nothing is loosened.  Kinds cross4 / seq2 at d_state 4 and 16, every padded
  dt_rank Sigma trains with, ragged maps, batch 1 / 2 / 3, L-segments 1, 2, 7, the library's choice, the cap, and a forward cut
  differently from its backward; outputs inside NaN-filled guards; the dt_r and padding columns of dxdbl 0.
* Kind cross (CroMB) the same way, element by element, at CroMB's training shapes at d_state 4 with 1-3 images
  (test_ss2d_bwd_fp64_gpu.CROSS_CASES) and at d_state 16.
* FusedSS2DCore.apply with the switch on under bf16 autocast: bf16 output, bf16 saved xc and delta', the saved bytes, all six
  gradients against the fp64 chain (kind cross chained per modality half); with the switch off, and under the deterministic
  switch, the fp32 entry points run.
* LayerNormFn with bf16 activations against fp64 at every width of ops._LN_WIDTHS."""
import math

import pytest
import torch

import procedural as P
from helpers import guard_ok as _guard_ok, guarded as _guarded, ptr as _p, record, ss2d_kind as _kid, ss2d_params, stream as _stream
from oracle import ss2d_ref64 as R64
from test_ss2d_bwd_fp64_gpu import CROSS_CASES

pytestmark = pytest.mark.gpu
S = 211
BF = torch.bfloat16


def _delta_ref(kind, xdbl, dtw, dtb, N):
    """fp64 softplus(dt_proj) slabs (K, B, Lseq, D) and the bound of a kernel delta' rounded to bf16"""
    ref, bnd = R64.delta_ref64(kind, xdbl, dtw, dtb, N)
    return ref, R64.delta_bound_bf16(ref, bnd)


def _check(tag, name, got, ref, bnd, worst):
    ok = ~ref.isnan()
    assert bool(torch.equal(got.isnan(), ~ok)), f"{tag} {name}: written where the kernel has nothing to write, or NaN"
    frac = R64.bound_fraction(got[ok], ref[ok], bnd[ok])
    worst[name] = max(worst.get(name, 0.0), frac)
    assert frac <= 1.0, f"{tag} {name}: {frac:.3f} of the per-element bound"


def _pair(kind, B, H, W, D, N, R, Cp, args16, fs, bs):
    """run the bf16 pair into guarded buffers; returns (buffers, outputs)"""
    from sigma_b200 import _lib
    L_ = _lib.lib()
    xc, xdbl, dtw, dtb, A, Ds, dy = args16
    K, Lseq = xdbl.shape[2], xc.shape[1]
    Kw = 2 if kind == "cross" else K
    T = L_.sigma_ss2d_scan_hs_bytes(_kid(kind), B, H, W, D, N) // (4 * K * B * D * N)
    bufs, outs = {}, {}
    for name, shape, dt in [("y", (K, B, Lseq, D), BF), ("delta", (K, B, Lseq, D), BF), ("hs", (K, B, T, D, N), torch.float32),
                            ("dxc", (B, Lseq, D), torch.float32), ("ddelta", (K, B, Lseq, D), torch.float32),
                            ("dxdbl", (B, Lseq, K, Cp), torch.float32), ("dA", (Kw * D, N), torch.float32), ("dDs", (Kw * D,), torch.float32),
                            ("ddtb", (Kw, D), torch.float32)]:
        bufs[name], outs[name] = _guarded(shape, dt)
    head = (_kid(kind), _p(xc), _p(xdbl), _p(dtw), _p(dtb), _p(A), _p(Ds))
    fwb = L_.sigma_ss2d_scan_workspace_bytes(_kid(kind), B, H, W, D, N)
    fws = torch.zeros(max(fwb, 4), dtype=torch.uint8, device="cuda")
    _lib.check(L_.sigma_ss2d_scan_fwd_save_bf16(*head, _p(outs["y"]), _p(outs["delta"]), _p(outs["hs"]), B, H, W, D, N, R, Cp, _p(fws), fwb,
                                                fs, _stream()), "sigma_ss2d_scan_fwd_save_bf16")
    wsb = L_.sigma_ss2d_scan_bwd_workspace_bytes(_kid(kind), B, H, W, D, N)
    ws = torch.full((wsb // 4,), float("nan"), device="cuda")
    tail = (_p(outs["dxc"]), _p(outs["ddelta"]), _p(outs["dxdbl"]), _p(outs["dA"]), _p(outs["dDs"]), _p(outs["ddtb"]), B, H, W, D, N, R, Cp,
            _p(ws), wsb)
    _lib.check(L_.sigma_ss2d_scan_bwd_saved_bf16(*head, _p(dy), _p(outs["delta"]), _p(outs["hs"]), *tail, bs, _stream()),
               "sigma_ss2d_scan_bwd_saved_bf16")
    torch.cuda.synchronize()
    return bufs, outs, (head, tail)


def _args16(kind, B, H, W, D, N, R, tag):
    (xc, xdbl, dtw, dtb, A, Ds, dy), Cp = ss2d_params(S, kind, B, H, W, D, N, R, tag)
    return [xc.to(BF), xdbl, dtw, dtb, A, Ds, dy.to(BF)], Cp


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
def test_bf16_pair_matches_fp64(kind, B, H, W, D, N, R):
    tag = f"{kind}/{B}/{H}x{W}/D{D}/N{N}/R{R}"
    args16, Cp = _args16(kind, B, H, W, D, N, R, tag)
    xc, xdbl, dtw, dtb, A, Ds, dy = args16
    dref, dbnd = _delta_ref(kind, xdbl, dtw, dtb, N)
    worst, refs = {}, {}
    for fs, bs in SPLITS:
        t = f"{tag} fwd={fs} bwd={bs}"
        bufs, outs, _ = _pair(kind, B, H, W, D, N, R, Cp, args16, fs, bs)
        _check(t, "delta", outs["delta"], dref, dbnd, worst)
        key = outs["delta"].view(torch.int16).clone()
        hit = [v for kk, v in refs.values() if torch.equal(kk, key)]       # delta' does not depend on the cut: one reference run
        if not hit:
            refs[fs] = (key, R64.ss2d_ref64(kind, xc, xdbl, dtw, dtb, A, Ds, dy.float(), H, W, delta=outs["delta"].double()))
            hit = [refs[fs][1]]
        ref, bnd = hit[0]
        for name in ("y", "hs", "dxc", "ddelta", "dA", "dDs", "ddtb"):
            _check(t, name, outs[name], ref[name], bnd[name], worst)
        dx = outs["dxdbl"]
        _check(t, "dB", dx[..., :N], ref["dB"], bnd["dB"], worst)
        _check(t, "dC", dx[..., N:2 * N], ref["dC"], bnd["dC"], worst)
        assert bool((dx[..., 2 * N:] == 0).all()), f"{t}: the dt_r / padding columns of dxdbl must stay 0"
        for name, buf in bufs.items():
            _guard_ok(buf, f"{t} {name}")
    assert len(refs) == 1, "delta' must not depend on the L-segment cut"
    record(f"ss2d bf16 train fp64 {tag}", **worst)


# Bt = 2·images, H, W, D, N, R: CroMB's training shapes at d_state 4 with 1-3 images, and two d_state 16 cases
CROSS = [(B, H, W, D, N, R) for _, B, H, W, D, N, R in CROSS_CASES] + [(2, 60, 80, 384, 16, 12), (4, 23, 30, 192, 16, 6)]


@pytest.mark.parametrize("B,H,W,D,N,R", CROSS)
def test_bf16_pair_cross(B, H, W, D, N, R):
    """kind cross: delta' against the fp64 softplus; every other output element by element against the reference run on the
    kernel's saved delta' (one reference: delta' must not depend on the L-segment cut)"""
    kind, tag = "cross", f"cross/{B}/{H}x{W}/D{D}/N{N}/R{R}"
    args16, Cp = _args16(kind, B, H, W, D, N, R, tag)
    xc, xdbl, dtw, dtb, A, Ds, dy = args16
    dref, dbnd = _delta_ref(kind, xdbl, dtw, dtb, N)
    worst, key, ref = {}, None, None
    for fs, bs in [(0, 0), (1, 1), (3, 7), (100, 100)]:
        t = f"{tag} fwd={fs} bwd={bs}"
        bufs, outs, _ = _pair(kind, B, H, W, D, N, R, Cp, args16, fs, bs)
        _check(t, "delta", outs["delta"], dref, dbnd, worst)
        if key is None:
            key = outs["delta"].view(torch.int16).clone()
            ref, bnd = R64.ss2d_ref64(kind, xc, xdbl, dtw, dtb, A, Ds, dy.float(), H, W, delta=outs["delta"].double())
        assert torch.equal(outs["delta"].view(torch.int16), key), f"{t}: delta' depends on the L-segment cut"
        for name in ("y", "hs", "dxc", "ddelta", "dA", "dDs", "ddtb"):
            _check(t, name, outs[name], ref[name], bnd[name], worst)
        dx = outs["dxdbl"]
        _check(t, "dB", dx[..., :N], ref["dB"], bnd["dB"], worst)
        _check(t, "dC", dx[..., N:2 * N], ref["dC"], bnd["dC"], worst)
        assert bool((dx[..., 2 * N:] == 0).all()), f"{t}: the dt_r / padding columns of dxdbl must stay 0"
        for name, buf in bufs.items():
            _guard_ok(buf, f"{t} {name}")
    record(f"ss2d bf16 train fp64 {tag}", **worst)


def _bf(t):
    return t.to(BF).float()


@pytest.mark.parametrize("kind,B,H,W,D,N,R", [("cross4", 2, 60, 80, 384, 16, 12), ("seq2", 2, 15, 20, 1536, 4, 48), ("cross4", 2, 30, 40, 768, 4, 24),
                                               ("cross", 4, 30, 40, 768, 4, 24)])
def test_fused_core_autograd_bf16_mode(kind, B, H, W, D, N, R, monkeypatch):
    from sigma_b200 import _lib, fused, ops
    from test_ss2d_bwd_fp64_gpu import core_chain64, core_xdbl
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    K = {"cross4": 4, "seq2": 2, "cross": 1}[kind]            # x_dbl rows per position
    Kw = 2 if kind == "cross" else K                          # parameter sets
    Lseq = H * W * (2 if kind == "seq2" else 1)
    Cp = _lib.lib().sigma_ss2d_padded_cp(N, R)
    tag = f"ag16/{kind}/{B}/{H}x{W}/D{D}/N{N}/R{R}"
    xc0 = P.randn(S, tag + "/xc", (B, Lseq, D)).cuda().to(BF)
    wgt = _bf(P.randn(S, tag + "/w", (B, Lseq, D)).cuda())
    xpw = _bf(P.randn(S, tag + "/xpw", (Kw, R + 2 * N, D), D ** -0.5).cuda())         # exact in the bf16 x_proj GEMM
    dtw = P.rand(S, tag + "/dtw", (Kw, D, R), -R ** -0.5, R ** -0.5).cuda()
    dt = torch.exp(P.rand(S, tag + "/dt", (Kw, D), math.log(1e-3), math.log(0.1)))
    dtb = (dt + torch.log(-torch.expm1(-dt))).cuda()
    Al = (torch.log(torch.arange(1, N + 1, dtype=torch.float32)).repeat(Kw * D, 1) + P.rand(S, tag + "/A", (Kw * D, N), -0.2, 0.2)).cuda()
    Ds = P.randn(S, tag + "/Ds", (Kw * D,), 0.1, 1.0).cuda()

    def run(on):
        leaves = [t.clone().requires_grad_(True) for t in (xc0, xpw, dtw, dtb, Al, Ds)]
        saved, calls = [], []
        s0, b0 = fused.ss2d_scan_save, ops._call_ss2d_bwd
        monkeypatch.setattr(fused, "ss2d_scan_save", lambda kd, xc, *a: (calls.append(("fwd", xc.dtype)), s0(kd, xc, *a))[1])
        monkeypatch.setattr(ops, "_call_ss2d_bwd", lambda args, sv=False, det=False: (calls.append(("bwd", sv, det)), b0(args, sv, det))[1])
        with torch.autograd.graph.saved_tensors_hooks(lambda t: (saved.append(t), t)[1], lambda t: t):
            with torch.autocast("cuda", dtype=BF):
                if on is None:
                    y = ops.FusedSS2DCore.apply(*leaves, _kid(kind), H, W)
                else:
                    with ops.bf16_training_core(on):
                        y = ops.FusedSS2DCore.apply(*leaves, _kid(kind), H, W)
        (y.float() * wgt).sum().backward()
        monkeypatch.setattr(fused, "ss2d_scan_save", s0)
        monkeypatch.setattr(ops, "_call_ss2d_bwd", b0)
        return y.detach(), [t.grad for t in leaves], saved, calls

    y0, g0, _, c0 = run(None)                     # the switch never touched
    y1, g1, saved, c1 = run(True)
    y2, g2, _, c2 = run(False)
    # off: the fp32 entry points, the same output bits, gradients the same up to the order of the backward's atomic sums
    assert c0 == c2 == [("fwd", torch.float32), ("bwd", True, False)] and y0.dtype == torch.float32 and torch.equal(y0, y2)
    for a, b in zip(g0, g2):          # (the bf16 leaf xc gets the fp32 dxc rounded by autograd: a last-bit difference there is one bf16 ulp)
        tol = 2.0 ** -7 if a.dtype == BF else 1e-4
        assert a.dtype == b.dtype and float((a.float() - b.float()).abs().max()) <= tol * float(a.float().abs().max())
    # on: bf16 in, out and saved
    assert c1 == [("fwd", BF), ("bwd", ops._SAVED_BF16, False)] and y1.dtype == BF
    assert g1[0].dtype == BF and all(g.dtype == torch.float32 for g in g1[1:])
    slabs = [t for t in saved if t.shape == (K, B, Lseq, D)]
    assert len(slabs) == 1 and slabs[0].dtype == BF and [t.dtype for t in saved if t.shape == (B, Lseq, D)] == [BF]
    hs_bytes = _lib.lib().sigma_ss2d_scan_hs_bytes(_kid(kind), B, H, W, D, N)
    want = (B * Lseq * D * 2 + K * B * Lseq * D * 2 + B * Lseq * K * Cp * 4 + Kw * Cp * D * 4 + Kw * D * R * 4 + Kw * D * 4
            + Kw * D * N * 4 + Kw * D * 4 + hs_bytes)          # xc, delta' (bf16); x_dbl, xw, W_dt, bias, A, Ds, hs (fp32)
    assert sum(t.numel() * t.element_size() for t in saved) == want
    # the fp64 chain on the delta' the forward saved
    with torch.no_grad():
        xdbl, xw = core_xdbl(kind, xc0, xpw, N, R, Cp)                # the forward's own x_proj GEMM calls
        A = -torch.exp(Al)
        ref, _ = R64.ss2d_ref64(kind, xc0, xdbl, dtw, dtb, A, Ds, wgt, H, W, delta=slabs[0].double())
        want, _ = core_chain64(kind, ref, None, xc0, xdbl, xw, dtw, N, R, Cp)
        want[4] = want[4] * A.double()
        dxc = want[0]
        worst = {}
        # y: K directions each rounded to bf16, added in fp32, rounded once more; dxc: one rounding of the fp32 sum
        yr = ref["y"].sum(0)
        ey = float(((y1.double() - yr).abs() - R64.BF16_RN * (ref["y"].abs().sum(0) + yr.abs())).max()) / float(yr.abs().max())
        assert ey <= 1e-4, f"{tag} y: {ey:.2e} of scale beyond the roundings"
        edx = float(((g1[0].double() - dxc).abs() - R64.BF16_RN * dxc.abs()).max()) / float(dxc.abs().max())
        assert edx <= 1e-4, f"{tag} dxc: {edx:.2e} of scale beyond the rounding"
        for name, g, r in zip(["dx_proj_weight", "ddt_projs_weight", "ddt_projs_bias", "dA_logs", "dDs"], g1[1:], want[1:]):
            err = float((g.double() - r).abs().max()) / float(r.abs().max())
            worst[name] = err
            assert err <= 1e-3, f"{tag} {name}: {err:.2e} of its scale"
    record(f"ss2d bf16 autograd fp64 {tag}", y=ey, dxc=edx, **worst)


def test_deterministic_switch_keeps_the_fp32_det_path():
    from sigma_b200 import fused, ops
    kind, B, H, W, D, N, R = "cross4", 2, 15, 20, 192, 16, 6
    K, Lseq = 4, H * W
    g = torch.Generator().manual_seed(S)
    mk = lambda *s, sc=1.0: (torch.randn(*s, generator=g) * sc).cuda()
    leaves = [mk(B, Lseq, D).to(BF), mk(K, R + 2 * N, D, sc=D ** -0.5), mk(K, D, R, sc=R ** -0.5), mk(K, D) - 4.0,
              torch.log(torch.arange(1, N + 1, dtype=torch.float32)).repeat(K * D, 1).cuda(), mk(K * D)]
    leaves = [t.requires_grad_(True) for t in leaves]
    calls, b0 = [], ops._call_ss2d_bwd
    ops._call_ss2d_bwd = lambda args, sv=False, det=False: (calls.append((sv, det)), b0(args, sv, det))[1]
    torch.use_deterministic_algorithms(True)
    try:
        with torch.autocast("cuda", dtype=BF), ops.bf16_training_core():
            y = ops.FusedSS2DCore.apply(*leaves, _kid(kind), H, W)
        y.float().sum().backward()
    finally:
        torch.use_deterministic_algorithms(False)
        ops._call_ss2d_bwd = b0
    assert y.dtype == torch.float32 and calls == [(True, True)]
    assert all(t.grad is not None and bool(t.grad.isfinite().all()) for t in leaves)


@pytest.mark.parametrize("C", sorted({32, 64, 96, 128, 192, 256, 384, 512, 768, 1024, 1536}))
@pytest.mark.parametrize("rows", [2 * 120 * 160, 2 * 15 * 20, 7])
def test_layernorm_bf16_matches_fp64(C, rows):
    from sigma_b200 import ops
    assert C in ops._LN_WIDTHS
    if rows * C > 2 * 120 * 160 * 384:
        rows = 2 * 30 * 40                                   # Sigma's widths above 384 only occur from stage 2 on
    tag = f"ln16/{rows}x{C}"
    x = (P.randn(S, tag + "/x", (rows, C)) * 1.5 + 0.3).cuda().to(BF).requires_grad_(True)
    w = P.randn(S, tag + "/w", (C,), 0.2, 1.0).cuda().requires_grad_(True)
    b = P.randn(S, tag + "/b", (C,), 0.2).cuda().requires_grad_(True)
    dy = P.randn(S, tag + "/dy", (rows, C)).cuda().to(BF)
    norm = torch.nn.LayerNorm(C).cuda()
    with torch.no_grad():
        norm.weight.copy_(w); norm.bias.copy_(b)
    with torch.autocast("cuda", dtype=BF), ops.bf16_training_core():
        y = ops.layer_norm(norm, x)
    assert y.dtype == BF
    y.backward(dy)
    assert x.grad.dtype == BF and norm.weight.grad.dtype == torch.float32
    xd = x.detach().double().requires_grad_(True)
    wd, bd = w.detach().double().requires_grad_(True), b.detach().double().requires_grad_(True)
    yr = torch.nn.functional.layer_norm(xd, (C,), wd, bd, norm.eps)
    yr.backward(dy.double())
    tol = lambda r: R64.BF16_RN * r.abs() + 1e-5 * (1.0 + r.abs())
    assert bool(((y.double() - yr).abs() <= tol(yr.detach())).all())
    assert bool(((x.grad.double() - xd.grad).abs() <= tol(xd.grad) + 1e-5 * float(xd.grad.abs().max())).all())
    for got, ref in ((norm.weight.grad, wd.grad), (norm.bias.grad, bd.grad)):
        assert float((got.double() - ref).abs().max()) <= 1e-4 * float(ref.abs().max()) + 1e-4 * math.sqrt(rows)
    # with the switch off the same call widens: fp32 out, as before
    x2 = x.detach().clone().requires_grad_(True)
    with torch.autocast("cuda", dtype=BF):
        assert ops.layer_norm(norm, x2).dtype == torch.float32
