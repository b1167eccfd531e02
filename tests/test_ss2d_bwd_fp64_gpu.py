"""GPU: the fused SS2D scan's training pair (sigma_ss2d_scan_fwd_save + sigma_ss2d_scan_bwd_saved) against the fp64 reference of
oracle/ss2d_ref64.py, element by element inside that module's per-element error bounds, at Sigma's training shapes:
* every padded dt_rank Sigma trains with (6 .. 64), so every x_dbl tile size and shared-memory layout runs;
* ragged maps (15 x 20: every column tile has 15 rows; 23 x 30 odd in both), batch 1, 2 and 3;
* kind CROSS (CroMB) at its training shapes (d_state 4): Sigma-tiny / small 120x160/192/R6, 60x80/384/12, 30x40/768/24,
  15x20/1536/48 and Sigma-base 180x240/256/8, 23x30/2048/64, with 1, 2 and 3 images (a batch of 2·images);
* backward L-segments 1, 2, 7, the library's choice and the 64 cap, a count that leaves the shorter walks an empty trailing
  segment, and a training forward cut differently from its backward.  The premises (more than one segment at stage 0 by default,
  the empty segment) are asserted through the backward's planner (sigma_test_ss2d_bwd_plan);
* every output inside NaN-filled memory whose guard elements must stay bit-identical, the dt_r and padding columns of dxdbl 0, and
  NaN-filled workspaces;
* y, delta' and the tile-start states hs of the training forward too.
At the autograd level FusedSS2DCore.apply is checked through all six gradients against the reference chained with the fp64
x_proj / dt_proj algebra of its backward, kind cross included, chained per modality half.  Parameters: dt log-uniform in [1e-3, 0.1]
through the inverse softplus, A = -exp(A_log) around the S4D-real init, Ds near 1; one widened set (dt up to 0.5, |A| up to 4x).
Worst bound fractions go to helpers.record.  Also: the CROSS kernels exist in the library and use no local memory."""
import ctypes
import math
import re
import subprocess

import pytest
import torch

import procedural as P
from helpers import guard_ok as _guard_ok, guarded as _guarded, ptr as _p, record, ss2d_kind as _kid, ss2d_params, \
    stream as _stream
from oracle import ss2d_ref64 as R64

pytestmark = pytest.mark.gpu
S = 97
S_CROSS = 101
OUTS = ("y", "delta", "hs", "dxc", "ddelta", "dA", "dDs", "ddtb")
# d dt_bias sums the per-element bounds of ddelta over all B·L positions; at dt_rank 48 / 64 that leaves its bound at the largest
# element up to ~6x looser than 1e-3 of scale, so it must also meet that max-norm bar
MAXNORM_TOO = ("ddtb",)


def _plan(kind, B, H, W, D, N, nsplit):
    from sigma_b200 import _lib
    out = (ctypes.c_int64 * 4)()
    _lib.check(_lib.lib().sigma_test_ss2d_bwd_plan(_kid(kind), B, H, W, D, N, nsplit, out), "sigma_test_ss2d_bwd_plan")
    return dict(zip(("nsplit", "tiles_per_split", "max_tiles", "min_tiles"), (int(v) for v in out)))


def _params(kind, B, H, W, D, N, R, tag, wide=False):
    return ss2d_params(S, kind, B, H, W, D, N, R, tag, wide)


def _check(tag, name, got, ref, bnd, worst):
    ok = ~ref.isnan()
    assert bool(torch.equal(got.isnan(), ~ok)), f"{tag} {name}: written where the kernel has nothing to write, or NaN"
    frac = R64.bound_fraction(got[ok], ref[ok], bnd[ok])
    worst[name] = max(worst.get(name, 0.0), frac)
    assert frac <= 1.0, f"{tag} {name}: {frac:.3f} of the per-element bound"
    # per element, yet at the largest element no looser than 1e-3 of the tensor's scale (checked once the fractions are logged)
    if name in MAXNORM_TOO:
        err = float((got[ok].double() - ref[ok]).abs().max()) / float(ref[ok].abs().max())
        assert err <= 1e-3, f"{tag} {name}: {err:.2e} of its scale"
    i = int(ref[ok].abs().argmax())
    worst["at_max/" + name] = max(worst.get("at_max/" + name, 0.0), float(bnd[ok][i]) / (1e-3 * float(ref[ok].abs().max())))


def _finish(tag, worst, tight=True):
    record(tag, **worst)
    loose = {k: v for k, v in worst.items() if k.startswith("at_max/") and k[7:] not in MAXNORM_TOO and v > 1.0}
    assert not (tight and loose), f"{tag}: bound at the largest element looser than 1e-3 of scale: {loose}"


def _run_bwd(kind, B, H, W, D, N, R, Cp, args, ref, bnd, tag, worst, fwd_split=0, bwd_split=0):
    """the training forward with fwd_split L-segments followed by the backward with bwd_split (0: the library's choice) that
    consumes its delta' and states"""
    from sigma_b200 import _lib
    L_ = _lib.lib()
    xc, xdbl, dtw, dtb, A, Ds, dy = args
    K, Kw = xdbl.shape[2], dtw.shape[0]
    Lseq = xc.shape[1]
    T = L_.sigma_ss2d_scan_hs_bytes(_kid(kind), B, H, W, D, N) // (4 * K * B * D * N)
    assert T == ref["hs"].shape[2]
    bufs, outs = {}, {}
    for name, shape in [("delta", (K, B, Lseq, D)), ("dxc", (B, Lseq, D)), ("ddelta", (K, B, Lseq, D)), ("dxdbl", (B, Lseq, K, Cp)),
                        ("dA", (Kw * D, N)), ("dDs", (Kw * D,)), ("ddtb", (Kw, D)), ("y", (K, B, Lseq, D)), ("hs", (K, B, T, D, N))]:
        bufs[name], outs[name] = _guarded(shape)
    wsb = L_.sigma_ss2d_scan_bwd_workspace_bytes(_kid(kind), B, H, W, D, N)
    assert wsb > 0
    ws = torch.full((wsb // 4,), float("nan"), device="cuda")
    tail = (_p(outs["dxc"]), _p(outs["ddelta"]), _p(outs["dxdbl"]), _p(outs["dA"]), _p(outs["dDs"]), _p(outs["ddtb"]), B, H, W, D, N, R, Cp,
            _p(ws), wsb)
    head = (_kid(kind), _p(xc), _p(xdbl), _p(dtw), _p(dtb), _p(A), _p(Ds))
    fwb = L_.sigma_ss2d_scan_workspace_bytes(_kid(kind), B, H, W, D, N)
    fws = torch.full((max(fwb, 4) // 4,), float("nan"), device="cuda")
    _lib.check(L_.sigma_ss2d_scan_fwd_save(*head, _p(outs["y"]), _p(outs["delta"]), _p(outs["hs"]), B, H, W, D, N, R, Cp, _p(fws), fwb,
                                           fwd_split, _stream()), "sigma_ss2d_scan_fwd_save")
    _lib.check(L_.sigma_ss2d_scan_bwd_saved(*head, _p(dy), _p(outs["delta"]), _p(outs["hs"]), *tail, bwd_split, _stream()),
               "sigma_ss2d_scan_bwd_saved")
    torch.cuda.synchronize()
    for name in OUTS:
        _check(tag, name, outs[name], ref[name], bnd[name], worst)
    dx = outs["dxdbl"]
    _check(tag, "dB", dx[..., :N], ref["dB"], bnd["dB"], worst)
    _check(tag, "dC", dx[..., N:2 * N], ref["dC"], bnd["dC"], worst)
    assert bool((dx[..., 2 * N:] == 0).all()), f"{tag}: the dt_r / padding columns of dxdbl must stay 0"
    for name, buf in bufs.items():
        _guard_ok(buf, f"{tag} {name}")


# kind, B, H, W, D, N, R
CASES = [
    ("cross4", 2, 120, 160, 192, 16, 6), ("cross4", 2, 60, 80, 384, 16, 12), ("cross4", 2, 30, 40, 768, 16, 24),
    ("cross4", 2, 15, 20, 1536, 16, 48), ("cross4", 2, 45, 60, 1024, 16, 32), ("cross4", 2, 23, 30, 2048, 16, 64),   # SS2D
    ("seq2", 2, 120, 160, 192, 4, 6), ("seq2", 2, 15, 20, 1536, 4, 48), ("seq2", 2, 23, 30, 2048, 4, 64),              # ConMB
    ("cross4", 2, 120, 160, 192, 4, 6), ("cross4", 2, 60, 80, 384, 4, 12), ("cross4", 2, 30, 40, 768, 4, 24),          # decoder SS2D
    ("cross4", 1, 30, 40, 768, 16, 24), ("cross4", 3, 30, 40, 768, 16, 24),
]
# CroMB (kind cross, d_state 4, B = 2·images): H, W, d_inner, dt_rank, images
CROSS_CASES = [("cross", 2 * im, H, W, D, 4, R) for H, W, D, R, im in [
    (120, 160, 192, 6, 2), (60, 80, 384, 12, 2), (30, 40, 768, 24, 2), (15, 20, 1536, 48, 2), (180, 240, 256, 8, 1),
    (23, 30, 2048, 64, 2), (30, 40, 768, 24, 1), (30, 40, 768, 24, 3), (15, 20, 1536, 48, 3), (60, 80, 384, 12, 1)]]


@pytest.mark.parametrize("kind,B,H,W,D,N,R", CASES + CROSS_CASES)
def test_fused_bwd_matches_fp64(kind, B, H, W, D, N, R):
    if kind == "cross":
        seed, tag = S_CROSS, f"cross/{B // 2}/{H}x{W}/D{D}/R{R}"
    else:
        seed, tag = S, f"{kind}/{B}/{H}x{W}/D{D}/N{N}/R{R}"
    args, Cp = ss2d_params(seed, kind, B, H, W, D, N, R, tag)
    ref, bnd = R64.ss2d_ref64(kind, *args, H, W)
    worst = {}
    auto = _plan(kind, B, H, W, D, N, 0)
    if (H, W) == (120, 160):
        assert auto["nsplit"] > 1, auto                                  # stage 0 runs L-segments by default
    splits = [1, 2, 7, 0, 100]
    cap = _plan(kind, B, H, W, D, N, 100)
    assert cap["tiles_per_split"] == -(-cap["max_tiles"] // 64) and cap["nsplit"] <= 64     # 100 is capped at 64 segments
    if (H, W) == (15, 20):
        pl = _plan(kind, B, H, W, D, N, 20)
        if pl["min_tiles"] < pl["max_tiles"]:
            assert (pl["nsplit"] - 1) * pl["tiles_per_split"] >= pl["min_tiles"]   # the shorter walks end in an empty segment
            splits.append(20)
    for fs, bs in [(0, sp) for sp in splits] + [(3, 7), (1, 2)]:
        _run_bwd(kind, B, H, W, D, N, R, Cp, args, ref, bnd, f"{tag} fwd={fs} bwd={bs}", worst, fs, bs)
    # CroMB's bound at the largest element is recorded; only the other kinds are held to 1e-3 of scale there
    _finish(f"ss2d bwd fp64 {tag}", worst, tight=kind != "cross")


@pytest.mark.parametrize("kind,B,H,W,D,N,R", [("cross4", 2, 15, 20, 1536, 16, 48), ("seq2", 2, 60, 80, 384, 4, 12),
                                               ("cross4", 1, 120, 160, 192, 16, 6)])
def test_fused_bwd_matches_fp64_widened(kind, B, H, W, D, N, R):
    """larger steps and decays: dt up to 0.5, |A| up to 4x the S4D-real init"""
    tag = f"wide/{kind}/{B}/{H}x{W}/D{D}/N{N}/R{R}"
    args, Cp = _params(kind, B, H, W, D, N, R, tag, wide=True)
    ref, bnd = R64.ss2d_ref64(kind, *args, H, W)
    worst = {}
    for sp in [1, 0, 7]:
        _run_bwd(kind, B, H, W, D, N, R, Cp, args, ref, bnd, f"{tag} bwd={sp}", worst, bwd_split=sp)
    _finish(f"ss2d bwd fp64 {tag}", worst)


def _mm_bound(a, ea, b, n):
    """bound of the fp32 product a @ b (b exact) given a's element bound: propagated error plus accumulation"""
    return ea @ b.abs() + R64._gt(n) * (a.abs() @ b.abs())


def _mm_bound_positions(aT, eaT, b):
    """the same for a contraction over the B·L positions (aT (M, B·L), b (B·L, P)): the propagated first-order errors of
    16-position chunks are combined as independent (oracle.ss2d_ref64.tile_rss); the fp32 accumulation's partial sums are bounded
    by |result| + sqrt(sum of squared terms) (a drift plus a random walk), n roundings of them by LAMBDA·sqrt(n)·u of that"""
    M, n = aT.shape
    pad = (-n) % 16
    ea = torch.nn.functional.pad(eaT, (0, pad)).view(M, -1, 16).transpose(0, 1)          # (chunks, M, 16)
    bb = torch.nn.functional.pad(b.abs(), (0, 0, 0, pad)).view(-1, 16, b.shape[1])        # (chunks, 16, P)
    part = torch.bmm(ea, bb)                                                              # (chunks, M, P)
    rss = R64.LAMBDA * (part * part).sum(0).sqrt()
    return rss + R64.LAMBDA * R64.U * math.sqrt(n) * ((aT @ b).abs() + ((aT * aT) @ (b * b)).sqrt())


def core_chain64(kind, ref, bnd, xc, xdbl, xw, dtw, N, R, Cp):
    """FusedSS2DCore's backward after the scan, in fp64: the six gradients (dxc, dx_proj_weight, ddt_projs_weight, ddt_projs_bias,
    the scan's dA (the caller applies the dA·A step of dA_logs), dDs) from the scan reference `ref` (oracle/ss2d_ref64's layout),
    and with `bnd` their per-element bounds (else None).  dxdbl = [dB | dC | ddelta · W_dt | 0] per direction (cross: per modality
    half, its own W_dt), then dxc += dxdbl · xw and d xw = dxdbl^T · xc per x_proj GEMM (cross: one per half, its own xw rows)."""
    d = lambda t: t.double()
    B, Lseq, K, _ = xdbl.shape
    D = xc.shape[-1]
    BL = B * Lseq
    cross = kind == "cross"
    Kw = 2 if cross else K
    n = BL // 2
    # (positions, x_dbl row, weight set) of each dt_proj step; (positions, xw rows) of each x_proj GEMM
    steps = [(slice(m * n, (m + 1) * n), 0, m) for m in range(2)] if cross else [(slice(None), k, k) for k in range(K)]
    gemms = [(slice(m * n, (m + 1) * n), slice(m * Cp, (m + 1) * Cp)) for m in range(2)] if cross else [(slice(None), slice(None))]
    withb = bnd is not None
    z = lambda *s: torch.zeros(s, dtype=torch.float64, device=xc.device)
    dxd, edxd = z(BL, K, Cp), z(BL, K, Cp)
    dxd[..., :N], dxd[..., N:2 * N] = ref["dB"].reshape(BL, K, N), ref["dC"].reshape(BL, K, N)
    if withb:
        edxd[..., :N], edxd[..., N:2 * N] = bnd["dB"].reshape(BL, K, N), bnd["dC"].reshape(BL, K, N)
    dW, edW = z(Kw, D, R), z(Kw, D, R)
    xd = d(xdbl).view(BL, K, Cp)
    for rs, k, w in steps:
        dd = ref["ddelta"][k].reshape(BL, D)[rs]
        dtr = xd[rs, k, 2 * N:2 * N + R]
        dxd[rs, k, 2 * N:2 * N + R] = dd @ d(dtw[w])
        dW[w] = dd.t() @ dtr
        if withb:
            edd = bnd["ddelta"][k].reshape(BL, D)[rs]
            edxd[rs, k, 2 * N:2 * N + R] = _mm_bound(dd, edd, d(dtw[w]), D)
            edW[w] = _mm_bound_positions(dd.t(), edd.t(), dtr)
    d2, e2 = dxd.view(BL, K * Cp), edxd.view(BL, K * Cp)
    x2 = d(xc).reshape(BL, D)
    dxc = ref["dxc"].reshape(BL, D).clone()
    edxc = bnd["dxc"].reshape(BL, D).clone() if withb else None
    dxw, edxw = z(Kw * Cp, D), z(Kw * Cp, D)
    for rs, cs in gemms:
        a, w = d2[rs], d(xw[cs])
        dxc[rs] += a @ w
        dxw[cs] = a.t() @ x2[rs]
        if withb:
            edxc[rs] += _mm_bound(a, e2[rs], w, a.shape[1])
            edxw[cs] = _mm_bound_positions(a.t(), e2[rs].t(), x2[rs])
    order = lambda t: torch.cat([t[:, 2 * N:2 * N + R], t[:, 0:N], t[:, N:2 * N]], dim=1)
    want = [dxc.view(B, Lseq, D), order(dxw.view(Kw, Cp, D)), dW, ref["ddtb"], ref["dA"], ref["dDs"]]
    if not withb:
        return want, None
    edxc += R64.U * dxc.abs()
    return want, [edxc.view(B, Lseq, D), order(edxw.view(Kw, Cp, D)), edW, bnd["ddtb"], bnd["dA"], bnd["dDs"]]


def core_inputs(kind, B, H, W, D, N, R, tag):
    """leaves of FusedSS2DCore (xc, x_proj_weight, dt_projs_weight, dt_projs_bias, A_logs, Ds) and the output weight, fp32: one
    parameter set per direction, or per modality for cross"""
    K = {"cross4": 4, "seq2": 2, "cross": 2}[kind]
    Lseq = H * W * (2 if kind == "seq2" else 1)
    xc0 = P.randn(S, tag + "/xc", (B, Lseq, D)).cuda()
    wgt = P.randn(S, tag + "/w", (B, Lseq, D)).cuda()
    xpw = P.randn(S, tag + "/xpw", (K, R + 2 * N, D), D ** -0.5).cuda()
    dtw = P.rand(S, tag + "/dtw", (K, D, R), -R ** -0.5, R ** -0.5).cuda()
    dt = torch.exp(P.rand(S, tag + "/dt", (K, D), math.log(1e-3), math.log(0.1)))
    dtb = (dt + torch.log(-torch.expm1(-dt))).cuda()
    Al = (torch.log(torch.arange(1, N + 1, dtype=torch.float32)).repeat(K * D, 1) + P.rand(S, tag + "/A", (K * D, N), -0.2, 0.2)).cuda()
    Ds = P.randn(S, tag + "/Ds", (K * D,), 0.1, 1.0).cuda()
    return [xc0, xpw, dtw, dtb, Al, Ds], wgt


def core_xdbl(kind, xc, xpw, N, R, Cp):
    """x_dbl as FusedSS2DCore's forward computes it (the same GEMM calls): (B, Lseq, K, Cp), and the packed x_proj rows xw"""
    from sigma_b200 import fused
    B, Lseq, D = xc.shape
    xw = torch.cat([fused._pack_xproj(xpw[k], N, R, Cp) for k in range(xpw.shape[0])], dim=0).contiguous()
    if kind != "cross":
        return fused.linear(xc.reshape(B * Lseq, D), xw, kind="x_proj").view(B, Lseq, -1, Cp), xw
    n = B // 2 * Lseq
    xdbl = torch.empty((B * Lseq, Cp), dtype=torch.float32, device=xc.device)
    for m in range(2):
        fused.linear(xc.reshape(B * Lseq, D)[m * n:(m + 1) * n], xw[m * Cp:(m + 1) * Cp], out=xdbl[m * n:(m + 1) * n], kind="x_proj")
    return xdbl.view(B, Lseq, 1, Cp), xw


@pytest.mark.parametrize("kind,B,H,W,D,N,R", [("cross4", 2, 120, 160, 192, 16, 6), ("seq2", 2, 15, 20, 1536, 4, 48),
                                               ("cross4", 2, 15, 20, 1536, 16, 48), ("cross", 4, 30, 40, 768, 4, 24)])
def test_fused_core_autograd_matches_fp64(kind, B, H, W, D, N, R, monkeypatch):
    """FusedSS2DCore.apply: y and all six gradients against the reference chained with the fp64 x_proj / dt_proj algebra.  The
    reference takes the very x_dbl the forward computed (the same deterministic GEMM calls), so only the scan and the backward's
    own fp32 GEMMs are under test; this pins the [dt | B | C] row order and the dA·A step at a real shape.  Kind cross (CroMB, 2
    images): the x_proj GEMMs, dt_proj steps and weight gradients per modality half, dC credited to the other half's rows."""
    from sigma_b200 import _lib, ops
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    K = {"cross4": 4, "seq2": 2, "cross": 1}[kind]
    Cp = _lib.lib().sigma_ss2d_padded_cp(N, R)
    tag = f"ag/{kind}/{B}/{H}x{W}/D{D}/N{N}/R{R}"
    (xc0, xpw, dtw, dtb, Al, Ds), wgt = core_inputs(kind, B, H, W, D, N, R, tag)
    leaves = [t.clone().requires_grad_(True) for t in (xc0, xpw, dtw, dtb, Al, Ds)]
    y = ops.FusedSS2DCore.apply(*leaves, _kid(kind), H, W)
    (y * wgt).sum().backward()
    got = [t.grad for t in leaves]
    with torch.no_grad():
        xdbl, xw = core_xdbl(kind, xc0, xpw, N, R, Cp)
        A = -torch.exp(Al)
        ref, bnd = R64.ss2d_ref64(kind, xc0, xdbl, dtw, dtb, A, Ds, wgt, H, W)
        worst = {}
        yr = ref["y"].sum(0)
        yb = bnd["y"].sum(0) + (K if K > 1 else 0) * R64.U * ref["y"].abs().sum(0)     # the directions' fp32 sum
        _check(tag, "y", y.detach(), yr, yb, worst)
        want, bounds = core_chain64(kind, ref, bnd, xc0, xdbl, xw, dtw, N, R, Cp)
        A64 = A.double()
        want[4], bounds[4] = want[4] * A64, bounds[4] * A64.abs() + 2 * R64.U * (want[4] * A64).abs()
        for name, g, r, b in zip(["dxc", "dx_proj_weight", "ddt_projs_weight", "ddt_projs_bias", "dA_logs", "dDs"], got, want, bounds):
            _check(tag, name, g, r, b, worst)
            # the weight gradients contract the scan's per-element bounds over all B·L positions, which leaves their propagated
            # bound looser than 1e-3 of scale at the largest element: there the max-norm bar holds as well
            err = float((g.double() - r).abs().max()) / float(r.abs().max())
            assert err <= 1e-3, f"{tag} {name}: {err:.2e} of its scale"
    _finish(f"ss2d autograd fp64 {tag}", worst, tight=False)


def test_cross_instances_exist_without_local_memory():
    from sigma_b200 import build
    out = subprocess.run(["cuobjdump", "-res-usage", build.LIB], capture_output=True, text=True, check=True).stdout
    use = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out))
    names = [f"_ZN5sigma21ss2d_bwd_cross_kernelILi{n}ELi{m}EEEvNS_13Ss2dBwdParamsE" for n in (4, 16) for m in (0, 1, 2)]
    for n in names:
        assert n in use, f"missing CROSS kernel {n}"
        assert re.search(r"\bSTACK:0\b", use[n]) and re.search(r"\bLOCAL:0\b", use[n]), f"{n}: {use[n]}"
    assert not [n for n in use if "cross" in n and "_det" in n]
    # the backward recomputes no states (the training forward saved them): every kernel of its parameter block is a reverse sweep
    assert all(n.startswith("_ZN5sigma") and "ss2d_bwd" in n for n in use if "Ss2dBwdParams" in n)
