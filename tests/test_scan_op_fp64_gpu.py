"""GPU: the op-level selective scan (sigma_scan_fwd_split, sigma_scan_bwd_split, sigma_scan_bwd_det: the drop-in
selective_scan_cuda_core.fwd / bwd) against the fp64 reference of oracle/scan_ref64.py, element by element inside that module's
per-element error bounds, at the calls Sigma trains with:
* CroMB (its backward runs through this op at every stage): (B, 192·2^i, L) for L = 19200, 4800, 1200, 300, d_state 4, and at
  Sigma-base's width, its 720 x 960 stage 0 (L = 43200, forward) and its 23 x 30 stage (L = 690: fp32 rows not 16-byte aligned,
  the generic kernels); the drop-in graph's SS2D (4 groups, d_state 16) and ConMB (2 groups, L = 38400) calls;
* forward L-segments: the library's choice, 1, 2, 7, 64 and 100 (capped at 64), and a count whose segment boundaries fall inside
  a 2048-position chunk of `x`; backward: the library's choice, 1, 3, 64; the deterministic build at its choice and a forced count;
* fp16 and bf16 at CroMB stages 0 and 3 (stage 3 takes the widened route), at L = 690 (generic) and at the SS2D stage-0 call;
  SIGMA_OP_GENERIC=1 on a TMA-eligible shape; a forward on padded-row views of u / delta / out, 16-byte aligned and not;
* Sigma's parameters (dt log-uniform in [1e-3, 0.1] through the inverse softplus, A around S4D-real, D near 1), a widened set,
  the reference test's distribution at one shape, and one call with softplus, D and delta_bias off.
The premises (routes, more than one segment by default at stage 0, the cap, a segment boundary inside a chunk) are asserted
through the library's planner (sigma_test_scan_plan).  Every output sits in NaN-filled memory whose guard elements must stay
untouched, every element of `x` must be written, and the workspace is NaN-filled scratch.  Worst fractions go to helpers.record."""
import ctypes

import pytest
import torch

from helpers import guard_ok, guarded, op_scan_params, ptr as _p, record, scan_plan, stream as _stream
from oracle import scan_ref64 as R

pytestmark = pytest.mark.gpu
S = 101
_DT = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
SUMMED = ("dA", "dD", "ddelta_bias")         # sums over batch·L: also held to a max-norm bar of 1e-3 of their scale


def _check(tag, name, got, ref, bnd, worst):
    got = got.double()
    assert not bool(got.isnan().any()), f"{tag} {name}: elements left unwritten (NaN)"
    frac = R.bound_fraction(got, ref, bnd)
    worst[name] = max(worst.get(name, 0.0), frac)
    assert frac <= 1.0, f"{tag} {name}: {frac:.3f} of the per-element bound"
    scale = float(ref.abs().max())
    if name in SUMMED:
        err = float((got - ref).abs().max()) / scale
        assert err <= 1e-3, f"{tag} {name}: {err:.2e} of its scale"
    i = int(ref.abs().argmax())
    worst["at_max/" + name] = max(worst.get("at_max/" + name, 0.0), float(bnd.reshape(-1)[i]) / (1e-3 * scale))


def _finish(tag, worst, tight=True):
    """the bound at each tensor's largest element no looser than 1e-3 of its scale; the batch·L sums, whose bounds add up the
    per-position ones, meet the max-norm bar of _check instead (as dt_bias's gradient in test_ss2d_bwd_fp64_gpu.py)"""
    record(tag, **worst)
    loose = {k: v for k, v in worst.items() if k.startswith("at_max/") and k[7:] not in SUMMED and v > 1.0}
    assert not (tight and loose), f"{tag}: bound at the largest element looser than 1e-3 of scale: {loose}"


def _strides(u, delta, A, B, C, out):
    from sigma_b200 import _lib
    return _lib.ScanStrides(u.stride(0), u.stride(1), delta.stride(0), delta.stride(1), A.stride(0), A.stride(1), B.stride(0),
                            B.stride(1), B.stride(2), C.stride(0), C.stride(1), C.stride(2), out.stride(0), out.stride(1))


def _fwd(args, softplus, ref, bnd, tag, worst, nsplit, u=None, delta=None):
    """sigma_scan_fwd_split into guarded out / x; u / delta / out may be padded-row views (u, delta given: out padded alike)"""
    from sigma_b200 import _lib
    L_ = _lib.lib()
    u0, delta0, A, B, C, D, bias, _ = args
    bt, dim, L = u0.shape
    G, N = B.shape[1], B.shape[2]
    dt = u0.dtype
    if u is None:
        u, delta = u0, delta0
        obuf, out = guarded((bt, dim, L), dt)
    else:
        Lp = u.stride(1)
        obuf, outp = guarded((bt, dim, Lp), dt)
        out = outp[:, :, :L]
    xbuf, x = guarded((bt, dim, -(-L // R.CHUNK), 2 * N))
    wsb = L_.sigma_scan_fwd_workspace_bytes(bt, dim, L, N, G, _DT[dt])
    ws = torch.full((wsb // 4 + 1,), float("nan"), device="cuda")
    st = _strides(u, delta, A, B, C, out)
    _lib.check(L_.sigma_scan_fwd_split(_p(u), _p(delta), _p(A), _p(B), _p(C), _p(D), _p(bias), _p(out), _p(x), bt, dim, L, N, G,
                                       _DT[dt], int(softplus), ctypes.byref(st), _p(ws), wsb, nsplit, _stream()), "sigma_scan_fwd_split")
    torch.cuda.synchronize()
    _check(tag, "out", out, ref["out"], bnd["out"], worst)
    _check(tag, "x", x, ref["x"], bnd["x"], worst)
    guard_ok(obuf if u is u0 else obuf, f"{tag} out")
    guard_ok(xbuf, f"{tag} x")
    if u is not u0:
        assert bool(outp[:, :, L:].isnan().all()), f"{tag}: the padding of out's rows was written"


def _bwd(args, softplus, ref, bnd, tag, worst, nsplit, det=False):
    from sigma_b200 import _lib
    L_ = _lib.lib()
    u, delta, A, B, C, D, bias, dout = args
    bt, dim, L = u.shape
    G, N = B.shape[1], B.shape[2]
    dt = u.dtype
    shapes = dict(du=((bt, dim, L), dt), ddelta=((bt, dim, L), dt), dA=((dim, N), torch.float32), dB=((bt, G, N, L), torch.float32),
                  dC=((bt, G, N, L), torch.float32))
    if D is not None:
        shapes["dD"] = ((dim,), torch.float32)
    if bias is not None:
        shapes["ddelta_bias"] = ((dim,), torch.float32)
    bufs, outs = {}, {}
    for k, (s, t) in shapes.items():
        bufs[k], outs[k] = guarded(s, t)
    wsb = (L_.sigma_scan_bwd_det_workspace_bytes if det else L_.sigma_scan_bwd_workspace_bytes)(bt, dim, L, N, G, _DT[dt])
    ws = torch.full((wsb // 4 + 1,), float("nan"), device="cuda")
    o = lambda k: _p(outs.get(k))
    fn = L_.sigma_scan_bwd_det if det else L_.sigma_scan_bwd_split
    _lib.check(fn(_p(u), _p(delta), _p(A), _p(B), _p(C), _p(D), _p(bias), _p(dout), o("du"), o("ddelta"), o("dA"), o("dB"), o("dC"),
                  o("dD"), o("ddelta_bias"), bt, dim, L, N, G, _DT[dt], int(softplus), _p(ws), wsb, nsplit, _stream()),
               "sigma_scan_bwd")
    torch.cuda.synchronize()
    for k in shapes:
        _check(tag, k, outs[k], ref[k], bnd[k], worst)
        guard_ok(bufs[k], f"{tag} {k}")


def _case(shape, tag, dist="sigma", dtype=torch.float32, softplus=True, has_D=True, has_bias=True):
    bt, dim, L, N, G = shape
    args = [None if t is None else t.cuda() for t in op_scan_params(S, bt, dim, L, N, G, tag, dist, dtype, has_D, has_bias, softplus)]
    ref, bnd = R.scan_ref64(*args[:7], softplus, args[7])
    return args, ref, bnd


def _pos_per_tile(plan, dtype):
    return 16 if plan["route"] == "widened" or (plan["route"] == "tma" and dtype == torch.float32) else 32


# (batch, dim, L, d_state, groups)
CASES = [
    (2, 192, 19200, 4, 1), (2, 384, 4800, 4, 1), (2, 768, 1200, 4, 1), (2, 1536, 300, 4, 1),      # CroMB, Sigma-tiny/small
    (1, 768, 1200, 4, 1), (3, 768, 1200, 4, 1),
    (1, 256, 19200, 4, 1), (1, 2048, 690, 4, 1),                                                 # CroMB at Sigma-base's width
    (2, 768, 19200, 16, 4), (2, 6144, 300, 16, 4),                                               # drop-in SS2D
    (2, 384, 38400, 4, 2),                                                                       # drop-in ConMB
]


@pytest.mark.parametrize("shape", CASES)
def test_op_scan_matches_fp64(shape):
    bt, dim, L, N, G = shape
    tag = "op/" + "/".join(map(str, shape))
    args, ref, bnd = _case(shape, tag)
    worst = {}
    auto = scan_plan("fwd", *shape)
    if L == 690:
        assert auto["route"] == "generic" and scan_plan("bwd", *shape)["route"] == "generic", auto
    else:
        assert auto["route"] == "tma", auto
    if L == 19200:
        assert auto["nsplit"] > 1 and scan_plan("bwd", *shape)["nsplit"] > 1                    # stage 0 runs L-segments by default
    cap = scan_plan("fwd", *shape, nsplit=100)
    assert cap["nsplit"] <= 64 and cap["tiles_per_split"] == -(-cap["ntiles"] // 64), cap      # 100 is capped at 64 segments
    splits = [0, 1, 2, 7, 64, 100]
    if L > R.CHUNK:                                   # a segment boundary inside a chunk of x: that chunk's state is the APPLY pass's
        p7 = scan_plan("fwd", *shape, nsplit=7)
        assert p7["nsplit"] == 7 and (p7["tiles_per_split"] * _pos_per_tile(p7, torch.float32)) % R.CHUNK != 0, p7
    for sp in splits:
        _fwd(args, True, ref, bnd, f"{tag} fwd split={sp}", worst, sp)
    for sp in [0, 1, 3, 64]:
        _bwd(args, True, ref, bnd, f"{tag} bwd split={sp}", worst, sp)
    for sp in [0, 5]:
        _bwd(args, True, ref, bnd, f"{tag} bwd det split={sp}", worst, sp, det=True)
    _finish(f"scan op fp64 {tag}", worst)


def test_op_scan_forward_sigma_base_stage0():
    """Sigma-base 720 x 960 stage 0, CroMB's forward: L = 43200 (22 chunks of x)"""
    shape = (1, 256, 43200, 4, 1)
    tag = "op/" + "/".join(map(str, shape))
    bt, dim, L, N, G = shape
    args = [None if t is None else t.cuda() for t in op_scan_params(S, bt, dim, L, N, G, tag)]
    ref, bnd = R.scan_ref64(*args[:7], True)
    worst = {}
    assert scan_plan("fwd", *shape)["nsplit"] > 1
    for sp in [0, 1, 64]:
        _fwd(args, True, ref, bnd, f"{tag} fwd split={sp}", worst, sp)
    _finish(f"scan op fp64 {tag}", worst)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("shape,route", [((2, 192, 19200, 4, 1), "tma"), ((2, 1536, 300, 4, 1), "widened"),
                                         ((1, 2048, 690, 4, 1), "generic"), ((2, 768, 19200, 16, 4), "tma")])
def test_op_scan_16bit_matches_fp64(shape, route, dtype):
    tag = f"op16/{str(dtype)[6:]}/" + "/".join(map(str, shape))
    for sweep in ("fwd", "bwd", "bwd_det"):
        assert scan_plan(sweep, *shape, dtype)["route"] == route
    args, ref, bnd = _case(shape, tag, dtype=dtype)
    worst = {}
    for sp in [0, 1, 7]:
        _fwd(args, True, ref, bnd, f"{tag} fwd split={sp}", worst, sp)
    p7 = scan_plan("fwd", *shape, dtype, nsplit=7)
    if route != "generic" or shape[2] > 32 * 7:
        assert p7["nsplit"] > 1, p7                  # the 16-bit forward really runs its summary / apply instances
    _bwd(args, True, ref, bnd, f"{tag} bwd", worst, 0)
    _bwd(args, True, ref, bnd, f"{tag} bwd det", worst, 0, det=True)
    _finish(f"scan op fp64 {tag}", worst, tight=dtype != torch.bfloat16)   # bf16's 2^-8 store rounding exceeds 1e-3 of scale


@pytest.mark.parametrize("shape,dist,opts", [
    ((2, 1536, 300, 4, 1), "wide", {}), ((2, 192, 19200, 4, 1), "wide", {}), ((2, 768, 1200, 16, 4), "wide", {}),
    ((2, 384, 4800, 4, 1), "ref", {}),
    ((2, 768, 1200, 4, 1), "sigma", dict(softplus=False, has_D=False, has_bias=False))])
def test_op_scan_other_parameters_match_fp64(shape, dist, opts):
    """larger steps and decays (dt up to 0.5, |A| up to 4x), the reference test's distribution (near-zero A), and a call with
    softplus, D and delta_bias off"""
    tag = f"op/{dist}/{opts}/" + "/".join(map(str, shape))
    args, ref, bnd = _case(shape, tag, dist, **opts)
    sp = opts.get("softplus", True)
    worst = {}
    for n in [0, 1, 7]:
        _fwd(args, sp, ref, bnd, f"{tag} fwd split={n}", worst, n)
    for n in [0, 3]:
        _bwd(args, sp, ref, bnd, f"{tag} bwd split={n}", worst, n)
    _bwd(args, sp, ref, bnd, f"{tag} bwd det", worst, 0, det=True)
    _finish(f"scan op fp64 {tag}", worst)


def test_op_scan_generic_kernels_on_a_tma_shape(monkeypatch):
    """SIGMA_OP_GENERIC=1: the generic forward (1, 7 and 100 segments, capped at 64) and backward on a TMA-eligible call"""
    shape = (2, 768, 1200, 4, 1)
    tag = "op/generic/" + "/".join(map(str, shape))
    args, ref, bnd = _case(shape, tag)
    monkeypatch.setenv("SIGMA_OP_GENERIC", "1")
    assert scan_plan("fwd", *shape)["route"] == "generic" and scan_plan("bwd", *shape)["route"] == "generic"
    cap = scan_plan("fwd", *shape, nsplit=100)
    assert cap["nsplit"] <= 64 and cap["tiles_per_split"] == -(-cap["ntiles"] // 64), cap
    worst = {}
    for sp in [1, 7, 100]:
        _fwd(args, True, ref, bnd, f"{tag} fwd split={sp}", worst, sp)
    _bwd(args, True, ref, bnd, f"{tag} bwd", worst, 0)
    _bwd(args, True, ref, bnd, f"{tag} bwd det", worst, 0, det=True)
    _finish(f"scan op fp64 {tag}", worst)


@pytest.mark.parametrize("pad", [4, 1])
def test_op_scan_forward_on_padded_rows(pad):
    """u / delta / out as views of rows padded by `pad` positions: 16-byte aligned rows (pad 4) stay on the TMA kernels, the
    others (pad 1) take the generic ones; the padding of out's rows must stay untouched"""
    shape = (2, 768, 1200, 4, 1)
    bt, dim, L, N, G = shape
    tag = f"op/pad{pad}/" + "/".join(map(str, shape))
    args, ref, bnd = _case(shape, tag)
    views = []
    for t in args[:2]:
        full = torch.zeros(bt, dim, L + pad, device="cuda")
        full[:, :, :L] = t
        views.append(full[:, :, :L])
    worst = {}
    for sp in [0, 1, 7]:
        _fwd(args, True, ref, bnd, f"{tag} fwd split={sp}", worst, sp, u=views[0], delta=views[1])
    _finish(f"scan op fp64 {tag}", worst)
