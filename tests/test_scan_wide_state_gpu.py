"""GPU: the op-level selective scan backward at 16 < d_state <= 256 (scan_op_bwd_wide.cu: one deterministic kernel behind
sigma_scan_bwd, sigma_scan_bwd_split and sigma_scan_bwd_det).

* Against the fp64 reference of oracle/scan_ref64.py, element by element inside its per-element bounds, every output in
  NaN-filled memory with guard elements and a NaN-filled workspace: d_state 17 .. 256 (every padded width), 1 / 2 / 3 / 4
  groups, channel groups that are not a multiple of 32, ragged and > 2048 lengths, batch 1 - 3, fp32 / fp16 / bf16 at every
  padded width, the d_state="auto" SS2D calls of Sigma-tiny stages 1 - 3 and Sigma-base stage 3 (batch 1), Sigma's parameters,
  larger steps, the reference test's distribution and a call with softplus, D and delta_bias off.
* Every call through all three entry points (with forced L-segment counts, which have no effect): bitwise equal to each other
  and to a repeated call.
* Autograd (ops.SelectiveScan, ops.selective_scan_fn) and the Mamba blocks with wide states: training gradients against the
  pure-torch scan, eval forwards on the composed path, and bitwise-repeatable gradients under the deterministic switch.
* Against the reference CUDA extension (where oracle/_ref was built): all seven gradients within 1e-3 (fp32) / 1e-2 (bf16) of
  each output's scale."""
import ctypes

import pytest
import torch

import procedural as P
from helpers import SEED, assert_close, guard_ok, guarded, op_scan_params, ptr as _p, scan_plan, stream as _stream
from oracle import scan_ref64 as R, sigma_ref
from test_ref_ext_gpu import load_ext
from test_scan_bwd_gpu import TOL
from test_scan_op_fp64_gpu import _DT, _check, _finish

pytestmark = pytest.mark.gpu
S = 173
NAMES = ("du", "ddelta", "dA", "dB", "dC", "dD", "ddelta_bias")
F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16


def _run(args, softplus, entry, nsplit=0):
    """one backward through `entry` ("bwd", "split" or "det") into guarded outputs, NaN-filled workspace -> (outs, bufs)"""
    from sigma_b200 import _lib
    L_ = _lib.lib()
    u, delta, A, B, C, D, bias, dout = args
    bt, dim, L = u.shape
    G, N = B.shape[1], B.shape[2]
    dt = u.dtype
    shapes = dict(du=((bt, dim, L), dt), ddelta=((bt, dim, L), dt), dA=((dim, N), F32), dB=((bt, G, N, L), F32), dC=((bt, G, N, L), F32))
    if D is not None:
        shapes["dD"] = ((dim,), F32)
    if bias is not None:
        shapes["ddelta_bias"] = ((dim,), F32)
    bufs, outs = {}, {}
    for k, (s, t) in shapes.items():
        bufs[k], outs[k] = guarded(s, t)
    det = entry == "det"
    wsb = (L_.sigma_scan_bwd_det_workspace_bytes if det else L_.sigma_scan_bwd_workspace_bytes)(bt, dim, L, N, G, _DT[dt])
    assert wsb > 0
    ws = torch.full((wsb // 4 + 1,), float("nan"), device="cuda")
    o = lambda k: _p(outs.get(k))
    common = (_p(u), _p(delta), _p(A), _p(B), _p(C), _p(D), _p(bias), _p(dout), o("du"), o("ddelta"), o("dA"), o("dB"), o("dC"),
              o("dD"), o("ddelta_bias"), bt, dim, L, N, G, _DT[dt], int(softplus), _p(ws), wsb)
    if entry == "bwd":
        rc = L_.sigma_scan_bwd(*common, _stream())
    else:
        rc = (L_.sigma_scan_bwd_det if det else L_.sigma_scan_bwd_split)(*common, nsplit, _stream())
    _lib.check(rc, "sigma_scan_bwd " + entry)
    torch.cuda.synchronize()
    return outs, bufs


def _bwd_all(args, softplus, ref, bnd, tag, worst):
    """every entry point against the oracle; the five calls bitwise equal"""
    runs = []
    for entry, ns in (("bwd", 0), ("split", 3), ("det", 0), ("det", 5), ("bwd", 0)):
        outs, bufs = _run(args, softplus, entry, ns)
        for k in outs:
            _check(f"{tag} {entry}/{ns}", k, outs[k], ref[k], bnd[k], worst)
            guard_ok(bufs[k], f"{tag} {entry}/{ns} {k}")
        err = float((outs["ddelta"].double() - ref["ddelta"]).abs().max()) / float(ref["ddelta"].abs().max())
        worst["ddelta/maxnorm"] = max(worst.get("ddelta/maxnorm", 0.0), err)
        runs.append(outs)
    for i, r in enumerate(runs[1:], 1):
        for k in r:
            assert torch.equal(r[k], runs[0][k]), f"{tag}: {k} of call {i} differs bitwise from the first call"


def _plan_ok(shape, dtype):
    bt, dim, L, N, G = shape
    for sweep in ("bwd", "bwd_det"):
        for ns in (0, 7):
            p = scan_plan(sweep, *shape, dtype, nsplit=ns)
            assert (p["route"], p["nsplit"], p["ntiles"], p["tiles_per_split"], p["channels"], p["state_nsplit"]) == \
                ("generic", 1, -(-L // 32), -(-L // 32), 32, 1), p


def _case(shape, tag, dtype=F32, dist="sigma", **opts):
    bt, dim, L, N, G = shape
    args = [None if t is None else t.cuda() for t in op_scan_params(S, bt, dim, L, N, G, tag, dist, dtype, **opts)]
    sp = opts.get("softplus", True)
    ref, bnd = R.scan_ref64(*args[:7], sp, args[7])
    return args, sp, ref, bnd


def _one(shape, dtype=F32, dist="sigma", **opts):
    tag = f"wide/{str(dtype)[6:]}/{dist}/{opts}/" + "/".join(map(str, shape))
    _plan_ok(shape, dtype)
    args, sp, ref, bnd = _case(shape, tag, dtype, dist, **opts)
    worst = {}
    _bwd_all(args, sp, ref, bnd, tag, worst)
    if shape[3] > 64:
        # ddelta's bound carries an (N + 5)·u term for its sum over the states, past 64 states looser than 1e-3 of its scale at
        # the largest element: there it is held to the max-norm bar of the summed outputs instead
        if dtype != BF16:
            assert worst["ddelta/maxnorm"] <= 1e-3, worst
        worst.pop("at_max/ddelta")
    _finish(f"scan wide fp64 {tag}", worst, tight=dtype != BF16)   # bf16's 2^-8 store rounding exceeds 1e-3 of scale


# (batch, dim, L, d_state, groups): d_state 17 .. 256 across every padded width (odd, just past a width, at a width, "auto"
# values), the layouts spread over them
LAYOUTS = [(2, 64, 300, 17, 1), (1, 96, 77, 22, 2), (3, 36, 130, 32, 3), (2, 128, 2100, 48, 4), (1, 64, 257, 64, 2),
           (2, 96, 200, 100, 2), (1, 128, 190, 128, 4), (2, 64, 100, 171, 1), (1, 64, 333, 256, 2)]


@pytest.mark.parametrize("shape", LAYOUTS)
def test_wide_bwd_matches_fp64(shape):
    _one(shape)


@pytest.mark.parametrize("dtype", [F16, BF16])
@pytest.mark.parametrize("n", [32, 64, 128, 256])
def test_wide_bwd_16bit_matches_fp64(n, dtype):
    """every padded width in fp16 and bf16 (fp32 above); 72 channels in 2 groups: a full and a partial channel tile per group"""
    _one((2, 72, 150, n, 2), dtype)


# Sigma's d_state="auto" SS2D calls, batch 1: tiny stages 1 - 3 (N 32, 64, 128) and base stage 3 (N 171 -> 256 states padded)
AUTO = [(1, 1536, 4800, 32, 4), (1, 3072, 1200, 64, 4), (1, 6144, 300, 128, 4), (1, 8192, 690, 171, 4)]


@pytest.mark.parametrize("shape", AUTO)
def test_wide_bwd_auto_shapes_match_fp64(shape):
    _one(shape)


@pytest.mark.parametrize("shape,dist,opts", [((2, 64, 300, 32, 1), "ref", {}), ((2, 96, 200, 128, 2), "wide", {}),
                                             ((2, 64, 300, 64, 2), "sigma", dict(softplus=False, has_D=False, has_bias=False))])
def test_wide_bwd_other_parameters_match_fp64(shape, dist, opts):
    """the reference test's distribution, larger steps and decays, and a call with softplus, D and delta_bias off"""
    _one(shape, F32, dist, **opts)


# ---------------------------------------------------------------------------------------------------------------------------
# autograd and the Mamba blocks
# ---------------------------------------------------------------------------------------------------------------------------
def _autograd(n, api, leaves_cpu, seed_tag):
    from sigma_b200 import ops
    leaves_ref = [t.clone().requires_grad_(True) for t in leaves_cpu]
    out_ref = sigma_ref.selective_scan_torch(*leaves_ref, True)
    w = P.randn(SEED, seed_tag + "/w", tuple(out_ref.shape))
    (out_ref * w).sum().backward()
    leaves = [t.clone().cuda().requires_grad_(True) for t in leaves_cpu]
    fn = ops.SelectiveScan.apply if api == "SelectiveScan" else ops.selective_scan_fn
    out = fn(*leaves, True, 1)
    (out * w.cuda()).sum().backward()
    assert_close(out, out_ref.detach(), 6e-4, 2e-3, "fwd")
    for name, a_, r_ in zip(["du", "ddelta", "dA", "dB", "dC", "dD", "dbias"], leaves, leaves_ref):
        rt, at = TOL[name]
        assert_close(a_.grad, r_.grad, rt, at * max(1.0, float(r_.grad.abs().max()) / 50.0), f"autograd {api} N={n} {name}")


@pytest.mark.parametrize("api", ["SelectiveScan", "selective_scan_fn"])
@pytest.mark.parametrize("n", [32, 64])
def test_autograd_wide_state(n, api):
    """the autograd functions at d_state 32 / 64 against the autograd of the pure-torch scan (Sigma's parameters)"""
    tag = f"wide-ag/{n}/{api}"
    u, delta, A, B, C, D, bias, _ = op_scan_params(S, 2, 64, 130, n, 2, tag)
    _autograd(n, api, [u, delta, A, B, C, D, bias], tag)


def test_autograd_wide_state_reference_distribution():
    """the reference test's input distribution (procedural.scan_inputs), d_state 48"""
    u, dl, A, Bm, Cm, D, bias = P.scan_inputs(SEED + 17, 2, 64, 48, 130, 2)
    _autograd(48, "SelectiveScan", [u, dl, A, Bm, Cm, D, bias], "wide-ag/ref")


def _swap_scan_for_torch(monkeypatch):
    """the op-level scans of the composed path replaced by the differentiable torch restatement (runs on the CPU)"""
    from sigma_b200 import ops
    g4 = lambda t: t.unsqueeze(1) if t.dim() == 3 else t                     # (B, N, L) -> one group, as SelectiveScanFn does
    f = lambda u_, d_, A_, B_, C_, D_=None, db_=None, sp_=False, nr_=1: sigma_ref.selective_scan_torch(u_, d_, A_, g4(B_), g4(C_), D_,
                                                                                                        db_, sp_)
    monkeypatch.setattr(ops.SelectiveScan, "apply", staticmethod(f))
    monkeypatch.setattr(ops.SelectiveScanFn, "apply", staticmethod(f))


def _outs(y):
    return list(y) if isinstance(y, tuple) else [y]


def _train_vs_cpu(make, xs_shape, nin, tag, monkeypatch):
    """one training step of the block on the GPU (composed path: the wide-state op-level backward) against the same block on the
    CPU with the torch scan: outputs, input gradients and every parameter gradient"""
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    blk = make()
    P.fill_state_dict(blk, SEED)
    ref_blk = make()
    ref_blk.load_state_dict(blk.state_dict())
    xs = [P.randn(SEED, f"{tag}/x{i}", xs_shape) for i in range(nin)]
    with monkeypatch.context() as m:
        _swap_scan_for_torch(m)
        xr = [x.clone().requires_grad_(True) for x in xs]
        yr = _outs(ref_blk(*xr))
        sum(y.square().sum() for y in yr).backward()
    blk = blk.cuda().train()
    xg = [x.clone().cuda().requires_grad_(True) for x in xs]
    yg = _outs(blk(*xg))
    sum(y.square().sum() for y in yg).backward()
    for a, r in zip(yg, yr):
        assert_close(a, r.detach(), 1e-4, 1e-4 * float(r.abs().max()), f"{tag} train fwd")
    for a, r in zip(xg, xr):
        assert_close(a.grad, r.grad, 2e-3, 2e-3 * float(r.grad.abs().max()), f"{tag} train dx")
    for (k, pg), (_, pr) in zip(blk.named_parameters(), ref_blk.named_parameters()):
        if pr.grad is None:
            continue
        assert pg.grad is not None, k
        assert_close(pg.grad, pr.grad, 2e-3, 2e-3 * float(pr.grad.abs().max()) + 1e-6, f"{tag} train grad {k}")


def test_ss2d_auto_state_trains(monkeypatch):
    """SS2D(d_model=192, d_state="auto"): d_state 32"""
    from sigma_b200 import modules as M
    assert M.SS2D(d_model=192, d_state="auto").d_state == 32
    _train_vs_cpu(lambda: M.SS2D(d_model=192, d_state="auto"), (1, 5, 6, 192), 1, "wide-ss2d", monkeypatch)


@pytest.mark.parametrize("block", ["ConcatMambaFusionBlock", "CrossMambaFusionBlock"])
def test_fusion_blocks_wide_state_train(block, monkeypatch):
    from sigma_b200 import modules as M
    _train_vs_cpu(lambda: getattr(M, block)(hidden_dim=48, d_state=32), (1, 5, 6, 48), 2, f"wide-{block}", monkeypatch)


@pytest.mark.parametrize("block,nin", [("VSSBlock", 1), ("CVSSDecoderBlock", 1), ("ConcatMambaFusionBlock", 2),
                                       ("CrossMambaFusionBlock", 2)])
def test_blocks_wide_state_eval_take_the_composed_path(block, nin):
    """under no_grad a block whose d_state the fused scan lacks returns the composed path's output instead of raising"""
    from sigma_b200 import modules as M
    kw = dict(hidden_dim=48, d_state=32)
    if block == "VSSBlock":
        kw = dict(hidden_dim=192, d_state="auto", mlp_ratio=0.0)
    blk = getattr(M, block)(**kw)
    P.fill_state_dict(blk, SEED)
    blk = blk.cuda().eval()
    C = kw["hidden_dim"]
    xs = [P.randn(SEED, f"wide-eval/{block}/x{i}", (2, 6, 7, C)).cuda() for i in range(nin)]
    with torch.no_grad():
        got = _outs(blk(*xs))
        with M.composed_path():
            ref = _outs(blk(*xs))
    assert len(got) == len(ref)
    for a, r in zip(got, ref):
        assert bool(a.isfinite().all())
        assert torch.equal(a, r), block


def test_auto_state_block_and_backbone_train_and_eval():
    """d_state="auto" end to end at 64 x 96: a VSSBlock (d_state 32) and a Backbone_VSSM (16, 32, 64, 128 by stage) run a
    training step and an eval forward"""
    from sigma_b200 import modules as M
    torch.manual_seed(SEED)
    blk = M.VSSBlock(hidden_dim=192, d_state="auto").cuda().train()
    x = torch.randn(1, 16, 24, 192, device="cuda", requires_grad=True)
    blk(x).square().mean().backward()
    assert bool(x.grad.isfinite().all()) and all(bool(p.grad.isfinite().all()) for p in blk.parameters() if p.grad is not None)
    with torch.no_grad():
        assert bool(blk.eval()(x.detach()).isfinite().all())
    net = M.Backbone_VSSM(depths=[1, 1, 2, 1], d_state="auto").cuda().train()
    assert [L.blocks[0].op.d_state for L in net.layers] == [16, 32, 64, 128]
    img = torch.randn(1, 3, 64, 96, device="cuda")
    sum(o.square().mean() for o in net(img)).backward()
    assert all(bool(p.grad.isfinite().all()) for p in net.parameters() if p.grad is not None)
    with torch.no_grad():
        assert all(bool(o.isfinite().all()) for o in net.eval()(img))


def test_wide_state_deterministic_training_steps(monkeypatch):
    """under torch.use_deterministic_algorithms(True) two training steps of one block give bitwise-equal gradients"""
    from sigma_b200 import modules as M
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")      # torch requires it for cuBLAS under the switch
    blk = M.ConcatMambaFusionBlock(hidden_dim=48, d_state=32)
    P.fill_state_dict(blk, SEED)
    blk = blk.cuda().train()
    xs = [P.randn(SEED, f"wide-det/x{i}", (2, 6, 7, 48)).cuda() for i in range(2)]
    runs = []
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(2):
            blk.zero_grad(set_to_none=True)
            xg = [x.clone().requires_grad_(True) for x in xs]
            blk(*xg).square().sum().backward()
            runs.append([x.grad.clone() for x in xg] + [p.grad.clone() for p in blk.parameters() if p.grad is not None])
    finally:
        torch.use_deterministic_algorithms(False)
    assert len(runs[0]) == len(runs[1]) > 2
    assert all(torch.equal(a, b) for a, b in zip(*runs))


# ---------------------------------------------------------------------------------------------------------------------------
# against the reference CUDA extension
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [F32, BF16])
@pytest.mark.parametrize("n", [32, 64, 128, 256])
def test_wide_bwd_matches_reference_extension(n, dtype):
    ext = load_ext()
    if ext is None:
        pytest.skip("the reference extension was not built (oracle/build_ref_ext.py)")
    from sigma_b200 import ops
    tag = f"wide-ext/{n}/{str(dtype)[6:]}"
    u, delta, A, B, C, D, bias, dout = [t.cuda() for t in op_scan_params(S, 2, 256, 600, n, 4, tag, dtype=dtype)]
    _, x = ext.fwd(u, delta, A, B, C, D, bias, True, 1)
    ref = ext.bwd(u, delta, A, B, C, D, bias, dout, x, True, 1)
    got = ops.selective_scan_cuda_core_bwd(u, delta, A, B, C, D, bias, dout, None, True, 1)
    bar = 1e-3 if dtype == F32 else 1e-2
    for name, g, r in zip(NAMES, got, ref):
        scale = float(r.float().abs().max())
        err = float((g.float() - r.float()).abs().max()) / scale
        assert err <= bar, f"{tag} {name}: {err:.2e} of its scale"
