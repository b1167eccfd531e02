"""GPU: training under torch.use_deterministic_algorithms(True).

* Bitwise repeatability of every `_det` backward: three calls on the same inputs, one of them while another stream keeps the SMs
  busy with GEMMs, must give torch.equal outputs.  The fused SS2D backward at the training shapes and dt_ranks of
  test_ss2d_bwd_fp64_gpu (after the training forward, auto and forced L-segment plans); the op-level backward in fp32 / fp16 /
  bf16 at d_state 4, 8, 16 and the generic kernel at L = 690; LayerNorm at every instantiated width; bilinear upsampling at
  Sigma's x2, x4 and size= cases.
* Accuracy: the fused `_det` outputs inside the per-element fp64 bounds of oracle/ss2d_ref64.py; the op-level ones at the
  reference tolerances of test_scan_bwd_gpu; the bilinear backward against fp64 CPU autograd of F.interpolate; the deterministic
  cross-entropy against nn.CrossEntropyLoss (value and gradient, ignore_index pixels present).
* End to end: two Sigma-tiny training steps in a subprocess with the switch on (fp32 and bf16 autocast), run twice from the
  same seeds: loss, every gradient and every updated parameter bitwise equal, and no torch op on the path raises."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import procedural as P
import test_ss2d_bwd_fp64_gpu as F64
from helpers import SEED
from oracle import scan_oracle, ss2d_ref64 as R64

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S = 131


def _busy():
    """queue GEMMs on a second stream so that the next launches on the current stream share the SMs with them"""
    det = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(False)          # the load itself need not be reproducible
    s = torch.cuda.Stream()
    a = torch.randn(4096, 4096, device="cuda")
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(8):
            a = a @ a * 1e-3
    torch.use_deterministic_algorithms(det)
    return s, a


def _three(run):
    """run() three times (the second while another stream is busy) -> the three lists of output tensors, cloned"""
    outs = []
    for i in range(3):
        keep = _busy() if i == 1 else None
        outs.append([t.clone() for t in run()])
        if keep is not None:
            torch.cuda.current_stream().wait_stream(keep[0])
    torch.cuda.synchronize()
    return outs


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32) if t.is_floating_point() else t


def _equal3(outs, tag):
    """bitwise equality (slots an entry leaves unwritten stay the same NaN, which torch.equal would call unequal)"""
    for i in (1, 2):
        for j, (a, b) in enumerate(zip(outs[0], outs[i])):
            assert torch.equal(_bits(a), _bits(b)), f"{tag}: output {j} of run {i} differs from run 0"


# ---- fused SS2D backward ----
def _ss2d_det(kind, B, H, W, D, N, R, Cp, args, nsplit):
    from sigma_b200 import _lib
    L_ = _lib.lib()
    xc, xdbl, dtw, dtb, A, Ds, dy = args
    K = xdbl.shape[2]
    Lseq = xc.shape[1]
    kid = F64._kid(kind)
    T = L_.sigma_ss2d_scan_hs_bytes(kid, B, H, W, D, N) // (4 * K * B * D * N)
    bufs, outs = {}, {}
    for name, shape in [("delta", (K, B, Lseq, D)), ("dxc", (B, Lseq, D)), ("ddelta", (K, B, Lseq, D)), ("dxdbl", (B, Lseq, K, Cp)),
                        ("dA", (K * D, N)), ("dDs", (K * D,)), ("ddtb", (K, D)), ("y", (K, B, Lseq, D)), ("hs", (K, B, T, D, N))]:
        bufs[name], outs[name] = F64._guarded(shape)
    wsb = L_.sigma_ss2d_scan_bwd_det_workspace_bytes(kid, B, H, W, D, N)
    assert wsb > L_.sigma_ss2d_scan_bwd_workspace_bytes(kid, B, H, W, D, N)
    ws = torch.full((wsb // 4,), float("nan"), device="cuda")
    head = (kid, F64._p(xc), F64._p(xdbl), F64._p(dtw), F64._p(dtb), F64._p(A), F64._p(Ds))
    tail = tuple(F64._p(outs[n]) for n in ("dxc", "ddelta", "dxdbl", "dA", "dDs", "ddtb")) + (B, H, W, D, N, R, Cp, F64._p(ws), wsb)
    fwb = L_.sigma_ss2d_scan_workspace_bytes(kid, B, H, W, D, N)
    fws = torch.zeros(max(fwb, 4), dtype=torch.uint8, device="cuda")
    _lib.check(L_.sigma_ss2d_scan_fwd_save(*head, F64._p(outs["y"]), F64._p(outs["delta"]), F64._p(outs["hs"]), B, H, W, D, N, R, Cp,
                                           F64._p(fws), fwb, 0, F64._stream()), "sigma_ss2d_scan_fwd_save")
    _lib.check(L_.sigma_ss2d_scan_bwd_saved_det(*head, F64._p(dy), F64._p(outs["delta"]), F64._p(outs["hs"]), *tail, nsplit, F64._stream()),
               "sigma_ss2d_scan_bwd_saved_det")
    torch.cuda.synchronize()
    for name, buf in bufs.items():
        F64._guard_ok(buf, f"{kind} det {name}")
    return outs


@pytest.mark.parametrize("kind,B,H,W,D,N,R", F64.CASES)
def test_fused_bwd_det_repeatable_and_within_fp64_bounds(kind, B, H, W, D, N, R):
    tag = f"{kind}/{B}/{H}x{W}/D{D}/N{N}/R{R}"                # the inputs of test_ss2d_bwd_fp64_gpu at this case
    args, Cp = F64._params(kind, B, H, W, D, N, R, tag)
    ref, bnd = R64.ss2d_ref64(kind, *args, H, W)
    worst = {}
    names = ("dxc", "ddelta", "dA", "dDs", "ddtb")
    plans = [0, 7, 1]
    if (H, W) == (15, 20):
        plans.append(20)                         # the shorter walks end in an empty segment (asserted in test_ss2d_bwd_fp64_gpu)
    for nsplit in plans:
        t = f"{tag} split={nsplit}"
        runs = _three(lambda: list(_ss2d_det(kind, B, H, W, D, N, R, Cp, args, nsplit).values()))
        _equal3(runs, t)
        outs = _ss2d_det(kind, B, H, W, D, N, R, Cp, args, nsplit)
        for name in names:
            F64._check(t, name, outs[name], ref[name], bnd[name], worst)
        dx = outs["dxdbl"]
        F64._check(t, "dB", dx[..., :N], ref["dB"], bnd["dB"], worst)
        F64._check(t, "dC", dx[..., N:2 * N], ref["dC"], bnd["dC"], worst)
        assert bool((dx[..., 2 * N:] == 0).all()), f"{t}: the dt_r / padding columns of dxdbl must stay 0"
    F64._finish(f"ss2d bwd det fp64 {tag}", worst)


def test_fused_core_autograd_switches_to_det(monkeypatch):
    """FusedSS2DCore.backward calls the _det entry under the switch: gradients repeat bitwise and stay within 1e-5 of the
    default build's"""
    from sigma_b200 import ops
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")      # torch requires it for cuBLAS under the switch
    kind, B, H, W, D, N, R = "cross4", 2, 30, 40, 768, 16, 24
    tag = "det/ag"
    K = 4
    xc0 = P.randn(S, tag + "/xc", (B, H * W, D)).cuda()
    wgt = P.randn(S, tag + "/w", (B, H * W, D)).cuda()
    xpw = P.randn(S, tag + "/xpw", (K, R + 2 * N, D), D ** -0.5).cuda()
    dtw = P.rand(S, tag + "/dtw", (K, D, R), -R ** -0.5, R ** -0.5).cuda()
    dtb = torch.full((K, D), -4.0).cuda()
    Al = torch.log(torch.arange(1, N + 1, dtype=torch.float32)).repeat(K * D, 1).cuda()
    Ds = torch.ones(K * D).cuda()
    calls = []
    orig = ops._call_ss2d_bwd
    monkeypatch.setattr(ops, "_call_ss2d_bwd", lambda args, saved=False, det=False: (calls.append(det), orig(args, saved, det))[1])

    def grads():
        leaves = [t.clone().requires_grad_(True) for t in (xc0, xpw, dtw, dtb, Al, Ds)]
        (ops.FusedSS2DCore.apply(*leaves, F64._kid(kind), H, W) * wgt).sum().backward()
        return [t.grad for t in leaves]

    plain = grads()
    torch.use_deterministic_algorithms(True)
    try:
        runs = _three(grads)
    finally:
        torch.use_deterministic_algorithms(False)
    assert calls == [False, True, True, True]
    _equal3(runs, "FusedSS2DCore det")
    for g, r in zip(runs[0], plain):
        assert float((g - r).abs().max()) <= 1e-5 * float(r.abs().max()) + 1e-30


# ---- op-level backward ----
RT, AT = 6e-4, 2e-3
TOL = {"du": (RT * 2, AT * 2), "ddelta": (RT * 5, AT * 10), "dA": (1e-3, 5e-3), "dB": (RT, AT), "dC": (RT, AT),
       "dD": (1e-3, 1e-3), "dbias": (1e-3, 1e-3)}
NAMES = ["du", "ddelta", "dA", "dB", "dC", "dD", "dbias"]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("b,d,n,L,G,split", [(2, 192, 4, 4800, 1, 0), (2, 96, 8, 1024, 2, 3), (2, 384, 16, 2048, 1, 0),
                                             (1, 128, 16, 1200, 1, 5), (2, 64, 16, 690, 1, 0), (2, 48, 4, 690, 2, 0)])
def test_op_bwd_det_repeatable_and_accurate(dtype, b, d, n, L, G, split):
    from sigma_b200 import ops
    u, dl, A, Bm, Cm, D, bias = P.scan_inputs(SEED + 21, b, d, n, L, G)
    dout = P.randn(SEED + 21, f"det/do/{b}/{d}/{n}/{L}", (b, d, L))
    q = lambda t: t.to(dtype).cuda()
    args = (q(u), q(dl), A.cuda(), q(Bm), q(Cm), D.cuda(), bias.cuda(), q(dout), None, True, 1)
    torch.use_deterministic_algorithms(True)
    try:
        runs = _three(lambda: ops.selective_scan_cuda_core_bwd(*args, _force_split=split))
    finally:
        torch.use_deterministic_algorithms(False)
    _equal3(runs, f"op bwd det {dtype} {(b, d, n, L, G, split)}")
    f = lambda t: t.to(dtype).float().numpy()
    ref = scan_oracle.scan_bwd(f(u), f(dl), A.numpy(), f(Bm), f(Cm), D.numpy(), bias.numpy(), f(dout), True)
    loose = dtype != torch.float32
    assert runs[0][3].dtype == dtype and runs[0][0].dtype == dtype
    for name, got, r in zip(NAMES, runs[0], ref):
        rt, at = (3e-2, 5e-2) if loose else TOL[name]
        err = np.abs(got.float().cpu().numpy() - r)
        lim = at * max(1.0, float(np.abs(r).max()) / 50.0) + rt * np.abs(r)
        assert bool((err <= lim).all()), f"{name}: max err {float(err.max()):.3e}"


def test_op_bwd_generic_det_runs_the_generic_kernel():
    """L = 690 rows are not 16-byte aligned: the generic kernel (shared-memory warp-ordered dB / dC) runs, deterministically"""
    from sigma_b200 import _lib, ops
    u, dl, A, Bm, Cm, D, bias = P.scan_inputs(SEED + 22, 2, 96, 16, 690, 1)
    dout = P.randn(SEED + 22, "det/gen/do", (2, 96, 690))
    c = lambda t: t.cuda()
    torch.use_deterministic_algorithms(True)
    try:
        n0 = _lib.launch_count()
        runs = _three(lambda: ops.selective_scan_cuda_core_bwd(c(u), c(dl), c(A), c(Bm), c(Cm), c(D), c(bias), c(dout), None, True, 1))
    finally:
        torch.use_deterministic_algorithms(False)
    assert _lib.launch_count() > n0
    _equal3(runs, "generic det")
    ref = scan_oracle.scan_bwd(u.numpy(), dl.numpy(), A.numpy(), Bm.numpy(), Cm.numpy(), D.numpy(), bias.numpy(), dout.numpy(), True)
    for name, got, r in zip(NAMES, runs[0], ref):
        rt, at = TOL[name]
        err = np.abs(got.cpu().numpy() - r)
        assert bool((err <= at * max(1.0, float(np.abs(r).max()) / 50.0) + rt * np.abs(r)).all()), name


# ---- LayerNorm ----
@pytest.mark.parametrize("C", [32, 64, 96, 128, 192, 256, 384, 512, 768, 1024, 1536])
@pytest.mark.parametrize("rows", [7, 38400])
def test_layernorm_bwd_det(C, rows):
    from sigma_b200 import ops
    ln = torch.nn.LayerNorm(C).cuda()
    with torch.no_grad():
        ln.weight.copy_(P.rand(S, f"ln/w/{C}", (C,), 0.5, 1.5))
    x0 = (P.randn(S, f"ln/x/{C}/{rows}", (rows, C)) * 2 + 0.3).cuda()
    wgt = P.randn(S, f"ln/g/{C}/{rows}", (rows, C)).cuda()

    def grads():
        ln.weight.grad = ln.bias.grad = None
        x = x0.clone().requires_grad_(True)
        (ops.layer_norm(ln, x) * wgt).sum().backward()
        return [x.grad, ln.weight.grad, ln.bias.grad]

    ref = grads()
    torch.use_deterministic_algorithms(True)
    try:
        runs = _three(grads)
    finally:
        torch.use_deterministic_algorithms(False)
    _equal3(runs, f"layernorm det C={C} rows={rows}")
    for g, r in zip(runs[0], ref):
        assert float((g - r).abs().max()) <= 2e-5 * (float(r.abs().max()) + 1e-20)


# ---- bilinear upsampling ----
BILINEAR = [((2, 96, 30, 40), dict(scale_factor=2), False), ((2, 96, 30, 40), dict(scale_factor=4), False),
            ((2, 40, 30, 40), dict(size=(120, 160)), True), ((2, 40, 18, 26), dict(size=(72, 104)), True),
            ((1, 96, 9, 13), dict(scale_factor=2), False), ((1, 192, 5, 7), dict(size=(9, 13)), False),
            ((2, 48, 17, 25), dict(scale_factor=4), True), ((1, 3, 23, 17), dict(size=(72, 104)), True)]


@pytest.mark.parametrize("shape,kw,nchw", BILINEAR)
def test_bilinear_bwd_det(shape, kw, nchw):
    from sigma_b200 import ops
    x0 = P.randn(S, f"bil/x/{shape}", shape)
    xc = x0.cuda() if nchw else x0.permute(0, 2, 3, 1).contiguous().cuda().permute(0, 3, 1, 2)    # channels-last view
    xr = x0.double().requires_grad_(True)
    yr = F.interpolate(xr, mode="bilinear", align_corners=False, **kw)
    g = P.randn(S, f"bil/g/{shape}", tuple(yr.shape))
    (yr * g.double()).sum().backward()
    torch.use_deterministic_algorithms(True)
    try:
        def run():
            x = xc.detach().clone().requires_grad_(True) if nchw else \
                xc.detach().permute(0, 2, 3, 1).clone().permute(0, 3, 1, 2).requires_grad_(True)
            y = ops.upsample_bilinear(x, **kw)
            assert "UpsampleBilinearFn" in type(y.grad_fn).__name__
            (y * g.cuda()).sum().backward()
            assert x.grad.is_contiguous(memory_format=torch.contiguous_format if nchw else torch.channels_last)
            return [y.detach(), x.grad]
        runs = _three(run)
    finally:
        torch.use_deterministic_algorithms(False)
    _equal3(runs, f"bilinear {shape} {kw}")
    y_plain = F.interpolate(xc, mode="bilinear", align_corners=False, **kw)
    assert torch.equal(runs[0][0], y_plain)                    # the forward is F.interpolate's kernel without the switch
    ref = xr.grad
    xa = x0.double().requires_grad_(True)
    (F.interpolate(xa, mode="bilinear", align_corners=False, **kw) * g.double().abs()).sum().backward()
    err = (runs[0][1].double().cpu() - ref).abs()
    # against fp64: a few fp32 roundings of the sum of |weight·dy| over the taps, plus the fp32 source index (torch's CUDA rule)
    # whose error of up to 2 ulps of its magnitude (< max(Hin, Win)) moves every weight by that much
    tol = 1e-6 + max(shape[2:]) * 2.0 ** -21
    assert bool((err <= tol * xa.grad + 1e-12).all()), f"max err {float(err.max()):.3e}"


# ---- cross-entropy ----
def test_deterministic_cross_entropy_matches_nn():
    from sigma_b200 import ops
    B, K, H, W = 2, 9, 48, 64
    logits0 = (P.randn(S, "ce/x", (B, K, H, W)) * 3).cuda()
    lab = torch.from_numpy(np.random.default_rng(S).integers(0, K, size=(B, H, W))).cuda()
    lab[:, :10, :] = 255
    crit = torch.nn.CrossEntropyLoss(reduction="mean", ignore_index=255)
    assert ops.plain_cross_entropy(crit) == 255
    assert ops.plain_cross_entropy(torch.nn.CrossEntropyLoss(label_smoothing=0.1)) is None
    assert ops.plain_cross_entropy(torch.nn.CrossEntropyLoss(weight=torch.ones(K))) is None
    a = logits0.clone().requires_grad_(True)
    la = crit(a, lab)
    la.backward()
    torch.use_deterministic_algorithms(True)
    try:
        def run():
            b = logits0.clone().requires_grad_(True)
            lb = ops.deterministic_cross_entropy(b, lab, 255)
            lb.backward()
            return [lb.detach(), b.grad]
        runs = _three(run)
    finally:
        torch.use_deterministic_algorithms(False)
    _equal3(runs, "cross-entropy")
    assert abs(float(runs[0][0]) - float(la)) <= 1e-6 * abs(float(la))
    assert float((runs[0][1] - a.grad).abs().max()) <= 1e-6 * float(a.grad.abs().max())


# ---- end to end ----
@pytest.mark.parametrize("amp", ["fp32", "bf16"])
def test_training_steps_bitwise_reproducible(amp, tmp_path):
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    script = os.path.join(ROOT, "scripts", "det_train_steps.py")
    outs = []
    for i in range(2):
        path = str(tmp_path / f"run{i}.pt")
        r = subprocess.run([sys.executable, script, "--amp", amp, "--out", path], cwd=ROOT, env=env, capture_output=True, text=True,
                           timeout=900)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
        outs.append(torch.load(path))
    a, b = outs
    assert a.keys() == b.keys() and len(a) > 100
    diff = [k for k in a if not torch.equal(a[k], b[k])]
    assert not diff, f"{len(diff)} tensors differ, e.g. {diff[:5]}"
    for k, v in a.items():
        if k.startswith("loss"):
            assert bool(torch.isfinite(v).all()), k
