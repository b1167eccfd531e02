"""GPU: the training kernels of the ChannelAttentionBlock's 3x3 convs (sigma_conv3x3_gelu_save_tf32, sigma_conv3x3_dgrad_tf32,
sigma_conv3x3_wgrad_tf32) and the autograd node and block route built on them (ops.CabConvFn, CVSSDecoderBlock).

* Op level against torch CPU float64 autograd of F.conv2d -> F.gelu -> F.conv2d, element by element: y, pre, dx, dW1, db1, dW2, db2
  at every Sigma-tiny / Sigma-small decoder stage at 480 x 640 with batch 2, the PST900 720 x 1280 stages (45 x 80 is ragged in H),
  the 72 x 104 model's stages, H = 1, W = 1 and channel counts that are multiples of 4 but not of 32; TF32 and tf32x3.  Each bound
  scales with the output's sum of |terms| (r = the precision's per-product bound + the terms added in sequence times u), with the
  errors of the pre-activation carried through GELU, GELU' and the second conv.  NaN guards around every output keep their bits.
* Two backward calls give the same bits, with torch.use_deterministic_algorithms(True) off and on, and equal bits between the two.
* Block level at Sigma's decoder widths: CVSSDecoderBlock's loss, input gradient and every parameter gradient on the new route match
  the cuDNN route (FUSED_CAB_TRAINING = False) at fp32 grade; no 3x3 convolution runs in the block's forward or backward; the saved
  tensors of its training forward fall.
* The route is not taken at hidden 32, under bf16 / fp16 autocast, under composed_path() or with the switch off.
The whole-model graph-replayed step runs the route through tests/test_train_graph_gpu.py (its decoder's CAB has C = 96)."""
import contextlib
import math

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from helpers import SEED, guard_ok, guarded, record

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
PREC = {"tf32": 2 * 2.0 ** -10 + 2.0 ** -20, "tf32x3": 4 * 2.0 ** -20}   # per-product relative bound of each mode
GELU2 = 0.8                                                               # max |GELU''| = 2·φ(0)
GELU1 = 1.13                                                              # max |GELU'|

# (B, H, W, C): the first conv maps C -> C // 3 (given as C1 where C is not a multiple of 3), the second C1 -> C
SIGMA = [(2, 120, 160, 96, 32), (2, 60, 80, 192, 64), (2, 30, 40, 384, 128)]
PST900 = [(1, 180, 320, 96, 32), (1, 90, 160, 192, 64), (1, 45, 80, 384, 128)]
ODD = [(1, 18, 26, 96, 32), (1, 9, 13, 192, 64), (1, 5, 7, 384, 128)]
EDGE = [(1, 1, 1, 12, 4), (1, 1, 37, 36, 12), (2, 29, 1, 36, 12), (1, 13, 21, 60, 20), (2, 9, 17, 44, 68)]


@contextlib.contextmanager
def _precision(mode):
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = mode == "tf32"
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32 = prev


def _inputs(B, H, W, C, C1, seed=SEED):
    g = torch.Generator().manual_seed(seed + 7 * C + H)
    x = torch.randn(B, H, W, C, generator=g)
    w1 = torch.randn(C1, C, 3, 3, generator=g) / math.sqrt(9 * C)
    b1 = torch.randn(C1, generator=g) * 0.1
    w2 = torch.randn(C, C1, 3, 3, generator=g) / math.sqrt(9 * C1)
    b2 = torch.randn(C, generator=g) * 0.1
    dy = torch.randn(B, H, W, C, generator=g)
    return x, w1, b1, w2, b2, dy


def _nchw(t):
    return t.double().permute(0, 3, 1, 2).contiguous()


def _ref64(x, w1, b1, w2, b2, dy, mode, n):
    """float64 autograd on CPU -> values and bounds of (y, pre, dx, dW1, db1, dW2, db2), channels-last where an activation"""
    xd, w1d, b1d, w2d, b2d = (t.double().requires_grad_(True) for t in (_nchw(x), w1, b1, w2, b2))
    pre = F.conv2d(xd, w1d, b1d, padding=1)
    y = F.conv2d(F.gelu(pre), w2d, b2d, padding=1)
    dyd = _nchw(dy)
    dx, dw1, db1, dw2, db2 = torch.autograd.grad(y, (xd, w1d, b1d, w2d, b2d), dyd)
    r = PREC[mode] + n * U
    cin, cout = torch.nn.grad.conv2d_input, torch.nn.grad.conv2d_weight
    with torch.no_grad():
        pre = pre.detach()
        ax, aw1, ab1, aw2, ab2, ady = xd.detach().abs(), w1d.detach().abs(), b1d.detach().abs(), w2d.detach().abs(), b2d.detach().abs(), dyd.abs()
        e_pre = r * (F.conv2d(ax, aw1, ab1, padding=1))
        h = F.gelu(pre)
        e_h = GELU1 * e_pre + U * h.abs()
        b_y = r * F.conv2d(h.abs(), aw2, ab2, padding=1) + F.conv2d(e_h, aw2, padding=1)
        g = cin((xd.shape[0], w1.shape[0], *xd.shape[2:]), w2d.detach(), dyd, padding=1)
        m_g = cin(g.shape, aw2, ady, padding=1)
        gp = 0.5 * (1 + torch.erf(pre / math.sqrt(2))) + pre * torch.exp(-0.5 * pre * pre) / math.sqrt(2 * math.pi)
        dpre = g * gp
        e_dpre = r * GELU1 * m_g + GELU2 * g.abs() * e_pre + U * dpre.abs()
        b_dx = r * cin(xd.shape, aw1, dpre.abs(), padding=1) + cin(xd.shape, aw1, e_dpre, padding=1)
        b_dw1 = r * cout(ax, w1.shape, dpre.abs(), padding=1) + cout(ax, w1.shape, e_dpre, padding=1)
        b_db1 = n * U * dpre.abs().sum((0, 2, 3)) + e_dpre.sum((0, 2, 3))
        b_dw2 = r * cout(h.abs(), w2.shape, ady, padding=1) + cout(e_h, w2.shape, ady, padding=1)
        b_db2 = n * U * ady.sum((0, 2, 3))
    cl = lambda t: t.permute(0, 2, 3, 1)   # noqa: E731
    vals = [cl(y.detach()), cl(pre), cl(dx), dw1, db1, dw2, db2]
    bounds = [cl(b_y), cl(e_pre), cl(b_dx), b_dw1, b_db1, b_dw2, b_db2]
    return vals, bounds


def _run(x, w1, b1, w2, b2, dy, mode):
    """the node's calls, each output in a NaN-guarded buffer -> (outputs, guard buffers)"""
    from sigma_b200 import _lib, ops
    from sigma_b200._lib import ptr, stream
    L = _lib.lib()
    B, H, W, C = x.shape
    C1 = w1.shape[0]
    x3 = mode == "tf32x3"
    x, w1, b1, w2, b2, dy = (t.cuda().contiguous() for t in (x, w1, b1, w2, b2, dy))
    shapes = dict(h=(B, H, W, C1), pre=(B, H, W, C1), y=(B, H, W, C), dpre=(B, H, W, C1), dx=(B, H, W, C),
                  dw1=(C1, C, 3, 3), db1=(C1,), dw2=(C, C1, 3, 3), db2=(C,))
    bufs, o = {}, {}
    for k, s in shapes.items():
        bufs[k], o[k] = guarded(s)
    hi, lo = ops._w9(w1, x3)
    _lib.check(L.sigma_conv3x3_gelu_save_tf32(ptr(x), ptr(hi), ptr(lo), ptr(b1), ptr(o["h"]), ptr(o["pre"]), B, H, W, C, C1, stream()), "save")
    hi, lo = ops._w9(w2, x3)
    _lib.check(L.sigma_conv3x3_tf32(ptr(o["h"]), ptr(hi), ptr(lo), ptr(b2), 0, ptr(o["y"]), B, H, W, C1, C, stream()), "conv")

    def wgrad(xin, gelu_x, g, dw, db, cin, cout_):
        wsb = L.sigma_conv3x3_wgrad_workspace_bytes(B, H, W, cin, cout_)
        ws = torch.full((wsb,), 255, dtype=torch.uint8, device="cuda")
        _lib.check(L.sigma_conv3x3_wgrad_tf32(ptr(xin), gelu_x, ptr(g), ptr(dw), ptr(db), B, H, W, cin, cout_, int(x3), ptr(ws), wsb,
                                              stream()), "wgrad")

    wgrad(o["pre"], 1, dy, o["dw2"], o["db2"], C1, C)
    hi, lo = ops._w9(w2, x3, grad=True)
    _lib.check(L.sigma_conv3x3_dgrad_tf32(ptr(dy), ptr(hi), ptr(lo), ptr(o["pre"]), ptr(o["dpre"]), B, H, W, C1, C, stream()), "dgrad2")
    wgrad(x, 0, o["dpre"], o["dw1"], o["db1"], C, C1)
    hi, lo = ops._w9(w1, x3, grad=True)
    _lib.check(L.sigma_conv3x3_dgrad_tf32(ptr(o["dpre"]), ptr(hi), ptr(lo), None, ptr(o["dx"]), B, H, W, C, C1, stream()), "dgrad1")
    torch.cuda.synchronize()
    return o, bufs


def _seq_terms(B, H, W, C, C1):
    """the longest chain of additions in sequence behind any output: the convs' K (9·C and 9·C1, chained through dpre) plus the
    weight gradient's pixels per partial row and the rows of the partial sum"""
    from sigma_b200 import _lib
    import ctypes
    worst = 0
    for cin, cout in ((C, C1), (C1, C)):
        out = (ctypes.c_int64 * 4)()
        assert _lib.lib().sigma_test_conv3x3_wgrad_plan(B, H, W, cin, cout, out) == 0
        npatch = B * math.ceil(H / 8) * math.ceil(W / 16)
        worst = max(worst, 128 * math.ceil(npatch / out[2]) + out[2])
    return 9 * (C + C1) + worst + 2


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("B,H,W,C,C1", SIGMA + PST900 + ODD + EDGE)
def test_ops_against_fp64(B, H, W, C, C1, mode):
    x, w1, b1, w2, b2, dy = _inputs(B, H, W, C, C1)
    o, bufs = _run(x, w1, b1, w2, b2, dy, mode)
    vals, bounds = _ref64(x, w1, b1, w2, b2, dy, mode, _seq_terms(B, H, W, C, C1))
    worst = {}
    for name, got, ref, bound in zip(("y", "pre", "dx", "dW1", "db1", "dW2", "db2"),
                                     (o["y"], o["pre"], o["dx"], o["dw1"], o["db1"], o["dw2"], o["db2"]), vals, bounds):
        err = (got.cpu().double() - ref).abs()
        ratio = float((err / (bound + 1e-30)).max())
        worst[name] = ratio
        assert bool(got.isfinite().all()), name
        assert ratio <= 1.0, (name, ratio, float(err.max()))
    for k, b in bufs.items():
        guard_ok(b, k)
    record("cab_conv_fp64", shape=[B, H, W, C, C1], mode=mode, **{k: round(v, 4) for k, v in worst.items()})


def _node_grads(x, w1, b1, w2, b2, dy):
    from sigma_b200 import ops
    args = [t.cuda().requires_grad_(True) for t in (x, w1, b1, w2, b2)]
    y = ops.CabConvFn.apply(*args)
    y.backward(dy.cuda())
    return [y.detach()] + [a.grad for a in args]


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
def test_backward_is_bitwise_reproducible(mode):
    inp = _inputs(2, 60, 80, 192, 64)
    prev = torch.are_deterministic_algorithms_enabled()
    runs = []
    try:
        with _precision(mode):
            for det in (False, False, True, True):
                torch.use_deterministic_algorithms(det)
                runs.append(_node_grads(*inp))
    finally:
        torch.use_deterministic_algorithms(prev)
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def _block(C, seed=SEED):
    from sigma_b200 import modules as M
    torch.manual_seed(seed)
    blk = M.CVSSDecoderBlock(hidden_dim=C, norm_layer=nn.LayerNorm, d_state=16).cuda().train()
    with torch.no_grad():
        for p in blk.parameters():
            if p.dim() == 1:                  # biases, scales and norm weights off their initial values
                p.add_(0.05 * torch.randn_like(p))
    return blk


def _block_step(blk, x):
    x = x.clone().requires_grad_(True)
    y = blk(x)
    loss = (y * torch.linspace(-1, 1, y.numel(), device=y.device).view_as(y)).sum()
    loss.backward()
    grads = {n: p.grad.clone() for n, p in blk.named_parameters()}
    blk.zero_grad(set_to_none=True)
    return loss.detach(), x.grad, grads


@contextlib.contextmanager
def _switch(on):
    from sigma_b200 import ops
    prev = ops.FUSED_CAB_TRAINING
    ops.FUSED_CAB_TRAINING = on
    try:
        yield
    finally:
        ops.FUSED_CAB_TRAINING = prev


@pytest.mark.parametrize("C,HW", [(96, (30, 40)), (192, (15, 20)), (384, (8, 10))])
def test_block_matches_the_cudnn_route(C, HW, monkeypatch):
    from sigma_b200 import ops
    blk = _block(C)
    x = torch.randn(2, *HW, C, generator=torch.Generator().manual_seed(SEED + C)).cuda()
    calls = []
    apply0 = ops.CabConvFn.apply
    monkeypatch.setattr(ops.CabConvFn, "apply", lambda *a: (calls.append(1), apply0(*a))[1])
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with _precision("tf32x3"):
            with _switch(True):
                new = _block_step(blk, x)
            assert calls == [1]
            with _switch(False):
                old = _block_step(blk, x)
            assert calls == [1]
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    worst = {}
    for name, a, b in [("loss", new[0], old[0]), ("dx", new[1], old[1])] + [(n, new[2][n], old[2][n]) for n in new[2]]:
        scale = float(b.abs().max()) + 1e-30
        rel = float((a - b).abs().max()) / scale
        worst[name] = rel
        assert rel < 1e-4, (name, rel)
    record("cab_block_vs_cudnn", C=C, worst=max(worst.values()), worst_param=max(worst, key=worst.get))


def test_block_runs_no_3x3_conv_and_saves_less(monkeypatch):
    blk = _block(96)
    x = torch.randn(2, 30, 40, 96, generator=torch.Generator().manual_seed(SEED)).cuda()
    conv0, convs = F.conv2d, []

    def counting(inp, weight, *a, **k):
        convs.append(tuple(weight.shape[-2:]))
        return conv0(inp, weight, *a, **k)

    params = {p.untyped_storage().data_ptr() for p in blk.parameters()}

    def saved_bytes():
        seen = {}

        def pack(t):
            s = t.untyped_storage()
            if s.data_ptr() not in params:
                seen[s.data_ptr()] = s.nbytes()
            return t
        with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
            y = blk(x.clone().requires_grad_(True))
        # the kernel sizes of the graph's convolution nodes: what the backward will run
        nodes, stack, seen_nodes = [], [y.grad_fn], set()
        while stack:
            n = stack.pop()
            if n is None or n in seen_nodes:
                continue
            seen_nodes.add(n)
            nodes.append(n)
            stack.extend(f for f, _ in n.next_functions)
        kernels = [tuple(n._saved_weight.shape[-2:]) for n in nodes if "Convolution" in type(n).__name__]
        y.sum().backward()
        return sum(seen.values()), kernels

    monkeypatch.setattr(F, "conv2d", counting)
    with _switch(True):
        new, kernels = saved_bytes()
    assert all(s == (1, 1) for s in convs), convs                    # forward: only the attention's 1x1 convs
    assert kernels and all(k == (1, 1) for k in kernels), kernels     # backward: no 3x3 convolution node in the graph
    with _switch(False):
        old, _ = saved_bytes()
    assert new < old, (new, old)
    record("cab_saved_bytes", new=new, old=old)


@pytest.mark.parametrize("case", ["hidden32", "bf16", "fp16", "composed", "switch_off"])
def test_fallbacks_do_not_take_the_route(case, monkeypatch):
    from sigma_b200 import modules as M, ops
    blk = _block(32 if case == "hidden32" else 96)
    x = torch.randn(2, 12, 16, blk.norm2.normalized_shape[0], device="cuda", requires_grad=True)
    calls = []
    apply0 = ops.CabConvFn.apply
    monkeypatch.setattr(ops.CabConvFn, "apply", lambda *a: (calls.append(1), apply0(*a))[1])
    ctx = {"bf16": torch.autocast("cuda", dtype=torch.bfloat16), "fp16": torch.autocast("cuda", dtype=torch.float16),
           "composed": M.composed_path(), "switch_off": _switch(False)}.get(case, contextlib.nullcontext())
    with ctx:
        y = blk(x)
    y.float().sum().backward()
    assert calls == []
    if case != "hidden32":                                    # the same block outside the fallback's condition takes it
        with _switch(True):
            blk(x)
        assert calls == [1]
