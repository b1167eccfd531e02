"""GPU: the pitched 3x3 conv entry points (sigma_conv3x3_{,gelu_save_,dgrad_,wgrad_}pitched_tf32) and what runs on them: the
training node ops.CabConvPitchedFn and the inference route fused.cab_convs_pitched, for ChannelAttentionBlocks whose C/3 is not a
multiple of 4 (Sigma-base's 42 / 85 / 170, hidden 32's 10).

* Op level against torch CPU float64 autograd, element by element, with the bounds of test_cab_conv_train_gpu._ref64: y, pre, dx,
  dW1, db1, dW2, db2 at Sigma-base's decoder stages (720 x 960 batch 1, 480 x 640 batch 2), hidden 32 and edge shapes (C1 = 1, 2,
  3, 5, 33; H = 1; W = 1; H, W not multiples of 8 / 16); TF32 and tf32x3.  NaN guards around every output keep their bits.
* Pad poisoning: the pad channels of h, pre, dpre and of the padded weights filled with 0, NaN and +inf give bit-identical kept
  outputs, and no call writes a pad channel.
* With every pitch equal to its count (Sigma-tiny's multiples of 4), the pitched entry points give the unpitched ones' bits: the
  plans are the same.
* Two backward calls of the node give the same bits, with torch.use_deterministic_algorithms(True) off and on.
* CVSSDecoderBlock at hidden 128 / 256 / 512 / 32 takes CabConvPitchedFn, matches the cuDNN route at fp32 grade, and runs no 3x3
  convolution forward or backward.
* A Sigma-base model's fused inference forward runs no 3x3 F.conv2d and matches the cuDNN route.
* A graph-replayed Sigma-base training step runs with no host synchronisation, a finite loss, and agrees with the eager step."""
import contextlib
import io
import math

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import procedural as P
from helpers import SEED, cfg_tiny, guard_ok, guarded, record
from test_cab_conv_train_gpu import _block, _block_step, _inputs, _precision, _ref64, _run, _seq_terms, _switch

pytestmark = pytest.mark.gpu

# (B, H, W, C, C1): the first conv maps C -> C1, the second C1 -> C
BASE_720 = [(1, 180, 240, 128, 42), (1, 90, 120, 256, 85), (1, 45, 60, 512, 170)]
BASE_480 = [(2, 120, 160, 128, 42), (2, 60, 80, 256, 85), (2, 30, 40, 512, 170)]
HIDDEN32 = [(2, 12, 16, 32, 10)]
EDGE = [(1, 1, 1, 12, 1), (1, 1, 37, 8, 2), (2, 29, 1, 12, 3), (1, 13, 21, 20, 5), (2, 9, 17, 100, 33), (1, 5, 7, 64, 21)]
TINY = [(2, 120, 160, 96, 32), (2, 60, 80, 192, 64), (2, 30, 40, 384, 128)]
NAMES = ("y", "pre", "dx", "dW1", "db1", "dW2", "db2")


def _r4(n):
    return (n + 3) // 4 * 4


def _weights(w, x3, grad, pitch, fill):
    """ops._w9 with the pad columns of hi (and lo) set to `fill`"""
    from sigma_b200 import ops
    hi, lo = ops._w9(w, x3, grad=grad, pitch=pitch)
    width = w.shape[0] if grad else w.shape[1]
    for t in (hi, lo):
        if t is not None and pitch > width:
            t[:, width:] = fill
    return hi, lo


def _run_pitched(x, w1, b1, w2, b2, dy, mode, fill=float("nan"), k1=None):
    """the node's calls on the pitched entry points, each output in a NaN-guarded buffer whose interior starts as `fill` (so the
    pads of h, pre and dpre hold it), the padded weights' pads `fill` too -> (outputs with h / pre / dpre at pitch k1, guards)"""
    from sigma_b200 import _lib
    from sigma_b200._lib import ptr, stream
    L = _lib.lib()
    B, H, W, C = x.shape
    C1 = w1.shape[0]
    k1 = k1 or _r4(C1)
    x3 = mode == "tf32x3"
    x, w1, b1, w2, b2, dy = (t.cuda().contiguous() for t in (x, w1, b1, w2, b2, dy))
    shapes = dict(h=(B, H, W, k1), pre=(B, H, W, k1), y=(B, H, W, C), dpre=(B, H, W, k1), dx=(B, H, W, C),
                  dw1=(C1, C, 3, 3), db1=(C1,), dw2=(C, C1, 3, 3), db2=(C,))
    bufs, o = {}, {}
    for k, s in shapes.items():
        bufs[k], o[k] = guarded(s)
        o[k].fill_(fill)
    hi, lo = _weights(w1, x3, False, C, fill)
    _lib.check(L.sigma_conv3x3_gelu_save_pitched_tf32(ptr(x), C, ptr(hi), C, ptr(lo), ptr(b1), ptr(o["h"]), ptr(o["pre"]), k1, B, H, W,
                                                      C, C1, stream()), "save")
    hi, lo = _weights(w2, x3, False, k1, fill)
    _lib.check(L.sigma_conv3x3_pitched_tf32(ptr(o["h"]), k1, ptr(hi), k1, ptr(lo), ptr(b2), 0, ptr(o["y"]), C, B, H, W, C1, C, stream()),
               "conv")

    def wgrad(xin, xp, gelu_x, g, gp, dw, db, cin, cout):
        wsb = L.sigma_conv3x3_wgrad_workspace_bytes(B, H, W, cin, cout)
        ws = torch.full((wsb,), 255, dtype=torch.uint8, device="cuda")
        _lib.check(L.sigma_conv3x3_wgrad_pitched_tf32(ptr(xin), xp, gelu_x, ptr(g), gp, ptr(dw), ptr(db), B, H, W, cin, cout, int(x3),
                                                      ptr(ws), wsb, stream()), "wgrad")

    wgrad(o["pre"], k1, 1, dy, C, o["dw2"], o["db2"], C1, C)
    hi, lo = _weights(w2, x3, True, C, fill)
    _lib.check(L.sigma_conv3x3_dgrad_pitched_tf32(ptr(dy), C, ptr(hi), C, ptr(lo), ptr(o["pre"]), ptr(o["dpre"]), k1, B, H, W, C1, C,
                                                  stream()), "dgrad2")
    wgrad(x, C, 0, o["dpre"], k1, o["dw1"], o["db1"], C, C1)
    hi, lo = _weights(w1, x3, True, k1, fill)
    _lib.check(L.sigma_conv3x3_dgrad_pitched_tf32(ptr(o["dpre"]), k1, ptr(hi), k1, ptr(lo), None, ptr(o["dx"]), C, B, H, W, C, C1,
                                                  stream()), "dgrad1")
    torch.cuda.synchronize()
    return o, bufs


def _kept(o, C1):
    return [o["y"], o["pre"][..., :C1], o["dx"], o["dw1"], o["db1"], o["dw2"], o["db2"]]


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("B,H,W,C,C1", BASE_720 + BASE_480 + HIDDEN32 + EDGE)
def test_ops_against_fp64(B, H, W, C, C1, mode):
    x, w1, b1, w2, b2, dy = _inputs(B, H, W, C, C1)
    o, bufs = _run_pitched(x, w1, b1, w2, b2, dy, mode)
    vals, bounds = _ref64(x, w1, b1, w2, b2, dy, mode, _seq_terms(B, H, W, C, C1))
    worst = {}
    for name, got, ref, bound in zip(NAMES, _kept(o, C1), vals, bounds):
        err = (got.cpu().double() - ref).abs()
        ratio = float((err / (bound + 1e-30)).max())
        worst[name] = ratio
        assert bool(got.isfinite().all()), name
        assert ratio <= 1.0, (name, ratio, float(err.max()))
    for k, b in bufs.items():
        guard_ok(b, k)
    record("cab_conv_pitched_fp64", shape=[B, H, W, C, C1], mode=mode, **{k: round(v, 4) for k, v in worst.items()})


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("B,H,W,C,C1", [(1, 45, 60, 512, 170), (2, 9, 17, 100, 33), (1, 13, 21, 20, 5)])
def test_pad_contents_never_reach_a_kept_output(B, H, W, C, C1, mode):
    inp = _inputs(B, H, W, C, C1)
    runs = {}
    for name, fill in (("zero", 0.0), ("nan", float("nan")), ("inf", float("inf"))):
        o, bufs = _run_pitched(*inp, mode, fill=fill)
        for k, b in bufs.items():
            guard_ok(b, k)
        for k in ("h", "pre", "dpre"):                          # no call writes a pad channel
            pad = o[k][..., C1:]
            assert torch.equal(_bits(pad), _bits(torch.full_like(pad, fill))), (name, k)
        runs[name] = _kept(o, C1)
        assert all(bool(t.isfinite().all()) for t in runs[name]), name
    for name in ("nan", "inf"):
        for k, a, b in zip(NAMES, runs["zero"], runs[name]):
            assert torch.equal(_bits(a), _bits(b)), (name, k)


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("B,H,W,C,C1", TINY)
def test_pitch_equal_to_count_gives_the_unpitched_bits(B, H, W, C, C1, mode):
    inp = _inputs(B, H, W, C, C1)
    new, _ = _run_pitched(*inp, mode, k1=C1)
    old, _ = _run(*inp, mode)
    for k in old:
        assert torch.equal(_bits(new[k]), _bits(old[k])), k


def _node_grads(x, w1, b1, w2, b2, dy):
    from sigma_b200 import ops
    args = [t.cuda().requires_grad_(True) for t in (x, w1, b1, w2, b2)]
    y = ops.CabConvPitchedFn.apply(*args)
    y.backward(dy.cuda())
    return [y.detach()] + [a.grad for a in args]


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
def test_backward_is_bitwise_reproducible(mode):
    inp = _inputs(2, 60, 80, 256, 85)
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
            assert torch.equal(_bits(a), _bits(b))


BLOCKS = [(128, (30, 40)), (256, (15, 20)), (512, (8, 10)), (32, (12, 16))]
# Both routes are fp32 grade but not the same arithmetic: tf32x3's products carry up to 4·2^-20 relative error where cuDNN's fp32 has
# 2^-24, and a conv output is a sum of 9·C signed terms (at C = 512, sqrt(9·C) ~ 68 times its value in magnitude), so an element of
# t may differ by ~2.6e-4 of itself.  The bias and attention gradients then sum such elements over the pixels with the loss's signed
# weights.  CabConvFn's own block test reaches 7.9e-5 of the largest gradient at C = 384; 2e-4 leaves room for C = 512 and for
# hidden 32's short sums.  The op-level test bounds every kernel output element by element.
BLOCK_BAR = 2e-4


@pytest.mark.parametrize("C,HW", BLOCKS, ids=[f"hidden{c}" for c, _ in BLOCKS])
def test_block_matches_the_cudnn_route(C, HW, monkeypatch):
    from sigma_b200 import ops
    blk = _block(C)
    x = torch.randn(2, *HW, C, generator=torch.Generator().manual_seed(SEED + C)).cuda()
    calls, other = [], []
    apply0, apply1 = ops.CabConvPitchedFn.apply, ops.CabConvFn.apply
    monkeypatch.setattr(ops.CabConvPitchedFn, "apply", lambda *a: (calls.append(1), apply0(*a))[1])
    monkeypatch.setattr(ops.CabConvFn, "apply", lambda *a: (other.append(1), apply1(*a))[1])
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with _precision("tf32x3"):
            with _switch(True):
                new = _block_step(blk, x)
            assert calls == [1] and other == []
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
        assert rel < BLOCK_BAR, (name, rel)
    record("cab_pitched_block_vs_cudnn", C=C, worst=max(worst.values()), worst_param=max(worst, key=worst.get))


@pytest.mark.parametrize("C", [128, 32])
def test_block_runs_no_3x3_conv(C, monkeypatch):
    blk = _block(C)
    x = torch.randn(2, 12, 16, C, generator=torch.Generator().manual_seed(SEED)).cuda()
    conv0, convs = F.conv2d, []

    def counting(inp, weight, *a, **k):
        convs.append(tuple(weight.shape[-2:]))
        return conv0(inp, weight, *a, **k)

    monkeypatch.setattr(F, "conv2d", counting)
    with _switch(True):
        y = blk(x.clone().requires_grad_(True))
    nodes, stack, seen = [], [y.grad_fn], set()
    while stack:
        n = stack.pop()
        if n is None or n in seen:
            continue
        seen.add(n)
        nodes.append(n)
        stack.extend(f for f, _ in n.next_functions)
    kernels = [tuple(n._saved_weight.shape[-2:]) for n in nodes if "Convolution" in type(n).__name__]
    y.sum().backward()
    assert all(s == (1, 1) for s in convs), convs                    # forward: only the attention's 1x1 convs
    assert kernels and all(k == (1, 1) for k in kernels), kernels     # backward: no 3x3 convolution node in the graph
    assert any(type(n).__name__ == "CabConvPitchedFnBackward" for n in nodes)


def _base_model(Hh, Ww, train=False):
    from sigma_b200 import modules as M
    torch.manual_seed(SEED)
    crit = nn.CrossEntropyLoss(reduction="mean", ignore_index=255) if train else None
    with contextlib.redirect_stdout(io.StringIO()):
        model = M.EncoderDecoder(cfg_tiny(Hh, Ww, num_classes=9 if train else 40, backbone="sigma_base"), criterion=crit)
    model = model.cuda()
    if train:
        for m in model.modules():
            if isinstance(m, M.DropPath):
                m.drop_prob = 0.0
        return model.train()
    P.fill_state_dict(model, SEED)
    return model.eval()


@pytest.mark.parametrize("mode", ["tf32x3", "tf32"])
def test_sigma_base_inference_runs_no_3x3_conv(mode, monkeypatch):
    from sigma_b200 import fused
    Hh, Ww = 96, 160
    model = _base_model(Hh, Ww)
    rgb = torch.randn(1, 3, Hh, Ww, device="cuda", generator=torch.Generator(device="cuda").manual_seed(SEED))
    mx = torch.randn(1, 3, Hh, Ww, device="cuda", generator=torch.Generator(device="cuda").manual_seed(SEED + 1))
    conv0, convs = F.conv2d, []

    def counting(inp, weight, *a, **k):
        convs.append(tuple(weight.shape[-2:]))
        return conv0(inp, weight, *a, **k)

    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = mode == "tf32"
    try:
        with _precision(mode), torch.no_grad():
            monkeypatch.setattr(F, "conv2d", counting)
            got = model(rgb, mx)
            assert (3, 3) not in convs, convs
            monkeypatch.setattr(fused, "cab_convs_pitched", lambda *a: None)     # the cuDNN route
            ref = model(rgb, mx)
            assert (3, 3) in convs
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    scale = float(ref.abs().max())
    err = float((got - ref).abs().max())
    record("cab_pitched_sigma_base_logits", mode=mode, err=err, scale=scale)
    assert err <= (1e-3 if mode == "tf32x3" else 1e-2) * scale, (err, scale)


def test_sigma_base_graphed_step_has_no_host_sync_and_matches_eager(monkeypatch):
    from sigma_b200 import ops, train_util
    Hh, Ww = 64, 96
    calls = []
    apply0 = ops.CabConvPitchedFn.apply
    monkeypatch.setattr(ops.CabConvPitchedFn, "apply", lambda *a: (calls.append(1), apply0(*a))[1])
    state = {k: v.clone() for k, v in _base_model(Hh, Ww, train=True).state_dict().items()}
    me, mg = _base_model(Hh, Ww, train=True), _base_model(Hh, Ww, train=True)
    me.load_state_dict(state)
    mg.load_state_dict(state)

    def batch(tag):
        rgb = P.randn(SEED, f"cabp/{tag}/rgb", (2, 3, Hh, Ww)).cuda()
        mx = P.randn(SEED, f"cabp/{tag}/x", (2, 3, Hh, Ww)).cuda()
        gt = (P.rand(SEED, f"cabp/{tag}/gt", (2, Hh, Ww), 0, 9).long() % 9).cuda()
        return rgb, mx, gt

    eager = train_util.TrainStep(me, train_util.make_optimizer(me, capturable=True))
    graphed = train_util.GraphedTrainStep(mg, train_util.make_optimizer(mg, capturable=True), batch("example"))
    assert calls                                                    # the decoder's CABs took the pitched node
    losses = []
    for i in range(2):
        b = batch(f"step{i}")
        le = eager(*b)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            lg = graphed(*b)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        torch.cuda.synchronize()
        losses.append((float(le), float(lg)))
    record("cab_pitched_graphed_step", losses=losses)
    for le, lg in losses:
        assert math.isfinite(lg) and abs(le - lg) <= 1e-4 * abs(le), losses
