"""GPU: the depthwise conv3x3 + SiLU backward (sigma_dwconv3x3_silu_bwd[_bf16|_fp16]) and the autograd node that trains the Mamba
blocks through it (ops.DwConvSiLUFn).

* Op level against torch CPU float64 autograd of F.conv2d(groups=D) + SiLU, element by element: every Sigma-tiny training shape at
  480 x 640 with batch 2 (SS2D's encoder stages as 4 images, ConMB per modality, CroMB at 2B, the decoder's stages), Sigma-base's
  23 x 30 stage, ragged tiles (H % 8, W % 16, H = 1, W = 1, D not a multiple of 32).  The fp32 bounds scale with the sum of |terms|
  of each output (as the forward's test does), with the sums of dw / db held to (terms added in sequence)·u; 16-bit adds one store
  of dx.  Layouts: x as the strided x half of [x | z] rows; dy and dx as the second half of each image of a (B, 2L, D) buffer (the
  ConMB slice).  NaN guards around dx, and the first halves of the ConMB buffer, must keep their bits.
* Two backward calls give the same bits, with and without torch.use_deterministic_algorithms(True).
* Blocks: no depthwise F.conv2d runs on the fused-core route in fp32, bf16 and fp16 autocast (core on and off), and the saved
  tensors of a block's training forward fall by one conv output per conv against the torch conv.
* A whole-model Sigma-tiny fp16 step with the fp16 core and a GradScaler, with cuDNN enabled, after a ConMB block's fp16 training
  step in the same process."""
import contextlib
import io
import math

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import procedural as P
from helpers import SEED, cfg_tiny, guard_ok, guarded, record

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
ROUND16 = {torch.bfloat16: (2.0 ** -8, 0.0), torch.float16: (2.0 ** -11, 2.0 ** -25)}   # relative half-ulp store bound, subnormal step
BWD = {torch.float32: "sigma_dwconv3x3_silu_bwd", torch.bfloat16: "sigma_dwconv3x3_silu_bwd_bf16",
       torch.float16: "sigma_dwconv3x3_silu_bwd_fp16"}

# (B, H, W, D, layout): Sigma-tiny at 480 x 640, batch 2 -- SS2D encoder (rgb and x batched: 4 images, x the half of [x | z]),
# CroMB (2B = 4 images), ConMB per modality and the decoder (2 images, dy / dx slices of the (B, 2L, D) core input)
TINY = [(4, 120, 160, 192, "ss2d"), (4, 60, 80, 384, "ss2d"), (4, 30, 40, 768, "ss2d"), (4, 15, 20, 1536, "ss2d"),
        (4, 30, 40, 768, "plain"),
        (2, 120, 160, 192, "conmb"), (2, 60, 80, 384, "conmb"), (2, 30, 40, 768, "conmb"), (2, 15, 20, 1536, "conmb"),
        (2, 60, 80, 384, "plain")]
OTHER = [(2, 23, 30, 2048, "ss2d"),                                                   # Sigma-base's 23 x 30 stage
         (1, 13, 21, 136, "plain"), (3, 1, 37, 136, "conmb"), (2, 29, 1, 136, "ss2d"), (1, 1, 1, 8, "plain"), (2, 9, 17, 40, "ss2d")]


def _parts(B, H, W, D):
    """the launch plan's persistent CTAs per channel block, as dwconv_bwd_parts computes it"""
    ntiles = B * math.ceil(W / 16) * math.ceil(H / 8)
    return max(1, min(ntiles, 132 * 2 // math.ceil(D / 32))), ntiles


def _ref64(x, w, b, dy):
    """float64 autograd of F.conv2d(groups=D) + SiLU on CPU (x, dy (B, H, W, D) exact widened values), and the bounds of the kernel's
    fp32 arithmetic: y, dx, dw, db and their bounds"""
    D = x.shape[-1]
    xn = x.double().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    wd, bd = w.double().requires_grad_(True), b.double().requires_grad_(True)
    pre = F.conv2d(xn, wd, bd, padding=1, groups=D)
    y = F.silu(pre)
    dyn = dy.double().permute(0, 3, 1, 2)
    dx, dw, db = torch.autograd.grad(y, (xn, wd, bd), dyn)
    with torch.no_grad():
        pre = pre.detach()
        mag = F.conv2d(xn.detach().abs(), wd.detach().abs(), bd.detach().abs(), padding=1, groups=D)
        y_b = 1.1 * 10 * U * mag + 2.0 ** -19 * y.detach().abs() + 1e-12
        s = torch.sigmoid(pre)
        g = dyn * s * (1 + pre * (1 - s))
        # g: the recomputed pre (<= 10u·mag, |SiLU''| <= 0.5), ex2.approx / fast division and the four products (a few ulp)
        e_g = dyn.abs() * (0.5 * 10 * U * mag + 2.0 ** -18 * (1 + pre.abs()))
        aw = wd.detach().abs()
        dx_b = torch.nn.grad.conv2d_input(xn.shape, aw, e_g + 10 * U * g.abs(), padding=1, groups=D) + 1e-12
        B, _, H, W = xn.shape
        ny, ntiles = _parts(B, H, W, D)
        nadd = math.ceil(ntiles / ny) * 8 + 16 + ny + 2             # terms one dw / db element adds in sequence
        ax = xn.detach().abs()
        dw_b = torch.nn.grad.conv2d_weight(ax, wd.shape, e_g + nadd * U * g.abs(), padding=1, groups=D) + 1e-12
        db_b = (e_g + nadd * U * g.abs()).sum(dim=(0, 2, 3)) + 1e-12
    cl = lambda t: t.permute(0, 2, 3, 1)
    return cl(y.detach()), cl(y_b), cl(dx), cl(dx_b), dw, dw_b, db, db_b


def _store16(ref, e, dtype):
    rel, sub = ROUND16[dtype]
    return e + rel * (ref.abs() + e) + sub


def _check(tag, got, ref, bound):
    got = got.double().cpu()
    assert bool(torch.isfinite(got).all()), f"{tag}: non-finite values (not written?)"
    err = (got - ref).abs()
    bad = err > bound
    assert not bool(bad.any()), (f"{tag}: {int(bad.sum())}/{bad.numel()} out of bound; max err {float(err.max()):.3e}, "
                                 f"worst err/bound {float((err / bound).max()):.2f}")
    return float((err / bound).max())


def _inputs(B, H, W, D, dtype, tag):
    x = P.randn(SEED, f"dwt/{tag}/x", (B, H, W, D)).to(dtype)
    w = P.randn(SEED, f"dwt/{tag}/w", (D, 1, 3, 3), scale=0.3)
    b = P.randn(SEED, f"dwt/{tag}/b", (D,), scale=0.5)
    dy = P.randn(SEED, f"dwt/{tag}/dy", (B, H, W, D)).to(dtype)
    return x, w, b, dy


def _bwd(dtype, x, w, b, dy, layout):
    """the C backward with the layout's strides -> dx (B, H, W, D), dw, db, after checking that nothing outside them was written"""
    from sigma_b200 import _lib
    from sigma_b200._lib import ptr, stream
    B, H, W, D = x.shape
    L = H * W
    if layout == "ss2d":
        xz = torch.full((B, H, W, 2 * D), float("nan"), dtype=dtype, device="cuda")
        xz[..., :D] = x.cuda()
        xd, xrs, xbs = xz[..., :D], 2 * D, L * 2 * D
    else:
        xd, xrs, xbs = x.cuda().contiguous(), D, L * D
    if layout == "conmb":                        # dy and dx: the second half of every image of (B, 2L, D)
        dyb = torch.full((B, 2 * L, D), float("nan"), dtype=dtype, device="cuda")
        dyb[:, L:] = dy.cuda().reshape(B, L, D)
        dyd, dybs = dyb[:, L:], 2 * L * D
        dxbuf, dxall = guarded((B, 2 * L, D), dtype)
        dxd, dxbs = dxall[:, L:], 2 * L * D
    else:
        dyd, dybs = dy.cuda().contiguous(), L * D
        dxbuf, dxall = guarded((B, L, D), dtype)
        dxd, dxbs = dxall, L * D
    wc, bc = w.cuda(), b.cuda()
    dwbuf, dw = guarded((D, 1, 3, 3))
    dbbuf, db = guarded((D,))
    L_ = _lib.lib()
    wsb = L_.sigma_dwconv3x3_silu_bwd_workspace_bytes(B, H, W, D)
    ws = torch.full((wsb,), 0xFF, dtype=torch.uint8, device="cuda")
    fn = BWD[dtype]
    _lib.check(getattr(L_, fn)(ptr(xd), xrs, xbs, ptr(wc), ptr(bc), ptr(dyd), dybs, ptr(dxd), dxbs, ptr(dw), ptr(db), B, H, W, D, ptr(ws),
                               wsb, stream()), fn)
    torch.cuda.synchronize()
    guard_ok(dxbuf, f"{fn} dx")
    guard_ok(dwbuf, f"{fn} dw")
    guard_ok(dbbuf, f"{fn} db")
    if layout == "conmb":                        # the first halves are another tensor's: untouched
        guard_ok(torch.cat([torch.full((64,), float("nan"), dtype=dtype, device="cuda"), dxall[:, :L].reshape(-1),
                            torch.full((64,), float("nan"), dtype=dtype, device="cuda")]), f"{fn} dx first halves")
    return dxd.reshape(B, H, W, D), dw, db


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("B,H,W,D,layout", TINY + OTHER)
def test_backward_against_fp64(B, H, W, D, layout, dtype):
    tag = f"{B}x{H}x{W}x{D}/{layout}"
    x, w, b, dy = _inputs(B, H, W, D, dtype, tag)
    dx, dw, db = _bwd(dtype, x, w, b, dy, layout)
    _, _, rdx, dx_b, rdw, dw_b, rdb, db_b = _ref64(x.float(), w, b, dy.float())
    if dtype != torch.float32:
        dx_b = _store16(rdx, dx_b, dtype)
    worst = {"dx": _check(f"{tag} dx", dx, rdx, dx_b), "dw": _check(f"{tag} dw", dw, rdw, dw_b), "db": _check(f"{tag} db", db, rdb, db_b)}
    ny, ntiles = _parts(B, H, W, D)
    record("dwconv_bwd", case=tag, dtype=str(dtype), tiles_per_cta=round(ntiles / ny, 2), **worst)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=["fp32", "bf16", "fp16"])
def test_node_forward_backward_against_fp64(dtype):
    """ops.DwConvSiLUFn on the x half of [x | z] rows, under autocast of its dtype (which must not cast the fp32 weights)"""
    from sigma_b200 import ops
    B, H, W, D = 2, 30, 40, 192
    x, w, b, dy = _inputs(B, H, W, D, dtype, "node")
    xz = torch.cat([x, x], dim=-1).cuda().requires_grad_(True)
    conv = nn.Conv2d(D, D, 3, padding=1, groups=D).cuda()
    with torch.no_grad():
        conv.weight.copy_(w)
        conv.bias.copy_(b)
    amp = dtype != torch.float32
    with torch.autocast("cuda", dtype=dtype if amp else torch.bfloat16, enabled=amp):
        y = ops.DwConvSiLUFn.apply(xz[..., :D], conv.weight, conv.bias)
    assert y.dtype == dtype and y.shape == (B, H * W, D)
    y.backward(dy.cuda().reshape(B, H * W, D))
    ry, y_b, rdx, dx_b, rdw, dw_b, rdb, db_b = _ref64(x.float(), w, b, dy.float())
    if amp:
        y_b, dx_b = _store16(ry, y_b, dtype), _store16(rdx, dx_b, dtype)
    assert conv.weight.grad.dtype == conv.bias.grad.dtype == torch.float32
    assert conv.weight.grad.shape == (D, 1, 3, 3) and conv.bias.grad.shape == (D,)
    assert float(xz.grad[..., D:].abs().max()) == 0.0
    worst = {"y": _check("node y", y.reshape(B, H, W, D), ry, y_b), "dx": _check("node dx", xz.grad[..., :D], rdx, dx_b),
             "dw": _check("node dw", conv.weight.grad, rdw, dw_b), "db": _check("node db", conv.bias.grad, rdb, db_b)}
    record("dwconv_node", dtype=str(dtype), **worst)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=["fp32", "bf16", "fp16"])
def test_backward_is_bitwise_reproducible(dtype):
    """the same bits from two calls, and from a call under torch.use_deterministic_algorithms(True): one kernel either way"""
    from sigma_b200 import ops
    B, H, W, D = 4, 60, 80, 384
    x, w, b, dy = _inputs(B, H, W, D, dtype, "det")
    xc, dyc = x.cuda(), dy.cuda().reshape(B, H * W, D)
    conv = nn.Conv2d(D, D, 3, padding=1, groups=D).cuda()
    outs = []
    for det in (False, False, True):
        prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(det)
        try:
            xi = xc.clone().requires_grad_(True)
            conv.zero_grad(set_to_none=True)
            ops.DwConvSiLUFn.apply(xi, conv.weight, conv.bias).backward(dyc)
            torch.cuda.synchronize()
            outs.append((xi.grad.clone(), conv.weight.grad.clone(), conv.bias.grad.clone()))
        finally:
            torch.use_deterministic_algorithms(prev)
    bits = lambda t: t.view({4: torch.int32, 2: torch.int16}[t.element_size()])
    for o in outs[1:]:
        for a, r in zip(o, outs[0]):
            assert torch.equal(bits(a), bits(r))


def _blocks():
    from sigma_b200 import modules as M
    x1 = P.randn(SEED, "dwt/blk/x", (2, 12, 10, 32)).cuda()
    x2 = P.randn(SEED, "dwt/blk/x2", (2, 12, 10, 32)).cuda()
    return {
        "vssblock": (lambda: M.VSSBlock(hidden_dim=32, norm_layer=nn.LayerNorm, mlp_ratio=0.0, d_state=16), (x1,), 1),
        "conmb": (lambda: M.ConcatMambaFusionBlock(hidden_dim=32, mlp_ratio=0.0, d_state=4), (x1, x2), 2),
        "cromb": (lambda: M.CrossMambaFusionBlock(hidden_dim=32, mlp_ratio=0.0, d_state=4), (x1, x2), 1),
        "cvss_dec": (lambda: M.CVSSDecoderBlock(hidden_dim=32, norm_layer=nn.LayerNorm, d_state=4, mlp_ratio=4.0), (x1,), 1),
    }


MODES = {"fp32": (None, None), "bf16": (torch.bfloat16, False), "bf16_core": (torch.bfloat16, True), "fp16": (torch.float16, False),
         "fp16_core": (torch.float16, True)}


def _mode_ctx(mode):
    from sigma_b200 import ops
    dt, core = MODES[mode]
    if dt is None:
        return contextlib.nullcontext()
    stack = contextlib.ExitStack()
    stack.enter_context(torch.autocast("cuda", dtype=dt))
    stack.enter_context((ops.bf16_training_core if dt == torch.bfloat16 else ops.fp16_training_core)(core))
    return stack


def _flat(y):
    return torch.cat([t.float().reshape(-1) for t in (y if isinstance(y, (tuple, list)) else (y,))])


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", ["vssblock", "conmb", "cromb", "cvss_dec"])
def test_blocks_make_no_depthwise_torch_conv(name, mode, monkeypatch):
    from sigma_b200 import ops
    make, xs, nconv = _blocks()[name]
    torch.manual_seed(SEED)
    blk = make().cuda().train()
    depthwise, node, conv0, apply0 = [], [], F.conv2d, ops.DwConvSiLUFn.apply

    def counting_conv(inp, weight, bias=None, stride=1, padding=0, dilation=1, groups=1):
        if groups > 1 and groups == inp.shape[1]:
            depthwise.append(tuple(inp.shape))
        return conv0(inp, weight, bias, stride, padding, dilation, groups)

    monkeypatch.setattr(F, "conv2d", counting_conv)
    monkeypatch.setattr(ops.DwConvSiLUFn, "apply", lambda *a: (node.append(a[0].dtype), apply0(*a))[1])
    xs = [x.clone().requires_grad_(True) for x in xs]
    with _mode_ctx(mode):
        y = _flat(blk(*xs))
    y.sum().backward()
    torch.cuda.synchronize()
    assert depthwise == [], depthwise
    assert len(node) == nconv, node
    assert all(p.grad is not None and bool(p.grad.isfinite().all()) for n, p in blk.named_parameters() if "conv2d" in n)
    record("dwconv_route", block=name, mode=mode, node_calls=len(node), node_dtypes=str(sorted(set(map(str, node)))))


def _torch_conv_node(x, weight, bias):
    """the torch route the node replaced: channels-last x through nn.Conv2d's F.conv2d and F.silu -> (B, H·W, D)"""
    B, H, W, D = x.shape
    return F.silu(F.conv2d(x.permute(0, 3, 1, 2), weight, bias, padding=1, groups=D)).permute(0, 2, 3, 1).reshape(B, H * W, D)


@pytest.mark.parametrize("name", ["vssblock", "conmb", "cromb"])
def test_saved_tensors_fall_by_one_conv_output_per_conv(name, monkeypatch):
    from sigma_b200 import ops
    make, xs, nconv = _blocks()[name]
    torch.manual_seed(SEED)
    blk = make().cuda().train()
    B, H, W, C = xs[0].shape
    per_conv = (2 * B if name == "cromb" else B) * H * W * 2 * C * 4            # one fp32 conv output (D = 2·C)

    params = {p.untyped_storage().data_ptr() for p in blk.parameters()}

    def saved_bytes():
        """bytes of the distinct activation storages the forward saves (parameters excluded: they are held anyway)"""
        seen = {}

        def pack(t):
            s = t.untyped_storage()
            if s.data_ptr() not in params:
                seen[s.data_ptr()] = s.nbytes()
            return t
        with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
            y = _flat(blk(*[x.clone().requires_grad_(True) for x in xs]))
        y.sum().backward()
        return sum(seen.values())

    new = saved_bytes()
    with monkeypatch.context() as m:
        m.setattr(ops.DwConvSiLUFn, "apply", _torch_conv_node)
        old = saved_bytes()
    record("dwconv_saved_bytes", block=name, torch_conv=old, node=new, per_conv=per_conv, convs=nconv)
    assert old - new == nconv * per_conv, (old, new, per_conv)


def test_fp16_whole_model_step_with_cudnn_enabled():
    """With cuDNN on: a ConMB block takes an fp16 training step, then a whole Sigma-tiny step with TrainStep(fp16_core=True,
    scaler=GradScaler()) gives a finite loss, applies the step, and lands within 1e-2 of the same step with cuDNN off."""
    from sigma_b200 import modules as M, train_util
    assert torch.backends.cudnn.enabled
    torch.manual_seed(SEED)
    blk = M.ConcatMambaFusionBlock(hidden_dim=32, mlp_ratio=0.0, d_state=4).cuda().train()
    xs = [P.randn(SEED, f"dwt/cudnn/{k}", (2, 12, 10, 32)).cuda().requires_grad_(True) for k in ("x", "x2")]
    with _mode_ctx("fp16_core"):
        y = _flat(blk(*xs))
    y.sum().backward()
    assert all(bool(p.grad.isfinite().all()) for p in blk.parameters() if p.grad is not None)
    H, W, ncls = 64, 96, 9
    rgb = P.randn(SEED, "dwt/cudnn/rgb", (2, 3, H, W)).cuda()
    mx = P.randn(SEED, "dwt/cudnn/mx", (2, 3, H, W)).cuda()
    gt = (P.rand(SEED, "dwt/cudnn/gt", (2, H, W), 0, ncls).long() % ncls).cuda()
    losses, decision = {}, {}
    for cudnn in (True, False):
        torch.manual_seed(SEED)
        with contextlib.redirect_stdout(io.StringIO()):
            model = M.EncoderDecoder(cfg_tiny(H, W, num_classes=ncls),
                                     criterion=nn.CrossEntropyLoss(reduction="mean", ignore_index=255)).cuda().train()
        scaler = torch.amp.GradScaler("cuda")
        step = train_util.TrainStep(model, train_util.make_optimizer(model), amp_dtype=torch.float16, fp16_core=True, scaler=scaler)
        scale0 = scaler.get_scale()
        with torch.backends.cudnn.flags(enabled=cudnn):
            loss = step(rgb, mx, gt)
        losses[cudnn] = float(loss.detach())
        decision[cudnn] = "applied" if scaler.get_scale() >= scale0 else "skipped"
    record("fp16 step with cudnn", loss_on=losses[True], loss_off=losses[False], scaler_on=decision[True], scaler_off=decision[False])
    assert math.isfinite(losses[True]) and decision[True] == "applied", (losses, decision)
    assert abs(losses[True] - losses[False]) <= 1e-2 * abs(losses[False]), losses
