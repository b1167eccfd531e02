"""GPU: the fp16 training mode at block and model level.  VSSBlock, ConMB, CroMB and CVSSDecoderBlock forward + backward under fp16
autocast with the switch on and off, both against the same fp32 run without autocast: the new mode's error in the output, the input
gradients and every parameter gradient is at most 2 x the switch-off error + fused.BF16_FLOOR of the tensor's scale (the convention
of fused.logits_bar, which the fp16 inference mode shares).  Then one whole-model step of Sigma-tiny 64 x 96 through
TrainStep(amp_dtype=torch.float16, fp16_core=True, scaler=GradScaler()) against the same step with the switch off."""
import contextlib
import io

import pytest
import torch
import torch.nn as nn

import procedural as P
from helpers import SEED, cfg_tiny, record

pytestmark = pytest.mark.gpu
F16 = torch.float16


def _cases():
    from sigma_b200 import modules as M
    x1 = P.randn(SEED, "f16t/x", (2, 12, 10, 32)).cuda()
    x2 = P.randn(SEED, "f16t/x2", (2, 12, 10, 32)).cuda()
    return {
        "vssblock": (lambda: M.VSSBlock(hidden_dim=32, norm_layer=nn.LayerNorm, mlp_ratio=0.0, d_state=16), (x1,)),
        "conmb": (lambda: M.ConcatMambaFusionBlock(hidden_dim=32, mlp_ratio=0.0, d_state=4), (x1, x2)),
        "cromb": (lambda: M.CrossMambaFusionBlock(hidden_dim=32, mlp_ratio=0.0, d_state=4), (x1, x2)),
        "cvss_dec": (lambda: M.CVSSDecoderBlock(hidden_dim=32, norm_layer=nn.LayerNorm, d_state=4, mlp_ratio=4.0), (x1,)),
    }


def _flat(y):
    """a block's output (CroMB returns one tensor per modality) as one fp32 vector"""
    return torch.cat([t.float().reshape(-1) for t in (y if isinstance(y, (tuple, list)) else (y,))])


def _run(blk, xs, wgt, amp, on):
    from sigma_b200 import ops
    blk.zero_grad(set_to_none=True)
    xs = [x.clone().requires_grad_(True) for x in xs]
    with torch.autocast("cuda", dtype=F16, enabled=amp), ops.fp16_training_core(on):
        y = _flat(blk(*xs))
    (y * wgt).sum().backward()
    out = {"y": y.detach()}
    out.update({f"dx{i}": x.grad.float() for i, x in enumerate(xs)})
    out.update({"d/" + n: p.grad.float().clone() for n, p in blk.named_parameters() if p.grad is not None})
    return out


@pytest.mark.parametrize("name", ["vssblock", "conmb", "cromb", "cvss_dec"])
def test_blocks_flag_on_vs_off_against_fp32(name, monkeypatch):
    from sigma_b200 import fused, ops
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    make, xs = _cases()[name]
    torch.manual_seed(SEED)
    blk = make().cuda().train()
    calls, b0 = [], ops._call_ss2d_bwd
    monkeypatch.setattr(ops, "_call_ss2d_bwd", lambda args, sv=False, det=False: (calls.append(sv), b0(args, sv, det))[1])
    with torch.no_grad():
        wgt = P.randn(SEED, f"f16t/{name}/w", tuple(_flat(blk(*xs)).shape)).cuda()
    ref = _run(blk, xs, wgt, False, False)
    off = _run(blk, xs, wgt, True, False)
    on = _run(blk, xs, wgt, True, True)
    assert calls == [True, True, ops._SAVED_FP16], calls           # the fused core ran all three times; the fp16 pair only when asked
    worst = {}
    assert set(on) == set(off) == set(ref)
    for key, r in ref.items():
        assert bool(on[key].isfinite().all()), key
        scale = float(r.abs().max())
        if scale == 0.0:
            assert float(on[key].abs().max()) == 0.0, key
            continue
        e_off, e_on = float((off[key] - r).abs().max()) / scale, float((on[key] - r).abs().max()) / scale
        worst[key] = e_on / (2.0 * e_off + fused.BF16_FLOOR)
        assert e_on <= 2.0 * e_off + fused.BF16_FLOOR, f"{name} {key}: on {e_on:.3e}, off {e_off:.3e} of scale"
    record(f"fp16 training block {name}", **worst)


def test_whole_model_step_through_trainstep_with_gradscaler():
    """The step runs with cuDNN off, so its depthwise convolutions take torch's own kernel.  With cuDNN 9.22 (torch 2.11) on an
    H100, once a ConMB block has taken a training step under fp16 autocast in the process (as test_blocks_flag_on_vs_off_against_fp32[conmb] does), cuDNN's
    fp16 depthwise 3x3 convolution of an NCHW input returns wrong values in a later model: ConMB's conv2d / conv2d_modalx here
    come out with an error of 1.7x their scale and the loss is NaN, with the switch off as much as on, and at the parent commit
    too (INTEGRATION.md §3).  With cuDNN off the same step is right whatever ran before, which is what this test compares."""
    from sigma_b200 import modules as M, ops, train_util
    H, W, ncls = 64, 96, 9
    losses, have, decision = {}, {}, {}
    for on in (False, True):
        torch.manual_seed(SEED)
        with contextlib.redirect_stdout(io.StringIO()):
            model = M.EncoderDecoder(cfg_tiny(H, W, num_classes=ncls), criterion=nn.CrossEntropyLoss(reduction="mean", ignore_index=255)).cuda().train()
        rgb = P.randn(SEED, "f16t/step/rgb", (2, 3, H, W)).cuda()
        mx = P.randn(SEED, "f16t/step/x", (2, 3, H, W)).cuda()
        gt = (P.rand(SEED, "f16t/step/gt", (2, H, W), 0, ncls).long() % ncls).cuda()
        calls, b0 = [], ops._call_ss2d_bwd
        ops._call_ss2d_bwd = lambda args, sv=False, det=False: (calls.append(sv), b0(args, sv, det))[1]
        scaler = torch.amp.GradScaler("cuda")
        try:
            step = train_util.TrainStep(model, train_util.make_optimizer(model), amp_dtype=F16, fp16_core=on, scaler=scaler)
            scale0 = scaler.get_scale()
            with torch.backends.cudnn.flags(enabled=False):
                loss = step(rgb, mx, gt)
        finally:
            ops._call_ss2d_bwd = b0
        assert ops.FP16_TRAINING_CORE is False
        assert calls and all(c == (ops._SAVED_FP16 if on else True) for c in calls), calls
        losses[on] = float(loss.detach())
        assert torch.isfinite(loss), losses
        grads = {n: p.grad for n, p in model.named_parameters() if p.requires_grad}
        assert all(g is None or bool(g.isfinite().all()) for g in grads.values())   # scaler.step unscaled them: finite at this scale
        have[on] = {n for n, g in grads.items() if g is not None}
        decision[on] = "applied" if scaler.get_scale() >= scale0 else "skipped"
    assert have[True] == have[False] and have[True]                 # every parameter the step reaches has a gradient in both modes
    assert decision[True] == decision[False] == "applied", decision
    # one fp16 step's loss is a mean over 2 x 64 x 96 pixels of logits that differ within the fp16 bar
    assert abs(losses[True] - losses[False]) <= 1e-2 * abs(losses[False]), losses
    record("fp16 training whole-model step", loss_off=losses[False], loss_on=losses[True], scaler_off=decision[False], scaler_on=decision[True])
