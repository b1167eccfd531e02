"""GPU: train_util.GraphedTrainStep, the training step replayed from one CUDA graph, against the eager TrainStep.

* Under torch.use_deterministic_algorithms(True), Sigma-tiny 64 x 96, batch 2: three graphed and three eager steps from one
  state_dict on the same three batches (none of them the example the graph was captured with) give bitwise-equal losses,
  parameters and AdamW state.
* The bf16 core and the fp16 core with a GradScaler: graphed against eager over three steps, within the whole-model bar of
  tests/test_fp16_training_blocks_gpu.py for the losses (1e-2 of the loss); the parameters' update within 2 x the spread between
  two eager runs + fused.BF16_FLOOR of its norm (the default backward kernels use atomics, so no two runs are bitwise equal).
* GradScaler inside the graph: a batch holding an inf leaves every parameter and the AdamW step count as they were and halves
  the scale; the next finite batch updates.
* Weights after replay: the fused inference forward (tf32x3 and bf16) and InferencePipeline equal a fresh model loaded with the
  trained state_dict, bit for bit.
* Every rejection of GraphedTrainStep; one eager step of each mode with no host synchronisation; DropPath's masks drawn afresh on
  each replay.
Every test but the DropPath one sets each DropPath.drop_prob to 0."""
import contextlib
import io

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import procedural as P
from helpers import SEED, cfg_tiny, record

pytestmark = pytest.mark.gpu
H, W, NCLS = 64, 96, 9
F16, BF16 = torch.float16, torch.bfloat16


def _model(state=None, drop=False):
    from sigma_b200 import modules as M
    torch.manual_seed(SEED)
    with contextlib.redirect_stdout(io.StringIO()):
        model = M.EncoderDecoder(cfg_tiny(H, W, num_classes=NCLS), criterion=nn.CrossEntropyLoss(reduction="mean", ignore_index=255))
    model = model.cuda().train()
    if state is not None:
        model.load_state_dict(state)
    if not drop:
        for m in model.modules():
            if isinstance(m, M.DropPath):
                m.drop_prob = 0.0
    return model


def _batch(tag):
    rgb = P.randn(SEED, f"tg/{tag}/rgb", (2, 3, H, W)).cuda()
    mx = P.randn(SEED, f"tg/{tag}/x", (2, 3, H, W)).cuda()
    gt = (P.rand(SEED, f"tg/{tag}/gt", (2, H, W), 0, NCLS).long() % NCLS).cuda()
    gt[:, : H // 8] = 255                                   # ignored pixels
    return rgb, mx, gt


@contextlib.contextmanager
def _deterministic(monkeypatch):
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")      # torch requires it for cuBLAS under the switch
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(False)


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32) if t.is_floating_point() else t


def _opt_state(opt):
    return [(k, v) for g in opt.param_groups for p in g["params"] for k, v in sorted(opt.state[p].items()) if torch.is_tensor(v)]


def _pair(mode_kw, opt_kw, scaler_fn=None):
    """an eager and a graphed step on two models from one state_dict; the graph captured on an example batch of its own"""
    from sigma_b200 import train_util
    state = {k: v.clone() for k, v in _model().state_dict().items()}
    me, mg = _model(state), _model(state)
    oe, og = train_util.make_optimizer(me, **opt_kw), train_util.make_optimizer(mg, **opt_kw)
    se, sg = (scaler_fn(), scaler_fn()) if scaler_fn else (None, None)
    eager = train_util.TrainStep(me, oe, scaler=se, **mode_kw)
    graphed = train_util.GraphedTrainStep(mg, og, _batch("example"), scaler=sg, **mode_kw)
    return (me, oe, se, eager), (mg, og, sg, graphed)


def test_bitwise_equal_to_eager_under_deterministic_switch(monkeypatch):
    with _deterministic(monkeypatch):
        (me, oe, _, eager), (mg, og, _, graphed) = _pair({}, dict(capturable=True))
        for i in range(3):
            b = _batch(f"step{i}")
            le, lg = eager(*b), graphed(*b)
            assert torch.equal(_bits(le.detach()), _bits(lg)), (i, float(le), float(lg))
        torch.cuda.synchronize()
    for (n, a), b in zip(me.named_parameters(), mg.parameters()):
        assert torch.equal(_bits(a.detach()), _bits(b.detach())), n
    se, sg = _opt_state(oe), _opt_state(og)
    assert len(se) == len(sg) > 0
    for (k, a), (_, b) in zip(se, sg):
        assert torch.equal(_bits(a), _bits(b)), k
    assert {float(v) for k, v in sg if k == "step"} == {3.0}      # the warm-up steps of the construction were put back


@pytest.mark.parametrize("mode", ["bf16", "fp16"])
def test_16bit_modes_match_eager(mode):
    """fp16 runs with cuDNN off, as tests/test_fp16_training_blocks_gpu.py explains (INTEGRATION.md §3)."""
    if mode == "bf16":
        kw, opt_kw, scaler_fn, flags = dict(amp_dtype=BF16, bf16_core=True), dict(capturable=True), None, contextlib.nullcontext()
    else:
        kw, opt_kw = dict(amp_dtype=F16, fp16_core=True), dict(capturable=True, fused=True)
        scaler_fn, flags = (lambda: torch.amp.GradScaler("cuda")), torch.backends.cudnn.flags(enabled=False)
    from sigma_b200 import fused, train_util
    with flags:
        p0 = {n: p.detach().clone() for n, p in _model().named_parameters()}
        (me, _, se, eager), (mg, _, sg, graphed) = _pair(kw, opt_kw, scaler_fn)
        m2 = _model()                                      # a second eager run: the atomics' own run-to-run spread
        eager2 = train_util.TrainStep(m2, train_util.make_optimizer(m2, **opt_kw), scaler=scaler_fn() if scaler_fn else None, **kw)
        losses = []
        for i in range(3):
            b = _batch(f"step{i}")
            losses.append((float(eager(*b).detach()), float(graphed(*b)), float(eager2(*b).detach())))
    for le, lg, _ in losses:
        assert abs(lg - le) <= 1e-2 * abs(le), losses
    if se is not None:
        assert se.get_scale() == sg.get_scale()
    update = lambda m: torch.cat([(p.detach() - p0[n]).reshape(-1) for n, p in m.named_parameters()])   # noqa: E731
    de, dg, d2 = update(me), update(mg), update(m2)
    rel, spread = float((dg - de).norm() / de.norm()), float((d2 - de).norm() / de.norm())
    # AdamW divides by sqrt(v): a parameter whose gradient is near zero moves by up to lr whatever the sign the atomics leave it,
    # so the bar on the update is the eager run-to-run spread, in the convention of fused.logits_bar
    assert float(de.norm()) > 0 and rel <= 2.0 * spread + fused.BF16_FLOOR, (rel, spread)
    record(f"graphed train step {mode}", losses=losses, update_rel_err=rel, eager_spread=spread)


def test_gradscaler_skips_an_inf_batch_in_the_graph_then_applies():
    from sigma_b200 import train_util
    with torch.backends.cudnn.flags(enabled=False):
        model = _model()
        opt = train_util.make_optimizer(model, capturable=True, fused=True)
        scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 10)
        step = train_util.GraphedTrainStep(model, opt, _batch("example"), amp_dtype=F16, fp16_core=True, scaler=scaler)
        rgb, mx, gt = _batch("step0")
        before = [p.detach().clone() for p in model.parameters()]
        assert scaler.get_scale() == 2.0 ** 10                   # construction put the scaler back as it found it
        bad = rgb.clone()
        bad[0, 0, 3, 5] = float("inf")
        step(bad, mx, gt)
        torch.cuda.synchronize()
        assert all(torch.equal(p.detach(), q) for p, q in zip(model.parameters(), before))
        assert scaler.get_scale() == 2.0 ** 9
        steps = {float(s["step"]) for s in opt.state.values()}
        assert steps == {0.0}, steps
        loss = step(rgb, mx, gt)
        torch.cuda.synchronize()
    assert torch.isfinite(loss)
    assert any(not torch.equal(p.detach(), q) for p, q in zip(model.parameters(), before))
    assert scaler.get_scale() == 2.0 ** 9
    assert {float(s["step"]) for s in opt.state.values()} == {1.0}


@pytest.mark.parametrize("mode", ["tf32x3", "bf16"])
def test_fused_inference_and_pipeline_see_replayed_weights(mode, monkeypatch):
    from sigma_b200 import fused, train_util
    from sigma_b200.pipeline import InferencePipeline
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    amp = BF16 if mode == "bf16" else None
    ctx = lambda: torch.autocast("cuda", dtype=BF16) if amp else contextlib.nullcontext()   # noqa: E731
    model = _model()
    step = train_util.GraphedTrainStep(model, train_util.make_optimizer(model, capturable=True), _batch("example"))
    rgb, mx, _ = _batch("eval")
    model.eval()
    with torch.no_grad(), ctx():          # after the construction: from here on only the replays change the weights
        assert fused.precision() == mode
        stale = model(rgb, mx)            # fills the derived-weight caches
    pipe = InferencePipeline(model, 2, H, W, amp_dtype=amp)
    model.train()
    for i in range(2):
        step(*_batch(f"step{i}"))
    torch.cuda.synchronize()
    model.eval()
    fresh = _model({k: v.clone() for k, v in model.state_dict().items()}).eval()
    with torch.no_grad(), ctx():
        got, want = model(rgb, mx), fresh(rgb, mx)
    assert not torch.equal(want, stale)
    assert torch.equal(got, want)
    h_out = torch.empty((2,) + pipe.out_shape[1:], dtype=pipe.out.dtype).pin_memory()
    pipe.submit(rgb.cpu().pin_memory(), mx.cpu().pin_memory(), h_out)
    pipe.drain()
    assert torch.equal(h_out, want.cpu())


class _Toy(nn.Module):
    """a two-layer segmentation head over rgb + modal_x; `fail_capture` raises inside the capture only"""

    def __init__(self, fail_capture=False):
        super().__init__()
        self.a, self.b, self.fail = nn.Conv2d(6, 8, 1), nn.Conv2d(8, NCLS, 1), fail_capture

    def forward(self, rgb, modal_x, label):
        if self.fail and torch.cuda.is_current_stream_capturing():
            raise RuntimeError("this forward cannot be captured")
        return F.cross_entropy(self.b(F.relu(self.a(torch.cat([rgb, modal_x], 1)))), label, ignore_index=255)


def test_rejections():
    from sigma_b200 import train_util
    b = _batch("example")
    model = _Toy().cuda()
    with pytest.raises(ValueError, match="capturable=True or fused=True"):
        train_util.GraphedTrainStep(model, train_util.make_optimizer(model), b)
    with pytest.raises(ValueError, match="fused=True"):
        train_util.GraphedTrainStep(model, train_util.make_optimizer(model, capturable=True), b, scaler=torch.amp.GradScaler("cuda"))
    with pytest.raises(ValueError, match="CUDA tensors"):
        train_util.GraphedTrainStep(model, train_util.make_optimizer(model, capturable=True), tuple(t.cpu() for t in b))
    bad = _Toy(fail_capture=True).cuda()
    with pytest.raises(ValueError, match="capturing the step failed"):
        train_util.GraphedTrainStep(bad, train_util.make_optimizer(bad, capturable=True), b)
    step = train_util.GraphedTrainStep(model, train_util.make_optimizer(model, capturable=True), b)
    rgb, mx, gt = b
    for args in ((rgb[:1], mx[:1], gt[:1]), (rgb.double(), mx, gt), (rgb, mx, gt.int()), (rgb.cpu(), mx, gt)):
        with pytest.raises(ValueError, match="captured for"):
            step(*args)
    assert torch.isfinite(step(rgb, mx, gt))


def test_fused_optimizer_without_capturable_flag_is_accepted():
    from sigma_b200 import train_util
    model = _Toy().cuda()
    opt = train_util.make_optimizer(model, fused=True)
    step = train_util.GraphedTrainStep(model, opt, _batch("example"))
    w0 = model.a.weight.detach().clone()
    step(*_batch("step0"))
    torch.cuda.synchronize()
    assert not torch.equal(model.a.weight.detach(), w0)


@pytest.mark.parametrize("mode", ["fp32", "bf16", "fp16", "deterministic"])
def test_eager_step_has_no_host_sync(mode, monkeypatch):
    """one warm-up step, then one step under torch.cuda.set_sync_debug_mode("error"), which raises at any synchronising call"""
    from sigma_b200 import train_util
    model = _model()
    kw, scaler, stack = {}, None, contextlib.ExitStack()
    opt = train_util.make_optimizer(model, capturable=True, fused=mode == "fp16")
    if mode == "bf16":
        kw = dict(amp_dtype=BF16, bf16_core=True)
    elif mode == "fp16":
        scaler = torch.amp.GradScaler("cuda")
        kw = dict(amp_dtype=F16, fp16_core=True, scaler=scaler)
        stack.enter_context(torch.backends.cudnn.flags(enabled=False))
    elif mode == "deterministic":
        stack.enter_context(_deterministic(monkeypatch))
    with stack:
        step = train_util.TrainStep(model, opt, **kw)
        b = _batch("sync")
        step(*b)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            loss = step(*b)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        torch.cuda.synchronize()
    assert torch.isfinite(loss)


def test_droppath_draws_fresh_masks_on_each_replay(monkeypatch):
    """lr = 0 keeps the weights, so only the masks can change the loss; the control without DropPath repeats it bit for bit"""
    from sigma_b200 import modules as M, train_util
    losses = {}
    with _deterministic(monkeypatch):
        for drop in (True, False):
            model = _model(drop=drop)
            assert any(m.drop_prob > 0 for m in model.modules() if isinstance(m, M.DropPath)) == drop
            step = train_util.GraphedTrainStep(model, train_util.make_optimizer(model, lr=0.0, capturable=True), _batch("example"))
            b = _batch("step0")
            losses[drop] = [float(step(*b)) for _ in range(2)]
    assert losses[True][0] != losses[True][1], losses
    assert losses[False][0] == losses[False][1], losses
