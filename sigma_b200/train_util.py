"""Training-step plumbing around the hot path, mirroring the reference's train.py (reference file:line cited per function).
The arithmetic is the modules' composed path (torch autograd over the op-level sigma_scan_fwd / sigma_scan_bwd kernels);
multi-GPU is torch DDP over NCCL exactly as train.py:103-108 — one bucketed all-reduce of the fp32 gradients per step."""
import contextlib
import time

import torch
import torch.distributed as dist
import torch.nn as nn


def group_weight(module, lr, norm_layer=nn.BatchNorm2d):
    """utils/init_func.py:33-56: weights of Linear / Conv layers decay, their biases and every norm parameter do not.
    As in the reference, bare nn.Parameters (x_proj_weight, dt_projs_*, A_logs, Ds, scale1/2) are in NEITHER group —
    `module.modules()` never yields them — so the reference's optimizer does not update them; kept for drop-in behaviour."""
    decay, no_decay = [], []
    for m in module.modules():
        if isinstance(m, (nn.Linear, nn.Conv1d, nn.Conv2d, nn.Conv3d, nn.ConvTranspose2d, nn.ConvTranspose3d)):
            decay.append(m.weight)
            if m.bias is not None:
                no_decay.append(m.bias)
        elif isinstance(m, (norm_layer, nn.BatchNorm1d, nn.BatchNorm2d, nn.BatchNorm3d, nn.GroupNorm, nn.LayerNorm)):
            if m.weight is not None:
                no_decay.append(m.weight)
            if m.bias is not None:
                no_decay.append(m.bias)
    return [dict(params=decay, lr=lr), dict(params=no_decay, weight_decay=0.0, lr=lr)]


def make_optimizer(model, lr=6e-5, weight_decay=0.01, capturable=False, fused=False):
    """train.py:84-93 with configs/config_MFNet.py:53-59 (AdamW, lr 6e-5, betas (0.9, 0.999), weight decay 0.01).
    capturable=True keeps the step counters on the device so the whole step can live in a CUDA graph.  fused=True runs torch's
    fused AdamW, which also takes a GradScaler's scale and inf flag on the device (what GraphedTrainStep needs with a scaler)."""
    return torch.optim.AdamW(group_weight(model, lr), lr=lr, betas=(0.9, 0.999), weight_decay=weight_decay, capturable=capturable,
                             fused=fused or None)


def wrap_ddp(model, device_index=None, single_bucket=False):
    """train.py:103-108.  device_index None = CPU (gloo tests).
    single_bucket: ONE gradient bucket that aliases the .grad tensors (bucket_cap_mb 1024, gradient_as_bucket_view).  On
    NVSwitch the whole 193-279 MB payload is a 0.5-0.8 ms all-reduce (617-648 GB/s bus bandwidth measured), cheaper than the
    per-bucket copies / launches / stream hand-offs of the default 25 MB buckets (measured: 11 ms exposed at 8 GPUs), so
    there is nothing to gain from overlapping it with the backward."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return model
    from torch.nn.parallel import DistributedDataParallel
    kw = dict(find_unused_parameters=False)
    if single_bucket:
        kw.update(bucket_cap_mb=1024, gradient_as_bucket_view=True)
    if device_index is None:
        return DistributedDataParallel(model, **kw)
    return DistributedDataParallel(model, device_ids=[device_index], output_device=device_index, **kw)


class TrainStep:
    """One iteration of train.py:164-172: loss = model(imgs, modal_xs, gts); zero_grad; backward; optimizer.step.
    `amp_dtype` = torch.bfloat16 runs the dense layers under autocast (the scan casts itself to fp32, vmamba.py:36).
    `bf16_core` = True switches the bf16 training mode of the fused core on around the step (ops.bf16_training_core); False
    leaves ops.BF16_TRAINING_CORE as it is.  `fp16_core` does the same for the fp16 training mode (ops.fp16_training_core), which
    applies under amp_dtype = torch.float16.
    `scaler` (a torch.amp.GradScaler, the usual companion of fp16 autocast): the step back-propagates the scaled loss and lets the
    scaler unscale the gradients, skip the optimizer step when one of them is inf / NaN, and update its scale.  The returned loss
    is unscaled either way."""

    def __init__(self, model, optimizer, amp_dtype=None, device_type="cuda", bf16_core=False, fp16_core=False, scaler=None):
        self.model, self.opt, self.amp, self.device_type = model, optimizer, amp_dtype, device_type
        self.bf16_core = bf16_core
        self.fp16_core, self.scaler = fp16_core, scaler

    def __call__(self, rgb, modal_x, label, sync=True):
        from . import ops
        ctx = self.model.no_sync() if (not sync and hasattr(self.model, "no_sync")) else contextlib.nullcontext()
        with ctx, (ops.bf16_training_core() if self.bf16_core else contextlib.nullcontext()), \
                (ops.fp16_training_core() if self.fp16_core else contextlib.nullcontext()):
            with torch.autocast(self.device_type, dtype=self.amp, enabled=self.amp is not None):
                loss = self.model(rgb, modal_x, label)
            self.opt.zero_grad(set_to_none=True)
            if self.scaler is None:
                loss.backward()
            else:
                self.scaler.scale(loss).backward()
        if self.scaler is None:
            self.opt.step()
        else:
            self.scaler.step(self.opt)
            self.scaler.update()
        return loss


class GraphedTrainStep:
    """TrainStep replayed from one CUDA graph: forward, backward and optimizer step (with a scaler, also its unscale / inf check,
    the skipped or applied step and the scale update) are captured once and each call replays them, so the host issues one graph
    launch per step instead of every kernel.  Same arguments as TrainStep, plus `example` = (rgb, modal_x, label), a batch whose
    shapes, dtypes and device every later batch must have.

    Construction copies the example into static input buffers, runs `warmup` eager steps on a side stream (lazy optimizer and
    scaler state, cuBLAS / cuDNN handles, kernel attributes), captures one step, then puts back the parameters, gradients,
    buffers, optimizer state and scaler state it found, so the first replay is the first step.  Random draws (DropPath) are not
    put back; each replay draws fresh ones from torch's generator.

    Conditions, each a ValueError: every param group of the optimizer is capturable=True or fused=True (make_optimizer(capturable=
    True) builds one); with an enabled scaler the optimizer is fused=True, whose kernel unscales and skips the step on the device;
    the model is not DistributedDataParallel (its all-reduce is not captured); a call's batch matches the example; and the capture
    itself succeeds (there is no eager fallback).  Hyper-parameters given as Python numbers (lr, betas, weight decay) are fixed at
    capture.

    A call returns the unscaled loss as a new device tensor and never waits for the GPU.  After each replay the updated tensors'
    `_version` is bumped (fused.weights_updated), so the fused inference forward, InferencePipeline and DeviceEvaluator see the new
    weights."""

    def __init__(self, model, optimizer, example, amp_dtype=None, bf16_core=False, fp16_core=False, scaler=None, warmup=3):
        from torch.nn.parallel import DistributedDataParallel
        if isinstance(model, DistributedDataParallel):
            raise ValueError("GraphedTrainStep: a DistributedDataParallel model cannot be captured (its gradient all-reduce is not "
                             "part of the graph); train multi-GPU with TrainStep")
        groups = optimizer.param_groups
        if not all(g.get("capturable") or g.get("fused") for g in groups):
            raise ValueError(f"GraphedTrainStep: {type(optimizer).__name__} cannot be captured: every param group needs "
                             "capturable=True or fused=True (make_optimizer(model, capturable=True))")
        if scaler is not None and scaler.is_enabled() and not getattr(optimizer, "_step_supports_amp_scaling", False):
            raise ValueError("GraphedTrainStep: with a GradScaler the optimizer must take the scale and inf flag on the device "
                             "(fused=True, e.g. make_optimizer(model, capturable=True, fused=True)); otherwise scaler.step "
                             "reads the inf flag on the host")
        if warmup < 1:
            raise ValueError("GraphedTrainStep: warmup must be >= 1 (the optimizer's and scaler's state must exist before the capture, "
                             "or the graph would re-initialise it on every replay)")
        if len(example) != 3 or not all(torch.is_tensor(t) and t.is_cuda for t in example) or len({t.device for t in example}) != 1:
            raise ValueError("GraphedTrainStep: the example batch must be three CUDA tensors (rgb, modal_x, label) on one device")
        for g in groups:
            if g.get("fused"):
                g["capturable"] = True   # fused kernels keep `step` on the device either way; torch's capture check reads the flag
        self.model, self.opt, self.scaler = model, optimizer, scaler
        self.static = tuple(t.detach().clone() for t in example)
        self.step = TrainStep(model, optimizer, amp_dtype=amp_dtype, bf16_core=bf16_core, fp16_core=fp16_core, scaler=scaler)
        self.updated = [p for g in groups for p in g["params"]]
        saved = self._snapshot()
        side = torch.cuda.Stream(device=self.static[0].device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):
                self.step(*self.static)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        try:
            with torch.cuda.graph(self.graph):
                self.loss = self.step(*self.static).detach()
        except Exception as e:
            raise ValueError(f"GraphedTrainStep: capturing the step failed ({type(e).__name__}: {e})") from e
        torch.cuda.synchronize()
        self._restore(saved)

    def _snapshot(self):
        clone = lambda t: None if t is None else t.detach().clone()   # noqa: E731
        sc = self.scaler
        return dict(params=[clone(p) for p in self.model.parameters()], grads=[clone(p.grad) for p in self.model.parameters()],
                    buffers=[clone(b) for b in self.model.buffers()],
                    opt={p: {k: clone(v) if torch.is_tensor(v) else v for k, v in self.opt.state[p].items()}
                         for p in self.updated if p in self.opt.state},
                    scaler=None if sc is None or getattr(sc, "_scale", None) is None else (clone(sc._scale), clone(sc._growth_tracker)))

    @torch.no_grad()
    def _restore(self, saved):
        """Put back what _snapshot saw, in place (the graph reads and writes these very tensors).  State that did not exist then
        (a fresh optimizer's moments and step, a fresh scaler) goes back to the values its lazy initialisation gives: zeros and the
        initial scale."""
        for p, v in zip(self.model.parameters(), saved["params"]):
            p.copy_(v)
        for p, g in zip(self.model.parameters(), saved["grads"]):
            if p.grad is not None:
                p.grad.copy_(g) if g is not None else p.grad.zero_()
        for b, v in zip(self.model.buffers(), saved["buffers"]):
            b.copy_(v)
        for p in self.updated:
            old = saved["opt"].get(p)
            for k, v in self.opt.state[p].items():
                if torch.is_tensor(v):
                    v.copy_(old[k]) if old is not None else v.zero_()
        sc = self.scaler
        if sc is not None and getattr(sc, "_scale", None) is not None:
            if saved["scaler"] is not None:
                sc._scale.copy_(saved["scaler"][0])
                sc._growth_tracker.copy_(saved["scaler"][1])
            else:
                sc._scale.fill_(sc._init_scale)
                sc._growth_tracker.fill_(sc._init_growth_tracker)
        torch.cuda.synchronize()

    def __call__(self, rgb, modal_x, label):
        from . import fused
        for name, t, s in zip(("rgb", "modal_x", "label"), (rgb, modal_x, label), self.static):
            if not torch.is_tensor(t) or t.shape != s.shape or t.dtype != s.dtype or t.device != s.device:
                got = (tuple(t.shape), t.dtype, t.device) if torch.is_tensor(t) else type(t).__name__
                raise ValueError(f"GraphedTrainStep: {name} is {got}; the graph was captured for {(tuple(s.shape), s.dtype, s.device)}")
            if t is not s:
                s.copy_(t, non_blocking=True)
        self.graph.replay()
        fused.weights_updated(self.updated)
        return self.loss.clone()


def grad_bytes(model):
    return sum(p.numel() * p.element_size() for p in model.parameters() if p.requires_grad)


def allreduce_bus_bandwidth(nbytes, device, reps=10):
    """Time a flat fp32 all-reduce of the gradient payload by itself: (seconds, bus GB/s = 2(N-1)/N · bytes / t)."""
    world = dist.get_world_size() if dist.is_initialized() else 1
    if world == 1:
        return 0.0, None
    buf = torch.zeros(nbytes // 4, dtype=torch.float32, device=device)
    for _ in range(3):
        dist.all_reduce(buf)
    if device.type == "cuda":
        torch.cuda.synchronize(device)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            dist.all_reduce(buf)
        e1.record()
        torch.cuda.synchronize(device)
        t = e0.elapsed_time(e1) * 1e-3 / reps
    else:
        t0 = time.perf_counter()
        for _ in range(reps):
            dist.all_reduce(buf)
        t = (time.perf_counter() - t0) / reps
    return t, 2 * (world - 1) / world * nbytes / t / 1e9
