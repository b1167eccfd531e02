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


def make_optimizer(model, lr=6e-5, weight_decay=0.01, capturable=False):
    """train.py:84-93 with configs/config_MFNet.py:53-59 (AdamW, lr 6e-5, betas (0.9, 0.999), weight decay 0.01).
    capturable=True keeps the step counters on the device so the whole step can live in a CUDA graph."""
    return torch.optim.AdamW(group_weight(model, lr), lr=lr, betas=(0.9, 0.999), weight_decay=weight_decay, capturable=capturable)


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
