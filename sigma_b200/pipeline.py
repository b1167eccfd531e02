"""Batched inference with host buffers: the serving-side call around `EncoderDecoder.forward`.

The reference's evaluator (engine/evaluator.py:433-522) feeds the model one host batch at a time: copy in, forward,
`.cpu()`.  A batch of 32 images moves 236 MB in and 354 MB of fp32 logits out over PCIe, which a serial loop spends with
the GPU idle.  `InferencePipeline` keeps the
same contract (host RGB / X batches in, host logits out, every batch copied both ways) and overlaps the three
stages of neighbouring batches on three streams:

    copy-in stream :  H2D(i+1) ───────────►
    compute stream :  [stage_in -> graph inputs] forward(i) [logits -> stage_out]
    copy-out stream:  ◄─────────── D2H(i-1)

The forward is one CUDA graph (captured once); the graph's static input / output tensors are decoupled from the
transfers by device-side staging buffers (two of each), so a transfer never touches a tensor the graph is using.
"""
import contextlib

import torch


class InferencePipeline:
    """pipe = InferencePipeline(model, batch, height, width); pipe.submit(h_rgb, h_x, h_out) per batch; pipe.drain().

    `h_rgb`, `h_x`: pinned host tensors (batch, 3, H, W) fp32; `h_out`: pinned host tensor (batch, classes, H, W) that
    receives the logits of THAT batch.  `submit` returns immediately; results are valid after `drain()` (or after a
    later `submit` that reuses the same staging slot has been drained — use `drain()` before reading `h_out`).

    The model must be in eval mode.  The captured graph holds the device pointers of the model's parameters AND of the
    packed SSM tensors the fused path derives from them (x_proj / dt / A = -exp(A_logs) / D copies, fused._cache): when
    any parameter is modified in place afterwards (load_state_dict, an optimizer step) `submit` notices the changed
    version counters and re-captures the graph, so stale packed copies are never replayed.

    amp_dtype=torch.bfloat16 runs the forward (warm-up, capture and any re-capture) under torch.autocast("cuda", dtype=amp_dtype),
    so the captured graph is the one of the fused path's bf16 mode (sigma_b200.fused.precision); None runs it as called.
    fp8=True runs them inside sigma_b200.fused.fp8_inference(), so the graph is the one of the FP8 mode (the per-channel e4m3
    weights it reads are re-quantized, like the packed SSM tensors, when a re-capture follows a weight change).  fp16=True runs
    them inside sigma_b200.fused.fp16_inference() (the fp16 mode; its fp16 weight copies are refreshed the same way); fp8 and fp16
    together are a ValueError."""

    def __init__(self, model, batch, height, width, use_graph=True, amp_dtype=None, fp8=False, fp16=False):
        if fp8 and fp16:
            raise ValueError("sigma_b200.InferencePipeline: fp8=True and fp16=True select two modes; choose one")
        self.model = model
        self.amp_dtype = amp_dtype
        self.fp8 = fp8
        self.fp16 = fp16
        p = next(model.parameters())
        if p.device.type != "cuda":
            raise RuntimeError("sigma_b200.InferencePipeline needs the model on a CUDA device (there is no CPU path)")
        if model.training:
            raise RuntimeError("sigma_b200.InferencePipeline: call model.eval() first (the fused inference path has no DropPath / dropout)")
        self.dev = p.device
        self.use_graph = use_graph
        self.shape = (batch, 3, height, width)
        self.rgb = torch.zeros(self.shape, device=self.dev)
        self.x = torch.zeros(self.shape, device=self.dev)
        self.compute = torch.cuda.Stream(self.dev)
        self.copy_in = torch.cuda.Stream(self.dev)
        self.copy_out = torch.cuda.Stream(self.dev)
        self.graph = None
        self.out = None
        self._capture()
        self.stage_in = [(torch.empty_like(self.rgb), torch.empty_like(self.x)) for _ in range(2)]
        self.stage_out = [torch.empty_like(self.out) for _ in range(2)]
        self.ev_in = [torch.cuda.Event() for _ in range(2)]        # H2D into stage_in[s] finished
        self.ev_in_free = [torch.cuda.Event() for _ in range(2)]   # compute has consumed stage_in[s]
        self.ev_out = [torch.cuda.Event() for _ in range(2)]       # compute has filled stage_out[s]
        self.ev_out_free = [torch.cuda.Event() for _ in range(2)]  # D2H out of stage_out[s] finished
        self.n = 0

    def _versions(self):
        return sum(p._version for p in self.model.parameters())

    def _autocast(self):
        """the forward's precision context: autocast (amp_dtype) and / or the FP8 or fp16 mode"""
        from . import fused
        stack = contextlib.ExitStack()
        if self.amp_dtype is not None:
            stack.enter_context(torch.autocast("cuda", dtype=self.amp_dtype))
        if self.fp8:
            stack.enter_context(fused.fp8_inference())
        if self.fp16:
            stack.enter_context(fused.fp16_inference())
        return stack

    def _capture(self):
        with torch.cuda.stream(self.compute), torch.no_grad(), self._autocast():
            for _ in range(2):                       # warm-up: allocator, kernel attributes, cuDNN algorithm choice, packed-parameter cache
                out = self.model(self.rgb, self.x)
        self.compute.synchronize()
        if self.use_graph:
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph, stream=self.compute), torch.no_grad(), self._autocast():
                out = self.model(self.rgb, self.x)
            self.compute.synchronize()
        self.out = out                               # the graph's static output tensor
        self._ver = self._versions()

    @property
    def out_shape(self):
        return tuple(self.out.shape)

    def submit(self, h_rgb, h_x, h_out):
        if self._versions() != self._ver:            # weights changed in place since the capture
            self.drain()
            self._capture()
        s = self.n & 1
        first_use = self.n < 2
        with torch.cuda.stream(self.copy_in):
            if not first_use:
                self.copy_in.wait_event(self.ev_in_free[s])
            self.stage_in[s][0].copy_(h_rgb, non_blocking=True)
            self.stage_in[s][1].copy_(h_x, non_blocking=True)
            self.ev_in[s].record(self.copy_in)
        with torch.cuda.stream(self.compute), torch.no_grad():
            self.compute.wait_event(self.ev_in[s])
            self.rgb.copy_(self.stage_in[s][0], non_blocking=True)
            self.x.copy_(self.stage_in[s][1], non_blocking=True)
            self.ev_in_free[s].record(self.compute)
            if self.graph is not None:
                self.graph.replay()
            else:
                with self._autocast():
                    self.out = self.model(self.rgb, self.x)
            if not first_use:
                self.compute.wait_event(self.ev_out_free[s])
            self.stage_out[s].copy_(self.out, non_blocking=True)
            self.ev_out[s].record(self.compute)
        with torch.cuda.stream(self.copy_out):
            self.copy_out.wait_event(self.ev_out[s])
            h_out.copy_(self.stage_out[s], non_blocking=True)
            self.ev_out_free[s].record(self.copy_out)
        self.n += 1

    def drain(self):
        self.copy_out.synchronize()
        self.compute.synchronize()
        self.copy_in.synchronize()
