"""Time the ChannelAttentionBlock's dense convs in training: ops.CabConvFn (sigma_conv3x3_gelu_save_tf32 + sigma_conv3x3_tf32 forward,
sigma_conv3x3_wgrad_tf32 / sigma_conv3x3_dgrad_tf32 backward), or ops.CabConvPitchedFn (the same on the pitched entry points) where
C/3 is not a multiple of 4, against the route it replaces in CVSSDecoderBlock (an NCHW copy of the
LayerNorm output, nn.Conv2d -> nn.GELU -> nn.Conv2d on cuDNN, and the copy back to channels-last), and the whole training step with
each (ops.FUSED_CAB_TRAINING on / off).

    python scripts/bench_cab_train.py [--out DIR (default: a temporary directory)] [--rounds 5] [--iters 20] [--steps 10] [--models sigma_tiny,sigma_small]
                                      [--stages tiny|base] [--skip-step] [--skip-profile]

Op arm: the Sigma-tiny / Sigma-small (--stages tiny: C = 96 / 192 / 384) or Sigma-base (--stages base: C = 128 / 256 / 512, C/3 =
42 / 85 / 170) decoder stages at 480 x 640, batch 2, fp32 with torch's default precision for convolutions
(cudnn.allow_tf32 = True: TF32 on both routes), forward + backward.  CUDA events around --iters back-to-back calls, median [min, max]
of --rounds rounds, the two routes alternating.  Algorithmic FLOPs, counted from the shapes: 2·(B·H·W)·9·C·C1 per conv pass, three
passes per conv (forward, data and weight gradient); FLOP/s over the measured time, next to the H100 SXM's dense TF32 rate (495
TFLOP/s).  A torch.profiler run of each route (separate from the timed rounds) gives the per-kernel device time.
Whole-step arm: each of --models (Sigma-base takes CabConvPitchedFn) at 480 x 640, batch 2, fp32 (TF32 dense layers), AdamW through GraphedTrainStep, the
switch on and off captured as two graphs in one process and replayed alternately, --rounds x --steps; eager peak memory
(max_memory_allocated over two eager steps) of both.  Profile arm: torch.profiler over one eager Sigma-tiny step per setting; the
device time of the kernels that belong to the CAB convs (by name) against the step's total.  The card's name and power limit are read
in the same run (nothing is set).  Needs a GPU."""
import argparse
import contextlib
import io
import json
import os
import statistics
import subprocess
import sys
import tempfile
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {"tiny": [(2, 120, 160, 96), (2, 60, 80, 192), (2, 30, 40, 384)], "base": [(2, 120, 160, 128), (2, 60, 80, 256), (2, 30, 40, 512)]}
TF32_PEAK = 495e12
# kernel names of the dense convs on either route: ours (the conv instances of gemm_tf32_kernel, the epilogue variants, the weight
# gradient, and their pitched twins), cuDNN's convolution, gradient and layout kernels, torch's GELU and its backward.  The patch-embed conv's cuDNN kernels
# match too, in both settings alike; the partial sums (sum_parts_det, shared with the depthwise conv's backward) and torch's permute
# copies are not counted.
CAB_KERNELS = ("conv3x3_epi", "conv3x3_wgrad", "cab_conv_pitched", "cab_wgrad_pitched", ", true, false>(sigma::GemmParams)", "ImplicitGemmConvolution", "implicit_gemm",
               "s1688wgrad", "nchwToNhwc", "nhwcToNchw", "GeluCUDAKernelImpl", "GeluBackwardCUDAKernelImpl")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def stats(v):
    return {"median_ms": round(statistics.median(v), 4), "min_ms": round(min(v), 4), "max_ms": round(max(v), 4)}


@contextlib.contextmanager
def cab_switch(on):
    from sigma_b200 import ops
    prev = ops.FUSED_CAB_TRAINING
    ops.FUSED_CAB_TRAINING = on
    try:
        yield
    finally:
        ops.FUSED_CAB_TRAINING = prev


def cudnn_route(xn, cab):
    """CVSSDecoderBlock's route without the switch: NCHW copy in, cuDNN conv -> GELU -> conv, channels-last copy out"""
    return cab[2](cab[1](cab[0](xn.permute(0, 3, 1, 2).contiguous()))).permute(0, 2, 3, 1).contiguous()


def op_arm(a):
    import torch
    from sigma_b200 import ops
    out = []
    for B, H, W, C in SHAPES[a.stages]:
        g = torch.Generator(device="cuda").manual_seed(0)
        xn = torch.randn(B, H, W, C, device="cuda", generator=g).requires_grad_(True)
        dy = torch.randn(B, H, W, C, device="cuda", generator=g)
        cab = torch.nn.Sequential(torch.nn.Conv2d(C, C // 3, 3, 1, 1), torch.nn.GELU(), torch.nn.Conv2d(C // 3, C, 3, 1, 1)).cuda()
        node = ops.CabConvFn if (C // 3) % 4 == 0 else ops.CabConvPitchedFn
        arms = {"ours": lambda: node.apply(xn, cab[0].weight, cab[0].bias, cab[2].weight, cab[2].bias),
                "cudnn": lambda: cudnn_route(xn, cab)}

        def run(fn):
            fn().backward(dy)
        times = {k: [] for k in arms}
        for fn in arms.values():
            for _ in range(3):
                run(fn)
        for _ in range(a.rounds):
            for k, fn in arms.items():
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.iters):
                    run(fn)
                e1.record()
                torch.cuda.synchronize()
                times[k].append(e0.elapsed_time(e1) / a.iters)
        flops = 3 * 2 * 2 * B * H * W * 9 * C * (C // 3)
        row = {"shape": [B, H, W, C, C // 3], "alg_GFLOP": round(flops / 1e9, 2)}
        for k, v in times.items():
            s = stats(v)
            s["TFLOPs"] = round(flops / (s["median_ms"] * 1e-3) / 1e12, 1)
            s["of_tf32_peak"] = round(flops / (s["median_ms"] * 1e-3) / TF32_PEAK, 3)
            row[k] = s
        # per-kernel device time of one forward + backward of each route, from the profiler (a run of its own)
        for k, fn in arms.items():
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(a.iters):
                    run(fn)
                torch.cuda.synchronize()
            kern = {}
            for e in prof.events():
                if e.device_type == torch.autograd.DeviceType.CUDA:
                    kern[e.name[:90]] = kern.get(e.name[:90], 0.0) + e.device_time_total / 1e3 / a.iters
            row[k]["kernel_ms"] = round(sum(kern.values()), 4)
            row[k]["kernel_TFLOPs"] = round(flops / (row[k]["kernel_ms"] * 1e-3) / 1e12, 1)
            row[k]["kernels"] = {n: round(t, 4) for n, t in sorted(kern.items(), key=lambda kv: -kv[1])[:8]}
        out.append(row)
        del xn, dy, cab
    return out


def _model(backbone):
    import torch
    from sigma_b200 import modules as M
    B, Hh, Ww, ncls = 2, 480, 640, 40
    cfg = types.SimpleNamespace(backbone=backbone, decoder="MambaDecoder", num_classes=ncls, image_height=Hh, image_width=Ww,
                                pretrained_model=None, bn_eps=1e-3, bn_momentum=0.1)
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        model = M.EncoderDecoder(cfg, criterion=torch.nn.CrossEntropyLoss(reduction="mean", ignore_index=255)).cuda().train()
    g = torch.Generator(device="cuda").manual_seed(1)
    batch = (torch.randn(B, 3, Hh, Ww, device="cuda", generator=g), torch.randn(B, 3, Hh, Ww, device="cuda", generator=g),
             torch.randint(0, ncls, (B, Hh, Ww), device="cuda", generator=g))
    return model, batch


def step_arm(a, backbone):
    import torch
    from sigma_b200 import train_util
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    model, batch = _model(backbone)
    opt = train_util.make_optimizer(model, capturable=True)
    eager = train_util.TrainStep(model, opt)
    peak = {}
    for on in (False, True):
        with cab_switch(on):
            for _ in range(2):
                eager(*batch)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            for _ in range(2):
                eager(*batch)
            torch.cuda.synchronize()
            peak["on" if on else "off"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 3)
    with cab_switch(False):
        g_off = train_util.GraphedTrainStep(model, opt, batch)
    with cab_switch(True):
        g_on = train_util.GraphedTrainStep(model, opt, batch)
    arms = {"graph/cudnn": g_off, "graph/ours": g_on}
    res = {k: [] for k in arms}
    for fn in arms.values():
        for _ in range(3):
            fn(*batch)
    torch.cuda.synchronize()
    for _ in range(a.rounds):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                fn(*batch)
            e1.record()
            torch.cuda.synchronize()
            res[k].append(e0.elapsed_time(e1) / a.steps)
    out = {k: stats(v) | {"rounds": [round(t, 3) for t in v]} for k, v in res.items()}
    out["eager_peak_GiB"] = peak
    del g_off, g_on, eager, opt, model
    torch.cuda.empty_cache()
    return out


def profile_arm(a):
    import torch
    from sigma_b200 import train_util
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    model, batch = _model("sigma_tiny")
    step = train_util.TrainStep(model, train_util.make_optimizer(model, capturable=True))
    out = {}
    for on in (False, True):
        with cab_switch(on):
            for _ in range(2):
                step(*batch)
            torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                step(*batch)
                torch.cuda.synchronize()
        total, cab, names = 0.0, 0.0, {}
        for e in prof.events():
            if e.device_type != torch.autograd.DeviceType.CUDA:
                continue
            t = e.device_time_total / 1e3
            total += t
            if any(s in e.name for s in CAB_KERNELS):
                cab += t
                names[e.name[:90]] = names.get(e.name[:90], 0.0) + t
        out["ours" if on else "cudnn"] = {"step_kernel_ms": round(total, 3), "cab_kernel_ms": round(cab, 3), "cab_share": round(cab / total, 4),
                                          "cab_kernels": {n: round(t, 3) for n, t in sorted(names.items(), key=lambda kv: -kv[1])[:12]}}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "bench_cab_train"))
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--models", default="sigma_tiny,sigma_small")
    ap.add_argument("--stages", choices=sorted(SHAPES), default="tiny")
    ap.add_argument("--skip-step", action="store_true")
    ap.add_argument("--skip-profile", action="store_true")
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_cab_train.py needs a GPU"
    os.makedirs(a.out, exist_ok=True)
    res = {"card": card(), "op": op_arm(a)}
    print(json.dumps({"card": res["card"], "op": res["op"]}, indent=1), flush=True)
    if not a.skip_profile:
        res["profile"] = profile_arm(a)
        print(json.dumps({"profile": res["profile"]}, indent=1), flush=True)
    if not a.skip_step:
        res["step"] = {m: step_arm(a, m) for m in a.models.split(",")}
        print(json.dumps({"step": res["step"]}, indent=1), flush=True)
    with open(os.path.join(a.out, "bench_cab_train.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
