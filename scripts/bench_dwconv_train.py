"""Time the Mamba blocks' depthwise conv3x3 + SiLU in training: ops.DwConvSiLUFn (sigma_dwconv3x3_silu_fwd + _bwd) against the torch
route it replaced (F.conv2d(groups=D) on the channels-last view + F.silu, cuDNN / torch kernels), and the whole training step with
each.

    python scripts/bench_dwconv_train.py [--out DIR] [--rounds 5] [--iters 20] [--steps 10] [--models sigma_tiny,sigma_small]
                                         [--skip-step]

Op arm: every Sigma-tiny training shape at 480 x 640, batch 2 (SS2D encoder stages and CroMB as 4 images, ConMB and the decoder as 2),
fp32, bf16 and fp16, forward + backward of one conv + SiLU from a channels-last x.  CUDA events around --iters calls, median [min, max]
of --rounds rounds, every shape warmed, the two arms alternating round by round.  Algorithmic bytes, counted from the shapes: the
fused forward reads x and writes y, the fused backward reads x and dy and writes dx, so 5 activations of B·H·W·D elements; the GB/s
of each arm is those bytes over its time, against the H100 SXM's 3.35 TB/s.  16-bit runs under autocast of its dtype, as training
does.
Whole-step arm: Sigma-tiny and Sigma-small at 480 x 640, batch 2, eager TrainStep and GraphedTrainStep, fp32 (TF32 dense layers), bf16
core and fp16 core + GradScaler; the torch route is substituted for the node in this process by replacing ops.DwConvSiLUFn.apply
(the eager arm while it runs, the graphed arm while it is captured), and the arms alternate round by round.  Peak memory: eager
max_memory_allocated over its rounds.  The card's name and power limit are read in the same run (nothing is set).  Needs a GPU."""
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

SHAPES = [(4, 120, 160, 192), (4, 60, 80, 384), (4, 30, 40, 768), (4, 15, 20, 1536),
          (2, 120, 160, 192), (2, 60, 80, 384), (2, 30, 40, 768), (2, 15, 20, 1536)]
HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def torch_route(x, weight, bias):
    """the route ops.DwConvSiLUFn replaced: channels-last x through F.conv2d(groups=D) and F.silu -> (B, H·W, D)"""
    import torch.nn.functional as F
    B, H, W, D = x.shape
    return F.silu(F.conv2d(x.permute(0, 3, 1, 2), weight, bias, padding=1, groups=D)).permute(0, 2, 3, 1).reshape(B, H * W, D)


@contextlib.contextmanager
def torch_conv():
    from sigma_b200 import ops
    prev = ops.DwConvSiLUFn.apply
    ops.DwConvSiLUFn.apply = torch_route
    try:
        yield
    finally:
        ops.DwConvSiLUFn.apply = prev


def stats(v):
    return {"median_ms": round(statistics.median(v), 4), "min_ms": round(min(v), 4), "max_ms": round(max(v), 4)}


def op_arm(a):
    import torch
    from sigma_b200 import ops
    out = []
    for dt in (torch.float32, torch.bfloat16, torch.float16):
        for B, H, W, D in SHAPES:
            g = torch.Generator(device="cuda").manual_seed(0)
            x = torch.randn(B, H, W, D, device="cuda", generator=g).to(dt).requires_grad_(True)
            dy = torch.randn(B, H * W, D, device="cuda", generator=g).to(dt)
            conv = torch.nn.Conv2d(D, D, 3, padding=1, groups=D).cuda()
            arms = {"ours": ops.DwConvSiLUFn.apply, "torch": torch_route}

            def run(fn):        # 16-bit: under autocast, as in training (it casts the torch conv's fp32 weights; the node keeps them)
                with torch.autocast("cuda", dtype=dt, enabled=dt != torch.float32):
                    y = fn(x, conv.weight, conv.bias)
                y.backward(dy)
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
            nbytes = 5 * B * H * W * D * x.element_size()
            row = {"dtype": str(dt).split(".")[1], "shape": [B, H, W, D], "alg_MB": round(nbytes / 1e6, 2)}
            for k, v in times.items():
                s = stats(v)
                s["GBps"] = round(nbytes / (s["median_ms"] * 1e-3) / 1e9, 1)
                s["of_hbm"] = round(nbytes / (s["median_ms"] * 1e-3) / HBM, 3)
                row[k] = s
            out.append(row)
            del x, dy, conv
    return out


def step_arm(a, backbone):
    import torch
    from sigma_b200 import modules as M, train_util
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    B, Hh, Ww, ncls = 2, 480, 640, 40
    g = torch.Generator(device="cuda").manual_seed(1)
    batch = (torch.randn(B, 3, Hh, Ww, device="cuda", generator=g), torch.randn(B, 3, Hh, Ww, device="cuda", generator=g),
             torch.randint(0, ncls, (B, Hh, Ww), device="cuda", generator=g))
    out = {}
    for mode in a.modes.split(","):
        cfg = types.SimpleNamespace(backbone=backbone, decoder="MambaDecoder", num_classes=ncls, image_height=Hh, image_width=Ww,
                                    pretrained_model=None, bn_eps=1e-3, bn_momentum=0.1)
        torch.manual_seed(0)
        with contextlib.redirect_stdout(io.StringIO()):
            model = M.EncoderDecoder(cfg, criterion=torch.nn.CrossEntropyLoss(reduction="mean", ignore_index=255)).cuda().train()
        kw = {"fp32": {}, "bf16": dict(amp_dtype=torch.bfloat16, bf16_core=True),
              "fp16": dict(amp_dtype=torch.float16, fp16_core=True, scaler=torch.amp.GradScaler("cuda"))}[mode]
        opt = train_util.make_optimizer(model, capturable=True, fused=mode == "fp16")
        eager = train_util.TrainStep(model, opt, **kw)
        with torch_conv():
            graph_old = train_util.GraphedTrainStep(model, opt, batch, **kw)
        graph_new = train_util.GraphedTrainStep(model, opt, batch, **kw)

        def eager_old(*b):
            with torch_conv():
                return eager(*b)
        arms = {"eager/torch_conv": eager_old, "eager/node": eager, "graph/torch_conv": graph_old, "graph/node": graph_new}
        res = {k: {"rounds": [], "peak": 0} for k in arms}
        for fn in arms.values():
            for _ in range(3):
                fn(*batch)
        torch.cuda.synchronize()
        for _ in range(a.rounds):
            for k, fn in arms.items():
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.steps):
                    fn(*batch)
                e1.record()
                torch.cuda.synchronize()
                res[k]["rounds"].append(e0.elapsed_time(e1) / a.steps)
                res[k]["peak"] = max(res[k]["peak"], torch.cuda.max_memory_allocated())
        for k, r in res.items():
            r.update(stats(r.pop("rounds")))
            r["peak_mem_GB"] = round(r.pop("peak") / 2 ** 30, 2)
        out[mode] = res
        del arms, graph_old, graph_new, eager, model, opt
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "bench_dwconv_train"))
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--models", default="sigma_tiny,sigma_small")
    ap.add_argument("--modes", default="fp32,bf16,fp16")
    ap.add_argument("--skip-step", action="store_true")
    ap.add_argument("--backbone", help=argparse.SUPPRESS)       # the whole-step arm of one backbone, in a child process
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_dwconv_train.py needs a CUDA device"
    if a.backbone:
        print(json.dumps(step_arm(a, a.backbone)))
        return
    os.makedirs(a.out, exist_ok=True)
    result = {"card": card(), "rounds": a.rounds, "iters": a.iters, "op": op_arm(a), "step": {}}
    print(f"card: {result['card']}")
    print("| dtype | B, H, W, D | alg. MB | ours ms | torch ms | ours GB/s (of 3.35 TB/s) | torch GB/s |")
    print("|---|---|---|---|---|---|---|")
    for r in result["op"]:
        o, t = r["ours"], r["torch"]
        print(f"| {r['dtype']} | {r['shape']} | {r['alg_MB']} | {o['median_ms']} [{o['min_ms']}, {o['max_ms']}] | {t['median_ms']} "
              f"[{t['min_ms']}, {t['max_ms']}] | {o['GBps']} ({o['of_hbm']:.0%}) | {t['GBps']} |")
    if not a.skip_step:
        for bb in a.models.split(","):     # one process per backbone, so each starts with a fresh allocator and cuDNN
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--backbone", bb, "--modes", a.modes, "--rounds", str(a.rounds),
                                "--steps", str(a.steps)], capture_output=True, text=True)
            if r.returncode != 0:
                raise SystemExit(f"{bb} failed:\n{r.stderr[-4000:]}")
            result["step"][bb] = json.loads(r.stdout.strip().splitlines()[-1])
        print("| model | mode | arm | ms/step | peak GB |")
        print("|---|---|---|---|---|")
        for bb, modes in result["step"].items():
            for mode, arms in modes.items():
                for k, r in arms.items():
                    print(f"| {bb} | {mode} | {k} | {r['median_ms']} [{r['min_ms']}, {r['max_ms']}] | {r['peak_mem_GB']} |")
    with open(os.path.join(a.out, "bench_dwconv_train.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
