"""Measure the training step replayed from one CUDA graph (train_util.GraphedTrainStep) against the eager TrainStep, in one process
per backbone, alternating the two after warming both up.

    python scripts/bench_train_graph.py [--out DIR] [--models sigma_tiny,sigma_small] [--modes fp32,bf16,fp16] [--rounds 5] [--steps 10]

Sigma at 480 x 640, batch 2 (Sigma's recipe: 2 images per GPU), 40 classes, AdamW (make_optimizer(capturable=True); fused=True
as well in the fp16 mode, whose GradScaler needs it inside the graph).  Modes:
  fp32  TF32 dense layers (torch.backends.cuda.matmul / cudnn allow_tf32 = True), no autocast;
  bf16  bf16 autocast with the bf16 training core;
  fp16  fp16 autocast with the fp16 training core and a GradScaler.
Both arms share one model and optimizer per mode.  Per arm: step time from CUDA events over rounds of --steps steps (median
[min, max] of --rounds rounds, the arms alternating round by round), host time per step (perf_counter around the same rounds,
up to the last enqueue), sigma_b200 kernel launches the host issues per step (_lib.launch_count(); a replay issues none of its
own: the graph holds them) and peak memory.  Eager: torch.cuda.max_memory_allocated over its timed rounds (it includes the graph's
gradient buffers, one parameter-sized set).  Graph: torch.cuda.memory_reserved right after the capture, before any eager step,
with the cache emptied: model, optimizer state and the graph's private pool, whose freed blocks max_memory_allocated would
miss.  The card's name and power limit are read in the same run (nothing is set).
The backbones run in separate processes so that each starts with a fresh cuDNN (INTEGRATION.md §3: an fp16 training step of a
ConMB block can spoil cuDNN's fp16 depthwise convolution for a model built later in the process).  Needs a GPU."""
import argparse
import contextlib
import io
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def run_backbone(a):
    import torch
    from sigma_b200 import _lib, modules as M, train_util
    assert torch.cuda.is_available(), "bench_train_graph.py needs a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    B, Hh, Ww, ncls = 2, 480, 640, 40
    g = torch.Generator(device="cuda").manual_seed(1)
    batch = (torch.randn(B, 3, Hh, Ww, device="cuda", generator=g), torch.randn(B, 3, Hh, Ww, device="cuda", generator=g),
             torch.randint(0, ncls, (B, Hh, Ww), device="cuda", generator=g))
    out = {}
    for mode in a.modes.split(","):
        cfg = types.SimpleNamespace(backbone=a.backbone, decoder="MambaDecoder", num_classes=ncls, image_height=Hh, image_width=Ww,
                                    pretrained_model=None, bn_eps=1e-3, bn_momentum=0.1)
        torch.manual_seed(0)
        with contextlib.redirect_stdout(io.StringIO()):
            model = M.EncoderDecoder(cfg, criterion=torch.nn.CrossEntropyLoss(reduction="mean", ignore_index=255)).cuda().train()
        kw = {"fp32": {}, "bf16": dict(amp_dtype=torch.bfloat16, bf16_core=True),
              "fp16": dict(amp_dtype=torch.float16, fp16_core=True, scaler=torch.amp.GradScaler("cuda"))}[mode]
        opt = train_util.make_optimizer(model, capturable=True, fused=mode == "fp16")
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        graph = train_util.GraphedTrainStep(model, opt, batch, **kw)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()                        # what stays reserved: model, optimizer state, the graph's private pool
        graph_mem = torch.cuda.memory_reserved()
        arms = {"eager": train_util.TrainStep(model, opt, **kw), "graph": graph}
        res = {k: {"rounds": [], "host": [], "peak": 0} for k in arms}
        for k, fn in arms.items():
            for _ in range(3):
                fn(*batch)
            torch.cuda.synchronize()
            n0 = _lib.launch_count()
            fn(*batch)
            res[k]["launches_per_step"] = _lib.launch_count() - n0
            torch.cuda.synchronize()
        for _ in range(a.rounds):
            for k, fn in arms.items():
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0 = time.perf_counter()
                e0.record()
                for _ in range(a.steps):
                    fn(*batch)
                e1.record()
                t1 = time.perf_counter()
                torch.cuda.synchronize()
                res[k]["rounds"].append(e0.elapsed_time(e1) / a.steps)
                res[k]["host"].append((t1 - t0) * 1e3 / a.steps)
                res[k]["peak"] = max(res[k]["peak"], torch.cuda.max_memory_allocated() if k == "eager" else graph_mem)
        for k, r in res.items():
            v = r.pop("rounds")
            r.update(median_ms=round(statistics.median(v), 3), min_ms=round(min(v), 3), max_ms=round(max(v), 3),
                     host_ms=round(statistics.median(r.pop("host")), 3), peak_mem_GB=round(r.pop("peak") / 2 ** 30, 2))
        out[mode] = res
        del arms, graph, fn, model, opt
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "bench_train_graph"))
    ap.add_argument("--models", default="sigma_tiny,sigma_small")
    ap.add_argument("--modes", default="fp32,bf16,fp16")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--backbone", help=argparse.SUPPRESS)       # set in the per-backbone child process
    a = ap.parse_args()
    if a.steps < 10 or a.rounds < 1:
        raise SystemExit("--steps must be >= 10 and --rounds >= 1")
    if a.backbone:
        print(json.dumps(run_backbone(a)))
        return
    os.makedirs(a.out, exist_ok=True)
    result = {"card": card(), "batch": 2, "size": "480x640", "steps_per_round": a.steps, "rounds": a.rounds, "models": {}}
    for bb in a.models.split(","):
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--backbone", bb, "--modes", a.modes, "--rounds", str(a.rounds),
                            "--steps", str(a.steps)], capture_output=True, text=True)
        if r.returncode != 0:
            raise SystemExit(f"{bb} failed:\n{r.stderr[-4000:]}")
        result["models"][bb] = json.loads(r.stdout.strip().splitlines()[-1])
    with open(os.path.join(a.out, "bench_train_graph.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(f"card: {result['card']}")
    print("| model | mode | eager ms/step | graphed ms/step | speed-up | host ms/step eager / graphed | sigma launches/step eager / graphed "
          "| peak GB eager / graphed |")
    print("|---|---|---|---|---|---|---|---|")
    for bb, modes in result["models"].items():
        for mode, r in modes.items():
            e, g = r["eager"], r["graph"]
            print(f"| {bb} | {mode} | {e['median_ms']} [{e['min_ms']}, {e['max_ms']}] | {g['median_ms']} [{g['min_ms']}, {g['max_ms']}] "
                  f"| {e['median_ms'] / g['median_ms']:.2f}x | {e['host_ms']} / {g['host_ms']} | {e['launches_per_step']} / "
                  f"{g['launches_per_step']} | {e['peak_mem_GB']} / {g['peak_mem_GB']} |")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
