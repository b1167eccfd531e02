"""CroMB training: the fused CROSS scan core against the composed path (op-level scans).

    python scripts/bench_cromb_train.py [--rounds 7] [--iters 10] [--steps 5] [--out result.json]

1. The CroMB block (CrossMambaFusionBlock) forward + backward at the four Sigma-tiny 480 x 640 stage shapes, 2 images per GPU.
2. One whole Sigma-tiny 480 x 640 training step (train_util.TrainStep, AdamW, TF32 dense layers as bench.py --mode train), batch 2.
Each is timed with CUDA events, fused and composed alternating within one process, every shape warmed first; the median over the
rounds is reported.  Only CroMB is switched: the composed arm runs CrossMambaFusion_SS2D_SSM.forward with ops.FUSED_TRAINING off,
every other block trains through the fused core in both arms.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from sigma_b200 import modules as M, ops, train_util  # noqa: E402

STAGES = [(120, 160, 96), (60, 80, 192), (30, 40, 384), (15, 20, 768)]     # Sigma-tiny at 480 x 640: (H/4^.., W/4^.., C)
_fused_forward = M.CrossMambaFusion_SS2D_SSM.forward


def _composed_forward(self, *a, **k):
    prev = ops.FUSED_TRAINING
    ops.FUSED_TRAINING = False
    try:
        return _fused_forward(self, *a, **k)
    finally:
        ops.FUSED_TRAINING = prev


def route(fused):
    M.CrossMambaFusion_SS2D_SSM.forward = _fused_forward if fused else _composed_forward


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[0] if q else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--images", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_cromb_train: needs a CUDA GPU")
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = True
    torch.manual_seed(0)
    res = dict(card=card(), images=a.images, rounds=a.rounds, block_ms={}, step_ms={})

    blocks = []
    for H, W, C in STAGES:
        blk = M.CrossMambaFusionBlock(hidden_dim=C, mlp_ratio=0.0, d_state=4, drop_path=0.0).cuda().train()
        xs = [torch.randn(a.images, H, W, C, device="cuda", requires_grad=True) for _ in range(2)]
        wts = [torch.randn(a.images, H, W, C, device="cuda") for _ in range(2)]

        def fb(blk=blk, xs=xs, wts=wts):
            o = blk(*xs)
            sum((t * w).sum() for t, w in zip(o, wts)).backward()
        blocks.append((f"{H}x{W}xC{C}", fb))
    times = {(n, f): [] for n, _ in blocks for f in (True, False)}
    for fused in (True, False):            # warm every shape on both routes
        route(fused)
        for _, fb in blocks:
            timed(fb, 2)
    for _ in range(a.rounds):
        for fused in (True, False):
            route(fused)
            for n, fb in blocks:
                times[(n, fused)].append(timed(fb, a.iters))
    for n, _ in blocks:
        f, c = statistics.median(times[(n, True)]), statistics.median(times[(n, False)])
        res["block_ms"][n] = dict(fused=round(f, 3), composed=round(c, 3), speedup=round(c / f, 3))
        print(f"CroMB block {n:>16}: fused {f:8.3f} ms  composed {c:8.3f} ms  x{c / f:.2f}", flush=True)
    del blocks

    cfg = types.SimpleNamespace(backbone="sigma_tiny", decoder="MambaDecoder", num_classes=40, image_height=480, image_width=640,
                                pretrained_model=None, bn_eps=1e-3, bn_momentum=0.1)
    model = M.EncoderDecoder(cfg, criterion=torch.nn.CrossEntropyLoss(reduction="mean", ignore_index=255)).cuda().train()
    step = train_util.TrainStep(model, train_util.make_optimizer(model))
    rgb = torch.randn(a.images, 3, 480, 640, device="cuda")
    mx = torch.randn(a.images, 3, 480, 640, device="cuda")
    gt = torch.randint(0, 40, (a.images, 480, 640), device="cuda")
    st = {True: [], False: []}
    for fused in (True, False):
        route(fused)
        timed(lambda: step(rgb, mx, gt), 2)
    for _ in range(a.rounds):
        for fused in (True, False):
            route(fused)
            st[fused].append(timed(lambda: step(rgb, mx, gt), a.steps))
    f, c = statistics.median(st[True]), statistics.median(st[False])
    res["step_ms"] = dict(fused=round(f, 2), composed=round(c, 2), speedup=round(c / f, 3))
    print(f"Sigma-tiny 480x640 training step, batch {a.images}: CroMB fused {f:.2f} ms  composed {c:.2f} ms  x{c / f:.3f}", flush=True)
    route(True)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
