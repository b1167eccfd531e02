"""Sigma-tiny 480x640 inference at B = 74 by CUDA-graph replay in the fused path's five modes — tf32x3 (default), tf32
(torch.backends.cuda.matmul.allow_tf32), bf16 (torch.autocast("cuda", dtype=torch.bfloat16)), fp8
(sigma_b200.fused.fp8_inference()) and fp16 (sigma_b200.fused.fp16_inference()) — alternating in one process
after warm-up.  Prints one JSON line: images/s per mode (median of the rounds), each mode's logits error against tf32x3 on
the same seeded inputs (max |diff| / max |logit|), peak memory per mode, and the card name and power limit read in the same run.

    python scripts/bench_precision.py [--batch 74] [--rounds 5] [--steps 10]
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        name, limit = [v.strip() for v in q.split(",")]
        return name, limit
    except Exception as e:   # noqa: BLE001 - reported, not hidden
        return torch.cuda.get_device_name(0), f"unknown ({e})"


def _mode_ctx(mode):
    from sigma_b200 import fused
    torch.backends.cuda.matmul.allow_tf32 = mode == "tf32"
    if mode == "fp8":
        return fused.fp8_inference()
    if mode == "fp16":
        return fused.fp16_inference()
    return torch.autocast("cuda", dtype=torch.bfloat16) if mode == "bf16" else contextlib.nullcontext()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=74)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_precision.py needs a CUDA device")
    import procedural as P
    from helpers import cfg_tiny
    from sigma_b200 import fused, modules as M
    B, H, W = args.batch, args.height, args.width
    with contextlib.redirect_stdout(io.StringIO()):
        model = M.EncoderDecoder(cfg_tiny(H, W), criterion=None)
    P.fill_state_dict(model, 7)
    model = model.cuda().eval()
    rgb = P.randn(7, "bench/rgb", (B, 3, H, W)).cuda()
    x = P.randn(7, "bench/x", (B, 3, H, W)).cuda()
    modes = ["tf32x3", "tf32", "bf16", "fp8", "fp16"]
    graphs, outs, peak = {}, {}, {}
    stream = torch.cuda.Stream()
    pool = torch.cuda.graph_pool_handle()            # one memory pool for the five graphs (replayed one at a time): five
                                                     # private pools of a B = 74 forward do not fit in 80 GB
    for m in modes:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        with torch.cuda.stream(stream), torch.no_grad(), _mode_ctx(m):
            assert fused.precision() == m, (fused.precision(), m)
            for _ in range(2):
                model(rgb, x)
            stream.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream, pool=pool):
                outs[m] = model(rgb, x)
        stream.synchronize()
        graphs[m] = g
        peak[m] = torch.cuda.max_memory_allocated() / 2 ** 30
    torch.backends.cuda.matmul.allow_tf32 = False
    times = {m: [] for m in modes}
    with torch.cuda.stream(stream):
        for m in modes:                              # warm-up replays
            for _ in range(3):
                graphs[m].replay()
        for _ in range(args.rounds):                 # alternate modes round by round
            for m in modes:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(args.steps):
                    graphs[m].replay()
                e1.record(stream)
                e1.synchronize()
                times[m].append(e0.elapsed_time(e1) / args.steps)
        final = {}
        for m in modes:                              # a graph's output can share pool memory with another's intermediates:
            graphs[m].replay()                       # read each right after its own replay
            final[m] = outs[m].float().clone()
        stream.synchronize()
    outs = final
    ref = outs["tf32x3"].float()
    scale = float(ref.abs().max())
    name, limit = _card()
    res = {"workload": f"sigma_tiny {H}x{W} B={B} CUDA-graph replay", "gpu": name, "power_limit": limit}
    for m in modes:
        ms = sorted(times[m])[len(times[m]) // 2]
        res[m] = {"images_per_s": round(B / ms * 1e3, 2), "ms_per_step": round(ms, 3),
                  "ms_all_rounds": [round(t, 3) for t in times[m]],
                  "logits_err_vs_tf32x3_of_scale": float((outs[m].float() - ref).abs().max()) / scale,
                  "labels_equal_vs_tf32x3": float((outs[m].argmax(1) == ref.argmax(1)).float().mean()),
                  "peak_mem_gib": round(peak[m], 2)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
