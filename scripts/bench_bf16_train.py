"""Measure the bf16 training mode of the fused core (ops.BF16_TRAINING_CORE) against the default under bf16 autocast, in one process,
alternating the two after warming both up: median and spread of `--rounds` rounds of `--steps` steps, timed with CUDA events.
With --amp fp16, the fp16 training mode (ops.FP16_TRAINING_CORE) against the default under fp16 autocast, both arms stepping through
a torch.amp.GradScaler (fp16 autocast's usual recipe).

    python scripts/bench_bf16_train.py [--amp bf16|fp16] [--out DIR] [--rounds 5] [--steps 10] [--models sigma_small,sigma_tiny] [--profile]

* whole training step (forward + backward + AdamW) at 480 x 640, batch 2: step time, peak memory (torch.cuda.max_memory_allocated)
  and the loss of both modes on the same seeded batch;
* per call at the four stage shapes of Sigma-tiny (SS2D, d_state 16): the core's forward-save and backward, fp32 and bf16 (fp16
  with --amp fp16), with the ALGORITHMIC bytes computed from the shapes below and the GB/s that follow from them (not a measured memory traffic);
* the card's name and power limit, queried in the same run (nothing is set);
* --profile: a separate torch.profiler pass of one step per mode, top kernels by time, written under --out.
Needs a GPU: there is no CPU fallback."""
import argparse
import contextlib
import io
import json
import os
import statistics
import subprocess
import sys
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

STAGES = [(120, 160, 192, 6), (60, 80, 384, 12), (30, 40, 768, 24), (15, 20, 1536, 48)]   # H, W, d_inner, dt_rank of Sigma-tiny at 480 x 640


def core_bytes(B, H, W, D, N, R, Cp, K, bf16):
    """algorithmic bytes of one forward-save and one backward of the core (kind CROSS4): every tensor once per direction that
    reads or writes it.  e = bytes of an xc / y / delta' / dy element (bf16: any 16-bit element type)."""
    e = 2 if bf16 else 4
    pos = B * H * W
    hs = K * B * -(-H * W // 16) * D * N * 4                      # one state per 16-position block and direction (upper bound: row tiles)
    fwd = K * pos * (D * e + Cp * 4 + 2 * D * e) + hs             # read xc + x_dbl row, write y + delta'; write hs
    bwd = K * pos * (3 * D * e + Cp * 4 + 2 * D * 4 + 2 * N * 4) + hs   # read xc, dy, delta', x_dbl; write ddelta, add du, add dB / dC; read hs
    return fwd, bwd


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def med(v):
    return {"median_ms": round(statistics.median(v), 3), "min_ms": round(min(v), 3), "max_ms": round(max(v), 3)}


def bench_steps(a, backbone, out):
    import torch
    from sigma_b200 import modules as M, ops, train_util
    cfg = types.SimpleNamespace(backbone=backbone, decoder="MambaDecoder", num_classes=40, image_height=480, image_width=640,
                                pretrained_model=None, bn_eps=1e-3, bn_momentum=0.1)
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        model = M.EncoderDecoder(cfg, criterion=torch.nn.CrossEntropyLoss(reduction="mean", ignore_index=255)).cuda().train()
    opt = train_util.make_optimizer(model)
    g = torch.Generator(device="cuda").manual_seed(1)
    rgb = torch.randn(2, 3, 480, 640, device="cuda", generator=g)
    mx = torch.randn(2, 3, 480, 640, device="cuda", generator=g)
    gt = torch.randint(0, 40, (2, 480, 640), device="cuda", generator=g)
    if a.amp == "fp16":
        steps = {on: train_util.TrainStep(model, opt, amp_dtype=torch.float16, fp16_core=on, scaler=torch.amp.GradScaler("cuda"))
                 for on in (False, True)}
    else:
        steps = {on: train_util.TrainStep(model, opt, amp_dtype=torch.bfloat16, bf16_core=on) for on in (False, True)}
    state = {k: v.clone() for k, v in model.state_dict().items()}
    res = {}
    for on in (False, True):      # the loss of both modes from the same weights on the same batch, and their peak memory
        model.load_state_dict(state)
        torch.cuda.synchronize(); torch.cuda.reset_peak_memory_stats()
        loss = float(steps[on](rgb, mx, gt))
        torch.cuda.synchronize()
        res[on] = {"first_step_loss": loss, "peak_mem_MB": round(torch.cuda.max_memory_allocated() / 2 ** 20, 1), "rounds": []}
    for on in (False, True):
        timed(lambda: steps[on](rgb, mx, gt), 3)
    for _ in range(a.rounds):
        for on in (False, True):
            res[on]["rounds"].append(timed(lambda: steps[on](rgb, mx, gt), a.steps))
    for on in (False, True):
        res[on].update(med(res[on].pop("rounds")))
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        for on in (False, True):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                steps[on](rgb, mx, gt)
                torch.cuda.synchronize()
            with open(os.path.join(out, f"profile_{backbone}_{a.amp + 'core' if on else 'default'}.txt"), "w") as f:
                f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=30, max_name_column_width=90))
    del model, opt, steps
    torch.cuda.empty_cache()
    return {"default": res[False], f"{a.amp}_core": res[True]}


def bench_calls(a):
    import torch
    from sigma_b200 import _lib, fused, ops
    from sigma_b200._lib import ptr, stream
    L_ = _lib.lib()
    rows = []
    B, N, K, kind = 2, 16, 4, _lib.DIRS_CROSS4
    for H, W, D, R in STAGES:
        Cp = L_.sigma_ss2d_padded_cp(N, R)
        g = torch.Generator(device="cuda").manual_seed(H)
        rn = lambda *s: torch.randn(*s, device="cuda", generator=g)
        xdbl = rn(B * H * W, K * Cp)
        dtw, dtb = rn(K, D, R) * R ** -0.5, rn(K, D) - 4.0
        A = -torch.arange(1, N + 1, device="cuda", dtype=torch.float32).repeat(K * D, 1)
        Ds = rn(K * D)
        wsb = L_.sigma_ss2d_scan_bwd_workspace_bytes(kind, B, H, W, D, N)
        ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
        f32 = lambda *s: torch.empty(*s, device="cuda")
        outs = (f32(B, H * W, D), f32(K, B, H * W, D), f32(B * H * W, K, Cp), f32(K * D, N), f32(K * D), f32(K, D))
        row = {"stage": f"{H}x{W} D{D} R{R}"}
        for bf16 in (False, True):
            dt = (torch.float16 if a.amp == "fp16" else torch.bfloat16) if bf16 else torch.float32
            xc, dy = rn(B, H * W, D).to(dt), rn(B, H * W, D).to(dt)
            y, delta, hs = fused.ss2d_scan_save(kind, xc, xdbl, dtw, dtb, A, Ds, B, H, W, D, N, R, Cp)
            fwd = lambda: fused.ss2d_scan_save(kind, xc, xdbl, dtw, dtb, A, Ds, B, H, W, D, N, R, Cp)
            fn = getattr(L_, f"sigma_ss2d_scan_bwd_saved_{a.amp}") if bf16 else L_.sigma_ss2d_scan_bwd_saved
            bwd = lambda: _lib.check(fn(kind, ptr(xc), ptr(xdbl), ptr(dtw), ptr(dtb), ptr(A), ptr(Ds), ptr(dy), ptr(delta), ptr(hs),
                                        *(ptr(o) for o in outs), B, H, W, D, N, R, Cp, ptr(ws), wsb, 0, stream()), "bwd")
            fb, bb = core_bytes(B, H, W, D, N, R, Cp, K, bf16)
            for name, call, nb in (("fwd_save", fwd, fb), ("bwd", bwd, bb)):
                timed(call, 5)
                t = [timed(call, max(a.steps, 20)) for _ in range(a.rounds)]
                m = statistics.median(t)
                row[f"{name}_{a.amp if bf16 else 'f32'}"] = {**med(t), "algorithmic_MB": round(nb / 1e6, 1), "algorithmic_GBps": round(nb / m / 1e6, 1)}
        rows.append(row)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--amp", choices=("bf16", "fp16"), default="bf16", help="autocast dtype, and the 16-bit training mode compared")
    ap.add_argument("--out", default=None, help="directory for the JSON result and the profiles (default: a temporary directory)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--models", default="sigma_small,sigma_tiny")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--shapes-only", action="store_true", help="print the algorithmic bytes per stage and exit (needs no GPU)")
    a = ap.parse_args()
    if a.rounds < 5 or a.steps < 10:
        ap.error("at least 5 rounds of at least 10 steps")
    if a.shapes_only:
        for H, W, D, R in STAGES:
            Cp = 2 * 16 + (R if R in (4, 8, 12, 16, 24, 32, 48, 64) else {6: 8}[R])
            print(H, W, D, R, [core_bytes(2, H, W, D, 16, R, Cp, 4, b) for b in (False, True)])
        return
    import tempfile
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_bf16_train.py measures on a GPU; none is visible")
    out = a.out or tempfile.mkdtemp(prefix="bench_bf16_train_")
    os.makedirs(out, exist_ok=True)
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    res = {"card": card(), "rounds": a.rounds, "steps_per_round": a.steps, "calls": bench_calls(a), "steps": {}}
    if a.amp == "fp16":
        res["amp"] = "fp16 autocast, GradScaler in both arms"
    for m in [m for m in a.models.split(",") if m]:
        res["steps"][m] = bench_steps(a, m, out)
    with open(os.path.join(out, "bench_bf16_train.json" if a.amp == "bf16" else "bench_fp16_train.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
