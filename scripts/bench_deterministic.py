"""Cost of torch.use_deterministic_algorithms(True): the Sigma-tiny training step at `bench.py --mode train`'s shape (480x640,
batch 2, fp32 with TF32 dense layers, AdamW), default and deterministic, alternating in one process; then each backward kernel
per call, default entry vs `_det` entry, at that step's stage-0 shapes.  Prints the card and its power limit with the numbers.

    CUBLAS_WORKSPACE_CONFIG=:4096:8 python scripts/bench_deterministic.py [--steps 20] [--rounds 3] [--out det.json]
"""
import argparse
import contextlib
import ctypes
import io
import json
import os
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # the numbers still stand; say what could not be read
        return f"nvidia-smi unavailable ({e})"


def events_ms(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def step_times(a):
    from sigma_b200 import modules as M, train_util
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    torch.manual_seed(0)
    cfg = types.SimpleNamespace(backbone="sigma_tiny", decoder="MambaDecoder", num_classes=9, image_height=a.height,
                                image_width=a.width, pretrained_model=None, bn_eps=1e-3, bn_momentum=0.1)
    with contextlib.redirect_stdout(io.StringIO()):
        model = M.EncoderDecoder(cfg, criterion=torch.nn.CrossEntropyLoss(reduction="mean", ignore_index=255)).cuda().train()
    step = train_util.TrainStep(model, train_util.make_optimizer(model))
    g = torch.Generator().manual_seed(1234)
    rgb = torch.randn(a.batch, 3, a.height, a.width, generator=g).cuda()
    mx = torch.randn(a.batch, 3, a.height, a.width, generator=g).cuda()
    gt = torch.randint(0, 9, (a.batch, a.height, a.width), generator=g).cuda()
    res = {"default": [], "deterministic": []}
    for mode in ("default", "deterministic"):          # warm both
        torch.use_deterministic_algorithms(mode == "deterministic")
        for _ in range(3):
            step(rgb, mx, gt)
    for _ in range(a.rounds):
        for mode in ("default", "deterministic"):
            torch.use_deterministic_algorithms(mode == "deterministic")
            res[mode].append(events_ms(lambda: step(rgb, mx, gt), a.steps))
    torch.use_deterministic_algorithms(False)
    return res


def kernel_times(a):
    """each backward entry per call, default vs _det, at Sigma-tiny stage-0 training shapes (batch 2, 120x160)"""
    import procedural as P
    from sigma_b200 import _lib, ops
    import test_ss2d_bwd_fp64_gpu as F64
    L_ = _lib.lib()
    out = {}
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    st = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    for kind, D, N, R in [("cross4", 192, 16, 6), ("seq2", 192, 4, 6)]:
        B, H, W = a.batch, a.height // 4, a.width // 4
        args, Cp = F64._params(kind, B, H, W, D, N, R, f"bench/{kind}")
        xc, xdbl, dtw, dtb, A, Ds, dy = args
        K = xdbl.shape[2]
        Lseq = xc.shape[1]
        kid = F64._kid(kind)
        delta = torch.empty(K, B, Lseq, D, device="cuda")
        hs = torch.empty(L_.sigma_ss2d_scan_hs_bytes(kid, B, H, W, D, N) // 4, device="cuda")
        fwb = L_.sigma_ss2d_scan_workspace_bytes(kid, B, H, W, D, N)
        fws = torch.empty(max(fwb, 4), dtype=torch.uint8, device="cuda")
        y = torch.empty(K, B, Lseq, D, device="cuda")
        head = (kid, p(xc), p(xdbl), p(dtw), p(dtb), p(A), p(Ds))
        _lib.check(L_.sigma_ss2d_scan_fwd_save(*head, p(y), p(delta), p(hs), B, H, W, D, N, R, Cp, p(fws), fwb, 0, st()), "fwd_save")
        outs = [torch.empty(B, Lseq, D, device="cuda"), torch.empty(K, B, Lseq, D, device="cuda"), torch.empty(B, Lseq, K, Cp, device="cuda"),
                torch.empty(K * D, N, device="cuda"), torch.empty(K * D, device="cuda"), torch.empty(K, D, device="cuda")]
        for det in (False, True):
            wsb = (L_.sigma_ss2d_scan_bwd_det_workspace_bytes if det else L_.sigma_ss2d_scan_bwd_workspace_bytes)(kid, B, H, W, D, N)
            ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
            tail = tuple(p(o) for o in outs) + (B, H, W, D, N, R, Cp, p(ws), wsb, 0, st())
            fn = L_.sigma_ss2d_scan_bwd_saved_det if det else L_.sigma_ss2d_scan_bwd_saved
            call = lambda: fn(*head, p(dy), p(delta), p(hs), *tail)
            call()
            out[f"ss2d_bwd_saved {kind} B{B} {H}x{W} D{D} N{N}" + (" det" if det else "")] = events_ms(call, a.calls)
    # op-level backward (CroMB's scan): batch 2, dim 192, d_state 4, L = 120·160
    u, dl, A, Bm, Cm, D_, bias = P.scan_inputs(5, a.batch, 192, 4, (a.height // 4) * (a.width // 4), 1)
    dout = P.randn(5, "bench/dout", tuple(u.shape))
    c = [t.cuda() for t in (u, dl, A, Bm, Cm, D_, bias, dout)]
    for det in (False, True):
        torch.use_deterministic_algorithms(det)
        call = lambda: ops.selective_scan_cuda_core_bwd(*c[:7], c[7], None, True, 1)
        call()
        out["scan_op_bwd B2 dim192 N4 L19200" + (" det" if det else "")] = events_ms(call, a.calls)
    # LayerNorm backward at stage 0: 2·120·160 rows of 96
    ln = torch.nn.LayerNorm(96).cuda()
    x = torch.randn(a.batch * (a.height // 4) * (a.width // 4), 96, device="cuda", requires_grad=True)
    gy = torch.randn_like(x)
    for det in (False, True):
        torch.use_deterministic_algorithms(det)
        yv = ops.layer_norm(ln, x)
        call = lambda: torch.autograd.grad(yv, (x, ln.weight, ln.bias), gy, retain_graph=True)
        call()
        out["layernorm_bwd rows38400 C96" + (" det" if det else "")] = events_ms(call, a.calls)
    # bilinear backward of the logits upsample (x4, NCHW, 9 classes) vs torch's atomic backward
    z = torch.randn(a.batch, 9, a.height // 4, a.width // 4, device="cuda", requires_grad=True)
    for det in (False, True):
        torch.use_deterministic_algorithms(det)
        yv = ops.upsample_bilinear(z, size=(a.height, a.width))
        gz = torch.randn_like(yv)
        call = lambda: torch.autograd.grad(yv, z, gz, retain_graph=True)
        call()
        out["bilinear_bwd x4 logits" + (" det (sigma)" if det else " (torch)")] = events_ms(call, a.calls)
    torch.use_deterministic_algorithms(False)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if os.environ.get("CUBLAS_WORKSPACE_CONFIG") is None:
        sys.exit("set CUBLAS_WORKSPACE_CONFIG=:4096:8 (torch requires it for cuBLAS under use_deterministic_algorithms)")
    res = {"card": card(), "shape": f"sigma_tiny {a.height}x{a.width} batch {a.batch}, fp32 + TF32 dense, AdamW"}
    st = step_times(a)
    res["step_ms"] = st
    res["step_ms_best"] = {k: min(v) for k, v in st.items()}
    res["ratio"] = res["step_ms_best"]["deterministic"] / res["step_ms_best"]["default"]
    res["kernel_ms_per_call"] = kernel_times(a)
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
