"""Dense-projection GEMMs of Sigma-tiny at `--images` per GPU: our wgmma kernel vs cuBLAS (torch.mm), in the precision of
`--precision` (tf32: one TF32 MMA per k-step, cuBLAS TF32; tf32x3: three TF32 MMAs per k-step, cuBLAS fp32).
Reports ms, effective GB/s over (A read once + C written once [+ residual read]) and TFLOP/s over 2·M·N·K; for our tf32x3
kernel also the TF32 tensor-core rate, 3 x 2·M·N·K (A_lo·W_hi + A_hi·W_lo + A_hi·W_hi).
--precision fp8 times, at the GEMMs the FP8 inference mode quantizes (in_proj, out_proj, the patch-merge reduction), our
bf16 instance (bf16 A, as in the bf16 mode) against our e4m3 instance (A already quantized, as the fused producers emit it);
bytes count A at 2 or 1 byte per element (+ 4 per row of scales), C fp32."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sigma_b200 import fused  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--images", type=int, default=16)
ap.add_argument("--only", nargs="*", default=None)
ap.add_argument("--precision", default="tf32", choices=["tf32", "tf32x3", "fp8"])
a = ap.parse_args()
torch.backends.cuda.matmul.allow_tf32 = a.precision == "tf32"
S = 2 * a.images
# name, M, N, K, residual
SHAPES = [
    ("in_proj0", S * 19200, 384, 96, False), ("x_proj0", S * 19200, 160, 192, False), ("out_proj0", S * 19200, 96, 192, True),
    ("in_proj1", S * 4800, 768, 192, False), ("x_proj1", S * 4800, 176, 384, False), ("out_proj1", S * 4800, 192, 384, True),
    ("in_proj2", S * 1200, 1536, 384, False), ("x_proj2", S * 1200, 224, 768, False), ("out_proj2", S * 1200, 384, 768, True),
    ("in_proj3", S * 300, 3072, 768, False), ("x_proj3", S * 300, 320, 1536, False), ("out_proj3", S * 300, 768, 1536, True),
    ("merge0", S * 4800, 192, 384, False), ("dec_x_proj", a.images * 19200, 64, 192, False),
]
print(f"precision {fused.precision()}, {torch.cuda.get_device_name()}", flush=True)
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
for name, M, N, K, res in SHAPES:
    if a.only and name not in a.only:
        continue
    if a.precision == "fp8":
        if "x_proj" in name:                         # x_proj stays bf16 in the FP8 mode
            continue
        A = torch.randn(M, K, device="cuda")
        W = torch.randn(N, K, device="cuda") * K ** -0.5
        R = torch.randn(M, N, device="cuda") if res else None
        out = torch.empty(M, N, device="cuda")
        operands = {"bf16": A.to(torch.bfloat16), "e4m3": fused.quantize_rows(A)}
        line = f"{name:11s} M={M:7d} N={N:5d} K={K:5d}: "
        for mode, op in operands.items():
            byt = (2 if mode == "bf16" else 1) * M * K + (4 * M if mode == "e4m3" else 0) + 4 * M * N * (2 if res else 1)
            ts = []
            for _ in range(7):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fused.linear(op, W, None, out=out, residual=R)
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            ms = sorted(ts[1:])[3]
            line += f"{mode} {ms:7.3f} ms {byt / ms / 1e6:7.1f} GB/s {2 * M * N * K / ms / 1e9:6.1f} TFLOP/s   "
        print(line, flush=True)
        continue
    A = torch.randn(M, K, device="cuda")
    W = torch.randn(N, K, device="cuda") * K ** -0.5
    R = torch.randn(M, N, device="cuda") if res else None
    out = torch.empty(M, N, device="cuda")
    byt = 4 * (M * K + M * N * (2 if res else 1) + N * K)
    flop = 2 * M * N * K
    line = f"{name:11s} M={M:7d} N={N:5d} K={K:5d}: "
    for mode in ("wgmma", "cublas"):
        fused.USE_OWN_GEMM = mode == "wgmma"
        ts = []
        for _ in range(5):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fused.linear(A, W, None, out=out, residual=R)
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ms = sorted(ts[1:])[2]
        line += f"{mode} {ms:7.3f} ms {byt / ms / 1e6:7.1f} GB/s {flop / ms / 1e9:6.1f} TFLOP/s"
        if mode == "wgmma" and a.precision == "tf32x3":
            line += f" ({3 * flop / ms / 1e9:6.1f} tensor)"
        line += "   "
    print(line, flush=True)
