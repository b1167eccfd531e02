"""Time the op-level selective scan backward at wide states (scan_op_bwd_wide.cu) against the reference CUDA extension
(selective_scan_cuda_core built for sm_90a into oracle/_ref by oracle/build_ref_ext.py), on the same GPU and the same tensors.

    python scripts/bench_scan_wide_state.py [--rounds 7] [--dtypes f32 bf16] [--out results.json]

One JSON line per (shape, dtype) on stdout; --out also writes the card and all rows to that file.

Shapes: the d_state="auto" SS2D calls (K = 4 directions, so G = 4) at batch 2: Sigma-tiny stages 1 - 3 and Sigma-base stage 3.
Per call: the backward alone (ours: sigma_scan_bwd through ops.selective_scan_cuda_core_bwd; the reference: its bwd, given the
chunk states of its own forward) and forward + backward.  CUDA events; every shape warmed; ours and the reference alternate
within each round; median and range over the rounds.  The card's name and power limit are read in the same run, and the two
backwards' outputs are compared (max error over each output's scale)."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle", "_ref")]
from sigma_b200 import ops  # noqa: E402

# name, batch, dim (= 4 directions x d_inner), L, d_state
SHAPES = [("tiny-s1", 2, 1536, 4800, 32), ("tiny-s2", 2, 3072, 1200, 64), ("tiny-s3", 2, 6144, 300, 128),
          ("base-s3", 2, 8192, 690, 171)]
DT = {"f32": torch.float32, "bf16": torch.bfloat16}
G = 4


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def inputs(b, dim, L, N, dt):
    g = torch.Generator(device="cuda").manual_seed(dim * 1000 + N)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    u, dout = r(b, dim, L).to(dt), r(b, dim, L).to(dt)
    delta = (0.5 * r(b, dim, L)).to(dt)
    dtv = torch.exp(torch.rand(dim, device="cuda", generator=g) * (torch.log(torch.tensor(0.1)) - torch.log(torch.tensor(1e-3)))
                    + torch.log(torch.tensor(1e-3, device="cuda")))
    bias = dtv + torch.log(-torch.expm1(-dtv))
    A = -torch.exp(torch.log(torch.arange(1, N + 1, device="cuda", dtype=torch.float32)).repeat(dim, 1))
    B, C = r(b, G, N, L).to(dt), r(b, G, N, L).to(dt)
    D = torch.ones(dim, device="cuda")
    return u, delta, A, B, C, D, bias, dout


def time_pair(fns, rounds):
    """each fn warmed; then `rounds` rounds, the fns alternating within a round -> per fn (median, min, max) in ms"""
    for f in fns:
        f()
        f()
    torch.cuda.synchronize()
    ts = [[] for _ in fns]
    for _ in range(rounds):
        for i, f in enumerate(fns):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            torch.cuda.synchronize()
            ts[i].append(e0.elapsed_time(e1))
    return [(sorted(t)[len(t) // 2], min(t), max(t)) for t in ts]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--dtypes", nargs="+", default=["f32", "bf16"])
    ap.add_argument("--out", default=None, help="also write the card and every row to this JSON file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a GPU")
    import selective_scan_cuda_core as ref   # the reference extension, built for sm_90a
    rows = []
    gpu = card()
    print("card:", gpu)
    for name, b, dim, L, N in SHAPES:
        for dn in a.dtypes:
            args = inputs(b, dim, L, N, DT[dn])
            u, delta, A, B, C, D, bias, dout = args
            _, x_ref = ref.fwd(u, delta, A, B, C, D, bias, True, 1)
            ours_b = lambda: ops.selective_scan_cuda_core_bwd(u, delta, A, B, C, D, bias, dout, None, True, 1)
            ref_b = lambda: ref.bwd(u, delta, A, B, C, D, bias, dout, x_ref, True, 1)

            def ours_fb():
                _, x = ops.selective_scan_cuda_core_fwd(u, delta, A, B, C, D, bias, True, 1)
                return ops.selective_scan_cuda_core_bwd(u, delta, A, B, C, D, bias, dout, x, True, 1)

            def ref_fb():
                _, x = ref.fwd(u, delta, A, B, C, D, bias, True, 1)
                return ref.bwd(u, delta, A, B, C, D, bias, dout, x, True, 1)

            err = {}
            for k, g_, r_ in zip(("du", "ddelta", "dA", "dB", "dC", "dD", "ddelta_bias"), ours_b(), ref_b()):
                err[k] = float((g_.float() - r_.float()).abs().max()) / float(r_.float().abs().max())
            (ob, rb) = time_pair([ours_b, ref_b], a.rounds)
            (ofb, rfb) = time_pair([ours_fb, ref_fb], a.rounds)
            row = dict(shape=name, batch=b, dim=dim, L=L, N=N, G=G, dtype=dn,
                       ours_bwd_ms=[round(v, 3) for v in ob], ref_bwd_ms=[round(v, 3) for v in rb],
                       bwd_speedup=round(rb[0] / ob[0], 2),
                       ours_fwd_bwd_ms=[round(v, 3) for v in ofb], ref_fwd_bwd_ms=[round(v, 3) for v in rfb],
                       fwd_bwd_speedup=round(rfb[0] / ofb[0], 2), max_err_over_scale={k: float(f"{v:.2e}") for k, v in err.items()})
            rows.append(row)
            print(json.dumps(row), flush=True)
            del args, u, delta, A, B, C, D, bias, dout, x_ref
            torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(card=gpu, rounds=a.rounds, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
