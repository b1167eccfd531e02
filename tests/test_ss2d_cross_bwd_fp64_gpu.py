"""GPU: the fused scan backward of kind CROSS (CroMB: sigma_ss2d_scan_bwd / _bwd_split with its state sweep, and the training pair
sigma_ss2d_scan_fwd_save + sigma_ss2d_scan_bwd_saved) against the fp64 reference of tests/ss2d_cross_ref64.py, element by element
inside its per-element error bounds, at CroMB's training shapes (d_state 4): Sigma-tiny / small 120x160/192/R6, 60x80/384/12,
30x40/768/24, 15x20/1536/48 and Sigma-base 180x240/256/8, 23x30/2048/64, with 1, 2 and 3 images (a batch of 2·images).
* L-segments 1, 2, 7, 64 and the library's choice for the state sweep; the training forward and backward cut alike and differently;
* every output inside NaN-filled memory whose guard elements must stay bit-identical, the dt_r and padding columns of dxdbl 0, and
  a NaN-filled workspace;
* delta' and the tile-start states of the training forward against those of the state sweep.
Worst bound fractions go to helpers.record.  Also: the CROSS kernels exist in the library and use no local memory."""
import ctypes
import re
import subprocess

import pytest
import torch

from helpers import guard_ok, guarded, ptr as _p, record, ss2d_kind, ss2d_params, stream as _stream
from oracle import ss2d_ref64 as R64
from ss2d_cross_ref64 import ss2d_cross_ref64

pytestmark = pytest.mark.gpu
S = 101
N = 4
MAXNORM_TOO = ("ddtb",)     # d dt_bias sums ddelta's per-element bounds over every position: its max-norm error is checked too


def _check(tag, name, got, ref, bnd, worst):
    ok = ~ref.isnan()
    assert bool(torch.equal(got.isnan(), ~ok)), f"{tag} {name}: written where the kernel has nothing to write, or NaN"
    frac = R64.bound_fraction(got[ok], ref[ok], bnd[ok])
    worst[name] = max(worst.get(name, 0.0), frac)
    assert frac <= 1.0, f"{tag} {name}: {frac:.3f} of the per-element bound"
    if name in MAXNORM_TOO:
        err = float((got[ok].double() - ref[ok]).abs().max()) / float(ref[ok].abs().max())
        assert err <= 1e-3, f"{tag} {name}: {err:.2e} of its scale"


def _plan(Bt, H, W, D, nsplit):
    from sigma_b200 import _lib
    out = (ctypes.c_int64 * 4)()
    _lib.check(_lib.lib().sigma_test_ss2d_bwd_plan(_lib.DIRS_CROSS, Bt, H, W, D, N, nsplit, out), "sigma_test_ss2d_bwd_plan")
    return dict(zip(("nsplit", "tiles_per_split", "max_tiles", "min_tiles"), (int(v) for v in out)))


def _run(Bt, H, W, D, R, Cp, args, ref, bnd, tag, worst, split=None, saved=None):
    """split: the state-sweep backward with that L-segment count (0: the library's choice).  saved = (fwd_split, bwd_split): the
    training forward followed by the backward that consumes its delta' and states.  Returns (delta, hs) as the route left them."""
    from sigma_b200 import _lib
    L_ = _lib.lib()
    kind = ss2d_kind("cross")
    xc, xdbl, dtw, dtb, A, Ds, dy = args
    L = H * W
    T = L_.sigma_ss2d_scan_hs_bytes(kind, Bt, H, W, D, N) // (4 * Bt * D * N)
    assert T == -(-L // 16)
    bufs, outs = {}, {}
    for name, shape in [("delta", (1, Bt, L, D)), ("dxc", (Bt, L, D)), ("ddelta", (1, Bt, L, D)), ("dxdbl", (Bt, L, 1, Cp)),
                        ("dA", (2 * D, N)), ("dDs", (2 * D,)), ("ddtb", (2, D)), ("y", (1, Bt, L, D)), ("hs", (1, Bt, T, D, N))]:
        bufs[name], outs[name] = guarded(shape)
    wsb = L_.sigma_ss2d_scan_bwd_workspace_bytes(kind, Bt, H, W, D, N)
    assert wsb > 0
    ws = torch.full((wsb // 4,), float("nan"), device="cuda")
    head = (kind, _p(xc), _p(xdbl), _p(dtw), _p(dtb), _p(A), _p(Ds))
    tail = (_p(outs["dxc"]), _p(outs["ddelta"]), _p(outs["dxdbl"]), _p(outs["dA"]), _p(outs["dDs"]), _p(outs["ddtb"]), Bt, H, W, D, N, R, Cp,
            _p(ws), wsb)
    if saved is None:
        if split:
            rc = L_.sigma_ss2d_scan_bwd_split(*head, _p(dy), _p(outs["delta"]), *tail, split, _stream())
        else:
            rc = L_.sigma_ss2d_scan_bwd(*head, _p(dy), _p(outs["delta"]), *tail, _stream())
        _lib.check(rc, "sigma_ss2d_scan_bwd")
        hs = ws[:Bt * T * D * N].view(1, Bt, T, D, N)
        names = ("delta", "hs", "dxc", "ddelta", "dA", "dDs", "ddtb")
    else:
        fwb = L_.sigma_ss2d_scan_workspace_bytes(kind, Bt, H, W, D, N)
        fws = torch.full((max(fwb, 4) // 4,), float("nan"), device="cuda")
        _lib.check(L_.sigma_ss2d_scan_fwd_save(*head, _p(outs["y"]), _p(outs["delta"]), _p(outs["hs"]), Bt, H, W, D, N, R, Cp, _p(fws), fwb,
                                               saved[0], _stream()), "sigma_ss2d_scan_fwd_save")
        _lib.check(L_.sigma_ss2d_scan_bwd_saved(*head, _p(dy), _p(outs["delta"]), _p(outs["hs"]), *tail, saved[1], _stream()),
                   "sigma_ss2d_scan_bwd_saved")
        hs = outs["hs"]
        names = ("y", "delta", "hs", "dxc", "ddelta", "dA", "dDs", "ddtb")
    torch.cuda.synchronize()
    for name in names:
        _check(tag, name, hs if name == "hs" else outs[name], ref[name], bnd[name], worst)
    dx = outs["dxdbl"]
    _check(tag, "dB", dx[..., :N], ref["dB"], bnd["dB"], worst)
    _check(tag, "dC", dx[..., N:2 * N], ref["dC"], bnd["dC"], worst)
    assert bool((dx[..., 2 * N:] == 0).all()), f"{tag}: the dt_r / padding columns of dxdbl must stay 0"
    for name, buf in bufs.items():
        guard_ok(buf, f"{tag} {name}")
    return outs["delta"].clone(), hs.clone()


# H, W, d_inner, dt_rank, images
CASES = [(120, 160, 192, 6, 2), (60, 80, 384, 12, 2), (30, 40, 768, 24, 2), (15, 20, 1536, 48, 2), (180, 240, 256, 8, 1),
         (23, 30, 2048, 64, 2), (30, 40, 768, 24, 1), (30, 40, 768, 24, 3), (15, 20, 1536, 48, 3), (60, 80, 384, 12, 1)]


@pytest.mark.parametrize("H,W,D,R,images", CASES)
def test_cross_bwd_matches_fp64(H, W, D, R, images):
    Bt = 2 * images
    tag = f"cross/{images}/{H}x{W}/D{D}/R{R}"
    args, Cp = ss2d_params(S, "cross", Bt, H, W, D, N, R, tag)
    ref, bnd = ss2d_cross_ref64(*args, H, W)
    worst = {}
    if (H, W) == (120, 160):
        assert _plan(Bt, H, W, D, 0)["nsplit"] > 1                      # stage 0 runs L-segments by default
    sweep = {}
    for sp in (1, 2, 7, 0, 64):
        sweep[sp] = _run(Bt, H, W, D, R, Cp, args, ref, bnd, f"{tag} split={sp}", worst, split=sp)
    for fs, bs in [(0, 0), (3, 7), (1, 2)]:
        delta, hs = _run(Bt, H, W, D, R, Cp, args, ref, bnd, f"{tag} saved fwd={fs} bwd={bs}", worst, saved=(fs, bs))
        # the training forward keeps what the state sweep would recompute: the same delta' and tile-start states, within the bound
        d0, h0 = sweep[1]
        for name, a, b in (("delta", delta, d0), ("hs", hs, h0)):
            frac = float(((a.double() - b.double()).abs() / (2 * bnd[name]).clamp_min(1e-300)).max())
            worst["fwd_vs_sweep/" + name] = max(worst.get("fwd_vs_sweep/" + name, 0.0), frac)
            assert frac <= 1.0, f"{tag} fwd={fs}: {name} of the training forward vs the state sweep: {frac:.3f} of twice the bound"
    record(f"ss2d cross bwd fp64 {tag}", **worst)


def test_cross_instances_exist_without_local_memory():
    from sigma_b200 import build
    out = subprocess.run(["cuobjdump", "-res-usage", build.LIB], capture_output=True, text=True, check=True).stdout
    use = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out))
    names = [f"_ZN5sigma{len(k)}{k}ILi{n}ELi{m}EEEvNS_13Ss2dBwdParamsE" for k in ("ss2d_bwd_cross_kernel", "ss2d_state_cross_kernel")
             for n in (4, 16) for m in (0, 1, 2)]
    for n in names:
        assert n in use, f"missing CROSS kernel {n}"
        assert re.search(r"\bSTACK:0\b", use[n]) and re.search(r"\bLOCAL:0\b", use[n]), f"{n}: {use[n]}"
    assert not [n for n in use if "cross" in n and "_det" in n]
