"""CPU: the fp64 reference of the CROSS (CroMB) scan backward (tests/ss2d_cross_ref64.py) that the fused backward's GPU tests compare
with, and the backward's launch plan for kind CROSS.
* every output and the tile-start states against torch.autograd in fp64 through a literal restatement of CroMB's two scans (each
  modality's half with its own weights and B, C from the other half; a loop over L), at ragged maps and at L > 2048; the same on a
  given (bf16-rounded) delta' through delta=, and without delta' the same bits as on the oracle's own forward;
* its error bound against an fp32 emulation whose decays are perturbed by the ex2.approx bound and whose forward runs in L-segments
  with carries formed as the summary pass forms them (an fp32 sum of delta'): the emulation must stay inside the bound;
* three plausible kernel mistakes (dC credited to the image's own row, the other weight set's rows for dA / dDs / d dt_bias, C read
  from the image's own half) land outside it;
* sigma_test_ss2d_bwd_plan, the state and workspace sizes for CROSS at every CroMB training shape and 1, 2, 3, 8 images, and the
  rejection of an odd batch."""
import ctypes

import numpy as np
import pytest
import torch

import procedural as P
from helpers import record
from oracle import ss2d_ref64 as R64
from ss2d_cross_ref64 import MISTAKES, ss2d_cross_ref64

S = 89


def _inputs(Bt, H, W, D, N, R, tag, wide=False):
    Lseq = H * W
    Cp = 2 * N + R + 3                                                       # 3 padding columns, as the packed x_proj leaves
    xc = P.randn(S, tag + "/xc", (Bt, Lseq, D))
    xdbl = P.randn(S, tag + "/xdbl", (Bt, Lseq, 1, Cp))
    xdbl[..., 2 * N + R:] = 0.0
    dtw = P.rand(S, tag + "/dtw", (2, D, R), -R ** -0.5, R ** -0.5)
    dt = torch.exp(P.rand(S, tag + "/dt", (2, D), np.log(1e-3), np.log(0.5 if wide else 0.1)))
    dtb = dt + torch.log(-torch.expm1(-dt))                                  # inverse softplus
    A = -torch.arange(1, N + 1, dtype=torch.float32).repeat(2 * D, 1) * P.rand(S, tag + "/A", (2 * D, N), 0.8, 4.0 if wide else 1.25)
    Ds = P.randn(S, tag + "/Ds", (2 * D,), 0.1, 1.0)
    dy = P.randn(S, tag + "/dy", (Bt, Lseq, D))
    return xc, xdbl, dtw, dtb, A, Ds, dy


def _literal(xc, xdbl, dtw, dtb, A, Ds, dy, H, W, delta=None):
    """CroMB's two scans restated (vmamba.py:1530,1536): fp64 autograd over a loop along L; the state entering every 16-position
    block too.  delta (1, Bt, L, D): run on this delta' instead of the softplus; ddelta is then the gradient at delta' times the
    softplus derivative 1 - exp(-delta') and d dt_bias its sum, as the backward kernel forms them"""
    t = [v.double().clone().requires_grad_(True) for v in (xc, xdbl, dtw, dtb, A, Ds)]
    xc_, xdbl_, dtw_, dtb_, A_, Ds_ = t
    Bt, L, D = xc.shape
    N, R = A.shape[1], dtw.shape[2]
    h2 = Bt // 2
    total, pres = 0.0, []
    hs = torch.full((1, Bt, -(-L // 16), D, N), float("nan"), dtype=torch.float64)
    for m in range(2):
        sl, osl = slice(m * h2, (m + 1) * h2), slice((1 - m) * h2, (2 - m) * h2)
        if delta is None:
            pre = xdbl_[sl, :, 0, 2 * N:2 * N + R] @ dtw_[m].t() + dtb_[m]
            pre.retain_grad()
            dl = torch.nn.functional.softplus(pre)
        else:
            dl = pre = delta[0, sl].double().clone().requires_grad_(True)
        Am, Dm = A_[m * D:(m + 1) * D], Ds_[m * D:(m + 1) * D]
        u, Bm, Cm = xc_[sl], xdbl_[sl, :, 0, :N], xdbl_[osl, :, 0, N:2 * N]
        h = torch.zeros(h2, D, N, dtype=torch.float64)
        ys = []
        for l in range(L):
            if l % 16 == 0:
                hs[0, sl, l // 16] = h.detach()
            h = torch.exp(dl[:, l, :, None] * Am) * h + (dl[:, l] * u[:, l])[..., None] * Bm[:, l, None, :]
            ys.append((h * Cm[:, l, None, :]).sum(-1) + Dm * u[:, l])
        total = total + (torch.stack(ys, 1) * dy.double()[sl]).sum()
        pres.append((sl, pre))
    total.backward()
    ddelta = torch.zeros(1, Bt, L, D, dtype=torch.float64)
    for sl, pre in pres:
        ddelta[0, sl] = pre.grad if delta is None else pre.grad * -torch.expm1(-pre.detach())
    g = xdbl_.grad
    ddtb = dtb_.grad if delta is None else torch.stack([ddelta[0, :h2].sum((0, 1)), ddelta[0, h2:].sum((0, 1))])
    return dict(dxc=xc_.grad, ddelta=ddelta, dB=g[..., :N], dC=g[..., N:2 * N], dA=A_.grad, dDs=Ds_.grad, ddtb=ddtb), hs


@pytest.mark.parametrize("H,W,N,Bt", [(5, 7, 4, 2), (9, 11, 4, 4), (9, 11, 16, 2), (1, 9, 16, 4), (42, 50, 4, 2)])
def test_backward_and_states_match_autograd(H, W, N, Bt):
    D, R = 8 if H * W < 2048 else 4, 3
    args = _inputs(Bt, H, W, D, N, R, f"b/{H}/{W}/{N}/{Bt}")
    ref, bnd = ss2d_cross_ref64(*args, H, W)
    want, hs = _literal(*args, H, W)
    for name, w in want.items():
        err = float((ref[name] - w).abs().max()) / float(w.abs().max())
        assert err < 1e-12, f"{name}: {err:.2e}"
    assert float((ref["hs"] - hs).abs().max()) <= 1e-12 * float(hs.abs().max())
    y, by = R64.ss2d_fwd_ref64("cross", *args[:6], H, W)                   # the forward is the oracle's, bit for bit
    assert torch.equal(y, ref["y"]) and torch.equal(by, bnd["y"])


@pytest.mark.parametrize("H,W,N,Bt", [(5, 7, 4, 2), (9, 11, 16, 4)])
def test_given_delta_matches_the_literal_loop(H, W, N, Bt):
    """delta=: every output against the literal loop run on the same delta' (a softplus value rounded to bf16, as the bf16 training
    mode saves it); ref["delta"] is the given one with bound 0; and with delta' = the fp64 softplus, the delta= path agrees with
    the reference that forms delta' itself"""
    D, R = 8, 3
    args = _inputs(Bt, H, W, D, N, R, f"d/{H}/{W}/{N}/{Bt}")
    full, _ = ss2d_cross_ref64(*args, H, W)
    given = full["delta"].to(torch.bfloat16).double()
    ref, bnd = ss2d_cross_ref64(*args, H, W, delta=given)
    want, hs = _literal(*args, H, W, delta=given)
    for name, w in want.items():
        err = float((ref[name] - w).abs().max()) / float(w.abs().max())
        assert err < 1e-12, f"{name}: {err:.2e}"
    assert float((ref["hs"] - hs).abs().max()) <= 1e-12 * float(hs.abs().max())
    assert torch.equal(ref["delta"], given) and not bool(bnd["delta"].any())
    same, _ = ss2d_cross_ref64(*args, H, W, delta=full["delta"])
    for name in ("y", "dxc", "ddelta", "dB", "dC", "dA", "dDs", "ddtb"):
        err = float((same[name] - full[name]).abs().max()) / float(full[name].abs().max())
        assert err < 1e-12, f"{name}: {err:.2e}"


def test_without_delta_the_oracle_forward_bit_for_bit(monkeypatch):
    """without delta the reference is what it was when it ran on oracle/ss2d_ref64.ss2d_fwd_ref64: every output and bound the same
    bits"""
    import ss2d_cross_ref64 as C
    H, W, N, Bt, D, R = 9, 11, 4, 4, 16, 6
    args = _inputs(Bt, H, W, D, N, R, "bits")
    ref, bnd = ss2d_cross_ref64(*args, H, W)
    monkeypatch.setattr(C.RD, "ss2d_fwd_ref64", lambda *a, delta=None, **kw: R64.ss2d_fwd_ref64(*a, **kw))
    ref0, bnd0 = ss2d_cross_ref64(*args, H, W)
    for name in ref:
        assert torch.equal(ref[name].nan_to_num(7.0), ref0[name].nan_to_num(7.0)), name
        assert torch.equal(bnd[name].nan_to_num(7.0), bnd0[name].nan_to_num(7.0)), name


def _emulate32(xc, xdbl, dtw, dtb, A, Ds, dy, H, W, seed, nseg):
    """fp32 emulation of the CROSS kernels: each decay perturbed by a seeded ±E2 relative error; the forward cut into nseg
    L-segments whose carried decay is ex2(a2 · the fp32 sum of the segment's delta') (also perturbed), as the summary pass forms it"""
    f = lambda t: t.numpy().astype(np.float32)
    xc, xdbl, dtw, dtb, A, Ds, dy = map(f, (xc, xdbl, dtw, dtb, A, Ds, dy))
    rng = np.random.default_rng(seed)
    f32 = np.float32
    Bt, L, D = xc.shape
    N, R = A.shape[1], dtw.shape[2]
    h2 = Bt // 2
    out = dict(y=np.zeros((1, Bt, L, D), f32), delta=np.zeros((1, Bt, L, D), f32), dxc=np.zeros((Bt, L, D), f32),
               ddelta=np.zeros((1, Bt, L, D), f32), dB=np.zeros((Bt, L, 1, N), f32), dC=np.zeros((Bt, L, 1, N), f32),
               dA=np.zeros((2 * D, N), f32), dDs=np.zeros(2 * D, f32), ddtb=np.zeros((2, D), f32),
               hs=np.zeros((1, Bt, -(-L // 16), D, N), f32))
    tiles = -(-L // 16)
    tps = -(-tiles // nseg)
    bounds = [(s * tps * 16, min(L, (s + 1) * tps * 16)) for s in range(nseg) if s * tps * 16 < L]
    pert = lambda shape: (1 + f32(R64.E2) * rng.choice([-1, 1], shape)).astype(f32)
    for m in range(2):
        sl, osl = slice(m * h2, (m + 1) * h2), slice((1 - m) * h2, (2 - m) * h2)
        Am, Dm = A[m * D:(m + 1) * D], Ds[m * D:(m + 1) * D]
        a2 = (Am * f32(1.4426950408889634)).astype(f32)
        pre = (xdbl[sl, :, 0, 2 * N:2 * N + R] @ dtw[m].T + dtb[m]).astype(f32)
        dl = np.logaddexp(f32(0), pre).astype(f32)
        u, Bm, Cm, dyk = xc[sl], xdbl[sl, :, 0, :N], xdbl[osl, :, 0, N:2 * N], dy[sl]
        dec = np.exp2(dl[..., None] * a2).astype(f32) * pert((h2, L, D, N))
        # summary pass: each segment from a zero state, its end state and carried decay; combine; then every step from the starts
        starts, cur = [], np.zeros((h2, D, N), f32)
        for lo, hi in bounds:
            starts.append(cur)
            h = np.zeros((h2, D, N), f32)
            for l in range(lo, hi):
                h = dec[:, l] * h + (dl[:, l] * u[:, l])[..., None] * Bm[:, l, None, :]
            S_ = dl[:, lo:hi].sum(1, dtype=f32)
            carry = np.exp2(S_[..., None] * a2).astype(f32) * pert((h2, D, N))
            cur = (carry * cur + h).astype(f32)
        hsave = np.zeros((h2, L, D, N), f32)
        for (lo, hi), h in zip(bounds, starts):
            for l in range(lo, hi):
                if l % 16 == 0:
                    out["hs"][0, sl, l // 16] = h
                h = dec[:, l] * h + (dl[:, l] * u[:, l])[..., None] * Bm[:, l, None, :]
                hsave[:, l] = h
                out["y"][0, sl, l] = (h * Cm[:, l, None, :]).sum(-1, dtype=f32) + Dm * u[:, l]
        out["delta"][0, sl] = dl
        dh = np.zeros((h2, D, N), f32)
        for l in range(L - 1, -1, -1):
            dhn = dyk[:, l, :, None] * Cm[:, l, None, :] + dh
            hp = hsave[:, l - 1] if l > 0 else np.zeros_like(dh)
            ah = dec[:, l] * hp
            s1 = (dhn * Bm[:, l, None, :]).sum(-1, dtype=f32)
            s2 = (dhn * ah * Am).sum(-1, dtype=f32)
            out["dC"][osl, l, 0] = (dyk[:, l, :, None] * hsave[:, l]).sum(1, dtype=f32)
            out["dB"][sl, l, 0] = (dhn * (dl[:, l] * u[:, l])[..., None]).sum(1, dtype=f32)
            out["dxc"][sl, l] += dyk[:, l] * Dm + dl[:, l] * s1
            dd = (1 - np.exp(-dl[:, l])).astype(f32) * (u[:, l] * s1 + s2)
            out["ddelta"][0, sl, l] = dd
            out["dA"][m * D:(m + 1) * D] += (dhn * ah * dl[:, l, :, None]).sum(0, dtype=f32)
            out["dDs"][m * D:(m + 1) * D] += (dyk[:, l] * u[:, l]).sum(0, dtype=f32)
            out["ddtb"][m] += dd.sum(0, dtype=f32)
            dh = (dhn * dec[:, l]).astype(f32)
    return out


@pytest.mark.parametrize("H,W,N,Bt,wide,nseg", [(9, 11, 4, 4, False, 1), (9, 11, 4, 2, True, 3), (17, 20, 16, 2, False, 7),
                                                (5, 7, 4, 6, False, 2)])
def test_bound_covers_an_fp32_emulation(H, W, N, Bt, wide, nseg):
    D, R = 16, 6
    tag = f"e/{H}/{W}/{N}/{Bt}/{wide}/{nseg}"
    args = _inputs(Bt, H, W, D, N, R, tag, wide)
    ref, bnd = ss2d_cross_ref64(*args, H, W)
    emu = _emulate32(*args, H, W, seed=len(tag), nseg=nseg)
    worst = {}
    for name, v in emu.items():
        v = torch.from_numpy(v).double()
        frac = R64.bound_fraction(v, ref[name], bnd[name])
        worst[name] = frac
        assert frac <= 1.0, f"{name}: {frac:.3f} of the bound"
        # per element, yet no looser than 1e-3 of scale at the largest element; d dt_bias sums ddelta's bounds over all positions, so
        # there (as in the GPU tests) the max-norm bar is checked instead
        i = int(ref[name].abs().argmax())
        if name == "ddtb":
            assert float((v - ref[name]).abs().max()) <= 1e-3 * float(ref[name].abs().max()), name
        else:
            assert float(bnd[name].reshape(-1)[i]) <= 1e-3 * float(ref[name].abs().max()), name
    record(f"ss2d_cross_ref64 bound self-check {tag}", **worst)


@pytest.mark.parametrize("mistake", MISTAKES)
def test_plausible_mistakes_land_outside_the_bound(mistake):
    H, W, N, Bt, D, R = 9, 11, 4, 4, 16, 6
    args = _inputs(Bt, H, W, D, N, R, "m")
    ref, bnd = ss2d_cross_ref64(*args, H, W)
    bad, _ = ss2d_cross_ref64(*args, H, W, mistake=mistake)
    fracs = {k: R64.bound_fraction(bad[k], ref[k], bnd[k]) for k in ("dxc", "ddelta", "dB", "dC", "dA", "dDs", "ddtb")}
    assert max(fracs.values()) > 100.0, fracs
    want = {"dC_own": "dC", "wset": "dA", "C_own": "dxc"}[mistake]
    assert fracs[want] > 100.0, fracs


# CroMB's training shapes (one block per encoder stage; d_inner = 2·C): Sigma-tiny / small at 480 x 640 and Sigma-base at 720 x 960
CROMB = [(120, 160, 192, 6), (60, 80, 384, 12), (30, 40, 768, 24), (15, 20, 1536, 48), (180, 240, 256, 8), (23, 30, 2048, 64)]


def _lib():
    from sigma_b200 import _lib
    return _lib


@pytest.mark.parametrize("H,W,D,R", CROMB)
@pytest.mark.parametrize("images", [1, 2, 3, 8])
def test_cross_backward_plan_and_sizes(H, W, D, R, images):
    L_, lib = _lib().lib(), _lib()
    Bt, N, L = 2 * images, 4, H * W
    tiles = -(-L // 16)
    for force in (0, 1, 2, 7, 64, 100):
        out = (ctypes.c_int64 * 4)()
        lib.check(L_.sigma_test_ss2d_bwd_plan(lib.DIRS_CROSS, Bt, H, W, D, N, force, out), "sigma_test_ss2d_bwd_plan")
        nsplit, tps, mx, mn = (int(v) for v in out)
        assert mx == mn == tiles                                          # one row-major walk of ceil(L / 16) tiles
        assert 1 <= nsplit <= 64 and nsplit * tps >= tiles and (nsplit - 1) * tps < tiles, (force, nsplit, tps)
        if force:
            assert nsplit == len(range(0, tiles, -(-tiles // min(force, 64, tiles))))
    hsb = L_.sigma_ss2d_scan_hs_bytes(lib.DIRS_CROSS, Bt, H, W, D, N)
    assert hsb == Bt * tiles * D * N * 4
    assert L_.sigma_ss2d_scan_bwd_workspace_bytes(lib.DIRS_CROSS, Bt, H, W, D, N) >= hsb
    assert L_.sigma_ss2d_scan_bwd_det_workspace_bytes(lib.DIRS_CROSS, Bt, H, W, D, N) == 0     # no deterministic build


def test_cross_backward_rejects_an_odd_batch():
    L_, lib = _lib().lib(), _lib()
    out = (ctypes.c_int64 * 4)()
    assert L_.sigma_test_ss2d_bwd_plan(lib.DIRS_CROSS, 3, 30, 40, 768, 4, 0, out) != 0
    assert L_.sigma_test_ss2d_bwd_plan(lib.DIRS_CROSS, 4, 30, 40, 768, 4, 0, out) == 0
    assert L_.sigma_ss2d_scan_hs_bytes(lib.DIRS_CROSS, 3, 30, 40, 768, 4) == 0
    assert L_.sigma_ss2d_scan_bwd_workspace_bytes(lib.DIRS_CROSS, 3, 30, 40, 768, 4) == 0
