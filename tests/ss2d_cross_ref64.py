"""fp64 reference of the fused scan backward for kind "cross" (CroMB, sigma_ss2d_scan_bwd{,_saved} with SIGMA_DIRS_CROSS), with a
per-element error bound for each output of the fp32 kernels.  Test infrastructure only.

It extends oracle/ss2d_ref64.py, whose ss2d_ref64 covers "cross4" and "seq2": the forward, its tiling and every error term are that
module's (ss2d_fwd_ref64 with its on_walk hook), and the backward below is ss2d_ref64's, run once per modality half.  The batch is
Bt = 2·images; image b uses weight set w = [b >= Bt/2] and its own B and dt_r, and reads C from image b' = (b + Bt/2) mod Bt.  So,
relative to one walk of ss2d_ref64:
  * dC of image b is credited to the C columns of dxdbl[b'] (the image whose x_dbl row supplied C);
  * dA, dDs and d dt_bias are sums over the images of one modality, into rows w·D + d of (2D, N), (2D) and (2, D).
`mistake` computes the result of a plausible kernel bug instead (for tests that the bound tells it apart): "dC_own" credits dC to
the image's own row, "wset" sends dA / dDs / d dt_bias to the other weight set's rows, "C_own" reads C from the image's own half.
`delta` runs the forward and the backward on a given delta' (the bf16 training mode's saved one), through
tests/ss2d_delta_ref64.ss2d_fwd_ref64 as ss2d_delta_ref64.ss2d_ref64 does for cross4 / seq2; without it the forward is the
oracle's, bit for bit.
"""
import math

import torch

import ss2d_delta_ref64 as RD
from oracle import ss2d_ref64 as R

MISTAKES = ("dC_own", "wset", "C_own")


def ss2d_cross_ref64(xc, xdbl, dtw, dtb, A, Ds, dy, H, W, device=None, mistake=None, delta=None):
    """The inputs of ss2d_fwd_ref64 for kind "cross" (xc (Bt, L, D), xdbl (Bt, L, 1, Cp), dtw (2, D, R), dtb (2, D), A (2D, N), Ds
    (2D)) and dy (Bt, L, D).  Returns (ref, bound) as ss2d_ref64 does: y / delta / ddelta (1, Bt, L, D), hs (1, Bt, ceil(L/16), D,
    N), dxc (Bt, L, D), dB / dC (Bt, L, 1, N), dA (2D, N), dDs (2D), ddtb (2, D).
    delta (1, Bt, L, D): the delta' to run with instead of the softplus (taken as exact; ref["delta"] is then it, bound 0)."""
    assert mistake in (None,) + MISTAKES, mistake
    dev = torch.device(device) if device is not None else xc.device
    Bt, Lseq, D = xc.shape
    N = A.shape[1]
    assert Bt % 2 == 0 and xdbl.shape[2] == 1, "cross: the batch holds 2·images, one x_dbl row per position"
    hb = Bt // 2
    if mistake == "C_own":   # swap the halves' C columns: the forward below then reads each image's own C
        xdbl = xdbl.clone()
        xdbl[:, :, :, N:2 * N] = torch.cat([xdbl[hb:, :, :, N:2 * N], xdbl[:hb, :, :, N:2 * N]])
    T = R.walk_tiles("cross", H, W)[0].shape[0]
    LT, U = R.LT, R.U
    z = lambda *s: torch.zeros(s, dtype=torch.float64, device=dev)
    ref = dict(delta=z(1, Bt, Lseq + 1, D), hs=torch.full((1, Bt, T, D, N), math.nan, dtype=torch.float64, device=dev),
               dxc=z(Bt, Lseq + 1, D), ddelta=z(1, Bt, Lseq + 1, D), dB=z(Bt, Lseq + 1, 1, N), dC=z(Bt, Lseq + 1, 1, N), dA=z(2 * D, N),
               dDs=z(2 * D), ddtb=z(2, D))
    bnd = {k: torch.zeros_like(v) for k, v in ref.items()}
    bnd["hs"].fill_(math.nan)
    dxc_mag = z(Bt, Lseq + 1, D)
    dyp = R._pad(dy.detach().to(dev, torch.float64))
    groups = iter(R.walk_groups("cross", Bt))

    def backward(g):
        _, bs, kw, cs = next(groups)
        ws = 1 - kw if mistake == "wset" else kw          # rows the weight-set sums go to
        cdst = bs if mistake == "dC_own" else cs           # images whose dxdbl C columns receive dC
        nb, m, p, pf, u, Bm, Cm, dl, edl, sig = g.nb, g.m, g.p, g.pf, g.u, g.Bm, g.Cm, g.dl, g.edl, g.sig
        Ak, Dk, absA, slot, P, h0, h_all, e_all = g.Ak, g.Dk, g.absA, g.slot, g.P, g.h0, g.h_all, g.e_all
        b = u.shape[0]
        sh = (b, nb, D, N)
        put = lambda dst, src: dst.index_copy_(1, pf, src.reshape(b, nb * LT, *src.shape[3:]))
        ref["hs"][0, bs, :nb], bnd["hs"][0, bs, :nb] = h0, g.e0
        put(ref["delta"][0, bs], dl); put(bnd["delta"][0, bs], edl)
        dyk = dyp[bs][:, p]

        def wslot(s):
            return dyk[:, :, s, :, None] * Cm[:, :, s, None, :]

        # ---- as ss2d_ref64's backward: the gradient entering each tile from the right (levels 1 + 2), then every step ----
        ql = z(*sh)
        for s in range(LT - 1, -1, -1):
            a, _, _, _ = slot(s)
            ql = a * (wslot(s) + ql)
        q0 = R._chain(P, ql, rev=True)
        q, eql = q0, z(*sh)
        for s in range(LT - 1, -1, -1):
            a, rho, _, _ = slot(s)
            gg = wslot(s) + q
            eg = eql + U * gg.abs()
            eql, q = a * eg + a * rho * gg.abs() + U * (a * gg).abs(), a * gg
        eq0 = R._chain(P, eql, rev=True)
        del ql, eql
        q, eq = q0, eq0
        dd_k, edd_k = torch.empty_like(u), torch.empty_like(u)
        du_k, edu_k, dum_k = torch.empty_like(u), torch.empty_like(u), torch.empty_like(u)
        dB_k, dC_k, edB_k, edC_k = z(b, nb, LT, N), z(b, nb, LT, N), z(b, nb, LT, N), z(b, nb, LT, N)
        dA_k, edA_k, dA_tot, dA_abs = z(D, N), z(*sh), z(*sh), z(*sh)
        gD = R._gt(D)
        for s in range(LT - 1, -1, -1):
            a, rho, v, _ = slot(s)
            gg = wslot(s) + q
            G = gg.abs()
            eg = eq + U * G
            h, eh = h_all[:, :, s], e_all[:, :, s].double()
            hp = h_all[:, :, s - 1] if s > 0 else h0
            Mh, Mp = h.abs(), hp.abs()
            dys, us, ds, es = dyk[:, :, s, :, None], u[:, :, s, :, None], dl[:, :, s, :, None], edl[:, :, s, :, None]
            Bs = Bm[:, :, s, None, :]
            dC_k[:, :, s] = (dys * h).sum(2)
            edC_k[:, :, s] = R.chan(dys.abs() * (eh + U * Mh)) + gD * (dys.abs() * Mh).sum(2)
            dlus = (ds * us).abs()
            dB_k[:, :, s] = (gg * ds * us).sum(2)
            edB_k[:, :, s] = R.chan(dlus * eg + us.abs() * G * es + 2 * U * G * dlus) + gD * (G * dlus).sum(2)
            s1, S1m = (gg * Bs).sum(-1), (G * Bs.abs()).sum(-1)
            es1 = (Bs.abs() * eg).sum(-1) + (N + 1) * U * S1m
            dyD = (dyk[:, :, s] * Dk).abs()
            du_k[:, :, s] = dyk[:, :, s] * Dk + dl[:, :, s] * s1
            dum_k[:, :, s] = dyD + dl[:, :, s] * S1m
            edu_k[:, :, s] = dl[:, :, s] * es1 + edl[:, :, s] * S1m + 2 * U * dum_k[:, :, s]
            ah, ahm = a * hp, a * Mp
            eah = eh + es * (us * Bs).abs() + 2 * U * v.abs() + U * ahm
            t, tm = gg * ah, G * ahm
            et = G * eah + eg * ahm + U * tm
            s2, S2m = (t * Ak).sum(-1), (tm * absA).sum(-1)
            es2 = (et * absA).sum(-1) + (N + 3) * U * S2m
            X = u[:, :, s] * s1 + s2
            Xm = u[:, :, s].abs() * S1m + S2m
            eX = u[:, :, s].abs() * es1 + es2 + 2 * U * Xm
            sg = sig[:, :, s]
            esg = torch.exp(-dl[:, :, s]) * (R.E2 + 2 * U * dl[:, :, s] + edl[:, :, s]) + U
            dd_k[:, :, s] = sg * X
            edd_k[:, :, s] = (sg * eX + Xm * esg + U * sg * Xm) * m[:, :, s]
            dA_k += (t * ds).sum((0, 1))
            dA_tot += t * ds
            dA_abs += (t * ds).abs()
            edA_k += ds * et + tm * es + U * ds * tm
            q, eq = a * gg, a * eg + a * rho * G + U * a * G
        put(ref["ddelta"][0, bs], dd_k * m); put(bnd["ddelta"][0, bs], edd_k)
        put(ref["dB"][bs, :, 0], dB_k); put(bnd["dB"][bs, :, 0], edB_k)
        put(ref["dC"][cdst, :, 0], dC_k); put(bnd["dC"][cdst, :, 0], edC_k)
        mm = m.expand_as(u).reshape(b, nb * LT, D)
        ref["dxc"][bs].index_add_(1, pf, du_k.reshape(b, nb * LT, D) * mm)
        bnd["dxc"][bs].index_add_(1, pf, edu_k.reshape(b, nb * LT, D) * mm)
        dxc_mag[bs].index_add_(1, pf, dum_k.reshape(b, nb * LT, D) * mm)
        rows = slice(ws * D, (ws + 1) * D)
        ref["dA"][rows] = dA_k
        bnd["dA"][rows] = R.tile_rss(edA_k) + R._acc(dA_tot, dA_abs, Lseq)
        dyu = dyk * u
        ref["dDs"][rows] = dyu.sum((0, 1, 2))
        bnd["dDs"][rows] = U * dyu.abs().sum((0, 1, 2)) + R._acc(dyu.sum(2), dyu.abs().sum(2), Lseq)
        dd_k *= m
        ref["ddtb"][ws] = dd_k.sum((0, 1, 2))
        bnd["ddtb"][ws] = R.tile_rss(edd_k.sum(2)) + R._acc(dd_k.sum(2), (dd_k.abs() + edd_k).sum(2), Lseq)

    y, ey = RD.ss2d_fwd_ref64("cross", xc, xdbl, dtw, dtb, A, Ds, H, W, device=dev, on_walk=backward, delta=delta)
    bnd["dxc"] += U * dxc_mag
    for key in ("delta", "dxc", "ddelta", "dB", "dC"):
        sl = (slice(None), slice(0, Lseq)) if key in ("dxc", "dB", "dC") else (slice(None), slice(None), slice(0, Lseq))
        ref[key], bnd[key] = ref[key][sl].contiguous(), bnd[key][sl].contiguous()
    for key in bnd:
        bnd[key] = bnd[key] * R.SAFETY
    ref["y"], bnd["y"] = y, ey
    return ref, bnd
