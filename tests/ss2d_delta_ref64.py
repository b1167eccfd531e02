"""fp64 reference of the fused SS2D scan core run on a GIVEN delta' (the bf16 training mode: sigma_ss2d_scan_fwd_save_bf16 /
sigma_ss2d_scan_bwd_saved_bf16), with per-element error bounds.  Test infrastructure only; a sibling of oracle/ss2d_ref64.py (whose
tiling, helpers and error model it imports and whose documentation it relies on) in the way tests/ss2d_cross_ref64.py is.

The kernels of the mode round delta' = softplus(dt_proj) to bf16 before the recurrence uses it and save that value.  The reference
here runs the recurrence and the backward on an fp64 copy of the saved values, so err(delta') = 0 in every term of the error model,
and the softplus derivative is 1 - exp(-delta') of the given value, as the backward kernel forms it.  delta' itself is checked apart,
against the softplus and inside its fp32 bound + BF16_RN·|delta'| (delta_bound_bf16).  With delta=None both functions compute what
oracle/ss2d_ref64.py computes (tests/test_bf16_training_cpu.py holds them to it)."""
import math
import types

import torch

from oracle.ss2d_ref64 import (BF16_RN, E2, KINDS, LT, SAFETY, SP, U, _acc, _chain, _gt, _pad, chan, tile_rss, walk_groups,
                               walk_tiles)


def delta_bound_bf16(ref_delta, bnd_delta):
    """per-element bound of a delta' the kernel rounded to bf16, from the fp64 softplus and its fp32 bound (SAFETY applied)"""
    return bnd_delta + BF16_RN * (ref_delta.abs() + bnd_delta)


def ss2d_fwd_ref64(kind, xc, xdbl, dtw, dtb, A, Ds, H, W, device=None, on_walk=None, delta=None):
    """The forward alone.  kind "cross4" / "seq2" / "cross"; xc (B, Lseq, D) fp32 or bf16, xdbl (B, Lseq, K, Cp) = [B | C | dt_r |
    padding], dtw (Kw, D, R), dtb (Kw, D), A (Kw·D, N), Ds (Kw·D), Kw = K or 2 (modalities) for "cross".  Returns (y, bound), float64
    (K, B, Lseq, D): direction k's output at the position it belongs to, and its per-element bound (SAFETY applied; with bf16 xc it
    includes the final rounding to bf16).
    on_walk(g): called after each walk with its tensors (tiles, inputs, delta', the states at every step and their bounds); the
    states are only kept when it is given.  ss2d_ref64 runs its backward from there.
    delta (K, B, Lseq, D): the delta' to run the recurrence with instead of the softplus (taken as exact)."""
    bf16 = xc.dtype == torch.bfloat16
    dev = torch.device(device) if device is not None else xc.device
    f = lambda t: t.detach().to(dev, torch.float64)
    xc, xdbl, dtw, dtb, A, Ds = map(f, (xc, xdbl, dtw, dtb, A, Ds))
    Bt, Lseq, D = xc.shape
    K, N, R = xdbl.shape[2], A.shape[1], dtw.shape[2]
    assert K == KINDS[kind]
    tiles = walk_tiles(kind, H, W)
    z = lambda *s: torch.zeros(s, dtype=torch.float64, device=dev)
    y, ey = z(K, Bt, Lseq + 1, D), z(K, Bt, Lseq + 1, D)
    xcp, xdp = _pad(xc), _pad(xdbl)
    dgiven = _pad(f(delta).flatten(0, 1)).view(K, Bt, Lseq + 1, D) if delta is not None else None
    for k, bs, kw, cs in walk_groups(kind, Bt):
        blk = torch.from_numpy(tiles[k]).to(dev)
        nb = blk.shape[0]
        m = (blk >= 0).double()[None, :, :, None]                               # (1, nb, 16, 1)
        p = torch.where(blk >= 0, blk, torch.full_like(blk, Lseq))
        u = xcp[bs][:, p]                                                       # (b, nb, 16, D)
        xk = xdp[bs][:, p, k]
        Bm, dtr = xk[..., :N], xk[..., 2 * N:2 * N + R]
        Cm = xdp[cs][:, p, k, N:2 * N]
        pre = dtr @ dtw[kw].t() + dtb[kw]
        Tm = dtr.abs() @ dtw[kw].abs().t() + dtb[kw].abs()
        dl = torch.nn.functional.softplus(pre) * m
        sig = torch.sigmoid(pre)
        edl = (sig * (R + 2) * U * Tm + SP * dl) * m
        if dgiven is not None:
            dl = dgiven[k, bs][:, p] * m
            edl = torch.zeros_like(dl)
            sig = -torch.expm1(-dl)
        del Tm, dtr, xk
        Ak, Dk = A[kw * D:(kw + 1) * D], Ds[kw * D:(kw + 1) * D]
        dlu = dl * u
        absA = Ak.abs()
        b = u.shape[0]

        def slot(s):
            d_, e_ = dl[:, :, s, :, None], edl[:, :, s, :, None]
            a = torch.exp(d_ * Ak)
            rho = E2 + 2 * U * (d_ * absA) + absA * e_
            v = dlu[:, :, s, :, None] * Bm[:, :, s, None, :]
            ein = u[:, :, s, :, None].abs() * Bm[:, :, s, None, :].abs() * e_ + 3 * U * v.abs()
            return a, rho, v, ein

        # ---- h (levels 1 + 2), its error e (levels 1 + 2), then both at every step (level 3) ----
        sh = (b, nb, D, N)
        hl, P = z(*sh), torch.ones(sh, dtype=torch.float64, device=dev)
        for s in range(LT):
            a, _, v, _ = slot(s)
            hl, P = a * hl + v, P * a
        h0 = _chain(P, hl)
        h, el = h0, z(*sh)
        for s in range(LT):
            a, rho, v, ein = slot(s)
            hn = a * h + v
            el = a * el + a * rho * h.abs() + ein + U * hn.abs()
            h = hn
        e0 = _chain(P, el)
        del hl, el
        keep = on_walk is not None
        if keep:
            h_all = torch.empty((b, nb, LT, D, N), dtype=torch.float64, device=dev)
            e_all = torch.empty(h_all.shape, dtype=torch.float32, device=dev)  # a bound: 24 bits are plenty
        h, e = h0, e0
        yk, eyk = torch.empty_like(u), torch.empty_like(u)
        for s in range(LT):
            a, rho, v, ein = slot(s)
            hn = a * h + v
            e = a * e + a * rho * h.abs() + ein + U * hn.abs()
            h = hn
            if keep:
                h_all[:, :, s], e_all[:, :, s] = h, e
            C = Cm[:, :, s, None, :]
            du_ = Dk * u[:, :, s]
            yk[:, :, s] = (C * h).sum(-1) + du_
            eyk[:, :, s] = (C.abs() * e).sum(-1) + (N + 2) * U * ((C * h).abs().sum(-1) + du_.abs())
        pf = p.reshape(-1)
        y[k, bs].index_copy_(1, pf, yk.reshape(b, nb * LT, D))
        ey[k, bs].index_copy_(1, pf, eyk.reshape(b, nb * LT, D))
        del yk, eyk
        if keep:
            on_walk(types.SimpleNamespace(k=k, nb=nb, m=m, p=p, pf=pf, u=u, Bm=Bm, Cm=Cm, dl=dl, edl=edl, sig=sig, Ak=Ak, Dk=Dk,
                                          absA=absA, slot=slot, P=P, h0=h0, e0=e0, h_all=h_all, e_all=e_all))
            del h_all, e_all
    y, ey = y[:, :, :Lseq].contiguous(), ey[:, :, :Lseq] * SAFETY
    if bf16:
        ey = ey + BF16_RN * (y.abs() + ey)
    return y, ey.contiguous()


def ss2d_ref64(kind, xc, xdbl, dtw, dtb, A, Ds, dy, H, W, device=None, delta=None):
    """kind "cross4" / "seq2"; the inputs of ss2d_fwd_ref64 (fp32) and dy (B, Lseq, D).  Returns (ref, bound): two dicts of float64
    tensors with keys y, delta, hs, dxc, ddelta, dB, dC, dA, dDs, ddtb.  y / delta / ddelta (K, B, Lseq, D), hs (K, B, max_tiles, D,
    N), dB / dC (B, Lseq, K, N).  y and its bound are ss2d_fwd_ref64's, bit for bit.
    delta: as in ss2d_fwd_ref64; the forward and the backward both run on it (ref["delta"] is then the given one, bound 0)."""
    assert kind in ("cross4", "seq2"), "the fused backward covers CROSS4 and SEQ2"
    dev = torch.device(device) if device is not None else xc.device
    Bt, Lseq, D = xc.shape
    K, N = xdbl.shape[2], A.shape[1]
    T = max(t.shape[0] for t in walk_tiles(kind, H, W))
    z = lambda *s: torch.zeros(s, dtype=torch.float64, device=dev)
    ref = dict(delta=z(K, Bt, Lseq + 1, D), hs=torch.full((K, Bt, T, D, N), math.nan, dtype=torch.float64, device=dev),
               dxc=z(Bt, Lseq + 1, D), ddelta=z(K, Bt, Lseq + 1, D), dB=z(Bt, Lseq + 1, K, N), dC=z(Bt, Lseq + 1, K, N), dA=z(K * D, N),
               dDs=z(K * D), ddtb=z(K, D))
    bnd = {k: torch.zeros_like(v) for k, v in ref.items()}
    bnd["hs"].fill_(math.nan)
    dxc_mag = z(Bt, Lseq + 1, D)
    dyp = _pad(dy.detach().to(dev, torch.float64))

    def backward(g):
        k, nb, m, p, pf, u, Bm, Cm, dl, edl, sig = g.k, g.nb, g.m, g.p, g.pf, g.u, g.Bm, g.Cm, g.dl, g.edl, g.sig
        Ak, Dk, absA, slot, P, h0, h_all, e_all = g.Ak, g.Dk, g.absA, g.slot, g.P, g.h0, g.h_all, g.e_all
        sh = (Bt, nb, D, N)
        put = lambda dst, src: dst.index_copy_(1, pf, src.reshape(Bt, nb * LT, *src.shape[3:]))
        ref["hs"][k, :, :nb], bnd["hs"][k, :, :nb] = h0, g.e0
        put(ref["delta"][k], dl); put(bnd["delta"][k], edl)
        dyk = dyp[:, p]

        # ---- backward: q = a·g entering each step from the right, and its error, tile by tile from the right ----
        def wslot(s):
            return dyk[:, :, s, :, None] * Cm[:, :, s, None, :]

        ql = z(*sh)
        for s in range(LT - 1, -1, -1):
            a, _, _, _ = slot(s)
            ql = a * (wslot(s) + ql)
        q0 = _chain(P, ql, rev=True)
        q, eql = q0, z(*sh)
        for s in range(LT - 1, -1, -1):
            a, rho, _, _ = slot(s)
            g = wslot(s) + q
            eg = eql + U * g.abs()
            eql, q = a * eg + a * rho * g.abs() + U * (a * g).abs(), a * g
        eq0 = _chain(P, eql, rev=True)
        del ql, eql
        q, eq = q0, eq0
        dd_k, edd_k = torch.empty_like(u), torch.empty_like(u)
        du_k, edu_k, dum_k = torch.empty_like(u), torch.empty_like(u), torch.empty_like(u)
        dB_k, dC_k = z(Bt, nb, LT, N), z(Bt, nb, LT, N)
        edB_k, edC_k = z(Bt, nb, LT, N), z(Bt, nb, LT, N)
        dA_k, edA_k = z(D, N), z(*sh)
        dA_tot, dA_abs = z(*sh), z(*sh)
        gD = _gt(D)
        for s in range(LT - 1, -1, -1):
            a, rho, v, _ = slot(s)
            w = wslot(s)
            g = w + q
            G = g.abs()
            eg = eq + U * G
            h, eh = h_all[:, :, s], e_all[:, :, s].double()
            hp = h_all[:, :, s - 1] if s > 0 else h0
            Mh, Mp = h.abs(), hp.abs()
            dys, us, ds, es = dyk[:, :, s, :, None], u[:, :, s, :, None], dl[:, :, s, :, None], edl[:, :, s, :, None]
            Bs, Cs = Bm[:, :, s, None, :], Cm[:, :, s, None, :]
            # dC = sum_d dy h,  dB = sum_d g delta' u
            dC_k[:, :, s] = (dys * h).sum(2)
            edC_k[:, :, s] = chan(dys.abs() * (eh + U * Mh)) + gD * (dys.abs() * Mh).sum(2)
            dlus = (ds * us).abs()
            dB_k[:, :, s] = (g * ds * us).sum(2)
            edB_k[:, :, s] = chan(dlus * eg + us.abs() * G * es + 2 * U * G * dlus) + gD * (G * dlus).sum(2)
            # du = dy Ds + delta' sum_n g B
            s1, S1m = (g * Bs).sum(-1), (G * Bs.abs()).sum(-1)
            es1 = (Bs.abs() * eg).sum(-1) + (N + 1) * U * S1m
            dyD = (dyk[:, :, s] * Dk).abs()
            du_k[:, :, s] = dyk[:, :, s] * Dk + dl[:, :, s] * s1
            dum_k[:, :, s] = dyD + dl[:, :, s] * S1m
            edu_k[:, :, s] = dl[:, :, s] * es1 + edl[:, :, s] * S1m + 2 * U * dum_k[:, :, s]
            # ddelta = sigmoid(x)·(u sum_n g B + sum_n g A a h_prev)
            ah, ahm = a * hp, a * Mp
            eah = eh + es * (us * Bs).abs() + 2 * U * v.abs() + U * ahm
            t, tm = g * ah, G * ahm
            et = G * eah + eg * ahm + U * tm
            s2, S2m = (t * Ak).sum(-1), (tm * absA).sum(-1)
            es2 = (et * absA).sum(-1) + (N + 3) * U * S2m
            X = u[:, :, s] * s1 + s2
            Xm = u[:, :, s].abs() * S1m + S2m
            eX = u[:, :, s].abs() * es1 + es2 + 2 * U * Xm
            sg = sig[:, :, s]
            esg = torch.exp(-dl[:, :, s]) * (E2 + 2 * U * dl[:, :, s] + edl[:, :, s]) + U
            dd_k[:, :, s] = sg * X
            edd_k[:, :, s] = (sg * eX + Xm * esg + U * sg * Xm) * m[:, :, s]
            # dA = sum_{b,l} g delta' a h_prev
            dA_k += (t * ds).sum((0, 1))
            dA_tot += t * ds
            dA_abs += (t * ds).abs()
            edA_k += ds * et + tm * es + U * ds * tm
            q, eq = a * g, a * eg + a * rho * G + U * a * G
        put(ref["ddelta"][k], dd_k * m); put(bnd["ddelta"][k], edd_k)
        ref["dB"][:, :, k].index_copy_(1, pf, dB_k.reshape(Bt, nb * LT, N)); bnd["dB"][:, :, k].index_copy_(1, pf, edB_k.reshape(Bt, nb * LT, N))
        ref["dC"][:, :, k].index_copy_(1, pf, dC_k.reshape(Bt, nb * LT, N)); bnd["dC"][:, :, k].index_copy_(1, pf, edC_k.reshape(Bt, nb * LT, N))
        mm = m.expand_as(u).reshape(Bt, nb * LT, D)
        ref["dxc"].index_add_(1, pf, (du_k.reshape(Bt, nb * LT, D) * mm))
        bnd["dxc"].index_add_(1, pf, (edu_k.reshape(Bt, nb * LT, D) * mm))
        dxc_mag.index_add_(1, pf, (dum_k.reshape(Bt, nb * LT, D) * mm))
        ref["dA"][k * D:(k + 1) * D] = dA_k
        bnd["dA"][k * D:(k + 1) * D] = tile_rss(edA_k) + _acc(dA_tot, dA_abs, Lseq)
        dyu = dyk * u
        ref["dDs"][k * D:(k + 1) * D] = dyu.sum((0, 1, 2))
        bnd["dDs"][k * D:(k + 1) * D] = U * dyu.abs().sum((0, 1, 2)) + _acc(dyu.sum(2), dyu.abs().sum(2), Lseq)
        dd_k *= m
        ref["ddtb"][k] = dd_k.sum((0, 1, 2))
        bnd["ddtb"][k] = tile_rss(edd_k.sum(2)) + _acc(dd_k.sum(2), (dd_k.abs() + edd_k).sum(2), Lseq)

    y, ey = ss2d_fwd_ref64(kind, xc, xdbl, dtw, dtb, A, Ds, H, W, device=dev, on_walk=backward, delta=delta)
    bnd["dxc"] += K * U * dxc_mag
    for key in ("delta", "dxc", "ddelta", "dB", "dC"):
        sl = (slice(None), slice(0, Lseq)) if key in ("dxc", "dB", "dC") else (slice(None), slice(None), slice(0, Lseq))
        ref[key], bnd[key] = ref[key][sl].contiguous(), bnd[key][sl].contiguous()
    for key in bnd:
        bnd[key] = bnd[key] * SAFETY
    ref["y"], bnd["y"] = y, ey
    return ref, bnd
