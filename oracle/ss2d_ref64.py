"""fp64 reference of the fused SS2D scan core (sigma_ss2d_scan_fwd_save, sigma_ss2d_scan_bwd{,_saved}) with a per-element error
bound for each output of the fp32 kernels.  ORACLE — test infrastructure only.  Plain torch float64, device-agnostic.

Operation (kind "cross4": four directions over an H x W map; "seq2": forward and reversed walks over [rgb ‖ x], Lseq = 2·H·W).
For direction k, walk step l visits position p = idx_k[l] (row-major, column-major l = w·H + h, and their reverses):
    delta'_l = softplus(dt_r[p] · W_dt[k]^T + bias[k])                  (K, B, Lseq, D) slabs, stored at position p
    h_l = exp(delta'_l · A) ⊙ h_{l-1} + delta'_l · u_l · B_l,  y_l = C_l · h_l + Ds · u_l
and the hand-written backward of sum over k and l of dy[p] · y_l: dxc (summed over directions), ddelta (pre-softplus), dB / dC (the
B and C columns of dxdbl), dA (with respect to A), dDs and ddtb.  `hs` is the state entering every 16-position block of each walk,
indexed as FbWalk::tile / ss2d_save_tiles define it: tile tau of a reversed walk is memory tile ntiles-1-tau, a column-major tile
holds min(16, H - i0) positions of one column.  Blocks a direction's walk does not reach are NaN.

Memory and time.  Each walk is cut into its 16-position tiles (ragged tiles padded with identity steps: delta' = 0, u = B = C =
dy = 0).  A scan runs in three levels: (1) every tile from a zero state, 16 steps vectorised over the tiles, keeping its end state
and decay product; (2) the tile-start states, sequentially over the tiles; (3) the 16 steps again from those states.  Only one
direction's states (h in fp64 and its error bound in fp32, (B, tiles, 16, D, N) each) are held at a time.  The largest case,
Sigma-tiny stage 0 (B 2, 120 x 160, D 192, N 16), takes about 2 s and under 8 GB on an H100.

Error bound.  A first-order running error analysis in fp64, carried through both recurrences alongside the values, in units of
u = 2^-24 (fp32 rounding) and E2 = 2^-22 (the relative error bound the PTX ISA documents for ex2.approx.f32):
  * delta':  |err| <= sigmoid(x)·(R+2)·u·(|bias| + sum_q |W_q dt_q|) + 6e-7·delta'  (dot product; softplus20's polynomial < 2.5e-7
    relative, its ex2 and the fma chain's roundings).
  * decay a = ex2(delta'·A·log2 e): relative error rho = E2 + 2u·|delta' A| + |A|·err(delta') (the ex2 bound, the two roundings
    of the argument, and delta' itself).
  * state:  e_l = a_l e_{l-1} + a_l rho_l |h_{l-1}| + |u B| err(delta') + 3u|delta' u B| + u |h_l|  (the fma and the two
    products): to first order the error of h_l is exactly the decayed sum of these local perturbations.
    In the long-memory regime (delta' near dt_min = 1e-3, A = -1) e_l sums about 1/(delta'|A|) = 1000 decay errors before they
    fade, and so does the bound.
  * backward: g_l = dy_l C_l + a_{l+1} g_{l+1} (the gradient reaching h_l) with error
    e^g_l = a_{l+1} e^g_{l+1} + a_{l+1} rho_{l+1} |g_{l+1}| + 2u |g_l|.  Every output is then a short expression in h, g, delta', u,
    B, C; its bound is the first-order sum of |partial| x error of each operand plus u per rounding on the magnitudes.
  * accumulation order: the atomics and per-thread sums of dA, dDs, ddtb (B·L terms), dB / dC (D terms), and the 2-4 direction
    terms of dxc.  Sums of more than 16 terms use the probabilistic model of Higham & Mary (SIAM J. Sci. Comput. 2019): the
    rounding errors of a sum behave as independent, so n roundings of partial sums bounded by S err by at most 4·sqrt(n)·u·S.
    Over the D channels S = sum|terms|; over the B·L positions S is the largest partial sum the kernel can form (_acc), because
    sum|terms| is ~sqrt(B·L) times the result when the terms' signs vary and 4·sqrt(n)·u·sum|terms| would exceed the whole
    1e-3-of-scale bar at B·L = 38400.  Up to 16 terms (dxc's directions) the bound is the rigorous n·u·sum|terms|.
  * the first-order errors of the D channel terms of dB and dC: the smaller of their absolute sum and LAMBDA·sqrt of their sum of
    squares (chan), since every channel runs its own recurrence.
  * the first-order errors of the B·L terms of dA and ddtb: added in absolute value within a 16-position tile, and as independent
    across tiles (tile_rss).  Summed in absolute value over all 38400 terms they would again exceed the 1e-3-of-scale bar.
All first-order terms are multiplied by SAFETY = 1.5 to cover second-order terms and the few roundings not itemised above (the L-segment
summaries' sum of delta' and the combine kernels, whose carry is a product of decays applied to a segment's start state rather than
to each step's state).  Every bound is per element; none is a fraction of the tensor's maximum.
"""
import math

import numpy as np
import torch

U = 2.0 ** -24
E2 = 2.0 ** -22
SP = 6e-7
SAFETY = 1.5
LAMBDA = 6.0
LT = 16


def dir_index(kind, H, W):
    """position visited at walk step l, per direction"""
    L = H * W
    if kind == "cross4":
        row = np.arange(L)
        col = (np.arange(H)[None, :] * W + np.arange(W)[:, None]).reshape(-1)      # l = w·H + h -> position h·W + w
        return [row, col, row[::-1].copy(), col[::-1].copy()]
    a = np.arange(2 * L)
    return [a, a[::-1].copy()]


def walk_tiles(kind, H, W):
    """per direction: (ntiles, 16) positions of each walk-order tile in walk order, -1 past a ragged tile's end"""
    out = []
    Lseq = H * W * (2 if kind == "seq2" else 1)
    for k, idx in enumerate(dir_index(kind, H, W)):
        colmajor = kind == "cross4" and k % 2 == 1
        rev = k >= 2 if kind == "cross4" else k == 1
        I, O = (H, W) if colmajor else (Lseq, 1)
        tpo = -(-I // LT)
        ntiles = O * tpo
        o, i = (idx % W, idx // W) if colmajor else (np.zeros_like(idx), idx)
        tm = o * tpo + i // LT
        tau = ntiles - 1 - tm if rev else tm
        assert np.all(np.diff(tau) >= 0)
        start = np.searchsorted(tau, np.arange(ntiles))
        blk = np.full((ntiles, LT), -1, np.int64)
        blk[tau, np.arange(len(idx)) - start[tau]] = idx
        out.append(blk)
    return out


def bound_fraction(got, ref, bound):
    """largest |got - ref| / bound; an element whose bound is 0 (a state that is exactly 0) must be exact"""
    err = (got.to(ref.device, torch.float64) - ref).abs()
    frac = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    return float(frac.max()) if frac.numel() else 0.0


def _gt(n):
    """relative bound of an n-term sum's accumulation error"""
    return U * (n if n <= 16 else 4.0 * math.sqrt(n))


def tile_rss(e):
    """bound of a sum over positions of terms with first-order error bounds e (B, tiles, ...): added in absolute value within a
    16-position tile, treated as independent across tiles (LAMBDA·sqrt of the sum of squares; Hoeffding's inequality puts the
    chance of exceeding it below 2·exp(-LAMBDA²/2) = 3e-8)"""
    return LAMBDA * (e * e).sum((0, 1)).sqrt()


def chan(e):
    """bound of a sum over the D channels (dim 2) of terms with first-order error bounds e: the channels' recurrences round
    independently, so the smaller of the absolute sum and LAMBDA·sqrt of the sum of squares"""
    return torch.minimum(e.sum(2), LAMBDA * (e * e).sum(2).sqrt())


def _acc(tot, absb, L):
    """accumulation-order bound of a B·L-term sum (dA, dDs, ddtb) from per-tile totals and absolute sums (B, tiles, ...) in walk
    order: every partial sum the kernel forms (a segment's running sum, walked backwards, then one atomic per image and segment)
    is within 2·Smax of 0, Smax = the largest |sum of a walk's suffix|, bounded per tile by the suffix after it plus the tile's
    absolute sum.  4·sqrt(L)·u per running partial sum (probabilistic) and 64·u per atomic (up to 64 segments, rigorous)."""
    after = tot.flip(1).cumsum(1).flip(1) - tot
    smax = (after.abs() + absb).amax(1)
    return U * (8.0 * math.sqrt(L) + 128.0) * smax.sum(0)


def _chain(P, loc, rev=False):
    """level 2: the state entering every tile, given each tile's decay product P and zero-start end state loc"""
    starts = torch.empty_like(loc)
    cur = torch.zeros_like(loc[:, 0])
    order = range(loc.shape[1] - 1, -1, -1) if rev else range(loc.shape[1])
    for t in order:
        starts[:, t] = cur
        cur = P[:, t] * cur + loc[:, t]
    return starts


def ss2d_ref64(kind, xc, xdbl, dtw, dtb, A, Ds, dy, H, W, device=None):
    """kind "cross4" / "seq2"; xc, dy (B, Lseq, D), xdbl (B, Lseq, K, Cp) = [B | C | dt_r | padding], dtw (K, D, R), dtb (K, D),
    A (K·D, N), Ds (K·D).  Returns (ref, bound): two dicts of float64 tensors with keys y, delta, hs, dxc, ddelta, dB, dC, dA, dDs,
    ddtb.  y / delta / ddelta (K, B, Lseq, D), hs (K, B, max_tiles, D, N), dB / dC (B, Lseq, K, N)."""
    dev = torch.device(device) if device is not None else xc.device
    f = lambda t: t.detach().to(dev, torch.float64)
    xc, xdbl, dtw, dtb, A, Ds, dy = map(f, (xc, xdbl, dtw, dtb, A, Ds, dy))
    Bt, Lseq, D = xc.shape
    K, N, R = xdbl.shape[2], A.shape[1], dtw.shape[2]
    tiles = walk_tiles(kind, H, W)
    assert len(tiles) == K
    T = max(t.shape[0] for t in tiles)
    z = lambda *s: torch.zeros(s, dtype=torch.float64, device=dev)
    ref = dict(y=z(K, Bt, Lseq + 1, D), delta=z(K, Bt, Lseq + 1, D), hs=torch.full((K, Bt, T, D, N), math.nan, dtype=torch.float64, device=dev),
               dxc=z(Bt, Lseq + 1, D), ddelta=z(K, Bt, Lseq + 1, D), dB=z(Bt, Lseq + 1, K, N), dC=z(Bt, Lseq + 1, K, N), dA=z(K * D, N),
               dDs=z(K * D), ddtb=z(K, D))
    bnd = {k: torch.zeros_like(v) for k, v in ref.items()}
    bnd["hs"].fill_(math.nan)
    dxc_mag = z(Bt, Lseq + 1, D)
    pad = lambda t: torch.cat([t, torch.zeros_like(t[:, :1])], 1)          # position Lseq = the padding's zero row
    xcp, dyp, xdp = pad(xc), pad(dy), pad(xdbl)
    for k in range(K):
        blk = torch.from_numpy(tiles[k]).to(dev)
        nb = blk.shape[0]
        m = (blk >= 0).double()[None, :, :, None]                               # (1, nb, 16, 1)
        p = torch.where(blk >= 0, blk, torch.full_like(blk, Lseq))
        u = xcp[:, p]                                                           # (B, nb, 16, D)
        xk = xdp[:, p, k]
        Bm, Cm, dtr = xk[..., :N], xk[..., N:2 * N], xk[..., 2 * N:2 * N + R]
        pre = dtr @ dtw[k].t() + dtb[k]
        Tm = dtr.abs() @ dtw[k].abs().t() + dtb[k].abs()
        dl = torch.nn.functional.softplus(pre) * m
        sig = torch.sigmoid(pre)
        edl = (sig * (R + 2) * U * Tm + SP * dl) * m
        del Tm, dtr, xk
        dyk = dyp[:, p]
        Ak, Dk = A[k * D:(k + 1) * D], Ds[k * D:(k + 1) * D]
        dlu = dl * u
        absA = Ak.abs()

        def slot(s):
            d_, e_ = dl[:, :, s, :, None], edl[:, :, s, :, None]
            a = torch.exp(d_ * Ak)
            rho = E2 + 2 * U * (d_ * absA) + absA * e_
            v = dlu[:, :, s, :, None] * Bm[:, :, s, None, :]
            ein = u[:, :, s, :, None].abs() * Bm[:, :, s, None, :].abs() * e_ + 3 * U * v.abs()
            return a, rho, v, ein

        # ---- forward: h (levels 1 + 2), its error e (levels 1 + 2), then both at every step (level 3) ----
        sh = (Bt, nb, D, N)
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
        h_all = torch.empty((Bt, nb, LT, D, N), dtype=torch.float64, device=dev)
        e_all = torch.empty(h_all.shape, dtype=torch.float32, device=dev)      # a bound: 24 bits are plenty
        h, e = h0, e0
        yk, ey = torch.empty_like(u), torch.empty_like(u)
        for s in range(LT):
            a, rho, v, ein = slot(s)
            hn = a * h + v
            e = a * e + a * rho * h.abs() + ein + U * hn.abs()
            h = hn
            h_all[:, :, s], e_all[:, :, s] = h, e
            C = Cm[:, :, s, None, :]
            du_ = Dk * u[:, :, s]
            yk[:, :, s] = (C * h).sum(-1) + du_
            ey[:, :, s] = (C.abs() * e).sum(-1) + (N + 2) * U * ((C * h).abs().sum(-1) + du_.abs())
        ntk = nb
        ref["hs"][k, :, :ntk], bnd["hs"][k, :, :ntk] = h0, e0
        pf = p.reshape(-1)
        put = lambda dst, src: dst.index_copy_(1, pf, src.reshape(Bt, nb * LT, *src.shape[3:]))
        put(ref["y"][k], yk); put(bnd["y"][k], ey)
        put(ref["delta"][k], dl); put(bnd["delta"][k], edl)
        del yk, ey

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
        del h_all, e_all
    bnd["dxc"] += K * U * dxc_mag
    for key in ("y", "delta", "dxc", "ddelta", "dB", "dC"):
        sl = (slice(None), slice(0, Lseq)) if key in ("dxc", "dB", "dC") else (slice(None), slice(None), slice(0, Lseq))
        ref[key], bnd[key] = ref[key][sl].contiguous(), bnd[key][sl].contiguous()
    for key in bnd:
        bnd[key] = bnd[key] * SAFETY
    return ref, bnd
