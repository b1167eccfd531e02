"""fp64 reference of the op-level selective scan (sigma_scan_fwd{,_split}, sigma_scan_bwd{,_split,_det}, i.e. the drop-in
selective_scan_cuda_core.fwd / bwd) with a per-element error bound for each output of the kernels.  ORACLE — test infrastructure
only.  Plain torch float64, device-agnostic.

Operation, in the op's layout: u, delta (b, dim, L); A (dim, N); B, C (b, G, N, L), channel d reads group g = d // (dim / G);
D, delta_bias (dim) nullable.  16-bit u / delta / B / C / dout are taken at their exact values.
    delta'_l = softplus(delta_l + bias)   (or delta_l + bias without softplus)
    h_l = exp(delta'_l · A) ⊙ h_{l-1} + delta'_l · u_l · B_l,   out_l = C_l · h_l + D · u_l
`x` holds (prod of the decays since the sequence start, h) at every 2048-position chunk end and at L, interleaved per state, as
the kernels write it.  With dout: du, ddelta (pre-softplus), dA, dB, dC, dD, ddelta_bias of sum(dout · out).

The error model is oracle/ss2d_ref64.py's: the same constants (U, E2, SP, SAFETY, LAMBDA), the same first-order recurrences for
the state (e) and the gradient reaching it (e^g), the same accumulation-order bounds (_gt, _acc, tile_rss and the channel sum
chan), and the same 3-level evaluation over 16-position tiles.  That module's walk core is written around its direction gather
and dt_proj dot product, so this one restates the core for the op's layout rather than reshaping it (its outputs stay bit for
bit what its tests pin).  What differs from the SS2D model:
  * delta':  one fp32 add (delta + bias), then softplus20: err <= sigmoid(x)·u·|x| + SP·delta'; without softplus u·|x|.
  * ddelta's sigmoid factor is __fdividef(1, 1 + ex2(-x·log2 e)) on the pre-activation x: relative error
    (1 - s)·(E2 + 3u|x|) + 3u (the ex2, the argument's roundings and x's own, the add and the fast division), and the factor is
    skipped (taken as 1) above x = 20.  The backward's A·log2 e and ·ln 2 add two roundings to the sum over the states.
  * dB / dC: sums over the dim / G channels of a group (chan + _gt(dim / G)), returned in fp32.
  * dA / dD / ddelta_bias: sums over batch·L (per-thread sums, one atomic per (batch, segment), or the deterministic build's
    partials): _acc and tile_rss, as for dA / dDs / ddtb there.
  * 16-bit outputs (out, du, ddelta) are rounded once to fp16 (2^-11 relative) or bf16 (2^-8) on top of the fp32 bound; fp16
    also 2^-25 absolute, its rounding error among the subnormals (ddelta = sigmoid(x)·X sits there at delta' ~ 1e-3).
  * x: h carries the state bound.  The product is ex2(a2·S), S the fp32 running sum of delta' since the CTA's segment start,
    times the fp32 product of the preceding segments' ex2(a2·S_s) (up to 64 factors).  Its error, in units of the exponent:
    65·(E2 + u) (an ex2 and a multiply per segment), 2u·|A|·S (the argument's roundings), |A|·(_gt(n)·sum|delta'| + sum of the
    delta' errors) (the sums' roundings, any cut into segments, and delta' itself), applied as P·expm1(.); plus an absolute 2^-125
    for ex2.approx.ftz's flush below 2^-126 (a product of factors <= 1 that flushes is itself below that).
Memory: channels recur independently, so they are evaluated in blocks of at most `block_bytes` of states (h in fp64 and its bound
in fp32 per position); dB / dC accumulate across the blocks of a group.  The (2, 768, 19200, N 16) backward takes ~2 GB per block.
"""
import math

import torch

from .ss2d_ref64 import BF16_RN, E2, LAMBDA, SAFETY, SP, U, _acc, _chain, _gt, bound_fraction, tile_rss  # noqa: F401

LT = 16
CHUNK = 2048
F16_RN = 2.0 ** -11
F16_SUB = 2.0 ** -25          # half the spacing of fp16's subnormals: the rounding error below its smallest normal, 2^-14
FTZ = 2.0 ** -125
MAX_SEGMENTS = 64
OUTS = ("out", "x", "du", "ddelta", "dA", "dB", "dC", "dD", "ddelta_bias")


def rounding(dtype):
    """relative error of rounding an fp32 value to `dtype` to nearest (0 for fp32)"""
    return {torch.float16: F16_RN, torch.bfloat16: BF16_RN}.get(dtype, 0.0)


def _gtv(n):
    """_gt for a tensor of term counts"""
    n = n.double()
    return U * torch.where(n <= 16, n, 4.0 * n.sqrt())


def _tiles(t, nt):
    """(b, c, L) -> (b, nt, LT, c), zero past L"""
    b, c, L = t.shape
    return torch.nn.functional.pad(t, (0, nt * LT - L)).view(b, c, nt, LT).permute(0, 2, 3, 1)


def _untile(t, L):
    """(b, nt, LT, c) -> (b, c, L)"""
    b, nt, lt, c = t.shape
    return t.permute(0, 3, 1, 2).reshape(b, c, nt * lt)[:, :, :L]


def scan_ref64(u, delta, A, B, C, D=None, delta_bias=None, softplus=True, dout=None, device=None, block_bytes=2e9):
    """Returns (ref, bound): dicts of float64 tensors, keys out, x and, with dout, du, ddelta, dA, dB, dC and dD / ddelta_bias when
    D / delta_bias are given.  out / du / ddelta (b, dim, L), x (b, dim, ceil(L / 2048), 2·N), dA (dim, N), dB / dC (b, G, N, L).
    Bounds are per element, SAFETY applied, 16-bit roundings of out / du / ddelta included for 16-bit u."""
    odt = u.dtype
    rn = rounding(odt)
    dev = torch.device(device) if device is not None else u.device
    f = lambda t: None if t is None else t.detach().to(dev, torch.float64)
    u, delta, A, B, C, D, bias, dout = map(f, (u, delta, A, B, C, D, delta_bias, dout))
    b, dim, L = u.shape
    G, N = B.shape[1], B.shape[2]
    dpg = dim // G
    nt = -(-L // LT)
    nch = -(-L // CHUNK)
    ends = torch.tensor([min((c + 1) * CHUNK, L) - 1 for c in range(nch)], device=dev)
    bwd = dout is not None
    z = lambda *s: torch.zeros(s, dtype=torch.float64, device=dev)
    ref = dict(out=z(b, dim, L), x=z(b, dim, nch, 2 * N))
    if bwd:
        ref.update(du=z(b, dim, L), ddelta=z(b, dim, L), dA=z(dim, N), dB=z(b, G, N, L), dC=z(b, G, N, L))
        if D is not None:
            ref["dD"] = z(dim)
        if bias is not None:
            ref["ddelta_bias"] = z(dim)
    bnd = {k: torch.zeros_like(v) for k, v in ref.items()}
    m = _tiles(torch.ones(b, 1, L, dtype=torch.float64, device=dev), nt)                  # (b, nt, LT, 1): 0 past L
    cb = max(1, min(dpg, int(block_bytes // (b * nt * LT * N * 12))))
    gD = _gt(dpg)

    for g in range(G):
        Bg, Cg = _tiles(B[:, g], nt), _tiles(C[:, g], nt)                                    # (b, nt, LT, N)
        if bwd:
            grp = {k: z(b, nt, LT, N) for k in ("dB", "edB", "qB", "mB", "dC", "edC", "qC", "mC")}
        for d0 in range(g * dpg, (g + 1) * dpg, cb):
            d1 = min(d0 + cb, (g + 1) * dpg)
            ub = _tiles(u[:, d0:d1], nt)                                                   # (b, nt, LT, c)
            pre = _tiles(delta[:, d0:d1], nt) + (bias[d0:d1] if bias is not None else 0.0)
            if softplus:
                dl = torch.nn.functional.softplus(pre) * m
                sig = torch.sigmoid(pre)
                edl = (sig * U * pre.abs() + SP * dl) * m
            else:
                dl, sig = pre * m, None
                edl = U * pre.abs() * m
            Ak = A[d0:d1]
            absA = Ak.abs()
            Dk = D[d0:d1] if D is not None else torch.zeros(d1 - d0, dtype=torch.float64, device=dev)
            dlu = dl * ub
            c = d1 - d0

            def slot(s):
                d_, e_ = dl[:, :, s, :, None], edl[:, :, s, :, None]
                a = torch.exp(d_ * Ak)
                rho = E2 + 2 * U * (d_ * absA) + absA * e_
                v = dlu[:, :, s, :, None] * Bg[:, :, s, None, :]
                ein = ub[:, :, s, :, None].abs() * Bg[:, :, s, None, :].abs() * e_ + 3 * U * v.abs()
                return a, rho, v, ein

            # ---- h (levels 1 + 2), its error e (levels 1 + 2), then both at every step (level 3) ----
            sh = (b, nt, c, N)
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
            if bwd:
                h_all = torch.empty((b, nt, LT, c, N), dtype=torch.float64, device=dev)
                e_all = torch.empty(h_all.shape, dtype=torch.float32, device=dev)      # a bound: 24 bits are plenty
            h, e = h0, e0
            yk, eyk = torch.empty_like(ub), torch.empty_like(ub)
            xh, xe = z(b, c, nch, N), z(b, c, nch, N)
            for s in range(LT):
                a, rho, v, ein = slot(s)
                hn = a * h + v
                e = a * e + a * rho * h.abs() + ein + U * hn.abs()
                h = hn
                if bwd:
                    h_all[:, :, s], e_all[:, :, s] = h, e
                for ci in range(nch):
                    t_c, s_c = divmod(int(ends[ci]), LT)
                    if s_c == s:
                        xh[:, :, ci], xe[:, :, ci] = h[:, t_c], e[:, t_c]
                Cs = Cg[:, :, s, None, :]
                du_ = Dk * ub[:, :, s]
                yk[:, :, s] = (Cs * h).sum(-1) + du_
                eyk[:, :, s] = (Cs.abs() * e).sum(-1) + (N + 2) * U * ((Cs * h).abs().sum(-1) + du_.abs())
            ref["out"][:, d0:d1] = _untile(yk, L)
            bnd["out"][:, d0:d1] = _untile(eyk, L)
            del yk, eyk
            # ---- x: (prod of the decays since the sequence start, h) at the chunk ends ----
            flat = lambda t: t.reshape(b, nt * LT, c)
            S = flat(dl).cumsum(1)[:, ends]                                                # (b, nch, c)
            Sa = flat(dl.abs()).cumsum(1)[:, ends]
            Se = flat(edl).cumsum(1)[:, ends]
            Px = torch.exp(S[..., None] * Ak)                                              # (b, nch, c, N)
            rel = (MAX_SEGMENTS + 1) * (E2 + U) + 2 * U * absA * Sa[..., None] + \
                absA * (_gtv(ends + 1)[None, :, None, None] * Sa[..., None] + Se[..., None])
            eP = Px * torch.expm1(rel) + FTZ
            ref["x"][:, d0:d1, :, 0::2] = Px.permute(0, 2, 1, 3)
            bnd["x"][:, d0:d1, :, 0::2] = eP.permute(0, 2, 1, 3)
            ref["x"][:, d0:d1, :, 1::2] = xh
            bnd["x"][:, d0:d1, :, 1::2] = xe
            if not bwd:
                continue

            # ---- backward: q = a·g entering each step from the right, and its error, tile by tile from the right ----
            dyk = _tiles(dout[:, d0:d1], nt)

            def wslot(s):
                return dyk[:, :, s, :, None] * Cg[:, :, s, None, :]

            ql = z(*sh)
            for s in range(LT - 1, -1, -1):
                a, _, _, _ = slot(s)
                ql = a * (wslot(s) + ql)
            q0 = _chain(P, ql, rev=True)
            q, eql = q0, z(*sh)
            for s in range(LT - 1, -1, -1):
                a, rho, _, _ = slot(s)
                gg = wslot(s) + q
                eg = eql + U * gg.abs()
                eql, q = a * eg + a * rho * gg.abs() + U * (a * gg).abs(), a * gg
            eq0 = _chain(P, eql, rev=True)
            del ql, eql
            q, eq = q0, eq0
            dd_k, edd_k = torch.empty_like(ub), torch.empty_like(ub)
            du_k, edu_k = torch.empty_like(ub), torch.empty_like(ub)
            dA_k, edA_k = z(c, N), z(*sh)
            dA_tot, dA_abs = z(*sh), z(*sh)
            for s in range(LT - 1, -1, -1):
                a, rho, v, _ = slot(s)
                gg = wslot(s) + q
                Gm = gg.abs()
                eg = eq + U * Gm
                h, eh = h_all[:, :, s], e_all[:, :, s].double()
                hp = h_all[:, :, s - 1] if s > 0 else h0
                Mh, Mp = h.abs(), hp.abs()
                dys, us, ds, es = dyk[:, :, s, :, None], ub[:, :, s, :, None], dl[:, :, s, :, None], edl[:, :, s, :, None]
                Bs = Bg[:, :, s, None, :]
                # dC = sum over the group's channels of dy h,  dB = the same of g delta' u
                ec = dys.abs() * (eh + U * Mh)
                grp["dC"][:, :, s] += (dys * h).sum(2)
                grp["edC"][:, :, s] += ec.sum(2)
                grp["qC"][:, :, s] += (ec * ec).sum(2)
                grp["mC"][:, :, s] += (dys.abs() * Mh).sum(2)
                dlus = (ds * us).abs()
                eb = dlus * eg + us.abs() * Gm * es + 2 * U * Gm * dlus
                grp["dB"][:, :, s] += (gg * ds * us).sum(2)
                grp["edB"][:, :, s] += eb.sum(2)
                grp["qB"][:, :, s] += (eb * eb).sum(2)
                grp["mB"][:, :, s] += (Gm * dlus).sum(2)
                # du = dy D + delta' sum_n g B
                s1, S1m = (gg * Bs).sum(-1), (Gm * Bs.abs()).sum(-1)
                es1 = (Bs.abs() * eg).sum(-1) + (N + 1) * U * S1m
                dum = (dyk[:, :, s] * Dk).abs() + dl[:, :, s] * S1m
                du_k[:, :, s] = dyk[:, :, s] * Dk + dl[:, :, s] * s1
                edu_k[:, :, s] = dl[:, :, s] * es1 + edl[:, :, s] * S1m + 2 * U * dum
                # ddelta = sigmoid(x)·(u sum_n g B + sum_n g A a h_prev)
                ah, ahm = a * hp, a * Mp
                eah = eh + es * (us * Bs).abs() + 2 * U * v.abs() + U * ahm
                t, tm = gg * ah, Gm * ahm
                et = Gm * eah + eg * ahm + U * tm
                s2, S2m = (t * Ak).sum(-1), (tm * absA).sum(-1)
                es2 = (et * absA).sum(-1) + (N + 5) * U * S2m
                X = ub[:, :, s] * s1 + s2
                Xm = ub[:, :, s].abs() * S1m + S2m
                eX = ub[:, :, s].abs() * es1 + es2 + 2 * U * Xm
                if softplus:
                    x_, sg = pre[:, :, s], sig[:, :, s]
                    esg = sg * ((1 - sg) * (E2 + 3 * U * x_.abs()) + 3 * U) + torch.where(x_ > 20, 1 - sg, 0.0)
                    dd_k[:, :, s] = sg * X
                    edd_k[:, :, s] = (sg * eX + Xm * esg + U * sg * Xm) * m[:, :, s]
                else:
                    dd_k[:, :, s] = X
                    edd_k[:, :, s] = eX * m[:, :, s]
                # dA = sum_{b,l} g delta' a h_prev
                dA_k += (t * ds).sum((0, 1))
                dA_tot += t * ds
                dA_abs += (t * ds).abs()
                edA_k += ds * et + tm * es + U * ds * tm
                q, eq = a * gg, a * eg + a * rho * Gm + U * a * Gm
            del h_all, e_all
            dd_k *= m
            ref["du"][:, d0:d1], bnd["du"][:, d0:d1] = _untile(du_k, L), _untile(edu_k, L)
            ref["ddelta"][:, d0:d1], bnd["ddelta"][:, d0:d1] = _untile(dd_k, L), _untile(edd_k, L)
            ref["dA"][d0:d1] = dA_k
            bnd["dA"][d0:d1] = tile_rss(edA_k) + _acc(dA_tot, dA_abs, L)
            if D is not None:
                dyu = dyk * ub
                ref["dD"][d0:d1] = dyu.sum((0, 1, 2))
                bnd["dD"][d0:d1] = U * dyu.abs().sum((0, 1, 2)) + _acc(dyu.sum(2), dyu.abs().sum(2), L)
            if bias is not None:
                ref["ddelta_bias"][d0:d1] = dd_k.sum((0, 1, 2))
                bnd["ddelta_bias"][d0:d1] = tile_rss(edd_k.sum(2)) + _acc(dd_k.sum(2), (dd_k.abs() + edd_k).sum(2), L)
        if bwd:
            for k in ("dB", "dC"):
                eb = torch.minimum(grp["e" + k], LAMBDA * grp["q" + k[1:]].sqrt()) + gD * grp["m" + k[1:]]
                ref[k][:, g] = _untile(grp[k], L)
                bnd[k][:, g] = _untile(eb, L)
    for k in bnd:
        bnd[k] = bnd[k] * SAFETY
    for k in ("out", "du", "ddelta"):
        if k in bnd and rn:
            bnd[k] = bnd[k] + rn * (ref[k].abs() + bnd[k]) + (F16_SUB if odt == torch.float16 else 0.0)
    return ref, bnd
