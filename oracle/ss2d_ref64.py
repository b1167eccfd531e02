"""fp64 reference of the fused SS2D scan core (sigma_ss2d_scan_fwd{,_split,_bf16,_save{,_bf16}}, sigma_ss2d_scan_bwd_saved{,_bf16,_det})
with a per-element error bound for each output of the fp32 kernels.  ORACLE — test infrastructure only.  Plain torch float64,
device-agnostic.  ss2d_fwd_ref64 is the forward alone (y and its bound, every kind, fp32 or bf16 xc); ss2d_ref64 runs it and
adds the backward (every kind).

Operation (kind "cross4": four directions over an H x W map; "seq2": forward and reversed walks over [rgb ‖ x], Lseq = 2·H·W;
"cross": the cross-modality scan, one row-major walk over the batch Bt = 2·images, images [0, Bt/2) of modality 0 and
[Bt/2, Bt) of modality 1: image b runs with weight set w = [b >= Bt/2] (its rows of A, Ds, dt_proj and bias, A (2·D, N)) and its
own B and dt_r, but takes C from the other modality's image b' = (b + Bt/2) mod Bt (vmamba.py:1530,1536)).  walk_groups lists
the walks: (direction, images, weight set, images C is read from).  Each walk's backward credits dB and dxc to its own images,
dC to the images that supplied C (under "cross" the other half's rows of dxdbl), and dA, dDs and d dt_bias to its weight set's
rows: K sets for "cross4" / "seq2", the two modalities' for "cross" (dA (2D, N), dDs (2D), ddtb (2, D)).
For direction k, walk step l visits position p = idx_k[l] (row-major, column-major l = w·H + h, and their reverses):
    delta'_l = softplus(dt_r[p] · W_dt[k]^T + bias[k])                  (K, B, Lseq, D) slabs, stored at position p
    h_l = exp(delta'_l · A) ⊙ h_{l-1} + delta'_l · u_l · B_l,  y_l = C_l · h_l + Ds · u_l
and the hand-written backward of sum over k and l of dy[p] · y_l: dxc (summed over directions), ddelta (pre-softplus), dB / dC (the
B and C columns of dxdbl), dA (with respect to A), dDs and ddtb.  `hs` is the state entering every 16-position block of each walk,
indexed as FbWalk::tile / ss2d_save_tiles define it: tile tau of a reversed walk is memory tile ntiles-1-tau, a column-major tile
holds min(16, H - i0) positions of one column.  Blocks a direction's walk does not reach are NaN.

Memory and time.  Each walk is cut into its 16-position tiles (ragged tiles padded with identity steps: delta' = 0, u = B = C =
dy = 0).  The reference's tiling is its own: the kernels' tiles are 32 positions at d_state 4 and 8.  A scan runs in three levels:
(1) every tile from a zero state, 16 steps vectorised over the tiles, keeping its end state and decay product; (2) the tile-start
states, sequentially over the tiles; (3) the 16 steps again from those states.  Only one direction's states (h in fp64 and its
error bound in fp32, (B, tiles, 16, D, N) each) are held at a time, and the forward alone keeps none of them.  The largest
backward case, Sigma-tiny stage 0 (B 2, 120 x 160, D 192, N 16), takes about 2 s and under 8 GB on an H100.

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
  * y = C·h + Ds·u:  sum_n |C| e_l + (N+2)·u·(sum_n |C h| + |Ds u|)  (the N-term dot product and the skip's fma).  With bf16 xc
    the reference takes xc's exact bf16 values (the kernel widens them exactly), and the bf16 store's round-to-nearest adds
    2^-8·|y| relative, on the fp32 value: 2^-8·(|y| + its fp32 bound), after SAFETY.
  * L-segments (the forward's summary / combine / apply passes): a segment's carried decay is ex2(a2·S), S the fp32 sum of the
    segment's delta' (up to 32·tiles_per_split terms), in place of the product of the per-step decays.  Its relative error is one
    E2, two roundings of the argument, |A|·(the sum's rounding, at most n·u·S for n terms) and |A|·(sum of the delta' errors).
    The last is the per-step |A|·err(delta') summed; the rest replaces n per-step E2 terms, n·E2 = 4n·u, applied to the same
    carried state.  |A|·S·n·u exceeds 4n·u only when |A|·S > 4, where the carried state has decayed below e^-4 of its value and
    the per-step terms of the positions after it dominate, so the itemised per-step bound covers the segmented walk (checked by
    an fp32 emulation that forms 32-segment carries the way the summary pass does, tests/test_ss2d_ref64_cpu.py).
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
All first-order terms are multiplied by SAFETY = 1.5 to cover second-order terms and the few roundings not itemised above (the
combine kernels, whose carry is a product of decays applied to a segment's start state rather than to each step's state).  Every
bound is per element; none is a fraction of the tensor's maximum.

A given delta' (delta=, the bf16 training mode: its kernels round delta' = softplus(dt_proj) to bf16 before the recurrence uses it
and save that value).  The recurrence and the backward then run on an fp64 copy of the given values, taken as exact: err(delta') =
0 in every term above, and the softplus derivative is 1 - exp(-delta') of the given value, as the backward kernel forms it.  delta'
itself is checked apart, against the softplus and inside its fp32 bound + BF16_RN·|delta'| (delta_ref64, delta_bound_bf16).

`mistake` (kind "cross" only) computes the result of a plausible kernel bug instead, for tests that the bound tells it apart:
"dC_own" credits dC to the image's own row, "wset" sends dA / dDs / d dt_bias to the other weight set's rows, "C_own" reads C from
the image's own half.
"""
import math
import types

import numpy as np
import torch

U = 2.0 ** -24
E2 = 2.0 ** -22
BF16_RN = 2.0 ** -8          # relative error of rounding to bf16 (8 significand bits) to nearest
SP = 6e-7
SAFETY = 1.5
LAMBDA = 6.0
LT = 16
KINDS = {"cross4": 4, "seq2": 2, "cross": 1}     # directions (x_dbl rows per position)
MISTAKES = ("dC_own", "wset", "C_own")


def dir_index(kind, H, W):
    """position visited at walk step l, per direction"""
    L = H * W
    if kind == "cross4":
        row = np.arange(L)
        col = (np.arange(H)[None, :] * W + np.arange(W)[:, None]).reshape(-1)      # l = w·H + h -> position h·W + w
        return [row, col, row[::-1].copy(), col[::-1].copy()]
    if kind == "cross":
        return [np.arange(L)]
    a = np.arange(2 * L)
    return [a, a[::-1].copy()]


def walk_tiles(kind, H, W, lt=LT):
    """per direction: (ntiles, lt) positions of each walk-order tile in walk order, -1 past a ragged tile's end"""
    out = []
    Lseq = H * W * (2 if kind == "seq2" else 1)
    for k, idx in enumerate(dir_index(kind, H, W)):
        colmajor = kind == "cross4" and k % 2 == 1
        rev = (k >= 2) if kind == "cross4" else (k == 1 and kind == "seq2")
        I, O = (H, W) if colmajor else (Lseq, 1)
        tpo = -(-I // lt)
        ntiles = O * tpo
        o, i = (idx % W, idx // W) if colmajor else (np.zeros_like(idx), idx)
        tm = o * tpo + i // lt
        tau = ntiles - 1 - tm if rev else tm
        assert np.all(np.diff(tau) >= 0)
        start = np.searchsorted(tau, np.arange(ntiles))
        blk = np.full((ntiles, lt), -1, np.int64)
        blk[tau, np.arange(len(idx)) - start[tau]] = idx
        out.append(blk)
    return out


def walk_groups(kind, Bt):
    """(direction k, images, weight set, images C is read from) of every walk the kernels run: each direction over the whole
    batch, or for "cross" each modality's half with its own weights and the other half's C"""
    if kind != "cross":
        return [(k, slice(0, Bt), k, slice(0, Bt)) for k in range(KINDS[kind])]
    assert Bt % 2 == 0, "cross: the batch holds 2·images"
    h = Bt // 2
    return [(0, slice(0, h), 0, slice(h, Bt)), (0, slice(h, Bt), 1, slice(0, h))]


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


def _pad(t):
    return torch.cat([t, torch.zeros_like(t[:, :1])], 1)          # position Lseq = the padding's zero row


def _softplus64(dtr, dtw, dtb):
    """delta' = softplus(dt_r · W_dt^T + bias) in fp64 (dt_r (..., R), dtw (D, R), dtb (D)), the sigmoid of its argument, and
    delta''s first-order error bound in the fp32 kernels (before SAFETY)"""
    pre = dtr @ dtw.t() + dtb
    Tm = dtr.abs() @ dtw.abs().t() + dtb.abs()
    dl = torch.nn.functional.softplus(pre)
    sig = torch.sigmoid(pre)
    return dl, sig, sig * (dtr.shape[-1] + 2) * U * Tm + SP * dl


def delta_ref64(kind, xdbl, dtw, dtb, N):
    """delta' (K, B, Lseq, D) at every position in fp64 and its per-element bound (SAFETY applied), for checking a kernel's delta'
    on its own; xdbl (B, Lseq, K, Cp) and the weights as ss2d_fwd_ref64 takes them"""
    f = lambda t: t.detach().double()
    xdbl, dtw, dtb = f(xdbl), f(dtw), f(dtb)
    Bt, Lseq, K, _ = xdbl.shape
    D, R = dtw.shape[1], dtw.shape[2]
    dl, bnd = (torch.empty((K, Bt, Lseq, D), dtype=torch.float64, device=xdbl.device) for _ in range(2))
    for k, bs, kw, _ in walk_groups(kind, Bt):
        dl[k, bs], _, e = _softplus64(xdbl[bs, :, k, 2 * N:2 * N + R], dtw[kw], dtb[kw])
        bnd[k, bs] = SAFETY * e
    return dl, bnd


def delta_bound_bf16(ref_delta, bnd_delta):
    """per-element bound of a delta' the kernel rounded to bf16, from the fp64 softplus and its fp32 bound (SAFETY applied)"""
    return bnd_delta + BF16_RN * (ref_delta.abs() + bnd_delta)


def ss2d_fwd_ref64(kind, xc, xdbl, dtw, dtb, A, Ds, H, W, device=None, on_walk=None, delta=None):
    """The forward alone.  kind "cross4" / "seq2" / "cross"; xc (B, Lseq, D) fp32 or bf16, xdbl (B, Lseq, K, Cp) = [B | C | dt_r |
    padding], dtw (Kw, D, R), dtb (Kw, D), A (Kw·D, N), Ds (Kw·D), Kw = K or 2 (modalities) for "cross".  Returns (y, bound), float64
    (K, B, Lseq, D): direction k's output at the position it belongs to, and its per-element bound (SAFETY applied; with bf16 xc it
    includes the final rounding to bf16).
    on_walk(g): called after each walk with its tensors (walk group, tiles, inputs, delta', the states at every step and their
    bounds); the states are only kept when it is given.  ss2d_ref64 runs its backward from there.
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
        Bm = xk[..., :N]
        Cm = xdp[cs][:, p, k, N:2 * N]
        if dgiven is None:
            dl, sig, edl = _softplus64(xk[..., 2 * N:2 * N + R], dtw[kw], dtb[kw])
            dl, edl = dl * m, edl * m
        else:
            dl = dgiven[k, bs][:, p] * m
            edl = torch.zeros_like(dl)
            sig = -torch.expm1(-dl)
        del xk
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
            on_walk(types.SimpleNamespace(k=k, bs=bs, kw=kw, cs=cs, nb=nb, m=m, p=p, pf=pf, u=u, Bm=Bm, Cm=Cm, dl=dl, edl=edl, sig=sig,
                                          Ak=Ak, Dk=Dk, absA=absA, slot=slot, P=P, h0=h0, e0=e0, h_all=h_all, e_all=e_all))
            del h_all, e_all
    y, ey = y[:, :, :Lseq].contiguous(), ey[:, :, :Lseq] * SAFETY
    if bf16:
        ey = ey + BF16_RN * (y.abs() + ey)
    return y, ey.contiguous()


def ss2d_ref64(kind, xc, xdbl, dtw, dtb, A, Ds, dy, H, W, device=None, delta=None, mistake=None):
    """The inputs of ss2d_fwd_ref64 (fp32 xc) and dy (B, Lseq, D).  Returns (ref, bound): two dicts of float64 tensors with keys y,
    delta, hs, dxc, ddelta, dB, dC, dA, dDs, ddtb.  y / delta / ddelta (K, B, Lseq, D), hs (K, B, max_tiles, D, N), dxc (B, Lseq, D),
    dB / dC (B, Lseq, K, N), dA (Kw·D, N), dDs (Kw·D), ddtb (Kw, D).  y and its bound are ss2d_fwd_ref64's, bit for bit.
    delta: as in ss2d_fwd_ref64; the forward and the backward both run on it (ref["delta"] is then the given one, bound 0).
    mistake: one of MISTAKES (kind "cross")."""
    assert mistake is None or (kind == "cross" and mistake in MISTAKES), mistake
    dev = torch.device(device) if device is not None else xc.device
    Bt, Lseq, D = xc.shape
    K, N, Kw = xdbl.shape[2], A.shape[1], dtw.shape[0]
    if mistake == "C_own":   # swap the halves' C columns: the forward then reads each image's own C
        hb = Bt // 2
        xdbl = xdbl.clone()
        xdbl[:, :, :, N:2 * N] = torch.cat([xdbl[hb:, :, :, N:2 * N], xdbl[:hb, :, :, N:2 * N]])
    T = max(t.shape[0] for t in walk_tiles(kind, H, W))
    z = lambda *s: torch.zeros(s, dtype=torch.float64, device=dev)
    ref = dict(delta=z(K, Bt, Lseq + 1, D), hs=torch.full((K, Bt, T, D, N), math.nan, dtype=torch.float64, device=dev),
               dxc=z(Bt, Lseq + 1, D), ddelta=z(K, Bt, Lseq + 1, D), dB=z(Bt, Lseq + 1, K, N), dC=z(Bt, Lseq + 1, K, N), dA=z(Kw * D, N),
               dDs=z(Kw * D), ddtb=z(Kw, D))
    bnd = {k: torch.zeros_like(v) for k, v in ref.items()}
    bnd["hs"].fill_(math.nan)
    dxc_mag = z(Bt, Lseq + 1, D)
    dyp = _pad(dy.detach().to(dev, torch.float64))

    def backward(wk):
        k, bs, nb, m, p, pf, u, Bm, Cm, dl, edl, sig = wk.k, wk.bs, wk.nb, wk.m, wk.p, wk.pf, wk.u, wk.Bm, wk.Cm, wk.dl, wk.edl, wk.sig
        Ak, Dk, absA, slot, P, h0, h_all, e_all = wk.Ak, wk.Dk, wk.absA, wk.slot, wk.P, wk.h0, wk.h_all, wk.e_all
        ws = 1 - wk.kw if mistake == "wset" else wk.kw              # rows the weight set's sums go to
        cdst = bs if mistake == "dC_own" else wk.cs                 # images whose dxdbl C columns receive dC
        b = u.shape[0]
        sh = (b, nb, D, N)
        put = lambda dst, src: dst.index_copy_(1, pf, src.reshape(b, nb * LT, *src.shape[3:]))
        ref["hs"][k, bs, :nb], bnd["hs"][k, bs, :nb] = h0, wk.e0
        put(ref["delta"][k, bs], dl); put(bnd["delta"][k, bs], edl)
        dyk = dyp[bs][:, p]

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
        dB_k, dC_k, edB_k, edC_k = z(b, nb, LT, N), z(b, nb, LT, N), z(b, nb, LT, N), z(b, nb, LT, N)
        dA_k, edA_k, dA_tot, dA_abs = z(D, N), z(*sh), z(*sh), z(*sh)
        gD = _gt(D)
        for s in range(LT - 1, -1, -1):
            a, rho, v, _ = slot(s)
            g = wslot(s) + q
            G = g.abs()
            eg = eq + U * G
            h, eh = h_all[:, :, s], e_all[:, :, s].double()
            hp = h_all[:, :, s - 1] if s > 0 else h0
            Mh, Mp = h.abs(), hp.abs()
            dys, us, ds, es = dyk[:, :, s, :, None], u[:, :, s, :, None], dl[:, :, s, :, None], edl[:, :, s, :, None]
            Bs = Bm[:, :, s, None, :]
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
        put(ref["ddelta"][k, bs], dd_k * m); put(bnd["ddelta"][k, bs], edd_k)
        put(ref["dB"][bs, :, k], dB_k); put(bnd["dB"][bs, :, k], edB_k)
        put(ref["dC"][cdst, :, k], dC_k); put(bnd["dC"][cdst, :, k], edC_k)
        mm = m.expand_as(u).reshape(b, nb * LT, D)
        ref["dxc"][bs].index_add_(1, pf, du_k.reshape(b, nb * LT, D) * mm)
        bnd["dxc"][bs].index_add_(1, pf, edu_k.reshape(b, nb * LT, D) * mm)
        dxc_mag[bs].index_add_(1, pf, dum_k.reshape(b, nb * LT, D) * mm)
        rows = slice(ws * D, (ws + 1) * D)
        ref["dA"][rows] = dA_k
        bnd["dA"][rows] = tile_rss(edA_k) + _acc(dA_tot, dA_abs, Lseq)
        dyu = dyk * u
        ref["dDs"][rows] = dyu.sum((0, 1, 2))
        bnd["dDs"][rows] = U * dyu.abs().sum((0, 1, 2)) + _acc(dyu.sum(2), dyu.abs().sum(2), Lseq)
        dd_k *= m
        ref["ddtb"][ws] = dd_k.sum((0, 1, 2))
        bnd["ddtb"][ws] = tile_rss(edd_k.sum(2)) + _acc(dd_k.sum(2), (dd_k.abs() + edd_k).sum(2), Lseq)

    y, ey = ss2d_fwd_ref64(kind, xc, xdbl, dtw, dtb, A, Ds, H, W, device=dev, on_walk=backward, delta=delta)
    bnd["dxc"] += K * U * dxc_mag
    for key in ("delta", "dxc", "ddelta", "dB", "dC"):
        sl = (slice(None), slice(0, Lseq)) if key in ("dxc", "dB", "dC") else (slice(None), slice(None), slice(0, Lseq))
        ref[key], bnd[key] = ref[key][sl].contiguous(), bnd[key][sl].contiguous()
    for key in bnd:
        bnd[key] = bnd[key] * SAFETY
    ref["y"], bnd["y"] = y, ey
    return ref, bnd
