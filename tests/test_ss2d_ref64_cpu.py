"""CPU: the fp64 reference of the fused SS2D scan core (oracle/ss2d_ref64.py) that the fused scan's GPU tests compare with.
* its forward y, all three kinds, against the C oracle composed per direction (the forward tests' own reference), and CROSS
  against the same composition restated in fp64, to 1e-12; the forward entry ss2d_fwd_ref64 is ss2d_ref64's forward bit for bit;
* every backward output, all three kinds, against torch.autograd in fp64 through a literal restatement of the op (per walk a
  gather, a loop over the walk with its weight set and its C images, a scatter), to 1e-12 relative, and `hs` against the
  restatement's state at every tile start, ragged column tiles and CROSS at L > 2048 included;
* the same on a given delta' (delta=, a softplus value rounded to bf16 as the bf16 training mode saves it): the rounded delta' lies
  inside delta_bound_bf16, the bounds lose only the delta' terms, and given the reference's own delta' nothing changes;
* its error bound against an fp32 emulation of the recurrences whose decay factors are perturbed by the ex2.approx bound (forwards
  and backwards run in L-segments whose carried decays come from an fp32 sum of delta' as the summary pass forms them): the
  emulation must stay inside the bound.  The worst fraction is logged with helpers.record;
* three plausible mistakes of the CROSS backward (dC credited to the image's own row, the other weight set's rows for dA / dDs /
  d dt_bias, C read from the image's own half) land outside the bound."""
import numpy as np
import pytest
import torch

import procedural as P
from helpers import record
from oracle import ss2d_ref64 as R64

S = 83              # seeds: the SS2D / ConMB cases,
S_CROSS = 89        # the CROSS backward cases,
S16 = 131           # and the cases drawn as the bf16 training mode's inputs
SHAPES = [(5, 7), (1, 9), (17, 3)]


def _inputs(kind, B, H, W, D, N, R, tag, wide=False, seed=S):
    """B: the batch (for "cross" 2·images); "cross" has one x_dbl row per position and two weight sets (modalities).  Seed S16:
    xc and dy are bf16 values and dt lies in [1e-3, 0.1]"""
    K = R64.KINDS[kind]
    Kw = 2 if kind == "cross" else K
    Lseq = H * W * (2 if kind == "seq2" else 1)
    Cp = 2 * N + R + 3                                                       # 3 padding columns, as the packed x_proj leaves
    bf = (lambda t: t.bfloat16().float()) if seed == S16 else (lambda t: t)
    xc = bf(P.randn(seed, tag + "/xc", (B, Lseq, D)))
    xdbl = P.randn(seed, tag + "/xdbl", (B, Lseq, K, Cp))
    xdbl[..., 2 * N + R:] = 0.0
    dtw = P.rand(seed, tag + "/dtw", (Kw, D, R), -R ** -0.5, R ** -0.5)
    lo, hi = (-6.9, -2.3) if seed == S16 else (np.log(1e-3), np.log(0.5 if wide else 0.1))
    dt = torch.exp(P.rand(seed, tag + "/dt", (Kw, D), lo, hi))
    dtb = dt + torch.log(-torch.expm1(-dt))                                  # inverse softplus
    A = -torch.arange(1, N + 1, dtype=torch.float32).repeat(Kw * D, 1) * (P.rand(seed, tag + "/A", (Kw * D, N), 0.8, 4.0 if wide else 1.25))
    Ds = P.randn(seed, tag + "/Ds", (Kw * D,), 0.1, 1.0)
    dy = bf(P.randn(seed, tag + "/dy", (B, Lseq, D)))
    return xc, xdbl, dtw, dtb, A, Ds, dy


def _tile_starts(tiles):
    """walk step -> index of the tile it starts, for a walk's (ntiles, 16) tile table (its tiles are consecutive in walk order)"""
    steps = np.concatenate([[0], np.cumsum((tiles >= 0).sum(1))])
    return {int(s): j for j, s in enumerate(steps[:-1])}, steps


def _literal(kind, xc, xdbl, dtw, dtb, A, Ds, dy, H, W, delta=None):
    """the op restated: per walk a gather, a loop over the walk (its weight set's parameters, C from its C images), a scatter;
    fp64 autograd.  Also the state entering every walk tile (NaN where a walk has no tile).  delta (K, B, Lseq, D): run on this
    delta' as a leaf instead of the softplus; ddelta is then the gradient at delta' times the softplus derivative 1 - exp(-delta')
    and d dt_bias its sum, as the backward kernel forms them"""
    t = [v.double().clone().requires_grad_(True) for v in (xc, xdbl, dtw, dtb, A, Ds)]
    xc_, xdbl_, dtw_, dtb_, A_, Ds_ = t
    Bt, Lseq, D = xc.shape
    K, N, R = xdbl.shape[2], A.shape[1], dtw.shape[2]
    tiles = R64.walk_tiles(kind, H, W)
    hs = torch.full((K, Bt, max(len(b) for b in tiles), D, N), float("nan"), dtype=torch.float64)
    total, pres = 0.0, []
    for k, bs, kw, cs in R64.walk_groups(kind, Bt):
        idx = R64.dir_index(kind, H, W)[k]
        starts, _ = _tile_starts(tiles[k])
        u, xk = xc_[bs][:, idx], xdbl_[bs][:, idx, k]
        if delta is None:
            pre = xk[..., 2 * N:2 * N + R] @ dtw_[kw].t() + dtb_[kw]
            pre.retain_grad()
            dl = torch.nn.functional.softplus(pre)
        else:
            dl = pre = delta[k, bs][:, idx].double().clone().requires_grad_(True)
        Ak, Dk = A_[kw * D:(kw + 1) * D], Ds_[kw * D:(kw + 1) * D]
        Cm = xdbl_[cs][:, idx, k, N:2 * N]
        h = torch.zeros(u.shape[0], D, N, dtype=torch.float64)
        ys = []
        for l in range(Lseq):
            if l in starts:
                hs[k, bs, starts[l]] = h.detach()
            h = torch.exp(dl[:, l, :, None] * Ak) * h + (dl[:, l] * u[:, l])[..., None] * xk[:, l, None, :N]
            ys.append((h * Cm[:, l, None, :]).sum(-1) + Dk * u[:, l])
        total = total + (torch.stack(ys, 1) * dy.double()[bs][:, idx]).sum()
        pres.append((k, bs, kw, idx, pre))
    total.backward()
    ddelta = torch.zeros(K, Bt, Lseq, D, dtype=torch.float64)
    ddtb = torch.zeros(dtb.shape, dtype=torch.float64)
    for k, bs, kw, idx, pre in pres:
        gd = pre.grad if delta is None else pre.grad * -torch.expm1(-pre.detach())
        ddelta[k, bs][:, idx] = gd
        ddtb[kw] += gd.sum((0, 1))
    g = xdbl_.grad
    return dict(dxc=xc_.grad, ddelta=ddelta, dB=g[..., :N], dC=g[..., N:2 * N], dA=A_.grad, dDs=Ds_.grad,
                ddtb=dtb_.grad if delta is None else ddtb), hs


def _matches_autograd(kind, args, H, W, delta=None):
    """ss2d_ref64 against _literal: every output to 1e-12 of its scale, and each direction's hs (NaN exactly in the blocks its
    walk does not reach)"""
    ref, bnd = R64.ss2d_ref64(kind, *args, H, W, delta=delta)
    want, hs = _literal(kind, *args, H, W, delta=delta)
    for name, w in want.items():
        err = float((ref[name] - w).abs().max()) / float(w.abs().max())
        assert err < 1e-12, f"{name}: {err:.2e}"
    for k, hk in enumerate(hs):
        ok = ~hk.isnan()
        assert torch.equal(ref["hs"][k].isnan(), ~ok), f"hs, direction {k}"
        assert float((ref["hs"][k][ok] - hk[ok]).abs().max()) <= 1e-12 * float(hk[ok].abs().max()), f"hs, direction {k}"
    return ref, bnd


@pytest.mark.parametrize("kind", ["cross4", "seq2", "cross"])
@pytest.mark.parametrize("H,W", SHAPES)
def test_forward_matches_the_composed_oracle(kind, H, W):
    from test_ss2d_scan_gpu import _reference
    B, D, N, R = 2, 8, 4, 3
    xc, xdbl, dtw, dtb, A, Ds, dy = _inputs(kind, B, H, W, D, N, R, f"f/{kind}/{H}/{W}")
    y, bnd = R64.ss2d_fwd_ref64(kind, xc, xdbl, dtw, dtb, A, Ds, H, W)
    want = torch.from_numpy(_reference(kind, xc, xdbl, dtw, dtb, A, Ds, H, W, N, R)).double()
    err = float((y - want).abs().max()) / float(want.abs().max())
    assert err < 2e-5, err                                                   # the C oracle runs in fp32
    assert bool((bnd > 0).all())


def _scan64(u, dl, A, Bm, Cm, Ds):
    """one selective scan in fp64, step by step: u, dl (b, L, D), A (D, N), Bm, Cm (b, L, N), Ds (D)"""
    h = torch.zeros(u.shape[0], u.shape[2], A.shape[1], dtype=torch.float64)
    ys = []
    for l in range(u.shape[1]):
        h = torch.exp(dl[:, l, :, None] * A) * h + (dl[:, l] * u[:, l])[..., None] * Bm[:, l, None, :]
        ys.append((h * Cm[:, l, None, :]).sum(-1) + Ds * u[:, l])
    return torch.stack(ys, 1)


@pytest.mark.parametrize("H,W", SHAPES + [(40, 3)])
@pytest.mark.parametrize("N", [4, 16])
def test_cross_matches_the_composition_in_fp64(H, W, N):
    """CROSS composed as the C oracle's test composes it (test_ss2d_scan_gpu._reference): each modality's half of the batch runs
    one row-major scan with its own weights and B, and the other half's C.  Restated in fp64, the reference must agree to 1e-12."""
    Bt, D, R = 4, 8, 3
    xc, xdbl, dtw, dtb, A, Ds, _ = _inputs("cross", Bt, H, W, D, N, R, f"c/{H}/{W}/{N}")
    y, _ = R64.ss2d_fwd_ref64("cross", xc, xdbl, dtw, dtb, A, Ds, H, W)
    x64, d64 = xc.double(), xdbl.double()
    want = torch.empty(1, Bt, H * W, D, dtype=torch.float64)
    h = Bt // 2
    for m in range(2):
        sl, osl = slice(m * h, (m + 1) * h), slice((1 - m) * h, (2 - m) * h)
        dl = torch.nn.functional.softplus(d64[sl, :, 0, 2 * N:2 * N + R] @ dtw[m].double().t() + dtb[m].double())
        want[0, sl] = _scan64(x64[sl], dl, A[m * D:(m + 1) * D].double(), d64[sl, :, 0, :N], d64[osl, :, 0, N:2 * N],
                              Ds[m * D:(m + 1) * D].double())
    err = float((y - want).abs().max()) / float(want.abs().max())
    assert err < 1e-12, err


@pytest.mark.parametrize("kind,H,W,N", [("cross4", 17, 3, 16), ("seq2", 5, 7, 4), ("cross4", 5, 7, 4)])
def test_forward_entry_is_the_training_reference_forward(kind, H, W, N):
    """ss2d_fwd_ref64 is ss2d_ref64's forward: y and its bound bit for bit"""
    args = _inputs(kind, 2, H, W, 8, N, 3, f"e/{kind}/{H}/{W}/{N}")
    ref, bnd = R64.ss2d_ref64(kind, *args, H, W)
    y, by = R64.ss2d_fwd_ref64(kind, *args[:6], H, W)
    assert torch.equal(y, ref["y"]) and torch.equal(by, bnd["y"])


@pytest.mark.parametrize("kind", ["cross4", "seq2"])
@pytest.mark.parametrize("H,W", SHAPES)
@pytest.mark.parametrize("N", [4, 16])
def test_backward_and_states_match_autograd(kind, H, W, N):
    B, D, R = 2, 8, 3
    _matches_autograd(kind, _inputs(kind, B, H, W, D, N, R, f"b/{kind}/{H}/{W}/{N}"), H, W)
    if kind == "cross4" and H % 16:
        assert len(R64.walk_tiles(kind, H, W)[1]) == W * -(-H // 16)              # ragged column tiles were among them


@pytest.mark.parametrize("H,W,N,Bt", [(5, 7, 4, 2), (9, 11, 4, 4), (9, 11, 16, 2), (1, 9, 16, 4), (42, 50, 4, 2)])
def test_cross_backward_and_states_match_autograd(H, W, N, Bt):
    """CroMB's two scans: each modality's half with its own weights and B, C from the other half; ragged maps and L > 2048"""
    D, R = 8 if H * W < 2048 else 4, 3
    args = _inputs("cross", Bt, H, W, D, N, R, f"b/{H}/{W}/{N}/{Bt}", seed=S_CROSS)
    ref, bnd = _matches_autograd("cross", args, H, W)
    y, by = R64.ss2d_fwd_ref64("cross", *args[:6], H, W)                  # the forward is the forward entry's, bit for bit
    assert torch.equal(y, ref["y"]) and torch.equal(by, bnd["y"])


# kind, batch, H, W, d_state, seed, tag
GIVEN = [("cross4", 2, 5, 7, 16, S16, "bf16train/cross4/5x7/N16"), ("seq2", 2, 5, 7, 4, S16, "bf16train/seq2/5x7/N4"),
         ("cross4", 2, 17, 3, 4, S16, "bf16train/cross4/17x3/N4"), ("cross", 2, 5, 7, 4, S_CROSS, "d/5/7/4/2"),
         ("cross", 4, 9, 11, 16, S_CROSS, "d/9/11/16/4")]


@pytest.mark.parametrize("kind,B,H,W,N,seed,tag", GIVEN, ids=[f"{c[0]}-{c[1]}-{c[2]}-{c[3]}-{c[4]}" for c in GIVEN])
def test_given_delta_matches_autograd(kind, B, H, W, N, seed, tag):
    _given_delta(kind, B, H, W, N, seed, tag)


def test_given_own_delta_changes_nothing():
    _given_delta("cross4", 2, 5, 7, 4, S16, "bf16train/self")


def _given_delta(kind, B, H, W, N, seed, tag):
    """delta=: the reference's delta' rounded to bf16 (through fp32, as the bf16 training mode stores it) lies inside the bound the
    GPU tests hold the kernel's delta' to; run on it, every output matches the literal loop on the same delta', ref["delta"] is the
    given one with bound 0, and the bounds only lose the delta' error terms.  Given the reference's own fp64 delta', nothing changes."""
    args = _inputs(kind, B, H, W, 8, N, 3, tag, seed=seed)
    plain, pb = R64.ss2d_ref64(kind, *args, H, W)
    given = plain["delta"].float().bfloat16().double()
    assert R64.bound_fraction(given, plain["delta"], R64.delta_bound_bf16(plain["delta"], pb["delta"])) <= 1.0
    assert float((given - plain["delta"]).abs().max()) > 0                        # and the rounding is really there
    ref, bnd = _matches_autograd(kind, args, H, W, delta=given)
    assert torch.equal(ref["delta"], given) and not bool(bnd["delta"].any())
    for key in ("y", "dxc", "ddelta", "dA"):
        assert bool((bnd[key] >= 0).all()) and float(bnd[key].max()) <= 1.5 * float(pb[key].max()), key
    same, _ = R64.ss2d_ref64(kind, *args, H, W, delta=plain["delta"])
    for name in ("y", "dxc", "ddelta", "dB", "dC", "dA", "dDs", "ddtb"):
        err = float((same[name] - plain[name]).abs().max()) / float(plain[name].abs().max())
        assert err < 1e-12, f"{name}: {err:.2e}"


def _emulate32(kind, xc, xdbl, dtw, dtb, A, Ds, dy, H, W, seed, nseg=1):
    """fp32 emulation of the kernels' recurrences over every walk, each decay factor perturbed by a seeded ±E2 relative error.
    nseg > 1 cuts the forward into L-segments of ceil(longest walk's tiles / nseg) 16-position tiles: a summary pass per segment
    from a zero state whose carried decay is ex2(a2 · the fp32 sum of the segment's delta') (also perturbed), the combine's chain,
    then every step from the segments' start states"""
    f = lambda t: t.numpy().astype(np.float32)
    xc, xdbl, dtw, dtb, A, Ds, dy = map(f, (xc, xdbl, dtw, dtb, A, Ds, dy))
    f32 = np.float32
    rng = np.random.default_rng(seed)
    pert = lambda shape: (1 + f32(R64.E2) * rng.choice([-1, 1], shape)).astype(f32)
    Bt, Lseq, D = xc.shape
    K, N, R, Kw = xdbl.shape[2], A.shape[1], dtw.shape[2], dtw.shape[0]
    out = dict(y=np.zeros((K, Bt, Lseq, D), f32), delta=np.zeros((K, Bt, Lseq, D), f32), dxc=np.zeros((Bt, Lseq, D), f32),
               ddelta=np.zeros((K, Bt, Lseq, D), f32), dB=np.zeros((Bt, Lseq, K, N), f32), dC=np.zeros((Bt, Lseq, K, N), f32),
               dA=np.zeros((Kw * D, N), f32), dDs=np.zeros(Kw * D, f32), ddtb=np.zeros((Kw, D), f32))
    tiles = R64.walk_tiles(kind, H, W)
    out["hs"] = np.full((K, Bt, max(len(t) for t in tiles), D, N), np.nan, f32)
    tps = -(-max(len(t) for t in tiles) // nseg)
    for k, bs, kw, cs in R64.walk_groups(kind, Bt):
        idx = R64.dir_index(kind, H, W)[k]
        starts, steps = _tile_starts(tiles[k])
        nt = len(tiles[k])
        segs = [(steps[s * tps], steps[min((s + 1) * tps, nt)]) for s in range(nseg) if s * tps < nt]
        Ak, Dk = A[kw * D:(kw + 1) * D], Ds[kw * D:(kw + 1) * D]
        a2 = (Ak * f32(1.4426950408889634)).astype(f32)
        pre = (xdbl[bs][:, idx, k, 2 * N:2 * N + R] @ dtw[kw].T + dtb[kw]).astype(f32)
        dl = np.logaddexp(f32(0), pre).astype(f32)
        u, Bm, Cm, dyk = xc[bs][:, idx], xdbl[bs][:, idx, k, :N], xdbl[cs][:, idx, k, N:2 * N], dy[bs][:, idx]
        b = u.shape[0]
        dec = np.exp2(dl[..., None] * a2).astype(f32) * pert((b, Lseq, D, N))
        # summary pass (with more than one segment): each segment from a zero state, its end state and carried decay; combine
        h0s, cur = [np.zeros((b, D, N), f32)], np.zeros((b, D, N), f32)
        if len(segs) > 1:
            h0s = []
            for lo, hi in segs:
                h0s.append(cur)
                h = np.zeros((b, D, N), f32)
                for l in range(lo, hi):
                    h = dec[:, l] * h + (dl[:, l] * u[:, l])[..., None] * Bm[:, l, None, :]
                carry = np.exp2(dl[:, lo:hi].sum(1, dtype=f32)[..., None] * a2).astype(f32) * pert((b, D, N))
                cur = (carry * cur + h).astype(f32)
        hsave = np.zeros((b, Lseq, D, N), f32)
        for (lo, hi), h in zip(segs, h0s):
            for l in range(lo, hi):
                if l in starts:
                    out["hs"][k, bs, starts[l]] = h
                h = dec[:, l] * h + (dl[:, l] * u[:, l])[..., None] * Bm[:, l, None, :]
                hsave[:, l] = h
                out["y"][k, bs, idx[l]] = (h * Cm[:, l, None, :]).sum(-1, dtype=f32) + Dk * u[:, l]
        out["delta"][k, bs][:, idx] = dl
        dh = np.zeros((b, D, N), f32)
        for l in range(Lseq - 1, -1, -1):
            p = idx[l]
            dhn = dyk[:, l, :, None] * Cm[:, l, None, :] + dh
            hp = hsave[:, l - 1] if l > 0 else np.zeros_like(dh)
            ah = dec[:, l] * hp
            s1 = (dhn * Bm[:, l, None, :]).sum(-1, dtype=f32)
            s2 = (dhn * ah * Ak).sum(-1, dtype=f32)
            out["dC"][cs, p, k] = (dyk[:, l, :, None] * hsave[:, l]).sum(1, dtype=f32)
            out["dB"][bs, p, k] = (dhn * (dl[:, l] * u[:, l])[..., None]).sum(1, dtype=f32)
            out["dxc"][bs, p] += dyk[:, l] * Dk + dl[:, l] * s1
            dd = (1 - np.exp(-dl[:, l])).astype(f32) * (u[:, l] * s1 + s2)
            out["ddelta"][k, bs, p] = dd
            out["dA"][kw * D:(kw + 1) * D] += (dhn * ah * dl[:, l, :, None]).sum(0, dtype=f32)
            out["dDs"][kw * D:(kw + 1) * D] += (dyk[:, l] * u[:, l]).sum(0, dtype=f32)
            out["ddtb"][kw] += dd.sum(0, dtype=f32)
            dh = (dhn * dec[:, l]).astype(f32)
    return out


def _covers_emulation(kind, args, H, W, tag, nseg=1, maxnorm=()):
    """the bound covers _emulate32 element by element, and at each tensor's largest element it is no looser than 1e-3 of the
    tensor's scale; the tensors in `maxnorm` meet that bar in the max norm instead"""
    ref, bnd = R64.ss2d_ref64(kind, *args, H, W)
    emu = _emulate32(kind, *args, H, W, seed=len(tag), nseg=nseg)
    worst = {}
    for name, v in emu.items():
        v = torch.from_numpy(v).double()
        ok = ~ref[name].isnan()
        r, b = ref[name][ok], bnd[name][ok]
        frac = R64.bound_fraction(v[ok], r, b)
        worst[name] = frac
        assert frac <= 1.0, f"{name}: {frac:.3f} of the bound"
        if name in maxnorm:
            assert float((v[ok] - r).abs().max()) <= 1e-3 * float(r.abs().max()), name
        else:
            assert float(b[int(r.abs().argmax())]) <= 1e-3 * float(r.abs().max()), name
    record(f"ss2d_ref64 bound self-check {tag}", **worst)


@pytest.mark.parametrize("kind,H,W,N,wide", [("cross4", 17, 3, 16, False), ("cross4", 5, 7, 4, True), ("seq2", 5, 7, 4, False),
                                             ("seq2", 1, 9, 16, True)])
def test_bound_covers_an_fp32_emulation(kind, H, W, N, wide):
    B, D, R = 2, 16, 6
    tag = f"e/{kind}/{H}/{W}/{N}/{wide}"
    _covers_emulation(kind, _inputs(kind, B, H, W, D, N, R, tag, wide), H, W, tag)


@pytest.mark.parametrize("H,W,N,Bt,wide,nseg", [(9, 11, 4, 4, False, 1), (9, 11, 4, 2, True, 3), (17, 20, 16, 2, False, 7),
                                                (5, 7, 4, 6, False, 2)])
def test_cross_bound_covers_an_fp32_emulation(H, W, N, Bt, wide, nseg):
    """CROSS, its forward in L-segments; d dt_bias sums ddelta's bounds over all positions, so there (as in the GPU tests) the
    max-norm bar is checked instead"""
    D, R = 16, 6
    tag = f"e/{H}/{W}/{N}/{Bt}/{wide}/{nseg}"
    _covers_emulation("cross", _inputs("cross", Bt, H, W, D, N, R, tag, wide, seed=S_CROSS), H, W, tag, nseg, maxnorm=("ddtb",))


@pytest.mark.parametrize("mistake", R64.MISTAKES)
def test_plausible_mistakes_land_outside_the_bound(mistake):
    H, W, N, Bt, D, R = 9, 11, 4, 4, 16, 6
    args = _inputs("cross", Bt, H, W, D, N, R, "m", seed=S_CROSS)
    ref, bnd = R64.ss2d_ref64("cross", *args, H, W)
    bad, _ = R64.ss2d_ref64("cross", *args, H, W, mistake=mistake)
    fracs = {k: R64.bound_fraction(bad[k], ref[k], bnd[k]) for k in ("dxc", "ddelta", "dB", "dC", "dA", "dDs", "ddtb")}
    assert max(fracs.values()) > 100.0, fracs
    want = {"dC_own": "dC", "wset": "dA", "C_own": "dxc"}[mistake]
    assert fracs[want] > 100.0, fracs


def _emulate32_fwd(kind, xc, xdbl, dtw, dtb, A, Ds, H, W, seed, nseg=1):
    """fp32 emulation of the inference forward, each decay factor perturbed by a seeded ±E2 relative error.  nseg > 1 runs it as the
    kernels run L-segments: the walk cut into the kernel's LT-position tiles (32 at d_state 4, 16 at 16), tiles_per_split =
    ceil(longest walk's tiles / segments) for every direction; a summary pass per segment from a zero state that also sums delta'
    in fp32 and forms the carried decay ex2(a2·sum) (perturbed like every ex2), the combine's fp32 chain over the segments, and
    the apply pass from the carried state."""
    f = lambda t: t.numpy().astype(np.float32)
    xc, xdbl, dtw, dtb, A, Ds = map(f, (xc, xdbl, dtw, dtb, A, Ds))
    rng = np.random.default_rng(seed)
    f32 = np.float32
    Bt, Lseq, D = xc.shape
    K, N, R = xdbl.shape[2], A.shape[1], dtw.shape[2]
    lt = 16 if N >= 16 else 32
    tiles = R64.walk_tiles(kind, H, W, lt)
    max_tiles = max(len(t) for t in tiles)
    nsplit = min(nseg, 32, max_tiles)
    tps = -(-max_tiles // nsplit)
    y = np.zeros((K, Bt, Lseq, D), f32)
    pm = lambda *s: (1 + f32(R64.E2) * rng.choice([-1, 1], s)).astype(f32)
    for k, bs, kw, cs in R64.walk_groups(kind, Bt):
        a2 = (A[kw * D:(kw + 1) * D] * f32(1.4426950408889634)).astype(f32)
        Dk = Ds[kw * D:(kw + 1) * D]
        segs = [t[t >= 0] for t in (tiles[k][s * tps:(s + 1) * tps].reshape(-1) for s in range(nsplit))]
        idx = np.concatenate(segs)
        pre = (xdbl[bs][:, idx, k, 2 * N:2 * N + R] @ dtw[kw].T + dtb[kw]).astype(f32)
        dl = np.logaddexp(f32(0), pre).astype(f32)
        u, Bm, Cm = xc[bs][:, idx], xdbl[bs][:, idx, k, :N], xdbl[cs][:, idx, k, N:2 * N]
        b = u.shape[0]
        dec = np.exp2((dl[..., None] * a2).astype(f32)).astype(f32) * pm(b, len(idx), D, N)

        def walk(h, l0, l1, out):
            for l in range(l0, l1):
                h = (dec[:, l] * h + (dl[:, l] * u[:, l])[..., None] * Bm[:, l, None, :]).astype(f32)
                if out:
                    y[k, bs, idx[l]] = (h * Cm[:, l, None, :]).sum(-1, dtype=f32) + Dk * u[:, l]
            return h

        ends = np.cumsum([0] + [len(s) for s in segs])
        carry = np.zeros((b, D, N), f32)
        for s in range(nsplit):
            l0, l1 = ends[s], ends[s + 1]
            walk(carry, l0, l1, True)                                        # the apply pass (a serial walk when nsplit = 1)
            if s + 1 < nsplit:                                               # summary, then one step of the combine's chain
                hl = walk(np.zeros((b, D, N), f32), l0, l1, False)
                sdl = np.zeros((b, D), f32)
                for l in range(l0, l1):
                    sdl = (sdl + dl[:, l]).astype(f32)
                P = np.exp2((a2 * sdl[..., None]).astype(f32)).astype(f32) * pm(b, D, N)
                carry = (P * carry + hl).astype(f32)
    return y


@pytest.mark.parametrize("kind,B,H,W,N,wide,nseg", [
    ("cross", 4, 5, 7, 4, False, 1), ("cross", 2, 17, 3, 16, True, 1), ("cross", 2, 9, 11, 16, False, 1),
    ("cross", 2, 32, 33, 4, True, 32), ("cross4", 2, 33, 32, 4, False, 32), ("cross4", 2, 33, 32, 4, True, 32),
    ("seq2", 2, 16, 32, 16, False, 32), ("cross4", 2, 16, 18, 16, True, 32)])
def test_bound_covers_an_fp32_forward_emulation(kind, B, H, W, N, wide, nseg):
    """the forward bound (ss2d_fwd_ref64) against the fp32 emulation: CROSS, and 32 L-segments whose carries come from the fp32
    delta' sum as the summary pass forms them (the 33 x 32 map's row walk ends in empty segments)"""
    D, R = 16, 6
    tag = f"fe/{kind}/{B}/{H}/{W}/{N}/{wide}/{nseg}"
    args = _inputs(kind, B, H, W, D, N, R, tag, wide)[:6]
    y, bnd = R64.ss2d_fwd_ref64(kind, *args, H, W)
    emu = torch.from_numpy(_emulate32_fwd(kind, *args, H, W, seed=len(tag), nseg=nseg)).double()
    frac = R64.bound_fraction(emu, y, bnd)
    record(f"ss2d_ref64 forward bound self-check {tag}", y=frac)
    assert frac <= 1.0, f"{frac:.3f} of the bound"
    i = int(y.abs().argmax())
    assert float(bnd.reshape(-1)[i]) <= 1e-3 * float(y.abs().max())
