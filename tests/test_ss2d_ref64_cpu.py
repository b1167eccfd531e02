"""CPU: the fp64 reference of the fused SS2D scan core (oracle/ss2d_ref64.py) that the fused scan's GPU tests compare with.
* its forward y, all three kinds, against the C oracle composed per direction (the forward tests' own reference), and CROSS
  against the same composition restated in fp64, to 1e-12; the forward entry ss2d_fwd_ref64 is ss2d_ref64's forward bit for bit;
* every backward output against torch.autograd in fp64 through a literal restatement of the op (gather, a loop over the walk,
  scatter), to ~1e-12 relative, and `hs` against the restatement's state at every tile start, ragged column tiles included;
* its error bound against an fp32 emulation of the recurrences whose decay factors are perturbed by the ex2.approx bound (CROSS
  included, and a forward run in 32 L-segments whose carried decays come from an fp32 sum of delta' as the summary pass forms
  them): the emulation must stay inside the bound.  The worst fraction is logged with helpers.record."""
import numpy as np
import pytest
import torch

import procedural as P
from helpers import record
from oracle import ss2d_ref64 as R64

S = 83
SHAPES = [(5, 7), (1, 9), (17, 3)]


def _inputs(kind, B, H, W, D, N, R, tag, wide=False):
    """B: the batch (for "cross" 2·images); "cross" has one x_dbl row per position and two weight sets (modalities)"""
    K = R64.KINDS[kind]
    Kw = 2 if kind == "cross" else K
    Lseq = H * W * (2 if kind == "seq2" else 1)
    Cp = 2 * N + R + 3                                                       # 3 padding columns, as the packed x_proj leaves
    xc = P.randn(S, tag + "/xc", (B, Lseq, D))
    xdbl = P.randn(S, tag + "/xdbl", (B, Lseq, K, Cp))
    xdbl[..., 2 * N + R:] = 0.0
    dtw = P.rand(S, tag + "/dtw", (Kw, D, R), -R ** -0.5, R ** -0.5)
    dt = torch.exp(P.rand(S, tag + "/dt", (Kw, D), np.log(1e-3), np.log(0.5 if wide else 0.1)))
    dtb = dt + torch.log(-torch.expm1(-dt))                                  # inverse softplus
    A = -torch.arange(1, N + 1, dtype=torch.float32).repeat(Kw * D, 1) * (P.rand(S, tag + "/A", (Kw * D, N), 0.8, 4.0 if wide else 1.25))
    Ds = P.randn(S, tag + "/Ds", (Kw * D,), 0.1, 1.0)
    dy = P.randn(S, tag + "/dy", (B, Lseq, D))
    return xc, xdbl, dtw, dtb, A, Ds, dy


def _literal(kind, xc, xdbl, dtw, dtb, A, Ds, dy, H, W):
    """the op restated: per direction gather, walk, scatter; fp64 autograd.  Also the state entering every walk tile."""
    t = [v.double().clone().requires_grad_(True) for v in (xc, xdbl, dtw, dtb, A, Ds)]
    xc_, xdbl_, dtw_, dtb_, A_, Ds_ = t
    Bt, Lseq, D = xc.shape
    N, R = A.shape[1], dtw.shape[2]
    tiles = R64.walk_tiles(kind, H, W)
    total, pres, hs = 0.0, [], []
    for k, idx in enumerate(R64.dir_index(kind, H, W)):
        step_of = np.empty(Lseq, np.int64)
        step_of[idx] = np.arange(Lseq)
        starts = {int(step_of[b[0]]): j for j, b in enumerate(tiles[k])}
        u, xk = xc_[:, idx], xdbl_[:, idx, k]
        pre = xk[..., 2 * N:2 * N + R] @ dtw_[k].t() + dtb_[k]
        pre.retain_grad()
        dl = torch.nn.functional.softplus(pre)
        Ak, Dk = A_[k * D:(k + 1) * D], Ds_[k * D:(k + 1) * D]
        h = torch.zeros(Bt, D, N, dtype=torch.float64)
        ys, hk = [], torch.full((Bt, len(tiles[k]), D, N), float("nan"), dtype=torch.float64)
        for l in range(Lseq):
            if l in starts:
                hk[:, starts[l]] = h.detach()
            h = torch.exp(dl[:, l, :, None] * Ak) * h + (dl[:, l] * u[:, l])[..., None] * xk[:, l, None, :N]
            ys.append((h * xk[:, l, None, N:2 * N]).sum(-1) + Dk * u[:, l])
        total = total + (torch.stack(ys, 1) * dy.double()[:, idx]).sum()
        pres.append((idx, pre))
        hs.append(hk)
    total.backward()
    ddelta = torch.zeros(len(pres), Bt, Lseq, D, dtype=torch.float64)
    for k, (idx, pre) in enumerate(pres):
        ddelta[k][:, idx] = pre.grad
    g = xdbl_.grad
    return dict(dxc=xc_.grad, ddelta=ddelta, dB=g[..., :N], dC=g[..., N:2 * N], dA=A_.grad, dDs=Ds_.grad, ddtb=dtb_.grad), hs


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
    xc, xdbl, dtw, dtb, A, Ds, dy = _inputs(kind, B, H, W, D, N, R, f"b/{kind}/{H}/{W}/{N}")
    ref, _ = R64.ss2d_ref64(kind, xc, xdbl, dtw, dtb, A, Ds, dy, H, W)
    want, hs = _literal(kind, xc, xdbl, dtw, dtb, A, Ds, dy, H, W)
    for name, w in want.items():
        err = float((ref[name] - w).abs().max()) / float(w.abs().max())
        assert err < 1e-12, f"{name}: {err:.2e}"
    for k, hk in enumerate(hs):
        got = ref["hs"][k, :, :hk.shape[1]]
        assert float((got - hk).abs().max()) <= 1e-12 * float(hk.abs().max()), f"hs, direction {k}"
        assert bool(ref["hs"][k, :, hk.shape[1]:].isnan().all())             # blocks this walk does not reach
    if kind == "cross4" and H % 16:
        assert hs[1].shape[1] == W * -(-H // 16)                                 # ragged column tiles were among them


def _emulate32(kind, xc, xdbl, dtw, dtb, A, Ds, dy, H, W, seed):
    """fp32 emulation of the kernels' recurrences, each decay factor perturbed by a seeded ±E2 relative error"""
    f = lambda t: t.numpy().astype(np.float32)
    xc, xdbl, dtw, dtb, A, Ds, dy = map(f, (xc, xdbl, dtw, dtb, A, Ds, dy))
    rng = np.random.default_rng(seed)
    Bt, Lseq, D = xc.shape
    K, N, R = xdbl.shape[2], A.shape[1], dtw.shape[2]
    f32 = np.float32
    out = dict(y=np.zeros((K, Bt, Lseq, D), f32), delta=np.zeros((K, Bt, Lseq, D), f32), dxc=np.zeros((Bt, Lseq, D), f32),
               ddelta=np.zeros((K, Bt, Lseq, D), f32), dB=np.zeros((Bt, Lseq, K, N), f32), dC=np.zeros((Bt, Lseq, K, N), f32),
               dA=np.zeros((K * D, N), f32), dDs=np.zeros(K * D, f32), ddtb=np.zeros((K, D), f32))
    tiles = R64.walk_tiles(kind, H, W)
    out["hs"] = np.full((K, Bt, max(len(t) for t in tiles), D, N), np.nan, f32)
    for k, idx in enumerate(R64.dir_index(kind, H, W)):
        step_of = np.empty(Lseq, np.int64)
        step_of[idx] = np.arange(Lseq)
        starts = {int(step_of[b[0]]): j for j, b in enumerate(tiles[k])}
        a2 = (A[k * D:(k + 1) * D] * f32(1.4426950408889634)).astype(f32)
        Dk = Ds[k * D:(k + 1) * D]
        pre = (xdbl[:, idx, k, 2 * N:2 * N + R] @ dtw[k].T + dtb[k]).astype(f32)
        dl = np.logaddexp(f32(0), pre).astype(f32)
        u, Bm, Cm, dyk = xc[:, idx], xdbl[:, idx, k, :N], xdbl[:, idx, k, N:2 * N], dy[:, idx]
        dec = np.exp2(dl[..., None] * a2).astype(f32) * (1 + f32(R64.E2) * rng.choice([-1, 1], (Bt, Lseq, D, N))).astype(f32)
        hsave = np.zeros((Bt, Lseq, D, N), f32)
        h = np.zeros((Bt, D, N), f32)
        for l in range(Lseq):
            if l in starts:
                out["hs"][k, :, starts[l]] = h
            h = dec[:, l] * h + (dl[:, l] * u[:, l])[..., None] * Bm[:, l, None, :]
            hsave[:, l] = h
            out["y"][k][:, idx[l]] = (h * Cm[:, l, None, :]).sum(-1, dtype=f32) + Dk * u[:, l]
        out["delta"][k][:, idx] = dl
        dh = np.zeros((Bt, D, N), f32)
        for l in range(Lseq - 1, -1, -1):
            p = idx[l]
            dhn = dyk[:, l, :, None] * Cm[:, l, None, :] + dh
            hp = hsave[:, l - 1] if l > 0 else np.zeros_like(h)
            ah = dec[:, l] * hp
            s1 = (dhn * Bm[:, l, None, :]).sum(-1, dtype=f32)
            s2 = (dhn * ah * A[k * D:(k + 1) * D]).sum(-1, dtype=f32)
            out["dC"][:, p, k] = (dyk[:, l, :, None] * hsave[:, l]).sum(1, dtype=f32)
            out["dB"][:, p, k] = (dhn * (dl[:, l] * u[:, l])[..., None]).sum(1, dtype=f32)
            out["dxc"][:, p] += dyk[:, l] * Dk + dl[:, l] * s1
            sig = (1 - np.exp(-dl[:, l])).astype(f32)
            dd = sig * (u[:, l] * s1 + s2)
            out["ddelta"][k][:, p] = dd
            out["dA"][k * D:(k + 1) * D] += (dhn * ah * dl[:, l, :, None]).sum(0, dtype=f32)
            out["dDs"][k * D:(k + 1) * D] += (dyk[:, l] * u[:, l]).sum(0, dtype=f32)
            out["ddtb"][k] += dd.sum(0, dtype=f32)
            dh = (dhn * dec[:, l]).astype(f32)
    return out


@pytest.mark.parametrize("kind,H,W,N,wide", [("cross4", 17, 3, 16, False), ("cross4", 5, 7, 4, True), ("seq2", 5, 7, 4, False),
                                             ("seq2", 1, 9, 16, True)])
def test_bound_covers_an_fp32_emulation(kind, H, W, N, wide):
    B, D, R = 2, 16, 6
    tag = f"e/{kind}/{H}/{W}/{N}/{wide}"
    args = _inputs(kind, B, H, W, D, N, R, tag, wide)
    ref, bnd = R64.ss2d_ref64(kind, *args, H, W)
    emu = _emulate32(kind, *args, H, W, seed=len(tag))
    worst = {}
    for name, v in emu.items():
        v = torch.from_numpy(v).double()
        ok = ~ref[name].isnan()
        frac = R64.bound_fraction(v[ok], ref[name][ok], bnd[name][ok])
        worst[name] = frac
        assert frac <= 1.0, f"{name}: {frac:.3f} of the bound"
        # per element, yet no looser than 1e-3 of the tensor's scale at its largest element
        i = int(ref[name][ok].abs().argmax())
        assert float(bnd[name][ok][i]) <= 1e-3 * float(ref[name][ok].abs().max()), name
    record(f"ss2d_ref64 bound self-check {tag}", **worst)


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
