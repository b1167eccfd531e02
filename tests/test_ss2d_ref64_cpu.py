"""CPU: the fp64 reference of the fused SS2D scan core (oracle/ss2d_ref64.py) that the fused backward's GPU tests compare with.
* its forward y against the C oracle composed per direction (the forward tests' own reference);
* every backward output against torch.autograd in fp64 through a literal restatement of the op (gather, a loop over the walk,
  scatter), to ~1e-12 relative, and `hs` against the restatement's state at every tile start, ragged column tiles included;
* its error bound against an fp32 emulation of the recurrences whose decay factors are perturbed by the ex2.approx bound: the
  emulation must stay inside the bound.  The worst fraction is logged with helpers.record."""
import numpy as np
import pytest
import torch

import procedural as P
from helpers import record
from oracle import ss2d_ref64 as R64

S = 83
SHAPES = [(5, 7), (1, 9), (17, 3)]


def _inputs(kind, B, H, W, D, N, R, tag, wide=False):
    K = 4 if kind == "cross4" else 2
    Lseq = H * W * (2 if kind == "seq2" else 1)
    Cp = 2 * N + R + 3                                                       # 3 padding columns, as the packed x_proj leaves
    xc = P.randn(S, tag + "/xc", (B, Lseq, D))
    xdbl = P.randn(S, tag + "/xdbl", (B, Lseq, K, Cp))
    xdbl[..., 2 * N + R:] = 0.0
    dtw = P.rand(S, tag + "/dtw", (K, D, R), -R ** -0.5, R ** -0.5)
    dt = torch.exp(P.rand(S, tag + "/dt", (K, D), np.log(1e-3), np.log(0.5 if wide else 0.1)))
    dtb = dt + torch.log(-torch.expm1(-dt))                                  # inverse softplus
    A = -torch.arange(1, N + 1, dtype=torch.float32).repeat(K * D, 1) * (P.rand(S, tag + "/A", (K * D, N), 0.8, 4.0 if wide else 1.25))
    Ds = P.randn(S, tag + "/Ds", (K * D,), 0.1, 1.0)
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


@pytest.mark.parametrize("kind", ["cross4", "seq2"])
@pytest.mark.parametrize("H,W", SHAPES)
def test_forward_matches_the_composed_oracle(kind, H, W):
    from test_ss2d_scan_gpu import _reference
    B, D, N, R = 2, 8, 4, 3
    xc, xdbl, dtw, dtb, A, Ds, dy = _inputs(kind, B, H, W, D, N, R, f"f/{kind}/{H}/{W}")
    ref, bnd = R64.ss2d_ref64(kind, xc, xdbl, dtw, dtb, A, Ds, dy, H, W)
    want = torch.from_numpy(_reference(kind, xc, xdbl, dtw, dtb, A, Ds, H, W, N, R)).double()
    err = float((ref["y"] - want).abs().max()) / float(want.abs().max())
    assert err < 2e-5, err                                                   # the C oracle runs in fp32
    assert bool((bnd["y"] > 0).all())


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
