"""CPU: the fp64 reference of the op-level selective scan (oracle/scan_ref64.py) that the op scan's fp64 GPU tests compare with.
* its out against the C oracle (which accumulates in double) on small ragged shapes: L not a multiple of 16 / 32, groups,
  d_state 4 / 8 / 16, Sigma's parameters and the reference test's, at fp32-rounding level;
* every gradient and the chunk states `x` against torch.autograd in fp64 through a literal loop-over-L restatement of the op, to
  ~1e-12 relative: L crossing 2048 (three chunks of `x`), and D / delta_bias / softplus off;
* its error bound against an fp32 emulation of the kernels whose decay factors and ex2 calls are perturbed by the ex2.approx bound,
  with a forward run in L-segments whose carries come from an fp32 sum of delta' as the summary pass forms them: the emulation must
  stay inside the bound, Sigma's parameters and a widened set.  Worst fractions go to helpers.record."""
import math

import numpy as np
import pytest
import torch

from helpers import op_scan_params, record
from oracle import scan_oracle
from oracle import scan_ref64 as R

S = 89
LOG2E = 1.4426950408889634


@pytest.mark.parametrize("b,dim,L,N,G,dist", [(2, 8, 37, 4, 1, "sigma"), (1, 12, 75, 8, 3, "sigma"), (2, 8, 50, 16, 2, "wide"),
                                              (2, 6, 97, 16, 1, "ref")])
def test_out_matches_the_c_oracle(b, dim, L, N, G, dist):
    u, delta, A, B, C, D, bias, _ = op_scan_params(S, b, dim, L, N, G, f"o/{b}/{dim}/{L}/{N}/{G}/{dist}", dist)
    ref, bnd = R.scan_ref64(u, delta, A, B, C, D, bias, True)
    want = torch.from_numpy(scan_oracle.scan_fwd(u.numpy(), delta.numpy(), A.numpy(), B.numpy(), C.numpy(), D.numpy(),
                                                 bias.numpy(), True)).double()
    err = float((ref["out"] - want).abs().max()) / float(want.abs().max())
    assert err < 2e-5, err                                                   # the oracle takes and returns fp32
    assert bool((bnd["out"] > 0).all())


def _literal(u, delta, A, B, C, D, bias, softplus, dout):
    """the op restated: a loop over L in fp64 autograd; also x = (prod of decays since the start, h) at every chunk end"""
    t = [None if v is None else v.double().clone().requires_grad_(True) for v in (u, delta, A, B, C, D, bias)]
    u_, dl_, A_, B_, C_, D_, b_ = t
    bt, dim, L = u.shape
    G, N = B.shape[1], B.shape[2]
    Bx, Cx = B_.repeat_interleave(dim // G, 1), C_.repeat_interleave(dim // G, 1)         # (b, dim, N, L)
    pre = dl_ + (b_[:, None] if b_ is not None else 0.0)
    d = torch.nn.functional.softplus(pre) if softplus else pre
    h = torch.zeros(bt, dim, N, dtype=torch.float64)
    cum = torch.zeros(bt, dim, dtype=torch.float64)
    ys, xs = [], []
    for l in range(L):
        h = torch.exp(d[:, :, l, None] * A_) * h + (d[:, :, l] * u_[:, :, l])[..., None] * Bx[..., l]
        cum = cum + d[:, :, l].detach()
        ys.append((h * Cx[..., l]).sum(-1) + (D_ * u_[:, :, l] if D_ is not None else 0.0))
        if (l + 1) % R.CHUNK == 0 or l + 1 == L:
            xs.append(torch.stack([torch.exp(cum[..., None] * A_.detach()), h.detach()], -1).reshape(bt, dim, 2 * N))
    out = torch.stack(ys, -1)
    (out * dout.double()).sum().backward()
    grads = dict(du=u_.grad, ddelta=dl_.grad, dA=A_.grad, dB=B_.grad, dC=C_.grad)
    if D_ is not None:
        grads["dD"] = D_.grad
    if b_ is not None:
        grads["ddelta_bias"] = b_.grad
    return dict(out=out.detach(), x=torch.stack(xs, 2), **grads)


@pytest.mark.parametrize("b,dim,L,N,G,has_D,has_bias,softplus", [
    (1, 4, 4200, 4, 1, True, True, True),                  # three chunks of x, the last ragged
    (2, 6, 37, 8, 2, False, False, False),                 # D, delta_bias and softplus off
    (2, 4, 2049, 16, 2, True, False, True),                # a one-position last chunk
    (1, 6, 75, 4, 3, False, True, False)])
def test_gradients_and_chunk_states_match_autograd(b, dim, L, N, G, has_D, has_bias, softplus):
    tag = f"g/{b}/{dim}/{L}/{N}/{G}/{has_D}/{has_bias}/{softplus}"
    u, delta, A, B, C, D, bias, dout = op_scan_params(S, b, dim, L, N, G, tag, "wide", has_D=has_D, has_bias=has_bias,
                                                      softplus=softplus)
    ref, _ = R.scan_ref64(u, delta, A, B, C, D, bias, softplus, dout)
    want = _literal(u, delta, A, B, C, D, bias, softplus, dout)
    assert set(ref) == set(want)
    for name, w in want.items():
        err = float((ref[name] - w).abs().max()) / float(w.abs().max())
        assert err < 1e-12, f"{name}: {err:.2e}"


def _emulate32(u, delta, A, B, C, D, bias, softplus, dout, seed, nseg=1, lt=16):
    """fp32 emulation of the kernels: every decay ex2 and every ex2 of a carried product or of the sigmoid perturbed by a seeded
    ±E2 relative error.  The forward runs in the L-segments of the TMA forward's plan for nseg (lt-position tiles, segments of
    ceil(tiles / nseg) tiles, at most 64): a summary pass per segment from a zero state that sums delta' in fp32 and forms the
    carried decay ex2(a2·sum), the combine's fp32 chain, and the apply pass from the carried state, which writes out and the
    chunk states `x` (its own ex2(a2·running sum) times the product of the preceding segments).  The backward walks serially."""
    f32 = torch.float32
    gen = torch.Generator().manual_seed(seed)
    pm = lambda *s: 1 + R.E2 * (torch.randint(0, 2, s, generator=gen) * 2 - 1).to(f32)
    u, delta, B, C, dout = (t.float() for t in (u, delta, B, C, dout))
    bt, dim, L = u.shape
    G, N = B.shape[1], B.shape[2]
    Bx, Cx = B.repeat_interleave(dim // G, 1), C.repeat_interleave(dim // G, 1)
    Dv = D if D is not None else torch.zeros(dim)
    pre = delta + (bias[:, None] if bias is not None else 0.0)
    dl = torch.where(pre > 20, pre, torch.log1p(torch.exp(pre))) if softplus else pre
    a2 = A * f32_const(LOG2E)
    dec = torch.exp2(dl[:, :, None, :] * a2[..., None]) * pm(bt, dim, N, L)
    ntl = -(-L // lt)
    nsplit = min(nseg, R.MAX_SEGMENTS, ntl)
    tps = -(-ntl // nsplit)
    segs = [(s * tps * lt, min(L, (s + 1) * tps * lt)) for s in range(-(-ntl // tps))]
    out = torch.zeros(bt, dim, L)
    x = torch.zeros(bt, dim, -(-L // R.CHUNK), 2 * N)
    hsave = torch.zeros(bt, dim, N, L)
    H, Pc = torch.zeros(bt, dim, N), torch.ones(bt, dim, N)
    for si, (l0, l1) in enumerate(segs):
        h, sdl = H, torch.zeros(bt, dim)
        for l in range(l0, l1):
            h = dec[..., l] * h + (dl[:, :, l] * u[:, :, l])[..., None] * Bx[..., l]
            sdl = sdl + dl[:, :, l]
            hsave[..., l] = h
            out[:, :, l] = (h * Cx[..., l]).sum(-1) + Dv * u[:, :, l]
            if (l + 1) % R.CHUNK == 0 or l + 1 == L:
                P = torch.exp2(a2 * sdl[..., None]) * pm(bt, dim, N)
                x[:, :, l // R.CHUNK, 0::2] = P * Pc if si else P
                x[:, :, l // R.CHUNK, 1::2] = h
        if si + 1 < len(segs):                                                # summary, then one step of the combine's chain
            hl = torch.zeros(bt, dim, N)
            for l in range(l0, l1):
                hl = dec[..., l] * hl + (dl[:, :, l] * u[:, :, l])[..., None] * Bx[..., l]
            Ps = torch.exp2(a2 * sdl[..., None]) * pm(bt, dim, N)
            H, Pc = Ps * H + hl, Pc * Ps
    res = dict(out=out, x=x)
    if dout is None:
        return res
    du, dd = torch.zeros(bt, dim, L), torch.zeros(bt, dim, L)
    dB, dC = torch.zeros(bt, G, N, L), torch.zeros(bt, G, N, L)
    dA, dD, db = torch.zeros(dim, N), torch.zeros(dim), torch.zeros(dim)
    dh = torch.zeros(bt, dim, N)
    ln2 = f32_const(math.log(2.0))
    for l in range(L - 1, -1, -1):
        dhn = dout[:, :, l, None] * Cx[..., l] + dh
        hp = hsave[..., l - 1] if l else torch.zeros(bt, dim, N)
        ah = dec[..., l] * hp
        s1 = (dhn * Bx[..., l]).sum(-1)
        s2 = (dhn * ah * a2).sum(-1) * ln2
        du[:, :, l] = dout[:, :, l] * Dv + dl[:, :, l] * s1
        X = u[:, :, l] * s1 + s2
        if softplus:
            sgf = 1 / (1 + torch.exp2(-pre[:, :, l] * f32_const(LOG2E)) * pm(bt, dim))
            X = torch.where(pre[:, :, l] <= 20, X * sgf, X)
        dd[:, :, l] = X
        dB[..., l] = (dhn * (dl[:, :, l] * u[:, :, l])[..., None]).view(bt, G, dim // G, N).sum(2)
        dC[..., l] = (dout[:, :, l, None] * hsave[..., l]).view(bt, G, dim // G, N).sum(2)
        dA += (dhn * ah * dl[:, :, l, None]).sum(0)
        dD += (dout[:, :, l] * u[:, :, l]).sum(0)
        db += X.sum(0)
        dh = dhn * dec[..., l]
    res.update(du=du, ddelta=dd, dA=dA, dB=dB, dC=dC)
    if D is not None:
        res["dD"] = dD
    if bias is not None:
        res["ddelta_bias"] = db
    return res


def f32_const(v):
    return float(np.float32(v))


@pytest.mark.parametrize("b,dim,L,N,G,dist,nseg", [
    (2, 16, 2100, 16, 2, "sigma", 1), (2, 16, 2100, 16, 2, "sigma", 7), (1, 32, 2500, 4, 1, "sigma", 64),
    (2, 16, 700, 4, 2, "wide", 1), (2, 16, 700, 8, 1, "wide", 11), (2, 8, 300, 16, 1, "ref", 5)])
def test_bound_covers_an_fp32_emulation(b, dim, L, N, G, dist, nseg):
    tag = f"e/{b}/{dim}/{L}/{N}/{G}/{dist}/{nseg}"
    u, delta, A, B, C, D, bias, dout = op_scan_params(S, b, dim, L, N, G, tag, dist)
    ref, bnd = R.scan_ref64(u, delta, A, B, C, D, bias, True, dout)
    emu = _emulate32(u, delta, A, B, C, D, bias, True, dout, seed=len(tag), nseg=nseg)
    if nseg > 1:                                  # the backward's hs come from the serial walk: compare its outputs once
        emu = {k: v for k, v in emu.items() if k in ("out", "x")}
    worst = {}
    for name, v in emu.items():
        v = v.double()
        frac = R.bound_fraction(v, ref[name], bnd[name])
        worst[name] = frac
        assert frac <= 1.0, f"{name}: {frac:.3f} of the bound"
        # per element, yet no looser than 1e-3 of the tensor's scale at its largest element
        i = int(ref[name].abs().argmax())
        assert float(bnd[name].reshape(-1)[i]) <= 1e-3 * float(ref[name].abs().max()), name
    record(f"scan_ref64 bound self-check {tag}", **worst)
