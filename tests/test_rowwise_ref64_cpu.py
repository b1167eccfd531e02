"""CPU: the fp64 references and error bounds of the row-wise and decoder-tail kernels (oracle/rowwise_ref64.py) that
tests/test_rowwise_fp64_gpu.py compares the kernels with.
* agreement: every reference against torch's own fp64 composition (F.layer_norm, F.interpolate(bilinear, align_corners=False),
  reshape / permute for the gather and the pixel shuffle, a 1x1 conv, autograd for the LayerNorm backward) to ~1e-12;
* soundness: an fp32 emulation of each kernel's operation order (its lane layout, float4 sums, butterflies, fmaf epilogues; rsqrtf,
  ex2 and __fdividef perturbed by their documented error) stays inside the bound on every input family;
* sharpness: each plausible kernel mistake, emulated in fp32 the same way, lands outside the bound on the designed inputs;
* coverage: the kernel instances of the built library, the oracle's tables of them and the GPU test's parameter lists agree, so a
  new instantiation fails here until the oracle lists it and the GPU test has a case for it."""
import math
import re
import subprocess

import pytest
import torch
import torch.nn.functional as F

import test_rowwise_fp64_gpu as G
from helpers import record
from oracle import rowwise_ref64 as R

F32 = torch.float32
BF = torch.bfloat16
LOG2E_F32 = torch.tensor(1.4426950408889634, dtype=F32)
EPS = 1e-5


# ---------------------------------------------------------------- fp32 emulation of the kernels
def _fma(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def _lane_sum(t4, lanes):
    """t4 (rows, V, lanes, 4) fp32: every lane adds its float4s as s += (x+y)+(z+w), then the xor butterfly"""
    s = torch.zeros(t4.shape[0], lanes, dtype=F32)
    for v in range(t4.shape[1]):
        f = t4[:, v]
        s = s + ((f[..., 0] + f[..., 1]) + (f[..., 2] + f[..., 3]))
    o = lanes // 2
    while o:
        s = s + s[:, torch.arange(lanes) ^ o]
        o //= 2
    return s[:, 0]


def _rsqrt(v):
    return (1.0 / torch.sqrt(v.double()) * (1 - R.E_RSQRT)).float()


def _silu(z):
    e = (torch.exp2((-z * LOG2E_F32).double()) * (1 + R.E2)).float()
    return (z.double() / (1.0 + e).double() * (1 - R.E_FDIV)).float()


def _bf(t):
    """fp32 -> bf16 -> fp32, round to nearest even (the kernels' st4 / __floats2bfloat162_rn)"""
    return t.to(BF).float()


def _bf_rz(t):
    """fp32 -> bf16 rounding toward zero (the low 16 bits dropped), as fp32"""
    return (t.contiguous().view(torch.int32) & -65536).view(F32)


def emu_norm(y, gamma, beta, eps, plan, z=None, gate_r=None, mut=()):
    """row_norm_{fast_,}kernel on y (K, rows, D) fp32: the K-sum, the lane-ordered mean / variance, rsqrtf, the fmaf epilogue,
    SiLU(z) and the gate (gate_r: the gate row of every row).  Also the normalisation of the head / upsample kernels.
    mut: "one_pass" (var = E[x^2] - mean^2), "eps_on_sigma" (rstd = 1/(sqrt(var) + eps)), "k_sum_bf16" (each partial K-sum rounded
    to bf16), "stats_bf16" (mean and variance from a bf16-rounded copy of the row)"""
    K, rows, D = y.shape
    lanes, vecs = plan[:2]
    a = y[0].clone()
    for k in range(1, K):
        a = a + y[k]
        if "k_sum_bf16" in mut:
            a = _bf(a)
    Dp = 4 * lanes * vecs
    xp = torch.zeros(rows, Dp, dtype=F32)
    xp[:, :D] = a
    mask = torch.zeros(Dp, dtype=F32)
    mask[:D] = 1
    view = lambda t: t.view(rows, vecs, lanes, 4)
    xs = _bf(xp) if "stats_bf16" in mut else xp
    mean = _lane_sum(view(xs), lanes) / float(D)
    d = xp - mean[:, None]
    if "one_pass" in mut:
        var = _lane_sum(view(xp * xp), lanes) / float(D) - mean * mean
    else:
        dm = (xs - mean[:, None]) * mask
        var = _lane_sum(view(dm * dm), lanes) / float(D)
    if "eps_on_sigma" in mut:
        rstd = (1.0 / (torch.sqrt(var.clamp_min(0)) + eps)).float()
    else:
        rstd = _rsqrt(var + eps)
    o = _fma(d[:, :D] * rstd[:, None], gamma, beta)
    if z is not None:
        o = o * _silu(z)
    if gate_r is not None:
        o = o * gate_r
    return o


def _taps32(n, mut=()):
    o = torch.arange(2 * n, dtype=F32)
    if "align_corners" in mut:
        s = (o.double() * (n - 1) / max(2 * n - 1, 1)).float()
    else:
        s = (o + 0.5) * 0.5 - 0.5
        if "unclamped" not in mut:
            s = s.clamp_min(0.0)
    i0 = torch.trunc(s).long()
    return i0, (i0 + 1).clamp_max(n - 1), s - i0.float()


def emu_bilinear(x, mut=()):
    """upsample2x_plain_kernel / the taps of the norm and head kernels, fp32, the kernel's association.
    mut: "unclamped", "align_corners", "seam" (the head's last tile column reads tap w0 for w1: a halo one column short)"""
    B, H, W, C = x.shape
    h0, h1, fh = _taps32(H, mut)
    w0, w1, fw = _taps32(W, mut)
    if "seam" in mut:
        seam = (torch.arange(2 * W) % 32 == 31) & (torch.arange(2 * W) < 2 * W - 1)
        w1 = torch.where(seam, w0, w1)
    fh, fw = fh[:, None, None], fw[:, None]
    r0, r1 = x[:, h0], x[:, h1]
    a, b, c, d = r0[:, :, w0], r0[:, :, w1], r1[:, :, w0], r1[:, :, w1]
    return (1 - fh) * ((1 - fw) * a + fw * b) + fh * ((1 - fw) * c + fw * d)


def emu_head(x, gamma, beta, eps, wcls, plan, mut=()):
    """upsample2x_norm_head_{fast_,}kernel: bilinear, the normalisation, then per lane an fmaf chain over its channels (w, z, y, x
    of every float4, float4 by float4) and the butterfly; NCHW"""
    B, H, W, C = x.shape
    lanes, vecs = plan[:2]
    up = emu_bilinear(x, mut).reshape(-1, C)
    o = emu_norm(up[None], gamma, beta, eps, plan)
    Cp = 4 * lanes * vecs
    op = torch.zeros(o.shape[0], Cp, dtype=F32)
    op[:, :C] = o
    wp = torch.zeros(wcls.shape[0], Cp, dtype=F32)
    wp[:, :C] = wcls
    o4 = op.view(-1, 1, vecs, lanes, 4)
    w4 = wp.view(1, -1, vecs, lanes, 4)
    acc = torch.zeros(o.shape[0], wcls.shape[0], lanes, dtype=F32)
    for v in range(vecs):
        for j in (3, 2, 1, 0):
            acc = _fma(o4[:, :, v, :, j], w4[:, :, v, :, j], acc)
    s = lanes // 2
    while s:
        acc = acc + acc[..., torch.arange(lanes) ^ s]
        s //= 2
    return acc[..., 0].view(B, 2 * H, 2 * W, -1).permute(0, 3, 1, 2)


def emu_pool(x, nslice, mut=()):
    """pool_avgmax_partial_kernel + fused.pool_avgmax: per thread a sequential sum / max over positions pr, pr + rows, ...; the rows
    partials in order; the slices' sums in order, / L.  mut: "max_from_0", "mean_per_x_nslice" (/ ceil(L/nslice)·nslice)"""
    B, L, C = x.shape
    rows = R.pool_rows(C)
    sums, maxs = [], []
    for l0, l1 in R.pool_slices(L, nslice):
        a = torch.zeros(B, C, dtype=F32)
        m = torch.full((B, C), 0.0 if "max_from_0" in mut else -math.inf, dtype=F32)
        for pr in range(rows):
            t = torch.zeros(B, C, dtype=F32)
            for l in range(l0 + pr, l1, rows):
                t = t + x[:, l]
                m = torch.maximum(m, x[:, l])
            a = a + t
        sums.append(a)
        maxs.append(m)
    tot = torch.zeros(B, C, dtype=F32)
    for a in sums:
        tot = tot + a
    div = -(-L // nslice) * nslice if "mean_per_x_nslice" in mut else L
    return tot / float(div), torch.stack(maxs, 1).amax(1), torch.stack(sums, 1)


def emu_ln_bwd(x, dy, gamma, eps, mut=()):
    """layernorm_bwd_body: dx of every row, dgamma / dbeta as the grid's warps accumulate them (rows in warp order).
    mut: "dx_bf16_before_rstd" (dx = bf16(bf16(gamma dy - m1 - xhat m2)·rstd): a bf16 kernel rounding before the last product)"""
    rows, D = x.shape
    lpr, vecs, nw, _ = R.bwd_plan(rows, D)
    view = lambda t: t.view(rows, vecs, lpr, 4)
    invD = torch.tensor(1.0 / D, dtype=F32)
    mean = _lane_sum(view(x), lpr) * invD
    xc = x - mean[:, None]
    rstd = _rsqrt(_lane_sum(view(xc * xc), lpr) * invD + eps)
    xh = xc * rstd[:, None]
    a = gamma * dy
    m1 = _lane_sum(view(a), lpr) * invD
    m2 = _lane_sum(view(a * xh), lpr) * invD
    inner = a - m1[:, None] - xh * m2[:, None]
    dx = _bf(rstd[:, None] * _bf(inner)) if "dx_bf16_before_rstd" in mut else rstd[:, None] * inner
    rpw = 32 // lpr
    steps = -(-rows // rpw)
    dg, db = torch.zeros(D, dtype=F32), torch.zeros(D, dtype=F32)
    for w in range(min(nw, steps)):
        pg, pb = torch.zeros(rpw, D, dtype=F32), torch.zeros(rpw, D, dtype=F32)
        for st in range(w, steps, nw):
            for sub in range(rpw):
                r = min(st * rpw + sub, rows - 1)
                if st * rpw + sub < rows:
                    pg[sub] = _fma(dy[r], xh[r], pg[sub])
                    pb[sub] = pb[sub] + dy[r]
        o = 1
        while o < rpw:
            pg = pg + pg[torch.arange(rpw) ^ o]
            pb = pb + pb[torch.arange(rpw) ^ o]
            o <<= 1
        dg, db = dg + pg[0], db + pb[0]
    return dx, dg, db


# ---------------------------------------------------------------- agreement
def test_layer_norm_and_merge_match_torch():
    x = R.hard_rows(1, 40, 96)
    g, b = R.affine(2, 96)
    ref = F.layer_norm(x.double(), (96,), g.double(), b.double(), EPS)
    assert torch.allclose(R.layer_norm_ref64(x, g, b, EPS), ref, rtol=0, atol=1e-12 * float(ref.abs().max()))
    y = torch.randn(3, 40, 96, dtype=torch.float64)
    z = torch.randn(40, 96, dtype=torch.float64)
    gate = torch.randn(5, 96, dtype=torch.float64)
    want = F.layer_norm(y.sum(0), (96,), g.double(), b.double(), EPS) * F.silu(z) * gate.repeat_interleave(8, 0)
    assert torch.allclose(R.merge_norm_ref64(y, g, b, EPS, z, gate, 8), want, rtol=0, atol=1e-12 * float(want.abs().max()))


@pytest.mark.parametrize("H,W", [(4, 6), (5, 7)])
def test_patch_merge_gather_matches_reshape(H, W):
    x = torch.randn(2, H, W, 8, dtype=torch.float64)
    xp = F.pad(x, (0, 0, 0, W % 2, 0, H % 2))
    B, Hp, Wp, C = xp.shape
    # PatchMerging2D: x0 = x[0::2, 0::2], x1 = x[1::2, 0::2], x2 = x[0::2, 1::2], x3 = x[1::2, 1::2] -> (dw dh c) order
    want = xp.view(B, Hp // 2, 2, Wp // 2, 2, C).permute(0, 1, 3, 4, 2, 5).reshape(-1, 4 * C)
    assert torch.equal(R.patch_merge_gather64(x), want)


def test_pixel_shuffle_matches_rearrange():
    B, H, W, C = 2, 3, 5, 6
    y = torch.randn(B, H, W, 4 * C, dtype=torch.float64)
    want = torch.empty(B, 2 * H, 2 * W, C, dtype=torch.float64)
    for p1 in range(2):
        for p2 in range(2):
            want[:, p1::2, p2::2] = y[..., (2 * p1 + p2) * C:(2 * p1 + p2 + 1) * C]
    assert torch.equal(R.pixel_shuffle64(y, B, H, W), want)


@pytest.mark.parametrize("H,W", [(1, 1), (1, 5), (4, 7), (13, 49)])
def test_upsample_and_head_match_torch(H, W):
    x = torch.randn(2, H, W, 48, dtype=torch.float64)
    want = F.interpolate(x.permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
    assert torch.allclose(R.upsample2x_ref64(x), want, rtol=0, atol=1e-12)
    g, b = R.affine(3, 48)
    wc = torch.randn(9, 48, dtype=torch.float64)
    up = F.layer_norm(want, (48,), g.double(), b.double(), EPS)
    logits = F.conv2d(up.permute(0, 3, 1, 2), wc[:, :, None, None])
    assert torch.allclose(R.head_ref64(x, g, b, EPS, wc), logits, rtol=0, atol=1e-12 * float(logits.abs().max()))


def test_pool_scale_add_match_torch():
    x = R.pool_input(4, 2, 2049, 8)
    mean, mx = R.pool_avgmax_ref64(x)
    xd = x.double()
    assert torch.allclose(mean, F.adaptive_avg_pool2d(xd.permute(0, 2, 1)[..., None], 1)[..., 0, 0], rtol=0, atol=1e-12)
    assert torch.equal(mx, F.adaptive_max_pool2d(xd.permute(0, 2, 1)[..., None], 1)[..., 0, 0])
    part = R.pool_partial_ref64(x, 64)
    assert torch.allclose(part[:, :, 0].sum(1) / 2049, mean, rtol=0, atol=1e-12) and torch.equal(part[:, :, 1].amax(1), mx)
    assert bool((part[:, 63, 0] == 0).all()) and bool((part[:, 63, 1] == -math.inf).all())   # 63 slices of 33 cover 2049
    a, b = torch.randn(12, 8, dtype=torch.float64), torch.randn(12, 8, dtype=torch.float64)
    sa, sb = torch.randn(3, 8, dtype=torch.float64), torch.randn(8, dtype=torch.float64)
    assert torch.equal(R.scale_add_ref64(a, sa, b, sb, 4), a * sa.repeat_interleave(4, 0) + b * sb)
    assert torch.equal(R.scale_add_ref64(None, None, b, sb, 4), b * sb)


def test_layernorm_bwd_matches_autograd():
    x = R.hard_rows(5, 30, 96).double().requires_grad_(True)
    g, b = (t.double().requires_grad_(True) for t in R.affine(6, 96))
    dy = torch.randn(30, 96, dtype=torch.float64)
    F.layer_norm(x, (96,), g, b, EPS).backward(dy)
    dx, dg, db = R.layernorm_bwd_ref64(x, dy, g, EPS)
    for got, want in ((dx, x.grad), (dg, g.grad), (db, b.grad)):
        assert torch.allclose(got, want, rtol=0, atol=1e-12 * float(want.abs().max()))


# ---------------------------------------------------------------- soundness
@pytest.mark.parametrize("D", [32, 64, 96, 200, 384, 1000, 2048])
def test_layer_norm_bound_covers_fp32_emulation(D):
    x = R.hard_rows(10 + D, 50, D)
    g, b = R.affine(11, D)
    plan = R.row_plan(D)
    got = emu_norm(x[None], g, b, EPS, plan)
    ref = R.layer_norm_ref64(x, g, b, EPS)
    frac = R.bound_fraction(got, ref, R.layer_norm_bound(x, g, b, EPS, plan))
    record("rowwise_ref64_cpu/ln_soundness", D=D, plan=list(plan), bound_used=frac)
    assert frac <= 1.0
    const = R.constant_rows(50)
    assert torch.equal(got[const], b.expand(int(const.sum()), D)), "a constant row must give beta exactly"


@pytest.mark.parametrize("K", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("D", [96, 200])
def test_merge_norm_bound_covers_fp32_emulation(K, D):
    rows, rpb = 60, 7
    y = torch.stack([R.hard_rows(20 + k, rows, D) for k in range(K)])
    z = torch.randn(rows, D) * 3
    gate = torch.randn(-(-rows // rpb), D)
    g, b = R.affine(21, D)
    plan = R.row_plan(D, K)
    got = emu_norm(y, g, b, EPS, plan, z, gate[torch.arange(rows) // rpb])
    ref = R.merge_norm_ref64(y, g, b, EPS, z, gate, rpb)
    frac = R.bound_fraction(got, ref, R.merge_norm_bound(y, g, b, EPS, plan, z, gate, rpb))
    record("rowwise_ref64_cpu/merge_soundness", K=K, D=D, bound_used=frac)
    assert frac <= 1.0


@pytest.mark.parametrize("H,W,C,ncls", [(5, 20, 96, 9), (3, 17, 64, 21), (4, 9, 48, 40), (1, 1, 96, 2)])
def test_upsample_head_bounds_cover_fp32_emulation(H, W, C, ncls):
    x = torch.randn(2, H, W, C) * 2 + torch.randn(2, H, W, 1) * 40          # per-pixel offsets: large means after the taps
    g, b = R.affine(30, C)
    wc = torch.randn(ncls, C) / math.sqrt(C)
    up = emu_bilinear(x)
    assert R.bound_fraction(up, R.upsample2x_ref64(x), R.upsample2x_bound(x)) <= 1.0
    plan0 = R.head_plan(C, 0)
    un = emu_norm(up.reshape(1, -1, C), g, b, EPS, plan0).view(up.shape)
    assert R.bound_fraction(un, R.upsample2x_norm_ref64(x, g, b, EPS), R.upsample2x_norm_bound(x, g, b, EPS, plan0)) <= 1.0
    plan = R.head_plan(C, ncls)
    got = emu_head(x, g, b, EPS, wc, plan)
    frac = R.bound_fraction(got, R.head_ref64(x, g, b, EPS, wc), R.head_bound(x, g, b, EPS, wc, plan))
    record("rowwise_ref64_cpu/head_soundness", H=H, W=W, C=C, ncls=ncls, bound_used=frac)
    assert frac <= 1.0


@pytest.mark.parametrize("L,C,nslice", [(2049, 4, 64), (300, 40, 7), (97, 1000, 3)])
def test_pool_bound_covers_fp32_emulation(L, C, nslice):
    x = R.pool_input(40, 2, L, C)
    mean, mx, part = emu_pool(x, nslice)
    rm, rx = R.pool_avgmax_ref64(x)
    assert torch.equal(mx.double(), rx)
    assert R.bound_fraction(mean, rm, R.pool_mean_bound(x, nslice)) <= 1.0
    assert R.bound_fraction(part, R.pool_partial_ref64(x, nslice)[:, :, 0], R.pool_partial_bound(x, nslice)) <= 1.0


def test_scale_add_bound_covers_fp32_emulation():
    a, b = torch.randn(30, 16), torch.randn(30, 16) * 100
    sa, sb = torch.randn(3, 16), torch.randn(16)
    got = _fma(a, sa[torch.arange(30) // 10], b * sb)
    assert R.bound_fraction(got, R.scale_add_ref64(a, sa, b, sb, 10), R.scale_add_bound(a, sa, b, sb, 10)) <= 1.0
    assert R.bound_fraction(b * sb, R.scale_add_ref64(None, None, b, sb, 10), R.scale_add_bound(None, None, b, sb, 10)) <= 1.0


@pytest.mark.parametrize("D", [32, 96, 384])
def test_layernorm_bwd_bound_covers_fp32_emulation(D):
    rows = 203
    x = R.hard_rows(50 + D, rows, D)
    g, _ = R.affine(51, D)
    dy = torch.randn(rows, D)
    got = emu_ln_bwd(x, dy, g, EPS)
    ref = R.layernorm_bwd_ref64(x, dy, g, EPS)
    for name, gt, rf, bd in zip(("dx", "dgamma", "dbeta"), got, ref, R.layernorm_bwd_bound(x, dy, g, EPS)):
        frac = R.bound_fraction(gt, rf, bd)
        record("rowwise_ref64_cpu/ln_bwd_soundness", D=D, out=name, bound_used=frac)
        assert frac <= 1.0, name


def _bf16_case(io, K, D, rows=60, seed=70):
    """inputs of a bf16 instance as its GPU test draws them: y (K, rows, D) bf16-exact for io 2 (fp32 for io 1, K = 1), z bf16-exact"""
    y = torch.stack([R.hard_rows(seed + k, rows, D, bf16=io == 2).float() for k in range(K)])
    z = _bf(torch.randn(rows, D, generator=torch.Generator().manual_seed(seed)) * 3) if io == 2 else None
    return y, z


@pytest.mark.parametrize("io,K,D", [(1, 1, 96), (1, 1, 200), (1, 1, 2048), (2, 1, 64), (2, 2, 384), (2, 3, 200), (2, 4, 96), (2, 8, 1000)])
def test_bf16_norm_bound_covers_fp32_then_bf16_emulation(io, K, D):
    """the fp32 emulation on bf16-exact inputs, its output rounded to bf16 once: inside bf16_store_bound of the fp32 bound; a constant
    row gives bf16(beta) exactly"""
    rows, rpb = 60, 7
    y, z = _bf16_case(io, K, D, rows)
    gate = torch.randn(-(-rows // rpb), D) if io == 2 else None
    g, b = R.affine(71, D)
    plan = R.row_plan(D, K, io=io)
    got = emu_norm(y, g, b, EPS, plan, z, gate[torch.arange(rows) // rpb] if gate is not None else None).to(BF)
    ref = R.merge_norm_ref64(y, g, b, EPS, z, gate, rpb)
    frac = R.bound_fraction(got, ref, R.bf16_store_bound(ref, R.merge_norm_bound(y, g, b, EPS, plan, z, gate, rpb)))
    record("rowwise_ref64_cpu/bf16_soundness", io=io, K=K, D=D, bound_used=frac)
    assert frac <= 1.0
    const = R.constant_rows(rows)
    got_c = emu_norm(y, g, b, EPS, plan).to(BF)[const]
    assert torch.equal(got_c, b.to(BF).expand(int(const.sum()), D)), "a constant row must give bf16(beta) exactly"


def test_bf16_hard_rows_stay_hard():
    """the bf16 form of hard_rows: var_eps rows keep sigma^2 ~ eps after rounding (not flattened to a few values), constant rows
    stay constant and exact"""
    D = 384
    x = R.hard_rows(72, 50, D, bf16=True)
    assert x.dtype == BF
    fam = torch.arange(50) % len(R.ROW_FAMILIES)
    var = x.double().var(-1, unbiased=False)
    ve = var[fam == R.ROW_FAMILIES.index("var_eps")]
    assert bool((ve > 0.3 * EPS).all() and (ve < 3 * EPS).all()), ve
    distinct = [len(torch.unique(r)) for r in x[fam == R.ROW_FAMILIES.index("var_eps")]]
    assert min(distinct) >= 20, distinct
    x32 = R.hard_rows(72, 50, D)
    const = R.constant_rows(50)
    assert torch.equal(x[const].float(), x32[const])


@pytest.mark.parametrize("D", [32, 96, 384])
def test_layernorm_bwd_bf16_bound_covers_emulation(D):
    """sigma_layernorm_bwd_bf16: bf16-exact x and dy, the fp32 body, dx rounded once: dx inside bf16_store_bound, dgamma / dbeta
    inside the unchanged fp32 bound"""
    rows = 203
    x = R.hard_rows(80 + D, rows, D, bf16=True).float()
    g, _ = R.affine(81, D)
    dy = _bf(torch.randn(rows, D, generator=torch.Generator().manual_seed(82)))
    dx, dg, db = emu_ln_bwd(x, dy, g, EPS)
    ref = R.layernorm_bwd_ref64(x, dy, g, EPS)
    bnd = R.layernorm_bwd_bound(x, dy, g, EPS)
    for name, gt, rf, bd in zip(("dx", "dgamma", "dbeta"), (dx.to(BF), dg, db), ref, (R.bf16_store_bound(ref[0], bnd[0]),) + bnd[1:]):
        frac = R.bound_fraction(gt, rf, bd)
        record("rowwise_ref64_cpu/ln_bwd_bf16_soundness", D=D, out=name, bound_used=frac)
        assert frac <= 1.0, name


# ---------------------------------------------------------------- sharpness: plausible mistakes land outside the bound
def _outside(got, ref, bound, what):
    frac = R.bound_fraction(got, ref, bound)
    record("rowwise_ref64_cpu/mutation", mutation=what, bound_used=frac)
    assert frac > 1.0, f"{what}: the bound does not reject it ({frac:.3g})"


@pytest.mark.parametrize("mut,family", [("one_pass", "large_mean"), ("eps_on_sigma", "var_eps")])
def test_variance_mistakes_are_rejected(mut, family):
    D = 96
    x = R.hard_rows(60, 40, D, families=(family,))
    g, b = R.affine(61, D)
    plan = R.row_plan(D)
    _outside(emu_norm(x[None], g, b, EPS, plan, mut=(mut,)), R.layer_norm_ref64(x, g, b, EPS),
             R.layer_norm_bound(x, g, b, EPS, plan), mut)


@pytest.mark.parametrize("mut,io,K,family", [("round_toward_zero", 2, 1, "ordinary"), ("k_sum_bf16", 2, 4, "ordinary"),
                                             ("stats_bf16", 1, 1, "large_mean")])
def test_bf16_norm_mistakes_are_rejected(mut, io, K, family):
    """a bf16 store that truncates, the K-direction sum kept in bf16, statistics taken from a bf16-rounded copy of an fp32 row"""
    D = 96
    y = torch.stack([R.hard_rows(90 + k, 40, D, families=(family,), bf16=io == 2).float() for k in range(K)])
    g, b = R.affine(91, D)
    plan = R.row_plan(D, K, io=io)
    o = emu_norm(y, g, b, EPS, plan, mut=(mut,))
    got = _bf_rz(o) if mut == "round_toward_zero" else o.to(BF)
    ref = R.merge_norm_ref64(y, g, b, EPS)
    bound = R.bf16_store_bound(ref, R.merge_norm_bound(y, g, b, EPS, plan))
    assert R.bound_fraction(emu_norm(y, g, b, EPS, plan).to(BF), ref, bound) <= 1.0
    _outside(got, ref, bound, mut)


def test_bf16_ln_bwd_double_rounding_is_rejected():
    """dx rounded to bf16 before the final rstd product (and again on the store)"""
    D, rows = 96, 203
    x = R.hard_rows(92, rows, D, families=("ordinary",), bf16=True).float()
    g, _ = R.affine(93, D)
    dy = _bf(torch.randn(rows, D, generator=torch.Generator().manual_seed(94)))
    ref = R.layernorm_bwd_ref64(x, dy, g, EPS)
    bound = R.bf16_store_bound(ref[0], R.layernorm_bwd_bound(x, dy, g, EPS)[0])
    _outside(emu_ln_bwd(x, dy, g, EPS, mut=("dx_bf16_before_rstd",))[0], ref[0], bound, "dx rounded before rstd")


def test_gate_and_z_mistakes_are_rejected():
    D, rows, rpb = 96, 42, 7
    y = R.hard_rows(62, rows, D, families=("ordinary",))[None]
    xz = torch.randn(rows, 2 * D)
    gate = torch.randn(rows // rpb, D)
    g, b = R.affine(63, D)
    plan = R.row_plan(D)
    ref = R.merge_norm_ref64(y, g, b, EPS, xz[:, D:], gate, rpb)
    bound = R.merge_norm_bound(y, g, b, EPS, plan, xz[:, D:], gate, rpb)
    shifted = gate[(torch.arange(rows) - 1).clamp_min(0) // rpb]                # image b's gate from one row past its boundary
    _outside(emu_norm(y, g, b, EPS, plan, xz[:, D:], shifted), ref, bound, "gate one row past the batch boundary")
    _outside(emu_norm(y, g, b, EPS, plan, xz[:, :D], gate[torch.arange(rows) // rpb]), ref, bound, "z read from the x half")


@pytest.mark.parametrize("mut", ["unclamped", "align_corners"])
def test_tap_mistakes_are_rejected(mut):
    x = torch.randn(2, 5, 7, 16)
    _outside(emu_bilinear(x, (mut,)), R.upsample2x_ref64(x), R.upsample2x_bound(x), mut)


def test_head_seam_mistake_is_rejected():
    x = torch.randn(1, 4, 40, 96)                                              # Wo = 80: seams at columns 31 and 63
    g, b = R.affine(64, 96)
    wc = torch.randn(9, 96) / math.sqrt(96)
    plan = R.head_plan(96, 9)
    ref, bound = R.head_ref64(x, g, b, EPS, wc), R.head_bound(x, g, b, EPS, wc, plan)
    assert R.bound_fraction(emu_head(x, g, b, EPS, wc, plan), ref, bound) <= 1.0
    _outside(emu_head(x, g, b, EPS, wc, plan, ("seam",)), ref, bound, "head halo one column short at the tile seam")


def test_pool_mistakes_are_rejected():
    L, nslice = 2049, 64                                                       # 63 slices of 33 positions, the last one empty
    x = R.pool_input(65, 2, L, 8)
    rm, rx = R.pool_avgmax_ref64(x)
    _, mx, _ = emu_pool(x, nslice, ("max_from_0",))
    assert not torch.equal(mx.double(), rx), "a max that starts at 0 must differ on all-negative channels"
    mean, _, _ = emu_pool(x, nslice, ("mean_per_x_nslice",))
    _outside(mean, rm, R.pool_mean_bound(x, nslice), "mean divided by slice length x slices")


def test_shuffle_and_gather_mistakes_are_rejected():
    B, H, W, C = 2, 3, 5, 96
    g, b = R.affine(66, C)
    plan = R.row_plan(C, mode=2)
    y = torch.randn(B, H, W, 4 * C)
    rows = y.reshape(-1, C)                                                     # the kernel normalises (b h w p1 p2) sub-rows
    ref = R.pixel_shuffle64(R.layer_norm_ref64(rows, g, b, EPS).reshape(B, H, W, 4 * C), B, H, W)
    bound = R.pixel_shuffle64(R.layer_norm_bound(rows, g, b, EPS, plan).reshape(B, H, W, 4 * C), B, H, W)
    o = emu_norm(rows[None], g, b, EPS, plan).reshape(B, H, W, 2, 2, C)
    assert R.bound_fraction(R.pixel_shuffle64(o.reshape(B, H, W, -1), B, H, W), ref, bound) <= 1.0
    _outside(R.pixel_shuffle64(o.transpose(3, 4).reshape(B, H, W, -1), B, H, W), ref, bound, "p1 / p2 swapped")
    Cq = 24
    g4, b4 = R.affine(67, 4 * Cq)
    plan4 = R.row_plan(4 * Cq, mode=1)
    x = torch.randn(B, 5, 7, Cq)
    cat = R.patch_merge_gather64(x).float()
    ref, bound = R.layer_norm_ref64(cat, g4, b4, EPS), R.layer_norm_bound(cat, g4, b4, EPS, plan4)
    swapped = cat.view(-1, 4, Cq)[:, [0, 2, 1, 3]].reshape(-1, 4 * Cq)
    _outside(emu_norm(swapped[None], g4, b4, EPS, plan4), ref, bound, "patch-merge quadrants swapped")


# ---------------------------------------------------------------- coverage cross-check, against the built library
_ELEM = {"float": "f32", "__nv_bfloat16": "bf16", "__half": "f16", "sigma::E4M3Rows": "e4m3"}
_BWD = ("layernorm_bwd_kernel", "layernorm_bwd_det_kernel", "layernorm_bwd_bf16_kernel", "layernorm_bwd_fp16_kernel")


@pytest.fixture(scope="module")
def instances():
    """{kernel: set of template-argument tuples} of the row-wise kernels in libsigma_b200.so (`cuobjdump -sass`, demangled by
    cu++filt); integer arguments as ints, element types by the oracle's names"""
    from sigma_b200 import _lib
    out = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    names = subprocess.run(["cu++filt"], input="\n".join(re.findall(r"Function : (\S+)", out)), capture_output=True, text=True,
                           check=True).stdout
    inst = {}
    for kernel, args in re.findall(r"sigma::(row_norm\w*|layernorm_bwd\w*|upsample2x_norm\w*)<([^<>]*)>\(", names):
        inst.setdefault(kernel, set()).add(tuple(int(a[5:]) if a.startswith("(int)") else _ELEM[a] for a in args.split(", ")))
    return inst


def test_instantiation_tables_are_covered(instances):
    row = {(l, v) for l, v, *_ in instances["row_norm_fast_kernel"]}
    head = instances["upsample2x_norm_head_fast_kernel"]
    cases = sorted({n for _, n in instances["upsample2x_norm_kernel"]} - {0})
    fast_ncls = {n for n in cases if n <= R.HEAD_FAST_MAX_NCLS}
    assert row == set(R.ROW_FAST) and cases == R.HEAD_NCLS
    assert all(instances[k] == set(R.BWD_FAST) for k in _BWD)
    # the fast head at every class count up to HEAD_FAST_MAX_NCLS (NCLS 1: the placeholder the larger class counts compile)
    assert head == {(l, v, n) for l, v in R.HEAD_FAST for n in fast_ncls | {1}}
    # the GPU test reaches every instantiation
    assert {4 * l * v for l, v in row} <= set(G.LN_FAST_D)
    assert {R.row_plan(D)[1] for D in G.LN_GENERIC_D if not R.row_plan(D)[2]} == set(R.MAXV_GENERIC)
    assert all(R.row_plan(D)[2] for D in G.MERGE_D) and set(G.MERGE_K) == set(range(1, 9))
    assert {4 * l * v for l, v in R.HEAD_FAST} <= set(G.HEAD_FAST_C)
    assert fast_ncls <= set(G.HEAD_FAST_NCLS) and set(cases) - fast_ncls <= set(G.HEAD_GENERIC_NCLS)
    assert all(not R.head_plan(C, 9)[2] for C in G.HEAD_GENERIC_C)
    assert {R.head_plan(C, 0)[1] for C in G.UPSAMPLE_C} == {1, 2, 4, 8}
    assert all(R.row_plan(4 * c, mode=1)[2] for c in G.PATCH_MERGE_C) and not any(4 * G.PATCH_MERGE_UNSUPPORTED_C == 4 * l * v for l, v in row)
    assert {4 * l * v for l, v in row} <= set(G.SHUFFLE_D)


def test_row_norm_instances_are_the_oracles_and_covered(instances):
    """The built row_norm_fast_kernel and row_norm_kernel instances are exactly the oracle's: every fast width at each (mode, K) of
    ROW_FAST_PAIRS, and the generic kernel at each MAXV of ROW_GENERIC_MAXV, for all seven element pairs.  The GPU test's parameter
    lists reach every fp32 / bf16 instance of them at every fast width, and its bf16 LayerNorm backward runs every BWD_FAST width."""
    fast, generic = instances["row_norm_fast_kernel"], instances["row_norm_kernel"]
    assert fast == {(l, v, k, mode, *pair) for pair, modes in R.ROW_FAST_PAIRS.items() for mode, ks in modes.items() for k in ks
                    for l, v in R.ROW_FAST}
    assert generic == {(mv, *pair) for pair, mvs in R.ROW_GENERIC_MAXV.items() for mv in mvs}
    assert len(fast) == 209 and len(generic) == 38
    # what the GPU cases reach: fast (lanes, vecs, K, mode, pair) and generic (MAXV, pair)
    cases = [(D, 1, 0, io) for D in G.LN_FAST_D + G.LN_GENERIC_D for io in G.LN_IO]
    cases += [(D, K, 0, io) for K in G.MERGE_K for D in G.MERGE_D for io in G.MERGE_IO]
    cases += [(4 * C, 1, 1, io) for C in G.PATCH_MERGE_C for io in G.PATCH_MERGE_IO]
    cases += [(D, 1, 2, 0) for D in G.SHUFFLE_D]
    reached = set()
    for D, K, mode, io in cases:
        lanes, vecs, is_fast = R.row_plan(D, K, mode, io)
        reached.add((lanes, vecs, K, mode, *R.IO_PAIRS[io]) if is_fast else (vecs, *R.IO_PAIRS[io]))
    want = {i for i in fast | generic if i[-2:] in set(R.IO_PAIRS.values())}
    assert want <= reached, sorted(want - reached)
    assert set(G.BWD_BF16_D) == {4 * l * v for l, v in R.BWD_FAST}
