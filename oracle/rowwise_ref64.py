"""fp64 references of the row-wise and decoder-tail kernels (sigma_b200/csrc/rowwise.cu) with a per-element error bound for each
fp32 output.  ORACLE — test infrastructure only.  Plain torch float64, device-agnostic; nothing here calls the library.

Operations (x a row of D channels; every kernel normalises with a divisor of D):
  layer_norm_ref64    LN(x) = (x - mean)/sqrt(var + eps)·gamma + beta, mean and var in two passes
  merge_norm_ref64    LN(sum_k y_k) [· SiLU(z)] [· gate[row // rows_per_batch]]   (sigma_merge_norm_gate_fwd, sigma_layernorm_fwd)
  patch_merge_gather64   the 2x2 gather of PatchMerging2D, quadrants (dh, dw) = (0,0), (1,0), (0,1), (1,1), zeros past odd H / W
  pixel_shuffle64     "b h w (p1 p2 c) -> b (h p1) (w p2) c" (PatchExpand)
  upsample2x_ref64    bilinear x2, align_corners=False, source index clamped at 0; upsample2x_norm_ref64 = LN of it
  head_ref64          the (NCLS, C) 1x1 projection of upsample2x_norm_ref64, NCHW
  pool_avgmax_ref64, pool_partial_ref64, scale_add_ref64, layernorm_bwd_ref64 (dx, dgamma, dbeta)

Lane layouts (*_plan, mirroring rowwise.cu's dispatch; tests/test_rowwise_ref64_cpu.py checks the tables against the built library):
a row is held by LPR lanes with V float4 each (fast kernels, D = 4·LPR·V) or by the 32 lanes of a warp with MAXV float4 slots
(generic kernels).  Lane l holds float4 number l + LPR·v.

Error bound.  u = 2^-24 (fp32 rounding to nearest).  First-order running-error analysis of the kernels' own fp32 operation order,
written out per step; every rounding contributes u times the magnitude of the value it rounds, an exact-operand product is
rounded once, and a compiler-contracted FMA rounds less often than the separate operations counted here.
  * K-direction sum: a = y_0 + y_1 + ... + y_{K-1} in order: |err a_i| <= (K-1)·u·sum_k |y_k,i| (= dx_i, the LN input error).
  * bilinear x2: (1-fh)·((1-fw)·a + fw·b) + fh·((1-fw)·c + fw·d); the weights are 0, 1/4, 3/4, 1 (exact).  Two products and a
    sum per inner bracket, one product per outer term and the outer sum: |err| <= 4u·M, M = sum of |weight·tap| (= dx_i).
  * row sum s: each lane adds its float4s as s += (x+y)+(z+w) (3 roundings per float4, then the running sum), V of them, then a
    log2(LPR)-step butterfly (fast) or a 5-step warp_sum (generic, MAXV slots).  Every partial sum is at most S = sum |x~_i|, so
    |err s| <= n_s·u·S + sum dx_i, n_s = 2 + V + log2(LPR) (generic: 2 + MAXV + 5).
  * mean m = s / D (IEEE division; the backward multiplies by fl(1/D): one more rounding): dm = |err s|/D + u|m|.
  * d_i = x~_i - m: |err d_i| = dd_i <= dx_i + dm + u|d_i|.
  * q = sum d~_i^2 in the order of s.  The mean's error is the same for every i and sum d_i = 0, so it enters q only to second
    order (D·dm^2): |err q| <= sum [2|d_i|(dx_i + u|d_i|) + dd_i^2] + (n_s + 1)·u·sum (|d_i| + dd_i)^2 (the squares, the sum).
    This is what amplifies a mean error by |mean|/sigma in a one-pass E[x^2] - E[x]^2, and why the two-pass kernels do not.
  * v = q/D + eps: dv = |err q|/D + 2u·v;  rstd = rsqrtf(v): relative error dv/(2v) + E_RSQRT (rsqrt.approx.f32, 2 ulp).
  * o = fmaf((x~ - m)·rstd, gamma, beta): |err o_i| <= |gamma|·(rstd·dd_i + |d_i|·rstd·(rel_rstd + u)) + u|o_i|.
  * · SiLU(z) = z / (1 + ex2(-z·log2e)) (__fdividef): relative error 2·E2 + u + 2u|z| (ex2.approx, __fdividef's 2 ulp, the
    1 + e, and the argument's product with a rounded log2e), then one product: err·|s| + |o s|(rel + u).  · gate: one product.
  * head: logit_k = sum_c o_c W_kc as an fmaf chain over a lane's 4·V channels, then the log2(LPR)-step butterfly (generic:
    4·MAXV channels, 5 steps): sum_c |W_kc|·err o_c + (4V + log2 LPR)·u·sum_c |o_c W_kc|.
  * pool slice sum: thread pr of a slice adds positions pr, pr + rows, ... (rows = 256 / (C/4) position rows), then the rows
    partial sums are added in order: (ceil(len/rows) + rows)·u·sum_slice |x|.  The max is exact.  pool_avgmax's mean adds the
    nslice partial sums (nslice·u) and divides (u).
  * scale_add: out = fmaf(a, sa, b·sb): u|b sb| + u|out| (a = NULL: u|out|).
  * layernorm_bwd: xhat = (x - m)·rstd, m1 = mean(gamma dy), m2 = mean(gamma dy xhat), dx = rstd·(gamma dy - m1 - xhat m2) with
    every product, sum and rounding of the body itemised the same way (layernorm_bwd_bound).  dgamma / dbeta sum B·L terms: each
    warp's fmaf chain over its rows (n_w of them, rigorous n_w·u per term), a fold over its 32/LPR sub-rows, then one atomic (or
    one term of the deterministic warp-order sum) per warp.  Over more than 16 roundings the bound uses the probabilistic model of
    Higham & Mary (SIAM J. Sci. Comput. 2019): n roundings of partial sums bounded by S err by at most 4·sqrt(n)·u·S, S = sum |terms|.
Every first-order bound is multiplied by SAFETY = 1.25 for the second-order products of the itemised errors (each below 1e-4 of
the first-order total on these inputs).  Every bound is per element; none is a fraction of a tensor's maximum.

bf16 instances (element pairs (f32, bf16): fp32 in, bf16 out; (bf16, bf16): bf16 y / z in, bf16 out; layernorm_bwd with bf16 x, dy, dx;
dwconv3x3_silu_tma_kernel<__nv_bfloat16>).  Every bf16 operand is widened exactly and all arithmetic is the fp32 kernel's, so the
inputs are rounded to bf16 first and the reference and its fp32 bound e are computed from those exact values: operand rounding
never enters the comparison.  A bf16 store rounds the kernel's fp32 value v, |v - ref| <= e, to nearest even, which moves it by at
most BF16_RN·|v| <= BF16_RN·(|ref| + e) (BF16_RN = 2^-8: 8 significand bits; bf16 has fp32's exponent range):
  * bf16_store_bound(ref, e) = e + BF16_RN·(|ref| + e), once per store; dgamma / dbeta of the bf16 backward stay fp32 (e alone).
A constant row of dyadic k/8 (exact in bf16) still normalises to beta exactly, stored as bf16(beta).  hard_rows(bf16=True) builds
the var_eps rows around a mean of order 2^-6, where bf16's spacing (<= 2^-14) still resolves a sigma of ~3e-3; at a mean of order
1 (spacing 2^-8) rounding would leave a few distinct values per row."""
import math

import torch

U = 2.0 ** -24
E_RSQRT = 2.0 ** -22      # rsqrtf / rsqrt.approx.f32: 2 ulp (CUDA C++ Programming Guide, mathematical functions)
E2 = 2.0 ** -22           # ex2.approx.f32 relative error (PTX ISA)
E_FDIV = 2.0 ** -22       # __fdividef: 2 ulp
SAFETY = 1.25
BF16_RN = 2.0 ** -8       # relative error of a round-to-nearest bf16 store (= oracle/ss2d_ref64.BF16_RN)
NUM_SMS = 132             # kNumSMs of common.cuh: the grid caps of layernorm_bwd and scale_add

# rowwise.cu's instantiation tables: (lanes per row, float4 per lane)
ROW_FAST = [(8, 2), (8, 3), (8, 4), (16, 3), (16, 4), (32, 3), (32, 4), (32, 6), (32, 8), (32, 12), (32, 16)]
ROW_FAST_K = (1, 2, 4)
MAXV_GENERIC = (1, 2, 4, 8, 16, 32)
# row_norm_launch's dispatch per element pair (y / z, out): mode -> the K with a fast instance, and the generic kernel's float4
# slots per lane (plain rows only, D <= 128·MAXV; e4m3 output holds the whole row in registers and stops at MAXV 8)
ROW_FAST_PAIRS = {
    ("f32", "f32"): {0: ROW_FAST_K, 1: (1,), 2: (1,)},
    ("f32", "bf16"): {0: (1,), 1: (1,)},
    ("f32", "f16"): {0: (1,), 1: (1,)},
    ("f32", "e4m3"): {0: (1,), 1: (1,)},
    ("bf16", "bf16"): {0: ROW_FAST_K},
    ("f16", "f16"): {0: ROW_FAST_K},
    ("bf16", "e4m3"): {0: (1, 4)},
}
ROW_GENERIC_MAXV = {pair: MAXV_GENERIC[:4] if pair[1] == "e4m3" else MAXV_GENERIC for pair in ROW_FAST_PAIRS}
ROW_E4M3_K = (1, 4)        # the only K of e4m3 output, fast or generic
# the integer element labels of tests/test_rowwise_fp64_gpu.py
IO_PAIRS = {0: ("f32", "f32"), 1: ("f32", "bf16"), 2: ("bf16", "bf16")}
HEAD_FAST = [(8, 2), (8, 3), (8, 4), (16, 3), (16, 4)]
HEAD_FAST_MAX_NCLS = 24
HEAD_NCLS = [2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 16, 19, 20, 21, 37, 40, 41]
BWD_FAST = [(8, 1), (8, 2), (8, 3), (8, 4), (16, 3), (16, 4), (32, 3), (32, 4), (32, 6), (32, 8), (32, 12)]


# ---------------------------------------------------------------- launch plans (lane layouts)
def _maxv(nvec, cap=32):
    for mv in MAXV_GENERIC:
        if mv <= cap and nvec <= 32 * mv:
            return mv
    raise ValueError(f"{4 * nvec} channels: no generic instantiation")


def row_plan(D, K=1, mode=0, io=0):
    """(lanes, float4 per lane, fast) of row_norm_launch for D channels, K directions, mode 0 / 1 (gather) / 2 (pixel shuffle) and
    element pair io (a key of ROW_FAST_PAIRS, or an IO_PAIRS label)"""
    pair = IO_PAIRS.get(io, io)
    if pair[1] == "e4m3" and K not in ROW_E4M3_K:
        raise ValueError(f"e4m3 output: K={K} has no instantiation")
    nvec = D // 4
    for lpr, v in ROW_FAST:
        if nvec == lpr * v and K in ROW_FAST_PAIRS[pair].get(mode, ()):
            return lpr, v, True
    if mode != 0:
        raise ValueError(f"mode {mode}: D={D} has no fast instantiation")
    return 32, _maxv(nvec, cap=ROW_GENERIC_MAXV[pair][-1]), False


def head_plan(C, ncls):
    """(lanes, float4 per lane, fast) of upsample2x_norm_launch; ncls 0 = the LayerNorm-only kernel"""
    nvec = C // 4
    if 0 < ncls <= HEAD_FAST_MAX_NCLS:
        for lpr, v in HEAD_FAST:
            if nvec == lpr * v:
                return lpr, v, True
    return 32, _maxv(nvec, cap=8), False


def bwd_plan(rows, D):
    """(lanes, float4 per lane, warps in the grid, grid-stride steps per warp) of layernorm_bwd_launch"""
    nvec = D // 4
    lpr, v = next((l, v) for l, v in BWD_FAST if nvec == l * v)
    glpr = 32 if nvec % 32 == 0 and nvec >= 96 else 16 if nvec % 16 == 0 and nvec >= 48 else 8   # layernorm_bwd_grid's rule
    nsteps_g = -(-rows // (32 // glpr))
    grid = max(1, min(NUM_SMS * 8, -(-nsteps_g // 32)))
    nw = grid * 8
    nsteps = -(-rows // (32 // lpr))
    return lpr, v, nw, -(-nsteps // nw)


def sum_depth(plan):
    """n_s: roundings on the way from one float4 to the row sum (the butterfly of the generic kernels is a 32-lane warp_sum)"""
    lanes, vecs = plan[0], plan[1]
    return 2 + vecs + int(math.log2(lanes))


def dot_depth(plan):
    lanes, vecs = plan[0], plan[1]
    return 4 * vecs + int(math.log2(lanes))


def _gt(n):
    """relative bound of the accumulation error of n roundings (rigorous up to 16, Higham & Mary above)"""
    return U * (n if n <= 16 else 4.0 * math.sqrt(n))


def bound_fraction(got, ref, bound):
    """largest |got - ref| / bound; an element whose bound is 0 must be exact"""
    err = (got.to(ref.device, torch.float64) - ref).abs()
    frac = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    return float(frac.max()) if frac.numel() else 0.0


def bf16_store_bound(ref, e):
    """bound of a bf16 store of a value the fp32 bound e holds to ref (module docstring): e + BF16_RN·(|ref| + e)"""
    return e + BF16_RN * (_f(ref).abs() + e)


def _f(t):
    return t.detach().to(torch.float64) if t is not None else None


# ---------------------------------------------------------------- references
def layer_norm_ref64(x, gamma, beta, eps):
    x = _f(x)
    d = x - x.mean(-1, keepdim=True)
    return d / torch.sqrt((d * d).mean(-1, keepdim=True) + eps) * _f(gamma) + _f(beta)


def silu64(z):
    z = _f(z)
    return z * torch.sigmoid(z)


def gate_rows(gate, rows, rows_per_batch):
    """the gate row of every output row: gate[row // rows_per_batch]"""
    idx = torch.arange(rows, device=gate.device) // rows_per_batch
    return _f(gate)[idx]


def merge_norm_ref64(y, gamma, beta, eps, z=None, gate=None, rows_per_batch=None):
    """y (K, rows, D): LN(sum_k y_k) [· SiLU(z)] [· gate[row // rows_per_batch]]"""
    o = layer_norm_ref64(_f(y).sum(0), gamma, beta, eps)
    if z is not None:
        o = o * silu64(z)
    if gate is not None:
        o = o * gate_rows(gate, o.shape[0], rows_per_batch)
    return o


def patch_merge_gather64(x):
    """(B, H, W, C) -> (B·ceil(H/2)·ceil(W/2), 4C): quadrants (0,0), (1,0), (0,1), (1,1), zeros past odd H / W"""
    x = _f(x)
    B, H, W, C = x.shape
    xp = torch.nn.functional.pad(x, (0, 0, 0, W % 2, 0, H % 2))
    return torch.cat([xp[:, 0::2, 0::2], xp[:, 1::2, 0::2], xp[:, 0::2, 1::2], xp[:, 1::2, 1::2]], -1).reshape(-1, 4 * C)


def pixel_shuffle64(y, B, H, W):
    """rows of 4C = (p1 p2 c) at pixel (b, h, w) -> (B, 2H, 2W, C)"""
    y = _f(y)
    C = y.shape[-1] // 4
    return y.reshape(B, H, W, 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B, 2 * H, 2 * W, C)


def bilinear2x_taps(n, device=None):
    """per output index o of 2n: (i0, i1, w1) with src = max((o + 0.5)/2 - 0.5, 0), i0 = floor(src), i1 = min(i0 + 1, n - 1)"""
    s = ((torch.arange(2 * n, dtype=torch.float64, device=device) + 0.5) * 0.5 - 0.5).clamp_min(0.0)
    i0 = s.floor().long()
    return i0, (i0 + 1).clamp_max(n - 1), s - i0


def _bilinear(x, H, W):
    h0, h1, fh = bilinear2x_taps(H, x.device)
    w0, w1, fw = bilinear2x_taps(W, x.device)
    fh, fw = fh[:, None, None], fw[:, None]
    r0, r1 = x[:, h0], x[:, h1]
    return (1 - fh) * ((1 - fw) * r0[:, :, w0] + fw * r0[:, :, w1]) + fh * ((1 - fw) * r1[:, :, w0] + fw * r1[:, :, w1])


def upsample2x_ref64(x):
    """(B, H, W, C) -> (B, 2H, 2W, C) bilinear, align_corners=False"""
    x = _f(x)
    return _bilinear(x, x.shape[1], x.shape[2])


def upsample2x_norm_ref64(x, gamma, beta, eps):
    return layer_norm_ref64(upsample2x_ref64(x), gamma, beta, eps)


def head_ref64(x, gamma, beta, eps, wcls):
    """(B, H, W, C) -> NCHW logits (B, NCLS, 2H, 2W) of the (NCLS, C) projection of upsample2x_norm_ref64"""
    o = upsample2x_norm_ref64(x, gamma, beta, eps)
    return torch.einsum("bhwc,kc->bkhw", o, _f(wcls))


def pool_avgmax_ref64(x):
    """(B, L, C) -> (mean, max) over L, each (B, C)"""
    x = _f(x)
    return x.mean(1), x.amax(1)


def pool_slices(L, nslice):
    """[l0, l1) of every slice: ceil(L / nslice) positions each, the trailing ones possibly empty"""
    per = -(-L // nslice)
    return [(min(L, s * per), min(L, (s + 1) * per)) for s in range(nslice)]


def pool_partial_ref64(x, nslice):
    """(B, L, C) -> (B, nslice, 2, C): the sum and the max over each slice (0 and -inf for an empty slice)"""
    x = _f(x)
    B, L, C = x.shape
    out = torch.empty((B, nslice, 2, C), dtype=torch.float64, device=x.device)
    for s, (l0, l1) in enumerate(pool_slices(L, nslice)):
        out[:, s, 0] = x[:, l0:l1].sum(1)
        out[:, s, 1] = x[:, l0:l1].amax(1) if l1 > l0 else -math.inf
    return out


def scale_add_ref64(a, sa, b, sb, rows_per_batch):
    """a (rows, C) · sa[row // rows_per_batch] + b · sb; a = None: b · sb"""
    out = _f(b) * _f(sb)
    if a is not None:
        out = out + _f(a) * gate_rows(sa, a.shape[0], rows_per_batch)
    return out


def layernorm_bwd_ref64(x, dy, gamma, eps):
    """(rows, D) -> dx, dgamma, dbeta of LN(x)·gamma + beta"""
    x, dy, g = _f(x), _f(dy), _f(gamma)
    d = x - x.mean(-1, keepdim=True)
    r = 1.0 / torch.sqrt((d * d).mean(-1, keepdim=True) + eps)
    xh = d * r
    a = g * dy
    dx = r * (a - a.mean(-1, keepdim=True) - xh * (a * xh).mean(-1, keepdim=True))
    return dx, (dy * xh).sum(0), dy.sum(0)


# ---------------------------------------------------------------- bounds
def _ln_err(x, dx, gamma, beta, eps, n_s, recip_mul=False):
    """the first-order analysis of the module docstring: (o, err o, d, dd, rstd, rel rstd), x the exact LN input (fp64) and
    dx the bound of the kernel's error in it.  recip_mul: the mean and variance are multiplied by fl(1/D) (layernorm_bwd)"""
    D = x.shape[-1]
    div_u = 2 * U if recip_mul else U
    S = (x.abs() + dx).sum(-1, keepdim=True)
    m = x.mean(-1, keepdim=True)
    es = n_s * U * S + dx.sum(-1, keepdim=True)
    dm = es / D + div_u * m.abs()
    d = x - m
    dd = dx + dm + U * d.abs()
    eq = (2 * d.abs() * (dx + U * d.abs()) + dd * dd).sum(-1, keepdim=True) + (n_s + 1) * U * ((d.abs() + dd) ** 2).sum(-1, keepdim=True)
    v = (d * d).mean(-1, keepdim=True) + eps
    dv = eq / D + (div_u + U) * v
    r = 1.0 / torch.sqrt(v)
    rel_r = dv / (2 * v) + E_RSQRT
    g = _f(gamma)
    o = d * r * g + _f(beta)
    eo = g.abs() * (r * dd + d.abs() * r * (rel_r + U)) + U * o.abs()
    return o, eo, d, dd, r, rel_r


def _silu_gate(o, eo, z, gate, rows_per_batch):
    if z is not None:
        z = _f(z)
        s = silu64(z)
        rel = 2 * E2 + U + 2 * U * z.abs()
        eo = eo * s.abs() + (o * s).abs() * (rel + U)
        o = o * s
    if gate is not None:
        gr = gate_rows(gate, o.shape[0], rows_per_batch)
        o = o * gr
        eo = eo * gr.abs() + U * o.abs()
    return o, eo


def merge_norm_bound(y, gamma, beta, eps, plan, z=None, gate=None, rows_per_batch=None):
    """bound of sigma_merge_norm_gate_fwd / sigma_layernorm_fwd (K = 1) / the gather and pixel-shuffle modes (y = the rows they
    normalise): y (K, rows, D), plan = row_plan(...)"""
    y = _f(y)
    K = y.shape[0]
    x = y.sum(0)
    dx = (K - 1) * U * y.abs().sum(0)
    o, eo, *_ = _ln_err(x, dx, gamma, beta, eps, sum_depth(plan))
    _, eo = _silu_gate(o, eo, z, gate, rows_per_batch)
    return SAFETY * eo


def layer_norm_bound(x, gamma, beta, eps, plan):
    return merge_norm_bound(_f(x)[None], gamma, beta, eps, plan)


def _bilinear_err(x):
    xa = _f(x)
    return _bilinear(xa, xa.shape[1], xa.shape[2]), 4 * U * _bilinear(xa.abs(), xa.shape[1], xa.shape[2])


def upsample2x_bound(x):
    return SAFETY * _bilinear_err(x)[1]


def upsample2x_norm_bound(x, gamma, beta, eps, plan):
    up, dx = _bilinear_err(x)
    return SAFETY * _ln_err(up, dx, gamma, beta, eps, sum_depth(plan))[1]


def head_bound(x, gamma, beta, eps, wcls, plan):
    """bound of every logit (B, NCLS, 2H, 2W)"""
    up, dx = _bilinear_err(x)
    o, eo, *_ = _ln_err(up, dx, gamma, beta, eps, sum_depth(plan))
    wa = _f(wcls).abs()
    return SAFETY * (torch.einsum("bhwc,kc->bkhw", eo, wa) + dot_depth(plan) * U * torch.einsum("bhwc,kc->bkhw", o.abs(), wa))


def pool_rows(C):
    """position rows of pool_avgmax_partial_kernel (256 threads over C/4 float4 columns)"""
    return 256 // (C // 4)


def _pool_partial_err(x, nslice):
    B, L, C = x.shape
    rows = pool_rows(C)
    out = torch.zeros((B, nslice, C), dtype=torch.float64, device=x.device)
    for s, (l0, l1) in enumerate(pool_slices(L, nslice)):
        out[:, s] = (-(-(l1 - l0) // rows) + rows) * U * x[:, l0:l1].abs().sum(1)
    return out


def pool_partial_bound(x, nslice):
    """bound of the slice sums of pool_partial_ref64 (B, nslice, C); the maxima must be exact"""
    return SAFETY * _pool_partial_err(_f(x), nslice)


def pool_mean_bound(x, nslice):
    """bound of pool_avgmax's mean: the slice sums, their fp32 sum over nslice, the division by L"""
    x = _f(x)
    L = x.shape[1]
    tot = _pool_partial_err(x, nslice).sum(1)
    return SAFETY * (tot / L + nslice * U * x.abs().sum(1) / L + U * x.mean(1).abs())


def scale_add_bound(a, sa, b, sb, rows_per_batch):
    bs = (_f(b) * _f(sb)).abs()
    out = scale_add_ref64(a, sa, b, sb, rows_per_batch).abs()
    return SAFETY * (U * out + (U * bs if a is not None else 0.0))


def layernorm_bwd_bound(x, dy, gamma, eps):
    """bounds of (dx, dgamma, dbeta) of layernorm_bwd for (rows, D) x and dy, from bwd_plan's lane layout and grid"""
    x, dy, g = _f(x), _f(dy), _f(gamma)
    rows, D = x.shape
    lpr, v, nw, nsteps_w = bwd_plan(rows, D)
    n_s = sum_depth((lpr, v))
    zero = torch.zeros_like(x)
    _, _, d, dd, r, rel_r = _ln_err(x, zero, g, torch.zeros_like(g), eps, n_s, recip_mul=True)
    xh = d * r
    dxh = r * dd + xh.abs() * (rel_r + U)                                # xv -= mean; xv *= rstd
    a = g * dy
    da = U * a.abs()
    m1 = a.mean(-1, keepdim=True)
    dm1 = (n_s * U * a.abs().sum(-1, keepdim=True) + da.sum(-1, keepdim=True)) / D + 2 * U * m1.abs()
    t = a * xh
    m2 = t.mean(-1, keepdim=True)
    et = a.abs() * dxh + xh.abs() * da + U * t.abs()
    dm2 = (et.sum(-1, keepdim=True) + n_s * U * t.abs().sum(-1, keepdim=True)) / D + 2 * U * m2.abs()
    inner = a - m1 - xh * m2
    ei = da + dm1 + m2.abs() * dxh + xh.abs() * dm2 + U * ((a - m1).abs() + (xh * m2).abs() + inner.abs())
    edx = r * ei + inner.abs() * r * (rel_r + U)
    n_acc = nsteps_w + int(math.log2(32 // lpr)) + nw
    tg = dy * xh
    edg = (dy.abs() * dxh).sum(0) + U * tg.abs().sum(0) + _gt(n_acc) * tg.abs().sum(0)
    edb = _gt(n_acc) * dy.abs().sum(0)
    return SAFETY * edx, SAFETY * edg, SAFETY * edb


# ---------------------------------------------------------------- inputs
ROW_FAMILIES = ("ordinary", "large_mean", "var_eps", "constant", "outlier")


def hard_rows(seed, rows, D, eps=1e-5, families=ROW_FAMILIES, device="cpu", bf16=False):
    """(rows, D) fp32 on `device` (its own generator, seeded), row i of family families[i % len(families)]:
      ordinary     N(0, 1) scaled by a per-row sigma in [0.5, 2]
      large_mean   mean = ±(30..100)·sigma: the one-pass variance's cancellation
      var_eps      sigma^2 in [0.5, 2]·eps around a mean of order 1 (bf16: of order 2^-6): where eps's placement matters
      constant     a dyadic constant k/8 (every partial sum exact): the output must be beta exactly
      outlier      N(0, 1) with one channel at ±(20..40)
    bf16: the same draws, var_eps's mean scaled by 2^-6, returned rounded to bf16 (module docstring)"""
    g = torch.Generator(device=device).manual_seed(seed)
    kw = dict(generator=g, device=device)
    n = torch.randn(rows, D, dtype=torch.float32, **kw)
    u = lambda lo, hi: torch.rand(rows, 1, **kw) * (hi - lo) + lo
    sign = torch.where(torch.rand(rows, 1, **kw) < 0.5, -1.0, 1.0)
    fam = torch.arange(rows, device=device) % len(families)
    out = torch.empty(rows, D, dtype=torch.float32, device=device)
    sig, sig_eps = u(0.5, 2.0), torch.sqrt(u(0.5, 2.0) * eps)
    mu, big = torch.randn(rows, 1, **kw), sign * u(30.0, 100.0)
    kconst = torch.randint(-64, 65, (rows, 1), **kw).float() / 8
    spike_at = torch.randint(0, D, (rows,), **kw)
    spike = sign[:, 0] * u(20.0, 40.0)[:, 0]
    for f, name in enumerate(families):
        m = fam == f
        if name == "ordinary":
            out[m] = n[m] * sig[m]
        elif name == "large_mean":
            out[m] = (n[m] + big[m]) * sig[m]
        elif name == "var_eps":
            out[m] = mu[m] * (2.0 ** -6 if bf16 else 1.0) + n[m] * sig_eps[m]
        elif name == "constant":
            out[m] = kconst[m].expand(-1, D)
        elif name == "outlier":
            o = n[m]
            o[torch.arange(o.shape[0], device=device), spike_at[m]] = spike[m]
            out[m] = o
        else:
            raise ValueError(name)
    return out.to(torch.bfloat16) if bf16 else out


def constant_rows(rows, families=ROW_FAMILIES, device="cpu"):
    """mask of the rows hard_rows makes constant"""
    if "constant" not in families:
        return torch.zeros(rows, dtype=torch.bool, device=device)
    return torch.arange(rows, device=device) % len(families) == families.index("constant")


def affine(seed, D):
    """LayerNorm weight of mixed sign (N(0, 1)) and bias N(0, 0.5^2), fp32 on the CPU"""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(D, generator=g), 0.5 * torch.randn(D, generator=g)


def pool_input(seed, B, L, C, device="cpu"):
    """(B, L, C) fp32 on `device`: N(1, 1) (a mean away from 0), and every third channel negative everywhere with its maximum at
    the last position L - 1 (the last position of the last non-empty slice), so a max that starts at 0 cannot pass"""
    g = torch.Generator(device=device).manual_seed(seed)
    x = torch.randn(B, L, C, generator=g, device=device) + 1.0
    neg = torch.arange(C, device=device) % 3 == 1
    x[:, :, neg] = -x[:, :, neg].abs() - 0.5
    x[:, L - 1, neg] = -0.25
    return x
