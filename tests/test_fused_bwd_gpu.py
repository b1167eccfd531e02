"""GPU: f1 — the fused SS2D core under autograd (ops.FusedSS2DCore: x_proj GEMM + the state-saving pair sigma_ss2d_scan_fwd_save /
sigma_ss2d_scan_bwd_saved) against the composed path (CrossScan + einsums + the op-level scan kernels, itself pinned to the
reference's autograd goldens): output and EVERY gradient, kinds CROSS4 (SS2D) and SEQ2 (ConMB), ragged maps, 1 / 3 / auto
L-segments.  fp32-grade projections on both sides (TF32 off); bar 1e-3 of each tensor's scale.  Also: the state-saving forward's y
is the inference forward's, bit for bit."""
import numpy as np
import pytest
import torch

import procedural as P

pytestmark = pytest.mark.gpu
S = 51


def _params(K, D, N, R, tag):
    xpw = P.randn(S, tag + "/xpw", (K, R + 2 * N, D), D ** -0.5).cuda().requires_grad_(True)
    dtw = P.rand(S, tag + "/dtw", (K, D, R), -R ** -0.5, R ** -0.5).cuda().requires_grad_(True)
    dtb = P.rand(S, tag + "/dtb", (K, D), -5.0, -1.0).cuda().requires_grad_(True)
    Al = torch.log(P.rand(S, tag + "/A", (K * D, N), 0.5, N + 0.5)).cuda().requires_grad_(True)
    Ds = P.randn(S, tag + "/Ds", (K * D,), 0.2, 1.0).cuda().requires_grad_(True)
    return xpw, dtw, dtb, Al, Ds


def _cmp(name, got, ref, bar=1e-3):
    sc = float(ref.abs().max()) + 1e-20
    err = float((got - ref).abs().max()) / sc
    assert err <= bar, f"{name}: {err:.2e} of its scale"


@pytest.mark.parametrize("B,H,W,D,N,R", [(2, 6, 5, 64, 16, 2), (1, 30, 40, 128, 16, 8), (2, 9, 13, 64, 4, 4), (1, 17, 33, 192, 16, 6),
                                         (1, 40, 21, 64, 4, 4), (1, 30, 40, 768, 16, 24)])   # last: Sigma stage 2 (CTAS = 4 budget)
@pytest.mark.parametrize("split", [0, 1, 3])
def test_fused_core_cross4_matches_composed(B, H, W, D, N, R, split):
    from sigma_b200 import _lib, fused, ops
    torch.backends.cuda.matmul.allow_tf32 = False
    tag = f"fb4/{B}/{H}/{W}/{D}/{N}/{R}"
    xc0 = P.randn(S, tag + "/xc", (B, H * W, D)).cuda()
    wgt = P.randn(S, tag + "/w", (B, H * W, D)).cuda()
    pr = _params(4, D, N, R, tag)
    # composed reference: the reference's formulation on NCHW + op-level kernels
    x_ref = xc0.clone().requires_grad_(True)
    xn = x_ref.view(B, H, W, D).permute(0, 3, 1, 2).contiguous()
    y_ref = ops.cross_selective_scan(xn, pr[0], None, pr[1], pr[2], pr[3], pr[4], out_norm=lambda t: t)       # (B,H,W,D)
    (y_ref.reshape(B, H * W, D) * wgt).sum().backward()
    ref = [x_ref.grad.clone()] + [t.grad.clone() for t in pr]
    for t in pr:
        t.grad = None
    x_f = xc0.clone().requires_grad_(True)
    fused._FORCE_SPLIT = split
    try:
        y = ops.FusedSS2DCore.apply(x_f, pr[0], pr[1], pr[2], pr[3], pr[4], _lib.DIRS_CROSS4, H, W)
        (y * wgt).sum().backward()
    finally:
        fused._FORCE_SPLIT = 0
    _cmp("y", y.detach(), y_ref.detach().reshape(B, H * W, D))
    for nm, g, r in zip(["dxc", "dx_proj_weight", "ddt_projs_weight", "ddt_projs_bias", "dA_logs", "dDs"], [x_f.grad] + [t.grad for t in pr], ref):
        _cmp(f"{tag} split={split} {nm}", g, r)


@pytest.mark.parametrize("B,H,W,D,N,R", [(2, 6, 5, 64, 4, 2), (1, 15, 20, 128, 4, 12)])
@pytest.mark.parametrize("split", [0, 2])
def test_fused_core_seq2_matches_composed(B, H, W, D, N, R, split):
    from sigma_b200 import _lib, fused, ops
    torch.backends.cuda.matmul.allow_tf32 = False
    tag = f"fb2/{B}/{H}/{W}/{D}/{N}/{R}"
    L = H * W
    xr0, xe0 = P.randn(S, tag + "/xr", (B, L, D)).cuda(), P.randn(S, tag + "/xe", (B, L, D)).cuda()
    wgt = P.randn(S, tag + "/w", (B, 2 * L, D)).cuda()
    pr = _params(2, D, N, R, tag)
    xr, xe = xr0.clone().requires_grad_(True), xe0.clone().requires_grad_(True)
    nchw = lambda t: t.view(B, H, W, D).permute(0, 3, 1, 2).contiguous()
    y_r, y_e = ops.cross_selective_scan_multimodal_k2(nchw(xr), nchw(xe), pr[0], None, pr[1], pr[2], pr[3], pr[4],
                                                       out_norm1=lambda t: t, out_norm2=lambda t: t)
    y_ref = torch.cat([y_r.reshape(B, L, D), y_e.reshape(B, L, D)], dim=1)
    (y_ref * wgt).sum().backward()
    ref = [torch.cat([xr.grad, xe.grad], dim=1)] + [t.grad.clone() for t in pr]
    for t in pr:
        t.grad = None
    x_f = torch.cat([xr0, xe0], dim=1).clone().requires_grad_(True)
    fused._FORCE_SPLIT = split
    try:
        y = ops.FusedSS2DCore.apply(x_f, pr[0], pr[1], pr[2], pr[3], pr[4], _lib.DIRS_SEQ2, H, W)
        (y * wgt).sum().backward()
    finally:
        fused._FORCE_SPLIT = 0
    _cmp("y", y.detach(), y_ref.detach())
    for nm, g, r in zip(["dxc", "dx_proj_weight", "ddt_projs_weight", "ddt_projs_bias", "dA_logs", "dDs"], [x_f.grad] + [t.grad for t in pr], ref):
        _cmp(f"{tag} split={split} {nm}", g, r)


@pytest.mark.parametrize("kind_name,B,H,W,D,N,R", [("cross4", 2, 9, 13, 64, 4, 4), ("cross4", 1, 40, 21, 64, 4, 4), ("cross4", 1, 17, 33, 128, 16, 6),
                                                   ("seq2", 2, 7, 9, 64, 4, 3)])
@pytest.mark.parametrize("split", [0, 3])
def test_saving_forward_keeps_y_bitwise(kind_name, B, H, W, D, N, R, split):
    """the training forward (sigma_ss2d_scan_fwd_save) writes the y of the inference forward (sigma_ss2d_scan_fwd) bit for bit:
    keeping delta' and the block-start states changes nothing else"""
    from sigma_b200 import _lib, fused
    L_ = _lib.lib()
    kind = _lib.DIRS_CROSS4 if kind_name == "cross4" else _lib.DIRS_SEQ2
    K = 4 if kind_name == "cross4" else 2
    Lseq = H * W if kind_name == "cross4" else 2 * H * W
    tag = f"sv/{kind_name}/{B}/{H}/{W}/{D}/{N}/{R}"
    Cp = L_.sigma_ss2d_padded_cp(N, R)
    xc = P.randn(S, tag + "/xc", (B, Lseq, D)).cuda()
    xdbl = P.randn(S, tag + "/xdbl", (B, Lseq, K, Cp)).cuda()
    dtw = P.rand(S, tag + "/dtw", (K, D, R), -R ** -0.5, R ** -0.5).cuda()
    dtb = P.rand(S, tag + "/dtb", (K, D), -5.0, -1.0).cuda()
    A = -P.rand(S, tag + "/A", (K * D, N), 0.5, N + 0.5).cuda()
    Ds = P.randn(S, tag + "/Ds", (K * D,)).cuda()
    fused._FORCE_SPLIT = split
    try:
        y, _, _ = fused.ss2d_scan_save(kind, xc, xdbl, dtw, dtb, A, Ds, B, H, W, D, N, R, Cp)
        y0 = fused.ss2d_scan(kind, xc, xdbl, dtw, dtb, A, Ds, B, H, W, D, N, R, Cp)
    finally:
        fused._FORCE_SPLIT = 0
    assert torch.equal(y, y0), "the state-saving forward must not change y"
