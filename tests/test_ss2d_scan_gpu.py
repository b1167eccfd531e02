"""GPU: the fused channels-last multi-direction scan (sigma_ss2d_scan_fwd) and the row-wise kernels
through the C-ABI, against the CPU oracle built from the reference's own definitions:
direction maps vmamba.py:80-121 / 123-163, dt_proj vmamba.py:199, selective_scan_ref."""
import ctypes

import numpy as np
import pytest
import torch

import procedural as P
from helpers import assert_close
from oracle import scan_oracle

pytestmark = pytest.mark.gpu
S = 21


def _dir_index(kind, H, W):
    """position visited at scan step l, per direction (SURVEY.md App. A 'Direction maps')."""
    L = H * W
    if kind == "cross4":
        row = np.arange(L)
        col = (np.arange(H)[None, :] * W + np.arange(W)[:, None]).reshape(-1)      # l1 = w·H + h -> h·W + w
        return [row, col, row[::-1].copy(), col[::-1].copy()]
    if kind == "seq2":
        a = np.arange(2 * L)
        return [a, a[::-1].copy()]
    return [np.arange(L)]


def _reference(kind, xc, xdbl, dtw, dtb, A, Ds, H, W, N, R):
    xc, xdbl, dtw, dtb, A, Ds = (t.numpy() for t in (xc, xdbl, dtw, dtb, A, Ds))
    Bt, Ls, D = xc.shape
    idx = _dir_index(kind, H, W)
    K = len(idx)
    y = np.zeros((K, Bt, Ls, D), np.float32)
    if kind == "cross":
        half = Bt // 2
        for m in range(2):
            sl = slice(m * half, (m + 1) * half)
            osl = slice((1 - m) * half, (2 - m) * half)
            u = xc[sl].transpose(0, 2, 1)                                             # (b, D, L)
            dt = np.einsum("blr,dr->bdl", xdbl[sl, :, 0, 2 * N:2 * N + R], dtw[m])
            Bm = xdbl[sl, :, 0, 0:N].transpose(0, 2, 1)[:, None]
            Cm = xdbl[osl, :, 0, N:2 * N].transpose(0, 2, 1)[:, None]                   # C of the other modality
            o = scan_oracle.scan_fwd(u, dt, A[m * D:(m + 1) * D], Bm, Cm, Ds[m * D:(m + 1) * D], dtb[m], True)
            y[0, sl] = o.transpose(0, 2, 1)
        return y
    us, dts, Bs, Cs = [], [], [], []
    for k, ix in enumerate(idx):
        us.append(xc[:, ix].transpose(0, 2, 1))
        dts.append(np.einsum("blr,dr->bdl", xdbl[:, ix, k, 2 * N:2 * N + R], dtw[k]))
        Bs.append(xdbl[:, ix, k, 0:N].transpose(0, 2, 1))
        Cs.append(xdbl[:, ix, k, N:2 * N].transpose(0, 2, 1))
    u = np.concatenate(us, 1)
    dt = np.concatenate(dts, 1)
    o = scan_oracle.scan_fwd(u, dt, A, np.stack(Bs, 1), np.stack(Cs, 1), Ds, dtb.reshape(-1), True)
    for k, ix in enumerate(idx):
        y[k][:, ix] = o[:, k * D:(k + 1) * D].transpose(0, 2, 1)
    return y


CASES = [  # kind, B(images), H, W, D, N, R
    ("cross4", 2, 6, 5, 64, 16, 2), ("cross4", 1, 15, 20, 192, 16, 6), ("cross4", 2, 40, 33, 96, 4, 6),
    ("cross4", 1, 30, 40, 80, 16, 12), ("cross4", 1, 7, 9, 768, 4, 24), ("cross4", 1, 9, 13, 128, 8, 5),
    ("seq2", 2, 6, 5, 64, 4, 2), ("seq2", 1, 30, 41, 384, 4, 12), ("cross", 2, 6, 5, 64, 4, 2), ("cross", 1, 31, 40, 192, 4, 6),
    ("cross4", 1, 10, 12, 64, 16, 48), ("cross4", 1, 10, 12, 64, 4, 64),
    ("cross4", 1, 30, 40, 768, 16, 24), ("cross4", 2, 30, 40, 768, 16, 24),     # Sigma stage 2: the CTAS = 4 register budget
]


@pytest.mark.parametrize("kind,B,H,W,D,N,R", CASES)
@pytest.mark.parametrize("split", [0, 1, 3])
def test_fused_scan_matches_oracle(kind, B, H, W, D, N, R, split):
    from sigma_b200 import _lib, fused
    L = H * W
    Kx = {"cross4": 4, "seq2": 2, "cross": 1}[kind]
    Kw = 2 if kind == "cross" else Kx
    Bt = 2 * B if kind == "cross" else B
    Ls = 2 * L if kind == "seq2" else L
    Cp = _lib.lib().sigma_ss2d_padded_cp(N, R)
    tag = f"{kind}/{B}/{H}/{W}/{D}/{N}/{R}"
    xc = P.randn(S, tag + "/xc", (Bt, Ls, D))
    xdbl = P.randn(S, tag + "/xdbl", (Bt, Ls, Kx, Cp))
    xdbl[..., 2 * N + R:] = 0.0                                   # zero padding columns, as the packed x_proj produces
    dtw = P.rand(S, tag + "/dtw", (Kw, D, R), -R ** -0.5, R ** -0.5)
    dtb = P.rand(S, tag + "/dtb", (Kw, D), -6.0, -1.0)
    A = -P.rand(S, tag + "/A", (Kw * D, N), 0.3, N + 0.5)
    Ds = P.randn(S, tag + "/Ds", (Kw * D,))
    ref = _reference(kind, xc, xdbl, dtw, dtb, A, Ds, H, W, N, R)
    kid = {"cross4": _lib.DIRS_CROSS4, "seq2": _lib.DIRS_SEQ2, "cross": _lib.DIRS_CROSS}[kind]
    fused._FORCE_SPLIT = split
    try:
        y = fused.ss2d_scan(kid, xc.cuda(), xdbl.cuda(), dtw.cuda(), dtb.cuda(), A.cuda(), Ds.cuda(), Bt, H, W, D, N, R, Cp)
        torch.cuda.synchronize()
    finally:
        fused._FORCE_SPLIT = 0
    scale = float(np.abs(ref).max())
    assert_close(y, ref, 6e-4, 1e-3 * scale, f"{tag} split={split}")


@pytest.mark.parametrize("kind,B,H,W,D,N,R", [c for c in CASES if c[5] == 16] + [
    ("cross4", 1, 10, 12, 64, 16, 16), ("cross4", 1, 10, 12, 64, 16, 32), ("cross4", 1, 10, 12, 64, 16, 64)])
def test_fused_scan_ctas4_budget_matches_oracle(kind, B, H, W, D, N, R, monkeypatch):
    """The second register budget of the d_state-16 scan (`CTAS = 4` of ss2d_scan_kernel; ss2d_pick_ctas runs it only at
    dt_rank 17..24), forced with SIGMA_SCAN_CTAS=4 at every padded dt_rank (4, 8, 12, 16, 24, 32, 48, 64)."""
    monkeypatch.setenv("SIGMA_SCAN_CTAS", "4")
    test_fused_scan_matches_oracle(kind, B, H, W, D, N, R, 0)


@pytest.mark.parametrize("rows,C", [(7, 32), (100, 96), (33, 192), (5, 768), (9, 3072), (3, 4096)])
def test_layernorm(rows, C):
    from sigma_b200 import fused
    x = P.randn(S, f"ln/{rows}/{C}", (rows, C), 2.0, 0.5)
    ln = torch.nn.LayerNorm(C)
    with torch.no_grad():
        ln.weight.copy_(P.randn(S, "ln/w", (C,), 0.1, 1.0))
        ln.bias.copy_(P.randn(S, "ln/b", (C,), 0.1))
        ref = ln(x)
        got = fused.layernorm(x.cuda(), ln.cuda())
    assert_close(got, ref, 1e-5, 2e-5, f"layernorm {rows}x{C}")


@pytest.mark.parametrize("B,H,W,D", [(2, 6, 5, 64), (1, 15, 20, 192), (3, 1, 7, 8), (1, 9, 1, 132)])
def test_dwconv_silu(B, H, W, D):
    from sigma_b200 import fused
    conv = torch.nn.Conv2d(D, D, 3, padding=1, groups=D)
    xz = P.randn(S, f"dw/{B}/{H}/{W}/{D}", (B, H, W, 2 * D))            # x is the first half of [x | z] rows
    with torch.no_grad():
        conv.weight.copy_(P.randn(S, "dw/w", (D, 1, 3, 3), 0.4))
        conv.bias.copy_(P.randn(S, "dw/b", (D,), 0.2))
        ref = torch.nn.functional.silu(conv(xz[..., :D].permute(0, 3, 1, 2))).permute(0, 2, 3, 1)
        out = torch.empty((B, H * W, D), device="cuda")
        fused.dwconv3x3_silu(xz.cuda(), 2 * D, H * W * 2 * D, conv.cuda(), out, H * W * D, B, H, W, D)
    assert_close(out.view(B, H, W, D), ref, 1e-5, 1e-5, "dwconv+silu")


def test_merge_norm_gate():
    from sigma_b200 import fused
    K, B, L, D = 4, 2, 37, 192
    y = P.randn(S, "mng/y", (K, B * L, D))
    z = P.randn(S, "mng/z", (B * L, 2 * D))
    gate = P.rand(S, "mng/g", (B, D))
    ln = torch.nn.LayerNorm(D)
    with torch.no_grad():
        ln.weight.copy_(P.randn(S, "mng/w", (D,), 0.1, 1.0))
        ln.bias.copy_(P.randn(S, "mng/b", (D,), 0.1))
        ref = ln(y.sum(0)) * torch.nn.functional.silu(z[:, D:]) * gate.repeat_interleave(L, 0)
        out = torch.empty((B * L, D), device="cuda")
        zc = z.cuda()
        fused.merge_norm_gate(y.cuda(), K, B * L * D, L * D, ln.cuda(), ctypes.c_void_p(zc.data_ptr() + 4 * D), 2 * D,
                              gate.cuda(), out, L * D, D, B * L, L, D)
    assert_close(out, ref, 2e-5, 5e-5, "merge+norm+gate")


@pytest.mark.parametrize("B,H,W,C,ncls", [(2, 5, 7, 32, 0), (1, 30, 40, 192, 0), (2, 6, 4, 96, 9), (1, 15, 20, 32, 5), (1, 3, 3, 128, 40),
                                          (3, 7, 5, 96, 9), (2, 9, 11, 128, 9), (1, 13, 3, 64, 2), (1, 6, 5, 192, 19), (1, 4, 4, 256, 12)])
def test_upsample2x_norm_and_head(B, H, W, C, ncls):
    from sigma_b200 import fused
    x = P.randn(S, f"up/{B}/{H}/{W}/{C}", (B, H, W, C))
    ln = torch.nn.LayerNorm(C)
    conv = torch.nn.Conv2d(C, max(ncls, 1), 1, bias=False)
    with torch.no_grad():
        ln.weight.copy_(P.randn(S, "up/w", (C,), 0.1, 1.0))
        ln.bias.copy_(P.randn(S, "up/b", (C,), 0.1))
        conv.weight.copy_(P.randn(S, "up/cw", tuple(conv.weight.shape), C ** -0.5))
        up = torch.nn.functional.interpolate(x.permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=False)
        ref = ln(up.permute(0, 2, 3, 1))
        if ncls:
            ref = conv(ref.permute(0, 3, 1, 2))
            got = fused.upsample2x_norm_head(x.cuda(), ln.cuda(), conv.cuda())
        else:
            got = fused.upsample2x_norm(x.cuda(), ln.cuda())
    assert_close(got, ref, 2e-5, 5e-5, f"upsample2x_norm ncls={ncls}")


@pytest.mark.parametrize("B,H,W,C", [(2, 5, 7, 32), (1, 30, 40, 96), (3, 1, 1, 8)])
def test_upsample2x_plain(B, H, W, C):
    """w = b = NULL: plain bilinear x2 (FinalUpsample_X4's first interpolate, MambaDecoder.py:92)."""
    from sigma_b200 import fused
    x = P.randn(S, f"upp/{B}/{H}/{W}/{C}", (B, H, W, C))
    ref = torch.nn.functional.interpolate(x.permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=False)
    got = fused.upsample2x_norm(x.cuda(), None)
    assert_close(got, ref.permute(0, 2, 3, 1), 1e-6, 1e-6, "upsample2x plain")


@pytest.mark.parametrize("B,H,W,C", [(2, 6, 8, 96), (1, 7, 5, 96), (2, 15, 20, 192), (1, 3, 3, 128), (1, 1, 1, 32)])
def test_patch_merging_fused(B, H, W, C):
    """PatchMerging2D (vmamba.py:619-636) incl. odd H / W: gather + LayerNorm kernel + wgmma GEMM vs the composed module."""
    from sigma_b200 import fused, modules as M
    m = M.PatchMerging2D(C, 2 * C).cuda()
    with torch.no_grad():
        for n, prm in m.named_parameters():
            prm.copy_(P.randn(S, f"pm/{C}/{n}", tuple(prm.shape), 0.2 if prm.dim() > 1 else 0.1, 1.0 if n.endswith("norm.weight") else 0.0))
        x = P.randn(S, f"pm/x/{B}/{H}/{W}/{C}", (B, H, W, C)).cuda()
        with M.composed_path():
            ref = m(x)
        got = fused.patch_merging(m, x)
    assert_close(got, ref, 5e-3, 1e-2, "patch_merging (tf32 GEMM)")
    # the LayerNorm'd gather alone, exactly
    H2, W2 = (H + 1) // 2, (W + 1) // 2
    xp = torch.nn.functional.pad(x, (0, 0, 0, W % 2, 0, H % 2))
    cat = torch.cat([xp[:, 0::2, 0::2], xp[:, 1::2, 0::2], xp[:, 0::2, 1::2], xp[:, 1::2, 1::2]], -1)
    xn = torch.empty((B * H2 * W2, 4 * C), device="cuda")
    from sigma_b200 import _lib
    _lib.check(_lib.lib().sigma_patch_merge_norm_fwd(x.data_ptr(), m.norm.weight.data_ptr(), m.norm.bias.data_ptr(), xn.data_ptr(),
                                                      B, H, W, C, float(m.norm.eps), torch.cuda.current_stream().cuda_stream), "pm")
    assert_close(xn.view(B, H2, W2, 4 * C), m.norm(cat), 2e-5, 5e-5, "patch merge gather + LN")


@pytest.mark.parametrize("B,H,W,C", [(2, 3, 5, 192), (1, 15, 20, 384), (1, 2, 2, 768), (1, 1, 3, 256)])
def test_patch_expand_fused(B, H, W, C):
    """PatchExpand (MambaDecoder.py:12-30): Linear C->2C, pixel shuffle, LayerNorm(C/2); the shuffle is the store address."""
    from sigma_b200 import fused, modules as M
    m = M.PatchExpand((H, W), C).cuda()
    with torch.no_grad():
        for n, prm in m.named_parameters():
            prm.copy_(P.randn(S, f"pe/{C}/{n}", tuple(prm.shape), C ** -0.5 if prm.dim() > 1 else 0.1, 1.0 if n.endswith("norm.weight") else 0.0))
        x = P.randn(S, f"pe/x/{B}/{H}/{W}/{C}", (B, H, W, C)).cuda()
        with M.composed_path():
            ref = m(x)
        got = fused.patch_expand(m, x)
    assert_close(got, ref, 5e-3, 8e-3, "patch_expand (tf32 GEMM)")


def test_pool_and_scale_add():
    from sigma_b200 import fused
    B, H, W, C = 2, 33, 40, 96
    t = P.randn(S, "pool/t", (B, H, W, C))
    avg, mx = fused.pool_avgmax(t.cuda())
    assert_close(avg, t.mean(dim=(1, 2)), 1e-5, 1e-5, "avg pool")
    assert_close(mx, t.amax(dim=(1, 2)), 0, 0, "max pool")
    a, bq = P.randn(S, "sa/a", (B, H, W, C)), P.randn(S, "sa/b", (B, H, W, C))
    sa, sb = P.rand(S, "sa/sa", (B, C)), P.randn(S, "sa/sb", (C,))
    got = fused.scale_add(a.cuda(), sa.cuda(), bq.cuda(), sb.cuda(), H * W)
    assert_close(got, a * sa[:, None, None, :] + bq * sb, 1e-6, 1e-6, "scale_add")
    got = fused.scale_add(None, None, bq.cuda(), sb.cuda(), H * W)
    assert_close(got, bq * sb, 1e-6, 1e-6, "scale only")


@pytest.mark.parametrize("M,N,K,extras", [
    (1000, 384, 96, ""), (77, 160, 192, "b"), (300, 96, 192, "r"), (513, 192, 384, "rs"), (129, 40, 64, "br"),
    (64, 32, 16, ""), (2500, 768, 1536, "r"), (4096, 320, 1536, ""), (1, 16, 32, "b"), (700, 3072, 768, ""),
])
@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
def test_tcgen05_tf32_gemm(M, N, K, extras, mode):
    """sigma_linear_tf32 / sigma_linear_tf32x3 (the wgmma GEMM of gemm_tf32.cu; the test keeps the name of the kernel's first,
    Blackwell version) vs fp64 matmul.  tf32: tolerance = TF32 input rounding (2^-10 relative per
    product); tf32x3 (error-compensated split, 3 MMAs per k-step): fp32-grade — 2^-20 of the sum of |products| plus fp32
    accumulation."""
    from sigma_b200 import fused
    torch.backends.cuda.matmul.allow_tf32 = mode == "tf32"
    assert fused.precision() == mode
    tag = f"gemm/{M}/{N}/{K}"
    A = P.randn(S, tag + "/A", (M, K))
    Wt = P.randn(S, tag + "/W", (N, K), K ** -0.5)
    bias = P.randn(S, tag + "/b", (N,)) if "b" in extras else None
    res = P.randn(S, tag + "/r", (M, N)) if "r" in extras else None
    rs = P.randn(S, tag + "/s", (N,), 0.2, 1.0) if "s" in extras else None
    ref = A.double() @ Wt.double().t()
    if bias is not None:
        ref = ref + bias.double()
    if res is not None:
        ref = ref + res.double() * (rs.double() if rs is not None else 1.0)
    c = lambda t: None if t is None else t.cuda()
    assert fused.USE_OWN_GEMM
    got = fused.linear(c(A), c(Wt), c(bias), residual=c(res), rscale=c(rs))
    torch.cuda.synchronize()
    bound = (2.5e-3 if mode == "tf32" else 4e-6) * float((A.abs().double() @ Wt.abs().double().t()).max()) + 1e-5
    err = float((got.cpu().double() - ref).abs().max())
    assert err < bound, f"{tag}: max abs err {err:.3e} > {bound:.3e}"
    # strided A (the x half of [x | z] rows) and strided output
    if K % 4 == 0 and M > 4:
        big = torch.zeros(M, 2 * K + 4, device="cuda")
        big[:, :K] = A.cuda()
        out = torch.zeros(M, N + 8, device="cuda")
        fused.linear(big[:, :K], c(Wt), None, out=out[:, :N])
        ref2 = A.double() @ Wt.double().t()
        assert float((out[:, :N].cpu().double() - ref2).abs().max()) < bound and float(out[:, N:].abs().max()) == 0.0


@pytest.mark.parametrize("B,H,W,Cin,Cout,gelu", [(2, 30, 40, 96, 32, True), (1, 15, 20, 32, 96, False), (3, 9, 17, 128, 384, False),
                                                 (1, 60, 80, 192, 64, True), (2, 8, 16, 64, 192, False), (1, 1, 5, 32, 32, True)])
@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
def test_tcgen05_conv3x3_implicit_gemm(B, H, W, Cin, Cout, gelu, mode):
    """sigma_conv3x3_tf32 (3x3 conv as 9 shifted TMA boxes x Cin blocks on the wgmma kernel; zero padding = TMA out-of-bounds
    fill; bias + exact GELU in the epilogue) vs torch's conv2d in fp64, ragged image sizes included."""
    from sigma_b200 import fused
    torch.backends.cudnn.allow_tf32 = mode == "tf32"      # convolutions follow torch's cuDNN switch
    tag = f"conv/{B}/{H}/{W}/{Cin}/{Cout}"
    conv = torch.nn.Conv2d(Cin, Cout, 3, 1, 1)
    x = P.randn(S, tag + "/x", (B, H, W, Cin))
    with torch.no_grad():
        conv.weight.copy_(P.randn(S, tag + "/w", (Cout, Cin, 3, 3), (9 * Cin) ** -0.5))
        conv.bias.copy_(P.randn(S, tag + "/b", (Cout,), 0.2))
        ref = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).double(), conv.weight.double(), conv.bias.double(), padding=1)
        if gelu:
            ref = torch.nn.functional.gelu(ref)
        ref = ref.permute(0, 2, 3, 1)
        got = fused.conv3x3(x.cuda(), conv.cuda(), gelu=gelu)
    assert got is not None and tuple(got.shape) == (B, H, W, Cout)
    mag = float(torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).abs().double(), conv.weight.abs().double().cpu(), padding=1).max())
    bound = (2.5e-3 if mode == "tf32" else 4e-6) * mag + 1e-5
    err = float((got.cpu().double() - ref).abs().max())
    assert err < bound, f"{tag} {mode}: max abs err {err:.3e} > {bound:.3e}"
