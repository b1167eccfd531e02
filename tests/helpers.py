"""Shared helpers for the parity tests."""
import os
import types
import zlib

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SEED = 7


def golden(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"))


def cfg_tiny(H, W, num_classes=9, backbone="sigma_tiny"):
    return types.SimpleNamespace(backbone=backbone, decoder="MambaDecoder", num_classes=num_classes, image_height=H,
                                 image_width=W, pretrained_model=None, bn_eps=1e-3, bn_momentum=0.1)


def max_err(a, b):
    a = a.detach().float().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    b = b.detach().float().cpu().numpy() if torch.is_tensor(b) else np.asarray(b)
    return float(np.abs(a - b).max())


def assert_close(a, b, rtol, atol, what=""):
    a = a.detach().float().cpu().numpy() if torch.is_tensor(a) else np.asarray(a, dtype=np.float32)
    b = b.detach().float().cpu().numpy() if torch.is_tensor(b) else np.asarray(b, dtype=np.float32)
    assert a.shape == b.shape, f"{what}: shape {a.shape} vs {b.shape}"
    err = np.abs(a - b)
    tol = atol + rtol * np.abs(b)
    bad = err > tol
    assert not bad.any(), (f"{what}: {bad.sum()}/{bad.size} elements out of tolerance; max abs err {err.max():.3e} "
                           f"(|ref| max {np.abs(b).max():.3e}), rtol={rtol} atol={atol}")


def record(name, **kv):
    """Append one JSON line of measured parity numbers to $SIGMA_PARITY_LOG (set by the GPU run scripts)."""
    import json
    path = os.environ.get("SIGMA_PARITY_LOG")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps(dict(test=name, **kv)) + "\n")


def gemm_plan(M, N, K, x3, conv=None):
    """The launch plan sigma_linear_tf32{,x3} (conv=None) or sigma_conv3x3_tf32 (conv=(B, H, W): input (B, H, W, K), N output
    channels) would use under the current environment (SIGMA_GEMM_BN included), from the library's own planner."""
    import ctypes
    from sigma_b200 import _lib
    out = (ctypes.c_int64 * 6)()
    B, H, W = conv if conv is not None else (0, 0, 0)
    _lib.check(_lib.lib().sigma_test_gemm_plan(M, N, K, int(bool(x3)), B, H, W, out), "sigma_test_gemm_plan")
    return dict(zip(("bn", "stages", "grid", "tiles", "smem", "ctas_per_sm"), (int(v) for v in out)))


def sample_index(key, numel, k):
    """A fixed, seeded set of min(k, numel) flat indices for `key`: the positions at which a golden file stores a large output."""
    rng = np.random.default_rng(zlib.crc32(key.encode()))
    return np.sort(rng.choice(numel, size=min(k, numel), replace=False))


# ---- the fused SS2D scan through its C-ABI (the fp64 tests of its forward and backward) ----
SS2D_GUARD = 64                          # guard elements on each side of every output (keeps 16-byte alignment)
_NAN_BITS = {torch.float32: (torch.int32, 0x7FC00000), torch.bfloat16: (torch.int16, 0x7FC0), torch.float16: (torch.int16, 0x7E00)}


def ptr(t):
    import ctypes
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def stream():
    import ctypes
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def ss2d_kind(kind):
    from sigma_b200 import _lib
    return {"cross4": _lib.DIRS_CROSS4, "seq2": _lib.DIRS_SEQ2, "cross": _lib.DIRS_CROSS}[kind]


def guarded(shape, dtype=torch.float32):
    """(buffer, interior view): NaN-filled device memory with SS2D_GUARD elements on each side of `shape`"""
    import math
    n = math.prod(shape)
    buf = torch.full((n + 2 * SS2D_GUARD,), float("nan"), dtype=dtype, device="cuda")
    return buf, buf[SS2D_GUARD:SS2D_GUARD + n].view(shape)


def guard_ok(buf, what):
    """no guard element of a `guarded` buffer was written: every one still has the bits of the NaN it was filled with"""
    n = buf.numel() - 2 * SS2D_GUARD
    ity, nan = _NAN_BITS[buf.dtype]
    bits = torch.cat([buf[:SS2D_GUARD], buf[SS2D_GUARD + n:]]).view(ity)
    bad = int((bits != nan).sum())
    assert bad == 0, f"{what}: {bad} guard elements were written"


def ss2d_params(seed, kind, B, H, W, D, N, R, tag, wide=False):
    """inputs of the fused scan at Sigma's scales: dt log-uniform in [1e-3, 0.1] (0.5 when wide) through the inverse softplus,
    A = -exp(A_log) around the S4D-real init (|A| up to 4x when wide), Ds near 1, x_dbl's padding columns 0.  B is the batch
    (2·images for "cross", which has two weight sets).  Returns ([xc, xdbl, dtw, dtb, A, Ds, dy] on the GPU, Cp)."""
    import math
    import procedural as P
    from sigma_b200 import _lib
    K = {"cross4": 4, "seq2": 2, "cross": 1}[kind]
    Kw = 2 if kind == "cross" else K
    Lseq = H * W * (2 if kind == "seq2" else 1)
    Cp = _lib.lib().sigma_ss2d_padded_cp(N, R)
    xc = P.randn(seed, tag + "/xc", (B, Lseq, D))
    xdbl = P.randn(seed, tag + "/xdbl", (B, Lseq, K, Cp))
    xdbl[..., 2 * N:2 * N + R] *= 2.0
    xdbl[..., 2 * N + R:] = 0.0                                          # padding columns, as the packed x_proj leaves them
    dtw = P.rand(seed, tag + "/dtw", (Kw, D, R), -R ** -0.5, R ** -0.5)
    dt = torch.exp(P.rand(seed, tag + "/dt", (Kw, D), math.log(1e-3), math.log(0.5 if wide else 0.1)))
    dtb = dt + torch.log(-torch.expm1(-dt))                              # inverse softplus
    A_log = torch.log(torch.arange(1, N + 1, dtype=torch.float32)).repeat(Kw * D, 1) + P.rand(seed, tag + "/A", (Kw * D, N), -0.2,
                                                                                                   1.4 if wide else 0.2)
    A = -torch.exp(A_log)
    Ds = P.randn(seed, tag + "/Ds", (Kw * D,), 0.1, 1.0)
    dy = P.randn(seed, tag + "/dy", (B, Lseq, D))
    return [t.cuda() for t in (xc, xdbl, dtw, dtb, A, Ds, dy)], Cp


def op_scan_params(seed, batch, dim, L, N, G, tag, dist="sigma", dtype=torch.float32, has_D=True, has_bias=True, softplus=True):
    """inputs of the op-level scan, on the CPU: [u, delta, A, B, C, D, delta_bias, dout]; u / delta / B / C / dout in `dtype`.
    dist "sigma": delta = a small dt_proj-like term (0.5·randn) + delta_bias, delta_bias = the inverse softplus of dt log-uniform
    in [1e-3, 0.1] per channel (folded into delta when has_bias is False); A = -exp(A_log) around the S4D-real init; D near 1.
    "wide": dt up to 0.5, |A| up to 4x.  Without softplus, delta' = delta (+ bias) must be a step itself: dt · exp(0.3·randn).
    "ref": the reference test's distribution (procedural.scan_inputs: delta, bias in [0, 0.5), A in [-0.5, 0])."""
    import math
    import procedural as P
    if dist == "ref":
        u, delta, A, B, C, D, bias = P.scan_inputs(seed, batch, dim, N, L, G, dtype, has_D, has_bias)
        dout = P.randn(seed, tag + "/dout", (batch, dim, L)).to(dtype)
        return [u, delta, A, B, C, D, bias, dout]
    wide = dist == "wide"
    dt = torch.exp(P.rand(seed, tag + "/dt", (dim,), math.log(1e-3), math.log(0.5 if wide else 0.1)))
    if softplus:
        isp = dt + torch.log(-torch.expm1(-dt))                          # inverse softplus
        delta = 0.5 * P.randn(seed, tag + "/delta", (batch, dim, L)) + (0.0 if has_bias else isp[:, None])
        bias = isp if has_bias else None
    else:
        delta = dt[:, None] * torch.exp(0.3 * P.randn(seed, tag + "/delta", (batch, dim, L)))
        bias = 0.1 * dt if has_bias else None
    A_log = torch.log(torch.arange(1, N + 1, dtype=torch.float32)).repeat(dim, 1) + P.rand(seed, tag + "/A", (dim, N), -0.2,
                                                                                            1.4 if wide else 0.2)
    A = -torch.exp(A_log)
    D = P.randn(seed, tag + "/D", (dim,), 0.1, 1.0) if has_D else None
    u = P.randn(seed, tag + "/u", (batch, dim, L))
    B = P.randn(seed, tag + "/B", (batch, G, N, L))
    C = P.randn(seed, tag + "/C", (batch, G, N, L))
    dout = P.randn(seed, tag + "/dout", (batch, dim, L))
    return [t.to(dtype) if i in (0, 1, 3, 4, 7) else t for i, t in enumerate((u, delta, A, B, C, D, bias, dout))]


SCAN_PLAN = ("route", "nsplit", "tiles_per_split", "ntiles", "channels", "stages", "state_nsplit", "state_tiles_per_split")
SCAN_ROUTES = ("tma", "widened", "generic")
_SCAN_SWEEPS = {"fwd": 0, "bwd": 1, "bwd_det": 2}


def scan_plan(sweep, batch, dim, L, N, G, dtype=torch.float32, nsplit=0, ws_bytes=None):
    """The launch plan the op-level scan would use (sigma_test_scan_plan), route as a name.  sweep "fwd" / "bwd" / "bwd_det";
    ws_bytes: the workspace the call gets (None: what sigma_b200.ops allocates, 0: none)."""
    import ctypes
    from sigma_b200 import _lib
    L_ = _lib.lib()
    dt = {torch.float32: _lib.F32, torch.float16: _lib.F16, torch.bfloat16: _lib.BF16}[dtype]
    if ws_bytes is None:
        ws_bytes = {"fwd": L_.sigma_scan_fwd_workspace_bytes, "bwd": L_.sigma_scan_bwd_workspace_bytes,
                    "bwd_det": L_.sigma_scan_bwd_det_workspace_bytes}[sweep](batch, dim, L, N, G, dt)
    out = (ctypes.c_int64 * 8)()
    _lib.check(L_.sigma_test_scan_plan(_SCAN_SWEEPS[sweep], batch, dim, L, N, G, dt, nsplit, ws_bytes, out), "sigma_test_scan_plan")
    plan = dict(zip(SCAN_PLAN, (int(v) for v in out)))
    plan["route"] = SCAN_ROUTES[plan["route"]]
    return plan


SS2D_FWD_PLAN = ("nsplit", "tiles_per_split", "max_tiles", "min_tiles", "warps", "nst", "ctas", "smem")


def ss2d_fwd_plan(kind, B, H, W, D, N, R, bf16=False, force=0, ws_bytes=None):
    """The launch plan sigma_ss2d_scan_fwd{,_split,_bf16} would use under the current environment (SIGMA_SCAN_* included), from the
    library's own planner.  ws_bytes: the workspace the call gets (None: sigma_ss2d_scan_workspace_bytes, 0: none)."""
    import ctypes
    from sigma_b200 import _lib
    L = _lib.lib()
    if ws_bytes is None:
        ws_bytes = L.sigma_ss2d_scan_workspace_bytes(ss2d_kind(kind), B, H, W, D, N)
    out = (ctypes.c_int64 * 8)()
    _lib.check(L.sigma_test_ss2d_fwd_plan(ss2d_kind(kind), B, H, W, D, N, R, int(bool(bf16)), force, ws_bytes, out),
               "sigma_test_ss2d_fwd_plan")
    return dict(zip(SS2D_FWD_PLAN, (int(v) for v in out)))
