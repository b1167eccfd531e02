"""Op surface of the reference on top of libsigma_b200 (no torch arithmetic on these paths).

`selective_scan_cuda_core_fwd/bwd` have the exact pybind signatures of the reference extension
(csrc/selective_scan/selective_scan.cpp:364-367); `sigma_b200/dropin/selective_scan_cuda_core.py`
re-exports them under the reference's module name.
"""
import contextlib
import ctypes
import functools
import os

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib
from ._lib import ptr, stream

_DTYPE = {torch.float32: _lib.F32, torch.float16: _lib.F16, torch.bfloat16: _lib.BF16}


def deterministic():
    """True when torch.use_deterministic_algorithms(True) is in effect: the backward kernels then run their `_det` builds, which
    keep every cross-CTA sum as partials and add them in a fixed order (bitwise reproducible for the same inputs, GPU model and
    launch plan)."""
    return torch.are_deterministic_algorithms_enabled()


def _require_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("sigma_b200 ops run on CUDA tensors only (there is no CPU path)")


def selective_scan_cuda_core_fwd(u, delta, A, B, C, D=None, delta_bias=None, delta_softplus=False, nrows=1,
                                 _force_split=0):
    """Drop-in for selective_scan_cuda_core.fwd (selective_scan.cpp:165-249) -> [out, x]."""
    _require_cuda(u, delta, A, B, C, D, delta_bias)
    if u.dtype not in _DTYPE:
        raise RuntimeError(f"selective_scan fwd: unsupported dtype {u.dtype}")
    if not (delta.dtype == u.dtype and B.dtype == u.dtype and C.dtype == u.dtype):
        raise RuntimeError("selective_scan fwd: u, delta, B, C must share one dtype (selective_scan.cpp:177-180)")
    if A.dtype != torch.float32 or (D is not None and D.dtype != torch.float32) or \
            (delta_bias is not None and delta_bias.dtype != torch.float32):
        raise RuntimeError("selective_scan fwd: A, D, delta_bias must be float32 (selective_scan.cpp:176,211,219)")
    if u.dim() != 3 or delta.shape != u.shape or B.dim() != 4 or C.shape != B.shape:
        raise RuntimeError("selective_scan fwd: expected u,delta (B,D,L) and B,C (B,G,N,L)")
    for t, n in ((u, "u"), (delta, "delta"), (B, "B"), (C, "C")):
        if t.stride(-1) != 1 and t.size(-1) != 1:
            raise RuntimeError(f"selective_scan fwd: {n} must have unit stride along seqlen (selective_scan.cpp:191-194)")
    batch, dim, L = u.shape
    G, N = B.shape[1], B.shape[2]
    if A.shape != (dim, N) or B.shape[0] != batch or B.shape[3] != L:
        raise RuntimeError("selective_scan fwd: shape mismatch")
    if dim % (G * nrows) != 0:
        raise RuntimeError(f"selective_scan fwd: dim={dim} must be divisible by ngroups*nrows={G * nrows}")
    if N > 256 // nrows:
        raise RuntimeError("selective_scan fwd: dstate too large (selective_scan.cpp:198)")
    if D is not None:
        D = D.contiguous()
    if delta_bias is not None:
        delta_bias = delta_bias.contiguous()
    out = torch.empty_like(delta)
    if out.stride(-1) != 1:
        out = torch.empty(delta.shape, dtype=delta.dtype, device=delta.device)
    nchunks = (L + 2047) // 2048
    x = torch.empty((batch, dim, nchunks, 2 * N), dtype=torch.float32, device=u.device)
    st = _lib.ScanStrides(u.stride(0), u.stride(1), delta.stride(0), delta.stride(1), A.stride(0), A.stride(1),
                          B.stride(0), B.stride(1), B.stride(2), C.stride(0), C.stride(1), C.stride(2),
                          out.stride(0), out.stride(1))
    L_ = _lib.lib()
    dt = _DTYPE[u.dtype]
    wsb = L_.sigma_scan_fwd_workspace_bytes(batch, dim, L, N, G, dt)
    ws = torch.empty(wsb, dtype=torch.uint8, device=u.device)
    if _force_split:
        rc = L_.sigma_scan_fwd_split(ptr(u), ptr(delta), ptr(A), ptr(B), ptr(C), ptr(D), ptr(delta_bias),
                                     ptr(out), ptr(x), batch, dim, L, N, G, dt, int(bool(delta_softplus)),
                                     ctypes.byref(st), ptr(ws), wsb, int(_force_split), stream())
    else:
        rc = L_.sigma_scan_fwd(ptr(u), ptr(delta), ptr(A), ptr(B), ptr(C), ptr(D), ptr(delta_bias),
                               ptr(out), ptr(x), batch, dim, L, N, G, dt, int(bool(delta_softplus)),
                               ctypes.byref(st), ptr(ws), wsb, stream())
    _lib.check(rc, "sigma_scan_fwd")
    return [out, x]


def selective_scan_cuda_core_bwd(u, delta, A, B, C, D, delta_bias, dout, x, delta_softplus, nrows=1, _force_split=0):
    """Drop-in for selective_scan_cuda_core.bwd (selective_scan.cpp:251-362)
    -> [du, ddelta, dA, dB, dC, dD, ddelta_bias]."""
    _require_cuda(u, delta, A, B, C, D, delta_bias, dout)
    if u.dtype not in _DTYPE:
        raise RuntimeError(f"selective_scan bwd: unsupported dtype {u.dtype}")
    batch, dim, L = u.shape
    G, N = B.shape[1], B.shape[2]
    u, delta, B, C, dout = (t.contiguous() for t in (u, delta, B, C, dout))
    A = A.contiguous()
    D = D.contiguous() if D is not None else None
    delta_bias = delta_bias.contiguous() if delta_bias is not None else None
    du, ddelta = torch.empty_like(u), torch.empty_like(delta)
    dA = torch.empty((dim, N), dtype=torch.float32, device=u.device)
    dB = torch.empty((batch, G, N, L), dtype=torch.float32, device=u.device)
    dC = torch.empty((batch, G, N, L), dtype=torch.float32, device=u.device)
    dD = torch.empty(dim, dtype=torch.float32, device=u.device) if D is not None else None
    dbias = torch.empty(dim, dtype=torch.float32, device=u.device) if delta_bias is not None else None
    L_ = _lib.lib()
    dt = _DTYPE[u.dtype]
    if deterministic():
        wsb = L_.sigma_scan_bwd_det_workspace_bytes(batch, dim, L, N, G, dt)
        ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=u.device)
        rc = L_.sigma_scan_bwd_det(ptr(u), ptr(delta), ptr(A), ptr(B), ptr(C), ptr(D), ptr(delta_bias), ptr(dout),
                                   ptr(du), ptr(ddelta), ptr(dA), ptr(dB), ptr(dC), ptr(dD), ptr(dbias),
                                   batch, dim, L, N, G, dt, int(bool(delta_softplus)), ptr(ws), wsb, int(_force_split), stream())
        _lib.check(rc, "sigma_scan_bwd_det")
        return [du, ddelta, dA, dB.to(u.dtype), dC.to(u.dtype), dD, dbias]
    wsb = L_.sigma_scan_bwd_workspace_bytes(batch, dim, L, N, G, dt)
    ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=u.device)
    if _force_split:
        rc = L_.sigma_scan_bwd_split(ptr(u), ptr(delta), ptr(A), ptr(B), ptr(C), ptr(D), ptr(delta_bias), ptr(dout),
                                     ptr(du), ptr(ddelta), ptr(dA), ptr(dB), ptr(dC), ptr(dD), ptr(dbias),
                                     batch, dim, L, N, G, dt, int(bool(delta_softplus)), ptr(ws), wsb, int(_force_split), stream())
    else:
        rc = L_.sigma_scan_bwd(ptr(u), ptr(delta), ptr(A), ptr(B), ptr(C), ptr(D), ptr(delta_bias), ptr(dout),
                               ptr(du), ptr(ddelta), ptr(dA), ptr(dB), ptr(dC), ptr(dD), ptr(dbias),
                               batch, dim, L, N, G, dt, int(bool(delta_softplus)), ptr(ws), wsb, stream())
    _lib.check(rc, "sigma_scan_bwd")
    # the reference returns dB/dC cast to the input dtype (selective_scan.cpp:360)
    return [du, ddelta, dA, dB.to(u.dtype), dC.to(u.dtype), dD, dbias]


class SelectiveScan(torch.autograd.Function):
    """vmamba.py:34-78 — fp32 cast under AMP, contiguity fix-ups, 3-D B/C unsqueeze; backward with nrows=1."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, u, delta, A, B, C, D=None, delta_bias=None, delta_softplus=False, nrows=1):
        assert nrows in (1, 2, 3, 4), f"{nrows}"
        assert u.shape[1] % (B.shape[1] * nrows) == 0, f"{nrows}, {u.shape}, {B.shape}"
        ctx.delta_softplus, ctx.nrows = delta_softplus, nrows
        u, delta, B, C = (t if t.stride(-1) == 1 else t.contiguous() for t in (u, delta, B, C))
        ctx.squeeze_B = B.dim() == 3
        ctx.squeeze_C = C.dim() == 3
        if ctx.squeeze_B:
            B = B.unsqueeze(1)
        if ctx.squeeze_C:
            C = C.unsqueeze(1)
        out, x = selective_scan_cuda_core_fwd(u, delta, A, B, C, D, delta_bias, delta_softplus, nrows)
        ctx.save_for_backward(u, delta, A, B, C, D, delta_bias, x)
        return out

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, dout, *args):
        u, delta, A, B, C, D, delta_bias, x = ctx.saved_tensors
        du, ddelta, dA, dB, dC, dD, dbias = selective_scan_cuda_core_bwd(
            u, delta, A, B, C, D, delta_bias, dout, x, ctx.delta_softplus, 1)
        dB = dB.squeeze(1) if ctx.squeeze_B else dB
        dC = dC.squeeze(1) if ctx.squeeze_C else dC
        return du, ddelta, dA, dB, dC, dD, dbias, None, None


class SelectiveScanFn(torch.autograd.Function):
    """selective_scan_interface.py:10-75 (no AMP cast: dtype follows the input, D/bias promoted to fp32)."""

    @staticmethod
    def forward(ctx, u, delta, A, B, C, D=None, delta_bias=None, delta_softplus=False, nrows=1):
        u, delta, B, C = (t if t.stride(-1) == 1 else t.contiguous() for t in (u, delta, B, C))
        ctx.squeeze_B = B.dim() == 3
        ctx.squeeze_C = C.dim() == 3
        if ctx.squeeze_B:
            B = B.unsqueeze(1)
        if ctx.squeeze_C:
            C = C.unsqueeze(1)
        ctx.d_dtype = D.dtype if D is not None else None
        ctx.bias_dtype = delta_bias.dtype if delta_bias is not None else None
        D = D.float() if D is not None else None
        delta_bias = delta_bias.float() if delta_bias is not None else None
        assert u.shape[1] % (B.shape[1] * nrows) == 0
        assert nrows in (1, 2, 3, 4)
        out, x = selective_scan_cuda_core_fwd(u, delta, A, B, C, D, delta_bias, delta_softplus, nrows)
        ctx.delta_softplus, ctx.nrows = delta_softplus, nrows
        ctx.save_for_backward(u, delta, A, B, C, D, delta_bias, x)
        return out

    @staticmethod
    def backward(ctx, dout, *args):
        u, delta, A, B, C, D, delta_bias, x = ctx.saved_tensors
        du, ddelta, dA, dB, dC, dD, dbias = selective_scan_cuda_core_bwd(
            u, delta, A, B, C, D, delta_bias, dout, x, ctx.delta_softplus, 1)
        dB = dB.squeeze(1) if ctx.squeeze_B else dB
        dC = dC.squeeze(1) if ctx.squeeze_C else dC
        dD = dD.to(ctx.d_dtype) if dD is not None else None
        dbias = dbias.to(ctx.bias_dtype) if dbias is not None else None
        return du, ddelta, dA, dB, dC, dD, dbias, None, None


def selective_scan_fn(u, delta, A, B, C, D=None, delta_bias=None, delta_softplus=False, nrows=1):
    """selective_scan_interface.py:78-83."""
    return SelectiveScanFn.apply(u, delta, A, B, C, D, delta_bias, delta_softplus, nrows)


# ---- direction maps (pure index shuffles; the fused inference path never materialises them) ----
class CrossScan(torch.autograd.Function):
    """vmamba.py:80-98.  (B,C,H,W) -> (B,4,C,L): row-major, column-major, and both reversed."""

    @staticmethod
    def forward(ctx, x):
        B, C, H, W = x.shape
        ctx.shape = (B, C, H, W)
        xs = x.new_empty((B, 4, C, H * W))
        xs[:, 0] = x.flatten(2, 3)
        xs[:, 1] = x.transpose(2, 3).flatten(2, 3)
        xs[:, 2:4] = xs[:, 0:2].flip(-1)
        return xs

    @staticmethod
    def backward(ctx, ys):
        B, C, H, W = ctx.shape
        return _merge4(ys, H, W).view(B, C, H, W)


def _merge4(ys, H, W):
    B, K, D, L = ys.shape
    ys = ys[:, 0:2] + ys[:, 2:4].flip(-1)
    return ys[:, 0] + ys[:, 1].reshape(B, D, W, H).transpose(2, 3).reshape(B, D, L)


def _scan4(x, H, W):
    B, C, L = x.shape
    xs = x.new_empty((B, 4, C, L))
    xs[:, 0] = x
    xs[:, 1] = x.view(B, C, H, W).transpose(2, 3).flatten(2, 3)
    xs[:, 2:4] = xs[:, 0:2].flip(-1)
    return xs


class CrossMerge(torch.autograd.Function):
    """vmamba.py:100-121.  (B,4,D,H,W) -> (B,D,L)."""

    @staticmethod
    def forward(ctx, ys):
        B, K, D, H, W = ys.shape
        ctx.shape = (H, W)
        return _merge4(ys.view(B, K, D, -1), H, W)

    @staticmethod
    def backward(ctx, x):
        H, W = ctx.shape
        B, C, L = x.shape
        return _scan4(x, H, W).view(B, 4, C, H, W)


class CrossScan_multimodal(torch.autograd.Function):
    """vmamba.py:123-141.  two (B,C,H,W) -> (B,2,C,2L): [rgb ‖ x] and its reverse."""

    @staticmethod
    def forward(ctx, x_rgb, x_e):
        B, C, H, W = x_rgb.shape
        ctx.shape = (B, C, H, W)
        xs = x_rgb.new_empty((B, 2, C, 2 * H * W))
        xs[:, 0, :, :H * W] = x_rgb.flatten(2, 3)
        xs[:, 0, :, H * W:] = x_e.flatten(2, 3)
        xs[:, 1] = xs[:, 0].flip(-1)
        return xs

    @staticmethod
    def backward(ctx, ys):
        B, C, H, W = ctx.shape
        y = ys[:, 0] + ys[:, 1].flip(-1)
        return y[:, :, :H * W].reshape(B, C, H, W), y[:, :, H * W:].reshape(B, C, H, W)


class CrossMerge_multimodal(torch.autograd.Function):
    """vmamba.py:143-163.  (B,2,D,2L) -> two (B,D,L)."""

    @staticmethod
    def forward(ctx, ys):
        B, K, D, L2 = ys.shape
        y = ys[:, 0] + ys[:, 1].flip(-1)
        return y[:, :, :L2 // 2], y[:, :, L2 // 2:]

    @staticmethod
    def backward(ctx, x1, x2):
        B, C, L = x1.shape
        xs = x1.new_empty((B, 2, C, 2 * L))
        xs[:, 0, :, :L] = x1
        xs[:, 0, :, L:] = x2
        xs[:, 1] = xs[:, 0].flip(-1)
        return xs


def _pick_nrows(D, nrows, N=1):
    """vmamba.py:183-191's automatic rows per block, stopping at a count whose d_state bound (N <= 256 / nrows,
    selective_scan.cpp:198) the call meets: d_state="auto" past 64 states runs instead of failing the check.  Unchanged for N <= 64."""
    if nrows >= 1:
        return nrows
    return next(r for r in (4, 3, 2, 1) if D % r == 0 and N <= 256 // r)


def _scan_core(xs, x_proj_weight, x_proj_bias, dt_projs_weight, dt_projs_bias, A_logs, Ds, nrows, delta_softplus):
    """x_proj / dt_proj einsums + SelectiveScan, shared by the two composed paths (vmamba.py:195-215, 401-421)."""
    B, K, D, L = xs.shape
    R, N = dt_projs_weight.shape[2], A_logs.shape[1]
    x_dbl = torch.einsum("bkdl,kcd->bkcl", xs, x_proj_weight)
    if x_proj_bias is not None:
        x_dbl = x_dbl + x_proj_bias.view(1, K, -1, 1)
    dts, Bs, Cs = torch.split(x_dbl, [R, N, N], dim=2)
    dts = torch.einsum("bkrl,kdr->bkdl", dts, dt_projs_weight)
    ys = SelectiveScan.apply(xs.reshape(B, K * D, L).float(), dts.reshape(B, K * D, L).float(),
                             -torch.exp(A_logs.float()), Bs.float().contiguous(), Cs.float().contiguous(),
                             Ds.float(), dt_projs_bias.reshape(-1).float(), delta_softplus, nrows)
    return ys.view(B, K, D, L)


def cross_selective_scan(x, x_proj_weight=None, x_proj_bias=None, dt_projs_weight=None, dt_projs_bias=None,
                         A_logs=None, Ds=None, out_norm=None, softmax_version=False, nrows=-1, delta_softplus=True):
    """vmamba.py:165-226 (composed path: used when autograd is recording)."""
    B, D, H, W = x.shape
    nrows = _pick_nrows(D, nrows, A_logs.shape[1])
    ys = _scan_core(CrossScan.apply(x), x_proj_weight, x_proj_bias, dt_projs_weight, dt_projs_bias, A_logs, Ds,
                    nrows, delta_softplus)
    y = CrossMerge.apply(ys.view(B, 4, D, H, W))
    y = y.transpose(1, 2).contiguous().view(B, H, W, D)
    if softmax_version:
        return y.softmax(dim=-1).to(x.dtype)
    return out_norm(y).to(x.dtype)


def cross_selective_scan_multimodal_k2(x_rgb, x_e, x_proj_weight=None, x_proj_bias=None, dt_projs_weight=None,
                                       dt_projs_bias=None, A_logs=None, Ds=None, out_norm1=None, out_norm2=None,
                                       softmax_version=False, nrows=-1, delta_softplus=True):
    """vmamba.py:369-430 (composed path)."""
    B, D, H, W = x_rgb.shape
    nrows = _pick_nrows(D, nrows, A_logs.shape[1])
    ys = _scan_core(CrossScan_multimodal.apply(x_rgb, x_e), x_proj_weight, x_proj_bias, dt_projs_weight,
                    dt_projs_bias, A_logs, Ds, nrows, delta_softplus)
    y_r, y_e = CrossMerge_multimodal.apply(ys)
    y_r = y_r.transpose(1, 2).contiguous().view(B, H, W, D)
    y_e = y_e.transpose(1, 2).contiguous().view(B, H, W, D)
    return out_norm1(y_r).to(x_rgb.dtype), out_norm2(y_e).to(x_e.dtype)


# ---- f1: the fused SS2D core under autograd (training) ----
FUSED_TRAINING = True   # False: the composed path (CrossScan + einsum + op-level scan), kept for A/B and as the general fallback


def fused_core_ok(xc, D, N):
    """The fused training core covers the Sigma configurations: fp32 CUDA activations, d_state in {4, 16}, d_inner % 64 == 0."""
    return FUSED_TRAINING and xc.is_cuda and N in (4, 16) and D % 64 == 0


# ---- bf16 training mode of the fused core (opt-in) ----
# On, the fused core and the LayerNorm pair keep bf16 activations under bf16 autocast instead of widening them to fp32: bf16 xc, y,
# dy, dxc and saved delta' (x_dbl, the states, every accumulator and every parameter gradient stay fp32).  Off (the default), autocast
# does not change those two autograd nodes.  SIGMA_BF16_TRAINING_CORE=1 sets the initial value.
BF16_TRAINING_CORE = os.environ.get("SIGMA_BF16_TRAINING_CORE", "0") == "1"


@contextlib.contextmanager
def bf16_training_core(on=True):
    """Switch the bf16 training mode of the fused core on (or off) inside the block."""
    global BF16_TRAINING_CORE
    prev, BF16_TRAINING_CORE = BF16_TRAINING_CORE, bool(on)
    try:
        yield
    finally:
        BF16_TRAINING_CORE = prev


# ---- fp16 training mode of the fused core (opt-in) ----
# The same under fp16 autocast, with fp16 in place of bf16.  fp16 keeps 11 significant bits where bf16 keeps 8, but its range ends at
# ±65504: a store past it gives ±inf (nothing saturates), so the mode is meant to run with a loss scaler (torch.amp.GradScaler), which
# sees the inf and skips the step.  SIGMA_FP16_TRAINING_CORE=1 sets the initial value.  The two switches are independent; the
# autocast dtype decides which of them can apply.
FP16_TRAINING_CORE = os.environ.get("SIGMA_FP16_TRAINING_CORE", "0") == "1"


@contextlib.contextmanager
def fp16_training_core(on=True):
    """Switch the fp16 training mode of the fused core on (or off) inside the block."""
    global FP16_TRAINING_CORE
    prev, FP16_TRAINING_CORE = FP16_TRAINING_CORE, bool(on)
    try:
        yield
    finally:
        FP16_TRAINING_CORE = prev


def _autocast_mode16():
    """the 16-bit training mode in effect: torch.bfloat16 / torch.float16 when autocast on CUDA runs that dtype and its switch is
    on, outside the deterministic switch; else None"""
    if not torch.is_autocast_enabled("cuda") or deterministic():
        return None
    dt = torch.get_autocast_dtype("cuda")
    on = {torch.bfloat16: BF16_TRAINING_CORE, torch.float16: FP16_TRAINING_CORE}.get(dt, False)
    return dt if on else None


def _mode16_fwd(takes16):
    """torch.amp.custom_fwd(cast_inputs=torch.float32) for an autograd forward, except when `takes16(ctx, dtype, *args)` holds
    under a 16-bit training mode of that dtype: then the arguments are passed as they are (autocast off inside, as custom_fwd
    does) and ctx.mode16 is the dtype (None otherwise)."""
    def decorate(fwd):
        widened = torch.amp.custom_fwd(fwd, device_type="cuda", cast_inputs=torch.float32)

        @functools.wraps(fwd)
        def wrapper(ctx, *args):
            dt = _autocast_mode16()
            ctx.mode16 = dt if dt is not None and takes16(ctx, dt, *args) else None
            if ctx.mode16 is None:
                return widened(ctx, *args)
            ctx._dtype, ctx._fwd_used_autocast = dt, False    # what custom_bwd reads
            with torch.autocast("cuda", enabled=False):
                return fwd(ctx, *args)
        return wrapper
    return decorate


_LN_WIDTHS = {32, 64, 96, 128, 192, 256, 384, 512, 768, 1024, 1536}   # C with an instantiation of sigma_layernorm_bwd
FUSED_LAYERNORM = True


class LayerNormFn(torch.autograd.Function):
    """nn.LayerNorm over the last dim under autograd: forward = sigma_layernorm_fwd, backward = sigma_layernorm_bwd (dx, dweight, dbias in
    one pass over x and dy; nothing saved but x).  Numerics as F.layer_norm in fp32.  In the bf16 (fp16) training mode a bf16 (fp16)
    x stays 16-bit (sigma_layernorm_fwd_bf16io / sigma_layernorm_bwd_bf16, or the _fp16io / _fp16 pair: 16-bit x, y, dy, dx; fp32
    statistics, parameters and their gradients)."""

    @staticmethod
    @_mode16_fwd(lambda ctx, dt, x, weight, bias, eps: x.dtype == dt and weight.dtype == torch.float32)
    def forward(ctx, x, weight, bias, eps):
        x2 = x.contiguous().view(-1, x.shape[-1])
        y = torch.empty_like(x2)
        w, b = weight.contiguous(), bias.contiguous()
        fn = {torch.bfloat16: "sigma_layernorm_fwd_bf16io", torch.float16: "sigma_layernorm_fwd_fp16io"}.get(ctx.mode16, "sigma_layernorm_fwd")
        _lib.check(getattr(_lib.lib(), fn)(ptr(x2), ptr(w), ptr(b), ptr(y), x2.shape[0], x2.shape[1], float(eps), stream()), fn)
        ctx.save_for_backward(x2, w)
        ctx.eps = float(eps)
        return y.view(x.shape)

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, dy):
        x2, w = ctx.saved_tensors
        dx = torch.empty_like(x2)
        dw, db = torch.empty_like(w), torch.empty_like(w)
        if ctx.mode16 is not None:
            dy2 = dy.contiguous().to(ctx.mode16).view(-1, x2.shape[1])
            fn = "sigma_layernorm_bwd_bf16" if ctx.mode16 == torch.bfloat16 else "sigma_layernorm_bwd_fp16"
            _lib.check(getattr(_lib.lib(), fn)(ptr(x2), ptr(dy2), ptr(w), ptr(dx), ptr(dw), ptr(db), x2.shape[0], x2.shape[1], ctx.eps,
                                               stream()), fn)
            return dx.view(dy.shape), dw, db, None
        dy2 = dy.contiguous().float().view(-1, x2.shape[1])
        if deterministic():
            L_ = _lib.lib()
            wsb = L_.sigma_layernorm_bwd_det_workspace_bytes(x2.shape[0], x2.shape[1])
            ws = torch.empty(max(wsb, 16), dtype=torch.uint8, device=x2.device)
            _lib.check(L_.sigma_layernorm_bwd_det(ptr(x2), ptr(dy2), ptr(w), ptr(dx), ptr(dw), ptr(db), x2.shape[0], x2.shape[1],
                                                  ctx.eps, ptr(ws), wsb, stream()), "sigma_layernorm_bwd_det")
            return dx.view(dy.shape), dw, db, None
        _lib.check(_lib.lib().sigma_layernorm_bwd(ptr(x2), ptr(dy2), ptr(w), ptr(dx), ptr(dw), ptr(db), x2.shape[0], x2.shape[1], ctx.eps,
                                                 stream()), "sigma_layernorm_bwd")
        return dx.view(dy.shape), dw, db, None


def layer_norm(norm, x):
    """`norm(x)` for an nn.LayerNorm over the last dim: the library pair under autograd when the width has an instantiation, the module
    itself otherwise (other widths, no affine parameters, CPU tensors are the caller's error elsewhere)."""
    if (FUSED_LAYERNORM and x.is_cuda and torch.is_grad_enabled() and isinstance(norm, torch.nn.LayerNorm) and norm.elementwise_affine
            and norm.bias is not None and len(norm.normalized_shape) == 1 and x.shape[-1] in _LN_WIDTHS
            and (x.dtype == torch.float32 or torch.is_autocast_enabled())):
        return LayerNormFn.apply(x, norm.weight, norm.bias, norm.eps)
    return norm(x)


_DWCONV_FWD = {torch.float32: "sigma_dwconv3x3_silu_fwd", torch.bfloat16: "sigma_dwconv3x3_silu_fwd_bf16",
               torch.float16: "sigma_dwconv3x3_silu_fwd_fp16"}
_DWCONV_BWD = {torch.float32: "sigma_dwconv3x3_silu_bwd", torch.bfloat16: "sigma_dwconv3x3_silu_bwd_bf16",
               torch.float16: "sigma_dwconv3x3_silu_bwd_fp16"}


def _rows_ok(t, row_stride):
    """t (B, ..., D) can be passed as rows `row_stride` elements apart with a batch stride: unit channel stride and 16-byte aligned
    pointer and strides, as the library's TMA maps need"""
    q = 16 // t.element_size()
    return t.stride(-1) == 1 and t.data_ptr() % 16 == 0 and row_stride % q == 0 and t.stride(0) % q == 0


class DwConvSiLUFn(torch.autograd.Function):
    """SiLU(nn.Conv2d(D, D, 3, padding=1, groups=D)(x)) of a channels-last activation under autograd: x (B, H, W, D), whose pixel rows
    may be a strided view (the x half of in_proj's [x | z] output) -> xc (B, H·W, D) in x's dtype (fp32, bf16 or fp16).  Forward =
    sigma_dwconv3x3_silu_fwd[_bf16|_fp16] with the fp32 weights as given (autocast is off inside, so it does not cast them); backward
    = sigma_dwconv3x3_silu_bwd[_bf16|_fp16], which recomputes the pre-activation from x, so the node saves nothing but x.  dweight and
    dbias are fp32 in the parameters' shapes.  The backward is deterministic by construction: one kernel with or without
    torch.use_deterministic_algorithms(True)."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        B, H, W, D = x.shape
        if x.dtype not in _DWCONV_FWD or weight.shape != (D, 1, 3, 3) or weight.dtype != torch.float32 or \
                (bias is not None and bias.dtype != torch.float32):
            raise RuntimeError(f"DwConvSiLUFn: a 3x3 depthwise conv with fp32 weights over fp32 / bf16 / fp16 x, got x {x.dtype}, "
                               f"weight {tuple(weight.shape)} {weight.dtype}")
        if not (_rows_ok(x, x.stride(2)) and x.stride(1) == W * x.stride(2)):
            x = x.contiguous()
        w = weight.contiguous()
        b = bias.contiguous() if bias is not None else None
        y = torch.empty((B, H * W, D), dtype=x.dtype, device=x.device)
        fn = _DWCONV_FWD[x.dtype]
        with torch.autocast("cuda", enabled=False):
            _lib.check(getattr(_lib.lib(), fn)(ptr(x), x.stride(2), x.stride(0), ptr(w), ptr(b), ptr(y), H * W * D, B, H, W, D, stream()),
                       fn)
        ctx.save_for_backward(x, w, b)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, b = ctx.saved_tensors
        B, H, W, D = x.shape
        dy = dy.to(x.dtype)
        if not (_rows_ok(dy, D) and dy.stride(1) == D):
            dy = dy.contiguous()                 # a slice of the (B, 2L, D) core gradient (ConMB) passes as it is
        dx = torch.empty((B, H, W, D), dtype=x.dtype, device=x.device)
        dw = torch.empty_like(w)
        db = torch.empty_like(b) if b is not None else None
        L_ = _lib.lib()
        wsb = L_.sigma_dwconv3x3_silu_bwd_workspace_bytes(B, H, W, D)
        ws = torch.empty(wsb, dtype=torch.uint8, device=x.device)
        fn = _DWCONV_BWD[x.dtype]
        _lib.check(getattr(L_, fn)(ptr(x), x.stride(2), x.stride(0), ptr(w), ptr(b), ptr(dy), dy.stride(0), ptr(dx), H * W * D, ptr(dw),
                                   ptr(db), B, H, W, D, ptr(ws), wsb, stream()), fn)
        return dx, dw, db


# ---- the ChannelAttentionBlock's dense convs under autograd ----
# On, CVSSDecoderBlock's training forward runs cab[0] -> GELU -> cab[2] as one CabConvFn (or, where C/3 is not a multiple of 4,
# CabConvPitchedFn) on channels-last tensors (library kernels forward and backward); off, it runs nn.Conv2d (cuDNN) on an NCHW copy.
# Applies to fp32 without autocast (cab_conv_fn).
FUSED_CAB_TRAINING = True


def _conv3x3_ok(conv, pitched=False):
    """a 3x3 / pad 1 / stride 1 conv with bias whose channel counts are multiples of 4 (pitched: any counts)"""
    return (isinstance(conv, torch.nn.Conv2d) and conv.kernel_size == (3, 3) and conv.stride == (1, 1) and conv.padding == (1, 1)
            and conv.dilation == (1, 1) and conv.groups == 1 and (pitched or (conv.in_channels % 4 == 0 and conv.out_channels % 4 == 0))
            and conv.bias is not None and conv.padding_mode == "zeros")


def _cab_ok(cab, x, pitched):
    return (FUSED_TRAINING and FUSED_CAB_TRAINING and torch.is_grad_enabled() and x.is_cuda and x.dtype == torch.float32
            and not torch.is_autocast_enabled("cuda") and isinstance(cab[1], torch.nn.GELU) and cab[1].approximate == "none"
            and _conv3x3_ok(cab[0], pitched) and _conv3x3_ok(cab[2], pitched) and cab[0].out_channels == cab[2].in_channels)


def cab_conv_ok(cab, x):
    """CabConvFn takes `cab` (the nn.Sequential of ChannelAttentionBlock) on x: autograd recording, both switches on, fp32 CUDA x with
    autocast off, an exact nn.GELU between two 3x3 / pad 1 / stride 1 convs whose channel counts are multiples of 4"""
    return _cab_ok(cab, x, False)


def cab_conv_fn(cab, x):
    """the autograd node that runs `cab` on x in training: CabConvFn where cab_conv_ok; CabConvPitchedFn where only C/3 (cab[0]'s
    output channels) is not a multiple of 4 (Sigma-base's 42 / 85 / 170, hidden 32's 10); None: the cuDNN route"""
    if cab_conv_ok(cab, x):
        return CabConvFn
    if _cab_ok(cab, x, True) and cab[0].in_channels % 4 == 0 and cab[2].out_channels % 4 == 0:
        return CabConvPitchedFn
    return None


def _round4(n):
    return (n + 3) // 4 * 4


def _tf32_split(w):
    """(hi, lo) of sigma_split_tf32_fwd, computed per call (inside a captured graph, so a replayed optimizer step is seen)"""
    hi, lo = torch.empty_like(w), torch.empty_like(w)
    _lib.check(_lib.lib().sigma_split_tf32_fwd(ptr(w), ptr(hi), ptr(lo), w.numel(), stream()), "sigma_split_tf32_fwd")
    return hi, lo


def _w9(w, x3, grad=False, pitch=None):
    """the nn.Conv2d weight (Cout, Cin, 3, 3) as the conv kernel's (9, Cout, Cin) or, grad, the data gradient's flipped and transposed
    (9, Cin, Cout), with its tf32x3 split when x3 (else lo = None); pitch: rows zero-padded to that many elements"""
    w = w.detach()
    w9 = (w.flip(2, 3).permute(2, 3, 1, 0) if grad else w.permute(2, 3, 0, 1)).reshape(-1, w.shape[0] if grad else w.shape[1])
    if pitch is not None and pitch > w9.shape[1]:
        w9 = F.pad(w9, (0, pitch - w9.shape[1]))
    w9 = w9.contiguous()
    return _tf32_split(w9) if x3 else (w9, None)


def _cab_forward(x, w1, b1, w2, b2, x3, pitched):
    """(y, pre) of the CAB node's forward.  pitched: h and pre are (B, H, W, round4(C1)) and the pitched entry points run"""
    B, H, W, C = x.shape
    C1, C2 = w1.shape[0], w2.shape[0]
    k1 = _round4(C1) if pitched else C1
    L_ = _lib.lib()
    pre = torch.empty((B, H, W, k1), dtype=torch.float32, device=x.device)
    h = torch.empty_like(pre)
    y = torch.empty((B, H, W, C2), dtype=torch.float32, device=x.device)
    hi, lo = _w9(w1, x3)
    if pitched:
        _lib.check(L_.sigma_conv3x3_gelu_save_pitched_tf32(ptr(x), C, ptr(hi), C, ptr(lo), ptr(b1), ptr(h), ptr(pre), k1, B, H, W, C, C1,
                                                           stream()), "sigma_conv3x3_gelu_save_pitched_tf32")
        hi, lo = _w9(w2, x3, pitch=k1)
        _lib.check(L_.sigma_conv3x3_pitched_tf32(ptr(h), k1, ptr(hi), k1, ptr(lo), ptr(b2), 0, ptr(y), C2, B, H, W, C1, C2, stream()),
                   "sigma_conv3x3_pitched_tf32")
    else:
        _lib.check(L_.sigma_conv3x3_gelu_save_tf32(ptr(x), ptr(hi), ptr(lo), ptr(b1), ptr(h), ptr(pre), B, H, W, C, C1, stream()),
                   "sigma_conv3x3_gelu_save_tf32")
        hi, lo = _w9(w2, x3)
        _lib.check(L_.sigma_conv3x3_tf32(ptr(h), ptr(hi), ptr(lo), ptr(b2), 0, ptr(y), B, H, W, C1, C2, stream()), "sigma_conv3x3_tf32")
    return y, pre


def _cab_backward(x, pre, w1, w2, dy, x3, pitched):
    """(dx, dw1, db1, dw2, db2) of the CAB node from the saved x and pre-activation.  Every activation's row pitch is its last
    dimension (pitched: pre and dpre at round4(C1))."""
    B, H, W, C = x.shape
    C1, C2 = w1.shape[0], w2.shape[0]
    L_ = _lib.lib()

    def wgrad(xin, gelu_x, g, cin, cout):
        dw = torch.empty((cout, cin, 3, 3), dtype=torch.float32, device=x.device)
        db = torch.empty(cout, dtype=torch.float32, device=x.device)
        wsb = L_.sigma_conv3x3_wgrad_workspace_bytes(B, H, W, cin, cout)
        ws = torch.empty(wsb, dtype=torch.uint8, device=x.device)
        if pitched:
            _lib.check(L_.sigma_conv3x3_wgrad_pitched_tf32(ptr(xin), xin.shape[-1], gelu_x, ptr(g), g.shape[-1], ptr(dw), ptr(db), B, H,
                                                           W, cin, cout, int(x3), ptr(ws), wsb, stream()),
                       "sigma_conv3x3_wgrad_pitched_tf32")
        else:
            _lib.check(L_.sigma_conv3x3_wgrad_tf32(ptr(xin), gelu_x, ptr(g), ptr(dw), ptr(db), B, H, W, cin, cout, int(x3), ptr(ws), wsb,
                                                   stream()), "sigma_conv3x3_wgrad_tf32")
        return dw, db

    def dgrad(g, w, gelu_pre, cin, cout):
        ld = _round4(cin) if pitched else cin
        dx = torch.empty((B, H, W, ld), dtype=torch.float32, device=x.device)
        if pitched:
            hi, lo = _w9(w, x3, grad=True, pitch=g.shape[-1])
            _lib.check(L_.sigma_conv3x3_dgrad_pitched_tf32(ptr(g), g.shape[-1], ptr(hi), g.shape[-1], ptr(lo), ptr(gelu_pre), ptr(dx), ld,
                                                           B, H, W, cin, cout, stream()), "sigma_conv3x3_dgrad_pitched_tf32")
        else:
            hi, lo = _w9(w, x3, grad=True)
            _lib.check(L_.sigma_conv3x3_dgrad_tf32(ptr(g), ptr(hi), ptr(lo), ptr(gelu_pre), ptr(dx), B, H, W, cin, cout, stream()),
                       "sigma_conv3x3_dgrad_tf32")
        return dx

    dw2, db2 = wgrad(pre, 1, dy, C1, C2)
    dpre = dgrad(dy, w2, pre, C1, C2)          # the gradient at conv 1's pre-activation
    dw1, db1 = wgrad(x, 0, dpre, C, C1)
    dx = dgrad(dpre, w1, None, C, C1)
    return dx, dw1, db1, dw2, db2


class CabConvFn(torch.autograd.Function):
    """cab[2](GELU(cab[0](x))) of ChannelAttentionBlock on a channels-last fp32 x (B, H, W, C) -> (B, H, W, C) under autograd, both
    convs 3x3 / pad 1 with bias.  Forward = sigma_conv3x3_gelu_save_tf32 (conv 1 + bias, keeping the pre-activation, and its GELU)
    + sigma_conv3x3_tf32 (conv 2 + bias); backward = sigma_conv3x3_wgrad_tf32 of conv 2 (GELU applied to the saved pre-activation as
    it is staged), sigma_conv3x3_dgrad_tf32 of conv 2 times GELU', then the wgrad and dgrad of conv 1.  It saves x and the
    pre-activation, not the GELU output.  Precision follows torch.backends.cudnn.allow_tf32 at the forward, as nn.Conv2d's does (True:
    one TF32 MMA per k-step; False: tf32x3).  The weights are re-ordered (and split) per call, never from an inference cache, so a
    graph-replayed step sees the optimizer's updates.  The weight gradients are deterministic by construction (fixed-order partial
    sums), with or without torch.use_deterministic_algorithms(True)."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2):
        x = x.contiguous()
        ctx.x3 = not torch.backends.cudnn.allow_tf32
        y, pre = _cab_forward(x, w1, b1, w2, b2, ctx.x3, False)
        ctx.save_for_backward(x, pre, w1, w2)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, pre, w1, w2 = ctx.saved_tensors
        return _cab_backward(x, pre, w1, w2, dy.contiguous(), ctx.x3, False)


class CabConvPitchedFn(torch.autograd.Function):
    """CabConvFn for C1 = cab[0].out_channels that is not a multiple of 4 (C still is): the same calls, order, precision rule and
    determinism on the pitched entry points (sigma_conv3x3_*_pitched_tf32).  The GELU output and the saved pre-activation are
    (B, H, W, round4(C1)), as is the gradient at the pre-activation; their pad channels are never written and never reach an output.
    The weights that are read along C1 (conv 2's, and conv 1's transposed for its data gradient) are re-ordered per call with their
    rows zero-padded to round4(C1)."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2):
        x = x.contiguous()
        ctx.x3 = not torch.backends.cudnn.allow_tf32
        y, pre = _cab_forward(x, w1, b1, w2, b2, ctx.x3, True)
        ctx.save_for_backward(x, pre, w1, w2)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, pre, w1, w2 = ctx.saved_tensors
        return _cab_backward(x, pre, w1, w2, dy.contiguous(), ctx.x3, True)


_SAVED_BF16 = 2               # `saved` of _call_ss2d_bwd: the arguments are those of sigma_ss2d_scan_bwd_saved_bf16
_SAVED_FP16 = 3               # ... of sigma_ss2d_scan_bwd_saved_fp16 (the same layout)


def _call_ss2d_bwd(args, saved=True, det=False):
    """The native call of the fused backward, sigma_ss2d_scan_bwd_saved (_det when det; _bf16 / _fp16 when saved is _SAVED_BF16 /
    _SAVED_FP16).  A module-level function so that bench.py can bracket it with events, through a wrapper that passes (args, saved)
    on: so the 16-bit training modes are values of `saved`, not another argument."""
    from . import fused
    fn = ("sigma_ss2d_scan_bwd_saved_bf16" if saved == _SAVED_BF16 else
          "sigma_ss2d_scan_bwd_saved_fp16" if saved == _SAVED_FP16 else
          "sigma_ss2d_scan_bwd_saved_det" if det else "sigma_ss2d_scan_bwd_saved")
    _lib.check(getattr(_lib.lib(), fn)(*args, int(fused._FORCE_SPLIT or 0), stream()), fn)


class FusedSS2DCore(torch.autograd.Function):
    """cross_selective_scan (vmamba.py:165-226, kind CROSS4) / cross_selective_scan_multimodal_k2 (:369-430, kind SEQ2) without
    out_norm, on channels-last activations:  xc (B, Lseq, D) -> y (B, Lseq, D) = sum over directions of the scan outputs, each at
    the position it belongs to (CrossMerge).  Forward = the inference kernels (x_proj GEMM + the fused scan) in their state-saving
    build (sigma_ss2d_scan_fwd_save: also keeps delta' and the scan state entering every 16-position block); backward =
    sigma_ss2d_scan_bwd_saved (one reverse sweep; no CrossScan / CrossMerge tensors) + the x_proj / dt_proj weight-gradient GEMMs.
    Kind CROSS is Cross_Mamba_Attention_SSM.forward (vmamba.py:1508-1545): xc (2·images, L, D) modality-major, the parameters of
    the two modalities stacked (x_proj_weight (2, R+2N, D), dt_projs_weight (2, D, R), dt_projs_bias (2, D), A_logs (2D, N), Ds
    (2D)); each half runs its own x_proj and weights and reads C from the other half.  It has no deterministic backward.
    The bf16 training mode (BF16_TRAINING_CORE, bf16 autocast, not deterministic, some input needs a gradient):
    xc is taken (or cast to) bf16 and never widened, x_proj runs the bf16 GEMM with fp32 x_dbl out, sigma_ss2d_scan_fwd_save_bf16
    writes bf16 y and the bf16 delta' its own recurrence ran on, and the backward (sigma_ss2d_scan_bwd_saved_bf16) takes a bf16 dy
    and returns a bf16 dxc rounded once from the fp32 sum of the directions and the x_proj term; parameter gradients are fp32.
    The fp16 training mode (FP16_TRAINING_CORE, fp16 autocast, the same conditions) is the same with fp16 for bf16: the x_proj GEMM is
    sigma_linear_fp16, the pair sigma_ss2d_scan_fwd_save_fp16 / sigma_ss2d_scan_bwd_saved_fp16; a dxc past ±65504 becomes ±inf."""

    @staticmethod
    @_mode16_fwd(lambda ctx, dt, xc, *a: any(ctx.needs_input_grad) and fused_core_ok(xc, xc.shape[-1], a[3].shape[1])
                 and all(t.dtype == torch.float32 for t in a[:5]))
    def forward(ctx, xc, x_proj_weight, dt_projs_weight, dt_projs_bias, A_logs, Ds, kind, H, W):
        from . import fused
        Kw, _, D = x_proj_weight.shape
        cross = kind == _lib.DIRS_CROSS
        K = 1 if cross else Kw                   # x_dbl rows per position
        N, R = A_logs.shape[1], dt_projs_weight.shape[2]
        Cp = _lib.lib().sigma_ss2d_padded_cp(N, R)
        xc = xc.contiguous()
        if ctx.mode16 is not None:
            xc = xc.to(ctx.mode16)               # a 16-bit xc of that dtype (the conv + SiLU under autocast) passes through untouched
        B, Lseq, _ = xc.shape
        xw = torch.cat([fused._pack_xproj(x_proj_weight[k], N, R, Cp) for k in range(Kw)], dim=0).contiguous()     # (Kw·Cp, D)
        if cross:   # each modality's half of the batch through its own x_proj
            if B % 2:
                raise RuntimeError(f"FusedSS2DCore: kind CROSS needs a batch of 2·images, got {B}")
            n = B // 2 * Lseq
            xdbl = torch.empty((B * Lseq, Cp), dtype=torch.float32, device=xc.device)
            for m in range(2):
                fused.linear(xc.view(B * Lseq, D)[m * n:(m + 1) * n], xw[m * Cp:(m + 1) * Cp], out=xdbl[m * n:(m + 1) * n], kind="x_proj")
        else:
            xdbl = fused.linear(xc.view(B * Lseq, D), xw, kind="x_proj")                                            # (B·Lseq, K·Cp)
        dtw, dtb = dt_projs_weight.contiguous(), dt_projs_bias.contiguous()
        A = (-torch.exp(A_logs)).contiguous()
        Dsc = Ds.contiguous()
        y, delta, hs = fused.ss2d_scan_save(kind, xc, xdbl, dtw, dtb, A, Dsc, B, H, W, D, N, R, Cp)                  # y (K, B, Lseq, D)
        ctx.save_for_backward(xc, xdbl, xw, dtw, dtb, A, Dsc, delta, hs)
        ctx.meta = (kind, H, W, K, D, N, R, Cp)
        return y[0] if cross else y.sum(0)

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, dy):
        from . import fused
        xc, xdbl, xw, dtw, dtb, A, Ds, delta, hs = ctx.saved_tensors
        kind, H, W, K, D, N, R, Cp = ctx.meta
        cross = kind == _lib.DIRS_CROSS
        Kw = 2 if cross else K                   # parameter sets
        det = deterministic()
        if cross and det:
            raise RuntimeError("FusedSS2DCore: kind CROSS has no deterministic backward; under torch.use_deterministic_algorithms(True) "
                               "CroMB trains through the op-level _det kernels (CrossMambaFusion_SS2D_SSM routes there itself)")
        B, Lseq, _ = xc.shape
        m16 = ctx.mode16
        dy = dy.contiguous().to(m16) if m16 is not None else dy.contiguous().float()
        dev = xc.device
        ddelta = torch.empty((K, B, Lseq, D), dtype=torch.float32, device=dev)
        dxc = torch.empty((B, Lseq, D), dtype=torch.float32, device=dev)
        dxdbl = torch.empty((B * Lseq, K, Cp), dtype=torch.float32, device=dev)
        dA = torch.empty((Kw * D, N), dtype=torch.float32, device=dev)
        dDs = torch.empty(Kw * D, dtype=torch.float32, device=dev)
        ddtb = torch.empty((Kw, D), dtype=torch.float32, device=dev)
        L_ = _lib.lib()
        wsb = (L_.sigma_ss2d_scan_bwd_det_workspace_bytes if det else L_.sigma_ss2d_scan_bwd_workspace_bytes)(kind, B, H, W, D, N)
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        args = (kind, ptr(xc), ptr(xdbl), ptr(dtw), ptr(dtb), ptr(A), ptr(Ds), ptr(dy), ptr(delta), ptr(hs),
                ptr(dxc), ptr(ddelta), ptr(dxdbl), ptr(dA), ptr(dDs), ptr(ddtb), B, H, W, D, N, R, Cp, ptr(ws), wsb)
        # det only when set: bench.py --mode train brackets this call with a wrapper that takes (args, saved)
        if m16 is not None:
            _call_ss2d_bwd(args, _SAVED_BF16 if m16 == torch.bfloat16 else _SAVED_FP16)
            xc = xc.float()                      # only the x_proj weight gradient below (a torch matmul) needs the widened copy
        else:
            _call_ss2d_bwd(args, True, True) if det else _call_ss2d_bwd(args, True)
        if cross:   # the same two steps per modality half m (its rows of dxdbl / ddelta / xc, its weight set)
            n = B // 2 * Lseq
            xd, dxd, dd = xdbl.view(2, n, Cp), dxdbl.view(2, n, Cp), ddelta.view(2, n, D)
            xcm, dxcm, xw3 = xc.view(2, n, D), dxc.view(2, n, D), xw.view(2, Cp, D)
            dW, dxw = torch.empty_like(dtw), torch.empty_like(xw3)
            for m in range(2):
                dxd[m, :, 2 * N:2 * N + R].copy_(dd[m] @ dtw[m])
                dW[m] = dd[m].t() @ xd[m, :, 2 * N:2 * N + R]
                dxcm[m].addmm_(dxd[m], xw3[m])
                dxw[m] = dxd[m].t() @ xcm[m]
            dxpw = torch.cat([dxw[:, 2 * N:2 * N + R], dxw[:, 0:N], dxw[:, N:2 * N]], dim=1)
            return (dxc.to(m16) if m16 is not None else dxc), dxpw, dW, ddtb, dA * A, dDs, None, None, None
        # dt_proj: d dt_r = ddelta_k · W_dt[k]  (into the dt_r columns of dxdbl),  dW_dt[k] = ddelta_k^T · dt_r_k
        xd3 = xdbl.view(B * Lseq, K, Cp)
        dW = torch.empty_like(dtw)
        for k in range(K):
            ddk = ddelta[k].view(B * Lseq, D)
            dxdbl[:, k, 2 * N:2 * N + R].copy_(ddk @ dtw[k])
            dW[k] = ddk.t() @ xd3[:, k, 2 * N:2 * N + R]
        # x_proj: dxc += dxdbl · xw,  d xw = dxdbl^T · xc
        d2 = dxdbl.view(B * Lseq, K * Cp)
        dxc2 = dxc.view(B * Lseq, D)
        dxc2.addmm_(d2, xw)
        dxw = (d2.t() @ xc.view(B * Lseq, D)).view(K, Cp, D)
        dxpw = torch.cat([dxw[:, 2 * N:2 * N + R], dxw[:, 0:N], dxw[:, N:2 * N]], dim=1)          # back to [dt | B | C] rows
        return (dxc.to(m16) if m16 is not None else dxc), dxpw, dW, ddtb, dA * A, dDs, None, None, None


# ---- deterministic training: bilinear upsampling and cross-entropy ----
def _pair(v):
    return (v, v) if not isinstance(v, (tuple, list)) else tuple(v)


class UpsampleBilinearFn(torch.autograd.Function):
    """F.interpolate(mode="bilinear", align_corners=False) of a CUDA tensor with a deterministic backward: forward is the kernel
    F.interpolate runs without the switch (same bits); backward is sigma_upsample_bilinear_bwd, a gather in which every input
    pixel sums the output pixels that tap it in a fixed order (torch's own backward adds them with atomics; under
    use_deterministic_algorithms torch falls back to a slower index_put decomposition with other forward bits).
    NCHW and channels-last inputs; `size=` or `scale_factor=` with torch's source-index rule for each."""

    @staticmethod
    def forward(ctx, x, size, scale_factor):
        # the native kernel F.interpolate calls (under the switch F.interpolate itself would route to a decomposition with other bits)
        y = torch._C._nn.upsample_bilinear2d(x, list(_pair(size)) if size is not None else None, False,
                                             [float(s) for s in _pair(scale_factor)] if scale_factor is not None else None)
        Hin, Win = x.shape[2:]
        Hout, Wout = y.shape[2:]
        if scale_factor is not None:   # torch passes the scale to the kernel: ratio = (float) (1.0 / scale)
            rh, rw = (float(np.float32(1.0 / float(s))) for s in _pair(scale_factor))
        else:                          # ratio = (float) in / out, in fp32
            rh, rw = float(np.float32(Hin) / np.float32(Hout)), float(np.float32(Win) / np.float32(Wout))
        ctx.meta = (tuple(x.shape), x.dtype, rh, rw, x.is_contiguous(memory_format=torch.channels_last) and not x.is_contiguous())
        return y

    @staticmethod
    def backward(ctx, dy):
        (B, C, Hin, Win), dtype, rh, rw, cl = ctx.meta
        Hout, Wout = dy.shape[2:]
        fmt = torch.channels_last if cl else torch.contiguous_format
        dy = dy.float().contiguous(memory_format=fmt)
        dx = torch.empty((B, C, Hin, Win), dtype=torch.float32, device=dy.device, memory_format=fmt)
        _lib.check(_lib.lib().sigma_upsample_bilinear_bwd(ptr(dy), ptr(dx), B, C, Hin, Win, Hout, Wout, rh, rw, int(cl), stream()),
                   "sigma_upsample_bilinear_bwd")
        return dx.to(dtype), None, None


def upsample_bilinear(x, size=None, scale_factor=None):
    """F.interpolate(x, size, scale_factor, mode="bilinear", align_corners=False); under autograd with
    torch.use_deterministic_algorithms(True), through UpsampleBilinearFn (same forward, deterministic backward)."""
    if deterministic() and torch.is_grad_enabled() and x.requires_grad and x.is_cuda:
        return UpsampleBilinearFn.apply(x, size, scale_factor)
    return F.interpolate(x, size=size, scale_factor=scale_factor, mode="bilinear", align_corners=False)


def plain_cross_entropy(criterion):
    """The ignore_index of an nn.CrossEntropyLoss that deterministic_cross_entropy computes exactly (no class weights, no label
    smoothing, reduction "mean"), else None."""
    if (type(criterion) is torch.nn.CrossEntropyLoss and criterion.weight is None and criterion.label_smoothing == 0.0
            and criterion.reduction == "mean"):
        return criterion.ignore_index
    return None


def deterministic_cross_entropy(logits, target, ignore_index):
    """nn.CrossEntropyLoss(ignore_index=ignore_index)(logits, target) for (B, K, ...) logits without nll_loss, whose CUDA
    backward raises under use_deterministic_algorithms: log-softmax over K, gather of the target class (torch makes gather's
    backward deterministic under the switch), then the mean over the pixels whose target is not ignore_index."""
    keep = target != ignore_index
    t = torch.where(keep, target, torch.zeros_like(target)).unsqueeze(1)
    nll = -torch.gather(F.log_softmax(logits, dim=1), 1, t).squeeze(1)
    nll = torch.where(keep, nll, torch.zeros_like(nll))
    return nll.sum() / keep.sum().to(nll.dtype)
