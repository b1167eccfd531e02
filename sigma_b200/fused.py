"""Inference pipeline of the Sigma hot path over libsigma_b200 (channels-last, fp32 storage).

Per SS2D block (vmamba.py:1067-1089 + cross_selective_scan :165-226) the kernels are
    LayerNorm -> in_proj GEMM -> dwconv3x3+SiLU -> x_proj GEMM (all 4 directions in one) ->
    fused 4-direction scan (CrossScan index math + dt_proj + softplus + scan, TMA-staged) ->
    merge(4) + out_norm + ·SiLU(z) -> out_proj GEMM (+ residual)
so neither CrossScan's (B,4,D,L) copy, nor delta (B,4D,L), nor CrossMerge's transposes ever exist.
Dense projections go through `linear()` (see there).  Everything here assumes no autograd.

Storage in the bf16 mode (`precision() == "bf16"`, selected by torch.autocast("cuda", dtype=torch.bfloat16) with autograd off):
the residual stream between blocks stays fp32, as do the LayerNorm statistics, the scan state and every accumulator.  Inside
SS2D, ConMB_SS2D, CrossMambaFusion_SS2D_SSM and PatchMerging2D, the LayerNorm output that feeds a GEMM, xz / tr / te,
xc / seq, the scan output y and the gated yg / ycat / yn are stored in bf16 (each value rounded once, to nearest even).
x_dbl stays fp32 (it carries dt, B and C into softplus and exp, and it is small), the SE gates of ConMB average in fp32, and
out_proj, the PatchMerging reduction and x_proj write fp32, so their residual and rscale epilogues read fp32.  Everything
else (the decoder's CAB convs, patch embed, PatchExpand, UpsampleExpand, the final head, the pools) runs in the dense mode
torch's matmul switch selects, with autocast switched off around the torch ops the fused path calls.

The FP8 mode (`precision() == "fp8"`, selected by `fp8_inference()` with autograd off, autocast or not) stores exactly what the
bf16 mode stores, and runs the in_proj / in_proj_modalx and out_proj / out_proj_rgb / out_proj_e GEMMs of SS2D, ConMB and CroMB
and the PatchMerging2D reduction on e4m3 operands (sigma_linear_fp8): activations with one fp32 scale per row, weights with one
per output channel (the formula in include/sigma_b200.h).  The LayerNorms in front of in_proj, the patch-merge LayerNorm and
SS2D's / CroMB's merge + norm + gate emit the e4m3 rows and scales themselves; ConMB's and CroMB's in_proj operands and ConMB's
two-part ycat go through the standalone row quantizer.  x_proj stays bf16 (it feeds softplus and exp).

The fp16 mode (`precision() == "fp16"`, selected by `fp16_inference()` with autograd off, autocast or not) stores exactly what
the bf16 mode stores, in fp16 instead of bf16, and runs the same GEMMs on fp16 operands (sigma_linear_fp16).  fp16 keeps 11
significant bits where bf16 keeps 8, but its range ends at ±65504: a stored value past it becomes ±inf, as torch's .half() does
(there is no saturating conversion).  torch.autocast with fp16 is not this mode: it keeps the fp32 path.
"""
import contextlib
import ctypes
from typing import NamedTuple

import torch
import torch.nn.functional as F

from . import _lib
from ._lib import ptr, stream

EPS = 1e-5
_FORCE_SPLIT = 0  # test hook: force the number of L-segments of the fused scan


# ---------------------------------------------------------------- primitive wrappers
class E4M3Rows(NamedTuple):
    """An FP8-mode GEMM operand: q (rows, ...) torch.float8_e4m3fn and one fp32 scale per row, s (rows,); row r is q[r]·s[r]."""
    q: torch.Tensor
    s: torch.Tensor

    def view(self, *shape):
        return E4M3Rows(self.q.view(*shape), self.s)


def _e4m3_empty(rows, C, device):
    return E4M3Rows(torch.empty((rows, C), dtype=torch.float8_e4m3fn, device=device),
                    torch.empty((rows,), dtype=torch.float32, device=device))


def quantize_rows(x2d, out=None):
    """(rows, C) fp32 or bf16 with unit column stride -> E4M3Rows (sigma_quantize_e4m3_rows; per-row scale)."""
    rows, C = x2d.shape
    out = out if out is not None else _e4m3_empty(rows, C, x2d.device)
    xd = _lib.BF16 if x2d.dtype == torch.bfloat16 else _lib.F32
    _lib.check(_lib.lib().sigma_quantize_e4m3_rows(ptr(x2d), xd, x2d.stride(0), ptr(out.q), out.q.stride(0), ptr(out.s), rows, C,
                                                   stream()), "sigma_quantize_e4m3_rows")
    return out


def _entry(fn, dtype):
    """the entry point of `fn` for an element type: fp32 `fn`, bf16 `fn`_bf16, fp16 `fn`_fp16"""
    return fn + {torch.bfloat16: "_bf16", torch.float16: "_fp16"}.get(dtype, "")


def layernorm(x2d, ln, dtype=torch.float32):
    """nn.LayerNorm over the last dim of a contiguous (rows, C) fp32 tensor; dtype=torch.bfloat16 / torch.float16 stores the
    output as bf16 / fp16, dtype=torch.float8_e4m3fn returns E4M3Rows (sigma_layernorm_fwd_fp8: the fp32 result quantized per row)."""
    rows, C = x2d.shape
    if dtype == torch.float8_e4m3fn:
        y = _e4m3_empty(rows, C, x2d.device)
        _lib.check(_lib.lib().sigma_layernorm_fwd_fp8(ptr(x2d), ptr(ln.weight), ptr(ln.bias), ptr(y.q), ptr(y.s), rows, C, float(ln.eps),
                                                      stream()), "sigma_layernorm_fwd_fp8")
        return y
    y = torch.empty((rows, C), dtype=dtype, device=x2d.device)
    fn = _entry("sigma_layernorm_fwd", dtype)
    _lib.check(getattr(_lib.lib(), fn)(ptr(x2d), ptr(ln.weight), ptr(ln.bias), ptr(y), rows, C, float(ln.eps), stream()), fn)
    return y


USE_OWN_GEMM = True  # False: cuBLAS through torch (library GEMM, precision by torch's switch), kept for A/B timing only


FP8_INFERENCE = False
FP16_INFERENCE = False


@contextlib.contextmanager
def fp8_inference(on=True):
    """Switch the FP8 inference mode of the fused path on (or off) inside the block: with autograd off, precision() is "fp8"."""
    global FP8_INFERENCE
    prev, FP8_INFERENCE = FP8_INFERENCE, bool(on)
    try:
        yield
    finally:
        FP8_INFERENCE = prev


@contextlib.contextmanager
def fp16_inference(on=True):
    """Switch the fp16 inference mode of the fused path on (or off) inside the block: with autograd off, precision() is "fp16"
    (module docstring; values past ±65504 become ±inf where the mode stores fp16)."""
    global FP16_INFERENCE
    prev, FP16_INFERENCE = FP16_INFERENCE, bool(on)
    try:
        yield
    finally:
        FP16_INFERENCE = prev


def precision():
    """Precision of the fused path.  Inside fp8_inference() with autograd off it is "fp8": the bf16 mode's storage, with the
    in_proj / out_proj / PatchMerging GEMMs on e4m3 operands scaled per row and per output channel (module docstring); logits
    within 2x the error of the reference's layers under bf16 autocast with the same e4m3 quantize-dequantize at those GEMMs.
    With autograd off and torch.autocast("cuda", dtype=torch.bfloat16) active it is "bf16": the
    SS2D / ConMB / CroMB / PatchMerging interiors store bf16 and their GEMMs run bf16 wgmma (module docstring); logits within
    2x the error of the reference's own layers under the same autocast.  Inside fp16_inference() with autograd off it is "fp16",
    with or without autocast: the bf16 mode's storage and GEMMs in fp16 (11 significant bits, range ±65504); logits within 2x the
    error of the reference's layers under fp16 autocast.  fp16_inference() and fp8_inference() together are a ValueError.
    torch.autocast with fp16 is not a mode of the fused path: it keeps the fp32 modes below.  With autograd on (training) neither
    autocast nor the contexts change the fused core.
    Otherwise the dense-projection precision (the scan, LayerNorms and the convolutions' accumulation are fp32 regardless)
    follows torch's own switch, exactly like the reference's nn.Linear layers do:
      torch.backends.cuda.matmul.allow_tf32 = False (torch's default) -> "tf32x3": fp32-GRADE products on the tensor cores — the
          hand-written wgmma GEMM with the error-compensated operand split (3 MMAs per k-step, sigma_linear_tf32x3); logits agree
          with the reference's fp32 results to ~1e-6 of their scale (1e-3 bar);
      torch.backends.cuda.matmul.allow_tf32 = True -> "tf32": the same kernel, one TF32 MMA per k-step (10-bit mantissa
          operands, fp32 accumulate in registers); logits within ~3e-3 of the reference's (1e-2 bar)."""
    if not torch.is_grad_enabled() and FP8_INFERENCE and FP16_INFERENCE:
        raise ValueError("fused.precision(): fp8_inference() and fp16_inference() are both on; choose one")
    if not torch.is_grad_enabled() and FP8_INFERENCE:
        return "fp8"
    if not torch.is_grad_enabled() and FP16_INFERENCE:
        return "fp16"
    if not torch.is_grad_enabled() and torch.is_autocast_enabled("cuda") and torch.get_autocast_dtype("cuda") == torch.bfloat16:
        return "bf16"
    return _dense_precision()


def _dense_precision():
    return "tf32" if torch.backends.cuda.matmul.allow_tf32 else "tf32x3"


BF16_FLOOR = 1e-3   # fraction of the logit scale added to the bf16 bar


def logits_bar(composed_err=None):
    """Parity bar for end-to-end logits of the fused path, as a fraction of the logit scale (tests state it through this).
    bf16 has no fixed bar: it is 2 x `composed_err` + BF16_FLOOR, where `composed_err` is the error (same fraction of the
    scale) of the reference's op composition (modules.composed_path()) on the same inputs under the same autocast — so the
    caller measures it first (tests/test_bf16_gpu.py).  fp8 likewise, with the composed path run under bf16 autocast and the
    mode's e4m3 quantize-dequantize at the GEMMs it quantizes (tests/test_fp8_gpu.py); fp16 with the composed path under fp16
    autocast (tests/test_fp16_gpu.py)."""
    mode = precision()
    if mode in ("bf16", "fp8", "fp16"):
        if composed_err is None:
            raise ValueError(f"logits_bar(): the {mode} bar is relative; pass the composed path's error under the same autocast")
        return 2.0 * composed_err + BF16_FLOOR
    return 1e-2 if mode == "tf32" else 1e-3


def _fp8_mode():
    return precision() == "fp8"


def _no_autocast():
    """Context for the torch ops the fused path calls itself (SE / channel-attention gates, cuDNN fallbacks): they stay fp32."""
    return torch.autocast("cuda", enabled=False)


_FP32_KINDS = set()   # experiment hook (scripts/tf32_error_budget.py): kinds of projections forced to full precision in tf32 mode
_SPLIT = {}           # id(weight) -> (weakref, version, W_hi, W_lo): the tf32x3 operand split of a weight, made once per version
_LOWP = {}            # id(weight) -> (weakref, version, {form: copy}): the bf16 / fp16 copies ("bf16", "fp16") and the
                      # per-channel e4m3 rows and scales ("e4m3") of a weight, each made once per version


def weights_updated(tensors):
    """Record that `tensors` (parameters) were written in place where autograd did not see it, as a replayed CUDA graph's
    optimizer step does (train_util.GraphedTrainStep calls this after every replay).  It bumps each tensor's `_version`, the key
    of every derived-weight cache here (_SPLIT, _LOWP, _W9, the packed SSM parameters of _cache) and of InferencePipeline's
    re-capture, so the next inference forward rebuilds them from the new values.  One host call for the list; no kernel runs."""
    torch.autograd.graph.increment_version(tensors)


def _split_weight(w):
    import weakref
    ent = _SPLIT.get(id(w))
    if ent is not None and ent[0]() is w and ent[1] == w._version:
        return ent[2], ent[3]
    hi, lo = torch.empty_like(w), torch.empty_like(w)
    _lib.check(_lib.lib().sigma_split_tf32_fwd(ptr(w), ptr(hi), ptr(lo), w.numel(), stream()), "sigma_split_tf32_fwd")
    key = id(w)
    _SPLIT[key] = (weakref.ref(w, lambda _r, k=key: _SPLIT.pop(k, None)), w._version, hi, lo)
    return hi, lo


def _lowp_weight(w, form):
    import weakref
    ent = _LOWP.get(id(w))
    if ent is None or ent[0]() is not w or ent[1] != w._version:
        key = id(w)
        ent = (weakref.ref(w, lambda _r, k=key: _LOWP.pop(k, None)), w._version, {})
        _LOWP[key] = ent
    forms = ent[2]
    if form not in forms:
        wc = w.detach().contiguous()
        if form == "e4m3":
            forms[form] = quantize_rows(wc.float() if wc.dtype != torch.float32 else wc)
        else:
            forms[form] = wc.to(torch.bfloat16 if form == "bf16" else torch.float16)
    return forms[form]


def _bf16_weight(w):
    return _lowp_weight(w, "bf16")


def _fp16_weight(w):
    return _lowp_weight(w, "fp16")


def _e4m3_weight(w):
    """E4M3Rows of a (N, K) weight: one scale per output channel"""
    return _lowp_weight(w, "e4m3")


def linear(x2d, weight, bias=None, out=None, residual=None, rscale=None, kind="dense", out_dtype=torch.float32):
    """Dense projection out = x·W^T (+bias) (+residual·rscale) through the hand-written wgmma GEMM (csrc/gemm_tf32.cu: TMA-fed,
    register accumulators, fused epilogue), in the precision `precision()` names.  x2d (M, K) with unit column stride, row stride
    % 4 == 0; weight (N, K).  Shapes the kernel cannot take (K or N not a multiple of 4) go to torch.mm.

    Limitation: in tf32x3 mode the weight's hi / lo split is cached per weight and refreshed when `weight._version` changes
    (optimizer steps, in-place ops under torch.no_grad(), load_state_dict).  A write through `weight.data` does not change
    `_version`, so the next call still uses the split of the old values (conv3x3's re-ordered weight likewise).

    A bf16 x2d runs the bf16 instance (sigma_linear_bf16: bf16 operands, fp32 accumulation) whatever `precision()` says, with a
    bf16 copy of the weight cached on `_version` exactly like the tf32x3 split (same `.data` limitation); the output is fp32 or
    (out_dtype=torch.bfloat16) bf16.  Rows whose byte stride is not a multiple of 16 go to torch.mm.  An fp16 x2d likewise runs the
    fp16 instance (sigma_linear_fp16) with a cached fp16 copy of the weight; its output is fp32 or (out_dtype=torch.float16) fp16.

    An E4M3Rows x2d runs the e4m3 instance (sigma_linear_fp8) with the weight's per-channel e4m3 rows, cached the same way; K and
    the row stride must be multiples of 16 and N of 4 (there is no other path for it)."""
    if isinstance(x2d, E4M3Rows):
        return _linear_fp8(x2d, weight, bias, out, residual, rscale, out_dtype)
    M, K = x2d.shape
    N = weight.shape[0]
    if x2d.dtype in (torch.bfloat16, torch.float16):
        return _linear_16bit(x2d, weight, bias, out, residual, rscale, out_dtype)
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=x2d.device)
    if not USE_OWN_GEMM or K % 4 or x2d.stride(1) != 1 or x2d.stride(0) % 4 or N % 4:
        with _no_autocast():
            torch.mm(x2d, weight.t(), out=out)
        if bias is not None:
            out += bias
        if residual is not None:
            out += residual * rscale if rscale is not None else residual
        return out
    w = weight if weight.is_contiguous() else weight.contiguous()
    ldr = residual.stride(0) if residual is not None else 0
    if _dense_precision() == "tf32" and kind not in _FP32_KINDS:
        rc = _lib.lib().sigma_linear_tf32(ptr(x2d), x2d.stride(0), ptr(w), ptr(bias), ptr(residual), ldr, ptr(rscale), ptr(out),
                                          out.stride(0), M, N, K, stream())
        _lib.check(rc, "sigma_linear_tf32")
    else:
        hi, lo = _split_weight(w)
        rc = _lib.lib().sigma_linear_tf32x3(ptr(x2d), x2d.stride(0), ptr(hi), ptr(lo), ptr(bias), ptr(residual), ldr, ptr(rscale), ptr(out),
                                            out.stride(0), M, N, K, stream())
        _lib.check(rc, "sigma_linear_tf32x3")
    return out


def _linear_16bit(x2d, weight, bias, out, residual, rscale, out_dtype):
    """the bf16 or fp16 instance, by the dtype of x2d"""
    M, K = x2d.shape
    N = weight.shape[0]
    f16 = x2d.dtype == torch.float16
    if out is None:
        out = torch.empty((M, N), dtype=out_dtype, device=x2d.device)
    w = _fp16_weight(weight) if f16 else _bf16_weight(weight)
    if not USE_OWN_GEMM or K % 8 or x2d.stride(1) != 1 or x2d.stride(0) % 8 or N % 4 or out.stride(0) % 4:
        with _no_autocast():
            t = torch.mm(x2d.float(), w.float().t())              # bf16 / fp16 values are exact in fp32
            if bias is not None:
                t += bias
            if residual is not None:
                t += residual * rscale if rscale is not None else residual
            out.copy_(t)
        return out
    ldr = residual.stride(0) if residual is not None else 0
    c_dtype = {torch.bfloat16: _lib.BF16, torch.float16: _lib.F16}.get(out.dtype, _lib.F32)
    fn = "sigma_linear_fp16" if f16 else "sigma_linear_bf16"
    rc = getattr(_lib.lib(), fn)(ptr(x2d), x2d.stride(0), ptr(w), ptr(bias), ptr(residual), ldr, ptr(rscale), ptr(out), out.stride(0),
                                 c_dtype, M, N, K, stream())
    _lib.check(rc, fn)
    return out


def _linear_fp8(xq, weight, bias, out, residual, rscale, out_dtype):
    q = xq.q
    M, K = q.shape
    N = weight.shape[0]
    if K % 16 or q.stride(1) != 1 or q.stride(0) % 16 or N % 4:
        raise ValueError(f"fused.linear: the e4m3 GEMM needs K and the row stride % 16 == 0 and N % 4 == 0 (K={K}, N={N})")
    if out is None:
        out = torch.empty((M, N), dtype=out_dtype, device=q.device)
    w = _e4m3_weight(weight)
    ldr = residual.stride(0) if residual is not None else 0
    c_dtype = _lib.BF16 if out.dtype == torch.bfloat16 else _lib.F32
    rc = _lib.lib().sigma_linear_fp8(ptr(q), q.stride(0), ptr(xq.s), ptr(w.q), ptr(w.s), ptr(bias), ptr(residual), ldr, ptr(rscale),
                                     ptr(out), out.stride(0), c_dtype, M, N, K, stream())
    _lib.check(rc, "sigma_linear_fp8")
    return out


def patch_embed(conv, x):
    """The patch-embedding convolution (vmamba.py:1967-1971: Conv2d(3, C, kernel 4, stride 4)) as a GEMM: non-overlapping
    patches make im2col a pure re-ordering, (B, 3, H, W) -> (B·H/4·W/4, 3·4·4) rows in the (c, ky, kx) order of the conv
    weight, then the wgmma GEMM with the bias in its epilogue.  Returns (B, H/4, W/4, C) channels-last.  None when the
    convolution is not of that form (caller falls back to cuDNN)."""
    p = conv.kernel_size[0]
    B, Cin, H, W = x.shape
    if conv.kernel_size != (p, p) or conv.stride != (p, p) or conv.padding != (0, 0) or conv.groups != 1 or H % p or W % p or (Cin * p * p) % 4:
        return None
    cols = x.reshape(B, Cin, H // p, p, W // p, p).permute(0, 2, 4, 1, 3, 5).reshape(B * (H // p) * (W // p), Cin * p * p)
    return linear(cols, conv.weight.reshape(conv.out_channels, Cin * p * p), conv.bias, kind="patch_embed").view(B, H // p, W // p, conv.out_channels)


_W9 = {}   # id(conv.weight) -> (weakref, version, w9): the (9, Cout, Cin) re-ordering of a 3x3 conv weight


def conv3x3(x, conv, gelu=False):
    """Dense 3x3 convolution (pad 1) + bias (+ exact GELU) on a channels-last (B, H, W, Cin) tensor through the implicit-GEMM
    variant of the wgmma kernel (sigma_conv3x3_tf32).  Precision follows torch's switch for CONVOLUTIONS, as the reference's
    nn.Conv2d does: torch.backends.cudnn.allow_tf32 = True (torch's default) -> one TF32 MMA per k-step; False -> tf32x3.
    Returns (B, H, W, Cout), or None when the convolution is not of that form (caller falls back to cuDNN)."""
    import weakref
    if conv.kernel_size != (3, 3) or conv.stride != (1, 1) or conv.padding != (1, 1) or conv.dilation != (1, 1) or conv.groups != 1 \
            or conv.in_channels % 4 or conv.out_channels % 4 or not USE_OWN_GEMM:
        return None
    x = x.contiguous()
    B, H, W, Cin = x.shape
    w = conv.weight
    ent = _W9.get(id(w))
    if ent is None or ent[0]() is not w or ent[1] != w._version:
        key = id(w)
        ent = (weakref.ref(w, lambda _r, k=key: _W9.pop(k, None)), w._version,
               w.detach().permute(2, 3, 0, 1).reshape(9 * conv.out_channels, Cin).contiguous())
        _W9[key] = ent
    w9 = ent[2]
    y = torch.empty((B, H, W, conv.out_channels), dtype=torch.float32, device=x.device)
    if torch.backends.cudnn.allow_tf32:
        hi, lo = w9, None
    else:
        hi, lo = _split_weight(w9)
    rc = _lib.lib().sigma_conv3x3_tf32(ptr(x), ptr(hi), ptr(lo), ptr(conv.bias), 1 if gelu else 0, ptr(y), B, H, W, Cin, conv.out_channels, stream())
    _lib.check(rc, "sigma_conv3x3_tf32")
    return y


_W9P = {}   # id(conv.weight) -> (weakref, version, w9): the (9, Cout, Cin) re-ordering with rows padded to a multiple of 4


def _conv3x3_form(conv):
    return (conv.kernel_size == (3, 3) and conv.stride == (1, 1) and conv.padding == (1, 1) and conv.dilation == (1, 1)
            and conv.groups == 1 and conv.padding_mode == "zeros")


def cab_convs_pitched(x, cab):
    """cab[2](GELU(cab[0](x))) of ChannelAttentionBlock on a channels-last fp32 x (B, H, W, C) when C1 = cab[0].out_channels is not a
    multiple of 4 (Sigma-base's 42 / 85 / 170), which conv3x3 cannot take: conv 1 + bias + GELU into h (B, H, W, round4(C1)), whose
    pad channels the second conv never reads (sigma_conv3x3_pitched_tf32), then conv 2 + bias from h at that pitch.  The second
    conv's weight is cached re-ordered with its rows padded to round4(C1), on the weight's _version as _W9 is.  Precision as
    conv3x3's.  Returns (B, H, W, C), or None when C is not a multiple of 4 or the convs are not of that form (cuDNN fallback)."""
    import weakref
    c1, c2 = cab[0], cab[2]
    if not (USE_OWN_GEMM and _conv3x3_form(c1) and _conv3x3_form(c2)) or c1.in_channels % 4 or c2.out_channels % 4 \
            or c1.out_channels != c2.in_channels:
        return None
    x = x.contiguous()
    B, H, W, C = x.shape
    C1, C2 = c1.out_channels, c2.out_channels
    k1 = (C1 + 3) // 4 * 4
    ws = []
    for conv, cin in ((c1, C), (c2, C1)):
        w, kp = conv.weight, (cin + 3) // 4 * 4
        ent = _W9P.get(id(w))
        if ent is None or ent[0]() is not w or ent[1] != w._version:
            key = id(w)
            w9 = F.pad(w.detach().permute(2, 3, 0, 1).reshape(9 * conv.out_channels, cin), (0, kp - cin)).contiguous()
            ent = (weakref.ref(w, lambda _r, k=key: _W9P.pop(k, None)), w._version, w9)
            _W9P[key] = ent
        ws.append((ent[2], None) if torch.backends.cudnn.allow_tf32 else _split_weight(ent[2]))
    L_ = _lib.lib()
    h = torch.empty((B, H, W, k1), dtype=torch.float32, device=x.device)
    (hi, lo), (hi2, lo2) = ws
    _lib.check(L_.sigma_conv3x3_pitched_tf32(ptr(x), C, ptr(hi), C, ptr(lo), ptr(c1.bias), 1, ptr(h), k1, B, H, W, C, C1, stream()),
               "sigma_conv3x3_pitched_tf32")
    y = torch.empty((B, H, W, C2), dtype=torch.float32, device=x.device)
    _lib.check(L_.sigma_conv3x3_pitched_tf32(ptr(h), k1, ptr(hi2), k1, ptr(lo2), ptr(c2.bias), 0, ptr(y), C2, B, H, W, C1, C2, stream()),
               "sigma_conv3x3_pitched_tf32")
    return y


def dwconv3x3_silu(x, x_row_stride, x_batch_stride, conv, out, out_batch_stride, batch, H, W, D):
    """x and out both fp32, both bf16 (sigma_dwconv3x3_silu_fwd_bf16) or both fp16 (sigma_dwconv3x3_silu_fwd_fp16)."""
    fn = _entry("sigma_dwconv3x3_silu_fwd", x.dtype)
    _lib.check(getattr(_lib.lib(), fn)(ptr(x), x_row_stride, x_batch_stride, ptr(conv.weight), ptr(conv.bias),
                                       ptr(out), out_batch_stride, batch, H, W, D, stream()), fn)
    return out


def ss2d_scan(kind, xc, xdbl, dtw, dtb, A, Ds, batch, H, W, D, N, R, Cp):
    L_ = _lib.lib()
    ndir = {_lib.DIRS_CROSS4: 4, _lib.DIRS_SEQ2: 2, _lib.DIRS_CROSS: 1}[kind]
    Lseq = 2 * H * W if kind == _lib.DIRS_SEQ2 else H * W
    y = torch.empty((ndir, batch, Lseq, D), dtype=xc.dtype, device=xc.device)      # bf16 / fp16 xc -> bf16 / fp16 y
    wsb = L_.sigma_ss2d_scan_workspace_bytes(kind, batch, H, W, D, N)
    ws = torch.empty(wsb, dtype=torch.uint8, device=xc.device)
    if xc.dtype in (torch.bfloat16, torch.float16):
        fn = _entry("sigma_ss2d_scan_fwd", xc.dtype)
        rc = getattr(L_, fn)(kind, ptr(xc), ptr(xdbl), ptr(dtw), ptr(dtb), ptr(A), ptr(Ds), ptr(y), batch, H, W, D, N, R, Cp,
                             ptr(ws), wsb, stream())
        _lib.check(rc, fn)
        return y
    if _FORCE_SPLIT:
        rc = L_.sigma_ss2d_scan_fwd_split(kind, ptr(xc), ptr(xdbl), ptr(dtw), ptr(dtb), ptr(A), ptr(Ds), ptr(y), batch, H, W, D, N,
                                          R, Cp, ptr(ws), wsb, _FORCE_SPLIT, stream())
    else:
        rc = L_.sigma_ss2d_scan_fwd(kind, ptr(xc), ptr(xdbl), ptr(dtw), ptr(dtb), ptr(A), ptr(Ds), ptr(y), batch, H, W, D, N, R, Cp,
                                    ptr(ws), wsb, stream())
    _lib.check(rc, "sigma_ss2d_scan_fwd")
    return y


def ss2d_scan_save(kind, xc, xdbl, dtw, dtb, A, Ds, batch, H, W, D, N, R, Cp):
    """Training forward: ss2d_scan that also returns delta' (K, batch, Lseq, D) and the block-start states `hs` for
    sigma_ss2d_scan_bwd_saved (no state sweep in the backward).  A bf16 (fp16) xc runs the bf16 (fp16) training mode: y and delta'
    are bf16 (fp16) too, and delta' is the rounded value the recurrence itself used (sigma_ss2d_scan_fwd_save_bf16 / _fp16)."""
    L_ = _lib.lib()
    ndir = {_lib.DIRS_CROSS4: 4, _lib.DIRS_SEQ2: 2, _lib.DIRS_CROSS: 1}[kind]
    Lseq = 2 * H * W if kind == _lib.DIRS_SEQ2 else H * W
    y = torch.empty((ndir, batch, Lseq, D), dtype=xc.dtype, device=xc.device)
    delta = torch.empty_like(y)
    hs = torch.empty(L_.sigma_ss2d_scan_hs_bytes(kind, batch, H, W, D, N) // 4, dtype=torch.float32, device=xc.device)
    wsb = L_.sigma_ss2d_scan_workspace_bytes(kind, batch, H, W, D, N)
    ws = torch.empty(wsb, dtype=torch.uint8, device=xc.device)
    fn = _entry("sigma_ss2d_scan_fwd_save", xc.dtype)
    rc = getattr(L_, fn)(kind, ptr(xc), ptr(xdbl), ptr(dtw), ptr(dtb), ptr(A), ptr(Ds), ptr(y), ptr(delta), ptr(hs), batch, H, W, D,
                         N, R, Cp, ptr(ws), wsb, int(_FORCE_SPLIT or 0), stream())
    _lib.check(rc, fn)
    return y, delta, hs


def merge_norm_gate(y, K, k_stride, in_batch_stride, ln, z, z_row_stride, gate, out, out_batch_stride, out_row_stride,
                    rows, rows_per_batch, D, y_offset=0, out_offset=0):
    """y, z and out all fp32, all bf16 (sigma_merge_norm_gate_fwd_bf16) or all fp16 (sigma_merge_norm_gate_fwd_fp16); offsets
    and strides count elements.  out = E4M3Rows
    (y, z bf16): sigma_merge_norm_gate_fwd_fp8, whose row r's scale lands at out.s[out_offset / out_row_stride + r]."""
    yp = ctypes.c_void_p(y.data_ptr() + y.element_size() * y_offset)
    if isinstance(out, E4M3Rows):
        qp = ctypes.c_void_p(out.q.data_ptr() + out_offset)
        sp = ctypes.c_void_p(out.s.data_ptr() + 4 * (out_offset // out_row_stride))
        rc = _lib.lib().sigma_merge_norm_gate_fwd_fp8(yp, K, k_stride, in_batch_stride, ptr(ln.weight), ptr(ln.bias), z, z_row_stride,
                                                      ptr(gate), qp, sp, out_batch_stride, out_row_stride, rows, rows_per_batch, D,
                                                      float(ln.eps), stream())
        _lib.check(rc, "sigma_merge_norm_gate_fwd_fp8")
        return out
    fn = _entry("sigma_merge_norm_gate_fwd", y.dtype)
    op = ctypes.c_void_p(out.data_ptr() + out.element_size() * out_offset)
    rc = getattr(_lib.lib(), fn)(yp, K, k_stride, in_batch_stride, ptr(ln.weight), ptr(ln.bias), z, z_row_stride,
                                 ptr(gate), op, out_batch_stride, out_row_stride, rows, rows_per_batch, D, float(ln.eps), stream())
    _lib.check(rc, fn)
    return out


# ---------------------------------------------------------------- per-module packed parameters
def _pack_xproj(w, N, R, Cp):
    """x_proj rows [dt (R) | B (N) | C (N)] (vmamba.py:198) -> kernel row order [B | C | dt | 0-pad]."""
    pad = w.new_zeros((Cp - 2 * N - R, w.shape[1]))
    return torch.cat([w[R:R + N], w[R + N:R + 2 * N], w[:R], pad], dim=0)


def _cache(m, key, versions, build):
    c = m.__dict__.setdefault("_sigma_cache", {})
    ent = c.get(key)
    if ent is None or ent[0] != versions:
        ent = (versions, build())
        c[key] = ent
    return ent[1]


def _ssm_params(m):
    """Packed, contiguous fp32 SSM parameters of SS2D / ConMB_SS2D (K directions)."""
    ps = (m.x_proj_weight, m.dt_projs_weight, m.dt_projs_bias, m.A_logs, m.Ds)
    ver = tuple((p._version, p.data_ptr()) for p in ps)

    def build():
        N, R = m.d_state, m.dt_rank
        Cp = _lib.lib().sigma_ss2d_padded_cp(N, R)
        if Cp < 0:
            raise RuntimeError(f"dt_rank={R} > 64 is not supported by the fused scan")
        xw = torch.cat([_pack_xproj(m.x_proj_weight[k].float(), N, R, Cp) for k in range(m.K)], dim=0).contiguous()
        return dict(Cp=Cp, xproj=xw, dtw=m.dt_projs_weight.float().contiguous(), dtb=m.dt_projs_bias.float().contiguous(),
                    A=(-torch.exp(m.A_logs.float())).contiguous(), Ds=m.Ds.float().contiguous())
    return _cache(m, "ssm", ver, build)


def _cma_params(cm):
    """Cross_Mamba_Attention_SSM: modality 0 = rgb (x_proj_1, ...), modality 1 = x."""
    ps = (cm.x_proj_1.weight, cm.x_proj_2.weight, cm.dt_proj_1.weight, cm.dt_proj_2.weight, cm.dt_proj_1.bias,
          cm.dt_proj_2.bias, cm.A_log_1, cm.A_log_2, cm.D_1, cm.D_2)
    ver = tuple((p._version, p.data_ptr()) for p in ps)

    def build():
        N, R = cm.d_state, cm.dt_rank
        Cp = _lib.lib().sigma_ss2d_padded_cp(N, R)
        return dict(Cp=Cp, xproj1=_pack_xproj(cm.x_proj_1.weight.float(), N, R, Cp).contiguous(),
                    xproj2=_pack_xproj(cm.x_proj_2.weight.float(), N, R, Cp).contiguous(),
                    dtw=torch.stack([cm.dt_proj_1.weight, cm.dt_proj_2.weight]).float().contiguous(),
                    dtb=torch.stack([cm.dt_proj_1.bias, cm.dt_proj_2.bias]).float().contiguous(),
                    A=(-torch.exp(torch.cat([cm.A_log_1, cm.A_log_2]).float())).contiguous(),
                    Ds=torch.cat([cm.D_1, cm.D_2]).float().contiguous())
    return _cache(cm, "cma", ver, build)


# ---------------------------------------------------------------- blocks
def ss2d(m, x, residual=None, rscale=None):
    """SS2D.forward (vmamba.py:1067-1089); x (B,H,W,C) contiguous.  Returns (B,H,W,C) [+ residual (· rscale)], the
    residual being added in the out_proj GEMM epilogue."""
    dt = _interior_dtype()                                      # storage of the block's interior (module docstring)
    fp8 = _fp8_mode()
    if isinstance(x, E4M3Rows):                                 # the FP8 mode's LayerNorm output (vss_block, cvss_decoder_block)
        B, H, W, C = x.q.shape
        xa = x.view(B * H * W, C)
    else:
        x = x.contiguous() if fp8 else x.to(dt).contiguous()
        B, H, W, C = x.shape
        xa = quantize_rows(x.view(B * H * W, C)) if fp8 else x.view(B * H * W, C)
    D, N, R, L = m.d_inner, m.d_state, m.dt_rank, H * W
    c = _ssm_params(m)
    dev = xa.q.device if fp8 else xa.device
    xz = linear(xa, m.in_proj.weight, m.in_proj.bias, kind="in_proj", out_dtype=dt)                   # (BL, 2D): [x | z]
    xc = torch.empty((B, L, D), dtype=dt, device=dev)
    dwconv3x3_silu(xz, 2 * D, L * 2 * D, m.conv2d, xc, L * D, B, H, W, D)
    xdbl = linear(xc.view(B * L, D), c["xproj"], kind="x_proj")                                        # (BL, 4·Cp) fp32
    y = ss2d_scan(_lib.DIRS_CROSS4, xc, xdbl, c["dtw"], c["dtb"], c["A"], c["Ds"], B, H, W, D, N, R, c["Cp"])
    yg = _e4m3_empty(B * L, D, dev) if fp8 else torch.empty((B * L, D), dtype=dt, device=dev)
    z = ctypes.c_void_p(xz.data_ptr() + xz.element_size() * D)
    merge_norm_gate(y, 4, B * L * D, 0, m.out_norm, z, 2 * D, None, yg, 0, D, B * L, B * L, D)
    res2d = residual.reshape(B * L, C) if residual is not None else None
    return linear(yg, m.out_proj.weight, m.out_proj.bias, residual=res2d, rscale=rscale, kind="out_proj").view(B, H, W, C)


def _interior_dtype():
    mode = precision()
    return torch.bfloat16 if mode in ("bf16", "fp8") else torch.float16 if mode == "fp16" else torch.float32


def _ln_out_dtype():
    """the dtype of a LayerNorm output that feeds in_proj: E4M3Rows in the FP8 mode, else the interior storage"""
    return torch.float8_e4m3fn if _fp8_mode() else _interior_dtype()


def vss_block(blk, x):
    """VSSBlock._forward (vmamba.py:1712-1716), mlp_ratio = 0."""
    x = x.contiguous()
    B, H, W, C = x.shape
    xn = layernorm(x.view(-1, C), blk.norm, _ln_out_dtype()).view(B, H, W, C)
    return ss2d(blk.op, xn, residual=x)


def patch_merging(m, x):
    """PatchMerging2D (vmamba.py:619-636)."""
    x = x.contiguous()
    B, H, W, C = x.shape
    H2, W2 = (H + 1) // 2, (W + 1) // 2
    if _fp8_mode():                                                  # the same kernel, quantizing its rows
        xq = _e4m3_empty(B * H2 * W2, 4 * C, x.device)
        _lib.check(_lib.lib().sigma_patch_merge_norm_fwd_fp8(ptr(x), ptr(m.norm.weight), ptr(m.norm.bias), ptr(xq.q), ptr(xq.s), B, H, W, C,
                                                             float(m.norm.eps), stream()), "sigma_patch_merge_norm_fwd_fp8")
        return linear(xq, m.reduction.weight).view(B, H2, W2, -1)
    dt = _interior_dtype()
    xn = torch.empty((B * H2 * W2, 4 * C), dtype=dt, device=x.device)
    # 2x2 gather (+ zero padding of odd sizes) + LayerNorm(4C) in one kernel: no concatenated tensor
    fn = _entry("sigma_patch_merge_norm_fwd", dt)
    _lib.check(getattr(_lib.lib(), fn)(ptr(x), ptr(m.norm.weight), ptr(m.norm.bias), ptr(xn), B, H, W, C, float(m.norm.eps), stream()), fn)
    return linear(xn, m.reduction.weight).view(B, H2, W2, -1)


def cromb_ss2d(m, x_rgb, x_e, residual=False):
    """CrossMambaFusion_SS2D_SSM.forward (vmamba.py:1622-1640) + Cross_Mamba_Attention_SSM.forward (:1508-1545)."""
    x_rgb, x_e = x_rgb.contiguous(), x_e.contiguous()
    B, H, W, C = x_rgb.shape
    D, L = m.d_inner, H * W
    cm = m.CMA_ssm
    N, R = cm.d_state, cm.dt_rank
    c = _cma_params(cm)
    dev = x_rgb.device
    dt = _interior_dtype()
    fp8 = _fp8_mode()
    if fp8:                                                                    # GEMM operands (the residuals below stay fp32)
        a_r, a_e = quantize_rows(x_rgb.view(B * L, C)), quantize_rows(x_e.view(B * L, C))
    else:
        a_r, a_e = x_rgb.to(dt).view(B * L, C), x_e.to(dt).view(B * L, C)
    xp = torch.empty((2, B * L, D), dtype=dt, device=dev)                     # modality-major
    linear(a_r, m.in_proj.weight, m.in_proj.bias, out=xp[0])
    linear(a_e, m.in_proj_modalx.weight, m.in_proj_modalx.bias, out=xp[1])
    xc = torch.empty((2 * B, L, D), dtype=dt, device=dev)
    dwconv3x3_silu(xp, D, L * D, m.conv2d, xc, L * D, 2 * B, H, W, D)         # ONE conv for both modalities (:1629-1630)
    xdbl = torch.empty((2, B * L, c["Cp"]), dtype=torch.float32, device=dev)
    linear(xc[:B].view(B * L, D), c["xproj1"], out=xdbl[0], kind="x_proj")
    linear(xc[B:].view(B * L, D), c["xproj2"], out=xdbl[1], kind="x_proj")
    y = ss2d_scan(_lib.DIRS_CROSS, xc, xdbl, c["dtw"], c["dtb"], c["A"], c["Ds"], 2 * B, H, W, D, N, R, c["Cp"])  # (1,2B,L,D)
    yn = _e4m3_empty(2 * B * L, D, dev) if fp8 else torch.empty((2 * B * L, D), dtype=dt, device=dev)
    merge_norm_gate(y, 1, 0, 0, cm.out_norm_1, None, 0, None, yn, 0, D, B * L, B * L, D)
    merge_norm_gate(y, 1, 0, 0, cm.out_norm_2, None, 0, None, yn, 0, D, B * L, B * L, D, y_offset=B * L * D, out_offset=B * L * D)
    if fp8:
        yn_r, yn_e = E4M3Rows(yn.q[:B * L], yn.s[:B * L]), E4M3Rows(yn.q[B * L:], yn.s[B * L:])
    else:
        yn_r, yn_e = yn[:B * L], yn[B * L:]
    r_r = x_rgb.view(B * L, C) if residual else None
    r_e = x_e.view(B * L, C) if residual else None
    o_r = linear(yn_r, m.out_proj_rgb.weight, m.out_proj_rgb.bias, residual=r_r).view(B, H, W, C)
    o_e = linear(yn_e, m.out_proj_e.weight, m.out_proj_e.bias, residual=r_e).view(B, H, W, C)
    return o_r, o_e


def conmb_ss2d(m, x_rgb, x_e, residual=None):
    """ConMB_SS2D.forward (vmamba.py:1265-1284) + cross_selective_scan_multimodal_k2 (:369-430)."""
    x_rgb, x_e = x_rgb.contiguous(), x_e.contiguous()
    B, H, W, C = x_rgb.shape
    D, N, R, L = m.d_inner, m.d_state, m.dt_rank, H * W
    c = _ssm_params(m)
    dev = x_rgb.device
    dt = _interior_dtype()
    fp8 = _fp8_mode()
    if fp8:
        a_r, a_e = quantize_rows(x_rgb.view(B * L, C)), quantize_rows(x_e.view(B * L, C))
    else:
        a_r, a_e = x_rgb.to(dt).view(B * L, C), x_e.to(dt).view(B * L, C)
    tr = linear(a_r, m.in_proj.weight, m.in_proj.bias, out_dtype=dt)
    te = linear(a_e, m.in_proj_modalx.weight, m.in_proj_modalx.bias, out_dtype=dt)
    seq = torch.empty((B, 2 * L, D), dtype=dt, device=dev)                    # [rgb ‖ x] along L (vmamba.py:130)
    dwconv3x3_silu(tr, D, L * D, m.conv2d, seq, 2 * L * D, B, H, W, D)
    dwconv3x3_silu(te, D, L * D, m.conv2d_modalx, seq[:, L:], 2 * L * D, B, H, W, D)
    xdbl = linear(seq.view(B * 2 * L, D), c["xproj"], kind="x_proj")          # (B·2L, 2·Cp)
    y = ss2d_scan(_lib.DIRS_SEQ2, seq, xdbl, c["dtw"], c["dtb"], c["A"], c["Ds"], B, H, W, D, N, R, c["Cp"])  # (2,B,2L,D)
    # SE gates from the PRE-conv projections, applied crosswise (vmamba.py:1276-1281)
    with _no_autocast():                                                      # the gates average and run in fp32
        g_r = m.fc1(tr.view(B, L, D).mean(dim=1, dtype=torch.float32))
        g_e = m.fc2(te.view(B, L, D).mean(dim=1, dtype=torch.float32))
    ycat = torch.empty((B * L, 2 * D), dtype=dt, device=dev)
    ks = B * 2 * L * D
    merge_norm_gate(y, 2, ks, 2 * L * D, m.out_norm1, None, 0, g_e, ycat, L * 2 * D, 2 * D, B * L, L, D)
    merge_norm_gate(y, 2, ks, 2 * L * D, m.out_norm2, None, 0, g_r, ycat, L * 2 * D, 2 * D, B * L, L, D,
                    y_offset=L * D, out_offset=D)
    res2d = residual.reshape(B * L, C) if residual is not None else None
    if fp8:                                                                   # the two halves come from two calls: quantize the row here
        ycat = quantize_rows(ycat)
    return linear(ycat, m.out_proj.weight, m.out_proj.bias, residual=res2d).view(B, H, W, C)


# ---------------------------------------------------------------- decoder pieces
def ln_nhwc(ln, x):
    """nn.LayerNorm over the last dim of a channels-last tensor of any rank."""
    x = x.contiguous()
    return layernorm(x.view(-1, x.shape[-1]), ln).view(x.shape)


def upsample2x_norm(x, ln):
    """LayerNorm(bilinear x2 (x)) in one pass (UpsampleExpand tail, MambaDecoder.py:47-49); ln=None: plain bilinear x2."""
    x = x.contiguous()
    B, H, W, C = x.shape
    y = torch.empty((B, 2 * H, 2 * W, C), dtype=torch.float32, device=x.device)
    wp, bp, eps = (ptr(ln.weight), ptr(ln.bias), float(ln.eps)) if ln is not None else (None, None, 0.0)
    _lib.check(_lib.lib().sigma_upsample2x_norm_fwd(ptr(x), wp, bp, ptr(y), B, H, W, C, eps, stream()),
               "sigma_upsample2x_norm_fwd")
    return y


def upsample2x_norm_head(x, ln, conv1x1):
    """Conv1x1(LayerNorm(bilinear x2 (x))) -> NCHW logits (MambaDecoder.py:95-96,276-279)."""
    x = x.contiguous()
    B, H, W, C = x.shape
    ncls = conv1x1.weight.shape[0]
    w = conv1x1.weight.view(ncls, C)
    out = torch.empty((B, ncls, 2 * H, 2 * W), dtype=torch.float32, device=x.device)
    _lib.check(_lib.lib().sigma_upsample2x_norm_head_fwd(ptr(x), ptr(ln.weight), ptr(ln.bias), ptr(w), ncls, ptr(out), B, H, W, C,
                                                          float(ln.eps), stream()), "sigma_upsample2x_norm_head_fwd")
    return out


def pool_avgmax(t):
    """(B, H, W, C) channels-last -> mean and max over H·W, each (B, C)."""
    B, H, W, C = t.shape
    L = H * W
    # slices of positions per image: enough CTAs (B·nslice >= 2 per SM) that a single image does not walk its map with a handful
    # of them (B = 1, 30x40 map: 4 CTAs took 74 us), at least 32 positions per slice
    nslice = max(1, min(64, L // 32, max(L // 256, -(-296 // B))))
    part = torch.empty((B, nslice, 2, C), dtype=torch.float32, device=t.device)
    _lib.check(_lib.lib().sigma_pool_avgmax_partial_fwd(ptr(t), ptr(part), B, L, C, nslice, stream()), "sigma_pool_avgmax_partial_fwd")
    return part[:, :, 0].sum(1) / L, part[:, :, 1].amax(1)


def scale_add(a, sa, b, sb, rows_per_batch):
    """a·sa[batch] + b·sb, all channels-last with C = last dim."""
    out = torch.empty_like(b)
    C = b.shape[-1]
    rows = b.numel() // C
    _lib.check(_lib.lib().sigma_scale_add_fwd(ptr(a), ptr(sa), ptr(b), ptr(sb), ptr(out), rows, rows_per_batch, C, stream()),
               "sigma_scale_add_fwd")
    return out


def cvss_decoder_block(blk, x):
    """CVSSDecoderBlock._forward (vmamba.py:1800-1805) with ChannelAttentionBlock (vmamba.py:1725-1757)."""
    x = x.contiguous()
    B, H, W, C = x.shape
    xn = layernorm(x.view(-1, C), blk.norm1, _ln_out_dtype()).view(B, H, W, C)
    x1 = ss2d(blk.op, xn, residual=x, rscale=blk.scale1)            # x·scale1 + SS2D(LN(x)) in the GEMM epilogue
    xn2 = layernorm(x1.view(-1, C), blk.norm2).view(B, H, W, C)
    cab = blk.conv_blk.cab
    t = None
    if isinstance(cab[1], torch.nn.GELU) and getattr(cab[1], "approximate", "none") == "none":
        h1 = conv3x3(xn2, cab[0], gelu=True)                         # conv3x3 + bias + GELU: implicit GEMM on the wgmma kernel
        t = conv3x3(h1, cab[2]) if h1 is not None else None
        if h1 is None:                                               # C/3 not a multiple of 4 (Sigma-base): pitched rows
            t = cab_convs_pitched(xn2, cab)
    with _no_autocast():                                             # CAB stays in the dense mode under autocast
        if t is None:                                                # other conv forms: cuDNN on a channels_last view
            t = cab[2](cab[1](cab[0](xn2.permute(0, 3, 1, 2)))).permute(0, 2, 3, 1).contiguous()
        avg, mx = pool_avgmax(t)
        fc = cab[3].fc
        attn = torch.sigmoid(fc(avg.view(B, C, 1, 1)) + fc(mx.view(B, C, 1, 1))).view(B, C).contiguous()
    return scale_add(t, attn, x1, blk.scale2, H * W)               # CAB(x)·attn + x·scale2


def patch_expand(m, x):
    """PatchExpand (MambaDecoder.py:12-30)."""
    B, H, W, C = x.shape
    y = linear(x.reshape(B * H * W, C), m.expand.weight)             # (B·H·W, 2C) = "b h w (p1 p2 c)"
    out = torch.empty((B, 2 * H, 2 * W, C // 2), dtype=torch.float32, device=x.device)
    _lib.check(_lib.lib().sigma_pixel_shuffle_norm_fwd(ptr(y), ptr(m.norm.weight), ptr(m.norm.bias), ptr(out), B, H, W, C // 2,
                                                        float(m.norm.eps), stream()), "sigma_pixel_shuffle_norm_fwd")
    return out


def upsample_expand(m, x):
    """UpsampleExpand (MambaDecoder.py:33-51)."""
    B, H, W, C = x.shape
    y = linear(x.reshape(B * H * W, C), m.linear.weight).view(B, H, W, C // 2)
    return upsample2x_norm(y, m.norm)


def final_head(dec, x):
    """MambaDecoder.up_x4 (MambaDecoder.py:272-280) = FinalUpsample_X4 (:87-97) + 1x1 conv.  linear2 is applied before
    the first bilinear x2 instead of after it: both are linear maps over different axes (channels vs space), so
    they commute exactly in real arithmetic and the 240x320 GEMM shrinks 4x."""
    B, H, W, C = x.shape
    t = linear(x.reshape(B * H * W, C), dec.up.linear1.weight)
    t = linear(t, dec.up.linear2.weight).view(B, H, W, C)
    t = upsample2x_norm(t, None)   # plain bilinear x2
    return upsample2x_norm_head(t, dec.up.norm, dec.output)
