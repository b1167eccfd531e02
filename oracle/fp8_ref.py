"""Host emulation of the FP8 inference mode's quantization (include/sigma_b200.h, "FP8 inference mode"), bit for bit.

e4m3 (torch.float8_e4m3fn): 1 sign, 4 exponent (bias 7), 3 mantissa bits; normals from 2^-6, subnormals in steps of 2^-9, largest
finite 448, no infinities.  `e4m3` rounds fp32 to nearest even with saturation to ±448 (cvt.rn.satfinite.e4m3x2.f32); float64
arithmetic on the step makes every rounding exact.  `quantize_rows` applies the per-row formula with numpy float32 operations,
which round like the kernels' IEEE fp32 division and multiplication.
"""
import numpy as np

E4M3_MAX = 448.0
FLT_MAX = np.float32(3.4028234663852886e38)


def e4m3(x):
    """fp32 array -> the e4m3 values it rounds to (float32; NaN stays NaN), round to nearest even, saturating to ±448."""
    x = np.asarray(x, dtype=np.float32).astype(np.float64)
    a = np.abs(x)
    e = np.frexp(np.where(a > 0, a, 1.0))[1] - 1.0         # floor(log2 a), exactly
    step = np.exp2(np.maximum(e, -6.0) - 3.0)              # 3 mantissa bits; below 2^-6 the subnormal step 2^-9
    q = np.rint(a / step) * step                           # a / step is exact (power-of-two step); rint = half to even
    q = np.minimum(q, E4M3_MAX)
    return (np.sign(x) * q).astype(np.float32)


def quantize_rows(x):
    """(rows, C) fp32 -> (q (rows, C) float32 holding e4m3 values, s (rows,) float32): the formula of sigma_b200.h."""
    x = np.asarray(x, dtype=np.float32)
    amax = np.abs(x).max(axis=1).astype(np.float32)
    zero = amax == 0
    safe = np.where(zero, np.float32(1), amax).astype(np.float32)
    with np.errstate(over="ignore"):                       # a subnormal amax: 448 / amax overflows, then clamps to FLT_MAX
        inv = np.minimum(np.float32(E4M3_MAX) / safe, FLT_MAX).astype(np.float32)
    inv = np.where(zero, np.float32(1), inv).astype(np.float32)
    s = np.where(zero, np.float32(1), safe / np.float32(E4M3_MAX)).astype(np.float32)
    q = e4m3((x * inv[:, None]).astype(np.float32))
    return q, s


def fake_quant_rows(x):
    """quantize-dequantize per row in fp32 (q·s): what the FP8 mode's GEMMs see of an operand"""
    q, s = quantize_rows(x)
    return (q * s[:, None]).astype(np.float32)
