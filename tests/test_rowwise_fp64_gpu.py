"""GPU: the row-wise and decoder-tail kernels of rowwise.cu (every LayerNorm of the model, the SS2D / CroMB / ConMB direction merge
+ out_norm + gate, patch merging, patch expanding, the decoder's upsampling, the logits head, channel-attention pooling, the decoder
block's tail and the LayerNorm backward) against the fp64 references of oracle/rowwise_ref64.py, element by element inside their
per-element error bounds, at every instantiation and at Sigma's shapes.
* LayerNorm at every fast width and every generic MAXV, 1 row, a row count ragged against the rows of a warp and a CTA, and >= 3
  waves of CTAs; every row family of rowwise_ref64.hard_rows (large means, variance ~ eps, constant rows that must give beta
  exactly, outliers) and a LayerNorm weight of mixed sign;
* merge + norm + gate at K = 1..8 (K = 3, 5..8 run the generic kernel), z and gate on and off, with padded output rows, and the
  three production calls with the strides and offsets of fused.ss2d, fused.cromb_ss2d and fused.conmb_ss2d;
* the patch-merge gather (odd sizes, Sigma-base's 45 x 60 map) and the pixel shuffle, called directly;
* bilinear x2 with and without LayerNorm (1-pixel maps too), the head's fast kernel at several 8 x 32 tiles per direction with a
  ragged last tile and at Sigma's 240 x 320 -> 480 x 640, its generic kernel, the whole logit tensor compared;
* pool_avgmax (forced slice counts with empty trailing slices, idle threads), scale_add past 3 grid-stride passes, layernorm_bwd
  past its grid cap (the deterministic build bitwise repeatable);
* the benchmark's batch of 74: every image of the LayerNorm and of the head bit-identical to a batch-1 run of it.
* The bf16 instances (rowwise_ref64's docstring: inputs rounded to bf16 first, the fp32 bound plus one bf16 store) on the same
  cases through an io axis: io 1 (fp32 in, bf16 out: sigma_layernorm_fwd_bf16 at every width and the benchmark's batch, the
  patch-merge gather at every width it takes, and fused.layernorm's routing to both), io 2 (bf16 in and out:
  sigma_layernorm_fwd_bf16io at every width, merge + norm + gate at K = 1..8 and the three production calls); hard rows in their
  bf16 form; constant rows give bf16(beta) exactly.  sigma_layernorm_bwd_bf16 at every instantiation past its grid cap.
Outputs sit in NaN-filled buffers (helpers.guarded): every interior element must be written, every guard stay untouched.  Inputs
are generated on the GPU from fixed seeds; the references run there in torch float64.  Worst bound fractions go to
helpers.record."""
import ctypes
import types

import pytest
import torch

from helpers import guard_ok, guarded, ptr, record, stream
from oracle import rowwise_ref64 as R

pytestmark = pytest.mark.gpu
S = 97
EPS = 1e-5
SIGMA_EUNSUPPORTED = -4

LN_FAST_D = [64, 96, 128, 192, 256, 384, 512, 768, 1024, 1536, 2048]
LN_GENERIC_D = [32, 200, 400, 1000, 2000, 4000, 4096]
MERGE_K = [1, 2, 3, 4, 5, 6, 7, 8]
MERGE_D = [96, 192, 384, 768, 1536, 256, 512, 1024, 2048, 64, 128]
PATCH_MERGE_C = [96, 192, 384, 128, 256, 512, 16, 24, 32, 48, 64]
# element pairs each test runs (oracle/rowwise_ref64.IO_PAIRS): 0 fp32, 1 fp32 in / bf16 out, 2 bf16 in and out
LN_IO = [0, 1, 2]
MERGE_IO = [0, 2]
PATCH_MERGE_IO = [0, 1]
BWD_BF16_D = [32, 64, 96, 128, 192, 256, 384, 512, 768, 1024, 1536]
BF = torch.bfloat16
PATCH_MERGE_UNSUPPORTED_C = 40
SHUFFLE_D = [384, 512] + [d for d in LN_FAST_D if d not in (384, 512)]
UPSAMPLE_C = [48, 192, 384, 1024]
HEAD_FAST_C = [64, 96, 128, 192, 256]
HEAD_FAST_NCLS = [2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 16, 19, 20, 21]
HEAD_GENERIC_NCLS = [37, 40, 41]
HEAD_GENERIC_C = [32, 48, 320]
WAVE_WARPS = 3 * 132 * 64          # three waves of fully occupied SMs, one row per warp


def _lib():
    from sigma_b200 import _lib
    return _lib


def _call(fn, *args):
    L = _lib()
    rc = getattr(L.lib(), fn)(*args)
    L.check(rc, fn)
    torch.cuda.synchronize()


def _off(t, elems):
    return ctypes.c_void_p(t.data_ptr() + t.element_size() * elems)


def _randn(seed, shape, scale=1.0, shift=0.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(shape, generator=g, device="cuda") * scale + shift


def _affine(seed, D):
    return [t.cuda() for t in R.affine(seed, D)]


def _check(tag, got, ref, bnd, worst, key):
    """written everywhere and inside the bound; the worst fraction kept under `key`"""
    assert not bool(got.isnan().any()), f"{tag}: output not written everywhere"
    frac = R.bound_fraction(got, ref, bnd)
    worst[key] = max(worst.get(key, 0.0), frac)
    assert frac <= 1.0, f"{tag}: {frac:.3f} of the per-element bound"


def _with_io(cases, ios):
    """pytest parameters (*case, io): io 0 keeps the fp32 test's ids, a bf16 io is appended to them as -io1 / -io2"""
    out = []
    for io in ios:
        for c in cases:
            c = c if isinstance(c, tuple) else (c,)
            ident = "-".join(str(v) for v in c)
            out.append(pytest.param(*c, io, id=ident if io == 0 else f"{ident}-io{io}"))
    return out


def _rows(seed, rows, D, io, **kw):
    """hard_rows as the instance reads them: bf16 (their bf16 form) when y is bf16 (io 2)"""
    return R.hard_rows(seed, rows, D, device="cuda", bf16=io == 2, **kw)


def _bound(io, ref, e):
    """the fp32 bound e, plus the bf16 store of a bf16 output"""
    return R.bf16_store_bound(ref, e) if io else e


def _out_dtype(io):
    return BF if io else torch.float32


_LN_FN = {0: "sigma_layernorm_fwd", 1: "sigma_layernorm_fwd_bf16", 2: "sigma_layernorm_fwd_bf16io"}


def _layernorm(x, g, b, io=0):
    rows, D = x.shape
    buf, y = guarded((rows, D), _out_dtype(io))
    _call(_LN_FN[io], ptr(x), ptr(g), ptr(b), ptr(y), rows, D, EPS, stream())
    guard_ok(buf, f"layernorm io={io} {rows}x{D}")
    return y


# ---------------------------------------------------------------- LayerNorm
def _ln_counts(D):
    lpr, _, fast = R.row_plan(D)
    rpw = 32 // lpr if fast else 1
    return [1, 8 * rpw * 5 + rpw - 1 if rpw > 1 else 8 * 5 + 3, WAVE_WARPS * rpw + 5]


@pytest.mark.parametrize("D,io", _with_io(LN_FAST_D + LN_GENERIC_D, LN_IO))
def test_layernorm(D, io):
    from sigma_b200 import fused
    plan = R.row_plan(D, io=io)
    g, b = _affine(S + D, D)
    worst = {}
    for rows in _ln_counts(D):
        x = _rows(S * D + rows, rows, D, io)
        y = _layernorm(x, g, b, io)
        ref = R.layer_norm_ref64(x, g, b, EPS)
        _check(f"D={D} io={io} rows={rows}", y, ref, _bound(io, ref, R.layer_norm_bound(x, g, b, EPS, plan)), worst, "y")
        const = R.constant_rows(rows, device="cuda")
        assert torch.equal(y[const], b.to(y.dtype).expand(int(const.sum()), D)), f"D={D} io={io}: constant rows must give beta exactly"
        if io < 2:      # fused.layernorm routes an fp32 row block to the instance of the output dtype: the same bits
            assert torch.equal(fused.layernorm(x, types.SimpleNamespace(weight=g, bias=b, eps=EPS), y.dtype), y), f"D={D} io={io}"
    record("rowwise_fp64/layernorm", D=D, io=io, plan=list(plan), rows=_ln_counts(D), bound_used=worst["y"])


# ---------------------------------------------------------------- merge + norm + gate
def _merge_inputs(seed, K, rows, D, io=0):
    y = torch.stack([_rows(seed + k, rows, D, io) for k in range(K)])
    xz = _randn(seed + 100, (rows, 2 * D), 2.0)
    return y, xz.to(BF) if io == 2 else xz


def _merge(io, *args):
    _call("sigma_merge_norm_gate_fwd_bf16" if io else "sigma_merge_norm_gate_fwd", *args)


@pytest.mark.parametrize("K,D,io", _with_io([(K, D) for K in MERGE_K for D in MERGE_D], MERGE_IO))
def test_merge_norm_gate(K, D, io):
    """y (K, B·L, D) in direction-major slabs, z the second half of [x | z] rows, out rows padded to D + 8 per row"""
    Bn, L = 3, 407
    rows, ld = Bn * L, D + 8
    y, xz = _merge_inputs(S + 10 * K + D, K, rows, D, io)
    gate = _randn(S + K + D, (Bn, D), 0.5, 1.0)
    g, b = _affine(S + 2 * D + K, D)
    plan = R.row_plan(D, K, io=io)
    worst = {}
    for with_z in (False, True):
        for with_gate in (False, True):
            tag = f"K={K} D={D} io={io} z={with_z} gate={with_gate}"
            buf, o = guarded((rows, ld), _out_dtype(io))
            z = xz[:, D:] if with_z else None
            gt = gate if with_gate else None
            _merge(io, ptr(y), K, rows * D, L * D, ptr(g), ptr(b), _off(xz, D) if with_z else None, 2 * D if with_z else 0, ptr(gt),
                   ptr(o), L * ld, ld, rows, L, D, EPS, stream())
            guard_ok(buf, tag)
            assert bool(o[:, D:].isnan().all()), f"{tag}: row padding written"
            ref = R.merge_norm_ref64(y, g, b, EPS, z, gt, L)
            _check(tag, o[:, :D], ref, _bound(io, ref, R.merge_norm_bound(y, g, b, EPS, plan, z, gt, L)), worst, "y")
    record("rowwise_fp64/merge_norm_gate", K=K, D=D, io=io, plan=list(plan), bound_used=worst["y"])


@pytest.mark.parametrize("B,H,W,D,io", _with_io([(2, 30, 40, 192), (3, 15, 20, 384), (1, 15, 20, 1536)], MERGE_IO))
def test_merge_ss2d_call(B, H, W, D, io):
    """fused.ss2d: K = 4 slabs of B·L rows, z from [x | z] rows, one dense output"""
    L = H * W
    rows = B * L
    y, xz = _merge_inputs(S + D, 4, rows, D, io)
    g, b = _affine(S + D + 1, D)
    buf, o = guarded((rows, D), _out_dtype(io))
    _merge(io, ptr(y), 4, B * L * D, 0, ptr(g), ptr(b), _off(xz, D), 2 * D, None, ptr(o), 0, D, rows, rows, D, EPS, stream())
    guard_ok(buf, "ss2d merge")
    worst = {}
    ref = R.merge_norm_ref64(y, g, b, EPS, xz[:, D:])
    _check(f"ss2d merge io={io}", o, ref, _bound(io, ref, R.merge_norm_bound(y, g, b, EPS, R.row_plan(D, 4, io=io), xz[:, D:])),
           worst, "y")
    record("rowwise_fp64/merge_ss2d", B=B, H=H, W=W, D=D, io=io, bound_used=worst["y"])


@pytest.mark.parametrize("B,H,W,D,io", _with_io([(2, 30, 40, 192), (1, 15, 20, 768)], MERGE_IO))
def test_merge_cromb_calls(B, H, W, D, io):
    """fused.cromb_ss2d: y (1, 2B, L, D) modality-major; two K = 1 launches, the second at offsets B·L·D of y and out"""
    L = H * W
    rows = B * L
    y = _rows(S + D + 2, 2 * rows, D, io)
    (g1, b1), (g2, b2) = _affine(S + 3, D), _affine(S + 4, D)
    buf, o = guarded((2, rows, D), _out_dtype(io))
    _merge(io, ptr(y), 1, 0, 0, ptr(g1), ptr(b1), None, 0, None, ptr(o), 0, D, rows, rows, D, EPS, stream())
    assert bool(o[1].isnan().all()), "cromb: the first launch wrote the second modality's half"
    _merge(io, _off(y, rows * D), 1, 0, 0, ptr(g2), ptr(b2), None, 0, None, _off(o, rows * D), 0, D, rows, rows, D, EPS, stream())
    guard_ok(buf, "cromb merge")
    plan, worst = R.row_plan(D, io=io), {}
    for m, (g, b) in enumerate(((g1, b1), (g2, b2))):
        ym = y[m * rows:(m + 1) * rows]
        ref = R.layer_norm_ref64(ym, g, b, EPS)
        _check(f"cromb io={io} modality {m}", o[m], ref, _bound(io, ref, R.layer_norm_bound(ym, g, b, EPS, plan)), worst, "y")
    record("rowwise_fp64/merge_cromb", B=B, H=H, W=W, D=D, io=io, bound_used=worst["y"])


@pytest.mark.parametrize("B,H,W,D,io", _with_io([(2, 30, 40, 192), (3, 15, 20, 384), (1, 15, 20, 768)], MERGE_IO))
def test_merge_conmb_calls(B, H, W, D, io):
    """fused.conmb_ss2d: y (2, B, 2L, D) = two directions over [rgb ‖ x]; out rows [rgb half | x half] of 2D; K = 2,
    rows_per_batch = L, in_batch_stride 2·L·D, out_row_stride 2D, the second launch at y offset L·D and out offset D, gates
    crosswise per image"""
    L = H * W
    rows = B * L
    y = torch.stack([_rows(S + D + k, B * 2 * L, D, io) for k in range(2)])                        # (2, B·2L, D)
    g_e, g_r = _randn(S + 5, (B, D), 0.5, 1.0), _randn(S + 6, (B, D), 0.5, 1.0)
    (w1, b1), (w2, b2) = _affine(S + 7, D), _affine(S + 8, D)
    ks = B * 2 * L * D
    buf, o = guarded((rows, 2 * D), _out_dtype(io))
    _merge(io, ptr(y), 2, ks, 2 * L * D, ptr(w1), ptr(b1), None, 0, ptr(g_e), ptr(o), L * 2 * D, 2 * D, rows, L, D, EPS, stream())
    assert bool(o[:, D:].isnan().all()), "conmb: the first launch wrote the second launch's half"
    _merge(io, _off(y, L * D), 2, ks, 2 * L * D, ptr(w2), ptr(b2), None, 0, ptr(g_r), _off(o, D), L * 2 * D, 2 * D, rows, L, D, EPS,
           stream())
    guard_ok(buf, "conmb merge")
    yv = y.view(2, B, 2, L, D)
    plan, worst = R.row_plan(D, 2, io=io), {}
    for half, (w, b, gate) in enumerate(((w1, b1, g_e), (w2, b2, g_r))):
        yh = yv[:, :, half].reshape(2, rows, D)
        ref = R.merge_norm_ref64(yh, w, b, EPS, None, gate, L)
        _check(f"conmb io={io} half {half}", o[:, half * D:(half + 1) * D], ref,
               _bound(io, ref, R.merge_norm_bound(yh, w, b, EPS, plan, None, gate, L)), worst, "y")
    record("rowwise_fp64/merge_conmb", B=B, H=H, W=W, D=D, io=io, bound_used=worst["y"])


# ---------------------------------------------------------------- patch merge, pixel shuffle
@pytest.mark.parametrize("C,io", _with_io(PATCH_MERGE_C, PATCH_MERGE_IO))
def test_patch_merge_norm(C, io):
    g, b = _affine(S + C, 4 * C)
    plan, worst = R.row_plan(4 * C, mode=1, io=io), {}
    fn = "sigma_patch_merge_norm_fwd_bf16" if io else "sigma_patch_merge_norm_fwd"
    for B, H, W in ((1, 45, 60), (3, 16, 22), (3, 15, 21), (1, 1, 1)):
        x = R.hard_rows(S + C + H, B * H * W, C, device="cuda").view(B, H, W, C)
        rows = B * ((H + 1) // 2) * ((W + 1) // 2)
        buf, y = guarded((rows, 4 * C), _out_dtype(io))
        _call(fn, ptr(x), ptr(g), ptr(b), ptr(y), B, H, W, C, EPS, stream())
        guard_ok(buf, f"patch merge io={io} {B}x{H}x{W}x{C}")
        cat = R.patch_merge_gather64(x)
        ref = R.layer_norm_ref64(cat, g, b, EPS)
        _check(f"patch merge io={io} {B}x{H}x{W}x{C}", y, ref, _bound(io, ref, R.layer_norm_bound(cat, g, b, EPS, plan)), worst, "y")
    record("rowwise_fp64/patch_merge", C=C, io=io, bound_used=worst["y"])


def test_patch_merge_without_instantiation_is_refused():
    C = PATCH_MERGE_UNSUPPORTED_C
    x = _randn(S, (1, 6, 6, C))
    g, b = _affine(S, 4 * C)
    buf, y = guarded((9, 4 * C))
    rc = _lib().lib().sigma_patch_merge_norm_fwd(ptr(x), ptr(g), ptr(b), ptr(y), 1, 6, 6, C, EPS, stream())
    torch.cuda.synchronize()
    assert rc == SIGMA_EUNSUPPORTED
    assert bool(buf.isnan().all()), "a refused call wrote its output"


@pytest.mark.parametrize("D", SHUFFLE_D)
def test_pixel_shuffle_norm(D):
    g, b = _affine(S + D + 9, D)
    plan, worst = R.row_plan(D, mode=2), {}
    shapes = [(2, 7, 9)] + ([(2, 15, 20)] if D in (384, 512) else [])
    for B, H, W in shapes:
        y = R.hard_rows(S + D + H, B * H * W * 4, D, device="cuda")           # rows (b h w p1 p2) of D channels
        buf, o = guarded((B, 2 * H, 2 * W, D))
        _call("sigma_pixel_shuffle_norm_fwd", ptr(y), ptr(g), ptr(b), ptr(o), B, H, W, D, EPS, stream())
        guard_ok(buf, f"pixel shuffle {B}x{H}x{W}x{D}")
        ref = R.pixel_shuffle64(R.layer_norm_ref64(y, g, b, EPS).view(B, H, W, 4 * D), B, H, W)
        bnd = R.pixel_shuffle64(R.layer_norm_bound(y, g, b, EPS, plan).view(B, H, W, 4 * D), B, H, W)
        _check(f"pixel shuffle {B}x{H}x{W}x{D}", o, ref, bnd, worst, "y")
    record("rowwise_fp64/pixel_shuffle", D=D, bound_used=worst["y"])


# ---------------------------------------------------------------- bilinear x2, its LayerNorm, the head
def _upsample_input(seed, B, H, W, C):
    """N(0, 4) plus a per-pixel offset N(0, 40^2): after the taps, rows with a mean far from 0"""
    return _randn(seed, (B, H, W, C), 2.0) + _randn(seed + 1, (B, H, W, 1), 40.0)


@pytest.mark.parametrize("C", UPSAMPLE_C)
def test_upsample2x_norm(C):
    g, b = _affine(S + C, C)
    plan, worst = R.head_plan(C, 0), {}
    for B, H, W in ((2, 7, 9), (1, 1, 1), (1, 1, 5), (1, 5, 1)):
        x = _upsample_input(S + C + H + W, B, H, W, C)
        buf, o = guarded((B, 2 * H, 2 * W, C))
        _call("sigma_upsample2x_norm_fwd", ptr(x), ptr(g), ptr(b), ptr(o), B, H, W, C, EPS, stream())
        guard_ok(buf, f"upsample norm {B}x{H}x{W}x{C}")
        _check(f"upsample norm {B}x{H}x{W}x{C}", o, R.upsample2x_norm_ref64(x, g, b, EPS), R.upsample2x_norm_bound(x, g, b, EPS, plan),
               worst, "norm")
        buf, o = guarded((B, 2 * H, 2 * W, C))
        _call("sigma_upsample2x_norm_fwd", ptr(x), None, None, ptr(o), B, H, W, C, 0.0, stream())
        guard_ok(buf, f"upsample {B}x{H}x{W}x{C}")
        _check(f"upsample {B}x{H}x{W}x{C}", o, R.upsample2x_ref64(x), R.upsample2x_bound(x), worst, "plain")
    record("rowwise_fp64/upsample2x", C=C, plan=list(plan), bound_used=worst)


@pytest.mark.parametrize("B,H,W,C", [(2, 15, 20, 384), (2, 30, 40, 192), (1, 60, 80, 96), (2, 120, 160, 96)])
def test_upsample2x_decoder_shapes(B, H, W, C):
    """UpsampleExpand's upsample2x_norm at the decoder's maps, and final_head's plain x2 (120 x 160 -> 240 x 320 at C = 96)"""
    x = _upsample_input(S + H, B, H, W, C)
    g, b = _affine(S + C, C)
    worst = {}
    buf, o = guarded((B, 2 * H, 2 * W, C))
    _call("sigma_upsample2x_norm_fwd", ptr(x), None, None, ptr(o), B, H, W, C, 0.0, stream())
    guard_ok(buf, "plain x2")
    _check("plain x2", o, R.upsample2x_ref64(x), R.upsample2x_bound(x), worst, "plain")
    if H < 120:
        buf, o = guarded((B, 2 * H, 2 * W, C))
        _call("sigma_upsample2x_norm_fwd", ptr(x), ptr(g), ptr(b), ptr(o), B, H, W, C, EPS, stream())
        guard_ok(buf, "x2 norm")
        _check("x2 norm", o, R.upsample2x_norm_ref64(x, g, b, EPS), R.upsample2x_norm_bound(x, g, b, EPS, R.head_plan(C, 0)), worst,
               "norm")
    record("rowwise_fp64/upsample2x_decoder", B=B, H=H, W=W, C=C, bound_used=worst)


def _head(x, g, b, wc):
    B, H, W, C = x.shape
    ncls = wc.shape[0]
    buf, o = guarded((B, ncls, 2 * H, 2 * W))
    _call("sigma_upsample2x_norm_head_fwd", ptr(x), ptr(g), ptr(b), ptr(wc), ncls, ptr(o), B, H, W, C, EPS, stream())
    guard_ok(buf, f"head {B}x{H}x{W}x{C} ncls {ncls}")
    return o


def _head_case(C, ncls, B=2, H=13, W=49, tag="head"):
    """13 x 49 -> 26 x 98: 4 x 4 tiles of 8 x 32 outputs, the last ones ragged in both directions"""
    x = _upsample_input(S + C + ncls, B, H, W, C)
    g, b = _affine(S + ncls, C)
    wc = _randn(S + C * ncls, (ncls, C), C ** -0.5)
    o = _head(x, g, b, wc)
    plan, worst = R.head_plan(C, ncls), {}
    _check(f"{tag} C={C} ncls={ncls}", o, R.head_ref64(x, g, b, EPS, wc), R.head_bound(x, g, b, EPS, wc, plan), worst, "logits")
    record(f"rowwise_fp64/{tag}", C=C, ncls=ncls, H=H, W=W, plan=list(plan), bound_used=worst["logits"])


@pytest.mark.parametrize("ncls", [2, 9, 21])
@pytest.mark.parametrize("C", HEAD_FAST_C)
def test_head_fast_widths(C, ncls):
    assert R.head_plan(C, ncls)[2]
    _head_case(C, ncls)


@pytest.mark.parametrize("ncls", [n for n in HEAD_FAST_NCLS if n not in (2, 9, 21)])
def test_head_fast_classes(ncls):
    _head_case(96, ncls)


@pytest.mark.parametrize("C,ncls", [(96, n) for n in HEAD_GENERIC_NCLS] + [(c, 9) for c in HEAD_GENERIC_C])
def test_head_generic(C, ncls):
    assert not R.head_plan(C, ncls)[2]
    _head_case(C, ncls)


@pytest.mark.parametrize("ncls", [9, 40])
def test_head_sigma_size(ncls):
    """Sigma's head: 240 x 320 -> 480 x 640 at C = 96 (15 x 60 tiles with a seam every 32 columns), the whole logit tensor"""
    _head_case(96, ncls, B=1, H=240, W=320, tag="head_full")


# ---------------------------------------------------------------- pool_avgmax
@pytest.mark.parametrize("B", [1, 2, 74])
@pytest.mark.parametrize("C,H,W", [(768, 15, 20), (384, 30, 40), (192, 60, 80), (96, 120, 160)])
def test_pool_avgmax_decoder(C, H, W, B):
    """through fused.pool_avgmax, whose slice count depends on B: compared with fp64 only (no batch-1 identity)"""
    from sigma_b200 import fused
    L = H * W
    x = R.pool_input(S + C + B, B, L, C, device="cuda")
    mean, mx = fused.pool_avgmax(x.view(B, H, W, C))
    torch.cuda.synchronize()
    nslice = max(1, min(64, L // 32, max(L // 256, -(-296 // B))))      # fused.pool_avgmax's slice count
    rm, rx = R.pool_avgmax_ref64(x)
    assert torch.equal(mx.double(), rx), "max differs from the fp64 max"
    worst = {}
    _check(f"pool {B}x{L}x{C}", mean, rm, R.pool_mean_bound(x, nslice), worst, "mean")
    record("rowwise_fp64/pool_avgmax", B=B, L=L, C=C, nslice=nslice, bound_used=worst["mean"])


@pytest.mark.parametrize("C", [4, 1000, 1024])
@pytest.mark.parametrize("L,nslice", [(2049, 1), (2049, 64), (300, 7)])
def test_pool_partial_forced_slices(L, nslice, C):
    """the partial kernel at a forced slice count: 1, 64 slices of 33 over 2049 positions (the last one empty), 7 of 43 over
    300; C = 1000 leaves 6 of 256 threads idle"""
    B = 2
    x = R.pool_input(S + L + C, B, L, C, device="cuda")
    buf, part = guarded((B, nslice, 2, C))
    _call("sigma_pool_avgmax_partial_fwd", ptr(x), ptr(part), B, L, C, nslice, stream())
    guard_ok(buf, f"pool partial {L}/{nslice}/{C}")
    ref = R.pool_partial_ref64(x, nslice)
    assert torch.equal(part[:, :, 1].double(), ref[:, :, 1]), "slice maxima differ from fp64 (empty slices: -inf)"
    worst = {}
    _check(f"pool partial {L}/{nslice}/{C}", part[:, :, 0], ref[:, :, 0], R.pool_partial_bound(x, nslice), worst, "sum")
    empty = [s for s, (l0, l1) in enumerate(R.pool_slices(L, nslice)) if l1 == l0]
    assert (nslice == 64) == bool(empty)
    record("rowwise_fp64/pool_partial", L=L, nslice=nslice, C=C, empty_slices=len(empty), bound_used=worst["sum"])


# ---------------------------------------------------------------- scale_add
@pytest.mark.parametrize("with_a", [True, False])
def test_scale_add_grid_stride(with_a):
    C, rpb, Bn = 96, 19200, 8
    rows = Bn * rpb
    passes = rows * C // 4 / (132 * 32 * 256)
    assert passes >= 3 and (132 * 32 * 256 * 4 // C) % rpb != 0
    a = _randn(S + 1, (rows, C)) if with_a else None
    sa = _randn(S + 2, (Bn, C)) if with_a else None
    bq = _randn(S + 3, (rows, C), 10.0)
    sb = _randn(S + 4, (C,))
    buf, o = guarded((rows, C))
    _call("sigma_scale_add_fwd", ptr(a), ptr(sa), ptr(bq), ptr(sb), ptr(o), rows, rpb, C, stream())
    guard_ok(buf, "scale_add")
    worst = {}
    _check("scale_add", o, R.scale_add_ref64(a, sa, bq, sb, rpb), R.scale_add_bound(a, sa, bq, sb, rpb), worst, "out")
    record("rowwise_fp64/scale_add", with_a=with_a, passes=passes, bound_used=worst["out"])


# ---------------------------------------------------------------- layernorm_bwd
def test_layernorm_bwd_past_grid_cap():
    rows, C = 150000, 96
    lpr, v, nw, steps = R.bwd_plan(rows, C)
    assert nw == 132 * 8 * 8 and steps >= 5, "premise: the grid is capped and every warp walks >= 5 steps"
    x = R.hard_rows(S + 11, rows, C, device="cuda")
    dy = _randn(S + 12, (rows, C))
    g, _ = _affine(S + 13, C)
    L_ = _lib().lib()
    outs = {}
    for det in (False, True, True):
        bx, dx = guarded((rows, C))
        bg, dg = guarded((C,))
        bb, db = guarded((C,))
        if det:
            wsb = L_.sigma_layernorm_bwd_det_workspace_bytes(rows, C)
            ws = torch.full((wsb // 4,), float("nan"), device="cuda")
            _call("sigma_layernorm_bwd_det", ptr(x), ptr(dy), ptr(g), ptr(dx), ptr(dg), ptr(db), rows, C, EPS, ptr(ws), wsb, stream())
        else:
            _call("sigma_layernorm_bwd", ptr(x), ptr(dy), ptr(g), ptr(dx), ptr(dg), ptr(db), rows, C, EPS, stream())
        for buf, what in ((bx, "dx"), (bg, "dgamma"), (bb, "dbeta")):
            guard_ok(buf, f"layernorm_bwd det={det} {what}")
        outs.setdefault(det, []).append((dx.clone(), dg.clone(), db.clone()))
    (a, b) = outs[True]
    assert all(torch.equal(p, q) for p, q in zip(a, b)), "the deterministic backward is not bitwise repeatable"
    assert torch.equal(outs[False][0][0], a[0]), "dx differs between the atomic and the deterministic build"
    ref = R.layernorm_bwd_ref64(x, dy, g, EPS)
    bnd = R.layernorm_bwd_bound(x, dy, g, EPS)
    worst = {}
    for det in (False, True):
        for name, got, rf, bd in zip(("dx", "dgamma", "dbeta"), outs[det][0], ref, bnd):
            _check(f"layernorm_bwd det={det} {name}", got, rf, bd, worst, name)
    record("rowwise_fp64/layernorm_bwd", rows=rows, C=C, warps=nw, steps_per_warp=steps, bound_used=worst)


@pytest.mark.parametrize("D", BWD_BF16_D)
def test_layernorm_bwd_bf16(D):
    """sigma_layernorm_bwd_bf16 (bf16 x, dy and dx; fp32 gamma, dgamma, dbeta) at every instantiation, its grid capped and every
    warp walking 5 steps, on the bf16 form of every hard_rows family: dx inside layernorm_bwd_bound plus its bf16 store, dgamma /
    dbeta inside the unchanged fp32 bound"""
    lpr = R.bwd_plan(1, D)[0]
    rows = 5 * R.NUM_SMS * 8 * 32 * (32 // lpr) // 4 - 3          # the last warp step ragged where a step holds several rows
    _, _, nw, steps = R.bwd_plan(rows, D)
    assert nw == R.NUM_SMS * 8 * 8 and steps == 5, "premise: the grid is capped and every warp walks 5 steps"
    x = R.hard_rows(S + 31 + D, rows, D, device="cuda", bf16=True)
    dy = _randn(S + 32 + D, (rows, D)).to(BF)
    g, _ = _affine(S + 33 + D, D)
    bx, dx = guarded((rows, D), BF)
    bg, dg = guarded((D,))
    bb, db = guarded((D,))
    _call("sigma_layernorm_bwd_bf16", ptr(x), ptr(dy), ptr(g), ptr(dx), ptr(dg), ptr(db), rows, D, EPS, stream())
    for buf, what in ((bx, "dx"), (bg, "dgamma"), (bb, "dbeta")):
        guard_ok(buf, f"layernorm_bwd_bf16 D={D} {what}")
    ref = R.layernorm_bwd_ref64(x, dy, g, EPS)
    bnd = list(R.layernorm_bwd_bound(x, dy, g, EPS))
    bnd[0] = R.bf16_store_bound(ref[0], bnd[0])
    worst = {}
    for name, got, rf, bd in zip(("dx", "dgamma", "dbeta"), (dx, dg, db), ref, bnd):
        _check(f"layernorm_bwd_bf16 D={D} {name}", got, rf, bd, worst, name)
    record("rowwise_fp64/layernorm_bwd_bf16", rows=rows, D=D, warps=nw, steps_per_warp=steps, bound_used=worst)


# ---------------------------------------------------------------- the benchmark's batch
BENCH_B = 74
CHECK_IMAGES = (0, 37, 73)


def test_bench_batch_layernorm():
    """C = 96 on 74 x 19200 rows (120 x 160 maps), fp32 and bf16 out (sigma_layernorm_fwd_bf16, the bf16 inference mode's): every
    image bit-identical to a batch-1 run; images 0, 37, 73 against fp64"""
    C, L = 96, 120 * 160
    x = R.hard_rows(S + 21, BENCH_B * L, C, device="cuda")
    g, b = _affine(S + 22, C)
    worst = {}
    for io in (0, 1):
        y = _layernorm(x, g, b, io)
        for i in range(BENCH_B):
            assert torch.equal(_layernorm(x[i * L:(i + 1) * L].contiguous(), g, b, io), y[i * L:(i + 1) * L]), f"io={io} image {i}"
        for i in CHECK_IMAGES:
            xi = x[i * L:(i + 1) * L]
            ref = R.layer_norm_ref64(xi, g, b, EPS)
            _check(f"bench ln io={io} image {i}", y[i * L:(i + 1) * L], ref,
                   _bound(io, ref, R.layer_norm_bound(xi, g, b, EPS, R.row_plan(C, io=io))), worst, f"y_io{io}")
    record("rowwise_fp64/bench_layernorm", B=BENCH_B, bound_used=worst["y_io0"], bound_used_bf16=worst["y_io1"])


def test_bench_batch_head():
    """the head at B = 74, 240 x 320 -> 480 x 640, C = 96, 9 classes: every image bit-identical to a batch-1 run; images 0, 37,
    73 against fp64"""
    C, H, W, ncls = 96, 240, 320, 9
    x = torch.empty((BENCH_B, H, W, C), device="cuda")
    for i in range(BENCH_B):
        x[i] = _upsample_input(S + 1000 + i, 1, H, W, C)[0]
    g, b = _affine(S + 23, C)
    wc = _randn(S + 24, (ncls, C), C ** -0.5)
    o = _head(x, g, b, wc)
    for i in range(BENCH_B):
        assert torch.equal(_head(x[i:i + 1].contiguous(), g, b, wc), o[i:i + 1]), f"image {i}"
    worst = {}
    plan = R.head_plan(C, ncls)
    for i in CHECK_IMAGES:
        xi = x[i:i + 1]
        _check(f"bench head image {i}", o[i:i + 1], R.head_ref64(xi, g, b, EPS, wc), R.head_bound(xi, g, b, EPS, wc, plan), worst,
               "logits")
    record("rowwise_fp64/bench_head", B=BENCH_B, bound_used=worst["logits"])
