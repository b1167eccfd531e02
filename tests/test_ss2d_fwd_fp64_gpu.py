"""GPU: the fused SS2D scan's inference forward (sigma_ss2d_scan_fwd, _split and _bf16: the kernels the inference benchmark times)
against the fp64 reference of oracle/ss2d_ref64.py (ss2d_fwd_ref64), element by element inside its per-element error bound, at
Sigma's inference shapes and all three scan kinds: the SS2D blocks (CROSS4, d_state 16), CroMB (CROSS, d_state 4: C from the other
modality), ConMB (SEQ2, d_state 4) and the decoder (CROSS4, d_state 4).
* launch plans: the library's choice, forced 1, 2, 7, 32 and 100 L-segments, a count that leaves only the shorter walks an empty
  trailing segment and one whose last segment is empty in every direction (both found through the plan query
  sigma_test_ss2d_fwd_plan), and the library's choice without a workspace;
* both register budgets of d_state 16 at every padded dt_rank, CTAs of 1-4 warps, ring depths 2 and 8, ragged D whose last CTA is
  partly filled (its surplus channels must write nowhere but the sink);
* bf16 xc / y on both sides of the split decision;
* the benchmark's batch of 74 images (148 for CROSS): every image bit-identical to a batch-1 run of it (its pair for CROSS) under
  the same plan, and a sample of images, the last ones included, against the reference.
y sits in NaN-filled memory whose guard elements must stay bit-identical and whose interior must be written everywhere; the
workspace is NaN-filled too, so no result can depend on its contents.  Parameters: dt log-uniform in [1e-3, 0.1] through the
inverse softplus, A = -exp(A_log) around the S4D-real init, Ds near 1; one widened set (dt up to 0.5, |A| up to 4x).  Worst bound
fractions go to helpers.record."""
import pytest
import torch

from helpers import guard_ok, guarded, ptr, record, ss2d_fwd_plan, ss2d_kind, ss2d_params, stream
from oracle import ss2d_ref64 as R64

pytestmark = pytest.mark.gpu
S = 89
SCAN_ENV = ("SIGMA_SCAN_WARPS", "SIGMA_SCAN_NST", "SIGMA_SCAN_CTAS", "SIGMA_SCAN_SPLIT_RULE")


@pytest.fixture(autouse=True)
def _library_plans(monkeypatch):
    for e in SCAN_ENV:
        monkeypatch.delenv(e, raising=False)


def _lseq(kind, H, W):
    return H * W * (2 if kind == "seq2" else 1)


def _run(kind, args, B, H, W, D, N, R, Cp, force=None, ws=True, tag=""):
    """one forward into NaN-guarded y with a NaN-filled workspace (ws=False: none).  force None: sigma_ss2d_scan_fwd, or
    sigma_ss2d_scan_fwd_bf16 when xc is bf16; otherwise sigma_ss2d_scan_fwd_split with that count.  Checks the guards."""
    from sigma_b200 import _lib
    L_ = _lib.lib()
    xc, xdbl, dtw, dtb, A, Ds = args[:6]
    bf16 = xc.dtype == torch.bfloat16
    buf, y = guarded((R64.KINDS[kind], B, _lseq(kind, H, W), D), xc.dtype)
    wsb = L_.sigma_ss2d_scan_workspace_bytes(ss2d_kind(kind), B, H, W, D, N) if ws else 0
    wsbuf = torch.full((wsb // 4,), float("nan"), device="cuda") if ws else None
    head = (ss2d_kind(kind), ptr(xc), ptr(xdbl), ptr(dtw), ptr(dtb), ptr(A), ptr(Ds), ptr(y), B, H, W, D, N, R, Cp, ptr(wsbuf), wsb)
    if bf16:
        assert force is None
        rc = L_.sigma_ss2d_scan_fwd_bf16(*head, stream())
    elif force is None:
        rc = L_.sigma_ss2d_scan_fwd(*head, stream())
    else:
        rc = L_.sigma_ss2d_scan_fwd_split(*head, force, stream())
    _lib.check(rc, f"sigma_ss2d_scan_fwd {tag}")
    torch.cuda.synchronize()
    guard_ok(buf, tag)
    return y


def _check(tag, got, ref, bnd, worst, key="y"):
    """every element written and inside its bound; at the largest |y| the error is also within 1e-3 of scale (bf16: plus the
    2^-8 of its rounding)"""
    assert not bool(got.isnan().any()), f"{tag}: y not written everywhere"
    frac = R64.bound_fraction(got, ref, bnd)
    worst[key] = max(worst.get(key, 0.0), frac)
    assert frac <= 1.0, f"{tag}: {frac:.3f} of the per-element bound"
    i = int(ref.abs().argmax())
    scale = float(ref.reshape(-1)[i].abs())
    bar = 1e-3 + (R64.BF16_RN if got.dtype == torch.bfloat16 else 0.0)
    err = abs(float(got.reshape(-1)[i].double()) - float(ref.reshape(-1)[i]))
    assert err <= bar * scale, f"{tag}: {err / scale:.2e} of scale at the largest element"
    worst["at_max/" + key] = max(worst.get("at_max/" + key, 0.0), float(bnd.reshape(-1)[i]) / (bar * scale))


def _forced_empty(kind, B, H, W, D, N, R):
    """from the plan query: the smallest forced count whose trailing segments are empty for the shorter walks only, and the
    smallest whose last segment is empty in every direction (None where no count up to 32 does that)"""
    short = every = None
    for n in range(2, 33):
        pl = ss2d_fwd_plan(kind, B, H, W, D, N, R, force=n)
        last0 = (pl["nsplit"] - 1) * pl["tiles_per_split"]
        if short is None and pl["min_tiles"] <= last0 < pl["max_tiles"]:
            short = n
        if every is None and last0 >= pl["max_tiles"]:
            every = n
    return short, every


SS2D = [(120, 160, 192, 6), (60, 80, 384, 12), (30, 40, 768, 24), (15, 20, 1536, 48), (45, 60, 1024, 32), (23, 30, 2048, 64)]
SMALL4 = [(120, 160, 192, 6), (60, 80, 384, 12), (30, 40, 768, 24), (15, 20, 1536, 48), (23, 30, 2048, 64)]
DEC = [(120, 160, 192, 6), (60, 80, 384, 12), (30, 40, 768, 24)]
SHAPES = ([("cross4", H, W, D, 16, R) for H, W, D, R in SS2D] + [("cross", H, W, D, 4, R) for H, W, D, R in SMALL4]
          + [("seq2", H, W, D, 4, R) for H, W, D, R in SMALL4] + [("cross4", H, W, D, 4, R) for H, W, D, R in DEC])
CASES = [(k, im, H, W, D, N, R) for k, H, W, D, N, R in SHAPES for im in (1, 2)] + [("cross4", 3, 30, 40, 768, 16, 24)]


@pytest.mark.parametrize("kind,images,H,W,D,N,R", CASES)
def test_fused_fwd_matches_fp64(kind, images, H, W, D, N, R):
    B = 2 * images if kind == "cross" else images
    tag = f"{kind}/{images}/{H}x{W}/D{D}/N{N}/R{R}"
    args, Cp = ss2d_params(S, kind, B, H, W, D, N, R, tag)
    ref, bnd = R64.ss2d_fwd_ref64(kind, *args[:6], H, W)
    auto = ss2d_fwd_plan(kind, B, H, W, D, N, R)
    if (H, W) == (15, 20) and images == 1:
        assert auto["nsplit"] > 1, auto                                  # stage 3 of one image runs L-segments by default
    cap = ss2d_fwd_plan(kind, B, H, W, D, N, R, force=100)
    assert cap["nsplit"] == min(32, cap["max_tiles"]), cap              # 100 is capped at 32 segments
    short, every = _forced_empty(kind, B, H, W, D, N, R)
    runs = [None, 1, 2, 7, 32, 100] + [n for n in (short, every) if n is not None]
    if (H, W, N) == (15, 20, 16):
        pl = ss2d_fwd_plan(kind, B, H, W, D, N, R, force=8)
        assert (pl["nsplit"], pl["tiles_per_split"], pl["max_tiles"]) == (8, 3, 20)      # segment 7 would start at tile 21 of 20
        runs.append(8)
    worst = {}
    for force in runs:
        y = _run(kind, args, B, H, W, D, N, R, Cp, force=force, tag=f"{tag} split={force}")
        _check(f"{tag} split={force}", y, ref, bnd, worst)
        del y
    if auto["nsplit"] > 1:                                               # without a workspace the same call runs one segment
        assert ss2d_fwd_plan(kind, B, H, W, D, N, R, ws_bytes=0)["nsplit"] == 1
        _check(f"{tag} no workspace", _run(kind, args, B, H, W, D, N, R, Cp, ws=False, tag=f"{tag} no ws"), ref, bnd, worst)
    record(f"ss2d fwd fp64 {tag}", short=short, every=every, **worst)


@pytest.mark.parametrize("kind,images,H,W,D,N,R", [("cross4", 1, 15, 20, 1536, 16, 48), ("seq2", 2, 60, 80, 384, 4, 12),
                                                   ("cross", 1, 120, 160, 192, 4, 6), ("cross4", 1, 120, 160, 192, 16, 6)])
def test_fused_fwd_matches_fp64_widened(kind, images, H, W, D, N, R):
    """larger steps and decays: dt up to 0.5, |A| up to 4x the S4D-real init"""
    B = 2 * images if kind == "cross" else images
    tag = f"wide/{kind}/{images}/{H}x{W}/D{D}/N{N}/R{R}"
    args, Cp = ss2d_params(S, kind, B, H, W, D, N, R, tag, wide=True)
    ref, bnd = R64.ss2d_fwd_ref64(kind, *args[:6], H, W)
    worst = {}
    for force in (None, 1, 7, 32):
        _check(f"{tag} split={force}", _run(kind, args, B, H, W, D, N, R, Cp, force=force, tag=tag), ref, bnd, worst)
    record(f"ss2d fwd fp64 {tag}", **worst)


@pytest.mark.parametrize("R", [4, 8, 12, 16, 24, 32, 48, 64])
def test_register_budgets_match_fp64(R, monkeypatch):
    """d_state 16 under both register budgets (128 and 168 registers: `CTAS` 4 and 3) at every padded dt_rank"""
    kind, B, H, W, D, N = "cross4", 1, 30, 40, 384, 16
    tag = f"ctas/{kind}/{H}x{W}/D{D}/N{N}/R{R}"
    args, Cp = ss2d_params(S, kind, B, H, W, D, N, R, tag)
    ref, bnd = R64.ss2d_fwd_ref64(kind, *args[:6], H, W)
    worst = {}
    for ctas in (3, 4):
        monkeypatch.setenv("SIGMA_SCAN_CTAS", str(ctas))
        for force in (1, 3):
            pl = ss2d_fwd_plan(kind, B, H, W, D, N, R, force=force)
            assert pl["ctas"] == ctas and pl["nsplit"] == force, pl
            _check(f"{tag} ctas={ctas} split={force}", _run(kind, args, B, H, W, D, N, R, Cp, force=force, tag=tag), ref, bnd, worst,
                   key=f"y/ctas{ctas}")
    record(f"ss2d fwd fp64 {tag}", **worst)


@pytest.mark.parametrize("kind,N,R", [("cross4", 16, 24), ("cross", 4, 12), ("seq2", 4, 12)])
def test_cta_shapes_and_ring_depths_match_fp64(kind, N, R, monkeypatch):
    """CTAs of 1-4 warps, TMA rings of 2 and 8 stages, and ragged D (100, 132: a partly filled last CTA whose surplus channels
    store to the sink; the guards and the every-element check would see a store anywhere else)"""
    images, H, W = 1, 30, 40
    B = 2 * images if kind == "cross" else images
    worst = {}
    for D in (384, 288, 100, 132):                                       # 288: 3-warp CTAs
        tag = f"cta/{kind}/{H}x{W}/D{D}/N{N}/R{R}"
        args, Cp = ss2d_params(S, kind, B, H, W, D, N, R, tag)
        ref, bnd = R64.ss2d_fwd_ref64(kind, *args[:6], H, W)
        envs = [("SIGMA_SCAN_WARPS", w) for w in (1, 2, 3, 4)] + [("SIGMA_SCAN_NST", n) for n in (2, 8)] if D == 384 else [(None, None)]
        for name, val in envs:
            if name:
                monkeypatch.setenv(name, str(val))
            for force in (1, 3):
                pl = ss2d_fwd_plan(kind, B, H, W, D, N, R, force=force)
                if name == "SIGMA_SCAN_NST":
                    assert pl["nst"] == val
                if name == "SIGMA_SCAN_WARPS":
                    assert pl["warps"] == next(x for x in (4, 2, 3, 1) if x <= val and D % (32 * x) == 0)
                if D == 288:
                    assert pl["warps"] == 3, pl
                if D in (100, 132):
                    assert D % (32 * pl["warps"]) != 0, pl                   # the last CTA is partly filled
                _check(f"{tag} {name}={val} split={force}", _run(kind, args, B, H, W, D, N, R, Cp, force=force, tag=tag), ref, bnd,
                       worst)
            if name:
                monkeypatch.delenv(name)
    record(f"ss2d fwd fp64 cta/{kind}", **worst)


@pytest.mark.parametrize("kind,N", [("cross4", 16), ("cross", 4), ("seq2", 4)])
@pytest.mark.parametrize("H,W,D,R", [(120, 160, 192, 6), (15, 20, 1536, 48)])
@pytest.mark.parametrize("images", [1, 2])
def test_bf16_fwd_matches_fp64(kind, N, H, W, D, R, images):
    """sigma_ss2d_scan_fwd_bf16 against the reference run on the exact bf16 values of xc, whose bound adds y's final rounding"""
    B = 2 * images if kind == "cross" else images
    tag = f"bf16/{kind}/{images}/{H}x{W}/D{D}/N{N}/R{R}"
    args, Cp = ss2d_params(S, kind, B, H, W, D, N, R, tag)
    args[0] = args[0].to(torch.bfloat16)
    pl = ss2d_fwd_plan(kind, B, H, W, D, N, R, bf16=True)
    if H == 15:
        assert (pl["nsplit"] > 1) == (images == 1), pl                   # both sides of the split decision
    assert pl["ctas"] == 3
    ref, bnd = R64.ss2d_fwd_ref64(kind, *args[:6], H, W)
    worst = {}
    _check(tag, _run(kind, args, B, H, W, D, N, R, Cp, tag=tag), ref, bnd, worst, key="y_bf16")
    record(f"ss2d fwd fp64 {tag}", nsplit=pl["nsplit"], **worst)


def _batch_inputs(kind, B, H, W, D, N, R, tag):
    """the benchmark's batch: per-image xc / x_dbl drawn on the device (the procedural generator is too slow for 4 GB), one
    parameter set"""
    args, Cp = ss2d_params(S, kind, 2 if kind == "cross" else 1, 1, 1, D, N, R, tag)
    g = torch.Generator(device="cuda")
    g.manual_seed(S)
    Lseq = _lseq(kind, H, W)
    xc = torch.randn((B, Lseq, D), generator=g, device="cuda")
    xdbl = torch.randn((B, Lseq, R64.KINDS[kind], Cp), generator=g, device="cuda")
    xdbl[..., 2 * N:2 * N + R] *= 2.0
    xdbl[..., 2 * N + R:] = 0.0
    return [xc, xdbl] + args[2:6], Cp


@pytest.mark.parametrize("kind,N,R", [("cross4", 16, 6), ("cross", 4, 6), ("seq2", 4, 6)])
def test_benchmark_batch(kind, N, R):
    """stage 0 at 74 images: every image as a batch-1 run computes it, bit for bit (same plan: warps, ring, register budget and
    segments), and images 0, 1, 37, 72, 73 (and their CROSS partners) inside the fp64 bound under the library's plan"""
    images, H, W, D = 74, 120, 160, 192
    cross = kind == "cross"
    B = 2 * images if cross else images
    tag = f"batch/{kind}/{images}/{H}x{W}/D{D}/N{N}/R{R}"
    torch.cuda.reset_peak_memory_stats()
    args, Cp = _batch_inputs(kind, B, H, W, D, N, R, tag)
    xc, xdbl = args[0], args[1]
    b1 = 2 if cross else 1
    members = (lambda i: [i, i + images]) if cross else (lambda i: [i])
    for force in (1, 3):
        big, one = ss2d_fwd_plan(kind, B, H, W, D, N, R, force=force), ss2d_fwd_plan(kind, b1, H, W, D, N, R, force=force)
        same = ("nsplit", "tiles_per_split", "warps", "nst", "ctas", "smem")
        assert {k: big[k] for k in same} == {k: one[k] for k in same}, (big, one)
        y = _run(kind, args, B, H, W, D, N, R, Cp, force=force, tag=f"{tag} split={force}")
        assert not bool(y.isnan().any()), f"{tag} split={force}: y not written everywhere"
        for i in range(images):
            sel = members(i)
            sub = [xc[sel].contiguous(), xdbl[sel].contiguous()] + args[2:]
            y1 = _run(kind, sub, b1, H, W, D, N, R, Cp, force=force, tag=f"{tag} image {i} split={force}")
            same = torch.equal(y[:, sel], y1)
            assert same, f"{tag} split={force}: image {i} differs from its batch-1 run"
        del y
    y = _run(kind, args, B, H, W, D, N, R, Cp, tag=f"{tag} auto")
    worst = {}
    for i in (0, 1, 37, 72, 73):
        sel = members(i)
        ref, bnd = R64.ss2d_fwd_ref64(kind, xc[sel], xdbl[sel], *args[2:], H, W)
        _check(f"{tag} image {i}", y[:, sel], ref, bnd, worst)
    record(f"ss2d fwd fp64 {tag}", peak_gb=torch.cuda.max_memory_allocated() / 2 ** 30, **worst)


@pytest.mark.parametrize("kind,N", [("cross4", 16), ("cross", 4), ("seq2", 4)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_wrapper_matches_fp64(kind, N, dtype):
    """fused.ss2d_scan: its workspace sizing (the library's plan splits at this shape) and its output dtype"""
    from sigma_b200 import fused
    images, H, W, D, R = 1, 60, 80, 384, 12
    B = 2 * images if kind == "cross" else images
    tag = f"wrapper/{kind}/{dtype}"
    args, Cp = ss2d_params(S, kind, B, H, W, D, N, R, tag)
    args[0] = args[0].to(dtype)
    assert ss2d_fwd_plan(kind, B, H, W, D, N, R, bf16=dtype == torch.bfloat16)["nsplit"] > 1
    ref, bnd = R64.ss2d_fwd_ref64(kind, *args[:6], H, W)
    y = fused.ss2d_scan(ss2d_kind(kind), *args[:6], B, H, W, D, N, R, Cp)
    torch.cuda.synchronize()
    assert y.dtype == dtype and y.shape == ref.shape
    worst = {}
    _check(tag, y, ref, bnd, worst)
    record(f"ss2d fwd fp64 {tag}", **worst)
