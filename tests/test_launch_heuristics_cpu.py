"""CPU: the two launch heuristics of the latency regime, held to a recorded H100 sweep through host-only test hooks.
* `ss2d_pick_segments` (L-segment count of the fused scan, a cost model of the busiest SM): replayed on every row of
  tests/golden/ss2d_split_sweep_h100.txt (scripts/bench_ss2d_splits.py on an H100 SXM at 400 W: 15 call shapes x {1,2,4,8}
  images x 10 forced counts) its choices must stay within 6 % of the per-row optimum in total and well ahead of the old rule.
* `pick_bn` (GEMM tile width): the widest divisor in the throughput regime, narrower tiles when few row tiles exist.
* `plan_gemm` (the whole launch plan of the GEMM / implicit-GEMM conv, SIGMA_GEMM_BN included, through sigma_test_gemm_plan):
  every plan is launchable — grid within the tile count, 2-8 ring stages, shared memory within the H100's limits.
* the fused scan forward's whole launch plan (through sigma_test_ss2d_fwd_plan) at every Sigma inference shape and 1, 2, 8 and 74
  images: segments capped at 32 and never empty for the longest walk by choice, one segment without a workspace, the 4-CTA register
  budget only where it is built and chosen, a ring of 2-8 stages whose shared memory fits the CTAs the budget puts on an SM.
* the fused scan backward's plan for kind CROSS (sigma_test_ss2d_bwd_plan), its state and workspace sizes at every CroMB training
  shape and 1, 2, 3, 8 images, and the rejection of an odd batch."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPLITS = [1, 2, 3, 4, 6, 8, 12, 16, 24, 32]
# name -> (streams per image, H, W, D, d_state, directions, sequence factor)
SHAPES = {"enc0": (2, 120, 160, 192, 16, 4, 1), "enc1": (2, 60, 80, 384, 16, 4, 1), "enc2": (2, 30, 40, 768, 16, 4, 1),
          "enc3": (2, 15, 20, 1536, 16, 4, 1), "dec0": (1, 120, 160, 192, 4, 4, 1), "dec1": (1, 60, 80, 384, 4, 4, 1),
          "dec2": (1, 30, 40, 768, 4, 4, 1), "conmb0": (1, 120, 160, 192, 4, 2, 2), "cromb0": (2, 120, 160, 192, 4, 1, 1),
          "conmb1": (1, 60, 80, 384, 4, 2, 2), "cromb1": (2, 60, 80, 384, 4, 1, 1), "conmb2": (1, 30, 40, 768, 4, 2, 2),
          "cromb2": (2, 30, 40, 768, 4, 1, 1), "conmb3": (1, 15, 20, 1536, 4, 2, 2), "cromb3": (2, 15, 20, 1536, 4, 1, 1)}


@pytest.fixture(scope="module")
def L():
    from sigma_b200 import _lib
    return _lib.lib()


def _rows():
    rows = []
    for ln in open(os.path.join(ROOT, "tests", "golden", "ss2d_split_sweep_h100.txt")):
        p = ln.split()
        if len(p) == 15 and p[1].isdigit() and p[0] in SHAPES:
            rows.append((p[0], int(p[1]), [float(v) for v in p[2:12]], float(p[12]), float(p[14])))
    return rows


def test_segment_model_tracks_the_recorded_sweep(L):
    rows = _rows()
    assert len(rows) == 60
    tot_model = tot_best = tot_old = 0.0
    for name, images, times, t_old, t_best in rows:
        spi, H, W, D, N, K, seq = SHAPES[name]
        LT = 16 if N >= 16 else 32
        nw = next(w for w in (4, 2, 3, 1) if D % (32 * w) == 0)          # pick_warps (ss2d_scan_host.cu)
        ctas = (D // (32 * nw)) * K * images * spi
        ntiles = max(-(-(H * W * seq) // LT), W * (-(-H // LT)) if K == 4 else 0)
        n = L.sigma_test_pick_segments(ctas, nw, ntiles, N)
        assert 1 <= n <= 32
        lo = max(s for s in SPLITS if s <= n)
        hi = min(s for s in SPLITS if s >= n)
        tot_model += max(times[SPLITS.index(lo)], times[SPLITS.index(hi)])          # conservative between measured counts
        tot_best += t_best
        tot_old += t_old
    assert tot_model <= 1.06 * tot_best, (tot_model, tot_best)
    assert tot_model <= 0.85 * tot_old, (tot_model, tot_old)


def test_segment_model_leaves_full_grids_alone(L):
    # B = 74 shapes: every sub-partition has its warps already; a second pass can only lose
    assert L.sigma_test_pick_segments(3 * 4 * 132, 2, 1280, 16) == 1       # enc0
    assert L.sigma_test_pick_segments(6 * 4 * 132, 4, 80, 16) == 1         # enc2
    assert L.sigma_test_pick_segments(2 * 4 * 74, 2, 640, 4) == 1          # dec0
    assert L.sigma_test_pick_segments(1, 4, 1, 16) == 1                    # one tile cannot be cut


@pytest.mark.parametrize("N,want", [(96, 96), (160, 160), (176, 192), (192, 192), (384, 192), (768, 256), (1536, 256), (3072, 256), (9, 32)])
def test_gemm_tile_width_throughput_regime(L, N, want):
    assert L.sigma_test_pick_bn(N, 1 << 30) == want


@pytest.mark.parametrize("N", [96, 192, 384, 768, 1536, 3072])
@pytest.mark.parametrize("m_tiles", [1, 2, 5, 19, 75, 300, 22200])
def test_gemm_tile_width_is_a_valid_tile(L, N, m_tiles):
    bn = L.sigma_test_pick_bn(N, m_tiles)
    assert bn % 32 == 0 and 32 <= bn <= 256
    wide = L.sigma_test_pick_bn(N, 1 << 30)
    assert bn <= wide                                   # never wider than the throughput choice
    if m_tiles * -(-N // wide) >= 132 * 4:
        assert bn == wide                               # enough tiles for every persistent CTA: nothing to gain from narrow tiles
    if m_tiles <= 5 and N >= 768:
        assert bn <= 128                                # a handful of row tiles: spread the columns over more CTAs


# ---- the launch plan of the wgmma GEMM / implicit-GEMM conv (sigma_test_gemm_plan = the planner the launches use) ----
SMEM_PER_BLOCK = 227 * 1024      # H100: opt-in dynamic shared memory per block
SMEM_PER_SM = 228 * 1024
GEMM_SHAPES = [(1, 16, 32), (77, 160, 192), (1000, 384, 96), (4096, 320, 1536), (38417, 768, 384), (102401, 4, 36),
               (355200, 768, 192), (355200, 176, 384), (700, 3072, 768), (38401, 260, 100)]
CONV_SHAPES = [(6, 120, 160, 96, 32), (6, 120, 160, 32, 96), (20, 60, 80, 192, 64), (66, 30, 40, 384, 128), (20, 57, 75, 100, 36),
               (1, 1, 5, 32, 32), (3, 9, 17, 128, 384)]


def _check_plan(pl, x3):
    assert pl["bn"] % 32 == 0 and 32 <= pl["bn"] <= 256
    assert 1 <= pl["grid"] <= pl["tiles"]                                   # a persistent CTA never starts without a tile
    assert 2 <= pl["stages"] <= 8
    stage = (128 * 32 * 4 + -(-pl["bn"] * 32 * 4 // 1024) * 1024) * (2 if x3 else 1)
    assert pl["smem"] == pl["stages"] * stage + 1024
    assert pl["smem"] <= SMEM_PER_BLOCK
    assert pl["ctas_per_sm"] * (pl["smem"] + 1024) <= SMEM_PER_SM          # the CTAs the grid counts on fit an SM together
    assert pl["grid"] <= 132 * pl["ctas_per_sm"]


@pytest.mark.parametrize("x3", [False, True])
@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_plan_is_launchable(L, M, N, K, x3, monkeypatch):
    from helpers import gemm_plan
    monkeypatch.delenv("SIGMA_GEMM_BN", raising=False)
    pl = gemm_plan(M, N, K, x3)
    _check_plan(pl, x3)
    mt = -(-M // 128)
    assert pl["bn"] == L.sigma_test_pick_bn(N, mt)                        # the plan's width is the heuristic's
    assert pl["tiles"] == mt * -(-N // pl["bn"])
    for bn in range(32, 257, 32):
        monkeypatch.setenv("SIGMA_GEMM_BN", str(bn))
        pl = gemm_plan(M, N, K, x3)
        assert pl["bn"] == bn and pl["tiles"] == mt * -(-N // bn)
        _check_plan(pl, x3)


@pytest.mark.parametrize("x3", [False, True])
@pytest.mark.parametrize("B,H,W,Cin,Cout", CONV_SHAPES)
def test_conv_plan_is_launchable(L, B, H, W, Cin, Cout, x3, monkeypatch):
    from helpers import gemm_plan
    monkeypatch.delenv("SIGMA_GEMM_BN", raising=False)
    patches = B * -(-H // 8) * -(-W // 16)                                  # 8 x 16 pixel patches
    for bn in [None] + list(range(32, 257, 32)):
        if bn is not None:
            monkeypatch.setenv("SIGMA_GEMM_BN", str(bn))
        pl = gemm_plan(0, Cout, Cin, x3, conv=(B, H, W))
        _check_plan(pl, x3)
        assert pl["bn"] == (bn or L.sigma_test_pick_bn(Cout, 1 << 30))
        assert pl["tiles"] == patches * -(-Cout // pl["bn"])


@pytest.mark.parametrize("value", ["0", "16", "48", "257", "288", "-32", "64x", "wide"])
def test_forced_tile_width_rejects_bad_values(L, value, monkeypatch):
    """SIGMA_GEMM_BN takes a multiple of 32 in [32, 256]; anything else is an error with a message, never a silent clamp."""
    import ctypes
    from sigma_b200 import _lib
    monkeypatch.setenv("SIGMA_GEMM_BN", value)
    out = (ctypes.c_int64 * 6)()
    for conv in [(0, 0, 0), (2, 30, 40)]:
        rc = L.sigma_test_gemm_plan(1000, 768, 192, 1, *conv, out)
        assert rc == -1                                                     # SIGMA_EINVAL
        assert "SIGMA_GEMM_BN" in _lib.lib().sigma_last_error().decode()
    monkeypatch.delenv("SIGMA_GEMM_BN")
    assert L.sigma_test_gemm_plan(1000, 768, 192, 1, 0, 0, 0, out) == 0



# ---- the L-segment plan of the fused scan backward (sigma_test_ss2d_bwd_plan = the planner sigma_ss2d_scan_bwd* launch with) ----
# Sigma's training shapes: (kind, H, W, D, d_state) — encoder SS2D stages of tiny / small (D 192..1536) and base (45 x 60, 23 x 30),
# ConMB (SEQ2, d_state 4) and the decoder's SS2D (d_state 4)
BWD_SHAPES = [("cross4", 120, 160, 192, 16), ("cross4", 60, 80, 384, 16), ("cross4", 30, 40, 768, 16), ("cross4", 15, 20, 1536, 16),
              ("cross4", 45, 60, 1024, 16), ("cross4", 23, 30, 2048, 16), ("seq2", 120, 160, 192, 4), ("seq2", 60, 80, 384, 4),
              ("seq2", 30, 40, 768, 4), ("seq2", 15, 20, 1536, 4), ("seq2", 23, 30, 2048, 4), ("cross4", 120, 160, 192, 4),
              ("cross4", 60, 80, 384, 4), ("cross4", 30, 40, 768, 4)]


def ss2d_bwd_plan(kind, B, H, W, D, N, nsplit=0):
    import ctypes
    from sigma_b200 import _lib
    out = (ctypes.c_int64 * 4)()
    k = _lib.DIRS_CROSS4 if kind == "cross4" else _lib.DIRS_SEQ2
    _lib.check(_lib.lib().sigma_test_ss2d_bwd_plan(k, B, H, W, D, N, nsplit, out), "sigma_test_ss2d_bwd_plan")
    return dict(zip(("nsplit", "tiles_per_split", "max_tiles", "min_tiles"), (int(v) for v in out)))


@pytest.mark.parametrize("kind,H,W,D,N", BWD_SHAPES)
@pytest.mark.parametrize("B", [1, 2, 3, 8])
def test_ss2d_bwd_plan_invariants(L, kind, H, W, D, N, B):
    rows = -(-H * W * (2 if kind == "seq2" else 1) // 16)
    for force in [0, 1, 2, 7, 20, 64, 100]:
        pl = ss2d_bwd_plan(kind, B, H, W, D, N, force)
        assert pl["max_tiles"] == (max(rows, W * -(-H // 16)) if kind == "cross4" else rows)
        assert pl["min_tiles"] == (min(rows, W * -(-H // 16)) if kind == "cross4" else rows)
        assert 1 <= pl["nsplit"] <= 64
        assert pl["tiles_per_split"] * pl["nsplit"] >= pl["max_tiles"]                 # every tile of the longest walk is covered
        assert (pl["nsplit"] - 1) * pl["tiles_per_split"] < pl["max_tiles"]             # and none of its segments is empty
        if force:
            assert pl["nsplit"] <= min(force, 64)


def test_ss2d_bwd_plan_rejects_bad_arguments(L):
    import ctypes
    out = (ctypes.c_int64 * 4)()
    assert L.sigma_test_ss2d_bwd_plan(2, 1, 15, 20, 1536, 4, 0, out) != 0            # CROSS has no fused backward
    assert L.sigma_test_ss2d_bwd_plan(0, 1, 15, 20, 96, 16, 0, out) != 0              # D % 64
    assert L.sigma_test_ss2d_bwd_plan(0, 1, 15, 20, 1536, 8, 0, out) != 0             # d_state
    assert L.sigma_test_ss2d_bwd_plan(0, 1, 15, 20, 1536, 16, -1, out) != 0


# ---- the launch plan of the fused scan forward (sigma_test_ss2d_fwd_plan = the planner sigma_ss2d_scan_fwd* launch with) ----
# Sigma's inference shapes: (kind, H, W, D, d_state, dt_rank) — the SS2D blocks of tiny / small (D 192..1536) and base (45 x 60,
# 23 x 30), CroMB (CROSS) and ConMB (SEQ2) at d_state 4, and the decoder's SS2D (d_state 4)
FWD_SHAPES = ([("cross4", 120, 160, 192, 16, 6), ("cross4", 60, 80, 384, 16, 12), ("cross4", 30, 40, 768, 16, 24),
               ("cross4", 15, 20, 1536, 16, 48), ("cross4", 45, 60, 1024, 16, 32), ("cross4", 23, 30, 2048, 16, 64)]
              + [(k, H, W, D, 4, R) for k in ("cross", "seq2")
                 for H, W, D, R in [(120, 160, 192, 6), (60, 80, 384, 12), (30, 40, 768, 24), (15, 20, 1536, 48), (23, 30, 2048, 64)]]
              + [("cross4", 120, 160, 192, 4, 6), ("cross4", 60, 80, 384, 4, 12), ("cross4", 30, 40, 768, 4, 24)])
SCAN_ENV = ("SIGMA_SCAN_WARPS", "SIGMA_SCAN_NST", "SIGMA_SCAN_CTAS", "SIGMA_SCAN_SPLIT_RULE")


def _reg_cap(ctas):
    return (65536 // (ctas * 128)) // 8 * 8                                  # ss2d_reg_cap (ss2d_scan.cuh)


def _walk_tiles(kind, H, W, N):
    lt = 16 if N >= 16 else 32
    rows = -(-H * W * (2 if kind == "seq2" else 1) // lt)
    return (max(rows, W * -(-H // lt)), min(rows, W * -(-H // lt))) if kind == "cross4" else (rows, rows)


def _check_fwd_plan(pl, kind, H, W, D, N, R, bf16):
    from sigma_b200 import _lib
    assert (pl["max_tiles"], pl["min_tiles"]) == _walk_tiles(kind, H, W, N)
    assert 1 <= pl["nsplit"] <= min(32, pl["max_tiles"])
    assert pl["tiles_per_split"] == -(-pl["max_tiles"] // pl["nsplit"])
    assert 1 <= pl["warps"] <= 4 and 2 <= pl["nst"] <= 8
    assert pl["ctas"] in (3, 4)
    lt = 16 if N >= 16 else 32
    stage = lt * 32 * pl["warps"] * (2 if bf16 else 4) + lt * _lib.lib().sigma_ss2d_padded_cp(N, R) * 4 * (2 if kind == "cross" else 1)
    assert pl["smem"] == pl["nst"] * stage + 128
    assert pl["smem"] <= SMEM_PER_BLOCK
    return stage


@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("kind,H,W,D,N,R", FWD_SHAPES)
@pytest.mark.parametrize("images", [1, 2, 8, 74])
def test_ss2d_fwd_plan_invariants(L, kind, H, W, D, N, R, images, bf16, monkeypatch):
    from helpers import ss2d_fwd_plan
    for e in SCAN_ENV:
        monkeypatch.delenv(e, raising=False)
    B = 2 * images if kind == "cross" else images
    auto = ss2d_fwd_plan(kind, B, H, W, D, N, R, bf16)
    _check_fwd_plan(auto, kind, H, W, D, N, R, bf16)
    assert (auto["nsplit"] - 1) * auto["tiles_per_split"] < auto["max_tiles"]      # no segment of the longest walk is empty
    # the register budget: 4 CTAs (128 registers) only for d_state 16 at padded dt_rank 24, and only in fp32
    assert auto["ctas"] == (4 if N == 16 and L.sigma_ss2d_padded_cp(N, R) == 2 * N + 24 and not bf16 else 3)
    # the ring fits the shared memory of the CTAs the register budget puts on an SM together
    ctas_sm = max(auto["ctas"], min(16, 65536 // (32 * auto["warps"] * _reg_cap(auto["ctas"]))))
    assert ctas_sm * (auto["smem"] + 1024) <= SMEM_PER_SM
    capped = ss2d_fwd_plan(kind, B, H, W, D, N, R, bf16, force=100)
    _check_fwd_plan(capped, kind, H, W, D, N, R, bf16)
    assert capped["nsplit"] == min(32, capped["max_tiles"])                        # 100 is capped at 32 segments
    for force in (1, 2, 7, 8, 20):
        pl = ss2d_fwd_plan(kind, B, H, W, D, N, R, bf16, force=force)
        _check_fwd_plan(pl, kind, H, W, D, N, R, bf16)
        assert pl["nsplit"] == min(force, pl["max_tiles"])                         # a forced count is kept, even if segments end empty
        assert {k: pl[k] for k in ("warps", "nst", "ctas", "smem")} == {k: auto[k] for k in ("warps", "nst", "ctas", "smem")}
    # without a workspace: one segment, and a forced count above 1 is an error
    assert ss2d_fwd_plan(kind, B, H, W, D, N, R, bf16, ws_bytes=0)["nsplit"] == 1
    assert ss2d_fwd_plan(kind, B, H, W, D, N, R, bf16, force=1, ws_bytes=0)["nsplit"] == 1
    import ctypes
    from helpers import ss2d_kind
    out = (ctypes.c_int64 * 8)()
    assert L.sigma_test_ss2d_fwd_plan(ss2d_kind(kind), B, H, W, D, N, R, int(bf16), 2, 0, out) == -3   # SIGMA_EWORKSPACE


@pytest.mark.parametrize("kind", ["cross4", "seq2", "cross"])
def test_ss2d_fwd_split_without_workspace_is_an_error(L, kind):
    """sigma_ss2d_scan_fwd_split with more than one forced segment and no workspace returns SIGMA_EWORKSPACE before it touches the
    device (the plan comes first), so the pointers here are never dereferenced"""
    import ctypes
    from sigma_b200 import _lib
    from helpers import ss2d_kind
    fake = ctypes.c_void_p(1 << 20)                                                # non-null and 16-byte aligned, never read
    rc = L.sigma_ss2d_scan_fwd_split(ss2d_kind(kind), *[fake] * 7, 2, 30, 40, 384, 4, 12, L.sigma_ss2d_padded_cp(4, 12), None, 0, 3,
                                     None)
    assert rc == -3, rc                                                            # SIGMA_EWORKSPACE
    assert "workspace" in _lib.lib().sigma_last_error().decode()


def test_ss2d_fwd_plan_honours_the_environment(L, monkeypatch):
    from helpers import ss2d_fwd_plan
    for e in SCAN_ENV:
        monkeypatch.delenv(e, raising=False)
    shape = ("cross4", 1, 30, 40, 768, 16, 24)
    assert ss2d_fwd_plan(*shape)["warps"] == 4 and ss2d_fwd_plan(*shape)["ctas"] == 4
    for w in (1, 2, 3, 4):
        monkeypatch.setenv("SIGMA_SCAN_WARPS", str(w))
        # SIGMA_SCAN_WARPS caps the width; pick_warps tries 4, 2, 3, 1 warps for one that divides D
        assert ss2d_fwd_plan(*shape)["warps"] == next(x for x in (4, 2, 3, 1) if x <= w and 768 % (32 * x) == 0)
    monkeypatch.delenv("SIGMA_SCAN_WARPS")
    for n in (2, 8):
        monkeypatch.setenv("SIGMA_SCAN_NST", str(n))
        assert ss2d_fwd_plan(*shape)["nst"] == n
    monkeypatch.delenv("SIGMA_SCAN_NST")
    for c in (3, 4):
        monkeypatch.setenv("SIGMA_SCAN_CTAS", str(c))
        assert ss2d_fwd_plan(*shape)["ctas"] == c
        assert ss2d_fwd_plan("cross4", 1, 30, 40, 768, 16, 24, bf16=True)["ctas"] == 3        # bf16 builds one budget
        assert ss2d_fwd_plan("cross4", 1, 30, 40, 768, 4, 24)["ctas"] == 3                    # d_state 4 builds one budget
    # ragged D: enough warps to cover it, the last CTA partly filled
    monkeypatch.delenv("SIGMA_SCAN_CTAS")
    assert ss2d_fwd_plan("cross4", 1, 30, 40, 100, 16, 6)["warps"] == 4
    assert ss2d_fwd_plan("cross4", 1, 30, 40, 132, 16, 6)["warps"] == 4


def test_ss2d_fwd_plan_rejects_bad_arguments(L):
    import ctypes
    out = (ctypes.c_int64 * 8)()
    assert L.sigma_test_ss2d_fwd_plan(2, 3, 15, 20, 1536, 4, 48, 0, 0, 1 << 30, out) != 0      # CROSS: batch = 2·images
    assert L.sigma_test_ss2d_fwd_plan(0, 1, 15, 20, 100, 4, 48, 1, 0, 1 << 30, out) != 0       # bf16: D % 8
    assert L.sigma_test_ss2d_fwd_plan(0, 1, 15, 20, 1536, 12, 48, 0, 0, 1 << 30, out) != 0     # d_state
    assert L.sigma_test_ss2d_fwd_plan(0, 1, 15, 20, 1536, 16, 65, 0, 0, 1 << 30, out) != 0     # dt_rank
    assert L.sigma_test_ss2d_fwd_plan(0, 1, 15, 20, 1536, 16, 48, 0, -1, 1 << 30, out) != 0


# ---- the op-level selective scan's launch plan (sigma_test_scan_plan): the routes, the 64-segment cap on every route, the
# segments covering the tiles, and the backward's two sweeps.  (batch, dim, L, N, G) of Sigma's calls and a few ragged ones.
OP_SHAPES = [(2, 192, 19200, 4, 1), (2, 384, 4800, 4, 1), (2, 768, 1200, 4, 1), (2, 1536, 300, 4, 1), (1, 256, 43200, 4, 1),
             (1, 2048, 690, 4, 1), (2, 768, 19200, 16, 4), (2, 6144, 300, 16, 4), (2, 384, 38400, 4, 2), (3, 64, 1001, 8, 2),
             (1, 96, 77, 16, 1), (2, 40, 500, 4, 1)]


def test_op_scan_plan_routes(monkeypatch):
    import torch
    from helpers import scan_plan
    monkeypatch.delenv("SIGMA_OP_GENERIC", raising=False)
    for sweep in ("fwd", "bwd", "bwd_det"):
        assert scan_plan(sweep, 1, 2048, 690, 4, 1)["route"] == "generic"                  # fp32 rows of 690 are not 16-byte aligned
        for dt in (torch.float16, torch.bfloat16):
            assert scan_plan(sweep, 2, 1536, 300, 4, 1, dt)["route"] == "widened"            # 16-bit rows of 300: fp32 copies are
            assert scan_plan(sweep, 2, 192, 19200, 4, 1, dt)["route"] == "tma"
            assert scan_plan(sweep, 1, 2048, 690, 4, 1, dt)["route"] == "generic"
        assert scan_plan(sweep, 2, 768, 19200, 16, 4)["route"] == "tma"
        assert scan_plan(sweep, 2, 40, 500, 4, 1)["route"] == "generic"                     # channel groups not a multiple of 32
    assert scan_plan("fwd", 2, 1536, 300, 4, 1, torch.bfloat16, ws_bytes=0)["route"] == "generic"   # widening needs scratch
    monkeypatch.setenv("SIGMA_OP_GENERIC", "1")
    for sweep in ("fwd", "bwd"):
        assert scan_plan(sweep, 2, 192, 19200, 4, 1)["route"] == "generic"
    p = scan_plan("fwd", 2, 192, 19200, 4, 1, nsplit=100)                                     # the generic forward's cap
    assert p["nsplit"] <= 64 and p["tiles_per_split"] == -(-p["ntiles"] // 64) == 10, p


def test_op_scan_plan_segments(monkeypatch):
    import torch
    from helpers import scan_plan
    for generic in ("0", "1"):
        monkeypatch.setenv("SIGMA_OP_GENERIC", generic)
        for shape in OP_SHAPES:
            for dt in (torch.float32, torch.bfloat16):
                for sweep in ("fwd", "bwd", "bwd_det"):
                    if sweep != "fwd" and shape[3] > 16:
                        continue
                    for ns in (0, 1, 2, 7, 64, 100):
                        p = scan_plan(sweep, *shape, dt, nsplit=ns)
                        what = (generic, shape, dt, sweep, ns, p)
                        assert 1 <= p["nsplit"] <= 64, what
                        assert p["nsplit"] * p["tiles_per_split"] >= p["ntiles"] > (p["nsplit"] - 1) * p["tiles_per_split"], what
                        seg = not (sweep != "fwd" and p["route"] == "generic")
                        if ns == 1 or not seg:
                            assert p["nsplit"] == 1, what                                    # the generic backward has no segments
                        if ns == 100 and seg:
                            assert p["tiles_per_split"] == -(-p["ntiles"] // 64), what
                        if sweep == "fwd":
                            assert p["state_nsplit"] == 0, what
                            continue
                        # the state sweep: the forward planner with the same forced count (its own choice at nsplit = 0)
                        assert 1 <= p["state_nsplit"] <= 64, what
                        if not seg:
                            assert p["state_nsplit"] == 1, what
                        elif ns:
                            f = scan_plan("fwd", *shape, dt if p["route"] == "tma" else torch.float32, nsplit=ns, ws_bytes=1 << 40)
                            assert (p["state_nsplit"], p["state_tiles_per_split"]) == (f["nsplit"], f["tiles_per_split"]), what
    monkeypatch.delenv("SIGMA_OP_GENERIC")
    # no workspace: one segment whatever is asked; a backward without its workspace is refused as the launch would be
    assert scan_plan("fwd", 2, 192, 19200, 4, 1, nsplit=7, ws_bytes=0)["nsplit"] == 1
    with pytest.raises(RuntimeError):
        scan_plan("bwd", 2, 192, 19200, 4, 1, ws_bytes=0)
    # the drop-in CroMB stage-0 call runs L-segments by default, forward and backward
    assert scan_plan("fwd", 2, 192, 19200, 4, 1)["nsplit"] > 1 and scan_plan("bwd", 2, 192, 19200, 4, 1)["nsplit"] > 1


# CroMB's training shapes (one block per encoder stage; d_inner = 2·C): Sigma-tiny / small at 480 x 640 and Sigma-base at 720 x 960
CROMB = [(120, 160, 192, 6), (60, 80, 384, 12), (30, 40, 768, 24), (15, 20, 1536, 48), (180, 240, 256, 8), (23, 30, 2048, 64)]


def _lib():
    from sigma_b200 import _lib
    return _lib


@pytest.mark.parametrize("H,W,D,R", CROMB)
@pytest.mark.parametrize("images", [1, 2, 3, 8])
def test_cross_backward_plan_and_sizes(H, W, D, R, images):
    L_, lib = _lib().lib(), _lib()
    Bt, N, L = 2 * images, 4, H * W
    tiles = -(-L // 16)
    for force in (0, 1, 2, 7, 64, 100):
        out = (ctypes.c_int64 * 4)()
        lib.check(L_.sigma_test_ss2d_bwd_plan(lib.DIRS_CROSS, Bt, H, W, D, N, force, out), "sigma_test_ss2d_bwd_plan")
        nsplit, tps, mx, mn = (int(v) for v in out)
        assert mx == mn == tiles                                          # one row-major walk of ceil(L / 16) tiles
        assert 1 <= nsplit <= 64 and nsplit * tps >= tiles and (nsplit - 1) * tps < tiles, (force, nsplit, tps)
        if force:
            assert nsplit == len(range(0, tiles, -(-tiles // min(force, 64, tiles))))
    hsb = L_.sigma_ss2d_scan_hs_bytes(lib.DIRS_CROSS, Bt, H, W, D, N)
    assert hsb == Bt * tiles * D * N * 4
    for kind, K in ((lib.DIRS_CROSS, 1), (lib.DIRS_CROSS4, 4), (lib.DIRS_SEQ2, 2)):   # the reverse carries of 64 segments, no more
        assert L_.sigma_ss2d_scan_bwd_workspace_bytes(kind, Bt, H, W, D, N) == -(-Bt * K * D * 64 * 2 * N * 4 // 256) * 256
    assert L_.sigma_ss2d_scan_bwd_det_workspace_bytes(lib.DIRS_CROSS, Bt, H, W, D, N) == 0     # no deterministic build


def test_cross_backward_rejects_an_odd_batch():
    L_, lib = _lib().lib(), _lib()
    out = (ctypes.c_int64 * 4)()
    assert L_.sigma_test_ss2d_bwd_plan(lib.DIRS_CROSS, 3, 30, 40, 768, 4, 0, out) != 0
    assert L_.sigma_test_ss2d_bwd_plan(lib.DIRS_CROSS, 4, 30, 40, 768, 4, 0, out) == 0
    assert L_.sigma_ss2d_scan_hs_bytes(lib.DIRS_CROSS, 3, 30, 40, 768, 4) == 0
    assert L_.sigma_ss2d_scan_bwd_workspace_bytes(lib.DIRS_CROSS, 3, 30, 40, 768, 4) == 0
