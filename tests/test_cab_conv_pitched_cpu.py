"""CPU: the pitched 3x3 conv entry points (the ChannelAttentionBlock convs of Sigma-base, whose C/3 is 42 / 85 / 170), as far as
they go without a device.
* the header declares the four entry points and `_lib` binds them: one pitch (int) after each activation and weight;
* argument validation returns its codes before any CUDA call: null pointers, sizes, pitches below the count or not multiples of 4,
  16-byte alignment, the workspace; the unpitched entry points still refuse counts that are not multiples of 4;
* the launch plans at Sigma-base's decoder stages: the weight gradient's (one wave, the workspace query of the unpitched call) and
  the inference conv's tile widths;
* `cuobjdump -sass` of the built library: the pitched conv's 32 instances run wgmma (GMMA), the pitched weight gradient's 4 run
  mma.sync (HMMA) and hold no float atomic and no bulk-tensor reduce."""
import ctypes

import pytest
import torch

from test_cab_conv_train_cpu import sass  # noqa: F401  (the module's cuobjdump fixture)
from test_deterministic_sass_cpu import FLOAT_ATOMIC

NEW = ("sigma_conv3x3_pitched_tf32", "sigma_conv3x3_gelu_save_pitched_tf32", "sigma_conv3x3_dgrad_pitched_tf32",
       "sigma_conv3x3_wgrad_pitched_tf32")
CONV = [f"_ZN5sigma23cab_conv_pitched_kernelILi{bn}ELb{x3}ELi{e}EEEvNS_10GemmParamsE" for x3 in (0, 1)
        for e, widths in ((0, range(32, 257, 32)), (1, range(32, 129, 32)), (2, range(32, 129, 32))) for bn in widths]
WGRAD = [f"_ZN5sigma24cab_wgrad_pitched_kernelILi{co}ELb{x3}EEEvNS_11WgradParamsE" for co in (32, 64) for x3 in (0, 1)]
EINVAL, EWORKSPACE = -1, -3

# (B, H, W, C) of Sigma-base's decoder stages at 720 x 960, batch 1, and at 480 x 640, batch 2; the convs map C -> C // 3 -> C
BASE_STAGES = [(1, 180, 240, 128), (1, 90, 120, 256), (1, 45, 60, 512), (2, 120, 160, 128), (2, 60, 80, 256), (2, 30, 40, 512)]


def test_header_declares_and_lib_binds_the_pitched_entry_points():
    from sigma_b200 import _lib
    L = _lib.lib()
    I, P, Z = ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t
    for name in NEW:
        assert name in _lib.SIGNATURES, name
        assert getattr(L, name).argtypes == _lib.SIGNATURES[name][1]
        assert _lib.SIGNATURES[name][0] is I
    sig = {n: _lib.SIGNATURES[n][1] for n in NEW}
    assert sig["sigma_conv3x3_pitched_tf32"] == [P, I, P, I, P, P, I, P, I] + [I] * 5 + [P]
    assert sig["sigma_conv3x3_gelu_save_pitched_tf32"] == [P, I, P, I, P, P, P, P, I] + [I] * 5 + [P]
    assert sig["sigma_conv3x3_dgrad_pitched_tf32"] == [P, I, P, I, P, P, P, I] + [I] * 5 + [P]
    assert sig["sigma_conv3x3_wgrad_pitched_tf32"] == [P, I, I, P, I, P, P] + [I] * 6 + [P, Z, P]


def test_argument_validation_needs_no_device():
    from sigma_b200 import _lib
    L = _lib.lib()
    buf = torch.zeros(64, dtype=torch.float32)
    p = ctypes.c_void_p(buf.data_ptr())                       # a non-null, 16-byte aligned host pointer: never dereferenced
    p4 = ctypes.c_void_p(buf.data_ptr() + 4)
    B, H, W, C, C1 = 1, 9, 17, 128, 42
    err = lambda: L.sigma_last_error().decode()              # noqa: E731

    def conv(x=p, xp=C, w=p, wp=C, wlo=None, bias=p, act=1, y=p, yp=44, sizes=(B, H, W), cin=C, cout=C1):
        return L.sigma_conv3x3_pitched_tf32(x, xp, w, wp, wlo, bias, act, y, yp, *sizes, cin, cout, None)

    def save(x=p, xp=C, w=p, wp=C, wlo=None, bias=p, y=p, pre=p, yp=44, sizes=(B, H, W), cin=C, cout=C1):
        return L.sigma_conv3x3_gelu_save_pitched_tf32(x, xp, w, wp, wlo, bias, y, pre, yp, *sizes, cin, cout, None)

    def dgrad(dy=p, dyp=C, w=p, wp=C, wlo=None, aux=p, dx=p, dxp=44, sizes=(B, H, W), cin=C1, cout=C):
        return L.sigma_conv3x3_dgrad_pitched_tf32(dy, dyp, w, wp, wlo, aux, dx, dxp, *sizes, cin, cout, None)

    for fn, ptrs, opt, pitches in ((conv, ("x", "w", "y"), ("wlo", "bias"), ("xp", "wp", "yp")),
                                   (save, ("x", "w", "y", "pre"), ("wlo", "bias"), ("xp", "wp", "yp")),
                                   (dgrad, ("dy", "w", "dx"), ("wlo", "aux"), ("dyp", "wp", "dxp"))):
        for k in ptrs:
            assert fn(**{k: None}) == EINVAL, (fn.__name__, k)
            assert "null pointer" in err()
        for sizes in ((-1, H, W), (B, 0, W), (B, H, 0)):
            assert fn(sizes=sizes) == EINVAL, (fn.__name__, sizes)
        assert fn(cin=0) == EINVAL and fn(cout=0) == EINVAL
        for k in pitches:                                      # below the count (C = 128, C1 = 42) or not a multiple of 4
            for bad in ((40, 42, 46) if k in ("yp", "dxp") else (0, 124, 126, 130)):
                assert fn(**{k: bad}) == EINVAL, (fn.__name__, k, bad)
                assert "pitches" in err()
        for k in ptrs + opt:
            assert fn(**{k: p4}) == EINVAL, (fn.__name__, k)
            assert "16-byte aligned" in err()
    assert conv(act=2) == EINVAL
    # an odd count at a pitch of round4(count), and any larger multiple of 4, gets past the checks: the call then returns at
    # batch 0 before any CUDA call
    assert conv(sizes=(0, H, W), cout=43, yp=44) == 0 and conv(sizes=(0, H, W), cout=1, yp=64) == 0
    assert save(sizes=(0, H, W), cout=85, yp=88) == 0 and dgrad(sizes=(0, H, W), cin=170, dxp=172) == 0

    wsb = L.sigma_conv3x3_wgrad_workspace_bytes(B, H, W, C, C1)
    assert wsb > 0 and wsb % 256 == 0

    def wgrad(x=p, xp=C, gelu_x=0, dy=p, dyp=44, dw=p, db=p, sizes=(B, H, W), cin=C, cout=C1, x3=0, ws=p, n=wsb):
        return L.sigma_conv3x3_wgrad_pitched_tf32(x, xp, gelu_x, dy, dyp, dw, db, *sizes, cin, cout, x3, ws, n, None)

    for k in ("x", "dy", "dw"):
        assert wgrad(**{k: None}) == EINVAL, k
        assert "null pointer" in err()
    for sizes in ((0, H, W), (B, 0, W), (B, H, 0)):
        assert wgrad(sizes=sizes) == EINVAL, sizes
    for kw in ({"xp": 126}, {"xp": 130}, {"dyp": 40}, {"dyp": 42}, {"dyp": 45}):
        assert wgrad(**kw) == EINVAL, kw
        assert "pitches" in err()
    assert wgrad(gelu_x=2) == EINVAL and wgrad(x3=-1) == EINVAL
    for k in ("x", "dy"):
        assert wgrad(**{k: p4}) == EINVAL, k
        assert "16-byte aligned" in err()
    assert wgrad(ws=None) == EWORKSPACE and wgrad(n=wsb - 1) == EWORKSPACE and wgrad(ws=p4) == EWORKSPACE
    assert "workspace" in err()
    assert wgrad(db=None, ws=None) == EWORKSPACE              # db is optional
    # the unpitched weight gradient keeps its rule
    assert L.sigma_conv3x3_wgrad_tf32(p, 0, p, p, p, B, H, W, C, C1, 0, p, wsb, None) == EINVAL
    assert "multiples of 4" in err()


def _wgrad_plan(*shape):
    from sigma_b200 import _lib
    out = (ctypes.c_int64 * 4)()
    assert _lib.lib().sigma_test_conv3x3_wgrad_plan(*shape, out) == 0
    return list(out)


def _conv_plan(B, H, W, cin, cout, x3):
    from sigma_b200 import _lib
    out = (ctypes.c_int64 * 6)()
    assert _lib.lib().sigma_test_gemm_plan(0, cout, cin, int(x3), B, H, W, out) == 0
    return list(out)


@pytest.mark.parametrize("B,H,W,C", BASE_STAGES)
@pytest.mark.parametrize("first", [True, False], ids=["conv1", "conv2"])
def test_plans_at_sigma_base_stages(B, H, W, C, first):
    from sigma_b200 import _lib
    C1 = C // 3
    cin, cout = (C, C1) if first else (C1, C)
    co, tiles, nsplit, ctas = _wgrad_plan(B, H, W, cin, cout)
    assert co == (64 if cout % 64 == 0 else 32)
    assert tiles == -(-cin // 32) * -(-cout // co) and ctas == tiles * nsplit and 132 - tiles < ctas <= 132
    wsb = _lib.lib().sigma_conv3x3_wgrad_workspace_bytes(B, H, W, cin, cout)
    assert wsb >= nsplit * (9 * cin + 1) * cout * 4 and wsb % 256 == 0
    # the inference conv (sigma_conv3x3_pitched_tf32 at EPI 0 plans as sigma_conv3x3_tf32): one tile spans C/3, and C = 512
    # takes the 256-wide instance
    for x3 in (False, True):
        bn = _conv_plan(B, H, W, cin, cout, x3)[0]
        assert bn == {42: 64, 85: 96, 170: 192, 128: 128, 256: 256, 512: 256}[cout], (cout, bn)


def test_pitched_kernels_run_on_the_tensor_cores_and_the_wgrad_holds_no_float_atomics(sass):  # noqa: F811
    assert sorted(n for n in sass if "cab_conv_pitched" in n) == sorted(CONV)
    assert sorted(n for n in sass if "cab_wgrad_pitched" in n) == sorted(WGRAD)
    for name in CONV:
        assert any("HGMMA" in l for l in sass[name]), name
    for name in WGRAD:
        assert any("HMMA" in l for l in sass[name]), name
        bad = [l.strip() for l in sass[name] if FLOAT_ATOMIC.search(l)]
        assert not bad, (name, bad[:3])
