"""CPU: the training kernels of the ChannelAttentionBlock's 3x3 convs, as far as they go without a device.
* the header declares the new entry points and `_lib` binds them; the data gradient and the saving forward take the plain conv's
  arguments in its order;
* the weight gradient's workspace query (0 for empty shapes) and its launch plan at Sigma's decoder shapes: one wave of CTAs that
  leaves fewer SMs idle than one CTA per output tile would fill, a plan that depends on the shape alone (the same with the
  deterministic switch on);
* argument validation returns its codes before any CUDA call: null pointers, channel counts, 16-byte alignment, the workspace;
* `cuobjdump -sass` of the built library: the new kernels exist, the weight gradient and the partial-sum kernel hold no float atomic
  and no bulk-tensor reduce, and the inference conv's instances keep their names."""
import ctypes
import re
import subprocess

import pytest
import torch

from test_deterministic_sass_cpu import FLOAT_ATOMIC

NEW = ("sigma_conv3x3_gelu_save_tf32", "sigma_conv3x3_dgrad_tf32", "sigma_conv3x3_wgrad_tf32", "sigma_conv3x3_wgrad_workspace_bytes",
       "sigma_test_conv3x3_wgrad_plan")
WGRAD = [f"_ZN5sigma20conv3x3_wgrad_kernelILi{co}ELb{x3}EEEvNS_11WgradParamsE" for co in (32, 64) for x3 in (0, 1)]
EPI = [f"_ZN5sigma18conv3x3_epi_kernelILi{bn}ELb{x3}ELi{e}EEEvNS_10GemmParamsE" for bn in (32, 64, 96, 128) for x3 in (0, 1)
       for e in (1, 2)]
CONV = [f"_ZN5sigma16gemm_tf32_kernelILi{bn}ELb{x3}ELb1ELb0EEEvNS_10GemmParamsE" for bn in range(32, 257, 32) for x3 in (0, 1)]
SUM = "_ZN5sigma20sum_parts_det_kernelEPKfixxxPf"
EINVAL, EWORKSPACE = -1, -3

# (B, H, W, C) of every Sigma-tiny / Sigma-small decoder stage at 480 x 640, batch 2; both convs: C -> C/3 and C/3 -> C
SIGMA_STAGES = [(2, 120, 160, 96), (2, 60, 80, 192), (2, 30, 40, 384)]


def test_header_declares_and_lib_binds_the_new_entry_points():
    from sigma_b200 import _lib
    L = _lib.lib()
    for name in NEW:
        assert name in _lib.SIGNATURES, name
        assert getattr(L, name).argtypes == _lib.SIGNATURES[name][1]
    assert _lib.SIGNATURES["sigma_conv3x3_dgrad_tf32"] == _lib.SIGNATURES["sigma_conv3x3_tf32"][:1] + (
        _lib.SIGNATURES["sigma_conv3x3_tf32"][1][:4] + _lib.SIGNATURES["sigma_conv3x3_tf32"][1][5:],)
    assert _lib.SIGNATURES["sigma_conv3x3_wgrad_workspace_bytes"] == (ctypes.c_size_t, [ctypes.c_int] * 5)


def _plan(*shape):
    from sigma_b200 import _lib
    out = (ctypes.c_int64 * 4)()
    assert _lib.lib().sigma_test_conv3x3_wgrad_plan(*shape, out) == 0
    return list(out)


@pytest.mark.parametrize("B,H,W,C", SIGMA_STAGES)
@pytest.mark.parametrize("first", [True, False], ids=["conv1", "conv2"])
def test_wgrad_plan_fills_the_sms_in_one_wave_and_ignores_the_deterministic_switch(B, H, W, C, first):
    from sigma_b200 import _lib
    cin, cout = (C, C // 3) if first else (C // 3, C)
    plan = _plan(B, H, W, cin, cout)
    co, tiles, nsplit, ctas = plan
    assert co == (64 if cout % 64 == 0 else 32)
    assert tiles == -(-cin // 32) * -(-cout // co) and ctas == tiles * nsplit and 132 - tiles < ctas <= 132
    npatch = B * -(-H // 8) * -(-W // 16)
    assert 1 <= nsplit <= npatch
    wsb = _lib.lib().sigma_conv3x3_wgrad_workspace_bytes(B, H, W, cin, cout)
    assert wsb >= nsplit * (9 * cin + 1) * cout * 4 and wsb % 256 == 0
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        assert _plan(B, H, W, cin, cout) == plan
        assert _lib.lib().sigma_conv3x3_wgrad_workspace_bytes(B, H, W, cin, cout) == wsb
    finally:
        torch.use_deterministic_algorithms(prev)


def test_wgrad_plan_of_small_and_ragged_shapes():
    assert _plan(1, 1, 1, 4, 4) == [32, 1, 1, 1]             # one patch: one range
    co, tiles, nsplit, _ = _plan(1, 45, 80, 36, 12)           # ragged H, channel counts that are not multiples of 32
    assert co == 32 and tiles == 2 and nsplit == 30        # ranges capped at the 6 x 5 patches


def test_argument_validation_needs_no_device():
    from sigma_b200 import _lib
    L = _lib.lib()
    buf = torch.zeros(64, dtype=torch.float32)
    p = ctypes.c_void_p(buf.data_ptr())                       # a non-null, 16-byte aligned host pointer: never dereferenced
    p4 = ctypes.c_void_p(buf.data_ptr() + 4)
    B, H, W, Cin, Cout = 2, 9, 17, 64, 32
    wsb = L.sigma_conv3x3_wgrad_workspace_bytes(B, H, W, Cin, Cout)
    assert wsb > 0 and wsb % 256 == 0
    for shape in ((0, H, W, Cin, Cout), (B, 0, W, Cin, Cout), (B, H, 0, Cin, Cout), (B, H, W, 0, Cout), (B, H, W, Cin, 0)):
        assert L.sigma_conv3x3_wgrad_workspace_bytes(*shape) == 0, shape

    def wgrad(x=p, dy=p, dw=p, db=p, cin=Cin, cout=Cout, gelu_x=0, x3=0, ws=p, n=wsb, sizes=(B, H, W)):
        return L.sigma_conv3x3_wgrad_tf32(x, gelu_x, dy, dw, db, *sizes, cin, cout, x3, ws, n, None)

    for k in ("x", "dy", "dw"):
        assert wgrad(**{k: None}) == EINVAL, k
        assert "null pointer" in L.sigma_last_error().decode()
    for sizes in ((0, H, W), (B, 0, W), (B, H, 0)):
        assert wgrad(sizes=sizes) == EINVAL, sizes
    assert wgrad(cin=6) == EINVAL and wgrad(cout=30) == EINVAL and wgrad(cin=0) == EINVAL
    assert "multiples of 4" in L.sigma_last_error().decode()
    assert wgrad(gelu_x=2) == EINVAL and wgrad(x3=-1) == EINVAL
    for k in ("x", "dy"):
        assert wgrad(**{k: p4}) == EINVAL, k
        assert "16-byte aligned" in L.sigma_last_error().decode()
    assert wgrad(ws=None) == EWORKSPACE and wgrad(n=wsb - 1) == EWORKSPACE and wgrad(ws=p4) == EWORKSPACE
    assert "workspace" in L.sigma_last_error().decode()
    # db is optional: without it the call gets as far as the workspace check
    assert wgrad(db=None, ws=None) == EWORKSPACE

    def save(x=p, w=p, wlo=None, bias=p, y=p, pre=p, cin=Cin, cout=Cout):
        return L.sigma_conv3x3_gelu_save_tf32(x, w, wlo, bias, y, pre, B, H, W, cin, cout, None)

    def dgrad(dy=p, w=p, wlo=None, aux=p, dx=p, cin=Cin, cout=Cout):
        return L.sigma_conv3x3_dgrad_tf32(dy, w, wlo, aux, dx, B, H, W, cin, cout, None)

    for fn, ptrs in ((save, ("x", "w", "y", "pre")), (dgrad, ("dy", "w", "dx"))):
        for k in ptrs:
            assert fn(**{k: None}) == EINVAL, (fn.__name__, k)
            assert "null pointer" in L.sigma_last_error().decode()
        assert fn(cin=6) == EINVAL and fn(cout=34) == EINVAL
        assert "multiples of 4" in L.sigma_last_error().decode()
        for k in ptrs + (("wlo", "bias") if fn is save else ("wlo", "aux")):
            assert fn(**{k: p4}) == EINVAL, (fn.__name__, k)
            assert "16-byte aligned" in L.sigma_last_error().decode()


@pytest.fixture(scope="module")
def sass():
    from sigma_b200 import build
    lib = build.build()
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs.setdefault(cur, [])
        elif cur is not None and "/*" in line:
            funcs[cur].append(line)
    return funcs


def test_new_kernels_exist_and_the_wgrad_sums_hold_no_float_atomics(sass):
    for name in WGRAD + EPI:
        assert name in sass, name
    assert sorted(n for n in sass if "conv3x3_wgrad" in n) == sorted(WGRAD)
    assert sorted(n for n in sass if "conv3x3_epi" in n) == sorted(EPI)
    for name in WGRAD + [SUM]:
        bad = [l.strip() for l in sass[name] if FLOAT_ATOMIC.search(l)]
        assert not bad, (name, bad[:3])
        assert any("HMMA" in l for l in sass[name]) or name == SUM, name     # the weight gradient runs on the tensor cores


def test_inference_conv_instances_keep_their_names(sass):
    for name in CONV:
        assert name in sass, name
