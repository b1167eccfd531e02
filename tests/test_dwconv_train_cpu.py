"""CPU: the depthwise conv3x3 + SiLU backward, as far as it goes without a device.
* the header declares the four entry points and `_lib` binds them; the 16-bit pair shares the fp32 argument list's shape;
* argument validation returns its codes before any CUDA call: null pointers, sizes, D % 4 (fp32) / D % 8 (16-bit), 16-byte alignment
  of pointers and strides, bias / dbias given together, the workspace;
* `cuobjdump -sass` of the built library: one kernel instance per element type, none of them (nor the sum kernel they launch) holds a
  float atomic or a bulk-tensor reduce, and no new symbol is named `_det` (the default call is the deterministic one)."""
import ctypes
import re
import subprocess

import pytest
import torch

from test_deterministic_sass_cpu import FLOAT_ATOMIC

NEW = ("sigma_dwconv3x3_silu_bwd", "sigma_dwconv3x3_silu_bwd_bf16", "sigma_dwconv3x3_silu_bwd_fp16",
       "sigma_dwconv3x3_silu_bwd_workspace_bytes")
KERNELS = [f"_ZN5sigma29dwconv3x3_silu_bwd_tma_kernelI{t}EEvNS_11DwBwdParamsE" for t in ("f", "13__nv_bfloat16", "6__half")]
SUM = "_ZN5sigma20sum_parts_det_kernelEPKfixxxPf"


def test_header_declares_and_lib_binds_the_new_entry_points():
    from sigma_b200 import _lib
    L = _lib.lib()
    for name in NEW:
        assert name in _lib.SIGNATURES, name
        assert getattr(L, name).argtypes == _lib.SIGNATURES[name][1]
    assert _lib.SIGNATURES["sigma_dwconv3x3_silu_bwd_bf16"] == _lib.SIGNATURES["sigma_dwconv3x3_silu_bwd_fp16"] \
        == _lib.SIGNATURES["sigma_dwconv3x3_silu_bwd"]
    assert _lib.SIGNATURES["sigma_dwconv3x3_silu_bwd_workspace_bytes"] == (ctypes.c_size_t, [ctypes.c_int] * 4)


def test_argument_validation_needs_no_device():
    from sigma_b200 import _lib
    L = _lib.lib()
    buf = torch.zeros(64, dtype=torch.float32)
    p = ctypes.c_void_p(buf.data_ptr())                             # a non-null, 16-byte aligned host pointer: never dereferenced
    p4 = ctypes.c_void_p(buf.data_ptr() + 4)
    B, H, W = 2, 9, 17
    wsb = L.sigma_dwconv3x3_silu_bwd_workspace_bytes(B, H, W, 64)
    assert wsb > 0 and wsb % 256 == 0
    assert L.sigma_dwconv3x3_silu_bwd_workspace_bytes(0, H, W, 64) == 0 == L.sigma_dwconv3x3_silu_bwd_workspace_bytes(B, H, W, 0)

    def call(fn, D=64, x=p, dy=p, dx=p, w=p, bias=p, dbias=p, dw=p, xrs=None, xbs=None, dybs=None, dxbs=None, ws=p, n=wsb, sizes=None):
        xrs = 2 * D if xrs is None else xrs
        xbs = H * W * 2 * D if xbs is None else xbs
        dybs = H * W * D if dybs is None else dybs
        dxbs = H * W * D if dxbs is None else dxbs
        b, h, w_ = sizes or (B, H, W)
        return getattr(L, fn)(x, xrs, xbs, w, bias, dy, dybs, dx, dxbs, dw, dbias, b, h, w_, D, ws, n, None)

    for fn, q in (("sigma_dwconv3x3_silu_bwd", 4), ("sigma_dwconv3x3_silu_bwd_bf16", 8), ("sigma_dwconv3x3_silu_bwd_fp16", 8)):
        for k in ("x", "dy", "dx", "w", "dw"):
            assert call(fn, **{k: None}) == -1, (fn, k)
        assert "null pointer" in L.sigma_last_error().decode()
        assert call(fn, bias=None) == -1 and call(fn, dbias=None) == -1          # bias and dbias go together
        for sizes in ((0, H, W), (B, 0, W), (B, H, 0)):
            assert call(fn, sizes=sizes) == -1, (fn, sizes)
        assert call(fn, D=0) == -1 and call(fn, D=q + 2) == -1 and call(fn, D=q // 2 + q) == -1
        assert "bad sizes" in L.sigma_last_error().decode()
        for k in ("x", "dy", "dx"):
            assert call(fn, **{k: p4}) == -1, (fn, k)
        for k in ("xrs", "xbs", "dybs", "dxbs"):
            assert call(fn, **{k: 64 * 2 + q // 2}) == -1, (fn, k)
        assert "16-byte aligned" in L.sigma_last_error().decode()
        assert call(fn, ws=None) == -1 and call(fn, n=wsb - 1) == -1 and call(fn, ws=p4) == -1
        assert "workspace" in L.sigma_last_error().decode()
    # fp32 rows need D % 4 only; 16-bit rows D % 8 (fp32 D = 68 passes the size check, so it fails on the workspace it was sized for)
    n68 = L.sigma_dwconv3x3_silu_bwd_workspace_bytes(B, H, W, 68)
    assert call("sigma_dwconv3x3_silu_bwd", D=68, ws=None, n=n68) == -1 and "workspace" in L.sigma_last_error().decode()
    assert call("sigma_dwconv3x3_silu_bwd_bf16", D=68, n=n68) == -1 and "bad sizes" in L.sigma_last_error().decode()


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


def test_every_instance_exists_without_float_atomics(sass):
    for name in KERNELS + [SUM]:
        assert name in sass, name
        bad = [l.strip() for l in sass[name] if FLOAT_ATOMIC.search(l)]
        assert not bad, (name, bad[:3])
    assert [n for n in sass if "dwconv3x3_silu_bwd" in n] == [n for n in sass if n in KERNELS]
    assert not [n for n in sass if "dwconv" in n and "_det" in n]
