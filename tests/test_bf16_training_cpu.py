"""CPU: the bf16 training mode of the fused core, as far as it goes without a device.
* the header declares the new entry points and `_lib` binds them;
* the forward planner reports the plan of sigma_ss2d_scan_fwd_save_bf16 (bf16 = 2) and refuses d_state 8 there; the backward's plan does
  not depend on the element type;
* argument validation of the new pair returns its codes before any CUDA call;
* the switch: default off, the context manager restores it;
* `cuobjdump -sass` of the built library: the fp32 training-forward / backward kernels and the bf16 inference kernels are still there
  under their names, and the bf16 training kernels are separate symbols."""
import ctypes
import subprocess

import pytest
import torch

NEW = ("sigma_ss2d_scan_fwd_save_bf16", "sigma_ss2d_scan_bwd_saved_bf16", "sigma_layernorm_fwd_bf16io", "sigma_layernorm_bwd_bf16")


def test_header_declares_and_lib_binds_the_new_entry_points():
    from sigma_b200 import _lib
    L = _lib.lib()
    for name in NEW:
        assert name in _lib.SIGNATURES, name
        assert getattr(L, name).argtypes == _lib.SIGNATURES[name][1]
    assert len(_lib.SIGNATURES["sigma_ss2d_scan_fwd_save_bf16"][1]) == len(_lib.SIGNATURES["sigma_ss2d_scan_fwd_save"][1])
    assert len(_lib.SIGNATURES["sigma_ss2d_scan_bwd_saved_bf16"][1]) == len(_lib.SIGNATURES["sigma_ss2d_scan_bwd_saved"][1])


def _fwd_plan(kind, B, H, W, D, N, R, bf16, split=0):
    from sigma_b200 import _lib
    out = (ctypes.c_int64 * 8)()
    rc = _lib.lib().sigma_test_ss2d_fwd_plan(kind, B, H, W, D, N, R, bf16, split, 1 << 40, out)
    return rc, [int(v) for v in out]


@pytest.mark.parametrize("kind,B,H,W,D,N,R", [(0, 2, 120, 160, 192, 16, 6), (1, 2, 15, 20, 1536, 4, 48), (2, 4, 30, 40, 768, 4, 24)])
def test_plan_hooks_report_the_new_pair(kind, B, H, W, D, N, R):
    rc, train = _fwd_plan(kind, B, H, W, D, N, R, 2)
    assert rc == 0
    rc, f32 = _fwd_plan(kind, B, H, W, D, N, R, 0)
    assert rc == 0
    # the same walk (segments, tiles, warps) as the fp32 training forward; the stage holds a 2-byte xc tile, so never a shallower ring
    assert train[:5] == f32[:5] and train[5] >= f32[5] and train[6] == 3
    rc, forced = _fwd_plan(kind, B, H, W, D, N, R, 2, split=7)
    assert rc == 0 and forced[0] == 7
    assert _fwd_plan(kind, B, H, W, D, 8, R, 2)[0] == -4            # SIGMA_EUNSUPPORTED: no d_state-8 training kernels
    assert _fwd_plan(kind, B, H, W, D, 8, R, 1)[0] == 0             # the inference plan is what it was


def test_argument_validation_needs_no_device():
    from sigma_b200 import _lib
    L = _lib.lib()
    x = torch.zeros(64, dtype=torch.float32)
    p = ctypes.c_void_p(x.data_ptr())                               # a non-null, 16-byte aligned host pointer: never dereferenced
    fwd = lambda D, N, Cp: L.sigma_ss2d_scan_fwd_save_bf16(0, p, p, p, p, p, p, p, p, p, 2, 8, 8, D, N, 4, Cp, None, 0, 0, None)
    bwd = lambda D, N, Cp, hs=p: L.sigma_ss2d_scan_bwd_saved_bf16(0, p, p, p, p, p, p, p, p, hs, p, p, p, p, p, p, 2, 8, 8, D, N, 4, Cp,
                                                                  None, 0, 0, None)
    assert fwd(64, 8, 20) == -4 and bwd(64, 8, 20) == -4            # d_state 8
    assert fwd(60, 16, 36) == -1                                    # bf16 rows need D % 8 == 0
    assert bwd(96, 16, 36) == -1                                    # the backward needs D % 64 == 0
    assert bwd(64, 16, 36, hs=None) == -1                           # the mode exists only with saved states
    assert fwd(64, 16, 35) == -1                                    # Cp must be the padded row length
    assert L.sigma_layernorm_fwd_bf16io(None, p, p, p, 4, 64, 1e-5, None) == -1
    assert L.sigma_layernorm_bwd_bf16(p, p, p, p, p, p, 4, 66, 1e-5, None) == -1


def test_switch_is_off_by_default_and_restored():
    from sigma_b200 import ops, train_util
    assert ops.BF16_TRAINING_CORE is False
    with ops.bf16_training_core():
        assert ops.BF16_TRAINING_CORE is True
        with ops.bf16_training_core(False):
            assert ops.BF16_TRAINING_CORE is False
        assert ops.BF16_TRAINING_CORE is True
    assert ops.BF16_TRAINING_CORE is False
    assert train_util.TrainStep(None, None).bf16_core is False


@pytest.fixture(scope="module")
def symbols():
    from sigma_b200 import build
    out = subprocess.run(["cuobjdump", "-sass", build.build()], capture_output=True, text=True, check=True).stdout
    return {line.split(":", 1)[1].strip() for line in out.splitlines() if line.strip().startswith("Function :")}


def test_existing_kernels_keep_their_names_and_new_ones_are_separate(symbols):
    rps = (4, 8, 12, 16, 24, 32, 48, 64)
    old = ([f"_ZN5sigma16ss2d_scan_kernelILi{n}ELi1ELi{rp}ELi{m}ELi3ELb1EfEEvNS_10Ss2dParamsE" for n in (4, 16) for rp in rps for m in (0, 2)]
           + [f"_ZN5sigma16ss2d_scan_kernelILi{n}ELi1ELi{rp}ELi{m}ELi3ELb0E13__nv_bfloat16EEvNS_10Ss2dParamsE"
              for n in (4, 8, 16) for rp in rps for m in (0, 1, 2)]
           + [f"_ZN5sigma{len(k)}{k}ILi{n}ELi{m}EEEvNS_13Ss2dBwdParamsE" for k in ("ss2d_bwd_kernel", "ss2d_bwd_cross_kernel")
              for n in (4, 16) for m in (0, 1, 2)])
    new = ([f"_ZN5sigma24ss2d_scan_train16_kernelILi{n}ELi1ELi{rp}ELi{m}ELi3ELb{int(m != 1)}EEEvNS_10Ss2dParamsE"
            for n in (4, 16) for rp in rps for m in (0, 1, 2)]
           + [f"_ZN5sigma{len(k)}{k}ILi{n}ELi{m}EEEvNS_13Ss2dBwdParamsE" for k in ("ss2d_bwd_bf16_kernel", "ss2d_bwd_cross_bf16_kernel")
              for n in (4, 16) for m in (0, 1, 2)])
    assert not [n for n in old if n not in symbols]
    assert not [n for n in new if n not in symbols]
    assert sum("layernorm_bwd_bf16_kernel" in n for n in symbols) == 11
    # no d_state-8 and no deterministic build of the mode
    assert not [n for n in symbols if "train16_kernelILi8E" in n or ("bf16" in n and "_det" in n and "ss2d" in n)]
