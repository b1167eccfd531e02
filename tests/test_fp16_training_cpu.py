"""CPU: the fp16 training mode of the fused core, as far as it goes without a device.
* the header declares the four new entry points and `_lib` binds them with the argument lists of their bf16 twins;
* the forward planner reports the plan of sigma_ss2d_scan_fwd_save_fp16 (bf16 = 4): the plan of the bf16 training forward (code 2),
  and refuses d_state 8 as code 2 does;
* argument validation of the new entry points returns its codes before any CUDA call;
* the switch: default off, the context manager restores it; TrainStep's new arguments default to the old behaviour;
* `cuobjdump -sass` of the built library: the fp16 training kernels are separate symbols (48 forward, 12 backward, 11 LayerNorm
  backward), there is no fp16 deterministic or d_state-8 training kernel, and the fp32 / bf16 training kernels and the fp16 inference
  scan are still there under their names."""
import ctypes
import subprocess

import pytest
import torch

NEW = ("sigma_ss2d_scan_fwd_save_fp16", "sigma_ss2d_scan_bwd_saved_fp16", "sigma_layernorm_fwd_fp16io", "sigma_layernorm_bwd_fp16")
RPS = (4, 8, 12, 16, 24, 32, 48, 64)


def test_header_declares_and_lib_binds_the_new_entry_points():
    from sigma_b200 import _lib
    L = _lib.lib()
    for name in NEW:
        assert name in _lib.SIGNATURES, name
        assert getattr(L, name).argtypes == _lib.SIGNATURES[name][1]
        twin = name.replace("fp16io", "bf16io").replace("_fp16", "_bf16")
        assert _lib.SIGNATURES[name] == _lib.SIGNATURES[twin], (name, twin)


def _fwd_plan(kind, B, H, W, D, N, R, code, split=0):
    from sigma_b200 import _lib
    out = (ctypes.c_int64 * 8)()
    rc = _lib.lib().sigma_test_ss2d_fwd_plan(kind, B, H, W, D, N, R, code, split, 1 << 40, out)
    return rc, [int(v) for v in out]


@pytest.mark.parametrize("kind,B,H,W,D,N,R", [(0, 2, 120, 160, 192, 16, 6), (0, 2, 23, 30, 2048, 16, 64), (1, 2, 15, 20, 1536, 4, 48),
                                               (2, 4, 30, 40, 768, 4, 24), (0, 1, 30, 40, 768, 4, 24)])
def test_plan_of_the_fp16_training_forward_is_the_bf16_one(kind, B, H, W, D, N, R):
    for split in (0, 1, 7):
        rc4, p4 = _fwd_plan(kind, B, H, W, D, N, R, 4, split)
        rc2, p2 = _fwd_plan(kind, B, H, W, D, N, R, 2, split)
        assert rc4 == rc2 == 0 and p4 == p2, (split, p4, p2)
    assert _fwd_plan(kind, B, H, W, D, 8, R, 4)[0] == -4 == _fwd_plan(kind, B, H, W, D, 8, R, 2)[0]   # SIGMA_EUNSUPPORTED
    assert _fwd_plan(kind, B, H, W, D, 8, R, 3)[0] == 0             # the fp16 inference plan is what it was


def test_argument_validation_needs_no_device():
    from sigma_b200 import _lib
    L = _lib.lib()
    x = torch.zeros(64, dtype=torch.float32)
    p = ctypes.c_void_p(x.data_ptr())                               # a non-null, 16-byte aligned host pointer: never dereferenced
    fwd = lambda D, N, Cp, hs=p, ns=0: L.sigma_ss2d_scan_fwd_save_fp16(0, p, p, p, p, p, p, p, p, hs, 2, 8, 8, D, N, 4, Cp, None, 0, ns, None)
    bwd = lambda D, N, Cp, hs=p, ns=0: L.sigma_ss2d_scan_bwd_saved_fp16(0, p, p, p, p, p, p, p, p, hs, p, p, p, p, p, p, 2, 8, 8, D, N, 4,
                                                                        Cp, None, 0, ns, None)
    assert fwd(64, 8, 20) == -4 and bwd(64, 8, 20) == -4            # d_state 8
    assert fwd(60, 16, 36) == -1                                    # fp16 rows need D % 8 == 0
    assert bwd(96, 16, 36) == -1                                    # the backward needs D % 64 == 0
    assert fwd(64, 16, 36, hs=None) == -1 and bwd(64, 16, 36, hs=None) == -1   # the mode exists only with saved states
    assert fwd(64, 16, 35) == -1 and bwd(64, 16, 35) == -1          # Cp must be the padded row length
    assert fwd(64, 16, 36, ns=-1) == -1 and bwd(64, 16, 36, ns=-1) == -1
    assert L.sigma_layernorm_fwd_fp16io(None, p, p, p, 4, 64, 1e-5, None) == -1
    assert L.sigma_layernorm_fwd_fp16io(p, p, p, p, 4, 66, 1e-5, None) == -1
    assert L.sigma_layernorm_bwd_fp16(p, p, p, p, p, p, 4, 66, 1e-5, None) == -1
    assert L.sigma_layernorm_bwd_fp16(p, p, p, None, p, p, 4, 64, 1e-5, None) == -1
    wb = lambda kind, B, N: L.sigma_ss2d_scan_bwd_workspace_bytes(kind, B, 30, 40, 768, N)
    assert wb(0, 2, 16) > 0 and wb(2, 3, 4) == 0                    # the workspace query is the one the bf16 pair uses


def test_switch_is_off_by_default_and_restored():
    from sigma_b200 import ops, train_util
    assert ops.FP16_TRAINING_CORE is False
    with ops.fp16_training_core():
        assert ops.FP16_TRAINING_CORE is True and ops.BF16_TRAINING_CORE is False   # the two switches are independent
        with ops.fp16_training_core(False):
            assert ops.FP16_TRAINING_CORE is False
        assert ops.FP16_TRAINING_CORE is True
    assert ops.FP16_TRAINING_CORE is False
    step = train_util.TrainStep(None, None)
    assert step.fp16_core is False and step.scaler is None and step.bf16_core is False
    assert ops._SAVED_FP16 not in (True, False, ops._SAVED_BF16)


@pytest.fixture(scope="module")
def symbols():
    from sigma_b200 import build
    out = subprocess.run(["cuobjdump", "-sass", build.build()], capture_output=True, text=True, check=True).stdout
    return {line.split(":", 1)[1].strip() for line in out.splitlines() if line.strip().startswith("Function :")}


def test_new_kernels_are_separate_and_existing_ones_keep_their_names(symbols):
    old = ([f"_ZN5sigma16ss2d_scan_kernelILi{n}ELi1ELi{rp}ELi{m}ELi3ELb1EfEEvNS_10Ss2dParamsE" for n in (4, 16) for rp in RPS for m in (0, 2)]
           + [f"_ZN5sigma24ss2d_scan_train16_kernelILi{n}ELi1ELi{rp}ELi{m}ELi3ELb{int(m != 1)}EEEvNS_10Ss2dParamsE"
              for n in (4, 16) for rp in RPS for m in (0, 1, 2)]
           + [f"_ZN5sigma16ss2d_scan_kernelILi{n}ELi1ELi{rp}ELi{m}ELi3ELb0E6__halfEEvNS_10Ss2dParamsE"
              for n in (4, 8, 16) for rp in RPS for m in (0, 1, 2)]
           + [f"_ZN5sigma{len(k)}{k}ILi{n}ELi{m}EEEvNS_13Ss2dBwdParamsE"
              for k in ("ss2d_bwd_kernel", "ss2d_bwd_cross_kernel", "ss2d_bwd_bf16_kernel", "ss2d_bwd_cross_bf16_kernel")
              for n in (4, 16) for m in (0, 1, 2)])
    new = ([f"_ZN5sigma27ss2d_scan_train_fp16_kernelILi{n}ELi1ELi{rp}ELi{m}ELi3ELb{int(m != 1)}EEEvNS_10Ss2dParamsE"
            for n in (4, 16) for rp in RPS for m in (0, 1, 2)]
           + [f"_ZN5sigma{len(k)}{k}ILi{n}ELi{m}EEEvNS_13Ss2dBwdParamsE" for k in ("ss2d_bwd_fp16_kernel", "ss2d_bwd_cross_fp16_kernel")
              for n in (4, 16) for m in (0, 1, 2)])
    assert len(new) == 48 + 12
    assert not [n for n in old if n not in symbols]
    assert not [n for n in new if n not in symbols]
    assert sum("ss2d_scan_train_fp16_kernel" in n for n in symbols) == 48
    assert sum("ss2d_bwd_fp16_kernel" in n or "ss2d_bwd_cross_fp16_kernel" in n for n in symbols) == 12
    assert sum("layernorm_bwd_fp16_kernel" in n for n in symbols) == 11
    assert sum("layernorm_bwd_bf16_kernel" in n for n in symbols) == 11
    # no d_state-8 and no deterministic build of the mode
    assert not [n for n in symbols if "train_fp16_kernelILi8E" in n or ("fp16" in n and "_det" in n)]
