"""CPU: the deterministic (`_det`) kernels of the built library contain no floating-point atomic or reduction instruction: no
float RED / ATOM (global or shared, including the CAS loop a shared float atomicAdd compiles to) and no bulk-tensor reduce.  The
only atomics left are the integer shared-memory counters of the TMA rings.  Every `_det` instance the entry points launch exists."""
import os
import re
import subprocess

import pytest

FLOAT_ATOMIC = re.compile(r"\b(RED|REDG|ATOM|ATOMG|ATOMS|REDAS)\.[A-Z0-9.]*(F32|F16|BF16|F64|FADD)|ATOMS\.CAST\.SPIN|ATOMG?\.E?\.?CAS|"
                          r"\bUTMAREDG\b|\bUBLKRED\b|\bREDUX\.F")

EXPECTED = (
    [f"_ZN5sigma19ss2d_bwd_det_kernelILi{n}ELi{m}EEEvNS_13Ss2dBwdParamsE" for n in (4, 16) for m in (0, 2)]
    + [f"_ZN5sigma26scan_op_bwd_tma_det_kernelI{t}Li{n}ELi{m}EEEvNS_16ScanBwdTmaParamsE"
       for t in ("f", "6__half", "13__nv_bfloat16") for n in (4, 8, 16) for m in (0, 2)]
    + [f"_ZN5sigma22scan_op_bwd_det_kernelI{t}Li4ELi{l}EEEvNS_13ScanBwdParamsE" for t in ("f", "6__half", "13__nv_bfloat16") for l in (1, 2, 4)]
    + [f"_ZN5sigma24layernorm_bwd_det_kernelILi{lpr}ELi{v}EEEvPKfS2_S2_PfxifS3_"
       for lpr, v in [(8, 1), (8, 2), (8, 3), (8, 4), (16, 3), (16, 4), (32, 3), (32, 4), (32, 6), (32, 8), (32, 12)]]
    + ["_ZN5sigma20sum_parts_det_kernelEPKfixxxPf"]
    + [f"_ZN5sigma32upsample_bilinear_bwd_det_kernelILb{b}EEEvPKfPfiiiiiiff" for b in (0, 1)]
)


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


def test_every_det_instance_exists(sass):
    missing = [n for n in EXPECTED if n not in sass]
    assert not missing, f"missing _det kernels: {missing}"
    assert sorted(n for n in sass if "_det" in n) == sorted(EXPECTED)


def test_det_kernels_have_no_float_atomics(sass):
    bad = {n: [l.strip() for l in body if FLOAT_ATOMIC.search(l)] for n, body in sass.items() if "_det" in n}
    bad = {n: v[:3] for n, v in bad.items() if v}
    assert not bad, f"float atomics / reductions in deterministic kernels: {bad}"


def test_the_pattern_sees_the_default_kernels_atomics(sass):
    """the same scan finds the atomics of the default builds (so a clean result above means something)"""
    for name in ("_ZN5sigma15ss2d_bwd_kernelILi16ELi0EEEvNS_13Ss2dBwdParamsE",
                 "_ZN5sigma18scan_op_bwd_kernelIfLi4ELi4EEEvNS_13ScanBwdParamsE",
                 "_ZN5sigma20layernorm_bwd_kernelILi8ELi1EEEvPKfS2_S2_PfS3_S3_xif"):
        assert name in sass, name
        assert any(FLOAT_ATOMIC.search(l) for l in sass[name]), name
    assert any("UTMAREDG" in l for l in sass["_ZN5sigma15ss2d_bwd_kernelILi16ELi0EEEvNS_13Ss2dBwdParamsE"])
