"""CPU: the tf32x3 GEMM instances (sigma_linear_tf32x3 and sigma_conv3x3_tf32 with a lo weight) keep their A fragments, the
split and 64-128 accumulators in registers: the built library's resource usage shows no local memory (no spills) for any of
them, at every tile width."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIDTHS = list(range(32, 257, 32))


@pytest.fixture(scope="module")
def res_usage():
    from sigma_b200 import build
    lib = build.build()
    out = subprocess.run(["cuobjdump", "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    # " Function <name>:\n  REG:96 STACK:0 SHARED:1024 LOCAL:0 ..."
    return dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out))


@pytest.mark.parametrize("conv", [False, True], ids=["linear", "conv"])
def test_x3_instances_do_not_spill(res_usage, conv):
    seen = {}
    for name, usage in res_usage.items():
        m = re.fullmatch(r"_ZN5sigma16gemm_tf32_kernelILi(\d+)ELb1ELb([01])ELb0EEEvNS_10GemmParamsE", name)
        if m and m.group(2) == ("1" if conv else "0"):
            seen[int(m.group(1))] = usage
    assert sorted(seen) == WIDTHS, f"X3 instances found: {sorted(seen)}"
    for bn, usage in sorted(seen.items()):
        fields = dict(kv.split(":", 1) for kv in usage.split())
        assert fields["LOCAL"] == "0" and fields["STACK"] == "0", f"BN={bn}: {usage}"
