"""CPU: the drop-in boundary.  The C-ABI library loads without a GPU or libcuda, exports every symbol that
include/sigma_b200.h declares, the ctypes binding declares the same set, and the reference's import paths resolve to
our modules.  No compute calls (there is no GPU here)."""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib_path():
    from sigma_b200 import build
    return build.build()


def _declared():
    src = open(os.path.join(ROOT, "include", "sigma_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return set(re.findall(r"\b(sigma_[a-z0-9_]+)\s*\(", src))


def test_library_exports_every_declared_symbol(lib_path):
    out = subprocess.run(["nm", "-D", "--defined-only", lib_path], capture_output=True, text=True, check=True).stdout
    exported = {ln.split()[-1] for ln in out.splitlines() if " T " in ln}
    declared = _declared()
    assert declared, "no declarations parsed"
    assert declared <= exported, f"declared but not exported: {sorted(declared - exported)}"
    extra = {s for s in exported - declared if s.startswith("sigma_")}
    assert not extra, f"undeclared exports: {sorted(extra)}"


def test_library_has_no_runtime_dependency_on_cuda_libs(lib_path):
    out = subprocess.run(["ldd", lib_path], capture_output=True, text=True, check=True).stdout
    assert "libcuda" not in out and "libcudart" not in out and "libtorch" not in out, out


def test_ctypes_binding_matches_header(lib_path):
    from sigma_b200 import _lib
    L = _lib.lib()
    assert L.sigma_abi_version() == 2
    assert set(_lib.SIGNATURES) == _declared()
    assert L.sigma_ss2d_padded_cp(16, 6) == 40 and L.sigma_ss2d_padded_cp(4, 24) == 32 and L.sigma_ss2d_padded_cp(4, 65) == -1
    assert L.sigma_scan_fwd_workspace_bytes(2, 768, 1024, 16, 4, 0) > 0
    assert L.sigma_launch_count() == 0


def test_ctypes_types_follow_header_conventions():
    """SIGNATURES is parsed from the header: host int64 arrays, the strides struct and the error string keep their types,
    every other pointer is a void pointer."""
    from ctypes import POINTER, c_char_p, c_int, c_int64, c_void_p
    from sigma_b200 import _lib
    S = _lib.SIGNATURES
    assert S["sigma_test_gemm_plan"] == (c_int, [c_int64] + [c_int] * 6 + [POINTER(c_int64)])
    assert S["sigma_image_pre_fwd"][1][3] is c_void_p                      # int64_t *labels_out: a device pointer
    assert POINTER(_lib.ScanStrides) in S["sigma_scan_fwd"][1]
    assert S["sigma_last_error"] == (c_char_p, [])
    src = open(os.path.join(ROOT, "include", "sigma_b200.h")).read()
    body = re.search(r"typedef struct sigma_scan_strides \{(.*?)\}", src, flags=re.S).group(1)
    decls = [d.split(None, 1) for d in body.split(";") if d.strip()]
    assert decls and all(t == "int64_t" for t, _ in decls)
    assert _lib.ScanStrides._fields_ == [(f.strip(), c_int64) for _, names in decls for f in names.split(",")]


def test_sm90a_tma_in_sass(lib_path):
    """the fused scan really is a TMA kernel (UTMALDG) compiled for sm_90a, and the GEMM runs on warpgroup MMAs (HGMMA)."""
    out = subprocess.run(["cuobjdump", "-lelf", lib_path], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    sass = subprocess.run(["cuobjdump", "-sass", os.path.join(ROOT, "sigma_b200", "build", "ss2d_scan_rp8.o")],
                          capture_output=True, text=True).stdout
    assert "UTMALDG" in sass and "SYNCS" in sass and "MUFU.EX2" in sass
    sass = subprocess.run(["cuobjdump", "-sass", os.path.join(ROOT, "sigma_b200", "build", "gemm_tf32.o")],
                          capture_output=True, text=True).stdout
    assert "HGMMA" in sass and "UTMALDG" in sass


def test_dropin_import_paths_resolve():
    code = ("import sys; sys.path[:0] = [%r, %r];"
            "import selective_scan_cuda_core as c, selective_scan as s;"
            "from models.builder import EncoderDecoder;"
            "from models.encoders.vmamba import SS2D, VSSBlock, ConMB_SS2D, CrossScan, SelectiveScan, Backbone_VSSM;"
            "from models.encoders.dual_vmamba import vssm_tiny, vssm_small, vssm_base;"
            "from models.decoders.MambaDecoder import MambaDecoder;"
            "import sigma_b200.modules as M;"
            "assert EncoderDecoder is M.EncoderDecoder and SS2D is M.SS2D and callable(c.fwd) and callable(c.bwd);"
            "assert callable(s.selective_scan_fn) and callable(s.selective_scan_ref); print('ok')") % (
        ROOT, os.path.join(ROOT, "sigma_b200", "dropin"))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr


def test_no_cpu_fallback():
    """product modules refuse CPU tensors instead of silently computing on the host."""
    import torch
    from sigma_b200 import modules as M, ops
    with pytest.raises(RuntimeError):
        ops.selective_scan_cuda_core_fwd(torch.zeros(1, 4, 8), torch.zeros(1, 4, 8), torch.zeros(4, 4),
                                         torch.zeros(1, 1, 4, 8), torch.zeros(1, 1, 4, 8), None, None, False, 1)
    blk = M.VSSBlock(hidden_dim=16, mlp_ratio=0.0, d_state=4)
    with pytest.raises(RuntimeError), torch.no_grad():
        blk(torch.zeros(1, 4, 4, 16))


def test_dropin_selective_scan_ref_matches_oracle():
    import numpy as np
    import torch
    sys.path.insert(0, os.path.join(ROOT, "sigma_b200", "dropin"))
    try:
        import selective_scan as s
    finally:
        sys.path.pop(0)
    import procedural as P
    from oracle import scan_oracle
    u, dl, A, Bm, Cm, D, bias = P.scan_inputs(3, 2, 8, 4, 40, 2)
    got = s.selective_scan_ref(u, dl, A, Bm, Cm, D, bias, True)
    ref = scan_oracle.scan_fwd(u.numpy(), dl.numpy(), A.numpy(), Bm.numpy(), Cm.numpy(), D.numpy(), bias.numpy(), True)
    assert np.abs(got.numpy() - ref).max() < 1e-4
