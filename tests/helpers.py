"""Shared helpers for the parity tests."""
import os
import types
import zlib

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SEED = 7


def golden(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"))


def cfg_tiny(H, W, num_classes=9, backbone="sigma_tiny"):
    return types.SimpleNamespace(backbone=backbone, decoder="MambaDecoder", num_classes=num_classes, image_height=H,
                                 image_width=W, pretrained_model=None, bn_eps=1e-3, bn_momentum=0.1)


def max_err(a, b):
    a = a.detach().float().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    b = b.detach().float().cpu().numpy() if torch.is_tensor(b) else np.asarray(b)
    return float(np.abs(a - b).max())


def assert_close(a, b, rtol, atol, what=""):
    a = a.detach().float().cpu().numpy() if torch.is_tensor(a) else np.asarray(a, dtype=np.float32)
    b = b.detach().float().cpu().numpy() if torch.is_tensor(b) else np.asarray(b, dtype=np.float32)
    assert a.shape == b.shape, f"{what}: shape {a.shape} vs {b.shape}"
    err = np.abs(a - b)
    tol = atol + rtol * np.abs(b)
    bad = err > tol
    assert not bad.any(), (f"{what}: {bad.sum()}/{bad.size} elements out of tolerance; max abs err {err.max():.3e} "
                           f"(|ref| max {np.abs(b).max():.3e}), rtol={rtol} atol={atol}")


def record(name, **kv):
    """Append one JSON line of measured parity numbers to $SIGMA_PARITY_LOG (set by the GPU run scripts)."""
    import json
    path = os.environ.get("SIGMA_PARITY_LOG")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps(dict(test=name, **kv)) + "\n")


def gemm_plan(M, N, K, x3, conv=None):
    """The launch plan sigma_linear_tf32{,x3} (conv=None) or sigma_conv3x3_tf32 (conv=(B, H, W): input (B, H, W, K), N output
    channels) would use under the current environment (SIGMA_GEMM_BN included), from the library's own planner."""
    import ctypes
    from sigma_b200 import _lib
    out = (ctypes.c_int64 * 6)()
    B, H, W = conv if conv is not None else (0, 0, 0)
    _lib.check(_lib.lib().sigma_test_gemm_plan(M, N, K, int(bool(x3)), B, H, W, out), "sigma_test_gemm_plan")
    return dict(zip(("bn", "stages", "grid", "tiles", "smem", "ctas_per_sm"), (int(v) for v in out)))


def sample_index(key, numel, k):
    """A fixed, seeded set of min(k, numel) flat indices for `key`: the positions at which a golden file stores a large output."""
    rng = np.random.default_rng(zlib.crc32(key.encode()))
    return np.sort(rng.choice(numel, size=min(k, numel), replace=False))
