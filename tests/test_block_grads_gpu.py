"""GPU: gradients of whole blocks through the training path (modules' composed path: torch autograd over the op-level
sigma_scan_fwd / sigma_scan_bwd kernels) against goldens from the UNMODIFIED reference's autograd
(tests/golden/make_golden_grads.py): VSSBlock (SS2D), CroMB, ConMB, CVSSDecoderBlock — loss, input gradients and the
gradient of EVERY parameter.  fp32 dense math (TF32 off): the op-level bar, 1e-3 of each gradient's scale."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import procedural as P
from helpers import SEED, golden

pytestmark = pytest.mark.gpu


def _cases():
    from sigma_b200 import modules as M
    return {
        "grad_vssblock": (lambda: M.VSSBlock(hidden_dim=32, norm_layer=nn.LayerNorm, mlp_ratio=0.0, d_state=16, drop_path=0.0), 1),
        "grad_cromb": (lambda: M.CrossMambaFusionBlock(hidden_dim=32, mlp_ratio=0.0, d_state=4, drop_path=0.0), 2),
        "grad_conmb": (lambda: M.ConcatMambaFusionBlock(hidden_dim=32, mlp_ratio=0.0, d_state=4, drop_path=0.0), 2),
        "grad_cvss_dec": (lambda: M.CVSSDecoderBlock(hidden_dim=32, norm_layer=nn.LayerNorm, d_state=4, mlp_ratio=4.0, drop_path=0.0), 1),
    }


@pytest.mark.parametrize("name", ["grad_vssblock", "grad_cromb", "grad_conmb", "grad_cvss_dec"])
@pytest.mark.parametrize("core", ["fused", "composed"])
def test_block_gradients_match_reference_autograd(name, core, monkeypatch):
    """core = fused: SS2D / ConMB train through ops.FusedSS2DCore (f1: sigma_ss2d_scan_bwd_saved); composed: CrossScan + einsums +
    the op-level scan kernels.  CroMB always uses the composed path (its scans read the other modality's C)."""
    from sigma_b200 import ops
    monkeypatch.setattr(ops, "FUSED_TRAINING", core == "fused")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    ctor, nin = _cases()[name]
    g = golden(name)
    mod = ctor()
    P.fill_state_dict(mod, SEED)
    mod = mod.cuda().train()
    xs = [P.randn(SEED, k, (2, 6, 5, 32)).cuda().requires_grad_(True) for k in ("mod/x", "mod/x2")[:nin]]
    out = mod(*xs)
    outs = out if isinstance(out, (tuple, list)) else (out,)
    loss = sum((o * P.randn(SEED, f"{name}/w{i}", tuple(o.shape)).cuda()).sum() for i, o in enumerate(outs))
    loss.backward()
    assert abs(float(loss) - float(g["loss"])) <= 1e-3 * max(1.0, abs(float(g["loss"]))), (float(loss), float(g["loss"]))
    checked = 0
    for i, x in enumerate(xs):
        r = g[f"dx{i}"]
        err = float(np.abs(x.grad.cpu().numpy() - r).max()) / (float(np.abs(r).max()) + 1e-20)
        assert err <= 1e-3, f"{name} dx{i}: {err:.2e} of its scale"
        checked += 1
    params = dict(mod.named_parameters())
    for k in g.files:
        if not k.startswith("g/"):
            continue
        p = params[k[2:]]
        assert p.grad is not None, k
        r = g[k]
        err = float(np.abs(p.grad.cpu().numpy() - r).max()) / (float(np.abs(r).max()) + 1e-20)
        assert err <= 1e-3, f"{name} {k}: {err:.2e} of its scale"
        checked += 1
    assert checked == len(g.files) - 1
