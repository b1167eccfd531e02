"""GPU: CroMB (CrossMambaFusionBlock) training through the fused scan core, kind CROSS.
* the block's loss, input gradients and every parameter gradient against the unmodified reference's autograd goldens (grad_cromb,
  1e-3 of each gradient's scale), with a spy on the fused backward's native call showing that the CROSS core ran;
* fused against the composed path (op-level scans) at a Sigma-tiny stage shape, 2 images, 30 x 40, hidden 384, with and without
  the residual: outputs and every gradient within 1e-3 of its scale;
* under torch.use_deterministic_algorithms(True): the fused core does not run (CroMB keeps the op-level _det kernels) and two
  backward passes are bitwise equal."""
import numpy as np
import pytest
import torch

import procedural as P
from helpers import SEED, golden

pytestmark = pytest.mark.gpu


def _spy(monkeypatch):
    from sigma_b200 import ops
    kinds = []
    real = ops._call_ss2d_bwd

    def spy(args, saved=False, det=False):
        kinds.append(args[0])
        return real(args, saved, det)
    monkeypatch.setattr(ops, "_call_ss2d_bwd", spy)
    return kinds


@pytest.fixture
def fp32_dense():
    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


def test_cromb_block_gradients_match_reference_through_the_cross_core(monkeypatch, fp32_dense):
    from sigma_b200 import _lib, modules as M, ops
    monkeypatch.setattr(ops, "FUSED_TRAINING", True)
    kinds = _spy(monkeypatch)
    g = golden("grad_cromb")
    mod = M.CrossMambaFusionBlock(hidden_dim=32, mlp_ratio=0.0, d_state=4, drop_path=0.0)
    P.fill_state_dict(mod, SEED)
    mod = mod.cuda().train()
    xs = [P.randn(SEED, k, (2, 6, 5, 32)).cuda().requires_grad_(True) for k in ("mod/x", "mod/x2")]
    outs = mod(*xs)
    loss = sum((o * P.randn(SEED, f"grad_cromb/w{i}", tuple(o.shape)).cuda()).sum() for i, o in enumerate(outs))
    loss.backward()
    assert kinds == [_lib.DIRS_CROSS], kinds
    assert abs(float(loss) - float(g["loss"])) <= 1e-3 * max(1.0, abs(float(g["loss"])))
    params = dict(mod.named_parameters())
    checked = 0
    for i, x in enumerate(xs):
        r = g[f"dx{i}"]
        assert float(np.abs(x.grad.cpu().numpy() - r).max()) <= 1e-3 * float(np.abs(r).max()), f"dx{i}"
        checked += 1
    for k in g.files:
        if k.startswith("g/"):
            r = g[k]
            err = float(np.abs(params[k[2:]].grad.cpu().numpy() - r).max()) / (float(np.abs(r).max()) + 1e-20)
            assert err <= 1e-3, f"{k}: {err:.2e} of its scale"
            checked += 1
    assert checked == len(g.files) - 1


def _block_grads(op, xs, wts, residual):
    op.zero_grad(set_to_none=True)
    xs = [x.detach().clone().requires_grad_(True) for x in xs]
    outs = op(*xs, residual=residual)
    sum((o * w).sum() for o, w in zip(outs, wts)).backward()
    return [o.detach() for o in outs], [x.grad for x in xs], {n: p.grad.clone() for n, p in op.named_parameters()}


@pytest.mark.parametrize("residual", [False, True])
def test_fused_matches_composed_at_a_stage_shape(residual, monkeypatch, fp32_dense):
    from sigma_b200 import _lib, modules as M, ops
    kinds = _spy(monkeypatch)
    images, H, W, C = 2, 30, 40, 384
    op = M.CrossMambaFusion_SS2D_SSM(d_model=C, d_state=4, ssm_ratio=2.0).cuda().train()
    xs = [P.randn(SEED, f"cromb/x{i}", (images, H, W, C)).cuda() for i in range(2)]
    wts = [P.randn(SEED, f"cromb/w{i}", (images, H, W, C)).cuda() for i in range(2)]
    monkeypatch.setattr(ops, "FUSED_TRAINING", False)
    ref = _block_grads(op, xs, wts, residual)
    assert kinds == []
    monkeypatch.setattr(ops, "FUSED_TRAINING", True)
    got = _block_grads(op, xs, wts, residual)
    assert kinds == [_lib.DIRS_CROSS]
    for what, a, b in [("out", got[0], ref[0]), ("dx", got[1], ref[1])]:
        for i, (x, y) in enumerate(zip(a, b)):
            err = float((x - y).abs().max()) / float(y.abs().max())
            assert err <= 1e-3, f"{what}{i}: {err:.2e} of its scale"
    assert got[2].keys() == ref[2].keys() and len(ref[2]) == len(list(op.parameters()))
    for n, r in ref[2].items():
        err = float((got[2][n] - r).abs().max()) / (float(r.abs().max()) + 1e-20)
        assert err <= 1e-3, f"{n}: {err:.2e} of its scale"


def test_deterministic_switch_keeps_the_op_level_path(monkeypatch, fp32_dense):
    from sigma_b200 import modules as M, ops
    monkeypatch.setattr(ops, "FUSED_TRAINING", True)
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")      # torch requires it for cuBLAS under the switch
    kinds = _spy(monkeypatch)
    images, H, W, C = 2, 15, 20, 96
    op = M.CrossMambaFusion_SS2D_SSM(d_model=C, d_state=4, ssm_ratio=2.0).cuda().train()
    xs = [P.randn(SEED, f"cromb-det/x{i}", (images, H, W, C)).cuda() for i in range(2)]
    wts = [P.randn(SEED, f"cromb-det/w{i}", (images, H, W, C)).cuda() for i in range(2)]
    torch.use_deterministic_algorithms(True)
    try:
        runs = [_block_grads(op, xs, wts, True) for _ in range(2)]
    finally:
        torch.use_deterministic_algorithms(False)
    assert kinds == []
    (o0, d0, p0), (o1, d1, p1) = runs
    assert all(torch.equal(a, b) for a, b in zip(o0 + d0, o1 + d1))
    assert all(torch.equal(p0[n], p1[n]) for n in p0)
