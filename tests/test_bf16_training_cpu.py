"""CPU: the bf16 training mode of the fused core, as far as it goes without a device.
* the header declares the new entry points and `_lib` binds them;
* the forward planner reports the plan of sigma_ss2d_scan_fwd_save_bf16 (bf16 = 2) and refuses d_state 8 there; the backward's plan does
  not depend on the element type;
* argument validation of the new pair returns its codes before any CUDA call;
* the fp64 reference on a given delta' (tests/ss2d_delta_ref64.py): with the reference's own delta' it changes nothing beyond the delta' error terms it
  drops, and with a bf16-rounded delta' every output matches fp64 autograd through a restatement of the op that runs on that delta'
  with the rounding passed straight through and the softplus derivative taken from the rounded value (the gradient the backward
  kernel computes);
* the switch: default off, the context manager restores it;
* `cuobjdump -sass` of the built library: the fp32 training-forward / backward kernels and the bf16 inference kernels are still there
  under their names, and the bf16 training kernels are separate symbols."""
import ctypes
import subprocess

import pytest
import torch

import procedural as P
import ss2d_delta_ref64 as RD
from oracle import ss2d_ref64 as R64

S = 131
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


def _inputs(kind, B, H, W, D, N, R, tag):
    K = R64.KINDS[kind]
    Lseq = H * W * (2 if kind == "seq2" else 1)
    Cp = 2 * N + R + 3
    bf = lambda t: t.bfloat16().float()
    xc = bf(P.randn(S, tag + "/xc", (B, Lseq, D)))
    xdbl = P.randn(S, tag + "/xdbl", (B, Lseq, K, Cp))
    xdbl[..., 2 * N + R:] = 0.0
    dtw = P.rand(S, tag + "/dtw", (K, D, R), -R ** -0.5, R ** -0.5)
    dt = torch.exp(P.rand(S, tag + "/dt", (K, D), -6.9, -2.3))
    dtb = dt + torch.log(-torch.expm1(-dt))
    A = -torch.arange(1, N + 1, dtype=torch.float32).repeat(K * D, 1) * P.rand(S, tag + "/A", (K * D, N), 0.8, 1.25)
    Ds = P.randn(S, tag + "/Ds", (K * D,), 0.1, 1.0)
    dy = bf(P.randn(S, tag + "/dy", (B, Lseq, D)))
    return xc, xdbl, dtw, dtb, A, Ds, dy


class _SoftplusRounded(torch.autograd.Function):
    """softplus rounded to bf16; backward as the kernel forms it: the derivative 1 - exp(-delta') of the ROUNDED delta', the
    rounding itself passed straight through"""

    @staticmethod
    def forward(ctx, x):
        dl = torch.nn.functional.softplus(x).float().bfloat16().double()
        ctx.save_for_backward(dl)
        return dl

    @staticmethod
    def backward(ctx, g):
        return g * -torch.expm1(-ctx.saved_tensors[0])


def _literal(kind, xc, xdbl, dtw, dtb, A, Ds, dy, H, W):
    """the op restated on a delta' rounded to bf16 before use: per direction gather, a loop over the walk, scatter; fp64 autograd"""
    t = [v.double().clone().requires_grad_(True) for v in (xc, xdbl, dtw, dtb, A, Ds)]
    xc_, xdbl_, dtw_, dtb_, A_, Ds_ = t
    Bt, Lseq, D = xc.shape
    N, R = A.shape[1], dtw.shape[2]
    total, pres, deltas = 0.0, [], []
    for k, idx in enumerate(R64.dir_index(kind, H, W)):
        u, xk = xc_[:, idx], xdbl_[:, idx, k]
        pre = xk[..., 2 * N:2 * N + R] @ dtw_[k].t() + dtb_[k]
        pre.retain_grad()
        dl = _SoftplusRounded.apply(pre)
        Ak, Dk = A_[k * D:(k + 1) * D], Ds_[k * D:(k + 1) * D]
        h = torch.zeros(Bt, D, N, dtype=torch.float64)
        ys = []
        for l in range(Lseq):
            h = torch.exp(dl[:, l, :, None] * Ak) * h + (dl[:, l] * u[:, l])[..., None] * xk[:, l, None, :N]
            ys.append((h * xk[:, l, None, N:2 * N]).sum(-1) + Dk * u[:, l])
        yk = torch.stack(ys, 1)
        total = total + (yk * dy.double()[:, idx]).sum()
        inv = torch.empty(Lseq, dtype=torch.long)
        inv[torch.from_numpy(idx.copy())] = torch.arange(Lseq)
        pres.append((pre, inv))
        deltas.append(dl.detach()[:, inv])
    total.backward()
    return t, pres, torch.stack(deltas)


@pytest.mark.parametrize("kind,H,W,N", [("cross4", 5, 7, 16), ("seq2", 5, 7, 4), ("cross4", 17, 3, 4)])
def test_oracle_with_a_given_delta_matches_autograd(kind, H, W, N):
    B, D, R = 2, 8, 3
    args = _inputs(kind, B, H, W, D, N, R, f"bf16train/{kind}/{H}x{W}/N{N}")
    (xc_, xdbl_, dtw_, dtb_, A_, Ds_), pres, delta = _literal(kind, *args, H, W)
    plain, pb = R64.ss2d_ref64(kind, *args, H, W)
    # the rounded delta' lies inside the bound the GPU test holds the kernel's delta' to
    assert R64.bound_fraction(delta, plain["delta"], RD.delta_bound_bf16(plain["delta"], pb["delta"])) <= 1.0
    assert float((delta - plain["delta"]).abs().max()) > 0                        # and the rounding is really there
    ref, bnd = RD.ss2d_ref64(kind, *args, H, W, delta=delta)
    assert torch.equal(ref["delta"], delta) and float(bnd["delta"].abs().max()) == 0.0
    close = lambda a, b: float((a - b).abs().max()) <= 1e-11 * (1.0 + float(b.abs().max()))
    assert close(ref["dxc"], xc_.grad)
    assert close(ref["dB"], xdbl_.grad[..., :N]) and close(ref["dC"], xdbl_.grad[..., N:2 * N])
    assert close(ref["dA"], A_.grad) and close(ref["dDs"], Ds_.grad) and close(ref["ddtb"], dtb_.grad)
    for k, (pre, inv) in enumerate(pres):
        assert close(ref["ddelta"][k], pre.grad[:, inv]), k
    # the bounds only lose the delta' error terms
    for key in ("y", "dxc", "ddelta", "dA"):
        assert bool((bnd[key] >= 0).all()) and float(bnd[key].max()) <= 1.5 * float(pb[key].max()), key


def test_given_own_delta_changes_nothing():
    args = _inputs("cross4", 2, 5, 7, 8, 4, 3, "bf16train/self")
    plain, _ = R64.ss2d_ref64("cross4", *args, 5, 7)
    again, _ = RD.ss2d_ref64("cross4", *args, 5, 7, delta=plain["delta"])
    for key in ("y", "dxc", "dB", "dC", "dA", "dDs"):
        assert float((again[key] - plain[key]).abs().max()) <= 1e-12 * (1.0 + float(plain[key].abs().max())), key
    # and without a delta' the module is the oracle, values and bounds, bit for bit
    same, sb = RD.ss2d_ref64("cross4", *args, 5, 7)
    _, pb = R64.ss2d_ref64("cross4", *args, 5, 7)
    for key in plain:
        assert torch.equal(same[key].nan_to_num(7.0), plain[key].nan_to_num(7.0)) and torch.equal(sb[key].nan_to_num(7.0), pb[key].nan_to_num(7.0)), key


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
