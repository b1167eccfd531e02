"""The reference's nn.Module surface for the Sigma hot path, re-implemented over libsigma_b200.

Same class names, constructor arguments, forward signatures and state_dict keys as the reference
(SURVEY.md §8b), so `sigma_b200/dropin/` can expose them under the reference's import paths and the
reference's train.py / eval.py / checkpoints work unchanged:

    models.encoders.vmamba       : PatchMerging2D, SS2D, ConMB_SS2D, Cross_Mamba_Attention_SSM,
                                   CrossMambaFusion_SS2D_SSM, VSSBlock, ChannelAttention(Block),
                                   CVSSDecoderBlock, CrossMambaFusionBlock, ConcatMambaFusionBlock,
                                   VSSM, Backbone_VSSM                      (vmamba.py:612-2212)
    models.encoders.dual_vmamba  : RGBXTransformer, vssm_tiny/small/base   (dual_vmamba.py:16-143)
    models.decoders.MambaDecoder : PatchExpand, UpsampleExpand, FinalUpsample_X4, Mamba_up,
                                   MambaDecoder                             (MambaDecoder.py:12-280)
    models.builder               : EncoderDecoder                          (builder.py:13-166)

Two execution paths share the parameters:
  * inference (no grad): `sigma_b200.fused` — channels-last activations end to end, hand-written
    kernels for LayerNorm / depthwise conv+SiLU / x_proj+dt_proj+4-direction scan / merge+norm+gate
    and wgmma GEMMs, no CrossScan/CrossMerge materialisation, RGB and X streams batched as 2B;
  * training (grad enabled): the reference's composition (CrossScan -> einsum -> SelectiveScan ->
    CrossMerge) with `sigma_b200.ops.SelectiveScan` (our fwd + bwd kernels) as the scan.
There is no CPU path: forward on CPU tensors raises.
"""
import math
from collections import OrderedDict
from functools import partial
from typing import Any, Callable

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops


def trunc_normal_(t, std=0.02):
    return nn.init.trunc_normal_(t, std=std, a=-2.0, b=2.0)


class DropPath(nn.Module):
    """Stochastic depth (timm.models.layers.DropPath as used at vmamba.py:1704): identity in eval."""

    def __init__(self, drop_prob: float = 0.0):
        super().__init__()
        self.drop_prob = float(drop_prob)

    def forward(self, x):
        if self.drop_prob == 0.0 or not self.training:
            return x
        keep = 1.0 - self.drop_prob
        mask = x.new_empty((x.shape[0],) + (1,) * (x.dim() - 1)).bernoulli_(keep)
        return x * mask / keep

    def extra_repr(self):
        return f"drop_prob={self.drop_prob}"


_FORCE_COMPOSED = False


class composed_path:
    """Context manager: run the reference's op composition (the training path) even under no_grad.
    Used by the parity tests to check both paths against the same goldens."""

    def __init__(self, on=True):
        self.on = on

    def __enter__(self):
        global _FORCE_COMPOSED
        self.prev, _FORCE_COMPOSED = _FORCE_COMPOSED, self.on

    def __exit__(self, *a):
        global _FORCE_COMPOSED
        _FORCE_COMPOSED = self.prev


def _lib_kinds():
    from . import _lib
    return _lib.DIRS_CROSS4, _lib.DIRS_SEQ2


def _fused_ok(*tensors):
    """The fused inference path is taken whenever autograd is not recording."""
    if _FORCE_COMPOSED or torch.is_grad_enabled():
        return False
    for t in tensors:
        if not t.is_cuda:
            raise RuntimeError("sigma_b200 modules run on CUDA tensors only (there is no CPU path)")
    return all(t.dtype == torch.float32 for t in tensors)


FUSED_SCAN_STATES = (4, 8, 16)   # the d_state values the fused channels-last scan is built for


def _fused_block_ok(op, *tensors):
    """The fused inference path of a Mamba block (SS2D, ConMB_SS2D, CrossMambaFusion_SS2D_SSM and the blocks around them): taken
    under _fused_ok when the block's scan `op` has a d_state the fused scan is built for; any other d_state (d_state="auto" at
    most widths) runs the composed path, as under composed_path()."""
    return _fused_ok(*tensors) and op.d_state in FUSED_SCAN_STATES


# --------------------------------------------------------------------------------------------
# SSM parameter initialisers (vmamba.py:728-782; identical in SS2D / ConMB_SS2D / CMA_SSM)
# --------------------------------------------------------------------------------------------
def _dt_init(dt_rank, d_inner, dt_scale=1.0, dt_init="random", dt_min=0.001, dt_max=0.1, dt_init_floor=1e-4):
    proj = nn.Linear(dt_rank, d_inner, bias=True)
    std = dt_rank ** -0.5 * dt_scale
    if dt_init == "constant":
        nn.init.constant_(proj.weight, std)
    elif dt_init == "random":
        nn.init.uniform_(proj.weight, -std, std)
    else:
        raise NotImplementedError(dt_init)
    dt = torch.exp(torch.rand(d_inner) * (math.log(dt_max) - math.log(dt_min)) + math.log(dt_min)).clamp(min=dt_init_floor)
    with torch.no_grad():
        proj.bias.copy_(dt + torch.log(-torch.expm1(-dt)))  # softplus^-1(dt)
    return proj


def _A_log_init(d_state, d_inner, copies=-1):
    A_log = torch.log(torch.arange(1, d_state + 1, dtype=torch.float32)).repeat(d_inner, 1)  # S4D-real
    if copies > 0:
        A_log = A_log.repeat(copies, 1)
    p = nn.Parameter(A_log.contiguous())
    p._no_weight_decay = True
    return p


def _D_init(d_inner, copies=-1):
    p = nn.Parameter(torch.ones(d_inner * max(copies, 1)))
    p._no_weight_decay = True
    return p


def _dwconv(d_inner, d_conv, conv_bias):
    return nn.Conv2d(d_inner, d_inner, kernel_size=d_conv, padding=(d_conv - 1) // 2, groups=d_inner, bias=conv_bias)


# --------------------------------------------------------------------------------------------
# vmamba.py
# --------------------------------------------------------------------------------------------
class PatchMerging2D(nn.Module):
    """vmamba.py:612-636 — pad odd H/W, 2x2 gather (order [0::2,0::2],[1::2,0::2],[0::2,1::2],[1::2,1::2]),
    LayerNorm(4C), Linear(4C->2C, no bias)."""

    def __init__(self, dim, out_dim=-1, norm_layer=nn.LayerNorm):
        super().__init__()
        self.dim = dim
        self.reduction = nn.Linear(4 * dim, (2 * dim) if out_dim < 0 else out_dim, bias=False)
        self.norm = norm_layer(4 * dim)

    def forward(self, x):
        if _fused_ok(x):
            from . import fused
            return fused.patch_merging(self, x)
        H, W = x.shape[-3:-1]
        if (W % 2) or (H % 2):
            x = F.pad(x, (0, 0, 0, W % 2, 0, H % 2))
        x = torch.cat([x[..., 0::2, 0::2, :], x[..., 1::2, 0::2, :], x[..., 0::2, 1::2, :], x[..., 1::2, 1::2, :]], -1)
        return self.reduction(ops.layer_norm(self.norm, x))


class SS2D(nn.Module):
    """vmamba.py:640-1089 (forward_core = forward_corev2, K = 4)."""

    def __init__(self, d_model=96, d_state=16, ssm_ratio=2, dt_rank="auto", d_conv=3, conv_bias=True, dropout=0.0,
                 bias=False, dt_min=0.001, dt_max=0.1, dt_init="random", dt_scale=1.0, dt_init_floor=1e-4,
                 softmax_version=False, **kwargs):
        super().__init__()
        if softmax_version or d_conv < 2:
            raise NotImplementedError("sigma_b200.SS2D covers the Sigma configuration: d_conv=3, softmax_version=False")
        self.softmax_version = False
        self.d_model = d_model
        self.d_state = math.ceil(d_model / 6) if d_state == "auto" else d_state
        self.d_conv = d_conv
        self.expand = ssm_ratio
        self.d_inner = int(ssm_ratio * d_model)
        self.dt_rank = math.ceil(d_model / 16) if dt_rank == "auto" else dt_rank
        self.K = self.K2 = 4

        self.in_proj = nn.Linear(d_model, self.d_inner * 2, bias=bias)
        self.conv2d = _dwconv(self.d_inner, d_conv, conv_bias)
        self.act = nn.SiLU()
        xp = [nn.Linear(self.d_inner, self.dt_rank + 2 * self.d_state, bias=False) for _ in range(self.K)]
        self.x_proj_weight = nn.Parameter(torch.stack([t.weight for t in xp], dim=0))          # (K, R+2N, D)
        dtp = [_dt_init(self.dt_rank, self.d_inner, dt_scale, dt_init, dt_min, dt_max, dt_init_floor) for _ in range(self.K)]
        self.dt_projs_weight = nn.Parameter(torch.stack([t.weight for t in dtp], dim=0))       # (K, D, R)
        self.dt_projs_bias = nn.Parameter(torch.stack([t.bias for t in dtp], dim=0))           # (K, D)
        self.A_logs = _A_log_init(self.d_state, self.d_inner, copies=self.K2)                  # (K*D, N)
        self.Ds = _D_init(self.d_inner, copies=self.K2)                                        # (K*D)
        self.out_norm = nn.LayerNorm(self.d_inner)
        self.out_proj = nn.Linear(self.d_inner, d_model, bias=bias)
        self.dropout = nn.Dropout(dropout) if dropout > 0.0 else nn.Identity()

    def forward_core(self, x, nrows=-1):
        """cross_selective_scan (vmamba.py:165-226): x (B,D,H,W) -> (B,H,W,D), out_norm applied."""
        return ops.cross_selective_scan(x, self.x_proj_weight, None, self.dt_projs_weight, self.dt_projs_bias,
                                        self.A_logs, self.Ds, self.out_norm, nrows=nrows)

    forward_corev2 = forward_core

    def forward(self, x, residual=None, **kwargs):
        if _fused_block_ok(self, x) and isinstance(self.dropout, nn.Identity):
            from . import fused
            return fused.ss2d(self, x, residual=residual)
        xz = self.in_proj(x)
        xi, z = xz.chunk(2, dim=-1)
        if ops.fused_core_ok(x, self.d_inner, self.d_state):
            # training through the fused core (f1): conv on the channels_last view, then x_proj + 4-direction scan + CrossMerge as
            # ONE autograd node over channels-last tensors (no CrossScan / delta / CrossMerge copies in either direction)
            B, H, W, _ = x.shape
            xc = ops.DwConvSiLUFn.apply(xi, self.conv2d.weight, self.conv2d.bias)   # (B, H·W, D), xi read in place
            y = ops.FusedSS2DCore.apply(xc, self.x_proj_weight, self.dt_projs_weight, self.dt_projs_bias, self.A_logs, self.Ds,
                                        _lib_kinds()[0], H, W)
            y = ops.layer_norm(self.out_norm, y.view(B, H, W, self.d_inner)).to(x.dtype) * F.silu(z)
        else:
            xi = self.act(self.conv2d(xi.permute(0, 3, 1, 2).contiguous()))
            y = self.forward_core(xi) * F.silu(z)
        out = self.dropout(self.out_proj(y))
        return out if residual is None else residual + out


class ConMB_SS2D(nn.Module):
    """vmamba.py:1092-1284 — concat-Mamba: [rgb ‖ x] along L, forward + reversed scan (K=2), SE cross-gating."""

    def __init__(self, d_model=96, d_state=4, ssm_ratio=2, dt_rank="auto", d_conv=3, conv_bias=True, dropout=0.0,
                 bias=False, dt_min=0.001, dt_max=0.1, dt_init="random", dt_scale=1.0, dt_init_floor=1e-4,
                 softmax_version=False, **kwargs):
        super().__init__()
        if softmax_version or d_conv < 2:
            raise NotImplementedError("sigma_b200.ConMB_SS2D covers d_conv=3, softmax_version=False")
        self.softmax_version = False
        self.d_model = d_model
        self.d_state = math.ceil(d_model / 6) if d_state == "auto" else d_state
        self.d_conv = d_conv
        self.expand = ssm_ratio
        self.d_inner = int(ssm_ratio * d_model)
        self.dt_rank = math.ceil(d_model / 16) if dt_rank == "auto" else dt_rank
        self.K = self.K2 = 2
        D = self.d_inner

        self.in_proj = nn.Linear(d_model, D, bias=bias)
        self.in_proj_modalx = nn.Linear(d_model, D, bias=bias)
        self.conv2d = _dwconv(D, d_conv, conv_bias)
        self.conv2d_modalx = _dwconv(D, d_conv, conv_bias)
        self.act = nn.SiLU()
        xp = [nn.Linear(D, self.dt_rank + 2 * self.d_state, bias=False) for _ in range(self.K)]
        self.x_proj_weight = nn.Parameter(torch.stack([t.weight for t in xp], dim=0))
        dtp = [_dt_init(self.dt_rank, D, dt_scale, dt_init, dt_min, dt_max, dt_init_floor) for _ in range(self.K)]
        self.dt_projs_weight = nn.Parameter(torch.stack([t.weight for t in dtp], dim=0))
        self.dt_projs_bias = nn.Parameter(torch.stack([t.bias for t in dtp], dim=0))
        self.A_logs = _A_log_init(self.d_state, D, copies=self.K2)
        self.Ds = _D_init(D, copies=self.K2)
        self.out_norm1 = nn.LayerNorm(D)
        self.out_norm2 = nn.LayerNorm(D)
        self.out_proj = nn.Linear(D * 2, d_model, bias=bias)
        self.dropout = nn.Dropout(dropout) if dropout > 0.0 else nn.Identity()
        self.avg_pool = nn.AdaptiveAvgPool2d(1)

        def se():
            return nn.Sequential(nn.Linear(D, D // 16, bias=False), nn.SiLU(inplace=True),
                                 nn.Linear(D // 16, D, bias=False), nn.Sigmoid())
        self.fc1, self.fc2 = se(), se()

    def forward_corev2_multimodal(self, x_rgb, x_e, nrows=-1):
        return ops.cross_selective_scan_multimodal_k2(
            x_rgb, x_e, self.x_proj_weight, None, self.dt_projs_weight, self.dt_projs_bias, self.A_logs, self.Ds,
            self.out_norm1, self.out_norm2, nrows=nrows)

    def forward(self, x_rgb, x_e, residual=None):
        if _fused_block_ok(self, x_rgb, x_e) and isinstance(self.dropout, nn.Identity):
            from . import fused
            return fused.conmb_ss2d(self, x_rgb, x_e, residual=residual)
        if ops.fused_core_ok(x_rgb, self.d_inner, self.d_state):
            # training through the fused core (f1), kind SEQ2: [rgb ‖ x] along L, forward + reversed scan, merged; channels-last
            # throughout (the conv + SiLU nodes read the in_proj outputs in place)
            B, H, W, _ = x_rgb.shape
            D, L = self.d_inner, H * W
            t_r, t_e = self.in_proj(x_rgb), self.in_proj_modalx(x_e)                                            # (B, H, W, D)
            c_r = ops.DwConvSiLUFn.apply(t_r, self.conv2d.weight, self.conv2d.bias)
            c_e = ops.DwConvSiLUFn.apply(t_e, self.conv2d_modalx.weight, self.conv2d_modalx.bias)
            ys = ops.FusedSS2DCore.apply(torch.cat([c_r, c_e], dim=1), self.x_proj_weight, self.dt_projs_weight, self.dt_projs_bias,
                                         self.A_logs, self.Ds, _lib_kinds()[1], H, W)                          # (B, 2L, D)
            y_r = ops.layer_norm(self.out_norm1, ys[:, :L].reshape(B, H, W, D)).to(x_rgb.dtype)
            y_e = ops.layer_norm(self.out_norm2, ys[:, L:].reshape(B, H, W, D)).to(x_e.dtype)
            hw = (1, 2)
        else:
            t_r = self.in_proj(x_rgb).permute(0, 3, 1, 2).contiguous()
            t_e = self.in_proj_modalx(x_e).permute(0, 3, 1, 2).contiguous()
            y_r, y_e = self.forward_corev2_multimodal(self.act(self.conv2d(t_r)), self.act(self.conv2d_modalx(t_e)))
            hw = (2, 3)
        g_r = self.fc1(t_r.mean(dim=hw))             # gates come from the PRE-conv projections (vmamba.py:1276-1279)
        g_e = self.fc2(t_e.mean(dim=hw))
        y = torch.cat([y_r * g_e[:, None, None, :], y_e * g_r[:, None, None, :]], dim=-1)  # cross-applied (:1280-1281)
        out = self.dropout(self.out_proj(y))
        return out if residual is None else residual + out


class Cross_Mamba_Attention_SSM(nn.Module):
    """vmamba.py:1407-1545 — two single-direction scans, each reading the OTHER modality's C."""

    def __init__(self, d_model=96, d_state=4, ssm_ratio=2, dt_rank="auto", dt_min=0.001, dt_max=0.1,
                 dt_init="random", dt_scale=1.0, dt_init_floor=1e-4, **kwargs):
        super().__init__()
        self.d_model = d_model
        self.d_state = math.ceil(d_model / 6) if d_state == "auto" else d_state
        self.expand = ssm_ratio
        self.d_inner = int(ssm_ratio * d_model)
        self.dt_rank = math.ceil(d_model / 16) if dt_rank == "auto" else dt_rank
        D = self.d_inner
        self.x_proj_1 = nn.Linear(D, self.dt_rank + 2 * self.d_state, bias=False)
        self.x_proj_2 = nn.Linear(D, self.dt_rank + 2 * self.d_state, bias=False)
        self.dt_proj_1 = _dt_init(self.dt_rank, D, dt_scale, dt_init, dt_min, dt_max, dt_init_floor)
        self.dt_proj_2 = _dt_init(self.dt_rank, D, dt_scale, dt_init, dt_min, dt_max, dt_init_floor)
        self.A_log_1 = _A_log_init(self.d_state, D)
        self.A_log_2 = _A_log_init(self.d_state, D)
        self.D_1 = _D_init(D)
        self.D_2 = _D_init(D)
        self.out_norm_1 = nn.LayerNorm(D)
        self.out_norm_2 = nn.LayerNorm(D)

    def forward(self, x_rgb, x_e):
        """x_*: (B, L, D) -> (B, L, D) each."""
        R, N = self.dt_rank, self.d_state

        def proj(x, xp, dtp):
            dt, Bm, Cm = torch.split(xp(x), [R, N, N], dim=-1)
            dt = F.linear(dt, dtp.weight).transpose(1, 2)                       # (B, D, L); bias goes in as delta_bias
            return dt, Bm.transpose(1, 2).contiguous(), Cm.transpose(1, 2).contiguous()

        dt_r, B_r, C_r = proj(x_rgb, self.x_proj_1, self.dt_proj_1)
        dt_e, B_e, C_e = proj(x_e, self.x_proj_2, self.dt_proj_2)
        y_r = ops.selective_scan_fn(x_rgb.transpose(1, 2), dt_r, -torch.exp(self.A_log_1.float()), B_r, C_e,
                                    self.D_1.float(), self.dt_proj_1.bias.float(), True)
        y_e = ops.selective_scan_fn(x_e.transpose(1, 2), dt_e, -torch.exp(self.A_log_2.float()), B_e, C_r,
                                    self.D_2.float(), self.dt_proj_2.bias.float(), True)
        return ops.layer_norm(self.out_norm_1, y_r.transpose(1, 2)), ops.layer_norm(self.out_norm_2, y_e.transpose(1, 2))


class CrossMambaFusion_SS2D_SSM(nn.Module):
    """vmamba.py:1549-1640.  Note the single conv2d shared by both modalities (:1629-1630)."""

    def __init__(self, d_model=96, d_state=16, ssm_ratio=2, dt_rank="auto", d_conv=3, conv_bias=True, dropout=0.0,
                 bias=False, dt_min=0.001, dt_max=0.1, dt_init="random", dt_scale=1.0, dt_init_floor=1e-4,
                 softmax_version=False, **kwargs):
        super().__init__()
        if d_conv < 2:
            raise NotImplementedError("sigma_b200.CrossMambaFusion_SS2D_SSM covers d_conv=3")
        self.softmax_version = softmax_version
        self.d_model = d_model
        self.d_state = math.ceil(d_model / 6) if d_state == "auto" else d_state
        self.d_conv = d_conv
        self.expand = ssm_ratio
        self.d_inner = int(ssm_ratio * d_model)
        self.dt_rank = math.ceil(d_model / 16) if dt_rank == "auto" else dt_rank
        D = self.d_inner
        self.in_proj = nn.Linear(d_model, D, bias=bias)
        self.in_proj_modalx = nn.Linear(d_model, D, bias=bias)
        self.conv2d = _dwconv(D, d_conv, conv_bias)
        self.act = nn.SiLU()
        self.out_proj_rgb = nn.Linear(D, d_model, bias=bias)
        self.out_proj_e = nn.Linear(D, d_model, bias=bias)
        self.dropout_rgb = nn.Dropout(dropout) if dropout > 0.0 else nn.Identity()
        self.dropout_e = nn.Dropout(dropout) if dropout > 0.0 else nn.Identity()
        self.CMA_ssm = Cross_Mamba_Attention_SSM(d_model=d_model, d_state=self.d_state, ssm_ratio=ssm_ratio,
                                                 dt_rank=dt_rank, dt_min=dt_min, dt_max=dt_max, dt_init=dt_init,
                                                 dt_scale=dt_scale, dt_init_floor=dt_init_floor, **kwargs)

    def forward(self, x_rgb, x_e, residual=False):
        if _fused_block_ok(self, x_rgb, x_e) and isinstance(self.dropout_rgb, nn.Identity):
            from . import fused
            return fused.cromb_ss2d(self, x_rgb, x_e, residual=residual)
        B, H, W, _ = x_rgb.shape
        if ops.fused_core_ok(x_rgb, self.d_inner, self.d_state) and not ops.deterministic():
            # training through the fused core (f1), kind CROSS: both modalities as one 2·B batch, channels-last throughout.  Under
            # the deterministic switch the composed path below runs (the op-level _det kernels; CROSS has no _det build)
            from . import _lib
            D, cm = self.d_inner, self.CMA_ssm
            t = torch.cat([self.in_proj(x_rgb), self.in_proj_modalx(x_e)], dim=0)             # (2B, H, W, D)
            xc = ops.DwConvSiLUFn.apply(t, self.conv2d.weight, self.conv2d.bias)                # one shared conv over 2B images
            y = ops.FusedSS2DCore.apply(xc, torch.stack([cm.x_proj_1.weight, cm.x_proj_2.weight]),
                                        torch.stack([cm.dt_proj_1.weight, cm.dt_proj_2.weight]),
                                        torch.stack([cm.dt_proj_1.bias, cm.dt_proj_2.bias]), torch.cat([cm.A_log_1, cm.A_log_2]),
                                        torch.cat([cm.D_1, cm.D_2]), _lib.DIRS_CROSS, H, W)                # (2B, L, D)
            y_r = ops.layer_norm(cm.out_norm_1, y[:B])
            y_e = ops.layer_norm(cm.out_norm_2, y[B:])
        else:
            c_r = self.act(self.conv2d(self.in_proj(x_rgb).permute(0, 3, 1, 2).contiguous()))
            c_e = self.act(self.conv2d(self.in_proj_modalx(x_e).permute(0, 3, 1, 2).contiguous()))
            y_r, y_e = self.CMA_ssm(c_r.flatten(2).transpose(1, 2), c_e.flatten(2).transpose(1, 2))
        o_r = self.dropout_rgb(self.out_proj_rgb(y_r.view(B, H, W, -1)))
        o_e = self.dropout_e(self.out_proj_e(y_e.view(B, H, W, -1)))
        return (x_rgb + o_r, x_e + o_e) if residual else (o_r, o_e)


class Permute(nn.Module):
    def __init__(self, *args):
        super().__init__()
        self.args = args

    def forward(self, x):
        return x.permute(*self.args)


class Mlp(nn.Module):
    """vmamba.py:1652-1670 (unused by Sigma: mlp_ratio = 0 everywhere on the path)."""

    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.GELU, drop=0.0,
                 channels_first=False):
        super().__init__()
        out_features = out_features or in_features
        hidden_features = hidden_features or in_features
        Linear = partial(nn.Conv2d, kernel_size=1, padding=0) if channels_first else nn.Linear
        self.fc1 = Linear(in_features, hidden_features)
        self.act = act_layer()
        self.fc2 = Linear(hidden_features, out_features)
        self.drop = nn.Dropout(drop)

    def forward(self, x):
        return self.drop(self.fc2(self.drop(self.act(self.fc1(x)))))


class VSSBlock(nn.Module):
    """vmamba.py:1673-1722 — x + DropPath(SS2D(LN(x))) [+ FFN when mlp_ratio > 0]."""

    def __init__(self, hidden_dim: int = 0, drop_path: float = 0, norm_layer: Callable[..., nn.Module] = partial(nn.LayerNorm, eps=1e-6),
                 attn_drop_rate: float = 0, d_state: int = 16, dt_rank: Any = "auto", ssm_ratio=2.0, shared_ssm=False,
                 softmax_version=False, use_checkpoint: bool = False, mlp_ratio=4.0, act_layer=nn.GELU, drop: float = 0.0,
                 **kwargs):
        super().__init__()
        self.use_checkpoint = use_checkpoint
        self.norm = norm_layer(hidden_dim)
        self.op = SS2D(d_model=hidden_dim, dropout=attn_drop_rate, d_state=d_state, ssm_ratio=ssm_ratio, dt_rank=dt_rank,
                       shared_ssm=shared_ssm, softmax_version=softmax_version, **kwargs)
        self.drop_path = DropPath(drop_path)
        self.mlp_branch = mlp_ratio > 0
        if self.mlp_branch:
            self.norm2 = norm_layer(hidden_dim)
            self.mlp = Mlp(in_features=hidden_dim, hidden_features=int(hidden_dim * mlp_ratio), act_layer=act_layer, drop=drop)

    def _forward(self, input):
        if _fused_block_ok(self.op, input) and not self.mlp_branch:
            from . import fused
            return fused.vss_block(self, input)
        x = input + self.drop_path(self.op(ops.layer_norm(self.norm, input)))
        if self.mlp_branch:
            x = x + self.drop_path(self.mlp(ops.layer_norm(self.norm2, x)))
        return x

    def forward(self, input):
        if self.use_checkpoint and torch.is_grad_enabled():
            return torch.utils.checkpoint.checkpoint(self._forward, input, use_reentrant=False)
        return self._forward(input)


class ChannelAttention(nn.Module):
    """vmamba.py:1725-1741."""

    def __init__(self, num_feat, squeeze_factor=16):
        super().__init__()
        self.avg_pool = nn.AdaptiveAvgPool2d(1)
        self.max_pool = nn.AdaptiveMaxPool2d(1)
        self.fc = nn.Sequential(nn.Conv2d(num_feat, num_feat // squeeze_factor, 1, bias=False), nn.SiLU(inplace=True),
                                nn.Conv2d(num_feat // squeeze_factor, num_feat, 1, bias=False))
        self.sigmoid = nn.Sigmoid()

    def forward(self, x):
        # global pools as plain reductions (same values and, away from exact ties, same gradients as AdaptiveAvg/MaxPool2d(1);
        # adaptive_max_pool2d's backward kernel alone cost 3.7 ms of the Sigma-tiny training step)
        avg, mx = x.mean(dim=(2, 3), keepdim=True), x.amax(dim=(2, 3), keepdim=True)
        return x * self.sigmoid(self.fc(avg) + self.fc(mx))


class ChannelAttentionBlock(nn.Module):
    """vmamba.py:1744-1757 — conv3x3(C->C/3), GELU, conv3x3(C/3->C), channel attention (squeeze 30)."""

    def __init__(self, num_feat, compress_ratio=3, squeeze_factor=30):
        super().__init__()
        self.cab = nn.Sequential(nn.Conv2d(num_feat, num_feat // compress_ratio, 3, 1, 1), nn.GELU(),
                                 nn.Conv2d(num_feat // compress_ratio, num_feat, 3, 1, 1),
                                 ChannelAttention(num_feat, squeeze_factor))

    def forward(self, x):
        return self.cab(x)


class CVSSDecoderBlock(nn.Module):
    """vmamba.py:1760-1811 — x·scale1 + SS2D(LN(x)); then CAB(LN(x)) + x·scale2.  mlp_ratio is ignored."""

    def __init__(self, hidden_dim: int = 0, drop_path: float = 0, norm_layer: Callable[..., nn.Module] = partial(nn.LayerNorm, eps=1e-6),
                 attn_drop_rate: float = 0, d_state: int = 16, dt_rank: Any = "auto", ssm_ratio=2.0, shared_ssm=False,
                 softmax_version=False, use_checkpoint: bool = False, mlp_ratio=4.0, act_layer=nn.GELU, drop: float = 0.0,
                 **kwargs):
        super().__init__()
        self.use_checkpoint = use_checkpoint
        self.norm1 = norm_layer(hidden_dim)
        self.scale1 = nn.Parameter(torch.ones(hidden_dim))
        self.op = SS2D(d_model=hidden_dim, dropout=attn_drop_rate, d_state=d_state, ssm_ratio=ssm_ratio, dt_rank=dt_rank,
                       shared_ssm=shared_ssm, softmax_version=softmax_version, **kwargs)
        self.drop_path = DropPath(drop_path)
        self.conv_blk = ChannelAttentionBlock(hidden_dim)
        self.norm2 = norm_layer(hidden_dim)
        self.scale2 = nn.Parameter(torch.ones(hidden_dim))

    def _forward(self, input):
        if _fused_block_ok(self.op, input):
            from . import fused
            return fused.cvss_decoder_block(self, input)
        x = input * self.scale1 + self.drop_path(self.op(ops.layer_norm(self.norm1, input)))
        cab = self.conv_blk.cab
        fn = None if _FORCE_COMPOSED else ops.cab_conv_fn(cab, x)
        if fn is not None:
            # channels-last throughout: the convs as one CabConvFn / CabConvPitchedFn, then ChannelAttention.forward's arithmetic
            # over (H, W)
            t = fn.apply(ops.layer_norm(self.norm2, x), cab[0].weight, cab[0].bias, cab[2].weight, cab[2].bias)
            ca = cab[3]
            avg, mx = t.mean(dim=(1, 2), keepdim=True), t.amax(dim=(1, 2), keepdim=True)
            attn = ca.sigmoid(ca.fc(avg.permute(0, 3, 1, 2)) + ca.fc(mx.permute(0, 3, 1, 2)))
            return t * attn.permute(0, 2, 3, 1) + x * self.scale2
        y = self.conv_blk(ops.layer_norm(self.norm2, x).permute(0, 3, 1, 2).contiguous()) + (x * self.scale2).permute(0, 3, 1, 2)
        return y.permute(0, 2, 3, 1).contiguous()

    def forward(self, input):
        if self.use_checkpoint and torch.is_grad_enabled():
            return torch.utils.checkpoint.checkpoint(self._forward, input, use_reentrant=False)
        return self._forward(input)


class CrossMambaFusionBlock(nn.Module):
    """vmamba.py:1814-1870 (CroMB)."""

    def __init__(self, hidden_dim: int = 0, drop_path: float = 0, norm_layer: Callable[..., nn.Module] = partial(nn.LayerNorm, eps=1e-6),
                 attn_drop_rate: float = 0, d_state: int = 4, dt_rank: Any = "auto", ssm_ratio=2.0, shared_ssm=False,
                 softmax_version=False, use_checkpoint: bool = False, mlp_ratio=0.0, act_layer=nn.GELU, drop: float = 0.0,
                 **kwargs):
        super().__init__()
        self.use_checkpoint = use_checkpoint
        self.op = CrossMambaFusion_SS2D_SSM(d_model=hidden_dim, dropout=attn_drop_rate, d_state=d_state, ssm_ratio=ssm_ratio,
                                            dt_rank=dt_rank, shared_ssm=shared_ssm, softmax_version=softmax_version, **kwargs)
        self.drop_path1 = DropPath(drop_path)
        self.drop_path2 = DropPath(drop_path)
        self.mlp_branch = mlp_ratio > 0
        if self.mlp_branch:
            self.norm2 = norm_layer(hidden_dim)
            self.mlp = Mlp(in_features=hidden_dim, hidden_features=int(hidden_dim * mlp_ratio), act_layer=act_layer, drop=drop)

    def _forward(self, x_rgb, x_e):
        if _fused_block_ok(self.op, x_rgb, x_e):
            return self.op(x_rgb, x_e, residual=True)
        c_r, c_e = self.op(x_rgb, x_e)
        return x_rgb + self.drop_path1(c_r), x_e + self.drop_path2(c_e)

    def forward(self, x_rgb, x_e):
        if self.use_checkpoint and torch.is_grad_enabled():
            return torch.utils.checkpoint.checkpoint(self._forward, x_rgb, x_e, use_reentrant=False)
        return self._forward(x_rgb, x_e)


class ConcatMambaFusionBlock(nn.Module):
    """vmamba.py:1873-1928 (ConMB): x_rgb + x_e + op(x_rgb, x_e)."""

    def __init__(self, hidden_dim: int = 0, drop_path: float = 0, norm_layer: Callable[..., nn.Module] = partial(nn.LayerNorm, eps=1e-6),
                 attn_drop_rate: float = 0, d_state: int = 4, dt_rank: Any = "auto", ssm_ratio=2.0, shared_ssm=False,
                 softmax_version=False, use_checkpoint: bool = False, mlp_ratio=0.0, act_layer=nn.GELU, drop: float = 0.0,
                 **kwargs):
        super().__init__()
        self.use_checkpoint = use_checkpoint
        self.op = ConMB_SS2D(d_model=hidden_dim, dropout=attn_drop_rate, d_state=d_state, ssm_ratio=ssm_ratio,
                             dt_rank=dt_rank, shared_ssm=shared_ssm, softmax_version=softmax_version, **kwargs)
        self.drop_path = DropPath(drop_path)
        self.mlp_branch = mlp_ratio > 0
        if self.mlp_branch:
            self.norm2 = norm_layer(hidden_dim)
            self.mlp = Mlp(in_features=hidden_dim, hidden_features=int(hidden_dim * mlp_ratio), act_layer=act_layer, drop=drop)

    def _forward(self, x_rgb, x_e):
        if _fused_block_ok(self.op, x_rgb, x_e) and not self.mlp_branch:
            return self.op(x_rgb, x_e, residual=x_rgb + x_e)     # the sum is added in the out_proj GEMM epilogue
        x = x_rgb + x_e + self.drop_path(self.op(x_rgb, x_e))
        if self.mlp_branch:
            x = x + self.drop_path(self.mlp(ops.layer_norm(self.norm2, x)))
        return x

    def forward(self, x_rgb, x_e):
        if self.use_checkpoint and torch.is_grad_enabled():
            return torch.utils.checkpoint.checkpoint(self._forward, x_rgb, x_e, use_reentrant=False)
        return self._forward(x_rgb, x_e)


class VSSM(nn.Module):
    """vmamba.py:1931-2147."""

    def __init__(self, patch_size=4, in_chans=3, num_classes=1000, depths=[2, 2, 9, 2], dims=[96, 192, 384, 768],
                 d_state=16, dt_rank="auto", ssm_ratio=2.0, attn_drop_rate=0.0, shared_ssm=False, softmax_version=False,
                 drop_rate=0.0, drop_path_rate=0.1, mlp_ratio=4.0, patch_norm=True, norm_layer=nn.LayerNorm,
                 downsample_version: str = "v2", use_checkpoint=False, **kwargs):
        super().__init__()
        self.num_classes = num_classes
        self.num_layers = len(depths)
        if isinstance(dims, int):
            dims = [int(dims * 2 ** i) for i in range(self.num_layers)]
        self.embed_dim, self.num_features, self.dims = dims[0], dims[-1], dims
        self.patch_embed = nn.Sequential(
            nn.Conv2d(in_chans, self.embed_dim, kernel_size=patch_size, stride=patch_size, bias=True),
            Permute(0, 2, 3, 1),
            norm_layer(self.embed_dim) if patch_norm else nn.Identity())
        dpr = [v.item() for v in torch.linspace(0, drop_path_rate, sum(depths))]
        self.layers = nn.ModuleList()
        for i in range(self.num_layers):
            if i < self.num_layers - 1:
                if downsample_version == "v2":
                    down = nn.Sequential(Permute(0, 3, 1, 2), nn.Conv2d(dims[i], dims[i + 1], kernel_size=2, stride=2),
                                         Permute(0, 2, 3, 1), norm_layer(dims[i + 1]))
                else:
                    down = PatchMerging2D(dims[i], dims[i + 1], norm_layer=norm_layer)
            else:
                down = nn.Identity()
            blocks = [VSSBlock(hidden_dim=dims[i], drop_path=dpr[sum(depths[:i]) + j], norm_layer=norm_layer,
                               attn_drop_rate=attn_drop_rate, d_state=d_state, dt_rank=dt_rank, ssm_ratio=ssm_ratio,
                               shared_ssm=shared_ssm, softmax_version=softmax_version, use_checkpoint=use_checkpoint,
                               mlp_ratio=mlp_ratio, act_layer=nn.GELU, drop=drop_rate) for j in range(depths[i])]
            self.layers.append(nn.Sequential(OrderedDict(blocks=nn.Sequential(*blocks), downsample=down)))
        self.classifier = nn.Sequential(OrderedDict(
            norm=norm_layer(self.num_features), permute=Permute(0, 3, 1, 2), avgpool=nn.AdaptiveAvgPool2d(1),
            flatten=nn.Flatten(1), head=nn.Linear(self.num_features, num_classes)))
        self.apply(self._init_weights)

    def _init_weights(self, m):
        if isinstance(m, nn.Linear):
            trunc_normal_(m.weight, std=0.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    def forward(self, x):
        x = self.patch_embed(x)
        for layer in self.layers:
            x = layer(x)
        return self.classifier(x)

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        """Accept checkpoints of the original VMamba training code (renames of vmamba.py:2111-2147)."""
        renames = [("patch_embed.proj", "patch_embed.0"), ("patch_embed.norm", "patch_embed.2")]
        for k in list(state_dict.keys()):
            if not k.startswith(prefix):
                continue
            new = k[len(prefix):]
            for src, dst in renames:
                if new.startswith(src):
                    new = dst + new[len(src):]
            new = new.replace(".ln_1.", ".norm.").replace(".self_attention.", ".op.")
            if new.startswith("norm."):
                new = "classifier." + new
            if new.startswith("head."):
                new = "classifier." + new
            if prefix + new != k:
                state_dict[prefix + new] = state_dict.pop(k)
        return super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs)


class Backbone_VSSM(VSSM):
    """vmamba.py:2151-2212 — per-stage outnorm{i}, NCHW outputs."""

    def __init__(self, patch_size=4, in_chans=3, num_classes=1000, depths=[2, 2, 9, 2], dims=[96, 192, 384, 768],
                 d_state=16, ssm_ratio=2.0, attn_drop_rate=0.0, drop_rate=0.0, drop_path_rate=0.1, mlp_ratio=4.0,
                 patch_norm=True, norm_layer=nn.LayerNorm, downsample_version: str = "v2", use_checkpoint=False,
                 out_indices=(0, 1, 2, 3), pretrained=None, **kwargs):
        super().__init__(patch_size=patch_size, in_chans=in_chans, num_classes=num_classes, depths=depths, dims=dims,
                         d_state=d_state, ssm_ratio=ssm_ratio, attn_drop_rate=attn_drop_rate, drop_rate=drop_rate,
                         drop_path_rate=drop_path_rate, mlp_ratio=mlp_ratio, patch_norm=patch_norm, norm_layer=norm_layer,
                         downsample_version=downsample_version, use_checkpoint=use_checkpoint, **kwargs)
        self.out_indices = out_indices
        for i in out_indices:
            self.add_module(f"outnorm{i}", norm_layer(self.dims[i]))
        del self.classifier
        self.load_pretrained(pretrained)

    def load_pretrained(self, ckpt=None, key="model"):
        if ckpt is None:
            return
        try:
            _ckpt = torch.load(open(ckpt, "rb"), map_location=torch.device("cpu"))
            print(f"Successfully load ckpt {ckpt}")
            print("incompatible:", self.load_state_dict(_ckpt[key], strict=False))
        except Exception as e:  # the reference swallows this too (vmamba.py:2190-2191)
            print(f"Failed loading checkpoint form {ckpt}: {e}")

    def forward_nhwc(self, x):
        """Stage outputs (after outnorm{i}) in channels-last (B,H,W,C) — used by the fused encoder."""
        fused_ln = None
        if _fused_ok(x):
            from . import fused
            fused_ln = fused.ln_nhwc
            pe = fused.patch_embed(self.patch_embed[0], x)      # 4x4 / stride-4 conv = re-ordering + our GEMM (no cuDNN)
            # otherwise: channels_last input -> cuDNN's NHWC kernel -> the (B,H,W,C) view is contiguous (no transposing copy)
            x = pe if pe is not None else self.patch_embed[0](x.contiguous(memory_format=torch.channels_last)).permute(0, 2, 3, 1)
            x = fused_ln(self.patch_embed[2], x) if isinstance(self.patch_embed[2], nn.LayerNorm) else x.contiguous()
        else:
            x = self.patch_embed(x)
        outs = []
        for i, layer in enumerate(self.layers):
            x = layer.blocks(x)
            if i in self.out_indices:
                norm = getattr(self, f"outnorm{i}")
                outs.append(fused_ln(norm, x) if fused_ln and isinstance(norm, nn.LayerNorm) else norm(x))
            x = layer.downsample(x)
        return outs

    def forward(self, x):
        if len(self.out_indices) == 0:
            x = self.patch_embed(x)
            for layer in self.layers:
                x = layer.downsample(layer.blocks(x))
            return x
        return [o.permute(0, 3, 1, 2).contiguous() for o in self.forward_nhwc(x)]


# --------------------------------------------------------------------------------------------
# dual_vmamba.py
# --------------------------------------------------------------------------------------------
class RGBXTransformer(nn.Module):
    """dual_vmamba.py:16-110 — Siamese VMamba encoder + CroMB + ConMB per stage."""

    def __init__(self, num_classes=1000, norm_layer=nn.LayerNorm, depths=[2, 2, 27, 2], dims=96, pretrained=None,
                 mlp_ratio=4.0, downsample_version="v1", ape=False, img_size=[480, 640], patch_size=4,
                 drop_path_rate=0.2, **kwargs):
        super().__init__()
        if ape:
            raise NotImplementedError("absolute position embedding is a discarded option of the reference (dual_vmamba.py:92)")
        self.ape = False
        self.vssm = Backbone_VSSM(pretrained=pretrained, norm_layer=norm_layer, num_classes=num_classes, depths=depths,
                                  dims=dims, mlp_ratio=mlp_ratio, downsample_version=downsample_version,
                                  drop_path_rate=drop_path_rate)
        self.cross_mamba = nn.ModuleList(CrossMambaFusionBlock(hidden_dim=dims * (2 ** i), mlp_ratio=0.0, d_state=4) for i in range(4))
        self.channel_attn_mamba = nn.ModuleList(ConcatMambaFusionBlock(hidden_dim=dims * (2 ** i), mlp_ratio=0.0, d_state=4) for i in range(4))

    def forward_features(self, x_rgb, x_e):
        B = x_rgb.shape[0]
        # Siamese: one weight set, both streams in one 2B batch (the reference runs them back to back,
        # dual_vmamba.py:85-86; LayerNorm-only network, so batching is exact)
        if _fused_ok(x_rgb):
            # the 2B batch is assembled directly in channels_last memory (what the patch-embed conv wants)
            x2 = torch.empty((2 * B,) + tuple(x_rgb.shape[1:]), dtype=x_rgb.dtype, device=x_rgb.device,
                             memory_format=torch.channels_last)
            x2[:B].copy_(x_rgb)
            x2[B:].copy_(x_e)
        else:
            x2 = torch.cat([x_rgb, x_e], dim=0)
        outs = self.vssm.forward_nhwc(x2)
        fused = []
        for i in range(4):
            o_r, o_x = outs[i][:B], outs[i][B:]
            c_r, c_x = self.cross_mamba[i](o_r, o_x)
            # NCHW-shaped like the reference's outputs, channels_last in memory: the decoder (and any 1x1 conv) reads it
            # without a transposing copy
            fused.append(self.channel_attn_mamba[i](c_r, c_x).permute(0, 3, 1, 2))
        return fused

    def forward(self, x_rgb, x_e):
        return self.forward_features(x_rgb, x_e)


class vssm_tiny(RGBXTransformer):
    def __init__(self, fuse_cfg=None, **kwargs):
        super().__init__(depths=[2, 2, 9, 2], dims=96, pretrained="pretrained/vmamba/vssmtiny_dp01_ckpt_epoch_292.pth",
                         mlp_ratio=0.0, downsample_version="v1", drop_path_rate=0.2)


class vssm_small(RGBXTransformer):
    def __init__(self, fuse_cfg=None, **kwargs):
        super().__init__(depths=[2, 2, 27, 2], dims=96, pretrained="pretrained/vmamba/vssmsmall_dp03_ckpt_epoch_238.pth",
                         mlp_ratio=0.0, downsample_version="v1", drop_path_rate=0.3)


class vssm_base(RGBXTransformer):
    def __init__(self, fuse_cfg=None, **kwargs):
        super().__init__(depths=[2, 2, 27, 2], dims=128, pretrained="pretrained/vmamba/vssmbase_dp06_ckpt_epoch_241.pth",
                         mlp_ratio=0.0, downsample_version="v1", drop_path_rate=0.6)


# --------------------------------------------------------------------------------------------
# MambaDecoder.py
# --------------------------------------------------------------------------------------------
def _bilinear_nhwc(x, size=None, scale_factor=None):
    """F.interpolate(bilinear, align_corners=False) on a channels-last tensor, staying channels-last."""
    t = x.permute(0, 3, 1, 2)  # NCHW view with channels_last strides: no copy
    t = ops.upsample_bilinear(t, size=size, scale_factor=scale_factor)
    return t.permute(0, 2, 3, 1).contiguous()


class PatchExpand(nn.Module):
    """MambaDecoder.py:12-30 — Linear(C->2C), pixel-shuffle 2x2, LayerNorm(C/2)."""

    def __init__(self, input_resolution, dim, dim_scale=2, norm_layer=nn.LayerNorm):
        super().__init__()
        self.input_resolution, self.dim = input_resolution, dim
        self.expand = nn.Linear(dim, 2 * dim, bias=False) if dim_scale == 2 else nn.Identity()
        self.norm = norm_layer(dim // dim_scale)

    def forward(self, x):
        if _fused_ok(x) and isinstance(self.norm, nn.LayerNorm) and isinstance(self.expand, nn.Linear):
            from . import fused
            return fused.patch_expand(self, x)
        x = self.expand(x)
        B, H, W, C = x.shape
        x = x.view(B, H, W, 2, 2, C // 4).permute(0, 1, 3, 2, 4, 5).reshape(B, 2 * H, 2 * W, C // 4)
        return ops.layer_norm(self.norm, x)


class UpsampleExpand(nn.Module):
    """MambaDecoder.py:33-51 — Linear(C->C/2), bilinear x2, LayerNorm."""

    def __init__(self, input_resolution, dim, patch_size=4, norm_layer=nn.LayerNorm):
        super().__init__()
        self.input_resolution, self.dim, self.patch_size = input_resolution, dim, patch_size
        self.linear = nn.Linear(dim, dim // 2, bias=False)
        self.output_dim = dim
        self.norm = norm_layer(dim // 2)

    def forward(self, x):
        if _fused_ok(x) and isinstance(self.norm, nn.LayerNorm):
            from . import fused
            return fused.upsample_expand(self, x)
        return ops.layer_norm(self.norm, _bilinear_nhwc(self.linear(x), scale_factor=2))


class FinalUpsample_X4(nn.Module):
    """MambaDecoder.py:76-97 — Linear, x2, Linear, x2, LayerNorm."""

    def __init__(self, input_resolution, dim, patch_size=4, norm_layer=nn.LayerNorm):
        super().__init__()
        self.input_resolution, self.dim, self.patch_size = input_resolution, dim, patch_size
        self.linear1 = nn.Linear(dim, dim, bias=False)
        self.linear2 = nn.Linear(dim, dim, bias=False)
        self.output_dim = dim
        self.norm = norm_layer(dim)

    def forward(self, x):
        x = _bilinear_nhwc(self.linear1(x), scale_factor=2)
        x = _bilinear_nhwc(self.linear2(x), scale_factor=2)
        return ops.layer_norm(self.norm, x)


class Mamba_up(nn.Module):
    """MambaDecoder.py:101-148 — depth x CVSSDecoderBlock (d_state=4) + optional UpsampleExpand."""

    def __init__(self, dim, input_resolution, depth, dt_rank="auto", d_state=4, ssm_ratio=2.0, attn_drop_rate=0.0,
                 drop_rate=0.0, mlp_ratio=4.0, drop_path=0.1, norm_layer=nn.LayerNorm, upsample=None, shared_ssm=False,
                 softmax_version=False, use_checkpoint=False, **kwargs):
        super().__init__()
        self.input_resolution, self.depth, self.use_checkpoint = input_resolution, depth, use_checkpoint
        self.blocks = nn.ModuleList([
            CVSSDecoderBlock(hidden_dim=dim, drop_path=drop_path[i], norm_layer=norm_layer, attn_drop_rate=attn_drop_rate,
                             d_state=d_state, dt_rank=dt_rank, ssm_ratio=ssm_ratio, shared_ssm=shared_ssm,
                             softmax_version=softmax_version, use_checkpoint=use_checkpoint, mlp_ratio=mlp_ratio,
                             act_layer=nn.GELU, drop=drop_rate) for i in range(depth)])
        self.upsample = UpsampleExpand(input_resolution, dim=dim, patch_size=2, norm_layer=norm_layer) if upsample is not None else None

    def forward(self, x):
        for blk in self.blocks:
            x = blk(x)
        return self.upsample(x) if self.upsample is not None else x


class MambaDecoder(nn.Module):
    """MambaDecoder.py:151-280 (deep_supervision=False is what builder.py:102 uses)."""

    def __init__(self, img_size=[480, 640], in_channels=[96, 192, 384, 768], num_classes=40, dropout_ratio=0.1,
                 embed_dim=96, align_corners=False, patch_size=4, depths=[4, 4, 4, 4], mlp_ratio=4.0, drop_rate=0.0,
                 attn_drop_rate=0.0, drop_path_rate=0.1, norm_layer=nn.LayerNorm, use_checkpoint=False,
                 deep_supervision=False, **kwargs):
        super().__init__()
        self.num_classes, self.num_layers, self.mlp_ratio, self.patch_size = num_classes, len(depths), mlp_ratio, patch_size
        self.patches_resolution = [img_size[0] // patch_size, img_size[1] // patch_size]
        self.deep_supervision = deep_supervision
        nl = self.num_layers
        dpr = [v.item() for v in torch.linspace(0, drop_path_rate, sum(depths))]
        self.layers_up = nn.ModuleList()
        for i in range(nl):
            res = (self.patches_resolution[0] // (2 ** (nl - 1 - i)), self.patches_resolution[1] // (2 ** (nl - 1 - i)))
            dim = int(embed_dim * 2 ** (nl - 1 - i))
            if i == 0:
                self.layers_up.append(PatchExpand(input_resolution=res, dim=dim, dim_scale=2, norm_layer=norm_layer))
            else:
                j = nl - 1 - i
                self.layers_up.append(Mamba_up(dim=dim, input_resolution=res, depth=depths[j], mlp_ratio=mlp_ratio,
                                               drop=drop_rate, attn_drop=attn_drop_rate,
                                               drop_path=dpr[sum(depths[:j]):sum(depths[:j + 1])], norm_layer=norm_layer,
                                               upsample=PatchExpand if i < nl - 1 else None, use_checkpoint=use_checkpoint))
        self.norm_up = norm_layer(embed_dim)
        if deep_supervision:
            self.norm_ds = nn.ModuleList([norm_layer(embed_dim * 2 ** (nl - 2 - i)) for i in range(nl - 1)])
            self.output_ds = nn.ModuleList([nn.Conv2d(embed_dim * 2 ** (nl - 2 - i), num_classes, kernel_size=1, bias=False)
                                            for i in range(nl - 1)])
        self.up = FinalUpsample_X4(input_resolution=(img_size[0] // patch_size, img_size[1] // patch_size), patch_size=4, dim=embed_dim)
        self.output = nn.Conv2d(embed_dim, num_classes, kernel_size=1, bias=False)

    def forward_up_features(self, inputs):
        ups = []
        y = None
        for inx, layer_up in enumerate(self.layers_up):
            skip = inputs[3 - inx].permute(0, 2, 3, 1)
            if inx == 0:
                y = layer_up(skip.contiguous())
            else:
                if not self.deep_supervision and y.shape[1:3] != skip.shape[1:3]:
                    y = _bilinear_nhwc(y, size=tuple(skip.shape[1:3]))     # odd sizes only (MambaDecoder.py:231-232)
                y = layer_up(y + skip)
            if self.deep_supervision and inx != self.num_layers - 1:
                ups.append(self.norm_ds[inx](y))
        if _fused_ok(y) and isinstance(self.norm_up, nn.LayerNorm):
            from . import fused
            x = fused.ln_nhwc(self.norm_up, y)
        else:
            x = ops.layer_norm(self.norm_up, y)
        return (x, ups) if self.deep_supervision else x

    def up_x4(self, x, pz):
        if _fused_ok(x) and isinstance(self.up.norm, nn.LayerNorm):
            from . import fused
            return fused.final_head(self, x)
        x = self.up(x)                                       # (B, 4H, 4W, C)
        return self.output(x.permute(0, 3, 1, 2))            # channels_last view; 1x1 conv = per-pixel linear

    def forward(self, inputs):
        if not self.deep_supervision:
            out = self.up_x4(self.forward_up_features(inputs), self.patch_size)
            return out.contiguous()
        x, ups = self.forward_up_features(inputs)
        outs = [self.up_x4(x, self.patch_size).contiguous()]
        for i, s in enumerate((16, 8, 4)):
            t = ops.upsample_bilinear(ups[i].permute(0, 3, 1, 2).contiguous(), scale_factor=s)
            outs.append(self.output_ds[i](t))
        return tuple(outs)


# --------------------------------------------------------------------------------------------
# builder.py
# --------------------------------------------------------------------------------------------
class EncoderDecoder(nn.Module):
    """builder.py:13-166, restricted to the Sigma path: cfg.backbone in {sigma_tiny, sigma_small, sigma_base},
    cfg.decoder == 'MambaDecoder'.  forward(rgb, modal_x, label=None) -> logits, or the loss when label is given."""

    _BACKBONES = {"sigma_tiny": (vssm_tiny, [96, 192, 384, 768]), "sigma_small": (vssm_small, [96, 192, 384, 768]),
                  "sigma_base": (vssm_base, [128, 256, 512, 1024])}

    def __init__(self, cfg=None, criterion=nn.CrossEntropyLoss(reduction="mean", ignore_index=255), norm_layer=nn.BatchNorm2d):
        super().__init__()
        self.norm_layer = norm_layer
        if cfg.backbone not in self._BACKBONES:
            raise NotImplementedError(f"sigma_b200 implements the Sigma (VMamba) backbones only, got cfg.backbone={cfg.backbone!r}; "
                                      "the CMX SegFormer/Swin baselines of the reference are out of scope")
        if cfg.decoder != "MambaDecoder":
            raise NotImplementedError(f"sigma_b200 implements cfg.decoder='MambaDecoder' only, got {cfg.decoder!r}")
        ctor, self.channels = self._BACKBONES[cfg.backbone]
        self.backbone = ctor()
        self.aux_head = None
        self.deep_supervision = False
        self.decode_head = MambaDecoder(img_size=[cfg.image_height, cfg.image_width], in_channels=self.channels,
                                        num_classes=cfg.num_classes, embed_dim=self.channels[0],
                                        deep_supervision=self.deep_supervision)
        self.criterion = criterion
        if self.criterion:
            self.init_weights(cfg, pretrained=cfg.pretrained_model)

    def init_weights(self, cfg, pretrained=None):
        """builder.py:112-126 + utils/init_func.py:10-19: kaiming-normal on the decoder's convs."""
        if pretrained and hasattr(self.backbone, "init_weights"):
            self.backbone.init_weights(pretrained=pretrained)
        for m in self.decode_head.modules():
            if isinstance(m, (nn.Conv1d, nn.Conv2d, nn.Conv3d)):
                nn.init.kaiming_normal_(m.weight, mode="fan_in", nonlinearity="relu")
            elif isinstance(m, self.norm_layer):
                m.eps, m.momentum = cfg.bn_eps, cfg.bn_momentum
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)

    def encode_decode(self, rgb, modal_x):
        out = self.decode_head(self.backbone(rgb, modal_x))
        if out.shape[2:] != rgb.shape[2:]:
            out = ops.upsample_bilinear(out, size=rgb.shape[2:])
        return out

    def forward(self, rgb, modal_x, label=None):
        if not rgb.is_cuda:
            raise RuntimeError("sigma_b200.EncoderDecoder runs on CUDA only (no CPU path)")
        out = self.encode_decode(rgb, modal_x)
        if label is not None:
            ignore = ops.plain_cross_entropy(self.criterion) if ops.deterministic() else None
            if ignore is not None:   # nll_loss's CUDA backward raises under torch.use_deterministic_algorithms(True)
                return ops.deterministic_cross_entropy(out, label.long(), ignore)
            return self.criterion(out, label.long())
        return out
