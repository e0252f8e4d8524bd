"""CPU emulation of the JK BatchNorm entry points (include/sgformer_b200.h: sgf_bn_fwd_jk, sgf_bn_bwd_reduce_jk /
sgf_bn_bwd_apply_jk) on top of tests/kernel_emu.py: `module()` is kernel_emu plus `bn_fwd_jk` / `bn_bwd_jk`, for running the
GCNJK schedule (engine.gcnjk_forward / _backward) without a GPU."""
import types

import torch

import kernel_emu
from dropout_mask import apply_kernel_dropout


def bn_fwd_jk(z, mean, rstd, gamma, beta, zbias, use_bn, use_relu, p, seed, want_y, mode, jk, jk_idx, layer):
    _, t = kernel_emu._bn_pre(z, mean, rstd, gamma, beta, zbias, use_bn)
    if use_relu:
        t = t.clamp_min(0)
    a = t.to(jk.dtype).float()                      # compared as stored
    h = z.shape[1]
    if mode == "max":
        if layer == 0:
            jk.copy_(a.to(jk.dtype))
            jk_idx[:, :h] = 0
        else:
            m = jk.float()
            upd = a > m                             # strict: a tie keeps the lower layer
            jk.copy_(torch.where(upd, a, m).to(jk.dtype))
            jk_idx[:, :h][upd] = layer
    else:
        jk.copy_(a.to(jk.dtype))
    t = apply_kernel_dropout(t, seed, p)
    return kernel_emu._st(kernel_emu.new_like(z), t) if want_y else None


def jk_addend(mode, jk_g, jk_idx, layer, h):
    add = jk_g.float()
    if mode == "max":
        add = add * (jk_idx[:, :h] == layer)
    return add


def bn_bwd_jk(dy, z, mean, rstd, gamma, beta, zbias, use_bn, use_relu, training, p, seed, mode, jk_g, jk_idx, layer,
              want_dz_colsum=False, out_row_scale=None):
    n, h = z.shape
    g = apply_kernel_dropout(dy.float(), seed, p) if dy is not None else torch.zeros(z.shape)
    g = g + jk_addend(mode, jk_g, jk_idx, layer, h)     # outside the dropout mask
    xh, pre = kernel_emu._bn_pre(z, mean, rstd, gamma, beta, zbias, use_bn)
    if use_relu:
        g = g * (pre > 0)
    sums = torch.cat([g.sum(0), (g * xh).sum(0)]) if use_bn else None
    if use_bn and training:
        d = gamma * rstd * (g - sums[:h] / n - xh * sums[h:] / n)
    elif use_bn:
        d = gamma * rstd * g
    else:
        d = g
    colsum = d.sum(0) if want_dz_colsum else None
    if out_row_scale is not None:
        d = d * out_row_scale[:, None]
    return kernel_emu._st(kernel_emu.new_like(z), d), sums, colsum


def module():
    m = types.ModuleType("kernel_emu_gcnjk")
    m.__dict__.update(kernel_emu.__dict__)
    m.bn_fwd_jk, m.bn_bwd_jk = bn_fwd_jk, bn_bwd_jk
    return m
