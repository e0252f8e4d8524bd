"""torch-CPU emulation of the GAT kernel contracts — TEST INFRASTRUCTURE ONLY.

Extends tests/kernel_emu_difformer.py (re-exported unchanged) with the entry points the GAT schedule uses: sgf_gat_logits,
sgf_gat_fwd, sgf_gat_bwd, sgf_dense_dropout, and the BatchNorm kernels' ELU activation code (2).  The edge softmax is restated
per edge from the CSR (rows = targets) with the formulas of include/sgformer_b200.h; attention dropout is emulated for p = 0
only.  Tests monkeypatch `engine.K` / `functional.K` with this module; it proves nothing about the CUDA kernels themselves."""
import torch

import kernel_emu as _base
from dropout_mask import apply_kernel_dropout
from kernel_emu import _st, new_like
from kernel_emu_difformer import *  # noqa: F401,F403

ACT_ELU = 2
GAT_MAX_HEADS = 8


def _edges(rowptr, col):
    n = rowptr.numel() - 1
    dst = torch.repeat_interleave(torch.arange(n), rowptr[1:] - rowptr[:-1])
    return col.long(), dst


def gat_logits(xp, heads, c, att_src, att_dst):
    x = xp.float().reshape(xp.shape[0], heads, c)
    return (x * att_src.view(heads, c)).sum(-1), (x * att_dst.view(heads, c)).sum(-1)


def _alpha(rowptr, col, a_src, a_dst, n):
    src, dst = _edges(rowptr, col)
    pre = a_src[src] + a_dst[dst]
    e = torch.nn.functional.leaky_relu(pre, 0.2)
    m = torch.full_like(a_dst, -float("inf")).scatter_reduce(0, dst[:, None].expand_as(e), e, "amax")
    lse = m + torch.zeros_like(a_dst).index_add(0, dst, (e - m[dst]).exp()).log()
    return src, dst, pre, (e - lse[dst]).exp(), lse


def gat_fwd(rowptr, col, xp, a_src, a_dst, heads, c, mean, bias, p, seed):
    if p > 0:
        raise NotImplementedError("kernel_emu_gat: attention dropout is not emulated")
    n = xp.shape[0]
    x = xp.float().reshape(n, heads, c)
    src, dst, _, alpha, lse = _alpha(rowptr, col, a_src, a_dst, n)
    y = torch.zeros_like(x).index_add(0, dst, alpha[..., None] * x[src])
    out = y.mean(1) if mean else y.reshape(n, heads * c)
    if bias is not None:
        out = out + bias
    return _st(_base.alloc_act(n, out.shape[1], xp.dtype, xp.device), out), lse


def gat_bwd(rowptr, col, rowptr_t, col_t, xp, a_src, a_dst, lse, g, att_src, att_dst, heads, c, mean, p, seed):
    if p > 0:
        raise NotImplementedError("kernel_emu_gat: attention dropout is not emulated")
    n = xp.shape[0]
    x = xp.float().reshape(n, heads, c)
    src, dst, pre, alpha, _ = _alpha(rowptr, col, a_src, a_dst, n)
    gh = (g.float() / heads).unsqueeze(1).expand(n, heads, c) if mean else g.float().reshape(n, heads, c)
    lg = torch.where(pre > 0, 1.0, 0.2)
    dalpha = (gh[dst] * x[src]).sum(-1)
    r = torch.zeros_like(a_dst).index_add(0, dst, alpha * dalpha)
    da_dst = torch.zeros_like(a_dst).index_add(0, dst, alpha * dalpha * lg) - r * torch.zeros_like(a_dst).index_add(0, dst, alpha * lg)
    da_src = torch.zeros_like(a_src).index_add(0, src, alpha * (dalpha - r[dst]) * lg)
    dxp = torch.zeros_like(x).index_add(0, src, alpha[..., None] * gh[dst])
    dxp = dxp + da_src[..., None] * att_src.view(heads, c) + da_dst[..., None] * att_dst.view(heads, c)
    return _st(new_like(xp), dxp.reshape(n, heads * c)), da_src.t().contiguous(), da_dst.t().contiguous()


def dense_dropout(x, p, seed):
    if p > 0:
        raise NotImplementedError("kernel_emu_gat: input dropout is not emulated")
    return x.clone()


def _act(t, code):
    if code == ACT_ELU:
        return torch.where(t > 0, t, torch.expm1(t))
    return t.clamp_min(0) if code else t


def _act_grad(g, pre, code):
    if code == ACT_ELU:
        return g * torch.where(pre > 0, torch.ones_like(pre), pre.exp())
    return g * (pre > 0) if code else g


def bn_fwd(z, res, mix, mean, rstd, gamma, beta, zbias, use_bn, use_relu, p, seed, gw, row_scale, want_y, want_scaled, ys_out=None):
    """sgf_bn_fwd with the activation code (0 none, 1 ReLU, 2 ELU)."""
    _, t = _base._bn_pre(z, mean, rstd, gamma, beta, zbias, use_bn)
    t = apply_kernel_dropout(_act(t, int(use_relu)), seed, p)
    if res is not None:
        t = t + res.float()
    ys = _st(new_like(z), t * row_scale[:, None]) if want_scaled else None
    if mix is not None:
        t = gw * t + (1 - gw) * mix.float()
    return (_st(new_like(z), t) if want_y else None), ys


def bn_bwd_sums(dy, dy2, row_scale2, z, mean, rstd, gamma, beta, zbias, use_bn, use_relu, p, seed, gscale):
    g = apply_kernel_dropout(_base._bn_g(dy, dy2, row_scale2, gscale), seed, p)
    xh, pre = _base._bn_pre(z, mean, rstd, gamma, beta, zbias, use_bn)
    g = _act_grad(g, pre, int(use_relu))
    return torch.cat([g.sum(0), (g * xh).sum(0)])


def bn_bwd(dy, dy2, row_scale2, z, mean, rstd, gamma, beta, zbias, use_bn, use_relu, training, p, seed, gscale, dres=None,
           dres_accumulate=False, want_dz_colsum=False, out_row_scale=None, reduce_fn=None, stat_rows=0):
    """sgf_bn_bwd_reduce + _apply with the activation code (0 none, 1 ReLU, 2 ELU)."""
    graw = _base._bn_g(dy, dy2, row_scale2, gscale)
    if dres is not None:
        _st(dres, graw + (dres.float() if dres_accumulate else 0.0))
    xh, pre = _base._bn_pre(z, mean, rstd, gamma, beta, zbias, use_bn)
    g = _act_grad(apply_kernel_dropout(graw, seed, p), pre, int(use_relu))
    sums = None
    if use_bn and training:
        sums = torch.cat([g.sum(0), (g * xh).sum(0)])
        if reduce_fn is not None:
            reduce_fn(sums)
        n = stat_rows if stat_rows > 0 else z.shape[0]
        d = gamma * rstd * (g - sums[:z.shape[1]] / n - xh * sums[z.shape[1]:] / n)
    elif use_bn:
        d = gamma * rstd * g
    else:
        d = g
    colsum = d.sum(0) if want_dz_colsum else None
    if out_row_scale is not None:
        d = d * out_row_scale[:, None]
    return _st(new_like(z), d), sums, colsum
