"""CPU contract of the fused attention kernels of csrc/attn_softmax.cu (include/sgformer_b200.h: sgf_attn_softmax_*) on top of
tests/kernel_emu.py, in both modes: the Frobenius-normalised scores of SGFormerSOFT (attn_softmax_*) and the scaled scores of
SGFormerGAT (attn_scaled_*).  `module()` is kernel_emu plus these entry points, for running the TransConv schedule with
trans_attention="softmax" / "gat" (engine.trans_forward / trans_backward) without a GPU.  The softmax runs over the heads of each
(node, key) pair; the backward is the exact derivative of the forward (autograd in the working precision).  Which shapes the
kernels take is not emulated: the engine asks the library's host-only query (kernels.attn_softmax_tile_rows) directly."""
import types

import torch

import kernel_emu
from kernel_emu import _f, _st, alloc_act


def _attend(q, k, v, heads, shared_v, scale):
    """o [N, H*D] and P [N, L, H]: scale q.k per head (scale None: q, k normalised by their Frobenius norms), softmax over heads."""
    n = q.shape[0]
    m = q.shape[1] // heads
    qh, kh = q.reshape(n, heads, m), k.reshape(n, heads, m)
    if scale is None:
        s = torch.einsum("nhm,lhm->nlh", qh / q.norm(), kh / k.norm())
    else:
        s = scale * torch.einsum("nhm,lhm->nlh", qh, kh)
    p = torch.softmax(s, dim=-1)
    vh = v.reshape(n, 1, -1).expand(-1, heads, -1) if shared_v else v.reshape(n, heads, -1)
    return torch.einsum("nlh,lhd->nhd", p, vh).reshape(n, -1), p


def _fwd(q, k, v, heads, shared_v, scale):
    o, _ = _attend(_f(q), _f(k), _f(v), heads, shared_v, scale)
    return _st(alloc_act(q.shape[0], o.shape[1], q.dtype, q.device), o)


def _bwd(q, k, v, heads, shared_v, scale, g, gscale, dq, dk, dv, dv_accumulate):
    qf, kf, vf = (_f(t).detach().clone().requires_grad_() for t in (q, k, v))
    with torch.enable_grad():
        o, _ = _attend(qf, kf, vf, heads, shared_v, scale)
        d = o.shape[1] // heads
        gf = _f(g)
        if gf.shape[1] == d and heads > 1:      # one gradient block shared by every head (the head mean's backward)
            gf = gf.repeat(1, heads)
        gq, gk, gv = torch.autograd.grad(o, (qf, kf, vf), gscale * gf)
    _st(dq, gq)
    _st(dk, gk)
    _st(dv, gv + (_f(dv) if dv_accumulate else 0.0))


def attn_softmax_fwd(q, k, v, heads, sq_q, sq_k, shared_v=False):
    return _fwd(q, k, v, heads, shared_v, None)


def attn_softmax_bwd(q, k, v, heads, sq_q, sq_k, shared_v, g, gscale, dq, dk, dv, dv_accumulate=False):
    _bwd(q, k, v, heads, shared_v, None, g, gscale, dq, dk, dv, dv_accumulate)


def attn_softmax_probs(q, k, heads, sq_q, sq_k):
    _, p = _attend(_f(q), _f(k), _f(k), heads, False, None)
    return p.mean(-1).float()


def attn_scaled_fwd(q, k, v, heads, scale):
    return _fwd(q, k, v, heads, False, float(scale))


def attn_scaled_bwd(q, k, v, heads, scale, g, gscale, dq, dk, dv, dv_accumulate=False):
    _bwd(q, k, v, heads, False, float(scale), g, gscale, dq, dk, dv, dv_accumulate)


def module():
    m = types.ModuleType("kernel_emu_attn_softmax")
    m.__dict__.update(kernel_emu.__dict__)
    for name in ("attn_softmax_fwd", "attn_softmax_bwd", "attn_softmax_probs",
                 "attn_scaled_fwd", "attn_scaled_bwd"):
        setattr(m, name, globals()[name])
    return m
