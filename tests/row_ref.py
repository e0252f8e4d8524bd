"""fp64 references of the row kernels (csrc/rowops.cu) and the comparison they are held to.

Each reference is autograd in fp64 of the formula a kernel implements, with the dropout mask passed in as a tensor
(mask * kernel scale, see tests/dropout_mask.py), so a test can replay the kernel's own mask.  Shared by
tests/test_gpu_dropout.py (every kernel pair at a few hundred rows) and tests/test_gpu_row_sweep.py (the same pairs at row counts
where every lane group of the capped grid processes several rows)."""
import math

import torch
import torch.nn.functional as F


def close(got, ref, tol, what, colsum_rows=0, elem=0.0):
    """max-abs error relative to the reference's max; column sums get a sqrt(rows) allowance and, where they cancel, are
    measured against their largest summand `elem`."""
    got, ref = got.detach().double().reshape(ref.shape), ref.detach().double()
    err = (got - ref).abs().max().item() if ref.numel() else 0.0
    scale = max(ref.abs().max().item(), float(elem), 1e-6)
    allow = tol * scale * (math.sqrt(colsum_rows) if colsum_rows else 1.0)
    assert err == err and err <= allow, f"{what}: max err {err:.3e} (ref max {scale:.3e}, allowed {allow:.3e})"


def ln_reference(x, r, gy, a, b, c, gamma, beta, use_ln, use_relu, M, dy, gscale):
    """fp64 autograd of y = dropout(relu?(LN?(a*x + b*r + c*gy))) -> y and the gradients of sum(gscale * dy * y)."""
    h = x.shape[1]
    xd = x.double().requires_grad_(True)
    rd = r.double().requires_grad_(True) if r is not None else None
    gd, bd = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    u = a * xd + (b * rd if rd is not None else 0.0) + (c * gy.double() if gy is not None else 0.0)
    u.retain_grad()
    t = F.layer_norm(u, (h,), gd, bd, 1e-5) if use_ln else u
    if use_relu:
        t = t.clamp_min(0)
    y = t * M
    (y * dy.double() * gscale).sum().backward()
    return dict(y=y.detach(), du=u.grad, dx=xd.grad, dr=rd.grad if rd is not None else None, dgamma=gd.grad, dbeta=bd.grad)


def untie(dy, x, r, a, b, gamma, beta, use_ln):
    """Zero the incoming gradient where the fp64 ReLU pre-activation LN?(a*x + b*r) is within 1e-3 of its largest magnitude of
    zero: there fp32 and fp64 may open the gate differently, and with no gradient through it the choice does not matter.  Every
    other output is then compared at the ordinary tolerance."""
    u = a * x.double() + (b * r.double() if r is not None else 0.0)
    pre = F.layer_norm(u, (u.shape[1],), gamma.double(), beta.double(), 1e-5) if use_ln else u
    return dy.masked_fill(pre.abs() <= 1e-3 * pre.abs().max(), 0)


def attn_reference(R, o, xa, a, den):
    """The Gram-attention row prologue of ln_bwd_attn on ga = a * du (R = ln_reference's result)."""
    ga = a * R["du"]
    gnum = ga / den.double()[:, None]
    gden = -(ga * o.double()).sum(1) / den.double()
    pgt = xa.double() * gden[:, None]
    return dict(gnum=gnum, gden=gden, cs=gnum.sum(0), pg=pgt.sum(0), sg=gden.sum().reshape(1),
                elem=dict(cs=gnum.abs().max().item(), pg=pgt.abs().max().item(), sg=gden.abs().max().item()))


BN_CASES = [   # (use_bn, training, relu, res, mix, dy2, dres_acc, out_row_scale)
    (True, True, True, True, False, True, True, False),       # GraphConv middle layer: residual, pre-scaled gradient
    (True, True, True, False, True, False, False, False),     # last layer: branch mix with gw
    (True, False, False, True, False, True, False, True),     # BatchNorm in eval mode
    (False, True, True, False, False, False, False, True),    # no BatchNorm (GCN backbone)
    (True, True, False, False, False, False, False, True),    # training BatchNorm, no ReLU, GCN-style row scale
]


def bn_untie(case, z, gamma, beta, rm, rv, dy, dy2):
    """As untie, for the BatchNorm chain: no gradient through a ReLU gate that fp32 and fp64 may decide differently."""
    use_bn, training, relu = case[:3]
    if not relu:
        return dy, dy2
    zz = z.double()
    if use_bn:
        mu, var = (zz.mean(0), zz.var(0, unbiased=False)) if training else (rm.double(), rv.double())
        pre = (zz - mu) / torch.sqrt(var + 1e-5) * gamma.double() + beta.double()
    else:
        pre = zz
    amb = pre.abs() <= 1e-3 * pre.abs().max()
    return dy.masked_fill(amb, 0), dy2.masked_fill(amb, 0)


def bn_reference(case, z, res, mix, dy, dy2, dres0, gamma, beta, rm, rv, rs, rs2, ors, gw, gscale, M):
    """fp64 of bn_fwd + bn_bwd for one BN_CASES flag set (unused operands are ignored as the flags say) -> dict of y, ys, dres,
    dz, colsum (of dz before out_row_scale), dbeta, dgamma."""
    use_bn, training, relu, with_res, with_mix, with_dy2, dres_acc, with_ors = case
    zd = z.double().requires_grad_(True)
    gd, bd = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    if use_bn:
        if training:
            mu, var = zd.mean(0), zd.var(0, unbiased=False)
        else:
            mu, var = rm.double(), rv.double()
        xh = (zd - mu) / torch.sqrt(var + 1e-5)
        t = xh * gd + bd
    else:
        t = zd
    if relu:
        t = t.clamp_min(0)
    t = t * M
    if with_res:
        t = t + res.double()
    G = gscale * (dy.double() + (rs2.double()[:, None] * dy2.double() if with_dy2 else 0.0))
    (t * G).sum().backward()
    return dict(y=(gw * t + (1 - gw) * mix.double()) if with_mix else t, ys=t * rs.double()[:, None],
                dres=G + (dres0.double() if dres_acc else 0.0), dz=zd.grad * (ors.double()[:, None] if with_ors else 1.0),
                colsum=zd.grad.sum(0), dbeta=bd.grad, dgamma=gd.grad)


def check_bn_chain(got, ref, case, tol, tag, rows, h):
    """got: the kernels' y, ys, dres, dz, colsum and sums ([dbeta, dgamma])."""
    use_bn, training = case[:2]
    close(got["y"], ref["y"], tol, f"y {tag}")
    close(got["ys"], ref["ys"], tol, f"ys {tag}")
    close(got["dres"], ref["dres"], tol, f"dres {tag}")
    # a training BatchNorm backward subtracts column means: its error is relative to the whole gradient's scale
    dz_tol = tol if not (use_bn and training) else 4 * tol
    close(got["dz"], ref["dz"], dz_tol, f"dz {tag}")
    cs_tol = 1e-5
    if not (use_bn and training):     # training: the column sums of dz are ~0 (the BatchNorm backward centres dz)
        close(got["colsum"], ref["colsum"], cs_tol, f"dz colsum {tag}", rows)
    if use_bn:
        close(got["sums"][:h], ref["dbeta"], cs_tol, f"dbeta {tag}", rows)
        close(got["sums"][h:], ref["dgamma"], cs_tol, f"dgamma {tag}", rows)
