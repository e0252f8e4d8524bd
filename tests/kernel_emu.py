"""torch-CPU emulation of sgformer_b200.kernels — TEST INFRASTRUCTURE ONLY.

Lets the hand-written forward/backward *schedules* of sgformer_b200/engine.py (which kernels run in which order, with
which scalings and accumulations) be checked against the oracle in the GPU-less build container: tests monkeypatch
`engine.K` / `functional.K` with this module.  It mirrors the documented semantics of every C-ABI entry point
(include/sgformer_b200.h) with plain tensor ops; it is never imported by the package and proves nothing about the CUDA
kernels themselves (those are checked by the `-m gpu` tests against the oracle)."""
from dataclasses import dataclass
from typing import Optional

import torch

from dropout_mask import apply_kernel_dropout

EPI_AFFINE, EPI_ATTN_APPLY, EPI_ATTN_GRAM = 0, 1, 2


def _use(t):
    pass


def ceil_to(x, m):
    return (x + m - 1) // m * m


def alloc_act(rows, h, dtype, device):
    return torch.zeros((rows, h), dtype=dtype, device=device)


def new_like(x):
    return torch.zeros(x.shape, dtype=x.dtype, device=x.device)


def _st(out, val):
    out.copy_(val.to(out.dtype))
    return out


@dataclass
class Operand:
    data: torch.Tensor  # logical fp32 [rows, k]
    rows: int
    k: int
    kp: int
    planes: int


def csr_build(edge_index, n, by_source=False, self_loop_mode=0, want_dinv=True, rows=None, col_rot=None):
    src, dst = edge_index[0], edge_index[1]
    if self_loop_mode == 1:
        keep = src != dst
        ar = torch.arange(n)
        src, dst = torch.cat([src[keep], ar]), torch.cat([dst[keep], ar])
    key, val = (src, dst) if by_source else (dst, src)
    if rows is not None:
        m = (key >= rows[0]) & (key < rows[1])
        key, val = key[m] - rows[0], val[m]
        nr = rows[1] - rows[0]
    else:
        nr = n
    if col_rot is not None:      # sgf_csr_build_rot: column ids stored as (col - rot) mod `mod`, rows sorted by them
        val = (val - col_rot[0]) % col_rot[1]
        n = max(n, col_rot[1])
    order = torch.argsort(key * n + val, stable=True)
    deg = torch.bincount(key, minlength=nr)
    n = nr
    rowptr = torch.zeros(n + 1, dtype=torch.int64)
    rowptr[1:] = torch.cumsum(deg, 0)
    d = deg.float()
    dinv = torch.where(d > 0, (1.0 / d).sqrt(), torch.zeros_like(d)) if (want_dinv and not by_source) else None
    return rowptr, val[order].to(torch.int32), dinv


def spmm(rowptr, col, row_scale, x, out=None, heavy=None):
    n = rowptr.numel() - 1
    rows = torch.repeat_interleave(torch.arange(n), rowptr[1:] - rowptr[:-1])
    y = torch.zeros((n, x.shape[1]), dtype=torch.float32).index_add_(0, rows, x.float()[col.long()])
    if row_scale is not None:
        y = y * row_scale[:, None]
    return _st(out if out is not None else alloc_act(n, x.shape[1], x.dtype, x.device), y)


def csr_row_splits(rowptr, col, thresholds):
    n = rowptr.numel() - 1
    rows = torch.repeat_interleave(torch.arange(n), rowptr[1:] - rowptr[:-1])
    out = torch.zeros((len(thresholds), n), dtype=torch.int32)
    for t, thr in enumerate(thresholds):
        out[t] = torch.zeros(n, dtype=torch.int64).index_add_(0, rows, (col.long() < thr).long()).to(torch.int32)
    return out


def spmm_range(rowptr, col, row_scale, x, lo, hi, part_in, part_out):
    n = rowptr.numel() - 1
    lens = rowptr[1:] - rowptr[:-1]
    rows = torch.repeat_interleave(torch.arange(n), lens)
    pos = torch.arange(col.numel()) - rowptr[:-1][rows]
    keep = torch.ones(col.numel(), dtype=torch.bool)
    if lo is not None:
        keep &= pos >= lo.long()[rows]
    if hi is not None:
        keep &= pos < hi.long()[rows]
    acc = torch.zeros((n, x.shape[1]), dtype=torch.float32).index_add_(0, rows[keep], x.float()[col.long()[keep]])
    if part_in is not None:
        acc = acc + part_in
    if part_out is not None:
        part_out.copy_(acc)
        return None
    if row_scale is not None:
        acc = acc * row_scale[:, None]
    return _st(alloc_act(n, x.shape[1], x.dtype, x.device), acc)


def operand_from_bf16(x):
    return Operand(x.float(), x.shape[0], x.shape[1], x.shape[1], 1)


def pack_operand(src, transpose=False, planes=1, colsum=None):
    if colsum is not None:
        colsum += src.sum(0)
    d = (src.t() if transpose else src).contiguous().float()
    if planes == 1:
        d = d.bfloat16().float()
    return Operand(d, d.shape[0], d.shape[1], ceil_to(d.shape[1], 64), planes)


def operand_memo_begin():
    pass


def operand_memo_clear():
    pass


def as_operand(x, planes, memo=False):
    if x.dtype == torch.bfloat16:
        return operand_from_bf16(x)
    return pack_operand(x, False, planes)


def gemm_nt(A, B, pairs, n_out, out, *, epi=EPI_AFFINE, bias=None, aux=None, row_scale=None, alpha=1.0, beta=0.0,
            alpha_dev=None, beta_dev=None, relu=False, accumulate=False, tail=None, nf=0.0, den_out=None, r1_row=None,
            r1_col=None, col_sum=None, col_sumsq=None, nf_dev=None, schedule=None):
    acc = 0
    for (ai, ak, bi, bk, klen) in pairs:
        acc = acc + A[ai].data[:, ak:ak + klen] @ B[bi].data[:, bk:bk + klen].t()
    assert acc.shape[1] == n_out
    if epi == EPI_ATTN_APPLY:
        den = (A[0].data @ tail.data.t())[:, 0] + nf
        if den_out is not None:
            den_out.copy_(den)
        v = (acc + nf * aux.float()) / den[:, None]
    elif epi == EPI_ATTN_GRAM:
        den = (A[0].data @ tail.data.t())[:, 0] + float(nf_dev)
        if den_out is not None:
            den_out.copy_(den)
        v = (acc + bias[:n_out]) / den[:, None]
    else:
        a = alpha * (float(alpha_dev) if alpha_dev is not None else 1.0)
        b = beta * (float(beta_dev) if beta_dev is not None else 1.0)
        v = a * acc
        if aux is not None:
            v = v + b * aux.float()
        if bias is not None:
            v = v + bias[:n_out]
        if r1_row is not None:
            v = v + r1_row[:, None] * r1_col[None, :n_out]
        if relu:
            v = v.clamp_min(0)
        if row_scale is not None:
            v = v * row_scale[:, None]
    if accumulate:
        v = v + out.float()
    _st(out, v)
    if col_sum is not None:
        col_sum += out.float().sum(0)
    if col_sumsq is not None:
        col_sumsq += (out.float() ** 2).sum(0)
    return out


def gemm_tn(A, B, out, *, transpose_out=False, alpha=1.0, beta=0.0, alpha_dev=None):
    r = alpha * (float(alpha_dev) if alpha_dev is not None else 1.0) * (A.data.t() @ B.data)
    if transpose_out:
        r = r.t()
    if beta != 0.0:
        r = r + beta * out
    return _st(out, r)


def colstats(x, w=None, want_sum=True, want_sumsq=True):
    xf = x.float()
    s = (xf * (w[:, None] if w is not None else 1.0)).sum(0) if want_sum else None
    q = (xf * xf).sum(0) if want_sumsq else None
    return s, q


def _f(t):
    """fp32 working precision of the kernels (fp64 inputs stay fp64: the math tests run the same contracts in double)."""
    return t if t.dtype == torch.float64 else t.float()


def _ln_core(x, r, a, b, gamma, beta, use_ln, use_relu):
    u = a * _f(x) + (b * _f(r) if r is not None else 0.0)
    mean = rstd = None
    xh = u
    if use_ln:
        mean = u.mean(1)
        rstd = (u.var(1, unbiased=False) + 1e-5).rsqrt()
        xh = (u - mean[:, None]) * rstd[:, None]
        t = xh * gamma + beta
    else:
        t = u
    return u, xh, t, mean, rstd


def ln_fwd(x, r, a, b, gamma, beta, use_ln, use_relu, p, seed, want_stats=True):
    u, xh, t, mean, rstd = _ln_core(x, r, a, b, gamma, beta, use_ln, use_relu)
    if use_relu:
        t = t.clamp_min(0)
    t = apply_kernel_dropout(t, seed, p)
    stats = torch.stack([mean, rstd], 1) if use_ln else None
    return _st(new_like(x), t), stats


def ln_bwd(dy, x, r, a, b, gamma, beta, stats, use_ln, use_relu, p, seed, gscale, want_dr, dgamma, dbeta):
    u, xh, t, mean, rstd = _ln_core(x, r, a, b, gamma, beta, use_ln, use_relu)
    g = apply_kernel_dropout(gscale * dy.float(), seed, p)
    if use_relu:
        g = g * (t > 0)
    if use_ln:
        dgamma += (g * xh).sum(0)
        dbeta += g.sum(0)
        gg = g * gamma
        du = rstd[:, None] * (gg - gg.mean(1, keepdim=True) - xh * (gg * xh).mean(1, keepdim=True))
    else:
        du = g
    dx = _st(new_like(x), a * du)
    dr = _st(new_like(x), b * du) if want_dr else None
    return dx, dr


def ln_bwd_attn(dy, o, r, xa, a, b, gamma, beta, stats, use_ln, use_relu, p, seed, gscale, want_dr, dgamma, dbeta, den):
    """sgf_ln_bwd_attn: LayerNorm backward of u = a*o + b*r fused with the attention-backward row prologue:
    g = a*du;  gnum' = g/den~;  gden' = -(g.o)/den~;  dr = b*du;  column sums cs = sum gnum', pg = sum xa*gden', sg = sum gden'."""
    u, xh, t, mean, rstd = _ln_core(o, r, a, b, gamma, beta, use_ln, use_relu)
    g = apply_kernel_dropout(gscale * _f(dy), seed, p)
    if use_relu:
        g = g * (t > 0)
    if use_ln:
        dgamma += (g * xh).sum(0)
        dbeta += g.sum(0)
        gg = g * gamma
        du = rstd[:, None] * (gg - gg.mean(1, keepdim=True) - xh * (gg * xh).mean(1, keepdim=True))
    else:
        du = g
    ga = a * du
    gnum_f = ga / den[:, None]
    gden = -(ga * _f(o)).sum(1) / den
    gnum = _st(new_like(o), gnum_f)
    dr = _st(new_like(o), b * du) if want_dr else None
    return gnum, gden, dr, gnum_f.sum(0), (_f(xa) * gden[:, None]).sum(0), gden.sum().reshape(1)


def bn_finalize(sum_, sumsq, rows, h, zbias, running_mean, running_var, device, eps=1e-5, momentum=0.1):
    if sum_ is not None:
        m = sum_ / rows
        var = (sumsq / rows - m * m).clamp_min(0)
        if zbias is not None:
            m = m + zbias
        if running_mean is not None:
            running_mean.mul_(1 - momentum).add_(momentum * m)
            running_var.mul_(1 - momentum).add_(momentum * var * rows / max(rows - 1, 1))
        return m, (var + eps).rsqrt()
    return running_mean.clone(), (running_var + eps).rsqrt()


def _bn_pre(z, mean, rstd, gamma, beta, zbias, use_bn):
    zz = z.float() + (zbias if zbias is not None else 0.0)
    if use_bn:
        xh = (zz - mean) * rstd
        return xh, xh * gamma + beta
    return zz, zz


def bn_fwd(z, res, mix, mean, rstd, gamma, beta, zbias, use_bn, use_relu, p, seed, gw, row_scale, want_y, want_scaled, ys_out=None):
    _, t = _bn_pre(z, mean, rstd, gamma, beta, zbias, use_bn)
    if use_relu:
        t = t.clamp_min(0)
    t = apply_kernel_dropout(t, seed, p)            # before the residual
    if res is not None:
        t = t + res.float()
    ys = _st(new_like(z), t * row_scale[:, None]) if want_scaled else None
    if mix is not None:
        t = gw * t + (1 - gw) * mix.float()
    y = _st(new_like(z), t) if want_y else None
    return y, ys


def _bn_g(dy, dy2, row_scale2, gscale):
    g = 0
    if dy is not None:
        g = g + dy.float()
    if dy2 is not None:
        g = g + dy2.float() * (row_scale2[:, None] if row_scale2 is not None else 1.0)
    return gscale * g


def bn_bwd_sums(dy, dy2, row_scale2, z, mean, rstd, gamma, beta, zbias, use_bn, use_relu, p, seed, gscale):
    g = apply_kernel_dropout(_bn_g(dy, dy2, row_scale2, gscale), seed, p)
    xh, pre = _bn_pre(z, mean, rstd, gamma, beta, zbias, use_bn)
    if use_relu:
        g = g * (pre > 0)
    return torch.cat([g.sum(0), (g * xh).sum(0)])


def bn_bwd(dy, dy2, row_scale2, z, mean, rstd, gamma, beta, zbias, use_bn, use_relu, training, p, seed, gscale, dres=None,
           dres_accumulate=False, want_dz_colsum=False, out_row_scale=None, reduce_fn=None, stat_rows=0):
    graw = _bn_g(dy, dy2, row_scale2, gscale)
    if dres is not None:
        _st(dres, graw + (dres.float() if dres_accumulate else 0.0))
    xh, pre = _bn_pre(z, mean, rstd, gamma, beta, zbias, use_bn)
    g = apply_kernel_dropout(graw, seed, p)           # dres takes the gradient before the dropout mask
    g = g * (pre > 0) if use_relu else g
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


def axpby(x, y, a, b, out_dtype=None, row_scale=None, out=None):
    v = a * x.float() + (b * y.float() if y is not None else 0.0)
    if row_scale is not None:
        v = v * row_scale[:, None]
    if out is None:
        out = torch.zeros(x.shape, dtype=out_dtype or x.dtype)
    return _st(out, v)


def head_mean(x, heads, d):
    return _st(alloc_act(x.shape[0], d, x.dtype, x.device), x.float().reshape(x.shape[0], heads, d).mean(1))


# ------------------------------------------------------------------------------------------------
# Gram-form linear attention (sgf_gram, sgf_attn_gram_prepare_fwd/bwd, sgf_ln_bwd_attn): contracts of include/sgformer_b200.h
# ------------------------------------------------------------------------------------------------
SC_NQ2, SC_NK2, SC_ALPHA, SC_BETA, SC_DEN, SC_N, SC_IP, SC_C, SC_CQ, SC_CK, SC_SG = 0, 1, 2, 3, 4, 5, 8, 9, 10, 11, 12


def gram(xop, x):
    xf = xop.data
    return xf.t() @ xf, xf.sum(0)


class GramState(dict):
    __getattr__ = dict.__getitem__


def attn_gram_prepare_fwd(G, s, wq, bq, wk, bk, wv, bv, n):
    nf = float(n)
    kx = wk @ G + torch.outer(bk, s)
    qx = wq @ G + torch.outer(bq, s)
    vx = wv @ G + torch.outer(bv, s)
    z1, q1, v1 = wk @ s + nf * bk, wq @ s + nf * bq, wv @ s + nf * bv
    S = kx @ wv.t() + torch.outer(z1, bv)
    nk2 = (kx * wk).sum() + z1 @ bk
    nq2 = (qx * wq).sum() + q1 @ bq
    alpha = nq2.rsqrt() * nk2.rsqrt()
    beta = alpha / nf
    Bt = beta * (S.t() @ wq) + wv                       # [d, h]: the apply GEMM's B operand (K-major over h)
    tail = G.new_zeros(16, wq.shape[1])
    tail[0] = beta * (wq.t() @ z1)
    bt = beta * (S.t() @ bq) + bv
    sc = G.new_zeros(16)
    sc[SC_NQ2], sc[SC_NK2], sc[SC_ALPHA], sc[SC_BETA], sc[SC_DEN], sc[SC_N] = nq2, nk2, alpha, beta, beta * (bq @ z1) + 1.0, nf
    return GramState(wq=wq, bq=bq, wk=wk, bk=bk, wv=wv, bv=bv, G=G, s=s, kx=kx, qx=qx, vx=vx, z1=z1, q1=q1, v1=v1, S=S, Bt=Bt,
                     tail=tail, bt=bt, sc=sc, n=n)


def attn_gram_prepare_bwd(st, P, pg, cs, sg):
    """P = x^T gnum' [h,d], pg = x^T gden' [h], cs = colsum(gnum') [d], sg = sum(gden') [1] with gnum' = g/den~, gden' = -(g.o)/den~."""
    wq, bq, wk, bk, wv, bv = st.wq, st.bq, st.wk, st.bk, st.wv, st.bv
    S, z1, kx, qx, vx, q1, v1, s = st.S, st.z1, st.kx, st.qx, st.vx, st.q1, st.v1, st.s
    beta, alpha, nq2, nk2 = st.sc[SC_BETA], st.sc[SC_ALPHA], st.sc[SC_NQ2], st.sc[SC_NK2]
    dS = wq @ P + torch.outer(bq, cs)
    dz = wq @ pg + bq * sg
    c = beta * ((dS * S).sum() + (dz * z1).sum())
    cq, ck = -c / nq2, -c / nk2
    dwq = beta * (S @ P.t()) + beta * torch.outer(z1, pg) + cq * qx
    dbq = beta * (S @ cs + sg * z1) + cq * q1
    dwk = beta * (dS @ vx) + beta * torch.outer(dz, s) + ck * kx
    dbk = beta * (dS @ v1) + alpha * dz + ck * z1
    dwv = beta * (dS.t() @ kx) + P.t()
    dbv = beta * (dS.t() @ z1) + cs
    U = dS @ wv
    A3 = cq * (wq.t() @ wq) + ck * (wk.t() @ wk) + beta * (wk.t() @ U + U.t() @ wk)
    a4 = cq * (wq.t() @ bq) + ck * (wk.t() @ bk) + beta * (wk.t() @ (dz + dS @ bv) + wv.t() @ (dS.t() @ bk))
    bcat = torch.cat([st.Bt.t(), A3], 1).contiguous()     # [h, d+h]: B operand of dx = gnum'.Bt + x.A3 (+ gden' (x) tail0 + a4)
    return dwq, dbq, dwk, dbk, dwv, dbv, bcat, a4


def attn_prepare_fwd(s_raw, z_raw, nq2v, nk2v, planes):
    inq, ink = nq2v.sum().rsqrt(), nk2v.sum().rsqrt()
    inv = inq * ink
    m, d = s_raw.shape
    bm = (s_raw.t() * inv).contiguous()
    bt = torch.zeros(16, m)
    bt[0] = z_raw * inv
    if planes == 1:
        bm, bt = bm.bfloat16().float(), bt.bfloat16().float()
    return Operand(bm, d, m, m, planes), Operand(bt, 16, m, m, planes), torch.stack([inq, ink, inv, torch.zeros(())])


def attn_bwd_prep(g, o, den, gscale):
    inv = gscale / den
    gnum = _st(alloc_act(g.shape[0], g.shape[1], g.dtype, g.device), g.float() * inv[:, None])
    gden = -(g.float() * o.float()).sum(1) * inv
    return gnum, gden


def attn_prepare_bwd(s_raw, z_raw, ds_raw, dz_raw, scal_fwd, planes, scal_bwd):
    inq, ink, alpha = scal_fwd[0], scal_fwd[1], scal_fwd[2]
    c = alpha * ((s_raw * ds_raw).sum() + (z_raw * dz_raw).sum())
    scal_bwd[0], scal_bwd[1], scal_bwd[2], scal_bwd[3] = alpha, -c * inq * inq, -c * ink * ink, c
    m, d = s_raw.shape

    def op(t):
        t = t.contiguous()
        if planes == 1:
            t = t.bfloat16().float()
        return Operand(t, t.shape[0], t.shape[1], t.shape[1], planes)

    return op(s_raw), op(ds_raw.t()), op(ds_raw), alpha * z_raw, alpha * dz_raw


def attn_combine_scal(scal_bwd_all, heads, scal_fwd):
    c = scal_bwd_all[:, 3].sum()
    scal_bwd_all[:, 1] = -c * scal_fwd[0] ** 2
    scal_bwd_all[:, 2] = -c * scal_fwd[1] ** 2


def softmax_nll(logits, labels, mask, scale, want_grad=True):
    lp = torch.log_softmax(logits.float(), 1)
    sel = torch.ones(logits.shape[0], dtype=torch.bool) if mask is None else mask.bool()
    loss = -(lp[torch.arange(logits.shape[0]), labels] * sel).sum() * scale
    d = None
    if want_grad:
        d = lp.exp()
        d[torch.arange(logits.shape[0]), labels] -= 1.0
        d = d * sel[:, None] * scale
    return loss.reshape(1), d


def launch_count():
    return 0


class EmuGraph:
    def __init__(self, edge_index, n, self_loop_mode=0, rows=None, col_rot=None):
        self.n, self.edge_index, self.self_loop_mode, self.rows, self.col_rot = n, edge_index, self_loop_mode, rows, col_rot
        self.rowptr, self.col, self.dinv = csr_build(edge_index, n, False, self_loop_mode, True, rows=rows, col_rot=col_rot)
        self.heavy = self.heavy_t = None

    def transpose(self):
        if not hasattr(self, "_t"):
            rp, cl, _ = csr_build(self.edge_index, self.n, True, self.self_loop_mode, False, rows=self.rows, col_rot=self.col_rot)
            self._t = (rp, cl)
        return self._t

    def row_splits(self, thresholds, transposed=False):
        rp, cl = self.transpose() if transposed else (self.rowptr, self.col)
        return csr_row_splits(rp, cl, thresholds)
