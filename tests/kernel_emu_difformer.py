"""torch-CPU emulation of the DIFFormer kernel modes — TEST INFRASTRUCTURE ONLY.

Extends tests/kernel_emu.py (which it re-exports unchanged) with the contracts of the entry points the DIFFormer schedules use:
the value-sum mode of the Gram h x h algebra (sgf_attn_gram_prepare_fwd_vsum / _bwd_vsum), the row pass with the graph term
(sgf_ln_fwd_graph), the LayerNorm backward + attention prologue that also writes the pre-scaled SpMM operand
(sgf_ln_bwd_attn_graph), and colstats accumulating into a given vector.  Tests monkeypatch `engine.K` / `functional.K` with
this module."""
import torch

import kernel_emu as _base
from dropout_mask import apply_kernel_dropout
from kernel_emu import *  # noqa: F401,F403
from kernel_emu import _f, _st, new_like

SC_NQ2, SC_NK2, SC_ALPHA, SC_BETA, SC_DEN, SC_N = (_base.SC_NQ2, _base.SC_NK2, _base.SC_ALPHA, _base.SC_BETA, _base.SC_DEN,
                                                   _base.SC_N)


def colstats(x, w=None, want_sum=True, want_sumsq=True, sum_out=None):
    """kernels.colstats; sum_out: the column sums are added to it (and returned)."""
    s, q = _base.colstats(x, w, want_sum or sum_out is not None, want_sumsq)
    if sum_out is not None:
        sum_out += s
        s = sum_out
    return s, q


def attn_gram_prepare_fwd(G, s, wq, bq, wk, bk, wv, bv, n, vsum=False):
    """vsum=True (sgf_attn_gram_prepare_fwd_vsum): the numerator adds sum_l v_l instead of N v_n, so
    Bt = beta S^T Wq (no Wv) and bt = beta S^T bq + v1 / N."""
    st = _base.attn_gram_prepare_fwd(G, s, wq, bq, wk, bk, wv, bv, n)
    st["vsum"] = bool(vsum)
    if vsum:
        beta = st.sc[SC_BETA]
        st["Bt"] = beta * (st.S.t() @ wq)
        st["bt"] = beta * (st.S.t() @ bq) + st.v1 / float(n)
    return st


def attn_gram_prepare_fwd_vsum(G, s, wq, bq, wk, bk, wv, bv, n):
    return attn_gram_prepare_fwd(G, s, wq, bq, wk, bk, wv, bv, n, vsum=True)


def attn_gram_prepare_bwd(st, P, pg, cs, sg):
    """vsum mode (sgf_attn_gram_prepare_bwd_vsum): dWv = beta dS^T kx + cs s^T / N instead of beta dS^T kx + P^T, and
    a4 += Wv^T cs / N; everything else as the base contract."""
    dwq, dbq, dwk, dbk, dwv, dbv, bcat, a4 = _base.attn_gram_prepare_bwd(st, P, pg, cs, sg)
    if st.get("vsum"):
        nf = float(st.n)
        dwv = dwv - P.t() + torch.outer(cs, st.s) / nf
        a4 = a4 + st.wv.t() @ cs / nf
    return dwq, dbq, dwk, dbk, dwv, dbv, bcat, a4


def ln_fwd_graph(x, r, gy, a, b, c, gamma, beta, use_ln, use_relu, p, seed, want_stats=True):
    """sgf_ln_fwd_graph: ln_fwd of u = a*x + b*r + c*gy."""
    u = a * _f(x) + (b * _f(r) if r is not None else 0.0) + c * _f(gy)
    return _base.ln_fwd(u, None, 1.0, 0.0, gamma, beta, use_ln, use_relu, p, seed, want_stats)


def ln_bwd_attn_graph(dy, o, r, xa, gy, a, b, c, gamma, beta, stats, use_ln, p, seed, gscale, want_dr, dgamma, dbeta, den, dinv):
    """sgf_ln_bwd_attn_graph: sgf_ln_bwd_attn for u = a*o + b*r + c*gy, plus ys = dinv (.) (c*du)."""
    u = a * _f(o) + (b * _f(r) if r is not None else 0.0) + c * _f(gy)
    g = apply_kernel_dropout(gscale * _f(dy), seed, p)
    if use_ln:
        mean = u.mean(1)
        rstd = (u.var(1, unbiased=False) + 1e-5).rsqrt()
        xh = (u - mean[:, None]) * rstd[:, None]
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
    ys = _st(new_like(o), (c * du) * dinv[:, None])
    return gnum, gden, dr, ys, gnum_f.sum(0), (_f(xa) * gden[:, None]).sum(0), gden.sum().reshape(1)
