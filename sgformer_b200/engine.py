"""Hand-scheduled forward / backward of the SGFormer encoder on the sm_90a kernels.

One schedule per branch — `trans_*` (TransConv: input MLP + linear-attention layers), `gconv_*` (GraphConv of
large/100M), `gcn_*` (PyG-GCN backbone of medium), `head_*` (branch mix + fc) — each a forward that records what the
backward needs in a `Tape`, and a backward that walks the tape and fills a gradient dict keyed by the reference's
parameter names.  There is no autograd inside: torch.autograd sees a single Function (functional.py) per call.

Reference semantics reproduced (paths in the reference repository): large/ours.py:25-42 (GraphConvLayer), :74-94 (GraphConv,
incl. the "residual always adds layer_[0]" quirk), :121-162 / medium/ours.py:14-46,74-100 (TransConvLayer +
full_attention_conv), :194-219 / medium/ours.py:133-160 / 100M/ours.py:247-272 (TransConv, the two residual rules),
medium/models.py:49-63 (GCN over PyG GCNConv), large/ours.py:265-276 (SGFormer.forward).
"""
from __future__ import annotations

import itertools
from collections import OrderedDict
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch

from . import kernels as K
from ._lib import EPI_ATTN_APPLY, EPI_ATTN_GRAM
from .dist import SINGLE, Comm
from .graph import Graph

Tensor = torch.Tensor


@dataclass
class Precision:
    """'bf16': bf16 activations, single-plane bf16 tensor-core operands (parity 1e-2).
    'fp32': fp32 activations, bf16x3 split operands — six tensor-core products per GEMM, fp32-accurate (parity 1e-4)."""
    name: str

    @property
    def act_dtype(self):
        return torch.bfloat16 if self.name == "bf16" else torch.float32

    @property
    def planes(self) -> int:
        return 1 if self.name == "bf16" else 3


BF16 = Precision("bf16")
FP32 = Precision("fp32")


def precision(name: str) -> Precision:
    if name in ("bf16", "bfloat16"):
        return BF16
    if name in ("fp32", "float32"):
        return FP32
    raise ValueError(f"unknown precision {name!r} (use 'bf16' or 'fp32')")


_seed_counter = itertools.count(1)


def next_seed() -> int:
    """Per-forward dropout seed: deterministic under torch.manual_seed, no device sync."""
    return ((torch.initial_seed() * 0x9E3779B1) ^ (next(_seed_counter) * 0x85EBCA6B)) & 0x7FFFFFFFFFFFFFFF


# Offsets of the dropout calls from the forward's seed (+ the layer index where marked).  A backward recomputes its
# forward's mask from the same seed, so both read these; changing a value changes every mask a training step draws.
_SEED_STEM = 101            # TransConv / DIFFormer input stem
_SEED_LAYER = 211           # + i: TransConv / DIFFormer layer i
_SEED_GCONV_STEM = 307      # GraphConv input layer
_SEED_GCONV_LAYER = 401     # + i: GraphConv layer i
_SEED_GCN_LAYER = 503       # + i: GCN layer i
_SEED_GAT_INPUT = 601       # GAT input dropout
_SEED_GAT_ACT = 611         # + i: dropout after GAT layer i's ELU
_SEED_GAT_ATT = 653         # + i: attention dropout of GAT layer i
_SEED_GCNJK_LAYER = 701     # + i: GCNJK layer i


def check_width(h: int, prec: Precision, what: str):
    """The row kernels move rows in 16-byte chunks, at most 128 chunks per row (csrc/rowops.cu make_geom): fail with a clear
    message instead of SGF_ERR_ARG from the first LayerNorm/BatchNorm launch.  (The reference has no such limit.)"""
    vn = 8 if prec.name == "bf16" else 4
    if h % vn != 0 or h > 128 * vn:
        raise ValueError(f"sgformer_b200: {what} = {h} is not supported in precision '{prec.name}': it must be a multiple of {vn} "
                         f"and at most {128 * vn}" + (" (use set_precision('bf16') for wider layers)" if prec.name != "bf16" and h % 8 == 0 and h <= 1024 else ""))


class Tape(dict):
    """Saved tensors / scalars of one forward."""
    pass


def _w(P: Dict[str, Tensor], name: str, prec: Precision, transpose: bool = False) -> K.Operand:
    return K.pack_operand(P[name], transpose, prec.planes)


def _b_blocks(w: Tensor, widths, prec: Precision):
    """B side of a GEMM that contracts each column block (of `widths`) of w [n_out, sum(widths)] with an A source of its own
    -> (operands, [(operand index, K offset)] per block).  A TMA load starts on a 16-byte boundary, so a block must start at a
    multiple of 8 bf16 columns of its operand (K.gemm_nt refuses anything else).  Where one does not (fp32 widths such as
    h = 100), every block is packed as an operand of its own and read from offset 0."""
    offs = [sum(widths[:j]) for j in range(len(widths))]
    if all(o % 8 == 0 for o in offs):
        return [K.pack_operand(w, False, prec.planes)], [(0, o) for o in offs]
    return [K.pack_operand(w[:, o:o + k], False, prec.planes) for o, k in zip(offs, widths)], [(j, 0) for j in range(len(widths))]


_xin_cache: "OrderedDict[tuple, tuple]" = OrderedDict()


def input_operand(x: Tensor, prec: Precision) -> K.Operand:
    """Raw node features fp32 [N, d_in] -> tensor-core operand (read by both branches' input Linear).  Full-batch
    training feeds the same feature tensor every step, so the packed operand is cached on the tensor's identity/version."""
    key = (x.data_ptr(), tuple(x.shape), x._version, str(x.dtype), prec.name, x.device.index)
    hit = _xin_cache.get(key)
    if hit is not None and hit[0] is x:
        _xin_cache.move_to_end(key)
        return hit[1]
    xs = x
    if xs.dtype != torch.float32:
        xs = xs.float()
    if xs.stride(-1) != 1:
        xs = xs.contiguous()
    op = K.pack_operand(xs.detach(), False, prec.planes)
    _xin_cache[key] = (x, op)
    while len(_xin_cache) > 2:
        _xin_cache.popitem(last=False)
    return op


# =================================================================================================
# linear attention core (full_attention_conv)
# =================================================================================================
def attention_forward(q: Tensor, k: Tensor, v: Tensor, heads: int, prec: Precision, tape: Optional[Tape],
                      comm: Comm = SINGLE, stats=None, shared_v: bool = False) -> Tensor:
    """q,k: [N, H*M], v: [N, H*D] activations (views allowed) -> o [N, H*D].  medium/ours.py:14-34.
    One Frobenius norm over all heads (medium/ours.py:16-17); N is the query count (the GLOBAL node count when the rows
    are sharded: the un-normalised partials {S', z', ||q||^2, ||k||^2} are all-reduced once, C1).
    shared_v: v is [N, D], one value for every head (the reference's one-head vs broadcast by einsum, medium/ours.py:21-23)."""
    n_loc = q.shape[0]
    n = comm.n_global if comm.active else n_loc
    m = q.shape[1] // heads
    d = v.shape[1] if shared_v else v.shape[1] // heads
    dev = q.device
    if stats is not None:        # (sum of squares of q columns, column sums of k, sum of squares of k columns) from the
        sq_q, z_raw, sq_k = stats    # producing GEMM's epilogue
    else:
        _, sq_q = K.colstats(q, want_sum=False)
        z_raw, sq_k = K.colstats(k)
    if shared_v:            # S'_h = k_h^T v of every head in one GEMM: [H*M, D], k and v read once
        s_all = torch.empty((heads * m, d), dtype=torch.float32, device=dev)
        K.gemm_tn(K.as_operand(k, prec.planes, memo=True), K.as_operand(v, prec.planes, memo=True), s_all)
        s_list = list(s_all.split(m))
        comm.allreduce_(sq_q, z_raw, sq_k, s_all)
    else:
        s_list = []
        for hd in range(heads):
            kh, vh = k[:, hd * m:(hd + 1) * m], v[:, hd * d:(hd + 1) * d]
            s_raw = torch.empty((m, d), dtype=torch.float32, device=dev)
            K.gemm_tn(K.as_operand(kh, prec.planes, memo=True), K.as_operand(vh, prec.planes, memo=True), s_raw)
            s_list.append(s_raw)
        comm.allreduce_(sq_q, z_raw, sq_k, *s_list)
    o = K.alloc_act(n_loc, heads * d, q.dtype, dev)
    den = torch.empty((heads, n_loc), dtype=torch.float32, device=dev)
    scal = None
    for hd in range(heads):
        qh, vh = q[:, hd * m:(hd + 1) * m], v if shared_v else v[:, hd * d:(hd + 1) * d]
        bmat, btail, scal = K.attn_prepare_fwd(s_list[hd], z_raw[hd * m:(hd + 1) * m], sq_q, sq_k, prec.planes)
        K.gemm_nt([K.as_operand(qh, prec.planes, memo=True)], [bmat], [(0, 0, 0, 0, m)], d, o[:, hd * d:(hd + 1) * d],
                  epi=EPI_ATTN_APPLY, aux=vh, tail=btail, nf=float(n), den_out=den[hd])
    if tape is not None:
        tape.update(q=q, k=k, v=v, o=o, den=den, s=s_list, z=z_raw, scal=scal, heads=heads, m=m, d=d, n=n, shared_v=shared_v)
    return o


def attention_backward(tape: Tape, g: Tensor, gscale: float, prec: Precision, dq: Tensor, dk: Tensor,
                       dv: Optional[Tensor], dv_accumulate: bool = False, comm: Comm = SINGLE):
    """g = dL/do [N, H*D] (times gscale), or [N, D] when every head receives the same gradient (the head mean's backward).
    Writes dq, dk [N, H*M] and dv [N, H*D] (+= if dv_accumulate).  With a shared v (attention_forward(shared_v=True)) dv is
    [N, D]: the heads' contributions are summed into it in head order (the first one += only if dv_accumulate).
    SURVEY.md Appendix A.1 in the raw-q/k form documented at sgf_attn_prepare_bwd; row-sharded: {dS', dz'} all-reduced (C2)."""
    q, k, v, o, den = tape["q"], tape["k"], tape["v"], tape["o"], tape["den"]
    heads, m, d, n = tape["heads"], tape["m"], tape["d"], tape["n"]
    shared_v = tape.get("shared_v", False)
    shared_g = g.shape[1] == d
    dev = q.device
    scal_bwd = torch.zeros((heads, 8), dtype=torch.float32, device=dev)
    part = []
    for hd in range(heads):
        qh = q[:, hd * m:(hd + 1) * m]
        gnum, gden = K.attn_bwd_prep(g if shared_g else g[:, hd * d:(hd + 1) * d], o[:, hd * d:(hd + 1) * d], den[hd], gscale)
        gnum_op = K.as_operand(gnum, prec.planes)
        ds_raw = torch.empty((m, d), dtype=torch.float32, device=dev)
        K.gemm_tn(K.as_operand(qh, prec.planes, memo=True), gnum_op, ds_raw)
        dz_raw, _ = K.colstats(qh, w=gden, want_sumsq=False)
        part.append((gnum, gden, gnum_op, ds_raw, dz_raw))
    comm.allreduce_(*[t for p_ in part for t in (p_[3], p_[4])])
    per_head = []
    for hd in range(heads):
        gnum, gden, gnum_op, ds_raw, dz_raw = part[hd]
        ops = K.attn_prepare_bwd(tape["s"][hd], tape["z"][hd * m:(hd + 1) * m], ds_raw, dz_raw, tape["scal"], prec.planes,
                                 scal_bwd[hd])
        per_head.append((gnum, gden, gnum_op, ops))
    if heads > 1:
        K.attn_combine_scal(scal_bwd, heads, tape["scal"])
    for hd in range(heads):
        gnum, gden, gnum_op, (b_dq, b_dv, b_dk, r1_col, dk_bias) = per_head[hd]
        qh, kh = q[:, hd * m:(hd + 1) * m], k[:, hd * m:(hd + 1) * m]
        vh = v if shared_v else v[:, hd * d:(hd + 1) * d]
        sb = scal_bwd[hd]
        K.gemm_nt([gnum_op], [b_dq], [(0, 0, 0, 0, d)], m, dq[:, hd * m:(hd + 1) * m], alpha_dev=sb[0:1], aux=qh, beta=1.0,
                  beta_dev=sb[1:2], r1_row=gden, r1_col=r1_col)
        K.gemm_nt([K.as_operand(vh, prec.planes, memo=True)], [b_dk], [(0, 0, 0, 0, d)], m, dk[:, hd * m:(hd + 1) * m], alpha_dev=sb[0:1],
                  aux=kh, beta=1.0, beta_dev=sb[2:3], bias=dk_bias)
        if dv is not None:
            K.gemm_nt([K.as_operand(kh, prec.planes, memo=True)], [b_dv], [(0, 0, 0, 0, m)], d,
                      dv if shared_v else dv[:, hd * d:(hd + 1) * d], alpha_dev=sb[0:1], aux=gnum, beta=float(n),
                      accumulate=dv_accumulate or (shared_v and hd > 0))


# =================================================================================================
# linear attention in Gram form (single head): projections + full_attention_conv without materialising q, k, v
# =================================================================================================
# With q = x Wq^T + bq, k = x Wk^T + bk, v = x Wv^T + bv every node-contracted quantity of full_attention_conv
# (medium/ours.py:16-31) is a function of the Gram matrix G = x^T x and the column sums s = x^T 1 of the layer input:
#   k^T v = Wk G Wv^T + (Wk s) bv^T + bk (Wv s)^T + N bk bv^T,   k^T 1 = Wk s + N bk,
#   ||k||^2 = <Wk G + bk s^T, Wk> + (k^T 1).bk   (same for q),
# so pass 1 is ONE node contraction x^T x (reads x once) and pass 2 ONE GEMM x . Bt^T with
#   Bt = (alpha/N) S'^T Wq + Wv,  out = (x Bt^T + bt) / (x ct + dt)      (alpha = 1/(||q|| ||k||); see sgf_attn_gram_prepare_fwd).
# The backward contracts P = x^T gnum', x^T gden' the same way: dWq, dWk, dWv come out of h x h algebra, dx is one
# two-segment GEMM [gnum' | x] . [Bt | A3] (sgf_attn_gram_prepare_bwd).  Forward traffic 3 N h b instead of 12 N h b,
# 4 N h^2 flops instead of 10 N h^2; identical mathematics (fp64 check: tests/test_gram_attention_math.py).
_eye_cache: dict = {}


def _identity_v(h: int, dev):
    """use_weight=False: V is the layer input itself (medium/ours.py:84) = projection by the identity with zero bias."""
    key = (h, str(dev))
    if key not in _eye_cache:
        _eye_cache[key] = (torch.eye(h, dtype=torch.float32, device=dev), torch.zeros(h, dtype=torch.float32, device=dev))
    return _eye_cache[key]


def attention_gram_forward(P: Dict[str, Tensor], lp: str, x: Tensor, use_weight: bool, prec: Precision, tape: Optional[Tape],
                           comm: Comm = SINGLE, vsum: bool = False) -> Tensor:
    """x: [N, h] layer input (activation) -> full_attention_conv(Wq x, Wk x, Wv x) [N, h], one head.
    vsum=True: DIFFormer's `simple` kernel (numerator + sum_l v_l instead of + N v_n, medium/difformer.py:18-39)."""
    n_loc, h = x.shape
    n = comm.n_global if comm.active else n_loc
    dev = x.device
    xop = K.as_operand(x, prec.planes, memo=True)
    G, s = K.gram(xop, x)
    comm.allreduce_(G, s)                                     # C1: h*h + h floats
    wv, bv = (P[lp + "Wv.weight"], P[lp + "Wv.bias"]) if use_weight else _identity_v(h, dev)
    prepare = K.attn_gram_prepare_fwd_vsum if vsum else K.attn_gram_prepare_fwd
    st = prepare(G, s, P[lp + "Wq.weight"], P[lp + "Wq.bias"], P[lp + "Wk.weight"], P[lp + "Wk.bias"], wv, bv, n)
    bop = K.pack_operand(st.Bt, False, prec.planes)
    btail = K.pack_operand(st.tail, False, prec.planes)
    d = st.Bt.shape[0]
    o = K.alloc_act(n_loc, d, x.dtype, dev)
    den = torch.empty(n_loc, dtype=torch.float32, device=dev)
    K.gemm_nt([xop], [bop], [(0, 0, 0, 0, h)], d, o, epi=EPI_ATTN_GRAM, bias=st.bt, tail=btail,
              nf_dev=st.sc[K.SC_DEN:K.SC_DEN + 1], den_out=den)
    if tape is not None:
        tape.update(st=st, den=den, xop=xop, n=n)
    return o


def attention_gram_backward(P: Dict[str, Tensor], lp: str, tape: Tape, x: Tensor, gnum: Tensor, gden: Tensor, cs: Tensor,
                            pg: Tensor, sg: Tensor, use_weight: bool, prec: Precision, dprev: Tensor, accumulate: bool,
                            grads: Dict[str, Tensor], comm: Comm = SINGLE, *, dv: Optional[Tensor] = None):
    """gnum' = g/den~ [N,h], gden' = -(g.o)/den~ [N] and their column sums (sgf_ln_bwd_attn) -> parameter gradients and
    dprev (+)= d/dx of the attention (through q, k and v).  dv: a further gradient of v = x Wv^T + bv (DIFFormer's graph
    term, from the transposed SpMM), added to dWv, dbv and dprev; single device only, as it is not all-reduced."""
    st = tape["st"]
    h = x.shape[1]
    d = gnum.shape[1]
    dev = x.device
    xop = tape["xop"]
    gnum_op = K.as_operand(gnum, prec.planes)
    pmat = torch.empty((h, d), dtype=torch.float32, device=dev)
    K.gemm_tn(xop, gnum_op, pmat)
    comm.allreduce_(pmat, pg, cs, sg)                         # C2
    dwq, dbq, dwk, dbk, dwv, dbv, bcat, a4 = K.attn_gram_prepare_bwd(st, pmat, pg, cs, sg)
    B, at = _b_blocks(bcat, [d, h], prec)
    A = [gnum_op, xop]
    pairs = [(0, 0, at[0][0], at[0][1], d), (1, 0, at[1][0], at[1][1], h)]
    if dv is not None:
        dv_op = K.as_operand(dv, prec.planes)
        if use_weight:
            K.gemm_tn(dv_op, xop, dwv, beta=1.0)
            K.colstats(dv, want_sumsq=False, sum_out=dbv)
        A.append(dv_op)
        B.append(K.pack_operand(P[lp + "Wv.weight"] if use_weight else _identity_v(h, dev)[0], True, prec.planes))
        if prec.planes == 1:            # dv Wv as a third segment of the dx GEMM
            pairs.append((2, 0, len(B) - 1, 0, d))
    grads[lp + "Wq.weight"], grads[lp + "Wq.bias"] = dwq, dbq
    grads[lp + "Wk.weight"], grads[lp + "Wk.bias"] = dwk, dbk
    names = [lp + "Wq.weight", lp + "Wq.bias", lp + "Wk.weight", lp + "Wk.bias"]
    if use_weight:
        grads[lp + "Wv.weight"], grads[lp + "Wv.bias"] = dwv, dbv
        names += [lp + "Wv.weight", lp + "Wv.bias"]
    _mark_global(grads, comm, *names)          # built from all-reduced contractions: already global sums
    K.gemm_nt(A, B, pairs, h, dprev, bias=a4, r1_row=gden, r1_col=st.tail[0], accumulate=accumulate)
    if dv is not None and prec.planes != 1:     # bf16x3: 3 x 6 partial products exceed the GEMM's 16 segments
        K.gemm_nt([A[2]], [B[-1]], [(0, 0, 0, 0, d)], h, dprev, accumulate=True)


# =================================================================================================
# TransConv branch
# =================================================================================================
def _res_coef(cfg: dict):
    if not cfg["trans_use_residual"]:
        return 1.0, 0.0, False
    if cfg["variant"] == "large":
        return 0.5, 0.5, True           # large/ours.py:211
    a = float(cfg["alpha"])
    return a, 1.0 - a, True             # medium/ours.py:152, 100M/ours.py:264


def _qkv_weight(P, pfx: str, use_weight: bool) -> (Tensor, Tensor):
    ws = [P[pfx + "Wq.weight"], P[pfx + "Wk.weight"]] + ([P[pfx + "Wv.weight"]] if use_weight else [])
    bs = [P[pfx + "Wq.bias"], P[pfx + "Wk.bias"]] + ([P[pfx + "Wv.bias"]] if use_weight else [])
    return torch.cat(ws, 0), torch.cat(bs, 0)


def _project_qkv(P, lp: str, xop: K.Operand, use_weight: bool, prec: Precision, stats: bool):
    """q | k (| v when use_weight) of a layer with materialised projections, in one GEMM of the layer input -> qkv [N, nout]
    and, with `stats`, the column sums and sums of squares its epilogue accumulates (else None, None)."""
    wcat, bcat = _qkv_weight(P, lp, use_weight)
    nout = wcat.shape[0]
    dev = wcat.device
    qkv = torch.empty((xop.rows, K.ceil_to(nout, 8)), dtype=prec.act_dtype, device=dev)[:, :nout]
    csum, csq = (torch.zeros(nout, dtype=torch.float32, device=dev), torch.zeros(nout, dtype=torch.float32, device=dev)) \
        if stats else (None, None)
    K.gemm_nt([xop], [K.pack_operand(wcat, False, prec.planes)], [(0, 0, 0, 0, xop.k)], nout, qkv, bias=bcat, col_sum=csum,
              col_sumsq=csq)
    return qkv, csum, csq


def _stem_forward(P, pfx: str, xin: K.Operand, h: int, use_ln: bool, prec: Precision, p: float = 0.0, seed: int = 0,
                  want_stats: bool = False):
    """Input Linear fcs.0, then LayerNorm?/ReLU/dropout (TransConv, DIFFormer) -> (t0, x, LayerNorm statistics)."""
    t0 = K.alloc_act(xin.rows, h, prec.act_dtype, xin.data.device)
    K.gemm_nt([xin], [_w(P, pfx + "fcs.0.weight", prec)], [(0, 0, 0, 0, xin.k)], h, t0, bias=P[pfx + "fcs.0.bias"])
    x, st = K.ln_fwd(t0, None, 1.0, 0.0, P.get(pfx + "bns.0.weight"), P.get(pfx + "bns.0.bias"), use_ln, True, p, seed, want_stats)
    return t0, x, st


def _stem_backward(P, pfx: str, tape: Tape, dout: Tensor, gscale: float, use_ln: bool, prec: Precision,
                   grads: Dict[str, Tensor], want_dx: bool) -> Optional[Tensor]:
    """Backward of _stem_forward (its t0, xin and statistics read from `tape`): fills the fcs.0 and bns.0 gradients and, with
    want_dx, returns the gradient of the raw features."""
    t0, xin = tape["t0"], tape["xin"]
    n, h = t0.shape
    d_in = xin.k
    dev = dout.device
    dg, db = (torch.zeros(h, dtype=torch.float32, device=dev), torch.zeros(h, dtype=torch.float32, device=dev)) if use_ln \
        else (None, None)
    dt0, _ = K.ln_bwd(dout, t0, None, 1.0, 0.0, P.get(pfx + "bns.0.weight"), P.get(pfx + "bns.0.bias"), tape["st0"], use_ln, True,
                      tape["p"], tape["seed"] + _SEED_STEM, gscale, False, dg, db)
    if use_ln:
        grads[pfx + "bns.0.weight"], grads[pfx + "bns.0.bias"] = dg, db
    dt0_op = K.as_operand(dt0, prec.planes)
    dw0 = torch.empty((h, d_in), dtype=torch.float32, device=dev)
    K.gemm_tn(dt0_op, xin, dw0)
    grads[pfx + "fcs.0.weight"] = dw0
    grads[pfx + "fcs.0.bias"], _ = K.colstats(dt0, want_sumsq=False)
    if not want_dx:
        return None
    dx = torch.empty((n, d_in), dtype=torch.float32, device=dev)
    K.gemm_nt([dt0_op], [_w(P, pfx + "fcs.0.weight", prec, transpose=True)], [(0, 0, 0, 0, h)], d_in, dx)
    return dx


def trans_forward(P: Dict[str, Tensor], cfg: dict, xin: K.Operand, prec: Precision, training: bool, seed: int,
                  tape: Optional[Tape], pfx: str = "trans_conv.", comm: Comm = SINGLE) -> Tensor:
    h, H = cfg["hidden"], cfg["num_heads"]
    check_width(h, prec, "hidden_channels")
    p = float(cfg["trans_dropout"]) if training else 0.0
    use_ln = bool(cfg["trans_use_bn"])
    t0, x, st = _stem_forward(P, pfx, xin, h, use_ln, prec, p, seed + _SEED_STEM, tape is not None)
    if tape is not None:
        tape.update(xin=xin, t0=t0, st0=st, layers=[], p=p, seed=seed, n=xin.rows)
    ca, cb, use_res = _res_coef(cfg)
    use_weight = bool(cfg["trans_use_weight"])
    for i in range(cfg["trans_num_layers"]):
        lp = f"{pfx}convs.{i}."
        at = Tape() if tape is not None else None
        if H == 1:
            a = attention_gram_forward(P, lp, x, use_weight, prec, at, comm)
            saved = dict(gram=True)
        else:
            # K^T 1, ||Q||^2, ||K||^2 fall out of the projection's epilogue.  use_weight=False: every head attends over the
            # layer input itself (the reference's one-head V broadcast across heads, medium/ours.py:84 and :21-23)
            qkv, csum, csq = _project_qkv(P, lp, K.as_operand(x, prec.planes, memo=True), use_weight, prec, stats=True)
            q, k = qkv[:, :H * h], qkv[:, H * h:2 * H * h]
            v = qkv[:, 2 * H * h:] if use_weight else x
            o = attention_forward(q, k, v, H, prec, at, comm, stats=(csq[:H * h], csum[H * h:2 * H * h], csq[H * h:2 * H * h]),
                                  shared_v=not use_weight)
            a = K.head_mean(o, H, h)
            saved = dict(nout=qkv.shape[1])
        y, st = K.ln_fwd(a, x if use_res else None, ca, cb, P.get(f"{pfx}bns.{i + 1}.weight"), P.get(f"{pfx}bns.{i + 1}.bias"),
                         use_ln, bool(cfg["trans_use_act"]), p, seed + _SEED_LAYER + i, tape is not None)
        if tape is not None:
            tape["layers"].append(dict(saved, x_in=x, attn=at, a=a, st=st))
        x = y
    return x


def trans_attentions(P: Dict[str, Tensor], cfg: dict, xin: K.Operand, prec: Precision, with_act: bool,
                     pfx: str = "trans_conv.") -> List[Tensor]:
    """TransConv.get_attentions (large/ours.py:221-238, medium/ours.py:162-177, 100M/ours.py:274-289): per attention layer the
    [N, N] visualisation matrix  mean_h(q~_h k~_h^T) / mean_h(q~_h . sum_l k~_l + N)  of large/ours.py:152-155.  The N x N product is one
    tensor-core GEMM of the concatenated heads (sum over heads of per-head dot products) with 1/(H ||q|| ||k||) read from the
    device and the row normaliser as its row scale; the layer stack itself runs the un-fused attention (q, k materialised).
    Inference only (no dropout, no tape), O(N^2) memory like the reference: meant for small graphs."""
    h, H = cfg["hidden"], cfg["num_heads"]
    check_width(h, prec, "hidden_channels")
    n = xin.rows
    dev = xin.data.device
    use_ln = bool(cfg["trans_use_bn"])
    ca, cb, use_res = _res_coef(cfg)
    use_weight = bool(cfg["trans_use_weight"])
    _, x, _ = _stem_forward(P, pfx, xin, h, use_ln, prec)
    out = []
    for i in range(cfg["trans_num_layers"]):
        lp = f"{pfx}convs.{i}."
        qkv, _, _ = _project_qkv(P, lp, K.as_operand(x, prec.planes), use_weight, prec, stats=False)
        q, k = qkv[:, :H * h], qkv[:, H * h:2 * H * h]
        v = qkv[:, 2 * H * h:] if use_weight else x
        at = Tape()
        o = attention_forward(q, k, v, H, prec, at, shared_v=not use_weight)
        inv_norm = at["den"].mean(dim=0).reciprocal_().contiguous()       # [N]: 1 / mean_h(den_h)  (an [N]-vector; not a hot path)
        att = K.alloc_act(n, n, torch.float32, dev)
        K.gemm_nt([K.as_operand(q, prec.planes)], [K.as_operand(k, prec.planes)], [(0, 0, 0, 0, H * h)], n, att, alpha=1.0 / H,
                  alpha_dev=at["scal"][2:3], row_scale=inv_norm)
        out.append(att)
        a = K.head_mean(o, H, h) if H > 1 else o
        x, _ = K.ln_fwd(a, x if use_res else None, ca, cb, P.get(f"{pfx}bns.{i + 1}.weight"), P.get(f"{pfx}bns.{i + 1}.bias"), use_ln,
                        with_act and bool(cfg["trans_use_act"]), 0.0, 0, False)
    return out


def trans_backward(P, cfg: dict, tape: Tape, dout: Tensor, gscale: float, prec: Precision, grads: Dict[str, Tensor],
                   pfx: str = "trans_conv.", want_dx: bool = False, comm: Comm = SINGLE) -> Optional[Tensor]:
    h, H = cfg["hidden"], cfg["num_heads"]
    n, p, seed = tape["n"], tape["p"], tape["seed"]
    dev = dout.device
    use_ln = bool(cfg["trans_use_bn"])
    ca, cb, use_res = _res_coef(cfg)
    use_weight = bool(cfg["trans_use_weight"])

    dcur, gs = dout, gscale
    for i in reversed(range(cfg["trans_num_layers"])):
        L = tape["layers"][i]
        lp, bn = f"{pfx}convs.{i}.", f"{pfx}bns.{i + 1}."
        x_in, at = L["x_in"], L["attn"]
        dg, db = (torch.zeros(h, dtype=torch.float32, device=dev), torch.zeros(h, dtype=torch.float32, device=dev)) if use_ln \
            else (None, None)
        if L.get("gram"):
            gnum, gden, dr, cs, pg, sg = K.ln_bwd_attn(dcur, L["a"], x_in if use_res else None, x_in, ca, cb, P.get(bn + "weight"),
                                                       P.get(bn + "bias"), L["st"], use_ln, bool(cfg["trans_use_act"]), p,
                                                       seed + _SEED_LAYER + i, gs, use_res, dg, db, at["den"])
            dprev = dr if dr is not None else K.new_like(x_in)
            attention_gram_backward(P, lp, at, x_in, gnum, gden, cs, pg, sg, use_weight, prec, dprev, dr is not None, grads, comm)
        else:       # materialised q, k (and v with use_weight): several heads
            nout = L["nout"]
            da, dr = K.ln_bwd(dcur, L["a"], x_in if use_res else None, ca, cb, P.get(bn + "weight"), P.get(bn + "bias"), L["st"],
                              use_ln, bool(cfg["trans_use_act"]), p, seed + _SEED_LAYER + i, gs, use_res, dg, db)
            dqkv = torch.empty((n, K.ceil_to(nout, 8)), dtype=prec.act_dtype, device=dev)[:, :nout]
            dprev = dr if dr is not None else K.new_like(x_in)
            if use_weight:
                # head mean: every head receives da / H; da has pitch h, per-head slices of g are the same columns for all heads
                attention_backward(at, _tile_heads(da, H), 1.0 / H, prec, dqkv[:, :H * h], dqkv[:, H * h:2 * H * h],
                                   dqkv[:, 2 * H * h:], comm=comm)
            else:
                # shared value v = x_in: every head reads the same da / H, and the heads' dv sum into dprev in head order
                attention_backward(at, da, 1.0 / H, prec, dqkv[:, :H * h], dqkv[:, H * h:], dprev, dv_accumulate=dr is not None,
                                   comm=comm)
            wcat, _ = _qkv_weight(P, lp, use_weight)
            dqkv_op = K.as_operand(dqkv, prec.planes)
            K.gemm_nt([dqkv_op], [K.pack_operand(wcat, True, prec.planes)], [(0, 0, 0, 0, nout)], h, dprev,
                      accumulate=dr is not None or not use_weight)
            dw = torch.empty((nout, h), dtype=torch.float32, device=dev)
            K.gemm_tn(dqkv_op, K.as_operand(x_in, prec.planes, memo=True), dw)
            dbias, _ = K.colstats(dqkv, want_sumsq=False)
            for j, nm in enumerate(("Wq", "Wk", "Wv")[:nout // (H * h)]):
                grads[lp + nm + ".weight"] = dw[j * H * h:(j + 1) * H * h]
                grads[lp + nm + ".bias"] = dbias[j * H * h:(j + 1) * H * h]
        if use_ln:
            grads[bn + "weight"], grads[bn + "bias"] = dg, db
        dcur, gs = dprev, 1.0
    return _stem_backward(P, pfx, tape, dcur, gs, use_ln, prec, grads, want_dx)


def _tile_heads(da: Tensor, heads: int) -> Tensor:
    """[N, h] -> [N, H*h] with the same block repeated (gradient of the head mean, before the 1/H factor)."""
    n, h = da.shape
    out = K.alloc_act(n, heads * h, da.dtype, da.device)
    for hd in range(heads):
        K.axpby(da, None, 1.0, 0.0, out=out[:, hd * h:(hd + 1) * h])
    return out


# =================================================================================================
# GraphConv branch (large / 100M)
# =================================================================================================
def _stat_bufs(use_bn: bool, training: bool, h: int, dev):
    """Zeroed (sum, sumsq) buffers for a GEMM epilogue to fill when batch statistics are needed, else (None, None)."""
    if use_bn and training:
        return torch.zeros(h, dtype=torch.float32, device=dev), torch.zeros(h, dtype=torch.float32, device=dev)
    return None, None


def _bn_stats(z: Tensor, P, name: str, use_bn: bool, training: bool, zbias: Optional[Tensor] = None, comm: Comm = SINGLE,
              pre=None):
    if not use_bn:
        return None, None
    h = z.shape[1]
    if training:
        s, q = pre if (pre is not None and pre[0] is not None) else K.colstats(z)
        comm.allreduce_(s, q)                                              # C3: batch statistics span all shards
        rows = comm.n_global if comm.active else z.shape[0]
        mean, rstd = K.bn_finalize(s, q, rows, h, zbias, P.get(name + "running_mean"), P.get(name + "running_var"),
                                   z.device)
        nbt = P.get(name + "num_batches_tracked")
        if nbt is not None:
            nbt += 1
    else:
        mean, rstd = K.bn_finalize(None, None, z.shape[0], h, None, P[name + "running_mean"], P[name + "running_var"],
                                   z.device)
    return mean, rstd


def gconv_forward(P, cfg: dict, xin: K.Operand, graph: Graph, prec: Precision, training: bool, seed: int,
                  tape: Optional[Tape], mix: Optional[Tensor] = None, gw: float = 1.0, pfx: str = "graph_conv.",
                  comm: Comm = SINGLE) -> Tensor:
    """Returns GraphConv(x) — or, when `mix` is given, gw*GraphConv(x) + (1-gw)*mix (the SGFormer branch sum fused
    into the last layer's epilogue pass)."""
    h, d_in, nl = cfg["hidden"], cfg["in_channels"], cfg["gnn_num_layers"]
    check_width(h, prec, "hidden_channels")
    n = xin.rows
    dev = xin.data.device
    p = float(cfg["gnn_dropout"]) if training else 0.0
    use_bn, use_res, use_act = bool(cfg["gnn_use_bn"]), bool(cfg["gnn_use_residual"]), bool(cfg["gnn_use_act"])
    use_init, use_weight = bool(cfg["gnn_use_init"]), bool(cfg["gnn_use_weight"])
    dinv = graph.dinv
    st0 = _stat_bufs(use_bn, training, h, dev)
    z0 = K.gemm_nt([xin], [_w(P, pfx + "fcs.0.weight", prec)], [(0, 0, 0, 0, d_in)], h,
                   K.alloc_act(n, h, prec.act_dtype, dev), bias=P[pfx + "fcs.0.bias"], col_sum=st0[0], col_sumsq=st0[1])
    mean0, rstd0 = _bn_stats(z0, P, pfx + "bns.0.", use_bn, training, comm=comm, pre=st0)
    last_is_input = nl == 0
    # the pre-scaled SpMM operand is written where the halo exchange wants it (slot 0 of the step's symmetric buffer when pushed)
    x0, cur_s = K.bn_fwd(z0, None, mix if last_is_input else None, mean0, rstd0, P.get(pfx + "bns.0.weight"),
                         P.get(pfx + "bns.0.bias"), None, use_bn, True, p, seed + _SEED_GCONV_STEM, gw, dinv, True, not last_is_input,
                         ys_out=None if last_is_input else comm.operand_out(n, h, prec.act_dtype, dev))
    if tape is not None:
        tape.update(xin=xin, z0=z0, mean0=mean0, rstd0=rstd0, x0=x0, layers=[], p=p, seed=seed, n=n, training=training,
                    mixed=mix is not None, gw=gw)
    out = x0
    for i in range(nl):
        last = i == nl - 1
        y = comm.spmm_gathered(K, graph, False, dinv, cur_s)    # C4: operand rows of every shard
        st = _stat_bufs(use_bn, training, h, dev)      # BatchNorm sums come out of the GEMM epilogue
        if use_init:
            w, at = _b_blocks(P[f"{pfx}convs.{i}.W.weight"], [h, h], prec)
            z = K.gemm_nt([K.as_operand(y, prec.planes, memo=True), K.as_operand(x0, prec.planes, memo=True)], w,
                          [(0, 0, at[0][0], at[0][1], h), (1, 0, at[1][0], at[1][1], h)], h, K.new_like(y), bias=P[f"{pfx}convs.{i}.W.bias"],
                          col_sum=st[0], col_sumsq=st[1])
        elif use_weight:
            w = _w(P, f"{pfx}convs.{i}.W.weight", prec)
            z = K.gemm_nt([K.as_operand(y, prec.planes, memo=True)], [w], [(0, 0, 0, 0, h)], h, K.new_like(y),
                          bias=P[f"{pfx}convs.{i}.W.bias"], col_sum=st[0], col_sumsq=st[1])
        else:
            z, st = y, (None, None)
        name = f"{pfx}bns.{i + 1}."
        mean, rstd = _bn_stats(z, P, name, use_bn, training, comm=comm, pre=st)
        yo, ys = K.bn_fwd(z, x0 if use_res else None, mix if last else None, mean, rstd, P.get(name + "weight"),
                          P.get(name + "bias"), None, use_bn, use_act, p, seed + _SEED_GCONV_LAYER + i, gw, dinv, last, not last,
                          ys_out=None if last else comm.operand_out(n, h, prec.act_dtype, dev))
        if tape is not None:
            tape["layers"].append(dict(y=y, z=z, mean=mean, rstd=rstd))
        if last:
            out = yo
        else:
            cur_s = ys
    return out


def gconv_backward(P, cfg: dict, tape: Tape, graph: Graph, dout: Tensor, prec: Precision, grads: Dict[str, Tensor],
                   pfx: str = "graph_conv.", want_dx: bool = False, comm: Comm = SINGLE) -> Optional[Tensor]:
    """dout = gradient w.r.t. the tensor gconv_forward returned (the mixed tensor when `mix` was given: the factor gw
    is applied here; the caller routes (1-gw)*dout to the other branch)."""
    h, d_in, nl = cfg["hidden"], cfg["in_channels"], cfg["gnn_num_layers"]
    n, p, seed, training = tape["n"], tape["p"], tape["seed"], tape["training"]
    dev = dout.device
    use_bn, use_res, use_act = bool(cfg["gnn_use_bn"]), bool(cfg["gnn_use_residual"]), bool(cfg["gnn_use_act"])
    use_init, use_weight = bool(cfg["gnn_use_init"]), bool(cfg["gnn_use_weight"])
    dinv = graph.dinv
    x0 = tape["x0"]
    red = comm.allreduce_ if comm.active else None
    nstat = comm.n_global if comm.active else 0
    gs = tape["gw"] if tape["mixed"] else 1.0
    dx0 = None            # accumulated gradient of x0 (act dtype)
    dy_plain, dy_scaled = dout, None   # gradient entering the current layer's epilogue: plain, or pre-SpMM (needs *dinv)
    for i in reversed(range(nl)):
        L = tape["layers"][i]
        name = f"{pfx}bns.{i + 1}."
        if use_res and dx0 is None:
            dx0 = K.new_like(x0)
            res_acc = False
        else:
            res_acc = True
        dz, sums, colsum = K.bn_bwd(dy_plain, dy_scaled, dinv if dy_scaled is not None else None, L["z"], L["mean"],
                                    L["rstd"], P.get(name + "weight"), P.get(name + "bias"), None, use_bn, use_act, training,
                                    p, seed + _SEED_GCONV_LAYER + i, gs, dres=dx0 if use_res else None, dres_accumulate=res_acc,
                                    want_dz_colsum=use_init or use_weight, reduce_fn=red, stat_rows=nstat)
        if use_bn:
            _bn_param_grads(grads, comm, P, name, sums, dy_plain, dy_scaled, dinv, L["z"], L["mean"], L["rstd"], use_act, gs)
        gs = 1.0
        if use_init or use_weight:
            wname = f"{pfx}convs.{i}.W.weight"
            dz_op = K.as_operand(dz, prec.planes)
            kin = 2 * h if use_init else h
            dw = torch.empty((h, kin), dtype=torch.float32, device=dev)
            K.gemm_tn(dz_op, K.as_operand(L["y"], prec.planes, memo=True), dw[:, :h])
            if use_init:
                K.gemm_tn(dz_op, K.as_operand(x0, prec.planes, memo=True), dw[:, h:])
            grads[wname] = dw
            grads[f"{pfx}convs.{i}.W.bias"] = colsum
            wt = _w(P, wname, prec, transpose=True)   # [kin, h]
            dys = comm.operand_out(n, h, prec.act_dtype, dev)
            if dys is None or dys.stride(0) != dz.stride(0):
                dys = K.new_like(dz)
            K.gemm_nt([dz_op], [_slice_rows(wt, 0, h)], [(0, 0, 0, 0, h)], h, dys, row_scale=dinv)
            if use_init:
                if dx0 is None:
                    dx0 = K.new_like(x0)
                    K.gemm_nt([dz_op], [_slice_rows(wt, h, 2 * h)], [(0, 0, 0, 0, h)], h, dx0)
                else:
                    K.gemm_nt([dz_op], [_slice_rows(wt, h, 2 * h)], [(0, 0, 0, 0, h)], h, dx0, accumulate=True)
        else:
            dys = K.axpby(dz, None, 1.0, 0.0, row_scale=dinv, out=comm.operand_out(n, h, prec.act_dtype, dev))
        # = A^T (dinv . dy): gradient w.r.t. the pre-scaled SpMM input (C4: gradient rows of every shard)
        dy_scaled = comm.spmm_gathered(K, graph, True, None, dys)
        dy_plain = None
    # input layer epilogue: gradient of x0 = accumulated dx0 (+ dinv * dy_scaled from layer 0's SpMM)
    if nl == 0:
        g_plain, g_scaled = dout, None
    else:
        g_plain, g_scaled = dx0, dy_scaled
    dz0, sums, colsum = K.bn_bwd(g_plain, g_scaled, dinv if g_scaled is not None else None, tape["z0"], tape["mean0"],
                                 tape["rstd0"], P.get(pfx + "bns.0.weight"), P.get(pfx + "bns.0.bias"), None, use_bn, True,
                                 training, p, seed + _SEED_GCONV_STEM, gs, want_dz_colsum=True, reduce_fn=red, stat_rows=nstat)
    if use_bn:
        _bn_param_grads(grads, comm, P, pfx + "bns.0.", sums, g_plain, g_scaled, dinv, tape["z0"], tape["mean0"], tape["rstd0"], True,
                        gs)
    dz0_op = K.as_operand(dz0, prec.planes)
    dw0 = torch.empty((h, d_in), dtype=torch.float32, device=dev)
    K.gemm_tn(dz0_op, tape["xin"], dw0)
    grads[pfx + "fcs.0.weight"] = dw0
    grads[pfx + "fcs.0.bias"] = colsum
    if want_dx:
        dx = torch.empty((n, d_in), dtype=torch.float32, device=dev)
        K.gemm_nt([dz0_op], [_w(P, pfx + "fcs.0.weight", prec, transpose=True)], [(0, 0, 0, 0, h)], d_in, dx)
        return dx
    return None


def _mark_global(grads: dict, comm: Comm, *names: str):
    """Gradients that are already sums over all shards (excluded from the C5 all-reduce)."""
    if comm.active:
        grads.setdefault("__global__", set()).update(names)


def _bn_param_grads(grads: dict, comm: Comm, P, name: str, sums: Optional[Tensor], dy, dy2, dinv, z: Tensor, mean, rstd,
                    use_relu: bool, gscale: float = 1.0, zbias: Optional[Tensor] = None):
    """Stores the affine gradients of the BatchNorm `name`.  Training: `sums` = (sum g, sum g*xhat) from bn_bwd, which
    all-reduced them between its phases.  Eval (sums is None; rare: eval-mode backward): computed here from the running
    statistics and the gradient gscale * (dy, dy2) that entered bn_bwd; `zbias` = the bias bn_fwd added to z (GCN layers)."""
    if sums is None:
        sums = K.bn_bwd_sums(dy, dy2, dinv if dy2 is not None else None, z, mean, rstd, P[name + "weight"], P[name + "bias"], zbias,
                             True, use_relu, 0.0, 0, gscale)
    else:
        _mark_global(grads, comm, name + "bias", name + "weight")
    h = z.shape[1]
    grads[name + "bias"], grads[name + "weight"] = sums[:h], sums[h:]


def _slice_rows(op: K.Operand, r0: int, r1: int) -> K.Operand:
    return K.Operand(op.data[r0:r1], r1 - r0, op.k, op.kp, op.planes)


# =================================================================================================
# GCN backbone (medium): PyG GCNConv stack
# =================================================================================================
# Weighted graphs (edge_weight, DESIGN.md §4.10): `graph` is the weighted Graph; layers < L-1 run on it (its weighted dinv is their
# pre / post scale, the SpMMs read its values), the last one on the unweighted pattern (graph.pattern()), as models.GCN passes
# edge_weight to every conv but the last (medium/models.py:53-62).  The edge-weight gradient (P[EDGE_WEIGHT] requiring grad) is
# summed over the weighted layers by sgf_edge_weight_grad, which needs each layer's t = dinv (.) x W^T from the forward.
EDGE_WEIGHT = "edge_weight"


def _is_weighted(graph) -> bool:
    return getattr(graph, "val", None) is not None


def _layer_graph(graph: Graph, last: bool) -> Graph:
    return graph.pattern() if _is_weighted(graph) and last else graph


def _weighted_spmm(g: Graph, transposed: bool, row_scale: Tensor, x: Tensor) -> Tensor:
    if transposed:
        rp, cl = g.transpose()
        return K.spmm(rp, cl, row_scale, x, heavy=g.heavy_t, val=g.val_t)
    return K.spmm(g.rowptr, g.col, row_scale, x, heavy=g.heavy, val=g.val)


def _gcn_spmm(g: Graph, transposed: bool, dinv: Optional[Tensor], x: Tensor, comm: Comm) -> Tensor:
    """Â x (or Âᵀ x) of one GCN layer; dinv None: the unnormalised conv (cfg gcn_normalize False), a plain sum over the edges as
    given (sgf_spmm_sum)."""
    if dinv is None:
        rp, cl = g.transpose() if transposed else (g.rowptr, g.col)
        return K.spmm_sum(rp, cl, x, heavy=g.heavy_t if transposed else g.heavy)
    if _is_weighted(g):
        return _weighted_spmm(g, transposed, dinv, x)
    return comm.spmm_gathered(K, g, transposed, dinv, x)


def _want_edge_grad(P) -> bool:
    w = P.get(EDGE_WEIGHT)
    return w is not None and w.requires_grad


def gcn_forward(P, cfg: dict, xin: K.Operand, graph: Graph, prec: Precision, training: bool, seed: int,
                tape: Optional[Tape], mix: Optional[Tensor] = None, gw: float = 1.0, pfx: str = "gnn.",
                comm: Comm = SINGLE) -> Tensor:
    """models.GCN.forward (medium/models.py:49-63).  `graph` is built with PyG self-loop semantics (gcn_norm).  With
    cfg["gcn_normalize"] False it is gnns.GCN(save_mem=True).forward (large/gnns.py:212-220): every conv is
    GCNConv(normalize=False), a plain sum over the edges of `graph` as built (self-loop mode 0), with no degree scaling."""
    nl = cfg["gcn_num_layers"]
    norm = bool(cfg.get("gcn_normalize", True))
    n = xin.rows
    dev = xin.data.device
    p = float(cfg["gcn_dropout"]) if training else 0.0
    use_bn = bool(cfg["gcn_use_bn"])
    if _is_weighted(graph) and comm.active:
        raise NotImplementedError("sgformer_b200: row sharding of a weighted graph is not supported")
    if not norm and (comm.active or _is_weighted(graph)):
        raise NotImplementedError("sgformer_b200: the unnormalised GCN runs unsharded on an unweighted graph")
    keep_t = tape is not None and _is_weighted(graph) and _want_edge_grad(P)
    cur_op, cur_k = xin, cfg["in_channels"]
    layers = []
    out = None
    for i in range(nl):
        last = i == nl - 1
        g = _layer_graph(graph, last)
        dinv = g.dinv if norm else None
        wname = f"{pfx}convs.{i}.lin.weight"
        hout = P[wname].shape[0]
        check_width(hout, prec, f"GCN layer {i} out_channels")
        t = K.gemm_nt([cur_op], [_w(P, wname, prec)], [(0, 0, 0, 0, cur_k)], hout, K.alloc_act(n, hout, prec.act_dtype, dev),
                      row_scale=dinv)
        s = _gcn_spmm(g, False, dinv, t, comm)
        zb = P.get(f"{pfx}convs.{i}.bias")
        if last:
            out, _ = K.bn_fwd(s, None, mix, None, None, None, None, zb, False, False, 0.0, 0, gw, None, True, False)
            layers.append(dict(s=s, cur_op=cur_op, cur_k=cur_k, hout=hout))
        else:
            name = f"{pfx}bns.{i}."
            mean, rstd = _bn_stats(s, P, name, use_bn, training, zbias=zb, comm=comm)
            y, _ = K.bn_fwd(s, None, None, mean, rstd, P.get(name + "weight"), P.get(name + "bias"), zb, use_bn, True, p,
                            seed + _SEED_GCN_LAYER + i, 1.0, None, True, False)
            layers.append(dict(s=s, cur_op=cur_op, cur_k=cur_k, hout=hout, mean=mean, rstd=rstd, t=t if keep_t else None))
            cur_op, cur_k = K.as_operand(y, prec.planes), hout
    if tape is not None:
        tape.update(layers=layers, p=p, seed=seed, n=n, training=training, mixed=mix is not None, gw=gw)
    return out


def gcn_backward(P, cfg: dict, tape: Tape, graph: Graph, dout: Tensor, prec: Precision, grads: Dict[str, Tensor],
                 pfx: str = "gnn.", want_dx: bool = False, comm: Comm = SINGLE) -> Optional[Tensor]:
    nl = cfg["gcn_num_layers"]
    n, p, seed, training = tape["n"], tape["p"], tape["seed"], tape["training"]
    dev = dout.device
    use_bn = bool(cfg["gcn_use_bn"])
    red = comm.allreduce_ if comm.active else None
    nstat = comm.n_global if comm.active else 0
    gs = tape["gw"] if tape["mixed"] else 1.0
    dcur = dout
    dx = None
    dew = None
    if _is_weighted(graph) and _want_edge_grad(P):
        dew = torch.zeros(graph.edge_index.shape[1], dtype=torch.float32, device=dev)
        grads[EDGE_WEIGHT] = dew
    for i in reversed(range(nl)):
        L = tape["layers"][i]
        last = i == nl - 1
        g = _layer_graph(graph, last)
        dinv = g.dinv if cfg.get("gcn_normalize", True) else None
        zb = P.get(f"{pfx}convs.{i}.bias")
        hout = L["hout"]
        if last:
            dzs, _, colsum = K.bn_bwd(dcur, None, None, L["s"], None, None, None, None, zb, False, False, training, 0.0, 0, gs,
                                      want_dz_colsum=zb is not None, out_row_scale=dinv)
        else:
            name = f"{pfx}bns.{i}."
            dzs, sums, colsum = K.bn_bwd(dcur, None, None, L["s"], L.get("mean"), L.get("rstd"), P.get(name + "weight"),
                                         P.get(name + "bias"), zb, use_bn, True, training, p, seed + _SEED_GCN_LAYER + i, gs,
                                         want_dz_colsum=zb is not None, out_row_scale=dinv, reduce_fn=red, stat_rows=nstat)
            if use_bn:
                _bn_param_grads(grads, comm, P, name, sums, dcur, None, None, L["s"], L["mean"], L["rstd"], True, gs, zb)
        gs = 1.0
        if zb is not None:
            grads[f"{pfx}convs.{i}.bias"] = colsum
        u = _gcn_spmm(g, True, dinv, dzs, comm)        # = Â^T dz = gradient of (x W^T)
        if _is_weighted(g) and dew is not None:     # dL/dw of this layer: <dzs_c, t_r> + the degree term of row c
            K.edge_weight_grad(g.rowptr, g.col, g.eid, dzs, L["t"], dew, y=L["s"], u=u, dinv=dinv, edge_index=g.edge_index,
                               loops=True)
        u_op = K.as_operand(u, prec.planes)
        wname = f"{pfx}convs.{i}.lin.weight"
        dw = torch.empty((hout, L["cur_k"]), dtype=torch.float32, device=dev)
        K.gemm_tn(u_op, L["cur_op"], dw)
        grads[wname] = dw
        if i > 0:
            dcur = K.alloc_act(n, L["cur_k"], prec.act_dtype, dev)
            K.gemm_nt([u_op], [_w(P, wname, prec, transpose=True)], [(0, 0, 0, 0, hout)], L["cur_k"], dcur)
        elif want_dx:
            dx = torch.empty((n, L["cur_k"]), dtype=torch.float32, device=dev)
            K.gemm_nt([u_op], [_w(P, wname, prec, transpose=True)], [(0, 0, 0, 0, hout)], L["cur_k"], dx)
    return dx


# =================================================================================================
# GCNJK baseline (medium): GCNConv stack + jumping knowledge + final Linear
# =================================================================================================
# models.GCNJK (medium/models.py:157-205) is the GCN stack above with BatchNorm on every conv but the last, no edge weights, and
# xs = [a_0 .. a_{L-1}] (each hidden layer's activation BEFORE its dropout, and the last conv's output) aggregated by
# JumpingKnowledge: 'max' = element-wise max over the layers (gradient to the first maximal layer), 'cat' = concatenation; then
# final_project.  The aggregation rides in the layers' bn_fwd passes (sgf_bn_fwd_jk: running max + uint8 layer index, or the
# layer's column block of the concatenation) and its gradient in their bn_bwd passes (sgf_bn_bwd_*_jk: an addend of dy after the
# dropout mask); the last conv's bias pass is a bn_fwd without BN/ReLU and finalises the max in place.  DESIGN.md §4.12.
def _gcnjk_dims(P, pfx: str, nl: int, jk: str):
    h = P[f"{pfx}convs.0.lin.weight"].shape[0]
    kfp = P[f"{pfx}final_project.weight"].shape[1]
    if kfp != (h * nl if jk == "cat" else h):
        raise ValueError(f"sgformer_b200: GCNJK final_project takes {kfp} inputs, but JumpingKnowledge('{jk}') over {nl} layers of "
                         f"{h} channels gives {h * nl if jk == 'cat' else h}")
    return h, kfp


def gcnjk_forward(P, cfg: dict, xin: K.Operand, graph: Graph, prec: Precision, training: bool, seed: int,
                  tape: Optional[Tape], mix: Optional[Tensor] = None, gw: float = 1.0, pfx: str = "gnn.",
                  comm: Comm = SINGLE, out_dtype=torch.float32) -> Tensor:
    """models.GCNJK.forward -> final_project(JK(xs)) [N, out] in `out_dtype` (gw*that + (1-gw)*mix when `mix` is given).  `graph`:
    the GCN's self-loop mode 1 graph, unweighted (GCNJK passes no edge weight)."""
    if comm.active:
        raise NotImplementedError("sgformer_b200: row sharding of GCNJK is not supported")
    nl, jk = cfg["gcn_num_layers"], cfg["gcn_jk"]
    n = xin.rows
    dev = xin.data.device
    p = float(cfg["gcn_dropout"]) if training else 0.0
    h, kfp = _gcnjk_dims(P, pfx, nl, jk)
    check_width(h, prec, "GCNJK hidden_channels")
    if nl > 256:
        raise ValueError("sgformer_b200: GCNJK runs at most 256 layers (uint8 layer index)")
    dinv = graph.dinv
    idx = None
    if jk == "max":
        jbuf = K.alloc_act(n, h, prec.act_dtype, dev)
        idx = torch.empty((n, jbuf.stride(0)), dtype=torch.uint8, device=dev)
    else:
        jbuf = K.alloc_act(n, nl * h, prec.act_dtype, dev)
    cur_op, cur_k = xin, cfg["in_channels"]
    layers = []
    for i in range(nl):
        last = i == nl - 1
        t = K.gemm_nt([cur_op], [_w(P, f"{pfx}convs.{i}.lin.weight", prec)], [(0, 0, 0, 0, cur_k)], h,
                      K.alloc_act(n, h, prec.act_dtype, dev), row_scale=dinv)
        s = _gcn_spmm(graph, False, dinv, t, comm)
        zb = P[f"{pfx}convs.{i}.bias"]
        blk = jbuf if jk == "max" else jbuf[:, i * h:(i + 1) * h]
        L = dict(s=s, cur_op=cur_op, cur_k=cur_k)
        if last:
            K.bn_fwd_jk(s, None, None, None, None, zb, False, False, 0.0, 0, False, jk, blk, idx, i)
        else:
            name = f"{pfx}bns.{i}."
            mean, rstd = _bn_stats(s, P, name, True, training, zbias=zb)
            # 'cat' without dropout: the next conv reads the activation from its block of the concatenation
            want_y = jk == "max" or p > 0.0
            y = K.bn_fwd_jk(s, mean, rstd, P[name + "weight"], P[name + "bias"], zb, True, True, p, seed + _SEED_GCNJK_LAYER + i,
                            want_y, jk, blk, idx, i)
            L.update(mean=mean, rstd=rstd)
            cur_op, cur_k = K.as_operand(y if want_y else blk, prec.planes), h
        layers.append(L)
    jk_op = K.as_operand(jbuf, prec.planes)
    c = P[f"{pfx}final_project.weight"].shape[0]
    out = K.alloc_act(n, c, out_dtype, dev)
    K.gemm_nt([jk_op], [_w(P, f"{pfx}final_project.weight", prec)], [(0, 0, 0, 0, kfp)], c, out, bias=P[f"{pfx}final_project.bias"])
    if mix is not None:
        out = K.axpby(out, mix, gw, 1.0 - gw)
    if tape is not None:
        tape.update(layers=layers, jk_op=jk_op, idx=idx, h=h, kfp=kfp, p=p, seed=seed, n=n, training=training,
                    mixed=mix is not None, gw=gw)
    return out


def gcnjk_backward(P, cfg: dict, tape: Tape, graph: Graph, dout: Tensor, prec: Precision, grads: Dict[str, Tensor],
                   pfx: str = "gnn.", want_dx: bool = False, comm: Comm = SINGLE) -> Optional[Tensor]:
    nl, jk = cfg["gcn_num_layers"], cfg["gcn_jk"]
    n, p, seed, training, h, kfp = tape["n"], tape["p"], tape["seed"], tape["training"], tape["h"], tape["kfp"]
    dev = dout.device
    gs = tape["gw"] if tape["mixed"] else 1.0
    dinv = graph.dinv
    # final_project: d bias = column sums of g_out (taken while packing), dW = g_out^T JK, g_jk = g_out W
    if gs != 1.0 or dout.dtype != torch.float32 or dout.stride(-1) != 1:
        dout = K.axpby(dout, None, gs, 0.0, out_dtype=torch.float32)
    c = dout.shape[1]
    db = torch.zeros(c, dtype=torch.float32, device=dev)
    dl_op = K.pack_operand(dout, False, prec.planes, colsum=db)
    wname = f"{pfx}final_project.weight"
    dw = torch.empty((c, kfp), dtype=torch.float32, device=dev)
    K.gemm_tn(dl_op, tape["jk_op"], dw)
    grads[wname], grads[f"{pfx}final_project.bias"] = dw, db
    g_jk = K.alloc_act(n, kfp, prec.act_dtype, dev)
    K.gemm_nt([dl_op], [_w(P, wname, prec, transpose=True)], [(0, 0, 0, 0, c)], kfp, g_jk)
    idx = tape["idx"]
    dcur = None
    dx = None
    for i in reversed(range(nl)):
        L = tape["layers"][i]
        last = i == nl - 1
        zb = P[f"{pfx}convs.{i}.bias"]
        blk = g_jk if jk == "max" else g_jk[:, i * h:(i + 1) * h]
        if last:
            dzs, _, colsum = K.bn_bwd_jk(None, L["s"], None, None, None, None, zb, False, False, training, 0.0, 0, jk, blk, idx, i,
                                         want_dz_colsum=True, out_row_scale=dinv)
        else:
            name = f"{pfx}bns.{i}."
            dzs, sums, colsum = K.bn_bwd_jk(dcur, L["s"], L["mean"], L["rstd"], P[name + "weight"], P[name + "bias"], zb, True, True,
                                            training, p, seed + _SEED_GCNJK_LAYER + i, jk, blk, idx, i, want_dz_colsum=True,
                                            out_row_scale=dinv)
            grads[name + "bias"], grads[name + "weight"] = sums[:h], sums[h:]
        grads[f"{pfx}convs.{i}.bias"] = colsum
        u = _gcn_spmm(graph, True, dinv, dzs, comm)        # = Â^T dz = gradient of (x W^T)
        u_op = K.as_operand(u, prec.planes)
        wname = f"{pfx}convs.{i}.lin.weight"
        dw = torch.empty((h, L["cur_k"]), dtype=torch.float32, device=dev)
        K.gemm_tn(u_op, L["cur_op"], dw)
        grads[wname] = dw
        if i > 0:
            dcur = K.alloc_act(n, L["cur_k"], prec.act_dtype, dev)
            K.gemm_nt([u_op], [_w(P, wname, prec, transpose=True)], [(0, 0, 0, 0, h)], L["cur_k"], dcur)
        elif want_dx:
            dx = torch.empty((n, L["cur_k"]), dtype=torch.float32, device=dev)
            K.gemm_nt([u_op], [_w(P, wname, prec, transpose=True)], [(0, 0, 0, 0, h)], L["cur_k"], dx)
    return dx


# =================================================================================================
# GAT backbone (medium): PyG GATConv stack
# =================================================================================================
# Layer i:  xp = x W^T [N, H*C] (GEMM),  a_src / a_dst = per-head dots of xp with att_src / att_dst (sgf_gat_logits, one row pass:
# the logits come from the same rounded xp the aggregation gathers, in either precision),  z = edge softmax aggregation + bias
# (sgf_gat_fwd; concat for the hidden layers, head mean for the last), then BatchNorm?/ELU/dropout in one bn_fwd pass whose
# statistics come from one colstats pass.  Backward: bn_bwd (ELU code), sgf_gat_bwd (two gathers: forward CSR, then transposed
# CSR) -> dxp incl. the logits' share, d att_* by per-head weighted column sums, dW and dx by the GEMMs.
# Wide layers (DESIGN.md §4.9): one launch of the GAT kernels serves at most SGF_GAT_MAX_HEADS heads and 2 KB of a row (512 fp32 /
# 1024 bf16 values), and so does one launch of the BatchNorm / ELU / dropout row kernels.  The edge softmax is independent per head,
# so a wider layer runs as a schedule over head groups (gat_groups): each group runs the unchanged kernels on column views of xp,
# att_*, z and g.  Group k draws its attention and post-ELU dropout under the layer's seed + k * _GAT_GROUP_SEED, so heads of
# different groups get independent masks and group 0 (all of a layer that fits one launch) keeps the layer's seeds.
_GAT_GROUP_SEED = 0x632BE59BD9B4E019       # odd 64-bit constant
_M64 = (1 << 64) - 1


def _gat_group_seed(seed: int, k: int) -> int:
    return (seed + k * _GAT_GROUP_SEED) & _M64 if k else seed


def gat_groups(dtype: str, heads: int, c: int) -> Tuple[int, List[Tuple[int, int]]]:
    """-> (cp, [(first head, head count), ...]): how a GAT layer of `heads` heads of `c` channels runs in precision `dtype` ('fp32' /
    'bf16').  cp is c rounded up to whole 16-byte chunks (4 fp32 / 8 bf16 values), the width every head runs at.  Each head is in
    exactly one group; a group has at most SGF_GAT_MAX_HEADS heads and 2 KB of a row (group heads * cp <= 512 fp32 / 1024 bf16);
    the groups are as few as that allows, in head order, sizes differing by at most one (larger first).  A layer that fits one
    launch is one group.  ValueError when a single head is wider than one launch."""
    if dtype not in ("fp32", "bf16"):
        raise ValueError(f"unknown precision {dtype!r}")
    vn = 8 if dtype == "bf16" else 4
    row_max = 128 * vn
    if heads < 1 or c < 1:
        raise ValueError(f"heads={heads}, out_channels={c}: both must be at least 1")
    cp = (c + vn - 1) // vn * vn
    per = min(K.GAT_MAX_HEADS, row_max // cp)
    if per < 1:
        raise ValueError(f"heads={heads}, out_channels={c} is not supported in precision '{dtype}': one head must fit one launch of the "
                         f"GAT kernels, out_channels at most {row_max}"
                         + (" (set_precision('bf16') runs heads of up to 1024 channels)" if dtype == "fp32" and cp <= 1024 else ""))
    ng = -(-heads // per)
    q, r = divmod(heads, ng)
    groups, h0 = [], 0
    for k in range(ng):
        hg = q + (k < r)
        groups.append((h0, hg))
        h0 += hg
    return cp, groups


@dataclass
class _GatPlan:
    """One GAT layer: heads x c channels run at cp (gat_groups); mean: a head-mean (concat=False) layer."""
    heads: int
    c: int
    cp: int
    mean: bool
    groups: List[Tuple[int, int]]

    def cols(self, grp) -> slice:
        """Columns of head group grp in xp / z / g of a concatenating layer (xp of either)."""
        return slice(grp[0] * self.cp, (grp[0] + grp[1]) * self.cp)


def _gat_plan(prec: Precision, heads: int, c: int, mean: bool, i: int) -> _GatPlan:
    try:
        cp, groups = gat_groups(prec.name, heads, c)
    except ValueError as e:
        raise ValueError(f"sgformer_b200 GAT layer {i}: {e}") from None
    return _GatPlan(heads, c, cp, mean, groups)


def _gat_dims(P, pfx: str, i: int):
    att = P[f"{pfx}convs.{i}.att_src"]
    return int(att.shape[-2]), int(att.shape[-1])


def _pad_heads(t: Tensor, heads: int, c: int, cp: int, dim: int = 0, fill: float = 0.0) -> Tensor:
    """t whose axis `dim` is `heads` blocks of c -> blocks of cp: each block's c values, then `fill` (fp32).  t itself when cp == c."""
    if cp == c:
        return t
    t = t.detach().movedim(dim, 0)
    rest = tuple(t.shape[1:])
    out = torch.full((heads, cp) + rest, fill, dtype=torch.float32, device=t.device)
    out[:, :c] = t.reshape((heads, c) + rest)
    return out.reshape((heads * cp,) + rest).movedim(0, dim).contiguous()


def _unpad_heads(t: Tensor, heads: int, c: int, cp: int, dim: int = 0) -> Tensor:
    """Inverse of _pad_heads: the real c of every cp-wide block along `dim`."""
    if cp == c:
        return t
    t = t.movedim(dim, 0)
    rest = tuple(t.shape[1:])
    return t.reshape((heads, cp) + rest)[:, :c].reshape((heads * c,) + rest).movedim(0, dim).contiguous()


def _gat_layer(P, lp: str, heads: int, c: int, mean: bool, prec: Precision, i: int, prev: Optional[_GatPlan] = None):
    """-> (cp, weight [heads*cp, in], att_src [heads*cp], att_dst [heads*cp], bias [heads*cp | cp]) of layer i at its run widths.
    The kernels move rows in 16-byte chunks per head, so a head whose width is not a multiple of 4 (fp32) / 8 (bf16) runs
    zero-padded to cp: the padded channels have zero weights, attention entries and bias, so they change neither the logits nor
    the real channels and stay exactly 0 (through BatchNorm too, whose padded affine is zero).  `prev`: the previous layer, whose
    padded channels this layer's weight reads through zero columns (`in` = its heads * cp)."""
    cp = _gat_plan(prec, heads, c, mean, i).cp
    w = _pad_heads(P[lp + "lin_src.weight"], heads, c, cp)
    if prev is not None:
        w = _pad_heads(w, prev.heads, prev.c, prev.cp, dim=1)
    a_s = _pad_heads(P[lp + "att_src"].reshape(-1), heads, c, cp)
    a_d = _pad_heads(P[lp + "att_dst"].reshape(-1), heads, c, cp)
    return cp, w, a_s, a_d, _pad_heads(P[lp + "bias"], 1 if mean else heads, c, cp)


def _sl(t: Optional[Tensor], cols: slice) -> Optional[Tensor]:
    return None if t is None else t[cols]


def _gat_conv_fwd(graph: Graph, xp: Tensor, lay: _GatPlan, att_s: Tensor, att_d: Tensor, bias: Tensor, p: float, seed: int):
    """Edge softmax aggregation of one layer over its head groups -> (z [N, heads*cp] | head mean [N, cp], [(a_src, a_dst, lse)] per
    group).  A concatenating group writes its own column block of z.  A head-mean layer of several groups sums the groups' means
    weighted by group heads / heads in group order (sgf_axpby) and adds the bias once (sgf_bn_fwd's zbias): no float atomics."""
    H, cp = lay.heads, lay.cp
    if len(lay.groups) == 1:
        a_s, a_d = K.gat_logits(xp, H, cp, att_s, att_d)
        z, lse = K.gat_fwd(graph.rowptr, graph.col, xp, a_s, a_d, H, cp, lay.mean, bias, p, seed)
        return z, [(a_s, a_d, lse)]
    n = xp.shape[0]
    z = None if lay.mean else K.alloc_act(n, H * cp, xp.dtype, xp.device)
    parts, means = [], []
    for k, grp in enumerate(lay.groups):
        cols, hg = lay.cols(grp), grp[1]
        xg = xp[:, cols]
        a_s, a_d = K.gat_logits(xg, hg, cp, att_s[cols], att_d[cols])
        if lay.mean:
            zk, lse = K.gat_fwd(graph.rowptr, graph.col, xg, a_s, a_d, hg, cp, True, None, p, _gat_group_seed(seed, k))
            means.append((zk, hg / H))
        else:
            _, lse = K.gat_fwd(graph.rowptr, graph.col, xg, a_s, a_d, hg, cp, False, bias[cols], p, _gat_group_seed(seed, k),
                               out=z[:, cols])
        parts.append((a_s, a_d, lse))
    if lay.mean:
        acc = K.axpby(means[0][0], means[1][0], means[0][1], means[1][1])
        for zk, wk in means[2:]:
            acc = K.axpby(zk, acc, wk, 1.0)
        z, _ = K.bn_fwd(acc, None, None, None, None, None, None, bias, False, False, 0.0, 0, 1.0, None, True, False)
    return z, parts


def _gat_conv_bwd(graph: Graph, rp_t: Tensor, col_t: Tensor, L: dict, g: Tensor, p: float, seed: int):
    """Backward of _gat_conv_fwd for g = dL/dz -> (dxp [N, heads*cp], [(da_src, da_dst) fp32 [group heads, N]] per group).  Group k
    of a concatenating layer reads its column block of g; of a head-mean layer, g * group heads / heads.  Each group writes its
    column block of dxp."""
    lay, xp = L["lay"], L["xp"]
    att_s, att_d = L["att"]
    H, cp = lay.heads, lay.cp
    if len(lay.groups) == 1:
        a_s, a_d, lse = L["parts"][0]
        dxp, da_s, da_d = K.gat_bwd(graph.rowptr, graph.col, rp_t, col_t, xp, a_s, a_d, lse, g, att_s, att_d, H, cp, lay.mean, p,
                                    seed)
        das = [(da_s, da_d)]
    else:
        dxp = K.new_like(xp)
        das, scaled = [], {}
        for k, (grp, (a_s, a_d, lse)) in enumerate(zip(lay.groups, L["parts"])):
            cols, hg = lay.cols(grp), grp[1]
            if lay.mean:
                if hg not in scaled:
                    scaled[hg] = K.axpby(g, None, hg / H, 0.0)
                gk = scaled[hg]
            else:
                gk = g[:, cols]
            _, da_s, da_d = K.gat_bwd(graph.rowptr, graph.col, rp_t, col_t, xp[:, cols], a_s, a_d, lse, gk, att_s[cols], att_d[cols],
                                      hg, cp, lay.mean, p, _gat_group_seed(seed, k), dxp_out=dxp[:, cols])
            das.append((da_s, da_d))
    return dxp, das


def _gat_att_grads(xp: Tensor, lay: _GatPlan, das) -> Tuple[Tensor, Tensor]:
    """d att_src, d att_dst [heads, cp]: per head, the column sums of xp's head block weighted by the head's da_src / da_dst."""
    H, cp = lay.heads, lay.cp
    datt_s = torch.zeros((H, cp), dtype=torch.float32, device=xp.device)
    datt_d = torch.zeros((H, cp), dtype=torch.float32, device=xp.device)
    for (h0, hg), (da_s, da_d) in zip(lay.groups, das):
        for j in range(hg):
            xh = xp[:, (h0 + j) * cp:(h0 + j + 1) * cp]
            K.colstats(xh, w=da_s[j], want_sumsq=False, sum_out=datt_s[h0 + j])
            K.colstats(xh, w=da_d[j], want_sumsq=False, sum_out=datt_d[h0 + j])
    return datt_s, datt_d


def _gat_bn_stats(z: Tensor, P, name: str, use_bn: bool, training: bool, lay: _GatPlan):
    """_bn_stats over the padded z of a concatenating layer: the running buffers are padded for the call (mean 0, variance 1 in the
    padding) and their real columns written back."""
    if not use_bn or lay.cp == lay.c:
        return _bn_stats(z, P, name, use_bn, training)
    H, c, cp = lay.heads, lay.c, lay.cp
    rm, rv = P[name + "running_mean"], P[name + "running_var"]
    Pp = {name + "running_mean": _pad_heads(rm, H, c, cp), name + "running_var": _pad_heads(rv, H, c, cp, fill=1.0)}
    if P.get(name + "num_batches_tracked") is not None:
        Pp[name + "num_batches_tracked"] = P[name + "num_batches_tracked"]
    mean, rstd = _bn_stats(z, Pp, name, True, training)
    if training:
        rm.copy_(_unpad_heads(Pp[name + "running_mean"], H, c, cp))
        rv.copy_(_unpad_heads(Pp[name + "running_var"], H, c, cp))
    return mean, rstd


def gat_forward(P, cfg: dict, xin: K.Operand, graph: Graph, prec: Precision, training: bool, seed: int,
                tape: Optional[Tape], mix: Optional[Tensor] = None, gw: float = 1.0, pfx: str = "gnn.",
                comm: Comm = SINGLE, x_raw: Optional[Tensor] = None) -> Tensor:
    """models.GAT.forward (medium/models.py:145-155).  `graph`: self_loop_mode 1 (remove_self_loops + add_self_loops); x_raw: the
    fp32 node features xin was packed from (input dropout)."""
    if comm.active:
        raise NotImplementedError("sgformer_b200: row sharding of the GAT branch is not supported")
    nl = cfg["gcn_num_layers"]
    n = xin.rows
    dev = xin.data.device
    p = float(cfg["gcn_dropout"]) if training else 0.0
    use_bn = bool(cfg["gcn_use_bn"])
    cur_op = xin
    if p > 0.0:
        xr = x_raw if x_raw.dtype == torch.float32 and x_raw.stride(-1) == 1 else x_raw.float().contiguous()
        cur_op = K.pack_operand(K.dense_dropout(xr, p, seed + _SEED_GAT_INPUT), False, prec.planes)
    layers = []
    out = None
    prev = None
    for i in range(nl):
        last = i == nl - 1
        H, C = _gat_dims(P, pfx, i)
        lp = f"{pfx}convs.{i}."
        lay = _gat_plan(prec, H, C, last, i)
        cp, w, att_s, att_d, bias = _gat_layer(P, lp, H, C, last, prec, i, prev)
        xp = K.gemm_nt([cur_op], [K.pack_operand(w, False, prec.planes)], [(0, 0, 0, 0, cur_op.k)], H * cp,
                       K.alloc_act(n, H * cp, prec.act_dtype, dev))
        z, parts = _gat_conv_fwd(graph, xp, lay, att_s, att_d, bias, p, seed + _SEED_GAT_ATT + i)
        L = dict(cur_op=cur_op, xp=xp, parts=parts, lay=lay, w=w, att=(att_s, att_d), prev=prev)
        if last:
            if cp != C:
                z = z[:, :C]
            out = K.axpby(z, mix, gw, 1.0 - gw) if mix is not None else z
        else:
            # BatchNorm / ELU / dropout per head group: column blocks of at most 2 KB (the row kernels' width); the statistics
            # are per column, so the blocks share one colstats / bn_finalize over the whole z
            name = f"{pfx}bns.{i}."
            mean, rstd = _gat_bn_stats(z, P, name, use_bn, training, lay)
            bw, bb = P.get(name + "weight"), P.get(name + "bias")
            if use_bn:
                bw, bb = _pad_heads(bw, H, C, cp), _pad_heads(bb, H, C, cp)
            if len(lay.groups) == 1:
                y, _ = K.bn_fwd(z, None, None, mean, rstd, bw, bb, None, use_bn, K.ACT_ELU, p, seed + _SEED_GAT_ACT + i, 1.0, None,
                                True, False)
            else:
                y = K.new_like(z)
                for k, grp in enumerate(lay.groups):
                    cs = lay.cols(grp)
                    K.bn_fwd(z[:, cs], None, None, _sl(mean, cs), _sl(rstd, cs), _sl(bw, cs), _sl(bb, cs), None, use_bn, K.ACT_ELU,
                             p, _gat_group_seed(seed + _SEED_GAT_ACT + i, k), 1.0, None, True, False, y_out=y[:, cs])
            L.update(z=z, mean=mean, rstd=rstd, bn=(bw, bb))
            cur_op = K.as_operand(y, prec.planes)
        layers.append(L)
        prev = lay
    if tape is not None:
        tape.update(layers=layers, p=p, seed=seed, n=n, training=training, mixed=mix is not None, gw=gw)
    return out


def gat_backward(P, cfg: dict, tape: Tape, graph: Graph, dout: Tensor, prec: Precision, grads: Dict[str, Tensor],
                 pfx: str = "gnn.", want_dx: bool = False, comm: Comm = SINGLE) -> Optional[Tensor]:
    nl = cfg["gcn_num_layers"]
    n, p, seed, training = tape["n"], tape["p"], tape["seed"], tape["training"]
    dev = dout.device
    use_bn = bool(cfg["gcn_use_bn"])
    rp_t, col_t = graph.transpose()
    gs = tape["gw"] if tape["mixed"] else 1.0
    dcur = dout
    dx = None
    for i in reversed(range(nl)):
        L = tape["layers"][i]
        last = i == nl - 1
        lp = f"{pfx}convs.{i}."
        lay, prev = L["lay"], L["prev"]
        H, C, cp = lay.heads, lay.c, lay.cp
        db = None
        if last:
            g = K.axpby(dcur, None, gs, 0.0) if gs != 1.0 else dcur
            if cp != C:        # zero-padded heads (see _gat_layer): the gradient of the padding columns is zero
                gp = torch.zeros((n, cp), dtype=g.dtype, device=dev)
                K.axpby(g, None, 1.0, 0.0, out=gp[:, :C])
                g = gp
        else:
            # the bias gradient is the column sum of dz taken in fp32 inside bn_bwd: in bf16, summing the stored dz would add its
            # rounding to a sum that a training BatchNorm makes exactly zero.  One bn_bwd per head group (<= 2 KB of a row).
            name = f"{pfx}bns.{i}."
            bw, bb = L["bn"]
            one = len(lay.groups) == 1
            if one:
                g, s_k, db = K.bn_bwd(dcur, None, None, L["z"], L["mean"], L["rstd"], bw, bb, None, use_bn, K.ACT_ELU, training, p,
                                      seed + _SEED_GAT_ACT + i, 1.0, want_dz_colsum=True)
                sums = [s_k]
            else:
                g = K.new_like(L["z"])
                sums, dbs = [], []
                for k, grp in enumerate(lay.groups):
                    cs = lay.cols(grp)
                    _, s_k, db_k = K.bn_bwd(dcur[:, cs], None, None, L["z"][:, cs], _sl(L["mean"], cs), _sl(L["rstd"], cs),
                                            _sl(bw, cs), _sl(bb, cs), None, use_bn, K.ACT_ELU, training, p,
                                            _gat_group_seed(seed + _SEED_GAT_ACT + i, k), 1.0, want_dz_colsum=True, dz_out=g[:, cs])
                    sums.append(s_k)
                    dbs.append(db_k)
                db = torch.cat(dbs)
            if use_bn and training:
                if one and cp == C:
                    _bn_param_grads(grads, comm, P, name, sums[0], dcur, None, None, L["z"], L["mean"], L["rstd"], K.ACT_ELU)
                else:
                    halves = [s.view(2, -1) for s in sums]
                    grads[name + "bias"] = _unpad_heads(torch.cat([s[0] for s in halves]), H, C, cp)
                    grads[name + "weight"] = _unpad_heads(torch.cat([s[1] for s in halves]), H, C, cp)
        if db is None:
            db, _ = K.colstats(g, want_sumsq=False)
        grads[lp + "bias"] = _unpad_heads(db, 1 if last else H, C, cp)
        dxp, das = _gat_conv_bwd(graph, rp_t, col_t, L, g, p, seed + _SEED_GAT_ATT + i)
        datt_s, datt_d = _gat_att_grads(L["xp"], lay, das)
        grads[lp + "att_src"], grads[lp + "att_dst"] = datt_s[:, :C], datt_d[:, :C]
        dxp_op = K.as_operand(dxp, prec.planes)
        cur_op = L["cur_op"]
        dw = torch.empty((H * cp, cur_op.k), dtype=torch.float32, device=dev)
        K.gemm_tn(dxp_op, cur_op, dw)
        dw = _unpad_heads(dw, H, C, cp)
        grads[lp + "lin_src.weight"] = dw if prev is None else _unpad_heads(dw, prev.heads, prev.c, prev.cp, dim=1)
        wt = K.pack_operand(L["w"], True, prec.planes)
        if i > 0:
            dcur = K.alloc_act(n, cur_op.k, prec.act_dtype, dev)
            K.gemm_nt([dxp_op], [wt], [(0, 0, 0, 0, H * cp)], cur_op.k, dcur)
        elif want_dx:
            dx = torch.empty((n, cur_op.k), dtype=torch.float32, device=dev)
            K.gemm_nt([dxp_op], [wt], [(0, 0, 0, 0, H * cp)], cur_op.k, dx)
            if p > 0.0:
                dx = K.dense_dropout(dx, p, seed + _SEED_GAT_INPUT)
    return dx


# =================================================================================================
# head: fc over the mixed / concatenated branches
# =================================================================================================
def head_forward(P, cfg: dict, feats: List[Tensor], prec: Precision, tape: Optional[Tape], pfx: str = "fc.") -> Tensor:
    """feats = [m] ('add', branches already mixed) or [x1, x2] ('cat').  large/ours.py:269-275.  Logits are fp32.
    pfx: the Linear's parameter prefix (DIFFormer's output Linear is "fcs.1.")."""
    h, c = cfg["hidden"], cfg["out_channels"]
    n = feats[0].shape[0]
    w, at = _b_blocks(P[pfx + "weight"], [h] * len(feats), prec)
    ops = [K.as_operand(f, prec.planes) for f in feats]
    pairs = [(j, 0, at[j][0], at[j][1], h) for j in range(len(feats))]
    # pitch padded to a 16-byte multiple (c = 47 -> 48 floats): the GEMM epilogue can then use its TMA-store path
    out = K.alloc_act(n, c, torch.float32, feats[0].device)
    K.gemm_nt(ops, w, pairs, c, out, bias=P[pfx + "bias"])
    if tape is not None:
        tape.update(ops=ops, nfeat=len(feats))
    return out


def head_backward(P, cfg: dict, tape: Tape, dlogits: Tensor, prec: Precision, grads: Dict[str, Tensor],
                  pfx: str = "fc.") -> List[Tensor]:
    h, c = cfg["hidden"], cfg["out_channels"]
    n = dlogits.shape[0]
    dev = dlogits.device
    dlogits = dlogits.contiguous().float()
    db = torch.zeros(c, dtype=torch.float32, device=dev)
    dl_op = K.pack_operand(dlogits, False, prec.planes, colsum=db)
    nf = tape["nfeat"]
    dw = torch.empty((c, nf * h), dtype=torch.float32, device=dev)
    wt = _w(P, pfx + "weight", prec, transpose=True)   # [nf*h, c]
    outs = []
    for j in range(nf):
        K.gemm_tn(dl_op, tape["ops"][j], dw[:, j * h:(j + 1) * h])
        dj = K.alloc_act(n, h, prec.act_dtype, dev)
        K.gemm_nt([dl_op], [_slice_rows(wt, j * h, (j + 1) * h)], [(0, 0, 0, 0, c)], h, dj)
        outs.append(dj)
    grads[pfx + "weight"], grads[pfx + "bias"] = dw, db
    return outs


# =================================================================================================
# DIFFormer (medium/difformer.py, kernel='simple', one head)
# =================================================================================================
# Layer i:  o = Gram-form attention in value-sum mode (sgf_attn_gram_prepare_fwd_vsum),  y = Â v  with v = x Wv^T + bv
# (gcn_conv, medium/difformer.py:63-79: in-degree normalisation over the edge targets, no self loops = Graph(self_loop_mode=0)),
#   u = a*o + b*r + c*y,   x' = dropout(LN?(u))                                          (sgf_ln_fwd_graph)
# with a, c the branch weights times alpha and b = 1-alpha (use_residual, r = layer input).  use_source adds alpha * x0 to u:
# r = (1-alpha) x + alpha x0 (one extra row pass for layers after the first).  Backward: sgf_ln_bwd_attn_graph writes the attention
# prologue and dinv (.) (c du); the transposed SpMM of that is dv, which adds dv^T x to dWv, 1^T dv to dbv and dv Wv to dx (a third
# segment of the dx GEMM).
def _difformer_coefs(cfg: dict, i: int):
    """-> (a, b, c, s): u = a*o + b*r + c*y + s*x0 of layer i."""
    gw = float(cfg["graph_weight"])
    if not cfg["use_graph"]:
        ca, cy = 1.0, 0.0
    elif gw > 0:
        ca, cy = 1.0 - gw, gw
    else:
        ca, cy = 1.0, 1.0
    al = float(cfg["alpha"])
    ka, kb = (al, 1.0 - al) if cfg["use_residual"] else (1.0, 0.0)
    ks = ka if cfg["use_source"] else 0.0
    return ka * ca, kb, ka * cy, ks


def _difformer_v_scaled(P, lp: str, x: Tensor, use_weight: bool, prec: Precision, dinv: Tensor) -> Tensor:
    """dinv (.) v: the pre-scaled SpMM operand of the graph term (row-scale epilogue of the V projection)."""
    if not use_weight:
        return K.axpby(x, None, 1.0, 0.0, row_scale=dinv)
    h = x.shape[1]
    return K.gemm_nt([K.as_operand(x, prec.planes, memo=True)], [_w(P, lp + "Wv.weight", prec)], [(0, 0, 0, 0, h)],
                     P[lp + "Wv.weight"].shape[0], K.new_like(x), bias=P[lp + "Wv.bias"], row_scale=dinv)


def _difformer_residual(x: Tensor, x0: Tensor, i: int, b: float, s: float):
    """-> (r, b): the residual operand of layer i and its coefficient in u, with use_source's s*x0 folded in."""
    if s and i > 0:
        return K.axpby(x, x0, b, s), 1.0
    if s or b:
        return x, b + s          # layer 0: x0 is the layer input
    return None, b


def difformer_forward(P: Dict[str, Tensor], cfg: dict, xin: K.Operand, graph: Optional[Graph], prec: Precision, training: bool,
                      seed: int, tape: Optional[Tape]) -> Tensor:
    """DIFFormer.forward (medium/difformer.py:184-211) -> fp32 logits [N, out_channels]."""
    h, nl = cfg["hidden"], cfg["num_layers"]
    check_width(h, prec, "hidden_channels")
    p = float(cfg["dropout"]) if training else 0.0
    use_ln, use_weight, use_graph = bool(cfg["use_bn"]), bool(cfg["use_weight"]), bool(cfg["use_graph"])
    t0, x, st0 = _stem_forward(P, "", xin, h, use_ln, prec, p, seed + _SEED_STEM, tape is not None)
    x0 = x
    layers = []
    # weighted graph (gcn_conv's edge_weight): value = w dinv[c] dinv[r] with the unweighted dinv; dL/dw needs dinv (.) v
    keep_v = tape is not None and use_graph and _is_weighted(graph) and _want_edge_grad(P)
    for i in range(nl):
        lp = f"convs.{i}."
        a, b, c, s_ = _difformer_coefs(cfg, i)
        at = Tape() if tape is not None else None
        o = attention_gram_forward(P, lp, x, use_weight, prec, at, vsum=True)
        r, b = _difformer_residual(x, x0, i, b, s_)
        gamma, beta = P.get(f"bns.{i + 1}.weight"), P.get(f"bns.{i + 1}.bias")
        vs = None
        if use_graph:
            vs = _difformer_v_scaled(P, lp, x, use_weight, prec, graph.dinv)
            y = _weighted_spmm(graph, False, graph.dinv, vs) if _is_weighted(graph) else \
                K.spmm(graph.rowptr, graph.col, graph.dinv, vs, heavy=graph.heavy)
            xn, st = K.ln_fwd_graph(o, r, y, a, b, c, gamma, beta, use_ln, False, p, seed + _SEED_LAYER + i, tape is not None)
        else:
            xn, st = K.ln_fwd(o, r, a, b, gamma, beta, use_ln, False, p, seed + _SEED_LAYER + i, tape is not None)
        layers.append(dict(x_in=x, attn=at, o=o, r=r, y=y if use_graph else None, st=st, coef=(a, b, c),
                           vs=vs if keep_v else None))
        x = xn
    logits = head_forward(P, cfg, [x], prec, tape, "fcs.1.")
    if tape is not None:
        tape.update(xin=xin, t0=t0, st0=st0, layers=layers, p=p, seed=seed, n=xin.rows)
    return logits


def difformer_backward(P: Dict[str, Tensor], cfg: dict, tape: Tape, graph: Optional[Graph], dlogits: Tensor, prec: Precision,
                       grads: Dict[str, Tensor], want_dx: bool = False) -> Optional[Tensor]:
    h, nl = cfg["hidden"], cfg["num_layers"]
    p, seed = tape["p"], tape["seed"]
    dev = dlogits.device
    use_ln, use_weight, use_graph = bool(cfg["use_bn"]), bool(cfg["use_weight"]), bool(cfg["use_graph"])
    dcur = head_backward(P, cfg, tape, dlogits, prec, grads, "fcs.1.")[0]
    dx0 = None                     # use_source: gradient of x0 collected from layers 1..L-1
    dew = None
    if use_graph:
        rp_t, col_t = graph.transpose()
        if _is_weighted(graph) and _want_edge_grad(P):
            dew = torch.zeros(graph.edge_index.shape[1], dtype=torch.float32, device=dev)
            grads[EDGE_WEIGHT] = dew
    for i in reversed(range(nl)):
        L = tape["layers"][i]
        lp = f"convs.{i}."
        a, b, c = L["coef"]
        _, _, _, s_ = _difformer_coefs(cfg, i)
        x_in, at, r = L["x_in"], L["attn"], L["r"]
        gamma, beta = P.get(f"bns.{i + 1}.weight"), P.get(f"bns.{i + 1}.bias")
        dg, db = (torch.zeros(h, dtype=torch.float32, device=dev), torch.zeros(h, dtype=torch.float32, device=dev)) if use_ln \
            else (None, None)
        if use_graph:
            gnum, gden, dr, ys, cs, pg, sg = K.ln_bwd_attn_graph(dcur, L["o"], r, x_in, L["y"], a, b, c, gamma, beta, L["st"], use_ln, p,
                                                                 seed + _SEED_LAYER + i, 1.0, r is not None, dg, db, at["den"],
                                                                 graph.dinv)
        else:
            gnum, gden, dr, cs, pg, sg = K.ln_bwd_attn(dcur, L["o"], r, x_in, a, b, gamma, beta, L["st"], use_ln, False, p,
                                                       seed + _SEED_LAYER + i, 1.0, r is not None, dg, db, at["den"])
        if use_ln:
            grads[f"bns.{i + 1}.weight"], grads[f"bns.{i + 1}.bias"] = dg, db
        # gradient of the layer input from r
        kb = 1.0 - float(cfg["alpha"]) if cfg["use_residual"] else 0.0
        if s_ and i > 0:           # r = kb*x + s*x0, b = 1: dr = du
            dx0 = K.axpby(dr, dx0, s_, 1.0) if dx0 is not None else K.axpby(dr, None, s_, 0.0)
            dprev, acc = (K.axpby(dr, None, kb, 0.0), True) if kb else (K.new_like(x_in), False)
        elif r is not None:
            dprev, acc = dr, True
        else:
            dprev, acc = K.new_like(x_in), False
        # attention (value-sum Gram form) + graph term: dv = dinv (.) A^T (dinv (.) c du)
        dv = None
        if use_graph:
            dv = _weighted_spmm(graph, True, graph.dinv, ys) if _is_weighted(graph) else \
                K.spmm(rp_t, col_t, graph.dinv, ys, heavy=graph.heavy_t)
        if dew is not None:        # dL/dw = dinv_c dinv_r <c du_c, v_r> = <ys_c, vs_r>
            K.edge_weight_grad(graph.rowptr, graph.col, graph.eid, ys, L["vs"], dew)
        attention_gram_backward(P, lp, at, x_in, gnum, gden, cs, pg, sg, use_weight, prec, dprev, acc, grads, dv=dv)
        if i == 0 and dx0 is not None:
            dprev = K.axpby(dprev, dx0, 1.0, 1.0)
        dcur = dprev
    return _stem_backward(P, "", tape, dcur, 1.0, use_ln, prec, grads, want_dx)


def difformer_attentions(P: Dict[str, Tensor], cfg: dict, xin: K.Operand, prec: Precision) -> List[Tensor]:
    """DIFFormer.get_attentions (medium/difformer.py:213-228) for use_graph=False: per layer the [N, N] matrix
    q~ k~^T / (q~ . sum_l k~_l + N).  The N x N product is one tensor-core GEMM of q and k with alpha = 1/(||q|| ||k||) read from
    the device and 1/den as its row scale (trans_attentions); the layer stack runs the Gram form.  Inference only, O(N^2) memory
    like the reference: meant for small graphs."""
    h, nl = cfg["hidden"], cfg["num_layers"]
    check_width(h, prec, "hidden_channels")
    n = xin.rows
    dev = xin.data.device
    use_ln, use_weight = bool(cfg["use_bn"]), bool(cfg["use_weight"])
    _, x, _ = _stem_forward(P, "", xin, h, use_ln, prec)
    x0 = x
    out = []
    for i in range(nl):
        lp = f"convs.{i}."
        a, b, _, s_ = _difformer_coefs(cfg, i)
        at = Tape()
        o = attention_gram_forward(P, lp, x, use_weight, prec, at, vsum=True)
        qk, _, _ = _project_qkv(P, lp, K.as_operand(x, prec.planes), False, prec, stats=False)
        inv_den = at["den"].reciprocal()        # [N]: the Gram denominator is the reference's normaliser / N
        att = K.alloc_act(n, n, torch.float32, dev)
        K.gemm_nt([K.as_operand(qk[:, :h], prec.planes)], [K.as_operand(qk[:, h:], prec.planes)], [(0, 0, 0, 0, h)], n, att,
                  alpha=1.0 / at["n"], alpha_dev=at["st"].sc[K.SC_ALPHA:K.SC_ALPHA + 1], row_scale=inv_den)
        out.append(att)
        r, b = _difformer_residual(x, x0, i, b, s_)
        x, _ = K.ln_fwd(o, r, a, b, P.get(f"bns.{i + 1}.weight"), P.get(f"bns.{i + 1}.bias"), use_ln, False, 0.0, 0, False)
    return out
