"""torch.autograd boundary: one Function per public op, each running a hand-scheduled forward/backward of engine.py.

`SGFormerFn` is the fused encoder (both branches + mix + fc in one schedule; what SGFormer.forward calls);
the others back the standalone modules/functions of the reference surface (TransConv, GraphConv, GCN,
full_attention_conv, GraphConvLayer's SpMM, nn.Linear on the tensor-core GEMM)."""
from __future__ import annotations

import functools
import threading
from typing import Dict, Optional, Sequence

import torch
from torch.autograd import Function

from . import engine as E
from . import kernels as K
from .dist import SINGLE, Comm
from .graph import Graph

Tensor = torch.Tensor

_outer = threading.local()


def _want_tape(ctx) -> bool:
    """Whether the forward must record its tape: some input requires grad AND the caller is not under torch.no_grad()
    (`needs_input_grad` ignores the grad mode, and inside Function.forward grad mode is always off: the caller's mode is sampled
    by `_TapeFunction.apply`).  Eval forwards (evaluate() is @torch.no_grad, large/eval.py) then keep no activations alive."""
    return getattr(_outer, "grad_enabled", True) and any(ctx.needs_input_grad)


class _TapeFunction(Function):
    @classmethod
    def apply(cls, *args, **kwargs):
        prev = getattr(_outer, "grad_enabled", True)
        _outer.grad_enabled = torch.is_grad_enabled()
        try:
            return super().apply(*args, **kwargs)
        finally:
            _outer.grad_enabled = prev


def _pdict(names: Sequence[str], tensors: Sequence[Tensor]) -> Dict[str, Tensor]:
    return {n: t for n, t in zip(names, tensors)}


def _grad_list(names, params, grads: Dict[str, Tensor]):
    out = []
    for n, p in zip(names, params):
        g = grads.get(n)
        if g is None or not p.requires_grad:
            out.append(None)
        else:
            if g.shape != p.shape:
                g = g.reshape(p.shape)
            out.append(g if g.dtype == p.dtype else g.to(p.dtype))
    return out


def _to_act(t: Tensor, prec: E.Precision) -> Tensor:
    """fp32/bf16 2-D tensor -> activation of the precision's dtype (cast kernel when needed)."""
    if t.dtype == prec.act_dtype and t.stride(-1) == 1 and t.stride(0) % (8 if t.dtype == torch.bfloat16 else 4) == 0 \
            and t.data_ptr() % 16 == 0:
        return t
    if t.dtype not in (torch.float32, torch.bfloat16):
        t = t.float()
    if t.stride(-1) != 1:
        t = t.contiguous()
    return K.axpby(t, None, 1.0, 0.0, out_dtype=prec.act_dtype)


def _from_act(t: Tensor, dtype) -> Tensor:
    if t.dtype == dtype and t.is_contiguous():
        return t
    out = torch.empty(t.shape, dtype=dtype, device=t.device)
    if dtype in (torch.float32, torch.bfloat16):
        K.axpby(t, None, 1.0, 0.0, out=out)
        return out
    return t.to(dtype)


_MEDIUM_GNN_BACKWARD = {"gcn": E.gcn_backward, "gat": E.gat_backward, "gcnjk": E.gcnjk_backward}


class SGFormerFn(_TapeFunction):
    """Fused encoder: logits = fc(mix(TransConv(x), GNN(x, graph))).  Returns fp32 [N, c]."""

    @staticmethod
    def forward(ctx, x: Tensor, graph: Optional[Graph], cfg: dict, prec: E.Precision, training: bool, comm: Comm, names,
                *params):
        """x: the rows this rank owns ([N, d_in], or its [N/P, d_in] block when `comm` is a row-sharding Comm)."""
        P = _pdict(names, params)
        need_tape = _want_tape(ctx)
        K.operand_memo_begin()       # fp32 activations shared by several GEMMs of this step are packed once
        xin = E.input_operand(x, prec)
        seed = E.next_seed()
        if comm.active:     # row shards hash local row ids: decorrelate the shards' dropout masks
            comm.begin_step()
            seed = (seed + comm.rank * 0x9E3779B97F4A7C15) & 0x7FFFFFFFFFFFFFFF
        tt, tg, th = (E.Tape(), E.Tape(), E.Tape()) if need_tape else (None, None, None)
        x1 = E.trans_forward(P, cfg, xin, prec, training, seed, tt, comm=comm)
        gw = float(cfg["graph_weight"])
        if cfg["use_graph"]:
            add = cfg["aggregate"] == "add"
            if cfg["variant"] != "medium":
                fwd = E.gconv_forward
            elif cfg["gnn_kind"] == "gat":
                fwd = functools.partial(E.gat_forward, x_raw=x)
            elif cfg["gnn_kind"] == "gcnjk":
                fwd = functools.partial(E.gcnjk_forward, out_dtype=prec.act_dtype)
            else:
                fwd = E.gcn_forward
            x2 = fwd(P, cfg, xin, graph, prec, training, seed, tg, mix=x1 if add else None, gw=gw, comm=comm)
            feats = [x2] if add else [x1, x2]
        else:
            feats = [x1]
        logits = E.head_forward(P, cfg, feats, prec, th)
        if need_tape:
            ctx.state = (cfg, prec, graph, comm, names, params, tt, tg, th, x.requires_grad)
        else:
            K.operand_memo_clear()
        return logits

    @staticmethod
    def backward(ctx, dlogits: Tensor):
        cfg, prec, graph, comm, names, params, tt, tg, th, want_dx = ctx.state
        P = _pdict(names, params)
        grads: Dict[str, Tensor] = {}
        dfeats = E.head_backward(P, cfg, th, dlogits, prec, grads)
        gw = float(cfg["graph_weight"])
        dx = None
        if cfg["use_graph"]:
            bwd = E.gconv_backward if cfg["variant"] != "medium" else _MEDIUM_GNN_BACKWARD[cfg["gnn_kind"]]
            if cfg["aggregate"] == "add":
                dm = dfeats[0]
                dxg = bwd(P, cfg, tg, graph, dm, prec, grads, want_dx=want_dx, comm=comm)
                dxt = E.trans_backward(P, cfg, tt, dm, 1.0 - gw, prec, grads, want_dx=want_dx, comm=comm)
            else:
                dxg = bwd(P, cfg, tg, graph, dfeats[1], prec, grads, want_dx=want_dx, comm=comm)
                dxt = E.trans_backward(P, cfg, tt, dfeats[0], 1.0, prec, grads, want_dx=want_dx, comm=comm)
            if want_dx:
                dx = K.axpby(dxt, dxg, 1.0, 1.0)
        else:
            dx = E.trans_backward(P, cfg, tt, dfeats[0], 1.0, prec, grads, want_dx=want_dx, comm=comm)
        if comm.active:
            # C5: every parameter gradient is a sum over rows -> one flattened all-reduce over the shards
            done = grads.get("__global__", ())
            comm.allreduce_(*[grads[n_] for n_ in names if n_ in grads and n_ not in done])
        ctx.state = None
        K.operand_memo_clear()
        return (dx, None, None, None, None, None, None, *_grad_list(names, params, grads))


class DIFFormerFn(_TapeFunction):
    """DIFFormer (medium/difformer.py:147-211, kernel='simple', one head): input MLP, Gram-form attention layers with the graph
    term, output Linear in one schedule (engine.difformer_forward / _backward).  Returns fp32 logits [N, c]."""

    @staticmethod
    def forward(ctx, x: Tensor, graph: Optional[Graph], cfg: dict, prec: E.Precision, training: bool, names, *params):
        P = _pdict(names, params)
        need_tape = _want_tape(ctx)
        K.operand_memo_begin()
        tape = E.Tape() if need_tape else None
        logits = E.difformer_forward(P, cfg, E.input_operand(x, prec), graph, prec, training, E.next_seed(), tape)
        if need_tape:
            ctx.state = (cfg, prec, graph, names, params, tape, x.requires_grad)
        else:
            K.operand_memo_clear()
        return logits

    @staticmethod
    def backward(ctx, dlogits: Tensor):
        cfg, prec, graph, names, params, tape, want_dx = ctx.state
        grads: Dict[str, Tensor] = {}
        dx = E.difformer_backward(_pdict(names, params), cfg, tape, graph, dlogits, prec, grads, want_dx=want_dx)
        ctx.state = None
        K.operand_memo_clear()
        return (dx, None, None, None, None, None, *_grad_list(names, params, grads))


class TransConvFn(_TapeFunction):
    """Standalone TransConv branch.  Returns [N, h] in x's dtype."""

    @staticmethod
    def forward(ctx, x, cfg, prec, training, names, *params):
        P = _pdict(names, params)
        need_tape = _want_tape(ctx)
        tape = E.Tape() if need_tape else None
        out = E.trans_forward(P, cfg, E.input_operand(x, prec), prec, training, E.next_seed(), tape)
        if need_tape:
            ctx.state = (cfg, prec, names, params, tape, x.requires_grad)
        return _from_act(out, x.dtype if x.dtype.is_floating_point else torch.float32)

    @staticmethod
    def backward(ctx, dout):
        cfg, prec, names, params, tape, want_dx = ctx.state
        grads: Dict[str, Tensor] = {}
        dx = E.trans_backward(_pdict(names, params), cfg, tape, _to_act(dout, prec), 1.0, prec, grads, want_dx=want_dx)
        ctx.state = None
        return (dx, None, None, None, None, *_grad_list(names, params, grads))


class GraphBranchFn(_TapeFunction):
    """Standalone GNN branch: GraphConv (large/100M), the PyG-GCN or the PyG-GAT backbone, or the GCNJK baseline (medium).
    Returns [N, h] in x's dtype."""

    @staticmethod
    def forward(ctx, x, graph, cfg, prec, training, kind, pfx, names, *params):
        P = _pdict(names, params)
        need_tape = _want_tape(ctx)
        tape = E.Tape() if need_tape else None
        if kind == "gat":
            fwd = functools.partial(E.gat_forward, x_raw=x)
        else:
            fwd = {"gcn": E.gcn_forward, "gcnjk": E.gcnjk_forward}.get(kind, E.gconv_forward)
        out = fwd(P, cfg, E.input_operand(x, prec), graph, prec, training, E.next_seed(), tape, pfx=pfx)
        if need_tape:
            ctx.state = (cfg, prec, graph, kind, pfx, names, params, tape, x.requires_grad)
        return _from_act(out, x.dtype if x.dtype.is_floating_point else torch.float32)

    @staticmethod
    def backward(ctx, dout):
        cfg, prec, graph, kind, pfx, names, params, tape, want_dx = ctx.state
        grads: Dict[str, Tensor] = {}
        bwd = {"gat": E.gat_backward, "gcn": E.gcn_backward, "gcnjk": E.gcnjk_backward}.get(kind, E.gconv_backward)
        # GCNJK returns fp32 logits and takes their gradient as it comes
        g = dout if kind == "gcnjk" else _to_act(dout, prec)
        dx = bwd(_pdict(names, params), cfg, tape, graph, g, prec, grads, pfx=pfx, want_dx=want_dx)
        ctx.state = None
        return (dx, None, None, None, None, None, None, None, *_grad_list(names, params, grads))


class HeadFn(Function):
    """fc over externally produced branch outputs (used when the GNN branch is a foreign nn.Module)."""

    @staticmethod
    def forward(ctx, x1, x2, cfg, prec, names, *params):
        P = _pdict(names, params)
        a1 = _to_act(x1, prec)
        gw = float(cfg["graph_weight"])
        if x2 is None:
            feats = [a1]
        else:
            a2 = _to_act(x2, prec)
            feats = [K.axpby(a2, a1, gw, 1.0 - gw)] if cfg["aggregate"] == "add" else [a1, a2]
        tape = E.Tape()
        out = E.head_forward(P, cfg, feats, prec, tape)
        ctx.state = (cfg, prec, names, params, tape, x1.dtype, None if x2 is None else x2.dtype)
        return out

    @staticmethod
    def backward(ctx, dlogits):
        cfg, prec, names, params, tape, dt1, dt2 = ctx.state
        grads: Dict[str, Tensor] = {}
        d = E.head_backward(_pdict(names, params), cfg, tape, dlogits, prec, grads)
        gw = float(cfg["graph_weight"])
        if dt2 is None:
            d1, d2 = _from_act(d[0], dt1), None
        elif cfg["aggregate"] == "add":
            d1 = K.axpby(d[0], None, 1.0 - gw, 0.0, out_dtype=dt1)
            d2 = K.axpby(d[0], None, gw, 0.0, out_dtype=dt2)
        else:
            d1, d2 = _from_act(d[0], dt1), _from_act(d[1], dt2)
        ctx.state = None
        return (d1, d2, None, None, None, *_grad_list(names, params, grads))


class SoftmaxAttentionFn(_TapeFunction):
    """softmax_attention(qs, ks, vs) -> [N, H, D]  (medium/ablation/oursSOFT.py:14-34).  A one-head vs [N, 1, D] is shared by all
    H heads, as the reference's einsum broadcasts it; its gradient is the sum over the heads."""

    @staticmethod
    def forward(ctx, q, k, v, prec, want_attn):
        n, heads, m = q.shape
        vh, d = v.shape[1], v.shape[2]
        if k.shape != q.shape or v.shape[0] != n or vh not in (1, heads):
            raise ValueError(f"softmax_attention: qs {tuple(q.shape)}, ks {tuple(k.shape)}, vs {tuple(v.shape)}: ks must match qs "
                             f"and vs must have {n} rows and 1 or {heads} heads")
        want = _want_tape(ctx)
        qa, ka, va = (_to_act(t.reshape(n, -1), prec) for t in (q, k, v))
        tape = E.Tape()
        # the backward passes each head its own gradient block: refuse here a shape whose backward could not run
        o = E.attention_softmax_forward(qa, ka, va, heads, prec, tape, shared_v=vh != heads, shared_g=False if want else None)
        att = K.attn_softmax_probs(qa, ka, heads, tape["sq_q"], tape["sq_k"]) if want_attn else None
        ctx.state = (tape, q.dtype, k.dtype, v.dtype, heads, vh, m, d, prec) if want else None
        out = _from_act(o, q.dtype).reshape(n, heads, d)
        if att is not None:
            ctx.mark_non_differentiable(att)
            return out, att
        return out

    @staticmethod
    def backward(ctx, g, *_):
        tape, dtq, dtk, dtv, heads, vh, m, d, prec = ctx.state
        n = g.shape[0]
        ga = _to_act(g.reshape(n, heads * d), prec)
        dq = K.alloc_act(n, heads * m, prec.act_dtype, g.device)
        dk = K.alloc_act(n, heads * m, prec.act_dtype, g.device)
        dv = K.alloc_act(n, vh * d, prec.act_dtype, g.device)
        E.attention_softmax_backward(tape, ga, 1.0, dq, dk, dv)
        ctx.state = None
        return (_from_act(dq, dtq).reshape(n, heads, m), _from_act(dk, dtk).reshape(n, heads, m),
                _from_act(dv, dtv).reshape(n, vh, d), None, None)


class ScaledAttentionFn(_TapeFunction):
    """GATAttention's scaled dot-product attention (medium/ablation/oursGAT.py:36-43) on q, k in the kernels' layout: q, k
    [N, H*mp], each head's dk columns followed by mp - dk zero columns (zero columns add nothing to q.k), v [N, H*D] ->
    [N, H, D], the softmax over the heads of q.k / sqrt(dk)."""

    @staticmethod
    def forward(ctx, q, k, v, heads, dk, prec):
        n = q.shape[0]
        mp, d = q.shape[1] // heads, v.shape[1] // heads
        if k.shape != q.shape or v.shape[0] != n or mp != E.gat_attn_pad(dk, prec):
            raise ValueError(f"GATAttention: q {tuple(q.shape)}, k {tuple(k.shape)}, v {tuple(v.shape)} do not hold {heads} heads of "
                             f"key width {dk} padded to {E.gat_attn_pad(dk, prec)}")
        E.check_attn_softmax(f"GAT attention with {heads} heads of key width {dk} and value width {d}", heads, mp, d, prec, False,
                             False if _want_tape(ctx) else None)
        qa, ka, va = (_to_act(t, prec) for t in (q, k, v))
        scale = E.gat_attn_scale(dk)
        o = K.attn_scaled_fwd(qa, ka, va, heads, scale)
        ctx.state = (qa, ka, va, scale, q.dtype, k.dtype, v.dtype, heads, prec) if _want_tape(ctx) else None
        return _from_act(o, q.dtype).reshape(n, heads, d)

    @staticmethod
    def backward(ctx, g):
        qa, ka, va, scale, dtq, dtk, dtv, heads, prec = ctx.state
        n, _, d = g.shape
        ga = _to_act(g.reshape(n, heads * d), prec)
        dq, dk = (K.alloc_act(n, qa.shape[1], prec.act_dtype, g.device) for _ in range(2))
        dv = K.alloc_act(n, heads * d, prec.act_dtype, g.device)
        K.attn_scaled_bwd(qa, ka, va, heads, scale, ga, 1.0, dq, dk, dv)
        ctx.state = None
        return _from_act(dq, dtq), _from_act(dk, dtk), _from_act(dv, dtv), None, None, None


class AttentionFn(_TapeFunction):
    """full_attention_conv(qs, ks, vs) -> [N, H, D]  (medium/ours.py:14-34, 100M/ours.py:12-43).  A one-head vs [N, 1, D]
    is shared by all H heads, as the reference's einsum broadcasts it; its gradient is the sum over the heads."""

    @staticmethod
    def forward(ctx, q, k, v, prec):
        n, heads, m = q.shape
        vh, d = v.shape[1], v.shape[2]
        if k.shape != q.shape or v.shape[0] != n or vh not in (1, heads):
            raise ValueError(f"full_attention_conv: qs {tuple(q.shape)}, ks {tuple(k.shape)}, vs {tuple(v.shape)}: ks must match qs "
                             f"and vs must have {n} rows and 1 or {heads} heads")
        qa, ka, va = (_to_act(t.reshape(n, -1), prec) for t in (q, k, v))
        need = _want_tape(ctx)
        tape = E.Tape() if need else None
        o = E.attention_forward(qa, ka, va, heads, prec, tape, shared_v=vh != heads)
        if need:
            ctx.state = (prec, tape, q.dtype, k.dtype, v.dtype, heads, vh, m, d)
        return _from_act(o, q.dtype).reshape(n, heads, d)

    @staticmethod
    def backward(ctx, g):
        prec, tape, dtq, dtk, dtv, heads, vh, m, d = ctx.state
        n = g.shape[0]
        ga = _to_act(g.reshape(n, heads * d), prec)
        dq = K.alloc_act(n, heads * m, prec.act_dtype, g.device)
        dk = K.alloc_act(n, heads * m, prec.act_dtype, g.device)
        dv = K.alloc_act(n, vh * d, prec.act_dtype, g.device)
        E.attention_backward(tape, ga, 1.0, prec, dq, dk, dv)
        ctx.state = None
        return (_from_act(dq, dtq).reshape(n, heads, m), _from_act(dk, dtk).reshape(n, heads, m),
                _from_act(dv, dtv).reshape(n, vh, d), None)


class LinearFn(Function):
    """y = x W^T + b on the wgmma GEMMs (nn.Linear forward / backward)."""

    @staticmethod
    def forward(ctx, x, w, b, prec):
        xa = _to_act(x, prec)
        xop = K.as_operand(xa, prec.planes)
        out = K.alloc_act(x.shape[0], w.shape[0], prec.act_dtype, x.device)
        K.gemm_nt([xop], [K.pack_operand(w, False, prec.planes)], [(0, 0, 0, 0, w.shape[1])], w.shape[0], out, bias=b)
        ctx.state = (prec, xop, w, b is not None, x.dtype)
        return _from_act(out, x.dtype)

    @staticmethod
    def backward(ctx, dy):
        prec, xop, w, has_b, dtx = ctx.state
        dya = _to_act(dy, prec)
        dop = K.as_operand(dya, prec.planes)
        dx = K.alloc_act(dy.shape[0], w.shape[1], prec.act_dtype, dy.device)
        K.gemm_nt([dop], [K.pack_operand(w, True, prec.planes)], [(0, 0, 0, 0, w.shape[0])], w.shape[1], dx)
        dw = torch.empty(w.shape, dtype=torch.float32, device=dy.device)
        K.gemm_tn(dop, xop, dw)
        db = K.colstats(dya, want_sumsq=False)[0] if has_b else None
        ctx.state = None
        return _from_act(dx, dtx), dw, db, None


class SpMMFn(Function):
    """y = Â x with Â = D^-1/2 A D^-1/2 of `graph` (GraphConvLayer.forward's matmul(adj, x), large/ours.py:26-34)."""

    @staticmethod
    def forward(ctx, x, graph: Graph, prec):
        xs = K.axpby(_to_act(x, prec), None, 1.0, 0.0, row_scale=graph.dinv)
        y = K.spmm(graph.rowptr, graph.col, graph.dinv, xs, heavy=graph.heavy)
        ctx.state = (graph, prec, x.dtype)
        return _from_act(y, x.dtype)

    @staticmethod
    def backward(ctx, dy):
        graph, prec, dtx = ctx.state
        rp, cl = graph.transpose()
        ds = K.axpby(_to_act(dy, prec), None, 1.0, 0.0, row_scale=graph.dinv)
        dx = K.spmm(rp, cl, graph.dinv, ds, heavy=graph.heavy_t)
        ctx.state = None
        return _from_act(dx, dtx), None, None


class SoftmaxNLLFn(Function):
    """mean NLL of log_softmax(logits) over the selected rows; the logits gradient is produced by the same pass."""

    @staticmethod
    def forward(ctx, logits, labels, mask, denom):
        loss, d = K.softmax_nll(logits, labels, mask, 1.0 / float(denom), want_grad=ctx.needs_input_grad[0])
        ctx.d = d
        return loss.reshape(())

    @staticmethod
    def backward(ctx, g):
        d = ctx.d
        ctx.d = None
        return (d if g is None else d * g), None, None, None
