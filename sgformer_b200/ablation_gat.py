"""SGFormerGAT, the GAT-attention ablation of the medium variant (medium/ablation/oursGAT.py, `--method ours --use_graph
--attention gat` of medium/ablation/parse.py): scaled dot-product attention, s = q.k / sqrt(dk), whose softmax runs over the
heads of each (node, key) pair as in the reference.  The attention runs on the scaled mode of the fused kernels of
csrc/attn_softmax.cu (engine config trans_attention="gat"); LayerNorm / residual / dropout passes, GNN branches, mix and head are
the medium SGFormer's.

The module tree is the reference's: each TransConvLayer holds a TransConvLayerGAT (`attention`: GATAttention's Wq, Wk, Wv, then
its own Wv with use_weight) and, after it, Wk, Wq and Wv of its own that never reach the output.  Those keep a `None` gradient,
as in the reference, so Adam skips them."""
from typing import Optional

import torch.nn as nn

from . import engine as E
from . import functional as Fn
from . import medium
from .modules import _Base, _require_cuda

__all__ = ["GATAttention", "TransConvLayerGAT", "TransConvLayer", "TransConv", "SGFormerGAT"]

_NO_ATTENTIONS = ("SGFormerGAT has no attention matrices to return: the reference's TransConvLayer (oursGAT.py:95-96) unpacks its "
                  "attention output into two names and raises")


class GATAttention(_Base):
    """oursGAT.py:13-44: q = Wq(qs), k = Wk(ks) with H heads of width dk = in_channels // H, v = Wv(vs) with H heads of width
    out_channels; softmax over the heads of q.k / sqrt(dk); -> [N, H, out_channels]."""

    def __init__(self, in_channels, out_channels, num_heads):
        super().__init__()
        self.num_heads = num_heads
        self.dk = in_channels // num_heads
        self.out_channels = out_channels
        self.Wq = nn.Linear(in_channels, num_heads * self.dk)
        self.Wk = nn.Linear(in_channels, num_heads * self.dk)
        self.Wv = nn.Linear(in_channels, num_heads * out_channels)
        self.softmax = nn.Softmax(dim=-1)

    def reset_parameters(self):
        self.Wq.reset_parameters()
        self.Wk.reset_parameters()
        self.Wv.reset_parameters()

    def forward(self, qs, ks, vs, precision: Optional[str] = None):
        if not qs.is_cuda:
            _require_cuda("GATAttention")
            raise RuntimeError("sgformer_b200.GATAttention needs CUDA tensors (no CPU fallback)")
        prec = E.precision(precision or self.precision)
        h, dk = self.num_heads, self.dk
        mp = E.gat_attn_pad(dk, prec)
        # q and k straight into the kernels' layout: each head's rows of Wq / Wk followed by zero rows (a copy of the weights;
        # autograd drops the pad rows from their gradients)
        q, k = (Fn.LinearFn.apply(x, E.gat_attn_pad_rows(lin.weight, h, dk, mp), E.gat_attn_pad_rows(lin.bias, h, dk, mp), prec)
                for x, lin in ((qs, self.Wq), (ks, self.Wk)))
        v = Fn.LinearFn.apply(vs, self.Wv.weight, self.Wv.bias, prec)
        return Fn.ScaledAttentionFn.apply(q, k, v, h, dk, prec)


class TransConvLayerGAT(_Base):
    """oursGAT.py:46-71: value = Wv(source) with use_weight (else the source itself), then GATAttention(query, key, value)."""

    def __init__(self, in_channels, out_channels, num_heads, use_weight=True):
        super().__init__()
        self.attention = GATAttention(in_channels, out_channels, num_heads)
        self.use_weight = use_weight
        if use_weight:
            self.Wv = nn.Linear(in_channels, out_channels)

    def reset_parameters(self):
        self.attention.reset_parameters()
        if self.use_weight:
            self.Wv.reset_parameters()

    def forward(self, query_input, source_input):
        value = source_input
        if self.use_weight:
            value = Fn.LinearFn.apply(source_input, self.Wv.weight, self.Wv.bias, E.precision(self.precision))
        return self.attention(query_input, source_input, value)


class TransConvLayer(_Base):
    """oursGAT.py:73-107: TransConvLayerGAT(x, x) and the head mean.  Wk, Wq and (with use_weight) Wv are registered after it and
    unused: the reference evaluates Wv and discards the result, which changes nothing and is skipped here."""

    def __init__(self, in_channels, out_channels, num_heads, use_weight=True):
        super().__init__()
        self.attention = TransConvLayerGAT(in_channels, out_channels, num_heads, use_weight)
        self.use_weight = use_weight
        self.Wk = nn.Linear(in_channels, out_channels * num_heads)
        self.Wq = nn.Linear(in_channels, out_channels * num_heads)
        if use_weight:
            self.Wv = nn.Linear(in_channels, out_channels * num_heads)

    def reset_parameters(self):
        self.attention.reset_parameters()

    def forward(self, query_input, source_input, edge_index=None, edge_weight=None, output_attn=False):
        if output_attn:
            raise ValueError(f"sgformer_b200: {_NO_ATTENTIONS}")
        return self.attention(query_input, source_input).mean(dim=1)


class TransConv(medium.TransConv):
    """oursGAT.py:110-183: the medium TransConv (stem, residual, LayerNorm, dropout; use_act is never passed, so False) with
    GAT-attention layers."""
    attention = "gat"
    _layer_cls = TransConvLayer

    def get_attentions(self, x):
        raise ValueError(f"sgformer_b200: {_NO_ATTENTIONS}")


class SGFormerGAT(medium.SGFormer):
    """oursGAT.py:185-229: the medium SGFormer with the GAT-attention TransConv; params1 / params2, reset_parameters, the native
    GCN, GAT and GCNJK branches and the foreign-GNN fallback are the medium SGFormer's."""
    _trans_conv_cls = TransConv
