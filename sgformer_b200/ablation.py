"""SGFormerSOFT, the softmax-attention ablation of the medium variant (medium/ablation/oursSOFT.py, `--method ours --attention
softmax` of medium/ablation/parse.py): the medium SGFormer's model tree with full_attention_conv replaced by softmax_attention.
The attention runs on the fused kernels of csrc/attn_softmax.cu (engine config trans_attention="softmax"); the projections,
LayerNorm / residual / dropout passes, GNN branches, mix and head are the medium SGFormer's."""
from typing import Optional

import torch

from . import engine as E
from . import functional as Fn
from . import medium
from .modules import _require_cuda, default_precision

__all__ = ["softmax_attention", "TransConvLayer", "TransConv", "SGFormerSOFT"]


def softmax_attention(qs, ks, vs, output_attn=False, precision: Optional[str] = None):
    """oursSOFT.py:14-34: qs, ks [N, H, M], vs [N, H, D] or [N, 1, D] (one value shared by every head) -> [N, H, D] (and, with
    output_attn, the [N, N] head mean of the softmax weights)."""
    if not qs.is_cuda:
        _require_cuda("softmax_attention")
        raise RuntimeError("sgformer_b200.softmax_attention needs CUDA tensors (no CPU fallback)")
    return Fn.SoftmaxAttentionFn.apply(qs, ks, vs, E.precision(precision or default_precision()), bool(output_attn))


class TransConvLayer(medium.TransConvLayer):
    """oursSOFT.py:37-88: Wq / Wk / (Wv) projections, softmax_attention, head mean."""

    def forward(self, query_input, source_input, edge_index=None, edge_weight=None, output_attn=False):
        prec = E.precision(self.precision)
        q = Fn.LinearFn.apply(query_input, self.Wq.weight, self.Wq.bias, prec).reshape(-1, self.num_heads, self.out_channels)
        k = Fn.LinearFn.apply(source_input, self.Wk.weight, self.Wk.bias, prec).reshape(-1, self.num_heads, self.out_channels)
        if self.use_weight:
            v = Fn.LinearFn.apply(source_input, self.Wv.weight, self.Wv.bias, prec).reshape(-1, self.num_heads, self.out_channels)
        else:       # oursSOFT.py:72: one value, the layer input, shared by every head
            v = source_input.reshape(-1, 1, self.out_channels)
        res = Fn.SoftmaxAttentionFn.apply(q, k, v, prec, bool(output_attn))
        if output_attn:
            out, attn = res
            return out.mean(dim=1), attn
        return res.mean(dim=1)


class TransConv(medium.TransConv):
    """oursSOFT.py:91-165: the medium TransConv (same parameters, order and initialisation) with softmax attention layers."""
    attention = "softmax"
    _layer_cls = TransConvLayer


class SGFormerSOFT(medium.SGFormer):
    """oursSOFT.py:167-211: the medium SGFormer with the softmax TransConv; params1 / params2, reset_parameters, the native GCN,
    GAT and GCNJK branches and the foreign-GNN fallback are the medium SGFormer's."""
    _trans_conv_cls = TransConv
