"""nn.Module surface shared by the three reference variants (large/, 100M/, medium/ `ours.py`).

The modules are *parameter containers with the reference's exact attribute tree* (so state_dict keys, default inits,
`.to()`, `copy.deepcopy`, `params1/params2` and `reset_parameters` behave as in the reference — SURVEY.md §8b) whose
`forward` hands the flat parameter list to the fused CUDA schedules in functional.py.  No torch op computes on the
hot path; there is no CPU implementation: a CPU call is executed on cuda:0 and its result copied back (how
large/eval.py:35-65 `evaluate_large(device="cpu")` keeps working), and fails loudly when no GPU exists.
"""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import engine as E
from . import functional as Fn
from .config import make_config
from .dist import SINGLE
from .graph import get_graph

Tensor = torch.Tensor


def default_precision() -> str:
    return os.environ.get("SGFORMER_B200_PRECISION", "fp32")


def _require_cuda(what: str):
    if not torch.cuda.is_available():
        raise RuntimeError(f"sgformer_b200: {what} needs a CUDA device (sm_90a); there is no CPU fallback")


class _Base(nn.Module):
    """Flat (name, tensor) views of parameters + buffers for the Functions; precision switch."""

    _precision: str = ""

    @property
    def precision(self) -> str:
        return self._precision or default_precision()

    def set_precision(self, name: str):
        E.precision(name)  # validate
        for m in self.modules():
            if isinstance(m, _Base):
                m._precision = name
        return self

    def _flat(self, prefix: str = ""):
        names, tensors = [], []
        for n, p in self.named_parameters():
            names.append(prefix + n)
            tensors.append(p)
        for n, b in self.named_buffers():
            names.append(prefix + n)
            tensors.append(b)
        return tuple(names), tensors


# =================================================================================================
# attention
# =================================================================================================
def full_attention_conv(qs: Tensor, ks: Tensor, vs: Tensor, output_attn: bool = False, precision: Optional[str] = None):
    """Reference free function (medium/ours.py:14-46, 100M/ours.py:12-53): qs,ks [N,H,M], vs [N,H,D] or [N,1,D] (one value
    shared by all heads) -> [N,H,D] (+ the [N,N] visualisation matrix when output_attn)."""
    if not qs.is_cuda:
        _require_cuda("full_attention_conv")
        raise RuntimeError("sgformer_b200.full_attention_conv needs CUDA tensors (no CPU fallback)")
    out = Fn.AttentionFn.apply(qs, ks, vs, E.precision(precision or default_precision()))
    if output_attn:
        return out, _attention_matrix(qs, ks)
    return out


def _attention_matrix(qs: Tensor, ks: Tensor) -> Tensor:
    """O(N^2) visualisation path (medium/ours.py:37-40) — out of the performance scope, plain tensor ops."""
    n = qs.shape[0]
    qn = qs / torch.linalg.vector_norm(qs)
    kn = ks / torch.linalg.vector_norm(ks)
    den = torch.einsum("nhm,hm->nh", qn, kn.sum(dim=0)) + n
    att = torch.einsum("nhm,lhm->nlh", qn, kn).mean(dim=-1)
    return att / den.mean(dim=-1, keepdim=True)


class TransConvLayerBase(_Base):
    """Wq/Wk/(Wv) projections + full_attention_conv + head mean (medium/ours.py:49-100, large/ours.py:96-162)."""

    def __init__(self, in_channels, out_channels, num_heads, use_weight=True):
        super().__init__()
        self.Wk = nn.Linear(in_channels, out_channels * num_heads)
        self.Wq = nn.Linear(in_channels, out_channels * num_heads)
        if use_weight:
            self.Wv = nn.Linear(in_channels, out_channels * num_heads)
        self.out_channels = out_channels
        self.num_heads = num_heads
        self.use_weight = use_weight

    def reset_parameters(self):
        self.Wk.reset_parameters()
        self.Wq.reset_parameters()
        if self.use_weight:
            self.Wv.reset_parameters()

    def _attend(self, query_input, source_input, output_attn=False):
        prec = E.precision(self.precision)
        q = Fn.LinearFn.apply(query_input, self.Wq.weight, self.Wq.bias, prec).reshape(-1, self.num_heads, self.out_channels)
        k = Fn.LinearFn.apply(source_input, self.Wk.weight, self.Wk.bias, prec).reshape(-1, self.num_heads, self.out_channels)
        if self.use_weight:
            v = Fn.LinearFn.apply(source_input, self.Wv.weight, self.Wv.bias, prec).reshape(-1, self.num_heads, self.out_channels)
        else:       # medium/ours.py:84: one value, the layer input, shared by every head
            v = source_input.reshape(-1, 1, self.out_channels)
        out = Fn.AttentionFn.apply(q, k, v, prec).mean(dim=1)
        if output_attn:
            return out, _attention_matrix(q, k)
        return out


class TransConvBase(_Base):
    variant = "large"
    attention = "linear"        # engine config `trans_attention`: "softmax" / "gat" for SGFormerSOFT's / SGFormerGAT's TransConv

    def _build(self, in_channels, hidden_channels, num_layers, num_heads, use_weight, layer_cls):
        self.convs = nn.ModuleList()
        self.fcs = nn.ModuleList()
        self.fcs.append(nn.Linear(in_channels, hidden_channels))
        self.bns = nn.ModuleList()
        self.bns.append(nn.LayerNorm(hidden_channels))
        for _ in range(num_layers):
            self.convs.append(layer_cls(hidden_channels, hidden_channels, num_heads=num_heads, use_weight=use_weight))
            self.bns.append(nn.LayerNorm(hidden_channels))
        self._dims = (in_channels, hidden_channels, num_layers, num_heads)

    def reset_parameters(self):
        for conv in self.convs:
            conv.reset_parameters()
        for bn in self.bns:
            bn.reset_parameters()
        for fc in self.fcs:
            fc.reset_parameters()

    def _cfg(self) -> dict:
        d, h, nl, nh = self._dims
        return make_config(self.variant, d, h, h, trans_num_layers=nl, num_heads=nh, trans_dropout=self.dropout,
                           trans_use_bn=self.use_bn, trans_use_residual=self._use_residual(),
                           trans_use_weight=self.convs[0].use_weight if nl else True, trans_use_act=self.use_act,
                           alpha=getattr(self, "alpha", 0.5), trans_attention=self.attention)

    def _use_residual(self):
        return getattr(self, "use_residual", getattr(self, "residual", True))

    def _run(self, x: Tensor) -> Tensor:
        if not x.is_cuda:
            raise RuntimeError("sgformer_b200.TransConv needs CUDA tensors (no CPU fallback)")
        names, tensors = self._flat("trans_conv.")
        return Fn.TransConvFn.apply(x, self._cfg(), E.precision(self.precision), self.training, names, *tensors)

    def _attentions(self, x: Tensor, with_act: bool) -> Tensor:
        """get_attentions (large/ours.py:221-238; medium/100M skip the activation) -> [layers, N, N], on the kernels
        (engine.trans_attentions).  CPU inputs are computed on cuda:0 and copied back, like forward."""
        _require_cuda("get_attentions")
        names, tensors = self._flat("trans_conv.")
        host = not x.is_cuda
        dev = torch.device("cuda", torch.cuda.current_device()) if host else x.device
        with torch.no_grad():
            P = {n_: (t.to(dev) if host else t) for n_, t in zip(names, tensors)}
            prec = E.precision(self.precision)
            atts = E.trans_attentions(P, self._cfg(), E.input_operand(x.to(dev), prec), prec, with_act)
            out = torch.stack([a.contiguous() for a in atts], dim=0)
        return out.to(x.device) if host else out


# =================================================================================================
# GCN branch of large / 100M
# =================================================================================================
class GraphConvLayerBase(_Base):
    def __init__(self, in_channels, out_channels, use_weight=True, use_init=False):
        super().__init__()
        self.use_init = use_init
        self.use_weight = use_weight
        self.W = nn.Linear(2 * in_channels if use_init else in_channels, out_channels)

    def reset_parameters(self):
        self.W.reset_parameters()

    def forward(self, x, edge_index, x0):
        """large/ours.py:25-42: Â·x (CSR SpMM, structure cached per edge_index) then W·[x || x0] / W·x / identity."""
        if not x.is_cuda:
            raise RuntimeError("sgformer_b200.GraphConvLayer needs CUDA tensors (no CPU fallback)")
        prec = E.precision(self.precision)
        graph = get_graph(edge_index, x.shape[0], 0)
        y = Fn.SpMMFn.apply(x, graph, prec)
        if self.use_init:
            return Fn.LinearFn.apply(torch.cat([y, x0], 1), self.W.weight, self.W.bias, prec)
        if self.use_weight:
            return Fn.LinearFn.apply(y, self.W.weight, self.W.bias, prec)
        return y


class GraphConvBase(_Base):
    variant = "large"

    def __init__(self, in_channels, hidden_channels, num_layers=2, dropout=0.5, use_bn=True, use_residual=True,
                 use_weight=True, use_init=False, use_act=True):
        super().__init__()
        self.convs = nn.ModuleList()
        self.fcs = nn.ModuleList()
        self.fcs.append(nn.Linear(in_channels, hidden_channels))
        self.bns = nn.ModuleList()
        self.bns.append(nn.BatchNorm1d(hidden_channels))
        for _ in range(num_layers):
            self.convs.append(self._layer_cls()(hidden_channels, hidden_channels, use_weight, use_init))
            self.bns.append(nn.BatchNorm1d(hidden_channels))
        self.dropout = dropout
        self.activation = F.relu
        self.use_bn = use_bn
        self.use_residual = use_residual
        self.use_act = use_act
        self._dims = (in_channels, hidden_channels, num_layers, use_weight, use_init)

    def _layer_cls(self):
        return GraphConvLayerBase

    def reset_parameters(self):
        for conv in self.convs:
            conv.reset_parameters()
        for bn in self.bns:
            bn.reset_parameters()
        for fc in self.fcs:
            fc.reset_parameters()

    def _cfg(self) -> dict:
        d, h, nl, uw, ui = self._dims
        return make_config(self.variant, d, h, h, gnn_num_layers=nl, gnn_dropout=self.dropout, gnn_use_weight=uw,
                           gnn_use_init=ui, gnn_use_bn=self.use_bn, gnn_use_residual=self.use_residual,
                           gnn_use_act=self.use_act)

    def forward(self, x, edge_index):
        if not x.is_cuda:
            raise RuntimeError("sgformer_b200.GraphConv needs CUDA tensors (no CPU fallback)")
        names, tensors = self._flat("graph_conv.")
        graph = get_graph(edge_index, x.shape[0], 0)
        return Fn.GraphBranchFn.apply(x, graph, self._cfg(), E.precision(self.precision), self.training, "gconv",
                                      "graph_conv.", names, *tensors)


# =================================================================================================
# encoder
# =================================================================================================
class SGFormerBase(_Base):
    variant = "large"
    _comm = SINGLE

    def set_row_sharding(self, comm):
        """Row-sharded multi-GPU execution (SURVEY.md §8e): `comm = sgformer_b200.dist.Comm(group, n_global)`.  forward then
        takes this rank's row block of x and the global edge_index and returns this rank's rows of the logits; parameter
        gradients come back already all-reduced.  `None` / `Comm(None)` restores single-GPU execution."""
        self._comm = comm if comm is not None else SINGLE
        return self

    _self_loop_mode = 0       # 1 in the medium variant (PyG gcn_norm adds the missing self loops)

    def prepare_graph(self, edge_index, num_nodes: int, backward: bool = True):
        """Builds (and caches) the structure forward() derives from `edge_index`: the CSR, its normalisation and, for training,
        the decision whether the backward SpMM shares it.  forward() does this itself on first sight of an edge_index; calling it
        ahead of time - e.g. on the copy stream of `HostFeeder(prepare=...)` - takes the graph build off the step's critical path."""
        if not getattr(self, "use_graph", True):
            return None
        comm = self._comm
        if comm.active:
            g = get_graph(edge_index, comm.n_global, self._self_loop_mode, rows=comm.rows, col_rot=comm.col_rot)
        else:
            g = get_graph(edge_index, num_nodes, self._self_loop_mode)
        if backward:
            g.transpose()
        return g

    def _finish_init(self, hidden_channels, out_channels, aggregate):
        if aggregate == "add":
            self.fc = nn.Linear(hidden_channels, out_channels)
        elif aggregate == "cat":
            self.fc = nn.Linear(2 * hidden_channels, out_channels)
        else:
            raise ValueError(f"Invalid aggregate type:{aggregate}")

    def get_attentions(self, x):
        return self.trans_conv.get_attentions(x)

    def _host_call(self, run, *tensors):
        """Inputs on the host (e.g. evaluate_large(device='cpu') after model.to('cpu')): compute on the GPU with
        temporary device copies of the parameters, return the result on the host.  Inference only."""
        _require_cuda("SGFormer.forward")
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise RuntimeError("sgformer_b200: training needs the model and inputs on a CUDA device (no CPU fallback)")
        dev = torch.device("cuda", torch.cuda.current_device())
        return run(dev, *[t.to(dev) for t in tensors]).cpu()
