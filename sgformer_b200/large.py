"""Drop-in for the reference's large/ours.py (`--method sgformer`, large/parse.py:35-39): same classes, constructor
and forward signatures, attribute names and state_dict keys; computation on the sm_90a kernels."""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import engine as E
from . import functional as Fn
from .config import make_config
from .dist import SINGLE
from .graph import Graph, get_graph
from .minibatch import MiniBatch
from .modules import GraphConvBase, GraphConvLayerBase, SGFormerBase, TransConvBase, TransConvLayerBase

__all__ = ["GraphConvLayer", "GraphConv", "TransConvLayer", "TransConv", "SGFormer"]


class GraphConvLayer(GraphConvLayerBase):
    """large/ours.py:10-42"""


class GraphConv(GraphConvBase):
    """large/ours.py:45-94"""
    variant = "large"

    def _layer_cls(self):
        return GraphConvLayer


class TransConvLayer(TransConvLayerBase):
    """large/ours.py:96-162"""

    def forward(self, query_input, source_input, output_attn=False):
        return self._attend(query_input, source_input, output_attn)


class TransConv(TransConvBase):
    """large/ours.py:165-238 (residual = (x + prev)/2, :211)"""
    variant = "large"

    def __init__(self, in_channels, hidden_channels, num_layers=2, num_heads=1, dropout=0.5, use_bn=True,
                 use_residual=True, use_weight=True, use_act=True):
        super().__init__()
        self._build(in_channels, hidden_channels, num_layers, num_heads, use_weight, TransConvLayer)
        self.dropout = dropout
        self.activation = F.relu
        self.use_bn = use_bn
        self.use_residual = use_residual
        self.use_act = use_act

    def forward(self, x):
        return self._run(x)

    def get_attentions(self, x):
        return self._attentions(x, with_act=True)


class SGFormer(SGFormerBase):
    """large/ours.py:241-286"""
    variant = "large"

    def __init__(self, in_channels, hidden_channels, out_channels,
                 trans_num_layers=1, trans_num_heads=1, trans_dropout=0.5, trans_use_bn=True, trans_use_residual=True,
                 trans_use_weight=True, trans_use_act=True,
                 gnn_num_layers=1, gnn_dropout=0.5, gnn_use_weight=True, gnn_use_init=False, gnn_use_bn=True,
                 gnn_use_residual=True, gnn_use_act=True,
                 use_graph=True, graph_weight=0.8, aggregate='add'):
        super().__init__()
        self.trans_conv = TransConv(in_channels, hidden_channels, trans_num_layers, trans_num_heads, trans_dropout,
                                    trans_use_bn, trans_use_residual, trans_use_weight, trans_use_act)
        self.graph_conv = GraphConv(in_channels, hidden_channels, gnn_num_layers, gnn_dropout, gnn_use_bn,
                                    gnn_use_residual, gnn_use_weight, gnn_use_init, gnn_use_act)
        self.use_graph = use_graph
        self.graph_weight = graph_weight
        self.aggregate = aggregate
        self._finish_init(hidden_channels, out_channels, aggregate)
        self.params1 = list(self.trans_conv.parameters())
        self.params2 = list(self.graph_conv.parameters()) if self.graph_conv is not None else []
        self.params2.extend(list(self.fc.parameters()))
        self._io = (in_channels, hidden_channels, out_channels)

    def _cfg(self) -> dict:
        d, h, c = self._io
        t, g = self.trans_conv, self.graph_conv
        _, _, tnl, tnh = t._dims
        _, _, gnl, guw, gui = g._dims
        return make_config(self.variant, d, h, c, trans_num_layers=tnl, num_heads=tnh, trans_dropout=t.dropout,
                           trans_use_bn=t.use_bn, trans_use_residual=t.use_residual,
                           trans_use_weight=t.convs[0].use_weight if tnl else True, trans_use_act=t.use_act,
                           alpha=getattr(self, "alpha", 0.5), gnn_num_layers=gnl, gnn_dropout=g.dropout,
                           gnn_use_weight=guw, gnn_use_init=gui, gnn_use_bn=g.use_bn, gnn_use_residual=g.use_residual,
                           gnn_use_act=g.use_act, use_graph=bool(self.use_graph), graph_weight=float(self.graph_weight),
                           aggregate=self.aggregate)

    def forward(self, x, edge_index=None):
        names, tensors = self._flat()
        if isinstance(x, MiniBatch):
            x, edge_index = x.features, x.graph
        if not x.is_cuda:
            def run(dev, xd, eid):
                graph = get_graph(eid, xd.shape[0], 0) if self.use_graph else None
                return Fn.SGFormerFn.apply(xd, graph, self._cfg(), E.precision(self.precision), self.training, SINGLE, names,
                                           *[t.to(dev) for t in tensors])
            with torch.no_grad():
                return self._host_call(run, x, edge_index)
        comm = self._comm
        if comm.active:
            # row-sharded: x holds this rank's row block, edge_index is the GLOBAL edge list
            if x.shape[0] != comm.rows[1] - comm.rows[0]:
                raise ValueError(f"row-sharded forward expects the {comm.rows[1] - comm.rows[0]} rows of this rank, got {x.shape[0]}")
            graph = get_graph(edge_index, comm.n_global, 0, rows=comm.rows, col_rot=comm.col_rot) if self.use_graph else None
        elif isinstance(edge_index, Graph):
            graph = edge_index      # a prebuilt structure (e.g. Graph.subset(idx) of a mini-batch) instead of an edge list
        else:
            graph = get_graph(edge_index, x.shape[0], 0) if self.use_graph else None
        return Fn.SGFormerFn.apply(x, graph, self._cfg(), E.precision(self.precision), self.training, comm, names, *tensors)

    def reset_parameters(self):
        # the reference never re-initialises self.fc (large/ours.py:283-286); kept.
        self.trans_conv.reset_parameters()
        if self.use_graph:
            self.graph_conv.reset_parameters()
