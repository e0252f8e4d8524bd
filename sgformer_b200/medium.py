"""Drop-in for the reference's medium/ours.py (`--method ours`, medium/parse.py:97-104) plus native `GCN`, `GAT` and `GCNJK`
backbones with the semantics of medium/models.py:14-63 (PyG GCNConv stack), :116-155 (PyG GATConv stack) and :157-205 (GCNConv
stack with JumpingKnowledge) for users without torch_geometric."""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import engine as E
from . import functional as Fn
from .config import make_config
from .dist import SINGLE
from .graph import Graph, get_graph
from .modules import SGFormerBase, TransConvBase, TransConvLayerBase, _Base, full_attention_conv

# GAT / GATConv / GCNJK stay out of __all__: the medium drop-in star-imports this module after the reference's `models`, and a star
# export would replace the reference's GAT / GCNJK in its parse.py (`--method gat|gcnjk`, `--backbone gat|gcnjk`) without being
# asked to (`launch --native-backbones` opts in)
__all__ = ["full_attention_conv", "TransConvLayer", "TransConv", "SGFormer", "GCN", "GCNConv"]


class TransConvLayer(TransConvLayerBase):
    """medium/ours.py:49-100"""

    def forward(self, query_input, source_input, edge_index=None, edge_weight=None, output_attn=False):
        return self._attend(query_input, source_input, output_attn)


class TransConv(TransConvBase):
    """medium/ours.py:103-177 (takes the dataset object; residual = alpha*x + (1-alpha)*prev, :152)"""
    variant = "medium"
    _layer_cls = TransConvLayer

    def __init__(self, in_channels, hidden_channels, num_layers=2, num_heads=1, alpha=0.5, dropout=0.5, use_bn=True,
                 use_residual=True, use_weight=True, use_act=False):
        super().__init__()
        self._build(in_channels, hidden_channels, num_layers, num_heads, use_weight, self._layer_cls)
        self.dropout = dropout
        self.activation = F.relu
        self.use_bn = use_bn
        self.residual = use_residual
        self.alpha = alpha
        self.use_act = use_act

    def forward(self, data):
        return self._run(data.graph['node_feat'])

    def get_attentions(self, x):
        return self._attentions(x, with_act=False)


class _Lin(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(cout, cin))


class GCNConv(nn.Module):
    """Parameter container with PyG>=2 GCNConv's names (`lin.weight` [out,in], `bias`) and inits (glorot / zeros)."""

    def __init__(self, in_channels, out_channels, cached=False, **kw):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.lin = _Lin(in_channels, out_channels)
        self.bias = nn.Parameter(torch.empty(out_channels))
        self.reset_parameters()

    def reset_parameters(self):
        a = math.sqrt(6.0 / (self.in_channels + self.out_channels))
        nn.init.uniform_(self.lin.weight, -a, a)
        nn.init.zeros_(self.bias)


class GCN(_Base):
    """models.GCN (medium/models.py:14-63): `num_layers` GCNConv layers, BN/ReLU/dropout between them."""

    def __init__(self, in_channels, hidden_channels, out_channels, num_layers=2, dropout=0.5, save_mem=True, use_bn=True):
        super().__init__()
        self.convs = nn.ModuleList()
        self.convs.append(GCNConv(in_channels, hidden_channels, cached=not save_mem))
        self.bns = nn.ModuleList()
        self.bns.append(nn.BatchNorm1d(hidden_channels))
        for _ in range(num_layers - 2):
            self.convs.append(GCNConv(hidden_channels, hidden_channels, cached=not save_mem))
            self.bns.append(nn.BatchNorm1d(hidden_channels))
        self.convs.append(GCNConv(hidden_channels, out_channels, cached=not save_mem))
        self.dropout = dropout
        self.activation = F.relu
        self.use_bn = use_bn

    def reset_parameters(self):
        for conv in self.convs:
            conv.reset_parameters()
        for bn in self.bns:
            bn.reset_parameters()

    def forward(self, data):
        x, edge_index = data.graph['node_feat'], data.graph['edge_index']
        if not x.is_cuda:
            raise RuntimeError("sgformer_b200.GCN needs CUDA tensors (no CPU fallback)")
        names, tensors = _gcn_flat(self, "gnn.")
        cfg = make_config("medium", x.shape[1], self.convs[0].out_channels, self.convs[-1].out_channels,
                          gcn_num_layers=len(self.convs), gcn_dropout=self.dropout, gcn_use_bn=self.use_bn)
        graph, names, tensors = _gcn_graph(data, x.shape[0], names, tensors)
        return Fn.GraphBranchFn.apply(x, graph, cfg, E.precision(self.precision), self.training, "gcn", "gnn.", names,
                                      *tensors)


def _gcn_graph(data, n, names, tensors):
    """The mode-1 Graph of data.graph: weighted when data.graph['edge_weight'] is set (models.GCN passes it to every conv but the
    last, medium/models.py:53-62); the weight then joins the autograd inputs under engine.EDGE_WEIGHT."""
    w = data.graph.get('edge_weight', None)
    if w is None:
        return get_graph(data.graph['edge_index'], n, 1), names, tensors
    return get_graph(data.graph['edge_index'], n, 1, edge_weight=w), tuple(names) + (E.EDGE_WEIGHT,), list(tensors) + [w]


def _is_gcn_like(gnn) -> bool:
    """A models.GCN-shaped module (ours, or the reference's over PyG GCNConv) whose layers we can run natively."""
    try:
        convs, bns = gnn.convs, gnn.bns
        if len(convs) < 1 or not hasattr(gnn, "dropout") or not hasattr(gnn, "use_bn"):
            return False
        for c in convs:
            w = c.lin.weight if hasattr(c, "lin") else c.weight
            if w.dim() != 2 or getattr(c, "bias", None) is None:
                return False
            if getattr(c, "improved", False) or not getattr(c, "normalize", True) or not getattr(c, "add_self_loops", True):
                return False
        return len(bns) >= len(convs) - 1
    except AttributeError:
        return False


def _gcn_out_dim(gnn) -> int:
    c = gnn.convs[-1]
    return c.lin.weight.shape[0] if hasattr(c, "lin") else c.weight.shape[1]


def _gcn_flat(gnn, prefix):
    """(names, tensors) with PyG>=2 naming; PyG 1.x stores GCNConv.weight as [in,out] -> transposed view (autograd
    carries the gradient back through the transpose)."""
    names, tensors = [], []
    for i, c in enumerate(gnn.convs):
        if hasattr(c, "lin"):
            w = c.lin.weight
        else:
            w = c.weight.t().contiguous()
        names.append(f"{prefix}convs.{i}.lin.weight"); tensors.append(w)
        names.append(f"{prefix}convs.{i}.bias"); tensors.append(c.bias)
    for i, bn in enumerate(gnn.bns):
        for nm in ("weight", "bias", "running_mean", "running_var", "num_batches_tracked"):
            names.append(f"{prefix}bns.{i}.{nm}"); tensors.append(getattr(bn, nm))
    return tuple(names), tensors


# PyG GATConv parameter names of other generations -> the 2.0-2.3 names used here (lin_src is lin_dst: one shared Linear)
_GAT_ALIASES = {"lin_l.weight": ("lin_src.weight", "lin_dst.weight"), "lin_r.weight": ("lin_src.weight", "lin_dst.weight"),
                "lin.weight": ("lin_src.weight", "lin_dst.weight"), "att_l": ("att_src",), "att_r": ("att_dst",)}


class GATConv(nn.Module):
    """Parameter container with PyG 2.0-2.3 GATConv's names and inits for `in_channels: int`: `lin_src` (= `lin_dst`, one shared
    bias-free Linear, weight [heads*out, in], glorot), `att_src` / `att_dst` [1, heads, out] (glorot), `bias` [heads*out] with
    concat else [out] (zeros).  load_state_dict also accepts PyG 1.7.2's `lin_l` / `lin_r` / `att_l` / `att_r` and PyG >= 2.4's
    `lin`.  It runs inside `GAT` (one schedule for the whole stack); calling a conv on its own is not supported."""

    def __init__(self, in_channels, out_channels, heads=1, concat=True, negative_slope=0.2, dropout=0.0, add_self_loops=True,
                 edge_dim=None, fill_value='mean', bias=True, **kw):
        super().__init__()
        if not isinstance(in_channels, int):
            raise NotImplementedError("sgformer_b200.GATConv: bipartite (tuple) in_channels are not supported")
        if edge_dim is not None:
            raise NotImplementedError("sgformer_b200.GATConv: edge_attr / edge_dim is not supported")
        if negative_slope != 0.2 or not add_self_loops or not bias:
            raise NotImplementedError("sgformer_b200.GATConv: only negative_slope=0.2, add_self_loops=True and bias=True are "
                                      "supported (PyG's defaults, as models.GAT uses them)")
        self.in_channels, self.out_channels, self.heads, self.concat = in_channels, out_channels, heads, concat
        self.negative_slope, self.dropout, self.add_self_loops = negative_slope, dropout, add_self_loops
        self.lin_src = _Lin(in_channels, heads * out_channels)
        self.lin_dst = self.lin_src
        self.att_src = nn.Parameter(torch.empty(1, heads, out_channels))
        self.att_dst = nn.Parameter(torch.empty(1, heads, out_channels))
        self.bias = nn.Parameter(torch.empty(heads * out_channels if concat else out_channels))
        self.reset_parameters()

    def reset_parameters(self):
        w = self.lin_src.weight
        a = math.sqrt(6.0 / (w.size(-2) + w.size(-1)))
        nn.init.uniform_(w, -a, a)
        for att in (self.att_src, self.att_dst):
            a = math.sqrt(6.0 / (att.size(-2) + att.size(-1)))
            nn.init.uniform_(att, -a, a)
        nn.init.zeros_(self.bias)

    def _load_from_state_dict(self, state_dict, prefix, *args, **kw):
        for old, new in _GAT_ALIASES.items():
            if prefix + old in state_dict:
                t = state_dict.pop(prefix + old)
                for nm in new:
                    state_dict.setdefault(prefix + nm, t)
        super()._load_from_state_dict(state_dict, prefix, *args, **kw)

    def forward(self, x, edge_index, edge_attr=None, size=None, return_attention_weights=None):
        if return_attention_weights:
            raise NotImplementedError("sgformer_b200.GATConv: return_attention_weights is not supported")
        raise NotImplementedError("sgformer_b200.GATConv runs inside sgformer_b200.medium.GAT (one schedule for the whole stack)")


class GAT(_Base):
    """models.GAT (medium/models.py:116-155): input dropout, GATConv(heads, concat) layers with BatchNorm?/ELU/dropout between them,
    a last GATConv(out_heads, concat=False)."""

    def __init__(self, in_channels, hidden_channels, out_channels, num_layers=2, dropout=0.5, use_bn=False, heads=2, out_heads=1):
        super().__init__()
        self.convs = nn.ModuleList()
        self.convs.append(GATConv(in_channels, hidden_channels, dropout=dropout, heads=heads, concat=True))
        self.bns = nn.ModuleList()
        self.bns.append(nn.BatchNorm1d(hidden_channels * heads))
        for _ in range(num_layers - 2):
            self.convs.append(GATConv(hidden_channels * heads, hidden_channels, dropout=dropout, heads=heads, concat=True))
            self.bns.append(nn.BatchNorm1d(hidden_channels * heads))
        self.convs.append(GATConv(hidden_channels * heads, out_channels, dropout=dropout, heads=out_heads, concat=False))
        self.dropout = dropout
        self.activation = F.elu
        self.use_bn = use_bn

    def reset_parameters(self):
        for conv in self.convs:
            conv.reset_parameters()
        for bn in self.bns:
            bn.reset_parameters()

    def _cfg_kw(self):
        return dict(gcn_num_layers=len(self.convs), gcn_dropout=float(self.dropout), gcn_use_bn=bool(self.use_bn), gnn_kind="gat")

    def forward(self, data):
        x, edge_index = data.graph['node_feat'], data.graph['edge_index']
        _check_gat_data(data)
        if not x.is_cuda:
            raise RuntimeError("sgformer_b200.GAT needs CUDA tensors (no CPU fallback)")
        return self._run(x, edge_index)

    def _run(self, x, edge_index, names=None, tensors=None):
        """The stack on CUDA x / edge_index (or a prebuilt self_loop_mode 1 Graph, from large_gnns.GAT); (names, tensors) default
        to this module's own (large_gnns.GAT passes device copies)."""
        if names is None:
            names, tensors = _gat_flat(self, "")
        cfg = make_config("medium", x.shape[1], self.convs[0].lin_src.weight.shape[0], self.convs[-1].out_channels, **self._cfg_kw())
        graph = edge_index if isinstance(edge_index, Graph) else get_graph(edge_index, x.shape[0], 1)
        return Fn.GraphBranchFn.apply(x, graph, cfg, E.precision(self.precision), self.training, "gat", "", names, *tensors)


def _check_gat_data(data):
    # models.GAT never reads edge_weight (medium/models.py:145-155): it is ignored here as well
    if data.graph.get('edge_attr', None) is not None:
        raise NotImplementedError("sgformer_b200.GAT: edge_attr is not supported")


def _gat_flat(gnn, prefix):
    """(names, tensors) of a GAT with PyG 2.0-2.3 GATConv naming."""
    names, tensors = [], []
    for i, c in enumerate(gnn.convs):
        for nm, t in (("lin_src.weight", c.lin_src.weight), ("att_src", c.att_src), ("att_dst", c.att_dst), ("bias", c.bias)):
            names.append(f"{prefix}convs.{i}.{nm}"); tensors.append(t)
    for i, bn in enumerate(gnn.bns[:len(gnn.convs) - 1]):
        for nm in ("weight", "bias", "running_mean", "running_var", "num_batches_tracked"):
            names.append(f"{prefix}bns.{i}.{nm}"); tensors.append(getattr(bn, nm))
    return tuple(names), tensors


class JumpingKnowledge(nn.Module):
    """PyG's JumpingKnowledge in 'max' / 'cat' mode: no parameters; it runs inside `GCNJK` (one schedule for the whole model)."""

    def __init__(self, mode, channels=None, num_layers=None):
        super().__init__()
        self.mode = mode.lower()
        if self.mode == "lstm":
            raise NotImplementedError("sgformer_b200.GCNJK: jk_type='lstm' is not supported (use 'max' or 'cat')")
        if self.mode not in ("max", "cat"):
            raise ValueError(f"JumpingKnowledge: unknown mode {mode!r}")

    def reset_parameters(self):
        pass

    def forward(self, xs):
        raise NotImplementedError("sgformer_b200.JumpingKnowledge runs inside sgformer_b200.medium.GCNJK")


class GCNJK(_Base):
    """models.GCNJK (medium/models.py:157-205): GCNConv(in, hidden), num_layers - 2 GCNConv(hidden, hidden) and a last
    GCNConv(hidden, hidden) (at least two convs), BatchNorm/ReLU/dropout after every conv but the last, JumpingKnowledge over the
    layers' activations (taken before their dropout) and final_project = Linear(hidden -> out) ('max') or Linear(hidden *
    num_layers -> out) ('cat').  No `use_bn` attribute (BatchNorm is always on), so SGFormer never mistakes it for a models.GCN;
    data.graph['edge_weight'] is ignored, as in the reference."""

    def __init__(self, in_channels, hidden_channels, out_channels, num_layers=2, dropout=0.5, save_mem=False, jk_type='max'):
        super().__init__()
        if save_mem:
            raise NotImplementedError("sgformer_b200.GCNJK: save_mem=True (GCNConv(normalize=False)) is not supported")
        jump = JumpingKnowledge(jk_type, channels=hidden_channels, num_layers=1)
        if jump.mode == "cat" and num_layers < 2:
            raise ValueError(f"GCNJK(jk_type='cat', num_layers={num_layers}) concatenates 2 layers of {hidden_channels} channels, "
                             f"but its final_project takes {hidden_channels * num_layers} (the reference fails here too)")
        self.convs = nn.ModuleList()
        self.convs.append(GCNConv(in_channels, hidden_channels, cached=not save_mem))
        self.bns = nn.ModuleList()
        self.bns.append(nn.BatchNorm1d(hidden_channels))
        for _ in range(num_layers - 2):
            self.convs.append(GCNConv(hidden_channels, hidden_channels, cached=not save_mem))
            self.bns.append(nn.BatchNorm1d(hidden_channels))
        self.convs.append(GCNConv(hidden_channels, hidden_channels, cached=not save_mem))
        self.dropout = dropout
        self.activation = F.relu
        self.jump = jump
        self.final_project = nn.Linear(hidden_channels * num_layers if jump.mode == "cat" else hidden_channels, out_channels)

    def reset_parameters(self):
        for conv in self.convs:
            conv.reset_parameters()
        for bn in self.bns:
            bn.reset_parameters()
        self.jump.reset_parameters()
        self.final_project.reset_parameters()

    def _cfg_kw(self):
        return dict(gcn_num_layers=len(self.convs), gcn_dropout=float(self.dropout), gcn_use_bn=True, gnn_kind="gcnjk",
                    gcn_jk=self.jump.mode)

    def forward(self, data):
        x, edge_index = data.graph['node_feat'], data.graph['edge_index']
        if not x.is_cuda:
            raise RuntimeError("sgformer_b200.GCNJK needs CUDA tensors (no CPU fallback)")
        names, tensors = _gcnjk_flat(self, "")
        cfg = make_config("medium", x.shape[1], self.convs[0].out_channels, self.final_project.out_features, **self._cfg_kw())
        graph = get_graph(edge_index, x.shape[0], 1)
        return Fn.GraphBranchFn.apply(x, graph, cfg, E.precision(self.precision), self.training, "gcnjk", "", names, *tensors)


def _gcnjk_flat(gnn, prefix):
    """(names, tensors) of a GCNJK (ours, or the reference's over PyG GCNConv): the GCN stack's, then final_project."""
    names, tensors = _gcn_flat(gnn, prefix)
    names = tuple(names) + (f"{prefix}final_project.weight", f"{prefix}final_project.bias")
    return names, list(tensors) + [gnn.final_project.weight, gnn.final_project.bias]


class SGFormer(SGFormerBase):
    """medium/ours.py:179-223: attention branch + an injected GNN (`gnn=`)."""
    variant = "medium"
    _self_loop_mode = 1
    _trans_conv_cls = TransConv

    def __init__(self, in_channels, hidden_channels, out_channels, num_layers=2, num_heads=1, alpha=0.5, dropout=0.5,
                 use_bn=True, use_residual=True, use_weight=True, use_graph=True, use_act=False, graph_weight=0.8,
                 gnn=None, aggregate='add'):
        super().__init__()
        # medium/ours.py:183 does not forward use_act to TransConv
        self.trans_conv = self._trans_conv_cls(in_channels, hidden_channels, num_layers, num_heads, alpha, dropout, use_bn,
                                               use_residual, use_weight)
        self.gnn = gnn
        self.use_graph = use_graph
        self.graph_weight = graph_weight
        self.use_act = use_act
        self.aggregate = aggregate
        self._finish_init(hidden_channels, out_channels, aggregate)
        self.params1 = list(self.trans_conv.parameters())
        self.params2 = list(self.gnn.parameters()) if self.gnn is not None else []
        self.params2.extend(list(self.fc.parameters()))
        self._io = (in_channels, hidden_channels, out_channels)

    def _cfg(self, gcn_layers=2, gcn_dropout=0.5, gcn_use_bn=True, gnn_kind="gcn", gcn_jk="max") -> dict:
        d, h, c = self._io
        t = self.trans_conv
        _, _, tnl, tnh = t._dims
        return make_config("medium", d, h, c, trans_num_layers=tnl, num_heads=tnh, trans_dropout=t.dropout,
                           trans_use_bn=t.use_bn, trans_use_residual=t.residual,
                           trans_use_weight=t.convs[0].use_weight if tnl else True, trans_use_act=False, alpha=t.alpha,
                           use_graph=bool(self.use_graph), graph_weight=float(self.graph_weight),
                           aggregate=self.aggregate, gcn_num_layers=gcn_layers, gcn_dropout=gcn_dropout,
                           gcn_use_bn=gcn_use_bn, gnn_kind=gnn_kind, gcn_jk=gcn_jk, trans_attention=t.attention)

    def forward(self, data):
        x, edge_index = data.graph['node_feat'], data.graph['edge_index']
        if not x.is_cuda:
            raise RuntimeError("sgformer_b200.SGFormer (medium) needs the dataset on a CUDA device (no CPU fallback)")
        prec = E.precision(self.precision)
        fused = bool(self.use_graph) and self.gnn is not None and _is_gcn_like(self.gnn) and \
            _gcn_out_dim(self.gnn) == self._io[1]
        tn, tt = self.trans_conv._flat("trans_conv.")
        fn, ft = self.fc._parameters.keys(), list(self.fc._parameters.values())
        names = list(tn) + ["fc." + k for k in fn]
        tensors = list(tt) + ft
        if not self.use_graph:
            return Fn.SGFormerFn.apply(x, None, self._cfg(), prec, self.training, self._comm, tuple(names), *tensors)
        if bool(self.use_graph) and isinstance(self.gnn, GAT) and self.gnn.convs[-1].out_channels == self._io[1]:
            _check_gat_data(data)
            if self._comm.active:
                raise NotImplementedError("sgformer_b200: row sharding of the GAT branch is not supported")
            gn, gt = _gat_flat(self.gnn, "gnn.")
            cfg = self._cfg(len(self.gnn.convs), float(self.gnn.dropout), bool(self.gnn.use_bn), "gat")
            graph = get_graph(edge_index, x.shape[0], 1)
            return Fn.SGFormerFn.apply(x, graph, cfg, prec, self.training, self._comm, tuple(names) + tuple(gn), *tensors, *gt)
        if isinstance(self.gnn, GCNJK) and self.gnn.final_project.out_features == self._io[1]:
            if self._comm.active:
                raise NotImplementedError("sgformer_b200: row sharding of the GCNJK branch is not supported")
            gn, gt = _gcnjk_flat(self.gnn, "gnn.")
            cfg = self._cfg(len(self.gnn.convs), float(self.gnn.dropout), True, "gcnjk", self.gnn.jump.mode)
            graph = get_graph(edge_index, x.shape[0], 1)
            return Fn.SGFormerFn.apply(x, graph, cfg, prec, self.training, self._comm, tuple(names) + tuple(gn), *tensors, *gt)
        if fused:
            gn, gt = _gcn_flat(self.gnn, "gnn.")
            cfg = self._cfg(len(self.gnn.convs), float(self.gnn.dropout), bool(self.gnn.use_bn))
            comm = self._comm
            if comm.active:
                if data.graph.get('edge_weight', None) is not None:
                    raise NotImplementedError("sgformer_b200: row sharding of a weighted graph (edge_weight) is not supported")
                graph = get_graph(edge_index, comm.n_global, 1, rows=comm.rows, col_rot=comm.col_rot)
            else:
                graph, gn, gt = _gcn_graph(data, x.shape[0], gn, gt)
            return Fn.SGFormerFn.apply(x, graph, cfg, prec, self.training, comm, tuple(names) + tuple(gn), *tensors, *gt)
        # foreign GNN module: run it as given, mix + fc on the GPU kernels
        x1 = Fn.TransConvFn.apply(x, self.trans_conv._cfg(), prec, self.training, tn, *tt)
        x2 = self.gnn(data)
        return Fn.HeadFn.apply(x1, x2, self._cfg(), prec, tuple("fc." + k for k in fn), *ft)

    def reset_parameters(self):
        self.trans_conv.reset_parameters()
        if self.use_graph:
            self.gnn.reset_parameters()
