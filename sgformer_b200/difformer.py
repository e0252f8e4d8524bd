"""Drop-in for the reference's medium/difformer.py (`--method difformer`, medium/parse.py:89-96) with kernel='simple' and one head.

`DIFFormer` keeps the reference's attribute tree (state_dict keys, `Wk` before `Wq`, inits, `reset_parameters` of convs, bns and
fcs), so `.to()`, `copy.deepcopy` and `load_state_dict` behave as there; its forward and backward run as one schedule on the CUDA
kernels (functional.DIFFormerFn).  `DIFFormer.forward(data, edge_weight)` runs its graph term on the weighted CSR build and SpMM.
Out of scope, each with an error: num_heads > 1, kernel='sigmoid' (O(N^2)), multi-dimensional edge attributes, and edge weights in
the standalone `gcn_conv`."""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import engine as E
from . import functional as Fn
from .graph import get_graph
from .modules import _Base, _require_cuda, default_precision

__all__ = ["full_attention_conv", "gcn_conv", "DIFFormerConv", "DIFFormer"]


def _check_kernel(kernel):
    if kernel == "sigmoid":
        raise NotImplementedError("sgformer_b200.DIFFormer: kernel='sigmoid' (O(N^2) attention) is not supported; use 'simple'")
    if kernel != "simple":
        raise ValueError(f"sgformer_b200.DIFFormer: unknown kernel {kernel!r}")


def full_attention_conv(qs, ks, vs, kernel, output_attn=False):
    """medium/difformer.py:10-61.  Runs only fused inside DIFFormer (the Gram form never materialises q, k, v)."""
    _check_kernel(kernel)
    raise NotImplementedError("sgformer_b200: DIFFormer's full_attention_conv runs fused inside DIFFormer.forward; "
                              "the standalone function on given q, k, v is not provided")


def gcn_conv(x, edge_index, edge_weight):
    """medium/difformer.py:63-79: y[:, h] = D^-1/2 A D^-1/2 x[:, h] (in-degree over edge targets, no self loops) on the CSR
    SpMM kernel.  x: [N, H, D].  Edge weights run inside DIFFormer.forward (the fused schedule), not through this function."""
    if edge_weight is not None:
        raise NotImplementedError("sgformer_b200.gcn_conv: edge_weight is not supported by the standalone function; "
                                  "DIFFormer.forward(data, edge_weight) runs weighted graphs")
    if not x.is_cuda:
        _require_cuda("gcn_conv")
        raise RuntimeError("sgformer_b200.gcn_conv needs CUDA tensors (no CPU fallback)")
    n = x.shape[0]
    graph = get_graph(edge_index, n, 0)
    prec = E.precision(default_precision())
    return Fn.SpMMFn.apply(x.reshape(n, -1), graph, prec).reshape(x.shape)


class DIFFormerConv(_Base):
    """medium/difformer.py:81-145: parameter container of one layer (Wk, Wq, Wv); the layer runs fused in DIFFormer.forward."""

    def __init__(self, in_channels, out_channels, num_heads, kernel='simple', use_graph=True, use_weight=True, graph_weight=-1,
                 use_source=False):
        super().__init__()
        self.Wk = nn.Linear(in_channels, out_channels * num_heads)
        self.Wq = nn.Linear(in_channels, out_channels * num_heads)
        if use_weight:
            self.Wv = nn.Linear(in_channels, out_channels * num_heads)
        self.out_channels = out_channels
        self.num_heads = num_heads
        self.kernel = kernel
        self.use_graph = use_graph
        self.use_weight = use_weight
        self.graph_weight = graph_weight
        self.use_source = use_source

    def reset_parameters(self):
        self.Wk.reset_parameters()
        self.Wq.reset_parameters()
        if self.use_weight:
            self.Wv.reset_parameters()

    def forward(self, query_input, source_input, edge_index=None, edge_weight=None, x_0=None, output_attn=False):
        raise NotImplementedError("sgformer_b200: DIFFormerConv runs fused inside DIFFormer.forward; a standalone layer call is "
                                  "not provided")


class DIFFormer(_Base):
    """medium/difformer.py:147-228."""

    def __init__(self, in_channels, hidden_channels, out_channels, num_layers=2, num_heads=1, kernel='simple', alpha=0.5,
                 dropout=0.5, use_bn=True, use_residual=True, use_weight=True, use_graph=True, graph_weight=-1, use_source=False):
        super().__init__()
        if num_heads != 1:
            raise ValueError(f"sgformer_b200.DIFFormer supports num_heads == 1 only (got {num_heads})")
        _check_kernel(kernel)
        self.convs = nn.ModuleList()
        self.fcs = nn.ModuleList()
        self.fcs.append(nn.Linear(in_channels, hidden_channels))
        self.bns = nn.ModuleList()
        self.bns.append(nn.LayerNorm(hidden_channels))
        for _ in range(num_layers):
            self.convs.append(DIFFormerConv(hidden_channels, hidden_channels, num_heads=num_heads, kernel=kernel, use_graph=use_graph,
                                            use_weight=use_weight, graph_weight=graph_weight, use_source=use_source))
            self.bns.append(nn.LayerNorm(hidden_channels))
        self.fcs.append(nn.Linear(hidden_channels, out_channels))
        self.dropout = dropout
        self.activation = F.relu
        self.use_bn = use_bn
        self.residual = use_residual
        self.alpha = alpha
        self._io = (in_channels, hidden_channels, out_channels)
        self._opts = dict(use_weight=use_weight, use_graph=use_graph, graph_weight=graph_weight, use_source=use_source)

    def reset_parameters(self):
        for conv in self.convs:
            conv.reset_parameters()
        for bn in self.bns:
            bn.reset_parameters()
        for fc in self.fcs:
            fc.reset_parameters()

    def _cfg(self) -> dict:
        d, h, c = self._io
        o = self._opts
        return dict(in_channels=d, hidden=h, out_channels=c, num_layers=len(self.convs), alpha=float(self.alpha),
                    dropout=float(self.dropout), use_bn=bool(self.use_bn), use_residual=bool(self.residual),
                    use_weight=bool(o["use_weight"]), use_graph=bool(o["use_graph"]),
                    graph_weight=float(o["graph_weight"]), use_source=bool(o["use_source"]))

    def forward(self, data, edge_weight=None):
        x, edge_index = data.graph['node_feat'], data.graph['edge_index']
        if not x.is_cuda:
            _require_cuda("DIFFormer")
            raise RuntimeError("sgformer_b200.DIFFormer needs the dataset on a CUDA device (no CPU fallback)")
        cfg = self._cfg()
        names, tensors = self._flat()
        graph = None
        if cfg["use_graph"]:       # edge_weight only reaches gcn_conv, which runs only with use_graph (medium/difformer.py:129)
            graph = get_graph(edge_index, x.shape[0], 0, edge_weight=edge_weight)
            if edge_weight is not None:
                names, tensors = tuple(names) + (E.EDGE_WEIGHT,), list(tensors) + [edge_weight]
        return Fn.DIFFormerFn.apply(x, graph, cfg, E.precision(self.precision), self.training, names, *tensors)

    def get_attentions(self, x):
        """[layers, N, N, 1] on the kernels (engine.difformer_attentions).  The reference calls its layers without edge_index
        here, which fails whenever use_graph=True; so does this, with a clear message."""
        if self._opts["use_graph"]:
            raise ValueError("DIFFormer.get_attentions needs use_graph=False: the reference calls its layers without edge_index "
                             "(medium/difformer.py:221), so the graph term cannot be computed")
        _require_cuda("get_attentions")
        names, tensors = self._flat()
        host = not x.is_cuda
        dev = torch.device("cuda", torch.cuda.current_device()) if host else x.device
        with torch.no_grad():
            P = {n_: (t.to(dev) if host else t) for n_, t in zip(names, tensors)}
            prec = E.precision(self.precision)
            atts = E.difformer_attentions(P, self._cfg(), E.input_operand(x.to(dev), prec), prec)
            out = torch.stack([a.contiguous() for a in atts], dim=0).unsqueeze(-1)
        return out.to(x.device) if host else out
