"""Native `GCN` and `GAT` with the constructor signatures, attribute trees and state_dict keys of the reference's large/gnns.py
(:177-220 and :272-310), the baselines `--method gcn|gat` builds in large/parse.py.  `python -m sgformer_b200.launch --variant large
--native-backbones` makes parse.py resolve to them.

`GCN` keeps gnns.GCN's `save_mem` switch: True (its default, and what parse.py passes) makes every conv GCNConv(normalize=False),
a plain sum over the edges as given (the drivers add one self loop per node beforehand, large/main.py:78-79), which runs on the
unscaled SpMM (DESIGN.md §4.11); False makes them normalize=True, exactly the medium GCNConv (gcn_norm), which runs on the medium
schedule.  `GAT` is the medium native GAT (same kernels, limits and errors) with gnns.GAT's `forward(x, edge_index)`.

A new edge_index (the mini-batch driver's per-batch `subgraph`) builds a new CSR; a repeated one hits the graph cache.  CPU inputs
(large/eval.py:35-65 `evaluate_large(device="cpu")`) are computed on cuda:0 with temporary device copies of the parameters and the
logits come back to the host."""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import engine as E
from . import functional as Fn
from . import medium as M
from .config import make_config
from .graph import get_graph
from .modules import _Base, _require_cuda

__all__ = ["GCN", "GAT", "GCNConv"]


def _on_host(module, name: str, run, x, edge_index):
    """Inference on host tensors: run(x, edge_index, tensors) on the GPU with device copies of `tensors`, result to the host."""
    _require_cuda(f"{name}.forward")
    if torch.is_grad_enabled() and any(p.requires_grad for p in module.parameters()):
        raise RuntimeError(f"sgformer_b200.{name}: training needs the model and inputs on a CUDA device (no CPU fallback)")
    dev = torch.device("cuda", torch.cuda.current_device())
    with torch.no_grad():
        return run(x.to(dev), edge_index.to(dev), lambda ts: [t.to(dev) for t in ts]).cpu()


class GCNConv(M.GCNConv):
    """PyG GCNConv parameter container (`lin.weight` [out, in], `bias`) that records `normalize`, as gnns.GCN sets it."""

    def __init__(self, in_channels, out_channels, cached=False, normalize=True, **kw):
        super().__init__(in_channels, out_channels, cached=cached, **kw)
        self.normalize = normalize


class GCN(_Base):
    """gnns.GCN (large/gnns.py:177-220): `num_layers` GCNConv(normalize=not save_mem), BatchNorm?/ReLU/dropout between them."""

    def __init__(self, in_channels, hidden_channels, out_channels, num_layers=2, dropout=0.5, save_mem=True, use_bn=True):
        super().__init__()
        self.convs = nn.ModuleList()
        self.convs.append(GCNConv(in_channels, hidden_channels, cached=not save_mem, normalize=not save_mem))
        self.bns = nn.ModuleList()
        self.bns.append(nn.BatchNorm1d(hidden_channels))
        for _ in range(num_layers - 2):
            self.convs.append(GCNConv(hidden_channels, hidden_channels, cached=not save_mem, normalize=not save_mem))
            self.bns.append(nn.BatchNorm1d(hidden_channels))
        self.convs.append(GCNConv(hidden_channels, out_channels, cached=not save_mem, normalize=not save_mem))
        self.dropout = dropout
        self.activation = F.relu
        self.use_bn = use_bn

    def reset_parameters(self):
        for conv in self.convs:
            conv.reset_parameters()
        for bn in self.bns:
            bn.reset_parameters()

    def forward(self, x, edge_index):
        names, tensors = M._gcn_flat(self, "")
        if not x.is_cuda:
            return _on_host(self, "GCN", lambda xd, ed, to_dev: self._run(xd, ed, names, to_dev(tensors)), x, edge_index)
        return self._run(x, edge_index, names, tensors)

    def _run(self, x, edge_index, names, tensors):
        norm = {bool(c.normalize) for c in self.convs}
        if len(norm) != 1:
            raise NotImplementedError("sgformer_b200.GCN: every conv must have the same `normalize` (as save_mem sets it)")
        norm = norm.pop()
        prec = E.precision(self.precision)
        # the row kernels move rows in 16-byte chunks: a last conv whose width (the class count, e.g. 2 on pokec) is not a multiple
        # of 4 (fp32) / 8 (bf16) runs on zero rows of weight and bias; its extra output columns are zero and are dropped
        c = self.convs[-1].out_channels
        cp = -(-c // (8 if prec.name == "bf16" else 4)) * (8 if prec.name == "bf16" else 4)
        if cp != c:
            tensors = list(tensors)
            li = 2 * (len(self.convs) - 1)
            tensors[li] = F.pad(tensors[li], (0, 0, 0, cp - c))
            tensors[li + 1] = F.pad(tensors[li + 1], (0, cp - c))
        cfg = make_config("large", x.shape[1], self.convs[0].out_channels, cp, gcn_num_layers=len(self.convs),
                          gcn_dropout=float(self.dropout), gcn_use_bn=bool(self.use_bn), gcn_normalize=norm)
        graph = get_graph(edge_index, x.shape[0], 1 if norm else 0)
        out = Fn.GraphBranchFn.apply(x, graph, cfg, prec, self.training, "gcn", "", names, *tensors)
        return out[:, :c] if cp != c else out


class GAT(M.GAT):
    """gnns.GAT (large/gnns.py:272-310): the medium native GAT (medium/models.py:116-155 is the same network) called as
    `forward(x, edge_index)`."""

    def forward(self, x, edge_index):
        if not x.is_cuda:
            names, tensors = M._gat_flat(self, "")
            return _on_host(self, "GAT", lambda xd, ed, to_dev: self._run(xd, ed, names, to_dev(tensors)), x, edge_index)
        return self._run(x, edge_index)
