"""Plain-torch restatement of PyG's GATConv as medium/models.py:116-155 uses it (defaults: negative_slope 0.2, add_self_loops,
bias, no edge features), and of models.GAT on top of it.  Runs on any device and dtype (fp64 on the CPU for references).

Parity with torch_geometric itself is not pinned here (it cannot be installed where the fixtures are made); this module states the
semantics the kernels implement:
  x' = x W^T viewed [N, H, C];  a_src = <x', att_src>, a_dst = <x', att_dst>  per head;
  edges = remove_self_loops(edge_index) + one (i, i) per node (duplicates kept);
  e_ij = leaky_relu(a_src[j] + a_dst[i], 0.2);  alpha = softmax of e over the in-edges of i;  alpha = dropout(alpha) in training;
  out_i = sum_j alpha_ij x'_j  -> concat [N, H*C] or head mean [N, C];  + bias."""
import math
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

Tensor = torch.Tensor


def gat_edges(edge_index: Tensor, n: int) -> Tensor:
    """remove_self_loops then add_self_loops (num_nodes = n): [2, E'] (source row 0, target row 1)."""
    ei = edge_index[:, edge_index[0] != edge_index[1]]
    loop = torch.arange(n, dtype=ei.dtype, device=ei.device)
    return torch.cat([ei, torch.stack([loop, loop])], dim=1)


def _glorot(t: Tensor):
    a = math.sqrt(6.0 / (t.size(-2) + t.size(-1)))
    with torch.no_grad():
        t.uniform_(-a, a)


class GATConv(nn.Module):
    """PyG 2.0-2.3 GATConv (in_channels: int) with the same parameter names: lin_src (= lin_dst), att_src, att_dst, bias.
    `edge_factor` (forward keyword, [E', H]): multiplies alpha instead of drawing F.dropout (replays a kernel's mask)."""

    def __init__(self, in_channels, out_channels, heads=1, concat=True, negative_slope=0.2, dropout=0.0, add_self_loops=True,
                 bias=True, **kw):
        super().__init__()
        assert add_self_loops and bias and kw.get("edge_dim") is None
        self.in_channels, self.out_channels, self.heads, self.concat = in_channels, out_channels, heads, concat
        self.negative_slope, self.dropout = negative_slope, dropout
        self.lin_src = nn.Linear(in_channels, heads * out_channels, bias=False)
        self.lin_dst = self.lin_src
        self.att_src = nn.Parameter(torch.empty(1, heads, out_channels))
        self.att_dst = nn.Parameter(torch.empty(1, heads, out_channels))
        self.bias = nn.Parameter(torch.empty(heads * out_channels if concat else out_channels))
        self.reset_parameters()

    def reset_parameters(self):
        _glorot(self.lin_src.weight)
        _glorot(self.att_src)
        _glorot(self.att_dst)
        nn.init.zeros_(self.bias)

    def forward(self, x: Tensor, edge_index: Tensor, edge_factor: Optional[Tensor] = None) -> Tensor:
        n = x.shape[0]
        H, C = self.heads, self.out_channels
        xp = self.lin_src(x).view(n, H, C)
        a_s = (xp * self.att_src).sum(-1)
        a_d = (xp * self.att_dst).sum(-1)
        src, dst = gat_edges(edge_index, n)
        e = F.leaky_relu(a_s[src] + a_d[dst], self.negative_slope)
        m = torch.full((n, H), -math.inf, dtype=e.dtype, device=e.device)
        m = m.scatter_reduce(0, dst[:, None].expand_as(e), e, "amax", include_self=True)
        ex = (e - m[dst]).exp()
        s = torch.zeros((n, H), dtype=e.dtype, device=e.device).index_add(0, dst, ex)
        alpha = ex / s[dst]
        if edge_factor is not None:
            alpha = alpha * edge_factor
        else:
            alpha = F.dropout(alpha, p=self.dropout, training=self.training)
        out = torch.zeros((n, H, C), dtype=xp.dtype, device=xp.device).index_add(0, dst, alpha[..., None] * xp[src])
        out = out.reshape(n, H * C) if self.concat else out.mean(dim=1)
        return out + self.bias


class GAT(nn.Module):
    """models.GAT (medium/models.py:116-155) over the GATConv above."""

    def __init__(self, in_channels, hidden_channels, out_channels, num_layers=2, dropout=0.5, use_bn=False, heads=2, out_heads=1):
        super().__init__()
        self.convs = nn.ModuleList([GATConv(in_channels, hidden_channels, dropout=dropout, heads=heads, concat=True)])
        self.bns = nn.ModuleList([nn.BatchNorm1d(hidden_channels * heads)])
        for _ in range(num_layers - 2):
            self.convs.append(GATConv(hidden_channels * heads, hidden_channels, dropout=dropout, heads=heads, concat=True))
            self.bns.append(nn.BatchNorm1d(hidden_channels * heads))
        self.convs.append(GATConv(hidden_channels * heads, out_channels, dropout=dropout, heads=out_heads, concat=False))
        self.dropout = dropout
        self.use_bn = use_bn

    def forward(self, data):
        x, ei = data.graph['node_feat'], data.graph['edge_index']
        x = F.dropout(x, p=self.dropout, training=self.training)
        for i, conv in enumerate(self.convs[:-1]):
            x = conv(x, ei)
            if self.use_bn:
                x = self.bns[i](x)
            x = F.elu(x)
            x = F.dropout(x, p=self.dropout, training=self.training)
        return self.convs[-1](x, ei)
