"""Functional torch-CPU restatement of the large variant's GCN baseline (large/gnns.py:177-220) driven by its state_dict names.
gnns.GAT (large/gnns.py:272-310) is the medium GAT network (oracle/gat_oracle.py) and needs nothing of its own here."""
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from .sgformer_oracle import _batch_norm, _dropout, pyg_gcn_adjacency

Tensor = torch.Tensor


def edge_sum_adjacency(edge_index: Tensor, n: int, dtype=torch.float32) -> Tensor:
    """GCNConv(normalize=False) with no edge weight: out[col] += x[row] for every edge as given (duplicates count, no self loops
    added, no degree scaling) -> CSR A with A[col, row] = the number of (row -> col) edges."""
    row, col = edge_index[0].long(), edge_index[1].long()
    w = torch.ones(row.numel(), dtype=dtype, device=row.device)
    return torch.sparse_coo_tensor(torch.stack([col, row]), w, (n, n)).coalesce().to_sparse_csr()


def gcn_large(x: Tensor, edge_index: Tensor, sd: Dict[str, Tensor], num_layers: int, use_bn: bool, save_mem: bool,
              training: bool, dropout: float = 0.0, stats_out: Optional[dict] = None) -> Tensor:
    """gnns.GCN.forward: conv -> [BN] -> ReLU -> dropout per hidden layer, then the last conv.  Every conv is GCNConv with
    normalize = not save_mem: (x W^T), aggregated by A (save_mem) or by gcn_norm's Â, + bias."""
    n = x.shape[0]
    adj = edge_sum_adjacency(edge_index, n, x.dtype) if save_mem else pyg_gcn_adjacency(edge_index.long(), n, None, x.dtype)
    for i in range(num_layers):
        x = torch.sparse.mm(adj, x @ sd[f"convs.{i}.lin.weight"].t()) + sd[f"convs.{i}.bias"]
        if i < num_layers - 1:
            if use_bn:
                x = _batch_norm(x, sd, f"bns.{i}.", training, stats_out)
            x = _dropout(F.relu(x), dropout, training)
    return x
