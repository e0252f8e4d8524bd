"""Functional torch-CPU restatement of the medium variant's JKNet baseline, models.GCNJK (medium/models.py:157-205), driven by its
state_dict names, in any float dtype (fp64 for the accuracy references).  The conv is the GCN oracle's (gcn_norm's Â, no edge
weight); JumpingKnowledge is PyG's 'max' (torch.stack(xs, -1).max(-1)[0]: the gradient goes to the first maximal layer) and 'cat'
(torch.cat(xs, -1))."""
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

from .sgformer_oracle import _batch_norm, pyg_gcn_adjacency, trans_conv

Tensor = torch.Tensor


def _dropout(x: Tensor, p: float, training: bool) -> Tensor:
    return F.dropout(x, p=p, training=training)


def jumping_knowledge(xs: List[Tensor], mode: str) -> Tensor:
    if mode == "max":
        return torch.stack(xs, dim=-1).max(dim=-1)[0]
    if mode == "cat":
        return torch.cat(xs, dim=-1)
    raise ValueError(f"unsupported JumpingKnowledge mode {mode!r}")


def gcnjk(x: Tensor, edge_index: Tensor, sd: Dict[str, Tensor], num_convs: int, jk: str, training: bool, dropout: float = 0.0,
          pfx: str = "", stats_out: Optional[dict] = None, xs_out: Optional[list] = None) -> Tensor:
    """GCNJK.forward: conv -> BN -> ReLU -> (into xs) -> dropout per conv but the last; the last conv into xs; JK; final_project.
    `xs_out`, when given, receives the layers' JK inputs."""
    adj = pyg_gcn_adjacency(edge_index.long(), x.shape[0], None, x.dtype)
    xs = []
    for i in range(num_convs):
        x = torch.sparse.mm(adj, x @ sd[f"{pfx}convs.{i}.lin.weight"].t()) + sd[f"{pfx}convs.{i}.bias"]
        if i < num_convs - 1:
            x = F.relu(_batch_norm(x, sd, f"{pfx}bns.{i}.", training, stats_out))
            xs.append(x)
            x = _dropout(x, dropout, training)
        else:
            xs.append(x)
    if xs_out is not None:
        xs_out.extend(xs)
    return F.linear(jumping_knowledge(xs, jk), sd[f"{pfx}final_project.weight"], sd[f"{pfx}final_project.bias"])


def sgformer_gcnjk(cfg: dict, sd: Dict[str, Tensor], x: Tensor, edge_index: Tensor, training: bool = False,
                   stats_out: Optional[dict] = None) -> Tensor:
    """medium SGFormer.forward (medium/ours.py:202-213) with gnn = GCNJK(d, h, h): cfg as sgformer_oracle's plus gcn_num_layers
    (the conv count), gcn_dropout and gcn_jk."""
    x1 = trans_conv(x, sd, cfg, training)
    x2 = gcnjk(x, edge_index, sd, cfg["gcn_num_layers"], cfg["gcn_jk"], training, cfg["gcn_dropout"], "gnn.", stats_out)
    if cfg["aggregate"] == "add":
        gw = cfg["graph_weight"]
        h = gw * x2 + (1.0 - gw) * x1
    else:
        h = torch.cat([x1, x2], dim=1)
    return F.linear(h, sd["fc.weight"], sd["fc.bias"])
