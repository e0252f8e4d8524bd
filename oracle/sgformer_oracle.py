"""CPU oracle for the SGFormer encoder hot path — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference` legs may
import this module. Nothing under `sgformer_b200/` imports it; the product path has no CPU fallback.

It is a *functional* torch-CPU restatement (no nn.Module clones) of the reference's three model
variants, driven by a plain config dict and a `state_dict` that uses the reference's parameter names,
so the same weights can be loaded into the reference, the oracle and the CUDA build.

Pinning: the reference has no tests or golden vectors of its own (SURVEY.md §4, §8c), so the oracle is
pinned against *outputs of the reference itself*: `tests/make_golden.py` imports the unmodified
the reference's `{medium,large,100M}/ours.py` (through `tests/ref_shims/`), runs seeded inputs and
commits inputs/outputs/gradients under `tests/golden/`; `tests/test_oracle_golden.py` checks this file
against those fixtures (and, in the build container, `tests/test_oracle_vs_reference.py` checks it
against the live reference).  The third-party ops the reference reaches through `torch_sparse` /
`torch_geometric` are not vendored (pins: torch_sparse==0.6.10, torch_geometric==1.7.2,
`large/requirements.txt:8-10`); their published semantics are restated here and cross-checked
against scipy / fp64 einsum in `oracle/np_ref.py`.

All citations are paths in the reference repository.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

Tensor = torch.Tensor

# --------------------------------------------------------------------------------------------
# configuration
# --------------------------------------------------------------------------------------------

_DEFAULTS = dict(
    variant="large", num_heads=1, trans_num_layers=1, trans_dropout=0.5, trans_use_bn=True,
    trans_use_residual=True, trans_use_weight=True, trans_use_act=True, alpha=0.5,
    gnn_num_layers=1, gnn_dropout=0.5, gnn_use_weight=True, gnn_use_init=False, gnn_use_bn=True,
    gnn_use_residual=True, gnn_use_act=True, use_graph=True, graph_weight=0.8, aggregate="add",
)


def make_config(variant: str, in_channels: int, hidden: int, out_channels: int, **kw) -> dict:
    """Normalised config.  `variant` in {'large','100M','medium'}.

    large : large/ours.py:242-245 kwargs (trans_*/gnn_*).
    100M  : 100M/ours.py:293-316 (large + alpha).
    medium: medium/ours.py:180-181 (num_layers,num_heads,alpha,dropout,use_bn,use_residual,use_weight,
            use_graph,use_act,graph_weight,aggregate) + the injected GCN backbone
            (medium/models.py:14-41: gcn_num_layers, gcn_dropout, gcn_use_bn).
    """
    cfg = dict(_DEFAULTS)
    cfg.update(variant=variant, in_channels=in_channels, hidden=hidden, out_channels=out_channels)
    if variant == "medium":
        # medium/ours.py:183 never forwards use_act to TransConv -> always False there.
        cfg.update(trans_num_layers=kw.pop("num_layers", 2), num_heads=kw.pop("num_heads", 1),
                   alpha=kw.pop("alpha", 0.5), trans_dropout=kw.pop("dropout", 0.5),
                   trans_use_bn=kw.pop("use_bn", True), trans_use_residual=kw.pop("use_residual", True),
                   trans_use_weight=kw.pop("use_weight", True), trans_use_act=False,
                   gcn_num_layers=kw.pop("gcn_num_layers", 2), gcn_dropout=kw.pop("gcn_dropout", 0.5),
                   gcn_use_bn=kw.pop("gcn_use_bn", True))
        kw.pop("use_act", None)
    else:
        if "trans_num_heads" in kw:
            cfg["num_heads"] = kw.pop("trans_num_heads")
    for k, v in kw.items():
        if k not in cfg:
            raise KeyError(f"unknown config key {k}")
        cfg[k] = v
    if cfg["aggregate"] not in ("add", "cat"):
        raise ValueError(f"Invalid aggregate type:{cfg['aggregate']}")  # large/ours.py:258-259
    return cfg


# --------------------------------------------------------------------------------------------
# linear attention  (medium/ours.py:14-34, 100M/ours.py:12-43, inlined at large/ours.py:130-151)
# --------------------------------------------------------------------------------------------

def attention_partials(q: Tensor, k: Tensor, v: Tensor) -> Dict[str, Tensor]:
    """Pass-1 quantities in the un-normalised ("sharded") form of SURVEY Appendix A.1:
    S' = k^T v [H,M,D], z' = k^T 1 [H,M], nq2 = ||q||_F^2, nk2 = ||k||_F^2 (one scalar over [N,H,M])."""
    return dict(S=torch.einsum("lhm,lhd->hmd", k, v), z=k.sum(dim=0),
                nq2=(q * q).sum(), nk2=(k * k).sum())


def full_attention(q: Tensor, k: Tensor, v: Tensor) -> Tensor:
    """out[n,h,:] = (q~ S + N v) / (q~ z + N),  q~ = q/||q||_F, k~ = k/||k||_F, S = k~^T v, z = k~^T 1.
    N is the *query* count (medium/ours.py:18).  Returns [N,H,D]."""
    n = q.shape[0]
    qn = q / torch.linalg.vector_norm(q)            # medium/ours.py:16
    kn = k / torch.linalg.vector_norm(k)            # medium/ours.py:17
    s = torch.einsum("lhm,lhd->hmd", kn, v)         # :21
    num = torch.einsum("nhm,hmd->nhd", qn, s) + n * v   # :22-23
    z = kn.sum(dim=0)                               # :26-27 (einsum with all-ones)
    den = torch.einsum("nhm,hm->nh", qn, z) + n     # :28-33
    return num / den.unsqueeze(-1)                  # :34


def attention_matrix(q: Tensor, k: Tensor) -> Tensor:
    """Visualisation path (medium/ours.py:37-40): mean_h(q~ k~^T) / mean_h(den) -> [N,N]."""
    n = q.shape[0]
    qn = q / torch.linalg.vector_norm(q)
    kn = k / torch.linalg.vector_norm(k)
    den = torch.einsum("nhm,hm->nh", qn, kn.sum(dim=0)) + n
    att = torch.einsum("nhm,lhm->nlh", qn, kn).mean(dim=-1)
    return att / den.mean(dim=-1, keepdim=True)


def trans_conv_layer(x: Tensor, sd: Dict[str, Tensor], pfx: str, heads: int, use_weight: bool,
                     return_attn: bool = False):
    """TransConvLayer.forward (medium/ours.py:74-100, large/ours.py:121-162): Wq/Wk/(Wv) projections,
    attention, mean over heads.  use_weight=False -> V is the input itself with one head (:84)."""
    h = sd[pfx + "Wq.weight"].shape[0] // heads
    q = F.linear(x, sd[pfx + "Wq.weight"], sd[pfx + "Wq.bias"]).reshape(-1, heads, h)
    k = F.linear(x, sd[pfx + "Wk.weight"], sd[pfx + "Wk.bias"]).reshape(-1, heads, h)
    if use_weight:
        v = F.linear(x, sd[pfx + "Wv.weight"], sd[pfx + "Wv.bias"]).reshape(-1, heads, h)
    else:
        v = x.reshape(-1, 1, h)
    out = full_attention(q, k, v).mean(dim=1)
    if return_attn:
        return out, attention_matrix(q, k)
    return out


def _dropout(x: Tensor, p: float, training: bool) -> Tensor:
    return F.dropout(x, p=p, training=training)


def trans_conv(x: Tensor, sd: Dict[str, Tensor], cfg: dict, training: bool, pfx: str = "trans_conv.") -> Tensor:
    """TransConv.forward: large/ours.py:194-219 (residual = (x+prev)/2, :211),
    medium/ours.py:133-160 and 100M/ours.py:247-272 (residual = alpha*x+(1-alpha)*prev, :152 / :264)."""
    hdim = cfg["hidden"]
    p = cfg["trans_dropout"]

    def ln(t, i):
        return F.layer_norm(t, (hdim,), sd[f"{pfx}bns.{i}.weight"], sd[f"{pfx}bns.{i}.bias"], 1e-5)

    x = F.linear(x, sd[pfx + "fcs.0.weight"], sd[pfx + "fcs.0.bias"])
    if cfg["trans_use_bn"]:
        x = ln(x, 0)
    x = _dropout(F.relu(x), p, training)
    prev = x
    for i in range(cfg["trans_num_layers"]):
        a = trans_conv_layer(prev, sd, f"{pfx}convs.{i}.", cfg["num_heads"], cfg["trans_use_weight"])
        if cfg["trans_use_residual"]:
            if cfg["variant"] == "large":
                a = (a + prev) / 2.0
            else:
                a = cfg["alpha"] * a + (1.0 - cfg["alpha"]) * prev
        if cfg["trans_use_bn"]:
            a = ln(a, i + 1)
        if cfg["trans_use_act"]:
            a = F.relu(a)
        prev = _dropout(a, p, training)
    return prev


def get_attentions(x: Tensor, sd: Dict[str, Tensor], cfg: dict, pfx: str = "trans_conv.") -> Tensor:
    """TransConv.get_attentions (large/ours.py:221-238; medium/100M omit the activation, medium/ours.py:162-177)."""
    hdim = cfg["hidden"]

    def ln(t, i):
        return F.layer_norm(t, (hdim,), sd[f"{pfx}bns.{i}.weight"], sd[f"{pfx}bns.{i}.bias"], 1e-5)

    x = F.linear(x, sd[pfx + "fcs.0.weight"], sd[pfx + "fcs.0.bias"])
    if cfg["trans_use_bn"]:
        x = ln(x, 0)
    prev = F.relu(x)
    atts = []
    for i in range(cfg["trans_num_layers"]):
        a, att = trans_conv_layer(prev, sd, f"{pfx}convs.{i}.", cfg["num_heads"], cfg["trans_use_weight"], True)
        atts.append(att)
        if cfg["trans_use_residual"]:
            a = (a + prev) / 2.0 if cfg["variant"] == "large" else cfg["alpha"] * a + (1 - cfg["alpha"]) * prev
        if cfg["trans_use_bn"]:
            a = ln(a, i + 1)
        if cfg["variant"] == "large" and cfg["trans_use_act"]:
            a = F.relu(a)
        prev = a
    return torch.stack(atts, dim=0)


# --------------------------------------------------------------------------------------------
# GCN branch, large/100M  (large/ours.py:25-42, 74-94)
# --------------------------------------------------------------------------------------------

def gcn_degree_inv_sqrt(edge_index: Tensor, n: int) -> Tensor:
    """d[i] = #{e: col_e = i} (in-degree over `col`, large/ours.py:28); d^-1/2 with 0 for isolated
    nodes (== the reference's inf -> nan_to_num(…, posinf=0) path, :29-32)."""
    d = torch.bincount(edge_index[1], minlength=n).to(torch.float32)
    dinv = d.rsqrt()
    return torch.where(d > 0, dinv, torch.zeros_like(dinv))


def normalized_adjacency(edge_index: Tensor, n: int, dtype=torch.float32) -> Tensor:
    """Â as a torch CSR tensor: Â[c, r] += w_e for each edge e=(r -> c), w_e = d[c]^-1/2 d[r]^-1/2
    (large/ours.py:29-33: SparseTensor(row=col, col=row, value=w)); duplicates accumulate."""
    row, col = edge_index[0], edge_index[1]
    d = torch.bincount(col, minlength=n).to(dtype)     # the reference uses fp32; fp64 only for accuracy studies in tests
    w = (1.0 / d[col]).sqrt() * (1.0 / d[row]).sqrt()
    w = torch.nan_to_num(w, nan=0.0, posinf=0.0, neginf=0.0)
    a = torch.sparse_coo_tensor(torch.stack([col, row]), w, (n, n)).coalesce()
    return a.to_sparse_csr()


def graph_conv_layer(x: Tensor, adj: Tensor, x0: Tensor, w: Tensor, b: Tensor, use_init: bool,
                     use_weight: bool) -> Tensor:
    """GraphConvLayer.forward after Â has been built (large/ours.py:34-42)."""
    y = torch.sparse.mm(adj, x)
    if use_init:
        return F.linear(torch.cat([y, x0], dim=1), w, b)
    if use_weight:
        return F.linear(y, w, b)
    return y


def _batch_norm(x: Tensor, sd: Dict[str, Tensor], pfx: str, training: bool, stats_out: Optional[dict]) -> Tensor:
    """nn.BatchNorm1d(eps=1e-5, momentum=0.1): batch stats (biased var) in train, running stats in eval.
    `stats_out`, when given, receives the would-be updated running buffers."""
    rm, rv = sd[pfx + "running_mean"], sd[pfx + "running_var"]
    if training:
        mean = x.mean(dim=0)
        var = x.var(dim=0, unbiased=False)
        if stats_out is not None:
            n = x.shape[0]
            stats_out[pfx + "running_mean"] = 0.9 * rm + 0.1 * mean.detach()
            stats_out[pfx + "running_var"] = 0.9 * rv + 0.1 * (var.detach() * n / max(n - 1, 1))
            stats_out[pfx + "num_batches_tracked"] = sd[pfx + "num_batches_tracked"] + 1
    else:
        mean, var = rm, rv
    return (x - mean) * torch.rsqrt(var + 1e-5) * sd[pfx + "weight"] + sd[pfx + "bias"]


def graph_conv(x: Tensor, edge_index: Tensor, sd: Dict[str, Tensor], cfg: dict, training: bool,
               pfx: str = "graph_conv.", stats_out: Optional[dict] = None) -> Tensor:
    """GraphConv.forward (large/ours.py:74-94).  Quirk kept: `layer_` is appended once, so the residual
    always adds the input-MLP output x0 (:83, :92-93)."""
    n = x.shape[0]
    p = cfg["gnn_dropout"]
    adj = normalized_adjacency(edge_index, n, x.dtype)
    x = F.linear(x, sd[pfx + "fcs.0.weight"], sd[pfx + "fcs.0.bias"])
    if cfg["gnn_use_bn"]:
        x = _batch_norm(x, sd, pfx + "bns.0.", training, stats_out)
    x = _dropout(F.relu(x), p, training)
    x0 = x
    for i in range(cfg["gnn_num_layers"]):
        x = graph_conv_layer(x, adj, x0, sd[f"{pfx}convs.{i}.W.weight"], sd[f"{pfx}convs.{i}.W.bias"],
                             cfg["gnn_use_init"], cfg["gnn_use_weight"])
        if cfg["gnn_use_bn"]:
            x = _batch_norm(x, sd, f"{pfx}bns.{i + 1}.", training, stats_out)
        if cfg["gnn_use_act"]:
            x = F.relu(x)
        x = _dropout(x, p, training)
        if cfg["gnn_use_residual"]:
            x = x + x0
    return x


# --------------------------------------------------------------------------------------------
# GCN backbone, medium  (medium/models.py:14-63 on top of PyG GCNConv / gcn_norm)
# --------------------------------------------------------------------------------------------

def pyg_gcn_adjacency(edge_index: Tensor, n: int, edge_weight: Optional[Tensor] = None) -> Tensor:
    """PyG gcn_norm(add_self_loops=True, improved=False): drop existing self loops, add one unit
    self loop per node (existing self-loop weights are kept when edge_weight is given),
    deg = scatter-add of weights at `col`, w_e = deg^-1/2[row] w_e deg^-1/2[col] (inf -> 0).
    Aggregation is out[col] += w_e x[row]  ->  CSR with row index = col."""
    row, col = edge_index[0], edge_index[1]
    w = torch.ones(row.numel(), dtype=torch.float32) if edge_weight is None else edge_weight.to(torch.float32)
    keep = row != col
    loop_w = torch.ones(n, dtype=torch.float32)
    if edge_weight is not None:
        loop_w[row[~keep]] = w[~keep]
    ar = torch.arange(n, dtype=row.dtype)
    row = torch.cat([row[keep], ar])
    col = torch.cat([col[keep], ar])
    w = torch.cat([w[keep], loop_w])
    deg = torch.zeros(n, dtype=torch.float32).scatter_add_(0, col, w)
    dis = deg.pow(-0.5)
    dis = torch.where(torch.isinf(dis), torch.zeros_like(dis), dis)
    w = dis[row] * w * dis[col]
    return torch.sparse_coo_tensor(torch.stack([col, row]), w, (n, n)).coalesce().to_sparse_csr()


def gcn_medium(x: Tensor, edge_index: Tensor, sd: Dict[str, Tensor], cfg: dict, training: bool,
               pfx: str = "gnn.", edge_weight: Optional[Tensor] = None,
               stats_out: Optional[dict] = None) -> Tensor:
    """models.GCN.forward (medium/models.py:49-63): GCNConv = (x W^T) then Â·, + bias; BN/ReLU/dropout
    between layers, none after the last."""
    n = x.shape[0]
    adj = pyg_gcn_adjacency(edge_index, n, edge_weight)
    # quirk kept: the last conv is called without edge_weight (medium/models.py:62)
    adj_last = adj if edge_weight is None else pyg_gcn_adjacency(edge_index, n, None)
    nl = cfg["gcn_num_layers"]
    for i in range(nl):
        a = adj_last if i == nl - 1 else adj
        x = torch.sparse.mm(a, x @ sd[f"{pfx}convs.{i}.lin.weight"].t()) + sd[f"{pfx}convs.{i}.bias"]
        if i < nl - 1:
            if cfg["gcn_use_bn"]:
                x = _batch_norm(x, sd, f"{pfx}bns.{i}.", training, stats_out)
            x = _dropout(F.relu(x), cfg["gcn_dropout"], training)
    return x


# --------------------------------------------------------------------------------------------
# whole encoder  (large/ours.py:265-276, medium/ours.py:202-213, 100M/ours.py:359-370)
# --------------------------------------------------------------------------------------------

def sgformer_forward(cfg: dict, sd: Dict[str, Tensor], x: Tensor, edge_index: Tensor,
                     training: bool = False, edge_weight: Optional[Tensor] = None,
                     stats_out: Optional[dict] = None) -> Tensor:
    x1 = trans_conv(x, sd, cfg, training)
    if cfg["use_graph"]:
        if cfg["variant"] == "medium":
            x2 = gcn_medium(x, edge_index, sd, cfg, training, edge_weight=edge_weight, stats_out=stats_out)
        else:
            x2 = graph_conv(x, edge_index, sd, cfg, training, stats_out=stats_out)
        if cfg["aggregate"] == "add":
            gw = cfg["graph_weight"]
            h = gw * x2 + (1.0 - gw) * x1
        else:
            h = torch.cat([x1, x2], dim=1)
    else:
        h = x1
    return F.linear(h, sd["fc.weight"], sd["fc.bias"])


# --------------------------------------------------------------------------------------------
# parameter construction (default torch inits; names == reference state_dict keys, SURVEY §8b)
# --------------------------------------------------------------------------------------------

def _linear_init(out_f: int, in_f: int, gen: torch.Generator):
    bound = 1.0 / math.sqrt(in_f)          # kaiming_uniform(a=sqrt(5)) == U(-1/sqrt(fan_in), +)
    w = (torch.rand(out_f, in_f, generator=gen) * 2 - 1) * bound
    b = (torch.rand(out_f, generator=gen) * 2 - 1) * bound
    return w, b


def init_state_dict(cfg: dict, seed: int = 0) -> Dict[str, Tensor]:
    """Random parameters with the reference's names/shapes (distributionally the torch defaults;
    not bit-identical to `reset_parameters()` — parity tests copy one state_dict into all models)."""
    g = torch.Generator().manual_seed(seed)
    h, d, c, heads = cfg["hidden"], cfg["in_channels"], cfg["out_channels"], cfg["num_heads"]
    sd: Dict[str, Tensor] = {}

    def lin(name, o, i):
        sd[name + ".weight"], sd[name + ".bias"] = _linear_init(o, i, g)

    lin("trans_conv.fcs.0", h, d)
    for i in range(cfg["trans_num_layers"] + 1):
        sd[f"trans_conv.bns.{i}.weight"] = 1.0 + 0.1 * torch.randn(h, generator=g)
        sd[f"trans_conv.bns.{i}.bias"] = 0.1 * torch.randn(h, generator=g)
    for i in range(cfg["trans_num_layers"]):
        lin(f"trans_conv.convs.{i}.Wk", h * heads, h)
        lin(f"trans_conv.convs.{i}.Wq", h * heads, h)
        if cfg["trans_use_weight"]:
            lin(f"trans_conv.convs.{i}.Wv", h * heads, h)

    def bn(name):
        sd[name + ".weight"] = 1.0 + 0.1 * torch.randn(h, generator=g)
        sd[name + ".bias"] = 0.1 * torch.randn(h, generator=g)
        sd[name + ".running_mean"] = 0.1 * torch.randn(h, generator=g)
        sd[name + ".running_var"] = 1.0 + 0.2 * torch.rand(h, generator=g)
        sd[name + ".num_batches_tracked"] = torch.zeros((), dtype=torch.long)

    if cfg["variant"] == "medium":
        nl = cfg["gcn_num_layers"]
        dims = [d] + [h] * nl
        for i in range(nl):
            a = math.sqrt(6.0 / (dims[i] + dims[i + 1]))
            sd[f"gnn.convs.{i}.lin.weight"] = (torch.rand(dims[i + 1], dims[i], generator=g) * 2 - 1) * a
            sd[f"gnn.convs.{i}.bias"] = 0.1 * torch.randn(dims[i + 1], generator=g)
        for i in range(nl - 1):
            bn(f"gnn.bns.{i}")
    else:
        lin("graph_conv.fcs.0", h, d)
        bn("graph_conv.bns.0")
        for i in range(cfg["gnn_num_layers"]):
            lin(f"graph_conv.convs.{i}.W", h, 2 * h if cfg["gnn_use_init"] else h)
            bn(f"graph_conv.bns.{i + 1}")
    lin("fc", c, 2 * h if cfg["aggregate"] == "cat" else h)
    return sd
