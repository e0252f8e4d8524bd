"""Generate tests/golden/gcn_weighted.pt from the UNMODIFIED reference (medium/models.py GCN, medium/ours.py SGFormer and
medium/difformer.py DIFFormer through tests/ref_shims) on weighted graphs (run where the reference checkout exists):

    SGFORMER_REFERENCE=/path/to/SGFormer python tests/make_golden_weighted.py

Writes only that file.  Per case: inputs, state_dict, eval logits, train logits, parameter gradients, edge_weight.grad of
sum(out_train * loss_weight), and the BatchNorm buffers after the train step."""
import importlib
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from make_golden import GOLD  # noqa: E402
from make_golden_difformer import _flat_dict  # noqa: E402


def weighted_graph(n, e, seed, directed=True, sym_asym=False):
    """Random weighted edge list over nodes 0..n-2 (node n-1 isolated) with duplicate edges, zero-weight edges, and self loops:
    node 0 none, node 1 one, node 2 two of different weights.  sym_asym: every edge in both directions (symmetric pattern) with
    independently drawn weights per direction."""
    g = torch.Generator().manual_seed(seed)
    hi = n - 1
    src = torch.randint(3, hi, (e,), generator=g)
    dst = torch.randint(3, hi, (e,), generator=g)
    keep = src != dst
    src, dst = src[keep], dst[keep]
    src = torch.cat([src, torch.tensor([0, 4, 1, 2, 5, 2])])
    dst = torch.cat([dst, torch.tensor([4, 0, 1, 2, 1, 2])])        # loops: (1,1) once, (2,2) twice
    if sym_asym:
        src, dst = torch.cat([src, dst]), torch.cat([dst, src])
    ei = torch.stack([src, dst])
    ei = torch.cat([ei, ei[:, :7]], 1)                              # duplicates
    perm = torch.randperm(ei.shape[1], generator=g)
    ei = ei[:, perm].contiguous()
    w = 0.2 + 1.8 * torch.rand(ei.shape[1], generator=g)
    w[torch.randperm(ei.shape[1], generator=g)[:5]] = 0.0           # zero-weight edges
    return ei, w


class Data:
    def __init__(self, x, ei, w):
        self.graph = {"node_feat": x, "edge_index": ei, "edge_weight": w, "num_nodes": x.shape[0]}


# the standalone GCN's last layer is out_channels wide: a multiple of 8 runs in both precisions
CASES = {
    "gcn_directed": dict(kind="gcn", n=40, d=8, h=16, c=8, graph=dict(), kw=dict(num_layers=3)),
    "gcn_sym_asym": dict(kind="gcn", n=40, d=8, h=16, c=8, graph=dict(sym_asym=True), kw=dict(num_layers=2)),
    "gcn_no_bn": dict(kind="gcn", n=36, d=8, h=16, c=8, graph=dict(), kw=dict(num_layers=3, use_bn=False)),
    "sgformer_add": dict(kind="sgformer", n=40, d=8, h=16, c=5, graph=dict(), kw=dict(aggregate="add", gcn_layers=3)),
    "sgformer_cat": dict(kind="sgformer", n=40, d=8, h=16, c=5, graph=dict(sym_asym=True), kw=dict(aggregate="cat", gcn_layers=2)),
    "difformer": dict(kind="difformer", n=40, d=8, h=16, c=5, graph=dict(), kw=dict()),
    "difformer_sym_asym": dict(kind="difformer", n=40, d=8, h=16, c=4, graph=dict(sym_asym=True), kw=dict(graph_weight=0.3)),
}


def _import(module):
    from _refload import REF_ROOT, SHIMS
    for name in ("ours", "models", "difformer"):
        sys.modules.pop(name, None)
    saved = list(sys.path)
    sys.path[:0] = [SHIMS, os.path.join(REF_ROOT, "medium")]
    try:
        return importlib.import_module(module)
    finally:
        sys.path[:] = saved
        for name in ("ours", "models", "difformer"):
            sys.modules.pop(name, None)


def build(kind, sp):
    kw = sp["kw"]
    if kind == "gcn":
        return _import("models").GCN(sp["d"], sp["h"], sp["c"], dropout=0.0, **kw)
    if kind == "sgformer":
        gnn = _import("models").GCN(sp["d"], sp["h"], sp["h"], num_layers=kw["gcn_layers"], dropout=0.0)
        return _import("ours").SGFormer(sp["d"], sp["h"], sp["c"], num_layers=1, alpha=0.5, dropout=0.0, use_residual=True,
                                        graph_weight=0.7, gnn=gnn, aggregate=kw["aggregate"])
    return _import("difformer").DIFFormer(sp["d"], sp["h"], sp["c"], num_layers=2, dropout=0.0, **kw)


def run(kind, model, x, ei, w):
    if kind == "difformer":
        return model(Data(x, ei, None), w)
    return model(Data(x, ei, w))


def weighted_cases():
    out = {}
    for i, (name, sp) in enumerate(CASES.items()):
        torch.manual_seed(700 + i)
        kind = sp["kind"]
        model = build(kind, sp)
        with torch.no_grad():              # move the BatchNorm / LayerNorm affine parameters off 1 / 0
            for nm, p_ in model.named_parameters():
                if "bns." in nm:
                    p_.add_(0.1 * torch.randn_like(p_))
        sd = {k: v.clone() for k, v in model.state_dict().items()}
        g = torch.Generator().manual_seed(800 + i)
        x = torch.randn(sp["n"], sp["d"], generator=g)
        ei, w = weighted_graph(sp["n"], 3 * sp["n"], 900 + i, **sp["graph"])
        lw = torch.randn(sp["n"], sp["c"], generator=g)
        model.eval()
        with torch.no_grad():
            out_eval = run(kind, model, x, ei, w).clone()
        model.train()
        wg = w.clone().requires_grad_(True)
        out_train = run(kind, model, x, ei, wg)
        (out_train * lw).sum().backward()
        grads = {k: p_.grad.clone() for k, p_ in model.named_parameters() if p_.grad is not None}
        buffers = {k: v.clone() for k, v in model.state_dict().items() if "running_" in k}
        out[name] = dict(kind=kind, kw=sp["kw"], in_channels=sp["d"], hidden=sp["h"], out_channels=sp["c"], x=x, edge_index=ei,
                         edge_weight=w, state_dict=_flat_dict(sd), loss_weight=lw, out_eval=out_eval,
                         out_train=out_train.detach().clone(), grads=_flat_dict(grads), ew_grad=wg.grad.clone(),
                         buffers=_flat_dict(buffers) if buffers else None)
    path = os.path.join(GOLD, "gcn_weighted.pt")
    torch.save(out, path)
    print("gcn_weighted", len(out), os.path.getsize(path), "bytes")


if __name__ == "__main__":
    weighted_cases()
