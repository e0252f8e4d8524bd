"""Generate tests/golden/large_gnns.pt from the UNMODIFIED reference's large/gnns.py GCN, imported through tests/ref_shims (whose
GCNConv honours `normalize`, so both `save_mem` settings run the reference's own stack):

    SGFORMER_REFERENCE=/path/to/SGFormer python tests/make_golden_large_gnns.py

Writes only that file."""
import importlib
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from make_golden import GOLD, synth_graph  # noqa: E402
from make_golden_difformer import _flat_dict  # noqa: E402
from make_golden_gat import _perturb  # noqa: E402

# (n, d, hidden, classes); gcn kw = gnns.GCN's; graph: synth_graph options, `driver_loops` = large/main.py:78-79 (remove_self_loops
# + add_self_loops: exactly one loop per node); without them the isolated nodes have no in-edges (zero rows of the sum)
CASES = {
    "savemem_l2_bn": dict(n=40, d=8, h=16, c=3, gcn=dict(num_layers=2, use_bn=True, save_mem=True),
                          graph=dict(directed=True, isolated=4, dup=11, driver_loops=True)),
    "savemem_l3_nobn": dict(n=48, d=12, h=16, c=8, gcn=dict(num_layers=3, use_bn=False, save_mem=True),
                            graph=dict(directed=True, isolated=5, dup=9, driver_loops=False)),
    "savemem_l3_bn_undirected": dict(n=48, d=8, h=24, c=5, gcn=dict(num_layers=3, use_bn=True, save_mem=True),
                                     graph=dict(isolated=3, dup=7, driver_loops=True)),
    "norm_l2_nobn": dict(n=40, d=8, h=16, c=3, gcn=dict(num_layers=2, use_bn=False, save_mem=False),
                         graph=dict(directed=True, isolated=4, dup=11, driver_loops=True)),
    "norm_l3_bn": dict(n=48, d=12, h=16, c=8, gcn=dict(num_layers=3, use_bn=True, save_mem=False),
                       graph=dict(directed=True, isolated=5, dup=9, driver_loops=False)),
}


def import_gnns():
    from _refload import REF_ROOT, SHIMS
    d = os.path.join(REF_ROOT, "large")
    sys.modules.pop("gnns", None)
    saved = list(sys.path)
    sys.path[:0] = [SHIMS, d]
    try:
        return importlib.import_module("gnns")
    finally:
        sys.path[:] = saved
        sys.modules.pop("gnns", None)


def graph(n, seed, directed=False, isolated=0, dup=0, driver_loops=False):
    ei = synth_graph(n, 3 * n, seed, directed=directed, isolated=isolated, dup=dup)
    if driver_loops:
        ei = ei[:, ei[0] != ei[1]]
        ar = torch.arange(n)
        ei = torch.cat([ei, torch.stack([ar, ar])], 1)
    return ei


# constructor calls whose parameter trees the native modules must reproduce
TREE_CASES = {"GCN": [dict(num_layers=2), dict(num_layers=3, use_bn=False), dict(num_layers=3, save_mem=False)],
              "GAT": [dict(num_layers=2), dict(num_layers=3, use_bn=True, heads=4, out_heads=2)]}


def reference_trees(gnns):
    """{class: (constructor signature, [(kwargs, {state_dict key: shape}, [conv.normalize])])} of gnns.GCN / gnns.GAT(12, 16, 5,
    **kwargs); GAT with oracle/gat_oracle.GATConv as its conv (the shims' GATConv is a stub), lin_dst (= lin_src) left out."""
    import inspect
    from oracle import gat_oracle
    gnns.GATConv = gat_oracle.GATConv
    out = {}
    for cls, kws in TREE_CASES.items():
        rows = []
        for kw in kws:
            m = getattr(gnns, cls)(12, 16, 5, **kw)
            rows.append((kw, {k: tuple(v.shape) for k, v in m.state_dict().items() if "lin_dst" not in k},
                         [getattr(c, "normalize", None) for c in m.convs]))
        out[cls] = (str(inspect.signature(getattr(gnns, cls).__init__)), rows)
    return out


def cases():
    gnns = import_gnns()
    out = {}
    for i, (name, sp) in enumerate(CASES.items()):
        torch.manual_seed(800 + i)
        model = gnns.GCN(sp["d"], sp["h"], sp["c"], dropout=0.0, **sp["gcn"])
        _perturb(model)
        sd = {k: v.clone() for k, v in model.state_dict().items()}
        g = torch.Generator().manual_seed(900 + i)
        x = torch.randn(sp["n"], sp["d"], generator=g)
        ei = graph(sp["n"], 1000 + i, **sp["graph"])
        model.eval()
        with torch.no_grad():
            out_eval = model(x, ei).clone()
        model.train()
        xg = x.clone().requires_grad_(True)
        out_train = model(xg, ei)
        lw = torch.randn(out_train.shape, generator=g)
        (out_train * lw).sum().backward()
        grads = {k: p_.grad.clone() for k, p_ in model.named_parameters() if p_.grad is not None}
        bufs = {k: v.clone() for k, v in model.state_dict().items() if "running" in k or "num_batches" in k}
        out[name] = dict(gcn=sp["gcn"], in_channels=sp["d"], hidden=sp["h"], out_channels=sp["c"], x=x,
                         edge_index=ei.to(torch.int32), state_dict=_flat_dict(sd), loss_weight=lw, out_eval=out_eval,
                         out_train=out_train.detach().clone(), grad_x=xg.grad.clone(), grads=_flat_dict(grads),
                         buffers_after_train=_flat_dict(bufs) if bufs else None)
    out["__trees__"] = reference_trees(gnns)
    path = os.path.join(GOLD, "large_gnns.pt")
    torch.save(out, path)
    print("large_gnns", len(out), os.path.getsize(path), "bytes")


if __name__ == "__main__":
    cases()
