"""Generate tests/golden/gat.pt from the UNMODIFIED reference's medium/models.py GAT and medium/ours.py SGFormer(gnn=GAT), with
oracle/gat_oracle.GATConv injected as models.py's `GATConv` (torch_geometric cannot be installed in the build container, so the
conv itself is the plain-torch restatement; the stack around it - input dropout, BatchNorm / ELU / dropout order, the heads *
hidden widths, the last conv's out_heads with concat=False, the branch mix - is the reference's own code):

    SGFORMER_REFERENCE=/path/to/SGFormer python tests/make_golden_gat.py

Writes only that file."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from make_golden import GOLD, synth_graph  # noqa: E402
from make_golden_difformer import _flat_dict  # noqa: E402

# (n, d, hidden, classes); gat kw = models.GAT's; graph: synth_graph options + `loops` existing self loops
GAT_CASES = {
    "h1_o1_bn": dict(n=40, d=8, h=8, c=3, gat=dict(num_layers=2, heads=1, out_heads=1, use_bn=True), graph={}),
    "h2_o2_nobn": dict(n=40, d=8, h=8, c=3, gat=dict(num_layers=3, heads=2, out_heads=2, use_bn=False), graph={}),
    "h8_o1_bn_directed": dict(n=48, d=8, h=8, c=4, gat=dict(num_layers=3, heads=8, out_heads=1, use_bn=True),
                              graph=dict(directed=True, isolated=5, dup=13, loops=6)),
    "h8_o2_nobn_directed": dict(n=48, d=8, h=8, c=4, gat=dict(num_layers=2, heads=8, out_heads=2, use_bn=False),
                                graph=dict(directed=True, isolated=4, dup=9, loops=4)),
}
# SGFormer(gnn=GAT): `sgformer` = medium/ours.py kwargs besides the GNN
SGFORMER_CASES = {
    "sgformer_add_h2_bn": dict(n=40, d=8, h=8, c=3, gat=dict(num_layers=2, heads=2, out_heads=1, use_bn=True),
                               sgformer=dict(aggregate="add", graph_weight=0.7), graph={}),
    "sgformer_cat_h8_o2_directed": dict(n=48, d=8, h=8, c=4, gat=dict(num_layers=2, heads=8, out_heads=2, use_bn=False),
                                        sgformer=dict(aggregate="cat"), graph=dict(directed=True, isolated=4, dup=9, loops=4)),
}


def _graph(n, seed, directed=False, isolated=0, dup=0, loops=0):
    ei = synth_graph(n, 3 * n, seed, directed=directed, isolated=isolated, dup=dup)
    if loops:
        ar = torch.arange(loops)
        ei = torch.cat([ei, torch.stack([ar, ar])], 1)
    return ei


def _perturb(model):
    """Move biases, BatchNorm affine parameters and running statistics off their inits."""
    with torch.no_grad():
        for nm, p_ in model.named_parameters():
            if nm.endswith("bias") or ".bns." in f".{nm}" or nm.startswith("bns."):
                p_.add_(0.1 * torch.randn_like(p_))
        for nm, b in model.named_buffers():
            if nm.endswith("running_mean"):
                b.normal_(0, 0.1)
            elif nm.endswith("running_var"):
                b.uniform_(0.5, 1.5)


def gat_cases():
    from _refload import FakeDataset, import_reference
    from oracle import gat_oracle as G
    ours, models = import_reference("medium")
    models.GATConv = G.GATConv                # the restated conv, injected where models.GAT looks it up
    out = {}
    for i, (name, sp) in enumerate({**GAT_CASES, **SGFORMER_CASES}.items()):
        torch.manual_seed(500 + i)
        # as medium/parse.py:99 builds the backbone of SGFormer: out_channels = hidden_channels
        gat = models.GAT(sp["d"], sp["h"], sp["h"] if "sgformer" in sp else sp["c"], dropout=0.0, **sp["gat"])
        if "sgformer" in sp:
            model = ours.SGFormer(sp["d"], sp["h"], sp["c"], num_layers=1, num_heads=1, alpha=0.5, dropout=0.0, use_bn=True,
                                  use_residual=True, use_weight=True, use_graph=True, gnn=gat, **sp["sgformer"])
        else:
            model = gat
        _perturb(model)
        sd = {k: v.clone() for k, v in model.state_dict().items()}
        g = torch.Generator().manual_seed(600 + i)
        x = torch.randn(sp["n"], sp["d"], generator=g)
        ei = _graph(sp["n"], 700 + i, **sp["graph"])
        model.eval()
        with torch.no_grad():
            out_eval = model(FakeDataset(x, ei)).clone()
        model.train()
        xg = x.clone().requires_grad_(True)
        out_train = model(FakeDataset(xg, ei))
        lw = torch.randn(out_train.shape, generator=g)
        (out_train * lw).sum().backward()
        grads = {k: p_.grad.clone() for k, p_ in model.named_parameters() if p_.grad is not None}
        bufs = {k: v.clone() for k, v in model.state_dict().items() if "running" in k or "num_batches" in k}
        out[name] = dict(gat=sp["gat"], sgformer=sp.get("sgformer"), in_channels=sp["d"], hidden=sp["h"], out_channels=sp["c"],
                         x=x, edge_index=ei.to(torch.int32), state_dict=_flat_dict({k: v for k, v in sd.items() if "lin_dst" not in k}),
                         loss_weight=lw, out_eval=out_eval, out_train=out_train.detach().clone(), grad_x=xg.grad.clone(),
                         grads=_flat_dict(grads), buffers_after_train=_flat_dict(bufs) if bufs else None)
    path = os.path.join(GOLD, "gat.pt")
    torch.save(out, path)
    print("gat", len(out), os.path.getsize(path), "bytes")


if __name__ == "__main__":
    gat_cases()
