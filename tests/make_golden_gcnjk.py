"""Generate tests/golden/gcnjk.pt from the UNMODIFIED reference's medium/models.py GCNJK, imported through tests/ref_shims:

    SGFORMER_REFERENCE=/path/to/SGFormer python tests/make_golden_gcnjk.py

The shims' JumpingKnowledge is an import-only stub, so this script puts a restatement of PyG's 'max' / 'cat' modes in its place
in the imported `models` module (the shim files stay as they are).  Writes only that file."""
import copy
import inspect
import os
import sys

import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from make_golden import GOLD, synth_graph  # noqa: E402
from make_golden_difformer import _flat_dict  # noqa: E402
from make_golden_gat import _perturb  # noqa: E402

# (n, d, hidden, classes, num_layers, jk_type); graphs: directed, isolated nodes, duplicate edges, existing self loops
CASES = {
    "max_l2": dict(n=40, d=8, h=16, c=3, num_layers=2, jk="max", graph=dict(directed=True, isolated=4, dup=11)),
    "max_l3": dict(n=48, d=12, h=16, c=5, num_layers=3, jk="max", graph=dict(isolated=3, dup=7)),
    "max_l4": dict(n=44, d=8, h=24, c=4, num_layers=4, jk="max", graph=dict(directed=True, isolated=5, dup=9)),
    "cat_l2": dict(n=40, d=8, h=16, c=3, num_layers=2, jk="cat", graph=dict(directed=True, isolated=4, dup=11)),
    "cat_l3": dict(n=48, d=12, h=16, c=6, num_layers=3, jk="cat", graph=dict(isolated=3, dup=7)),
    "cat_l4": dict(n=44, d=8, h=24, c=4, num_layers=4, jk="cat", graph=dict(directed=True, isolated=5, dup=9)),
}


class JumpingKnowledge(nn.Module):
    """PyG's JumpingKnowledge(mode, channels, num_layers) in 'max' / 'cat' mode (no parameters)."""

    def __init__(self, mode, channels=None, num_layers=None):
        super().__init__()
        self.mode = mode.lower()
        assert self.mode in ("cat", "max"), self.mode

    def reset_parameters(self):
        pass

    def forward(self, xs):
        if self.mode == "cat":
            return torch.cat(xs, dim=-1)
        return torch.stack(xs, dim=-1).max(dim=-1)[0]


class _Args:
    """The parse.py arguments parse_method reads for --method gcnjk / --method ours --backbone gcnjk."""
    hidden_channels, num_layers, dropout = 16, 3, 0.5
    ours_layers, alpha, ours_dropout, num_heads, use_bn, ours_use_residual, use_graph = 1, 0.5, 0.3, 1, True, True, True
    ours_use_weight, ours_use_act, graph_weight, aggregate, backbone = True, False, 0.8, "add", "gcnjk"


def import_models():
    from _refload import import_reference
    ours, models = import_reference("medium")
    models.JumpingKnowledge = JumpingKnowledge
    return ours, models


def reference_trees(ours, models):
    """Constructor signature, and ([state_dict key], [parameter name] in order) of GCNJK as parse.py builds it for --method gcnjk
    (d = 12, c = 5) and of SGFormer with --backbone gcnjk."""
    a = _Args()
    gj = models.GCNJK(in_channels=12, hidden_channels=a.hidden_channels, out_channels=5, num_layers=a.num_layers, dropout=a.dropout)
    gnn = models.GCNJK(in_channels=12, hidden_channels=a.hidden_channels, out_channels=a.hidden_channels, num_layers=a.num_layers,
                       dropout=a.dropout)
    sg = ours.SGFormer(12, a.hidden_channels, 5, num_layers=a.ours_layers, alpha=a.alpha, dropout=a.ours_dropout,
                       num_heads=a.num_heads, use_bn=a.use_bn, use_residual=a.ours_use_residual, use_graph=a.use_graph,
                       use_weight=a.ours_use_weight, use_act=a.ours_use_act, graph_weight=a.graph_weight, gnn=gnn,
                       aggregate=a.aggregate)
    cat = models.GCNJK(12, 16, 5, num_layers=2, jk_type="cat")

    def tree(m):
        return list(m.state_dict().keys()), [k for k, _ in m.named_parameters()], {k: tuple(v.shape) for k, v in m.state_dict().items()}

    return dict(signature=str(inspect.signature(models.GCNJK.__init__)), method=tree(gj), backbone=tree(sg), cat_l2=tree(cat),
                args=dict(hidden=a.hidden_channels, num_layers=a.num_layers, dropout=a.dropout))


def run(model, x, ei, lw):
    """eval logits, then one training forward / backward of sum(out * lw): logits, parameter and input gradients, BN buffers."""
    data = type("D", (), {})()
    model.eval()
    data.graph = {"node_feat": x, "edge_index": ei, "num_nodes": x.shape[0]}
    with torch.no_grad():
        out_eval = model(data).clone()
    model.train()
    xg = x.clone().requires_grad_(True)
    data.graph = {"node_feat": xg, "edge_index": ei, "num_nodes": x.shape[0]}
    out_train = model(data)
    (out_train * lw).sum().backward()
    grads = {k: p_.grad.clone() for k, p_ in model.named_parameters() if p_.grad is not None}
    bufs = {k: v.clone() for k, v in model.state_dict().items() if "running" in k or "num_batches" in k}
    return dict(out_eval=out_eval, out_train=out_train.detach().clone(), grad_x=xg.grad.clone(), grads=_flat(grads, x.dtype),
                buffers_after_train=_flat(bufs, x.dtype))


def _flat(d, dtype):
    """_flat_dict in `dtype` (the fp64 run keeps its precision)."""
    f = _flat_dict(d)
    f["flat"] = torch.cat([t.reshape(-1).to(dtype) for t in d.values()])
    return f


def cases():
    ours, models = import_models()
    out = {}
    for i, (name, sp) in enumerate(CASES.items()):
        torch.manual_seed(1200 + i)
        model = models.GCNJK(sp["d"], sp["h"], sp["c"], num_layers=sp["num_layers"], dropout=0.0, jk_type=sp["jk"])
        _perturb(model)
        sd = {k: v.clone() for k, v in model.state_dict().items()}
        g = torch.Generator().manual_seed(1300 + i)
        x = torch.randn(sp["n"], sp["d"], generator=g)
        ei = synth_graph(sp["n"], 3 * sp["n"], 1400 + i, **sp["graph"])
        ar = torch.arange(0, sp["n"] - sp["graph"]["isolated"], 5)
        ei = torch.cat([ei, torch.stack([ar, ar])], 1)                   # some existing self loops
        lw = torch.randn(sp["n"], sp["c"], generator=g)
        case = dict(num_layers=sp["num_layers"], jk=sp["jk"], in_channels=sp["d"], hidden=sp["h"], out_channels=sp["c"], x=x,
                    edge_index=ei.to(torch.int32), state_dict=_flat_dict(sd), loss_weight=lw)
        for dtype, sfx in ((torch.float32, ""), (torch.float64, "64")):     # the reference in fp32, and in fp64 for the fp64 oracle
            m = copy.deepcopy(model).to(dtype)
            case.update({k + sfx: v for k, v in run(m, x.to(dtype), ei, lw.to(dtype)).items()})
        out[name] = case
    out["__trees__"] = reference_trees(ours, models)
    path = os.path.join(GOLD, "gcnjk.pt")
    torch.save(out, path)
    print("gcnjk", len(out), os.path.getsize(path), "bytes")


if __name__ == "__main__":
    cases()
