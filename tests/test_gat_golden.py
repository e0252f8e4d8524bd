"""The GAT backbone pinned to the reference's own stack (tests/golden/gat.pt, tests/make_golden_gat.py: the unmodified
medium/models.py GAT and medium/ours.py SGFormer(gnn=GAT) over the restated GATConv): the oracle against the fixture, and the
hand-written GAT schedule (engine.gat_forward / gat_backward inside GraphBranchFn and SGFormerFn) with the kernels replaced by their
torch-CPU contracts (tests/kernel_emu_gat.py) against the fixture."""
import os

import pytest
import torch
import torch.nn.functional as F

import kernel_emu_gat as emu
from oracle import gat_oracle as G
from oracle import sgformer_oracle as O
from sgformer_b200 import engine as E
from sgformer_b200 import functional as Fn
from sgformer_b200 import medium as M
from sgformer_b200.dist import SINGLE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = torch.load(os.path.join(ROOT, "tests", "golden", "gat.pt"), weights_only=False)


def _unflat(d):
    out, o = {}, 0
    for k, shp in zip(d["names"], d["shapes"]):
        n = 1
        for s in shp:
            n *= s
        t = d["flat"][o:o + n].reshape(shp)
        out[k] = t.long() if k.endswith("num_batches_tracked") else t
        o += n
    return out


def _state_dict(c):
    sd = _unflat(c["state_dict"])
    for k in list(sd):
        if k.endswith("lin_src.weight"):
            sd[k.replace("lin_src", "lin_dst")] = sd[k]
    return sd


def _close(a, b, rtol, what, floor=1e-3):
    a, b = a.detach().double(), b.detach().double()
    assert a.shape == b.shape, f"{what}: shape {tuple(a.shape)} vs {tuple(b.shape)}"
    err = (a - b).abs().max().item()
    assert err <= rtol * max(b.abs().max().item(), floor), f"{what}: max err {err:.3e}"


class Data:
    def __init__(self, x, ei):
        self.graph = {"node_feat": x, "edge_index": ei, "num_nodes": x.shape[0]}


def test_fixture_covers_the_cases():
    gats = [c["gat"] for c in FIXTURE.values()]
    assert {g["heads"] for g in gats} >= {1, 2, 8} and {g["out_heads"] for g in gats} >= {1, 2}
    assert {g["use_bn"] for g in gats} == {True, False}
    assert {c["sgformer"]["aggregate"] for c in FIXTURE.values() if c["sgformer"]} == {"add", "cat"}
    directed = [c for name, c in FIXTURE.items() if "directed" in name]
    assert directed
    for c in directed:                  # existing self loops, duplicate edges, isolated nodes, not symmetric
        ei = c["edge_index"].long()
        assert (ei[0] == ei[1]).any()
        assert ei.t().unique(dim=0).shape[0] < ei.shape[1]
        assert torch.unique(ei).numel() < c["x"].shape[0]
        assert ei.flip(0).t().unique(dim=0).tolist() != ei.t().unique(dim=0).tolist()


def _models(c):
    d, h, cc = c["in_channels"], c["hidden"], c["out_channels"]
    sg = c["sgformer"]
    gnn_out = h if sg else cc
    ref_gat = G.GAT(d, h, gnn_out, dropout=0.0, **c["gat"])
    ours_gat = M.GAT(d, h, gnn_out, dropout=0.0, **c["gat"])
    if not sg:
        return ref_gat, ours_gat
    ours = M.SGFormer(d, h, cc, num_layers=1, num_heads=1, alpha=0.5, dropout=0.0, use_bn=True, use_residual=True, use_weight=True,
                      use_graph=True, gnn=ours_gat, **sg)
    return ref_gat, ours


def _oracle_forward(c, ref_gat, sd, x, ei, training):
    """models.GAT (or SGFormer(gnn=GAT)) restated: oracle GAT + the TransConv oracle + branch mix + fc."""
    sg = c["sgformer"]
    if not sg:
        return ref_gat(Data(x, ei))
    cfg = O.make_config("medium", c["in_channels"], c["hidden"], c["out_channels"], num_layers=1, num_heads=1, alpha=0.5,
                        dropout=0.0, use_bn=True, aggregate=sg["aggregate"], graph_weight=sg.get("graph_weight", 0.8))
    x1 = O.trans_conv(x, sd, cfg, training)
    x2 = ref_gat(Data(x, ei))
    gw = cfg["graph_weight"]
    hcat = gw * x2 + (1 - gw) * x1 if sg["aggregate"] == "add" else torch.cat([x1, x2], 1)
    return F.linear(hcat, sd["fc.weight"], sd["fc.bias"])


@pytest.mark.parametrize("name", sorted(FIXTURE))
def test_oracle_matches_fixture(name):
    c = FIXTURE[name]
    sd = _state_dict(c)
    ref_gat, _ = _models(c)
    gsd = {k[4:]: v for k, v in sd.items() if k.startswith("gnn.")} if c["sgformer"] else sd
    ref_gat.load_state_dict(gsd)
    x, ei = c["x"], c["edge_index"].long()
    ref_gat.eval()
    with torch.no_grad():
        _close(_oracle_forward(c, ref_gat, sd, x, ei, False), c["out_eval"], 1e-5, "eval logits")
    ref_gat.train()
    out = _oracle_forward(c, ref_gat, sd, x, ei, True)
    _close(out, c["out_train"], 1e-5, "train logits")
    exp = _unflat(c["grads"])
    (out * c["loss_weight"]).sum().backward()
    gmax = max(g.abs().max().item() for g in exp.values())
    pfx = "gnn." if c["sgformer"] else ""
    for k, p_ in ref_gat.named_parameters():
        if pfx + k in exp:
            _close(p_.grad, exp[pfx + k], 1e-5, k, floor=gmax)


def _run_emulated(c, model, x, ei, training):
    graph = emu.EmuGraph(ei, x.shape[0], 1)
    sg = c["sgformer"]
    if not sg:
        names, tensors = M._gat_flat(model, "gnn.")
        cfg = M.make_config("medium", x.shape[1], model.convs[0].lin_src.weight.shape[0], model.convs[-1].out_channels,
                            **model._cfg_kw())
        return Fn.GraphBranchFn.apply(x, graph, cfg, E.FP32, training, "gat", "gnn.", names, *tensors)
    tn, tt = model.trans_conv._flat("trans_conv.")
    fn = list(model.fc._parameters.keys())
    gn, gt = M._gat_flat(model.gnn, "gnn.")
    cfg = model._cfg(len(model.gnn.convs), float(model.gnn.dropout), bool(model.gnn.use_bn), "gat")
    names = tuple(tn) + tuple("fc." + k for k in fn) + tuple(gn)
    tensors = list(tt) + list(model.fc._parameters.values()) + list(gt)
    return Fn.SGFormerFn.apply(x, graph, cfg, E.FP32, training, SINGLE, names, *tensors)


@pytest.mark.parametrize("name", sorted(FIXTURE))
def test_emulated_schedule_matches_fixture(monkeypatch, name):
    monkeypatch.setattr(E, "K", emu)
    monkeypatch.setattr(Fn, "K", emu)
    c = FIXTURE[name]
    _, model = _models(c)
    model.load_state_dict(_state_dict(c))
    x, ei = c["x"], c["edge_index"].long()
    model.eval()
    with torch.no_grad():
        _close(_run_emulated(c, model, x, ei, False), c["out_eval"], 1e-5, "eval logits")
    model.train()
    xg = x.clone().requires_grad_(True)
    out = _run_emulated(c, model, xg, ei, True)
    _close(out, c["out_train"], 1e-5, "train logits")
    (out * c["loss_weight"]).sum().backward()
    _close(xg.grad, c["grad_x"], 1e-5, "grad_x")
    exp = _unflat(c["grads"])
    gmax = max(g.abs().max().item() for g in exp.values())
    got = dict(model.named_parameters())
    for k, g in exp.items():
        _close(got[k].grad, g, 1e-5, k, floor=gmax)
    if c["buffers_after_train"] is not None:
        sd = model.state_dict()
        for k, v in _unflat(c["buffers_after_train"]).items():
            _close(sd[k].float(), v.float(), 1e-5, k, floor=1.0)
