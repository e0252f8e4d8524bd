"""The medium variant's JKNet baseline (sgformer_b200.medium.GCNJK) without a GPU: the oracle against the fixture from the
unmodified reference (tests/make_golden_gcnjk.py), the GCNJK schedule on the emulated kernels (tests/kernel_emu_gcnjk.py) against
the fp64 oracle (alone and as SGFormer's graph branch), the parameter trees parse.py builds, and the refused options."""
import os

import pytest
import torch

import kernel_emu
import kernel_emu_gcnjk
from config_matrix import rel_err
from make_golden import synth_graph
from oracle import gcnjk_oracle as O
from sgformer_b200 import engine as E
from sgformer_b200 import functional as Fn
from sgformer_b200 import medium as M
from sgformer_b200.config import make_config
from sgformer_b200.dist import SINGLE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _unflat(d):
    out, o = {}, 0
    for name, shape in zip(d["names"], d["shapes"]):
        k = 1
        for s in shape:
            k *= s
        out[name] = d["flat"][o:o + k].reshape(shape).clone()
        o += k
    return out


def load():
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "gcnjk.pt"), weights_only=False)
    for name, c in fx.items():
        if name == "__trees__":
            continue
        for k in ("state_dict", "grads", "buffers_after_train", "grads64", "buffers_after_train64"):
            c[k] = _unflat(c[k])
        c["edge_index"] = c["edge_index"].long()
    return fx


FX = load()
TREES = FX.pop("__trees__")


def state_dict_as_loaded(c):
    return {k: (v.long() if k.endswith("num_batches_tracked") else v) for k, v in c["state_dict"].items()}


def oracle_run(c, dtype, training):
    sd = {k: (v.to(dtype).clone().requires_grad_(training and "running" not in k and "num_batches" not in k)
              if v.is_floating_point() else v) for k, v in state_dict_as_loaded(c).items()}
    x = c["x"].to(dtype).clone().requires_grad_(training)
    stats = {}
    out = O.gcnjk(x, c["edge_index"], sd, max(c["num_layers"], 2), c["jk"], training, stats_out=stats)
    if not training:
        return out.detach(), {}, None, {}
    (out * c["loss_weight"].to(dtype)).sum().backward()
    grads = {k: v.grad for k, v in sd.items() if isinstance(v, torch.Tensor) and v.grad is not None}
    return out.detach(), grads, x.grad, stats


def test_fixture_covers_the_cases():
    seen = {(c["num_layers"], c["jk"]) for c in FX.values()}
    assert seen == {(n, j) for n in (2, 3, 4) for j in ("max", "cat")}
    for c in FX.values():
        ei, n = c["edge_index"], c["x"].shape[0]
        assert ei.shape[1] > torch.unique(ei[0] * n + ei[1]).numel()                  # duplicate edges
        assert (ei[0] == ei[1]).any()                                                  # existing self loops
        assert (torch.bincount(ei[1], minlength=n) == 0).any()                         # isolated nodes
        assert set(c["buffers_after_train"]) == {f"bns.{i}.{b}" for i in range(c["num_layers"] - 1)
                                                for b in ("running_mean", "running_var", "num_batches_tracked")}


@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-10), (torch.float32, 1e-5)])
@pytest.mark.parametrize("name", sorted(FX))
def test_oracle_matches_fixture(name, dtype, tol):
    c = FX[name]

    sfx = "64" if dtype == torch.float64 else ""          # the reference run in the same dtype

    def close(a, b, msg):
        torch.testing.assert_close(a.double(), b.double(), rtol=tol, atol=tol, msg=msg)

    out_eval, _, _, _ = oracle_run(c, dtype, False)
    close(out_eval, c["out_eval" + sfx], "out_eval")
    out, grads, gx, stats = oracle_run(c, dtype, True)
    close(out, c["out_train" + sfx], "out_train")
    close(gx, c["grad_x" + sfx], "grad_x")
    assert set(grads) == set(c["grads" + sfx])
    for k, g in grads.items():
        close(g, c["grads" + sfx][k], k)
    for k, v in c["buffers_after_train" + sfx].items():
        close(stats[k].to(v.dtype), v, k)


def _relerr(a, b):
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / max(b.norm().item(), 1e-30)).item()


def _err(name, g, ref):
    return rel_err(name, g, ref) if "convs." in name and name.endswith(".bias") else _relerr(g, ref[name])


def _tol(name, nl):
    """The bias of a conv in front of a training BatchNorm has an exactly zero gradient: rel_err measures its fp32 rounding on
    1e-3 of its weight gradient's scale."""
    hidden_bias = any(name.endswith(f"convs.{i}.bias") for i in range(nl - 1))
    return 1e-3 if hidden_bias else 1e-4


def _emulate(monkeypatch):
    emu = kernel_emu_gcnjk.module()
    monkeypatch.setattr(E, "K", emu)
    monkeypatch.setattr(Fn, "K", emu)


def _run_gcnjk(m, x, ei):
    """GCNJK.forward's call with the emulated graph (the module itself refuses CPU tensors)."""
    names, tensors = M._gcnjk_flat(m, "")
    cfg = make_config("medium", x.shape[1], m.convs[0].out_channels, m.final_project.out_features, **m._cfg_kw())
    return Fn.GraphBranchFn.apply(x, kernel_emu.EmuGraph(ei, x.shape[0], 1), cfg, E.FP32, m.training, "gcnjk", "", names, *tensors)


@pytest.mark.parametrize("training", [False, True])
@pytest.mark.parametrize("name", sorted(FX))
def test_emulated_schedule_matches_fp64_oracle(name, training, monkeypatch):
    c = FX[name]
    m = M.GCNJK(c["in_channels"], c["hidden"], c["out_channels"], num_layers=c["num_layers"], dropout=0.0, jk_type=c["jk"])
    m.load_state_dict(state_dict_as_loaded(c))
    m.train(training)
    ref, rgrads, rgx, rstats = oracle_run(c, torch.float64, training)
    _emulate(monkeypatch)
    x = c["x"].clone().requires_grad_(training)
    out = _run_gcnjk(m, x, c["edge_index"])
    assert _relerr(out, ref) < 1e-5
    if not training:
        return
    (out * c["loss_weight"]).sum().backward()
    assert _relerr(x.grad, rgx) < 1e-4
    for k, p_ in m.named_parameters():
        assert _err(k, p_.grad, rgrads) < _tol(k, len(m.convs)), k
    for k, v in rstats.items():
        assert _relerr(m.state_dict()[k].double(), v) < 1e-5, k


def _sgformer_case(aggregate, jk, nl):
    torch.manual_seed(7)
    d, h, c, n = 10, 16, 4, 37
    m = M.SGFormer(d, h, c, num_layers=1, dropout=0.0, graph_weight=0.7, aggregate=aggregate,
                   gnn=M.GCNJK(d, h, h, num_layers=nl, dropout=0.0, jk_type=jk))
    with torch.no_grad():
        for k, p_ in m.named_parameters():
            if k.endswith("bias") or ".bns." in k:
                p_.add_(0.1 * torch.randn_like(p_))
    x = torch.randn(n, d)
    ei = synth_graph(n, 3 * n, 11, directed=True, isolated=3, dup=5)
    return m, x, ei


@pytest.mark.parametrize("aggregate,jk,nl", [("add", "max", 3), ("cat", "cat", 2), ("add", "cat", 4), ("cat", "max", 2)])
def test_emulated_sgformer_gcnjk_matches_fp64_oracle(aggregate, jk, nl, monkeypatch):
    m, x, ei = _sgformer_case(aggregate, jk, nl)
    m.train()
    cfg = m._cfg(len(m.gnn.convs), 0.0, True, "gcnjk", jk)
    sd = {k: (v.double().clone().requires_grad_(True) if v.is_floating_point() and "running" not in k else v)
          for k, v in m.state_dict().items()}
    lw = torch.randn(x.shape[0], 4)
    ref = O.sgformer_gcnjk(cfg, sd, x.double(), ei, training=True)
    (ref * lw.double()).sum().backward()
    _emulate(monkeypatch)
    tn, tt = m.trans_conv._flat("trans_conv.")
    gn, gt = M._gcnjk_flat(m.gnn, "gnn.")
    names = tuple(tn) + ("fc.weight", "fc.bias") + tuple(gn)
    out = Fn.SGFormerFn.apply(x, kernel_emu.EmuGraph(ei, x.shape[0], 1), cfg, E.FP32, True, SINGLE, names, *tt, m.fc.weight,
                              m.fc.bias, *gt)
    assert _relerr(out, ref) < 1e-5
    (out * lw).sum().backward()
    ref = {k: v.grad for k, v in sd.items() if isinstance(v, torch.Tensor) and v.grad is not None}
    for k, p_ in m.named_parameters():
        assert _err(k, p_.grad, ref) < _tol(k, len(m.gnn.convs)), k


def _tree(m):
    return list(m.state_dict().keys()), [k for k, _ in m.named_parameters()], {k: tuple(v.shape) for k, v in m.state_dict().items()}


def test_parameter_trees_match_parse_py():
    import inspect
    assert str(inspect.signature(M.GCNJK.__init__)) == TREES["signature"]
    a = TREES["args"]
    gj = M.GCNJK(in_channels=12, hidden_channels=a["hidden"], out_channels=5, num_layers=a["num_layers"], dropout=a["dropout"])
    assert list(_tree(gj)) == list(TREES["method"])
    gnn = M.GCNJK(12, a["hidden"], a["hidden"], num_layers=a["num_layers"], dropout=a["dropout"])
    sg = M.SGFormer(12, a["hidden"], 5, num_layers=1, alpha=0.5, dropout=0.3, num_heads=1, use_bn=True, use_residual=True,
                    use_graph=True, use_weight=True, use_act=False, graph_weight=0.8, gnn=gnn, aggregate="add")
    assert list(_tree(sg)) == list(TREES["backbone"])
    assert list(_tree(M.GCNJK(12, 16, 5, num_layers=2, jk_type="cat"))) == list(TREES["cat_l2"])


def test_reset_parameters_resets_convs_bns_and_final_project():
    m = M.GCNJK(8, 16, 3, num_layers=3)
    with torch.no_grad():
        for p_ in m.parameters():
            p_.fill_(3.0)
        for b in m.buffers():
            b.fill_(3)
    m.reset_parameters()
    for k, v in m.state_dict().items():
        assert not torch.all(v == 3), k


def test_is_not_gcn_like():
    assert not M._is_gcn_like(M.GCNJK(8, 16, 3, num_layers=3))
    from _refload import reference_available
    if reference_available():
        import make_golden_gcnjk
        _, models = make_golden_gcnjk.import_models()
        assert not M._is_gcn_like(models.GCNJK(8, 16, 3, num_layers=3))
    # what makes the reference's module not GCN-like: it has no use_bn (medium/models.py:157-190)
    assert not hasattr(M.GCNJK(8, 16, 3), "use_bn")


def test_refused_options():
    with pytest.raises(NotImplementedError, match="lstm"):
        M.GCNJK(8, 16, 3, jk_type="lstm")
    with pytest.raises(ValueError, match="cat"):
        M.GCNJK(8, 16, 3, num_layers=1, jk_type="cat")
    with pytest.raises(NotImplementedError, match="save_mem"):
        M.GCNJK(8, 16, 3, save_mem=True)
    assert len(M.GCNJK(8, 16, 3, num_layers=1).convs) == 2          # max with one layer: two convs, as the reference builds


def test_no_cpu_fallback():
    m = M.GCNJK(8, 16, 3)
    data = type("D", (), {"graph": {"node_feat": torch.randn(5, 8), "edge_index": torch.zeros(2, 0, dtype=torch.long)}})()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(data)


def test_gcnjk_stays_out_of_star_export():
    assert "GCNJK" not in M.__all__
