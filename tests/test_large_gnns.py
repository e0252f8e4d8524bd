"""The large variant's GCN / GAT baselines (sgformer_b200.large_gnns) without a GPU: the oracle against the reference's fixture,
the GCN schedule (both `save_mem` settings, the unscaled SpMM emulated) against the fp64 oracle through the module's own forward,
and the modules' constructors and parameter trees against large/gnns.py's."""
import inspect

import pytest
import torch

import kernel_emu
import large_gnns_fixture as LF
from config_matrix import FLOOR, rel_err
from sgformer_b200 import engine as E
from sgformer_b200 import functional as Fn
from sgformer_b200 import large_gnns as LG

FX = LF.load()
TREES = FX.pop("__trees__")


def test_fixture_covers_the_cases():
    seen = {(c["gcn"]["save_mem"], c["gcn"]["num_layers"], c["gcn"]["use_bn"]) for c in FX.values()}
    assert {s for s, _, _ in seen} == {True, False}
    assert {n for _, n, _ in seen} == {2, 3} and {b for _, _, b in seen} == {True, False}
    for c in FX.values():
        ei, n = c["edge_index"], c["x"].shape[0]
        assert ei.shape[1] > torch.unique(ei[0] * n + ei[1]).numel()                 # duplicate edges
        assert (torch.bincount(ei[1], minlength=n) <= (ei[0] == ei[1]).long().bincount(minlength=n)).any()  # a node with no other in-edge
    assert any(c["out_channels"] % 4 for c in FX.values())                            # a last conv the kernels run padded


@pytest.mark.parametrize("name", sorted(FX))
def test_oracle_matches_fixture(name):
    c = FX[name]
    out_eval, _, _, _ = LF.oracle_run(c, torch.float32, False)
    torch.testing.assert_close(out_eval, c["out_eval"], rtol=1e-5, atol=1e-5)
    out, grads, gx, stats = LF.oracle_run(c, torch.float32, True)
    torch.testing.assert_close(out, c["out_train"], rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(gx, c["grad_x"], rtol=1e-4, atol=1e-5)
    assert set(grads) == set(c["grads"])
    for k, g in grads.items():
        torch.testing.assert_close(g, c["grads"][k], rtol=1e-4, atol=1e-5, msg=k)
    for k, v in c["buffers_after_train"].items():
        if "running" in k and c["gcn"]["use_bn"]:
            torch.testing.assert_close(stats[k], v, rtol=1e-5, atol=1e-6, msg=k)


def _module(c):
    g = c["gcn"]
    m = LG.GCN(c["in_channels"], c["hidden"], c["out_channels"], dropout=0.0, **g)
    m.load_state_dict(LF.state_dict_as_loaded(c))
    return m.set_precision("fp32")


@pytest.mark.parametrize("name", sorted(FX))
def test_emulated_schedule_matches_fp64_oracle(name, monkeypatch):
    emu = LF.emulated_kernels()
    monkeypatch.setattr(E, "K", emu)
    monkeypatch.setattr(Fn, "K", emu)
    monkeypatch.setattr(LG, "get_graph", lambda ei, n, mode: kernel_emu.EmuGraph(ei, n, mode))
    c = FX[name]
    m = _module(c)
    names, tensors = LG.M._gcn_flat(m, "")
    m.eval()
    with torch.no_grad():
        out = m._run(c["x"], c["edge_index"], names, tensors)
    ref, _, _, _ = LF.oracle_run(c, torch.float64, False)
    assert (out.double() - ref).abs().max().item() <= 1e-4 * (1 + ref.abs().max().item())
    m.train()
    x = c["x"].clone().requires_grad_(True)
    out = m._run(x, c["edge_index"], names, tensors)
    (out * c["loss_weight"]).sum().backward()
    ref, grads, gx, stats = LF.oracle_run(c, torch.float64, True)
    assert (out.detach().double() - ref).abs().max().item() <= 1e-4 * (1 + ref.abs().max().item())
    ref_grads = dict(grads, __x=gx)
    got = {k: p.grad for k, p in m.named_parameters()}
    got["__x"] = x.grad
    for k in ref_grads:
        cls = "grad_x" if k == "__x" else ("affine" if k.endswith("bias") or k.startswith("bns.") else "bn_weight")
        e = rel_err("gnn." + k, got[k], {"gnn." + n: g for n, g in ref_grads.items()})
        assert e <= FLOOR[cls]["fp32"], f"{k}: relative error {e:.3e}"
    for k, v in stats.items():
        torch.testing.assert_close(m.state_dict()[k].double(), v.double(), rtol=1e-5, atol=1e-6, msg=k)


def _tree(m):
    return {k: tuple(v.shape) for k, v in m.state_dict().items() if "lin_dst" not in k}


@pytest.mark.parametrize("cls", ["GCN", "GAT"])
def test_modules_match_reference_trees(cls):
    """Constructor signature, state_dict keys and shapes (and the GCN convs' `normalize`) of large/gnns.py's classes, recorded
    in the fixture."""
    sig, rows = TREES[cls]
    native = getattr(LG, cls)
    assert str(inspect.signature(native.__init__)) == sig
    for kw, tree, norm in rows:
        m = native(12, 16, 5, **kw)
        assert _tree(m) == tree, kw
        assert [getattr(c, "normalize", None) for c in m.convs] == norm, kw
