"""Weighted graphs (edge_weight) on the CPU: the oracle against the reference fixture (tests/golden/gcn_weighted.pt), the
edge-weight gradient formulas of sgf_edge_weight_grad against fp64 autograd, and the CSR restatement's loop / order rules."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from oracle import sgformer_oracle as O  # noqa: E402
import kernel_emu_weighted as KW  # noqa: E402

FIXTURE = os.path.join(HERE, "golden", "gcn_weighted.pt")


def load_cases():
    return torch.load(FIXTURE, weights_only=False)


def unflat(d):
    out, off = {}, 0
    for name, shape in zip(d["names"], d["shapes"]):
        k = int(np.prod(shape)) if shape else 1
        out[name] = d["flat"][off:off + k].reshape(shape)
        off += k
    return out


def oracle_config(case):
    kw = case["kw"]
    d, h, c = case["in_channels"], case["hidden"], case["out_channels"]
    if case["kind"] == "gcn":
        return O.make_config("medium", d, h, c, gcn_num_layers=kw.get("num_layers", 2), gcn_dropout=0.0,
                             gcn_use_bn=kw.get("use_bn", True))
    return O.make_config("medium", d, h, c, num_layers=1, alpha=0.5, dropout=0.0, use_residual=True,
                         gcn_num_layers=kw["gcn_layers"], gcn_dropout=0.0, graph_weight=0.7, aggregate=kw["aggregate"])


@pytest.mark.parametrize("name", ["gcn_directed", "gcn_sym_asym", "gcn_no_bn", "sgformer_add", "sgformer_cat"])
def test_oracle_matches_weighted_fixture(name):
    case = load_cases()[name]
    cfg = oracle_config(case)
    sd = {k: v for k, v in unflat(case["state_dict"]).items()}
    if case["kind"] == "gcn":
        sd = {"gnn." + k: v for k, v in sd.items()}
        out = O.gcn_medium(case["x"], case["edge_index"], sd, cfg, False, edge_weight=case["edge_weight"])
    else:
        out = O.sgformer_forward(cfg, sd, case["x"], case["edge_index"], False, edge_weight=case["edge_weight"])
    torch.testing.assert_close(out, case["out_eval"], rtol=1e-5, atol=1e-5)


def test_fixture_covers_the_graph_cases():
    for name, case in load_cases().items():
        ei, w = case["edge_index"], case["edge_weight"]
        src, dst = ei[0], ei[1]
        loops = torch.bincount(src[src == dst], minlength=case["x"].shape[0])
        assert loops[0] == 0 and loops[1] >= 1 and loops[2] >= 2, name
        assert (w == 0).any() and ei.unique(dim=1).shape[1] < ei.shape[1], name
        deg = torch.bincount(torch.cat([src, dst]), minlength=case["x"].shape[0])
        assert deg[-1] == 0, name                                    # isolated node
        # the reference's gcn_conv differentiates w * inf (sources without in-edges) into NaN; the forward value is 0 there
        assert case["ew_grad"].nan_to_num().abs().sum() > 0, name


def _graph(seed, n=9, e=30):
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n - 1, (e,), generator=g)
    dst = torch.randint(0, n - 1, (e,), generator=g)
    src = torch.cat([src, torch.tensor([3, 3, 5])])
    dst = torch.cat([dst, torch.tensor([3, 3, 5])])                 # node 3: two self loops, node n-1 isolated
    w = (0.1 + torch.rand(src.numel(), generator=g, dtype=torch.float64))
    w[2] = 0.0
    return torch.stack([src, dst]), w


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_gcn_edge_grad_formula_matches_autograd(seed):
    ei, w = _graph(seed)
    n, h = 9, 5
    g = torch.Generator().manual_seed(100 + seed)
    t = torch.randn(n, h, generator=g, dtype=torch.float64)
    go = torch.randn(n, h, generator=g, dtype=torch.float64)
    wv = w.clone().requires_grad_(True)
    (go * (KW.dense_gcn_adjacency(ei, wv, n) @ t)).sum().backward()
    got = KW.edge_weight_grad(ei.numpy(), w.numpy(), n, t.numpy(), go.numpy(), self_loop_mode=1)
    np.testing.assert_allclose(got, wv.grad.numpy(), rtol=0, atol=1e-10)


@pytest.mark.parametrize("seed", [0, 1])
def test_gcn_conv_edge_grad_formula_matches_autograd(seed):
    ei, w = _graph(seed)
    n, h = 9, 4
    g = torch.Generator().manual_seed(200 + seed)
    v = torch.randn(n, h, generator=g, dtype=torch.float64)
    go = torch.randn(n, h, generator=g, dtype=torch.float64)
    wv = w.clone().requires_grad_(True)
    (go * (KW.dense_gcn_conv_adjacency(ei, wv, n) @ v)).sum().backward()
    got = KW.edge_weight_grad(ei.numpy(), w.numpy(), n, v.numpy(), go.numpy(), self_loop_mode=0)
    np.testing.assert_allclose(got, wv.grad.numpy(), rtol=0, atol=1e-10)


def test_csr_restatement_matches_the_oracle_adjacency():
    ei, w = _graph(3)
    n = 9
    rowptr, col, eid, val, dinv = KW.csr_weighted(ei.numpy(), w.float().numpy(), n, False, 1)
    assert (np.diff(rowptr) >= 1).all()                              # one added loop per node
    loop3 = [j for j in range(rowptr[3], rowptr[4]) if col[j] == 3]
    assert len(loop3) == 1 and eid[loop3[0]] == ei.shape[1] - 2   # the last of node 3's two self loops
    A = KW.scipy_weighted(rowptr, col, val, n).toarray() * dinv[:, None].astype(np.float64) * dinv[None, :]
    ref = O.pyg_gcn_adjacency(ei, n, w.float()).to_dense().double().numpy()
    np.testing.assert_allclose(A, ref, rtol=2e-6, atol=1e-7)
