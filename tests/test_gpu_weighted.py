"""Weighted graphs (edge_weight) on the H100: the weighted CSR build against the numpy restatement (tests/kernel_emu_weighted.py),
the weighted SpMM against scipy in fp64, GCN / SGFormer(gnn=GCN) / DIFFormer against the reference fixture
(tests/golden/gcn_weighted.pt, tests/make_golden_weighted.py), GAT ignoring the weight, determinism and CUDA-graph capture."""
import numpy as np
import pytest
import torch

import kernel_emu_weighted as KW
from test_weighted import load_cases, unflat

pytestmark = pytest.mark.gpu
DEV = "cuda"


class Data:
    def __init__(self, x, ei, w=None):
        self.graph = {"node_feat": x, "edge_index": ei, "edge_weight": w, "num_nodes": x.shape[0]}


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-3)


def _graph(n, e, seed, hub=0, loops=True, symmetric=False, asym_weights=False):
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n - 1, (e,), generator=g)
    dst = torch.randint(0, n - 1, (e,), generator=g)
    if hub:                                     # node 5 receives `hub` edges: a row over HEAVY_ROW entries
        src = torch.cat([src, torch.randint(0, n, (hub,), generator=g)])
        dst = torch.cat([dst, torch.full((hub,), 5)])
    if loops:                                   # node 1: one self loop, node 2: three (the last one wins)
        src = torch.cat([src, torch.tensor([1, 2, 2, 2])])
        dst = torch.cat([dst, torch.tensor([1, 2, 2, 2])])
    w = 0.1 + torch.rand(src.numel(), generator=g)
    w[::17] = 0.0
    if symmetric:
        src, dst = torch.cat([src, dst]), torch.cat([dst, src])
        w = torch.cat([w, 0.1 + torch.rand(w.numel(), generator=g) if asym_weights else w])
    perm = torch.randperm(src.numel(), generator=g)
    return torch.stack([src, dst])[:, perm].contiguous(), w[perm].contiguous()


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("by_source", [False, True])
@pytest.mark.parametrize("hub", [0, 3000])
def test_weighted_csr_build_matches_restatement(mode, by_source, hub):
    from sgformer_b200 import kernels as K
    n = 700
    ei, w = _graph(n, 5000, 1 + hub + mode, hub=hub)
    rp, col, eid, val, dinv = K.csr_build_weighted(ei.to(DEV), w.to(DEV), n, by_source, mode, want_dinv=not by_source)
    erp, ecol, eeid, evl, edinv = KW.csr_weighted(ei.numpy(), w.numpy(), n, by_source, mode)
    assert np.array_equal(rp.cpu().numpy(), erp)
    assert np.array_equal(col.cpu().numpy(), ecol)
    assert np.array_equal(eid.cpu().numpy(), eeid)
    assert np.array_equal(val.cpu().numpy(), evl)
    if mode == 1:
        loops2 = (ei[0] == 2) & (ei[1] == 2)
        j = [k for k in range(erp[2], erp[3]) if ecol[k] == 2]
        assert eid.cpu()[j[0]].item() == loops2.nonzero().max().item()      # the last of node 2's self loops
    if not by_source:
        if mode == 1:
            deg = np.array([evl[erp[i]:erp[i + 1]].astype(np.float64).sum() for i in range(n)])
            ref = np.where(deg == 0, 0.0, 1.0 / np.sqrt(np.where(deg == 0, 1.0, deg)))
        else:
            lens = np.diff(erp)
            ref = np.where(lens > 0, 1.0 / np.sqrt(np.maximum(lens, 1)), 0.0)
        got = dinv.cpu().numpy().astype(np.float64)
        assert np.all(np.abs(got - ref) <= 2e-7 * np.abs(ref))


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 1e-5), (torch.bfloat16, 1e-2)])
@pytest.mark.parametrize("hub", [0, 3000])
@pytest.mark.parametrize("h", [64, 256])
def test_weighted_spmm_matches_scipy(dtype, tol, hub, h):
    from sgformer_b200 import kernels as K
    from sgformer_b200.graph import Graph
    n = 1500
    ei, w = _graph(n, 12000, 7 + hub, hub=hub, loops=False)
    g = Graph(ei.to(DEV), n, 1, edge_weight=w.to(DEV))
    x = torch.randn(n, h, generator=torch.Generator().manual_seed(2)).to(DEV, dtype)
    rp, col, eid, val, dinv = KW.csr_weighted(ei.numpy(), w.numpy(), n, False, 1)
    A = KW.scipy_weighted(rp, col, val, n)
    xd = x.double().cpu().numpy()
    y = K.spmm(g.rowptr, g.col, g.dinv, x, heavy=g.heavy, val=g.val)
    assert (g.heavy is not None) == bool(hub)
    assert _rel(y, torch.from_numpy(dinv[:, None].astype(np.float64) * (A @ xd))) < tol
    rpt, colt = g.transpose()
    assert rpt is not g.rowptr                      # directed: the transpose is built
    yt = K.spmm(rpt, colt, None, x, heavy=g.heavy_t, val=g.val_t)
    assert _rel(yt, torch.from_numpy(A.T @ xd)) < tol


def test_weighted_transpose_shares_only_symmetric_weights():
    from sgformer_b200 import kernels as K
    from sgformer_b200.graph import Graph
    n, h = 600, 64
    x = torch.randn(n, h, generator=torch.Generator().manual_seed(4)).to(DEV)
    for asym, shared in ((False, True), (True, False)):
        ei, w = _graph(n, 4000, 11, loops=True, symmetric=True, asym_weights=asym)
        g = Graph(ei.to(DEV), n, 1, edge_weight=w.to(DEV))
        rpt, colt = g.transpose()
        assert (rpt is g.rowptr) == shared
        rp, col, eid, val, _ = KW.csr_weighted(ei.numpy(), w.numpy(), n, False, 1)
        ref = KW.scipy_weighted(rp, col, val, n).T @ x.double().cpu().numpy()
        assert _rel(K.spmm(rpt, colt, None, x, heavy=g.heavy_t, val=g.val_t), torch.from_numpy(ref)) < 1e-5


def _build(case, prec):
    from sgformer_b200 import difformer as D
    from sgformer_b200 import medium as M
    d, h, c, kw = case["in_channels"], case["hidden"], case["out_channels"], case["kw"]
    if case["kind"] == "gcn":
        m = M.GCN(d, h, c, dropout=0.0, **kw)
    elif case["kind"] == "sgformer":
        gnn = M.GCN(d, h, h, num_layers=kw["gcn_layers"], dropout=0.0)
        m = M.SGFormer(d, h, c, num_layers=1, alpha=0.5, dropout=0.0, use_residual=True, graph_weight=0.7, gnn=gnn,
                       aggregate=kw["aggregate"])
    else:
        m = D.DIFFormer(d, h, c, num_layers=2, dropout=0.0, **kw)
    m.load_state_dict(unflat(case["state_dict"]))
    return m.to(DEV).set_precision(prec)


def _run(case, m, x, ei, w):
    if case["kind"] == "difformer":
        return m(Data(x, ei), w)
    return m(Data(x, ei, w))


# bf16: 1e-2 on the logits.  The parameter gradients of these 40-node BatchNorm / LayerNorm stacks carry the rounding of every
# bf16 activation they pass through, and a BatchNorm bias gradient is a sum over rows that largely cancels: in bf16 they are checked
# together, by the relative Frobenius error of all of them (5e-2); edge_weight.grad at 1e-1 of its largest entry
@pytest.mark.parametrize("prec,tol,gtol", [("fp32", 1e-4, 1e-4), ("bf16", 1e-2, 1e-1)])
@pytest.mark.parametrize("name", ["gcn_directed", "gcn_sym_asym", "gcn_no_bn", "sgformer_add", "sgformer_cat", "difformer",
                                  "difformer_sym_asym"])
def test_model_matches_reference_fixture(name, prec, tol, gtol):
    case = load_cases()[name]
    m = _build(case, prec)
    x, ei, w = case["x"].to(DEV), case["edge_index"].to(DEV), case["edge_weight"].to(DEV)
    m.eval()
    with torch.no_grad():
        assert _rel(_run(case, m, x, ei, w), case["out_eval"]) < tol, "eval logits"
    m.train()
    wg = w.clone().requires_grad_(True)
    out = _run(case, m, x, ei, wg)
    (out * case["loss_weight"].to(DEV)).sum().backward()
    assert _rel(out.detach(), case["out_train"]) < tol, "train logits"
    ref_grads = unflat(case["grads"])
    pairs = [(k, p_.grad, ref_grads[k]) for k, p_ in m.named_parameters() if k in ref_grads]
    if prec == "bf16":
        a = torch.cat([g_.double().cpu().reshape(-1) for _, g_, _ in pairs])
        b = torch.cat([r.double().reshape(-1) for _, _, r in pairs])
        assert ((a - b).norm() / b.norm()).item() < 5e-2, "parameter gradients"
    for k, got, exp in pairs if prec == "fp32" else []:
        if exp.abs().max() < 1e-5:              # a conv bias in front of BatchNorm: its gradient is 0 up to rounding
            assert got.abs().max().item() < 1e-4, k
        else:
            assert _rel(got, exp) < gtol, k
    ref = case["ew_grad"]
    fin = torch.isfinite(ref)       # NaN in the reference: gcn_conv's w * inf for sources without in-edges (value 0 there)
    assert torch.all(wg.grad.cpu()[~fin] == 0)
    assert _rel(wg.grad.cpu()[fin], ref[fin]) < gtol, "edge_weight.grad"
    if case["buffers"] is not None and prec == "fp32":
        sd = m.state_dict()
        for k, v in unflat(case["buffers"]).items():
            assert _rel(sd[k], v) < tol, k


@pytest.mark.parametrize("hub", [0, 3000])
def test_weighted_gcn_conv_term_matches_fp64_autograd(hub):
    """The kernels of DIFFormer's weighted graph term (gcn_conv, medium/difformer.py:63-79, as engine.difformer_forward /
    _backward run it: pre-scaled operand, weighted SpMM, transposed weighted SpMM, sgf_edge_weight_grad without the degree term)
    against fp64 autograd of the dense restatement, on a directed graph with isolated nodes, duplicates and a hub row."""
    from sgformer_b200 import kernels as K
    from sgformer_b200.graph import Graph
    n, h = 1500, 32
    ei, w = _graph(n, 9000, 31 + hub, hub=hub)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(n, h, generator=g)
    gy = torch.randn(n, h, generator=g, dtype=torch.float64)
    xd, wd = x.double().requires_grad_(True), w.double().requires_grad_(True)
    yd = KW.dense_gcn_conv_adjacency(ei, wd, n) @ xd
    (yd * gy).sum().backward()
    gr = Graph(ei.to(DEV), n, 0, edge_weight=w.to(DEV))
    assert (gr.heavy is not None) == bool(hub)
    xs = K.axpby(x.to(DEV), None, 1.0, 0.0, row_scale=gr.dinv)
    y = K.spmm(gr.rowptr, gr.col, gr.dinv, xs, heavy=gr.heavy, val=gr.val)
    assert _rel(y, yd.detach()) < 1e-5
    ds = K.axpby(gy.float().to(DEV), None, 1.0, 0.0, row_scale=gr.dinv)
    rpt, colt = gr.transpose()
    dx = K.spmm(rpt, colt, gr.dinv, ds, heavy=gr.heavy_t, val=gr.val_t)
    assert _rel(dx, xd.grad) < 1e-5
    dw = torch.zeros(ei.shape[1], dtype=torch.float32, device=DEV)
    K.edge_weight_grad(gr.rowptr, gr.col, gr.eid, ds, xs, dw)
    assert _rel(dw, wd.grad) < 1e-5


def test_gat_ignores_edge_weight():
    from sgformer_b200 import medium as M
    n, d = 300, 16
    ei, w = _graph(n, 2000, 5)
    torch.manual_seed(0)
    m = M.GAT(d, 8, 4, num_layers=2, dropout=0.0, heads=2).to(DEV).eval()
    x = torch.randn(n, d, device=DEV)
    with torch.no_grad():
        a = m(Data(x, ei.to(DEV)))
        b = m(Data(x, ei.to(DEV), w.to(DEV)))
    assert torch.equal(a, b)


def _gcn_step(model, x, ei, wg, lw):
    for p_ in model.parameters():
        p_.grad = None
    wg.grad = None
    out = model(Data(x, ei, wg))
    (out * lw).sum().backward()
    return out.detach().clone(), [p_.grad.clone() for p_ in model.parameters()], wg.grad.clone()


def test_weighted_training_is_deterministic_and_capturable(monkeypatch):
    from sgformer_b200 import engine as E
    from sgformer_b200 import medium as M
    n, d, h = 2000, 32, 64
    ei, w = _graph(n, 16000, 21, hub=2500)
    ei, w = ei.to(DEV), w.to(DEV)
    torch.manual_seed(1)
    model = M.GCN(d, h, h, num_layers=3, dropout=0.0).to(DEV)
    x = torch.randn(n, d, device=DEV)
    lw = torch.randn(n, h, device=DEV)
    monkeypatch.setattr(E, "next_seed", lambda: 0x5EED)
    sd0 = {k: v.clone() for k, v in model.state_dict().items()}
    wg = w.clone().requires_grad_(True)        # one weight tensor throughout: its graph structure is cached
    a = _gcn_step(model, x, ei, wg, lw)
    model.load_state_dict(sd0)
    b = _gcn_step(model, x, ei, wg, lw)
    assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2])
    assert all(torch.equal(p, q) for p, q in zip(a[1], b[1]))
    model.load_state_dict(sd0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _gcn_step(model, x, ei, wg, lw)
    torch.cuda.current_stream().wait_stream(s)
    model.load_state_dict(sd0)
    for p_ in model.parameters():
        p_.grad = None
    wg.grad = None
    cg = torch.cuda.CUDAGraph()
    with torch.cuda.graph(cg):
        out = model(Data(x, ei, wg))
        (out * lw).sum().backward()
    model.load_state_dict(sd0)
    cg.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, a[0])
    assert torch.equal(wg.grad, a[2])
    assert all(torch.equal(p_.grad, g) for p_, g in zip(model.parameters(), a[1]))
