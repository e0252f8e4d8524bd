"""The large variant's GCN / GAT baselines on the device (`-m gpu`): the unscaled SpMM (sgf_spmm_sum) against scipy in fp64, the
modules against the reference's fixture, the GCN at the recipe widths against the fp64 oracle, run-to-run bit identity, a
CUDA-graph captured training step, and a main-batch.py-style loop (a fresh edge_index every step, then an evaluation on the host)."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import large_gnns_fixture as LF
from config_matrix import FLOOR, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _rand_graph(n, e, seed, hub=None, hub_len=0, zero_rows=0):
    """Directed random edges with duplicates; the last `zero_rows` nodes receive no edge and the first `zero_rows` send none (empty
    rows in both orientations); node `hub` receives hub_len edges."""
    g = torch.Generator().manual_seed(seed)
    hi = n - zero_rows
    src = torch.randint(zero_rows, n, (e,), generator=g)
    dst = torch.randint(0, hi, (e,), generator=g)
    ei = torch.stack([src, dst])
    ei = torch.cat([ei, ei[:, : e // 10]], 1)                     # duplicates
    if hub is not None:
        ei = torch.cat([ei, torch.stack([torch.randint(zero_rows, n, (hub_len,), generator=g), torch.full((hub_len,), hub)])], 1)
    return ei[:, torch.randperm(ei.shape[1], generator=g)].contiguous()


def _scipy_sum(ei, n):
    return sp.csr_matrix((np.ones(ei.shape[1]), (ei[1].numpy(), ei[0].numpy())), shape=(n, n))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("h", [8, 16, 40, 64, 128, 256, 512])
def test_spmm_sum_matches_scipy(dtype, h):
    from sgformer_b200 import kernels as K
    from sgformer_b200.graph import Graph
    n = 3000
    ei = _rand_graph(n, 20000, 7 + h, hub=5, hub_len=2600, zero_rows=40)
    g = Graph(ei.to(DEV), n, 0)
    assert g.heavy is not None                                     # the hub row takes the segment path
    x = torch.randn(n, h, device=DEV).to(dtype)
    xd = x.double().cpu().numpy()
    A = _scipy_sum(ei, n)
    for transposed, M in ((False, A), (True, A.T.tocsr())):
        rp, cl = g.transpose() if transposed else (g.rowptr, g.col)
        y = K.spmm_sum(rp, cl, x, heavy=g.heavy_t if transposed else g.heavy).double().cpu().numpy()
        ref = M @ xd
        tol = 1e-5 if dtype == torch.float32 else 8e-3
        assert np.abs(y - ref).max() <= tol * (1 + np.abs(ref).max()), (transposed, np.abs(y - ref).max())
        empty = np.diff(M.indptr) == 0
        assert empty.any() and (y[empty] == 0).all()               # rows without entries are exact zeros
    # deterministic run to run, bit for bit
    a = K.spmm_sum(g.rowptr, g.col, x, heavy=g.heavy)
    b = K.spmm_sum(g.rowptr, g.col, x, heavy=g.heavy)
    assert torch.equal(a, b)


FX = LF.load()
FX.pop("__trees__")


def _module(c, prec):
    from sgformer_b200 import large_gnns as LG
    m = LG.GCN(c["in_channels"], c["hidden"], c["out_channels"], dropout=0.0, **c["gcn"])
    m.load_state_dict(LF.state_dict_as_loaded(c))
    return m.to(DEV).set_precision(prec)


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("name", sorted(FX))
def test_gcn_matches_fixture(name, prec):
    c = FX[name]
    tol = 1e-4 if prec == "fp32" else 1e-2
    m = _module(c, prec).eval()
    x, ei = c["x"].to(DEV), c["edge_index"].to(DEV)
    with torch.no_grad():
        out = m(x, ei).cpu()
    ref = c["out_eval"]
    assert (out - ref).abs().max().item() <= tol * (1 + ref.abs().max().item())
    m.train()
    xg = x.clone().requires_grad_(True)
    out = m(xg, ei)
    (out * c["loss_weight"].to(DEV)).sum().backward()
    ref = c["out_train"]
    assert (out.detach().cpu() - ref).abs().max().item() <= tol * (1 + ref.abs().max().item())
    ref_g = {"gnn." + k: v for k, v in c["grads"].items()}
    ref_g["__x"] = c["grad_x"]
    got = {"gnn." + k: p.grad for k, p in m.named_parameters()}
    got["__x"] = xg.grad
    for k in ref_g:
        cls = "grad_x" if k == "__x" else ("affine" if k.endswith("bias") or ".bns." in k else "bn_weight")
        e = rel_err(k, got[k], ref_g)
        assert e <= FLOOR[cls][prec], f"{k}: relative error {e:.3e} > {FLOOR[cls][prec]}"


def test_gcn_cpu_inputs_come_back_on_the_host():
    c = FX["savemem_l2_bn"]
    m = _module(c, "fp32").eval()
    with torch.no_grad():
        ref = m(c["x"].to(DEV), c["edge_index"].to(DEV)).cpu()
    m.to("cpu")
    with torch.no_grad():
        out = m(c["x"], c["edge_index"])
    assert out.device.type == "cpu" and torch.equal(out, ref)


@pytest.mark.parametrize("n,d,h,c,save_mem", [(200_000, 128, 64, 40, True), (50_000, 100, 256, 47, True),
                                               (50_000, 100, 256, 47, False)])
def test_gcn_recipe_widths_match_fp64(n, d, h, c, save_mem):
    """3 layers with BatchNorm at arxiv / amazon2m-like widths, the driver's self loops added; logits and every gradient against
    the fp64 oracle."""
    from sgformer_b200 import large_gnns as LG
    torch.manual_seed(3)
    ei = _rand_graph(n, 6 * n, 11, zero_rows=0)
    ei = torch.cat([ei, ei.flip(0)], 1)
    ei = ei[:, ei[0] != ei[1]]
    ar = torch.arange(n)
    ei = torch.cat([ei, torch.stack([ar, ar])], 1)
    m = LG.GCN(d, h, c, num_layers=3, dropout=0.0, save_mem=save_mem, use_bn=True)
    fx = dict(gcn=dict(num_layers=3, use_bn=True, save_mem=save_mem), x=torch.randn(n, d) * 0.5, edge_index=ei,
              state_dict=dict(m.state_dict()), loss_weight=torch.randn(n, c))
    ref, grads, gx, _ = LF.oracle_run(fx, torch.float64, True)
    m = m.to(DEV).set_precision("fp32").train()
    xg = fx["x"].to(DEV).requires_grad_(True)
    out = m(xg, ei.to(DEV))
    (out * fx["loss_weight"].to(DEV)).sum().backward()
    assert (out.detach().cpu().double() - ref).abs().max().item() <= 1e-4 * (1 + ref.abs().max().item())
    ref_g = {"gnn." + k: v for k, v in grads.items()}
    ref_g["__x"] = gx
    got = {"gnn." + k: p.grad for k, p in m.named_parameters()}
    got["__x"] = xg.grad
    for k in ref_g:
        cls = "grad_x" if k == "__x" else ("affine" if k.endswith("bias") or ".bns." in k else "bn_weight")
        e = rel_err(k, got[k], ref_g)
        assert e <= FLOOR[cls]["fp32"], f"{k}: relative error {e:.3e}"


def _step(m, x, ei, wgt):
    for p in m.parameters():
        p.grad = None
    xg = x.clone().requires_grad_(True)
    out = m(xg, ei)
    (out * wgt).sum().backward()
    return out.detach().clone(), [p.grad.clone() for p in m.parameters()], xg.grad.clone()


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_gcn_training_step_is_bit_identical_run_to_run(prec, monkeypatch):
    from sgformer_b200 import engine as E
    from sgformer_b200 import large_gnns as LG
    monkeypatch.setattr(E, "next_seed", lambda: 0xBEEF)
    n, d = 20000, 64
    ei = _rand_graph(n, 8 * n, 5, hub=3, hub_len=3000).to(DEV)
    m = LG.GCN(d, 64, 40, num_layers=3, dropout=0.5).to(DEV).set_precision(prec).train()
    x, wgt = torch.randn(n, d, device=DEV), torch.randn(n, 40, device=DEV)
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    a = _step(m, x, ei, wgt)
    m.load_state_dict(sd0)
    b = _step(m, x, ei, wgt)
    assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2])
    assert all(torch.equal(u, v) for u, v in zip(a[1], b[1]))


def test_gcn_cuda_graph_step_matches_eager(monkeypatch):
    from sgformer_b200 import engine as E
    from sgformer_b200 import kernels as K
    from sgformer_b200 import large_gnns as LG
    n, d, c = 5000, 32, 40
    ei = _rand_graph(n, 8 * n, 9).to(DEV)
    m = LG.GCN(d, 64, c, num_layers=3, dropout=0.3).to(DEV).train()
    x, wgt = torch.randn(n, d, device=DEV), torch.randn(n, c, device=DEV)
    K.dropout_epoch()
    monkeypatch.setattr(E, "next_seed", lambda: 0x5EED)
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    eager = _step(m, x, ei, wgt)
    m.load_state_dict(sd0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _step(m, x, ei, wgt)
    torch.cuda.current_stream().wait_stream(s)
    m.load_state_dict(sd0)
    for p in m.parameters():
        p.grad = None
    xo = x.clone().requires_grad_(True)
    cg = torch.cuda.CUDAGraph()
    with torch.cuda.graph(cg):
        out = m(xo, ei)
        (out * wgt).sum().backward()
    m.load_state_dict(sd0)
    cg.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager[0])
    assert all(torch.equal(p.grad, g) for p, g in zip(m.parameters(), eager[1]))
    assert torch.equal(xo.grad, eager[2])


def _subgraph(idx, ei, n):
    """PyG subgraph(idx, edge_index, relabel_nodes=True) restated in torch (large/main-batch.py:139)."""
    mask = torch.zeros(n, dtype=torch.bool, device=ei.device)
    mask[idx] = True
    keep = mask[ei[0]] & mask[ei[1]]
    loc = torch.full((n,), -1, dtype=torch.long, device=ei.device)
    loc[idx] = torch.arange(idx.numel(), device=ei.device)
    return loc[ei[:, keep]]


@pytest.mark.parametrize("cls", ["GCN", "GAT"])
def test_minibatch_loop_then_host_evaluation(cls):
    """main-batch.py's loop: a random node batch and its fresh subgraph every step (a new CSR each time), an optimizer step, then
    evaluate_large(device="cpu")'s round trip: model.to("cpu") and a host forward whose logits equal the device forward's."""
    from sgformer_b200 import graph as G
    from sgformer_b200 import large_gnns as LG
    torch.manual_seed(0)
    n, d, c, bs = 6000, 32, 8, 2000
    ei = _rand_graph(n, 6 * n, 4)
    ei = torch.cat([ei[:, ei[0] != ei[1]], torch.arange(n).repeat(2, 1)], 1).to(DEV)
    x, y = torch.randn(n, d, device=DEV), torch.randint(0, c, (n,), device=DEV)
    m = (LG.GCN(d, 64, c, num_layers=3, dropout=0.5) if cls == "GCN" else
         LG.GAT(d, 16, c, num_layers=2, dropout=0.5, heads=4, out_heads=1)).to(DEV)
    opt = torch.optim.Adam(m.parameters(), lr=1e-2)
    m.train()
    seen = []
    for step in range(4):
        idx = torch.randperm(n, device=DEV)[:bs]
        ei_i = _subgraph(idx, ei, n)
        opt.zero_grad()
        loss = torch.nn.functional.cross_entropy(m(x[idx], ei_i), y[idx])
        loss.backward()
        opt.step()
        assert torch.isfinite(loss)
        mode = 0 if cls == "GCN" else 1
        g = G.get_graph(ei_i, bs, mode)
        assert g.edge_index is ei_i and g not in seen               # a new edge_index built a new CSR ...
        assert G.get_graph(ei_i, bs, mode) is g                    # ... and a repeated one hits the cache
        seen.append(g)
    m.eval()
    with torch.no_grad():
        ref = m(x, ei).cpu()
    m.to(torch.device("cpu"))
    with torch.no_grad():
        out = m(x.cpu(), ei.cpu())
    assert out.device.type == "cpu" and torch.equal(out, ref)


def test_gat_matches_medium_gat():
    """large_gnns.GAT is the medium native GAT called as forward(x, edge_index): same parameters, same logits and gradients."""
    from sgformer_b200 import medium as M
    from sgformer_b200 import large_gnns as LG

    class Data:
        def __init__(self, x, ei):
            self.graph = {"node_feat": x, "edge_index": ei}

    torch.manual_seed(1)
    n, d = 3000, 24
    ei = _rand_graph(n, 6 * n, 2).to(DEV)
    a = LG.GAT(d, 16, 8, num_layers=3, dropout=0.0, use_bn=True, heads=4, out_heads=2).to(DEV)
    b = M.GAT(d, 16, 8, num_layers=3, dropout=0.0, use_bn=True, heads=4, out_heads=2).to(DEV)
    b.load_state_dict(a.state_dict())
    x, wgt = torch.randn(n, d, device=DEV), torch.randn(n, 8, device=DEV)
    oa, ob = a(x, ei), b(Data(x, ei))
    (oa * wgt).sum().backward()
    (ob * wgt).sum().backward()
    assert torch.equal(oa, ob)
    assert all(torch.equal(p.grad, q.grad) for p, q in zip(a.parameters(), b.parameters()))
