"""The induced subset of a directed graph (sgf_csr_subset_pair, Graph.subset on a parent whose edge list is not symmetric),
checked without a GPU: a torch statement of the kernel contract against PyG `subgraph(relabel_nodes=True)` (tests/ref_shims)
followed by a CSR build of each orientation, and Graph.subset's plumbing with that statement in place of the kernels.  The
CUDA kernels themselves are compared with the same edge-list path bit for bit in tests/test_gpu_subset_directed.py."""
import os
import sys

import pytest
import torch

import kernel_emu as emu
from sgformer_b200 import engine as E
from sgformer_b200 import functional as Fn
from sgformer_b200 import graph as G
from sgformer_b200 import large as L
from sgformer_b200.dist import SINGLE

HERE = os.path.dirname(os.path.abspath(__file__))


def pyg_subgraph(idx, ei, n):
    sys.path.insert(0, os.path.join(HERE, "ref_shims"))
    try:
        from torch_geometric.utils import subgraph          # CPU restatement of PyG 1.7.2
    finally:
        sys.path.pop(0)
    return subgraph(idx, ei, num_nodes=n, relabel_nodes=True)[0]


def subset_half(rowptr, col, node_map, idx, capacity, want_dinv):
    """One orientation of sgf_csr_subset(_pair): the rows of `idx`, entries kept when their column is in the subset (mapped to
    its local id) in CSR order, row pointers clamped to `capacity` (a clamped row keeps its first entries), rows then sorted."""
    b = idx.numel()
    lens = rowptr[idx + 1] - rowptr[idx]
    owner = torch.repeat_interleave(torch.arange(b), lens)
    pos = torch.repeat_interleave(rowptr[idx] - torch.cumsum(lens, 0) + lens, lens) + torch.arange(int(lens.sum()))
    m = node_map[col[pos].long()]
    keep = m >= 0
    owner, m = owner[keep], m[keep]
    counts = torch.bincount(owner, minlength=b)
    full = torch.zeros(b + 1, dtype=torch.int64)
    full[1:] = torch.cumsum(counts, 0)
    needed = full[-1:].clone()
    rp = full.clamp(max=capacity)
    fits = torch.arange(owner.numel()) < rp[owner + 1]      # the k-th kept entry goes to position k unless its row is clamped
    owner, m = owner[fits], m[fits]
    order = torch.argsort(owner * max(b, 1) + m.long(), stable=True)
    out_col = m[order].to(torch.int32)
    d = (rp[1:] - rp[:-1]).float()
    dinv = torch.where(d > 0, (1.0 / d).sqrt(), torch.zeros_like(d)) if want_dinv else None
    return rp, out_col, dinv, needed


def csr_subset(rowptr, col, n, subset, node_map, capacity=None, transposed=None):
    """torch statement of kernels.csr_subset (node_map is filled for the call and restored, as the kernels do)."""
    assert bool((node_map == -1).all())
    node_map[subset] = torch.arange(subset.numel(), dtype=torch.int32)
    if capacity is None:
        capacity = int((rowptr[subset + 1] - rowptr[subset]).sum())
    rp, cl, dv, needed = subset_half(rowptr, col, node_map, subset, capacity, True)
    out = (rp, cl, dv, needed)
    if transposed is not None:
        rp_t, cl_t, _, needed_t = subset_half(transposed[0], transposed[1], node_map, subset, capacity, False)
        out += (rp_t, cl_t, needed_t)
    node_map[subset] = -1
    return out


class EmuKernels:
    csr_subset = staticmethod(csr_subset)


def parent_graph(ei, n):
    """A Graph of a directed edge list (CSR and transposed CSR built by the CPU statement of sgf_csr_build)."""
    rp, cl, dv = emu.csr_build(ei, n)
    g = G.Graph._from_parts(n, rp, cl, dv, False)
    rp_t, cl_t, _ = emu.csr_build(ei, n, by_source=True)
    g._t = (rp_t, cl_t)
    g.edge_index = ei
    return g


def directed_graph(n, e, seed, hub=0, isolated=0, dup=0, loops=0):
    g = torch.Generator().manual_seed(seed)
    hi = n - isolated
    src = torch.randint(0, hi, (e,), generator=g)
    dst = torch.randint(1, hi, (e,), generator=g)           # node 0 is a source with no in-edges
    if hub:
        dst[:hub] = 3                                       # a hub row of the forward CSR ...
        src[hub:2 * hub] = 5                                # ... and one of the transposed CSR
    ei = torch.stack([src, dst])
    if dup:
        ei = torch.cat([ei, ei[:, :dup]], 1)
    if loops:
        ar = torch.arange(loops)
        ei = torch.cat([ei, torch.stack([ar, ar])], 1)
    return ei[:, torch.randperm(ei.shape[1], generator=g)].contiguous()


CASES = {
    "dup_loops_isolated": dict(n=300, e=2500, dup=400, loops=40, isolated=17),
    "hub_rows": dict(n=400, e=6000, hub=1500),
    "sparse": dict(n=1000, e=300, isolated=200),
}


@pytest.mark.parametrize("case", list(CASES))
def test_emulated_pair_matches_pyg_subgraph_then_build(monkeypatch, case):
    c = dict(CASES[case])
    n, e = c.pop("n"), c.pop("e")
    ei = directed_graph(n, e, 3, **c)
    assert not bool(torch.equal(torch.sort(ei[0] * n + ei[1]).values, torch.sort(ei[1] * n + ei[0]).values))
    monkeypatch.setattr(G, "K", EmuKernels)
    parent = parent_graph(ei, n)
    gen = torch.Generator().manual_seed(7)
    for idx in (torch.tensor([0]), torch.tensor([3]), torch.randperm(n, generator=gen)[:n // 3], torch.randperm(n, generator=gen),
                torch.arange(n)):
        sub = parent.subset(idx)
        ei_sub = pyg_subgraph(idx, ei, n)
        b = idx.numel()
        rp, cl, dv = emu.csr_build(ei_sub, b)
        rp_t, cl_t, _ = emu.csr_build(ei_sub, b, by_source=True)
        sub_t = sub.transpose()
        assert sub_t[0] is not sub.rowptr and sub.heavy_t is None
        assert torch.equal(sub.rowptr, rp) and torch.equal(sub.col, cl), f"{case} b={b}: forward CSR differs"
        assert torch.equal(sub.dinv, dv), f"{case} b={b}: dinv differs"
        assert torch.equal(sub_t[0], rp_t) and torch.equal(sub_t[1], cl_t), f"{case} b={b}: transposed CSR differs"
        assert int(sub.nnz_needed) == int(sub.nnz_needed_t) == ei_sub.shape[1]
        assert bool((parent._node_map == -1).all())


def test_emulated_pair_capacity_truncates_each_half():
    """A capacity below the induced nnz clamps both halves to it, each keeps its rows that fit, and both report the full size."""
    n = 500
    ei = directed_graph(n, 8000, 4, hub=600)
    parent = parent_graph(ei, n)
    idx = torch.randperm(n, generator=torch.Generator().manual_seed(1))[:300]
    node_map = torch.full((n,), -1, dtype=torch.int32)
    exact = csr_subset(parent.rowptr, parent.col, n, idx, node_map, None, parent._t)
    nnz = int(exact[0][-1])
    for cap in (nnz - 1, nnz // 2, 0):
        rp, cl, dv, needed, rp_t, cl_t, needed_t = csr_subset(parent.rowptr, parent.col, n, idx, node_map, cap, parent._t)
        assert int(needed) == int(needed_t) == nnz
        for r, full in ((rp, exact[0]), (rp_t, exact[4])):
            assert int(r[-1]) == cap and bool((r[1:] >= r[:-1]).all())
            first = int((full <= cap).sum()) - 1
            assert torch.equal(r[:first + 1], full[:first + 1])
        assert cl.numel() == cl_t.numel() == cap


def test_two_batch_schedule_matches_edge_list_path(monkeypatch):
    """Two random-partition batches of a directed graph through the large SGFormer schedule (kernels emulated): the batch
    Graph from Graph.subset gives the same logits and parameter gradients, bit for bit, as the batch's `subgraph` edge list."""
    monkeypatch.setattr(E, "K", emu)
    monkeypatch.setattr(Fn, "K", emu)
    monkeypatch.setattr(G, "K", EmuKernels)
    torch.manual_seed(0)
    n, d, h, c = 240, 12, 16, 4
    ei = directed_graph(n, 1500, 5, dup=50, loops=30, isolated=9)
    x = torch.randn(n, d)
    y = torch.randint(0, c, (n,))
    model = L.SGFormer(d, h, c, gnn_num_layers=2, gnn_use_init=True, gnn_dropout=0.0, trans_dropout=0.0, graph_weight=0.5)
    cfg, (names, tensors) = model._cfg(), model._flat()
    parent = parent_graph(ei, n)
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(2))
    for idx in (perm[:n // 2], perm[n // 2:]):
        results = []
        for graph in (parent.subset(idx, capacity=int(ei.shape[1])), emu.EmuGraph(pyg_subgraph(idx, ei, n), idx.numel())):
            params = [t.detach().clone().requires_grad_(t.is_floating_point() and "running" not in k) for k, t in zip(names, tensors)]
            out = Fn.SGFormerFn.apply(x[idx], graph, cfg, E.FP32, True, SINGLE, names, *params)
            torch.nn.functional.cross_entropy(out, y[idx]).backward()
            results.append((out.detach(), [p.grad for p in params if p.requires_grad]))
        (out_a, g_a), (out_b, g_b) = results
        assert torch.equal(out_a, out_b), "logits differ"
        assert all(torch.equal(a, b) for a, b in zip(g_a, g_b)), "a parameter gradient differs"
