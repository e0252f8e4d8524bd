"""Mini-batch subsets of directed graphs on the H100 (sgf_csr_subset_pair through Graph.subset and RandomPartitionSampler): both
halves equal sgf_csr_build of the batch's `subgraph` edge list bit for bit, a too-small capacity truncates but never overruns
either half and is reported, and training on sampler batches is bit-identical to training on the batches' edge lists."""
import copy
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def K():
    from sgformer_b200 import kernels
    return kernels


def directed_graph(n, e, seed, kind="random", hub=0):
    """A directed edge list with duplicate edges, self loops, isolated nodes (the top 1 %) and a source with no in-edges (node
    n - 2).  "powerlaw": both endpoints skewed towards small ids; `hub` edges into node 0 and as many out of node 1 (hub rows of
    each orientation longer than one block's share of the sort scratch)."""
    g = torch.Generator().manual_seed(seed)
    hi = n - max(n // 100, 2)
    if kind == "powerlaw":
        src = (hi * torch.rand(e, generator=g) ** 2.5).long()
        dst = (hi * torch.rand(e, generator=g) ** 3).long()
    else:
        src = torch.randint(0, hi, (e,), generator=g)
        dst = torch.randint(0, hi, (e,), generator=g)
    dst[dst == n - 2] = 2
    src[-(e // 50):] = n - 2
    if hub:
        dst[:hub] = 0
        src[hub:2 * hub] = 1
    ei = torch.stack([src, dst])
    ar = torch.arange(0, hi, 7)
    ei = torch.cat([ei, ei[:, : e // 20], torch.stack([ar, ar])], 1)
    return ei[:, torch.randperm(ei.shape[1], generator=g)].contiguous()


def _check_against_edge_list(K, full, ei, n, idx):
    sub = full.subset(idx)
    b = idx.numel()
    ei_sub = K.subgraph(ei, n, idx)
    rp, cl, dv = K.csr_build(ei_sub, b)
    rp_t, cl_t, _ = K.csr_build(ei_sub, b, True)
    sub_t = sub.transpose()
    assert torch.equal(sub.rowptr, rp) and torch.equal(sub.col, cl), f"b={b}: forward CSR differs"
    assert torch.equal(sub.dinv, dv), f"b={b}: dinv differs (bitwise)"
    assert torch.equal(sub_t[0], rp_t) and torch.equal(sub_t[1], cl_t), f"b={b}: transposed CSR differs"
    assert sub.heavy_t is None
    assert int(sub.nnz_needed) == int(sub.nnz_needed_t) == ei_sub.shape[1]
    assert int((full._node_map != -1).sum()) == 0, "node_map not restored"
    return sub


@pytest.mark.parametrize("kind,n,e,hub", [("random", 20000, 150000, 0), ("powerlaw", 30000, 300000, 0),
                                          ("powerlaw", 6000, 60000, 20000)])
def test_directed_subset_pair_matches_subgraph_then_build(K, kind, n, e, hub):
    from sgformer_b200.graph import Graph
    ei = directed_graph(n, e, 11, kind, hub).to(DEV)
    full = Graph(ei, n)
    assert full.transpose()[0] is not full.rowptr
    g = torch.Generator().manual_seed(3)
    for b in (1, 2, 31, 256, 1000, 4097, n // 2, n):
        idx = torch.randperm(n, generator=g)[:b].to(DEV)
        sub = _check_against_edge_list(K, full, ei, n, idx)
        assert sub.transpose()[0] is not sub.rowptr
    for idx in (torch.tensor([n - 2]), torch.tensor([0]), torch.arange(n)):     # no in-edges, the hub row, every node in order
        _check_against_edge_list(K, full, ei, n, idx.to(DEV))


def _pair_into_guarded_buffers(K, full, n, idx, cap, guard=64):
    """sgf_csr_subset_pair with `cap` as capacity into column buffers `guard` entries longer, pre-filled with -7."""
    b = idx.numel()
    rp_t, col_t = full.transpose()
    out = [torch.empty(b + 1, dtype=torch.int64, device=DEV), torch.full((cap + guard,), -7, dtype=torch.int32, device=DEV)]
    out_t = [torch.empty(b + 1, dtype=torch.int64, device=DEV), torch.full((cap + guard,), -7, dtype=torch.int32, device=DEV)]
    dinv = torch.empty(b, dtype=torch.float32, device=DEV)
    needed = torch.empty(2, dtype=torch.int64, device=DEV)
    nbytes = C.c_size_t(0)
    K.check(K.lib().sgf_csr_subset_ws_bytes(b, cap, C.byref(nbytes)), "ws")
    ws = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=DEV)
    K.check(K.lib().sgf_csr_subset_pair(K._p(full.rowptr), K._p(full.col), K._p(rp_t), K._p(col_t), n, K._p(idx), b,
                                        K._p(full._node_map), K._p(out[0]), K._p(out[1]), K._p(out_t[0]), K._p(out_t[1]), cap,
                                        K._p(dinv), K._p(needed), K._p(needed[1:]), K._p(ws), nbytes.value, K._stream()),
            "sgf_csr_subset_pair")
    return out, out_t, needed


def test_directed_subset_capacity_below_at_and_above(K):
    """Each half is bounded by the capacity: below the induced nnz its row pointers are clamped, the rows that fit are exact and
    nothing is written past the buffer; at or above it the result is exact.  Both halves report the full size, and
    RandomPartitionSampler.check raises when a batch overflowed."""
    from sgformer_b200.graph import Graph
    from sgformer_b200.minibatch import RandomPartitionSampler
    n = 8000
    ei = directed_graph(n, 90000, 5, "powerlaw").to(DEV)
    full = Graph(ei, n)
    idx = torch.randperm(n, generator=torch.Generator().manual_seed(0))[:4000].to(DEV)
    exact = full.subset(idx)
    exact_t = exact.transpose()
    nnz = int(exact.rowptr[-1])
    assert int(exact_t[0][-1]) == nnz
    for cap in (0, 1, nnz // 3, nnz - 1, nnz, nnz + 100):
        out, out_t, needed = _pair_into_guarded_buffers(K, full, n, idx, cap)
        assert needed.tolist() == [nnz, nnz], f"cap={cap}: needed {needed.tolist()}"
        for (rp, cl), (rp_x, cl_x) in (((out[0], out[1]), (exact.rowptr, exact.col)), ((out_t[0], out_t[1]), exact_t)):
            assert bool((cl[cap:] == -7).all()), f"cap={cap}: written past the capacity"
            if cap >= nnz:
                assert torch.equal(rp, rp_x) and torch.equal(cl[:nnz], cl_x)
                continue
            assert int(rp[-1]) == cap and bool((rp[1:] >= rp[:-1]).all())
            first = int((rp_x <= cap).sum()) - 1                     # rows that fit entirely are untouched
            assert torch.equal(rp[:first + 1], rp_x[:first + 1])
            assert torch.equal(cl[:int(rp[first])], cl_x[:int(rp[first])])
        assert int((full._node_map != -1).sum()) == 0
    x = torch.randn(n, 8, device=DEV)
    gen = torch.Generator(device=DEV)
    sampler = RandomPartitionSampler(full, x, None, 4000, capacity=nnz // 2, generator=gen.manual_seed(1))
    with pytest.raises(RuntimeError, match="capacity"):
        for _ in sampler:
            pass
    sampler = RandomPartitionSampler(full, x, None, 4000, capacity=int(ei.shape[1]), generator=gen.manual_seed(1))
    assert sum(mb.idx.numel() for mb in sampler) == n


def test_symmetric_parent_still_shares_the_transpose(K, monkeypatch):
    """On a symmetric edge list the subset's transpose is its forward CSR (one symmetry check per parent graph), also with a
    hub row longer than one block's share of the sort scratch."""
    from sgformer_b200 import kernels
    from sgformer_b200.graph import Graph
    n = 6000
    d = directed_graph(n, 40000, 2, "powerlaw", hub=12000)
    ei = torch.cat([d, d.flip(0)], 1).to(DEV)
    calls = []
    sym = kernels.edge_symmetry
    monkeypatch.setattr(kernels, "edge_symmetry", lambda *a: calls.append(1) or sym(*a))
    full = Graph(ei, n)
    g = torch.Generator().manual_seed(4)
    for b in (500, 3000, n):
        idx = torch.randperm(n, generator=g)[:b].to(DEV)
        sub = full.subset(idx)
        assert sub.transpose()[0] is sub.rowptr and sub.transpose()[1] is sub.col and sub.nnz_needed_t is sub.nnz_needed
        rp, cl, dv = K.csr_build(K.subgraph(ei, n, idx), b)
        assert torch.equal(sub.rowptr, rp) and torch.equal(sub.col, cl) and torch.equal(sub.dinv, dv)
    assert len(calls) == 1


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_sampler_training_on_directed_graph_matches_edge_lists(K, precision):
    """The large SGFormer trained for a few RandomPartitionSampler steps of a directed graph (two-group Adam, as
    large/main-batch.py:118-147) computes the same logits, parameter gradients and Adam updates, bit for bit, as the same
    steps fed `subgraph(idx, edge_index, relabel_nodes=True)` edge lists."""
    from sgformer_b200 import large as L
    from sgformer_b200.graph import Graph
    from sgformer_b200.minibatch import RandomPartitionSampler
    from sgformer_b200.optim import Adam
    torch.manual_seed(0)
    n, d, c = 20000, 32, 5
    ei = directed_graph(n, 160000, 7).to(DEV)
    x = torch.randn(n, d, device=DEV)
    y = torch.randint(0, c, (n,), device=DEV)
    model = L.SGFormer(d, 64, c, gnn_num_layers=2, gnn_use_init=True, gnn_dropout=0.0, trans_dropout=0.0, graph_weight=0.5)
    model = model.to(DEV).set_precision(precision)
    ref = copy.deepcopy(model)
    model.train()
    ref.train()
    opts = [Adam([{"params": m.params1, "weight_decay": 1e-3}, {"params": m.params2, "weight_decay": 5e-4}], lr=0.01)
            for m in (model, ref)]
    full = Graph(ei, n)
    sampler = RandomPartitionSampler(full, x, y, 7000, capacity=int(ei.shape[1]),
                                     generator=torch.Generator(device=DEV).manual_seed(0))
    steps = 0
    for _ in range(2):
        for mb in sampler:
            outs = []
            for m, opt, args in ((model, opts[0], (mb,)), (ref, opts[1], (x[mb.idx], K.subgraph(ei, n, mb.idx)))):
                opt.zero_grad()
                out = m(*args)
                torch.nn.functional.cross_entropy(out, y[mb.idx]).backward()
                outs.append(out.detach())
            assert torch.equal(outs[0], outs[1]), f"step {steps}: logits differ"
            for (k, p), q in zip(model.named_parameters(), ref.parameters()):
                assert torch.equal(p.grad, q.grad), f"step {steps}: grad {k} differs"
            for opt in opts:
                opt.step()
            for (k, p), q in zip(model.named_parameters(), ref.parameters()):
                assert torch.equal(p, q), f"step {steps}: parameter {k} differs after Adam"
            steps += 1
    assert steps == 6
