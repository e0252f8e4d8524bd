"""Mini-batch subsets of self_loop_mode 1 graphs on the H100 (the structure of GCN(save_mem=False) and GAT): both halves of
Graph.subset equal sgf_csr_build(self_loop_mode = 1) of the batch's `subgraph` edge list bit for bit, a too-small capacity
truncates but never overruns, mode-0 subsets are unchanged, and large_gnns.GCN / GAT trained on RandomPartitionSampler batches
are bit-identical to the same steps fed edge lists."""
import copy
import ctypes as C

import pytest
import torch

from test_gpu_subset_directed import directed_graph

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def K():
    from sgformer_b200 import kernels
    return kernels


def with_loops(ei, n, loops):
    """`loops` "none": no self loop at all; "dup": every node's loop three times; "some": loops on every 7th node only."""
    ei = ei[:, ei[0] != ei[1]]
    ar = torch.arange(n, device=ei.device)
    if loops == "dup":
        return torch.cat([ei, torch.stack([ar, ar]).repeat(1, 3)], 1)
    if loops == "some":
        return torch.cat([ei, torch.stack([ar[::7], ar[::7]])], 1)
    return ei


def _check(K, full, ei, n, idx, directed):
    sub = full.subset(idx)
    b = idx.numel()
    ei_sub = K.subgraph(ei, n, idx)
    rp, cl, dv = K.csr_build(ei_sub, b, False, 1)
    assert sub.self_loop_mode == 1 and sub.heavy is None and sub.heavy_t is None
    assert torch.equal(sub.rowptr, rp) and torch.equal(sub.col, cl), f"b={b}: forward CSR differs"
    assert torch.equal(sub.dinv, dv), f"b={b}: dinv differs (bitwise)"
    if directed:
        rp_t, cl_t, _ = K.csr_build(ei_sub, b, True, 1)
        assert sub.transpose()[0] is not sub.rowptr
        assert torch.equal(sub.transpose()[0], rp_t) and torch.equal(sub.transpose()[1], cl_t), f"b={b}: transposed CSR differs"
    else:
        assert sub.transpose()[0] is sub.rowptr
    assert int(sub.nnz_needed) == int(sub.nnz_needed_t) == int(rp[-1])
    assert int((full._node_map != -1).sum()) == 0, "node_map not restored"


@pytest.mark.parametrize("directed", [False, True])
@pytest.mark.parametrize("kind,n,e,hub,loops", [("random", 20000, 150000, 0, "none"), ("powerlaw", 30000, 300000, 0, "dup"),
                                                ("powerlaw", 6000, 60000, 20000, "some")])
def test_mode1_subset_matches_subgraph_then_mode1_build(K, directed, kind, n, e, hub, loops):
    from sgformer_b200.graph import Graph
    d = directed_graph(n, e, 11, kind, hub)
    ei = with_loops(d if directed else torch.cat([d, d.flip(0)], 1), n, loops).to(DEV)
    full = Graph(ei, n, self_loop_mode=1)
    g = torch.Generator().manual_seed(3)
    for b in (0, 1, 2, 31, 256, 1000, 4097, n // 2, n):
        _check(K, full, ei, n, torch.randperm(n, generator=g)[:b].to(DEV), directed)
    for idx in (torch.tensor([n - 1]), torch.tensor([0, 1]), torch.arange(n)):   # an isolated node, the hub rows, all nodes
        _check(K, full, ei, n, idx.to(DEV), directed)


@pytest.mark.parametrize("directed", [False, True])
def test_mode1_subset_capacity_below_at_and_above(K, directed):
    """Mode-1 halves through sgf_csr_subset(_pair) into guarded buffers: clamped below the induced nnz, exact at and above it,
    nothing written past the capacity, the full size reported."""
    from sgformer_b200.graph import Graph
    n = 8000
    d = directed_graph(n, 90000, 5, "powerlaw")
    ei = with_loops(d if directed else torch.cat([d, d.flip(0)], 1), n, "dup").to(DEV)
    full = Graph(ei, n, self_loop_mode=1)
    idx = torch.randperm(n, generator=torch.Generator().manual_seed(0))[:4000].to(DEV)
    exact = full.subset(idx)
    halves = [(exact.rowptr, exact.col)] + ([exact.transpose()] if directed else [])
    nnz = int(exact.rowptr[-1])
    b, guard = idx.numel(), 64
    rp_t, col_t = full.transpose()
    for cap in (0, 1, nnz // 3, nnz - 1, nnz, nnz + 100):
        outs = [(torch.empty(b + 1, dtype=torch.int64, device=DEV), torch.full((cap + guard,), -7, dtype=torch.int32, device=DEV))
                for _ in halves]
        dinv = torch.empty(b, dtype=torch.float32, device=DEV)
        needed = torch.empty(2, dtype=torch.int64, device=DEV)
        nbytes = C.c_size_t(0)
        K.check(K.lib().sgf_csr_subset_ws_bytes(b, cap, C.byref(nbytes)), "ws")
        ws = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=DEV)
        if directed:
            K.check(K.lib().sgf_csr_subset_pair(K._p(full.rowptr), K._p(full.col), K._p(rp_t), K._p(col_t), n, K._p(idx), b,
                                                K._p(full._node_map), K._p(outs[0][0]), K._p(outs[0][1]), K._p(outs[1][0]),
                                                K._p(outs[1][1]), cap, K._p(dinv), K._p(needed), K._p(needed[1:]), K._p(ws),
                                                nbytes.value, K._stream()), "sgf_csr_subset_pair")
        else:
            needed[1] = nnz
            K.check(K.lib().sgf_csr_subset(K._p(full.rowptr), K._p(full.col), n, K._p(idx), b, K._p(full._node_map),
                                           K._p(outs[0][0]), K._p(outs[0][1]), cap, K._p(dinv), K._p(needed), K._p(ws),
                                           nbytes.value, K._stream()), "sgf_csr_subset")
        assert needed.tolist() == [nnz, nnz], f"cap={cap}: needed {needed.tolist()}"
        for (rp, cl), (rp_x, cl_x) in zip(outs, halves):
            assert bool((cl[cap:] == -7).all()), f"cap={cap}: written past the capacity"
            if cap >= nnz:
                assert torch.equal(rp, rp_x) and torch.equal(cl[:nnz], cl_x)
                continue
            assert int(rp[-1]) == cap and bool((rp[1:] >= rp[:-1]).all())
            first = int((rp_x <= cap).sum()) - 1
            assert torch.equal(rp[:first + 1], rp_x[:first + 1])
            assert torch.equal(cl[:int(rp[first])], cl_x[:int(rp[first])])
        if cap >= nnz:
            assert torch.equal(dinv, exact.dinv)
        assert int((full._node_map != -1).sum()) == 0


def test_mode0_subsets_unchanged(K):
    """A mode-0 parent's subsets are still the mode-0 build of the batch's edge list (no added loops), with mode 0."""
    from sgformer_b200.graph import Graph
    n = 10000
    d = directed_graph(n, 80000, 9, "powerlaw")
    for ei in (d.to(DEV), torch.cat([d, d.flip(0)], 1).to(DEV)):
        full = Graph(ei, n)
        for b in (0, 500, n):
            idx = torch.randperm(n, generator=torch.Generator().manual_seed(b))[:b].to(DEV)
            sub = full.subset(idx)
            ei_sub = K.subgraph(ei, n, idx)
            rp, cl, dv = K.csr_build(ei_sub, b)
            assert sub.self_loop_mode == 0
            assert torch.equal(sub.rowptr, rp) and torch.equal(sub.col, cl) and torch.equal(sub.dinv, dv)
            rp_t, cl_t, _ = K.csr_build(ei_sub, b, True)
            assert torch.equal(sub.transpose()[0], rp_t) and torch.equal(sub.transpose()[1], cl_t)


def _model(kind, d, c):
    from sgformer_b200 import large_gnns as LG
    torch.manual_seed(0)
    if kind == "gcn_save_mem":
        return LG.GCN(d, 64, c, num_layers=3, dropout=0.0, save_mem=True)
    if kind == "gcn_norm":
        return LG.GCN(d, 64, c, num_layers=3, dropout=0.0, save_mem=False)
    return LG.GAT(d, 16, c, num_layers=2, dropout=0.0, heads=2)


def training_graph(n, e, seed, directed):
    """Random edges with duplicates, self loops on every 7th node and isolated nodes (the top 1 %), and no hub row: a batch
    Graph carries no hub-row plan (planning one costs a host sync per batch), while the edge-list path plans the rows longer
    than kernels.HEAVY_ROW and sums them in segments, so the two agree bit for bit only where no batch row is that long."""
    g = torch.Generator().manual_seed(seed)
    hi = n - n // 100
    ei = torch.randint(0, hi, (2, e), generator=g)
    ar = torch.arange(0, hi, 7)
    ei = torch.cat([ei, ei[:, : e // 20], torch.stack([ar, ar])], 1)
    if not directed:
        ei = torch.cat([ei, ei.flip(0)], 1)
    return ei[:, torch.randperm(ei.shape[1], generator=g)].contiguous()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("directed", [False, True])
@pytest.mark.parametrize("kind", ["gcn_save_mem", "gcn_norm", "gat"])
def test_sampler_training_matches_edge_lists(K, kind, directed, precision):
    """Six RandomPartitionSampler Adam steps of large_gnns.GCN / GAT (main-batch.py:118-147, one parameter group) compute the
    same logits, gradients and parameters, bit for bit, as the same steps fed `(x[idx], subgraph(idx, edge_index))`."""
    from sgformer_b200.graph import Graph
    from sgformer_b200.minibatch import RandomPartitionSampler
    from sgformer_b200.optim import Adam
    n, d, c = 20000, 32, 5
    ei = training_graph(n, 160000, 7, directed).to(DEV)
    x = torch.randn(n, d, generator=torch.Generator().manual_seed(1)).to(DEV)
    y = torch.randint(0, c, (n,), generator=torch.Generator().manual_seed(2)).to(DEV)
    model = _model(kind, d, c).to(DEV).set_precision(precision)
    ref = copy.deepcopy(model)
    model.train()
    ref.train()
    opts = [Adam(m.parameters(), lr=0.01, weight_decay=5e-4) for m in (model, ref)]
    full = Graph(ei, n, model.self_loop_mode)
    assert full.heavy is None and full.transpose() is not None and full.heavy_t is None
    sampler = RandomPartitionSampler(full, x, y, 7000, capacity=int(ei.shape[1]) + n,
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
                if p.grad is None:          # GAT without BatchNorm keeps gnns.GAT's unused `bns`
                    assert q.grad is None, f"step {steps}: grad {k}"
                    continue
                assert torch.equal(p.grad, q.grad), f"step {steps}: grad {k} differs"
            for opt in opts:
                opt.step()
            for (k, p), q in zip(model.named_parameters(), ref.parameters()):
                assert torch.equal(p, q), f"step {steps}: parameter {k} differs after Adam"
            steps += 1
    assert steps == 6


def test_mode_mismatch_raises():
    from sgformer_b200 import large_gnns as LG
    from sgformer_b200.graph import Graph
    from sgformer_b200.minibatch import RandomPartitionSampler
    n, d = 500, 8
    ei = torch.randint(0, n, (2, 3000), generator=torch.Generator().manual_seed(0)).to(DEV)
    x = torch.randn(n, d, device=DEV)
    g0, g1 = Graph(ei, n, 0), Graph(ei, n, 1)
    cases = [(LG.GCN(d, 8, 3, save_mem=True), g1), (LG.GCN(d, 8, 3, save_mem=False), g0), (LG.GAT(d, 8, 3), g0)]
    for model, wrong in cases:
        model = model.to(DEV).eval()
        with pytest.raises(ValueError, match=f"self_loop_mode {wrong.self_loop_mode}.*self_loop_mode {1 - wrong.self_loop_mode}"):
            model(x, wrong)
        idx = torch.arange(0, n, 2, device=DEV)
        with pytest.raises(ValueError, match="self_loop_mode"):
            model(RandomPartitionSampler(wrong, x, None, 100).batch(idx))
        right = Graph(ei, n, model.self_loop_mode)
        with torch.no_grad():
            assert torch.equal(model(x, right), model(x, ei))
