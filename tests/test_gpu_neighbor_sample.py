"""The device neighbour sampler (sgformer_b200/csrc/sample.cu through minibatch.NeighborSampler) on the H100: every batch equals the
numpy restatement (tests/neighbor_sample_ref.py) bit for bit, idx and edge list, at the 100M recipe's fan-outs [15, 10, 5], at
k = 1, k = 64 and k = -1, on graphs with hub rows of more than 10^5 entries and frontiers past the kernels' grid cap; the batch
Graph equals Graph(edge_index, b, 0) field for field; batches replay from the generator state and leave the node map at -1; the
100M SGFormer on a batch matches its edge-list run and the fp64 oracle; inclusion rates are uniform; a short nb-sample.py-style
loop learns; an undersized capacity is reported by check()."""
import numpy as np
import pytest
import torch

import neighbor_sample_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"


def hub_graph(n, e, seed, hubs=(0, 1), hub_deg=120000):
    """Uniform random directed edges plus `hub_deg` in-edges into each hub (rows longer than 10^5 entries), duplicates, self loops
    and isolated nodes (the top 1 %)."""
    g = torch.Generator().manual_seed(seed)
    hi = n - n // 100
    src, dst = torch.randint(0, hi, (e,), generator=g), torch.randint(0, hi, (e,), generator=g)
    parts = [torch.stack([src, dst]), torch.stack([src[: e // 20], dst[: e // 20]]), torch.arange(0, hi, 5).repeat(2, 1)]
    for h in hubs:
        parts.append(torch.stack([torch.randint(0, hi, (hub_deg,), generator=g), torch.full((hub_deg,), h)]))
    return torch.cat(parts, 1).contiguous()


@pytest.fixture(scope="module")
def big():
    from sgformer_b200.graph import Graph
    n = 300000
    ei = hub_graph(n, 3000000, 1).to(DEV)
    g = Graph(ei, n)
    return g, g.rowptr.cpu().numpy(), g.col.cpu().numpy(), n


def _check_batch(mb, rowptr, col, seeds, fan, seed, capacity=None):
    idx, ei, need = R.sample(rowptr, col, seeds.cpu().numpy(), fan, seed, capacity)
    assert mb.idx.cpu().numpy().tolist() == idx.tolist(), "idx differs from the restatement"
    assert np.array_equal(mb.graph.edge_index.cpu().numpy(), ei), "edge list differs from the restatement"
    assert mb.num_seeds == seeds.numel()
    return need


def _check_graph(K, mb):
    from sgformer_b200.graph import Graph
    g, b = mb.graph, mb.idx.numel()
    ref = Graph(mb.graph.edge_index.contiguous(), b, 0)
    assert torch.equal(g.rowptr, ref.rowptr) and torch.equal(g.col, ref.col), "forward CSR differs"
    assert torch.equal(g.dinv, ref.dinv), "dinv differs (bitwise)"
    t, rt = g.transpose(), ref.transpose()
    assert torch.equal(t[0], rt[0]) and torch.equal(t[1], rt[1]), "transposed CSR differs"
    assert g.n == b and g.self_loop_mode == 0


@pytest.mark.parametrize("fan,bsz,capacity", [([15, 10, 5], 1000, None), ([1], 4096, None), ([1, 1, 1], 50000, None),
                                              ([64], 700, None), ([64, 2], 300, None), ([-1], 12, 130000),
                                              ([3, -1], 40, 130000), ([15, 10, -1], 16, 400)])
def test_batches_match_restatement_bit_for_bit(big, fan, bsz, capacity):
    from sgformer_b200 import kernels as K
    from sgformer_b200.minibatch import NeighborSampler
    g, rowptr, col, n = big
    x = torch.zeros(n, 4, device=DEV)
    s = NeighborSampler(g, x, None, fan, bsz, shuffle=True, generator=torch.Generator().manual_seed(7), capacity=capacity)
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(len(fan) + bsz))
    need = 0
    for i, seeds in enumerate([perm[:bsz], torch.cat([torch.tensor([0, 1]), perm[:bsz - 2]]), perm[bsz: bsz + bsz // 3 + 1]]):
        seed = 0xABCDEF + 977 * i
        mb = s.batch(seeds.to(DEV), seed=seed)
        need = max(need, _check_batch(mb, rowptr, col, seeds, fan, seed, capacity))
        _check_graph(K, mb)
        assert int((g._sample_map != -1).sum()) == 0, "node map not restored"
    if capacity is not None and need > capacity:
        with pytest.raises(RuntimeError, match=f"capacity >= {need}"):
            s.check()
    else:
        s.check()


def test_replay_from_generator_state_and_epochs(big):
    from sgformer_b200.minibatch import NeighborSampler
    g, rowptr, col, n = big
    x = torch.randn(n, 8, device=DEV)
    y = torch.randint(0, 5, (n,), device=DEV)
    split = torch.randperm(n, generator=torch.Generator().manual_seed(3))[:5500].to(DEV)

    def epoch(state_seed):
        s = NeighborSampler(g, x, y, [15, 10, 5], 1000, input_nodes=split, shuffle=True,
                            generator=torch.Generator().manual_seed(state_seed), num_workers=12)
        out = []
        for mb in s:
            assert int((g._sample_map != -1).sum()) == 0
            assert torch.equal(mb.features, x[mb.idx]) and torch.equal(mb.labels, y[mb.idx])
            out.append((mb.idx.clone(), mb.graph.edge_index.clone(), mb.graph.col.clone(), mb.num_seeds))
        return out
    a, b, c = epoch(11), epoch(11), epoch(12)
    assert len(a) == 6 and [m[3] for m in a] == [1000] * 5 + [500]
    assert sorted(torch.cat([m[0][:m[3]] for m in a]).tolist()) == sorted(split.tolist())
    for p, q in zip(a, b):
        assert all(torch.equal(u, v) for u, v in zip(p[:3], q[:3]))
    assert not torch.equal(a[0][0], c[0][0])
    empty = NeighborSampler(g, x, y, [15, 10, 5], 1000, input_nodes=split[:0])
    assert len(empty) == 0 and list(empty) == []


def test_capacity_too_small_is_reported_and_never_overrun(big):
    """k = -1 with a capacity below the hub rows: those rows are cut to their first `capacity` entries (the restatement with the
    same capacity), the buffers are the plan's, and check() raises."""
    from sgformer_b200.minibatch import NeighborSampler
    g, rowptr, col, n = big
    x = torch.zeros(n, 4, device=DEV)
    s = NeighborSampler(g, x, None, [-1, 2], 8, capacity=1000)
    seeds = torch.tensor([0, 1, 5, 9, 17, 33, 65, 129])
    mb = s.batch(seeds.to(DEV), seed=5)
    _check_batch(mb, rowptr, col, seeds, [-1, 2], 5, capacity=1000)
    assert mb.graph.col.numel() <= s.plan.max_edges and mb.idx.numel() <= s.plan.max_nodes
    with pytest.raises(RuntimeError, match="capacity >= 12"):
        s.check()
    assert int((g._sample_map != -1).sum()) == 0


def test_parent_graph_requirements():
    from sgformer_b200.graph import Graph
    from sgformer_b200.minibatch import NeighborSampler
    ei = hub_graph(1000, 5000, 2, hubs=()).to(DEV)
    x = torch.zeros(1000, 4, device=DEV)
    with pytest.raises(ValueError, match="self_loop_mode 1"):
        NeighborSampler(Graph(ei, 1000, 1), x, None, [2], 10)
    with pytest.raises(NotImplementedError):
        NeighborSampler(Graph(ei, 1000, 0, edge_weight=torch.rand(ei.shape[1], device=DEV)), x, None, [2], 10)
    with pytest.raises(ValueError, match="distinct"):
        NeighborSampler(Graph(ei, 1000), x, None, [2], 10, input_nodes=torch.tensor([1, 1], device=DEV))


def test_inclusion_rates_are_uniform():
    """T targets share the same D sources (row position p = source T + p).  Over T rows x 8 seeds, the count of each position is
    within a chi-square bound of T * 8 * k / D: chi2 over the D positions below the 99.99 % quantile of chi2(D - 1) (Floyd's draws
    are without replacement, which only lowers the spread)."""
    from sgformer_b200.graph import Graph
    from sgformer_b200.minibatch import NeighborSampler
    bound = {20: 50.8, 6: 25.7, 200: 281.9}     # the 99.99 % quantiles of chi2(D - 1)
    T = 4000
    for D, k in ((20, 5), (6, 5), (200, 15)):
        src = (T + torch.arange(D)).repeat(T)
        dst = torch.arange(T).repeat_interleave(D)
        ei = torch.stack([src, dst]).to(DEV)
        g = Graph(ei, T + D)
        s = NeighborSampler(g, torch.zeros(T + D, 4, device=DEV), None, [k], T)
        counts = torch.zeros(D, dtype=torch.float64)
        for seed in range(8):
            mb = s.batch(torch.arange(T, device=DEV), seed=1000 + seed)
            srcs = mb.idx[mb.graph.edge_index[0]] - T
            assert mb.graph.edge_index.shape[1] == T * k
            counts += torch.bincount(srcs.cpu(), minlength=D).double()
        exp = T * 8 * k / D
        chi2 = float(((counts - exp) ** 2 / exp).sum())
        assert chi2 < bound[D], f"D={D} k={k}: chi2 {chi2:.1f} over {bound[D]}"


def _model(d, c, precision):
    from sgformer_b200 import hundred_m as H
    torch.manual_seed(0)
    m = H.SGFormer(d, 32, c, trans_num_layers=1, gnn_num_layers=3, gnn_use_init=True, alpha=0.5, graph_weight=0.8,
                   gnn_dropout=0.0, trans_dropout=0.0)
    return m.to(DEV).set_precision(precision)


@pytest.mark.parametrize("precision,tol", [("fp32", 1e-4), ("bf16", 1e-2)])
def test_model_on_batch_equals_edge_list_and_oracle(precision, tol):
    """model(mb) == model(mb.features, mb.graph.edge_index) bit for bit (uniform graph: no batch row past the SpMM's hub-row
    threshold, so both runs take the same SpMM path), eval and train, and the eval logits match the fp64 oracle."""
    from oracle import sgformer_oracle as O
    from sgformer_b200.graph import Graph
    from sgformer_b200.minibatch import NeighborSampler
    n, d, c = 60000, 24, 6
    ei = hub_graph(n, 600000, 4, hubs=()).to(DEV)
    x = torch.randn(n, d, device=DEV)
    s = NeighborSampler(Graph(ei, n), x, None, [15, 10, 5], 200, generator=torch.Generator().manual_seed(1))
    mb = s.batch(torch.randperm(n, generator=torch.Generator().manual_seed(2))[:200].to(DEV))
    model = _model(d, c, precision)
    model.eval()
    with torch.no_grad():
        a, b = model(mb), model(mb.features, mb.graph.edge_index)
    assert torch.equal(a, b), "eval logits differ between the batch Graph and its edge list"
    sd = {k: v.detach().cpu() for k, v in model.state_dict().items()}     # before train mode moves the BatchNorm running stats
    model.train()
    outs = []
    for args in ((mb,), (mb.features, mb.graph.edge_index)):
        model.zero_grad()
        out = model(*args)
        out[:mb.num_seeds].square().sum().backward()
        outs.append((out.detach(), [p.grad.clone() for p in model.parameters()]))
    assert torch.equal(outs[0][0], outs[1][0])
    assert all(torch.equal(p, q) for p, q in zip(outs[0][1], outs[1][1])), "parameter gradients differ"
    ref = O.sgformer_forward(model._cfg(), {k: v.double() if v.is_floating_point() else v for k, v in sd.items()},
                             mb.features.cpu().double(), mb.graph.edge_index.cpu(), training=False)
    err = (a.double().cpu() - ref).abs().max().item()
    assert err <= tol * max(1.0, ref.abs().max().item()), f"{precision}: logits differ from the fp64 oracle by {err:.3e}"


def test_short_training_loop_learns():
    """nb-sample.py:27-46 / :125-150 on the device: pretrain 300 steps on a planted-label graph (80 % of the in-edges within the
    class, features = weak class signal + noise), loss on out[:num_seeds]; the loss falls and validation accuracy by argmax
    counts beats chance by a wide margin."""
    from sgformer_b200.graph import Graph
    from sgformer_b200.minibatch import NeighborSampler
    from sgformer_b200.optim import Adam
    n, d, c = 40000, 16, 4
    g = torch.Generator().manual_seed(0)
    y = torch.randint(0, c, (n,), generator=g)
    by_class = [torch.nonzero(y == k).flatten() for k in range(c)]
    dst = torch.randint(0, n, (400000,), generator=g)
    same = torch.rand(400000, generator=g) < 0.8
    src = torch.randint(0, n, (400000,), generator=g)
    for k in range(c):
        m = same & (y[dst] == k)
        src[m] = by_class[k][torch.randint(0, by_class[k].numel(), (int(m.sum()),), generator=g)]
    x = 0.4 * torch.nn.functional.one_hot(y, c).float().repeat(1, d // c) + torch.randn(n, d, generator=g)
    perm = torch.randperm(n, generator=g)
    ei, x, y = torch.stack([src, dst]).to(DEV), x.to(DEV), y.to(DEV)
    parent = Graph(ei, n)
    train = NeighborSampler(parent, x, y, [15, 10, 5], 256, input_nodes=perm[:30000], shuffle=True,
                            generator=torch.Generator().manual_seed(1))
    valid = NeighborSampler(parent, x, y, [15, 10, 5], 1000, input_nodes=perm[30000:35000], generator=torch.Generator().manual_seed(2))
    model = _model(d, c, "fp32")
    opt = Adam(model.parameters(), lr=0.005, weight_decay=1e-5)
    losses, steps = [], 0
    while steps < 300:
        for mb in train:
            model.train()
            out = model(mb)[:mb.num_seeds]
            loss = torch.nn.functional.cross_entropy(out, mb.labels[:mb.num_seeds])
            opt.zero_grad()
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
            steps += 1
            if steps == 300:
                break
    correct = total = 0
    model.eval()
    with torch.no_grad():
        for mb in valid:
            out = model(mb)[:mb.num_seeds]
            correct += int((out.argmax(-1) == mb.labels[:mb.num_seeds]).sum())
            total += mb.num_seeds
    assert total == 5000
    assert np.mean(losses[-30:]) < 0.8 * np.mean(losses[:10]), (losses[:10], losses[-30:])
    assert correct / total > 0.5, f"validation accuracy {correct / total:.3f} (chance 0.25)"
