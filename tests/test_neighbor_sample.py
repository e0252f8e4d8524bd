"""The neighbour sampler's semantics on the CPU: the numpy restatement of the device kernels (tests/neighbor_sample_ref.py) against a
brute-force statement of the rules on small graphs, the static buffer bounds, and the 100M SGFormer oracle on a sampled batch
against the reference's 100M/ours.py (tests/golden/neighbor_sample.pt, tests/make_golden_neighbor_sample.py)."""
import os

import numpy as np
import pytest
import torch

import neighbor_sample_ref as R
from oracle import sgformer_oracle as O

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "neighbor_sample.pt")


def small_graph():
    """12 nodes: node 11 isolated (no edges at all), node 10 has no in-edges, node 0 a row of 9 entries with a duplicate edge
    (3 -> 0 twice) and a self loop, seeds 0, 1, 2 are each other's neighbours, node 5 has one in-edge (deg < k)."""
    e = [(3, 0), (3, 0), (0, 0), (1, 0), (2, 0), (4, 0), (6, 0), (7, 0), (8, 0),
         (0, 1), (2, 1), (9, 1), (10, 1), (5, 5), (0, 2), (1, 2), (6, 3), (7, 3), (8, 3), (10, 4),
         (4, 5), (9, 6), (2, 7), (3, 8), (5, 9), (6, 9), (10, 9), (9, 9)]
    s, t = zip(*e)
    return np.array([s, t], dtype=np.int64), 12


CASES = [([0, 1, 2], [2, 2]), ([11, 0], [3, 1]), ([5], [1, 1, 1]), ([0, 4, 11, 9], [-1, 2]), ([3, 10], [-1, -1]),
         ([0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11], [15, 10, 5]), ([2, 8], [64]), ([], [2, 2]), ([7], [0, 3])]


@pytest.mark.parametrize("seeds,fanouts", CASES)
@pytest.mark.parametrize("seed", [0, 1, 0xDEADBEEF12345])
def test_restatement_matches_brute_force(seeds, fanouts, seed):
    edges, n = small_graph()
    rowptr, col = R.csr_of(edges, n)
    idx, ei, _ = R.sample(rowptr, col, np.array(seeds, dtype=np.int64), fanouts, seed, capacity=20)
    idx_b, ei_b = R.brute_force(edges, n, seeds, fanouts, seed, capacity=20)
    assert idx.tolist() == idx_b.tolist()
    assert ei.tolist() == ei_b.tolist()
    assert idx[:len(seeds)].tolist() == list(seeds) and len(set(idx.tolist())) == idx.size
    if ei.size:      # every edge is a drawn entry: source -> target is an edge of the parent
        parent = {(int(s), int(t)) for s, t in edges.T}
        assert all((int(idx[s]), int(idx[t])) in parent for s, t in ei.T)


def test_rules_on_random_graphs():
    """Per target: min(k, deg) distinct entry positions, every entry when deg <= k or k = -1, and a node seen only at the last hop
    has no in-edges in the batch."""
    rng = np.random.default_rng(0)
    for trial in range(20):
        n = int(rng.integers(5, 60))
        e = int(rng.integers(0, 6 * n))
        edges = rng.integers(0, n, (2, e))
        rowptr, col = R.csr_of(edges, n)
        seeds = rng.permutation(n)[:int(rng.integers(0, n))]
        fan = [int(rng.integers(-1, 6)) for _ in range(int(rng.integers(1, 4)))]
        idx, ei, need = R.sample(rowptr, col, seeds, fan, trial, capacity=10 ** 6)
        idx_b, ei_b = R.brute_force(edges, n, seeds.tolist(), fan, trial, capacity=10 ** 6)
        assert idx.tolist() == idx_b.tolist() and ei.tolist() == ei_b.tolist()
        indeg = np.bincount(ei[1], minlength=idx.size)
        deg = rowptr[idx + 1] - rowptr[idx]
        assert (indeg <= deg).all()
        b = seeds.size      # the seeds are hop 0's frontier: each takes min(k_0, deg) entries
        assert indeg[:b].tolist() == [int(d) if fan[0] < 0 else min(fan[0], int(d)) for d in deg[:b]]
        if len(fan) == 1:   # nodes first seen at the last hop are not expanded
            assert (indeg[b:] == 0).all()


def test_floyd_positions_are_distinct_and_vectorised_equals_scalar():
    for k, deg in [(1, 2), (5, 6), (15, 16), (15, 100000), (64, 65), (64, 3000)]:
        vs = np.arange(50) * 7919
        P = R.hop_positions(123, 2, vs, np.full(50, deg), k)
        for r, v in enumerate(vs):
            assert P[r].tolist() == R.row_positions(123, 2, int(v), deg, k, k)
            assert len(set(P[r].tolist())) == k and P[r].min() >= 0 and P[r].max() < deg


def test_static_bounds():
    from sgformer_b200.kernels import neighbor_sample_plan
    p = neighbor_sample_plan(1000, [15, 10, 5])
    assert p.max_nodes == 1000 * (1 + 15 + 150 + 750) and p.max_edges == 1000 * (15 + 150 + 750)
    assert p.frontier_caps == (1000, 15000, 150000) and p.slot_offsets == (0, 15000, 165000)
    q = neighbor_sample_plan(8, [-1, 2], capacity=100)
    assert q.widths == (100, 2) and q.max_edges == 8 * 100 + 800 * 2
    with pytest.raises(ValueError, match="capacity"):
        neighbor_sample_plan(8, [-1])
    with pytest.raises(ValueError, match="2\\^31"):
        neighbor_sample_plan(100000, [100, 100, 100])


def test_100M_oracle_on_a_sampled_batch_matches_reference():
    fx = torch.load(GOLD, weights_only=False)
    rowptr, col = R.csr_of(fx["edge_index"].numpy(), fx["n"])
    idx, ei, _ = R.sample(rowptr, col, fx["seeds"].numpy(), fx["num_neighbors"], fx["seed"])
    assert idx.tolist() == fx["idx"].tolist() and ei.tolist() == fx["sampled_edge_index"].tolist()
    indeg = np.bincount(ei[1], minlength=idx.size)
    assert (indeg == 0).any() and (indeg > 0).any()      # last-hop nodes carry no in-edges
    out = O.sgformer_forward(fx["cfg"], fx["state_dict"], fx["x"][fx["idx"]], fx["sampled_edge_index"], training=False)
    err = (out.double() - fx["out_eval"].double()).abs().max().item()
    assert err <= 1e-5 * max(1.0, fx["out_eval"].abs().max().item()), err
