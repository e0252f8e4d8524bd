"""The induced subset of a self_loop_mode 1 graph (Graph.subset of the structure GCN(save_mem=False) and GAT build), and the
count contract of sgformer_b200.eval.evaluate_batch, checked without a GPU.

The mode-1 contract, stated in torch: the subset of a mode-1 parent at the distinct nodes idx is PyG `subgraph(idx,
relabel_nodes=True)` followed by PyG `add_remaining_self_loops` (every self loop of the batch dropped, duplicates included, and
one added per node) as a CSR with rows sorted by source, and dinv = (1/deg).sqrt() (0 for an empty row) of gcn_norm's degree.
The subset kernels need no rule of their own for it (csr.cu, subset_half); the CPU statement of those kernels
(tests/test_subset_directed.py) applied to the emulated mode-1 parent CSR must meet the contract bit for bit.  The CUDA kernels
are compared with the edge-list path in tests/test_gpu_subset_mode1.py."""
import os
import sys

import pytest
import torch

import kernel_emu as emu
from make_golden_eval_batch import CASES, RoundedSum, make_case, split_logits
from sgformer_b200 import graph as G
from test_gpu_eval_batch import evaluate_batch_restated, split_counts
from test_subset_directed import EmuKernels, pyg_subgraph

HERE = os.path.dirname(os.path.abspath(__file__))


def pyg_utils():
    sys.path.insert(0, os.path.join(HERE, "ref_shims"))
    try:
        from torch_geometric import utils                      # CPU restatement of PyG 1.7.2
    finally:
        sys.path.pop(0)
    return utils


def mode1_contract(ei, n, idx):
    """(rowptr, col, dinv, rowptr_t, col_t) of the batch idx: subgraph -> add_remaining_self_loops -> CSR of each orientation."""
    U = pyg_utils()
    b = idx.numel()
    ei_b, _ = U.add_remaining_self_loops(pyg_subgraph(idx, ei, n), num_nodes=b)
    out = []
    for key, val in ((ei_b[1], ei_b[0]), (ei_b[0], ei_b[1])):
        order = torch.argsort(key * max(b, 1) + val, stable=True)
        rowptr = torch.zeros(b + 1, dtype=torch.int64)
        rowptr[1:] = torch.cumsum(torch.bincount(key, minlength=b), 0)
        out += [rowptr, val[order].to(torch.int32)]
    deg = U.degree(ei_b[1], b, dtype=torch.float32)            # gcn_norm's degree: the count of entries per target row
    dinv = torch.where(deg > 0, (1.0 / deg).sqrt(), torch.zeros_like(deg))
    return out[0], out[1], dinv, out[2], out[3]


def parent_graph(ei, n, symmetric):
    """A mode-1 Graph of `ei` built by the CPU statement of sgf_csr_build (and its transpose for a directed edge list)."""
    rp, cl, dv = emu.csr_build(ei, n, self_loop_mode=1)
    g = G.Graph._from_parts(n, rp, cl, dv, symmetric, 1)
    if not symmetric:
        rp_t, cl_t, _ = emu.csr_build(ei, n, by_source=True, self_loop_mode=1)
        g._t = (rp_t, cl_t)
    g.edge_index = ei
    return g


def edges(n, e, seed, symmetric, loops, isolated=0):
    g = torch.Generator().manual_seed(seed)
    ei = torch.randint(0, n - isolated, (2, e), generator=g)
    ei = torch.cat([ei, ei[:, : e // 10]], 1)                  # duplicate edges
    if symmetric:
        ei = torch.cat([ei, ei.flip(0)], 1)
    ar = torch.arange(n - isolated)
    if loops == "none":
        ei = ei[:, ei[0] != ei[1]]
    elif loops == "dup":                                        # every node's loop three times
        ei = torch.cat([ei, torch.stack([ar, ar]).repeat(1, 3)], 1)
    elif loops == "some":                                       # loops on every 5th node, twice on every 10th
        ei = torch.cat([ei, torch.stack([ar[::5], ar[::5]]), torch.stack([ar[::10], ar[::10]])], 1)
    return ei[:, torch.randperm(ei.shape[1], generator=g)].contiguous()


@pytest.mark.parametrize("symmetric", [True, False])
@pytest.mark.parametrize("loops", ["none", "dup", "some"])
def test_emulated_mode1_subset_meets_the_contract(monkeypatch, symmetric, loops):
    monkeypatch.setattr(G, "K", EmuKernels)
    n = 400
    ei = edges(n, 2500, 3, symmetric, loops, isolated=23)
    parent = parent_graph(ei, n, symmetric)
    gen = torch.Generator().manual_seed(7)
    batches = [torch.zeros(0, dtype=torch.int64), torch.tensor([n - 1]), torch.tensor([n - 1, n - 2, 0]),
               torch.randperm(n, generator=gen)[:n // 3], torch.randperm(n, generator=gen), torch.arange(n)]
    for idx in batches:
        b = idx.numel()
        sub = parent.subset(idx)
        rp, cl, dv, rp_t, cl_t = mode1_contract(ei, n, idx)
        assert sub.self_loop_mode == 1 and sub.heavy is None and sub.heavy_t is None
        assert torch.equal(sub.rowptr, rp) and torch.equal(sub.col, cl), f"b={b}: CSR differs"
        assert torch.equal(sub.dinv, dv), f"b={b}: dinv differs"
        sub_t = sub.transpose()
        assert (sub_t[0] is sub.rowptr) == symmetric
        assert torch.equal(sub_t[0], rp_t) and torch.equal(sub_t[1], cl_t), f"b={b}: transposed CSR differs"
        # the emulated mode-1 build of the batch's edge list is the same structure (what the edge-list path computes)
        rp_b, cl_b, dv_b = emu.csr_build(pyg_subgraph(idx, ei, n), b, self_loop_mode=1)
        assert torch.equal(rp_b, rp) and torch.equal(cl_b, cl) and torch.equal(dv_b, dv)
        # one loop per row, whatever the parent's edge list held
        rows = torch.repeat_interleave(torch.arange(b), rp[1:] - rp[:-1])
        assert torch.equal(torch.bincount(rows[cl.long() == rows], minlength=b), torch.ones(b, dtype=torch.int64))
        assert int(sub.nnz_needed) == int(sub.nnz_needed_t) == int(rp[-1])
        assert bool((parent._node_map == -1).all())


def test_mode1_dinv_is_gcn_norms_degree():
    """The kernels' dinv, (1/deg).sqrt(), is gcn_norm's deg^-1/2 of the same degrees to within one rounding."""
    U = pyg_utils()
    sys.path.insert(0, os.path.join(HERE, "ref_shims"))
    try:
        from torch_geometric.nn.conv.gcn_conv import gcn_norm
    finally:
        sys.path.pop(0)
    n = 300
    ei = edges(n, 2000, 5, False, "some", isolated=10)
    idx = torch.randperm(n, generator=torch.Generator().manual_seed(1))[:150]
    rp, cl, dv, _, _ = mode1_contract(ei, n, idx)
    ei_b, w = gcn_norm(pyg_subgraph(idx, ei, n), None, 150)
    deg = U.degree(ei_b[1], 150, dtype=torch.float32)
    assert torch.equal(deg, (rp[1:] - rp[:-1]).float())
    torch.testing.assert_close(dv, deg.pow(-0.5), rtol=2e-7, atol=0)
    torch.testing.assert_close(w, dv[ei_b[0]] * dv[ei_b[1]], rtol=1e-6, atol=0)


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(HERE, "golden", "eval_batch.pt"))


@pytest.mark.parametrize("case", list(CASES))
def test_split_counts_match_reference_eval_acc(golden, case):
    """The count contract of sgf_eval_acc_splits (split_counts, the torch count tests/test_gpu_eval_batch.py checks the kernel
    with) equals, split by split, the (rows, hits) of the reference's eval_acc on the same logits, planted ties included."""
    n, _, c, _, seed, _ = CASES[case]
    logits, label, code = split_logits(n, c, seed)
    counts = split_counts(logits, label, code, torch.arange(n))
    assert [tuple(counts[2 * k:2 * k + 2]) for k in range(3)] == [tuple(t) for t in golden[case]["eval_acc"]]


@pytest.mark.parametrize("case", list(CASES))
def test_restated_evaluate_batch_matches_reference(golden, case):
    """evaluate_batch_restated (the torch restatement of large/eval.py:67-118 the GPU test compares evaluate_batch with), fed
    PyG `subgraph` edge lists on the CPU, returns exactly the reference's own evaluate_batch accuracies under the same seed -
    with a partial last batch, an empty last batch and overlapping splits."""
    n, e, c, bs, seed, overlap = CASES[case]
    d = make_case(n, e, c, seed, overlap)
    model = RoundedSum(d["x"].shape[1], c, seed)
    torch.manual_seed(golden[case]["torch_seed"])
    got = evaluate_batch_restated(model, d["x"], d["edge_index"], n, d["label"], d["split"], bs,
                                  lambda ei, n_, idx: pyg_subgraph(idx, ei, n_))
    assert got == tuple(golden[case]["accuracies"])
