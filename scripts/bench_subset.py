"""One mini-batch structure of a directed graph at the pokec shape (1.63 M nodes, 30.6 M edges, batch 100 000), built three ways:
  subset    Graph.subset(idx, capacity): sgf_csr_subset_pair, the batch's CSR and transposed CSR from the graph's (no host sync)
  edges     K.subgraph (sgf_subgraph, O(E) device mask) + sgf_csr_build of both orientations of the batch's edge list
  pyg_cpu   PyG subgraph(idx, edge_index, num_nodes=n, relabel_nodes=True) on the host (large/main-batch.py:139), restated in
            torch ops as torch_geometric 1.7.2 computes it; the reference then still copies the batch and builds its CSR
    python scripts/bench_subset.py [--reps 20]
Device times from CUDA events over `reps` calls after 3 warm-ups, the host time from perf_counter; checks first that the subset
pair equals the edge-list path bit for bit.  Prints one JSON line with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sgformer_b200 import kernels as K  # noqa: E402
from sgformer_b200.graph import Graph  # noqa: E402

N, E, B = 1_632_803, 30_622_564, 100_000


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in q.split(","))
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except (OSError, subprocess.CalledProcessError, IndexError, ValueError):
        return dict(gpu=torch.cuda.get_device_name(), power_limit="unknown", max_sm_clock="unknown")


def device_ms(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def pyg_subgraph_cpu(idx, ei, n):
    node_mask = torch.zeros(n, dtype=torch.bool)
    node_mask[idx] = True
    edge_mask = node_mask[ei[0]] & node_mask[ei[1]]
    out = ei[:, edge_mask]
    relabel = torch.zeros(n, dtype=torch.long)
    relabel[idx] = torch.arange(idx.numel())
    return relabel[out]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_subset.py measures on a CUDA device; none found")
    gen = torch.Generator(device="cuda").manual_seed(0)
    ei = torch.stack([torch.randint(0, N, (E,), generator=gen, device="cuda"),
                      torch.randint(0, N, (E,), generator=gen, device="cuda")])
    full = Graph(ei, N)
    full.transpose()
    idx = torch.randperm(N, generator=gen, device="cuda")[:B]

    exact = full.subset(idx)
    ei_sub = K.subgraph(ei, N, idx)
    rp, cl, dv = K.csr_build(ei_sub, B)
    rp_t, cl_t, _ = K.csr_build(ei_sub, B, True)
    assert torch.equal(exact.rowptr, rp) and torch.equal(exact.col, cl) and torch.equal(exact.dinv, dv)
    assert torch.equal(exact.transpose()[0], rp_t) and torch.equal(exact.transpose()[1], cl_t)
    nnz = int(exact.rowptr[-1])
    capacity = 2 * nnz          # a sampler's no-sync bound: twice what this batch needs

    t_subset = device_ms(lambda: full.subset(idx, capacity), args.reps)

    def edges():
        s = K.subgraph(ei, N, idx)
        K.csr_build(s, B)
        K.csr_build(s, B, True)
    t_edges = device_ms(edges, args.reps)

    ei_cpu, idx_cpu = ei.cpu(), idx.cpu()
    pyg_subgraph_cpu(idx_cpu, ei_cpu, N)
    reps_cpu = max(3, args.reps // 5)
    t0 = time.perf_counter()
    for _ in range(reps_cpu):
        pyg_subgraph_cpu(idx_cpu, ei_cpu, N)
    t_cpu = (time.perf_counter() - t0) / reps_cpu * 1e3

    print(json.dumps(dict(**card(), nodes=N, edges=E, batch=B, induced_nnz=nnz, capacity=capacity,
                          subset_pair_ms=round(t_subset, 4), subgraph_plus_builds_ms=round(t_edges, 4),
                          pyg_cpu_subgraph_ms=round(t_cpu, 2), host_threads=torch.get_num_threads())))


if __name__ == "__main__":
    main()
