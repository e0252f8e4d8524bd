"""Time per neighbour-sampled batch (minibatch.NeighborSampler, 100M/nb-sample.py's NeighborLoader(num_neighbors=[15, 10, 5],
batch_size=1000)) on a synthetic papers100M-shaped slice, split into the sampling stage (draws + relabel + edge list) and the batch
structure (sgf_csr_build of both orientations), against the numpy restatement (tests/neighbor_sample_ref.py) on the host.
    python scripts/bench_neighbor_sample.py [--nodes 4000000] [--avg-deg 30] [--batches 50] [--out DIR]
Prints one JSON line (GPU name and power limit included) and writes it to DIR/bench_neighbor_sample.json when --out is given."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=4_000_000)
    ap.add_argument("--avg-deg", type=int, default=30)
    ap.add_argument("--batch-size", type=int, default=1000)
    ap.add_argument("--batches", type=int, default=50)
    ap.add_argument("--host-batches", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_neighbor_sample needs a CUDA device")
    from sgformer_b200 import kernels as K
    from sgformer_b200.graph import Graph
    from sgformer_b200.minibatch import NeighborSampler
    import neighbor_sample_ref as R

    n, e = a.nodes, a.nodes * a.avg_deg // 2
    g = torch.Generator(device="cuda").manual_seed(0)
    # skewed degrees both ways (sources and targets ~ u^2), symmetrised as nb-sample.py does with to_undirected
    src = (n * torch.rand(e, device="cuda", generator=g) ** 2).long().clamp_(max=n - 1)
    dst = torch.randint(0, n, (e,), device="cuda", generator=g)
    ei = torch.cat([torch.stack([src, dst]), torch.stack([dst, src])], 1)
    del src, dst
    graph = Graph(ei, n)
    del ei
    torch.cuda.synchronize()
    x = torch.randn(n, 128, device="cuda")
    fan = [15, 10, 5]
    s = NeighborSampler(graph, x, None, fan, a.batch_size, shuffle=True, generator=torch.Generator().manual_seed(1))
    plan, node_map = s.plan, graph._sample_map
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(2)).cuda()
    seed_sets = [perm[i * a.batch_size:(i + 1) * a.batch_size] for i in range(a.batches)]

    for sd in seed_sets[:5]:                       # warm-up
        s.batch(sd)
    torch.cuda.synchronize()
    # whole batches as yielded (kernels, count read-back, feature gather)
    t0 = time.perf_counter()
    sizes = []
    for sd in seed_sets:
        mb = s.batch(sd)
        sizes.append((mb.idx.numel(), mb.graph.col.numel()))
    torch.cuda.synchronize()
    per_batch_ms = (time.perf_counter() - t0) * 1e3 / a.batches

    # stage split by CUDA events: sampling (begin, hops, relabel, edges) | structure (both sgf_csr_build calls)
    samp, struct = [], []
    for i, sd in enumerate(seed_sets):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        ev[0].record()
        idx = torch.empty(plan.max_nodes, dtype=torch.int64, device="cuda")
        rowlen = torch.empty(plan.max_nodes, dtype=torch.int32, device="cuda")
        bounds = torch.empty(len(fan) + 2, dtype=torch.int64, device="cuda")
        cand = torch.empty(plan.max_edges, dtype=torch.int32, device="cuda")
        ein = torch.empty((2, plan.max_edges), dtype=torch.int64, device="cuda")
        counts = torch.empty(2, dtype=torch.int64, device="cuda")
        ws, wsb = K._ns_ws(plan, "cuda")
        K.check(K.lib().sgf_neighbor_begin(K._p(sd), sd.numel(), K._p(node_map), K._p(idx), K._p(bounds), K._p(rowlen),
                                           plan.max_nodes, K._stream()), "begin")
        for t in range(len(fan)):
            c = cand[plan.slot_offsets[t]:]
            K.neighbor_sample_hop(graph.rowptr, graph.col, idx, bounds, plan, t, 1234 + i, c, rowlen)
            K.neighbor_sample_relabel(c, rowlen, bounds, plan, t, node_map, idx, ws, wsb)
        K.neighbor_sample_edges(cand, plan, bounds, rowlen, node_map, idx, ein, counts, ws, wsb)
        ev[1].record()
        K.neighbor_sample(graph.rowptr, graph.col, node_map, sd, plan, 1234 + i)   # full path again; structure = difference
        ev[2].record()
        torch.cuda.synchronize()
        samp.append(ev[0].elapsed_time(ev[1]))
        struct.append(ev[1].elapsed_time(ev[2]) - ev[0].elapsed_time(ev[1]))
    samp.sort(); struct.sort()

    rowptr, col = graph.rowptr.cpu().numpy(), graph.col.cpu().numpy()
    t0 = time.perf_counter()
    for i in range(a.host_batches):
        R.sample(rowptr, col, seed_sets[i].cpu().numpy(), fan, 99 + i)
    host_ms = (time.perf_counter() - t0) * 1e3 / a.host_batches

    res = dict(bench="neighbor_sample", gpu=gpu_info(), nodes=n, edges=int(graph.col.numel()), batch_size=a.batch_size,
               num_neighbors=fan, batches=a.batches, per_batch_ms=round(per_batch_ms, 3),
               sampling_ms_median=round(samp[len(samp) // 2], 3), structure_ms_median=round(struct[len(struct) // 2], 3),
               mean_batch_nodes=int(sum(b for b, _ in sizes) / len(sizes)), mean_batch_edges=int(sum(e for _, e in sizes) / len(sizes)),
               max_nodes=plan.max_nodes, max_edges=plan.max_edges, host_restatement_ms=round(host_ms, 1))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_neighbor_sample.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
