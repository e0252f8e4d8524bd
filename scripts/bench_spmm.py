#!/usr/bin/env python
"""Per-launch timing of the CSR SpMM on a synthetic graph of a BASELINE shape (1 GPU, CUDA events), optionally for an
alternative build of the library (tuning variants from sgformer_b200._build.build_variant).

    python scripts/bench_spmm.py [--workload products] [--lib sgformer_b200/lib/libsgformer_b200_<name>.so] [--weighted]

--weighted also times the weighted SpMM (edge_weight, sgf_spmm_weighted) on the same graph with random weights, alternating it
with the unweighted one, and prints the card's name and power limit beside the numbers.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="products")
    ap.add_argument("--lib", default=None)
    ap.add_argument("--reps", type=int, default=6)
    ap.add_argument("--peak", type=float, default=3350.0, help="HBM GB/s (default: H100 SXM data sheet)")
    ap.add_argument("--check", action="store_true", help="compare with the main build's result (bitwise)")
    ap.add_argument("--weighted", action="store_true", help="also time the weighted SpMM (value array) against the unweighted one")
    args = ap.parse_args()
    if args.lib:
        from sgformer_b200 import _build
        _build.LIB_PATH = os.path.abspath(args.lib)
    from sgformer_b200 import kernels as K
    from sgformer_b200.graph import Graph
    from sgformer_b200.synth import SHAPES, make_graph
    dev = torch.device("cuda:0")
    n, _, e, _, h, _, _ = SHAPES[args.workload]
    ei = make_graph(n, e, seed=100, device=dev)
    g = Graph(ei, n)
    x = torch.randn(n, h, device=dev).to(torch.bfloat16)
    y = torch.empty_like(x)
    nnz = g.nnz
    alg = nnz * 4 + (n + 1) * 8 + nnz * h * 2 + n * h * 2
    if args.weighted:
        return bench_weighted(args, K, Graph, ei, n, h, x, y)
    for _ in range(2):
        K.spmm(g.rowptr, g.col, g.dinv, x, out=y)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.reps):
        K.spmm(g.rowptr, g.col, g.dinv, x, out=y)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.reps
    chk = float(y.float().abs().sum().item())
    print(f"{os.path.basename(args.lib) if args.lib else 'main':40s} n={n} nnz={nnz} h={h}: {ms:7.3f} ms/launch  "
          f"{alg / ms / 1e6:7.1f} GB/s algorithmic = {alg / ms / 1e6 / args.peak:5.3f} of the measured peak   checksum {chk:.6e}",
          flush=True)


def bench_weighted(args, K, Graph, ei, n, h, x, y):
    import subprocess
    dev = x.device
    w = torch.rand(ei.shape[1], device=dev, generator=torch.Generator(device=dev).manual_seed(5))
    gu = Graph(ei, n, 1)
    gw = Graph(ei, n, 1, edge_weight=w)
    nnz = gw.nnz
    runs = {"unweighted": lambda: K.spmm(gu.rowptr, gu.col, gu.dinv, x, out=y, heavy=gu.heavy),
            "weighted": lambda: K.spmm(gw.rowptr, gw.col, gw.dinv, x, out=y, heavy=gw.heavy, val=gw.val)}
    alg = {"unweighted": nnz * 4 + (n + 1) * 8 + nnz * h * 2 + n * h * 2,
           "weighted": nnz * 8 + (n + 1) * 8 + nnz * h * 2 + n * h * 2}
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    for f in runs.values():
        for _ in range(2):
            f()
    torch.cuda.synchronize()
    times = {k: [] for k in runs}
    for _ in range(3):                  # alternate the two variants
        for k, f in runs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                f()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / args.reps)
    print(f"card: {card}", flush=True)
    for k in runs:
        ms = min(times[k])
        print(f"{k:10s} n={n} nnz={nnz} h={h} bf16: {ms:7.3f} ms/launch (best of 3 x {args.reps}; all {['%.3f' % t for t in times[k]]})  "
              f"{alg[k] / ms / 1e6:7.1f} GB/s algorithmic = {alg[k] / ms / 1e6 / args.peak:5.3f} of {args.peak:.0f} GB/s", flush=True)


if __name__ == "__main__":
    main()
