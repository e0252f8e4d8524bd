#!/usr/bin/env python
"""Per-launch timing of the CSR SpMM on a synthetic graph of a BASELINE shape (1 GPU, CUDA events), optionally for an
alternative build of the library (tuning variants from sgformer_b200._build.build_variant).

    python scripts/bench_spmm.py [--workload products] [--lib sgformer_b200/lib/libsgformer_b200_<name>.so]
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


if __name__ == "__main__":
    main()
