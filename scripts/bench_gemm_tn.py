#!/usr/bin/env python
"""Per-launch timing of the node-contracting GEMMs of the products-shaped step (1 GPU): every gemm_tn shape the step runs and
the gram of its attention, plus one bf16x3 gemm_tn at the arxiv shape.  CUDA events, tensors far larger than L2.  Prints one
line per case with the algorithmic bytes over the time, as a fraction of the HBM data-sheet bandwidth.

    python scripts/bench_gemm_tn.py [--rows 2449029] [--diag N | --lib PATH]

--diag N builds and times a diagnostic variant of csrc/gemm_tc.cu (SGF_TN_DIAG, wrong results): 1 = no mid-loop flush,
2 = no MMAs (loads only), 3 = no loads (MMAs only).  What each variant gains over the shipped kernel is what that part costs.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=2449029)
    ap.add_argument("--arxiv-rows", type=int, default=169343)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--peak", type=float, default=3350.0, help="HBM GB/s (default: H100 SXM data sheet)")
    ap.add_argument("--lib", default=None, help="alternative build of libsgformer_b200.so to time (A/B of kernel versions)")
    ap.add_argument("--diag", type=int, default=0, choices=[0, 1, 2, 3], help="time the SGF_TN_DIAG=N variant")
    args = ap.parse_args()
    from sgformer_b200 import _build
    if args.diag:
        args.lib = _build.build_variant(f"tndiag{args.diag}", [f"-DSGF_TN_DIAG={args.diag}"], only=("gemm_tc.cu",))
    if args.lib:
        _build.LIB_PATH = os.path.abspath(args.lib)
    from sgformer_b200 import kernels as K

    dev = torch.device("cuda:0")
    n, h, b = args.rows, 256, 2
    g = torch.Generator(device=dev).manual_seed(0)

    def act(rows, cols):
        return torch.randn(rows, cols, generator=g, device=dev).to(torch.bfloat16)

    x, dz = act(n, h), act(n, h)
    X, DZ = K.operand_from_bf16(x), K.operand_from_bf16(dz)
    X100 = K.pack_operand(torch.randn(n, 100, generator=g, device=dev), False, 1)       # input features (padded to 104)
    D47 = K.pack_operand(torch.randn(n, 47, generator=g, device=dev), False, 1)         # head output gradient (48)
    na = args.arxiv_rows
    A3 = K.pack_operand(torch.randn(na, h, generator=g, device=dev), False, 3)
    B3 = K.pack_operand(torch.randn(na, h, generator=g, device=dev), False, 3)
    o256, o100, o47 = (torch.empty(r, c, device=dev) for r, c in ((h, h), (h, 100), (47, h)))
    cases = [
        # (name, call, algorithmic bytes: every operand element read once)
        ("gemm_tn 256x256 (GraphConv dW)", lambda: K.gemm_tn(DZ, X, o256), n * (h + h) * b),
        ("gemm_tn 256x104 (input dW)", lambda: K.gemm_tn(DZ, X100, o100), n * (h + 104) * b),
        ("gemm_tn 48x256 (head dW)", lambda: K.gemm_tn(D47, X, o47), n * (48 + h) * b),
        ("gemm_tn 256x256 bf16x3 arxiv", lambda: K.gemm_tn(A3, B3, o256), na * 3 * (h + h) * b),
        ("gram h=256 (G = x^T x)", lambda: K.gram(X, x), n * h * b),
    ]
    name = f"diag{args.diag}" if args.diag else (os.path.basename(args.lib) if args.lib else "shipped")
    smi = os.popen("nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv,noheader 2>/dev/null").read().strip()
    print(f"[{name}] rows={n}  peak={args.peak} GB/s  gpu: {smi}")
    for label, fn, alg in cases:
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.reps
        print(f"[{name}] {label:32s} {ms:7.3f} ms  roofline {alg / args.peak / 1e6:6.3f} ms  "
              f"frac {alg / ms / 1e6 / args.peak:4.2f}", flush=True)


if __name__ == "__main__":
    main()
