#!/usr/bin/env python
"""Per-launch timing of the gemm_nt shapes of the products-shaped step (1 GPU), for every schedule of
sgf_gemm_nt_args.schedule.  CUDA events, tensors far larger than L2.  Prints one line per (case, schedule) with the
HBM-roofline time of the algorithmic bytes next to it.

    python scripts/bench_gemm_nt.py [--rows 2449029] [--schedules 1,2]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from sgformer_b200 import kernels as K  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=2449029)
    ap.add_argument("--schedules", default="1,2")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--peak", type=float, default=3350.0, help="HBM GB/s (default: H100 SXM data sheet)")
    ap.add_argument("--lib", default=None, help="alternative build of libsgformer_b200.so to time (A/B of kernel versions)")
    args = ap.parse_args()
    if args.lib:
        from sgformer_b200 import _build
        _build.LIB_PATH = os.path.abspath(args.lib)
    dev = torch.device("cuda:0")
    n, h = args.rows, 256
    g = torch.Generator(device=dev).manual_seed(0)

    def act(cols):
        return torch.randn(n, cols, generator=g, device=dev).to(torch.bfloat16)

    def weight(rows, cols):
        return K.pack_operand(torch.randn(rows, cols, generator=g, device=dev) / cols ** 0.5, False, 1)

    x, x0, v = act(h), act(h), act(h)
    x100 = K.pack_operand(torch.randn(n, 100, generator=g, device=dev), False, 1)
    X, X0 = K.operand_from_bf16(x), K.operand_from_bf16(x0)
    w256, w768, w512, w100, w47 = weight(h, h), weight(3 * h, h), weight(h, 2 * h), weight(h, 100), weight(47, h)
    bias256, bias768, bias47 = (torch.randn(c, device=dev) for c in (h, 3 * h, 47))
    rs = torch.rand(n, device=dev)
    sdev = torch.tensor([0.5], device=dev)
    s_raw, z_raw = torch.randn(h, h, device=dev), torch.randn(h, device=dev)
    nq2, nk2 = torch.rand(h, device=dev) * n, torch.rand(h, device=dev) * n
    bmat, btail, _ = K.attn_prepare_fwd(s_raw, z_raw, nq2, nk2, 1)
    out256, out768 = K.alloc_act(n, h, torch.bfloat16, dev), K.alloc_act(n, 3 * h, torch.bfloat16, dev)
    out47 = torch.empty(n, 47, device=dev)
    den = torch.empty(n, device=dev)
    b = 2
    cases = [
        ("plain 256->256 +bias", lambda s: K.gemm_nt([X], [w256], [(0, 0, 0, 0, h)], h, out256, bias=bias256, schedule=s),
         n * (h + h) * b),
        ("row_scale 256->256", lambda s: K.gemm_nt([X], [w256], [(0, 0, 0, 0, h)], h, out256, row_scale=rs, schedule=s),
         n * (h + h) * b),
        ("accumulate 256->256", lambda s: K.gemm_nt([X], [w256], [(0, 0, 0, 0, h)], h, out256, accumulate=True, schedule=s),
         n * (h + 2 * h) * b),
        ("aux(beta) 256->256", lambda s: K.gemm_nt([X], [w256], [(0, 0, 0, 0, h)], h, out256, aux=v, beta=1.0, alpha_dev=sdev,
                                                   schedule=s), n * (h + 2 * h) * b),
        ("qkv 256->768 +bias", lambda s: K.gemm_nt([X], [w768], [(0, 0, 0, 0, h)], 3 * h, out768, bias=bias768, schedule=s),
         n * (h + 3 * h) * b),
        ("concat 512->256 +bias", lambda s: K.gemm_nt([X, X0], [w512], [(0, 0, 0, 0, h), (1, 0, 0, h, h)], h, out256,
                                                      bias=bias256, schedule=s), n * (2 * h + h) * b),
        ("attn apply 256->256", lambda s: K.gemm_nt([X], [bmat], [(0, 0, 0, 0, h)], h, out256, epi=1, aux=v, tail=btail,
                                                    nf=float(n), den_out=den, schedule=s), n * (3 * h) * b + n * 4),
        ("fcs0 100->256 relu", lambda s: K.gemm_nt([x100], [w100], [(0, 0, 0, 0, 100)], h, out256, bias=bias256, relu=True,
                                                   schedule=s), n * (104 + h) * b),
        ("head 256->47 fp32", lambda s: K.gemm_nt([X], [w47], [(0, 0, 0, 0, h)], 47, out47, bias=bias47, schedule=s),
         n * (h * b + 47 * 4)),
    ]
    scheds = [int(s) for s in args.schedules.split(",")]
    print(f"rows={n}  peak={args.peak} GB/s")
    for name, fn, alg_bytes in cases:
        line = f"{name:26s} roofline {alg_bytes / args.peak / 1e6:6.3f} ms |"
        for s in scheds:
            try:
                for _ in range(2):
                    fn(s)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.reps):
                    fn(s)
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / args.reps
                line += f"  sched{s}: {ms:6.3f} ms ({alg_bytes / ms / 1e6 / args.peak:4.2f})"
            except RuntimeError as exc:
                line += f"  sched{s}: {str(exc)[:40]}"
        print(line, flush=True)


if __name__ == "__main__":
    main()
