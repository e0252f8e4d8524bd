#!/usr/bin/env python
"""Per-launch timing of the row-streaming kernels (rowops.cu) at the products shape (2 449 029 rows, h = 256), in bf16 and
fp32, each next to a device-to-device copy (cudaMemcpyAsync via Tensor.copy_) of the same number of bytes: the copy reads
and writes bytes / 2 each.  CUDA events, tensors far larger than L2.  Algorithmic bytes = every activation read or
written once (row statistics and per-row vectors included).

    python scripts/bench_rowops.py [--rows 2449029] [--dtypes bf16,fp32] [--reps 5]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from sgformer_b200 import kernels as K  # noqa: E402


def timed(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def cases(n, h, dt, dev):
    g = torch.Generator(device=dev).manual_seed(0)

    def act():
        return torch.randn(n, h, generator=g, device=dev).to(dt)

    def vec(m, lo=0.5, hi=1.5):
        return torch.rand(m, generator=g, device=dev) * (hi - lo) + lo

    x, r, o, dy, dy2, z, res = (act() for _ in range(7))
    gamma, beta, mean, rstd = vec(h), vec(h, -0.5, 0.5), vec(h, -0.1, 0.1), vec(h)
    dinv, den = vec(n), vec(n)
    _, stats = K.ln_fwd(x, r, 0.5, 0.5, gamma, beta, True, False, 0.0, 0)
    dg, db = torch.zeros(h, device=dev), torch.zeros(h, device=dev)
    sums = K.bn_bwd_sums(dy, dy2, dinv, z, mean, rstd, gamma, beta, None, True, True, 0.0, 0, 1.0)
    A, b = n * h * x.element_size(), 4 * n          # one activation, one fp32 per-row value

    def bn_fwd(res_, mix, want_y, want_s):
        return K.bn_fwd(z, res_, mix, mean, rstd, gamma, beta, None, True, True, 0.0, 0, 0.5, dinv, want_y, want_s)

    def bn_apply(dy_, dy2_, dres=None):
        return K.bn_bwd(dy_, dy2_, dinv if dy2_ is not None else None, z, mean, rstd, gamma, beta, None, True, True, True,
                        0.0, 0, 1.0, dres=dres, dres_accumulate=dres is not None, want_dz_colsum=True)

    acc = act()
    return [
        ("colstats", lambda: K.colstats(z), A),
        ("ln_fwd  x,r -> y", lambda: K.ln_fwd(x, r, 0.5, 0.5, gamma, beta, True, False, 0.0, 0), 3 * A + 2 * b),
        ("ln_fwd_graph x,r,gy -> y", lambda: K.ln_fwd_graph(x, r, o, 0.5, 0.5, 0.3, gamma, beta, True, False, 0.0, 0),
         4 * A + 2 * b),
        ("ln_bwd  dy,x,r -> dx,dr", lambda: K.ln_bwd(dy, x, r, 0.5, 0.5, gamma, beta, stats, True, False, 0.0, 0, 1.0, True,
                                                     dg, db), 5 * A + 2 * b),
        ("ln_bwd_attn dy,o,r -> gnum,dr", lambda: K.ln_bwd_attn(dy, o, r, r, 0.5, 0.5, gamma, beta, stats, True, False, 0.0,
                                                                  0, 1.0, True, dg, db, den), 5 * A + 4 * b),
        ("bn_fwd stem z -> y,ys", lambda: bn_fwd(None, None, True, True), 3 * A + b),
        ("bn_fwd layer z,res -> ys", lambda: bn_fwd(res, None, False, True), 3 * A + b),
        ("bn_fwd last z,res,mix -> y", lambda: bn_fwd(res, x, True, False), 4 * A),
        ("bn_bwd_reduce dy,dy2,z", lambda: K.bn_bwd_sums(dy, dy2, dinv, z, mean, rstd, gamma, beta, None, True, True, 0.0, 0,
                                                         1.0), 3 * A + b),
        # training-mode bn_bwd = the reduce pass and the apply pass
        ("bn_bwd reduce+apply dy,dy2,z -> dz", lambda: bn_apply(dy, dy2), 7 * A + 2 * b),
        ("bn_bwd reduce+apply dy2,z,dres -> dz,dres+=", lambda: bn_apply(None, dy2, acc), 7 * A + 2 * b),
    ], sums


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=2449029)
    ap.add_argument("--h", type=int, default=256)
    ap.add_argument("--dtypes", default="bf16,fp32")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--peak", type=float, default=3350.0, help="HBM GB/s (default: H100 SXM data sheet)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_rowops.py needs a CUDA device")
    dev = torch.device("cuda:0")
    n, h = args.rows, args.h
    print(f"{torch.cuda.get_device_name(0)}; rows={n} h={h}  peak={args.peak} GB/s (fraction columns are of this)")
    for name in args.dtypes.split(","):
        dt = {"bf16": torch.bfloat16, "fp32": torch.float32}[name]
        cs, _ = cases(n, h, dt, dev)
        big = max(bts for _, _, bts in cs)
        src = torch.empty(big // 2 + 16, dtype=torch.uint8, device=dev)
        dst = torch.empty_like(src)
        for label, fn, bts in cs:
            ms = timed(fn, args.reps)
            half = bts // 2
            cms = timed(lambda: dst[:half].copy_(src[:half]), args.reps)
            print(f"{name} {label:38s} {ms:7.3f} ms  {bts / 1e9:6.2f} GB  {bts / ms / 1e6 / args.peak:5.2f} of peak | "
                  f"copy {cms:7.3f} ms ({bts / cms / 1e6 / args.peak:4.2f})  kernel/copy {ms / cms:5.2f}", flush=True)
        del cs, src, dst
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
