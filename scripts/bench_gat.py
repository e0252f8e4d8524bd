"""GAT layer micro-benchmark on the GPU: the kernels (projection GEMM + sgf_gat_logits + sgf_gat_fwd) against the plain-torch
GATConv restatement (oracle/gat_oracle.py) run as torch ops on the same GPU, on random graphs of the Cora / Actor / ogbn-arxiv
shapes with H = 8 heads of 64 channels (models.GAT's first layer at --hidden_channels 64 --gat_heads 8).  Reports the layer times,
sgf_gat_fwd's time and its algorithmic bytes/s against the H100 SXM's 3.35 TB/s, and the card's name and power limit.

    python scripts/bench_gat.py [--iters 50] [--precision fp32|bf16] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import gat_oracle as G  # noqa: E402
from sgformer_b200 import kernels as K  # noqa: E402
from sgformer_b200.graph import Graph  # noqa: E402

SHAPES = {"cora": (2708, 10556, 1433), "actor": (7600, 30019, 932), "arxiv": (169343, 2315598, 128)}
HBM_BPS = 3.35e12


def _time(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def fwd_bytes(n, nnz, heads, c, elt):
    """rowptr, column ids, a_src gathered per edge, x' rows gathered per edge, a_dst, out, lse.  Every gathered x' row is counted:
    when x' fits the 50 MB L2 (Cora, Actor shapes) the rate is an L2-served one, not a share of HBM bandwidth."""
    return (n + 1) * 8 + nnz * 4 + nnz * heads * 4 + nnz * heads * c * elt + n * heads * 4 + n * heads * c * elt + n * heads * 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--precision", choices=["fp32", "bf16"], default="fp32")
    ap.add_argument("--heads", type=int, default=8)
    ap.add_argument("--channels", type=int, default=64)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gat.py needs a CUDA GPU")
    dev = "cuda"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = smi.stdout.strip()
    H, C = a.heads, a.channels
    act = torch.bfloat16 if a.precision == "bf16" else torch.float32
    planes = 1 if a.precision == "bf16" else 3
    rows = []
    for name, (n, e, d) in SHAPES.items():
        g = torch.Generator().manual_seed(0)
        ei = torch.randint(0, n, (2, e), generator=g).to(dev)
        x = torch.randn(n, d, device=dev)
        conv = G.GATConv(d, C, heads=H).to(dev)
        graph = Graph(ei, n, 1)
        nnz = graph.nnz
        w_op = K.pack_operand(conv.lin_src.weight.detach(), False, planes)
        xin = K.pack_operand(x, False, planes)
        att_s, att_d = conv.att_src.detach().reshape(-1), conv.att_dst.detach().reshape(-1)
        bias = conv.bias.detach()
        xp = K.gemm_nt([xin], [w_op], [(0, 0, 0, 0, d)], H * C, K.alloc_act(n, H * C, act, dev))
        a_s, a_d = K.gat_logits(xp, H, C, att_s, att_d)

        def ours():
            xp_ = K.gemm_nt([xin], [w_op], [(0, 0, 0, 0, d)], H * C, K.alloc_act(n, H * C, act, dev))
            s_, d_ = K.gat_logits(xp_, H, C, att_s, att_d)
            return K.gat_fwd(graph.rowptr, graph.col, xp_, s_, d_, H, C, False, bias, 0.0, 0)

        def kernel():
            return K.gat_fwd(graph.rowptr, graph.col, xp, a_s, a_d, H, C, False, bias, 0.0, 0)

        with torch.no_grad():
            t_ref = _time(lambda: conv(x, ei), a.iters)
            t_ours = _time(ours, a.iters)
            t_k = _time(kernel, a.iters)
            err = (ours()[0].float() - conv(x, ei)).abs().max().item()
        tol = 1e-3 if a.precision == "fp32" else 1e-1
        if not err <= tol:
            raise SystemExit(f"{name}: native layer differs from the torch layer by {err:.3e} (> {tol})")
        nb = fwd_bytes(n, nnz, H, C, 2 if act == torch.bfloat16 else 4)
        rows.append(dict(graph=name, n=n, nnz=nnz, d=d, heads=H, channels=C, precision=a.precision, torch_layer_ms=t_ref,
                         native_layer_ms=t_ours, speedup=t_ref / t_ours, gat_fwd_ms=t_k, gat_fwd_bytes=nb,
                         gat_fwd_TBps=nb / (t_k * 1e-3) / 1e12, max_abs_err=err,
                         x_prime_fits_l2=n * H * C * (2 if act == torch.bfloat16 else 4) <= 50e6,
                         gat_fwd_share_of_hbm=nb / (t_k * 1e-3) / HBM_BPS))
        print(json.dumps(rows[-1]))
    out = dict(card=card, rows=rows)
    print(json.dumps(dict(card=card)))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
