"""Time one training step (forward + backward) of SGFormerSOFT's attention branch (medium/ablation/oursSOFT.py, use_graph=False)
in three forms: the native softmax attention, the same model as the reference's torch ops (until torch runs out of memory), and
the native linear attention (the medium SGFormer) of the same shape.  Also times the fused attention forward alone and reports
its FLOP/s from the reference's 4 N^2 H M flops (the kernel computes every head's scores for each head it writes, H times
the score work) against the dense BF16 data-sheet peak of the H100 SXM (989 TFLOP/s).  One JSON line per shape.

    python scripts/bench_softmax.py [--shapes cora,pubmed,deezer,arxiv] [--precision fp32|bf16] [--steps 5]

--attention gat times SGFormerGAT's attention branch (medium/ablation/oursGAT.py, use_graph=False) instead: the native step in
fp32 and in bf16, and the same model as the reference's torch einsums (oracle/gat_attention_oracle.py).  Flops are counted from
shapes: the kernels' score work is 2 N^2 H^2 dk (every head's scores for each head written), the reference's 2 N^2 H dk plus
2 N^2 H h for the values.

    python scripts/bench_softmax.py --attention gat [--shapes ...] [--steps 5]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import gat_attention_oracle as OG  # noqa: E402
from oracle import softmax_oracle as O  # noqa: E402
from sgformer_b200 import ablation, ablation_gat, medium  # noqa: E402
from sgformer_b200 import engine as E  # noqa: E402
from sgformer_b200 import kernels as K  # noqa: E402

# (nodes, features, hidden, classes): Cora, Pubmed and deezer as in medium/ablation/run.sh / the medium recipes; arxiv-shaped
SHAPES = {"cora": (2708, 1433, 64, 7), "pubmed": (19717, 500, 64, 3), "deezer": (28281, 128, 64, 2), "arxiv": (169343, 128, 64, 40)}
BF16_PEAK = 989e12


class _Data:
    def __init__(self, x):
        self.graph = {"node_feat": x, "edge_index": torch.zeros(2, 0, dtype=torch.long, device=x.device)}


def _time(fn, steps, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def _step(m, data):
    def f():
        m.zero_grad(set_to_none=True)
        m(data).sum().backward()
    return f


def _torch_step(sd, x, layers, heads):
    def f():
        for t in sd.values():
            t.grad = None
        O.sgformer_soft(sd, x, layers, heads).sum().backward()
    return f


def _gat_torch_step(sd, x, layers, heads):
    def f():
        for t in sd.values():
            t.grad = None
        OG.sgformer_gat(sd, x, layers, heads).sum().backward()
    return f


def _gat_shape(name, a, card):
    n, f, h, c = SHAPES[name]
    H, dk = a.heads, h // a.heads
    torch.manual_seed(0)
    x = torch.randn(n, f, device="cuda")
    data = _Data(x)
    rec = dict(attention="gat", shape=name, n=n, hidden=h, heads=H, layers=a.layers, card=card,
               kernel_score_flops=2.0 * n * n * H * H * dk * a.layers, reference_flops=(2.0 * n * n * H * dk + 2.0 * n * n * H * h) * a.layers)
    m = ablation_gat.SGFormerGAT(f, h, c, num_layers=a.layers, num_heads=H, dropout=0.0, use_graph=False).cuda().train()
    for prec in ("fp32", "bf16"):
        m.set_precision(prec)
        rec[f"native_{prec}_ms"] = _time(_step(m, data), a.steps)
    sd = {k: v.detach().clone().requires_grad_() for k, v in m.state_dict().items()}
    try:
        rec["torch_ms"] = _time(_gat_torch_step(sd, x, a.layers, H), a.steps, warmup=1)
    except torch.OutOfMemoryError:
        rec["torch_ms"] = "out of memory"
    print(json.dumps(rec), flush=True)
    del m, sd
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--attention", default="softmax", choices=["softmax", "gat"])
    ap.add_argument("--shapes", default="cora,pubmed,deezer,arxiv")
    ap.add_argument("--precision", default="fp32", choices=["fp32", "bf16"])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--heads", type=int, default=2)   # one head is degenerate: every weight is 1
    ap.add_argument("--layers", type=int, default=1)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    if a.attention == "gat":
        for name in a.shapes.split(","):
            _gat_shape(name, a, card)
        return
    for name in a.shapes.split(","):
        n, f, h, c = SHAPES[name]
        torch.manual_seed(0)
        x = torch.randn(n, f, device="cuda")
        data = _Data(x)
        rec = dict(shape=name, n=n, hidden=h, heads=a.heads, layers=a.layers, precision=a.precision, card=card)
        soft = ablation.SGFormerSOFT(f, h, c, num_layers=a.layers, num_heads=a.heads, dropout=0.0, use_graph=False).cuda()
        soft.set_precision(a.precision).train()
        rec["native_softmax_ms"] = _time(_step(soft, data), a.steps)
        lin = medium.SGFormer(f, h, c, num_layers=a.layers, num_heads=a.heads, dropout=0.0, use_graph=False).cuda()
        lin.set_precision(a.precision).train()
        rec["native_linear_ms"] = _time(_step(lin, data), a.steps)
        sd = {k: v.detach().clone().requires_grad_() for k, v in soft.state_dict().items()}
        try:
            rec["torch_softmax_ms"] = _time(_torch_step(sd, x, a.layers, a.heads), a.steps, warmup=1)
        except torch.OutOfMemoryError:
            rec["torch_softmax_ms"] = "out of memory"
        torch.cuda.empty_cache()
        # the fused forward kernel alone, on q, k, v of this shape
        prec = E.precision(a.precision)
        q, k, v = (torch.randn(n, a.heads * h, device="cuda").to(prec.act_dtype) for _ in range(3))
        sq = K.colstats(q, want_sum=False)[1], K.colstats(k, want_sum=False)[1]
        ms = _time(lambda: K.attn_softmax_fwd(q, k, v, a.heads, *sq), a.steps)
        flops = 4.0 * n * n * a.heads * h
        rec["attn_fwd_ms"] = ms
        rec["attn_fwd_tflops"] = flops / (ms * 1e-3) / 1e12
        rec["attn_fwd_share_of_bf16_peak"] = flops / (ms * 1e-3) / BF16_PEAK
        print(json.dumps(rec), flush=True)
        del soft, lin, sd, q, k, v
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
