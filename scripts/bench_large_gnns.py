"""Training-step benchmark of the large variant's baselines on the GPU: sgformer_b200.large_gnns.GCN (save_mem=True: the unscaled
SpMM) and GAT against their plain-torch restatement (oracle/large_gnns_oracle.py's GCN, oracle/gat_oracle.py's GATConv in
large/gnns.py's GAT stack) run as torch ops on the same GPU, on random undirected graphs of the ogbn-arxiv and pokec shapes with the
drivers' self loops.  One step = forward, a weighted-sum loss, backward.  Reports the step times, the SpMM launches' time in the
native GCN step and their algorithmic bytes/s against the H100 SXM's 3.35 TB/s, and the card's name and power limit.

    python scripts/bench_large_gnns.py [--iters 10] [--precision fp32|bf16] [--shapes arxiv,pokec] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import gat_oracle as G  # noqa: E402
from oracle import large_gnns_oracle as O  # noqa: E402
from sgformer_b200 import kernels as K  # noqa: E402
from sgformer_b200 import large_gnns as LG  # noqa: E402
from sgformer_b200.graph import get_graph  # noqa: E402

# nodes, undirected edges before symmetrisation, features, classes; GCN hidden / layers and GAT hidden / heads as the reference's
# large/run.sh family uses them
SHAPES = {"arxiv": dict(n=169343, e=1166243, d=128, c=40, gcn=(256, 3), gat=(64, 4)),
          "pokec": dict(n=1632803, e=22301964, d=65, c=2, gcn=(256, 3), gat=(32, 2))}
HBM_BPS = 3.35e12


def _graph(n, e, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    src = torch.randint(0, n, (e,), device="cuda", generator=g)
    dst = torch.randint(0, n, (e,), device="cuda", generator=g)
    ei = torch.cat([torch.stack([src, dst]), torch.stack([dst, src])], 1)
    ei = ei[:, ei[0] != ei[1]]
    ar = torch.arange(n, device="cuda")
    return torch.cat([ei, torch.stack([ar, ar])], 1).contiguous()


def _time(fn, iters):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


class TorchGAT(torch.nn.Module):
    """large/gnns.py:272-310's stack over the plain-torch GATConv restatement."""

    def __init__(self, d, h, c, heads):
        super().__init__()
        self.convs = torch.nn.ModuleList([G.GATConv(d, h, heads=heads, concat=True), G.GATConv(h * heads, c, heads=1, concat=False)])
        self.bns = torch.nn.ModuleList([torch.nn.BatchNorm1d(h * heads)])

    def forward(self, x, ei):
        x = F.dropout(x, 0.5, self.training)
        x = F.dropout(F.elu(self.convs[0](x, ei)), 0.5, self.training)
        return self.convs[1](x, ei)


def spmm_bytes(n, nnz, h, elt):
    """column ids, rowptr, one gathered feature row per entry, one written row per node."""
    return nnz * 4 + (n + 1) * 8 + nnz * h * elt + n * h * elt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--precision", default="fp32", choices=["fp32", "bf16"])
    ap.add_argument("--shapes", default="arxiv,pokec")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_large_gnns needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    rows = []
    for name in a.shapes.split(","):
        s = SHAPES[name]
        n, d, c = s["n"], s["d"], s["c"]
        ei = _graph(n, s["e"], 0)
        nnz = ei.shape[1]
        x = torch.randn(n, d, device="cuda")
        wgt = torch.randn(n, c, device="cuda")
        h, nl = s["gcn"]
        row = dict(shape=name, n=n, nnz=nnz, precision=a.precision, gpu=q)

        gcn = LG.GCN(d, h, c, num_layers=nl, dropout=0.5).cuda().set_precision(a.precision).train()
        sd = {k: v.clone() for k, v in gcn.state_dict().items()}

        def native_gcn():
            gcn.zero_grad(set_to_none=True)
            (gcn(x, ei) * wgt).sum().backward()
        get_graph(ei, n, 0).transpose()
        row["gcn_native_ms"] = _time(native_gcn, a.iters)
        K.spmm_events = []
        native_gcn()
        torch.cuda.synchronize()
        ev, K.spmm_events = K.spmm_events, None
        spmm_ms = sum(e0.elapsed_time(e1) for e0, e1 in ev)
        elt = 4 if a.precision == "fp32" else 2
        widths = [h] * (nl - 1) + [-(-c // (4 if elt == 4 else 8)) * (4 if elt == 4 else 8)]
        byts = 2 * sum(spmm_bytes(n, nnz, w, elt) for w in widths)     # forward + backward launch per layer
        row.update(gcn_spmm_launches=len(ev), gcn_spmm_ms=spmm_ms, gcn_spmm_TBps=byts / (spmm_ms * 1e-3) / 1e12,
                   gcn_spmm_share_of_peak=byts / (spmm_ms * 1e-3) / HBM_BPS)

        P = {k: v.detach().clone().requires_grad_(v.is_floating_point() and "running" not in k) for k, v in sd.items()}
        xt = x.clone()

        def torch_gcn():
            for v in P.values():
                v.grad = None
            (O.gcn_large(xt, ei, P, nl, True, True, True, 0.5) * wgt).sum().backward()
        try:
            row["gcn_torch_ms"] = _time(torch_gcn, a.iters)
        except torch.OutOfMemoryError:
            row["gcn_torch_ms"] = "out of memory"
        del P, gcn
        torch.cuda.empty_cache()

        hg, heads = s["gat"]
        gat = LG.GAT(d, hg, c, num_layers=2, dropout=0.5, use_bn=False, heads=heads).cuda().set_precision(a.precision).train()

        def native_gat():
            gat.zero_grad(set_to_none=True)
            (gat(x, ei) * wgt).sum().backward()
        row["gat_native_ms"] = _time(native_gat, a.iters)
        tg = TorchGAT(d, hg, c, heads).cuda().train()

        def torch_gat():
            tg.zero_grad(set_to_none=True)
            (tg(x, ei) * wgt).sum().backward()
        try:
            row["gat_torch_ms"] = _time(torch_gat, a.iters)
        except torch.OutOfMemoryError:
            row["gat_torch_ms"] = "out of memory"
        del gat, tg
        torch.cuda.empty_cache()
        rows.append(row)
        print(json.dumps(row), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
