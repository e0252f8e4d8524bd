"""One GCNJK training step (forward, cross-entropy, backward, Adam) on the kernels (fp32 and bf16) against the same model as plain
torch ops (oracle/gcnjk_oracle.py's restatement over a cached torch CSR Â, as PyG's GCNConv(cached=True) keeps it), on one GPU.

    python scripts/bench_gcnjk.py [--steps 20] [--warmup 5] [--out results/bench_gcnjk.json]

Shapes: Cora (2 708 nodes, 1 433 features, h = 64, 2 layers, 7 classes) and arxiv (169 343 nodes, 128 features, 1.17 M edges,
h = 256, 3 layers, 40 classes), both JK modes.  Prints one JSON line per case and the card's name, power limit and SM clock.  Beside
each time: the HBM bytes the JK aggregation adds to the GCN schedule's passes, from the shapes (jk_bytes)."""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.gcnjk_oracle import jumping_knowledge  # noqa: E402
from oracle.sgformer_oracle import pyg_gcn_adjacency  # noqa: E402

SHAPES = {"cora": dict(n=2708, d=1433, e=10556, h=64, layers=2, c=7),
          "arxiv": dict(n=169343, d=128, e=1166243, h=256, layers=3, c=40)}


def jk_bytes(n, h, layers, b, mode):
    """HBM bytes the JK aggregation adds to the GCN schedule's row passes, per step, for `layers` convs of width h and b-byte
    activations (the final projection is GEMM traffic and is not counted here).
    max, forward: layer 0 writes the running max m and the index (N h b + N h); every later layer reads and writes both
      (2 N h b + 2 N h).
    max, backward: each pass of bn_bwd reads g_jk and the index (N h b + N h): two passes (reduce, apply) per hidden layer, one for
      the last conv.
    cat, forward: a hidden layer writes its block of the concatenation when dropout is active (N h b); the last conv's pass writes
      its block in place of its output (0 extra).  cat, backward: each bn_bwd pass reads its block of g_jk (N h b)."""
    if mode == "max":
        fwd = (n * h * b + n * h) + (layers - 1) * 2 * (n * h * b + n * h)
        bwd = (2 * (layers - 1) + 1) * (n * h * b + n * h)
    else:
        fwd = (layers - 1) * n * h * b
        bwd = (2 * (layers - 1) + 1) * n * h * b
    return dict(fwd=fwd, bwd=bwd)


def gcn_bytes(n, h, layers, b):
    """HBM bytes of the GCN schedule's own row passes, per step: bn_fwd reads z and writes y (2 N h b per layer); a hidden layer's
    bn_bwd reads z and dy in its reduce pass and z and dy and writes dz in its apply pass (5 N h b); the last conv's reads z and dy
    and writes dz (3 N h b)."""
    return layers * 2 * n * h * b + (layers - 1) * 5 * n * h * b + 3 * n * h * b


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q


def graph(n, e, seed=0):
    g = torch.Generator().manual_seed(seed)
    ei = torch.stack([torch.randint(0, n, (e // 2,), generator=g), torch.randint(0, n, (e // 2,), generator=g)])
    return torch.cat([ei, ei.flip(0)], 1)


def time_steps(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        step()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def native_step(model, data, y, opt):
    def step():
        opt.zero_grad(set_to_none=True)
        F.cross_entropy(model(data), y).backward()
        opt.step()
    return step


def torch_step(params, x, adj, y, layers, jk, opt, p):
    """The plain-torch restatement: GCNConv = Â (x Wᵀ) + b; BatchNorm / ReLU / dropout; JK; final Linear."""
    bns = [torch.nn.BatchNorm1d(params["h"]).cuda() for _ in range(layers - 1)]

    def step():
        opt.zero_grad(set_to_none=True)
        h, xs = x, []
        for i in range(layers):
            h = torch.sparse.mm(adj, h @ params[f"w{i}"].t()) + params[f"b{i}"]
            if i < layers - 1:
                h = F.relu(bns[i](h))
                xs.append(h)
                h = F.dropout(h, p, True)
            else:
                xs.append(h)
        out = F.linear(jumping_knowledge(xs, jk), params["wf"], params["bf"])
        F.cross_entropy(out, y).backward()
        opt.step()
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--shapes", default="cora,arxiv")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gcnjk needs a CUDA device")
    from sgformer_b200 import medium as M
    info = card()
    print(json.dumps({"card": info}))
    rows = []
    for name in a.shapes.split(","):
        s = SHAPES[name]
        n, d, h, L, c = s["n"], s["d"], s["h"], s["layers"], s["c"]
        torch.manual_seed(0)
        x = torch.randn(n, d, device="cuda")
        ei = graph(n, s["e"]).cuda()
        y = torch.randint(0, c, (n,), device="cuda")
        adj = pyg_gcn_adjacency(ei.cpu(), n).cuda()
        data = type("D", (), {})()
        data.graph = {"node_feat": x, "edge_index": ei, "num_nodes": n}
        for jk in ("max", "cat"):
            res = dict(shape=name, jk=jk, n=n, d=d, h=h, layers=L, classes=c, steps=a.steps, warmup=a.warmup)
            for prec in ("fp32", "bf16"):
                m = M.GCNJK(d, h, c, num_layers=L, dropout=0.5, jk_type=jk).cuda().set_precision(prec).train()
                opt = torch.optim.Adam(m.parameters(), lr=1e-2)
                res[f"native_{prec}_ms"] = round(time_steps(native_step(m, data, y, opt), a.steps, a.warmup), 3)
                b = 4 if prec == "fp32" else 2
                res[f"jk_bytes_{prec}"] = jk_bytes(n, h, L, b, jk)
                res[f"gcn_rowpass_bytes_{prec}"] = gcn_bytes(n, h, L, b)
            params = {"h": h}
            dims = [d] + [h] * L
            for i in range(L):
                params[f"w{i}"] = (torch.randn(h, dims[i], device="cuda") / dims[i] ** 0.5).requires_grad_()
                params[f"b{i}"] = torch.zeros(h, device="cuda", requires_grad=True)
            kfp = h * L if jk == "cat" else h
            params["wf"] = (torch.randn(c, kfp, device="cuda") / kfp ** 0.5).requires_grad_()
            params["bf"] = torch.zeros(c, device="cuda", requires_grad=True)
            opt = torch.optim.Adam([v for k, v in params.items() if k != "h"], lr=1e-2)
            res["torch_fp32_ms"] = round(time_steps(torch_step(params, x, adj, y, L, jk, opt, 0.5), a.steps, a.warmup), 3)
            rows.append(res)
            print(json.dumps(res), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(card=info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
