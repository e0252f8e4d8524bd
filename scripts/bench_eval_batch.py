"""Mini-batch evaluation and GAT mini-batch training steps, each on device batches and on per-batch edge lists:
  eval      one evaluation epoch over a papers100M-shaped slice (2 M nodes, 28 M directed edges made symmetric, 128 features,
            172 classes, batch 400 000 as large/run.sh; the large SGFormer in bf16, 3 GraphConv layers, hidden 256):
              batch  sgformer_b200.eval.evaluate_batch: Graph.subset batches, sgf_eval_acc_splits, two host syncs per epoch
              edges  large/eval.py:67-118 on the device: K.subgraph (sgf_subgraph, an O(E) mask) per batch, the model on the
                     edge list (a CSR build per batch), three masked eval_acc counts per batch with a host sync each
  gat_step  one large_gnns.GAT training step (fwd, cross-entropy, bwd, Adam) of a pokec-shaped graph (1.63 M nodes, 30.6 M
            edges, 65 features, 2 classes, hidden 64 x 2 heads, batch 100 000), its batch from Graph.subset (RandomPartitionSampler)
            or from K.subgraph's edge list
    python scripts/bench_eval_batch.py [--reps 15] [--steps 20]
Host clock around whole epochs (each ends in a device synchronise), CUDA events around the steps, after warm-ups; the two ways
alternate; min / median / max of the epochs and the median step are printed, and the peak device memory (above what was
allocated before) of one epoch whose features, labels and edge list are on the host.  Checks first that both ways give the
same accuracies and the same step logits.  Prints one JSON line with the card's name and power limit."""
import argparse
import copy
import json
import os
import statistics
import sys
import time
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench_subset import card  # noqa: E402
from sgformer_b200 import kernels as K  # noqa: E402
from sgformer_b200 import large as L  # noqa: E402
from sgformer_b200 import large_gnns as LG  # noqa: E402
from sgformer_b200.eval import evaluate_batch  # noqa: E402
from sgformer_b200.graph import Graph  # noqa: E402
from sgformer_b200.minibatch import RandomPartitionSampler  # noqa: E402
from sgformer_b200.optim import Adam  # noqa: E402

EVAL = dict(n=2_000_000, e=28_000_000, d=128, c=172, h=256, batch=400_000)
STEP = dict(n=1_632_803, e=30_622_564, d=65, c=2, h=64, heads=2, batch=100_000)


def eval_edges(model, x, ei, n, label, split, bs):
    """large/eval.py:67-118 with the per-batch structure from K.subgraph and the three eval_acc counts of each batch."""
    masks = [torch.zeros(n, dtype=torch.bool, device=x.device) for _ in range(3)]
    for m, key in zip(masks, ("train", "valid", "test")):
        m[split[key]] = True
    idx = torch.randperm(n).to(x.device)
    tot, cor = [0, 0, 0], [0, 0, 0]
    with torch.no_grad():
        for i in range(n // bs + 1):
            idx_i = idx[i * bs:(i + 1) * bs]
            if idx_i.numel() == 0:
                continue
            out = model(x[idx_i], K.subgraph(ei, n, idx_i))
            y_i = label[idx_i]
            for k, m in enumerate(masks):
                m_i = m[idx_i]
                tot[k] += int(m_i.sum().item())
                cor[k] += (y_i[m_i] == torch.max(out[m_i], dim=1, keepdim=True)[1]).sum().item()
    return tuple(c / t for c, t in zip(cor, tot))


def host_s(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def bench_eval(reps):
    w = EVAL
    n, bs = w["n"], w["batch"]
    gen = torch.Generator(device="cuda").manual_seed(0)
    ei = torch.stack([torch.randint(0, n, (w["e"],), generator=gen, device="cuda"),
                      torch.randint(0, n, (w["e"],), generator=gen, device="cuda")])
    ei = ei[:, ei[0] != ei[1]]
    ar = torch.arange(n, device="cuda")
    ei = torch.cat([ei, ei.flip(0), torch.stack([ar, ar])], 1).contiguous()
    x = torch.randn(n, w["d"], generator=gen, device="cuda")
    label = torch.randint(0, w["c"], (n, 1), generator=gen, device="cuda")
    perm = torch.randperm(n, generator=gen, device="cuda")
    split = {"train": perm[: n // 10], "valid": perm[n // 10: n // 5], "test": perm[n // 5: n // 2]}
    torch.manual_seed(0)
    model = L.SGFormer(w["d"], w["h"], w["c"], trans_num_layers=1, gnn_num_layers=3, gnn_use_init=True, gnn_use_bn=True,
                       gnn_use_residual=True, graph_weight=0.5).cuda().set_precision("bf16").eval()
    ds = SimpleNamespace(graph={"edge_index": ei, "node_feat": x}, label=label)
    args = SimpleNamespace(batch_size=bs)
    graph = Graph(ei, n, 0)
    run_batch = lambda: evaluate_batch(model, ds, split, args, "cuda", n, label, graph=graph)[:3]  # noqa: E731
    run_edges = lambda: eval_edges(model, x, ei, n, label, split, bs)  # noqa: E731
    torch.manual_seed(1)
    a = run_batch()
    torch.manual_seed(1)
    b = run_edges()
    assert a == b, f"accuracies differ: {a} vs {b}"
    tb, te = [], []
    for _ in range(reps):
        tb.append(host_s(run_batch)[0])
        te.append(host_s(run_edges)[0])
    spread = lambda t: [round(1e3 * v, 1) for v in (min(t), statistics.median(t), max(t))]  # noqa: E731
    # peak device memory of one epoch with features, labels and edge list on the host (the parent CSR built inside)
    host_ds = SimpleNamespace(graph={"edge_index": ei.cpu(), "node_feat": x.cpu()}, label=label.cpu())
    del graph
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    evaluate_batch(model, host_ds, split, args, "cuda", n, host_ds.label)
    peak = torch.cuda.max_memory_allocated() - base
    return dict(eval_nodes=n, eval_edges=int(ei.shape[1]), eval_batch=bs, eval_batches=n // bs + 1, eval_reps=reps,
                eval_epoch_batch_ms_min_med_max=spread(tb), eval_epoch_edges_ms_min_med_max=spread(te),
                eval_host_inputs_peak_device_mb=round(peak / 2**20, 1))


def bench_gat_step(steps):
    w = STEP
    n, bs = w["n"], w["batch"]
    gen = torch.Generator(device="cuda").manual_seed(2)
    ei = torch.stack([torch.randint(0, n, (w["e"],), generator=gen, device="cuda"),
                      torch.randint(0, n, (w["e"],), generator=gen, device="cuda")])
    x = torch.randn(n, w["d"], generator=gen, device="cuda")
    y = torch.randint(0, w["c"], (n,), generator=gen, device="cuda")
    torch.manual_seed(0)
    model = LG.GAT(w["d"], w["h"], w["c"], num_layers=2, dropout=0.0, heads=w["heads"]).cuda().train()
    ref = copy.deepcopy(model)
    opts = [Adam(m.parameters(), lr=0.01) for m in (model, ref)]
    sampler = RandomPartitionSampler(Graph(ei, n, 1), x, y, bs, capacity=int(ei.shape[1]) + n)
    idx = torch.randperm(n, generator=gen, device="cuda")[:bs]

    def step(m, opt, from_subset):
        opt.zero_grad()
        out = m(sampler.batch(idx)) if from_subset else m(x[idx], K.subgraph(ei, n, idx))
        torch.nn.functional.cross_entropy(out, y[idx]).backward()
        opt.step()
        return out

    assert torch.equal(step(model, opts[0], True).detach(), step(ref, opts[1], False).detach())
    ts, te = [], []
    for _ in range(3):
        step(model, opts[0], True)
        step(ref, opts[1], False)
    for _ in range(steps):
        for m, opt, sub, acc in ((model, opts[0], True, ts), (ref, opts[1], False, te)):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            step(m, opt, sub)
            b.record()
            torch.cuda.synchronize()
            acc.append(a.elapsed_time(b))
    sampler.check()
    return dict(step_nodes=n, step_edges=w["e"], step_batch=bs, gat_step_subset_ms=round(statistics.median(ts), 3),
                gat_step_edges_ms=round(statistics.median(te), 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval_batch.py measures on a CUDA device; none found")
    res = dict(**card())
    res.update(bench_eval(args.reps))
    torch.cuda.empty_cache()
    res.update(bench_gat_step(args.steps))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
