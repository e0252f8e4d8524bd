"""`evaluate()` of the reference drivers with the metric computed on the device (SURVEY.md §8f-3).

Reference: large/eval.py:6-33 runs the model, then for each of the three splits gathers `out[split]`, takes the argmax, copies both
label and prediction arrays to the host and loops in numpy (`eval_acc`, large/data_utils.py:210-220); the validation loss is
`NLLLoss(log_softmax(out)[valid], label[valid])`.  Here one kernel launch per split (`sgf_eval_acc`, K11) reads the logits in
place through the split's index list and returns the hit count (and, for the validation split, the summed NLL); only those
scalars cross PCIe.  Same signature and return tuple as the reference, so `large/main.py:144` can call it unchanged:

    from sgformer_b200.eval import evaluate

Metrics other than `eval_acc` (rocauc / f1: host-side sklearn in the reference) and the multi-label datasets are delegated to the
caller's own `eval_func` / `criterion` exactly as the reference does.

`evaluate_batch` replaces large/eval.py:67-118, the mini-batch evaluation large/main-batch.py:154-155 runs on ogbn-papers100M,
with the same signature and return tuple:

    from sgformer_b200.eval import evaluate_batch
"""
from __future__ import annotations

from typing import Optional

import torch

from . import kernels as K
from .graph import Graph, get_graph
from .minibatch import MiniBatch

_BCE_DATASETS = ('yelp-chi', 'deezer-europe', 'twitch-e', 'fb100', 'ogbn-proteins')      # large/eval.py:21


@torch.no_grad()
def evaluate(model, dataset, split_idx, eval_func, criterion, args, result=None):
    if result is not None:
        out = result
    else:
        model.eval()
        out = model(dataset.graph['node_feat'], dataset.graph['edge_index'])
    label = dataset.label
    on_device = (getattr(eval_func, "__name__", "") == "eval_acc" and label.dim() == 2 and label.shape[1] == 1
                 and label.dtype == torch.int64 and getattr(args, "dataset", None) not in _BCE_DATASETS)
    if not on_device:
        # other metrics (rocauc, f1: sklearn on the host in the reference) and the multi-label datasets: the caller's own
        # eval_func / criterion, exactly as large/eval.py:13-31 - these are outside the accelerated path, not a fallback of K11
        train_acc = eval_func(label[split_idx['train']], out[split_idx['train']])
        valid_acc = eval_func(label[split_idx['valid']], out[split_idx['valid']])
        test_acc = eval_func(label[split_idx['test']], out[split_idx['test']])
        if getattr(args, "dataset", None) in _BCE_DATASETS:
            true_label = torch.nn.functional.one_hot(label, label.max() + 1).squeeze(1) if label.shape[1] == 1 else label
            valid_loss = criterion(out[split_idx['valid']], true_label.squeeze(1)[split_idx['valid']].to(torch.float))
        else:
            out = torch.log_softmax(out, dim=1)
            valid_loss = criterion(out[split_idx['valid']], label.squeeze(1)[split_idx['valid']])
        return train_acc, valid_acc, test_acc, valid_loss, out
    logits = out.float()
    if not logits.is_cuda:              # logits handed in from the host (e.g. `result=` of evaluate_large): K11 has no CPU path
        logits = logits.cuda()
    lab = label.to(logits.device)
    train_acc, _ = K.eval_acc(logits, lab, split_idx['train'])
    valid_acc, valid_loss = K.eval_acc(logits, lab, split_idx['valid'], want_loss=True)
    test_acc, _ = K.eval_acc(logits, lab, split_idx['test'])
    return train_acc, valid_acc, test_acc, torch.tensor(valid_loss, dtype=torch.float32), torch.log_softmax(out, dim=1)


_HOST_PARENT: dict = {}


def _host_parent(edge_index, n: int, mode: int, dev) -> Graph:
    """The parent Graph of a host edge list: built from a temporary device copy that is released after the build (only the CSR
    stays on the device), and kept for the next call with the same edge list tensor (identity and version), as get_graph
    keeps the Graph of a device edge list."""
    key = (edge_index.data_ptr(), tuple(edge_index.shape), edge_index._version, int(n), mode, str(dev))
    hit = _HOST_PARENT.get(key)
    if hit is not None and hit[0] is edge_index:
        return hit[1]
    _HOST_PARENT.clear()
    graph = Graph(edge_index.to(dev), n, mode)
    graph.transpose()               # the transposed CSR of a directed graph is built from the edge list ...
    graph.edge_index = None         # ... which is not needed after that: free its device copy
    _HOST_PARENT[key] = (edge_index, graph)
    return graph


@torch.no_grad()
def evaluate_batch(model, dataset, split_idx, args, device, n, true_label, graph: Optional[Graph] = None):
    """large/eval.py:67-118 with the batches and the counts on the device.  The reference cuts `torch.randperm(n)` into
    `n // batch_size + 1` slices and, per slice, runs PyG `subgraph` over every edge on the CPU, the model, and three masked
    `eval_acc` calls (three host syncs).  Here every slice of the same permutation is a `Graph.subset` batch fed to `model(mb)`,
    and one `sgf_eval_acc_splits` launch per batch adds the batch's rows and argmax hits of each split to six device counters.

    Host syncs: one before the loop, reading the largest per-slice sum of the parent's row lengths (the subsets' capacity, never
    exceeded, so no batch is truncated and none sizes itself with a sync), and one after it, reading the counters.  None per batch.

    Memory: node features stay where they are.  Host features (as the reference keeps them) are gathered per batch into pinned
    memory and copied to the device without a sync; device features are gathered on the device.  The parent graph is
    `graph` (in the model's `self_loop_mode`), else the cached Graph of a device edge list (get_graph), else the Graph of a
    host edge list, built once from a temporary device copy that is released after the build, so that only the CSR stays on
    the device, and reused by the next call with the same edge list.

    An empty last slice (n a multiple of batch_size) is skipped; it adds nothing in the reference either.  Returns
    (train_acc, valid_acc, test_acc, 0, None); an empty split gives nan.  Single-column integer labels only; the model must take
    a MiniBatch (large.SGFormer, large_gnns.GCN / GAT)."""
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("sgformer_b200.eval.evaluate_batch runs on a CUDA device (no CPU fallback)")
    label = true_label.reshape(-1) if true_label.dim() == 1 or true_label.shape[1] == 1 else None
    if label is None or label.dtype != torch.int64:
        raise ValueError("evaluate_batch: true_label must hold one int64 class per node ([n] or [n, 1])")
    batch_size = int(args.batch_size)
    num_batch = n // batch_size + 1                     # large/eval.py:68
    model.to(dev)
    model.eval()
    perm = torch.randperm(n)                            # the reference's permutation: same generator, same stream of draws
    mode = getattr(model, "self_loop_mode", 0)
    if graph is None:
        ei = dataset.graph['edge_index']
        graph = get_graph(ei, n, mode) if ei.is_cuda else _host_parent(ei, n, mode, dev)
    elif graph.self_loop_mode != mode:
        raise ValueError(f"evaluate_batch: the graph has self_loop_mode {graph.self_loop_mode} but the model builds self_loop_mode {mode}")
    graph.transpose()
    x = dataset.graph['node_feat']
    label = label.to(dev).contiguous()
    split = torch.zeros(n, dtype=torch.uint8, device=dev)
    for key, bit in (('train', K.SPLIT_TRAIN), ('valid', K.SPLIT_VALID), ('test', K.SPLIT_TEST)):
        rows = split_idx[key]
        split[rows.pin_memory().to(dev, non_blocking=True) if not rows.is_cuda else rows.to(dev)] |= bit
    idx = perm.pin_memory().to(dev, non_blocking=True)        # pinned: a pageable copy would wait for the stream
    # capacity: the largest sum of a slice's parent row lengths bounds its induced nnz (either half of a directed graph's)
    slot = torch.arange(n, device=dev) // batch_size
    rp, rp_t = graph.rowptr, graph.transpose()[0]
    bound = torch.zeros(num_batch, dtype=torch.int64, device=dev).index_add_(0, slot, (rp[1:] - rp[:-1])[idx])
    if rp_t is not rp:
        bound = torch.minimum(bound, torch.zeros_like(bound).index_add_(0, slot, (rp_t[1:] - rp_t[:-1])[idx]))
    capacity = int(bound.max().item()) if n else 0
    counts = torch.zeros(6, dtype=torch.int64, device=dev)
    for i in range(num_batch):
        lo, hi = i * batch_size, min((i + 1) * batch_size, n)
        if hi <= lo:
            continue
        idx_i = idx[lo:hi]
        if x.is_cuda:
            feats = x.index_select(0, idx_i)
        else:
            host = torch.empty((hi - lo, x.shape[1]), dtype=x.dtype, pin_memory=True)
            feats = torch.index_select(x, 0, perm[lo:hi], out=host).to(dev, non_blocking=True)
        out = model(MiniBatch(idx_i, feats, graph.subset(idx_i, capacity)))
        K.eval_acc_splits(out if out.dtype == torch.float32 else out.float(), label, split, idx_i, counts)
    total = counts.tolist()
    acc = [total[2 * k + 1] / total[2 * k] if total[2 * k] else float("nan") for k in range(3)]
    return acc[0], acc[1], acc[2], 0, None
