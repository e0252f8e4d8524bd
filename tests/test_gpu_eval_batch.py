"""Mini-batch evaluation on the H100: sgf_eval_acc_splits counts exactly, and sgformer_b200.eval.evaluate_batch returns exactly
the accuracies of `evaluate_batch_restated`, a torch restatement of the reference's large/eval.py:67-118 fed `subgraph` edge
lists (tests/test_subset_mode1.py pins the restatement to the reference's own evaluate_batch and eval_acc on the CPU)."""
import os
from types import SimpleNamespace

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def eval_acc(true, pred):
    """large/eval.py:120-131: (rows, hits), hits = label == torch.max(pred, dim=1) index (first maximum on ties)."""
    pred = torch.max(pred, dim=1, keepdim=True)[1]
    return true.shape[0], (true == pred).sum().item()


def evaluate_batch_restated(model, x, edge_index, n, label, split_idx, batch_size, subgraph):
    """large/eval.py:67-118 with `subgraph(edge_index, n, idx_i)` -> the batch's relabelled edge list (PyG `subgraph` order).
    x, edge_index and label live on the model's device; masks and the permutation on the host, as in the reference.  An
    empty last batch (n a multiple of batch_size) is skipped: it adds no rows to any split."""
    num_batch = n // batch_size + 1
    masks = []
    for key in ("train", "valid", "test"):
        m = torch.zeros(n, dtype=torch.bool)
        m[split_idx[key].cpu()] = True
        masks.append(m)
    model.eval()
    idx = torch.randperm(n)
    totals, corrects = [0, 0, 0], [0, 0, 0]
    with torch.no_grad():
        for i in range(num_batch):
            idx_i = idx[i * batch_size:(i + 1) * batch_size]
            if idx_i.numel() == 0:
                continue
            idx_d = idx_i.to(x.device)
            out_i = model(x[idx_d], subgraph(edge_index, n, idx_d))
            y_i = label[idx_d]
            for k, m in enumerate(masks):
                m_i = m[idx_i].to(x.device)
                t, c = eval_acc(y_i[m_i], out_i[m_i])
                totals[k] += t
                corrects[k] += c
    return tuple(c / t for c, t in zip(corrects, totals))


@pytest.fixture(scope="module")
def K():
    from sgformer_b200 import kernels
    return kernels


def split_counts(logits, label, code, idx):
    """Torch count of sgf_eval_acc_splits: per split bit, [rows, argmax hits] of the batch rows whose node carries the bit."""
    arg = torch.max(logits, dim=1)[1]
    lab, c = label.reshape(-1)[idx], code[idx]
    out = []
    for bit in (1, 2, 4):
        m = (c & bit) != 0
        out += [int(m.sum()), int((arg[m] == lab[m]).sum())]
    return out


@pytest.mark.parametrize("m,c", [(1, 3), (333, 2), (5000, 47), (140000, 172), (40000, 1)])
def test_eval_acc_splits_counts_exactly(K, m, c):
    """Exact counts against torch on random logits with planted ties, at row counts past the capped grid (8 blocks per SM, 8
    warps per block: 8448 rows per pass on 132 SMs), added into the counters over two launches, with and without idx."""
    g = torch.Generator().manual_seed(m + c)
    n = m + 777
    logits = torch.randint(-4, 5, (m, c), generator=g).float()          # integer logits: many ties
    rows = torch.randperm(m, generator=g)[: m // 3]
    logits[rows, rows % c] = logits[rows].max(dim=1).values
    label = torch.randint(-1, c + 1, (n,), generator=g)                  # includes labels outside [0, c): never hit
    code = torch.randint(0, 8, (n,), generator=g).to(torch.uint8)
    idx = torch.randperm(n, generator=g)[:m]
    ld, lb, cd, ix = logits.to(DEV), label.to(DEV), code.to(DEV), idx.to(DEV)
    counts = torch.zeros(6, dtype=torch.int64, device=DEV)
    K.eval_acc_splits(ld, lb, cd, ix, counts)
    assert counts.tolist() == split_counts(logits, label, code, idx)
    K.eval_acc_splits(ld, lb, cd, ix, counts)
    assert counts.tolist() == [2 * v for v in split_counts(logits, label, code, idx)]
    padded = torch.zeros(m, c + 5, device=DEV)
    padded[:, :c] = ld
    counts.zero_()
    K.eval_acc_splits(padded[:, :c], lb[:m].contiguous(), cd[:m].contiguous(), None, counts)     # strided logits, rows = nodes
    assert counts.tolist() == split_counts(logits, label[:m], code[:m], torch.arange(m))


def test_eval_acc_splits_refuses_bad_arguments(K):
    lg = torch.zeros(4, 3, device=DEV)
    lab = torch.zeros(10, dtype=torch.int64, device=DEV)
    code = torch.zeros(10, dtype=torch.uint8, device=DEV)
    counts = torch.zeros(6, dtype=torch.int64, device=DEV)
    with pytest.raises(TypeError):
        K.eval_acc_splits(lg.double(), lab, code, None, counts)
    with pytest.raises(ValueError):
        K.eval_acc_splits(lg, lab, code.int(), None, counts)
    with pytest.raises(ValueError):
        K.eval_acc_splits(lg, lab, code, torch.arange(3, device=DEV), counts)
    with pytest.raises(ValueError):
        K.eval_acc_splits(lg, lab, code, None, counts[:5])
    for host in ("labels", "split", "idx", "counts"):        # a host tensor is refused before any launch
        args = dict(labels=lab, split=code, idx=torch.arange(4, device=DEV), counts=counts)
        args[host] = args[host].cpu()
        with pytest.raises(ValueError, match=host):
            K.eval_acc_splits(lg, args["labels"], args["split"], args["idx"], args["counts"])


def _graph(n, e, seed, directed):
    g = torch.Generator().manual_seed(seed)
    ei = torch.randint(0, n - n // 50, (2, e), generator=g)
    ei = ei[:, ei[0] != ei[1]]
    if not directed:
        ei = torch.cat([ei, ei.flip(0)], 1)
    ar = torch.arange(n)
    return torch.cat([ei, torch.stack([ar, ar])], 1).contiguous()         # large/main-batch.py:97-98


def _models(d, c):
    from sgformer_b200 import large as L
    from sgformer_b200 import large_gnns as LG
    torch.manual_seed(0)
    return {"gcn_save_mem": LG.GCN(d, 32, c, num_layers=2, save_mem=True),
            "gcn_norm": LG.GCN(d, 32, c, num_layers=3, save_mem=False),
            "gat": LG.GAT(d, 16, c, num_layers=2, heads=2),
            "sgformer": L.SGFormer(d, 32, c, gnn_num_layers=2, gnn_use_init=True, graph_weight=0.5)}


@pytest.mark.parametrize("directed", [False, True])
@pytest.mark.parametrize("n,bs", [(9000, 2500), (6000, 2000)])          # a partial last batch; an empty one
def test_evaluate_batch_matches_restated_reference(K, directed, n, bs):
    from sgformer_b200.eval import evaluate_batch
    d, c = 16, 7
    ei = _graph(n, 8 * n, 3, directed).to(DEV)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(n, d, generator=g).to(DEV)
    label = torch.randint(0, c, (n, 1), generator=g).to(DEV)
    perm = torch.randperm(n, generator=g)
    split = {"train": perm[: n // 2], "valid": perm[n // 2: 3 * n // 4], "test": perm[3 * n // 4:]}
    ds = SimpleNamespace(graph={"edge_index": ei, "node_feat": x}, label=label)
    host_ds = SimpleNamespace(graph={"edge_index": ei.cpu(), "node_feat": x.cpu()}, label=label.cpu())
    for name, model in _models(d, c).items():
        model = model.to(DEV)
        torch.manual_seed(11)
        ref = evaluate_batch_restated(model, x, ei, n, label, split, bs, K.subgraph)
        torch.manual_seed(11)
        got = evaluate_batch(model, ds, split, SimpleNamespace(batch_size=bs), DEV, n, label)
        assert got[3:] == (0, None)
        assert got[:3] == ref, f"{name}: {got[:3]} != {ref}"
        torch.manual_seed(11)       # features and edge list on the host, as the reference keeps them
        got = evaluate_batch(model, host_ds, split, SimpleNamespace(batch_size=bs), DEV, n, label)
        assert got[:3] == ref, f"{name} (host inputs): {got[:3]} != {ref}"


def test_evaluate_batch_syncs_a_fixed_number_of_times():
    """An epoch syncs with the host twice whatever its number of batches: the capacity bound before the loop and the counters
    after it, none per batch (the synchronizing calls torch's sync debug mode reports from sgformer_b200, by source line)."""
    import warnings
    from sgformer_b200 import large_gnns as LG
    from sgformer_b200.eval import evaluate_batch
    from sgformer_b200.graph import Graph
    n, d, c = 12000, 16, 5
    ei = _graph(n, 80000, 2, True).to(DEV)
    x = torch.randn(n, d, device=DEV)
    label = torch.randint(0, c, (n, 1), device=DEV)
    split = {"train": torch.arange(0, 6000), "valid": torch.arange(6000, 9000), "test": torch.arange(9000, n)}
    ds = SimpleNamespace(graph={"edge_index": ei, "node_feat": x}, label=label)
    for model in (LG.GAT(d, 8, c).to(DEV), LG.GCN(d, 16, c, save_mem=False).to(DEV)):
        graph = Graph(ei, n, model.self_loop_mode)
        evaluate_batch(model, ds, split, SimpleNamespace(batch_size=4000), DEV, n, label, graph=graph)     # warm-up
        syncs = []
        for bs in (4000, 1000):                     # 4 and 13 batches
            with warnings.catch_warnings(record=True) as w:
                warnings.simplefilter("always")
                torch.cuda.set_sync_debug_mode("warn")
                try:
                    evaluate_batch(model, ds, split, SimpleNamespace(batch_size=bs), DEV, n, label, graph=graph)
                finally:
                    torch.cuda.set_sync_debug_mode("default")
            syncs.append(sorted(f"{os.path.basename(m.filename)}:{m.lineno}" for m in w
                                if "synchroniz" in str(m.message) and f"{os.sep}sgformer_b200{os.sep}" in m.filename))
        assert len(syncs[0]) == 2 and syncs[0] == syncs[1], f"host syncs of an epoch of 4 and of 13 batches: {syncs}"


def test_evaluate_batch_checks_graph_mode():
    from sgformer_b200 import large_gnns as LG
    from sgformer_b200.eval import evaluate_batch
    from sgformer_b200.graph import Graph
    n, d, c = 3000, 8, 3
    ei = _graph(n, 20000, 1, False).to(DEV)
    x = torch.randn(n, d, device=DEV)
    label = torch.randint(0, c, (n, 1), device=DEV)
    split = {"train": torch.arange(0, 1000), "valid": torch.arange(1000, 2000), "test": torch.arange(2000, 3000)}
    ds = SimpleNamespace(graph={"edge_index": ei, "node_feat": x}, label=label)
    model = LG.GAT(d, 8, c).to(DEV)
    with pytest.raises(ValueError, match="self_loop_mode 0.*self_loop_mode 1"):
        evaluate_batch(model, ds, split, SimpleNamespace(batch_size=1500), DEV, n, label, graph=Graph(ei, n, 0))
    got = evaluate_batch(model, ds, split, SimpleNamespace(batch_size=1500), DEV, n, label, graph=Graph(ei, n, 1))
    assert all(0.0 <= a <= 1.0 for a in got[:3])
    # a host edge list: the parent CSR is built once, holds no device copy of the edge list, and is reused by the next call
    from sgformer_b200 import eval as ev
    host_ds = SimpleNamespace(graph={"edge_index": ei.cpu(), "node_feat": x.cpu()}, label=label.cpu())
    first = evaluate_batch(model, host_ds, split, SimpleNamespace(batch_size=1500), DEV, n, label)
    (held, parent), = ev._HOST_PARENT.values()
    assert held is host_ds.graph["edge_index"] and parent.edge_index is None and parent.self_loop_mode == 1
    second = evaluate_batch(model, host_ds, split, SimpleNamespace(batch_size=1500), DEV, n, label)
    assert all(0.0 <= a <= 1.0 for a in first[:3] + second[:3])
    assert next(iter(ev._HOST_PARENT.values()))[1] is parent
