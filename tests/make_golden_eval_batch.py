"""Generate tests/golden/eval_batch.pt from the UNMODIFIED reference large/eval.py (evaluate_batch and its eval_acc) through
tests/ref_shims:  python tests/make_golden_eval_batch.py  (reference checkout in SGFORMER_REFERENCE or ../reference).

Per case (inputs regenerated from the seeds by make_case / split_logits): the accuracies the reference's evaluate_batch returns
on the CPU for `RoundedSum` under a fixed torch seed (its `randperm`), and the (rows, hits) its eval_acc returns for each split
of fixed logits with planted ties.  Pins the count contract of sgf_eval_acc_splits and the restatement of evaluate_batch that
tests/test_gpu_eval_batch.py compares sgformer_b200.eval.evaluate_batch with."""
import importlib
import os
import sys
from types import SimpleNamespace

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

OUT = os.path.join(HERE, "golden", "eval_batch.pt")
# name -> (n, e, classes, batch_size, seed, overlapping splits); "exact" has n a multiple of batch_size (an empty last batch)
CASES = {"partial": (1000, 6000, 5, 300, 0, False), "exact": (900, 5000, 3, 300, 1, False), "overlap": (700, 4000, 7, 128, 2, True)}


class RoundedSum(torch.nn.Module):
    """A deterministic stand-in model on any device: logits = round(sum over in-edges of x W), integer-valued, so that argmax
    ties with the row maximum are frequent and the batch structure changes the result."""

    def __init__(self, d, c, seed):
        super().__init__()
        self.w = torch.nn.Parameter(torch.randn(d, c, generator=torch.Generator().manual_seed(seed)), requires_grad=False)

    def forward(self, x, edge_index):
        h = x @ self.w.to(x.device)
        out = torch.zeros_like(h).index_add_(0, edge_index[1], h[edge_index[0]])
        return torch.round(out)


def make_case(n, e, c, seed, overlap):
    g = torch.Generator().manual_seed(100 + seed)
    ei = torch.randint(0, n - n // 50, (2, e), generator=g)          # the top 2 % of the nodes are isolated
    ar = torch.arange(n)
    ei = torch.cat([ei[:, ei[0] != ei[1]], torch.stack([ar, ar])], 1)  # main-batch.py:97-98: one self loop per node
    x = torch.randint(-2, 3, (n, 4), generator=g).float()
    label = torch.randint(0, c, (n, 1), generator=g)
    perm = torch.randperm(n, generator=g)
    split = {"train": perm[: n // 2], "valid": perm[n // 2: 3 * n // 4], "test": perm[3 * n // 4:]}
    if overlap:
        split["test"] = torch.cat([split["test"], perm[: n // 10]])
    return dict(edge_index=ei, x=x, label=label, split=split, classes=c, model_seed=seed)


def split_logits(n, c, seed):
    """Fixed logits with exact ties with the row maximum, labels, and split codes (bits 1 train, 2 valid, 4 test)."""
    g = torch.Generator().manual_seed(seed)
    logits = torch.randint(-3, 4, (n, c), generator=g).float()
    rows = torch.randperm(n, generator=g)[: n // 4]
    logits[rows, (rows % c)] = logits[rows].max(dim=1).values
    label = torch.randint(0, c, (n, 1), generator=g)
    code = torch.randint(0, 8, (n,), generator=g).to(torch.uint8)
    return logits, label, code


def main():
    from _refload import REF_ROOT, SHIMS
    for name in ("eval", "data_utils"):
        sys.modules.pop(name, None)
    saved = list(sys.path)
    sys.path[:0] = [SHIMS, os.path.join(REF_ROOT, "large")]
    try:
        ev = importlib.import_module("eval")
    finally:
        sys.path[:] = saved
    out = {}
    for name, (n, e, c, bs, seed, overlap) in CASES.items():
        case = make_case(n, e, c, seed, overlap)
        ds = SimpleNamespace(graph={"edge_index": case["edge_index"], "node_feat": case["x"]}, label=case["label"])
        model = RoundedSum(case["x"].shape[1], c, seed)
        torch.manual_seed(1000 + seed)
        res = ev.evaluate_batch(model, ds, case["split"], SimpleNamespace(batch_size=bs), "cpu", n, case["label"])
        logits, label, code = split_logits(n, c, seed)
        out[name] = dict(torch_seed=1000 + seed, accuracies=tuple(float(a) for a in res[:3]),
                         eval_acc=tuple(ev.eval_acc(label[(code & bit) != 0], logits[(code & bit) != 0]) for bit in (1, 2, 4)))
    torch.save(out, OUT)
    print({k: (v["accuracies"], v["eval_acc"]) for k, v in out.items()})


if __name__ == "__main__":
    main()
