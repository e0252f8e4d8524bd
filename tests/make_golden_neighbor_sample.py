"""Generate tests/golden/neighbor_sample.pt from the UNMODIFIED reference 100M/ours.py through tests/ref_shims:
    python tests/make_golden_neighbor_sample.py   (reference checkout in SGFORMER_REFERENCE or ../reference)

A neighbour-sampled batch of a small directed graph (the numpy restatement tests/neighbor_sample_ref.py at the 100M recipe's
fan-outs [15, 10, 5] on 40 seeds, with hub rows longer than the fan-outs), and the reference 100M SGFormer's eval output on
(x[idx], sampled edge_index), the forward nb-sample.py:27-46 runs per batch.  Pins the restatement's batch and the oracle's 100M
forward on a sampled edge list (in-degree 0 for the last hop's nodes)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from oracle import sgformer_oracle as O  # noqa: E402
from _refload import build_reference_model, run_reference  # noqa: E402
import neighbor_sample_ref as R  # noqa: E402

OUT = os.path.join(HERE, "golden", "neighbor_sample.pt")


def make_case():
    """n = 600 nodes, power-law-ish sources, hubs 0 and 1 (300 in-edges each), duplicates, self loops and isolated nodes."""
    g = torch.Generator().manual_seed(21)
    n, e = 600, 5000
    src = (580 * torch.rand(e, generator=g) ** 2).long()
    dst = torch.randint(0, 580, (e,), generator=g)
    dst[:300], dst[300:600] = 0, 1
    ei = torch.cat([torch.stack([src, dst]), torch.stack([src[:200], dst[:200]]), torch.arange(0, 580, 9).repeat(2, 1)], 1)
    seeds = torch.randperm(580, generator=g)[:40]
    seeds[:2] = torch.tensor([0, 1])
    return dict(n=n, edge_index=ei, seeds=seeds, num_neighbors=[15, 10, 5], seed=0x5EED1234ABCD)


def main():
    case = make_case()
    rowptr, col = R.csr_of(case["edge_index"].numpy(), case["n"])
    idx, ei, _ = R.sample(rowptr, col, case["seeds"].numpy(), case["num_neighbors"], case["seed"])
    idx, ei = torch.from_numpy(idx), torch.from_numpy(ei)
    d, h, c = 12, 16, 5
    cfg = O.make_config("100M", d, h, c, alpha=0.4, gnn_num_layers=3, gnn_use_init=True, graph_weight=0.8, gnn_dropout=0.0,
                        trans_dropout=0.0)
    torch.manual_seed(1234)
    model, _ = build_reference_model("100M", cfg)
    model.reset_parameters()
    x = torch.randn(case["n"], d, generator=torch.Generator().manual_seed(5))
    model.eval()
    with torch.no_grad():
        out = run_reference("100M", model, x[idx], ei).clone()
    torch.save(dict(case, cfg=cfg, state_dict={k: v.clone() for k, v in model.state_dict().items()}, x=x, idx=idx,
                    sampled_edge_index=ei, out_eval=out), OUT)
    print("neighbor_sample:", idx.numel(), "nodes", ei.shape[1], "edges", float(out.abs().mean()))


if __name__ == "__main__":
    main()
