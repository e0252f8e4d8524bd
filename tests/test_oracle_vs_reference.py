"""Property test: the oracle against the unmodified reference modules on randomly drawn configurations and graphs — isolated
nodes, directed/asymmetric edges, duplicates, self loops, odd sizes, 1-4 heads (SURVEY.md §4 'property' row).  The reference's
outputs for 25 seeded draws are stored in tests/golden/oracle_property.pt (tests/make_golden.py oracle_property)."""
import os

import torch

from oracle import sgformer_oracle as O

CASES = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_property.pt"), weights_only=False)


def test_oracle_equals_reference():
    assert len(CASES) == 25
    for i, c in enumerate(CASES):
        cfg, sd, ei, x = c["cfg"], c["state_dict"], c["edge_index"], c["x"]
        for training, ref in ((False, c["ref_eval"]), (True, c["ref_train"])):
            out = O.sgformer_forward(cfg, {k: v.clone() for k, v in sd.items()}, x, ei, training=training)
            err = (out - ref).abs().max().item()
            assert err <= 1e-4 * max(1.0, ref.abs().max().item()), f"case {i} ({cfg['variant']}) training={training}: {err:.3e}"
