"""The drop-in `ours.py` files export the reference's names and build our model from the reference's recorded constructor call
(construction is CPU-safe, no compute)."""
import importlib
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _import_from(paths, name):
    for m in ("ours", "models", "parse", "gnns"):
        sys.modules.pop(m, None)
    saved = list(sys.path)
    sys.path[:0] = paths
    try:
        return importlib.import_module(name)
    finally:
        sys.path[:] = saved
        for m in ("ours", "models", "parse", "gnns"):
            sys.modules.pop(m, None)


@pytest.mark.parametrize("variant,names", [
    ("large", ["SGFormer", "TransConv", "TransConvLayer", "GraphConv", "GraphConvLayer"]),
    ("100M", ["SGFormer", "TransConv", "TransConvLayer", "GraphConv", "GraphConvLayer", "full_attention_conv"]),
    ("medium", ["SGFormer", "TransConv", "TransConvLayer", "full_attention_conv"]),
])
def test_dropin_exports(variant, names):
    mod = _import_from([os.path.join(ROOT, "sgformer_b200", "dropin", variant)], "ours")
    for n in names:
        assert hasattr(mod, n), f"dropin/{variant}/ours.py lacks {n}"
    assert mod.SGFormer.__module__.startswith("sgformer_b200")


def test_reference_parse_builds_our_model_large():
    """The constructor call of the reference's own large/parse.py for the amazon2m recipe (large/run.sh:15-19), recorded in
    tests/golden/parse_large_sgformer.json by tests/make_golden.py parse_large, builds the drop-in model with that config."""
    import json
    with open(os.path.join(ROOT, "tests", "golden", "parse_large_sgformer.json")) as f:
        call = json.load(f)
    ours = _import_from([os.path.join(ROOT, "sgformer_b200", "dropin", "large")], "ours")
    model = ours.SGFormer(*call["args"], **call["kwargs"]).to("cpu")
    assert type(model).__module__ == "sgformer_b200.large"
    cfg = model._cfg()
    assert cfg["gnn_use_init"] and cfg["gnn_num_layers"] == 3 and cfg["hidden"] == 256 and cfg["graph_weight"] == 0.5
    assert cfg["trans_use_act"] is False and cfg["trans_use_bn"] is True
    assert len(model.params1) > 0 and len(model.params2) > 0
