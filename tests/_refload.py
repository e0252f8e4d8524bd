"""Helpers to import the UNMODIFIED reference modules from a reference checkout (SGFORMER_REFERENCE,
default ../reference beside this repository) through tests/ref_shims, for tests/make_golden.py; the tests themselves use the committed fixtures."""
import importlib
import os
import sys

REF_ROOT = os.environ.get("SGFORMER_REFERENCE",
                          os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))), "reference"))
SHIMS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_shims")
_VARIANT_DIR = {"large": "large", "100M": "100M", "medium": "medium"}


def reference_available() -> bool:
    return os.path.isdir(REF_ROOT)


def import_reference(variant: str):
    """Return the reference `ours` module of `variant` (fresh import; also returns `models` for medium)."""
    d = os.path.join(REF_ROOT, _VARIANT_DIR[variant])
    for name in ("ours", "models", "parse", "gnns", "data_utils", "dataset", "logger", "eval"):
        sys.modules.pop(name, None)
    saved = list(sys.path)
    sys.path[:0] = [SHIMS, d]
    try:
        ours = importlib.import_module("ours")
        models = importlib.import_module("models") if variant == "medium" else None
    finally:
        sys.path[:] = saved
        for name in ("ours", "models"):
            sys.modules.pop(name, None)
    return ours, models


def build_reference_model(variant: str, cfg: dict):
    """Instantiate the reference SGFormer for a normalised oracle config (oracle.make_config)."""
    ours, models = import_reference(variant)
    if variant == "medium":
        gnn = models.GCN(cfg["in_channels"], cfg["hidden"], cfg["hidden"], num_layers=cfg["gcn_num_layers"],
                         dropout=cfg["gcn_dropout"], use_bn=cfg["gcn_use_bn"])
        m = ours.SGFormer(cfg["in_channels"], cfg["hidden"], cfg["out_channels"],
                          num_layers=cfg["trans_num_layers"], num_heads=cfg["num_heads"], alpha=cfg["alpha"],
                          dropout=cfg["trans_dropout"], use_bn=cfg["trans_use_bn"],
                          use_residual=cfg["trans_use_residual"], use_weight=cfg["trans_use_weight"],
                          use_graph=cfg["use_graph"], graph_weight=cfg["graph_weight"], gnn=gnn,
                          aggregate=cfg["aggregate"])
    else:
        kw = dict(trans_num_layers=cfg["trans_num_layers"], trans_num_heads=cfg["num_heads"],
                  trans_dropout=cfg["trans_dropout"], trans_use_bn=cfg["trans_use_bn"],
                  trans_use_residual=cfg["trans_use_residual"], trans_use_weight=cfg["trans_use_weight"],
                  trans_use_act=cfg["trans_use_act"], gnn_num_layers=cfg["gnn_num_layers"],
                  gnn_dropout=cfg["gnn_dropout"], gnn_use_weight=cfg["gnn_use_weight"],
                  gnn_use_init=cfg["gnn_use_init"], gnn_use_bn=cfg["gnn_use_bn"],
                  gnn_use_residual=cfg["gnn_use_residual"], gnn_use_act=cfg["gnn_use_act"],
                  use_graph=cfg["use_graph"], graph_weight=cfg["graph_weight"], aggregate=cfg["aggregate"])
        if variant == "100M":
            kw["alpha"] = cfg["alpha"]
        m = ours.SGFormer(cfg["in_channels"], cfg["hidden"], cfg["out_channels"], **kw)
    return m, ours


class FakeDataset:
    """The `data` object medium/ours.py:134-136 reads."""

    def __init__(self, x, edge_index):
        self.graph = {"node_feat": x, "edge_index": edge_index, "num_nodes": x.shape[0]}


def run_reference(variant, model, x, edge_index):
    if variant == "medium":
        return model(FakeDataset(x, edge_index))
    return model(x, edge_index)
