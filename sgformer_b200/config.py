"""Normalised encoder configuration shared by the three reference variants (see SURVEY.md §8a "variant differences")."""

_DEFAULTS = dict(
    variant="large", num_heads=1, trans_num_layers=1, trans_dropout=0.5, trans_use_bn=True, trans_use_residual=True,
    trans_use_weight=True, trans_use_act=True, alpha=0.5, gnn_num_layers=1, gnn_dropout=0.5, gnn_use_weight=True,
    gnn_use_init=False, gnn_use_bn=True, gnn_use_residual=True, gnn_use_act=True, use_graph=True, graph_weight=0.8,
    aggregate="add", gcn_num_layers=2, gcn_dropout=0.5, gcn_use_bn=True, gcn_normalize=True, gnn_kind="gcn", gcn_jk="max",
)


def make_config(variant: str, in_channels: int, hidden: int, out_channels: int, **kw) -> dict:
    if variant not in ("large", "100M", "medium"):
        raise ValueError(f"unknown variant {variant}")
    cfg = dict(_DEFAULTS)
    cfg.update(variant=variant, in_channels=int(in_channels), hidden=int(hidden), out_channels=int(out_channels))
    for k, v in kw.items():
        if k not in cfg:
            raise KeyError(f"unknown config key {k}")
        cfg[k] = v
    if cfg["gnn_kind"] not in ("gcn", "gat", "gcnjk"):
        raise ValueError(f"unknown GNN kind {cfg['gnn_kind']!r}")
    if cfg["gcn_jk"] not in ("max", "cat"):
        raise ValueError(f"unknown JumpingKnowledge mode {cfg['gcn_jk']!r}")
    if cfg["aggregate"] not in ("add", "cat"):
        raise ValueError(f"Invalid aggregate type:{cfg['aggregate']}")
    return cfg
