"""Generate tests/golden/dropout.pt from the UNMODIFIED reference with dropout on (run in the build container only):

    SGFORMER_REFERENCE=/path/to/SGFormer python tests/make_golden_dropout.py

The reference's own imports must resolve (tests/ref_shims covers torch_geometric / torch_sparse; medium/models.py also imports
scipy).

Every dropout of the reference is a call `F.dropout(x, p=..., training=...)` (large/ours.py, 100M/ours.py, medium/ours.py,
medium/models.py, medium/difformer.py).  Here torch.nn.functional.dropout is patched for the training forward: each call
draws a Bernoulli keep mask from a seeded generator, records it and returns x * mask / (1 - p).  The fixture stores the
masks in call order (bit-packed) with the training logits, parameter gradients, grad_x and the BatchNorm buffers after the
step; tests/test_dropout_replay.py replays the masks in the oracles and checks that they reproduce these values, which pins
where the oracles place each dropout.

Inputs, weights and loss weights are not stored again: each case names the p = 0 fixture (model_<name>.pt or a case of
difformer.pt) whose state_dict, x, edge_index and loss_weight it reuses, with only the dropout rates changed.  Writes only
this file."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from dropout_mask import pack_mask  # noqa: E402
from make_golden import GOLD  # noqa: E402
from make_golden_difformer import _flat_dict  # noqa: E402

SGFORMER_CASES = {          # base fixture -> dropout rates (large/run.sh, 100M/run.sh, medium/run.sh use 0.2 - 0.6)
    "large_add_init": dict(trans_dropout=0.2, gnn_dropout=0.5),     # GraphConv with BN, use_init and residual
    "large_cat_heads2": dict(trans_dropout=0.5, gnn_dropout=0.3),   # two heads, 'cat', three GraphConv layers
    "large_nores": dict(trans_dropout=0.6, gnn_dropout=0.2),        # no residuals, no GraphConv activation
    "100M_alpha": dict(trans_dropout=0.3, gnn_dropout=0.6),
    "medium_gcn": dict(trans_dropout=0.2, gcn_dropout=0.6),          # GCN backbone, four layers
    "medium_res_heads2": dict(trans_dropout=0.4, gcn_dropout=0.5),   # two heads, residual
}
DIFFORMER_CASES = {         # case of difformer.pt -> dropout (medium/run.sh: 0.6 on Actor / Squirrel)
    "default": 0.6,
    "no_graph": 0.5,
    "no_res_no_bn": 0.2,
    "source": 0.4,
    "graph_weight": 0.3,
}


def _unflat(f):
    out, o = {}, 0
    for name, shape in zip(f["names"], f["shapes"]):
        k = int(torch.Size(shape).numel())
        out[name] = f["flat"][o:o + k].reshape(shape).clone()
        o += k
    return out


class _RecordingDropout:
    def __init__(self, seed):
        self.gen = torch.Generator().manual_seed(seed)
        self.masks = []

    def __call__(self, x, p=0.5, training=True, inplace=False):
        if not training or p == 0.0:
            return x
        m = torch.rand(x.shape, generator=self.gen) >= p
        self.masks.append((float(p), m))
        return x * m.to(x.dtype) / (1.0 - p)


def _train_step(run, seed):
    """Runs the training forward `run()` with the recording dropout -> (masks in call order, output); the caller runs the backward."""
    import torch.nn.functional as F
    rec = _RecordingDropout(seed)
    saved = F.dropout
    F.dropout = rec
    try:
        out = run()
    finally:
        F.dropout = saved
    return rec.masks, out


def sgformer_cases():
    from _refload import build_reference_model, run_reference
    out = {}
    for i, (name, rates) in enumerate(SGFORMER_CASES.items()):
        fx = torch.load(os.path.join(GOLD, f"model_{name}.pt"), weights_only=False)
        cfg = dict(fx["cfg"], **rates)
        model, _ = build_reference_model(cfg["variant"], cfg)
        model.load_state_dict(fx["state_dict"])
        model.train()
        xg = fx["x"].clone().requires_grad_(True)
        masks, y = _train_step(lambda: run_reference(cfg["variant"], model, xg, fx["edge_index"]), 500 + i)
        (y * fx["loss_weight"]).sum().backward()
        grads = {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}
        bufs = {k: v.clone() for k, v in model.state_dict().items() if "running" in k}
        out[name] = dict(base=f"model_{name}.pt", rates=rates, masks=[dict(p=p, **pack_mask(m.numpy())) for p, m in masks],
                         out_train=y.detach().clone(), grad_x=xg.grad.clone(), grads=_flat_dict(grads),
                         buffers_after_train=_flat_dict(bufs) if bufs else None)
        print(name, len(masks), "dropout calls")
    return out


def difformer_cases():
    import importlib
    from _refload import REF_ROOT, SHIMS, FakeDataset
    sys.modules.pop("difformer", None)
    saved = list(sys.path)
    sys.path[:0] = [SHIMS, os.path.join(REF_ROOT, "medium")]
    try:
        ref = importlib.import_module("difformer")
    finally:
        sys.path[:] = saved
        sys.modules.pop("difformer", None)
    base = torch.load(os.path.join(GOLD, "difformer.pt"), weights_only=False)
    out = {}
    for i, (name, p) in enumerate(DIFFORMER_CASES.items()):
        c = base[name]
        kw = dict(c["kw"], dropout=p)
        model = ref.DIFFormer(c["in_channels"], c["hidden"], c["out_channels"], **kw)
        model.load_state_dict(_unflat(c["state_dict"]))
        model.train()
        xg = c["x"].clone().requires_grad_(True)
        ei = c["edge_index"].long()
        masks, y = _train_step(lambda: model(FakeDataset(xg, ei)), 700 + i)
        (y * c["loss_weight"]).sum().backward()
        grads = {k: p_.grad.clone() for k, p_ in model.named_parameters() if p_.grad is not None}
        out[name] = dict(base=name, dropout=p, masks=[dict(p=pp, **pack_mask(m.numpy())) for pp, m in masks],
                         out_train=y.detach().clone(), grad_x=xg.grad.clone(), grads=_flat_dict(grads))
        print("difformer", name, len(masks), "dropout calls")
    return out


if __name__ == "__main__":
    torch.set_num_threads(1)        # the reference's sparse backward sums in thread order: one thread makes the file reproducible
    path = os.path.join(GOLD, "dropout.pt")
    torch.save(dict(sgformer=sgformer_cases(), difformer=difformer_cases()), path)
    print("dropout.pt", os.path.getsize(path), "bytes")
