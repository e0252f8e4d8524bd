"""Generate tests/golden/sgformer_softmax.pt from the UNMODIFIED reference medium/ablation/oursSOFT.py (and its models.GCN)
through tests/ref_shims:  python tests/make_golden_softmax.py  (reference checkout in SGFORMER_REFERENCE or ../reference).

Per case: the fp32 state_dict the reference initialises, inputs, and in fp64 and fp32 the eval and train logits (dropout 0),
the parameter gradients and grad_x of a fixed linear loss of the train logits, and get_attentions.  GAT backbones are not
covered: the shims stub PyG's GATConv, so the reference GAT cannot run here."""
import importlib
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from _refload import REF_ROOT, SHIMS  # noqa: E402

OUT = os.path.join(HERE, "golden", "sgformer_softmax.pt")
N, D_IN, HID, C = 24, 10, 8, 3
# (name, num_heads, use_weight, use_residual, use_bn, use_graph, aggregate)
CASES = [
    ("h1", 1, True, True, True, False, "add"),
    ("h2_noweight", 2, False, True, True, False, "add"),
    ("h4_nores", 4, True, False, True, False, "add"),
    ("h2_noln", 2, True, True, False, False, "add"),
    ("h2_gcn_add", 2, True, True, True, True, "add"),
    ("h4_gcn_cat", 4, False, True, True, True, "cat"),
]


class _Data:
    def __init__(self, x, ei):
        self.graph = {"node_feat": x, "edge_index": ei}


def _import():
    d = os.path.join(REF_ROOT, "medium", "ablation")
    for name in ("oursSOFT", "models"):
        sys.modules.pop(name, None)
    sys.path[:0] = [SHIMS, d]
    return importlib.import_module("oursSOFT"), importlib.import_module("models")


def _run(model, x, ei, wout, dtype):
    m = model.to(dtype)
    xd = x.to(dtype).clone().requires_grad_()
    data = _Data(xd, ei)
    m.eval()
    with torch.no_grad():
        eval_logits = m(_Data(x.to(dtype), ei)).detach()
        atts = m.get_attentions(x.to(dtype)).detach()
    m.train()
    m.zero_grad()
    train_logits = m(data)
    (train_logits * wout.to(dtype)).sum().backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}
    return dict(eval_logits=eval_logits, train_logits=train_logits.detach(), grads=grads, grad_x=xd.grad.detach(), attentions=atts)


def main():
    soft, models = _import()
    g = torch.Generator().manual_seed(0)
    x = torch.randn(N, D_IN, generator=g)
    src = torch.randint(0, N, (60,), generator=g)
    dst = torch.randint(0, N, (60,), generator=g)
    ei = torch.cat([torch.stack([src, dst]), torch.stack([dst, src])], 1)
    out = dict(x=x, edge_index=ei, cases={})
    for i, (name, heads, use_weight, use_res, use_bn, use_graph, agg) in enumerate(CASES):
        torch.manual_seed(100 + i)
        gnn = models.GCN(D_IN, HID, HID, num_layers=2, dropout=0.0, use_bn=True) if use_graph else None
        model = soft.SGFormerSOFT(D_IN, HID, C, num_layers=2, num_heads=heads, alpha=0.5, dropout=0.0, use_bn=use_bn,
                                  use_residual=use_res, use_weight=use_weight, use_graph=use_graph, graph_weight=0.8, gnn=gnn,
                                  aggregate=agg)
        sd = {k: v.clone() for k, v in model.state_dict().items()}
        wout = torch.randn(N, C, generator=g)
        rec = dict(config=dict(heads=heads, use_weight=use_weight, use_residual=use_res, use_bn=use_bn, use_graph=use_graph,
                               aggregate=agg), state_dict=sd, wout=wout)
        model64 = soft.SGFormerSOFT(D_IN, HID, C, num_layers=2, num_heads=heads, alpha=0.5, dropout=0.0, use_bn=use_bn,
                                    use_residual=use_res, use_weight=use_weight, use_graph=use_graph, graph_weight=0.8,
                                    gnn=models.GCN(D_IN, HID, HID, num_layers=2, dropout=0.0, use_bn=True) if use_graph else None,
                                    aggregate=agg)
        model64.load_state_dict(sd)
        rec["fp64"] = _run(model64, x, ei, wout, torch.float64)
        model.load_state_dict(sd)
        rec["fp32"] = _run(model, x, ei, wout, torch.float32)
        out["cases"][name] = rec
    torch.save(out, OUT)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
