"""Generate tests/golden/sgformer_gat_attention.pt from the UNMODIFIED reference medium/ablation/oursGAT.py (and its models.GCN)
through tests/ref_shims:  python tests/make_golden_gat_attention.py  (reference checkout in SGFORMER_REFERENCE or ../reference).

Per case: the fp32 state_dict the reference initialises under a seed and the one its reset_parameters() then draws, inputs, and in
fp64 and fp32 (from the initial state_dict) the eval and train logits (dropout 0), the parameter gradients and grad_x of a fixed
linear loss of the train logits, and the names whose gradient stays None.  Also the type of the exception the reference's
get_attentions raises.  GAT backbones are not covered: the shims stub PyG's GATConv, so the reference GAT cannot run here."""
import importlib
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from _refload import REF_ROOT, SHIMS  # noqa: E402

OUT = os.path.join(HERE, "golden", "sgformer_gat_attention.pt")
N, D_IN, C = 24, 10, 3
# (name, hidden, num_heads, use_weight, use_residual, use_bn, use_graph, aggregate, Wq scale)
CASES = [
    ("h1", 8, 1, True, True, True, False, "add", 1.0),
    ("h2_noweight", 8, 2, False, True, True, False, "add", 1.0),
    ("h4_nores", 8, 4, True, False, True, False, "add", 1.0),
    ("h2_noln", 8, 2, True, True, False, False, "add", 1.0),
    ("h3_dk5", 16, 3, True, True, True, False, "add", 1.0),
    ("h2_gcn_add", 8, 2, True, True, True, True, "add", 1.0),
    ("h4_gcn_cat", 8, 4, False, True, True, True, "cat", 1.0),
    ("h2_large_scores", 8, 2, True, True, True, False, "add", 150.0),
]


class _Data:
    def __init__(self, x, ei):
        self.graph = {"node_feat": x, "edge_index": ei}


def _import():
    d = os.path.join(REF_ROOT, "medium", "ablation")
    for name in ("oursGAT", "models"):
        sys.modules.pop(name, None)
    sys.path[:0] = [SHIMS, d]
    return importlib.import_module("oursGAT"), importlib.import_module("models")


def _max_score(model, x, dtype):
    """Largest |q.k / sqrt(dk)| of the first layer (hooked on GATAttention's projections)."""
    seen = {}
    att = model.trans_conv.convs[0].attention.attention
    hooks = [att.Wq.register_forward_hook(lambda m, i, o: seen.__setitem__("q", o)),
             att.Wk.register_forward_hook(lambda m, i, o: seen.__setitem__("k", o))]
    model.eval()
    with torch.no_grad():
        model(_Data(x.to(dtype), None))
    for h in hooks:
        h.remove()
    q = seen["q"].view(-1, att.num_heads, att.dk)
    k = seen["k"].view(-1, att.num_heads, att.dk)
    return (torch.einsum("nhm,lhm->nlh", q, k) / att.dk ** 0.5).abs().max().item()


def _run(model, x, ei, wout, dtype):
    m = model.to(dtype)
    xd = x.to(dtype).clone().requires_grad_()
    data = _Data(xd, ei)
    m.eval()
    with torch.no_grad():
        eval_logits = m(_Data(x.to(dtype), ei)).detach()
    m.train()
    m.zero_grad()
    train_logits = m(data)
    (train_logits * wout.to(dtype)).sum().backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}
    none = [k for k, p in m.named_parameters() if p.grad is None]
    return dict(eval_logits=eval_logits, train_logits=train_logits.detach(), grads=grads, grad_x=xd.grad.detach(),
                none_grads=none)


def main():
    gat, models = _import()
    g = torch.Generator().manual_seed(0)
    x = torch.randn(N, D_IN, generator=g)
    src = torch.randint(0, N, (60,), generator=g)
    dst = torch.randint(0, N, (60,), generator=g)
    ei = torch.cat([torch.stack([src, dst]), torch.stack([dst, src])], 1)
    out = dict(x=x, edge_index=ei, cases={})

    def build(hid, heads, use_weight, use_res, use_bn, use_graph, agg):
        gnn = models.GCN(D_IN, hid, hid, num_layers=2, dropout=0.0, use_bn=True) if use_graph else None
        return gat.SGFormerGAT(D_IN, hid, C, num_layers=2, num_heads=heads, alpha=0.5, dropout=0.0, use_bn=use_bn,
                               use_residual=use_res, use_weight=use_weight, use_graph=use_graph, graph_weight=0.8, gnn=gnn,
                               aggregate=agg)

    for i, (name, hid, heads, use_weight, use_res, use_bn, use_graph, agg, wq_scale) in enumerate(CASES):
        spec = (hid, heads, use_weight, use_res, use_bn, use_graph, agg)
        torch.manual_seed(100 + i)
        model = build(*spec)
        init_sd = {k: v.clone() for k, v in model.state_dict().items()}
        torch.manual_seed(200 + i)
        model.reset_parameters()
        reset_sd = {k: v.clone() for k, v in model.state_dict().items()}
        sd = {k: v.clone() for k, v in init_sd.items()}
        for j in range(2):
            for t in ("weight", "bias"):
                sd[f"trans_conv.convs.{j}.attention.attention.Wq.{t}"] *= wq_scale
        wout = torch.randn(N, C, generator=g)
        rec = dict(config=dict(hidden=hid, heads=heads, use_weight=use_weight, use_residual=use_res, use_bn=use_bn,
                               use_graph=use_graph, aggregate=agg, wq_scale=wq_scale),
                   init_state_dict=init_sd, reset_state_dict=reset_sd, state_dict=sd, wout=wout)
        model64 = build(*spec)
        model64.load_state_dict(sd)
        rec["fp64"] = _run(model64, x, ei, wout, torch.float64)
        model.load_state_dict(sd)
        rec["fp32"] = _run(model, x, ei, wout, torch.float32)
        if not use_graph:
            rec["max_abs_score"] = _max_score(model64, x, torch.float64)
        out["cases"][name] = rec
    m = build(8, 2, True, True, True, False, "add")
    try:
        m.get_attentions(x)
        out["get_attentions_error"] = None
    except Exception as e:  # noqa: BLE001 - the type is what is recorded
        out["get_attentions_error"] = type(e).__name__
    torch.save(out, OUT)
    print(OUT, os.path.getsize(OUT), "bytes", {k: round(v.get("max_abs_score", 0), 1) for k, v in out["cases"].items()},
          out["get_attentions_error"])


if __name__ == "__main__":
    main()
