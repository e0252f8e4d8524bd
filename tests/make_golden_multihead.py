"""Generate tests/golden/multihead_shared_value.pt from the UNMODIFIED reference (run in the build container only):

    python tests/make_golden_multihead.py

SGFormer attention with several heads and no value projection (use_weight=False, num_heads > 1): the reference's
`value = source_input.reshape(-1, 1, D)` is broadcast across the heads by full_attention_conv's einsum and `+ N * vs`
(medium/ours.py:21-23, 84; large/ours.py:128-157; 100M/ours.py), so every head attends with its own q and k over the layer input.
The fixture holds, per model configuration, the seeded inputs, the state_dict (no Wv keys), eval and train logits, every parameter
and input gradient, the LayerNorm / BatchNorm buffers after the training step and get_attentions; and full_attention_conv called
with a one-head vs, with its gradients."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from oracle import sgformer_oracle as O  # noqa: E402
from _refload import build_reference_model, import_reference, run_reference  # noqa: E402
from make_golden import perturb_  # noqa: E402

OUT = os.path.join(HERE, "golden", "multihead_shared_value.pt")

# name: variant, n, d, h, c, config keywords (oracle.make_config; dropout 0 everywhere, so train and eval differ by the
# BatchNorm statistics only)
_T = dict(trans_use_weight=False, trans_dropout=0.0, gnn_dropout=0.0)
_M = dict(use_weight=False, dropout=0.0, gcn_dropout=0.0)
CASES = {
    "large_h2_res_ln_add": ("large", 70, 9, 16, 4, dict(_T, trans_num_heads=2, trans_num_layers=2, gnn_num_layers=2, graph_weight=0.6)),
    "large_h3_cat_plain": ("large", 53, 7, 8, 3, dict(_T, trans_num_heads=3, trans_num_layers=1, trans_use_residual=False,
                                                      trans_use_bn=False, trans_use_act=False, gnn_num_layers=1, aggregate="cat")),
    "large_h4_nograph": ("large", 41, 6, 16, 5, dict(_T, trans_num_heads=4, trans_num_layers=2, trans_use_bn=False,
                                                     use_graph=False)),
    "100M_h3_res_ln_add": ("100M", 64, 8, 16, 3, dict(_T, trans_num_heads=3, trans_num_layers=2, alpha=0.3, gnn_num_layers=2,
                                                      gnn_use_init=True, graph_weight=0.7)),
    "100M_h2_cat_nores": ("100M", 47, 5, 8, 4, dict(_T, trans_num_heads=2, trans_num_layers=1, trans_use_residual=False, alpha=0.6,
                                                    gnn_num_layers=1, aggregate="cat")),
    "medium_h2_res_ln_add": ("medium", 60, 10, 16, 4, dict(_M, num_heads=2, num_layers=2, alpha=0.4, use_residual=True,
                                                           gcn_num_layers=2, graph_weight=0.8)),
    "medium_h4_cat_plain": ("medium", 45, 6, 8, 3, dict(_M, num_heads=4, num_layers=1, use_residual=False, use_bn=False,
                                                        gcn_num_layers=3, aggregate="cat")),
    "medium_h3_nograph": ("medium", 38, 7, 16, 5, dict(_M, num_heads=3, num_layers=2, alpha=0.7, use_residual=True, use_bn=False,
                                                       use_graph=False, gcn_num_layers=2)),
}


def graph(n, seed):
    """Directed edges with duplicates, self loops, and node n-1 isolated."""
    g = torch.Generator().manual_seed(seed)
    live = n - 1
    ei = torch.stack([torch.randint(0, live, (4 * n,), generator=g), torch.randint(0, live, (4 * n,), generator=g)])
    loops = torch.randint(0, live, (n // 6,), generator=g)
    ei = torch.cat([ei, ei[:, :n // 5], torch.stack([loops, loops])], 1)
    return ei[:, torch.randperm(ei.shape[1], generator=g)].contiguous()


def model_case(name, spec):
    variant, n, d, h, c, kw = spec
    torch.manual_seed(4321)
    cfg = O.make_config(variant, d, h, c, **kw)
    model, _ = build_reference_model(variant, cfg)
    model.reset_parameters()
    perturb_(model, 7)
    g = torch.Generator().manual_seed(55)
    x = torch.randn(n, d, generator=g)
    lw = torch.randn(n, c, generator=g)
    ei = graph(n, 17)
    sd0 = {k: v.clone() for k, v in model.state_dict().items()}
    assert not any(".Wv." in k for k in sd0)

    model.eval()
    with torch.no_grad():
        out_eval = run_reference(variant, model, x, ei).clone()
        att = model.get_attentions(x).clone()
    model.train()
    xg = x.clone().requires_grad_(True)
    out_train = run_reference(variant, model, xg, ei)
    (out_train * lw).sum().backward()
    grads = {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}
    sd1 = {k: v.clone() for k, v in model.state_dict().items() if "running" in k or "tracked" in k}
    print(name, "out_eval", tuple(out_eval.shape), float(out_eval.abs().mean()), "attentions", tuple(att.shape))
    return dict(cfg=cfg, state_dict=sd0, x=x, edge_index=ei, loss_weight=lw, out_eval=out_eval,
                out_train=out_train.detach().clone(), grad_x=xg.grad.clone(), grads=grads, buffers_after_train=sd1,
                attentions=att)


def attention_cases():
    """full_attention_conv(qs, ks, vs) with vs [N, 1, D] (what TransConvLayer passes when use_weight=False)."""
    ours, _ = import_reference("medium")
    out = {}
    for n, heads, m, d in [(40, 2, 8, 8), (65, 3, 16, 16), (33, 4, 8, 24)]:
        g = torch.Generator().manual_seed(n * 10 + heads)
        q = torch.randn(n, heads, m, generator=g, requires_grad=True)
        k = torch.randn(n, heads, m, generator=g, requires_grad=True)
        v = torch.randn(n, 1, d, generator=g, requires_grad=True)
        w = torch.randn(n, heads, d, generator=g)
        o = ours.full_attention_conv(q, k, v)
        (o * w).sum().backward()
        out[f"n{n}_h{heads}_m{m}_d{d}"] = dict(q=q.detach(), k=k.detach(), v=v.detach(), w=w, out=o.detach(), dq=q.grad, dk=k.grad,
                                               dv=v.grad)
    return out


if __name__ == "__main__":
    fx = dict(models={nm: model_case(nm, sp) for nm, sp in CASES.items()}, attention=attention_cases())
    torch.save(fx, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")
