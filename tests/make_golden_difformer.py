"""Generate tests/golden/difformer.pt from the UNMODIFIED reference's medium/difformer.py (run in the build container only):

    SGFORMER_REFERENCE=/path/to/SGFormer python tests/make_golden_difformer.py

Writes only that file; the other fixtures are tests/make_golden.py's."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from make_golden import GOLD, synth_graph  # noqa: E402

DIFFORMER_CASES = {        # sizes keep the file under 1 MB: the 8-layer h=64 case alone holds 2 x 100 k parameters
    "default": dict(n=32, d=8, h=8, c=5, graph={}, kw={}),
    "actor_recipe": dict(n=32, d=8, h=64, c=5, graph={}, kw=dict(num_layers=8)),
    "no_graph": dict(n=32, d=8, h=8, c=4, graph={}, kw=dict(use_graph=False, num_layers=3)),
    "graph_weight": dict(n=32, d=8, h=8, c=3, graph={}, kw=dict(graph_weight=0.3)),
    "no_weight": dict(n=32, d=8, h=8, c=3, graph={}, kw=dict(use_weight=False)),
    "no_res_no_bn": dict(n=32, d=8, h=8, c=3, graph={}, kw=dict(use_residual=False, use_bn=False)),
    "source": dict(n=32, d=8, h=8, c=3, graph={}, kw=dict(use_source=True, num_layers=3)),
    "directed": dict(n=40, d=8, h=8, c=4, graph=dict(directed=True, isolated=5, dup=11), kw={}),
}


def _flat_dict(d):
    """{name: tensor} as one flat fp32 tensor + names and shapes (one storage instead of one per tensor keeps the file small);
    tests/test_difformer.load_fixture inverts it."""
    return dict(names=list(d), shapes=[list(t.shape) for t in d.values()], flat=torch.cat([t.reshape(-1).float() for t in d.values()]))


def difformer_cases():
    """The reference's medium/difformer.py DIFFormer (kernel 'simple', one head, dropout 0) on the cases above: inputs,
    state_dict, eval / train logits, parameter gradients and grad_x of sum(out * loss_weight), and get_attentions where the
    reference can compute it (use_graph=False).  Pins oracle/difformer_oracle.py and the kernel path (tests/test_difformer.py,
    tests/test_gpu_difformer.py)."""
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
    out = {}
    for i, (name, sp) in enumerate(DIFFORMER_CASES.items()):
        torch.manual_seed(100 + i)
        kw = dict(dict(num_layers=2, dropout=0.0), **sp["kw"])
        model = ref.DIFFormer(sp["d"], sp["h"], sp["c"], **kw)
        with torch.no_grad():                      # move the LayerNorm affine parameters off 1 / 0
            for nm, p_ in model.named_parameters():
                if nm.startswith("bns."):
                    p_.add_(0.1 * torch.randn_like(p_))
        sd = {k: v.clone() for k, v in model.state_dict().items()}
        g = torch.Generator().manual_seed(200 + i)
        x = torch.randn(sp["n"], sp["d"], generator=g)
        ei = synth_graph(sp["n"], 3 * sp["n"], 300 + i, **sp["graph"]) if sp["graph"] else synth_graph(sp["n"], 3 * sp["n"], 300 + i)
        lw = torch.randn(sp["n"], sp["c"], generator=g)
        model.eval()
        with torch.no_grad():
            out_eval = model(FakeDataset(x, ei)).clone()
        model.train()
        xg = x.clone().requires_grad_(True)
        out_train = model(FakeDataset(xg, ei))
        (out_train * lw).sum().backward()
        grads = {k: p_.grad.clone() for k, p_ in model.named_parameters() if p_.grad is not None}
        case = dict(kw=kw, in_channels=sp["d"], hidden=sp["h"], out_channels=sp["c"], x=x, edge_index=ei.to(torch.int32),
                    state_dict=_flat_dict(sd), loss_weight=lw, out_eval=out_eval, out_train=out_train.detach().clone(),
                    grad_x=xg.grad.clone(), grads=_flat_dict(grads))
        if not kw.get("use_graph", True):
            model.eval()
            with torch.no_grad():
                case["attentions"] = model.get_attentions(x).clone()
        out[name] = case
    path = os.path.join(GOLD, "difformer.pt")
    torch.save(out, path)
    print("difformer", len(out), os.path.getsize(path), "bytes")


if __name__ == "__main__":
    difformer_cases()
