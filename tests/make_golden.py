"""Generate tests/golden/*.pt from the UNMODIFIED reference (run in the build container only):

    python tests/make_golden.py

Each fixture holds seeded inputs, the state_dict, and the reference's outputs / gradients.
The committed fixtures are what pins oracle/ (tests/test_oracle_golden.py) and what the `-m gpu`
parity tests compare the CUDA path with, without a reference checkout."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from oracle import sgformer_oracle as O  # noqa: E402
from _refload import build_reference_model, import_reference, run_reference  # noqa: E402

GOLD = os.path.join(HERE, "golden")


def synth_graph(n, e, seed, directed=False, isolated=0, dup=0):
    g = torch.Generator().manual_seed(seed)
    hi = n - isolated
    src = torch.randint(0, hi, (e,), generator=g)
    dst = torch.randint(0, hi, (e,), generator=g)
    ei = torch.stack([src, dst])
    if not directed:
        ei = torch.cat([ei, ei.flip(0)], 1)
        key = torch.unique(ei[0] * n + ei[1])
        ei = torch.stack([key // n, key % n])
        ei = ei[:, ei[0] != ei[1]]
        loops = torch.arange(hi)
        ei = torch.cat([ei, torch.stack([loops, loops])], 1)
    if dup:
        ei = torch.cat([ei, ei[:, :dup]], 1)
    perm = torch.randperm(ei.shape[1], generator=g)
    return ei[:, perm].contiguous()


CASES = {
    "large_add_init": dict(variant="large", n=257, d=24, h=32, c=7, e=900, graph={},
                           kw=dict(gnn_num_layers=2, gnn_use_init=True, graph_weight=0.5, gnn_dropout=0.0,
                                   trans_dropout=0.0)),
    "large_cat_heads2": dict(variant="large", n=130, d=10, h=16, c=5, e=400,
                             graph=dict(directed=True, isolated=3, dup=17),
                             kw=dict(trans_num_layers=2, trans_num_heads=2, gnn_num_layers=3, aggregate="cat",
                                     gnn_dropout=0.0, trans_dropout=0.0)),
    "large_noweight": dict(variant="large", n=64, d=12, h=16, c=3, e=200, graph={},
                           kw=dict(trans_use_weight=False, gnn_use_weight=False, gnn_use_bn=False,
                                   trans_use_bn=False, trans_use_act=False, gnn_num_layers=2, gnn_dropout=0.0,
                                   trans_dropout=0.0, graph_weight=0.3)),
    "large_nores": dict(variant="large", n=100, d=20, h=32, c=4, e=300, graph={},
                        kw=dict(trans_use_residual=False, gnn_use_residual=False, gnn_use_act=False,
                                gnn_num_layers=2, gnn_dropout=0.0, trans_dropout=0.0)),
    "100M_alpha": dict(variant="100M", n=200, d=16, h=32, c=6, e=700, graph={},
                       kw=dict(alpha=0.3, gnn_num_layers=3, gnn_use_init=True, graph_weight=0.8,
                               gnn_dropout=0.0, trans_dropout=0.0)),
    "medium_gcn": dict(variant="medium", n=150, d=40, h=16, c=7, e=400, graph={},
                       kw=dict(num_layers=1, alpha=0.5, dropout=0.0, use_residual=False, gcn_num_layers=4,
                               gcn_dropout=0.0, graph_weight=0.8)),
    "medium_res_heads2": dict(variant="medium", n=90, d=12, h=16, c=4, e=250, graph=dict(directed=True),
                              kw=dict(num_layers=2, num_heads=2, alpha=0.7, dropout=0.0, use_residual=True,
                                      gcn_num_layers=2, gcn_dropout=0.0, graph_weight=0.6)),
}


def perturb_(model, seed):
    """Make affine/BN buffers non-trivial so parity exercises them."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, t in list(model.named_parameters()) + list(model.named_buffers()):
            if ".bns." in name:
                if name.endswith("num_batches_tracked"):
                    continue
                if name.endswith("running_var") or name.endswith("weight"):
                    t.copy_(1.0 + 0.2 * torch.rand(t.shape, generator=g))
                else:
                    t.copy_(0.1 * torch.randn(t.shape, generator=g))
            elif name.endswith(".bias") and "gnn.convs" in name:
                t.copy_(0.1 * torch.randn(t.shape, generator=g))


def model_case(name, spec):
    torch.manual_seed(1234)
    cfg = O.make_config(spec["variant"], spec["d"], spec["h"], spec["c"], **spec["kw"])
    model, _ = build_reference_model(spec["variant"], cfg)
    model.reset_parameters()
    perturb_(model, 7)
    g = torch.Generator().manual_seed(99)
    x = torch.randn(spec["n"], spec["d"], generator=g)
    ei = synth_graph(spec["n"], spec["e"], 5, **spec["graph"])
    lw = torch.randn(spec["n"], spec["c"], generator=g)
    sd0 = {k: v.clone() for k, v in model.state_dict().items()}

    model.eval()
    with torch.no_grad():
        out_eval = run_reference(spec["variant"], model, x, ei).clone()

    model.train()
    xg = x.clone().requires_grad_(True)
    out_train = run_reference(spec["variant"], model, xg, ei)
    (out_train * lw).sum().backward()
    grads = {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}
    sd1 = {k: v.clone() for k, v in model.state_dict().items() if "running" in k or "tracked" in k}
    torch.save(dict(name=name, cfg=cfg, state_dict=sd0, x=x, edge_index=ei, loss_weight=lw,
                    out_eval=out_eval, out_train=out_train.detach().clone(), grad_x=xg.grad.clone(),
                    grads=grads, buffers_after_train=sd1), os.path.join(GOLD, f"model_{name}.pt"))
    print(name, "out_eval", tuple(out_eval.shape), float(out_eval.abs().mean()))


def attention_cases():
    ours, _ = import_reference("medium")
    out = {}
    for n, h, m in [(16, 1, 8), (64, 2, 16), (257, 1, 32), (33, 4, 8)]:
        g = torch.Generator().manual_seed(n * 100 + h)
        q = torch.randn(n, h, m, generator=g, dtype=torch.float64, requires_grad=True)
        k = torch.randn(n, h, m, generator=g, dtype=torch.float64, requires_grad=True)
        v = torch.randn(n, h, m, generator=g, dtype=torch.float64, requires_grad=True)
        w = torch.randn(n, h, m, generator=g, dtype=torch.float64)
        # the reference creates `all_ones` in fp32 (medium/ours.py:26); run it in fp32 as shipped,
        # the fp64 tensors above are only the seeded source of the inputs.
        q32, k32, v32 = (t.detach().float().requires_grad_(True) for t in (q, k, v))
        o = ours.full_attention_conv(q32, k32, v32)
        (o * w.float()).sum().backward()
        out[f"n{n}_h{h}_m{m}"] = dict(q=q32.detach(), k=k32.detach(), v=v32.detach(), w=w.float(), out=o.detach(),
                                      dq=q32.grad, dk=k32.grad, dv=v32.grad)
    torch.save(out, os.path.join(GOLD, "attention.pt"))
    print("attention", list(out))


def graphconv_layer_cases():
    ours, _ = import_reference("large")
    out = {}
    for name, n, h, e, gk, use_init, use_weight in [
        ("sym", 120, 16, 400, {}, True, True),
        ("directed_dup_iso", 77, 8, 300, dict(directed=True, isolated=5, dup=23), False, True),
        ("noweight", 50, 8, 150, dict(directed=True), False, False),
    ]:
        torch.manual_seed(3)
        layer = ours.GraphConvLayer(h, h, use_weight=use_weight, use_init=use_init)
        g = torch.Generator().manual_seed(11)
        x = torch.randn(n, h, generator=g, requires_grad=True)
        x0 = torch.randn(n, h, generator=g, requires_grad=True)
        w = torch.randn(n, h, generator=g)
        ei = synth_graph(n, e, 21, **gk)
        y = layer(x, ei, x0)
        (y * w).sum().backward()
        out[name] = dict(x=x.detach(), x0=x0.detach(), w=w, edge_index=ei, use_init=use_init,
                         use_weight=use_weight, W=layer.W.weight.detach().clone(), b=layer.W.bias.detach().clone(),
                         y=y.detach(), dx=x.grad.clone(), dx0=None if x0.grad is None else x0.grad.clone(),
                         dW=None if layer.W.weight.grad is None else layer.W.weight.grad.clone(),
                         db=None if layer.W.bias.grad is None else layer.W.bias.grad.clone())
    torch.save(out, os.path.join(GOLD, "graphconv_layer.pt"))
    print("graphconv_layer", list(out))


def import_reference_driver_modules():
    """`data_utils` (eval_acc) and `eval` (evaluate) of the reference's large/ directory, through the shims, unmodified."""
    import importlib
    from _refload import REF_ROOT, SHIMS
    for name in ("data_utils", "eval", "dataset", "logger", "parse", "ours", "gnns"):
        sys.modules.pop(name, None)
    saved = list(sys.path)
    sys.path[:0] = [SHIMS, os.path.join(REF_ROOT, "large")]
    try:
        du = importlib.import_module("data_utils")
        ev = importlib.import_module("eval")
    finally:
        sys.path[:] = saved
    return du, ev


def evaluate_cases():
    """The reference's own evaluate() / eval_acc (large/eval.py:6-33, large/data_utils.py:210-220) on fixed logits: pins K11
    (sgf_eval_acc) and sgformer_b200.eval.evaluate."""
    from types import SimpleNamespace
    du, ev = import_reference_driver_modules()
    out = {}
    for name, (n, c, seed, ties) in {"c7": (500, 7, 0, 0), "c47_ties": (1500, 47, 1, 200), "c2": (257, 2, 2, 40)}.items():
        g = torch.Generator().manual_seed(seed)
        logits = torch.randn(n, c, generator=g)
        if ties:
            rows = torch.randperm(n, generator=g)[:ties]
            logits[rows, (rows % c)] = logits[rows].max(dim=1).values      # exact ties with the row maximum
        label = torch.randint(0, c, (n, 1), generator=g)
        perm = torch.randperm(n, generator=g)
        split = {"train": perm[: n // 2], "valid": perm[n // 2: 3 * n // 4], "test": perm[3 * n // 4:]}

        class Fixed(torch.nn.Module):
            def forward(self, x, ei):
                return logits.clone()

        ds = SimpleNamespace(graph={"node_feat": torch.zeros(n, 1), "edge_index": torch.zeros(2, 0, dtype=torch.long)}, label=label)
        tr, va, te, vloss, lsm = ev.evaluate(Fixed(), ds, split, du.eval_acc, torch.nn.NLLLoss(), SimpleNamespace(dataset="synthetic"))
        out[name] = dict(logits=logits, label=label, split=split, train_acc=tr, valid_acc=va, test_acc=te, valid_loss=float(vloss),
                         log_softmax=lsm)
    torch.save(out, os.path.join(GOLD, "evaluate.pt"))
    print("evaluate", {k: (v["train_acc"], v["valid_acc"], v["test_acc"], v["valid_loss"]) for k, v in out.items()})


def graph_prep_cases():
    """to_undirected / remove_self_loops / add_self_loops of the torch_geometric restatement the reference drivers run through
    here (tests/ref_shims; the real package is not installable - SURVEY.md 8c): fixtures for K10."""
    from _refload import SHIMS
    saved = list(sys.path)
    sys.path.insert(0, SHIMS)
    try:
        from torch_geometric.utils import add_self_loops, remove_self_loops, to_undirected
    finally:
        sys.path[:] = saved
    out = {}
    for name, (n, e, seed, loops, dup) in {"small": (9, 30, 0, 4, 5), "mid": (400, 3000, 1, 60, 200), "isolated": (50, 40, 2, 0, 0),
                                           "hub": (3000, 9000, 3, 10, 0)}.items():
        g = torch.Generator().manual_seed(seed)
        hi = n if name != "isolated" else n // 2
        ei = torch.stack([torch.randint(0, hi, (e,), generator=g), torch.randint(0, hi, (e,), generator=g)])
        if name == "hub":
            ei[1, :5000] = 7
        ei[1, :loops] = ei[0, :loops]
        if dup:
            ei = torch.cat([ei, ei[:, :dup]], 1)
        und = to_undirected(ei, num_nodes=n)
        nsl, _ = remove_self_loops(und)
        full, _ = add_self_loops(nsl, num_nodes=n)
        out[name] = dict(n=n, edge_index=ei, to_undirected=und, remove_self_loops_raw=remove_self_loops(ei)[0],
                         add_self_loops_raw=add_self_loops(ei, num_nodes=n)[0], prepared=full)
    out = {k: {kk: v.to(torch.int32) if torch.is_tensor(v) else v for kk, v in c.items()} for k, c in out.items()}   # < 1 MB
    torch.save(out, os.path.join(GOLD, "graph_prep.pt"))
    print("graph_prep", {k: tuple(v["prepared"].shape) for k, v in out.items()})


def get_attentions_cases():
    """TransConv.get_attentions of the unmodified reference (large/ours.py:221-238 and the medium / 100M variants): the [layers, N, N]
    visualisation matrices, for the model fixtures whose graphs are small enough (N <= 257)."""
    out = {}
    for name in ("large_add_init", "large_cat_heads2", "large_noweight", "100M_alpha", "medium_res_heads2"):
        fx = torch.load(os.path.join(GOLD, f"model_{name}.pt"), weights_only=False)
        model, _ = build_reference_model(fx["cfg"]["variant"], fx["cfg"])
        model.load_state_dict(fx["state_dict"])
        model.eval()
        with torch.no_grad():
            att = model.get_attentions(fx["x"])
        out[name] = att.clone()
        print("get_attentions", name, tuple(att.shape), float(att.abs().max()))
    torch.save(out, os.path.join(GOLD, "get_attentions.pt"))


def property_graph(n, e, seed, directed, isolated, dup, loops):
    g = torch.Generator().manual_seed(seed)
    hi = max(n - isolated, 1)
    ei = torch.stack([torch.randint(0, hi, (e,), generator=g), torch.randint(0, hi, (e,), generator=g)])
    if not directed:
        ei = torch.cat([ei, ei.flip(0)], 1)
    if dup:
        ei = torch.cat([ei, ei[:, :dup]], 1)
    if loops:
        ar = torch.arange(hi)
        ei = torch.cat([ei, torch.stack([ar, ar])], 1)
    return ei


def oracle_property_cases(count=25):
    """Randomly drawn configurations and graphs (isolated nodes, directed/asymmetric edges, duplicates, self loops, odd sizes,
    1-4 heads; fixed seed) with the outputs of the reference, eval and train mode: pins oracle/ (tests/test_oracle_vs_reference.py)."""
    import random
    rnd = random.Random(0)
    out = []
    for _ in range(count):
        variant, n, h = rnd.choice(["large", "100M", "medium"]), rnd.randint(5, 90), rnd.choice([8, 16, 24])
        heads, seed, directed = rnd.choice([1, 2, 4]), rnd.randint(0, 10 ** 6), rnd.random() < 0.5
        isolated, dup, loops = rnd.randint(0, 3), rnd.randint(0, 9), rnd.random() < 0.5
        flags = [rnd.random() < 0.5 for _ in range(9)]
        aggregate, layers, tlayers = rnd.choice(["add", "cat"]), rnd.randint(1, 3), rnd.randint(1, 2)
        d, c = 7, 4
        use_weight = flags[0] or heads > 1        # use_weight=False forces one head (medium/ours.py:84)
        if variant == "medium":
            cfg = O.make_config("medium", d, h, c, num_layers=tlayers, num_heads=heads, alpha=0.3, dropout=0.0, use_bn=flags[1],
                                use_residual=flags[2], use_weight=use_weight, gcn_num_layers=layers + 1, gcn_dropout=0.0,
                                gcn_use_bn=flags[3], graph_weight=0.7, aggregate=aggregate)
        else:
            kw = dict(trans_num_layers=tlayers, trans_num_heads=heads, trans_dropout=0.0, trans_use_bn=flags[1],
                      trans_use_residual=flags[2], trans_use_weight=use_weight, trans_use_act=flags[4], gnn_num_layers=layers,
                      gnn_dropout=0.0, gnn_use_weight=flags[5], gnn_use_init=flags[6], gnn_use_bn=flags[3], gnn_use_residual=flags[7],
                      gnn_use_act=flags[8], graph_weight=0.7, aggregate=aggregate)
            if variant == "100M":
                kw["alpha"] = 0.3
            cfg = O.make_config(variant, d, h, c, **kw)
        torch.manual_seed(seed)
        model, _ = build_reference_model(variant, cfg)
        sd = {k: v.clone() for k, v in model.state_dict().items()}
        ei = property_graph(n, 3 * n, seed, directed, isolated, dup, loops)
        x = torch.randn(n, d, generator=torch.Generator().manual_seed(seed + 1))
        ref = {}
        for training in (False, True):
            model.train(training)
            with torch.no_grad():
                ref[training] = run_reference(variant, model, x, ei).clone()
            model.load_state_dict(sd)   # undo BatchNorm running-stat updates
        out.append(dict(cfg=cfg, state_dict=sd, edge_index=ei, x=x, ref_eval=ref[False], ref_train=ref[True]))
    torch.save(out, os.path.join(GOLD, "oracle_property.pt"))
    print("oracle_property", len(out))


def parse_large_case():
    """The SGFormer constructor call that the reference's own large/parse.py makes for the amazon2m recipe of large/run.sh:15-19
    (positional and keyword arguments as data): tests/test_dropin_plumbing.py replays it against the drop-in."""
    import argparse
    import importlib
    import json
    from _refload import REF_ROOT, SHIMS
    for name in ("parse", "ours", "gnns"):
        sys.modules.pop(name, None)
    saved = list(sys.path)
    sys.path[:0] = [SHIMS, os.path.join(REF_ROOT, "large")]
    try:
        parse = importlib.import_module("parse")
    finally:
        sys.path[:] = saved
    calls = []

    class Record:
        def __init__(self, *a, **kw):
            calls.append(dict(args=list(a), kwargs=kw))

        def to(self, device):
            return self

    parse.SGFormer = Record
    argv = ("--method sgformer --hidden_channels 256 --gnn_num_layers 3 --gnn_dropout 0. --gnn_use_residual --gnn_use_weight "
            "--gnn_use_bn --gnn_use_init --gnn_use_act --trans_num_layers 1 --trans_dropout 0. --trans_use_residual "
            "--trans_use_weight --trans_use_bn --use_graph --graph_weight 0.5")
    p = argparse.ArgumentParser()
    parse.parser_add_main_args(p)
    parse.parse_method(p.parse_args(argv.split()), 47, 100, "cpu")
    assert len(calls) == 1
    with open(os.path.join(GOLD, "parse_large_sgformer.json"), "w") as f:
        json.dump(dict(argv=argv, **calls[0]), f, indent=1, sort_keys=True)
        f.write("\n")
    print("parse_large", calls[0])


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] in ("get_attentions", "oracle_property", "parse_large"):   # add one fixture, keep the others
        {"get_attentions": get_attentions_cases, "oracle_property": oracle_property_cases, "parse_large": parse_large_case}[sys.argv[1]]()
        sys.exit(0)
    os.makedirs(GOLD, exist_ok=True)
    for nm, sp in CASES.items():
        model_case(nm, sp)
    attention_cases()
    graphconv_layer_cases()
    evaluate_cases()
    graph_prep_cases()
    get_attentions_cases()
    oracle_property_cases()
    parse_large_case()
