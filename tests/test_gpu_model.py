"""Module-level parity on the H100: the drop-in nn.Modules against the golden fixtures generated from the unmodified
reference (tests/make_golden.py) and against the CPU oracle on fresh seeded graphs.
fp32 precision: 1e-4; bf16 precision: 1e-2 (BASELINE.json north_star)."""
import glob
import os

import pytest
import torch

from oracle import sgformer_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MODEL_FILES = sorted(glob.glob(os.path.join(GOLD, "model_*.pt")))


def _close(a, b, rtol, atol, what):
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    assert a.shape == b.shape, f"{what}: shape {tuple(a.shape)} vs {tuple(b.shape)}"
    err = (a - b).abs().max().item()
    ref = b.abs().max().item()
    assert err == err and err <= atol + rtol * ref, f"{what}: max err {err:.3e} (ref max {ref:.3e})"


def _close_fro(a, b, tol, floor, what):
    """Relative Frobenius error; `floor` guards tensors whose true value is ~0 (e.g. biases feeding a BatchNorm)."""
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    assert a.shape == b.shape, f"{what}: shape {tuple(a.shape)} vs {tuple(b.shape)}"
    err = (a - b).norm().item() / max(b.norm().item(), floor)
    assert err == err and err <= tol, f"{what}: relative Frobenius error {err:.3e} > {tol}"


def _check_grads(named_got, ref_grads, precision, problems):
    """fp32: max-norm 2e-3.  bf16: the north-star's 1e-2 is an output tolerance; gradients of these tiny, ReLU/BatchNorm
    heavy fixtures carry ~10% inherent bf16 noise (measured with the CPU emulation of the same schedule), so they are
    bounded in relative Frobenius norm."""
    gmax = max(g.norm().item() for g in ref_grads.values())
    for k, g in ref_grads.items():
        try:
            assert named_got[k] is not None, f"missing grad {k}"
            if precision == "fp32":
                scale = max(g.abs().max().item(), 1e-3)
                _close(named_got[k], g, 2e-3, 2e-3 * scale * 0.05 + 3e-5, f"grad {k}")
            else:
                _close_fro(named_got[k], g, 0.25, 2e-2 * gmax, f"grad {k}")
        except AssertionError as e:
            problems.append(str(e))


class Data:
    def __init__(self, x, ei):
        self.graph = {"node_feat": x, "edge_index": ei, "num_nodes": x.shape[0]}


def build_model(cfg):
    """Instantiate our drop-in module for an oracle config (same constructor calls as the reference's parse.py)."""
    v = cfg["variant"]
    if v == "medium":
        from sgformer_b200 import medium as M
        gnn = M.GCN(cfg["in_channels"], cfg["hidden"], cfg["hidden"], num_layers=cfg["gcn_num_layers"],
                    dropout=cfg["gcn_dropout"], use_bn=cfg["gcn_use_bn"])
        return M.SGFormer(cfg["in_channels"], cfg["hidden"], cfg["out_channels"], num_layers=cfg["trans_num_layers"],
                          num_heads=cfg["num_heads"], alpha=cfg["alpha"], dropout=cfg["trans_dropout"],
                          use_bn=cfg["trans_use_bn"], use_residual=cfg["trans_use_residual"],
                          use_weight=cfg["trans_use_weight"], use_graph=cfg["use_graph"], graph_weight=cfg["graph_weight"],
                          gnn=gnn, aggregate=cfg["aggregate"])
    kw = dict(trans_num_layers=cfg["trans_num_layers"], trans_num_heads=cfg["num_heads"], trans_dropout=cfg["trans_dropout"],
              trans_use_bn=cfg["trans_use_bn"], trans_use_residual=cfg["trans_use_residual"],
              trans_use_weight=cfg["trans_use_weight"], trans_use_act=cfg["trans_use_act"],
              gnn_num_layers=cfg["gnn_num_layers"], gnn_dropout=cfg["gnn_dropout"], gnn_use_weight=cfg["gnn_use_weight"],
              gnn_use_init=cfg["gnn_use_init"], gnn_use_bn=cfg["gnn_use_bn"], gnn_use_residual=cfg["gnn_use_residual"],
              gnn_use_act=cfg["gnn_use_act"], use_graph=cfg["use_graph"], graph_weight=cfg["graph_weight"],
              aggregate=cfg["aggregate"])
    if v == "100M":
        from sgformer_b200 import hundred_m as H
        return H.SGFormer(cfg["in_channels"], cfg["hidden"], cfg["out_channels"], alpha=cfg["alpha"], **kw)
    from sgformer_b200 import large as L
    return L.SGFormer(cfg["in_channels"], cfg["hidden"], cfg["out_channels"], **kw)


def run(model, cfg, x, ei):
    return model(Data(x, ei)) if cfg["variant"] == "medium" else model(x, ei)


@pytest.mark.parametrize("path", MODEL_FILES, ids=[os.path.basename(p)[6:-3] for p in MODEL_FILES])
def test_state_dict_keys_match_reference(path):
    fx = torch.load(path, weights_only=False)
    model = build_model(fx["cfg"])
    assert list(model.state_dict().keys()) == list(fx["state_dict"].keys())
    for k, v in model.state_dict().items():
        assert tuple(v.shape) == tuple(fx["state_dict"][k].shape), k


@pytest.mark.parametrize("precision,rtol", [("fp32", 1e-4), ("bf16", 1e-2)])
@pytest.mark.parametrize("path", MODEL_FILES, ids=[os.path.basename(p)[6:-3] for p in MODEL_FILES])
def test_model_matches_reference_golden(path, precision, rtol):
    fx = torch.load(path, weights_only=False)
    cfg = fx["cfg"]
    model = build_model(cfg).to(DEV).set_precision(precision)
    model.load_state_dict(fx["state_dict"])
    x, ei = fx["x"].to(DEV), fx["edge_index"].to(DEV)
    model.eval()
    with torch.no_grad():
        out = run(model, cfg, x, ei)
    assert out.dtype == torch.float32 and out.shape == fx["out_eval"].shape
    _close(out, fx["out_eval"], rtol, rtol, "eval output")

    model.train()
    xg = x.clone().requires_grad_(True)
    out = run(model, cfg, xg, ei)
    _close(out, fx["out_train"], rtol, rtol, "train output")
    (out * fx["loss_weight"].to(DEV)).sum().backward()
    problems = []
    grads = {k: p.grad for k, p in model.named_parameters()}
    grads["__x__"] = xg.grad
    ref = dict(fx["grads"])
    ref["__x__"] = fx["grad_x"]
    _check_grads(grads, ref, precision, problems)
    assert not problems, "\n".join(problems)
    if precision == "fp32":
        sd = model.state_dict()
        for k, v in fx["buffers_after_train"].items():
            _close(sd[k].float(), v.float(), 1e-4, 1e-5, f"buffer {k}")


@pytest.mark.parametrize("precision,tol", [("fp32", 1e-4), ("bf16", 1e-2)])
def test_full_attention_conv_golden(precision, tol):
    from sgformer_b200.medium import full_attention_conv
    fx = torch.load(os.path.join(GOLD, "attention.pt"), weights_only=False)
    for name, c in fx.items():
        q, k, v = (c[t].to(DEV).requires_grad_(True) for t in "qkv")
        o = full_attention_conv(q, k, v, precision=precision)
        _close(o, c["out"], tol, tol, f"{name} out")
        (o * c["w"].to(DEV)).sum().backward()
        gt = 2e-3 if precision == "fp32" else 8e-2
        for t, g in (("dq", q.grad), ("dk", k.grad), ("dv", v.grad)):
            _close(g, c[t], gt, gt * c[t].abs().max().item() * 0.05 + 1e-7, f"{name} {t}")
    o, att = full_attention_conv(q, k, v, output_attn=True, precision=precision)
    assert att.shape == (q.shape[0], q.shape[0])


@pytest.mark.parametrize("precision,tol", [("fp32", 2e-4), ("bf16", 3e-2)])
def test_get_attentions_golden(precision, tol):
    """SGFormer.get_attentions on the kernels (engine.trans_attentions) == the reference's [layers, N, N] matrices
    (large/ours.py:221-238, medium/ours.py:162-177, 100M/ours.py:274-289), CUDA and CPU inputs."""
    fx = torch.load(os.path.join(GOLD, "get_attentions.pt"), weights_only=False)
    for name, ref in fx.items():
        m = torch.load(os.path.join(GOLD, f"model_{name}.pt"), weights_only=False)
        model = build_model(m["cfg"]).to(DEV).set_precision(precision)
        model.load_state_dict(m["state_dict"])
        model.eval()
        att = model.get_attentions(m["x"].to(DEV))
        assert att.shape == ref.shape and att.is_cuda
        _close(att, ref, tol, 0, f"{name} get_attentions")
    att_cpu = model.get_attentions(m["x"])          # host tensors: computed on the device, returned on the host
    assert not att_cpu.is_cuda
    _close(att_cpu, ref, tol, 0, "get_attentions (cpu input)")


def test_graphconv_layer_golden():
    from sgformer_b200.large import GraphConvLayer
    fx = torch.load(os.path.join(GOLD, "graphconv_layer.pt"), weights_only=False)
    for name, c in fx.items():
        h = c["x"].shape[1]
        layer = GraphConvLayer(h, h, use_weight=c["use_weight"], use_init=c["use_init"]).to(DEV)
        with torch.no_grad():
            layer.W.weight.copy_(c["W"])
            layer.W.bias.copy_(c["b"])
        x, x0 = c["x"].to(DEV).requires_grad_(True), c["x0"].to(DEV).requires_grad_(True)
        y = layer(x, c["edge_index"].to(DEV), x0)
        _close(y, c["y"], 1e-4, 1e-5, f"{name} y")
        (y * c["w"].to(DEV)).sum().backward()
        _close(x.grad, c["dx"], 1e-3, 1e-5, f"{name} dx")
        if c["dx0"] is not None:
            _close(x0.grad, c["dx0"], 1e-3, 1e-5, f"{name} dx0")
        if c["dW"] is not None:
            _close(layer.W.weight.grad, c["dW"], 1e-3, 1e-4, f"{name} dW")


MIDSIZE = [
    (12000, 90000, 128, 256, 40, dict(gnn_num_layers=3, graph_weight=0.5)),                       # arxiv recipe, large/run.sh:2-5
    (16000, 200000, 100, 256, 47, dict(gnn_num_layers=3, gnn_use_init=True, graph_weight=0.5)),    # amazon2m recipe, :15-19
    (14000, 160000, 65, 64, 2, dict(gnn_num_layers=2, gnn_use_init=True, graph_weight=0.5)),       # pokec recipe, :22-26
]
_midsize_cache = {}


def _midsize_oracle(i):
    """Oracle results of case i (computed once, shared by both precisions; the CPU oracle is the slow part)."""
    if i in _midsize_cache:
        return _midsize_cache[i]
    from sgformer_b200.synth import make_graph
    n, e, d, h, c, kw = MIDSIZE[i]
    cfg = O.make_config("large", d, h, c, gnn_dropout=0.0, trans_dropout=0.0, trans_use_act=False, **kw)
    sd = O.init_state_dict(cfg, seed=3)
    ei = make_graph(n, e, seed=1)
    g = torch.Generator().manual_seed(2)
    x = torch.randn(n, d, generator=g)
    y = torch.randint(0, c, (n,), generator=g)
    ref_eval = O.sgformer_forward(cfg, sd, x, ei, training=False)

    def grads(dtype):
        sdg = {k: (v.to(dtype).clone().requires_grad_(True) if v.is_floating_point() and "running" not in k else
                   (v.to(dtype) if v.is_floating_point() else v.clone())) for k, v in sd.items()}
        out = O.sgformer_forward(cfg, sdg, x.to(dtype), ei, training=True)
        loss = torch.nn.functional.cross_entropy(out, y)
        loss.backward()
        return out.detach(), loss.detach(), {k: v.grad for k, v in sdg.items() if v.is_floating_point() and v.grad is not None}

    ref_t, loss_ref, g32 = grads(torch.float32)
    _, _, g64 = grads(torch.float64)
    _midsize_cache[i] = dict(cfg=cfg, sd=sd, ei=ei, x=x, y=y, ref_eval=ref_eval, ref_t=ref_t, loss_ref=loss_ref, g32=g32, g64=g64)
    return _midsize_cache[i]


@pytest.mark.parametrize("precision,tol", [("fp32", 1e-4), ("bf16", 1e-2)])
@pytest.mark.parametrize("case", range(len(MIDSIZE)))
def test_model_matches_oracle_midsize(case, precision, tol):
    """Fresh seeded graph, reference hyper-parameters, sizes the CPU oracle finishes in seconds.
    Train-mode gradients: the weight gradients behind a BatchNorm are ill-conditioned (the fp32 torch reference itself is only
    good to ~2e-3 of their scale here), so they are judged against an fp64 run of the oracle.  The "fp32" precision evaluates
    every GEMM as bf16x3 partial products with tensor-core fp32 accumulation (effective epsilon ~2^-20, about 10x IEEE fp32), which
    the same cancellation amplifies: the CUDA path must be within max(3e-2 of the tensor's scale, 8x the fp32 oracle's own
    deviation, 1e-3 of the largest gradient entry of the model); in bf16 mode gradients are bounded in Frobenius norm."""
    from sgformer_b200 import large as L
    n, e, d, h, c, kw = MIDSIZE[case]
    r = _midsize_oracle(case)
    x, ei, y, g32, g64 = r["x"], r["ei"], r["y"], r["g32"], r["g64"]
    model = L.SGFormer(d, h, c, trans_dropout=0.0, gnn_dropout=0.0, trans_use_act=False, **kw).to(DEV).set_precision(precision)
    model.load_state_dict(r["sd"])
    model.eval()
    with torch.no_grad():
        out = model(x.to(DEV), ei.to(DEV))
    _close(out, r["ref_eval"], tol, tol, "eval logits")
    model.train()
    out_t = model(x.to(DEV), ei.to(DEV))
    loss = torch.nn.functional.cross_entropy(out_t, y.to(DEV))
    loss.backward()
    _close(out_t, r["ref_t"], tol, tol, "train logits")
    _close(loss, r["loss_ref"], tol, tol, "loss")
    problems = []
    gmax = max(v.norm().item() for v in g64.values())
    gabs = max(v.abs().max().item() for v in g64.values())
    for k, p in model.named_parameters():
        gref = g64[k]
        scale = gref.abs().max().item()
        try:
            if precision == "fp32":
                own = (g32[k].double() - gref).abs().max().item()
                err = (p.grad.detach().cpu().double() - gref).abs().max().item()
                assert err <= max(3e-2 * scale, 8.0 * own, 1e-3 * gabs), \
                    f"grad {k}: err {err:.3e} vs fp64 oracle (scale {scale:.3e}; fp32 oracle's own error {own:.3e})"
            else:
                _close_fro(p.grad, gref, 0.2, 1e-2 * gmax, f"grad {k}")
        except AssertionError as e:
            problems.append(str(e))
    assert not problems, "\n".join(problems)


def test_minibatch_path_matches_edge_list_path():
    """large/main-batch.py:136-143 semantics: a batch given as MiniBatch (CSR-subset structure) == the same batch given as
    (x[idx], subgraph(idx, edge_index, relabel_nodes=True))."""
    from sgformer_b200 import kernels as K
    from sgformer_b200 import large as L
    from sgformer_b200.graph import Graph
    from sgformer_b200.minibatch import RandomPartitionSampler
    from sgformer_b200.synth import make_graph
    n, d = 30000, 32
    ei = make_graph(n, 200000, seed=5).to(DEV)
    x = torch.randn(n, d, device=DEV)
    y = torch.randint(0, 5, (n,), device=DEV)
    model = L.SGFormer(d, 64, 5, gnn_num_layers=2, gnn_use_init=True, gnn_dropout=0.0, trans_dropout=0.0).to(DEV)
    model.train()
    sampler = RandomPartitionSampler(Graph(ei, n), x, y, batch_size=8000, generator=torch.Generator(device=DEV).manual_seed(0))
    assert len(sampler) == 4
    seen = 0
    for mb in sampler:
        out = model(mb)
        ref = model(x[mb.idx], K.subgraph(ei, n, mb.idx))
        _close(out, ref, 1e-5, 1e-6, "mini-batch logits")
        torch.nn.functional.cross_entropy(out, mb.labels).backward()
        seen += mb.idx.numel()
    assert seen == n


def test_host_resident_call_runs_on_gpu():
    """large/eval.py:35-65 `evaluate_large(device='cpu')` moves the model and data to the CPU and calls forward: the
    drop-in computes on the GPU and returns the logits on the host."""
    from sgformer_b200 import large as L
    from sgformer_b200.synth import make_graph
    model = L.SGFormer(16, 32, 5, gnn_num_layers=2).to(DEV)
    x, ei = torch.randn(500, 16), make_graph(500, 2000, seed=0)
    model.eval()
    with torch.no_grad():
        ref = model(x.to(DEV), ei.to(DEV)).cpu()
        model.to("cpu")
        out = model(x, ei)
    assert out.device.type == "cpu"
    _close(out, ref, 1e-6, 1e-6, "host call")


def test_reference_plumbing_methods():
    import copy
    from sgformer_b200 import large as L
    model = L.SGFormer(16, 32, 5, gnn_num_layers=2, gnn_use_init=True)
    assert len(model.params1) + len(model.params2) == len(list(model.parameters()))
    fc0 = model.fc.weight.clone()
    model.reset_parameters()
    assert torch.equal(fc0, model.fc.weight), "reset_parameters must not touch fc (large/ours.py:283-286)"
    m2 = copy.deepcopy(model).to(DEV)
    opt = torch.optim.Adam([{"params": m2.params1, "weight_decay": 1e-3}, {"params": m2.params2, "weight_decay": 0.0}], lr=0.01)
    from sgformer_b200.synth import make_graph
    x, ei = torch.randn(300, 16, device=DEV), make_graph(300, 1000, seed=0).to(DEV)
    y = torch.randint(0, 5, (300,), device=DEV)
    losses = []
    for _ in range(30):
        opt.zero_grad()
        loss = torch.nn.functional.nll_loss(torch.log_softmax(m2(x, ei), 1), y)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < losses[0], f"loss did not decrease: {losses[0]:.4f} -> {losses[-1]:.4f}"
    with pytest.raises(ValueError):
        L.SGFormer(16, 32, 5, aggregate="sum")
    assert model.get_attentions is not None and print(model) is None


def test_host_feeder_double_buffering():
    """HostFeeder hands out exactly what was submitted, in order, while the next submit overwrites the other slot."""
    from sgformer_b200.feed import HostFeeder
    dev = torch.device("cuda:0")
    feeder = HostFeeder(dev)
    host = [(torch.full((1 << 20,), float(i)).pin_memory(), torch.arange(i, i + 1000).pin_memory()) for i in range(6)]
    feeder.submit(host[0])
    with pytest.raises(RuntimeError):
        feeder.submit(host[1])          # one slot belongs to the consumer: only one submit may be outstanding with 2 slots
    sums = []
    for i in range(6):
        a, b = feeder.get()
        if i + 1 < 6:
            feeder.submit(host[i + 1])
        # a long-ish consumer on the compute stream: the following submit must not overwrite its inputs early
        acc = a.clone()
        for _ in range(20):
            acc = acc * 1.0 + 0.0
        sums.append((acc.sum(), b.sum()))
    torch.cuda.synchronize()
    for i, (sa, sb) in enumerate(sums):
        assert sa.item() == float(i) * (1 << 20)
        assert sb.item() == sum(range(i, i + 1000))
    with pytest.raises(RuntimeError):
        feeder.get()


def test_evaluate_on_device_matches_reference_formula():
    """sgformer_b200.eval.evaluate (K11) returns the tuple of large/eval.py:6-33: three accuracies, valid NLL, log_softmax(out)."""
    from types import SimpleNamespace

    from oracle import np_ref
    from sgformer_b200.eval import evaluate

    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    n, c = 3000, 11
    logits = torch.randn(n, c, generator=g)
    label = torch.randint(0, c, (n, 1), generator=g)
    perm = torch.randperm(n, generator=g)
    split = {"train": perm[:1500], "valid": perm[1500:2200], "test": perm[2200:]}

    class Fixed(torch.nn.Module):
        def forward(self, x, ei):
            return logits.to(dev)

    def eval_acc(y_true, y_pred):           # only the name is consulted on the device path
        raise AssertionError("host metric must not be called")

    ds = SimpleNamespace(graph={"node_feat": torch.zeros(n, 1, device=dev), "edge_index": torch.zeros(2, 0, dtype=torch.long, device=dev)},
                         label=label.to(dev))
    tr, va, te, vloss, out = evaluate(Fixed(), ds, {k: v.to(dev) for k, v in split.items()}, eval_acc, torch.nn.NLLLoss(),
                                      SimpleNamespace(dataset="ogbn-products"))
    for got, key in ((tr, "train"), (va, "valid"), (te, "test")):
        assert got == np_ref.eval_acc(label[split[key]].numpy(), logits[split[key]].numpy())
    lsm = torch.log_softmax(logits, 1)
    ref_loss = torch.nn.functional.nll_loss(lsm[split["valid"]], label.squeeze(1)[split["valid"]]).item()
    assert abs(vloss.item() - ref_loss) < 1e-5
    assert torch.allclose(out.cpu(), lsm, atol=1e-6)


def test_host_feeder_prepare_overlaps_graph_build():
    """get -> step -> submit order with prepare=model.prepare_graph: the CSR of the next batch is built on the copy stream while the
    current step runs; results equal the plain (build inside forward) loop and every slot is consumed before it is overwritten."""
    from sgformer_b200 import large as L
    from sgformer_b200.feed import HostFeeder
    from sgformer_b200.graph import clear_cache
    from sgformer_b200.synth import make_graph
    dev = torch.device("cuda:0")
    n, d, h, c = 20000, 32, 64, 5
    kw = dict(gnn_num_layers=2, gnn_dropout=0.0, trans_dropout=0.0)
    g = torch.Generator().manual_seed(0)
    batches = []
    for i in range(5):
        ei = make_graph(n, 80000 + 5000 * i, seed=i)
        if i == 3:
            ei = ei[:, ei[0] < ei[1]].contiguous()        # a directed one: the backward needs its own transposed CSR
        batches.append((torch.randn(n, d, generator=g).pin_memory(), ei.pin_memory(), torch.randint(0, c, (n,), generator=g).pin_memory()))

    def run(prefetch):
        clear_cache()
        torch.manual_seed(1)
        model = L.SGFormer(d, h, c, **kw).to(dev)
        model.train()
        opt = torch.optim.SGD(model.parameters(), lr=0.05)
        feeder = HostFeeder(dev, prepare=(lambda x, ei, y: model.prepare_graph(ei, x.shape[0])) if prefetch else None)
        feeder.submit(batches[0])
        losses = []
        for i in range(len(batches)):
            x, ei, y = feeder.get()
            opt.zero_grad()
            loss = torch.nn.functional.cross_entropy(model(x, ei), y)
            loss.backward()
            opt.step()
            if i + 1 < len(batches):
                feeder.submit(batches[i + 1])
            losses.append(loss)
        torch.cuda.synchronize()
        return torch.stack(losses).cpu(), [p.detach().clone() for p in model.parameters()]

    l0, p0 = run(False)
    l1, p1 = run(True)
    # same kernels on the same data; only the order of the float atomics inside the column reductions may differ
    assert torch.allclose(l0, l1, rtol=1e-5, atol=1e-6), (l0, l1)
    for a, b in zip(p0, p1):
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-6)
