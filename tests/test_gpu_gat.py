"""The GAT backbone on the H100: kernels against the plain-torch GATConv restatement (oracle/gat_oracle.py), the native GAT and
SGFormer(gnn=GAT) against that oracle in fp64 (fp32 1e-4, bf16 1e-2, dropout 0), hub rows, run-to-run bit identity, the attention
dropout mask replayed exactly, and a CUDA-graph captured training step."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import gat_oracle as G
from oracle import sgformer_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


class Data:
    def __init__(self, x, ei):
        self.graph = {"node_feat": x, "edge_index": ei, "num_nodes": x.shape[0]}


def _graph(n, e, seed, hub=0):
    """Directed graph with isolated nodes, duplicate edges and existing self loops; `hub` extra in-edges into node 0."""
    g = torch.Generator().manual_seed(seed)
    live = n - 3                                            # nodes n-3.. are isolated
    src = torch.randint(0, live, (e,), generator=g)
    dst = torch.randint(0, live, (e,), generator=g)
    src = torch.cat([src, src[:e // 10], torch.arange(5)])  # duplicates, self loops
    dst = torch.cat([dst, dst[:e // 10], torch.arange(5)])
    if hub:
        src = torch.cat([src, torch.randint(0, live, (hub,), generator=g)])
        dst = torch.cat([dst, torch.zeros(hub, dtype=torch.int64)])
    return torch.stack([src, dst])


def _close(a, b, rtol, what, floor=1e-3):
    """max |a - b| <= rtol * max(max |b|, floor): `floor` guards tensors whose true value is ~0 (the bias of a conv feeding a
    BatchNorm has a zero gradient)."""
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    assert a.shape == b.shape, f"{what}: shape {tuple(a.shape)} vs {tuple(b.shape)}"
    err = (a - b).abs().max().item()
    ref = b.abs().max().item()
    assert err == err and err <= rtol * max(ref, floor), f"{what}: max err {err:.3e} (ref max {ref:.3e})"


def _close_fro(a, b, tol, what, floor=1e-6):
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    err = (a - b).norm().item() / max(b.norm().item(), floor)
    assert err == err and err <= tol, f"{what}: relative Frobenius error {err:.3e} > {tol}"


# ---- CSR of the GAT edge set ---------------------------------------------------------------------------------------------------
def test_csr_self_loop_mode_matches_numpy():
    from sgformer_b200 import kernels as K
    n = 300
    ei = _graph(n, 2000, 1)
    e = G.gat_edges(ei, n).numpy()
    for by_source in (False, True):
        key, val = (e[0], e[1]) if by_source else (e[1], e[0])
        order = np.lexsort((val, key))
        rp_ref = np.concatenate([[0], np.cumsum(np.bincount(key, minlength=n))])
        rp, col, _ = K.csr_build(ei.to(DEV), n, by_source, 1, False)
        assert np.array_equal(rp.cpu().numpy(), rp_ref)
        assert np.array_equal(col.cpu().numpy(), val[order].astype(np.int32))


# ---- kernels against the oracle ------------------------------------------------------------------------------------------------
def _edge_keep(seed, n, ei_gat, heads, p):
    """fp64 replay of the attention-dropout factors of csrc/gat.cu (gat_keep) for the oracle's edge order."""
    M64 = (1 << 64) - 1

    def mix(x):
        x ^= x >> 33; x = (x * 0xff51afd7ed558ccd) & M64
        x ^= x >> 33; x = (x * 0xc4ceb9fe1a85ec53) & M64
        x ^= x >> 33
        return x
    thr = int(p * 65536.0 + 0.5)
    inv = 65536.0 / (65536.0 - thr)
    seen = {}
    out = torch.empty((ei_gat.shape[1], heads), dtype=torch.float64)
    for k, (s, d) in enumerate(ei_gat.t().tolist()):
        r = seen.get((s, d), 0)
        seen[(s, d)] = r + 1
        key = ((d << 32) | s) & M64
        for h in range(heads):
            x = mix((seed + key * 0x9E3779B97F4A7C15 + ((r << 8) | h) * 0xD1B54A32D192ED03) & M64)
            out[k, h] = inv if (x & 0xFFFF) >= thr else 0.0
    return out


@pytest.mark.parametrize("heads,c,mean,p", [(1, 8, False, 0.0), (2, 16, True, 0.0), (8, 8, False, 0.0), (8, 8, False, 0.5),
                                            (2, 16, True, 0.3)])
def test_gat_kernels_match_oracle(heads, c, mean, p):
    """sgf_gat_logits / fwd / bwd in fp32 against the fp64 oracle conv (attention dropout replayed from the kernel's hash)."""
    from sgformer_b200 import kernels as K
    from sgformer_b200.graph import Graph
    torch.manual_seed(0)
    n, d = 200, 24
    ei = _graph(n, 1500, 2, hub=1500)
    conv = G.GATConv(d, c, heads=heads, concat=not mean).double()
    with torch.no_grad():
        conv.bias.normal_()
    x = torch.randn(n, d, dtype=torch.float64, requires_grad=True)
    seed = 12345
    ep = K.dropout_epoch(create=False)          # the kernels add the registered dropout epoch to their seed
    seed_eff = (seed + (int(ep.item()) if ep is not None else 0) * 0xD1B54A32D192ED03) & ((1 << 64) - 1)
    factor = _edge_keep(seed_eff, n, G.gat_edges(ei, n), heads, p) if p > 0 else None
    out_ref = conv(x, ei, edge_factor=factor)
    gout = torch.randn_like(out_ref)
    out_ref.backward(gout)

    graph = Graph(ei.to(DEV), n, 1)
    xp = (x.detach() @ conv.lin_src.weight.detach().t()).float().to(DEV).contiguous()
    att_s, att_d = conv.att_src.detach().float().reshape(-1).to(DEV), conv.att_dst.detach().float().reshape(-1).to(DEV)
    a_s, a_d = K.gat_logits(xp, heads, c, att_s, att_d)
    xpr = (x.detach() @ conv.lin_src.weight.detach().t()).view(n, heads, c)
    _close(a_s, (xpr * conv.att_src.detach()).sum(-1), 1e-5, "a_src")
    _close(a_d, (xpr * conv.att_dst.detach()).sum(-1), 1e-5, "a_dst")
    out, lse = K.gat_fwd(graph.rowptr, graph.col, xp, a_s, a_d, heads, c, mean, conv.bias.detach().float().to(DEV), p, seed)
    _close(out, out_ref, 1e-5, "out")
    rp_t, col_t = graph.transpose()
    g = gout.float().to(DEV).contiguous()
    dxp, da_s, da_d = K.gat_bwd(graph.rowptr, graph.col, rp_t, col_t, xp, a_s, a_d, lse, g, att_s, att_d, heads, c, mean, p, seed)
    # dx = dxp W, d att_src = sum_j da_src[j] xp_j: compare the derived gradients with autograd
    w = conv.lin_src.weight.detach()
    _close(dxp.double().cpu() @ w, x.grad, 1e-5, "dx")
    _close((da_s.double().cpu()[:, :, None] * xpr.permute(1, 0, 2)).sum(1), conv.att_src.grad[0], 1e-5, "d att_src")
    _close((da_d.double().cpu()[:, :, None] * xpr.permute(1, 0, 2)).sum(1), conv.att_dst.grad[0], 1e-5, "d att_dst")


# ---- modules -------------------------------------------------------------------------------------------------------------------
def _pair(d, h, layers, heads, out_heads, use_bn):
    from sgformer_b200 import medium as M
    torch.manual_seed(7)
    ref = G.GAT(d, h, h, num_layers=layers, dropout=0.0, use_bn=use_bn, heads=heads, out_heads=out_heads).double()
    with torch.no_grad():
        for conv in ref.convs:
            conv.bias.normal_(0, 0.1)
        for bn in ref.bns:
            bn.weight.uniform_(0.5, 1.5); bn.bias.normal_(0, 0.1)
            bn.running_mean.normal_(0, 0.1); bn.running_var.uniform_(0.5, 1.5)
    ours = M.GAT(d, h, h, num_layers=layers, dropout=0.0, use_bn=use_bn, heads=heads, out_heads=out_heads)
    ours.load_state_dict({k: v.float() if v.is_floating_point() else v for k, v in ref.state_dict().items()})
    return ref, ours.to(DEV)


def _check_train_step(ref_fn, ours_fn, ref_mod, ours_mod, x, precision, what):
    rtol = 1e-4 if precision == "fp32" else 1e-2
    ref_mod.eval(); ours_mod.eval()
    with torch.no_grad():
        _close(ours_fn(x.float().to(DEV)), ref_fn(x), rtol, f"{what} eval output")
    ref_mod.train(); ours_mod.train()
    xr = x.clone().requires_grad_(True)
    xo = x.float().to(DEV).requires_grad_(True)
    out_r, out_o = ref_fn(xr), ours_fn(xo)
    _close(out_o, out_r, rtol, f"{what} train output")
    wgt = torch.randn(out_r.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(3))
    (out_r * wgt).sum().backward()
    (out_o * wgt.float().to(DEV)).sum().backward()
    got = dict(ours_mod.named_parameters())
    gmax = max(pr.grad.abs().max().item() for pr in ref_mod.parameters() if pr.grad is not None)
    gnorm = max(pr.grad.norm().item() for pr in ref_mod.parameters() if pr.grad is not None)
    for k, pr in ref_mod.named_parameters():
        if pr.grad is None:                      # BatchNorm affine parameters of a stack without BatchNorm
            assert got[k].grad is None, k
            continue
        if precision == "fp32":
            _close(got[k].grad, pr.grad, rtol, f"{what} grad {k}", floor=0.05 * gmax)
        else:
            # bf16: the 1e-2 bound is an output tolerance; the gradients of these small BatchNorm/ELU stacks carry ~10 % bf16 noise,
            # bounded in relative Frobenius norm as tests/test_gpu_model.py does
            _close_fro(got[k].grad, pr.grad, 0.25, f"{what} grad {k}", floor=2e-2 * gnorm)
    if precision == "fp32":
        _close(xo.grad, xr.grad, rtol, f"{what} grad_x")
        sd = ours_mod.state_dict()
        for k, v in ref_mod.state_dict().items():
            if "running" in k or "num_batches" in k:
                _close(sd[k].float(), v.float(), 1e-4, f"{what} buffer {k}")
    else:
        _close_fro(xo.grad, xr.grad, 0.25, f"{what} grad_x")


CASES = [(2, 1, 1, False), (2, 2, 2, True), (3, 8, 1, True), (3, 8, 2, False)]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("layers,heads,out_heads,use_bn", CASES)
def test_gat_module_matches_oracle(layers, heads, out_heads, use_bn, precision):
    n, d, h = 400, 20, 16
    ei = _graph(n, 3000, 4, hub=1200)
    ref, ours = _pair(d, h, layers, heads, out_heads, use_bn)
    ours.set_precision(precision)
    x = torch.randn(n, d, dtype=torch.float64, generator=torch.Generator().manual_seed(5))
    ei_d = ei.to(DEV)
    _check_train_step(lambda t: ref(Data(t, ei)), lambda t: ours(Data(t, ei_d)), ref, ours, x, precision, "GAT")


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("aggregate", ["add", "cat"])
def test_sgformer_gat_matches_oracle(aggregate, precision):
    from sgformer_b200 import medium as M
    n, d, h, c = 300, 20, 16, 5
    ei = _graph(n, 2000, 6)
    ref_gnn, gnn = _pair(d, h, 2, 2, 1, True)
    model = M.SGFormer(d, h, c, num_layers=1, num_heads=1, alpha=0.3, dropout=0.0, use_bn=True, gnn=gnn, aggregate=aggregate,
                       graph_weight=0.7).to(DEV).set_precision(precision)
    cfg = O.make_config("medium", d, h, c, num_layers=1, num_heads=1, alpha=0.3, dropout=0.0, use_bn=True, aggregate=aggregate,
                        graph_weight=0.7)
    sd = {k: v.detach().double().cpu().clone() for k, v in model.state_dict().items() if not k.startswith("gnn.")}

    class Ref(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.gnn = ref_gnn
            self.p = torch.nn.ParameterDict({k.replace(".", "__"): torch.nn.Parameter(v) for k, v in sd.items()
                                             if v.is_floating_point() and "running" not in k})

        def forward(self, x):
            P = {k.replace("__", "."): v for k, v in self.p.items()}
            P.update({k: v for k, v in sd.items() if "running" in k or "num_batches" in k})
            x1 = O.trans_conv(x, P, cfg, self.training)
            x2 = self.gnn(Data(x, ei))
            hcat = 0.7 * x2 + 0.3 * x1 if aggregate == "add" else torch.cat([x1, x2], 1)
            return F.linear(hcat, P["fc.weight"], P["fc.bias"])

    ref = Ref()
    x = torch.randn(n, d, dtype=torch.float64, generator=torch.Generator().manual_seed(8))
    rtol = 1e-4 if precision == "fp32" else 1e-2
    model.train(); ref.train()
    xr = x.clone().requires_grad_(True)
    xo = x.float().to(DEV).requires_grad_(True)
    out_r, out_o = ref(xr), model(Data(xo, ei.to(DEV)))
    _close(out_o, out_r, rtol, "SGFormer(gnn=GAT) train output")
    wgt = torch.randn(out_r.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(9))
    (out_r * wgt).sum().backward()
    (out_o * wgt.float().to(DEV)).sum().backward()
    got = dict(model.named_parameters())
    gnorm = max(pr.grad.norm().item() for pr in ref_gnn.parameters() if pr.grad is not None)
    # bf16: d att_* ends in the cancellation A - r B of the softmax backward over bf16-rounded x', so it is bounded against a
    # fifth of the branch's largest gradient norm rather than its own
    t, fl = (1e-3, 2e-2) if precision == "fp32" else (0.25, 0.2)
    for k, pr in ref_gnn.named_parameters():
        if pr.grad is None:
            continue
        _close_fro(got["gnn." + k].grad, pr.grad, t, f"grad gnn.{k}", floor=fl * gnorm)
    _close_fro(xo.grad, xr.grad, t, "grad_x")
    model.eval(); ref.eval()
    with torch.no_grad():
        _close(model(Data(x.float().to(DEV), ei.to(DEV))), ref(x), rtol, "SGFormer(gnn=GAT) eval output")


# ---- determinism, dropout, CUDA graphs -----------------------------------------------------------------------------------------
def _train_step(model, x, ei, wgt):
    for p_ in model.parameters():
        p_.grad = None
    xo = x.clone().requires_grad_(True)
    out = model(Data(xo, ei))
    (out * wgt).sum().backward()
    return out.detach().clone(), [p_.grad.clone() for p_ in model.parameters()], xo.grad.clone()


def test_gat_training_step_bit_identical(monkeypatch):
    """Two training steps with the same dropout seed (attention, ELU and input dropout on) give the same bits."""
    from sgformer_b200 import engine as E
    from sgformer_b200 import medium as M
    monkeypatch.setattr(E, "next_seed", lambda: 0x5EED)
    n, d, h = 2000, 32, 16
    ei = _graph(n, 20000, 10, hub=3000).to(DEV)
    model = M.GAT(d, h, h, num_layers=3, dropout=0.4, use_bn=True, heads=8, out_heads=2).to(DEV)
    x = torch.randn(n, d, device=DEV)
    wgt = torch.randn(n, h, device=DEV)
    runs = []
    for _ in range(2):
        torch.manual_seed(11)
        sd = {k: v.clone() for k, v in model.state_dict().items()}
        runs.append(_train_step(model, x, ei, wgt))
        model.load_state_dict(sd)
    (o1, g1, x1), (o2, g2, x2) = runs
    assert torch.equal(o1, o2) and torch.equal(x1, x2)
    assert all(torch.equal(a, b) for a, b in zip(g1, g2))


def test_gat_cuda_graph_step_matches_eager(monkeypatch):
    """A captured training step with input, attention and ELU dropout on: its first replay reproduces the eager step of the same
    seed and epoch bit for bit; a replay after the dropout epoch advanced draws other masks."""
    from sgformer_b200 import engine as E
    from sgformer_b200 import kernels as K
    from sgformer_b200 import medium as M
    n, d, h = 1000, 32, 16
    ei = _graph(n, 8000, 12).to(DEV)
    model = M.GAT(d, h, h, num_layers=2, dropout=0.3, use_bn=True, heads=4, out_heads=1).to(DEV)
    x = torch.randn(n, d, device=DEV)
    wgt = torch.randn(n, h, device=DEV)
    K.dropout_epoch()
    monkeypatch.setattr(E, "next_seed", lambda: 0x5EED)     # eager, warm-up and captured step: one host seed
    sd0 = {k: v.clone() for k, v in model.state_dict().items()}
    eager = _train_step(model, x, ei, wgt)            # also warms the graph-structure caches
    model.load_state_dict(sd0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _train_step(model, x, ei, wgt)
    torch.cuda.current_stream().wait_stream(s)
    model.load_state_dict(sd0)
    for p_ in model.parameters():
        p_.grad = None
    xo = x.clone().requires_grad_(True)
    cg = torch.cuda.CUDAGraph()
    with torch.cuda.graph(cg):
        out = model(Data(xo, ei))
        (out * wgt).sum().backward()
    model.load_state_dict(sd0)
    cg.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager[0])
    assert all(torch.equal(p_.grad, g) for p_, g in zip(model.parameters(), eager[1]))
    assert torch.equal(xo.grad, eager[2])
    K.advance_dropout_epoch()
    model.load_state_dict(sd0)
    cg.replay()
    torch.cuda.synchronize()
    assert not torch.equal(out, eager[0])


def test_dense_dropout_matches_replayed_mask():
    """sgf_dense_dropout (GAT's input dropout) against an fp64 replay of its hash, forward and as its own backward."""
    from sgformer_b200 import kernels as K
    M64 = (1 << 64) - 1
    rows, cols, p, seed = 37, 1433, 0.4, 987654321
    ep = K.dropout_epoch(create=False)
    s_eff = (seed + (int(ep.item()) if ep is not None else 0) * 0xD1B54A32D192ED03) & M64
    k = np.arange(rows * cols, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = np.uint64(s_eff) + k * np.uint64(0x9E3779B97F4A7C15)
        x ^= x >> np.uint64(33); x *= np.uint64(0xff51afd7ed558ccd)
        x ^= x >> np.uint64(33); x *= np.uint64(0xc4ceb9fe1a85ec53)
        x ^= x >> np.uint64(33)
    thr = int(p * 65536.0 + 0.5)
    keep = torch.from_numpy(((x & np.uint64(0xFFFF)) >= np.uint64(thr)).reshape(rows, cols))
    t = torch.randn(rows, cols, dtype=torch.float64)
    ref = t * keep * (65536.0 / (65536.0 - thr))
    got = K.dense_dropout(t.float().to(DEV), p, seed)
    _close(got, ref, 1e-6, "dense dropout")
    assert torch.equal(got.cpu() == 0, ~keep | (t.float() == 0))


# ---- the native modules against the reference's own stack (tests/golden/gat.pt) -----------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_native_modules_match_golden(precision):
    from test_gat_golden import FIXTURE, _models, _state_dict, _unflat
    rtol = 1e-4 if precision == "fp32" else 1e-2
    for name, c in FIXTURE.items():
        _, model = _models(c)
        model.load_state_dict(_state_dict(c))
        model = model.to(DEV).set_precision(precision)
        x, ei = c["x"].to(DEV), c["edge_index"].long().to(DEV)
        model.eval()
        with torch.no_grad():
            _close(model(Data(x, ei)), c["out_eval"], rtol, f"{name} eval")
        model.train()
        xg = x.clone().requires_grad_(True)
        out = model(Data(xg, ei))
        _close(out, c["out_train"], rtol, f"{name} train")
        (out * c["loss_weight"].to(DEV)).sum().backward()
        exp = _unflat(c["grads"])
        got = dict(model.named_parameters())
        gnorm = max(g.norm().item() for g in exp.values())
        tol = 1e-3 if precision == "fp32" else 0.25
        for k, g in exp.items():
            _close_fro(got[k].grad, g, tol, f"{name} grad {k}", floor=2e-2 * gnorm)
        _close_fro(xg.grad, c["grad_x"], tol, f"{name} grad_x")
