"""DIFFormer on the H100: the new kernel modes against their contracts (tests/kernel_emu_difformer.py), the model against the oracle
restatement (oracle/difformer_oracle.py, checked against the reference by tests/test_difformer.py), the attention term alone
against fp64, determinism, and a medium/main.py-style training loop."""
import copy
import itertools

import pytest
import torch
import torch.nn.functional as F

import kernel_emu_difformer as emu
from oracle import difformer_oracle as O
from test_difformer import CASES, FIXTURE, make_case, oracle_run

pytestmark = pytest.mark.gpu
DEV = "cuda"


class Data:
    def __init__(self, x, ei):
        self.graph = {"node_feat": x, "edge_index": ei}


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-3)


def _model(cfg, sd, prec):
    from sgformer_b200.difformer import DIFFormer
    kw = {k: cfg[k] for k in ("num_layers", "alpha", "dropout", "use_bn", "use_residual", "use_weight", "use_graph",
                              "graph_weight", "use_source")}
    m = DIFFormer(cfg["in_channels"], cfg["hidden"], cfg["out_channels"], **kw)
    m.load_state_dict(sd)
    return m.to(DEV).set_precision(prec)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_row_pass_modes_match_contracts(dtype):
    from sgformer_b200 import kernels as K
    g = torch.Generator().manual_seed(0)
    n, h = 1000, 64
    o, r, y, dy, xa = (torch.randn(n, h, generator=g).to(DEV, dtype) for _ in range(5))
    gamma, beta = (1 + 0.1 * torch.randn(h, generator=g)).to(DEV), (0.1 * torch.randn(h, generator=g)).to(DEV)
    den = (1 + torch.rand(n, generator=g)).to(DEV)
    dinv = torch.rand(n, generator=g).to(DEV)
    tol = 1e-5 if dtype == torch.float32 else 2e-2
    out, st = K.ln_fwd_graph(o, r, y, 0.3, 0.5, 0.7, gamma, beta, True, False, 0.0, 0)
    ref, _ = emu.ln_fwd_graph(o.cpu(), r.cpu(), y.cpu(), 0.3, 0.5, 0.7, gamma.cpu(), beta.cpu(), True, False, 0.0, 0)
    assert _rel(out, ref) < tol
    dg, db = torch.zeros(h, device=DEV), torch.zeros(h, device=DEV)
    got = K.ln_bwd_attn_graph(dy, o, r, xa, y, 0.3, 0.5, 0.7, gamma, beta, st, True, 0.0, 0, 1.0, True, dg, db, den, dinv)
    dge, dbe = torch.zeros(h), torch.zeros(h)
    exp = emu.ln_bwd_attn_graph(dy.cpu(), o.cpu(), r.cpu(), xa.cpu(), y.cpu(), 0.3, 0.5, 0.7, gamma.cpu(), beta.cpu(), None, True, 0.0,
                                0, 1.0, True, dge, dbe, den.cpu(), dinv.cpu())
    for name, a, b in zip(("gnum", "gden", "dr", "ys", "cs", "pg", "sg"), got, exp):
        assert _rel(a, b) < 10 * tol, name
    assert _rel(dg, dge) < 10 * tol and _rel(db, dbe) < 10 * tol


def test_value_sum_prepare_matches_contract():
    from sgformer_b200 import kernels as K
    g = torch.Generator().manual_seed(1)
    n, h = 500, 48
    x = torch.randn(n, h, generator=g, dtype=torch.float64)
    ws = [0.3 * torch.randn(h, h, generator=g, dtype=torch.float64) if i % 2 == 0 else 0.3 * torch.randn(h, generator=g, dtype=torch.float64)
          for i in range(6)]
    G, s = x.t() @ x, x.sum(0)
    st = K.attn_gram_prepare_fwd(G.float().to(DEV), s.float().to(DEV), *[w.float().to(DEV) for w in ws], n, vsum=True)
    se = emu.attn_gram_prepare_fwd(G, s, *ws, n, vsum=True)
    for f in ("Bt", "bt", "tail"):
        assert _rel(getattr(st, f), se[f]) < 1e-4, f
    P, pg, cs, sg = (torch.randn(h, h, generator=g, dtype=torch.float64), torch.randn(h, generator=g, dtype=torch.float64),
                     torch.randn(h, generator=g, dtype=torch.float64), torch.randn(1, generator=g, dtype=torch.float64))
    got = K.attn_gram_prepare_bwd(st, *[t.float().to(DEV) for t in (P, pg, cs, sg)])
    exp = emu.attn_gram_prepare_bwd(se, P, pg, cs, sg)
    for name, a, b in zip(("dwq", "dbq", "dwk", "dbk", "dwv", "dbv", "bcat", "a4"), got, exp):
        assert _rel(a, b) < 1e-4, name


@pytest.mark.parametrize("prec,tol", [("fp32", 1e-4), ("bf16", 1e-2)])
@pytest.mark.parametrize("name", sorted(CASES))
def test_model_matches_oracle(name, prec, tol):
    cfg, sd, x, ei = make_case(name)
    gw = torch.randn(x.shape[0], cfg["out_channels"], generator=torch.Generator().manual_seed(3))
    ref, gref, gxref = oracle_run(cfg, sd, x, ei, gw)
    m = _model(cfg, sd, prec)
    m.eval()
    with torch.no_grad():
        assert _rel(m(Data(x.to(DEV), ei.to(DEV))), ref) < tol, "eval logits"
    m.train()
    xg = x.to(DEV).requires_grad_(True)
    out = m(Data(xg, ei.to(DEV)))
    assert _rel(out, ref) < tol, "train logits"
    (out * gw.to(DEV)).sum().backward()
    got = dict(m.named_parameters())
    if prec == "fp32":
        assert _rel(xg.grad, gxref) < 5 * tol, "grad_x"
        for k, g in gref.items():
            assert (got[k].grad is None) if g is None else _rel(got[k].grad, g) < 5 * tol, k
        return
    # bf16: 1e-2 is an output tolerance.  Gradients carry the noise of bf16 activations (the CPU emulation of this schedule
    # with bf16 activations deviates from the fp32 oracle by up to 9 % in grad_x and more in near-zero parameter gradients), so
    # they are bounded in relative Frobenius norm as in test_gpu_model.py
    gmax = max(g.norm().item() for g in gref.values() if g is not None)
    assert _fro(xg.grad, gxref, 0.0) < 0.25, "grad_x"
    for k, g in gref.items():
        assert (got[k].grad is None) if g is None else _fro(got[k].grad, g, 2e-2 * gmax) < 0.25, k


def _fro(a, b, floor):
    a, b = a.double().cpu(), b.double().cpu()
    return (a - b).norm().item() / max(b.norm().item(), floor, 1e-30)


@pytest.mark.parametrize("prec,tol", [("fp32", 1e-4), ("bf16", 2e-2)])
@pytest.mark.parametrize("name", sorted(CASES))
def test_model_matches_reference_fixture(name, prec, tol):
    """Against the outputs of the unmodified reference (tests/golden/difformer.pt): eval and train logits, grad_x and every
    parameter gradient (bf16 gradients in relative Frobenius norm, see test_model_matches_oracle).  The small cases are h = 8 to
    keep the file small; there bf16 activations alone put the logits up to 1.7 % off (the CPU emulation of this schedule with
    bf16 activations, no_res_no_bn case), so bf16 is held to 2e-2 here and to 1e-2 at h >= 16 in test_model_matches_oracle."""
    cfg, sd, x, ei, lw, exp = FIXTURE[name]
    m = _model(cfg, sd, prec)
    m.eval()
    with torch.no_grad():
        assert _rel(m(Data(x.to(DEV), ei.to(DEV))), exp["out_eval"]) < tol, "eval logits"
    m.train()
    xg = x.to(DEV).requires_grad_(True)
    out = m(Data(xg, ei.to(DEV)))
    assert _rel(out, exp["out_train"]) < tol, "train logits"
    (out * lw.to(DEV)).sum().backward()
    got = dict(m.named_parameters())
    gmax = max(g.norm().item() for g in exp["grads"].values())
    for k, p in got.items():
        g = exp["grads"].get(k)
        if g is None:
            assert p.grad is None, k
        elif prec == "fp32":
            assert _rel(p.grad, g) < 5 * tol, k
        else:
            assert _fro(p.grad, g, 2e-2 * gmax) < 0.25, k
    assert (_rel(xg.grad, exp["grad_x"]) < 5 * tol) if prec == "fp32" else (_fro(xg.grad, exp["grad_x"], 0.0) < 0.25), "grad_x"
    if exp["attentions"] is not None:
        assert _rel(m.get_attentions(x.to(DEV)), exp["attentions"]) < (2e-4 if prec == "fp32" else 3e-2), "attentions"


def test_gcn_conv_matches_oracle():
    from sgformer_b200.difformer import gcn_conv
    g = torch.Generator().manual_seed(2)
    n, heads, d = 300, 1, 32
    x = torch.randn(n, heads, d, generator=g)
    ei = torch.randint(0, n - 7, (2, 1500), generator=g)              # directed, with isolated nodes and duplicates
    ei = torch.cat([ei, ei[:, :40]], 1)
    ref = O.gcn_aggregate(x.reshape(n, -1), ei, n).reshape(n, heads, d)
    assert _rel(gcn_conv(x.to(DEV), ei.to(DEV), None), ref) < 1e-5
    with pytest.raises(NotImplementedError):
        gcn_conv(x.to(DEV), ei.to(DEV), torch.ones(ei.shape[1], device=DEV))


def test_attentions_match_oracle():
    cfg, sd, x, _ = make_case("no_graph")
    m = _model(cfg, sd, "fp32")
    assert _rel(m.get_attentions(x.to(DEV)), O.difformer_attentions(cfg, sd, x)) < 1e-4
    assert m.get_attentions(x).device.type == "cpu"          # CPU input: computed on the GPU, returned on the CPU


@pytest.mark.parametrize("n,h", [(37, 16), (300, 24), (128, 64)])
def test_attention_term_vs_fp64(n, h):
    """The q~(k~^T v) part alone (output minus the sum-of-values term) against fp64: a wrong k^T v path cannot hide behind
    the sum-of-values term, which dominates the output.  fp32 only: a bf16 output rounds away more than this term's 2e-3."""
    prec = "fp32"
    from sgformer_b200 import engine as E
    g = torch.Generator().manual_seed(n + h)
    x = torch.randn(n, h, generator=g, dtype=torch.float64)
    P = {f"c.{nm}.weight": 0.4 * torch.randn(h, h, generator=g, dtype=torch.float64) for nm in ("Wq", "Wk", "Wv")}
    P.update({f"c.{nm}.bias": torch.randn(h, generator=g, dtype=torch.float64) for nm in ("Wq", "Wk", "Wv")})
    lin = lambda nm: x @ P[f"c.{nm}.weight"].t() + P[f"c.{nm}.bias"]          # noqa: E731
    q, k, v = lin("Wq"), lin("Wk"), lin("Wv")
    qn, kn = q / q.norm(), k / k.norm()
    den = qn @ kn.sum(0) + n
    term_ref = (qn @ (kn.t() @ v)) / den[:, None]
    pr = E.precision(prec)
    tape = E.Tape()
    xa = x.float().to(DEV).to(pr.act_dtype)
    o = E.attention_gram_forward({k_: t.float().to(DEV) for k_, t in P.items()}, "c.", xa, True, pr, tape, vsum=True)
    den_g = tape["den"].double().cpu() * n
    term = o.double().cpu() - v.sum(0) / den_g[:, None]
    assert (term - term_ref).abs().max().item() <= 2e-3 * term_ref.abs().max().item()


def test_actor_shape_fp32_matches_oracle():
    n, d, h, c = 7600, 932, 64, 5
    cfg = O.make_config(d, h, c, num_layers=8, dropout=0.0)
    sd = O.init_state_dict(cfg, seed=5)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(n, d, generator=g)
    ei = torch.randint(0, n, (2, 15000), generator=g)
    ei = torch.cat([ei, ei.flip(0)], 1)
    gw = torch.randn(n, c, generator=g)
    sdr = {k: v.double().to(DEV).requires_grad_(True) for k, v in sd.items()}
    xr = x.double().to(DEV).requires_grad_(True)
    ref = O.difformer_forward(cfg, sdr, xr, ei.to(DEV))
    (ref * gw.double().to(DEV)).sum().backward()
    m = _model(cfg, sd, "fp32")
    xg = x.to(DEV).requires_grad_(True)
    out = m(Data(xg, ei.to(DEV)))
    assert _rel(out, ref) < 1e-4
    (out * gw.to(DEV)).sum().backward()
    assert _rel(xg.grad, xr.grad) < 5e-4
    for k, p in m.named_parameters():
        assert _rel(p.grad, sdr[k].grad) < 5e-4, k


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_training_step_is_bit_identical(prec, monkeypatch):
    """Two runs of the same training step (dropout on, so the masks must repeat too) give identical logits and parameters."""
    from sgformer_b200 import engine as E
    cfg, sd, x, ei = make_case("default")
    cfg = dict(cfg, dropout=0.5)
    outs = []
    for _ in range(2):
        torch.manual_seed(0)
        monkeypatch.setattr(E, "_seed_counter", itertools.count(1))       # same dropout seed for both runs
        m = _model(cfg, sd, prec)
        m.train()
        opt = torch.optim.Adam(m.parameters(), lr=0.01)
        out = m(Data(x.to(DEV), ei.to(DEV)))
        F.cross_entropy(out, torch.arange(x.shape[0], device=DEV) % cfg["out_channels"]).backward()
        opt.step()
        outs.append((out.detach().clone(), [p.detach().clone() for p in m.parameters()]))
    assert torch.equal(outs[0][0], outs[1][0])
    assert all(torch.equal(a, b) for a, b in zip(outs[0][1], outs[1][1]))


def _planted(n, c, d, deg, seed):
    g = torch.Generator().manual_seed(seed)
    y = torch.randint(0, c, (n,), generator=g)
    x = torch.randn(c, d, generator=g)[y] + 2.0 * torch.randn(n, d, generator=g)
    src = torch.randint(0, n, (n * deg,), generator=g)
    same = torch.rand(n * deg, generator=g) < 0.8
    order = torch.argsort(y)
    starts = torch.searchsorted(y[order], torch.arange(c))
    counts = torch.bincount(y, minlength=c)
    pick = (starts[y[src]] + (torch.rand(n * deg, generator=g) * counts[y[src]]).long()).clamp_max(n - 1)
    dst = torch.where(same, order[pick], torch.randint(0, n, (n * deg,), generator=g))
    return x, torch.stack([torch.cat([src, dst]), torch.cat([dst, src])]), y


def test_medium_main_style_loop_trains():
    """medium/main.py's loop for --method difformer: reset_parameters, Adam with weight decay, per epoch
    train() + NLL(log_softmax(out)[train_idx]) + step, evaluation under no_grad."""
    from sgformer_b200.difformer import DIFFormer
    n, c, d = 3000, 5, 64
    x, ei, y = _planted(n, c, d, 6, 0)
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(1))
    tr, te = perm[: n // 2].to(DEV), perm[n // 2:].to(DEV)
    data = Data(x.to(DEV), ei.to(DEV))
    y = y.to(DEV)
    torch.manual_seed(0)
    model = DIFFormer(d, 64, c, num_layers=4, alpha=0.5, dropout=0.3, num_heads=1).to(DEV)
    model.reset_parameters()
    opt = torch.optim.Adam(model.parameters(), lr=0.01, weight_decay=5e-4)
    crit = torch.nn.NLLLoss()
    for _ in range(60):
        model.train()
        opt.zero_grad()
        out = F.log_softmax(model(data), dim=1)
        crit(out[tr], y[tr]).backward()
        opt.step()
    model.eval()
    with torch.no_grad():
        acc = (model(data).argmax(1)[te] == y[te]).float().mean().item()
    assert acc > 0.8, f"test accuracy {acc:.3f}"
    copy.deepcopy(model)(data)
