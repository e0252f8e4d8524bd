"""DIFFormer (medium/difformer.py, kernel='simple') without a GPU: the value-sum Gram algebra and the graph term in fp64 against
autograd, the forward/backward schedule with the kernels replaced by their emulation (tests/kernel_emu_difformer.py) against autograd of the
oracle restatement, and the module surface."""
import os
import sys

import pytest
import torch

import kernel_emu_difformer as emu
from oracle import difformer_oracle as O
from sgformer_b200 import engine as E
from sgformer_b200 import functional as Fn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DT = torch.float64


def _graph(n, e, seed, directed=False, isolated=0, dup=0):
    g = torch.Generator().manual_seed(seed)
    hi = n - isolated
    ei = torch.stack([torch.randint(0, hi, (e,), generator=g), torch.randint(0, hi, (e,), generator=g)])
    if not directed:
        ei = torch.cat([ei, ei.flip(0)], 1)
    if dup:
        ei = torch.cat([ei, ei[:, :dup]], 1)
    return ei


def _ref_layer(x, wq, bq, wk, bk, wv, bv, ei, cy):
    q, k, v = x @ wq.t() + bq, x @ wk.t() + bk, x @ wv.t() + bv
    return O.simple_attention(q, k, v) + cy * O.gcn_aggregate(v, ei, x.shape[0])


@pytest.mark.parametrize("n,h,use_weight,graph", [(5, 8, True, {}), (37, 12, True, dict(directed=True, isolated=4, dup=9)),
                                                  (64, 16, False, dict(directed=True, isolated=3)), (300, 24, True, {})])
def test_value_sum_gram_layer_with_graph_term_matches_autograd(n, h, use_weight, graph):
    """o + c*y of one layer from the contracts (value-sum Gram prepare, ln_bwd_attn_graph prologue, transposed SpMM, three-
    segment dx) against autograd of the reference formula in fp64: outputs, every parameter gradient and dx to 1e-10."""
    g = torch.Generator().manual_seed(n)
    ei = _graph(n, 3 * n, n, **graph)
    x = torch.randn(n, h, generator=g, dtype=DT).requires_grad_(True)
    mk = lambda *s: (0.4 * torch.randn(*s, generator=g, dtype=DT)).requires_grad_(True)      # noqa: E731
    wq, bq, wk, bk = mk(h, h), mk(h), mk(h, h), mk(h)
    wv, bv = (mk(h, h), mk(h)) if use_weight else (torch.eye(h, dtype=DT).requires_grad_(True), torch.zeros(h, dtype=DT).requires_grad_(True))
    cy = 0.7
    o_ref = _ref_layer(x, wq, bq, wk, bk, wv, bv, ei, cy)
    gout = torch.randn(n, h, generator=g, dtype=DT)
    (o_ref * gout).sum().backward()
    with torch.no_grad():
        xd = x.detach()
        rowptr, col, dinv = emu.csr_build(ei, n)
        rp_t, col_t, _ = emu.csr_build(ei, n, by_source=True, want_dinv=False)
        deg = (rowptr[1:] - rowptr[:-1]).to(DT)
        dinv = torch.where(deg > 0, deg.clamp_min(1).rsqrt(), torch.zeros_like(deg))
        st = emu.attn_gram_prepare_fwd(xd.t() @ xd, xd.sum(0), wq.detach(), bq.detach(), wk.detach(), bk.detach(), wv.detach(),
                                       bv.detach(), n, vsum=True)
        den = xd @ st.tail[0] + st.sc[emu.SC_DEN]
        o = (xd @ st.Bt.t() + st.bt) / den[:, None]
        vs = dinv[:, None] * (xd @ wv.detach().t() + bv.detach())
        rows = torch.repeat_interleave(torch.arange(n), rowptr[1:] - rowptr[:-1])
        y = dinv[:, None] * torch.zeros(n, h, dtype=DT).index_add_(0, rows, vs[col.long()])
        assert (o + cy * y - o_ref).abs().max() < 1e-12 * max(1.0, o_ref.abs().max().item())
        gnum, gden, _, ys, cs, pg, sg = emu.ln_bwd_attn_graph(gout, o, None, xd, y, 1.0, 0.0, cy, None, None, None, False, 0.0, 0,
                                                               1.0, False, None, None, den, dinv)
        dwq, dbq, dwk, dbk, dwv, dbv, bcat, a4 = emu.attn_gram_prepare_bwd(st, xd.t() @ gnum, pg, cs, sg)
        rows_t = torch.repeat_interleave(torch.arange(n), rp_t[1:] - rp_t[:-1])
        dv = dinv[:, None] * torch.zeros(n, h, dtype=DT).index_add_(0, rows_t, ys[col_t.long()])
        dwv = dwv + dv.t() @ xd
        dbv = dbv + dv.sum(0)
        dx = torch.cat([gnum, xd, dv], 1) @ torch.cat([bcat, wv.detach().t()], 1).t() + torch.outer(gden, st.tail[0]) + a4
    checks = [("dWq", dwq, wq.grad), ("dbq", dbq, bq.grad), ("dWk", dwk, wk.grad), ("dbk", dbk, bk.grad), ("dx", dx, x.grad)]
    if use_weight:
        checks += [("dWv", dwv, wv.grad), ("dbv", dbv, bv.grad)]
    for name, got, ref in checks:
        scale = max(ref.abs().max().item(), 1e-30)
        assert (got - ref).abs().max().item() <= 1e-10 * scale + 1e-16, f"{name}: {(got - ref).abs().max().item():.3e} vs {scale:.3e}"


CASES = {
    "default": dict(n=60, d=12, h=16, c=5, graph={}, kw=dict(num_layers=2)),
    "actor_recipe": dict(n=80, d=20, h=64, c=5, graph={}, kw=dict(num_layers=8)),
    "no_graph": dict(n=50, d=10, h=16, c=4, graph={}, kw=dict(use_graph=False, num_layers=3)),
    "graph_weight": dict(n=60, d=12, h=16, c=3, graph={}, kw=dict(graph_weight=0.3, num_layers=2)),
    "no_weight": dict(n=40, d=8, h=16, c=3, graph={}, kw=dict(use_weight=False, num_layers=2)),
    "no_res_no_bn": dict(n=40, d=8, h=16, c=3, graph={}, kw=dict(use_residual=False, use_bn=False, num_layers=2)),
    "source": dict(n=50, d=8, h=16, c=3, graph={}, kw=dict(use_source=True, num_layers=3)),
    "directed": dict(n=70, d=9, h=16, c=4, graph=dict(directed=True, isolated=5, dup=11), kw=dict(num_layers=2)),
}


def make_case(name, seed=0):
    cs = CASES[name]
    cfg = O.make_config(cs["d"], cs["h"], cs["c"], dropout=0.0, **cs["kw"])
    sd = O.init_state_dict(cfg, seed=seed + 1)
    g = torch.Generator().manual_seed(seed + 7)
    x = torch.randn(cs["n"], cs["d"], generator=g)
    ei = _graph(cs["n"], 3 * cs["n"], seed + 11, **cs["graph"])
    return cfg, sd, x, ei


def oracle_run(cfg, sd, x, ei, gw):
    sdr = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    xr = x.clone().requires_grad_(True)
    out = O.difformer_forward(cfg, sdr, xr, ei)
    (out * gw).sum().backward()
    return out.detach(), {k: v.grad for k, v in sdr.items()}, xr.grad


def _close(a, b, rtol, what, floor=1e-3):
    """max |a - b| <= rtol * max(max |b|, floor); `floor` = the model's largest gradient entry for near-zero gradients."""
    a, b = a.double(), b.double()
    err, ref = (a - b).abs().max().item(), b.abs().max().item()
    assert err <= rtol * max(ref, floor), f"{what}: max err {err:.3e} (ref max {ref:.3e})"


@pytest.mark.parametrize("name", sorted(CASES))
def test_emulated_schedule_matches_oracle(monkeypatch, name):
    monkeypatch.setattr(E, "K", emu)
    monkeypatch.setattr(Fn, "K", emu)
    cfg, sd, x, ei = make_case(name)
    gw = torch.randn(x.shape[0], cfg["out_channels"], generator=torch.Generator().manual_seed(3))
    ref, gref, gxref = oracle_run(cfg, sd, x, ei, gw)
    graph = emu.EmuGraph(ei, x.shape[0], 0) if cfg["use_graph"] else None
    names = tuple(sd)
    params = [sd[k].clone().requires_grad_(True) for k in names]
    xg = x.clone().requires_grad_(True)
    out = Fn.DIFFormerFn.apply(xg, graph, cfg, E.FP32, True, names, *params)
    _close(out, ref, 1e-5, "logits")
    (out * gw).sum().backward()
    _close(xg.grad, gxref, 1e-5, "grad_x")
    for k, p in zip(names, params):
        if gref[k] is None:               # LayerNorms of a use_bn=False model take no part
            assert p.grad is None, k
        else:
            _close(p.grad, gref[k], 1e-5, k)


def test_emulated_attentions_match_oracle(monkeypatch):
    monkeypatch.setattr(E, "K", emu)
    cfg, sd, x, _ = make_case("no_graph")
    att = E.difformer_attentions(sd, cfg, emu.pack_operand(x, False, 3), E.FP32)
    _close(torch.stack(att, 0).unsqueeze(-1), O.difformer_attentions(cfg, sd, x), 1e-5, "attentions")


def test_dropin_surface_and_parse_call():
    """`from difformer import *` of medium/parse.py finds the four names; the constructor call parse.py makes for the Actor line
    of medium/run.sh (--num_layers 8 --hidden_channels 64 --dropout 0.6 --alpha 0.5 --num_heads 1) builds the reference's
    parameter tree."""
    sys.path.insert(0, os.path.join(ROOT, "sgformer_b200", "dropin", "medium"))
    try:
        import difformer as D
    finally:
        sys.path.pop(0)
    for name in ("DIFFormer", "DIFFormerConv", "full_attention_conv", "gcn_conv"):
        assert hasattr(D, name), name
    m = D.DIFFormer(in_channels=932, hidden_channels=64, out_channels=5, num_layers=8, alpha=0.5, dropout=0.6, num_heads=1)
    cfg = O.make_config(932, 64, 5, num_layers=8)
    keys = sorted(m.state_dict())
    assert keys == sorted(O.init_state_dict(cfg))
    assert list(m.convs[0]._modules) == ["Wk", "Wq", "Wv"]
    fc0 = m.fcs[0].weight.clone()
    m.reset_parameters()
    assert not torch.equal(fc0, m.fcs[0].weight)          # fcs are reset too (unlike SGFormer's fc)


def test_out_of_scope_options_raise():
    from sgformer_b200.difformer import DIFFormer
    with pytest.raises(ValueError, match="num_heads"):
        DIFFormer(8, 16, 3, num_heads=2)
    with pytest.raises(NotImplementedError):
        DIFFormer(8, 16, 3, kernel="sigmoid")
    m = DIFFormer(8, 16, 3)
    with pytest.raises(ValueError, match="use_graph=False"):
        m.get_attentions(torch.randn(4, 8))


def test_no_cpu_fallback():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from sgformer_b200.difformer import DIFFormer, gcn_conv

    class Data:
        graph = {"node_feat": torch.randn(4, 8), "edge_index": torch.zeros(2, 3, dtype=torch.long)}

    with pytest.raises(RuntimeError, match="no CPU fallback"):
        DIFFormer(8, 16, 3)(Data)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        gcn_conv(torch.randn(4, 1, 8), Data.graph["edge_index"], None)


# ------------------------------------------------------------------------------------------------------------------------------
# tests/golden/difformer.pt: outputs of the unmodified reference (tests/make_golden_difformer.py)
# ------------------------------------------------------------------------------------------------------------------------------
def _unflat(f):
    out, o = {}, 0
    for name, shape in zip(f["names"], f["shapes"]):
        k = 1
        for s_ in shape:
            k *= s_
        out[name] = f["flat"][o:o + k].reshape(shape).clone()
        o += k
    return out


def load_fixture():
    """{case: (cfg, state_dict, x, edge_index, loss_weight, expected)} with expected = out_eval, out_train, grads, grad_x
    (+ attentions)."""
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "difformer.pt"), weights_only=False)
    out = {}
    for name, c in fx.items():
        cfg = O.make_config(c["in_channels"], c["hidden"], c["out_channels"], **c["kw"])
        exp = dict(out_eval=c["out_eval"], out_train=c["out_train"], grads=_unflat(c["grads"]), grad_x=c["grad_x"],
                   attentions=c.get("attentions"))
        out[name] = (cfg, _unflat(c["state_dict"]), c["x"], c["edge_index"].long(), c["loss_weight"], exp)
    return out


FIXTURE = load_fixture()


def test_fixture_covers_the_cases():
    assert set(FIXTURE) == set(CASES)
    cfg = FIXTURE["actor_recipe"][0]
    assert (cfg["num_layers"], cfg["hidden"]) == (8, 64)
    ei, n = FIXTURE["directed"][3], FIXTURE["directed"][2].shape[0]
    assert torch.bincount(ei.reshape(-1), minlength=n).eq(0).any()                     # isolated nodes
    assert ei.t().unique(dim=0).shape[0] < ei.shape[1]                                 # duplicate edges


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_fixture(name):
    cfg, sd, x, ei, lw, exp = FIXTURE[name]
    with torch.no_grad():
        _close(O.difformer_forward(cfg, sd, x, ei), exp["out_eval"], 1e-5, "eval logits")
    out, grads, gx = oracle_run(cfg, sd, x, ei, lw)
    _close(out, exp["out_train"], 1e-5, "train logits")
    _close(gx, exp["grad_x"], 1e-5, "grad_x")
    gmax = max(g.abs().max().item() for g in exp["grads"].values())
    for k, g in exp["grads"].items():
        _close(grads[k], g, 1e-5, k, floor=gmax)
    if exp["attentions"] is not None:
        _close(O.difformer_attentions(cfg, sd, x), exp["attentions"], 1e-5, "attentions")


@pytest.mark.parametrize("name", sorted(CASES))
def test_emulated_schedule_matches_fixture(monkeypatch, name):
    monkeypatch.setattr(E, "K", emu)
    monkeypatch.setattr(Fn, "K", emu)
    cfg, sd, x, ei, lw, exp = FIXTURE[name]
    graph = emu.EmuGraph(ei, x.shape[0], 0) if cfg["use_graph"] else None
    names = tuple(sd)
    params = [sd[k].clone().requires_grad_(True) for k in names]
    xg = x.clone().requires_grad_(True)
    out = Fn.DIFFormerFn.apply(xg, graph, cfg, E.FP32, True, names, *params)
    _close(out, exp["out_train"], 1e-5, "train logits")
    (out * lw).sum().backward()
    _close(xg.grad, exp["grad_x"], 1e-5, "grad_x")
    gmax = max(g.abs().max().item() for g in exp["grads"].values())
    for k, p in zip(names, params):
        if k in exp["grads"]:
            _close(p.grad, exp["grads"][k], 1e-5, k, floor=gmax)
        else:
            assert p.grad is None, k
