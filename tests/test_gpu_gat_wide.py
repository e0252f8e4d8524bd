"""GAT layers wider than one launch of the GAT kernels (engine.gat_groups) on the H100, against fp64.

  (a) one layer's head-group schedule (engine._gat_conv_fwd / _gat_conv_bwd) at the wide shapes on the directed test graph of
      tests/test_gpu_gat_widths.py (duplicates, self loops, a hub row), p = 0 and 0.5: out, lse, dxp, da_src, da_dst element by
      element in that file's bounds, each group's attention mask replayed under its own seed;
  (b) GAT and SGFormer(gnn=GAT) at the wide widths against oracle/gat_oracle.py in that file's gradient bounds;
  (c) a training step with input, attention and post-ELU dropout, the masks of heads in different groups replayed;
  (d) run-to-run bit identity, a CUDA-graph captured step equal to eager, a reference state_dict round trip at a padded width;
  (e) layers that fit one launch: the schedule's launches are the single direct kernel calls, bit for bit."""
import copy
import math

import pytest
import torch
import torch.nn.functional as F

import gat_widths as W
import test_gpu_gat_widths as GW
from dropout_mask import current_epoch, keep_mask, keep_scale
from oracle import gat_oracle as G

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS_BF16 = 2.0 ** -8


@pytest.fixture(scope="module")
def Kmod():
    from sgformer_b200 import kernels
    return kernels


def _plan(dtype, H, C, mean):
    from sgformer_b200 import engine as E
    return E._gat_plan(E.precision(dtype), H, C, mean, 0)


# ------------------------------------------------------------------------------------------------
# (a) one layer
# ------------------------------------------------------------------------------------------------
# (dtype, H, C, mean); C is the run width (padded widths such as 250 run at cp = 252)
LAYER_SHAPES = [("fp32", 4, 256, False), ("fp32", 8, 128, False), ("fp32", 16, 64, False), ("fp32", 3, 252, False),
                ("bf16", 8, 256, False), ("bf16", 16, 64, False), ("bf16", 3, 104, False), ("fp32", 10, 8, True),
                ("bf16", 10, 8, True), ("fp32", 4, 256, True), ("bf16", 16, 64, True)]


def run_layer(shape, p, seed=0x5EED):
    """The group schedule of one layer on the base graph -> (got, ref, S, lay)."""
    from sgformer_b200 import engine as E
    dtype, H, C, mean = shape
    lay = _plan(dtype, H, C, mean)
    assert lay.cp == C
    graph, n = GW._graph("base")
    xp, g, att_s, att_d, bias = GW._inputs(n, dtype, H, C, mean, 1000 * H + C + mean)
    z, parts = E._gat_conv_fwd(graph, xp, lay, att_s, att_d, bias, p, seed)
    rp_t, col_t = graph.transpose()
    dxp, das = E._gat_conv_bwd(graph, rp_t, col_t, dict(lay=lay, xp=xp, att=(att_s, att_d), parts=parts), g, p, seed)
    edges = GW._csr_edges(graph)
    factor = None
    if p > 0:
        ep = current_epoch()
        factor = torch.cat([W.edge_keep(W.with_epoch(E._gat_group_seed(seed, k), ep), n, edges, hg, p)
                            for k, (_, hg) in enumerate(lay.groups)], 1)
    a_s, a_d, lse = (torch.cat([pt[j] for pt in parts], 1) for j in range(3))
    ref, S = GW.reference(graph, n, xp, a_s, a_d, lse, att_s, att_d, bias, g, H, C, mean, factor)
    got = dict(a_src=a_s, a_dst=a_d, out=z, lse=lse, dxp=dxp, da_src=torch.cat([d[0] for d in das], 0),
               da_dst=torch.cat([d[1] for d in das], 0))
    return got, ref, S, lay


@pytest.mark.parametrize("shape", LAYER_SHAPES, ids=[W.shape_id(s) for s in LAYER_SHAPES])
def test_wide_layer_matches_fp64(shape):
    dtype, H, C, mean = shape
    bf = dtype == "bf16"
    problems = []
    for p in (0.0, 0.5):
        got, ref, S, lay = run_layer(shape, p)
        multi_mean = mean and len(lay.groups) > 1
        for name in GW.K:
            if name == "out" and multi_mean:
                continue
            problems += [f"{pr} [p={p}]" for pr in W.check_elementwise(name, got[name], ref[name], S[name], GW.K[name],
                                                                         bf and name in GW.STORED)]
        if multi_mean:
            # the groups' means, their weighted sum and the bias add are each stored in the activation dtype: one more rounding
            # of a value bounded by S per store (2 x groups - 1 more than the single launch)
            u = EPS_BF16 if bf else 2.0 ** -24
            o, r, s_ = got["out"].double(), ref["out"], S["out"]
            d = (o - r).abs() - (2 * len(lay.groups) - 1) * u * s_ - (W.bf16_ulp(r) if bf else 0.0)
            bad = d > GW.K["out"] * W.EPS32 * s_
            if bool(bad.any()):
                problems.append(f"out: {int(bad.sum())} elements above the grouped head-mean bound [p={p}]")
    assert not problems, "\n".join(problems)


def test_groups_draw_independent_attention_masks():
    """Two groups of 8 heads: the same head of different groups keeps different edges."""
    from sgformer_b200 import engine as E
    graph, n = GW._graph("base")
    edges = GW._csr_edges(graph)
    lay = _plan("fp32", 16, 64, False)
    ep = current_epoch()
    m = [W.edge_keep(W.with_epoch(E._gat_group_seed(0x5EED, k), ep), n, edges, 8, 0.5) for k in range(2)]
    assert not torch.equal(m[0] == 0, m[1] == 0)
    assert E._gat_group_seed(0x5EED, 0) == 0x5EED and len(lay.groups) == 2


# ------------------------------------------------------------------------------------------------
# (b) modules
# ------------------------------------------------------------------------------------------------
# (precision, heads, hidden, layers, use_bn, out_heads, out_channels)
MODULE_CASES = [("fp32", 4, 256, 2, True, 1, 7), ("fp32", 8, 128, 3, True, 10, 7), ("fp32", 16, 64, 2, False, 2, 7),
                ("fp32", 3, 250, 3, True, 2, 7), ("bf16", 8, 256, 2, True, 1, 7), ("bf16", 16, 64, 3, True, 10, 5),
                ("bf16", 3, 100, 2, True, 2, 7), ("fp32", 4, 256, 2, True, 4, 256)]


@pytest.mark.parametrize("case", MODULE_CASES, ids=[f"{c[0]}-{c[1]}x{c[2]}-L{c[3]}-bn{int(c[4])}-oh{c[5]}c{c[6]}" for c in MODULE_CASES])
def test_wide_gat_module_matches_oracle(case):
    precision, heads, h, layers, use_bn, out_heads, c = case
    n, d, ei = GW._cora()
    ref = GW._ref_gat(d, h, c, layers, heads, out_heads, use_bn)
    ours = GW._ours_gat(ref, d, h, c, layers, heads, out_heads, use_bn, precision)
    gen = torch.Generator().manual_seed(n + layers + heads)
    x = torch.randn(n, d, generator=gen, dtype=torch.float64)
    lw = torch.randn(n, c, generator=gen, dtype=torch.float64) / math.sqrt(n)
    r64, r32 = GW._oracle_step(ref, x, ei, lw, torch.float64), GW._oracle_step(ref, x, ei, lw, torch.float32)
    got = GW._ours_step(ours, x, ei, lw)
    problems = GW.compare_step(got, r64, r32, precision, layers, use_bn, f"{case}")
    assert not problems, "\n".join(problems)


@pytest.mark.parametrize("precision,h", [("fp32", 128), ("bf16", 256)])
@pytest.mark.parametrize("aggregate", ["add", "cat"])
def test_wide_sgformer_gat_matches_oracle(aggregate, precision, h):
    """`--method ours --backbone gat --hidden_channels 128` (8 x 128, fp32) and 8 x 256 in bf16: two head groups per hidden layer."""
    n, d, ei = GW._cora()
    c = 7
    ref, model, cfg = GW._sgformer_pair(d, h, c, aggregate, precision)
    gen = torch.Generator().manual_seed(19)
    x = torch.randn(n, d, generator=gen, dtype=torch.float64)
    lw = torch.randn(n, c, generator=gen, dtype=torch.float64) / math.sqrt(n)
    r64, r32 = GW._oracle_step(ref, x, ei, lw, torch.float64), GW._oracle_step(ref, x, ei, lw, torch.float32)
    got = GW._ours_step(model, x, ei, lw)
    rename = lambda r: dict(r, grads={GW.ref_name(k): v for k, v in r["grads"].items()})
    r64, r32 = rename(r64), rename(r32)
    problems = GW.compare_step(got, r64, r32, precision, 2, True, f"SGFormer(gnn=GAT) {aggregate} {precision} h={h}", ocfg=cfg)
    assert not problems, "\n".join(problems)


# ------------------------------------------------------------------------------------------------
# (c) dropout
# ------------------------------------------------------------------------------------------------
STEP_SEED = 0x5EED


def _masked_oracle(ref, x, ei, lw, p, seed, epoch, dtype, plans, offset=True):
    """models.GAT with the kernels' masks: input dropout, attention dropout per head group (group k: the layer's seed offset by
    engine._gat_group_seed), post-ELU dropout per column block of each group."""
    from sgformer_b200 import engine as E
    gseed = E._gat_group_seed if offset else (lambda s_, k: s_)
    mod = copy.deepcopy(ref).to(DEV, dtype)
    mod.train()
    n, d = x.shape
    xg = x.to(DEV, dtype).clone().requires_grad_(True)
    eid = ei.to(DEV)
    edges = G.gat_edges(ei, n)
    sc = keep_scale(p)
    h = xg * (W.dense_keep(W.with_epoch(seed + E._SEED_GAT_INPUT, epoch), n, d, p).to(DEV, dtype) * sc)
    for i, conv in enumerate(mod.convs):
        lay = plans[i]
        fac = torch.cat([W.edge_keep(W.with_epoch(gseed(seed + E._SEED_GAT_ATT + i, k), epoch), n, edges, hg, p)
                         for k, (_, hg) in enumerate(lay.groups)], 1).to(DEV, dtype)
        h = conv(h, eid, edge_factor=fac)
        if i < len(mod.convs) - 1:
            if mod.use_bn:
                h = mod.bns[i](h)
            h = F.elu(h)
            m = torch.cat([torch.from_numpy(keep_mask(gseed(seed + E._SEED_GAT_ACT + i, k), n, hg * lay.cp, p, epoch))
                           for k, (_, hg) in enumerate(lay.groups)], 1).to(DEV, dtype)
            h = h * (m * sc)
    (h * lw.to(DEV, dtype)).sum().backward()
    grads = {k: q.grad for k, q in mod.named_parameters() if q.grad is not None}
    grads["__x__"] = xg.grad
    buffers = {k: v for k, v in mod.state_dict().items() if "running" in k}
    return dict(out_train=h.detach(), grads=grads, buffers=buffers)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_wide_training_step_with_all_dropout_streams(monkeypatch, precision):
    """16 heads x 64 (two groups of 8 per hidden layer) and a last conv of 10 heads (two groups of 5)."""
    from sgformer_b200 import engine as E
    monkeypatch.setattr(E, "next_seed", lambda: STEP_SEED)
    n, d, ei = GW._cora()
    h, c, layers, p, heads, out_heads = 64, 8, 3, 0.5, 16, 10
    plans = [_plan(precision, heads, h, False)] * (layers - 1) + [_plan(precision, out_heads, c, True)]
    assert all(len(pl.groups) == 2 and pl.cp == pl.c for pl in plans)
    ref = GW._ref_gat(d, h, c, layers, heads, out_heads, True, dropout=p)
    ours = GW._ours_gat(ref, d, h, c, layers, heads, out_heads, True, precision, dropout=p)
    gen = torch.Generator().manual_seed(29)
    x = torch.randn(n, d, generator=gen, dtype=torch.float64)
    lw = torch.randn(n, c, generator=gen, dtype=torch.float64) / math.sqrt(n)
    ours.train()
    xg = x.to(DEV, torch.float32).clone().requires_grad_(True)
    out = ours(GW.Data(xg, ei.to(DEV)))
    epoch = current_epoch()
    (out * lw.to(DEV)).sum().backward()
    got = dict(out_train=out.detach(), grads=dict({k: q.grad for k, q in ours.named_parameters()}, __x__=xg.grad),
               buffers={k: v for k, v in ours.state_dict().items() if "running" in k})
    r64 = _masked_oracle(ref, x, ei, lw, p, STEP_SEED, epoch, torch.float64, plans)
    r32 = _masked_oracle(ref, x, ei, lw, p, STEP_SEED, epoch, torch.float32, plans)
    for r in (got, r64, r32):
        r["out_eval"] = r["out_train"]
    problems = GW.compare_step(got, r64, r32, precision, layers, True, f"wide dropout step {precision}")
    assert not problems, "\n".join(problems)
    # with every group drawing group 0's masks (a head index local to a launch) the oracle is far away
    r_same = _masked_oracle(ref, x, ei, lw, p, STEP_SEED, epoch, torch.float64, plans, offset=False)
    assert (r_same["out_train"] - r64["out_train"]).abs().max() > 100 * GW.LOGIT_TOL["fp32"] * r64["out_train"].abs().max()


# ------------------------------------------------------------------------------------------------
# (d) bit identity, CUDA graph, state_dict
# ------------------------------------------------------------------------------------------------
def _train_step(model, x, ei, wgt):
    for q in model.parameters():
        q.grad = None
    xo = x.clone().requires_grad_(True)
    out = model(GW.Data(xo, ei))
    (out * wgt).sum().backward()
    return out.detach().clone(), [q.grad.clone() for q in model.parameters()], xo.grad.clone()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_wide_training_step_bit_identical(monkeypatch, precision):
    from sgformer_b200 import engine as E
    monkeypatch.setattr(E, "next_seed", lambda: 0x5EED)
    n, d, ei = GW._cora()
    ref = GW._ref_gat(d, 250, 7, 3, 4, 10, True, dropout=0.4)
    model = GW._ours_gat(ref, d, 250, 7, 3, 4, 10, True, precision, dropout=0.4)
    x, wgt, eid = torch.randn(n, d, device=DEV), torch.randn(n, 7, device=DEV), ei.to(DEV)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    runs = []
    for _ in range(2):
        model.load_state_dict(sd)
        runs.append(_train_step(model, x, eid, wgt) + ([v.clone() for k, v in model.state_dict().items() if "running" in k],))
    (o1, g1, x1, b1), (o2, g2, x2, b2) = runs
    assert torch.equal(o1, o2) and torch.equal(x1, x2)
    assert all(torch.equal(a, b) for a, b in zip(g1, g2)) and all(torch.equal(a, b) for a, b in zip(b1, b2))


def test_wide_cuda_graph_step_matches_eager(monkeypatch):
    """4 x 250 fp32 (two padded head groups per hidden layer) and a 10-head mean, all dropout streams on: the first replay of a
    captured step reproduces the eager step bit for bit."""
    from sgformer_b200 import engine as E
    from sgformer_b200 import kernels as K
    from sgformer_b200 import medium as M
    n, d, h = 1000, 32, 250
    ei = GW._base_edges(n=n, e=8000, hub=500).to(DEV)
    model = M.GAT(d, h, 7, num_layers=3, dropout=0.3, use_bn=True, heads=4, out_heads=10).to(DEV)
    x, wgt = torch.randn(n, d, device=DEV), torch.randn(n, 7, device=DEV)
    K.dropout_epoch()
    monkeypatch.setattr(E, "next_seed", lambda: 0x5EED)
    sd0 = {k: v.clone() for k, v in model.state_dict().items()}
    eager = _train_step(model, x, ei, wgt)
    bufs = [v.clone() for k, v in model.state_dict().items() if "running" in k]
    model.load_state_dict(sd0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _train_step(model, x, ei, wgt)
    torch.cuda.current_stream().wait_stream(s)
    model.load_state_dict(sd0)
    for q in model.parameters():
        q.grad = None
    xo = x.clone().requires_grad_(True)
    cg = torch.cuda.CUDAGraph()
    with torch.cuda.graph(cg):
        out = model(GW.Data(xo, ei))
        (out * wgt).sum().backward()
    model.load_state_dict(sd0)
    cg.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager[0])
    assert all(torch.equal(q.grad, g) for q, g in zip(model.parameters(), eager[1]))
    assert torch.equal(xo.grad, eager[2])
    assert all(torch.equal(a, b) for a, b in zip([v for k, v in model.state_dict().items() if "running" in k], bufs))


@pytest.mark.parametrize("precision,h", [("fp32", 250), ("bf16", 100)])
def test_reference_state_dict_round_trip_at_a_padded_width(precision, h):
    """The module keeps the reference's unpadded parameters and buffers: a trained state_dict loads into the oracle, which then
    computes the module's eval logits."""
    n, d, ei = GW._cora()
    ref = GW._ref_gat(d, h, 7, 3, 3, 2, True)
    ours = GW._ours_gat(ref, d, h, 7, 3, 3, 2, True, precision)
    x = torch.randn(n, d, device=DEV)
    eid = ei.to(DEV)
    ours.train()
    opt = torch.optim.SGD(ours.parameters(), lr=0.05)
    (ours(GW.Data(x, eid)) ** 2).mean().backward()
    opt.step()
    sd = ours.state_dict()
    assert {k: tuple(v.shape) for k, v in sd.items()} == {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    back = copy.deepcopy(ref).to(DEV, torch.float64)
    back.load_state_dict({k: v.double() if v.is_floating_point() else v for k, v in sd.items()})
    back.eval()
    ours.eval()
    with torch.no_grad():
        want = back(GW.Data(x.double(), eid))
        got = ours(GW.Data(x, eid))
    e = (got.double() - want).abs().max().item() / want.abs().max().item()
    assert e <= GW.LOGIT_TOL[precision], e


# ------------------------------------------------------------------------------------------------
# (e) one group: the direct kernel calls
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [("fp32", 8, 64, False), ("bf16", 8, 64, True), ("fp32", 2, 8, True), ("bf16", 7, 136, False)],
                         ids=W.shape_id)
def test_one_group_is_the_direct_kernel_calls(Kmod, shape):
    from sgformer_b200 import engine as E
    dtype, H, C, mean = shape
    lay = _plan(dtype, H, C, mean)
    assert lay.groups == [(0, H)] and lay.cp == C
    graph, n = GW._graph("base")
    rp_t, col_t = graph.transpose()
    xp, g, att_s, att_d, bias = GW._inputs(n, dtype, H, C, mean, 77)
    for p in (0.0, 0.5):
        z, parts = E._gat_conv_fwd(graph, xp, lay, att_s, att_d, bias, p, 0x5EED)
        dxp, das = E._gat_conv_bwd(graph, rp_t, col_t, dict(lay=lay, xp=xp, att=(att_s, att_d), parts=parts), g, p, 0x5EED)
        a_s, a_d = Kmod.gat_logits(xp, H, C, att_s, att_d)
        z0, lse0 = Kmod.gat_fwd(graph.rowptr, graph.col, xp, a_s, a_d, H, C, mean, bias, p, 0x5EED)
        dxp0, ds0, dd0 = Kmod.gat_bwd(graph.rowptr, graph.col, rp_t, col_t, xp, a_s, a_d, lse0, g, att_s, att_d, H, C, mean, p, 0x5EED)
        for a, b in ((z, z0), (parts[0][0], a_s), (parts[0][1], a_d), (parts[0][2], lse0), (dxp, dxp0), (das[0][0], ds0),
                     (das[0][1], dd0)):
            assert torch.equal(a, b)
