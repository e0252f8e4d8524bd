"""The GCNJK baseline on the device (`-m gpu`): the JK BatchNorm kernels (sgf_bn_fwd_jk, sgf_bn_bwd_*_jk) against fp64 of the
operands they read at every row geometry, with planted ties; the module and SGFormer(gnn=GCNJK) against the fp64 oracle with
dropout masks replayed; run-to-run bit identity; a CUDA-graph captured training step; and planted errors that the checks must
name."""
import pytest
import torch

from config_matrix import C_OWN, FLOOR, LOGIT_TOL
from dropout_mask import MaskReplayer, current_epoch, keep_mask, keep_scale
from oracle import gcnjk_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


class Data:
    def __init__(self, x, ei):
        self.graph = {"node_feat": x, "edge_index": ei, "num_nodes": x.shape[0]}


# ---- kernels -------------------------------------------------------------------------------------------------------------------
# Operands on a grid of 1/16 with power-of-two BatchNorm scales: every fp32 product and sum of the row pass is exact, so the fp64
# reference sees the values the kernel compares, and ties between layers are frequent (besides the planted ones).
def _q(shape, lo, hi, g):
    return torch.randint(lo, hi, shape, generator=g).double() / 16


def _layer_operands(n, h, g, bn):
    z = _q((n, h), -48, 48, g)
    p = dict(zb=_q((h,), -8, 8, g))
    if bn:
        p.update(mean=_q((h,), -8, 8, g), rstd=2.0 ** torch.randint(-1, 2, (h,), generator=g).double(),
                 gamma=2.0 ** torch.randint(-1, 1, (h,), generator=g).double(), beta=_q((h,), -8, 8, g))
    return z, p


def _act(z, p, bn):
    v = z + p["zb"]
    if bn:
        v = ((v - p["mean"]) * p["rstd"] * p["gamma"] + p["beta"]).clamp_min(0)
    return v


def _widths(prec):
    """One width per chunks-per-lane geometry (1..4 chunks of 16 bytes per lane, lanes per row 1..32), up to check_width's limit."""
    vn = 4 if prec == "fp32" else 8
    return [vn, 3 * vn, 32 * vn, 33 * vn, 65 * vn, 97 * vn, 128 * vn]


def _jk_forward_case(prec, h, n=613, nl=3, fwd=None):
    """Runs the JK forward of nl layers on quantised operands; returns (kernel m, kernel idx, fp64 max, fp64 first argmax, y of
    layer 0, the fp64 activations)."""
    from sgformer_b200 import kernels as K
    fwd = fwd or K.bn_fwd_jk
    dt = torch.float32 if prec == "fp32" else torch.bfloat16
    g = torch.Generator().manual_seed(1000 + h)
    m = K.alloc_act(n, h, dt, DEV)
    idx = torch.empty((n, m.stride(0)), dtype=torch.uint8, device=DEV)
    acts, y0 = [], None
    for l in range(nl):
        bn = l < nl - 1
        z, p = _layer_operands(n, h, g, bn)
        if l == 1:                                   # planted ties: layer 1 repeats layer 0 on rows 0..19
            z[:20] = z0[:20]
            p = dict(p0)
        if bn:
            z[20:30] = -100.0                         # planted all-zero ReLU rows
        if l == 0:
            z0, p0 = z.clone(), dict(p)
        a = _act(z, p, bn)
        acts.append(a.to(dt).double())               # compared as stored
        zd = K.alloc_act(n, h, dt, DEV)
        zd.copy_(z.to(dt))
        f = {k: v.float().to(DEV) for k, v in p.items()}
        y = fwd(zd, f.get("mean"), f.get("rstd"), f.get("gamma"), f.get("beta"), f["zb"], bn, bn, 0.5 if bn else 0.0, 77 + l,
                l == 0, "max", m, idx, l)
        if l == 0:
            y0 = y
    st = torch.stack(acts, -1)
    ref_m, ref_i = st.max(-1)
    return m.double().cpu(), idx[:, :h].long().cpu(), ref_m, ref_i, y0, acts


def _kernel_problems(prec, h, fwd=None):
    m, idx, ref_m, ref_i, y0, acts = _jk_forward_case(prec, h, fwd=fwd)
    probs = []
    if not torch.equal(m, ref_m):
        probs.append(f"jk_max: {(m != ref_m).sum().item()} elements differ")
    if not torch.equal(idx, ref_i):
        probs.append(f"jk_idx: {(idx != ref_i).sum().item()} elements differ")
    mask = torch.from_numpy(keep_mask(77, acts[0].shape[0], h, 0.5, current_epoch()))
    ref_y = acts[0] * mask.double() * keep_scale(0.5)
    if not torch.allclose(y0.double().cpu(), ref_y, rtol=0, atol=0 if prec == "fp32" else 0.02):
        probs.append("y: dropout output differs")
    return probs


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_jk_max_forward_against_fp64(prec):
    for h in _widths(prec):
        assert _kernel_problems(prec, h) == [], h


def test_jk_max_ties_pick_the_lowest_layer():
    m, idx, ref_m, ref_i, _, acts = _jk_forward_case("fp32", 64)
    tie01 = (acts[0][:20] == acts[1][:20]) & (acts[0][:20] > 0)
    assert tie01.any()
    tie01 &= acts[2][:20] <= acts[0][:20]
    assert tie01.any() and (idx[:20][tie01] == 0).all()
    assert (idx[20:30] == torch.where(acts[2][20:30] > 0, 2, 0)).all()    # zero rows: layer 0 unless the last layer is positive


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_jk_cat_forward_writes_the_pre_dropout_block(prec):
    from sgformer_b200 import kernels as K
    dt = torch.float32 if prec == "fp32" else torch.bfloat16
    for h in _widths(prec):
        n, nl = 301, 3
        g = torch.Generator().manual_seed(h)
        buf = K.alloc_act(n, nl * h, dt, DEV)
        buf.fill_(7.0)
        z, p = _layer_operands(n, h, g, True)
        zd = K.alloc_act(n, h, dt, DEV)
        zd.copy_(z.to(dt))
        f = {k: v.float().to(DEV) for k, v in p.items()}
        y = K.bn_fwd_jk(zd, f["mean"], f["rstd"], f["gamma"], f["beta"], f["zb"], True, True, 0.5, 5, True, "cat",
                        buf[:, h:2 * h], None, 1)
        a = _act(z, p, True).to(dt).double()
        assert torch.equal(buf[:, h:2 * h].double().cpu(), a), h
        assert (buf[:, :h] == 7).all() and (buf[:, 2 * h:] == 7).all(), h
        mask = torch.from_numpy(keep_mask(5, n, h, 0.5, current_epoch())).double()
        torch.testing.assert_close(y.double().cpu(), (a * mask * keep_scale(0.5)).to(dt).double(), rtol=0, atol=0)


def _bwd_reference(dy, z, p, bn, training, drop_seed, pdrop, add):
    """fp64 of the contract: g = dropout(dy) + add, * relu', BatchNorm backward -> (dz, sums, colsum)."""
    n, h = z.shape
    g = torch.zeros_like(z) if dy is None else dy * torch.from_numpy(keep_mask(drop_seed, n, h, pdrop, current_epoch())).double() * \
        (keep_scale(pdrop) if pdrop > 0 else 1.0)
    g = g + add
    v = z + p["zb"]
    if not bn:
        return g, None, g.sum(0)
    xh = (v - p["mean"]) * p["rstd"]
    g = g * ((xh * p["gamma"] + p["beta"]) > 0)
    sums = torch.cat([g.sum(0), (g * xh).sum(0)])
    d = p["gamma"] * p["rstd"] * ((g - sums[:h] / n - xh * sums[h:] / n) if training else g)
    return d, sums, d.sum(0)


@pytest.mark.parametrize("mode", ["max", "cat"])
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_jk_backward_addend_against_fp64(prec, mode):
    from sgformer_b200 import kernels as K
    dt = torch.float32 if prec == "fp32" else torch.bfloat16
    tol = 1e-5 if prec == "fp32" else 2e-2
    for h in _widths(prec):
        n, nl, l = 517, 3, 1
        g = torch.Generator().manual_seed(3 * h)
        z, p = _layer_operands(n, h, g, True)
        p["mean"] = (z + p["zb"]).mean(0)              # batch statistics of z, as training sees them
        p["rstd"] = ((z + p["zb"]).var(0, unbiased=False) + 1e-5).rsqrt()
        dy = torch.randn(n, h, generator=g, dtype=torch.float64).to(dt).double()
        gj = torch.randn(n, h * (nl if mode == "cat" else 1), generator=g, dtype=torch.float64).to(dt).double()
        idx = torch.randint(0, nl, (n, h), generator=g, dtype=torch.uint8)
        idx[:25] = l                                   # rows routed to this layer only
        zd, dyd = K.alloc_act(n, h, dt, DEV), K.alloc_act(n, h, dt, DEV)
        zd.copy_(z.to(dt))
        dyd.copy_(dy.to(dt))
        gjd = K.alloc_act(n, gj.shape[1], dt, DEV)
        gjd.copy_(gj.to(dt))
        idxd = torch.zeros((n, gjd.stride(0)), dtype=torch.uint8, device=DEV)
        idxd[:, :h] = idx.to(DEV)
        blk = gjd if mode == "max" else gjd[:, l * h:(l + 1) * h]
        add = gj * (idx == l) if mode == "max" else gj[:, l * h:(l + 1) * h]
        f = {k: v.float().to(DEV) for k, v in p.items()}
        for training in (True, False):
            dz, sums, colsum = K.bn_bwd_jk(dyd, zd, f["mean"], f["rstd"], f["gamma"], f["beta"], f["zb"], True, True, training, 0.5,
                                          99, mode, blk, idxd if mode == "max" else None, l, want_dz_colsum=True)
            rd, rs, rc = _bwd_reference(dy, z, p, True, training, 99, 0.5, add)
            for name, a, b in (("dz", dz, rd), ("sums", sums, rs), ("colsum", colsum, rc)):
                e = (a.double().cpu() - b).abs().max().item()
                assert e <= tol * (1 + b.abs().max().item()), (h, training, name, e)
        # the last conv: no BatchNorm, no ReLU, no dy: dz is the addend and its column sum is the bias gradient
        dz, _, colsum = K.bn_bwd_jk(None, zd, None, None, None, None, f["zb"], False, False, True, 0.0, 0, mode, blk,
                                    idxd if mode == "max" else None, l, want_dz_colsum=True)
        assert torch.equal(dz.double().cpu(), add), h
        torch.testing.assert_close(colsum.double().cpu(), add.sum(0), rtol=1e-5, atol=1e-4)


# ---- modules against the fp64 oracle -----------------------------------------------------------------------------------------
def _graph(n, e, seed, hub=0):
    """Directed random edges with duplicates, isolated nodes (the last 7), existing self loops, and `hub` in-edges into node 3."""
    g = torch.Generator().manual_seed(seed)
    hi = n - 7
    ei = torch.stack([torch.randint(0, hi, (e,), generator=g), torch.randint(0, hi, (e,), generator=g)])
    ei = torch.cat([ei, ei[:, :e // 10], torch.stack([torch.arange(0, hi, 9)] * 2)], 1)
    if hub:
        ei = torch.cat([ei, torch.stack([torch.randint(0, hi, (hub,), generator=g), torch.full((hub,), 3)])], 1)
    return ei


def _cora():
    g = torch.Generator().manual_seed(5)
    n, d = 2708, 1433
    return (torch.rand(n, d, generator=g) < 0.013).float(), _graph(n, 5278, 6), 64, 7


def _hub():
    n = 2 * torch.cuda.get_device_properties(0).multi_processor_count * 128 + 7
    g = torch.Generator().manual_seed(8)
    return torch.randn(n, 48, generator=g), _graph(n, 6 * n, 9, hub=1500), 64, 10


def _cls(name, nl):
    """FLOOR class: the hidden convs' weights sit behind a BatchNorm ('bn_weight'), the last conv's and final_project's do not."""
    if name == "x":
        return "grad_x"
    if name.startswith("bns.") or name.endswith("bias"):
        return "affine"
    return "bn_weight" if any(name == f"convs.{i}.lin.weight" for i in range(nl - 1)) else "weight"


def check(got, ref64, ref32, prec):
    """Problems (one line each, starting with the tensor's name): logits by LOGIT_TOL, gradients and BatchNorm buffers by
    max(C_OWN * the fp32 oracle's own error, FLOOR of the tensor's class)."""
    probs = []
    nl = sum(1 for k in ref64["grads"] if k.endswith(".lin.weight")) or 4
    o, r = got["out"].double().cpu(), ref64["out"]
    tol = LOGIT_TOL[prec]
    err = (o - r).abs().max().item()
    if not err <= tol * (1 + r.abs().max().item()):
        probs.append(f"out: max err {err:.3e}")
    for k, g64 in ref64["grads"].items():
        g = got["grads"].get(k)
        if g is None:
            probs.append(f"{k}: missing")
            continue
        den = max(g64.norm().item(), 1e-3 * ref64["grads"].get(k.replace("bias", "lin.weight"), g64).norm().item(), 1e-30)
        e = (g.double().cpu() - g64).norm().item() / den
        own = (ref32["grads"][k].double() - g64).norm().item() / den
        bound = max(C_OWN[prec] * own, FLOOR[_cls(k, nl)][prec])
        if not e <= bound:
            probs.append(f"{k}: rel err {e:.3e} > {bound:.3e}")
    for k, b64 in ref64["stats"].items():
        if k.endswith("num_batches_tracked"):
            if int(got["stats"][k]) != int(b64):
                probs.append(f"{k}: {int(got['stats'][k])} vs {int(b64)}")
            continue
        e = (got["stats"][k].double().cpu() - b64).norm().item() / max(b64.norm().item(), 1e-30)
        if not e <= FLOOR["affine"][prec]:
            probs.append(f"{k}: rel err {e:.3e}")
    return probs


def _record_masks(monkeypatch):
    """Records (p, mask) of every dropout the JK forward draws, in call order."""
    from sgformer_b200 import kernels as K
    calls = []
    real = K.bn_fwd_jk

    def wrapped(z, mean, rstd, gamma, beta, zbias, use_bn, use_relu, p, seed, *a, **kw):
        if p > 0.0:
            calls.append((p, keep_mask(seed, z.shape[0], z.shape[1], p, current_epoch())))
        return real(z, mean, rstd, gamma, beta, zbias, use_bn, use_relu, p, seed, *a, **kw)
    monkeypatch.setattr(K, "bn_fwd_jk", wrapped)
    return calls


def _oracle(sd, x, ei, nl, jk, training, p, masks, dtype, monkeypatch):
    sdd = {k: (v.to(dtype).clone().requires_grad_(training) if v.is_floating_point() and "running" not in k else v.clone())
           for k, v in sd.items()}
    xd = x.to(dtype).clone().requires_grad_(training)
    rep = MaskReplayer(masks)
    monkeypatch.setattr(O, "_dropout", rep)
    stats = {}
    out = O.gcnjk(xd, ei, sdd, nl, jk, training, p, stats_out=stats)
    res = dict(out=out.detach().double(), grads={}, stats={k: v.double() for k, v in stats.items()})
    if training:
        rep.finish()
        (out * _WGT[out.shape].to(dtype)).sum().backward()
        res["grads"] = {k: v.grad.double() for k, v in sdd.items() if isinstance(v, torch.Tensor) and v.grad is not None}
        res["grads"]["x"] = xd.grad.double()
    return res


_WGT = {}


def _run_module(case, nl, jk, training, p, prec, monkeypatch, plant=None):
    from sgformer_b200 import medium as M
    x, ei, h, c = case
    torch.manual_seed(nl * 10 + len(jk))
    m = M.GCNJK(x.shape[1], h, c, num_layers=nl, dropout=p, jk_type=jk)
    with torch.no_grad():
        for k, v in m.named_parameters():
            if k.endswith("bias") or k.startswith("bns."):
                v.add_(0.1 * torch.randn_like(v))
        for k, b in m.named_buffers():
            if k.endswith("running_mean"):
                b.normal_(0, 0.1)
            elif k.endswith("running_var"):
                b.uniform_(0.5, 1.5)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    _WGT.setdefault((x.shape[0], c), torch.randn(x.shape[0], c, generator=torch.Generator().manual_seed(3)))
    m = m.to(DEV).set_precision(prec).train(training)
    masks = _record_masks(monkeypatch)
    if plant:
        plant(monkeypatch)
    xo = x.to(DEV).clone().requires_grad_(training)
    out = m(Data(xo, ei.to(DEV)))
    got = dict(out=out.detach(), grads={}, stats={k: v for k, v in m.state_dict().items() if "running" in k or "num_batches" in k})
    if training:
        (out * _WGT[out.shape].to(DEV)).sum().backward()
        got["grads"] = {k: v.grad for k, v in m.named_parameters()}
        got["grads"]["x"] = xo.grad
    monkeypatch.undo()
    ref64 = _oracle(sd, x, ei, len(m.convs), jk, training, p, masks, torch.float64, monkeypatch)
    ref32 = _oracle(sd, x, ei, len(m.convs), jk, training, p, masks, torch.float32, monkeypatch)
    monkeypatch.undo()
    if not training:
        ref64["stats"] = {}
    return got, ref64, ref32



@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("jk", ["max", "cat"])
@pytest.mark.parametrize("nl", [2, 3, 4])
def test_gcnjk_cora_against_fp64_oracle(nl, jk, prec, monkeypatch):
    case = _cora()
    for training, p in ((False, 0.0), (True, 0.0), (True, 0.5)):
        got, r64, r32 = _run_module(case, nl, jk, training, p, prec, monkeypatch)
        assert check(got, r64, r32, prec) == [], (training, p)


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("jk", ["max", "cat"])
def test_gcnjk_hub_graph_against_fp64_oracle(jk, prec, monkeypatch):
    case = _hub()
    got, r64, r32 = _run_module(case, 3, jk, True, 0.5, prec, monkeypatch)
    assert check(got, r64, r32, prec) == []


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("aggregate,jk,nl", [("add", "max", 3), ("cat", "cat", 2), ("add", "cat", 3), ("cat", "max", 4)])
def test_sgformer_with_gcnjk_against_fp64_oracle(aggregate, jk, nl, prec):
    from sgformer_b200 import medium as M
    x, ei, h, c = _cora()
    torch.manual_seed(nl)
    m = M.SGFormer(x.shape[1], h, c, num_layers=1, dropout=0.0, graph_weight=0.7, aggregate=aggregate,
                   gnn=M.GCNJK(x.shape[1], h, h, num_layers=nl, dropout=0.0, jk_type=jk))
    m.train()
    cfg = m._cfg(len(m.gnn.convs), 0.0, True, "gcnjk", jk)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    wgt = torch.randn(x.shape[0], c, generator=torch.Generator().manual_seed(4))
    refs = {}
    for dt in (torch.float64, torch.float32):
        sdd = {k: (v.to(dt).clone().requires_grad_(True) if v.is_floating_point() and "running" not in k else v) for k, v in sd.items()}
        out = O.sgformer_gcnjk(cfg, sdd, x.to(dt), ei, training=True)
        (out * wgt.to(dt)).sum().backward()
        refs[dt] = dict(out=out.detach().double(), grads={k: v.grad.double() for k, v in sdd.items()
                                                           if isinstance(v, torch.Tensor) and v.grad is not None}, stats={})
    m = m.to(DEV).set_precision(prec)
    out = m(Data(x.to(DEV), ei.to(DEV)))
    (out * wgt.to(DEV)).sum().backward()
    got = dict(out=out.detach(), grads={k: v.grad for k, v in m.named_parameters()}, stats={})
    assert check(got, refs[torch.float64], refs[torch.float32], prec) == []


# ---- determinism and capture ---------------------------------------------------------------------------------------------------
def _train_step(model, x, ei, wgt):
    for p_ in model.parameters():
        p_.grad = None
    xo = x.clone().requires_grad_(True)
    out = model(Data(xo, ei))
    (out * wgt).sum().backward()
    return out.detach().clone(), [p_.grad.clone() for p_ in model.parameters()], xo.grad.clone()


@pytest.mark.parametrize("jk", ["max", "cat"])
def test_gcnjk_training_step_bit_identical(jk, monkeypatch):
    from sgformer_b200 import engine as E
    from sgformer_b200 import medium as M
    monkeypatch.setattr(E, "next_seed", lambda: 0x5EED)
    x, ei, h, c = _hub()
    x, ei = x.to(DEV), ei.to(DEV)
    model = M.GCNJK(x.shape[1], h, c, num_layers=3, dropout=0.5, jk_type=jk).to(DEV)
    wgt = torch.randn(x.shape[0], c, device=DEV)
    runs = []
    for _ in range(2):
        sd = {k: v.clone() for k, v in model.state_dict().items()}
        runs.append(_train_step(model, x, ei, wgt))
        model.load_state_dict(sd)
    (o1, g1, x1), (o2, g2, x2) = runs
    assert torch.equal(o1, o2) and torch.equal(x1, x2)
    assert all(torch.equal(a, b) for a, b in zip(g1, g2))


@pytest.mark.parametrize("jk", ["max", "cat"])
def test_gcnjk_cuda_graph_step_matches_eager(jk, monkeypatch):
    from sgformer_b200 import engine as E
    from sgformer_b200 import kernels as K
    from sgformer_b200 import medium as M
    x, ei, h, c = _cora()
    x, ei = x.to(DEV), ei.to(DEV)
    model = M.GCNJK(x.shape[1], h, c, num_layers=3, dropout=0.5, jk_type=jk).to(DEV)
    wgt = torch.randn(x.shape[0], c, device=DEV)
    K.dropout_epoch()
    monkeypatch.setattr(E, "next_seed", lambda: 0x5EED)
    sd0 = {k: v.clone() for k, v in model.state_dict().items()}
    eager = _train_step(model, x, ei, wgt)
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


# ---- planted errors: the checks above must name the tensor they corrupt ----------------------------------------------------------
def _plant_last_index_ties(z, mean, rstd, gamma, beta, zbias, use_bn, use_relu, p, seed, want_y, mode, jk, jk_idx, layer):
    """The real kernel, then the tie rule flipped: where layer l equals the running max it takes the index."""
    from sgformer_b200 import kernels as K
    prev = jk.clone()
    y = K.bn_fwd_jk(z, mean, rstd, gamma, beta, zbias, use_bn, use_relu, p, seed, want_y, mode, jk, jk_idx, layer)
    if layer > 0:
        v = z.float() + zbias
        if use_bn:
            v = ((v - mean) * rstd * gamma + beta).clamp_min(0)
        h = z.shape[1]
        tie = v.to(z.dtype) == prev
        jk_idx[:, :h][tie] = layer
    return y


def test_planted_last_index_ties_are_reported():
    assert any(s.startswith("jk_idx") for s in _kernel_problems("fp32", 64, fwd=_plant_last_index_ties))


def _plant_routed_to_next_layer(monkeypatch):
    from sgformer_b200 import kernels as K
    real = K.bn_bwd_jk
    monkeypatch.setattr(K, "bn_bwd_jk", lambda *a, **kw: real(*a[:15], a[15] - 1 if a[15] > 0 else 255, **kw))


def _plant_cat_block_off_by_one(monkeypatch):
    """Layer l writes its activation into the concatenation's block l + 1 (mod L)."""
    from sgformer_b200 import kernels as K
    real = K.bn_fwd_jk

    def wrapped(z, *a):
        a = list(a)
        if a[10] == "cat":
            full, h, layer = a[11]._base, z.shape[1], a[13]
            k = (layer + 1) % (full.shape[1] // h)
            a[11] = full[:, k * h:(k + 1) * h]
        return real(z, *a)
    monkeypatch.setattr(K, "bn_fwd_jk", wrapped)


def _plant_colsum_without_addend(monkeypatch):
    from sgformer_b200 import kernels as K
    real = K.bn_bwd_jk

    def wrapped(dy, *a, **kw):
        dz, sums, colsum = real(dy, *a, **kw)
        if dy is None and colsum is not None:        # the last conv: its dz is only the JK addend
            colsum.zero_()
        return dz, sums, colsum
    monkeypatch.setattr(K, "bn_bwd_jk", wrapped)


@pytest.mark.parametrize("plant,jk,expect", [(_plant_routed_to_next_layer, "max", "convs.0.lin.weight"),
                                             (_plant_cat_block_off_by_one, "cat", "out"),
                                             (_plant_colsum_without_addend, "max", "convs.2.bias")])
def test_planted_errors_are_reported(plant, jk, expect, monkeypatch):
    got, r64, r32 = _run_module(_cora(), 3, jk, True, 0.0, "fp32", monkeypatch, plant=plant)
    probs = check(got, r64, r32, "fp32")
    assert any(s.startswith(expect + ":") for s in probs), probs
