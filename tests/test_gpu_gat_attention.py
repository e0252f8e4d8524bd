"""The scaled mode of the fused attention kernels (csrc/attn_softmax.cu) and SGFormerGAT, the GAT-attention ablation, on the
device.  ("GAT attention" is oursGAT.py's scaled dot-product attention; the GAT backbone is tested in test_gpu_gat*.py.)

The references are fp64: autograd through oracle/gat_attention_oracle.py on the operands the kernels read for the kernels, and
tests/golden/sgformer_gat_attention.pt (made from the unmodified oursGAT.py) for the modules.  Errors are max |x - ref| / max |ref|
per output: fp32 within 1e-4, bf16 within 1e-2.  Scores reach |s| ~ 200, where exp overflows fp32 unless each pair's maximum over
the heads is subtracted.  With one head every weight is exactly 1 and dq, dk exactly zero."""
import os

import pytest
import torch

from oracle import gat_attention_oracle as O
from sgformer_b200 import ablation_gat, medium
from sgformer_b200 import engine as E
from sgformer_b200 import kernels as K
from sgformer_b200.optim import Adam

pytestmark = pytest.mark.gpu
TOL = {"fp32": 1e-4, "bf16": 1e-2}
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sgformer_gat_attention.pt")


def _check(name, x, ref, tol, scale, exact_zero=True):
    """scale: the largest magnitude among the outputs of the same call; a reference below 1e-12 of it is an exact zero (one head),
    which the kernels return exactly.  exact_zero=False (the GCN conv bias ahead of a train-mode BatchNorm): within tol * scale."""
    assert torch.isfinite(x).all(), f"{name}: non-finite values"
    rmax = ref.abs().max().item()
    if rmax <= 1e-12 * scale:
        if exact_zero:
            assert torch.count_nonzero(x) == 0, f"{name}: the exact value is zero, got max {x.abs().max().item():.3g}"
        else:
            assert x.abs().max().item() <= tol * scale, f"{name}: the exact value is zero, got max {x.abs().max().item():.3g}"
        return
    err = ((x.double() - ref).abs().max() / rmax).item()
    assert err <= tol, f"{name}: relative error {err:.3g}"


def _kernel_case(n, heads, dk, d, prec_name, smax, seed=0, per_head_g=False, accumulate=False):
    """q, k in the kernels' layout (each head's dk columns padded with zeros to 16 bytes), scaled so that max |s| = smax.
    per_head_g: a gradient block per head (ScaledAttentionFn's) instead of the head mean's shared one.  accumulate: dv starts
    from random values and the backward adds to them."""
    prec = E.precision(prec_name)
    dt = prec.act_dtype
    mp = E.gat_attn_pad(dk, prec)
    g = torch.Generator(device="cuda").manual_seed(seed)
    q0 = torch.randn(n, heads, dk, device="cuda", generator=g, dtype=torch.float64) + 0.3
    k0 = torch.randn(n, heads, dk, device="cuda", generator=g, dtype=torch.float64) - 0.2
    scale = E.gat_attn_scale(dk)
    s0 = (scale * torch.einsum("nhm,lhm->nlh", q0, k0)).abs().max().item()
    q0 = q0 * (smax / s0)
    q, k = (torch.zeros(n, heads, mp, device="cuda", dtype=dt) for _ in range(2))
    q[:, :, :dk], k[:, :, :dk] = q0.to(dt), k0.to(dt)
    q, k = q.reshape(n, heads * mp), k.reshape(n, heads * mp)
    v = torch.randn(n, heads * d, device="cuda", generator=g).to(dt)
    gr = torch.randn(n, (heads if per_head_g else 1) * d, device="cuda", generator=g).to(dt)     # shared: the head mean's
    o = K.attn_scaled_fwd(q, k, v, heads, scale)
    dq, dkk = K.alloc_act(n, heads * mp, dt, "cuda"), K.alloc_act(n, heads * mp, dt, "cuda")
    dv = K.alloc_act(n, heads * d, dt, "cuda")
    if accumulate:
        dv.copy_(torch.randn(n, heads * d, device="cuda", generator=g) * 2)
    dv0 = dv.double() if accumulate else 0.0
    K.attn_scaled_bwd(q, k, v, heads, scale, gr, 1.0 if per_head_g else 1.0 / heads, dq, dkk, dv, dv_accumulate=accumulate)
    qr, kr = (t.double().reshape(n, heads, mp)[:, :, :dk].clone().requires_grad_() for t in (q, k))
    vr = v.double().reshape(n, heads, d).requires_grad_()
    ref = O.gat_attention(qr, kr, vr)
    gd = gr.double().reshape(n, -1, d).expand(n, heads, d)
    ref.backward(gd if per_head_g else gd / heads)
    torch.cuda.synchronize()
    unpad = lambda t: t.reshape(n, heads, mp)[:, :, :dk].reshape(n, -1)      # noqa: E731
    pads = lambda t: t.reshape(n, heads, mp)[:, :, dk:]                       # noqa: E731
    assert torch.count_nonzero(pads(dq)) == 0 and torch.count_nonzero(pads(dkk)) == 0
    return {"o": (o, ref.detach().reshape(n, -1)), "dq": (unpad(dq), qr.grad.reshape(n, -1)),
            "dk": (unpad(dkk), kr.grad.reshape(n, -1)), "dv": (dv, dv0 + vr.grad.reshape(n, -1))}


def _check_case(res, tol, heads):
    """With one head dq and dk are exactly zero; with several, a saturated softmax over the heads (|s| ~ 200) leaves a gradient far
    below rounding of the largest output, which is held to tol of that output."""
    scale = max(ref.abs().max().item() for _, ref in res.values())
    for name, (x, ref) in res.items():
        _check(name, x, ref, tol, scale, exact_zero=heads == 1)


# (heads, dk, value width per head, precisions): padded dk 5 and 21, 8 heads in bf16 (8 x 64 bf16 values fill 1 KB), 12 heads
GEOMS = [(1, 8, 32, ("fp32", "bf16")), (2, 64, 64, ("fp32", "bf16")), (3, 5, 16, ("fp32", "bf16")), (4, 21, 32, ("fp32", "bf16")),
         (8, 16, 64, ("bf16",)), (12, 4, 16, ("fp32", "bf16"))]
KCASES = [(h, dk, d, p) for h, dk, d, ps in GEOMS for p in ps]


def _tol(prec, smax):
    """fp32 products are bf16x3 (hi.hi + hi.lo + lo.hi): each carries about 2^-16 of its magnitude, so a score's error grows with
    |s|, and the softmax over the heads passes a score error d on as a relative weight error of about d.  Up to |s| ~ 25 that
    stays within 1e-4; beyond, the fp32 bound grows with |s| (8e-4 at 200).  bf16 operands are exact in the reference."""
    return TOL[prec] * max(1.0, smax / 25.0) if prec == "fp32" else TOL[prec]


@pytest.mark.parametrize("smax", [3.0, 200.0])
@pytest.mark.parametrize("heads,dk,d,prec", KCASES)
@pytest.mark.parametrize("n", [1, 63, 64, 65, 300])
def test_kernels_vs_fp64(n, heads, dk, d, prec, smax):
    _check_case(_kernel_case(n, heads, dk, d, prec, smax), _tol(prec, smax), heads)


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("smax", [3.0, 200.0])
def test_kernels_vs_fp64_many_tiles(prec, smax):
    n = 2 * torch.cuda.get_device_properties(0).multi_processor_count * 64 + 7
    _check_case(_kernel_case(n, 2, 32, 64, prec, smax, seed=1), _tol(prec, smax), 2)


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_one_head_weights_are_exactly_one(prec):
    """P = 1: with v = 1 every output is exactly the key count; dq and dk are exactly zero (checked in test_kernels_vs_fp64)."""
    n, dt = 300, E.precision(prec).act_dtype
    q = (100 * torch.randn(n, 8, device="cuda")).to(dt)
    v = torch.ones(n, 16, device="cuda", dtype=dt)
    o = K.attn_scaled_fwd(q, q, v, 1, E.gat_attn_scale(8))
    assert torch.equal(o.float(), torch.full_like(o.float(), float(n)))


def test_row_width_limit_is_a_clear_error():
    m = ablation_gat.SGFormerGAT(8, 64, 3, num_layers=1, num_heads=5, use_graph=False).cuda()     # 5 x 64 fp32 values > 1 KB
    data = _Data(torch.randn(10, 8, device="cuda"), torch.zeros(2, 0, dtype=torch.long, device="cuda"))
    with pytest.raises(ValueError, match="at most 1024 bytes"):
        m(data)


class _Data:
    def __init__(self, x, ei):
        self.graph = {"node_feat": x, "edge_index": ei}


GD = None


def _golden():
    global GD
    if GD is None:
        GD = torch.load(GOLDEN, weights_only=False)
    return GD


def _native_for(cfg, d, c):
    h = cfg["hidden"]
    gnn = medium.GCN(d, h, h, num_layers=2, dropout=0.0, use_bn=True) if cfg["use_graph"] else None
    return ablation_gat.SGFormerGAT(d, h, c, num_layers=2, num_heads=cfg["heads"], alpha=0.5, dropout=0.0, use_bn=cfg["use_bn"],
                                    use_residual=cfg["use_residual"], use_weight=cfg["use_weight"], use_graph=cfg["use_graph"],
                                    graph_weight=0.8, gnn=gnn, aggregate=cfg["aggregate"])


def _backward_rank(name, layers=2):
    """Order of the backward: head and GNN, then the TransConv layers from the last (bns.i+1, convs.i, ...), then the stem."""
    if not name.startswith("trans_conv."):
        return 0 if name.startswith("fc.") else 1
    kind, i = name.split(".")[1], int(name.split(".")[2])
    if kind == "bns":
        return 2 + 2 * (layers - i)
    return 3 + 2 * (layers - 1 - i) if kind == "convs" else 3 + 2 * layers


def _module_check(case, prec):
    gd = _golden()
    rec = gd["cases"][case]
    sd = rec["state_dict"]
    x, ei = gd["x"].cuda(), gd["edge_index"].cuda()
    m = _native_for(rec["config"], x.shape[1], sd["fc.weight"].shape[0]).cuda().set_precision(prec)
    m.load_state_dict(sd)                  # the reference's own checkpoint
    ref = rec["fp64"]
    # bf16: two attention layers of bf16 activations at h = 8 leave logits about 1e-2 off; 2e-2 for the module
    tol = 2e-2 if prec == "bf16" else _tol(prec, rec.get("max_abs_score", 1.0))
    m.eval()
    with torch.no_grad():
        _check("eval_logits", m(_Data(x, ei)).float(), ref["eval_logits"].cuda(), tol, 1.0)
    m.train()
    xg = x.clone().requires_grad_()
    out = m(_Data(xg, ei))
    _check("train_logits", out.detach().float(), ref["train_logits"].cuda(), tol, 1.0)
    (out * rec["wout"].cuda()).sum().backward()
    scale = max(g.abs().max().item() for g in ref["grads"].values())
    assert sorted(k for k, p in m.named_parameters() if p.grad is None) == sorted(ref["none_grads"])
    for name, p in sorted(m.named_parameters(), key=lambda kv: _backward_rank(kv[0])):      # where a backward error enters first
        if p.grad is None:
            continue
        if prec == "bf16":      # bf16: every gradient within tol of the model's largest gradient
            err = (p.grad.double() - ref["grads"][name].cuda()).abs().max().item() / scale
            assert err <= tol, f"{name}: error {err:.3g} of the largest gradient"
        else:
            _check(name, p.grad, ref["grads"][name].cuda(), tol, scale, exact_zero=False)
    _check("grad_x", xg.grad, ref["grad_x"].cuda(), tol, scale)


FX_CASES = ["h1", "h2_noweight", "h4_nores", "h2_noln", "h3_dk5", "h2_gcn_add", "h4_gcn_cat", "h2_large_scores"]


@pytest.mark.parametrize("case", FX_CASES)
def test_module_vs_reference_fixture_fp32(case):
    _module_check(case, "fp32")


# bf16 activations round q to 8 bits: at |s| ~ 120 (h2_large_scores) that moves a score by ~0.5, which no bf16 computation of
# that model can meet within 1e-2; that case runs in fp32 only
@pytest.mark.parametrize("case", [c for c in FX_CASES if c != "h2_large_scores"])
def test_module_vs_reference_fixture_bf16(case):
    _module_check(case, "bf16")


def test_adam_leaves_unused_layer_weights_untouched():
    gd = _golden()
    rec = gd["cases"]["h2_gcn_add"]
    x, ei = gd["x"].cuda(), gd["edge_index"].cuda()
    m = _native_for(rec["config"], x.shape[1], rec["state_dict"]["fc.weight"].shape[0]).cuda()
    m.load_state_dict(rec["state_dict"])
    opt = Adam([{"params": m.params1, "weight_decay": 0.05}, {"params": m.params2, "weight_decay": 0.01}], lr=0.01)
    unused = {k: p.detach().clone() for k, p in m.named_parameters() if k.startswith("trans_conv.convs.") and k.split(".")[3] in ("Wq", "Wk", "Wv")}
    assert len(unused) == 12
    opt.zero_grad()
    (m(_Data(x, ei)) * rec["wout"].cuda()).sum().backward()
    opt.step()
    torch.cuda.synchronize()
    params = dict(m.named_parameters())
    for k, v in unused.items():
        assert params[k].grad is None and torch.equal(params[k].detach(), v), k
    assert not torch.equal(params["trans_conv.convs.0.attention.attention.Wq.weight"].detach(),
                           rec["state_dict"]["trans_conv.convs.0.attention.attention.Wq.weight"].cuda())


def _model(heads=2, use_weight=True, d=24, h=32, c=5):
    return ablation_gat.SGFormerGAT(d, h, c, num_layers=2, num_heads=heads, alpha=0.5, dropout=0.5, use_weight=use_weight,
                                    use_graph=False)


def _train_step(m, x, ei, wgt):
    m.zero_grad(set_to_none=True)
    xg = x.clone().requires_grad_()
    out = m(_Data(xg, ei))
    (out * wgt).sum().backward()
    return out.detach().clone(), [p.grad.clone() for p in m.parameters() if p.grad is not None], xg.grad.clone()


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("use_weight", [True, False])
def test_training_step_bit_identical(prec, use_weight, monkeypatch):
    torch.manual_seed(1)
    m = _model(heads=4, use_weight=use_weight).cuda().set_precision(prec)
    x = torch.randn(1000, 24, device="cuda")
    ei = torch.zeros(2, 0, dtype=torch.long, device="cuda")
    wgt = torch.randn(1000, 5, device="cuda")
    monkeypatch.setattr(E, "next_seed", lambda: 0x5EED)
    a, b = _train_step(m, x, ei, wgt), _train_step(m, x, ei, wgt)
    assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2])
    assert len(a[1]) == len(b[1]) and all(torch.equal(p, q) for p, q in zip(a[1], b[1]))


def test_cuda_graph_training_step_matches_eager(monkeypatch):
    torch.manual_seed(2)
    m = _model(heads=2).cuda().set_precision("fp32")
    x = torch.randn(300, 24, device="cuda")
    ei = torch.zeros(2, 0, dtype=torch.long, device="cuda")
    wgt = torch.randn(300, 5, device="cuda")
    m.train()
    K.dropout_epoch()
    monkeypatch.setattr(E, "next_seed", lambda: 0x5EED)
    eager = _train_step(m, x, ei, wgt)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _train_step(m, x, ei, wgt)
    torch.cuda.current_stream().wait_stream(s)
    for p_ in m.parameters():
        p_.grad = None
    xo = x.clone().requires_grad_(True)
    cg = torch.cuda.CUDAGraph()
    with torch.cuda.graph(cg):
        out = m(_Data(xo, ei))
        (out * wgt).sum().backward()
    cg.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager[0])
    assert all(torch.equal(p_.grad, g) for p_, g in zip([p for p in m.parameters() if p.grad is not None], eager[1]))
    assert torch.equal(xo.grad, eager[2])


def test_no_quadratic_buffer_in_training():
    n, h = 50_000, 64
    torch.manual_seed(0)
    m = ablation_gat.SGFormerGAT(32, h, 8, num_layers=1, num_heads=2, dropout=0.1, use_graph=False).cuda().set_precision("fp32")
    data = _Data(torch.randn(n, 32, device="cuda"), torch.zeros(2, 0, dtype=torch.long, device="cuda"))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    m(data).sum().backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert peak < 200 * n * h * 4, f"peak {peak / 2**20:.0f} MiB"      # an [N, N] fp32 buffer alone would be 9.3 GiB


# ---- planted errors: the module check must report the output they corrupt ---------------------------------------------------
def test_planted_scale_one_over_dk_is_reported(monkeypatch):
    fwd, bwd = K.attn_scaled_fwd, K.attn_scaled_bwd
    monkeypatch.setattr(K, "attn_scaled_fwd", lambda q, k, v, h, s: fwd(q, k, v, h, s * s))
    monkeypatch.setattr(K, "attn_scaled_bwd", lambda q, k, v, h, s, *a, **kw: bwd(q, k, v, h, s * s, *a, **kw))
    with pytest.raises(AssertionError, match="eval_logits"):
        _module_check("h3_dk5", "fp32")


def test_planted_pad_rows_kept_in_weight_gradient_is_reported(monkeypatch):
    monkeypatch.setattr(E, "_gat_attn_unpad_rows", lambda t, heads, dk, mp: t[:heads * dk])
    with pytest.raises(AssertionError, match=r"convs\.1\.attention\.attention\.W[qk]\."):
        _module_check("h3_dk5", "fp32")


def test_planted_one_head_dv_scaled_is_reported(monkeypatch):
    bwd = K.attn_scaled_bwd

    def wrapped(q, k, v, heads, scale, g, gscale, dq, dk, dv, dv_accumulate=False):
        bwd(q, k, v, heads, scale, g, gscale, dq, dk, dv, dv_accumulate)
        d = dv.shape[1] // heads
        dv[:, d:2 * d] *= 1.01

    monkeypatch.setattr(K, "attn_scaled_bwd", wrapped)
    with pytest.raises(AssertionError, match=r"convs\.1\.attention\.attention\.Wv\."):
        _module_check("h2_noweight", "fp32")


@pytest.mark.parametrize("heads,use_weight", [(3, True), (2, False)])
def test_standalone_layer_vs_fp64(heads, use_weight):
    """A TransConvLayer called on its own (GATAttention.forward through ScaledAttentionFn, dk = 16 // 3 = 5 padded) against the
    oracle's layer in fp64."""
    torch.manual_seed(4)
    layer = ablation_gat.TransConvLayer(16, 16, heads, use_weight).cuda().set_precision("fp32")
    x = torch.randn(70, 16, device="cuda", requires_grad=True)
    out = layer(x, x)
    g = torch.randn_like(out)
    out.backward(g)
    sd = {"l." + k: v.detach().double().requires_grad_() for k, v in layer.state_dict().items()}
    xr = x.detach().double().requires_grad_()
    ref = O.layer(sd, "l.", xr, heads, use_weight)
    ref.backward(g.double())
    scale = max(v.grad.abs().max().item() for v in sd.values() if v.grad is not None)
    _check("out", out.detach(), ref.detach(), 1e-4, 1.0)
    _check("grad_x", x.grad, xr.grad, 1e-4, scale)
    for k, p in layer.named_parameters():
        assert (p.grad is None) == (sd["l." + k].grad is None), k
        if p.grad is not None:
            _check(k, p.grad, sd["l." + k].grad, 1e-4, scale, exact_zero=False)
