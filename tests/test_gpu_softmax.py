"""The fused softmax attention (csrc/attn_softmax.cu) and SGFormerSOFT on the device.  The references are fp64: autograd through
oracle/softmax_oracle.py for the kernels, and tests/golden/sgformer_softmax.pt (made from the unmodified oursSOFT.py) for the
modules.  Errors are max |x - ref| / max |ref| per output: fp32 within 1e-4, bf16 within 1e-2.  Where the exact gradient is zero
(one head: every weight is 1; a shared v under the head mean: every head has the same dP, and the softmax over heads passes
nothing back), the fp64 reference holds only rounding noise and the kernels must return exactly zero."""
import os

import pytest
import torch

from oracle import softmax_oracle as O
from sgformer_b200 import ablation, medium
from sgformer_b200 import engine as E
from sgformer_b200 import kernels as K

pytestmark = pytest.mark.gpu
TOL = {"fp32": 1e-4, "bf16": 1e-2}
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sgformer_softmax.pt")


def _check(name, x, ref, tol, scale, exact_zero=True):
    """scale: the largest magnitude among the outputs of the same call; a reference below 1e-12 of it is rounding noise of an
    exact zero, which the attention kernels return exactly.  exact_zero=False (the GCN conv bias ahead of a train-mode
    BatchNorm: zero gradient, which the unchanged GCN schedule forms as a cancelling column sum): within tol * scale."""
    rmax = ref.abs().max().item()
    if rmax <= 1e-12 * scale:
        if exact_zero:
            assert torch.count_nonzero(x) == 0, f"{name}: the exact value is zero, got max {x.abs().max().item():.3g}"
        else:
            assert x.abs().max().item() <= tol * scale, f"{name}: the exact value is zero, got max {x.abs().max().item():.3g}"
        return
    err = ((x.double() - ref).abs().max() / rmax).item()
    assert err <= tol, f"{name}: relative error {err:.3g}"


def _kernel_case(n, heads, m, shared_v, per_head_g, prec_name, seed=0, d=None, accumulate=False):
    """d: v's width per head (default m).  accumulate: dv starts from random values and the backward adds to them."""
    prec = E.precision(prec_name)
    g = torch.Generator(device="cuda").manual_seed(seed)
    d = m if d is None else d
    dt = prec.act_dtype
    q = (torch.randn(n, heads * m, device="cuda", generator=g) * 2 + 0.5).to(dt)
    k = (torch.randn(n, heads * m, device="cuda", generator=g) - 0.3).to(dt)
    v = torch.randn(n, (1 if shared_v else heads) * d, device="cuda", generator=g).to(dt)
    gr = torch.randn(n, (heads if per_head_g else 1) * d, device="cuda", generator=g).to(dt)
    gscale = 1.0 if per_head_g else 1.0 / heads
    tape = E.Tape()
    o = E.attention_softmax_forward(q, k, v, heads, prec, tape, shared_v=shared_v, shared_g=not per_head_g and heads > 1)
    dq, dk = K.alloc_act(n, heads * m, dt, "cuda"), K.alloc_act(n, heads * m, dt, "cuda")
    dv = K.alloc_act(n, v.shape[1], dt, "cuda")
    if accumulate:
        dv.copy_(torch.randn(n, v.shape[1], device="cuda", generator=g) * 2)
    dv0 = dv.double() if accumulate else 0.0
    E.attention_softmax_backward(tape, gr, gscale, dq, dk, dv, dv_accumulate=accumulate)
    qr, kr = (t.double().reshape(n, heads, m).requires_grad_() for t in (q, k))
    vr = v.double().reshape(n, -1, d).requires_grad_()
    ref, _ = O.softmax_attention(qr, kr, vr)
    ref.backward(gr.double().reshape(n, -1, d).expand(n, heads, d) * gscale)
    torch.cuda.synchronize()
    return {"o": (o, ref.detach().reshape(n, -1)), "dq": (dq, qr.grad.reshape(n, -1)), "dk": (dk, kr.grad.reshape(n, -1)),
            "dv": (dv, dv0 + vr.grad.reshape(n, -1))}


def _check_case(res, tol):
    scale = max(ref.abs().max().item() for _, ref in res.values())
    for name, (x, ref) in res.items():
        _check(name, x, ref, tol, scale)


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("shared_v,per_head_g", [(False, False), (True, False), (True, True), (False, True)])
@pytest.mark.parametrize("heads,m", [(1, 16), (2, 64), (8, 32), (1, 256), (2, 120)])
@pytest.mark.parametrize("n", [1, 63, 64, 65, 300])
def test_kernels_vs_fp64(n, heads, m, shared_v, per_head_g, prec):
    _check_case(_kernel_case(n, heads, m, shared_v, per_head_g, prec), TOL[prec])


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("shared_v,per_head_g", [(False, False), (True, True)])
def test_kernels_vs_fp64_many_tiles(shared_v, per_head_g, prec):
    n = 2 * torch.cuda.get_device_properties(0).multi_processor_count * 64 + 7
    _check_case(_kernel_case(n, 2, 64, shared_v, per_head_g, prec, seed=1), TOL[prec])


@pytest.mark.parametrize("shared_v", [False, True])
def test_more_than_eight_heads(shared_v):
    _check_case(_kernel_case(97, 12, 16, shared_v, True, "fp32"), 1e-4)


def test_row_width_limit_is_a_clear_error():
    x = torch.zeros(8, 4 * 128, device="cuda")
    with pytest.raises(ValueError, match="at most 1024 bytes"):
        E.attention_softmax_forward(x, x, x, 4, E.FP32, None)


class _Data:
    def __init__(self, x, ei):
        self.graph = {"node_feat": x, "edge_index": ei}


def _native_for(cfg, d, h, c):
    gnn = medium.GCN(d, h, h, num_layers=2, dropout=0.0, use_bn=True) if cfg["use_graph"] else None
    return ablation.SGFormerSOFT(d, h, c, num_layers=2, num_heads=cfg["heads"], alpha=0.5, dropout=0.0, use_bn=cfg["use_bn"],
                                 use_residual=cfg["use_residual"], use_weight=cfg["use_weight"], use_graph=cfg["use_graph"],
                                 graph_weight=0.8, gnn=gnn, aggregate=cfg["aggregate"])


GD = None


def _golden():
    global GD
    if GD is None:
        GD = torch.load(GOLDEN, weights_only=False)
    return GD


@pytest.mark.parametrize("case", ["h1", "h2_noweight", "h4_nores", "h2_noln", "h2_gcn_add", "h4_gcn_cat"])
def test_module_vs_reference_fixture(case):
    gd = _golden()
    rec = gd["cases"][case]
    sd = rec["state_dict"]
    x, ei = gd["x"].cuda(), gd["edge_index"].cuda()
    d, h, c = x.shape[1], sd["trans_conv.fcs.0.weight"].shape[0], sd["fc.weight"].shape[0]
    m = _native_for(rec["config"], d, h, c).cuda().set_precision("fp32")
    m.load_state_dict(sd)                  # the reference's own checkpoint
    ref = rec["fp64"]
    m.eval()
    with torch.no_grad():
        _check("eval_logits", m(_Data(x, ei)), ref["eval_logits"].cuda(), 1e-4, 1.0)
        _check("attentions", m.get_attentions(x), ref["attentions"].cuda(), 1e-4, 1.0)
    m.train()
    xg = x.clone().requires_grad_()
    out = m(_Data(xg, ei))
    _check("train_logits", out.detach(), ref["train_logits"].cuda(), 1e-4, 1.0)
    (out * rec["wout"].cuda()).sum().backward()
    scale = max(g.abs().max().item() for g in ref["grads"].values())
    _check("grad_x", xg.grad, ref["grad_x"].cuda(), 1e-4, scale)
    for name, p in m.named_parameters():
        if name not in ref["grads"]:        # unused by the reference (LayerNorms with use_bn=False)
            assert p.grad is None or torch.count_nonzero(p.grad) == 0, name
            continue
        _check(name, p.grad, ref["grads"][name].cuda(), 1e-4, scale, exact_zero=not name.startswith("gnn."))


def _model(heads=2, use_weight=True, d=24, h=32, c=5):
    return ablation.SGFormerSOFT(d, h, c, num_layers=2, num_heads=heads, alpha=0.5, dropout=0.5, use_weight=use_weight,
                                 use_graph=False)


def _train_step(m, x, ei, wgt):
    m.zero_grad(set_to_none=True)
    xg = x.clone().requires_grad_()
    out = m(_Data(xg, ei))
    (out * wgt).sum().backward()
    return out.detach().clone(), [p.grad.clone() for p in m.parameters()], xg.grad.clone()


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_training_step_bit_identical(prec, monkeypatch):
    torch.manual_seed(1)
    m = _model(heads=2, use_weight=False).cuda().set_precision(prec)
    x = torch.randn(1000, 24, device="cuda")
    ei = torch.zeros(2, 0, dtype=torch.long, device="cuda")
    wgt = torch.randn(1000, 5, device="cuda")
    monkeypatch.setattr(E, "next_seed", lambda: 0x5EED)
    a, b = _train_step(m, x, ei, wgt), _train_step(m, x, ei, wgt)
    assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2])
    assert all(torch.equal(p, q) for p, q in zip(a[1], b[1]))


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
    assert all(torch.equal(p_.grad, g) for p_, g in zip(m.parameters(), eager[1]))
    assert torch.equal(xo.grad, eager[2])


def test_no_quadratic_buffer_in_training():
    n, h = 50_000, 64
    torch.manual_seed(0)
    m = ablation.SGFormerSOFT(32, h, 8, num_layers=1, num_heads=2, dropout=0.1, use_graph=False).cuda().set_precision("fp32")
    data = _Data(torch.randn(n, 32, device="cuda"), torch.zeros(2, 0, dtype=torch.long, device="cuda"))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    m(data).sum().backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert peak < 200 * n * h * 4, f"peak {peak / 2**20:.0f} MiB"      # an [N, N] fp32 buffer alone would be 9.3 GiB
