"""Multi-head SGFormer attention without a value projection (use_weight=False, num_heads > 1) on the H100: every head attends
with its own q and k over one shared value, the layer input, as the reference's one-head `vs` broadcasts across heads
(medium/ours.py:21-23, 84).  The drop-in modules against the reference's fixture (tests/make_golden_multihead.py), the recipes'
widths against the fp64 oracle with the bounds of tests/config_matrix.py, the standalone layer and free function, run-to-run
bit identity, a CUDA-graph captured step and reference-format checkpoints."""
import io
import os

import pytest
import torch

import config_matrix as M
from oracle import sgformer_oracle as O
from test_gpu_model import _check_grads, build_model, run

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FX = torch.load(os.path.join(GOLD, "multihead_shared_value.pt"), weights_only=False)
MODELS = sorted(FX["models"])
TOL = {"fp32": 1e-4, "bf16": 1e-2}


def _close(a, b, rtol, atol, what):
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    assert a.shape == b.shape, f"{what}: shape {tuple(a.shape)} vs {tuple(b.shape)}"
    err = (a - b).abs().max().item()
    ref = b.abs().max().item()
    assert err == err and err <= atol + rtol * ref, f"{what}: max err {err:.3e} (ref max {ref:.3e})"


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", MODELS)
def test_module_matches_reference_fixture(name, precision):
    m = FX["models"][name]
    cfg, tol = m["cfg"], TOL[precision]
    model = build_model(cfg).to(DEV).set_precision(precision)
    model.load_state_dict(m["state_dict"])           # the reference's checkpoint: no Wv keys
    x, ei = m["x"].to(DEV), m["edge_index"].to(DEV)
    model.eval()
    with torch.no_grad():
        _close(run(model, cfg, x, ei), m["out_eval"], tol, tol, "eval output")
    _close(model.get_attentions(x), m["attentions"], tol, tol, "get_attentions")
    model.train()
    xg = x.clone().requires_grad_(True)
    out = run(model, cfg, xg, ei)
    _close(out, m["out_train"], tol, tol, "train output")
    if precision == "fp32":    # bf16 gradients are bounded at the recipes' widths below; on these tiny layers they carry its noise
        (out * m["loss_weight"].to(DEV)).sum().backward()
        grads = {k: p.grad for k, p in model.named_parameters()}
        grads["__x__"] = xg.grad
        problems = []
        _check_grads(grads, dict(m["grads"], __x__=m["grad_x"]), precision, problems)
        assert not problems, "\n".join(problems)
        sd = model.state_dict()
        for k, v in m["buffers_after_train"].items():
            _close(sd[k].float(), v.float(), 1e-4, 1e-5, f"buffer {k}")


# ------------------------------------------------------------------------------------------------
# the recipes' widths against the fp64 oracle (medium/run.sh and large/run.sh switches with several heads and no Wv)
# ------------------------------------------------------------------------------------------------
# Columns as tests/config_matrix.py's table: name, variant, tl, heads, t_bn, t_res, t_w, t_act, gl, g_w, g_init, g_bn, g_res, g_act,
# agg, ug, gw, alpha, h, d, c, n, hub, sym.
CASES = [M.Case(*r) for r in [
    ("cora_h2", "medium", 1, 2, 0, 0, 0, 0, 3, 1, 0, 0, 1, 1, "add", 1, 0.8, 0.5, 64, 1433, 7, 3001, 0, 1),
    ("deezer_h4_hub", "medium", 1, 4, 0, 1, 0, 0, 1, 1, 0, 0, 1, 1, "add", 1, 0.8, 0.5, 96, 602, 2, 8200, 1, 0),
    ("arxiv_h3", "large", 1, 3, 1, 1, 0, 1, 3, 1, 0, 1, 1, 1, "add", 1, 0.5, 0.5, 256, 128, 40, 20011, 0, 1),
    ("papers_h2_t2_cat", "100M", 2, 2, 1, 1, 0, 0, 2, 1, 1, 1, 1, 1, "cat", 1, 0.8, 0.5, 256, 128, 47, 3001, 1, 1),
]]


def _module_step(c, precision):
    inp = M.inputs(c)
    ocfg = inp["ocfg"]
    model = build_model(ocfg).to(DEV).set_precision(precision)
    model.load_state_dict(inp["sd"])
    x, ei = inp["x"].to(DEV), inp["ei"].to(DEV)
    model.train()
    xg = x.clone().requires_grad_(True)
    out = run(model, ocfg, xg, ei)
    (out * inp["lw"].to(DEV)).sum().backward()
    grads = {k: p.grad for k, p in model.named_parameters() if p.grad is not None}
    grads["__x__"] = xg.grad
    stats = {k: v for k, v in model.state_dict().items() if "running" in k or k.endswith("num_batches_tracked")}
    return dict(out=out, grads=grads, stats=stats)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("c", CASES, ids=[c.name for c in CASES])
def test_recipe_widths_match_fp64_oracle(c, precision):
    assert not M.oracle_config(c)["trans_use_weight"] and c.heads > 1
    got = _module_step(c, precision)
    problems = M.check(c, got, M.oracle_run(c, torch.float64), M.oracle_run(c, torch.float32), precision)
    assert not problems, "\n".join(problems)


def test_gradients_are_bit_identical_run_to_run():
    c = CASES[1]
    a, b = _module_step(c, "fp32"), _module_step(c, "fp32")
    assert torch.equal(a["out"], b["out"])
    for k, g in a["grads"].items():
        assert torch.equal(g, b["grads"][k]), f"{k} differs between two runs"


# ------------------------------------------------------------------------------------------------
# standalone surface
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision,tol", [("fp32", 1e-4), ("bf16", 1e-2)])
def test_full_attention_conv_one_head_value(precision, tol):
    from sgformer_b200.medium import full_attention_conv
    for name, c in FX["attention"].items():
        q, k, v = (c[t].to(DEV).requires_grad_(True) for t in "qkv")
        o = full_attention_conv(q, k, v, precision=precision)
        _close(o, c["out"], tol, tol, f"{name} out")
        (o * c["w"].to(DEV)).sum().backward()
        assert v.grad.shape == v.shape
        gt = 2e-3 if precision == "fp32" else 8e-2
        for t, g in (("dq", q.grad), ("dk", k.grad), ("dv", v.grad)):
            _close(g, c[t], gt, gt * c[t].abs().max().item() * 0.05 + 1e-7, f"{name} {t}")


@pytest.mark.parametrize("variant", ["large", "100M", "medium"])
def test_transconv_layer_alone_matches_fp64_oracle(variant):
    import importlib
    mod = importlib.import_module({"large": "sgformer_b200.large", "100M": "sgformer_b200.hundred_m",
                                   "medium": "sgformer_b200.medium"}[variant])
    n, h, heads = 3000, 64, 3
    torch.manual_seed(5)
    layer = mod.TransConvLayer(h, h, num_heads=heads, use_weight=False).to(DEV)
    assert not hasattr(layer, "Wv")
    x = torch.randn(n, h)
    w = torch.randn(n, h)
    sd = {k: v.detach().cpu().double().requires_grad_(True) for k, v in layer.state_dict().items()}
    x64 = x.double().requires_grad_(True)
    ref = O.trans_conv_layer(x64, sd, "", heads, False)
    (ref * w.double()).sum().backward()
    xg = x.to(DEV).requires_grad_(True)
    out = layer(xg, xg)
    _close(out, ref, 1e-4, 1e-4, "layer output")
    (out * w.to(DEV)).sum().backward()
    _close(xg.grad, x64.grad, 2e-3, 2e-3 * x64.grad.abs().max().item() * 0.05, "grad x")
    for k, p in layer.named_parameters():
        _close(p.grad, sd[k].grad, 2e-3, 2e-3 * sd[k].grad.abs().max().item() * 0.05 + 1e-7, f"grad {k}")


def test_row_kernels_refuse_too_few_head_columns():
    from sgformer_b200 import kernels as K
    x = torch.zeros(10, 16, device=DEV)
    with pytest.raises(ValueError, match="heads"):
        K.head_mean(x, 2, 16)
    assert K.head_mean(x, 2, 8).shape == (10, 8)
    with pytest.raises(ValueError, match="heads"):
        K.gat_logits(x, 4, 8, torch.zeros(32, device=DEV), torch.zeros(32, device=DEV))
    with pytest.raises(ValueError):
        K.attn_combine_scal(torch.zeros(2, 8, device=DEV), 3, torch.zeros(4, device=DEV))


def test_reference_checkpoint_round_trip():
    """A reference-format state_dict (no Wv keys) loads strictly, saves back with the same keys and values, and the reloaded
    model computes the same logits."""
    m = FX["models"]["large_h2_res_ln_add"]
    a = build_model(m["cfg"]).to(DEV)
    a.load_state_dict(m["state_dict"])
    sd = a.state_dict()
    assert list(sd) == list(m["state_dict"])
    assert all(torch.equal(sd[k].cpu(), v) for k, v in m["state_dict"].items())
    buf = io.BytesIO()
    torch.save(sd, buf)
    buf.seek(0)
    b = build_model(m["cfg"]).to(DEV)
    b.load_state_dict(torch.load(buf, weights_only=True))
    a.eval()
    b.eval()
    x, ei = m["x"].to(DEV), m["edge_index"].to(DEV)
    with torch.no_grad():
        assert torch.equal(run(a, m["cfg"], x, ei), run(b, m["cfg"], x, ei))


def test_cuda_graph_step_matches_eager():
    """A captured training step of an SGFormer with three shared-value heads replays to the eager step's values bit for bit."""
    from sgformer_b200 import large as L
    from sgformer_b200.synth import make_graph
    n, d, h, c = 3000, 48, 64, 7
    torch.manual_seed(9)
    model = L.SGFormer(d, h, c, trans_num_layers=2, trans_num_heads=3, trans_use_weight=False, trans_dropout=0.0, gnn_dropout=0.0,
                       gnn_num_layers=2).to(DEV)
    model.train()
    x = torch.randn(n, d, device=DEV)
    ei = make_graph(n, 20000, seed=4).to(DEV)
    wgt = torch.randn(n, c, device=DEV)
    sd0 = {k: v.clone() for k, v in model.state_dict().items()}

    def step():
        for p in model.parameters():
            p.grad = None
        out = model(x, ei)
        (out * wgt).sum().backward()
        return out

    eager = step().detach().clone()
    eager_grads = [p.grad.clone() for p in model.parameters()]
    model.load_state_dict(sd0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    cg = torch.cuda.CUDAGraph()
    with torch.cuda.graph(cg):
        out = step()
    model.load_state_dict(sd0)
    cg.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
    assert all(torch.equal(p.grad, g) for p, g in zip(model.parameters(), eager_grads))
