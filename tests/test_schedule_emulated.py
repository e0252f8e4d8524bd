"""Checks the forward/backward *schedules* (sgformer_b200/engine.py + functional.py) against the golden fixtures of
the reference, with the CUDA kernels replaced by their torch-CPU emulation (tests/kernel_emu.py).  Runs without a GPU.
The kernels themselves are verified on the H100 by the `-m gpu` tests."""
import glob
import os

import pytest
import torch

import kernel_emu
from sgformer_b200 import engine as E
from sgformer_b200 import functional as Fn
from sgformer_b200.config import make_config
from sgformer_b200.dist import SINGLE

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MODEL_FILES = sorted(glob.glob(os.path.join(GOLD, "model_*.pt")))


@pytest.fixture(autouse=True)
def emulated_kernels(monkeypatch):
    monkeypatch.setattr(E, "K", kernel_emu)
    monkeypatch.setattr(Fn, "K", kernel_emu)
    yield


def _cfg_from_oracle(c):
    keys = make_config("large", 1, 1, 1).keys()
    kw = {k: v for k, v in c.items() if k in keys and k not in ("variant", "in_channels", "hidden", "out_channels")}
    return make_config(c["variant"], c["in_channels"], c["hidden"], c["out_channels"], **kw)


def _close(a, b, rtol, atol, what):
    a, b = a.double(), b.double()
    err = (a - b).abs().max().item()
    ref = b.abs().max().item()
    assert err <= atol + rtol * ref, f"{what}: max err {err:.3e} (ref max {ref:.3e})"


@pytest.mark.parametrize("path", MODEL_FILES, ids=[os.path.basename(p)[6:-3] for p in MODEL_FILES])
def test_fused_schedule_fp32(path):
    fx = torch.load(path, weights_only=False)
    cfg = _cfg_from_oracle(fx["cfg"])
    sd = {k: v.clone() for k, v in fx["state_dict"].items()}
    names = tuple(sd.keys())
    n = fx["x"].shape[0]
    graph = kernel_emu.EmuGraph(fx["edge_index"], n, 1 if cfg["variant"] == "medium" else 0)

    out = Fn.SGFormerFn.apply(fx["x"], graph, cfg, E.FP32, False, SINGLE, names, *[sd[k] for k in names])
    _close(out, fx["out_eval"], 2e-5, 2e-6, "eval output")

    params = [sd[k].clone().requires_grad_(True) if (sd[k].is_floating_point() and "running" not in k) else sd[k].clone()
              for k in names]
    x = fx["x"].clone().requires_grad_(True)
    out = Fn.SGFormerFn.apply(x, graph, cfg, E.FP32, True, SINGLE, names, *params)
    _close(out, fx["out_train"], 2e-5, 2e-6, "train output")
    (out * fx["loss_weight"]).sum().backward()
    _close(x.grad, fx["grad_x"], 5e-4, 2e-6, "grad x")
    got = dict(zip(names, params))
    for k, g in fx["grads"].items():
        assert got[k].grad is not None, f"missing grad {k}"
        _close(got[k].grad, g, 5e-4, 3e-5, f"grad {k}")
    for k, v in fx["buffers_after_train"].items():
        _close(got[k].float(), v.float(), 1e-5, 1e-6, f"buffer {k}")


def test_attention_fn_matches_reference():
    fx = torch.load(os.path.join(GOLD, "attention.pt"), weights_only=False)
    for name, c in fx.items():
        q, k, v = (c[t].clone().requires_grad_(True) for t in "qkv")
        o = Fn.AttentionFn.apply(q, k, v, E.FP32)
        _close(o, c["out"], 2e-5, 2e-6, f"{name} out")
        (o * c["w"]).sum().backward()
        for t, g in (("dq", q.grad), ("dk", k.grad), ("dv", v.grad)):
            _close(g, c[t], 1e-3, 1e-7, f"{name} {t}")


def test_get_attentions_matches_reference():
    """engine.trans_attentions (kernel path of TransConv.get_attentions) against the reference's own get_attentions output."""
    fx = torch.load(os.path.join(GOLD, "get_attentions.pt"), weights_only=False)
    for name, ref in fx.items():
        m = torch.load(os.path.join(GOLD, f"model_{name}.pt"), weights_only=False)
        cfg = _cfg_from_oracle(m["cfg"])
        P = {k: v for k, v in m["state_dict"].items() if k.startswith("trans_conv.")}
        atts = E.trans_attentions(P, cfg, kernel_emu.pack_operand(m["x"], False, 3), E.FP32, with_act=cfg["variant"] == "large")
        got = torch.stack(atts, 0)
        assert got.shape == ref.shape
        _close(got, ref, 1e-4, 1e-9, f"get_attentions {name}")


def test_bf16_schedule_is_close():
    fx = torch.load(os.path.join(GOLD, "model_large_add_init.pt"), weights_only=False)
    cfg = _cfg_from_oracle(fx["cfg"])
    sd = fx["state_dict"]
    names = tuple(sd.keys())
    graph = kernel_emu.EmuGraph(fx["edge_index"], fx["x"].shape[0], 0)
    out = Fn.SGFormerFn.apply(fx["x"], graph, cfg, E.BF16, False, SINGLE, names, *[sd[k].clone() for k in names])
    _close(out, fx["out_eval"], 3e-2, 3e-2, "bf16 eval output")


# ------------------------------------------------------------------------------------------------
# property: random configurations / graphs, fused schedule (emulated kernels) vs the oracle's autograd
# ------------------------------------------------------------------------------------------------
from hypothesis import HealthCheck, given, settings  # noqa: E402
from hypothesis import strategies as st  # noqa: E402

from oracle import sgformer_oracle as O  # noqa: E402


@settings(max_examples=40, deadline=None, suppress_health_check=list(HealthCheck))
@given(variant=st.sampled_from(["large", "100M", "medium"]), n=st.integers(6, 70), h=st.sampled_from([8, 16]),
       heads=st.sampled_from([1, 2]), seed=st.integers(0, 10 ** 6), directed=st.booleans(), flags=st.lists(st.booleans(), min_size=9, max_size=9),
       aggregate=st.sampled_from(["add", "cat"]), layers=st.integers(0, 3), tlayers=st.integers(0, 2), use_graph=st.booleans())
def test_schedule_property(variant, n, h, heads, seed, directed, flags, aggregate, layers, tlayers, use_graph):
    d, c = 5, 3
    use_weight = flags[0] or heads > 1
    if variant == "medium":
        ocfg = O.make_config("medium", d, h, c, num_layers=tlayers, num_heads=heads, alpha=0.3, dropout=0.0, use_bn=flags[1],
                             use_residual=flags[2], use_weight=use_weight, gcn_num_layers=layers + 1, gcn_dropout=0.0,
                             gcn_use_bn=flags[3], graph_weight=0.7, aggregate=aggregate, use_graph=use_graph)
    else:
        kw = dict(trans_num_layers=tlayers, trans_num_heads=heads, trans_dropout=0.0, trans_use_bn=flags[1],
                  trans_use_residual=flags[2], trans_use_weight=use_weight, trans_use_act=flags[4], gnn_num_layers=layers,
                  gnn_dropout=0.0, gnn_use_weight=flags[5], gnn_use_init=flags[6], gnn_use_bn=flags[3], gnn_use_residual=flags[7],
                  gnn_use_act=flags[8], graph_weight=0.7, aggregate=aggregate, use_graph=use_graph)
        if variant == "100M":
            kw["alpha"] = 0.3
        ocfg = O.make_config(variant, d, h, c, **kw)
    if aggregate == "cat" and not use_graph:
        return   # the reference's fc would expect 2h inputs: invalid combination there as well
    cfg = _cfg_from_oracle(ocfg)
    sd = O.init_state_dict(ocfg, seed=seed)
    g = torch.Generator().manual_seed(seed)
    ei = torch.stack([torch.randint(0, n, (3 * n,), generator=g), torch.randint(0, n, (3 * n,), generator=g)])
    if not directed:
        ei = torch.cat([ei, ei.flip(0)], 1)
    x = torch.randn(n, d, generator=g)
    lw = torch.randn(n, c, generator=g)
    names = tuple(sd.keys())
    graph = kernel_emu.EmuGraph(ei, n, 1 if variant == "medium" else 0) if use_graph else None

    def leafs():
        return {k: (v.clone().requires_grad_(True) if v.is_floating_point() and "running" not in k else v.clone()) for k, v in sd.items()}

    ref_p = leafs()
    xr = x.clone().requires_grad_(True)
    ref = O.sgformer_forward(ocfg, ref_p, xr, ei, training=True)
    (ref * lw).sum().backward()
    got_p = leafs()
    xg = x.clone().requires_grad_(True)
    out = Fn.SGFormerFn.apply(xg, graph, cfg, E.FP32, True, SINGLE, names, *[got_p[k] for k in names])
    _close(out, ref.detach(), 1e-4, 1e-5, "logits")
    (out * lw).sum().backward()
    _close(xg.grad, xr.grad, 2e-3, 1e-5, "grad x")
    for k in names:
        if ref_p[k].is_floating_point() and ref_p[k].grad is not None:
            assert got_p[k].grad is not None, f"missing grad {k}"
            _close(got_p[k].grad, ref_p[k].grad, 2e-3, 2e-4, f"grad {k}")
