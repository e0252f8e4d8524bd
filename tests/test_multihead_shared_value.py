"""Multi-head SGFormer attention without a value projection (use_weight=False, num_heads > 1), on the CPU: the oracle pinned to
the reference's fixture (tests/make_golden_multihead.py), and the shared-value schedule of engine.py with the kernels replaced by
their torch-CPU emulation (tests/kernel_emu.py), single-process and row-sharded over gloo."""
import os

import pytest
import torch
import torch.multiprocessing as mp

import kernel_emu
from oracle import sgformer_oracle as O
from sgformer_b200 import engine as E
from sgformer_b200 import functional as Fn
from sgformer_b200.config import make_config
from sgformer_b200.dist import SINGLE
from test_row_sharding_gloo import _free_port, _worker

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FX = torch.load(os.path.join(GOLD, "multihead_shared_value.pt"), weights_only=False)
MODELS = sorted(FX["models"])


def _close(a, b, rtol, atol, what):
    a, b = a.detach().double(), b.detach().double()
    assert a.shape == b.shape, f"{what}: shape {tuple(a.shape)} vs {tuple(b.shape)}"
    err = (a - b).abs().max().item()
    ref = b.abs().max().item()
    assert err <= atol + rtol * ref, f"{what}: max err {err:.3e} (ref max {ref:.3e})"


def _cfg(c):
    keys = make_config("large", 1, 1, 1).keys()
    kw = {k: v for k, v in c.items() if k in keys and k not in ("variant", "in_channels", "hidden", "out_channels")}
    return make_config(c["variant"], c["in_channels"], c["hidden"], c["out_channels"], **kw)


def _leaves(sd):
    return {k: (v.clone().requires_grad_(True) if v.is_floating_point() and "running" not in k else v.clone()) for k, v in sd.items()}


def test_fixture_covers_the_configurations():
    cfgs = [FX["models"][k]["cfg"] for k in MODELS]
    assert {c["variant"] for c in cfgs} == {"large", "100M", "medium"}
    assert {c["num_heads"] for c in cfgs} == {2, 3, 4}
    assert {c["trans_num_layers"] for c in cfgs} == {1, 2}
    assert not any(c["trans_use_weight"] for c in cfgs)
    for key in ("trans_use_residual", "trans_use_bn", "use_graph"):
        assert {bool(c[key]) for c in cfgs} == {False, True}, key
    assert {c["aggregate"] for c in cfgs} == {"add", "cat"}
    for k in MODELS:
        m = FX["models"][k]
        assert not any(".Wv." in n for n in m["state_dict"])
        ei, n = m["edge_index"], m["x"].shape[0]
        pairs = set(map(tuple, ei.t().tolist()))
        assert any(a == b for a, b in pairs)                                # self loops
        assert any((b, a) not in pairs for a, b in pairs)                   # directed
        assert not bool((ei == n - 1).any())                                # isolated node
        assert torch.unique(ei[0] * n + ei[1]).numel() < ei.shape[1]     # duplicate edges


@pytest.mark.parametrize("name", MODELS)
def test_oracle_matches_reference(name):
    m = FX["models"][name]
    cfg, sd, x, ei = m["cfg"], m["state_dict"], m["x"], m["edge_index"]
    _close(O.sgformer_forward(cfg, sd, x, ei, training=False), m["out_eval"], 1e-5, 1e-6, "eval output")
    _close(O.get_attentions(x, sd, cfg), m["attentions"], 1e-5, 1e-7, "get_attentions")
    P = _leaves(sd)
    xg = x.clone().requires_grad_(True)
    stats = {}
    out = O.sgformer_forward(cfg, P, xg, ei, training=True, stats_out=stats)
    _close(out, m["out_train"], 1e-5, 1e-6, "train output")
    (out * m["loss_weight"]).sum().backward()
    _close(xg.grad, m["grad_x"], 2e-4, 1e-6, "grad x")
    for k, g in m["grads"].items():
        _close(P[k].grad, g, 2e-4, 2e-5, f"grad {k}")
    for k, v in m["buffers_after_train"].items():
        _close(stats.get(k, sd[k]), v, 1e-5, 1e-6, f"buffer {k}")


def test_oracle_attention_broadcasts_one_head_value():
    for name, c in FX["attention"].items():
        q, k, v = (c[t].clone().requires_grad_(True) for t in "qkv")
        o = O.full_attention(q, k, v)
        _close(o, c["out"], 1e-5, 1e-6, f"{name} out")
        (o * c["w"]).sum().backward()
        for t, g in (("dq", q.grad), ("dk", k.grad), ("dv", v.grad)):
            _close(g, c[t], 5e-4, 1e-7, f"{name} {t}")


# ------------------------------------------------------------------------------------------------
# the schedule on the emulated kernels
# ------------------------------------------------------------------------------------------------
@pytest.fixture
def emulated(monkeypatch):
    monkeypatch.setattr(E, "K", kernel_emu)
    monkeypatch.setattr(Fn, "K", kernel_emu)


@pytest.mark.parametrize("name", MODELS)
def test_schedule_matches_reference(emulated, name):
    m = FX["models"][name]
    cfg = _cfg(m["cfg"])
    sd = m["state_dict"]
    names = tuple(sd)
    n = m["x"].shape[0]
    graph = kernel_emu.EmuGraph(m["edge_index"], n, 1 if cfg["variant"] == "medium" else 0) if cfg["use_graph"] else None
    out = Fn.SGFormerFn.apply(m["x"], graph, cfg, E.FP32, False, SINGLE, names, *[sd[k].clone() for k in names])
    _close(out, m["out_eval"], 2e-5, 2e-6, "eval output")

    P = _leaves(sd)
    x = m["x"].clone().requires_grad_(True)
    out = Fn.SGFormerFn.apply(x, graph, cfg, E.FP32, True, SINGLE, names, *[P[k] for k in names])
    _close(out, m["out_train"], 2e-5, 2e-6, "train output")
    (out * m["loss_weight"]).sum().backward()
    _close(x.grad, m["grad_x"], 5e-4, 2e-6, "grad x")
    for k, g in m["grads"].items():
        assert P[k].grad is not None, f"missing grad {k}"
        _close(P[k].grad, g, 5e-4, 3e-5, f"grad {k}")
    assert not any(".Wv." in k for k in names)
    for k, v in m["buffers_after_train"].items():
        _close(P[k].float(), v.float(), 1e-5, 1e-6, f"buffer {k}")

    Pt = {k: v for k, v in sd.items() if k.startswith("trans_conv.")}
    atts = E.trans_attentions(Pt, cfg, kernel_emu.pack_operand(m["x"], False, 3), E.FP32, with_act=cfg["variant"] == "large")
    _close(torch.stack(atts, 0), m["attentions"], 1e-4, 1e-9, "get_attentions")


def test_attention_fn_broadcasts_one_head_value(emulated):
    for name, c in FX["attention"].items():
        q, k, v = (c[t].clone().requires_grad_(True) for t in "qkv")
        o = Fn.AttentionFn.apply(q, k, v, E.FP32)
        _close(o, c["out"], 2e-5, 2e-6, f"{name} out")
        (o * c["w"]).sum().backward()
        assert v.grad.shape == v.shape
        for t, g in (("dq", q.grad), ("dk", k.grad), ("dv", v.grad)):
            _close(g, c[t], 1e-3, 1e-7, f"{name} {t}")


def test_shared_value_dv_sums_heads_in_order(emulated, monkeypatch):
    """The heads' dv GEMMs write one [N, D] buffer: the first overwrites it (or adds, when the caller accumulates), the others add,
    in head order."""
    c = FX["attention"]["n65_h3_m16_d16"]
    n, heads, m = c["q"].shape
    d = c["v"].shape[2]
    tape = E.Tape()
    E.attention_forward(c["q"].reshape(n, -1), c["k"].reshape(n, -1), c["v"].reshape(n, d), heads, E.FP32, tape, shared_v=True)
    seen = []
    real = kernel_emu.gemm_nt

    def spy(A, B, pairs, n_out, out, **kw):
        if kw.get("aux") is not None and kw.get("beta") == float(n):
            seen.append((out.data_ptr(), out.shape, kw.get("accumulate", False)))
        return real(A, B, pairs, n_out, out, **kw)

    monkeypatch.setattr(kernel_emu, "gemm_nt", spy)
    for acc in (False, True):
        seen.clear()
        dq, dk, dv = torch.zeros(n, heads * m), torch.zeros(n, heads * m), torch.zeros(n, d)
        E.attention_backward(tape, c["w"].reshape(n, -1), 1.0, E.FP32, dq, dk, dv, dv_accumulate=acc)
        assert [s[2] for s in seen] == [acc] + [True] * (heads - 1)
        assert all(s[0] == dv.data_ptr() and tuple(s[1]) == (n, d) for s in seen)


# ------------------------------------------------------------------------------------------------
# row sharding over gloo: C1 / C2 carry the same partials as with one value per head; v is row-local
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("name", ["large_h2_res_ln_add", "100M_h3_res_ln_add", "medium_h4_cat_plain"])
def test_row_sharded_matches_single_process(tmp_path, world, name):
    m = FX["models"][name]
    fixture = str(tmp_path / "model.pt")
    torch.save(m, fixture)
    mp.spawn(_worker, args=(world, _free_port(), fixture, str(tmp_path)), nprocs=world, join=True)
    parts = [torch.load(str(tmp_path / f"rank{r}.pt"), weights_only=False) for r in range(world)]
    _close(torch.cat([p["out"] for p in parts]), m["out_train"], 5e-5, 5e-6, "sharded train logits")
    _close(torch.cat([p["grad_x"] for p in parts]), m["grad_x"], 1e-3, 5e-6, "sharded grad x")
    for k, g in m["grads"].items():
        for r, p in enumerate(parts):
            _close(p["grads"][k], g, 1e-3, 5e-5, f"rank {r} grad {k} (all-reduced)")
    for k, v in m["buffers_after_train"].items():
        if "running" in k:
            _close(parts[0]["buffers"][k].float(), v.float(), 1e-4, 1e-5, f"buffer {k}")
