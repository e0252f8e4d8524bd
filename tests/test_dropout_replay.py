"""Dropout without a GPU: the host restatement of the kernels' mask (tests/dropout_mask.py), the oracles' dropout placement
against the unmodified reference with its masks replayed (tests/golden/dropout.pt), and the engine's forward/backward
schedules in training mode with dropout on (kernels replaced by their emulation) against the oracles with the kernels' masks
replayed from the seeds the forward passed.  The last part checks the per-call seed bookkeeping of engine.py: a backward that
recomputes a different layer's mask fails it."""
import os

import numpy as np
import pytest
import torch

import kernel_emu
import kernel_emu_difformer
from dropout_mask import (DropoutRecorder, MaskReplayer, keep_mask, keep_scale, keep_threshold, unpack_mask)
from oracle import difformer_oracle as D
from oracle import sgformer_oracle as O
from sgformer_b200 import engine as E
from sgformer_b200 import functional as Fn
from sgformer_b200.dist import SINGLE

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RECIPE_P = (0.2, 0.3, 0.4, 0.5, 0.6)


# ------------------------------------------------------------------------------------------------
# the restatement itself
# ------------------------------------------------------------------------------------------------
def _mask_scalar(seed, epoch, r, c, h, p):
    """One element in plain Python integers (an independent statement of the numpy vectorisation)."""
    m = (1 << 64) - 1
    x = (seed + epoch * 0xD1B54A32D192ED03 + (r * (h // 4) + c // 4) * 0x9E3779B97F4A7C15) & m
    x ^= x >> 33
    x = (x * 0xFF51AFD7ED558CCD) & m
    x ^= x >> 33
    x = (x * 0xC4CEB9FE1A85EC53) & m
    x ^= x >> 33
    return ((x >> (16 * (c % 4))) & 0xFFFF) >= keep_threshold(p)


@pytest.mark.parametrize("seed,epoch", [(0, 0), (12345, 0), (7, 3), ((1 << 62) + 977, 0), ((1 << 63) - 5, 11), ((1 << 64) - 1, 2)])
def test_keep_mask_matches_scalar_statement(seed, epoch):
    rows, h, p = 9, 24, 0.5
    m = keep_mask(seed, rows, h, p, epoch)
    want = np.array([[_mask_scalar(seed, epoch, r, c, h, p) for c in range(h)] for r in range(rows)])
    assert np.array_equal(m, want)


def _binom_ok(k, n, q, z=5.0):
    return abs(k - n * q) <= z * np.sqrt(n * q * (1 - q)) + 1


@pytest.mark.parametrize("p", [0.1, 0.5, 0.6, 0.9])
def test_keep_rate_per_column_residue_and_row(p):
    rows, h = 4096, 64
    m = keep_mask(0xC0FFEE, rows, h, p)
    q = 1 - keep_threshold(p) / 65536
    for res in range(4):                       # the four 16-bit fields of one hash
        k = int(m[:, res::4].sum())
        assert _binom_ok(k, m[:, res::4].size, q), (res, k)
    per_row = m.sum(1)
    assert all(_binom_ok(int(k), h, q, z=5.5) for k in per_row)
    per_col = m.sum(0)
    assert all(_binom_ok(int(k), rows, q) for k in per_col)


@pytest.mark.parametrize("p", [0.2, 0.5, 0.6])
def test_masks_of_neighbouring_seeds_rows_and_epochs_are_uncorrelated(p):
    rows, h, s = 2048, 96, 987654321
    q = 1 - keep_threshold(p) / 65536
    a = keep_mask(s, rows + 1, h, p)
    pairs = {"seed s / s+1 (adjacent layers)": (a[:rows], keep_mask(s + 1, rows + 1, h, p)[:rows]),
             "row r / r+1": (a[:rows], a[1:rows + 1]),
             "epoch e / e+1": (keep_mask(s, rows, h, p, 5), keep_mask(s, rows, h, p, 6))}
    for what, (x, y) in pairs.items():
        both = int((x & y).sum())
        assert _binom_ok(both, x.size, q * q), f"{what}: {both / x.size:.4f} kept in both vs {q * q:.4f}"


@pytest.mark.parametrize("p", RECIPE_P)
def test_keep_scale_is_inverse_keep_probability(p):
    """The one deliberate departure from F.dropout: the scale is 65536 / (65536 - round(p * 65536)), not 1 / (1 - p)."""
    assert abs(keep_scale(p) * (1 - p) - 1) <= 2e-5


@pytest.mark.parametrize("p", [2.0 ** -18, 0.1, 0.9, 0.99])
def test_keep_scale_rounding_bound(p):
    """p is rounded to a multiple of 2^-16: the relative scale error is at most 2^-17 / (1 - p) (+ fp32 rounding)."""
    assert abs(keep_scale(p) * (1 - p) - 1) <= 2.0 ** -17 / (1 - p) + 1e-6
    assert keep_threshold(2.0 ** -18) == 0 and keep_scale(2.0 ** -18) == 1.0


# ------------------------------------------------------------------------------------------------
# the oracles against the reference, with the reference's masks replayed
# ------------------------------------------------------------------------------------------------
FX = torch.load(os.path.join(GOLD, "dropout.pt"), weights_only=False)


def _unflat(f):
    out, o = {}, 0
    for name, shape in zip(f["names"], f["shapes"]):
        k = int(torch.Size(shape).numel())
        out[name] = f["flat"][o:o + k].reshape(shape)
        o += k
    return out


def _close(a, b, rtol, atol, what):
    a, b = torch.as_tensor(a).detach().double(), torch.as_tensor(b).detach().double()
    assert a.shape == b.shape, f"{what}: shape {tuple(a.shape)} vs {tuple(b.shape)}"
    err = (a - b).abs().max().item()
    ref = b.abs().max().item()
    assert err <= atol + rtol * ref, f"{what}: max err {err:.3e} (ref max {ref:.3e})"


def _stored_masks(case):
    return [(m["p"], unpack_mask(m)) for m in case["masks"]]


def test_fixture_is_small_and_covers_the_variants():
    assert os.path.getsize(os.path.join(GOLD, "dropout.pt")) < 1 << 20
    assert {"large_add_init", "100M_alpha", "medium_gcn", "medium_res_heads2"} <= set(FX["sgformer"])
    assert {"default", "no_graph", "no_res_no_bn", "source"} <= set(FX["difformer"])
    ps = {m["p"] for grp in FX.values() for c in grp.values() for m in c["masks"]}
    assert min(ps) <= 0.2 and max(ps) >= 0.6


@pytest.mark.parametrize("name", sorted(FX["sgformer"]))
def test_sgformer_oracle_matches_reference_with_its_masks(monkeypatch, name):
    case = FX["sgformer"][name]
    fx = torch.load(os.path.join(GOLD, case["base"]), weights_only=False)
    cfg = dict(fx["cfg"], **case["rates"])
    sd = fx["state_dict"]
    replay = MaskReplayer(_stored_masks(case), scale="ref")
    monkeypatch.setattr(O, "_dropout", replay)
    sdg = {k: (v.clone().requires_grad_(True) if v.is_floating_point() and "running" not in k else v) for k, v in sd.items()}
    xg = fx["x"].clone().requires_grad_(True)
    stats = {}
    out = O.sgformer_forward(cfg, sdg, xg, fx["edge_index"], training=True, stats_out=stats)
    replay.finish()
    _close(out, case["out_train"], 1e-5, 1e-6, "train output")
    # not vacuous: the masks move the output far beyond the tolerance
    assert (case["out_train"] - fx["out_train"]).abs().max() > 100 * (1e-6 + 1e-5 * fx["out_train"].abs().max())
    (out * fx["loss_weight"]).sum().backward()
    _close(xg.grad, case["grad_x"], 2e-4, 1e-6, "grad x")
    for k, g in _unflat(case["grads"]).items():
        _close(sdg[k].grad, g, 2e-4, 2e-5, f"grad {k}")
    if case["buffers_after_train"] is not None:
        for k, v in _unflat(case["buffers_after_train"]).items():
            _close(stats.get(k, sd[k]), v, 1e-5, 1e-6, f"buffer {k}")


@pytest.mark.parametrize("name", sorted(FX["difformer"]))
def test_difformer_oracle_matches_reference_with_its_masks(monkeypatch, name):
    from test_difformer import FIXTURE
    case = FX["difformer"][name]
    cfg, sd, x, ei, lw, exp0 = FIXTURE[case["base"]]
    cfg = dict(cfg, dropout=case["dropout"])
    replay = MaskReplayer(_stored_masks(case), scale="ref")
    monkeypatch.setattr(D, "_dropout", replay)
    sdg = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    xg = x.clone().requires_grad_(True)
    out = D.difformer_forward(cfg, sdg, xg, ei, training=True)
    replay.finish()
    _close(out, case["out_train"], 1e-5, 1e-6, "train output")
    assert (case["out_train"] - exp0["out_train"]).abs().max() > 100 * (1e-6 + 1e-5 * exp0["out_train"].abs().max())
    (out * lw).sum().backward()
    _close(xg.grad, case["grad_x"], 2e-4, 1e-6, "grad x")
    for k, g in _unflat(case["grads"]).items():
        _close(sdg[k].grad, g, 2e-4, 2e-5, f"grad {k}")


# ------------------------------------------------------------------------------------------------
# engine schedules (emulated kernels) against the oracles with the kernels' masks replayed
# ------------------------------------------------------------------------------------------------
SEED = 0x1234_5678_9ABC


def expected_calls(cfg) -> int:
    """Dropout calls of one training forward: 1 + layers per TransConv / GraphConv, layers - 1 for the GCN backbone."""
    n = 1 + cfg["trans_num_layers"] if cfg["trans_dropout"] > 0 else 0
    if cfg["use_graph"]:
        if cfg["variant"] == "medium":
            n += cfg["gcn_num_layers"] - 1 if cfg["gcn_dropout"] > 0 else 0
        elif cfg["gnn_dropout"] > 0:
            n += 1 + cfg["gnn_num_layers"]
    return n


def _cfg_from_oracle(c):
    from test_schedule_emulated import _cfg_from_oracle as f
    return f(c)


def run_sgformer_pair(monkeypatch, ocfg, sd, x, ei, lw, rtol_out, atol_out, rtol_g, atol_g):
    """SGFormerFn on the emulated kernels in training mode (seed fixed, dropout calls recorded) against the oracle with those
    masks replayed at the kernels' scale."""
    monkeypatch.setattr(E, "K", kernel_emu)
    monkeypatch.setattr(Fn, "K", kernel_emu)
    monkeypatch.setattr(E, "next_seed", lambda: SEED)
    rec = DropoutRecorder(monkeypatch, kernel_emu)
    cfg = _cfg_from_oracle(ocfg)
    names = tuple(sd.keys())

    def leafs():
        return {k: (v.clone().requires_grad_(True) if v.is_floating_point() and "running" not in k else v.clone()) for k, v in sd.items()}

    got_p = leafs()
    xg = x.clone().requires_grad_(True)
    graph = kernel_emu.EmuGraph(ei, x.shape[0], 1 if cfg["variant"] == "medium" else 0) if cfg["use_graph"] else None
    out = Fn.SGFormerFn.apply(xg, graph, cfg, E.FP32, True, SINGLE, names, *[got_p[k] for k in names])
    (out * lw).sum().backward()
    assert len(rec.calls) == expected_calls(ocfg), [(c.fn, c.rows, c.h) for c in rec.calls]
    replay = MaskReplayer(rec.masks(), scale="kernel")
    monkeypatch.setattr(O, "_dropout", replay)
    ref_p = leafs()
    xr = x.clone().requires_grad_(True)
    stats = {}
    ref = O.sgformer_forward(ocfg, ref_p, xr, ei, training=True, stats_out=stats)
    replay.finish()
    (ref * lw).sum().backward()
    _close(out, ref, rtol_out, atol_out, "logits")
    _close(xg.grad, xr.grad, rtol_g, atol_g, "grad x")
    for k in names:
        if ref_p[k].is_floating_point() and ref_p[k].grad is not None:
            assert got_p[k].grad is not None, f"missing grad {k}"
            _close(got_p[k].grad, ref_p[k].grad, rtol_g, atol_g, f"grad {k}")
    for k, v in stats.items():
        if "running" in k:
            _close(got_p[k], v, 1e-5, 1e-6, f"buffer {k}")
    return out.detach(), ref.detach()


@pytest.mark.parametrize("name", sorted(FX["sgformer"]))
def test_sgformer_schedule_with_dropout_matches_oracle(monkeypatch, name):
    case = FX["sgformer"][name]
    fx = torch.load(os.path.join(GOLD, case["base"]), weights_only=False)
    ocfg = dict(fx["cfg"], **case["rates"])
    out, ref = run_sgformer_pair(monkeypatch, ocfg, fx["state_dict"], fx["x"], fx["edge_index"], fx["loss_weight"],
                                 2e-5, 2e-6, 5e-4, 3e-5)
    with torch.no_grad():
        ref0 = O.sgformer_forward(fx["cfg"], fx["state_dict"], fx["x"], fx["edge_index"], training=True)
    assert (ref - ref0).abs().max() > 100 * (2e-6 + 2e-5 * ref.abs().max()), "dropout changed nothing"


@pytest.mark.parametrize("variant", ["large", "100M", "medium"])
def test_deep_single_head_schedule_with_dropout_matches_oracle(monkeypatch, variant):
    """Three Gram-form attention layers and three graph layers: every layer's backward must recompute its own forward's mask."""
    n, d, h, c = 40, 6, 16, 3
    if variant == "medium":
        ocfg = O.make_config("medium", d, h, c, num_layers=3, num_heads=1, alpha=0.3, dropout=0.5, gcn_num_layers=3,
                             gcn_dropout=0.6, graph_weight=0.6)
    else:
        ocfg = O.make_config(variant, d, h, c, trans_num_layers=3, trans_num_heads=1, trans_dropout=0.5, gnn_num_layers=3,
                             gnn_dropout=0.6, gnn_use_init=variant == "100M", graph_weight=0.6)
    sd = O.init_state_dict(ocfg, seed=3)
    g = torch.Generator().manual_seed(4)
    ei = torch.stack([torch.randint(0, n, (3 * n,), generator=g), torch.randint(0, n, (3 * n,), generator=g)])
    run_sgformer_pair(monkeypatch, ocfg, sd, torch.randn(n, d, generator=g), torch.cat([ei, ei.flip(0)], 1),
                      torch.randn(n, c, generator=g), 2e-5, 2e-6, 5e-4, 3e-5)


def run_difformer_pair(monkeypatch, cfg, sd, x, ei, lw):
    monkeypatch.setattr(E, "K", kernel_emu_difformer)
    monkeypatch.setattr(Fn, "K", kernel_emu_difformer)
    monkeypatch.setattr(E, "next_seed", lambda: SEED)
    rec = DropoutRecorder(monkeypatch, kernel_emu_difformer)
    names = tuple(sd.keys())
    params = [sd[k].clone().requires_grad_(True) for k in names]
    xg = x.clone().requires_grad_(True)
    graph = kernel_emu_difformer.EmuGraph(ei, x.shape[0], 0) if cfg["use_graph"] else None
    out = Fn.DIFFormerFn.apply(xg, graph, cfg, E.FP32, True, names, *params)
    (out * lw).sum().backward()
    assert len(rec.calls) == 1 + cfg["num_layers"]
    replay = MaskReplayer(rec.masks(), scale="kernel")
    monkeypatch.setattr(D, "_dropout", replay)
    sdr = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    xr = x.clone().requires_grad_(True)
    ref = D.difformer_forward(cfg, sdr, xr, ei, training=True)
    replay.finish()
    (ref * lw).sum().backward()
    _close(out, ref, 2e-5, 2e-6, "logits")
    _close(xg.grad, xr.grad, 5e-4, 3e-5, "grad x")
    for k, p in zip(names, params):
        if sdr[k].grad is None:
            assert p.grad is None, k
        else:
            _close(p.grad, sdr[k].grad, 5e-4, 3e-5, f"grad {k}")
    return out.detach(), ref.detach()


@pytest.mark.parametrize("name", sorted(FX["difformer"]))
def test_difformer_schedule_with_dropout_matches_oracle(monkeypatch, name):
    from test_difformer import FIXTURE
    case = FX["difformer"][name]
    cfg, sd, x, ei, lw, _ = FIXTURE[case["base"]]
    run_difformer_pair(monkeypatch, dict(cfg, dropout=case["dropout"]), sd, x, ei, lw)


# ------------------------------------------------------------------------------------------------
# property: random configurations with dropout on
# ------------------------------------------------------------------------------------------------
from hypothesis import HealthCheck, given, settings  # noqa: E402
from hypothesis import strategies as st  # noqa: E402


@settings(max_examples=30, deadline=None, suppress_health_check=list(HealthCheck))
@given(variant=st.sampled_from(["large", "100M", "medium"]), n=st.integers(6, 70), h=st.sampled_from([8, 16]),
       heads=st.sampled_from([1, 2]), seed=st.integers(0, 10 ** 6), flags=st.lists(st.booleans(), min_size=9, max_size=9),
       aggregate=st.sampled_from(["add", "cat"]), layers=st.integers(0, 3), tlayers=st.integers(0, 2),
       p_t=st.sampled_from([0.0, 0.2, 0.5, 0.6]), p_g=st.sampled_from([0.0, 0.2, 0.5, 0.6]))
def test_schedule_property_with_dropout(variant, n, h, heads, seed, flags, aggregate, layers, tlayers, p_t, p_g):
    d, c = 5, 3
    use_weight = flags[0] or heads > 1
    if variant == "medium":
        ocfg = O.make_config("medium", d, h, c, num_layers=tlayers, num_heads=heads, alpha=0.3, dropout=p_t, use_bn=flags[1],
                             use_residual=flags[2], use_weight=use_weight, gcn_num_layers=layers + 1, gcn_dropout=p_g,
                             gcn_use_bn=flags[3], graph_weight=0.7, aggregate=aggregate, use_graph=True)
    else:
        kw = dict(trans_num_layers=tlayers, trans_num_heads=heads, trans_dropout=p_t, trans_use_bn=flags[1],
                  trans_use_residual=flags[2], trans_use_weight=use_weight, trans_use_act=flags[4], gnn_num_layers=layers,
                  gnn_dropout=p_g, gnn_use_weight=flags[5], gnn_use_init=flags[6], gnn_use_bn=flags[3], gnn_use_residual=flags[7],
                  gnn_use_act=flags[8], graph_weight=0.7, aggregate=aggregate, use_graph=True)
        if variant == "100M":
            kw["alpha"] = 0.3
        ocfg = O.make_config(variant, d, h, c, **kw)
    sd = O.init_state_dict(ocfg, seed=seed)
    g = torch.Generator().manual_seed(seed)
    ei = torch.stack([torch.randint(0, n, (3 * n,), generator=g), torch.randint(0, n, (3 * n,), generator=g)])
    ei = torch.cat([ei, ei.flip(0)], 1)
    x = torch.randn(n, d, generator=g)
    lw = torch.randn(n, c, generator=g)
    with pytest.MonkeyPatch.context() as mp:
        run_sgformer_pair(mp, ocfg, sd, x, ei, lw, 1e-4, 1e-5, 2e-3, 2e-4)


@settings(max_examples=15, deadline=None, suppress_health_check=list(HealthCheck))
@given(n=st.integers(5, 60), h=st.sampled_from([8, 16]), layers=st.integers(1, 3), p=st.sampled_from([0.2, 0.5, 0.6]),
       flags=st.lists(st.booleans(), min_size=5, max_size=5), gw=st.sampled_from([-1.0, 0.3]), seed=st.integers(0, 10 ** 6))
def test_difformer_schedule_property_with_dropout(n, h, layers, p, flags, gw, seed):
    cfg = D.make_config(6, h, 3, num_layers=layers, dropout=p, use_bn=flags[0], use_residual=flags[1], use_weight=flags[2],
                        use_graph=flags[3], use_source=flags[4], graph_weight=gw)
    sd = D.init_state_dict(cfg, seed=seed)
    g = torch.Generator().manual_seed(seed)
    ei = torch.stack([torch.randint(0, n, (3 * n,), generator=g), torch.randint(0, n, (3 * n,), generator=g)])
    x = torch.randn(n, 6, generator=g)
    lw = torch.randn(n, 3, generator=g)
    with pytest.MonkeyPatch.context() as mp:
        run_difformer_pair(mp, cfg, sd, x, ei, lw)
