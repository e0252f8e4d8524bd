"""SGFormerGAT (medium/ablation/oursGAT.py), the GAT-attention ablation, without a GPU: the module tree, seeded initialisation and
reset_parameters against the fixture from the unmodified oursGAT.py (tests/make_golden_gat_attention.py), the plain-torch
oracle against the fixture, the TransConv schedule on the emulated attention kernels (tests/kernel_emu_attn_softmax.py) against
the fixture's fp64 run (dk padding, the two-stage v, the unused layer weights left without a gradient), the same emulated schedule
for the softmax ablation, which SGFormerGAT the launcher resolves, and the refused options.  "GAT attention" here is scaled
dot-product attention; the GAT backbone is tested in test_gat*.py."""
import json
import os
import sys

import pytest
import torch

import kernel_emu
import kernel_emu_attn_softmax
from oracle import gat_attention_oracle as O
from sgformer_b200 import ablation, ablation_gat, medium
from sgformer_b200 import engine as E
from sgformer_b200 import functional as Fn
from sgformer_b200.config import make_config
from sgformer_b200.dist import SINGLE, Comm

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sgformer_gat_attention.pt")
GD = torch.load(GOLDEN, weights_only=False)
CASES = sorted(GD["cases"])


def _native(cls, cfg, d, c, graph=True):
    h = cfg["hidden"]
    gnn = medium.GCN(d, h, h, num_layers=2, dropout=0.0, use_bn=True) if cfg["use_graph"] and graph else None
    return cls(d, h, c, num_layers=2, num_heads=cfg["heads"], alpha=0.5, dropout=0.0, use_bn=cfg["use_bn"],
               use_residual=cfg["use_residual"], use_weight=cfg["use_weight"], use_graph=cfg["use_graph"], graph_weight=0.8,
               gnn=gnn, aggregate=cfg["aggregate"])


def _parse_call(d=12, h=16, c=5, heads=2, use_weight=True):
    # medium/ablation/parse.py:110-112
    return ablation_gat.SGFormerGAT(d, h, c, num_layers=2, alpha=0.5, dropout=0.3, num_heads=heads, use_bn=True,
                                    use_residual=True, use_graph=False, use_weight=use_weight, use_act=False, graph_weight=0.8,
                                    gnn=None, aggregate="add")


# ---- module structure ------------------------------------------------------------------------------------------------------
def test_fixture_covers_the_cases():
    cfgs = [GD["cases"][n]["config"] for n in CASES]
    assert {c["heads"] for c in cfgs} >= {1, 2, 3, 4}
    assert any(c["hidden"] // c["heads"] == 5 for c in cfgs)
    assert {c["use_weight"] for c in cfgs} == {True, False} and not all(c["use_residual"] for c in cfgs)
    assert not all(c["use_bn"] for c in cfgs) and {c["aggregate"] for c in cfgs if c["use_graph"]} == {"add", "cat"}
    assert max(GD["cases"][n].get("max_abs_score", 0.0) for n in CASES) > 100.0
    assert GD["get_attentions_error"] == "ValueError"


@pytest.mark.parametrize("name", CASES)
def test_state_dict_keys_shapes_and_order(name):
    rec = GD["cases"][name]
    d, c = GD["x"].shape[1], rec["state_dict"]["fc.weight"].shape[0]
    m = _native(ablation_gat.SGFormerGAT, rec["config"], d, c)
    sd = m.state_dict()
    assert list(sd.keys()) == list(rec["init_state_dict"].keys())
    assert {k: tuple(v.shape) for k, v in sd.items()} == {k: tuple(v.shape) for k, v in rec["init_state_dict"].items()}
    m.load_state_dict(rec["state_dict"], strict=True)


@pytest.mark.parametrize("name", CASES)
def test_seeded_init_and_reset_parameters_match_the_reference(name):
    rec = GD["cases"][name]
    order = [n for n, *_ in __import__("make_golden_gat_attention").CASES]
    i = order.index(name)
    d, c = GD["x"].shape[1], rec["state_dict"]["fc.weight"].shape[0]
    torch.manual_seed(100 + i)
    m = _native(ablation_gat.SGFormerGAT, rec["config"], d, c)
    for k, v in m.state_dict().items():
        assert torch.equal(v, rec["init_state_dict"][k]), k
    torch.manual_seed(200 + i)
    m.reset_parameters()
    for k, v in m.state_dict().items():
        assert torch.equal(v, rec["reset_state_dict"][k]), k


def test_params_groups_and_layer_types():
    m = _parse_call()
    assert [p.shape for p in m.params1] == [p.shape for p in m.trans_conv.parameters()]
    assert len(m.params2) == 2
    layer = m.trans_conv.convs[0]
    assert isinstance(layer, ablation_gat.TransConvLayer) and isinstance(layer.attention, ablation_gat.TransConvLayerGAT)
    assert isinstance(layer.attention.attention, ablation_gat.GATAttention) and layer.attention.attention.dk == 8
    keys = _parse_call(use_weight=False).state_dict()
    assert "trans_conv.convs.0.Wv.weight" not in keys and "trans_conv.convs.0.attention.Wv.weight" not in keys
    assert "trans_conv.convs.0.attention.attention.Wv.weight" in keys


# ---- refusals ----------------------------------------------------------------------------------------------------------------
def test_config_switch_and_unknown_attention():
    assert _parse_call()._cfg()["trans_attention"] == "gat"
    assert _parse_call().trans_conv._cfg()["trans_attention"] == "gat"
    assert make_config("medium", 4, 8, 2, trans_attention="gat")["trans_attention"] == "gat"
    with pytest.raises(ValueError, match="unknown TransConv attention"):
        make_config("medium", 4, 8, 2, trans_attention="nodeformer")


def test_get_attentions_raises_value_error():
    m = _parse_call()
    with pytest.raises(ValueError, match="no attention matrices"):
        m.get_attentions(torch.randn(5, 12))
    with pytest.raises(ValueError, match="no attention matrices"):
        m.trans_conv.convs[0](torch.randn(5, 16), torch.randn(5, 16), output_attn=True)
    cfg = m._cfg()
    with pytest.raises(ValueError, match="no attention matrices"):
        E.trans_attentions({}, cfg, None, E.FP32, False)


def test_row_sharding_raises(monkeypatch):
    class _Active(Comm):
        def __init__(self):
            pass

        @property
        def active(self):
            return True

    monkeypatch.setattr(E, "K", kernel_emu_attn_softmax.module())
    m = _parse_call()
    names, tensors = m.trans_conv._flat("trans_conv.")
    P = dict(zip(names, [t.detach() for t in tensors]))
    xin = kernel_emu.pack_operand(torch.randn(7, 12), False, 3)
    with pytest.raises(NotImplementedError, match="row sharding of the gat attention"):
        E.trans_forward(P, m.trans_conv._cfg(), xin, E.FP32, True, 1, None, comm=_Active())


# ---- oracle against the fixture ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-10), (torch.float32, 1e-5)])
@pytest.mark.parametrize("name", [n for n in CASES if not GD["cases"][n]["config"]["use_graph"]])
def test_oracle_matches_fixture(name, dtype, tol):
    rec = GD["cases"][name]
    cfg = rec["config"]
    ref = rec["fp64" if dtype == torch.float64 else "fp32"]
    sd = {k: v.to(dtype).requires_grad_() for k, v in rec["state_dict"].items()}
    xg = GD["x"].to(dtype).detach().clone().requires_grad_()
    out = O.sgformer_gat(sd, xg, 2, cfg["heads"], use_bn=cfg["use_bn"], use_residual=cfg["use_residual"],
                         use_weight=cfg["use_weight"])
    torch.testing.assert_close(out.detach(), ref["train_logits"], rtol=tol, atol=tol)
    (out * rec["wout"].to(dtype)).sum().backward()
    torch.testing.assert_close(xg.grad, ref["grad_x"], rtol=tol, atol=tol)
    assert sorted(k for k, v in sd.items() if v.grad is None) == sorted(ref["none_grads"])
    for k, g in ref["grads"].items():
        torch.testing.assert_close(sd[k].grad, g, rtol=tol, atol=tol, msg=lambda m: f"{name} {k}: {m}")


def test_one_head_weights_are_exactly_one():
    g = torch.Generator().manual_seed(0)
    q, k = (30 * torch.randn(9, 1, 5, generator=g, dtype=torch.float64) for _ in range(2))
    v = torch.randn(9, 1, 7, generator=g, dtype=torch.float64)
    o = O.gat_attention(q, k, v)
    torch.testing.assert_close(o, v.sum(0, keepdim=True).expand_as(o), rtol=0, atol=1e-12)     # one head: every weight is 1


# ---- the schedule on the emulated kernels --------------------------------------------------------------------------------------
def _relerr(a, b, floor=1e-30):
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / max(b.norm().item(), floor)).item()


def _check_grads(m, ref, tol):
    """Every parameter gradient against the reference's (None where the reference's is None).  Gradients that are zero in exact
    arithmetic or nearly so (a conv bias in front of a training BatchNorm, q / k under a saturated or uniform softmax over the
    heads) carry fp32 rounding only: errors are measured against at least 1% of the largest gradient's norm."""
    floor = 1e-2 * max(g.norm().item() for g in ref["grads"].values())
    for k, p in m.named_parameters():
        if p.grad is None:
            assert k not in ref["grads"], k
            continue
        assert _relerr(p.grad, ref["grads"][k], floor) < tol, k


def _run_emulated(m, x, ei, training, monkeypatch):
    monkeypatch.setattr(E, "K", kernel_emu_attn_softmax.module())
    monkeypatch.setattr(Fn, "K", E.K)
    m.train(training)
    tn, tt = m.trans_conv._flat("trans_conv.")
    names = tuple(tn) + ("fc.weight", "fc.bias")
    tensors = list(tt) + [m.fc.weight, m.fc.bias]
    if not m.use_graph:
        return Fn.SGFormerFn.apply(x, None, m._cfg(), E.FP32, training, SINGLE, names, *tensors)
    gn, gt = medium._gcn_flat(m.gnn, "gnn.")
    cfg = m._cfg(len(m.gnn.convs), float(m.gnn.dropout), bool(m.gnn.use_bn))
    graph = kernel_emu.EmuGraph(ei, x.shape[0], 1)
    return Fn.SGFormerFn.apply(x, graph, cfg, E.FP32, training, SINGLE, names + tuple(gn), *tensors, *gt)


@pytest.mark.parametrize("name", CASES)
def test_emulated_gat_schedule_matches_fp64_reference(name, monkeypatch):
    """The TransConv schedule (dk padded to the kernels' 16-byte blocks, [q | k | u] in one GEMM, v = Wv_att u + b) against the
    reference's own fp64 run; the layers' unused Wq / Wk / Wv get no gradient."""
    rec = GD["cases"][name]
    cfg = rec["config"]
    d, c = GD["x"].shape[1], rec["state_dict"]["fc.weight"].shape[0]
    m = _native(ablation_gat.SGFormerGAT, cfg, d, c)
    m.load_state_dict(rec["state_dict"])
    ref = rec["fp64"]
    tol = 1e-4 if cfg["wq_scale"] == 1.0 else 1e-3      # |s| ~ 120 scales the fp32 rounding of the scores in the weights
    out = _run_emulated(m, GD["x"], GD["edge_index"], False, monkeypatch)
    assert _relerr(out, ref["eval_logits"]) < tol
    x = GD["x"].clone().requires_grad_()
    out = _run_emulated(m, x, GD["edge_index"], True, monkeypatch)
    assert _relerr(out, ref["train_logits"]) < tol
    (out * rec["wout"]).sum().backward()
    assert _relerr(x.grad, ref["grad_x"]) < tol
    got_none = sorted(k for k, p in m.named_parameters() if p.grad is None)
    assert got_none == sorted(ref["none_grads"])
    assert any(".convs.0.Wq." in k for k in got_none)
    _check_grads(m, ref, tol)


def test_emulated_gat_schedule_one_head_has_no_qk_gradient(monkeypatch):
    rec = GD["cases"]["h1"]
    m = _native(ablation_gat.SGFormerGAT, rec["config"], GD["x"].shape[1], rec["state_dict"]["fc.weight"].shape[0])
    m.load_state_dict(rec["state_dict"])
    out = _run_emulated(m, GD["x"], GD["edge_index"], True, monkeypatch)
    (out * rec["wout"]).sum().backward()
    for i in range(2):
        for w in ("Wq", "Wk"):
            g = m.trans_conv.convs[i].attention.attention.get_submodule(w).weight.grad
            assert g.abs().max() < 1e-6, (i, w)


# the softmax ablation (SGFormerSOFT) on the same emulated kernels, against its own fixture made from oursSOFT.py
SOFT = torch.load(os.path.join(os.path.dirname(GOLDEN), "sgformer_softmax.pt"), weights_only=False)


@pytest.mark.parametrize("name", sorted(SOFT["cases"]))
def test_emulated_softmax_schedule_matches_fp64_reference(name, monkeypatch):
    rec = SOFT["cases"][name]
    cfg = dict(rec["config"], hidden=rec["state_dict"]["trans_conv.fcs.0.weight"].shape[0])
    d, c = SOFT["x"].shape[1], rec["state_dict"]["fc.weight"].shape[0]
    m = _native(ablation.SGFormerSOFT, cfg, d, c)
    m.load_state_dict(rec["state_dict"])
    ref = rec["fp64"]
    x = SOFT["x"].clone().requires_grad_()
    out = _run_emulated(m, x, SOFT["edge_index"], True, monkeypatch)
    assert _relerr(out, ref["train_logits"]) < 1e-5
    (out * rec["wout"]).sum().backward()
    assert _relerr(x.grad, ref["grad_x"]) < 1e-4
    _check_grads(m, ref, 1e-4)
    if not m.use_graph:       # get_attentions through engine.trans_attentions on the emulated probs
        with torch.no_grad():
            tn, tt = m.trans_conv._flat("trans_conv.")
            atts = E.trans_attentions(dict(zip(tn, tt)), m.trans_conv._cfg(), kernel_emu.pack_operand(SOFT["x"], False, 3),
                                      E.FP32, False)
        assert _relerr(torch.stack(atts), ref["attentions"]) < 1e-5


# ---- launcher ------------------------------------------------------------------------------------------------------------------
def test_launcher_resolves_native_sgformer_gat(tmp_path, monkeypatch):
    from sgformer_b200 import launch
    stubs = {
        "models.py": "class GAT:\n    pass\n\n\nclass GCN:\n    pass\n\n\nclass GCNJK:\n    pass\n",
        "parse.py": "from models import *\nfrom ours import *\nfrom oursSOFT import *\nfrom oursGAT import *\n",
        "main.py": ("import json, sys\nfrom parse import *\nimport parse\n"
                    "json.dump({'gat_attention': parse.SGFormerGAT.__module__, 'soft': parse.SGFormerSOFT.__module__, "
                    "'ours': parse.SGFormer.__module__, 'gcn': parse.GCN.__module__, 'gat': parse.GAT.__module__, "
                    "'gcnjk': parse.GCNJK.__module__, 'layer': parse.TransConvLayer.__module__}, open(sys.argv[1], 'w'))\n"),
    }
    for name, text in stubs.items():
        (tmp_path / name).write_text(text)
    mods = ("models", "parse", "ours", "oursSOFT", "oursGAT")
    out = tmp_path / "resolved.json"
    # the medium drop-in ours.py exports its GCN either way; GAT and GCNJK are the reference's unless --native-backbones
    for native, want in ((True, "sgformer_b200.medium"), (False, "models")):
        monkeypatch.setattr(sys, "path", list(sys.path))
        monkeypatch.setattr(sys, "argv", list(sys.argv))
        monkeypatch.chdir(os.getcwd())
        for m in mods:
            monkeypatch.delitem(sys.modules, m, raising=False)
        try:
            launch.main(["--variant", "medium"] + (["--native-backbones"] if native else []) + [str(tmp_path / "main.py"), str(out)])
        finally:
            for m in mods:
                sys.modules.pop(m, None)
        got = json.loads(out.read_text())
        assert got == {"gat_attention": "sgformer_b200.ablation_gat", "soft": "sgformer_b200.ablation", "ours": "sgformer_b200.medium",
                       "gcn": "sgformer_b200.medium", "gat": want, "gcnjk": want, "layer": "sgformer_b200.ablation_gat"}, native


# ---- ABI -----------------------------------------------------------------------------------------------------------------------
def test_attn_softmax_args_layout_matches_the_header(tmp_path):
    """_lib.AttnSoftmaxArgs mirrors sgf_attn_softmax_args field by field: a C compiler's offsets and size of the header's struct."""
    import ctypes
    import shutil
    import subprocess
    from sgformer_b200 import _lib
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    fields = [f for f, *_ in _lib.AttnSoftmaxArgs._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include <stdint.h>\n#include "sgformer_b200.h"\nint main(void) {\n'
                   + "".join(f'    printf("%zu\\n", offsetof(sgf_attn_softmax_args, {f}));\n' for f in fields)
                   + '    printf("%zu\\n", sizeof(sgf_attn_softmax_args));\n    return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", os.path.join(root, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    want = [getattr(_lib.AttnSoftmaxArgs, f).offset for f in fields] + [ctypes.sizeof(_lib.AttnSoftmaxArgs)]
    assert got == want
