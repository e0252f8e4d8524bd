"""SGFormerSOFT (medium/ablation/oursSOFT.py) without a GPU: the module tree and state_dict keys that parse.py's constructor call
builds, initialisation parity with the medium SGFormer (oursSOFT.py builds the same tree in the same order), the config switch,
the plain-torch oracle against a direct restatement and against the fixture from the unmodified oursSOFT.py, and which
SGFormerSOFT the launcher resolves."""
import json
import os
import sys

import pytest
import torch

from oracle import softmax_oracle as O
from sgformer_b200 import ablation, medium
from sgformer_b200.config import make_config


def _parse_call(d=12, h=16, c=5, layers=2, heads=2, use_weight=True, gnn=None, use_graph=False, aggregate="add"):
    # medium/ablation/parse.py:106-109
    return ablation.SGFormerSOFT(d, h, c, num_layers=layers, alpha=0.5, dropout=0.3, num_heads=heads, use_bn=True,
                                 use_residual=True, use_graph=use_graph, use_weight=use_weight, use_act=False,
                                 graph_weight=0.8, gnn=gnn, aggregate=aggregate)


def test_state_dict_keys_and_shapes():
    m = _parse_call()
    want = []
    for i in range(2):
        for w in ("Wk", "Wq", "Wv"):
            want += [f"trans_conv.convs.{i}.{w}.weight", f"trans_conv.convs.{i}.{w}.bias"]
    want += ["trans_conv.fcs.0.weight", "trans_conv.fcs.0.bias"]
    for i in range(3):
        want += [f"trans_conv.bns.{i}.weight", f"trans_conv.bns.{i}.bias"]
    want += ["fc.weight", "fc.bias"]
    sd = m.state_dict()
    assert list(sd.keys()) == want
    assert sd["trans_conv.convs.0.Wq.weight"].shape == (32, 16)
    assert isinstance(m.trans_conv.convs[0], ablation.TransConvLayer)
    nv = _parse_call(use_weight=False)
    assert not any("Wv" in k for k in nv.state_dict())


def test_init_matches_medium_sgformer():
    torch.manual_seed(3)
    a = _parse_call()
    torch.manual_seed(3)
    b = medium.SGFormer(12, 16, 5, num_layers=2, alpha=0.5, dropout=0.3, num_heads=2, use_graph=False)
    for (ka, va), (kb, vb) in zip(a.state_dict().items(), b.state_dict().items()):
        assert ka == kb and torch.equal(va, vb)
    assert [p.shape for p in a.params1] == [p.shape for p in b.params1]
    assert [p.shape for p in a.params2] == [p.shape for p in b.params2]


def test_params_groups_with_gnn_and_cat():
    gnn = medium.GCN(12, 16, 16, num_layers=2)
    m = _parse_call(gnn=gnn, use_graph=True, aggregate="cat")
    assert m.fc.weight.shape == (5, 32)
    assert len(m.params2) == len(list(gnn.parameters())) + 2
    m.reset_parameters()
    m.to("cpu")


def test_config_switch():
    assert make_config("medium", 4, 8, 2)["trans_attention"] == "linear"
    assert _parse_call()._cfg()["trans_attention"] == "softmax"
    assert medium.SGFormer(12, 16, 5)._cfg()["trans_attention"] == "linear"
    with pytest.raises(ValueError):
        make_config("medium", 4, 8, 2, trans_attention="soft")


@pytest.mark.parametrize("vh", [1, 3])
def test_oracle_softmax_matches_direct_formula(vh):
    g = torch.Generator().manual_seed(0)
    q, k = torch.randn(7, 3, 4, generator=g, dtype=torch.float64), torch.randn(7, 3, 4, generator=g, dtype=torch.float64)
    v = torch.randn(7, vh, 5, generator=g, dtype=torch.float64)
    o, att = O.softmax_attention(q, k, v)
    qn, kn = q / q.norm(), k / k.norm()
    s = torch.einsum("nhm,lhm->nlh", qn, kn)
    assert s.abs().max() <= 1.0             # the bound the kernels rely on
    p = torch.exp(s) / torch.exp(s).sum(2, keepdim=True)       # softmax over the heads, per (n, l)
    for h in range(3):
        torch.testing.assert_close(o[:, h], p[:, :, h] @ v[:, h if vh > 1 else 0], rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(att, p.mean(2), rtol=1e-12, atol=1e-12)


def test_launcher_resolves_native_sgformer_soft(tmp_path, monkeypatch):
    from sgformer_b200 import launch
    stubs = {
        "models.py": "class GAT:\n    pass\n\n\nclass GCN:\n    pass\n\n\nclass GCNJK:\n    pass\n",
        "parse.py": "from models import *\nfrom ours import *\nfrom oursSOFT import *\n",
        "main.py": ("import json, sys\nfrom parse import *\nimport parse\n"
                    "json.dump({'soft': parse.SGFormerSOFT.__module__, 'ours': parse.SGFormer.__module__, "
                    "'gcn': parse.GCN.__module__}, open(sys.argv[1], 'w'))\n"),
    }
    for name, text in stubs.items():
        (tmp_path / name).write_text(text)
    mods = ("models", "parse", "ours", "oursSOFT")
    monkeypatch.setattr(sys, "path", list(sys.path))
    monkeypatch.setattr(sys, "argv", list(sys.argv))
    monkeypatch.chdir(os.getcwd())
    for m in mods:
        monkeypatch.delitem(sys.modules, m, raising=False)
    out = tmp_path / "resolved.json"
    try:
        launch.main(["--variant", "medium", "--native-backbones", str(tmp_path / "main.py"), str(out)])
    finally:
        for m in mods:
            sys.modules.pop(m, None)
    assert json.loads(out.read_text()) == {"soft": "sgformer_b200.ablation", "ours": "sgformer_b200.medium",
                                           "gcn": "sgformer_b200.medium"}


# ---- against tests/golden/sgformer_softmax.pt (made from the unmodified oursSOFT.py by tests/make_golden_softmax.py) ----------
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sgformer_softmax.pt")


def _golden():
    return torch.load(GOLDEN, weights_only=False)


def _native_for(cfg, d, h, c):
    gnn = medium.GCN(d, h, h, num_layers=2, dropout=0.0, use_bn=True) if cfg["use_graph"] else None
    return ablation.SGFormerSOFT(d, h, c, num_layers=2, num_heads=cfg["heads"], alpha=0.5, dropout=0.0, use_bn=cfg["use_bn"],
                                 use_residual=cfg["use_residual"], use_weight=cfg["use_weight"], use_graph=cfg["use_graph"],
                                 graph_weight=0.8, gnn=gnn, aggregate=cfg["aggregate"])


def test_fixture_state_dicts_load_into_native_modules():
    gd = _golden()
    d, n = gd["x"].shape[1], gd["x"].shape[0]
    for name, rec in gd["cases"].items():
        sd = rec["state_dict"]
        h, c = sd["trans_conv.fcs.0.weight"].shape[0], sd["fc.weight"].shape[0]
        m = _native_for(rec["config"], d, h, c)
        m.load_state_dict(sd, strict=True)
        assert list(m.state_dict().keys()) == list(sd.keys()), name


def test_oracle_matches_fixture():
    """The oracle restates the reference's softmax over the head axis; with one head every weight is 1."""
    gd = _golden()
    x = gd["x"].double()
    for name, rec in gd["cases"].items():
        cfg = rec["config"]
        if cfg["use_graph"]:
            continue
        sd = {k: v.double().requires_grad_() for k, v in rec["state_dict"].items()}
        kw = dict(use_bn=cfg["use_bn"], use_residual=cfg["use_residual"], use_weight=cfg["use_weight"])
        atts = []
        O.trans_conv(sd, x, 2, cfg["heads"], attentions=atts, **kw)
        ref = rec["fp64"]
        torch.testing.assert_close(torch.stack(atts).detach(), ref["attentions"], rtol=1e-12, atol=1e-12)
        xg = x.clone().requires_grad_()
        out = O.sgformer_soft(sd, xg, 2, cfg["heads"], **kw)
        torch.testing.assert_close(out.detach(), ref["train_logits"], rtol=1e-10, atol=1e-10)
        (out * rec["wout"].double()).sum().backward()
        torch.testing.assert_close(xg.grad, ref["grad_x"], rtol=1e-10, atol=1e-10)
        for k, g in ref["grads"].items():
            torch.testing.assert_close(sd[k].grad, g, rtol=1e-10, atol=1e-12, msg=lambda m: f"{name} {k}: {m}")
    h1 = gd["cases"]["h1"]["fp64"]["attentions"]
    assert torch.equal(h1, torch.ones_like(h1))
