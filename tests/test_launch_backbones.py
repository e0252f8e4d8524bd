"""Which GAT / GCN classes the reference's medium parse.py resolves under `python -m sgformer_b200.launch --variant medium`, with
and without `--native-backbones`.  The reference's import order is restated by stub modules: parse.py star-imports models, the
drop-in ours and graphtrans (which defines its own GCN)."""
import json
import os
import sys

import pytest

STUBS = {
    "models.py": "class GAT:\n    pass\n\n\nclass GCN:\n    pass\n",
    "graphtrans.py": "class GCN:\n    pass\n",
    "parse.py": "from models import *\nfrom ours import *\nfrom graphtrans import *\n",
    "main.py": ("import json, sys\nfrom parse import *\nimport parse\n"
                "json.dump({k: getattr(parse, k).__module__ for k in ('GAT', 'GCN', 'SGFormer')}, open(sys.argv[1], 'w'))\n"),
}


@pytest.mark.parametrize("native", [False, True])
def test_backbone_resolution(tmp_path, monkeypatch, native):
    from sgformer_b200 import launch
    for name, text in STUBS.items():
        (tmp_path / name).write_text(text)
    monkeypatch.setattr(sys, "path", list(sys.path))
    monkeypatch.setattr(sys, "argv", list(sys.argv))
    monkeypatch.chdir(os.getcwd())
    for m in ("models", "parse", "ours", "graphtrans"):
        monkeypatch.delitem(sys.modules, m, raising=False)
    out = tmp_path / "resolved.json"
    try:
        launch.main(["--variant", "medium"] + (["--native-backbones"] if native else []) + [str(tmp_path / "main.py"), str(out)])
    finally:
        for m in ("models", "parse", "ours", "graphtrans"):
            sys.modules.pop(m, None)
    got = json.loads(out.read_text())
    assert got["SGFormer"] == "sgformer_b200.medium"
    if native:
        assert got == {"GAT": "sgformer_b200.medium", "GCN": "sgformer_b200.medium", "SGFormer": "sgformer_b200.medium"}
    else:
        assert got["GAT"] == "models" and got["GCN"] == "graphtrans"


def test_medium_star_export_leaves_gat_alone():
    import sgformer_b200.medium as M
    assert "GAT" not in M.__all__ and "GATConv" not in M.__all__
