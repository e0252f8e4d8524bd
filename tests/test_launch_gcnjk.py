"""Which GCNJK class the reference's medium parse.py resolves under `python -m sgformer_b200.launch --variant medium`, with and
without `--native-backbones`.  Stub modules restate the reference's import order: parse.py star-imports models (which defines
GCNJK), the drop-in ours and graphtrans."""
import json
import os
import sys

import pytest

STUBS = {
    "models.py": "class GAT:\n    pass\n\n\nclass GCN:\n    pass\n\n\nclass GCNJK:\n    pass\n",
    "graphtrans.py": "class GCN:\n    pass\n",
    "parse.py": "from models import *\nfrom ours import *\nfrom graphtrans import *\n",
    "main.py": ("import json, sys\nfrom parse import *\nimport parse, models\n"
                "json.dump({'parse': parse.GCNJK.__module__, 'models': models.GCNJK.__module__}, open(sys.argv[1], 'w'))\n"),
}


@pytest.mark.parametrize("native", [False, True])
def test_gcnjk_resolution(tmp_path, monkeypatch, native):
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
    want = "sgformer_b200.medium" if native else "models"
    assert json.loads(out.read_text()) == {"parse": want, "models": want}
