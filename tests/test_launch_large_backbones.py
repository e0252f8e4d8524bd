"""Which GCN / GAT classes the reference's large parse.py resolves under `python -m sgformer_b200.launch --variant large`, with and
without `--native-backbones`, and that `--variant 100M` still refuses the flag.  The reference's import order is restated by stub
modules: parse.py star-imports gnns and the drop-in ours."""
import json
import os
import sys

import pytest

STUBS = {
    "gnns.py": "class GAT:\n    pass\n\n\nclass GCN:\n    pass\n",
    "parse.py": "from gnns import *\nfrom ours import *\n",
    "main.py": ("import json, sys\nfrom parse import *\nimport parse, gnns\n"
                "json.dump({k: getattr(parse, k).__module__ for k in ('GAT', 'GCN', 'SGFormer')} | "
                "{'gnns.' + k: getattr(gnns, k).__module__ for k in ('GAT', 'GCN')}, open(sys.argv[1], 'w'))\n"),
}
MODS = ("gnns", "parse", "ours")


def _launch(tmp_path, monkeypatch, args):
    from sgformer_b200 import launch
    for name, text in STUBS.items():
        (tmp_path / name).write_text(text)
    monkeypatch.setattr(sys, "path", list(sys.path))
    monkeypatch.setattr(sys, "argv", list(sys.argv))
    monkeypatch.chdir(os.getcwd())
    for m in MODS:
        monkeypatch.delitem(sys.modules, m, raising=False)
    out = tmp_path / "resolved.json"
    try:
        launch.main(args + [str(tmp_path / "main.py"), str(out)])
    finally:
        for m in MODS:
            sys.modules.pop(m, None)
    return json.loads(out.read_text())


@pytest.mark.parametrize("native", [False, True])
def test_large_baseline_resolution(tmp_path, monkeypatch, native):
    got = _launch(tmp_path, monkeypatch, ["--variant", "large"] + (["--native-backbones"] if native else []))
    assert got["SGFormer"] == "sgformer_b200.large"
    want = "sgformer_b200.large_gnns" if native else "gnns"
    assert {k: v for k, v in got.items() if k != "SGFormer"} == {"GAT": want, "GCN": want, "gnns.GAT": want, "gnns.GCN": want}


def test_100M_refuses_native_backbones(tmp_path, monkeypatch):
    with pytest.raises(SystemExit):
        _launch(tmp_path, monkeypatch, ["--variant", "100M", "--native-backbones"])
