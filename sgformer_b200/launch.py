"""Run an UNMODIFIED reference training script with the H100 `ours.py` in front of its own:

    python -m sgformer_b200.launch --variant large /path/to/SGFormer/large/main-batch.py --method sgformer --dataset pokec ...

sys.path becomes [dropin/<variant>, <script dir>, ...] so `from ours import *` in the reference's parse.py picks the
drop-in while every other sibling import (logger, dataset, data_utils, eval, parse) stays the reference's."""
import argparse
import os
import runpy
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m sgformer_b200.launch")
    ap.add_argument("--variant", required=True, choices=["large", "medium", "100M"])
    ap.add_argument("--precision", choices=["bf16", "fp32"], default=None)
    ap.add_argument("--native-backbones", action="store_true",
                    help="medium: make the GAT, GCN and GCNJK that the reference's parse.py builds backbones from resolve to "
                         "sgformer_b200.medium.GAT / GCN / GCNJK, so that --backbone gat|gcn|gcnjk (and --method gat|gcn|gcnjk) "
                         "run on the kernels; "
                         "large: make parse.py's GCN and GAT (from gnns.py) resolve to sgformer_b200.large_gnns.GCN / GAT, so that "
                         "--method gcn|gat runs on the kernels (models.py / gnns.py still import torch_geometric)")
    ap.add_argument("script")
    ap.add_argument("script_args", nargs=argparse.REMAINDER)
    a = ap.parse_args(argv)
    if a.precision:
        os.environ["SGFORMER_B200_PRECISION"] = a.precision
    script = os.path.abspath(a.script)
    sdir = os.path.dirname(script)
    sys.path[:0] = [os.path.join(HERE, "dropin", a.variant), sdir]
    sys.argv = [script] + a.script_args
    os.chdir(sdir)
    if a.native_backbones:
        if a.variant == "100M":
            ap.error("--native-backbones applies to --variant medium and large")
        # parse.py star-imports models (medium) / gnns (large), ours, ... (medium's graphtrans has a GCN of its own that shadows
        # models.GCN); parse_method looks the classes up in parse's namespace, so that is where they are replaced (main.py's
        # `from parse import ...` then reuses this module)
        if a.variant == "medium":
            import models as gnn_mod
            from . import medium as native
        else:
            import gnns as gnn_mod
            from . import large_gnns as native
        import parse
        for mod in (gnn_mod, parse):
            mod.GAT, mod.GCN = native.GAT, native.GCN
            if a.variant == "medium":
                mod.GCNJK = native.GCNJK
    runpy.run_path(script, run_name="__main__")


if __name__ == "__main__":
    main()
