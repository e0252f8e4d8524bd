"""Shared case table, fp64/fp32 oracle runs and per-tensor checker for the schedule-switch tests — helper module, not collected.

`CASES` is a fixed pairwise covering of the SGFormer schedule switches (every value pair of two different switches that can
both take effect occurs in some case; `uncovered_pairs()` is asserted empty by tests/test_config_matrix_emulated.py), led by the
reference's own recipes.  `tests/test_gpu_config_matrix.py` runs it on the device at the recipes' widths,
`tests/test_config_matrix_emulated.py` runs the `small=True` view of it through the CPU emulation of the kernels.

Every gradient tensor is judged on its own scale against an fp64 run of the oracle: there is no term proportional to the
largest gradient of the model, so a small tensor (the attention's Wq / Wk gradients are O(1/N) of the others) cannot hide
behind a large one."""
import inspect
import itertools
import json
import os
import zlib
from collections import namedtuple

import torch

from oracle import sgformer_oracle as O
from sgformer_b200.config import make_config

# ------------------------------------------------------------------------------------------------
# the switch space
# ------------------------------------------------------------------------------------------------
FACTORS = dict(
    variant=("large", "100M", "medium"), tl=(0, 1, 2), heads=(1, 2), t_bn=(0, 1), t_res=(0, 1), t_w=(0, 1), t_act=(0, 1),
    gl=(0, 1, 2, 3), g_w=(0, 1), g_init=(0, 1), g_bn=(0, 1), g_res=(0, 1), g_act=(0, 1), agg=("add", "cat"), ug=(0, 1),
    gw=(0.3, 0.8), alpha=(0.3, 0.7),
)
# tl = trans_num_layers, gl = gnn_num_layers (medium: gcn_num_layers - 1), g_bn = gnn_use_bn (medium: gcn_use_bn), ug = use_graph

Case = namedtuple("Case", "name " + " ".join(FACTORS) + " h d c n hub sym")


def valid(a) -> bool:
    """num_heads > 1 needs the value projection (medium/ours.py:84); `cat` without a graph branch gives fc the wrong width;
    models.GCN always has an input and an output conv (medium/models.py:22-35), so the medium variant has gl >= 1."""
    return not (a["heads"] == 2 and not a["t_w"]) and not (a["agg"] == "cat" and not a["ug"]) and \
        not (a["variant"] == "medium" and a["gl"] == 0)


def active(a) -> set:
    """The switches that change what this configuration computes (a switch of a branch that does not run, of a layer stack
    of depth 0, or one the variant does not have, is inert and does not count towards the coverage)."""
    s = {"variant", "tl", "t_bn", "agg", "ug"}
    med = a["variant"] == "medium"
    if a["tl"] > 0:
        s |= {"heads", "t_res", "t_w"}
        if not med:
            s.add("t_act")          # medium/ours.py:183 never forwards use_act
        if a["t_res"] and a["variant"] != "large":
            s.add("alpha")          # large/ours.py:211 averages instead
    if a["ug"]:
        s.add("gl")
        if a["agg"] == "add":
            s.add("gw")
        s.add("g_bn")
        if not med and a["gl"] > 0:
            s |= {"g_init", "g_res", "g_act"}
            if not a["g_init"]:     # use_init applies W regardless of use_weight (large/ours.py:36-41)
                s.add("g_w")
    return s


_STRUCT = ("variant", "tl", "heads", "t_res", "t_w", "gl", "g_init", "agg", "ug")


def required_pairs() -> set:
    """{((f1, v1), (f2, v2))}: value pairs of two switches for which a valid configuration exists where both are active."""
    names = list(FACTORS)
    base = {f: FACTORS[f][-1] for f in names}
    req = set()
    for s in itertools.product(*[FACTORS[f] for f in _STRUCT]):
        a = dict(base, **dict(zip(_STRUCT, s)))
        if not valid(a):
            continue
        act = sorted(active(a), key=names.index)
        for f1, f2 in itertools.combinations(act, 2):
            for v1 in (FACTORS[f1] if f1 not in _STRUCT else (a[f1],)):
                for v2 in (FACTORS[f2] if f2 not in _STRUCT else (a[f2],)):
                    req.add(((f1, v1), (f2, v2)))
    return req


def covered_pairs(cases) -> set:
    names = list(FACTORS)
    cov = set()
    for c in cases:
        a = c._asdict()
        act = sorted(active(a), key=names.index)
        for f1, f2 in itertools.combinations(act, 2):
            cov.add(((f1, a[f1]), (f2, a[f2])))
    return cov


def uncovered_pairs(cases=None) -> list:
    return sorted(required_pairs() - covered_pairs(CASES if cases is None else cases), key=str)


# ------------------------------------------------------------------------------------------------
# the table.  Columns: name, then FACTORS in order, then hidden, d_in, classes, n, hub (one node with > 1024 in-edges and one
# with > 1024 out-edges: the segmented SpMM runs in the forward and in the transposed backward), sym (undirected edge list).
# h = 100 is not a multiple of 8: fp32 only.  Rows 0-6 are the reference's recipes (switches only; graph_weight as given there).
# ------------------------------------------------------------------------------------------------
_RECIPES = [
    # large/run.sh:2-5 (ogbn-arxiv)
    ("arxiv", "large", 1, 1, 1, 1, 1, 0, 3, 1, 0, 1, 1, 1, "add", 1, 0.5, 0.5, 256, 128, 40, 20011, 0, 1),
    # large/run.sh:8-12 (ogbn-proteins)
    ("proteins", "large", 1, 1, 1, 1, 1, 0, 2, 1, 0, 1, 1, 1, "add", 1, 0.5, 0.5, 64, 128, 2, 8200, 0, 1),
    # large/run.sh:15-19 (amazon2m)
    ("amazon2m", "large", 1, 1, 1, 1, 1, 0, 3, 1, 1, 1, 1, 1, "add", 1, 0.5, 0.5, 256, 100, 47, 8200, 1, 1),
    # large/run.sh:22-26 (pokec)
    ("pokec", "large", 1, 1, 1, 1, 1, 0, 2, 1, 1, 1, 1, 1, "add", 1, 0.5, 0.5, 64, 65, 2, 20011, 1, 0),
    # 100M/run.sh:3-7 (ogbn-papers100M pretraining)
    ("papers100M", "100M", 1, 1, 1, 1, 1, 0, 3, 1, 1, 1, 1, 1, "add", 1, 0.8, 0.5, 256, 128, 47, 3001, 1, 1),
    # medium/run.sh:2-7 (cora: h = 64, four GCN layers, no LayerNorm / residual / value projection)
    ("cora", "medium", 1, 1, 0, 0, 0, 0, 3, 1, 0, 0, 1, 1, "add", 1, 0.8, 0.5, 64, 1433, 7, 3001, 0, 1),
    # medium/run.sh:34-37 (deezer-europe: h = 96, two GCN layers, residual)
    ("deezer", "medium", 1, 1, 0, 1, 0, 0, 1, 1, 0, 0, 1, 1, "add", 1, 0.8, 0.5, 96, 602, 2, 8200, 1, 0),
]
_COVERING = [
    # greedy pairwise covering of what the recipes leave open (names: variant, index, trans layers, heads, gnn layers, aggregate)
    ('H00_t2h2_g1_add', '100M', 2, 2, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 'add', 1, 0.3, 0.7, 64, 65, 7, 1000, 0, 0),
    ('L01_t2h1_g2_cat', 'large', 2, 1, 0, 0, 0, 1, 2, 0, 0, 1, 1, 0, 'cat', 1, 0.3, 0.7, 256, 100, 40, 8200, 0, 1),
    ('H02_t1h2_g2_cat', '100M', 1, 2, 0, 1, 1, 0, 2, 1, 0, 0, 0, 0, 'cat', 1, 0.3, 0.3, 64, 128, 2, 3001, 0, 0),
    ('H03_t2h1_g3_add', '100M', 2, 1, 0, 1, 0, 1, 3, 0, 1, 0, 0, 1, 'add', 1, 0.3, 0.3, 256, 100, 47, 20011, 1, 1),
    ('L04_t2h2_g1_add', 'large', 2, 2, 1, 0, 1, 1, 1, 1, 0, 1, 0, 1, 'add', 1, 0.8, 0.3, 256, 1433, 7, 129, 0, 0),
    ('H05_t2h1_g0_cat', '100M', 2, 1, 1, 1, 0, 0, 0, 1, 0, 1, 0, 1, 'cat', 1, 0.8, 0.7, 64, 65, 40, 20011, 0, 1),
    ('L06_t0h1_g3_add', 'large', 0, 1, 0, 1, 0, 1, 3, 0, 0, 0, 1, 0, 'add', 1, 0.8, 0.3, 256, 100, 2, 129, 0, 0),
    ('L07_t1h2_g0_add', 'large', 1, 2, 0, 0, 1, 1, 0, 1, 0, 0, 1, 1, 'add', 1, 0.3, 0.3, 64, 128, 47, 3001, 0, 1),
    ('M08_t2h2_g1_add', 'medium', 2, 2, 1, 1, 1, 1, 1, 0, 0, 0, 0, 1, 'add', 0, 0.3, 0.3, 256, 602, 7, 1000, 0, 0),
    ('H09_t0h1_g1_cat', '100M', 0, 1, 1, 1, 1, 0, 1, 1, 1, 1, 0, 1, 'cat', 1, 0.3, 0.7, 96, 128, 40, 8200, 1, 1),
    ('H10_t2h2_g3_add', '100M', 2, 2, 0, 1, 1, 0, 3, 1, 0, 1, 1, 1, 'add', 1, 0.3, 0.7, 64, 65, 2, 1000, 0, 0),
    ('H11_t1h1_g1_add', '100M', 1, 1, 0, 0, 0, 0, 1, 0, 0, 1, 1, 0, 'add', 0, 0.3, 0.3, 256, 100, 47, 8200, 0, 1),
    ('H12_t1h1_g1_add', '100M', 1, 1, 1, 1, 0, 0, 1, 0, 0, 1, 1, 1, 'add', 1, 0.8, 0.3, 64, 128, 7, 3001, 1, 0),
    ('M13_t1h1_g2_add', 'medium', 1, 1, 0, 1, 0, 0, 2, 1, 1, 1, 0, 0, 'add', 1, 0.3, 0.7, 256, 100, 40, 20011, 0, 1),
    ('H14_t1h2_g3_cat', '100M', 1, 2, 0, 0, 1, 0, 3, 0, 1, 0, 1, 0, 'cat', 1, 0.8, 0.7, 256, 1433, 2, 129, 0, 0),
    ('M15_t0h2_g2_add', 'medium', 0, 2, 1, 1, 1, 0, 2, 0, 1, 0, 1, 0, 'add', 1, 0.8, 0.7, 64, 65, 47, 20011, 1, 1),
    ('L16_t1h2_g0_add', 'large', 1, 2, 0, 0, 1, 1, 0, 0, 0, 1, 1, 1, 'add', 0, 0.8, 0.7, 256, 100, 7, 129, 0, 0),
    ('H17_t0h1_g1_add', '100M', 0, 1, 1, 0, 1, 0, 1, 1, 0, 1, 1, 1, 'add', 1, 0.3, 0.7, 64, 128, 40, 3001, 0, 1),
    ('H18_t1h2_g0_add', '100M', 1, 2, 0, 1, 1, 0, 0, 1, 1, 1, 1, 0, 'add', 1, 0.8, 0.3, 256, 602, 2, 1000, 0, 0),
    ('H19_t1h2_g1_add', '100M', 1, 2, 1, 1, 1, 0, 1, 0, 1, 1, 1, 0, 'add', 1, 0.8, 0.7, 256, 128, 47, 8200, 0, 1),
    ('M20_t0h1_g1_add', 'medium', 0, 1, 1, 1, 0, 0, 1, 1, 1, 0, 1, 0, 'add', 0, 0.3, 0.7, 64, 65, 7, 1000, 0, 0),
    ('L21_t0h1_g0_add', 'large', 0, 1, 0, 0, 1, 1, 0, 1, 0, 1, 0, 1, 'add', 1, 0.3, 0.7, 256, 100, 40, 8200, 1, 1),
    ('M22_t1h2_g3_cat', 'medium', 1, 2, 1, 0, 1, 1, 3, 1, 0, 1, 1, 0, 'cat', 1, 0.8, 0.3, 64, 128, 2, 3001, 0, 0),
    ('H23_t2h1_g0_add', '100M', 2, 1, 0, 1, 1, 1, 0, 1, 1, 0, 1, 1, 'add', 0, 0.3, 0.7, 256, 100, 47, 20011, 0, 1),
    ('H24_t1h1_g1_add', '100M', 1, 1, 0, 0, 0, 1, 1, 1, 0, 1, 0, 0, 'add', 1, 0.8, 0.3, 100, 1433, 7, 129, 0, 0),
    # a second width that is not a multiple of 8, on the two-source GEMMs whose second block then starts off a 16-byte boundary
    # (use_init's [y | x0] W, the `cat` head) besides the Gram-form backward's [gnum' | x]
    ('L25_t1h1_g2_cat', 'large', 1, 1, 1, 1, 1, 1, 2, 1, 1, 1, 1, 1, 'cat', 1, 0.8, 0.5, 100, 65, 7, 1000, 0, 0),
]
CASES = [Case(*r) for r in _RECIPES + _COVERING]
BY_NAME = {c.name: c for c in CASES}
assert len(BY_NAME) == len(CASES)

_SMALL_H = {64: 16, 96: 24, 100: 20, 256: 32}     # 100 -> 20: still not a multiple of 8
_SMALL_N = {129: 61, 1000: 130, 3001: 187, 8200: 257, 20011: 300}
_SMALL_D = {65: 5, 100: 12, 128: 8, 602: 10, 1433: 9}


def small_view(c: Case) -> Case:
    """The same switches at n <= 300, h in {16, 20, 24, 32}: what the CPU emulation of the kernels runs."""
    return c._replace(h=_SMALL_H[c.h], n=_SMALL_N[c.n], d=_SMALL_D[c.d], hub=0)


def supports(c: Case, precision: str) -> bool:
    return precision == "fp32" or c.h % 8 == 0


def oracle_config(c: Case) -> dict:
    if c.variant == "medium":
        return O.make_config("medium", c.d, c.h, c.c, num_layers=c.tl, num_heads=c.heads, alpha=c.alpha, dropout=0.0,
                             use_bn=bool(c.t_bn), use_residual=bool(c.t_res), use_weight=bool(c.t_w), gcn_num_layers=c.gl + 1,
                             gcn_dropout=0.0, gcn_use_bn=bool(c.g_bn), graph_weight=c.gw, aggregate=c.agg, use_graph=bool(c.ug))
    kw = dict(trans_num_layers=c.tl, trans_num_heads=c.heads, trans_dropout=0.0, trans_use_bn=bool(c.t_bn),
              trans_use_residual=bool(c.t_res), trans_use_weight=bool(c.t_w), trans_use_act=bool(c.t_act), gnn_num_layers=c.gl,
              gnn_dropout=0.0, gnn_use_weight=bool(c.g_w), gnn_use_init=bool(c.g_init), gnn_use_bn=bool(c.g_bn),
              gnn_use_residual=bool(c.g_res), gnn_use_act=bool(c.g_act), graph_weight=c.gw, aggregate=c.agg, use_graph=bool(c.ug))
    if c.variant == "100M":
        kw["alpha"] = c.alpha
    return O.make_config(c.variant, c.d, c.h, c.c, **kw)


def package_config(ocfg: dict) -> dict:
    keys = make_config("large", 1, 1, 1).keys()
    kw = {k: v for k, v in ocfg.items() if k in keys and k not in ("variant", "in_channels", "hidden", "out_channels")}
    return make_config(ocfg["variant"], ocfg["in_channels"], ocfg["hidden"], ocfg["out_channels"], **kw)


def _seed(c: Case) -> int:
    return zlib.crc32(c.name.encode()) % 100000


def make_edges(c: Case) -> torch.Tensor:
    """Seeded edge list [2, E] (src, dst), ~6 edges per node: the last n/16 nodes are isolated, the first n/8 edges occur
    twice, n/20 nodes carry a self loop; `hub`: node 3 receives 1500 edges and node 5 sends 1300; `sym`: every edge also
    reversed (then the transposed CSR is the forward one), else the graph is directed."""
    g = torch.Generator().manual_seed(_seed(c))
    n = c.n
    live = n - n // 16
    ei = torch.stack([torch.randint(0, live, (6 * n,), generator=g), torch.randint(0, live, (6 * n,), generator=g)])
    loops = torch.randint(0, live, (n // 20,), generator=g)
    parts = [ei, ei[:, :n // 8], torch.stack([loops, loops])]
    if c.hub:
        parts.append(torch.stack([torch.randint(0, live, (1500,), generator=g), torch.full((1500,), 3)]))
        parts.append(torch.stack([torch.full((1300,), 5), torch.randint(0, live, (1300,), generator=g)]))
    ei = torch.cat(parts, 1)
    if c.sym:
        ei = torch.cat([ei, ei.flip(0)], 1)
    return ei.contiguous()


def make_inputs(c: Case) -> dict:
    """cfg, state_dict (LayerNorm / BatchNorm affines and running statistics away from their defaults, as
    make_golden.perturb_ does), features, edges and the seeded loss weight of loss = (logits * lw).sum()."""
    ocfg = oracle_config(c)
    sd = O.init_state_dict(ocfg, seed=_seed(c))
    g = torch.Generator().manual_seed(_seed(c) + 7)
    for k, t in sd.items():
        if ".bns." in k and not k.endswith("num_batches_tracked"):
            if k.endswith("running_var") or k.endswith("weight"):
                t.copy_(1.0 + 0.2 * torch.rand(t.shape, generator=g))
            else:
                t.copy_(0.1 * torch.randn(t.shape, generator=g))
    x = torch.randn(c.n, c.d, generator=g)
    lw = torch.randn(c.n, c.c, generator=g)
    lwh = torch.randn(c.n, c.h, generator=g)       # upstream gradient of a branch called alone
    x1, x2 = torch.randn(c.n, c.h, generator=g), torch.randn(c.n, c.h, generator=g)    # inputs of the head called alone
    return dict(ocfg=ocfg, cfg=package_config(ocfg), sd=sd, x=x, ei=make_edges(c), lw=lw, lwh=lwh, x1=x1, x2=x2)


def is_param(k: str, v: torch.Tensor) -> bool:
    return v.is_floating_point() and "running" not in k


# ------------------------------------------------------------------------------------------------
# oracle runs (cached: both precisions of the device, and the stage tests, share them)
# ------------------------------------------------------------------------------------------------
STAGES = ("model", "trans", "graph", "head")
EVAL_CASES = ("amazon2m", "L01_t2h1_g2_cat", "M13_t1h1_g2_add")    # backward of an eval-mode forward: one per GNN schedule / mix
_cache = {}


def _leaves(sd, dtype):
    return {k: (v.to(dtype).clone().requires_grad_(True) if is_param(k, v) else (v.to(dtype) if v.is_floating_point() else v.clone()))
            for k, v in sd.items()}


def _oracle_stage(c: Case, inp: dict, stage: str, dtype, training: bool) -> dict:
    ocfg, ei = inp["ocfg"], inp["ei"]
    P = _leaves(inp["sd"], dtype)
    stats = {}
    extra = {}
    if stage == "head":
        x1, x2 = (inp[k].to(dtype).clone().requires_grad_(True) for k in ("x1", "x2"))
        feat = x1 if not c.ug else (c.gw * x2 + (1.0 - c.gw) * x1 if c.agg == "add" else torch.cat([x1, x2], 1))
        out = torch.nn.functional.linear(feat, P["fc.weight"], P["fc.bias"])
        lw = inp["lw"]
        extra = {"__x1__": x1, "__x2__": x2}
    else:
        x = inp["x"].to(dtype).clone().requires_grad_(True)
        extra = {"__x__": x}
        if stage == "model":
            out = O.sgformer_forward(ocfg, P, x, ei, training=training, stats_out=stats)
            lw = inp["lw"]
        elif stage == "trans":
            out = O.trans_conv(x, P, ocfg, training)
            lw = inp["lwh"]
        elif c.variant == "medium":
            out = O.gcn_medium(x, ei, P, ocfg, training, stats_out=stats)
            lw = inp["lwh"]
        else:
            out = O.graph_conv(x, ei, P, ocfg, training, stats_out=stats)
            lw = inp["lwh"]
    (out * lw.to(dtype)).sum().backward()
    grads = {k: v.grad for k, v in P.items() if is_param(k, v) and v.grad is not None}
    grads.update({k: v.grad for k, v in extra.items() if v.grad is not None})
    return dict(out=out.detach(), grads=grads, stats={k: v.detach() for k, v in stats.items()})


def oracle_run(c: Case, dtype, stage: str = "model", training: bool = True) -> dict:
    """logits (or the stage's output), every parameter gradient, the input gradient(s) and the updated BatchNorm buffers of the
    oracle with leaf parameters in `dtype` (torch.float64: the reference value; torch.float32: what plain fp32 delivers)."""
    key = (c, dtype, stage, training)
    if key not in _cache:
        _cache[key] = _oracle_stage(c, inputs(c), stage, dtype, training)
    return _cache[key]


def inputs(c: Case) -> dict:
    if ("inputs", c) not in _cache:
        _cache["inputs", c] = make_inputs(c)
    return _cache["inputs", c]


# ------------------------------------------------------------------------------------------------
# checker
# ------------------------------------------------------------------------------------------------
def tensor_class(name: str, ocfg: dict) -> str:
    """bn_weight: a Linear weight whose output feeds a LayerNorm / BatchNorm (its gradient is a difference of large terms);
    qk / qk_bias: the attention's query / key projection weights / biases; affine: biases and LayerNorm / BatchNorm affines; grad_x: input gradients."""
    if name.startswith("__x"):
        return "grad_x"
    if ".Wq." in name or ".Wk." in name:
        return "qk_bias" if name.endswith("bias") else "qk"
    if not name.endswith("weight") or ".bns." in name:
        return "affine"
    if name.startswith("trans_conv.fcs.") and ocfg["trans_use_bn"]:
        return "bn_weight"
    if name.startswith("trans_conv.convs.") and ocfg["trans_use_bn"]:
        return "bn_weight"
    if name.startswith("graph_conv.") and ocfg["gnn_use_bn"]:
        return "bn_weight"
    if name.startswith("gnn.convs.") and ocfg.get("gcn_use_bn") and not name.startswith(f"gnn.convs.{ocfg['gcn_num_layers'] - 1}."):
        return "bn_weight"
    return "weight"


# Allowed relative Frobenius error of a gradient tensor against the fp64 oracle: max(C_OWN * own32, FLOOR[class][precision]),
# own32 = the fp32 oracle's own relative error for that tensor.  Beside each entry: the worst error measured through the drop-in
# modules and the stages over the table on an H100 80GB HBM3 (700 W limit; accuracy figures, not timings); a floor is at most 4x that.
# fp32 floors above 1e-3: the weights and affines behind a BatchNorm (a difference of large terms, which the bf16x3 GEMMs'
# epsilon of ~2^-20 amplifies; the fp32 oracle itself is off by 1e-3 there) and, through them, the input gradient.
# bf16 floors above 5e-2: every class; a bf16 activation carries 2^-9 per element and the BatchNorm / LayerNorm backward
# amplifies it.  The query / key projections' gradients are O(1/N) of the others: in bf16 the weights keep 14 % and of the
# biases only the order of magnitude survives (40 % measured); in fp32 they are the most accurate tensors of the model.
# What the bounds cannot see: on the tensors behind a BatchNorm the fp32 oracle is itself off by ~1e-3, so
# max(4 * own32, 5e-3) passes a missing term below about 0.5 % there; the planted 1 % bias error is caught on a bias with no
# BatchNorm behind it (trans_conv.fcs.0.bias).  The figures come from one run on one card; tests/test_gpu_config_matrix.py took
# 54 s there, the cached CPU oracle runs included.
C_OWN = {"fp32": 4.0, "bf16": 4.0}
FLOOR = {
    "weight":    {"fp32": 2e-3, "bf16": 0.2},    # measured 7.2e-4 (H03 convs.2.W.weight; own32 7.2e-4) / 9.1e-2 (cora gnn.convs.0)
    "bn_weight": {"fp32": 5e-3, "bf16": 0.3},    # measured 1.7e-3 (papers100M convs.0.W.weight; own32 1.2e-3) / 1.3e-1 (arxiv)
    "affine":    {"fp32": 5e-3, "bf16": 0.3},    # measured 2.0e-3 (papers100M bns.1.bias; own32 1.4e-3) / 1.4e-1 (arxiv bns.2.bias)
    "qk":        {"fp32": 1.2e-5, "bf16": 0.4},  # measured 3.2e-6 / 1.4e-1
    "qk_bias":   {"fp32": 3e-5, "bf16": 0.8},    # measured 8.1e-6 (H23 Wq.bias; own32 2.7e-4) / 4.0e-1 (L16 Wq.bias)
    "grad_x":    {"fp32": 2.5e-3, "bf16": 0.25},  # measured 9.9e-4 (papers100M; own32 9.8e-4) / 9.6e-2 (M22)
}
LOGIT_TOL = {"fp32": 1e-4, "bf16": 1e-2}


def _sibling_scale(name: str, ref: dict) -> float:
    """A bias that feeds a training-mode BatchNorm has an exactly zero gradient: such a tensor is measured on the scale of the
    weight gradient of its own layer (never on another layer's or the model's)."""
    if name.endswith(".bias") and ".bns." not in name:
        stem = name[:-len("bias")]
        for w in (stem + "weight", stem + "lin.weight"):
            if w in ref:
                return 1e-3 * ref[w].double().norm().item() / max(ref[w].shape[1], 1) ** 0.5
    return 0.0


def rel_err(name: str, a: torch.Tensor, ref: dict) -> float:
    b = ref[name].double()
    a = a.detach().cpu().double()
    if a.shape != b.shape:
        return float("inf")
    den = max(b.norm().item(), _sibling_scale(name, ref), 1e-30)
    e = (a - b).norm().item() / den
    return e if e == e else float("inf")


def check(c: Case, got: dict, ref64: dict, ref32: dict, precision: str, report: str = None) -> list:
    """got: dict(out=logits, grads={name: tensor}, stats={buffer name: tensor} (optional)).  Returns one line per violated bound,
    each starting with the name of the tensor it concerns."""
    ocfg = oracle_config(c)
    problems = []
    tol = LOGIT_TOL[precision]
    o, r = got["out"].detach().cpu().double(), ref64["out"].double()
    if o.shape != r.shape:
        return [f"out: shape {tuple(o.shape)} vs {tuple(r.shape)}"]
    err = (o - r).abs().max().item()
    if not err <= tol + tol * r.abs().max().item():
        problems.append(f"out: max err {err:.3e} (ref max {r.abs().max().item():.3e}, tolerance {tol})")
    rows = []
    for k, g64 in ref64["grads"].items():
        g = got["grads"].get(k)
        if g is None:
            problems.append(f"{k}: gradient missing")
            continue
        cls = tensor_class(k, ocfg)
        e = rel_err(k, g, ref64["grads"])
        own = rel_err(k, ref32["grads"][k], ref64["grads"])
        allowed = max(C_OWN[precision] * own, FLOOR[cls][precision])
        rows.append(dict(case=c.name, precision=precision, tensor=k, cls=cls, err=e, own32=own, allowed=allowed,
                         norm=g64.double().norm().item()))
        if not e <= allowed:
            problems.append(f"{k}: relative error {e:.3e} vs fp64 oracle > {allowed:.3e} "
                            f"(class {cls}, fp32 oracle's own error {own:.3e}, |ref| {g64.double().norm().item():.3e})")
    if precision == "fp32":
        for k, r in ref64["stats"].items():
            v, r = got["stats"][k], r.double()
            e = (v.detach().cpu().double() - r).abs().max().item()
            if not e <= 1e-5 + 1e-4 * r.abs().max().item():
                problems.append(f"{k}: buffer after the step off by {e:.3e}")
    if report:
        with open(report, "a") as f:
            for row in rows:
                f.write(json.dumps(row) + "\n")
    return problems


REPORT = os.environ.get("SGF_CONFIG_MATRIX_REPORT")     # path: append one JSON line per (case, precision, tensor) checked


# ------------------------------------------------------------------------------------------------
# running the schedules (kernel module `K` = sgformer_b200.kernels on the device, tests/kernel_emu.py on the CPU)
# ------------------------------------------------------------------------------------------------
def _params(inp: dict, dev, keep):
    sd = inp["sd"]
    names = tuple(k for k in sd if keep(k))
    tensors = [sd[k].clone().to(dev).requires_grad_(True) if is_param(k, sd[k]) else sd[k].clone().to(dev) for k in names]
    return names, tensors


def _collect(names, tensors, out, extra, want_stats=True):
    grads = {k: t.grad for k, t in zip(names, tensors) if t.requires_grad and t.grad is not None}
    grads.update({k: v.grad for k, v in extra.items() if v.grad is not None})
    stats = {k: t.detach() for k, t in zip(names, tensors) if "running" in k or k.endswith("num_batches_tracked")}
    return dict(out=out.detach(), grads=grads, stats=stats if want_stats else {})


def run_stage(c: Case, stage: str, prec, graph, dev="cpu", training: bool = True) -> dict:
    """The fused encoder (`model`) or one branch alone through sgformer_b200.functional, on whatever kernel module
    functional.K / engine.K currently are."""
    from sgformer_b200 import functional as Fn
    from sgformer_b200.dist import SINGLE
    inp = inputs(c)
    cfg = inp["cfg"]
    if stage == "head":
        names, tensors = _params(inp, dev, lambda k: k.startswith("fc."))
        x1 = inp["x1"].clone().to(dev).requires_grad_(True)
        x2 = inp["x2"].clone().to(dev).requires_grad_(True) if c.ug else None
        out = Fn.HeadFn.apply(x1, x2, cfg, prec, names, *tensors)
        (out * inp["lw"].to(dev)).sum().backward()
        return _collect(names, tensors, out, {"__x1__": x1, **({"__x2__": x2} if c.ug else {})})
    x = inp["x"].clone().to(dev).requires_grad_(True)
    if stage == "model":
        names, tensors = _params(inp, dev, lambda k: True)
        out = Fn.SGFormerFn.apply(x, graph if c.ug else None, cfg, prec, training, SINGLE, names, *tensors)
        lw = inp["lw"]
    elif stage == "trans":
        names, tensors = _params(inp, dev, lambda k: k.startswith("trans_conv."))
        out = Fn.TransConvFn.apply(x, cfg, prec, training, names, *tensors)
        lw = inp["lwh"]
    else:
        med = c.variant == "medium"
        pfx = "gnn." if med else "graph_conv."
        names, tensors = _params(inp, dev, lambda k: k.startswith(pfx))
        out = Fn.GraphBranchFn.apply(x, graph, cfg, prec, training, "gcn" if med else "gconv", pfx, names, *tensors)
        lw = inp["lwh"]
    (out * lw.to(dev)).sum().backward()
    return _collect(names, tensors, out, {"__x__": x}, want_stats=training)


def stage_applies(c: Case, stage: str) -> bool:
    return stage != "graph" or bool(c.ug)


# ------------------------------------------------------------------------------------------------
# planted errors: each wraps ONE correct entry point of the kernel module and alters its result (every launch stays valid).
# name -> (the case it runs on, make(K, graph) -> (attribute, wrapper), tensors check() must then name)
# ------------------------------------------------------------------------------------------------
def _plant_gemm_tn_drops_rows(K, graph):
    real = K.gemm_tn

    def gemm_tn(A, B, out, **kw):
        r = A.rows - 64
        return real(type(A)(A.data[:r], r, A.k, A.kp, A.planes), type(B)(B.data[:r], r, B.k, B.kp, B.planes), out, **kw)
    return "gemm_tn", gemm_tn


def _plant_gemm_nt_overwrites(K, graph):
    real = K.gemm_nt

    def gemm_nt(*a, **kw):
        kw["accumulate"] = False
        return real(*a, **kw)
    return "gemm_nt", gemm_nt


def _plant_bn_bwd_ignores_gscale(K, graph):
    real = K.bn_bwd
    sig = inspect.signature(real)

    def bn_bwd(*a, **kw):
        b = sig.bind(*a, **kw)
        b.arguments["gscale"] = 1.0
        return real(*b.args, **b.kwargs)
    return "bn_bwd", bn_bwd


def _plant_axpby_without_row_scale(K, graph):
    real = K.axpby

    def axpby(*a, **kw):
        kw["row_scale"] = None
        return real(*a, **kw)
    return "axpby", axpby


def _plant_spmm_not_transposed(K, graph):
    real = K.spmm
    rp_t = graph.transpose()[0]

    def spmm(rowptr, col, row_scale, x, **kw):
        if rowptr is rp_t:
            rowptr, col, kw["heavy"] = graph.rowptr, graph.col, graph.heavy
        return real(rowptr, col, row_scale, x, **kw)
    return "spmm", spmm


def _plant_colstats_bias_1pct(K, graph):
    real = K.colstats

    def colstats(*a, **kw):
        s, q = real(*a, **kw)
        return (s * 1.01 if s is not None else None), q
    return "colstats", colstats


def _plant_wq_grad_5pct(K, graph):
    real = K.attn_gram_prepare_bwd

    def attn_gram_prepare_bwd(*a, **kw):
        r = list(real(*a, **kw))
        r[0] = r[0] * 1.05
        return tuple(r)
    return "attn_gram_prepare_bwd", attn_gram_prepare_bwd


PLANTED = {
    "gemm_tn_drops_last_64_rows": ("plant_a", _plant_gemm_tn_drops_rows, ("fc.weight", "graph_conv.convs.0.W.weight")),
    "gemm_nt_accumulate_overwrites": ("plant_a", _plant_gemm_nt_overwrites, ("graph_conv.fcs.0.weight", "trans_conv.fcs.0.weight")),
    "bn_bwd_ignores_gscale": ("plant_a", _plant_bn_bwd_ignores_gscale, ("graph_conv.fcs.0.weight", "graph_conv.bns.2.weight")),
    "axpby_without_row_scale": ("plant_b", _plant_axpby_without_row_scale, ("graph_conv.fcs.0.weight",)),
    "spmm_forward_csr_in_backward": ("plant_a", _plant_spmm_not_transposed, ("graph_conv.fcs.0.weight",)),
    "colstats_bias_grad_1pct": ("plant_a", _plant_colstats_bias_1pct, ("trans_conv.fcs.0.bias",)),
    "wq_grad_scaled_1_05": ("plant_a", _plant_wq_grad_5pct, ("trans_conv.convs.0.Wq.weight",)),
}
# plant_a: two GraphConv layers with use_init on a directed graph, one Gram-form attention layer with residual, `add`;
# plant_b: GraphConv layers without a weight (the axpby branch of gconv_backward)
PLANT_CASES = {
    "plant_a": Case("plant_a", "large", 1, 1, 1, 1, 1, 1, 2, 1, 1, 1, 1, 1, "add", 1, 0.3, 0.5, 64, 65, 7, 1000, 0, 0),
    "plant_b": Case("plant_b", "large", 1, 1, 1, 1, 1, 0, 2, 0, 0, 1, 1, 1, "add", 1, 0.8, 0.5, 64, 65, 7, 1000, 0, 0),
}
