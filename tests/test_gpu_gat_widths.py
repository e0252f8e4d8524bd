"""The GAT kernels and backbone on the H100 at the reference's widths, against fp64.

  (a) sgf_gat_logits / gat_fwd / gat_bwd at every shape of gat_widths.SHAPES (all 32 instantiations), p = 0 and 0.5: a_src, a_dst,
      out, lse, dxp, da_src and da_dst element by element against an fp64 restatement of the operands each kernel reads (xp and g
      as stored; the logits and lse of the kernel that wrote them), bounded by gat_widths.check_elementwise;
  (b) duplicate runs of 32, 33 and 70 identical edges placed across the 32-entry batches of a row, differently in the CSR and
      its transpose, under attention dropout;
  (c) the grid-stride loops (more rows than the capped grid has warps);
  (d) ELU in bn_fwd / bn_bwd / bn_bwd_sums with dropout at gat_widths.ELU_WIDTHS (CPL 1-4 in both dtypes);
  (e) the GAT modules and SGFormer(gnn=GAT) at hidden 64 x 8 heads against oracle/gat_oracle.py in fp64;
  (f) one training step with input, attention and post-ELU dropout on against fp64 with the three masks replayed;
  (g) planted errors that the bounds must report by name, and run-to-run bit identity.

Set SGF_GAT_WIDTHS_REPORT to a path to have the worst measured ratio of every bound appended there as JSON (the calibration of
K and FLOOR below, DESIGN.md §6)."""
import copy
import json
import math
import os
import zlib

import pytest
import torch
import torch.nn.functional as F

import gat_widths as W
from dropout_mask import current_epoch, keep_mask, keep_scale
from oracle import gat_oracle as G

pytestmark = pytest.mark.gpu
DEV = "cuda"
DT = {"fp32": torch.float32, "bf16": torch.bfloat16}

# k of each kernel output's bound |got - ref| <= k 2^-24 S (gat_widths.check_elementwise).  Beside each: the worst ratio
# measured over (a)-(c) on an H100 80GB HBM3 (700 W limit), one run; k is 4x that, rounded up.
K = {
    "a_src": 10,        # 2.47
    "a_dst": 13,        # 3.17 (gat_logits at 32 rows per warp)
    "out": 94,          # 23.4
    "lse": 6,           # 1.34
    "dxp": 69,          # 17.1
    "da_src": 21,       # 5.16
    "da_dst": 16,       # 3.91
}
REPORT = os.environ.get("SGF_GAT_WIDTHS_REPORT")
_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if REPORT:
        with open(REPORT, "a") as f:
            f.write(json.dumps(_WORST, sort_keys=True) + "\n")


def _note(key, value):
    if value == value:
        _WORST[key] = max(_WORST.get(key, 0.0), float(value))


@pytest.fixture(scope="module")
def Kmod():
    from sgformer_b200 import kernels
    return kernels


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------
# graphs
# ------------------------------------------------------------------------------------------------
def _base_edges(n=1500, e=9000, hub=3200, seed=21):
    """Directed: duplicates (e/10 copied edges), 5 existing self loops, nodes n-3.. isolated, `hub` extra in-edges of node 0."""
    g = torch.Generator().manual_seed(seed)
    live = n - 3
    src, dst = torch.randint(0, live, (e,), generator=g), torch.randint(0, live, (e,), generator=g)
    src = torch.cat([src, src[:e // 10], torch.arange(5), torch.randint(0, live, (hub,), generator=g)])
    dst = torch.cat([dst, dst[:e // 10], torch.arange(5), torch.zeros(hub, dtype=torch.int64)])
    return torch.stack([src, dst])


def _run_edges():
    """Runs of identical edges across the 32-entry batches of a row.  Row 100 of the CSR: sources 0..19, then 70 x (50 -> 100)
    at entries 20..89 (across 32 and 64), then its self loop; row 50 of the transpose: 50, 60..64, then the same 70 edges at
    entries 6..75.  Row 200: sources 0..31, then exactly 32 x (150 -> 200) starting at entry 32.  Row 400: 33 x (5 -> 400) at
    entries 0..32 (entries 3..35 of row 5 of the transpose).  Plus random edges among nodes 450..599."""
    g = torch.Generator().manual_seed(5)
    n = 600
    full = lambda k, v: torch.full((k,), v, dtype=torch.int64)
    parts = [(torch.arange(20), full(20, 100)), (full(70, 50), full(70, 100)), (full(5, 50), torch.arange(60, 65)),
             (torch.arange(32), full(32, 200)), (full(32, 150), full(32, 200)), (full(33, 5), full(33, 400))]
    src = torch.cat([s for s, _ in parts] + [torch.randint(450, n, (2000,), generator=g)])
    dst = torch.cat([d for _, d in parts] + [torch.randint(450, n, (2000,), generator=g)])
    ei = torch.stack([src, dst])
    return ei[:, torch.randperm(ei.shape[1], generator=g)], n


_GRAPHS = {}


def _graph(kind):
    """-> (Graph, n).  'base': directed; 'undirected': the base edges and their reverses (graph.transpose() shares the CSR);
    'runs': _run_edges; 'grid<groups>': n = 2 * num_sms * 16 * 8 * groups + 7 rows, mean in-degree ~3."""
    from sgformer_b200.graph import Graph
    if kind not in _GRAPHS:
        if kind == "base":
            ei, n = _base_edges(), 1500
        elif kind == "undirected":
            ei = _base_edges(hub=0)
            ei, n = torch.cat([ei, ei.flip(0)], 1), 1500
        elif kind == "runs":
            ei, n = _run_edges()
        else:
            n = 2 * _sms() * 16 * 8 * int(kind[4:]) + 7
            g = torch.Generator().manual_seed(n)
            ei = torch.randint(0, n, (2, 2 * n), generator=g)
        gr = Graph(ei.to(DEV), n, 1)
        if kind == "undirected":
            assert gr.transpose()[0] is gr.rowptr, "a symmetric multigraph shares its CSR with the transpose"
        _GRAPHS[kind] = (gr, n)
    return _GRAPHS[kind]


# ------------------------------------------------------------------------------------------------
# fp64 reference of the three kernels
# ------------------------------------------------------------------------------------------------
def _lrelu(v):
    return torch.where(v > 0, v, 0.2 * v)


def _edges(rowptr, col):
    n = rowptr.numel() - 1
    return col.long(), torch.repeat_interleave(torch.arange(n, device=col.device), rowptr.diff())


def _seg(idx, vals, n):
    return torch.zeros((n,) + tuple(vals.shape[1:]), dtype=vals.dtype, device=vals.device).index_add_(0, idx, vals)


def _chunks(E, step=1 << 15):
    return [(a, min(a + step, E)) for a in range(0, E, step)]


def reference(graph, n, xp, a_s, a_d, lse, att_s, att_d, bias, g, H, C, mean, factor=None, transposed=None):
    """fp64 values and absolute sums S of the kernel outputs.  xp, g: as stored; a_s, a_d, lse: the kernels' own fp32 outputs
    (the operands gat_fwd and gat_bwd read).  `factor` [nnz, H]: attention-dropout factors in CSR order (None: 1).  Returns
    (ref, S) dicts keyed by output name; da_* are [H, n] as the kernel writes them."""
    d64 = lambda t: t.detach().double()
    xp, a_s, a_d, lse, g = d64(xp), d64(a_s), d64(a_d), d64(lse), d64(g)
    att_s, att_d = d64(att_s).view(H, C), d64(att_d).view(H, C)
    xh = xp.view(n, H, C)
    ref, S = {}, {}
    ref["a_src"], S["a_src"] = (xh * att_s).sum(-1), (xh.abs() * att_s.abs()).sum(-1)
    ref["a_dst"], S["a_dst"] = (xh * att_d).sum(-1), (xh.abs() * att_d.abs()).sum(-1)
    src, dst = _edges(graph.rowptr, graph.col)
    pre = a_s[src] + a_d[dst]
    e = _lrelu(pre)
    m = torch.full((n, H), -math.inf, dtype=torch.float64, device=DEV).scatter_reduce(0, dst[:, None].expand_as(e), e, "amax")
    lse_ref = m + torch.log(_seg(dst, torch.exp(e - m[dst]), n))
    pmax = torch.zeros((n, H), dtype=torch.float64, device=DEV).scatter_reduce(0, dst[:, None].expand_as(e), pre.abs(), "amax")
    ref["lse"], S["lse"] = lse_ref, 1.0 + lse_ref.abs() + pmax
    fac = torch.ones_like(e) if factor is None else factor.to(DEV).double()
    gsc = 1.0 / H if mean else 1.0
    gh = g.view(n, 1, C).expand(n, H, C) if mean else g.view(n, H, C)
    # forward: y_i = sum_j alpha_ij d_ij xp_j with lse from fp64
    y, ys = torch.zeros((n, H, C), dtype=torch.float64, device=DEV), torch.zeros((n, H, C), dtype=torch.float64, device=DEV)
    # backward: alpha from the kernel's lse
    al = torch.exp(e - lse[dst])
    dot = torch.empty_like(e)
    adot = torch.empty_like(e)
    for a, b in _chunks(len(src)):
        s_, d_ = src[a:b], dst[a:b]
        w = (torch.exp(e[a:b] - lse_ref[d_]) * fac[a:b])[:, :, None]
        y.index_add_(0, d_, w * xh[s_])
        ys.index_add_(0, d_, w * xh[s_].abs())
        dot[a:b] = (gh[d_] * xh[s_]).sum(-1)
        adot[a:b] = (gh[d_].abs() * xh[s_].abs()).sum(-1)
    da, ada = fac * dot * gsc, fac * adot * gsc
    lg = torch.where(pre > 0, torch.ones_like(pre), torch.full_like(pre, 0.2))
    R, SR = _seg(dst, al * da, n), _seg(dst, al * ada, n)
    A, SA, B = _seg(dst, al * da * lg, n), _seg(dst, al * ada * lg, n), _seg(dst, al * lg, n)
    ref["da_dst"], S["da_dst"] = (A - R * B).t(), (SA + SR * B).t()
    de = al * (da - R[dst])
    ref["da_src"] = _seg(src, de * lg, n).t()
    S["da_src"] = _seg(src, al * (ada + SR[dst]) * lg, n).t()
    dx, sdx = torch.zeros((n, H, C), dtype=torch.float64, device=DEV), torch.zeros((n, H, C), dtype=torch.float64, device=DEV)
    coef = al * fac * gsc
    for a, b in _chunks(len(src)):
        s_, d_ = src[a:b], dst[a:b]
        dx.index_add_(0, s_, coef[a:b, :, None] * gh[d_])
        sdx.index_add_(0, s_, coef[a:b, :, None] * gh[d_].abs())
    dx += ref["da_src"].t()[:, :, None] * att_s + ref["da_dst"].t()[:, :, None] * att_d
    sdx += S["da_src"].t()[:, :, None] * att_s.abs() + S["da_dst"].t()[:, :, None] * att_d.abs()
    ref["dxp"], S["dxp"] = dx.reshape(n, H * C), sdx.reshape(n, H * C)
    b64 = d64(bias)
    if mean:
        ref["out"], S["out"] = y.mean(1) + b64, ys.mean(1) + b64.abs()
    else:
        ref["out"], S["out"] = y.reshape(n, H * C) + b64, ys.reshape(n, H * C) + b64.abs()
    return ref, S


def _inputs(n, dtype, H, C, mean, seed, pitch=False):
    """xp ~ N(0, 1) and g ~ N(0, 1) in the activation dtype (column views of wider buffers when `pitch`), attention vectors
    ~ N(0, 1/C), bias ~ N(0, 0.1)."""
    gen = torch.Generator().manual_seed(seed)
    dt = DT[dtype]
    vn = 8 if dtype == "bf16" else 4
    gc = C if mean else H * C

    def mat(cols):
        t = torch.randn(n, cols, generator=gen)
        if not pitch:
            return t.to(DEV, dt).contiguous()
        buf = torch.full((n, cols + 6 * vn), float("nan"), dtype=dt, device=DEV)
        buf[:, 2 * vn:2 * vn + cols] = t.to(dt)
        return buf[:, 2 * vn:2 * vn + cols]
    xp, g = mat(H * C), mat(gc)
    att_s = (torch.randn(H * C, generator=gen) / math.sqrt(C)).to(DEV)
    att_d = (torch.randn(H * C, generator=gen) / math.sqrt(C)).to(DEV)
    bias = (0.1 * torch.randn(gc, generator=gen)).to(DEV)
    return xp, g, att_s, att_d, bias


def _csr_edges(graph):
    src, dst = _edges(graph.rowptr, graph.col)
    return torch.stack([src, dst]).cpu()


def run_kernels(Kmod, kind, shape, p, seed=0x5EED, pitch=False):
    """The three kernels on graph `kind` at `shape` -> (got, ref, S, ctx)."""
    dtype, H, C, mean = shape
    graph, n = _graph(kind)
    xp, g, att_s, att_d, bias = _inputs(n, dtype, H, C, mean, zlib.crc32(repr((shape, kind)).encode()), pitch)
    a_s, a_d = Kmod.gat_logits(xp, H, C, att_s, att_d)
    out, lse = Kmod.gat_fwd(graph.rowptr, graph.col, xp, a_s, a_d, H, C, mean, bias, p, seed)
    rp_t, col_t = graph.transpose()
    dxp, da_s, da_d = Kmod.gat_bwd(graph.rowptr, graph.col, rp_t, col_t, xp, a_s, a_d, lse, g, att_s, att_d, H, C, mean, p, seed)
    seed_eff = W.with_epoch(seed, current_epoch())
    edges = _csr_edges(graph)
    factor = W.edge_keep(seed_eff, n, edges, H, p) if p > 0 else None
    ref, S = reference(graph, n, xp, a_s, a_d, lse, att_s, att_d, bias, g, H, C, mean, factor)
    got = dict(a_src=a_s, a_dst=a_d, out=out, lse=lse, dxp=dxp, da_src=da_s, da_dst=da_d)
    ctx = dict(graph=graph, n=n, xp=xp, g=g, a_s=a_s, a_d=a_d, lse=lse, att_s=att_s, att_d=att_d, bias=bias, edges=edges,
               seed_eff=seed_eff)
    return got, ref, S, ctx


STORED = ("out", "dxp")       # outputs stored in the activation dtype; the rest are fp32


def check_outputs(got, ref, S, dtype, tag=""):
    problems = []
    for name in ("a_src", "a_dst", "out", "lse", "dxp", "da_src", "da_dst"):
        bf = dtype == "bf16" and name in STORED
        _note(name, W.ratio(got[name], ref[name], S[name], bf).max().item())
        problems += W.check_elementwise(name, got[name], ref[name], S[name], K[name], bf)
    return [f"{pr} [{tag}]" for pr in problems]


# ------------------------------------------------------------------------------------------------
# (a) every shape, p = 0 and 0.5
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", W.SHAPES, ids=[W.shape_id(s) for s in W.SHAPES])
def test_kernels_match_fp64_at_every_width(Kmod, shape):
    problems = []
    kinds = ["base"]
    if shape in (("fp32", 5, 32, False), ("bf16", 8, 64, False)):
        kinds.append("undirected")
    for kind in kinds:
        for p in (0.0, 0.5):
            got, ref, S, _ = run_kernels(Kmod, kind, shape, p)
            problems += check_outputs(got, ref, S, shape[0], f"{kind} p={p}")
    if W.geometry(*shape[:3])[2] == 4 and shape in (("fp32", 8, 64, False), ("bf16", 7, 136, False)):
        got, ref, S, ctx = run_kernels(Kmod, "base", shape, 0.5, pitch=True)
        assert ctx["xp"].stride(0) > ctx["xp"].shape[1] and ctx["g"].stride(0) > ctx["g"].shape[1]
        problems += check_outputs(got, ref, S, shape[0], "pitched xp and g, p=0.5")
    assert not problems, "\n".join(problems)


# ------------------------------------------------------------------------------------------------
# (b) duplicate runs across batch boundaries
# ------------------------------------------------------------------------------------------------
RUN_SHAPES = [("fp32", 8, 16, False), ("bf16", 8, 32, True), ("fp32", 8, 64, False), ("bf16", 8, 128, True)]


def test_run_graph_places_the_runs():
    graph, n = _graph("runs")
    rp, col = graph.rowptr.cpu(), graph.col.cpu().long()
    rp_t, col_t = (t.cpu() for t in graph.transpose())
    row = lambda r, c, i: c[r[i]:r[i + 1]].tolist()
    assert row(rp, col, 100)[20:90] == [50] * 70 and row(rp, col, 100)[19] == 19
    assert row(rp_t, col_t.long(), 50)[6:76] == [100] * 70
    assert row(rp, col, 200)[32:64] == [150] * 32 and row(rp, col, 200)[64] == 200
    assert row(rp, col, 400)[:33] == [5] * 33
    assert row(rp_t, col_t.long(), 5)[3:36] == [400] * 33


@pytest.mark.parametrize("shape", RUN_SHAPES, ids=[W.shape_id(s) for s in RUN_SHAPES])
def test_duplicate_runs_under_attention_dropout(Kmod, shape):
    got, ref, S, _ = run_kernels(Kmod, "runs", shape, 0.5, seed=0xD0B1E)
    problems = check_outputs(got, ref, S, shape[0], "runs p=0.5")
    assert not problems, "\n".join(problems)


# ------------------------------------------------------------------------------------------------
# (c) the grid-stride loops
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_grid_stride_rows(Kmod, dtype):
    """(8, 64): one row per warp in all three kernels; n = 2 * num_sms * 16 * 8 + 7 rows, so each warp of the capped grid runs
    two rows and the first 7 warps a third."""
    shape = (dtype, 8, 64, False)
    lpr = W.geometry(*shape[:3])[1]
    kind = f"grid{32 // lpr}"
    got, ref, S, ctx = run_kernels(Kmod, kind, shape, 0.5)
    assert ctx["n"] > 2 * _sms() * 16 * 8
    problems = check_outputs(got, ref, S, dtype, kind)
    assert not problems, "\n".join(problems)


def test_grid_stride_logits_32_rows_per_warp(Kmod):
    """(1, 4) fp32: a row is one chunk, 32 rows share a warp; n = 2 * num_sms * 16 * 8 * 32 + 7."""
    n = 2 * _sms() * 16 * 8 * 32 + 7
    gen = torch.Generator().manual_seed(4)
    xp = torch.randn(n, 4, generator=gen).to(DEV)
    att_s, att_d = torch.randn(4, generator=gen).to(DEV), torch.randn(4, generator=gen).to(DEV)
    a_s, a_d = Kmod.gat_logits(xp, 1, 4, att_s, att_d)
    x = xp.double()
    problems = []
    for name, got, att in (("a_src", a_s, att_s), ("a_dst", a_d, att_d)):
        ref, S = x @ att.double(), x.abs() @ att.double().abs()
        _note(name, W.ratio(got[:, 0], ref, S, False).max().item())
        problems += W.check_elementwise(name, got[:, 0], ref, S, K[name], False)
    assert not problems, "\n".join(problems)


# ------------------------------------------------------------------------------------------------
# (d) ELU in the BatchNorm / activation / dropout row kernels
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,h", W.ELU_WIDTHS, ids=[f"{d}-h{h}" for d, h in W.ELU_WIDTHS])
def test_bn_elu_dropout_matches_fp64(Kmod, dtype, h):
    """y = dropout(elu(BN?(z))) and its backward (dz, the BatchNorm sums, the running buffers) against fp64 autograd with the
    kernels' mask: training BatchNorm, eval BatchNorm and none, in the bounds of tests/test_gpu_dropout.py."""
    from test_gpu_dropout import _close, _rand, _tol, dmask
    K_ = Kmod
    dtype = DT[dtype]
    tol = _tol(dtype)
    for k, (use_bn, training) in enumerate([(True, True), (True, False), (False, True)]):
        rows, p, seed = 777, (0.5, 0.3, 0.6)[k], 900 + 13 * k + h
        gen = torch.Generator().manual_seed(seed)
        z, dy = _rand(rows, h, dtype, gen, 1.5), _rand(rows, h, dtype, gen)
        gamma, beta = (1 + 0.2 * torch.randn(h, generator=gen)).to(DEV), (0.2 * torch.randn(h, generator=gen)).to(DEV)
        rm, rv = (0.1 * torch.randn(h, generator=gen)).to(DEV), (1 + 0.3 * torch.rand(h, generator=gen)).to(DEV)
        rm_k, rv_k = rm.clone(), rv.clone()
        mean = rstd = None
        if use_bn:
            if training:
                s, q = K_.colstats(z)
                mean, rstd = K_.bn_finalize(s, q, rows, h, None, rm_k, rv_k, DEV)
            else:
                mean, rstd = K_.bn_finalize(None, None, rows, h, None, rm_k, rv_k, DEV)
        gm, bt = (gamma, beta) if use_bn else (None, None)
        y, _ = K_.bn_fwd(z, None, None, mean, rstd, gm, bt, None, use_bn, K_.ACT_ELU, p, seed, 1.0, None, True, False)
        dz, sums, _ = K_.bn_bwd(dy, None, None, z, mean, rstd, gm, bt, None, use_bn, K_.ACT_ELU, training, p, seed, 1.0)
        if use_bn and not training:
            sums = K_.bn_bwd_sums(dy, None, None, z, mean, rstd, gamma, beta, None, True, K_.ACT_ELU, p, seed, 1.0)
        zd = z.double().requires_grad_(True)
        gd, bd = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
        if use_bn:
            mu, var = (zd.mean(0), zd.var(0, unbiased=False)) if training else (rm.double(), rv.double())
            t = (zd - mu) / torch.sqrt(var + 1e-5) * gd + bd
        else:
            t = zd
        t = F.elu(t) * dmask(seed, rows, h, p)
        (t * dy.double()).sum().backward()
        tag = f"bn={use_bn} training={training} p={p}"
        _close(y, t, tol, f"y {tag}")
        _close(dz, zd.grad, tol if not (use_bn and training) else 4 * tol, f"dz {tag}")
        if use_bn:
            _close(sums[:h], bd.grad, 1e-5, f"dbeta {tag}", rows)
            _close(sums[h:], gd.grad, 1e-5, f"dgamma {tag}", rows)
            if training:
                zz = z.double()
                _close(rm_k, 0.9 * rm.double() + 0.1 * zz.mean(0), 1e-5, f"running_mean {tag}")
                _close(rv_k, 0.9 * rv.double() + 0.1 * zz.var(0, unbiased=True), 1e-5, f"running_var {tag}")
            else:
                assert torch.equal(rm_k, rm) and torch.equal(rv_k, rv), "eval BatchNorm changed its running buffers"


# ------------------------------------------------------------------------------------------------
# (e) modules at the recipe widths
# ------------------------------------------------------------------------------------------------
class Data:
    def __init__(self, x, ei):
        self.graph = {"node_feat": x, "edge_index": ei, "num_nodes": x.shape[0]}


# Allowed relative Frobenius error of a gradient against fp64: max(4 x the fp32 oracle's own error, FLOOR[class][precision]).
# Beside each floor: the worst error measured over (e) and (f) on an H100 80GB HBM3 (700 W limit), one run; a floor is at most
# 4x that.
FLOOR = {
    "weight":    {"fp32": 1.4e-5, "bf16": 0.14},   # 3.7e-6 / 3.7e-2
    "bn_weight": {"fp32": 1.4e-5, "bf16": 0.2},    # 3.5e-6 / 5.2e-2
    "att":       {"fp32": 1.8e-5, "bf16": 0.6},    # 4.6e-6 / 1.7e-1
    "affine":    {"fp32": 1.9e-3, "bf16": 0.25},   # 4.8e-4 / 6.4e-2
    "grad_x":    {"fp32": 8e-6, "bf16": 0.2},      # 2.0e-6 / 5.1e-2
}
# The bf16 attention-vector floor is wide because d att = sum_n d a_n xp_n ends in the cancellation A - r B of the softmax
# backward: the fp32 oracle's own 4.6e-6 is ~77 x its 2^-24 rounding, and 77 x the 2^-9 of a bf16-stored xp is ~0.15, the
# 0.17 measured.  The element-wise da_src / da_dst bounds of (a) carry the kernels' real precision there.
# SGFormer(gnn=GAT)'s attention-branch and head gradients keep the classes and floors of config_matrix.check.
LOGIT_TOL = {"fp32": 1e-4, "bf16": 1e-2}           # the project's logit tolerances; measured 2.3e-6 / 9.3e-3
BUFFER_TOL = {"fp32": 1.9e-6, "bf16": 1.8e-3}      # 4.8e-7 / 4.5e-4


def grad_class(name, layers, use_bn):
    """att: attention vectors; bn_weight: lin_src of a conv that feeds a BatchNorm; affine: biases and BatchNorm affines."""
    if name == "__x__":
        return "grad_x"
    if name.endswith("att_src") or name.endswith("att_dst"):
        return "att"
    if name.endswith("lin_src.weight"):
        i = int(name.split("convs.")[1].split(".")[0])
        return "bn_weight" if use_bn and i < layers - 1 else "weight"
    return "affine"


def rel_err(name, a, ref):
    """Relative Frobenius error.  A conv bias in front of a training BatchNorm has a zero true gradient: it is measured on
    1e-3 of its own layer's weight gradient (as config_matrix._sibling_scale)."""
    b = ref[name].double()
    a = a.detach().double().to(b.device)
    den = b.norm().item()
    if name.endswith(".bias") and ".bns." not in name and "convs." in name:
        w = ref[name[:-len("bias")] + "lin_src.weight"]
        den = max(den, 1e-3 * w.double().norm().item() / max(w.shape[1], 1) ** 0.5)
    e = (a - b).norm().item() / max(den, 1e-30)
    return e if e == e else float("inf")


def _max_rel(a, b):
    a, b = a.detach().double().to(b.device), b.double()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def _bound(k, got, ref64, ref32, precision, layers, use_bn, ocfg, ref64_cpu):
    """-> (report label, class, error, fp32 oracle's own error, floor) of gradient k.  With `ocfg` (an SGFormer config) the
    tensors outside the GAT branch are measured as config_matrix.check measures them."""
    if ocfg is not None and not k.startswith("gnn.") and k != "__x__":
        import config_matrix as CM
        cls = CM.tensor_class(k, ocfg)
        return ("sgformer", cls, CM.rel_err(k, got["grads"][k], ref64_cpu), CM.rel_err(k, ref32["grads"][k], ref64_cpu),
                CM.FLOOR[cls][precision])
    cls = grad_class(k, layers, use_bn)
    return ("module", cls, rel_err(k, got["grads"][k], ref64["grads"]), rel_err(k, ref32["grads"][k], ref64["grads"]),
            FLOOR[cls][precision])


def compare_step(got, ref64, ref32, precision, layers, use_bn, what, ocfg=None):
    """got / ref*: dict(out_eval, out_train, grads {name: tensor incl. '__x__'}, buffers {name: tensor}).  One line per bound
    violated, starting with the tensor's name."""
    problems = []
    tol = LOGIT_TOL[precision]
    for key in ("out_eval", "out_train"):
        e = _max_rel(got[key], ref64[key])
        _note(f"module {key} {precision}", e)
        if not e <= tol:
            problems.append(f"{key}: max err {e:.3e} of the reference's max > {tol} [{what}]")
    ref64_cpu = {k: v.detach().cpu() for k, v in ref64["grads"].items()} if ocfg is not None else None
    for k, g64 in ref64["grads"].items():
        if k not in got["grads"] or got["grads"][k] is None:
            problems.append(f"{k}: gradient missing [{what}]")
            continue
        label, cls, e, own, floor = _bound(k, got, ref64, ref32, precision, layers, use_bn, ocfg, ref64_cpu)
        allowed = max(4.0 * own, floor)
        _note(f"{label} {cls} {precision}", e)
        if not e <= allowed:
            problems.append(f"{k}: relative error {e:.3e} > {allowed:.3e} (class {cls}, fp32 oracle's own {own:.3e}) [{what}]")
    for k, v in ref64["buffers"].items():
        e = _max_rel(got["buffers"][k], v)
        _note(f"module buffer {precision}", e)
        if not e <= BUFFER_TOL[precision]:
            problems.append(f"{k}: buffer off by {e:.3e} of its max [{what}]")
    return problems


def _cora():
    g = torch.Generator().manual_seed(2708)
    n, d = 2708, 1433
    ei = torch.randint(0, n - 3, (2, 5278), generator=g)
    ei = torch.cat([ei, ei.flip(0), ei[:, :300], torch.arange(4).expand(2, 4)], 1)
    return n, d, ei


def _wide():
    n, d = 2 * _sms() * 128 + 7, 128
    g = torch.Generator().manual_seed(n)
    ei = torch.randint(0, n, (2, 4 * n), generator=g)
    hub = torch.stack([torch.randint(0, n, (3000,), generator=g), torch.full((3000,), 7)])
    return n, d, torch.cat([ei, hub], 1)


GRAPHS = {"cora": _cora, "wide": _wide}


def _ref_gat(d, h, c, layers, heads, out_heads, use_bn, dropout=0.0, seed=7):
    torch.manual_seed(seed)
    ref = G.GAT(d, h, c, num_layers=layers, dropout=dropout, use_bn=use_bn, heads=heads, out_heads=out_heads).double()
    with torch.no_grad():
        for conv in ref.convs:
            conv.bias.normal_(0, 0.1)
        for bn in ref.bns:
            bn.weight.uniform_(0.5, 1.5); bn.bias.normal_(0, 0.1)
            bn.running_mean.normal_(0, 0.1); bn.running_var.uniform_(0.5, 1.5)
    return ref


def _ours_gat(ref, d, h, c, layers, heads, out_heads, use_bn, precision, dropout=0.0):
    from sgformer_b200 import medium as M
    ours = M.GAT(d, h, c, num_layers=layers, dropout=dropout, use_bn=use_bn, heads=heads, out_heads=out_heads)
    ours.load_state_dict({k: v.float() if v.is_floating_point() else v for k, v in ref.state_dict().items()})
    return ours.to(DEV).set_precision(precision)


def _oracle_step(mod, x, ei, lw, dtype):
    """eval logits, train logits, gradients (incl. '__x__') and BatchNorm buffers of one oracle step on the device."""
    mod = copy.deepcopy(mod).to(DEV, dtype)
    xd, eid = x.to(DEV, dtype), ei.to(DEV)
    mod.eval()
    with torch.no_grad():
        out_eval = mod(Data(xd, eid))
    mod.train()
    xg = xd.clone().requires_grad_(True)
    out = mod(Data(xg, eid))
    (out * lw.to(DEV, dtype)).sum().backward()
    grads = {k: p.grad for k, p in mod.named_parameters() if p.grad is not None}
    grads["__x__"] = xg.grad
    buffers = {k: v for k, v in mod.state_dict().items() if "running" in k}
    return dict(out_eval=out_eval, out_train=out.detach(), grads=grads, buffers=buffers)


def _ours_step(mod, x, ei, lw):
    xd, eid = x.to(DEV, torch.float32), ei.to(DEV)
    mod.eval()
    with torch.no_grad():
        out_eval = mod(Data(xd, eid))
    mod.train()
    xg = xd.clone().requires_grad_(True)
    out = mod(Data(xg, eid))
    (out * lw.to(DEV)).sum().backward()
    grads = {k: p.grad for k, p in mod.named_parameters()}
    grads["__x__"] = xg.grad
    buffers = {k: v for k, v in mod.state_dict().items() if "running" in k}
    return dict(out_eval=out_eval, out_train=out.detach(), grads=grads, buffers=buffers)


# (layers, use_bn, out_heads, out_channels): the backbone (out = hidden 64) and the `--method gat` head (out = classes, a
# zero-padded head mean)
MODULE_CASES = [(2, True, 1, 64), (2, False, 2, 64), (3, True, 2, 64), (3, False, 1, 64), (2, True, 1, 7), (3, True, 2, 5)]
MODULE_PARAMS = [(gk, c, pr) for gk in GRAPHS for c in MODULE_CASES for pr in ("fp32", "bf16")]


@pytest.mark.parametrize("graph,case,precision", MODULE_PARAMS,
                         ids=[f"{gk}-L{c[0]}-bn{int(c[1])}-oh{c[2]}-c{c[3]}-{pr}" for gk, c, pr in MODULE_PARAMS])
def test_gat_module_at_recipe_width(graph, case, precision):
    layers, use_bn, out_heads, c = case
    n, d, ei = GRAPHS[graph]()
    h, heads = 64, 8
    ref = _ref_gat(d, h, c, layers, heads, out_heads, use_bn)
    ours = _ours_gat(ref, d, h, c, layers, heads, out_heads, use_bn, precision)
    gen = torch.Generator().manual_seed(n + layers)
    x = torch.randn(n, d, generator=gen, dtype=torch.float64)
    lw = torch.randn(n, c, generator=gen, dtype=torch.float64) / math.sqrt(n)
    r64, r32 = _oracle_step(ref, x, ei, lw, torch.float64), _oracle_step(ref, x, ei, lw, torch.float32)
    got = _ours_step(ours, x, ei, lw)
    problems = compare_step(got, r64, r32, precision, layers, use_bn, f"{graph} {case} {precision}")
    assert not problems, "\n".join(problems)


def _sgformer_pair(d, h, c, aggregate, precision):
    from oracle import sgformer_oracle as O
    from sgformer_b200 import medium as M
    ref_gnn = _ref_gat(d, h, h, 2, 8, 1, True)
    gnn = _ours_gat(ref_gnn, d, h, h, 2, 8, 1, True, "fp32")
    model = M.SGFormer(d, h, c, num_layers=1, num_heads=1, alpha=0.3, dropout=0.0, use_bn=True, gnn=gnn, aggregate=aggregate,
                       graph_weight=0.7).to(DEV).set_precision(precision)
    cfg = O.make_config("medium", d, h, c, num_layers=1, num_heads=1, alpha=0.3, dropout=0.0, use_bn=True, aggregate=aggregate,
                        graph_weight=0.7)
    sd = {k: v.detach().double().cpu().clone() for k, v in model.state_dict().items() if not k.startswith("gnn.")}
    assert all(v.is_floating_point() and "running" not in k for k, v in sd.items()), "the medium TransConv has LayerNorms only"

    class Ref(torch.nn.Module):
        """The GAT oracle as `gnn`; the attention branch and the head as parameters `p.<name with '.' -> '__'>` (ref_name)."""
        def __init__(self):
            super().__init__()
            self.gnn = ref_gnn
            self.p = torch.nn.ParameterDict({k.replace(".", "__"): torch.nn.Parameter(v) for k, v in sd.items()})

        def forward(self, data):
            x, ei = data.graph["node_feat"], data.graph["edge_index"]
            P = {k.replace("__", "."): v for k, v in self.p.items()}
            x1 = O.trans_conv(x, P, cfg, self.training)
            x2 = self.gnn(data)
            hcat = 0.7 * x2 + 0.3 * x1 if aggregate == "add" else torch.cat([x1, x2], 1)
            return F.linear(hcat, P["fc.weight"], P["fc.bias"])
    return Ref(), model, cfg


def ref_name(k):
    """Name of a Ref parameter in the SGFormer module: 'p.trans_conv__fcs__0__weight' -> 'trans_conv.fcs.0.weight'."""
    return k[len("p."):].replace("__", ".") if k.startswith("p.") else k


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("aggregate", ["add", "cat"])
def test_sgformer_gat_at_recipe_width(aggregate, precision):
    """SGFormer(gnn=GAT) with hidden 64 x 8 heads on the Cora-shaped graph: eval and train logits, every parameter gradient (the
    attention branch's and the head's in config_matrix.check's classes), the input gradient and the GAT branch's BatchNorm
    buffers."""
    n, d, ei = _cora()
    h, c = 64, 7
    ref, model, cfg = _sgformer_pair(d, h, c, aggregate, precision)
    gen = torch.Generator().manual_seed(17)
    x = torch.randn(n, d, generator=gen, dtype=torch.float64)
    lw = torch.randn(n, c, generator=gen, dtype=torch.float64) / math.sqrt(n)
    r64, r32 = _oracle_step(ref, x, ei, lw, torch.float64), _oracle_step(ref, x, ei, lw, torch.float32)
    got = _ours_step(model, x, ei, lw)
    rename = lambda r: dict(r, grads={ref_name(k): v for k, v in r["grads"].items()})
    r64, r32 = rename(r64), rename(r32)
    ours = {k for k, v in got["grads"].items() if v is not None}
    assert set(r64["grads"]) == ours, sorted(set(r64["grads"]) ^ ours)
    assert set(r64["buffers"]) == set(got["buffers"]) and any(k.startswith("gnn.bns.") for k in r64["buffers"])
    problems = compare_step(got, r64, r32, precision, 2, True, f"SGFormer(gnn=GAT) {aggregate} {precision}", ocfg=cfg)
    assert not problems, "\n".join(problems)


# ------------------------------------------------------------------------------------------------
# (f) a training step with all three dropout streams
# ------------------------------------------------------------------------------------------------
STEP_SEED = 0x5EED


def _masked_oracle(ref, x, ei, lw, p, seed, epoch, dtype):
    """fp64 / fp32 forward of models.GAT rebuilt layer by layer with the kernels' masks: input dropout (seed + _SEED_GAT_INPUT),
    attention dropout (seed + _SEED_GAT_ATT + i, through GATConv's edge_factor), post-ELU dropout (seed + _SEED_GAT_ACT + i)."""
    from sgformer_b200 import engine as E
    mod = copy.deepcopy(ref).to(DEV, dtype)
    mod.train()
    n, d = x.shape
    xg = x.to(DEV, dtype).clone().requires_grad_(True)
    eid = ei.to(DEV)
    edges = G.gat_edges(ei, n)
    sc = keep_scale(p)
    h = xg * (W.dense_keep(W.with_epoch(seed + E._SEED_GAT_INPUT, epoch), n, d, p).to(DEV, dtype) * sc)
    for i, conv in enumerate(mod.convs):
        fac = W.edge_keep(W.with_epoch(seed + E._SEED_GAT_ATT + i, epoch), n, edges, conv.heads, p).to(DEV, dtype)
        h = conv(h, eid, edge_factor=fac)
        if i < len(mod.convs) - 1:
            if mod.use_bn:
                h = mod.bns[i](h)
            h = F.elu(h)
            m = torch.from_numpy(keep_mask(seed + E._SEED_GAT_ACT + i, n, h.shape[1], p, epoch)).to(DEV, dtype)
            h = h * (m * sc)
    (h * lw.to(DEV, dtype)).sum().backward()
    grads = {k: q.grad for k, q in mod.named_parameters() if q.grad is not None}
    grads["__x__"] = xg.grad
    buffers = {k: v for k, v in mod.state_dict().items() if "running" in k}
    return dict(out_train=h.detach(), grads=grads, buffers=buffers)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_training_step_with_all_dropout_streams(monkeypatch, precision):
    from sgformer_b200 import engine as E
    monkeypatch.setattr(E, "next_seed", lambda: STEP_SEED)
    n, d, ei = _cora()
    h, c, layers, p = 64, 64, 3, 0.5
    ref = _ref_gat(d, h, c, layers, 8, 2, True, dropout=p)
    ours = _ours_gat(ref, d, h, c, layers, 8, 2, True, precision, dropout=p)
    gen = torch.Generator().manual_seed(23)
    x = torch.randn(n, d, generator=gen, dtype=torch.float64)
    lw = torch.randn(n, c, generator=gen, dtype=torch.float64) / math.sqrt(n)
    ours.train()
    xg = x.to(DEV, torch.float32).clone().requires_grad_(True)
    out = ours(Data(xg, ei.to(DEV)))
    epoch = current_epoch()
    (out * lw.to(DEV)).sum().backward()
    got = dict(out_train=out.detach(), grads=dict({k: q.grad for k, q in ours.named_parameters()}, __x__=xg.grad),
               buffers={k: v for k, v in ours.state_dict().items() if "running" in k})
    r64 = _masked_oracle(ref, x, ei, lw, p, STEP_SEED, epoch, torch.float64)
    r32 = _masked_oracle(ref, x, ei, lw, p, STEP_SEED, epoch, torch.float32)
    for r in (got, r64, r32):
        r["out_eval"] = r["out_train"]
    problems = compare_step(got, r64, r32, precision, layers, True, f"dropout step {precision}")
    assert not problems, "\n".join(problems)
    # the masks matter: without them the oracle is far away
    ref_p0 = copy.deepcopy(ref)
    ref_p0.dropout = 0.0
    for conv in ref_p0.convs:
        conv.dropout = 0.0
    ref0 = _oracle_step(ref_p0, x, ei, lw, torch.float64)["out_train"]
    assert (ref0 - r64["out_train"]).abs().max() > 100 * LOGIT_TOL["fp32"] * r64["out_train"].abs().max()


# ------------------------------------------------------------------------------------------------
# (g) planted errors and bit identity
# ------------------------------------------------------------------------------------------------
def test_planted_errors_are_reported_by_name(Kmod):
    # 1. the last valid chunk of one dxp row at (7, 72) fp32 (chunk 125 of 126), scaled by 1 + 1e-3
    shape = ("fp32", 7, 72, False)
    got, ref, S, _ = run_kernels(Kmod, "base", shape, 0.0)
    assert not check_outputs(got, ref, S, "fp32")
    cols = slice(125 * 4, 126 * 4)
    j = int(torch.argmax((ref["dxp"][:, cols].abs() / S["dxp"][:, cols]).min(1).values))
    bad = got["dxp"].clone()
    bad[j, cols] *= 1 + 1e-3
    lines = W.check_elementwise("dxp", bad, ref["dxp"], S["dxp"], K["dxp"], False)
    assert lines and lines[0].startswith("dxp:"), lines
    # 2. one head of lse on the hub row (node 0), + 1e-4; 3. one head of da_dst scaled by 1.01
    shape = ("fp32", 8, 64, False)
    got, ref, S, _ = run_kernels(Kmod, "base", shape, 0.5)
    assert not check_outputs(got, ref, S, "fp32")
    lse = got["lse"].clone()
    lse[0, 3] += 1e-4
    lines = W.check_elementwise("lse", lse, ref["lse"], S["lse"], K["lse"], False)
    assert lines and lines[0].startswith("lse:"), lines
    da = got["da_dst"].clone()
    da[5] *= 1.01
    lines = W.check_elementwise("da_dst", da, ref["da_dst"], S["da_dst"], K["da_dst"], False)
    assert lines and lines[0].startswith("da_dst:"), lines
    # 4. the reference with the duplicate rank shifted by one on the run of 70 that crosses entries 32 and 64 of row 100
    for shape in (("fp32", 8, 16, False), ("fp32", 8, 64, False)):
        got, ref, S, ctx = run_kernels(Kmod, "runs", shape, 0.5, seed=0xD0B1E)
        assert not check_outputs(got, ref, S, "fp32")
        n, edges = ctx["n"], ctx["edges"]
        rank = W.duplicate_rank(edges[0].numpy(), edges[1].numpy(), n)
        run = ((edges[0] == 50) & (edges[1] == 100)).numpy()
        assert run.sum() == 70
        rank[run] += 1
        fac = W.edge_keep(ctx["seed_eff"], n, edges, shape[1], 0.5, rank=rank)
        ref2, S2 = reference(ctx["graph"], n, ctx["xp"], ctx["a_s"], ctx["a_d"], ctx["lse"], ctx["att_s"], ctx["att_d"],
                             ctx["bias"], ctx["g"], shape[1], shape[2], shape[3], fac)
        lines = W.check_elementwise("out", got["out"], ref2["out"], S2["out"], K["out"], False)
        assert lines and lines[0].startswith("out:"), lines


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_training_step_bit_identical_at_recipe_width(monkeypatch, precision):
    from sgformer_b200 import engine as E
    monkeypatch.setattr(E, "next_seed", lambda: 0x5EED)
    n, d, ei = _cora()
    ref = _ref_gat(d, 64, 64, 3, 8, 2, True, dropout=0.4)
    model = _ours_gat(ref, d, 64, 64, 3, 8, 2, True, precision, dropout=0.4)
    x = torch.randn(n, d, device=DEV)
    wgt = torch.randn(n, 64, device=DEV)
    eid = ei.to(DEV)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    runs = []
    for _ in range(2):
        model.load_state_dict(sd)
        for q in model.parameters():
            q.grad = None
        xo = x.clone().requires_grad_(True)
        out = model(Data(xo, eid))
        (out * wgt).sum().backward()
        runs.append((out.detach().clone(), [q.grad.clone() for q in model.parameters()], xo.grad.clone(),
                     [v.clone() for k, v in model.state_dict().items() if "running" in k]))
    (o1, g1, x1, b1), (o2, g2, x2, b2) = runs
    assert torch.equal(o1, o2) and torch.equal(x1, x2)
    assert all(torch.equal(a, b) for a, b in zip(g1, g2))
    assert all(torch.equal(a, b) for a, b in zip(b1, b2))
