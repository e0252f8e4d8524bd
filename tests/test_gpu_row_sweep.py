"""The row kernels of csrc/rowops.cu against fp64 at row counts where every lane group of the capped grid processes several rows.

Each row kernel is software-pipelined: while a lane group works on row r, row r + row_step is already loading (packed registers,
or the cp.async ring of the BatchNorm backward), and column sums accumulate per lane across the rows.  `row_grid` caps the grid
at 8 blocks of 8 warps per SM, so row_step = 64 * SMs * rows-per-warp and a lane group sees a second row only when
rows > row_step: tens of thousands of rows at the wide geometries, hundreds of thousands at the narrow ones.  The plans below
restate the kernels' geometry and pick row counts past that point:

  ragged  3 * row_step + tail: every group runs 3 or 4 rows, and the last warp has live and dead groups;
  exact   3 * row_step: the last prefetch of every group lands on the `rn < rows` boundary;
  ring    6 * row_step + tail (BatchNorm backward, one chunk per lane): every group refills the 4-stage ring.

Inputs are random per row, so a row read in place of another shows as an O(1) error.  The checks: every kernel pair against
fp64 with the kernels' own dropout masks replayed; column-sliced (pitched) operands whose padding must stay untouched; the
non-default sides of the launch switches (SGF_BN_BWD_RING=0, SGF_LNATTN_BLOCKS=3, SGF_PACK_VEC=0) in a child process, bit
for bit against the default path (except the accumulated BatchNorm dres, which the two BatchNorm pipelines round differently,
see _one_product_rounding_apart); BatchNorm sharded by rows on one device; run-to-run bit identity of every reduction; and a
planted row swap that the comparison must report."""
import contextlib
import functools
import os
import subprocess
import sys
import tempfile

import pytest
import torch

from dropout_mask import current_epoch, keep_mask, keep_scale
from row_ref import BN_CASES, attn_reference, bn_reference, bn_untie, check_bn_chain, close, ln_reference, untie

gpu = pytest.mark.gpu
DEV = "cuda"
F32, B16 = torch.float32, torch.bfloat16

# ------------------------------------------------------------------------------------------------
# the row plan: make_geom / row_grid of csrc/rowops.cu
# ------------------------------------------------------------------------------------------------
ROW_BLOCK, BLOCKS_PER_SM, RING_DEPTH = 256, 8, 4

# (dtype, h) -> (lanes per row, chunks per lane): every geometry of the row kernels
SHAPES = {(F32, 4): (1, 1), (F32, 12): (4, 1), (F32, 64): (16, 1), (F32, 100): (32, 1), (F32, 256): (32, 2), (F32, 300): (32, 3),
          (F32, 512): (32, 4), (B16, 8): (1, 1), (B16, 24): (4, 1), (B16, 200): (32, 1), (B16, 256): (32, 1), (B16, 768): (32, 3),
          (B16, 1024): (32, 4)}
SHAPE_LIST = list(SHAPES)
SHAPE_IDS = [f"{'fp32' if d == F32 else 'bf16'}-h{h}" for d, h in SHAPE_LIST]


def geom(dtype, h, rows, sms):
    """make_geom + row_grid: chunks, lanes per row, chunks per lane, rows per warp, grid and row_step of a launch."""
    vn = 8 if dtype == B16 else 4
    assert h % vn == 0
    chunks = h // vn
    lpr_log2 = 0
    while (1 << lpr_log2) < chunks and lpr_log2 < 5:
        lpr_log2 += 1
    lpr = 1 << lpr_log2
    rpw = 32 // lpr
    warps = -(-rows // rpw)
    grid = max(1, min(-(-warps * 32 // ROW_BLOCK), sms * BLOCKS_PER_SM))
    return dict(chunks=chunks, lpr=lpr, cpl=-(-chunks // lpr), rpw=rpw, grid=grid, row_step=grid * (ROW_BLOCK // 32) * rpw)


def full_step(dtype, h, sms):
    """row_step of the capped grid."""
    return BLOCKS_PER_SM * (ROW_BLOCK // 32) * sms * geom(dtype, h, 1, sms)["rpw"]


def plan_rows(dtype, h, plan, sms):
    step = full_step(dtype, h, sms)
    tail = step // 2 + 1          # row_step is a multiple of rows-per-warp: the tail ends inside a warp
    return {"ragged": 3 * step + tail, "exact": 3 * step, "ring": 6 * step + tail}[plan]


def rows_per_group(rows, step):
    """(fewest, most) rows a lane group of the capped grid processes."""
    return rows // step, -(-rows // step)


def plans_for(dtype, h, bn=False):
    """The plans a kernel runs at: ragged and exact, and the ring plan for a BatchNorm backward with one chunk per lane."""
    return ["ragged", "exact"] + (["ring"] if bn and SHAPES[(dtype, h)][1] == 1 else [])


@pytest.mark.parametrize("sms", [132, 114])
def test_row_plan_sweeps_every_lane_group(sms):
    """The plans reach what the GPU tests below are for, on a 132-SM and a 114-SM H100: the capped grid, several rows per lane
    group, a ragged tail, the prefetch boundary and ring refills; and the shapes cover every geometry."""
    geoms = set()
    for (dtype, h), (lpr, cpl) in SHAPES.items():
        big = geom(dtype, h, 1 << 40, sms)
        assert (big["lpr"], big["cpl"]) == (lpr, cpl), (dtype, h, big)
        geoms.add((dtype, lpr, cpl))
        step = full_step(dtype, h, sms)
        assert step == big["row_step"] == 64 * sms * big["rpw"]
        for plan in plans_for(dtype, h, bn=True):
            rows = plan_rows(dtype, h, plan, sms)
            g = geom(dtype, h, rows, sms)
            assert g["grid"] == sms * BLOCKS_PER_SM and g["row_step"] == step, (dtype, h, plan, g)
            lo, hi = rows_per_group(rows, step)
            tail = rows % step
            if plan == "exact":
                assert tail == 0 and lo == hi == 3, (dtype, h, lo, hi)
            else:
                assert 0 < tail < step and hi == lo + 1, (dtype, h, plan, tail)
                assert g["rpw"] == 1 or tail % g["rpw"] != 0, "the tail must end inside a warp"
                assert lo >= (3 if plan == "ragged" else RING_DEPTH + 2), (dtype, h, plan, lo)
        if cpl == 1:
            assert "ring" in plans_for(dtype, h, bn=True)
    for dtype in (F32, B16):
        assert {(lpr, cpl) for d, lpr, cpl in geoms if d == dtype} >= {(1, 1), (4, 1), (32, 1), (32, 3), (32, 4)}
    assert (F32, 32, 2) in geoms and (F32, 16, 1) in geoms
    partial = [(d, h) for (d, h) in SHAPES if geom(d, h, 1, sms)["chunks"] % 32 and SHAPES[(d, h)][0] == 32]
    assert {(F32, 100), (F32, 300), (B16, 200)} <= set(partial), "dead lanes and partially live chunks"


# ------------------------------------------------------------------------------------------------
# inputs, masks, comparisons
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def K():
    from sgformer_b200 import kernels
    return kernels


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _tol(dtype):
    return 2e-5 if dtype == F32 else 5e-3


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _rand(rows, h, dtype, g, scale=1.0):
    return (scale * torch.randn(rows, h, generator=g, device=DEV)).to(dtype)


def _act(rows, h, dtype, g):
    """A LayerNorm operand: random per row plus a column ramp, so that no row of hundreds of thousands is nearly constant (the
    fp32 variance of such a row loses digits that have nothing to do with the pipeline)."""
    ramp = torch.linspace(-1.5, 1.5, h, device=DEV)
    return (0.8 * torch.randn(rows, h, generator=g, device=DEV) + ramp).to(dtype)


def _vec(h, g, lo, scale):
    return lo + scale * torch.randn(h, generator=g, device=DEV)


def _pos(rows, g, lo):
    return lo + torch.rand(rows, generator=g, device=DEV)


@functools.lru_cache(maxsize=24)
def _device_mask(seed, rows, h, p, epoch):
    return torch.from_numpy(keep_mask(seed, rows, h, p, epoch)).to(DEV)


def dmask(seed, rows, h, p):
    """fp64 mask * kernel scale for the epoch word as it stands (1 when p = 0: the no-dropout instantiation)."""
    if p == 0.0:
        return torch.ones((), dtype=torch.float64, device=DEV)
    return _device_mask(seed, rows, h, p, current_epoch()).double() * keep_scale(p)


def _same(a, b, what):
    """Bit identity of two runs' outputs (dicts of tensors / None)."""
    for k, v in a.items():
        if isinstance(v, torch.Tensor):
            assert torch.equal(v, b[k]), f"{what}: {k} differs between two runs"


@contextlib.contextmanager
def no_epoch_word(K):
    """Unregister the process-global dropout epoch word (another test may have registered it) for the duration, so a child
    process without one draws the same masks."""
    saved = K._epoch
    if saved is not None:
        K.lib().sgf_set_dropout_epoch(None)
        K._epoch = None
    try:
        yield
    finally:
        if saved is not None:
            K._epoch = saved
            K.lib().sgf_set_dropout_epoch(K._p(saved))


def _p_for(k):
    return (0.0, 0.5)[k % 2]      # both DROP instantiations


# ------------------------------------------------------------------------------------------------
# kernel runs (inputs -> outputs) and their fp64 checks
# ------------------------------------------------------------------------------------------------
def ln_inputs(dtype, rows, h, seed):
    g = _gen(seed)
    x, r, gy, xa = (_act(rows, h, dtype, g) for _ in range(4))
    dy = _rand(rows, h, dtype, g)
    return dict(x=x, r=r, gy=gy, xa=xa, dy=dy, gamma=_vec(h, g, 1.0, 0.2), beta=_vec(h, g, 0.0, 0.2), den=_pos(rows, g, 1.0),
                dinv=_pos(rows, g, 0.0))


def run_ln(K, I, relu, with_r, p, seed):
    h = I["x"].shape[1]
    r = I["r"] if with_r else None
    a, b = (0.7, 0.3) if with_r else (1.3, 0.0)
    y, st = K.ln_fwd(I["x"], r, a, b, I["gamma"], I["beta"], True, relu, p, seed)
    dg, db = torch.zeros(h, device=DEV), torch.zeros(h, device=DEV)
    dx, dr = K.ln_bwd(I["dy"], I["x"], r, a, b, I["gamma"], I["beta"], st, True, relu, p, seed, 0.75, with_r, dg, db)
    return dict(y=y, stats=st, dx=dx, dr=dr, dgamma=dg, dbeta=db)


def check_ln(I, out, relu, with_r, p, seed, tol, tag):
    rows, h = I["x"].shape
    r = I["r"] if with_r else None
    a, b = (0.7, 0.3) if with_r else (1.3, 0.0)
    R = ln_reference(I["x"], r, None, a, b, 0.0, I["gamma"], I["beta"], True, relu, dmask(seed, rows, h, p), I["dy"], 0.75)
    close(out["y"], R["y"], tol, f"y {tag}")
    close(out["dx"], R["dx"], tol, f"dx {tag}")
    if with_r:
        close(out["dr"], R["dr"], tol, f"dr {tag}")
    close(out["dgamma"], R["dgamma"], 1e-5, f"dgamma {tag}", rows)
    close(out["dbeta"], R["dbeta"], 1e-5, f"dbeta {tag}", rows)


ATTN_AB = (0.61, 0.37)


def run_ln_attn(K, I, relu, alias, p, seed):
    h = I["x"].shape[1]
    a, b = ATTN_AB
    xa = I["r"] if alias else I["xa"]
    y, st = K.ln_fwd(I["x"], I["r"], a, b, I["gamma"], I["beta"], True, relu, p, seed)
    dg, db = torch.zeros(h, device=DEV), torch.zeros(h, device=DEV)
    gnum, gden, dr, cs, pg, sg = K.ln_bwd_attn(I["dy"], I["x"], I["r"], xa, a, b, I["gamma"], I["beta"], st, True, relu, p, seed,
                                               1.5, True, dg, db, I["den"])
    return dict(y=y, gnum=gnum, gden=gden, dr=dr, cs=cs, pg=pg, sg=sg, dgamma=dg, dbeta=db)


def check_ln_attn(I, out, relu, alias, p, seed, tol, tag):
    rows, h = I["x"].shape
    a, b = ATTN_AB
    xa = I["r"] if alias else I["xa"]
    R = ln_reference(I["x"], I["r"], None, a, b, 0.0, I["gamma"], I["beta"], True, relu, dmask(seed, rows, h, p), I["dy"], 1.5)
    A = attn_reference(R, I["x"], xa, a, I["den"])
    close(out["y"], R["y"], tol, f"y {tag}")
    close(out["gnum"], A["gnum"], tol, f"gnum {tag}")
    close(out["dr"], R["dr"], tol, f"dr {tag}")
    close(out["gden"], A["gden"], 1e-4, f"gden {tag}")
    for what in ("cs", "pg", "sg"):
        close(out[what], A[what], 1e-5, f"{what} {tag}", rows, A["elem"][what])
    close(out["dgamma"], R["dgamma"], 1e-5, f"dgamma {tag}", rows)
    close(out["dbeta"], R["dbeta"], 1e-5, f"dbeta {tag}", rows)


GRAPH_ABC = (0.5, 0.3, 0.8)


def run_graph(K, I, alias, p, seed):
    h = I["x"].shape[1]
    a, b, c = GRAPH_ABC
    xa = I["r"] if alias else I["xa"]
    y, st = K.ln_fwd_graph(I["x"], I["r"], I["gy"], a, b, c, I["gamma"], I["beta"], True, False, p, seed)
    dg, db = torch.zeros(h, device=DEV), torch.zeros(h, device=DEV)
    gnum, gden, dr, ys, cs, pg, sg = K.ln_bwd_attn_graph(I["dy"], I["x"], I["r"], xa, I["gy"], a, b, c, I["gamma"], I["beta"], st,
                                                         True, p, seed, 1.0, True, dg, db, I["den"], I["dinv"])
    return dict(y=y, gnum=gnum, gden=gden, dr=dr, ys=ys, cs=cs, pg=pg, sg=sg, dgamma=dg, dbeta=db)


def check_graph(I, out, alias, p, seed, tol, tag):
    rows, h = I["x"].shape
    a, b, c = GRAPH_ABC
    xa = I["r"] if alias else I["xa"]
    R = ln_reference(I["x"], I["r"], I["gy"], a, b, c, I["gamma"], I["beta"], True, False, dmask(seed, rows, h, p), I["dy"], 1.0)
    A = attn_reference(R, I["x"], xa, a, I["den"])
    close(out["y"], R["y"], tol, f"y {tag}")
    close(out["gnum"], A["gnum"], tol, f"gnum {tag}")
    close(out["ys"], I["dinv"].double()[:, None] * c * R["du"], tol, f"ys {tag}")
    close(out["dr"], b * R["du"], tol, f"dr {tag}")
    close(out["gden"], A["gden"], 1e-4, f"gden {tag}")
    for what in ("cs", "pg", "sg"):
        close(out[what], A[what], 1e-5, f"{what} {tag}", rows, A["elem"][what])
    close(out["dgamma"], R["dgamma"], 1e-5, f"dgamma {tag}", rows)
    close(out["dbeta"], R["dbeta"], 1e-5, f"dbeta {tag}", rows)


def run_colstats(K, I):
    s_w, q_w = K.colstats(I["x"], I["w"])
    s, q = K.colstats(I["x"])
    return dict(sum_w=s_w, sumsq_w=q_w, sum=s, sumsq=q)


def check_colstats(I, out, tag):
    x, w = I["x"].double(), I["w"].double()
    rows = x.shape[0]
    xw = x * w[:, None]
    close(out["sum_w"], xw.sum(0), 1e-5, f"weighted sum {tag}", rows, xw.abs().max().item())
    close(out["sum"], x.sum(0), 1e-5, f"sum {tag}", rows, x.abs().max().item())
    for k in ("sumsq_w", "sumsq"):
        close(out[k], (x * x).sum(0), 1e-5, f"{k} {tag}", rows)


def bn_inputs(dtype, rows, h, case, seed):
    g = _gen(seed)
    z, res, mix, dy, dy2, dres0 = (_rand(rows, h, dtype, g, 1.5) for _ in range(6))
    I = dict(z=z, res=res, mix=mix, dy=dy, dy2=dy2, dres0=dres0, gamma=_vec(h, g, 1.0, 0.2), beta=_vec(h, g, 0.0, 0.2),
             rm=_vec(h, g, 0.0, 0.1), rv=1 + 0.3 * torch.rand(h, generator=g, device=DEV), rs=_pos(rows, g, 0.2),
             rs2=_pos(rows, g, 0.2), ors=_pos(rows, g, 0.2))
    I["dy"], I["dy2"] = bn_untie(case, z, I["gamma"], I["beta"], I["rm"], I["rv"], dy, dy2)
    return I


BN_GW, BN_GSCALE = 0.7, 0.9


def run_bn(K, I, case, p, seed):
    use_bn, training, relu, with_res, with_mix, with_dy2, dres_acc, with_ors = case
    rows, h = I["z"].shape
    mean = rstd = None
    if use_bn:
        if training:
            s, q = K.colstats(I["z"])
            mean, rstd = K.bn_finalize(s, q, rows, h, None, I["rm"].clone(), I["rv"].clone(), DEV)
        else:
            mean, rstd = K.bn_finalize(None, None, rows, h, None, I["rm"], I["rv"], DEV)
    gamma, beta = (I["gamma"], I["beta"]) if use_bn else (None, None)
    y, ys = K.bn_fwd(I["z"], I["res"] if with_res else None, I["mix"] if with_mix else None, mean, rstd, gamma, beta, None, use_bn,
                     relu, p, seed, BN_GW, I["rs"], True, True)
    dy2, rs2 = (I["dy2"], I["rs2"]) if with_dy2 else (None, None)
    dres = K.new_like(I["dres0"]).copy_(I["dres0"])
    dz, sums, colsum = K.bn_bwd(I["dy"], dy2, rs2, I["z"], mean, rstd, gamma, beta, None, use_bn, relu, training, p, seed, BN_GSCALE,
                                dres=dres, dres_accumulate=dres_acc, want_dz_colsum=True,
                                out_row_scale=I["ors"] if with_ors else None)
    if use_bn and not training:
        sums = K.bn_bwd_sums(I["dy"], dy2, rs2, I["z"], mean, rstd, gamma, beta, None, True, relu, p, seed, BN_GSCALE)
    return dict(y=y, ys=ys, dres=dres, dz=dz, colsum=colsum, sums=sums)


def check_bn(I, out, case, p, seed, tol, tag):
    rows, h = I["z"].shape
    ref = bn_reference(case, I["z"], I["res"], I["mix"], I["dy"], I["dy2"], I["dres0"], I["gamma"], I["beta"], I["rm"], I["rv"],
                       I["rs"], I["rs2"], I["ors"], BN_GW, BN_GSCALE, dmask(seed, rows, h, p))
    check_bn_chain(out, ref, case, tol, tag, rows, h)


# ---- jumping knowledge over 3 layers: operands on a grid of 1/16 with power-of-two BatchNorm scales, so that every fp32 product
# and sum of the forward row pass is exact and the maxima and layer indices can be compared bit for bit
JK_LAYERS = 3


def jk_inputs(dtype, rows, h, seed):
    g = _gen(seed)
    q = lambda shape, lo, hi: torch.randint(lo, hi, shape, generator=g, device=DEV).double() / 16
    layers = []
    for l in range(JK_LAYERS):
        bn = l < JK_LAYERS - 1                     # the last GCN layer has no BatchNorm and no ReLU
        P = dict(z=q((rows, h), -48, 48).to(dtype), zb=q((h,), -8, 8).float())
        if bn:
            P.update(mean=q((h,), -8, 8).float(), rstd=2.0 ** torch.randint(-1, 2, (h,), generator=g, device=DEV).float(),
                     gamma=2.0 ** torch.randint(-1, 1, (h,), generator=g, device=DEV).float(), beta=q((h,), -8, 8).float())
        P["dy"] = _rand(rows, h, dtype, g) if bn else None
        layers.append(P)
    g_out = _rand(rows, JK_LAYERS * h, dtype, g)     # cat: the gradient of the concatenation; max: its first block
    return dict(layers=layers, g_out=g_out)


def _jk_act(P):
    v = P["z"].double() + P["zb"].double()
    if "mean" in P:
        v = ((v - P["mean"].double()) * P["rstd"].double() * P["gamma"].double() + P["beta"].double()).clamp_min(0)
    return v


def run_jk(K, I, mode, p, seed):
    rows, h = I["layers"][0]["z"].shape
    dtype = I["layers"][0]["z"].dtype
    if mode == "max":
        buf = K.alloc_act(rows, h, dtype, DEV)
        idx = torch.zeros((rows, buf.stride(0)), dtype=torch.uint8, device=DEV)
        blocks = [buf] * JK_LAYERS
    else:
        buf = K.alloc_act(rows, JK_LAYERS * h, dtype, DEV)
        idx = None
        blocks = [buf[:, l * h:(l + 1) * h] for l in range(JK_LAYERS)]
    out = {}
    for l, P in enumerate(I["layers"]):
        bn = "mean" in P
        out[f"y{l}"] = K.bn_fwd_jk(P["z"], P.get("mean"), P.get("rstd"), P.get("gamma"), P.get("beta"), P["zb"], bn, bn,
                                   p if bn else 0.0, seed + l, True, mode, blocks[l], idx, l)
    out["jk"] = buf.clone()
    out["idx"] = idx[:, :h].clone() if idx is not None else None
    g_out = I["g_out"]
    gblocks = [g_out[:, :h].contiguous()] * JK_LAYERS if mode == "max" else [g_out[:, l * h:(l + 1) * h] for l in range(JK_LAYERS)]
    for l, P in enumerate(I["layers"]):
        bn = "mean" in P
        dz, sums, colsum = K.bn_bwd_jk(P["dy"], P["z"], P.get("mean"), P.get("rstd"), P.get("gamma"), P.get("beta"), P["zb"], bn,
                                       bn, True, p if bn else 0.0, seed + l, mode, gblocks[l], idx, l, want_dz_colsum=True)
        out[f"dz{l}"], out[f"sums{l}"], out[f"colsum{l}"] = dz, sums, colsum
    return out


def check_jk(I, out, mode, p, seed, tol, tag):
    rows, h = I["layers"][0]["z"].shape
    dtype = I["layers"][0]["z"].dtype
    acts = [_jk_act(P).to(dtype).double() for P in I["layers"]]           # as stored
    if mode == "max":
        ref_m, ref_i = torch.stack(acts, -1).max(-1)                        # first maximum: the lowest layer on ties
        assert torch.equal(out["jk"].double(), ref_m), f"jk max {tag}"
        assert torch.equal(out["idx"].long(), ref_i), f"jk layer index {tag}"
    else:
        assert torch.equal(out["jk"].double(), torch.cat(acts, 1)), f"jk cat {tag}"
    for l, P in enumerate(I["layers"]):
        bn = "mean" in P
        M = dmask(seed + l, rows, h, p if bn else 0.0)
        assert torch.equal(out[f"y{l}"].double(), (_jk_act(P) * M).to(dtype).double()), f"y of layer {l} {tag}"
        gj = I["g_out"][:, :h] if mode == "max" else I["g_out"][:, l * h:(l + 1) * h]
        add = gj.double() * (out["idx"].long() == l) if mode == "max" else gj.double()
        if not bn:                                  # no dy, no BatchNorm: dz is the JK gradient itself
            assert torch.equal(out[f"dz{l}"].double(), add), f"dz of layer {l} {tag}"
            close(out[f"colsum{l}"], add.sum(0), 1e-5, f"colsum of layer {l} {tag}", rows, add.abs().max().item())
            continue
        g = P["dy"].double() * M + add
        xh = (P["z"].double() + P["zb"].double() - P["mean"].double()) * P["rstd"].double()
        g = g * ((xh * P["gamma"].double() + P["beta"].double()) > 0)
        sums = torch.cat([g.sum(0), (g * xh).sum(0)])
        d = P["gamma"].double() * P["rstd"].double() * (g - sums[:h] / rows - xh * sums[h:] / rows)
        close(out[f"dz{l}"], d, 4 * tol, f"dz of layer {l} {tag}")
        close(out[f"sums{l}"][:h], sums[:h], 1e-5, f"dbeta of layer {l} {tag}", rows, g.abs().max().item())
        close(out[f"sums{l}"][h:], sums[h:], 1e-5, f"dgamma of layer {l} {tag}", rows, (g * xh).abs().max().item())
        close(out[f"colsum{l}"], d.sum(0), 1e-5, f"dz colsum of layer {l} {tag}", rows, d.abs().max().item())


def small_inputs(dtype, rows, h, seed):
    g = _gen(seed)
    return dict(g=_rand(rows, h, dtype, g), o=_rand(rows, h, dtype, g), den=_pos(rows, g, 1.0), heads=_rand(rows, 3 * h, dtype, g),
                x=_rand(rows, h, dtype, g), y=_rand(rows, h, dtype, g), rs=_pos(rows, g, 0.5))


AXPBY_AB = (0.25, -1.5)


def run_small(K, I, out_buf=None):
    """attn_bwd_prep, head_mean (3 heads of width h) and axpby (fp32 output; into out_buf when given)."""
    gnum, gden = K.attn_bwd_prep(I["g"], I["o"], I["den"], 0.5)
    hm = K.head_mean(I["heads"], 3, I["g"].shape[1])
    ax = K.axpby(I["x"], I["y"], *AXPBY_AB, out_dtype=F32, row_scale=I["rs"], out=out_buf)
    return dict(gnum=gnum, gden=gden, head_mean=hm, axpby=ax)


def check_small(I, out, tol, tag):
    rows, h = I["g"].shape
    gd, od, den = I["g"].double(), I["o"].double(), I["den"].double()[:, None]
    close(out["gnum"], 0.5 * gd / den, tol, f"attn_bwd_prep gnum {tag}")
    close(out["gden"], -0.5 * (gd * od).sum(1) / den[:, 0], 1e-4, f"attn_bwd_prep gden {tag}")
    close(out["head_mean"], I["heads"].double().reshape(rows, 3, h).mean(1), tol, f"head_mean {tag}")
    a, b = AXPBY_AB
    close(out["axpby"], (a * I["x"].double() + b * I["y"].double()) * I["rs"].double()[:, None], 2e-5, f"axpby {tag}")


# ------------------------------------------------------------------------------------------------
# the sweep: every kernel at every geometry and plan against fp64; the ragged plan runs twice (bit identity)
# ------------------------------------------------------------------------------------------------
def _sweep(shape, kernel_plans, run, check, seed0):
    """run(k, rows, seed) -> (inputs, outputs) and check(k, seed, inputs, outputs, tag) at every plan of the kernel."""
    dtype, h = shape
    for k, plan in enumerate(kernel_plans):
        rows = plan_rows(dtype, h, plan, _sms())
        seed = seed0 + 17 * k
        I, out = run(k, rows, seed)
        check(k, seed, I, out, f"{plan} rows={rows}")
        if plan == "ragged":
            _same(out, run(k, rows, seed)[1], f"{plan} rows={rows}")


@gpu
@pytest.mark.parametrize("dtype,h", SHAPE_LIST, ids=SHAPE_IDS)
def test_ln_pair_sweep(K, dtype, h):
    combos = [(True, True), (False, False)]          # (relu, with_r)

    def run(k, rows, seed):
        I = ln_inputs(dtype, rows, h, seed)
        relu, with_r = combos[k % 2]
        if relu:
            I["dy"] = untie(I["dy"], I["x"], I["r"] if with_r else None, 0.7, 0.3 if with_r else 0.0, I["gamma"], I["beta"], True)
        return I, run_ln(K, I, relu, with_r, _p_for(k), seed)

    def check(k, seed, I, out, tag):
        relu, with_r = combos[k % 2]
        check_ln(I, out, relu, with_r, _p_for(k), seed, _tol(dtype), f"{tag} relu={relu} r={with_r} p={_p_for(k)}")

    _sweep((dtype, h), plans_for(dtype, h), run, check, 1000 + h)


@gpu
@pytest.mark.parametrize("dtype,h", SHAPE_LIST, ids=SHAPE_IDS)
def test_ln_bwd_attn_pair_sweep(K, dtype, h):
    """Both ln_bwd_attn instantiations (with and without ReLU), with the layer input aliasing the residual and not."""
    for relu, alias in ((False, True), (True, False)):
        def run(k, rows, seed):
            I = ln_inputs(dtype, rows, h, seed)
            if relu:
                I["dy"] = untie(I["dy"], I["x"], I["r"], *ATTN_AB, I["gamma"], I["beta"], True)
            return I, run_ln_attn(K, I, relu, alias, _p_for(k + relu), seed)

        def check(k, seed, I, out, tag):
            p = _p_for(k + relu)
            check_ln_attn(I, out, relu, alias, p, seed, _tol(dtype), f"{tag} relu={relu} xa_is_r={alias} p={p}")

        _sweep((dtype, h), plans_for(dtype, h), run, check, 2000 + h + 100 * relu)


@gpu
@pytest.mark.parametrize("dtype,h", SHAPE_LIST, ids=SHAPE_IDS)
def test_ln_graph_pair_sweep(K, dtype, h):
    def run(k, rows, seed):
        I = ln_inputs(dtype, rows, h, seed)
        return I, run_graph(K, I, k % 2 == 0, _p_for(k + 1), seed)

    def check(k, seed, I, out, tag):
        p = _p_for(k + 1)
        check_graph(I, out, k % 2 == 0, p, seed, _tol(dtype), f"{tag} xa_is_r={k % 2 == 0} p={p}")

    _sweep((dtype, h), plans_for(dtype, h), run, check, 3000 + h)


@gpu
@pytest.mark.parametrize("dtype,h", SHAPE_LIST, ids=SHAPE_IDS)
def test_colstats_sweep(K, dtype, h):
    def run(k, rows, seed):
        g = _gen(seed)
        I = dict(x=_rand(rows, h, dtype, g, 2.0), w=torch.rand(rows, generator=g, device=DEV))
        return I, run_colstats(K, I)

    _sweep((dtype, h), plans_for(dtype, h), run, lambda k, seed, I, out, tag: check_colstats(I, out, tag), 4000 + h)


@gpu
@pytest.mark.parametrize("dtype,h", SHAPE_LIST, ids=SHAPE_IDS)
def test_bn_chain_sweep(K, dtype, h):
    """bn_fwd + bn_bwd (+ bn_bwd_sums) over every BN_CASES flag set; one chunk per lane also at the ring plan."""
    for c, case in enumerate(BN_CASES):
        def run(k, rows, seed):
            I = bn_inputs(dtype, rows, h, case, seed)
            return I, run_bn(K, I, case, _p_for(k + c), seed)

        def check(k, seed, I, out, tag):
            p = _p_for(k + c)
            check_bn(I, out, case, p, seed, _tol(dtype), f"{tag} case={case} p={p}")

        _sweep((dtype, h), plans_for(dtype, h, bn=True), run, check, 5000 + h + 100 * c)


@gpu
@pytest.mark.parametrize("mode", ["max", "cat"])
@pytest.mark.parametrize("dtype,h", SHAPE_LIST, ids=SHAPE_IDS)
def test_jk_sweep(K, dtype, h, mode):
    """bn_fwd_jk / bn_bwd_jk over 3 GCN layers (the register pipeline: the ring does not carry the JK addend)."""
    def run(k, rows, seed):
        I = jk_inputs(dtype, rows, h, seed)
        return I, run_jk(K, I, mode, _p_for(k + 1), seed)

    def check(k, seed, I, out, tag):
        check_jk(I, out, mode, _p_for(k + 1), seed, _tol(dtype), f"{tag} mode={mode}")

    _sweep((dtype, h), plans_for(dtype, h), run, check, 6000 + h)


@gpu
@pytest.mark.parametrize("dtype,h", SHAPE_LIST, ids=SHAPE_IDS)
def test_small_row_passes_sweep(K, dtype, h):
    """attn_bwd_prep, head_mean and axpby; axpby reads and writes three different pitches."""
    vn = 8 if dtype == B16 else 4

    def run(k, rows, seed):
        I = small_inputs(dtype, rows, h, seed)
        I["x"] = _pitched_copy(I["x"], h + vn)
        I["y"] = _pitched_copy(I["y"], h + 3 * vn)
        buf = torch.full((rows, h + 8), float("nan"), device=DEV)
        out = run_small(K, I, out_buf=buf[:, :h])
        assert torch.isnan(buf[:, h:]).all(), "axpby wrote into the padding of its output"
        return I, out

    _sweep((dtype, h), plans_for(dtype, h), run, lambda k, seed, I, out, tag: check_small(I, out, _tol(dtype), tag), 7000 + h)


def _pitched_copy(t, ld, fill=float("nan")):
    """t as the first t.shape[1] columns of a [rows, ld] buffer whose padding holds `fill`."""
    buf = torch.full((t.shape[0], ld), fill, dtype=t.dtype, device=t.device)
    buf[:, :t.shape[1]] = t
    return buf[:, :t.shape[1]]


# ------------------------------------------------------------------------------------------------
# pitched rows: column slices of wider buffers with NaN padding, inputs and outputs
# ------------------------------------------------------------------------------------------------
PITCH_SHAPES = [(F32, 300), (B16, 200)]          # partially live chunks at 3 chunks per lane; dead lanes in the ring geometry


class Canaries:
    """Pitched NaN-padded buffers: makes the inputs, stands in for kernels.new_like (every activation a kernel wrapper
    allocates), and checks afterwards that no padding was written."""

    def __init__(self, pad):
        self.pad, self.bufs = pad, []

    def copy(self, t):
        v = _pitched_copy(t, t.shape[1] + self.pad)
        self.bufs.append(v)
        return v

    def new_like(self, x):
        rows, h = x.shape
        buf = torch.full((rows, x.stride(0)), float("nan"), dtype=x.dtype, device=x.device)
        v = buf[:, :h]
        self.bufs.append(v)
        return v

    def check(self, what):
        for v in self.bufs:
            full = torch.as_strided(v, (v.shape[0], v.stride(0)), (v.stride(0), 1))
            assert torch.isnan(full[:, v.shape[1]:]).all(), f"{what}: padding of a pitched buffer was written"


def _pitch_inputs(C, I):
    return {k: (C.copy(v) if isinstance(v, torch.Tensor) and v.dim() == 2 and v.is_floating_point() else v) for k, v in I.items()}


@gpu
@pytest.mark.parametrize("kernel", ["ln", "ln_attn", "ln_attn_relu", "graph", "colstats", "bn", "bn_eval", "small"])
@pytest.mark.parametrize("dtype,h", PITCH_SHAPES, ids=[f"{'fp32' if d == F32 else 'bf16'}-h{h}" for d, h in PITCH_SHAPES])
def test_pitched_rows(K, monkeypatch, dtype, h, kernel):
    """Every kernel on column slices of wider buffers (NaN in the padding) computes exactly what it computes on contiguous rows,
    at the ragged plan, and writes nothing into the padding."""
    rows = plan_rows(dtype, h, "ragged", _sms())
    vn = 8 if dtype == B16 else 4
    seed = 8000 + h
    if kernel.startswith("bn"):
        case = BN_CASES[0] if kernel == "bn" else BN_CASES[2]
        I = bn_inputs(dtype, rows, h, case, seed)
        run = lambda J: run_bn(K, J, case, 0.5, seed)
    elif kernel == "colstats":
        g = _gen(seed)
        I = dict(x=_rand(rows, h, dtype, g), w=torch.rand(rows, generator=g, device=DEV))
        run = lambda J: run_colstats(K, J)
    elif kernel == "small":
        I = small_inputs(dtype, rows, h, seed)
        run = lambda J: run_small(K, J)
    else:
        I = ln_inputs(dtype, rows, h, seed)
        run = {"ln": lambda J: run_ln(K, J, True, True, 0.5, seed),
               "ln_attn": lambda J: run_ln_attn(K, J, False, False, 0.5, seed),
               "ln_attn_relu": lambda J: run_ln_attn(K, J, True, True, 0.5, seed),
               "graph": lambda J: run_graph(K, J, False, 0.5, seed)}[kernel]
    want = run(I)
    C = Canaries(3 * vn)
    J = _pitch_inputs(C, I)
    assert all(J[k].stride(0) == v.shape[1] + 3 * vn for k, v in I.items() if isinstance(v, torch.Tensor) and v.dim() == 2
               and v.is_floating_point())
    monkeypatch.setattr(K, "new_like", C.new_like)
    got = run(J)
    torch.cuda.synchronize()
    for k, v in want.items():
        if isinstance(v, torch.Tensor):
            assert torch.equal(got[k], v), f"{kernel}: {k} on pitched rows differs from contiguous rows"
    C.check(kernel)


# ------------------------------------------------------------------------------------------------
# launch switches: the non-default side in a child process, bit for bit against the default path
# ------------------------------------------------------------------------------------------------
RING_CASES = (BN_CASES[0], BN_CASES[2])          # training with residual, dy2 and dres accumulation; eval with out_row_scale
RING_SHAPES = [s for s in SHAPE_LIST if SHAPES[s][1] == 1]


def switch_outputs(K, name):
    """The outputs each launch switch changes the code path of, at the sweep plans (run in both processes)."""
    out = {}
    if name == "SGF_BN_BWD_RING":
        for (dtype, h) in RING_SHAPES:
            rows = plan_rows(dtype, h, "ring", _sms())
            for c, case in enumerate(RING_CASES):
                I = bn_inputs(dtype, rows, h, case, 9000 + h + c)
                o = run_bn(K, I, case, _p_for(c), 9000 + h + c)
                out[(dtype, h, c)] = {k: o[k] for k in ("dz", "dres", "colsum", "sums")}
    elif name == "SGF_LNATTN_BLOCKS":
        for (dtype, h) in SHAPE_LIST:
            rows = plan_rows(dtype, h, "ragged", _sms())
            I = ln_inputs(dtype, rows, h, 9100 + h)
            o = run_ln_attn(K, I, False, h % 3 == 0, _p_for(h // 4), 9100 + h)
            out[(dtype, h)] = {k: v for k, v in o.items() if k != "y"}
    elif name == "SGF_PACK_VEC":
        for (dtype, h) in SHAPE_LIST:
            if dtype != F32 or h % 8:
                continue
            rows = plan_rows(dtype, h, "ragged", _sms())
            src = _rand(rows, h, F32, _gen(9200 + h))
            idx = torch.randint(0, rows, (rows // 3,), generator=_gen(9300 + h), device=DEV)
            for planes in (1, 3):
                out[(h, planes)] = K.pack_operand(src, False, planes).data
                out[(h, planes, "gather")] = K.pack_operand(src, False, planes, row_index=idx).data
    else:
        raise KeyError(name)
    return out


def _switch_child(name, path):
    """Entry point of the child process (the switch's environment variable is set there)."""
    from sgformer_b200 import kernels
    torch.save(switch_outputs(kernels, name), path)


def _ulp(x, dtype):
    """The spacing of `dtype` at |x| (fp32 tensor)."""
    return torch.ldexp(torch.ones_like(x), torch.frexp(x.abs())[1] - (24 if dtype == F32 else 8))


def _one_product_rounding_apart(a, b, key):
    """The accumulated dres = dres + gscale * g of the two BatchNorm backward pipelines.  The register pipeline's instantiation
    contracts it into one FFMA; the ring's rounds the product first (FMUL + FADD; cuobjdump -sass of the two bn_bwd_kernel
    instances), so the two may differ by one fp32 rounding of the product and one rounding of the result, and by nothing more.
    dz, its column sums and the BatchNorm sums are compared bit for bit."""
    dtype, h, c = key
    I = bn_inputs(dtype, plan_rows(dtype, h, "ring", _sms()), h, RING_CASES[c], 9000 + h + c)
    prod = (BN_GSCALE * (I["dy"].double() + I["rs2"].double()[:, None] * I["dy2"].double())).float()
    m = torch.maximum(a.float().abs(), b.float().abs())
    return bool(((a.float() - b.float()).abs() <= _ulp(m, dtype) + _ulp(prod, F32)).all())


SWITCHES = {"SGF_BN_BWD_RING": "0", "SGF_LNATTN_BLOCKS": "3", "SGF_PACK_VEC": "0"}


def _check_pack(K, name_out, h, planes, gather):
    """The packed bf16 planes against the CPU emulation's rounding, exactly: plane 0 = bf16(v), plane 1 = bf16(v - plane 0),
    plane 2 = bf16(v - plane 0 - plane 1) in fp32; the K padding is zero."""
    import kernel_emu as emu
    rows = plan_rows(F32, h, "ragged", _sms())
    src = _rand(rows, h, F32, _gen(9200 + h))
    if gather:
        idx = torch.randint(0, rows, (rows // 3,), generator=_gen(9300 + h), device=DEV)
        src = src[idx]
    data = name_out.float().cpu()
    v = src.cpu()
    kp = data.shape[1] // planes
    p0 = emu.pack_operand(v, False, 1).data
    r1 = v - p0
    p1 = r1.bfloat16().float()
    p2 = (r1 - p1).bfloat16().float()
    for i, want in enumerate((p0, p1, p2)[:planes]):
        assert torch.equal(data[:, i * kp:i * kp + h], want), f"pack h={h} planes={planes} gather={gather}: plane {i}"
        assert torch.count_nonzero(data[:, i * kp + h:(i + 1) * kp]) == 0, "K padding must be zero"


@gpu
@pytest.mark.parametrize("var", list(SWITCHES))
def test_launch_switch_other_side(K, var):
    """The non-default side of a launch switch (read once per process) computes bit for bit what the default path computes, and
    both match fp64 (the pack: the emulation's rounding, exactly)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    tests = os.path.dirname(os.path.abspath(__file__))
    with tempfile.TemporaryDirectory() as tmp, no_epoch_word(K):
        path = os.path.join(tmp, "out.pt")
        code = (f"import sys; sys.path[:0] = [{tests!r}, {root!r}]; import test_gpu_row_sweep as T; "
                f"T._switch_child({var!r}, {path!r})")
        env = dict(os.environ, **{var: SWITCHES[var]})
        r = subprocess.run([sys.executable, "-c", code], env=env, cwd=root, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, f"child with {var}={SWITCHES[var]} failed:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
        other = torch.load(path, map_location=DEV)
        default = switch_outputs(K, var)
        assert other.keys() == default.keys()
        bad = []
        for key, o in other.items():
            d = default[key]
            pairs = o.items() if isinstance(o, dict) else [("data", o)]
            d = d if isinstance(d, dict) else {"data": d}
            for k, v in pairs:
                if v is None or d[k] is None:
                    same = v is None and d[k] is None
                elif var == "SGF_BN_BWD_RING" and k == "dres" and RING_CASES[key[2]][6]:
                    same = _one_product_rounding_apart(v, d[k], key)
                else:
                    same = torch.equal(v, d[k])
                if not same:
                    bad.append(f"{key} {k}: max |diff| {(v.double() - d[k].double()).abs().max().item():.3e}")
        assert not bad, f"{var}={SWITCHES[var]} differs from the default path:\n" + "\n".join(bad)
        # the outputs are equal: one check against fp64 covers both sides
        for key, o in other.items():
            if var == "SGF_BN_BWD_RING":
                dtype, h, c = key
                case = RING_CASES[c]
                I = bn_inputs(dtype, plan_rows(dtype, h, "ring", _sms()), h, case, 9000 + h + c)
                full = run_bn(K, I, case, _p_for(c), 9000 + h + c)       # y and ys of the same inputs (not switch-dependent)
                full.update(o)
                check_bn(I, full, case, _p_for(c), 9000 + h + c, _tol(dtype), f"ring plan {key}")
            elif var == "SGF_LNATTN_BLOCKS":
                dtype, h = key
                I = ln_inputs(dtype, plan_rows(dtype, h, "ragged", _sms()), h, 9100 + h)
                full = dict(o, y=run_ln_attn(K, I, False, h % 3 == 0, _p_for(h // 4), 9100 + h)["y"])
                check_ln_attn(I, full, False, h % 3 == 0, _p_for(h // 4), 9100 + h, _tol(dtype), f"ragged plan {key}")
            else:
                _check_pack(K, o, key[0], key[1], len(key) == 3)


# ------------------------------------------------------------------------------------------------
# BatchNorm sharded by rows on one device: statistics and backward sums reduced over the shards
# ------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype,h", [(F32, 100), (F32, 300), (B16, 256), (B16, 1024)],
                         ids=["fp32-h100", "fp32-h300", "bf16-h256", "bf16-h1024"])
def test_row_sharded_batchnorm(K, dtype, h):
    """Three unequal row shards: column statistics summed over the shards and finalised with the global row count; the backward
    sums replaced by their sum over the shards (reduce_fn) and applied with stat_rows = the global row count.  The concatenated
    y and dz and the summed dgamma / dbeta match fp64 of the unsharded BatchNorm."""
    case = BN_CASES[0]
    plan = "ring" if SHAPES[(dtype, h)][1] == 1 else "ragged"
    rows = plan_rows(dtype, h, plan, _sms())
    step = full_step(dtype, h, _sms())
    cuts = [0, 2 * step + 5, 2 * step + 5 + step // 3 + 2, rows]          # a shard over 2 sweeps, one under 1, the rest
    p, seed = 0.5, 9400 + h
    I = bn_inputs(dtype, rows, h, case, seed)
    sh = [slice(cuts[i], cuts[i + 1]) for i in range(3)]
    S = torch.zeros(h, device=DEV)
    Q = torch.zeros(h, device=DEV)
    for s in sh:
        a, b = K.colstats(I["z"][s])
        S += a
        Q += b
    mean, rstd = K.bn_finalize(S, Q, rows, h, None, I["rm"].clone(), I["rv"].clone(), DEV)
    args = lambda s: (I["dy"][s], I["dy2"][s], I["rs2"][s], I["z"][s], mean, rstd, I["gamma"], I["beta"], None, True, True)
    total = sum(K.bn_bwd_sums(*args(s), p, seed + i, BN_GSCALE) for i, s in enumerate(sh))
    ys, yss, dzs, dress, colsums = [], [], [], [], []
    for i, s in enumerate(sh):
        y, yscaled = K.bn_fwd(I["z"][s], I["res"][s], None, mean, rstd, I["gamma"], I["beta"], None, True, True, p, seed + i, BN_GW,
                              I["rs"][s].contiguous(), True, True)
        dres = I["dres0"][s].clone()
        dz, sums, colsum = K.bn_bwd(*args(s), True, p, seed + i, BN_GSCALE, dres=dres, dres_accumulate=True, want_dz_colsum=True,
                                    reduce_fn=lambda t: t.copy_(total), stat_rows=rows)
        assert torch.equal(sums, total)
        ys.append(y), yss.append(yscaled), dzs.append(dz), dress.append(dres), colsums.append(colsum)
    M = torch.cat([dmask(seed + i, s.stop - s.start, h, p).expand(s.stop - s.start, h) for i, s in enumerate(sh)])
    ref = bn_reference(case, I["z"], I["res"], I["mix"], I["dy"], I["dy2"], I["dres0"], I["gamma"], I["beta"], I["rm"], I["rv"],
                       I["rs"], I["rs2"], I["ors"], BN_GW, BN_GSCALE, M)
    got = dict(y=torch.cat(ys), ys=torch.cat(yss), dres=torch.cat(dress), dz=torch.cat(dzs), colsum=sum(colsums), sums=total)
    check_bn_chain(got, ref, case, _tol(dtype), f"3 shards {cuts}", rows, h)


# ------------------------------------------------------------------------------------------------
# the comparison sees the defect class this file is for
# ------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype,h", [(F32, 64), (B16, 256)], ids=["fp32-h64", "bf16-h256"])
def test_swapped_rows_are_reported(K, dtype, h):
    """Rows r and r + row_step of one lane group swapped in a real kernel output: the check that passes on the output as the
    kernel wrote it must fail on the swapped one."""
    rows = plan_rows(dtype, h, "ragged", _sms())
    step = full_step(dtype, h, _sms())
    I = ln_inputs(dtype, rows, h, 9500 + h)
    out = run_ln(K, I, False, True, 0.5, 9500 + h)
    check_ln(I, out, False, True, 0.5, 9500 + h, _tol(dtype), "as written")
    r = step // 3 + 1
    for k in ("y", "dx"):
        bad = dict(out)
        bad[k] = out[k].clone()
        bad[k][[r, r + step]] = out[k][[r + step, r]]
        with pytest.raises(AssertionError, match=k):
            check_ln(I, bad, False, True, 0.5, 9500 + h, _tol(dtype), "swapped")
