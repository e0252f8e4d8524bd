"""Dropout on the H100, value for value.  The kernels' mask is a pure function of (seed, epoch, row, column, h, p), restated on
the host by tests/dropout_mask.py, so every dropout kernel and every training step is compared with an fp64 reference that
applies the same mask:

  (a) the mask each kernel applies, extracted with all-ones inputs, bit-exact against `keep_mask` (fp32 and bf16, every row
      geometry, with and without the device epoch word);
  (b) the fused forward / backward pairs against fp64 autograd of the kernel's formula with the restated mask;
  (c) the same under CUDA-graph replay, where the epoch word advances inside the graph;
  (d) whole models in training mode against the fp64 oracle with the masks replayed from the seeds the forward passed;
  (e) guards against a vacuous pass (call counts, the masks' effect, eval mode)."""
import contextlib
import functools

import pytest
import torch

from dropout_mask import DropoutRecorder, MaskReplayer, current_epoch, keep_mask, keep_scale
from row_ref import BN_CASES, bn_reference, bn_untie, check_bn_chain, ln_reference
from row_ref import attn_reference as _attn_reference, close as _close, untie as _untie

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32, B16 = torch.float32, torch.bfloat16
WIDTHS = {F32: [4, 12, 64, 96, 100, 200, 256, 300, 384, 512], B16: [8, 24, 64, 96, 200, 256, 768, 1024]}   # cpl 1-4
TINY_P = 2.0 ** -18          # thr16 = 0: nothing is dropped, but the DROP instantiation runs
BIG_SEED = (1 << 62) + 0x5EED


@pytest.fixture(scope="module")
def K():
    from sgformer_b200 import kernels
    return kernels


@contextlib.contextmanager
def epoch_word(K, advances):
    """advances=None: no epoch word registered for the duration (restored afterwards); else the word is registered and advanced
    `advances` times before the body runs."""
    if advances is None:
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
    else:
        K.dropout_epoch()
        for _ in range(advances):
            K.advance_dropout_epoch()
        torch.cuda.synchronize()
        yield


@functools.lru_cache(maxsize=160)
def _device_mask(seed, rows, h, p, epoch):
    return torch.from_numpy(keep_mask(seed, rows, h, p, epoch)).to(DEV)


def dmask(seed, rows, h, p):
    """fp64 mask * kernel scale on the device, for the epoch word as it stands."""
    return torch.from_numpy(keep_mask(seed, rows, h, p, current_epoch())).to(DEV).double() * keep_scale(p)


def _sweep_rows(h, dtype):
    """Rows for which the capped grid (num_sms * 8 blocks of 8 warps) sweeps the rows at least twice at width h."""
    vn = 8 if dtype == B16 else 4
    lpr = 1
    while lpr < h // vn and lpr < 32:
        lpr *= 2
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return 2 * sms * 8 * 8 * (32 // lpr) + 7


# ------------------------------------------------------------------------------------------------
# (a) the mask of every dropout kernel, bit-exact
# ------------------------------------------------------------------------------------------------
def _extract(K, name, rows, h, dtype, p, seed):
    """-> list of (what, tensor that equals mask * scale)."""
    ones = torch.ones(rows, h, device=DEV, dtype=dtype)
    zeros = torch.zeros(rows, h, device=DEV, dtype=dtype)
    one_r = torch.ones(rows, device=DEV)
    if name == "ln_fwd":
        return [("y", K.ln_fwd(ones, None, 1.0, 0.0, None, None, False, False, p, seed)[0])]
    if name == "ln_fwd_graph":
        return [("y", K.ln_fwd_graph(ones, None, zeros, 1.0, 0.0, 1.0, None, None, False, False, p, seed)[0])]
    if name == "bn_fwd":
        y, ys = K.bn_fwd(ones, None, None, None, None, None, None, None, False, False, p, seed, 1.0, one_r, True, True)
        return [("y", y), ("y_scaled", ys)]
    if name == "ln_bwd":
        return [("dx", K.ln_bwd(ones, ones, None, 1.0, 0.0, None, None, None, False, False, p, seed, 1.0, False, None, None)[0])]
    if name == "ln_bwd_attn":
        gnum = K.ln_bwd_attn(ones, zeros, None, zeros, 1.0, 0.0, None, None, None, False, False, p, seed, 1.0, False, None, None,
                             one_r)[0]
        return [("gnum*den", gnum)]
    if name == "ln_bwd_attn_graph":
        ys = K.ln_bwd_attn_graph(ones, zeros, None, zeros, zeros, 1.0, 0.0, 1.0, None, None, None, False, p, seed, 1.0, False,
                                 None, None, one_r, one_r)[3]
        return [("ys", ys)]
    hz = torch.zeros(h, device=DEV)
    h1 = torch.ones(h, device=DEV)
    if name == "bn_bwd_apply":          # BatchNorm in eval mode with mean 0, rstd 1, gamma 1: dz = the masked gradient
        return [("dz", K.bn_bwd(ones, None, None, ones, hz, h1, h1, hz, None, True, False, False, p, seed, 1.0)[0])]
    if name == "bn_bwd_reduce":         # training BatchNorm: sums[:h] = column sums of the masked gradient
        sums = K.bn_bwd_sums(ones, None, None, ones, hz, h1, h1, hz, None, True, False, p, seed, 1.0)
        return [("colsum", sums[:h])]
    raise KeyError(name)


MASK_KERNELS = ["ln_fwd", "ln_fwd_graph", "bn_fwd", "ln_bwd", "ln_bwd_attn", "ln_bwd_attn_graph", "bn_bwd_apply", "bn_bwd_reduce"]


@pytest.mark.parametrize("epoch", [None, 3], ids=["no_epoch", "epoch"])
@pytest.mark.parametrize("dtype", [F32, B16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("name", MASK_KERNELS)
def test_kernel_mask_is_bit_exact(K, name, dtype, epoch):
    bad = []
    with epoch_word(K, epoch):
        for hi, h in enumerate(WIDTHS[dtype]):
            # the sweep plan uses p with an exact fp32 scale (2, 2.5): its column sums are exact and a single flip shows
            plan = [(1, 0.2), (5, 0.9), (777, TINY_P), (777, 0.6), (_sweep_rows(h, dtype), (0.5, 0.6)[hi % 2])]
            for j, (rows, p) in enumerate(plan):
                seed = BIG_SEED + 977 * hi if j % 2 else 1000 + 31 * hi + j
                m = _device_mask(seed, rows, h, p, current_epoch())
                sc = torch.tensor(keep_scale(p), dtype=dtype).float()        # bf16(scale) in bf16
                for what, got in _extract(K, name, rows, h, dtype, p, seed):
                    if what == "colsum":      # kept elements per column, as an integer count
                        count = m.double().sum(0)
                        ok = torch.equal(torch.round(got.double() / keep_scale(p)), count) and \
                            (got.double() - count * keep_scale(p)).abs().max().item() <= 1e-6 * count.max().item() * keep_scale(p)
                    else:
                        ok = torch.equal(got.float(), m.float() * sc)
                    if not ok:
                        bad.append(f"{what} h={h} rows={rows} p={p} seed={seed}")
    assert not bad, "\n".join(bad[:20])


@pytest.mark.parametrize("name", ["ln_fwd", "bn_fwd", "ln_bwd", "bn_bwd_apply"])
def test_same_seed_same_mask_in_both_dtypes(K, name):
    rows, h, p, seed = 777, 64, 0.5, BIG_SEED
    a = _extract(K, name, rows, h, F32, p, seed)[0][1] != 0
    b = _extract(K, name, rows, h, B16, p, seed)[0][1] != 0
    assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------
# (b) fused pairs against fp64 autograd with the restated mask
# ------------------------------------------------------------------------------------------------
def _tol(dtype):
    return 2e-5 if dtype == F32 else 5e-3


def _rand(rows, h, dtype, gen, scale=1.0):
    return (scale * torch.randn(rows, h, generator=gen)).to(DEV).to(dtype)


def _ln_inputs(rows, h, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x, r, gy, dy, xa = (_rand(rows, h, dtype, g) for _ in range(5))
    gamma = (1 + 0.2 * torch.randn(h, generator=g)).to(DEV)
    beta = (0.2 * torch.randn(h, generator=g)).to(DEV)
    den = (1 + torch.rand(rows, generator=g)).to(DEV)
    dinv = torch.rand(rows, generator=g).to(DEV)
    return x, r, gy, dy, xa, gamma, beta, den, dinv


PAIR_SHAPES = [(F32, h) for h in (4, 12, 96, 100, 256, 300, 384, 512)] + [(B16, h) for h in (8, 24, 96, 200, 768, 1024)]


@pytest.mark.parametrize("dtype,h", PAIR_SHAPES, ids=[f"{'fp32' if d == F32 else 'bf16'}-h{h}" for d, h in PAIR_SHAPES])
def test_ln_fwd_ln_bwd_pair(K, dtype, h):
    tol = _tol(dtype)
    for k, (use_ln, use_relu, with_r) in enumerate([(u, v, w) for u in (False, True) for v in (False, True) for w in (False, True)]):
        rows, p = (777, 5)[k % 2], (0.2, 0.5, 0.6)[k % 3]
        seed = 40 + k + h
        x, r, _, dy, _, gamma, beta, _, _ = _ln_inputs(rows, h, dtype, seed)
        r = r if with_r else None
        a, b = (0.7, 0.3) if with_r else (1.3, 0.0)
        if use_relu:
            dy = _untie(dy, x, r, a, b, gamma, beta, use_ln)
        y, st = K.ln_fwd(x, r, a, b, gamma, beta, use_ln, use_relu, p, seed)
        dg, db = torch.zeros(h, device=DEV), torch.zeros(h, device=DEV)
        dx, dr = K.ln_bwd(dy, x, r, a, b, gamma, beta, st, use_ln, use_relu, p, seed, 0.75, with_r, dg, db)
        R = ln_reference(x, r, None, a, b, 0.0, gamma, beta, use_ln, use_relu, dmask(seed, rows, h, p), dy, 0.75)
        tag = f"ln={use_ln} relu={use_relu} r={with_r} rows={rows} p={p}"
        _close(y, R["y"], tol, f"y {tag}")
        _close(dx, R["dx"], tol, f"dx {tag}")
        if with_r:
            _close(dr, R["dr"], tol, f"dr {tag}")
        if use_ln:
            _close(dg, R["dgamma"], 1e-5, f"dgamma {tag}", rows)
            _close(db, R["dbeta"], 1e-5, f"dbeta {tag}", rows)


@pytest.mark.parametrize("dtype,h", PAIR_SHAPES, ids=[f"{'fp32' if d == F32 else 'bf16'}-h{h}" for d, h in PAIR_SHAPES])
def test_ln_fwd_ln_bwd_attn_pair(K, dtype, h):
    tol = _tol(dtype)
    for k, (use_ln, use_relu, alias) in enumerate([(u, v, w) for u in (False, True) for v in (False, True) for w in (False, True)]):
        rows, p = (777, 5)[k % 2], (0.6, 0.2, 0.5)[k % 3]
        seed = 90 + k + h
        o, r, _, dy, xa, gamma, beta, den, _ = _ln_inputs(rows, h, dtype, seed)
        xa = r if alias else xa
        a, b = 0.61, 0.37        # no exact ties a*o + b*r = 0 between bf16 values (0.6 / 0.4 has many)
        if use_relu:
            dy = _untie(dy, o, r, a, b, gamma, beta, use_ln)
        y, st = K.ln_fwd(o, r, a, b, gamma, beta, use_ln, use_relu, p, seed)
        dg, db = torch.zeros(h, device=DEV), torch.zeros(h, device=DEV)
        gnum, gden, dr, cs, pg, sg = K.ln_bwd_attn(dy, o, r, xa, a, b, gamma, beta, st, use_ln, use_relu, p, seed, 1.5, True, dg, db,
                                                   den)
        R = ln_reference(o, r, None, a, b, 0.0, gamma, beta, use_ln, use_relu, dmask(seed, rows, h, p), dy, 1.5)
        A = _attn_reference(R, o, xa, a, den)
        tag = f"ln={use_ln} relu={use_relu} xa_is_r={alias} rows={rows} p={p}"
        _close(y, R["y"], tol, f"y {tag}")
        _close(gnum, A["gnum"], tol, f"gnum {tag}")
        _close(dr, R["dr"], tol, f"dr {tag}")
        _close(gden, A["gden"], 1e-4, f"gden {tag}")
        for what in ("cs", "pg", "sg"):
            _close({"cs": cs, "pg": pg, "sg": sg}[what], A[what], 1e-5, f"{what} {tag}", rows, A["elem"][what])
        if use_ln:
            _close(dg, R["dgamma"], 1e-5, f"dgamma {tag}", rows)
            _close(db, R["dbeta"], 1e-5, f"dbeta {tag}", rows)


def _graph_inputs(dtype, rows, h, with_r, alias, seed):
    o, r, gy, dy, xa, gamma, beta, den, dinv = _ln_inputs(rows, h, dtype, seed)
    r = r if with_r else None
    xa = r if (alias and with_r) else xa
    return o, r, gy, dy, xa, gamma, beta, den, dinv, 0.5, (0.3 if with_r else 0.0), 0.8


def _graph_pair(K, inputs, use_ln, with_r, p, seed):
    o, r, gy, dy, xa, gamma, beta, den, dinv, a, b, c = inputs
    h = o.shape[1]
    y, st = K.ln_fwd_graph(o, r, gy, a, b, c, gamma, beta, use_ln, False, p, seed)
    dg, db = torch.zeros(h, device=DEV), torch.zeros(h, device=DEV)
    got = K.ln_bwd_attn_graph(dy, o, r, xa, gy, a, b, c, gamma, beta, st, use_ln, p, seed, 1.0, with_r, dg, db, den, dinv)
    return y, got, dg, db


def _check_graph_pair(inputs, y, got, dg, db, use_ln, with_r, p, seed, tol, tag):
    o, r, gy, dy, xa, gamma, beta, den, dinv, a, b, c = inputs
    rows, h = o.shape
    gnum, gden, dr, ys, cs, pg, sg = got
    R = ln_reference(o, r, gy, a, b, c, gamma, beta, use_ln, False, dmask(seed, rows, h, p), dy, 1.0)
    A = _attn_reference(R, o, xa, a, den)
    _close(y, R["y"], tol, f"y {tag}")
    _close(gnum, A["gnum"], tol, f"gnum {tag}")
    _close(ys, dinv.double()[:, None] * c * R["du"], tol, f"ys {tag}")
    if with_r:
        _close(dr, b * R["du"], tol, f"dr {tag}")
    _close(gden, A["gden"], 1e-4, f"gden {tag}")
    for what, v in (("cs", cs), ("pg", pg), ("sg", sg)):
        _close(v, A[what], 1e-5, f"{what} {tag}", rows, A["elem"][what])
    if use_ln:
        _close(dg, R["dgamma"], 1e-5, f"dgamma {tag}", rows)
        _close(db, R["dbeta"], 1e-5, f"dbeta {tag}", rows)


@pytest.mark.parametrize("dtype,h", PAIR_SHAPES, ids=[f"{'fp32' if d == F32 else 'bf16'}-h{h}" for d, h in PAIR_SHAPES])
def test_ln_fwd_graph_ln_bwd_attn_graph_pair(K, dtype, h):
    for k, (use_ln, with_r, alias) in enumerate([(True, True, True), (True, True, False), (False, True, False), (True, False, False)]):
        rows, p, seed = (777, 5)[k % 2], (0.5, 0.6, 0.2)[k % 3], 300 + k + h
        inputs = _graph_inputs(dtype, rows, h, with_r, alias, seed)
        y, got, dg, db = _graph_pair(K, inputs, use_ln, with_r, p, seed)
        _check_graph_pair(inputs, y, got, dg, db, use_ln, with_r, p, seed, _tol(dtype),
                          f"ln={use_ln} r={with_r} xa_is_r={alias} rows={rows} p={p}")


def _bn_chain(K, dtype, rows, h, case, p, seed):
    use_bn, training, relu, with_res, with_mix, with_dy2, dres_acc, with_ors = case
    g = torch.Generator().manual_seed(seed)
    z, res, mix, dy, dy2, dres0 = (_rand(rows, h, dtype, g, 1.5) for _ in range(6))
    gamma = (1 + 0.2 * torch.randn(h, generator=g)).to(DEV)
    beta = (0.2 * torch.randn(h, generator=g)).to(DEV)
    rm, rv = (0.1 * torch.randn(h, generator=g)).to(DEV), (1 + 0.3 * torch.rand(h, generator=g)).to(DEV)
    rs, rs2, ors = (0.2 + torch.rand(rows, generator=g)).to(DEV), (0.2 + torch.rand(rows, generator=g)).to(DEV), \
        (0.2 + torch.rand(rows, generator=g)).to(DEV)
    gw, gscale = 0.7, 0.9
    dy, dy2 = bn_untie(case, z, gamma, beta, rm, rv, dy, dy2)
    mean = rstd = None
    if use_bn:
        if training:
            s, q = K.colstats(z)
            mean, rstd = K.bn_finalize(s, q, rows, h, None, rm.clone(), rv.clone(), DEV)
        else:
            mean, rstd = K.bn_finalize(None, None, rows, h, None, rm, rv, DEV)
    res_, mix_ = (res if with_res else None), (mix if with_mix else None)
    y, ys = K.bn_fwd(z, res_, mix_, mean, rstd, gamma if use_bn else None, beta if use_bn else None, None, use_bn, relu, p, seed,
                     gw, rs, True, True)
    dres = dres0.clone()
    dz, sums, colsum = K.bn_bwd(dy, dy2 if with_dy2 else None, rs2 if with_dy2 else None, z, mean, rstd,
                                gamma if use_bn else None, beta if use_bn else None, None, use_bn, relu, training, p, seed, gscale,
                                dres=dres, dres_accumulate=dres_acc, want_dz_colsum=True, out_row_scale=ors if with_ors else None)
    if use_bn and not training:
        sums = K.bn_bwd_sums(dy, dy2 if with_dy2 else None, rs2 if with_dy2 else None, z, mean, rstd, gamma, beta, None, True, relu,
                             p, seed, gscale)
    ref = bn_reference(case, z, res, mix, dy, dy2, dres0, gamma, beta, rm, rv, rs, rs2, ors, gw, gscale, dmask(seed, rows, h, p))
    return dict(y=y, ys=ys, dres=dres, dz=dz, colsum=colsum, sums=sums), ref


@pytest.mark.parametrize("dtype,h", PAIR_SHAPES, ids=[f"{'fp32' if d == F32 else 'bf16'}-h{h}" for d, h in PAIR_SHAPES])
def test_bn_fwd_bn_bwd_chain(K, dtype, h):
    tol = _tol(dtype)
    for k, case in enumerate(BN_CASES):
        for rows in (5, 777):
            p, seed = (0.2, 0.5, 0.6)[(k + rows) % 3], 500 + 7 * k + rows + h
            got, ref = _bn_chain(K, dtype, rows, h, case, p, seed)
            check_bn_chain(got, ref, case, tol, f"case={case} rows={rows} p={p}", rows, h)


# ------------------------------------------------------------------------------------------------
# (c) CUDA-graph replay with the epoch word advanced inside the graph
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [F32, B16], ids=["fp32", "bf16"])
def test_values_under_graph_replay(K, dtype):
    rows, h, p, seed = 777, 96, 0.5, BIG_SEED
    K.dropout_epoch()
    g = torch.Generator().manual_seed(11)
    z, res, dy = (_rand(rows, h, dtype, g) for _ in range(3))
    gamma, beta = (1 + 0.2 * torch.randn(h, generator=g)).to(DEV), (0.2 * torch.randn(h, generator=g)).to(DEV)
    rm, rv = (0.1 * torch.randn(h, generator=g)).to(DEV), (1 + 0.3 * torch.rand(h, generator=g)).to(DEV)
    rs = (0.2 + torch.rand(rows, generator=g)).to(DEV)
    mean, rstd = K.bn_finalize(None, None, rows, h, None, rm, rv, DEV)     # eval BatchNorm: no batch statistics in the graph
    pre = (z.double() - rm.double()) / torch.sqrt(rv.double() + 1e-5) * gamma.double() + beta.double()
    dy = dy.masked_fill(pre.abs() <= 1e-3 * pre.abs().max(), 0)           # as _untie
    inputs = _graph_inputs(dtype, rows, h, True, False, seed + 1)

    def step():
        K.advance_dropout_epoch()
        y, _ = K.bn_fwd(z, res, None, mean, rstd, gamma, beta, None, True, True, p, seed, 1.0, rs, True, False)
        dz = K.bn_bwd(dy, None, None, z, mean, rstd, gamma, beta, None, True, True, False, p, seed, 1.0)[0]
        y2, got, dg, db = _graph_pair(K, inputs, True, True, p, seed + 1)
        return y, dz, y2, got, dg, db

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()                                 # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step()
    tol = _tol(dtype)
    masks = []
    for rep in range(3):
        graph.replay()
        torch.cuda.synchronize()
        y, dz, y2, got, dg, db = outs
        M = dmask(seed, rows, h, p)
        masks.append(M != 0)
        _close(y, pre.clamp_min(0) * M + res.double(), tol, f"replay {rep}: bn_fwd y")
        _close(dz, dy.double() * M * (pre > 0) * gamma.double() / torch.sqrt(rv.double() + 1e-5), tol, f"replay {rep}: bn_bwd dz")
        _check_graph_pair(inputs, y2, got, dg, db, True, True, p, seed + 1, tol, f"replay {rep}: ln graph pair")
    assert not torch.equal(masks[0], masks[1]) and not torch.equal(masks[1], masks[2]), "the epoch did not advance"


# ------------------------------------------------------------------------------------------------
# (d) + (e) models on the kernels against the fp64 oracle with the kernels' masks replayed
# ------------------------------------------------------------------------------------------------
SEED = 0x0DD_5EED_1234


def _fixture_case(name, rates):
    import os
    fx = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"model_{name}.pt"), weights_only=False)
    return dict(fx["cfg"], **rates), fx["state_dict"], fx["x"], fx["edge_index"], fx["loss_weight"]


def _arxiv_case():
    from oracle import sgformer_oracle as O
    n, e, d, h, c = 12000, 90000, 128, 256, 40
    cfg = O.make_config("large", d, h, c, gnn_num_layers=3, graph_weight=0.5, trans_dropout=0.5, gnn_dropout=0.2,
                        trans_use_act=False)
    sd = O.init_state_dict(cfg, seed=5)
    g = torch.Generator().manual_seed(6)
    ei = torch.stack([torch.randint(0, n, (e,), generator=g), torch.randint(0, n, (e,), generator=g)])
    ei = torch.cat([ei, ei.flip(0)], 1)
    return cfg, sd, torch.randn(n, d, generator=g), ei, torch.randn(n, c, generator=g) / n ** 0.5


MODEL_CASES = {
    "large_add_init": lambda: _fixture_case("large_add_init", dict(trans_dropout=0.2, gnn_dropout=0.5)),
    "large_cat_heads2": lambda: _fixture_case("large_cat_heads2", dict(trans_dropout=0.5, gnn_dropout=0.3)),
    "100M_alpha": lambda: _fixture_case("100M_alpha", dict(trans_dropout=0.3, gnn_dropout=0.6)),
    "medium_gcn": lambda: _fixture_case("medium_gcn", dict(trans_dropout=0.2, gcn_dropout=0.6)),
    "medium_res_heads2": lambda: _fixture_case("medium_res_heads2", dict(trans_dropout=0.4, gcn_dropout=0.5)),
}


def _oracle_fp64(O, cfg, sd, x, ei, lw, masks):
    """fp64 oracle training step with `masks` replayed at the kernels' scale (None: no dropout patch)
    -> (out, grads incl. '__x__', stats)."""
    sdd = {k: (v.double().requires_grad_(True) if v.is_floating_point() and "running" not in k else
               (v.double() if v.is_floating_point() else v)) for k, v in sd.items()}
    xd = x.double().requires_grad_(True)
    stats = {}
    with pytest.MonkeyPatch.context() as mp:
        if masks is not None:
            replay = MaskReplayer(masks, scale="kernel")
            mp.setattr(O, "_dropout", replay)
        if hasattr(O, "sgformer_forward"):
            orig = O.pyg_gcn_adjacency
            mp.setattr(O, "pyg_gcn_adjacency", lambda *a, **k: orig(*a, **k).to(torch.float64))
            out = O.sgformer_forward(cfg, sdd, xd, ei, training=True, stats_out=stats)
        else:
            out = O.difformer_forward(cfg, sdd, xd, ei, training=True)
        if masks is not None:
            replay.finish()
    (out * lw.double()).sum().backward()
    grads = {k: v.grad for k, v in sdd.items() if getattr(v, "grad", None) is not None}
    grads["__x__"] = xd.grad
    return out.detach(), grads, stats


def _model_step(run, lw):
    """One training step on the kernels with the dropout seed fixed and the forward's dropout calls recorded -> (out, recorder)."""
    from sgformer_b200 import engine as E
    from sgformer_b200 import kernels as Kmod
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(E, "next_seed", lambda: SEED)
        rec = DropoutRecorder(mp, Kmod)
        out = run()
        (out * lw.to(DEV)).sum().backward()
    return out.detach(), rec


def _compare_model(model, out, ref, ref_grads, xg, precision, what, out_tol=None):
    from test_gpu_model import _check_grads, _close as _mclose
    tol = out_tol or (1e-4 if precision == "fp32" else 1e-2)
    _mclose(out, ref, tol, tol, f"{what} logits")
    named = {k: p.grad for k, p in model.named_parameters()}
    named["__x__"] = xg.grad
    problems = []
    _check_grads(named, {k: v.float() for k, v in ref_grads.items() if k in named}, precision, problems)
    assert not problems, "\n".join(problems)


# the arxiv-shaped case (h = 256, 12 k nodes) runs in fp32, where h = 256 takes the cpl = 2 kernel paths
SGF_MODEL_PARAMS = [(n, pr) for n in MODEL_CASES for pr in ("fp32", "bf16")] + [("arxiv_h256", "fp32")]


@pytest.mark.parametrize("name,precision", SGF_MODEL_PARAMS, ids=[f"{n}-{pr}" for n, pr in SGF_MODEL_PARAMS])
def test_sgformer_training_step_matches_oracle_with_masks(name, precision):
    from oracle import sgformer_oracle as O
    from test_dropout_replay import expected_calls
    from test_gpu_model import build_model, run
    cfg, sd, x, ei, lw = _arxiv_case() if name == "arxiv_h256" else MODEL_CASES[name]()
    model = build_model(cfg).to(DEV).set_precision(precision)
    model.load_state_dict(sd)
    model.train()
    xg = x.to(DEV).clone().requires_grad_(True)
    out, rec = _model_step(lambda: run(model, cfg, xg, ei.to(DEV)), lw)
    assert len(rec.calls) == expected_calls(cfg), [(c.fn, c.rows, c.h, c.p) for c in rec.calls]
    ref, ref_grads, stats = _oracle_fp64(O, cfg, sd, x, ei, lw, rec.masks())
    _compare_model(model, out, ref, ref_grads, xg, precision, name)
    if precision == "fp32":
        sdm = model.state_dict()
        for k, v in stats.items():
            if "running" in k:
                torch.testing.assert_close(sdm[k].cpu().double(), v.double(), rtol=1e-4, atol=1e-5, msg=f"buffer {k}")
    # (e) the masks matter: the p = 0 oracle is far away
    ref0, _, _ = _oracle_fp64(O, dict(cfg, trans_dropout=0.0, gnn_dropout=0.0, gcn_dropout=0.0), sd, x, ei, lw, None)
    assert (ref - ref0).abs().max() > 100 * 1e-4 * ref.abs().max(), "dropout changed nothing"


DIFF_CASES = {"default": 0.6, "no_graph": 0.5, "source": 0.4, "no_res_no_bn": 0.2, "actor_recipe": 0.6}


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", list(DIFF_CASES))
def test_difformer_training_step_matches_oracle_with_masks(name, precision):
    """bf16 logits: 1e-2 at h >= 16, 2e-2 on the h = 8 fixture cases, where bf16 activations alone reach 1.7 %
    (the tolerances of test_gpu_difformer.py)."""
    from oracle import difformer_oracle as D
    from test_difformer import FIXTURE
    from test_gpu_difformer import Data, _model
    cfg, sd, x, ei, lw, _ = FIXTURE[name]
    cfg = dict(cfg, dropout=DIFF_CASES[name])
    model = _model(cfg, sd, precision)
    model.train()
    xg = x.to(DEV).clone().requires_grad_(True)
    out, rec = _model_step(lambda: model(Data(xg, ei.to(DEV))), lw)
    assert len(rec.calls) == 1 + cfg["num_layers"]
    ref, ref_grads, _ = _oracle_fp64(D, cfg, sd, x, ei, lw, rec.masks())
    out_tol = 2e-2 if (precision == "bf16" and cfg["hidden"] < 16) else None
    _compare_model(model, out, ref, ref_grads, xg, precision, name, out_tol)
    ref0, _, _ = _oracle_fp64(D, dict(cfg, dropout=0.0), sd, x, ei, lw, None)
    assert (ref - ref0).abs().max() > 100 * 1e-4 * ref.abs().max(), "dropout changed nothing"


@pytest.mark.parametrize("name", ["large_add_init", "medium_gcn"])
def test_eval_ignores_dropout(name):
    """model.eval() with dropout > 0 == the same weights with dropout 0, bit for bit, and no dropout kernel runs with p > 0."""
    from test_gpu_model import build_model, run
    from sgformer_b200 import kernels as Kmod
    cfg, sd, x, ei, _ = MODEL_CASES[name]()
    outs = []
    for c in (cfg, dict(cfg, trans_dropout=0.0, gnn_dropout=0.0, gcn_dropout=0.0)):
        model = build_model(c).to(DEV)
        model.load_state_dict(sd)
        model.eval()
        with pytest.MonkeyPatch.context() as mp, torch.no_grad():
            rec = DropoutRecorder(mp, Kmod)
            outs.append(run(model, c, x.to(DEV), ei.to(DEV)))
        assert not rec.calls
    assert torch.equal(outs[0], outs[1])
