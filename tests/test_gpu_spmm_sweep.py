"""The CSR gather kernels (csrc/spmm.cu, csrc/edge_weight.cu) against exact sums and fp64, at every lane geometry of
tests/spmm_geometry.py and at work counts past every grid cap.

Every SpMM variant -- scaled (`row_scale` None or dinv), unscaled (`spmm_sum`) and weighted (`val=`), each without and with the
hub-row plan, on a CSR and on its transpose -- runs on a directed graph with isolated nodes, duplicate edges, single and repeated
self loops, rows of the lengths where the kernels change behaviour (the 32-id column batches, HEAVY_ROW = 1024 against 1025) and
a node with more than HEAVY_ROW out-edges, so the transpose has a hub row too; the graph has 3 x row_cap (+ tail) rows, so every
warp of the capped grid runs three or four rows.  Features are integers in [-2, 2] and weights dyadic (k / 4, |k| <= 8): every
fp32 sum is then exact in any order, and the output must equal the exact sum bit for bit (bf16: round-to-nearest-even of it; with
dinv: one fp32 rounding of the exact product).  Operands and outputs are column blocks of wider buffers: the operand's other
columns hold NaN (a read of them would show in the output) and the output's a sentinel bit pattern that must survive every call.

The edge-weight gradient (sgf_edge_weight_grad) runs at every width the layers admit, past its own (smaller) grid cap, in its
DIFFormer form and in its GCN form (degree term, duplicated self loops), against fp64 under a per-edge rounding bound."""
import pytest
import torch

import kernel_emu_weighted as KW
import spmm_geometry as G

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32, B16 = G.F32, G.B16
SENTINEL = {F32: 0x7FA5A5A5, B16: 0x7FA5}           # NaN bit patterns no kernel writes
SPECIAL_LENS = (1, 31, 32, 33, 64, 65, 1024, 1025, 2048, 2049, 3001)
HUB_OUT = 1500
ORIENTS = ("csr", "transpose")
PEAK_BUDGET = 8 * 2 ** 30


@pytest.fixture(scope="module")
def mem0():
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    return torch.cuda.memory_allocated()


@pytest.fixture(scope="module")
def sms(mem0):
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


# ------------------------------------------------------------------------------------------------
# graphs, operands, references
# ------------------------------------------------------------------------------------------------
class SweepGraph:
    pass


def _edge_list(n, seed):
    """Directed edge list (int64 [2, E] on the device) and dyadic weights, with: isolated nodes (i % 97 == 5), random rows of
    about 6 entries, 5 % duplicated edges, rows of exactly SPECIAL_LENS entries, a node with HUB_OUT out-edges, one self loop on
    every 13th ordinary node and three on every 26th."""
    g = torch.Generator().manual_seed(seed)
    ar = torch.arange(n)
    iso = ar % 97 == 5
    special = torch.tensor([n // 3 + 211 * k for k in range(6)] + [n - 1 - 389 * k for k in range(5)])
    assert not bool(iso[special].any()) and special.unique().numel() == len(SPECIAL_LENS)
    free = ~iso
    free[special] = False
    ordinary, live = ar[free], ar[~iso]
    e = 6 * n
    src = live[torch.randint(0, live.numel(), (e,), generator=g)]
    dst = ordinary[torch.randint(0, ordinary.numel(), (e,), generator=g)]
    dup = torch.randint(0, e, (e // 20,), generator=g)
    srcs, dsts = [src, src[dup]], [dst, dst[dup]]
    for r, length in zip(special.tolist(), SPECIAL_LENS):
        srcs.append(live[torch.randint(0, live.numel(), (length,), generator=g)])
        dsts.append(torch.full((length,), r))
    hub = int(ordinary[7])
    srcs.append(torch.full((HUB_OUT,), hub))
    dsts.append(ordinary[torch.randint(0, ordinary.numel(), (HUB_OUT,), generator=g)])
    one, three = ordinary[::13], ordinary[::26]
    srcs += [one, three, three]
    dsts += [one, three, three]
    src, dst = torch.cat(srcs), torch.cat(dsts)
    perm = torch.randperm(src.numel(), generator=g)
    ei = torch.stack([src, dst])[:, perm].contiguous()
    w = (torch.randint(-8, 9, (ei.shape[1],), generator=g).float() / 4)
    return ei.to(DEV), w.to(DEV), special.to(DEV), iso.to(DEV), hub


@pytest.fixture(scope="module")
def graphs(sms):
    """plan -> SweepGraph: the unweighted Graph, the weighted one (same edges, dyadic weights), both transposes, and a CSR with
    rotated column ids for the phased SpMM."""
    from sgformer_b200 import kernels as K
    from sgformer_b200.graph import Graph
    cache = {}

    def get(plan):
        if plan not in cache:
            s = SweepGraph()
            s.n = G.plan(G.row_cap(sms), plan)
            s.ei, s.w, s.special, s.iso, s.hub = _edge_list(s.n, 1 + G.PLANS.index(plan))
            s.g = Graph(s.ei, s.n)
            s.gw = Graph(s.ei, s.n, 0, edge_weight=s.w)
            s.g.transpose()
            s.gw.transpose()
            s.rot = s.n // 3
            s.rot_rowptr, s.rot_col, _ = K.csr_build(s.ei, s.n, col_rot=(s.rot, s.n))
            cache[plan] = s
        return cache[plan]
    return get


def _bits(t):
    return t.view(torch.int16 if t.dtype == B16 else torch.int32)


def _mismatch(got, want) -> int:
    """Elements whose bit patterns differ."""
    assert got.shape == want.shape and got.dtype == want.dtype
    return int((_bits(got) != _bits(want)).sum())


def _block(rows, h, dtype, pad=None):
    """(buffer [rows, h + 2 VN], its column block [:, VN:VN + h]): 16-byte aligned, pitch h + 2 VN.  The buffer holds NaN
    (operands) or the sentinel pattern (outputs)."""
    v = G.vn(dtype)
    buf = torch.empty((rows, h + 2 * v), dtype=dtype, device=DEV)
    if pad is None:
        buf.fill_(float("nan"))
    else:
        _bits(buf).fill_(pad)
    return buf, buf[:, v:v + h]


def _check_block(buf, h, want, what):
    v = G.vn(buf.dtype)
    bad = _mismatch(buf[:, v:v + h], want)
    assert bad == 0, f"{what}: {bad} elements differ"
    pads = torch.cat([_bits(buf[:, :v]), _bits(buf[:, v + h:])], 1)
    assert bool((pads == SENTINEL[buf.dtype]).all()), f"{what}: the columns beside the output block were written"


def _coo(rowptr, col):
    n = rowptr.numel() - 1
    return torch.repeat_interleave(torch.arange(n, device=DEV), rowptr[1:] - rowptr[:-1]), col.long()


def _coo_sum(rows, cols, x, n, w=None, acc=None, absolute=False):
    """out[rows[j]] += w[j] * x[cols[j]] (|w| |x| when `absolute`) in x's dtype or `acc` (int32: exact; fp64), in edge chunks."""
    acc = acc or x.dtype
    out = torch.zeros((n, x.shape[1]), dtype=acc, device=DEV)
    step = max(1, (1 << 24) // x.shape[1])
    for i in range(0, rows.numel(), step):
        v = x.index_select(0, cols[i:i + step]).to(acc)
        if w is not None:
            v = v * w[i:i + step, None].to(acc)
        out.index_add_(0, rows[i:i + step], v.abs() if absolute else v)
    return out


def _quarters(val):
    """Dyadic weights k / 4 as the integers k."""
    q = torch.round(val * 4).to(torch.int32)
    assert torch.equal(q.float() / 4, val)
    return q


def _want(ref, scale, dtype):
    """The kernel's output for the exact fp32 sum `ref`: unscaled, or one fp32 rounding of ref * scale (exact in fp64);
    then round-to-nearest-even to bf16."""
    if scale is not None:
        ref = (ref.double() * scale.double()[:, None]).float()
    return ref.to(dtype)


def _variants(s, orient):
    """[(label, run(x, out, with_hub_plan), weighted, row scale)] of one orientation."""
    from sgformer_b200 import kernels as K
    g, gw, dinv = s.g, s.gw, s.g.dinv
    if orient == "csr":
        rp, cl, hv = g.rowptr, g.col, g.heavy
        wrp, wcl, wv, whv = gw.rowptr, gw.col, gw.val, gw.heavy
    else:
        (rp, cl), hv = g.transpose(), g.heavy_t
        (wrp, wcl), wv, whv = gw.transpose(), gw.val_t, gw.heavy_t
    assert hv is not None and whv is not None

    def plan(p, on):
        return p if on else None
    return [
        ("spmm", lambda x, o, on: K.spmm(rp, cl, None, x, out=o, heavy=plan(hv, on)), False, None),
        ("spmm dinv", lambda x, o, on: K.spmm(rp, cl, dinv, x, out=o, heavy=plan(hv, on)), False, dinv),
        ("spmm_sum", lambda x, o, on: K.spmm_sum(rp, cl, x, out=o, heavy=plan(hv, on)), False, None),
        ("weighted dinv", lambda x, o, on: K.spmm(wrp, wcl, dinv, x, out=o, heavy=plan(whv, on), val=wv), True, dinv),
    ], (wrp, wcl, wv)


def _edges(s, orient):
    """(rows, cols) of the edge list in the orientation's row order."""
    return (s.ei[1], s.ei[0]) if orient == "csr" else (s.ei[0], s.ei[1])


def _int_features(n, h, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randint(-2, 3, (n, h), generator=gen, device=DEV, dtype=torch.int32)


# ------------------------------------------------------------------------------------------------
# the graph has what the sweep is for
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("plan", G.PLANS)
def test_sweep_graph_has_its_edges(graphs, sms, plan):
    from sgformer_b200 import kernels as K
    s = graphs(plan)
    assert s.n == G.plan(G.row_cap(sms), plan) and s.n > 3 * G.row_cap(sms) - 1
    lens = s.g.rowptr[1:] - s.g.rowptr[:-1]
    assert lens[s.special].tolist() == list(SPECIAL_LENS)
    assert bool((lens[s.iso] == 0).all()) and int((lens == 0).sum()) > int(s.iso.sum())
    assert sorted(s.g.heavy.rows.tolist()) == sorted(s.special[lens[s.special] > K.HEAVY_ROW].tolist())
    lens_t = s.g.transpose()[0].diff()
    assert bool((lens_t[s.iso] == 0).all()) and s.hub in s.g.heavy_t.rows.tolist()
    loops = s.ei[0] == s.ei[1]
    per_node = torch.bincount(s.ei[0][loops], minlength=s.n)
    assert int(per_node.max()) >= 3, "repeated self loops"
    key = s.ei[0] * s.n + s.ei[1]
    assert key.unique().numel() < key.numel(), "duplicate edges"
    assert torch.equal(s.gw.rowptr, s.g.rowptr) and torch.equal(s.gw.transpose()[0], s.g.transpose()[0])


# ------------------------------------------------------------------------------------------------
# every variant x every width, exactly
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,h", G.WIDTH_LIST, ids=G.WIDTH_IDS)
@pytest.mark.parametrize("plan", G.PLANS)
def test_spmm_variants_exact(graphs, plan, dtype, h):
    s = graphs(plan)
    n = s.n
    xi = _int_features(n, h, h)
    xbuf, x = _block(n, h, dtype)
    x.copy_(xi)
    ybuf, y = _block(n, h, dtype, SENTINEL[dtype])
    for orient in ORIENTS:
        calls, (wrp, wcl, wv) = _variants(s, orient)
        rows, cols = _edges(s, orient)
        ref = _coo_sum(rows, cols, xi, n).float()                  # exact: |sum| <= 2 * 3001
        wrows, wcols = _coo(wrp, wcl)
        wref = _coo_sum(wrows, wcols, xi, n, _quarters(wv)).double().div_(4).float()
        for label, run, weighted, scale in calls:
            want = _want(wref if weighted else ref, scale, dtype)
            for hub in (False, True):
                _bits(ybuf).fill_(SENTINEL[dtype])
                assert run(x, y, hub) is y
                _check_block(ybuf, h, want, f"{orient} {label} hub plan {hub}")
            del want
        del ref, wref


@pytest.mark.parametrize("dtype,h", G.FLOAT_WIDTHS, ids=[f"{G.name(d)}-h{h}" for d, h in G.FLOAT_WIDTHS])
def test_spmm_float_inputs_and_run_to_run(graphs, dtype, h):
    """Random features against fp64 under the bound of an fp32 sum of the row: (len + 2) u sum|x| (+ the bf16 rounding of the
    output); two runs are bit-identical, with and without the hub plan."""
    s = graphs("ragged")
    n = s.n
    gen = torch.Generator(device=DEV).manual_seed(100 + h)
    xbuf, x = _block(n, h, dtype)
    x.copy_(torch.randn(n, h, generator=gen, device=DEV))
    f64 = torch.float64
    out_ulp = 2.0 ** -8 if dtype == B16 else 0.0
    step = 1 << 14
    for orient in ORIENTS:
        calls, (wrp, wcl, wv) = _variants(s, orient)
        rows, cols = _edges(s, orient)
        lens = torch.bincount(rows, minlength=n).double()[:, None]
        for weighted in (False, True):
            if weighted:
                rows, cols = _coo(wrp, wcl)
            w = wv if weighted else None
            ref = _coo_sum(rows, cols, x, n, w, acc=f64)
            mag = _coo_sum(rows, cols, x, n, w, acc=f64, absolute=True)
            for label, run, wtd, scale in calls:
                if wtd != weighted:
                    continue
                sc = scale.double()[:, None] if scale is not None else torch.ones((n, 1), dtype=f64, device=DEV)
                for hub in (False, True):
                    a, b = run(x, None, hub), run(x, None, hub)
                    assert _mismatch(a, b) == 0, f"{orient} {label} hub plan {hub}: two runs differ"
                    for i in range(0, n, step):
                        r, m = ref[i:i + step] * sc[i:i + step], mag[i:i + step] * sc[i:i + step]
                        bound = (lens[i:i + step] + 2) * 2.0 ** -24 * m + out_ulp * r.abs()
                        err = (a[i:i + step].double() - r).abs()
                        assert bool((err <= bound).all()), f"{orient} {label} hub plan {hub}, rows from {i}: error " \
                                                           f"{(err / bound.clamp_min(1e-300)).max().item():.2f} x the bound"
            del ref, mag


# ------------------------------------------------------------------------------------------------
# grid-stride of the segment and finalize kernels (CSRs built directly: an edge list of 10^8 entries would cost gigabytes)
# ------------------------------------------------------------------------------------------------
def _direct_csr(lens, n_src, seed):
    lens = torch.tensor(lens, dtype=torch.int64, device=DEV)
    rowptr = torch.zeros(lens.numel() + 1, dtype=torch.int64, device=DEV)
    rowptr[1:] = torch.cumsum(lens, 0)
    gen = torch.Generator(device=DEV).manual_seed(seed)
    col = torch.randint(0, n_src, (int(rowptr[-1]),), generator=gen, device=DEV, dtype=torch.int32)
    val = torch.randint(-4, 5, (col.numel(),), generator=gen, device=DEV, dtype=torch.int32).float() / 4
    return rowptr, col, val


def _csr_ref(rowptr, col, xi, wq=None):
    """Exact int32 sum over a CSR, in entry chunks (no per-entry row array)."""
    n = rowptr.numel() - 1
    out = torch.zeros((n, xi.shape[1]), dtype=torch.int32, device=DEV)
    step = max(1 << 12, (1 << 24) // xi.shape[1])
    for i in range(0, col.numel(), step):
        pos = torch.arange(i, min(i + step, col.numel()), device=DEV)
        rows = torch.searchsorted(rowptr, pos, right=True) - 1
        v = xi.index_select(0, col[i:i + step].long())
        if wq is not None:
            v = v * wq[i:i + step, None]
        out.index_add_(0, rows, v)
    return out


def _hub_variants_exact(rowptr, col, val, heavy, n_src, dtype, h, seed):
    from sgformer_b200 import kernels as K
    n = rowptr.numel() - 1
    xi = _int_features(n_src, h, seed)
    xbuf, x = _block(n_src, h, dtype)
    x.copy_(xi)
    scale = torch.rand(n, generator=torch.Generator(device=DEV).manual_seed(seed), device=DEV) + 0.5
    ref = _csr_ref(rowptr, col, xi).float()                       # exact: |sum| < 2^22
    wref = _csr_ref(rowptr, col, xi, _quarters(val)).double().div_(4).float()
    ybuf, y = _block(n, h, dtype, SENTINEL[dtype])
    for label, run, r, sc in (
            ("spmm", lambda: K.spmm(rowptr, col, None, x, out=y, heavy=heavy), ref, None),
            ("spmm row_scale", lambda: K.spmm(rowptr, col, scale, x, out=y, heavy=heavy), ref, scale),
            ("spmm_sum", lambda: K.spmm_sum(rowptr, col, x, out=y, heavy=heavy), ref, None),
            ("weighted row_scale", lambda: K.spmm(rowptr, col, scale, x, out=y, heavy=heavy, val=val), wref, scale)):
        _bits(ybuf).fill_(SENTINEL[dtype])
        run()
        _check_block(ybuf, h, _want(r, sc, dtype), label)


@pytest.mark.parametrize("dtype,h", [(F32, 4), (B16, 8)], ids=["fp32-h4", "bf16-h8"])
def test_segment_kernel_grid_strides(sms, dtype, h):
    """More than 3 x row_cap hub segments: every warp of the capped segment grid runs three or four segments."""
    from sgformer_b200 import kernels as K
    sp = G.segment_plan(sms)
    lens = [sp["row_len"], 5] * sp["rows"]
    rowptr, col, val = _direct_csr(lens, 4096, 7)
    heavy = K.heavy_rows(rowptr)
    assert heavy.rows.numel() == sp["rows"] and heavy.seg_start.numel() == sp["n_seg"] > 3 * G.row_cap(sms)
    _hub_variants_exact(rowptr, col, val, heavy, 4096, dtype, h, 8)


@pytest.mark.parametrize("dtype,h", [(F32, 512), (B16, 1024)], ids=["fp32-h512", "bf16-h1024"])
def test_finalize_kernel_grid_strides(sms, dtype, h):
    """n_heavy x h > 3 x finalize_cap: every thread of the capped finalize grid adds up three or four hub-row values."""
    from sgformer_b200 import kernels as K
    fp = G.finalize_plan(dtype, h, sms)
    lens = [x for hub in fp["lens"] for x in (hub, 3)]
    rowptr, col, val = _direct_csr(lens, 4096, 9)
    heavy = K.heavy_rows(rowptr)
    assert heavy.rows.numel() == fp["n_heavy"] and fp["n_heavy"] * h > 3 * G.finalize_cap(sms)
    _hub_variants_exact(rowptr, col, val, heavy, 4096, dtype, h, 10)


# ------------------------------------------------------------------------------------------------
# phased SpMM over a rotated CSR
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,h", G.WIDTH_LIST, ids=G.WIDTH_IDS)
def test_phased_spmm_exact(graphs, dtype, h):
    """Rows split into three phases at per-row offsets (empty phases, a whole row in each phase, random cuts), the fp32 partials
    in a pitched buffer passed from phase to phase in place, over column ids rotated by n / 3 and the rotated operand."""
    from sgformer_b200 import kernels as K
    s = graphs("ragged")
    n, rp, cl = s.n, s.rot_rowptr, s.rot_col
    assert torch.equal(rp, s.g.rowptr)
    xi = _int_features(n, h, 50 + h)
    xbuf, x = _block(n, h, dtype)
    x.copy_(torch.roll(xi, -s.rot, 0))                 # row i of the rotated operand = node (i + rot) mod n
    ref = _coo_sum(s.ei[1], s.ei[0], xi, n).float()
    lens = rp.diff()
    gen = torch.Generator(device=DEV).manual_seed(h)
    a = (torch.rand(n, generator=gen, device=DEV) * (lens + 1)).long().clamp_max(lens)
    b = a + (torch.rand(n, generator=gen, device=DEV) * (lens - a + 1)).long().clamp_max(lens - a)
    kind = torch.arange(n, device=DEV) % 6
    a = torch.where(kind == 0, 0, torch.where(kind == 1, lens, torch.where(kind == 2, 0, a)))
    b = torch.where(kind == 0, 0, torch.where(kind == 1, lens, torch.where(kind == 2, lens, torch.where(kind == 3, a, b))))
    assert bool(((0 <= a) & (a <= b) & (b <= lens)).all())
    a, b = a.to(torch.int32).contiguous(), b.to(torch.int32).contiguous()
    pbuf = torch.empty((n, h + 4), dtype=torch.float32, device=DEV)
    part = pbuf[:, :h]
    for scale in (None, s.g.dinv):
        _bits(pbuf).fill_(SENTINEL[F32])
        assert K.spmm_range(rp, cl, None, x, None, a, None, part) is None
        assert K.spmm_range(rp, cl, None, x, a, b, part, part) is None
        out = K.spmm_range(rp, cl, scale, x, b, None, part, None)
        bad = _mismatch(out, _want(ref, scale, dtype))
        assert bad == 0, f"phased, row_scale {'dinv' if scale is not None else None}: {bad} elements differ"
        assert bool((_bits(pbuf[:, h:]) == SENTINEL[F32]).all()), "the partial buffer's padding was written"


# ------------------------------------------------------------------------------------------------
# refusals and the negative control
# ------------------------------------------------------------------------------------------------
def _heavy_direct(K, x, out, heavy, rowptr, col):
    """sgf_spmm_heavy on its own (the wrappers call it only after the row kernel accepted the operands)."""
    from sgformer_b200.kernels import _p, _stream, dcode, lib
    ns = heavy.seg_start.numel()
    partial = torch.empty((ns, max(x.shape[1], 1)), dtype=torch.float32, device=DEV)
    K.check(lib().sgf_spmm_heavy(_p(col), None, _p(x), x.stride(0), _p(out), out.stride(0), x.shape[1], dcode(x),
                                 _p(heavy.seg_start), _p(heavy.seg_len), ns, _p(partial), _p(heavy.rows), _p(heavy.seg_ptr),
                                 heavy.rows.numel(), _stream()), "sgf_spmm_heavy")


def test_refused_shapes_raise_and_leave_out_untouched(graphs):
    from sgformer_b200 import kernels as K
    s = graphs("exact")
    g, gw, n = s.g, s.gw, s.n
    cases = [(dtype, h, 0) for dtype, h in G.REFUSED] + [(F32, 64, 1), (B16, 64, 1)]   # (.., offset): x not 16-byte aligned
    for dtype, h, off in cases:
        v = G.vn(dtype)
        pitch = -(-(h + off) // v) * v + v
        xbuf = torch.zeros((n, pitch), dtype=dtype, device=DEV)
        x = xbuf[:, off:off + h]
        obuf = torch.empty((n, pitch), dtype=dtype, device=DEV)
        _bits(obuf).fill_(SENTINEL[dtype])
        out = obuf[:, :h]
        pbuf = torch.empty((n, -(-h // 4) * 4 + 4), dtype=torch.float32, device=DEV)
        _bits(pbuf).fill_(SENTINEL[F32])
        for label, run in (
                ("sgf_spmm", lambda: K.spmm(g.rowptr, g.col, g.dinv, x, out=out, heavy=g.heavy)),
                ("sgf_spmm_sum", lambda: K.spmm_sum(g.rowptr, g.col, x, out=out, heavy=g.heavy)),
                ("sgf_spmm_weighted", lambda: K.spmm(gw.rowptr, gw.col, g.dinv, x, out=out, heavy=gw.heavy, val=gw.val)),
                ("sgf_spmm_heavy", lambda: _heavy_direct(K, x, out, g.heavy, g.rowptr, g.col)),
                ("sgf_spmm_range", lambda: K.spmm_range(g.rowptr, g.col, None, x, None, None, None, pbuf[:, :h]))):
            with pytest.raises(RuntimeError, match=f"{label} failed: (invalid argument|unsupported shape)"):
                run()
            torch.cuda.synchronize()
            assert bool((_bits(obuf) == SENTINEL[dtype]).all()), f"{G.name(dtype)} h={h} offset {off}: {label} wrote out"
            assert bool((_bits(pbuf) == SENTINEL[F32]).all()), f"{G.name(dtype)} h={h} offset {off}: {label} wrote partials"


def test_exact_comparison_reports_swapped_columns(graphs):
    """Negative control: two column ids swapped between two rows must show as a mismatch in exactly those rows."""
    from sgformer_b200 import kernels as K
    s = graphs("ragged")
    g, n, h = s.g, s.n, 16
    xi = _int_features(n, h, 3)
    x = xi.float()
    want = _coo_sum(s.ei[1], s.ei[0], xi, n).float()
    assert _mismatch(K.spmm(g.rowptr, g.col, None, x), want) == 0
    lens = g.rowptr.diff()
    r1, r2 = [int(r) for r in (lens == 3).nonzero().flatten()[[0, -1]]]
    j1, j2 = int(g.rowptr[r1]), int(g.rowptr[r2])
    c1, c2 = int(g.col[j1]), int(g.col[j2])
    assert not torch.equal(xi[c1], xi[c2]), "pick rows whose swapped neighbours differ"
    col = g.col.clone()
    col[j1], col[j2] = c2, c1
    got = K.spmm(g.rowptr, col, None, x)
    bad_rows = (_bits(got) != _bits(want)).any(1).nonzero().flatten().tolist()
    assert bad_rows == sorted([r1, r2]), "the exact comparison must report the swap"


# ------------------------------------------------------------------------------------------------
# edge-weight gradient
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def edge_graphs(sms):
    """form -> (Graph, edge_index): DIFFormer (self-loop mode 0) and GCN (mode 1, positive weights) over 3 x edge_grad_cap
    (+ tail) rows."""
    from sgformer_b200.graph import Graph
    n = G.plan(G.edge_grad_cap(sms), "ragged")
    ei, w, *_ = _edge_list(n, 11)
    w = w.abs() + 0.25
    return {"difformer": (Graph(ei, n, 0, edge_weight=w), ei), "gcn": (Graph(ei, n, 1, edge_weight=w), ei)}


def _edge_grad_ref(gr, ei, a, b, y, u, dinv, loops):
    """fp64 restatement of sgf_edge_weight_grad over the same operands (kernel_emu_weighted.edge_weight_grad, vectorised):
    d_j = <a_c, b_r> + q_c per CSR entry j = (c, r), q_c = -1/2 dinv_c (<a_c, y_c> + <b_c, u_c>); the loop entries of a mode-1
    CSR go to every self-loop edge of their node.  -> (grad, magnitude) per edge: the sum and the sum of |terms|."""
    n = gr.rowptr.numel() - 1
    rows, cols = _coo(gr.rowptr, gr.col)
    A, B = a.double(), b.double()
    q = torch.zeros(n, dtype=torch.float64, device=DEV)
    qm = torch.zeros_like(q)
    if y is not None:
        Y, U, dv = y.double(), u.double(), dinv.double()
        q = -0.5 * dv * ((A * Y).sum(1) + (B * U).sum(1))
        qm = 0.5 * dv.abs() * ((A * Y).abs().sum(1) + (B * U).abs().sum(1))
    d = torch.empty(rows.numel(), dtype=torch.float64, device=DEV)
    m = torch.empty_like(d)
    step = max(1, (1 << 22) // a.shape[1])
    for i in range(0, rows.numel(), step):
        p = A.index_select(0, rows[i:i + step]) * B.index_select(0, cols[i:i + step])
        d[i:i + step] = p.sum(1) + q[rows[i:i + step]]
        m[i:i + step] = p.abs().sum(1) + qm[rows[i:i + step]]
    eid = gr.eid
    is_loop = (rows == cols) if loops else torch.zeros_like(rows, dtype=torch.bool)
    keep = ~is_loop & (eid >= 0)
    assert eid[keep].unique().numel() == int(keep.sum()), "one CSR entry per edge"
    grad = torch.zeros(ei.shape[1], dtype=torch.float64, device=DEV)
    mag = torch.zeros_like(grad)
    grad[eid[keep]], mag[eid[keep]] = d[keep], m[keep]
    if loops:
        assert torch.equal(rows[is_loop], torch.arange(n, device=DEV)), "one loop entry per node"
        self_loop = ei[0] == ei[1]
        grad[self_loop], mag[self_loop] = d[is_loop][ei[0][self_loop]], m[is_loop][ei[0][self_loop]]
    return grad, mag


@pytest.mark.parametrize("form", ["difformer", "gcn"])
@pytest.mark.parametrize("dtype,h", G.EDGE_GRAD_WIDTHS, ids=[f"{G.name(d)}-h{h}" for d, h in G.EDGE_GRAD_WIDTHS])
def test_edge_weight_grad(edge_graphs, sms, form, dtype, h):
    """Against fp64 under the bound of an fp32 dot product of h terms, (h + 16) u sum|terms|, per edge; pitched operands whose
    NaN padding must not leak in; two runs bit-identical; and a second run into the same `out` adds (doubles it exactly)."""
    from sgformer_b200 import kernels as K
    gr, ei = edge_graphs[form]
    n = gr.rowptr.numel() - 1
    assert n > 3 * G.edge_grad_cap(sms)
    gen = torch.Generator(device=DEV).manual_seed(h)
    ops = []
    for _ in range(4 if form == "gcn" else 2):
        buf, t = _block(n, h, dtype)
        t.copy_(torch.randn(n, h, generator=gen, device=DEV))
        ops.append((buf, t))
    a, b = ops[0][1], ops[1][1]
    kw = dict(y=ops[2][1], u=ops[3][1], dinv=gr.dinv, edge_index=ei, loops=True) if form == "gcn" else {}
    if form == "gcn":
        loops = ei[0] == ei[1]
        assert int(torch.bincount(ei[0][loops]).max()) >= 3, "duplicated self loops"
    out = torch.zeros(ei.shape[1], dtype=torch.float32, device=DEV)
    K.edge_weight_grad(gr.rowptr, gr.col, gr.eid, a, b, out, **kw)
    ref, mag = _edge_grad_ref(gr, ei, a, b, kw.get("y"), kw.get("u"), kw.get("dinv"), form == "gcn")
    err = (out.double() - ref).abs()
    bound = (h + 16) * 2.0 ** -24 * mag
    assert bool((err <= bound).all()), f"error {(err / bound.clamp_min(1e-300)).max().item():.2f} x the bound"
    assert bool((mag > 0).any()) and bool((out != 0).any())
    again = torch.zeros_like(out)
    K.edge_weight_grad(gr.rowptr, gr.col, gr.eid, a, b, again, **kw)
    assert torch.equal(_bits(again), _bits(out)), "two runs differ"
    K.edge_weight_grad(gr.rowptr, gr.col, gr.eid, a, b, again, **kw)
    assert torch.equal(again, 2 * out), "out is accumulated into"


class _Data:
    def __init__(self, x, ei, w):
        self.graph = {"node_feat": x, "edge_index": ei, "edge_weight": w, "num_nodes": x.shape[0]}


@pytest.mark.parametrize("prec,h,tol_max,tol_norm", [("bf16", 1024, 1e-1, 5e-2), ("fp32", 512, 1e-4, 1e-4)], ids=["bf16-h1024", "fp32-h512"])
def test_weighted_gcn_edge_weight_grad_at_widest_hidden(sms, prec, h, tol_max, tol_norm):
    """models.GCN at the widest hidden width of its precision (two layers, no BatchNorm, dropout 0; engine.gcn_forward /
    gcn_backward) with a learnable edge_weight: its gradient against fp64 autograd of the dense restatement (weighted gcn_norm
    for the first conv, the unweighted pattern for the last).  fp32 checks the chain tightly; bf16 the width only it reaches."""
    from sgformer_b200 import medium as M
    n, d, c = 1200, 32, 16
    g = torch.Generator().manual_seed(21)
    src = torch.cat([torch.randint(0, n, (9000,), generator=g), torch.tensor([1, 2, 2, 2])])
    dst = torch.cat([torch.randint(0, n - 50, (9000,), generator=g), torch.tensor([1, 2, 2, 2])])
    src = torch.cat([src, src[:400]])
    dst = torch.cat([dst, dst[:400]])
    ei = torch.stack([src, dst])
    w = 0.1 + torch.rand(ei.shape[1], generator=g)
    x = torch.randn(n, d, generator=g)
    lw = torch.randn(n, c, generator=g)
    torch.manual_seed(3)
    m = M.GCN(d, h, c, num_layers=2, dropout=0.0, use_bn=False)
    with torch.no_grad():
        m.convs[0].bias.uniform_(-0.1, 0.1)
    m = m.to(DEV).set_precision(prec)
    m.train()
    wg = w.to(DEV).requires_grad_(True)
    out = m(_Data(x.to(DEV), ei.to(DEV), wg))
    (out.float() * lw.to(DEV)).sum().backward()
    W0, b0, W1, b1 = (p.detach().double().cpu() for p in (m.convs[0].lin.weight, m.convs[0].bias, m.convs[1].lin.weight,
                                                           m.convs[1].bias))
    wd = w.double().requires_grad_(True)
    Aw = KW.dense_gcn_adjacency(ei, wd, n)
    A1 = KW.dense_gcn_adjacency(ei, torch.ones_like(wd).detach(), n)
    h1 = torch.relu(Aw @ (x.double() @ W0.t()) + b0)
    ref = A1 @ (h1 @ W1.t()) + b1
    (ref * lw.double()).sum().backward()
    assert (out.double().cpu() - ref.detach()).abs().max().item() < 2 * tol_norm * ref.abs().max().item()
    # bf16 rounds t, dz and the layer output before the kernel contracts them, and the degree term cancels most of <dz_c, t_r>:
    # its bound is the bf16 one of tests/test_gpu_weighted.py, per entry against the largest, and 5e-2 over the whole vector
    got, want = wg.grad.double().cpu(), wd.grad
    rel = (got - want).abs().max().item() / want.abs().max().item()
    rel_norm = ((got - want).norm() / want.norm()).item()
    print(f"{prec} GCN hidden {h}: edge_weight.grad error {rel:.2e} of the largest entry, {rel_norm:.2e} in norm")
    assert rel < tol_max and rel_norm < tol_norm, f"edge_weight.grad: {rel:.2e} of its largest entry, {rel_norm:.2e} in norm"


# ------------------------------------------------------------------------------------------------
def test_peak_device_memory(mem0):
    """The module keeps its device memory under 8 GiB above what it found (the GPU is shared)."""
    peak = torch.cuda.max_memory_allocated() - mem0
    print(f"test_gpu_spmm_sweep: peak device memory {peak / 2 ** 30:.2f} GiB above the module's start, "
          f"{torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count} SMs")
    assert peak < PEAK_BUDGET
