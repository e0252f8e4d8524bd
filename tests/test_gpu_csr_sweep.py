"""The graph-structure kernels (csrc/csr.cu) bit for bit against references that never call the library, on the graphs of
tests/csr_geometry.py: every row-sort tier on both sides of its edges, the capped scratch and the row past it, scans of one to
three block-sum passes, fill windows of the default size, of 1 MiB (past the 12-window cap) and of one launch, and grids past
their caps.

References: `ref_csr` restates every build on the device with torch's stable sort (rows = keys, entries ordered by column and
then edge position); on the small graph it is itself checked against oracle/np_ref.py, tests/kernel_emu.py and
tests/kernel_emu_weighted.py.  Edge lists carry duplicate edges, single and triple self loops, and rows whose sources are one
repeated node (runs of 31 to 65 equal columns in to_undirected's rows).  Weights are dyadic and positive, so the mode-1 degree sums
are exact in any order."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

import csr_geometry as G
import kernel_emu as emu
import kernel_emu_weighted as KW
from oracle import np_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
PEAK_BUDGET = 12 * 2 ** 30
TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)


@pytest.fixture(scope="module")
def mem0():
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    return torch.cuda.memory_allocated()


@pytest.fixture(scope="module")
def K(mem0):
    from sgformer_b200 import kernels
    return kernels


_CACHE = {}


def graph(name):
    """(edge_index int64 [2, E], weights fp32 [E]) of a table graph, on the device (seeded: the same in every process)."""
    if name not in _CACHE:
        _CACHE[name] = make_edges(G.GRAPHS[name], seed=1 + list(G.GRAPHS).index(name))
    return _CACHE[name]


def make_edges(spec, seed):
    lens_c = spec.lengths()
    n, e = spec.n, int(lens_c.sum())
    start_c = torch.cumsum(lens_c, 0) - lens_c
    g = torch.Generator(device=DEV).manual_seed(seed)
    lens = lens_c.to(DEV)
    dst = torch.repeat_interleave(torch.arange(n, device=DEV), lens)
    src = torch.randint(0, n, (e,), generator=g, device=DEV)
    # duplicate edges: every 50th entry repeats the one before it in its row
    start = start_c.to(DEV)
    pos = torch.arange(e, device=DEV) - start[dst]
    dup = (pos > 0) & (torch.arange(e, device=DEV) % 50 == 0)
    src[dup] = src[dup.nonzero().flatten() - 1]
    # self loops: one on rows r % 10 == 3, two on rows r % 20 == 3 (first entries of the row)
    r = torch.arange(n, device=DEV)
    one = (r % 10 == 3) & (lens >= 1)
    two = (r % 20 == 3) & (lens >= 2)
    src[start[one]] = r[one]
    src[start[two] + 1] = r[two]
    # special rows: the second row of each RUN_LENS length takes one source throughout; the others with >= 3 entries hold three
    # self loops (the mode-1 weight is the last one's)
    seen = {}
    idx, val = [], []
    for row, length in spec.special_rows():
        k = seen.get(length, 0)
        seen[length] = k + 1
        s = int(start_c[row])
        if length in G.RUN_LENS and k == 1:
            idx.append(torch.arange(s, s + length))
            val.append(torch.full((length,), (row * 7919 + 13) % n))
        elif length >= 3:
            idx.append(torch.arange(s, s + 3))
            val.append(torch.full((3,), row))
    if idx:
        src[torch.cat(idx).to(DEV)] = torch.cat(val).to(DEV)
    perm = torch.randperm(e, generator=g, device=DEV)
    ei = torch.stack([src[perm], dst[perm]]).contiguous()
    w = torch.randint(1, 9, (e,), generator=g, device=DEV).float() / 4
    return ei, w


# ------------------------------------------------------------------------------------------------
# references (device, torch only)
# ------------------------------------------------------------------------------------------------
def ref_csr(ei, n, by_source=False, mode=0, rows=None, col_rot=None, w=None):
    """The CSR every build entry point makes: rowptr, col int32, eid int64 (-1: an added loop without a source loop), dinv (the
    count-based one; with `w` in mode 1 the weighted one), val (with `w`)."""
    src, dst = ei[0], ei[1]
    e = src.numel()
    key, other = (src, dst) if by_source else (dst, src)
    eid = torch.arange(e, device=DEV)
    if mode == 1:
        keep = src != dst
        ar = torch.arange(n, device=DEV)
        last = torch.full((n,), -1, dtype=torch.int64, device=DEV)
        last.scatter_reduce_(0, src[~keep], eid[~keep], "amax")
        key, other, eid = torch.cat([key[keep], ar]), torch.cat([other[keep], ar]), torch.cat([eid[keep], last])
    nr = n
    if rows is not None:
        m = (key >= rows[0]) & (key < rows[1])
        key, other, eid = key[m] - rows[0], other[m], eid[m]
        nr = rows[1] - rows[0]
    span = n
    if col_rot is not None:
        other = (other - col_rot[0]) % col_rot[1]
        span = max(n, col_rot[1])
    order = torch.sort(key * span + other, stable=True).indices     # ties (duplicates) keep edge order: (col, eid)
    key, other, eid = key[order], other[order], eid[order]
    deg = torch.bincount(key, minlength=nr)
    rowptr = torch.zeros(nr + 1, dtype=torch.int64, device=DEV)
    rowptr[1:] = torch.cumsum(deg, 0)
    d = deg.float()
    dinv = torch.where(d > 0, (1.0 / d).sqrt(), torch.zeros_like(d))
    out = dict(rowptr=rowptr, col=other.to(torch.int32), eid=eid, dinv=dinv)
    if w is not None:
        val = torch.where(eid >= 0, w[eid.clamp(min=0)], torch.ones_like(eid, dtype=torch.float32))
        out["val"] = val
        if mode == 1:
            dd = torch.zeros(nr, dtype=torch.float64, device=DEV).index_add_(0, key, val.double()).float()
            out["dinv"] = torch.where(dd == 0, torch.zeros_like(dd), (1.0 / dd.double().sqrt()).float())
    return out


def ref_subgraph(ei, n, subset):
    mask = torch.zeros(n, dtype=torch.bool, device=DEV)
    mask[subset] = True
    relabel = torch.full((n,), -1, dtype=torch.int64, device=DEV)
    relabel[subset] = torch.arange(subset.numel(), device=DEV)
    keep = mask[ei[0]] & mask[ei[1]]
    return relabel[ei[:, keep]]


def _bits(t):
    return t.view(torch.int32)


def _keys(col, eid):
    return (col.long() << 32) | (eid + 1)


def unsorted_rows(rowptr, tot):
    """Rows past the capped scratch (left in fill order by the documented limit)."""
    lens = rowptr[1:] - rowptr[:-1]
    return (lens > G.scratch_elems(tot)).nonzero().flatten().tolist()


def row_mismatch(rowptr, got, want_rowptr, want, unsorted=()):
    """Rows whose entries differ from the reference's; a row in `unsorted` only when its entries are not a permutation of the
    reference's row.  rowptr must be equal."""
    assert torch.equal(rowptr, want_rowptr), "rowptr differs"
    assert got.shape == want.shape, f"{got.numel()} entries, reference {want.numel()}"
    pos = (got != want).nonzero().flatten()
    bad = set(torch.unique(torch.searchsorted(rowptr, pos, right=True) - 1).tolist()) if pos.numel() else set()
    for r in unsorted:
        s, e = int(rowptr[r]), int(rowptr[r + 1])
        bad.discard(r)
        if not torch.equal(torch.sort(got[s:e]).values, torch.sort(want[s:e]).values):
            bad.add(r)
    return sorted(bad)


def check_csr(got, want, tot, what, dinv=True):
    rowptr, col = got[0], got[1]
    unsorted = unsorted_rows(want["rowptr"], tot)
    bad = row_mismatch(rowptr, col, want["rowptr"], want["col"], unsorted)
    assert not bad, f"{what}: {len(bad)} rows differ, first {bad[:5]}"
    if dinv and got[2] is not None:
        assert torch.equal(_bits(got[2]), _bits(want["dinv"])), f"{what}: dinv bits differ"
    return unsorted


def check_weighted(got, want, w, tot, what):
    rowptr, col, eid, val, dinv = got
    unsorted = unsorted_rows(want["rowptr"], tot)
    bad = row_mismatch(rowptr, _keys(col, eid), want["rowptr"], _keys(want["col"], want["eid"]), unsorted)
    assert not bad, f"{what}: {len(bad)} rows differ in (col, eid), first {bad[:5]}"
    want_val = torch.where(eid >= 0, w[eid.clamp(min=0)], torch.ones_like(val))
    assert torch.equal(_bits(val), _bits(want_val)), f"{what}: val is not weight[eid]"
    if not unsorted:
        assert torch.equal(_bits(val), _bits(want["val"])), f"{what}: val differs"
    assert torch.equal(_bits(dinv), _bits(want["dinv"])), f"{what}: dinv bits differ"
    return unsorted


def _tot(ei, n):
    return ei.shape[1] + n


# ------------------------------------------------------------------------------------------------
# the reference against the CPU restatements, and the comparison helper against a planted defect
# ------------------------------------------------------------------------------------------------
def test_reference_matches_the_cpu_restatements():
    ei, w = graph("small")
    n = G.GRAPHS["small"].n
    eic, wc = ei.cpu(), w.cpu()
    for by_source in (False, True):
        rp, cl, dv = np_ref.gcn_csr((eic.flip(0) if by_source else eic).numpy(), n)
        r = ref_csr(ei, n, by_source)
        assert np.array_equal(r["rowptr"].cpu().numpy(), rp) and np.array_equal(r["col"].cpu().numpy(), cl)
        assert np.array_equal(r["dinv"].cpu().numpy().view(np.int32), dv.view(np.int32))
        rp1, cl1, _ = emu.csr_build(eic, n, by_source, 1)
        r1 = ref_csr(ei, n, by_source, 1)
        assert torch.equal(r1["rowptr"].cpu(), rp1) and torch.equal(r1["col"].cpu(), cl1)
        for mode in (0, 1):
            rp, cl, eid, val, dv = KW.csr_weighted(eic.numpy(), wc.numpy(), n, by_source, mode)
            r = ref_csr(ei, n, by_source, mode, w=w)
            for k, v in (("rowptr", rp), ("col", cl), ("eid", eid)):
                assert np.array_equal(r[k].cpu().numpy(), v), (by_source, mode, k)
            assert np.array_equal(r["val"].cpu().numpy().view(np.int32), val.view(np.int32))
            if not by_source:
                assert np.array_equal(r["dinv"].cpu().numpy().view(np.int32), dv.view(np.int32)), (by_source, mode)
    rows, rot = (1000, 3001), (1234, n + 5)
    rp, cl, _ = emu.csr_build(eic, n, False, 1, False, rows=rows, col_rot=rot)
    r = ref_csr(ei, n, False, 1, rows=rows, col_rot=rot)
    assert torch.equal(r["rowptr"].cpu(), rp) and torch.equal(r["col"].cpu(), cl)


def test_comparison_helper_reports_a_swapped_pair():
    ei, _ = graph("small")
    n = G.GRAPHS["small"].n
    r = ref_csr(ei, n)
    lens = r["rowptr"][1:] - r["rowptr"][:-1]
    row = int((lens == 257).nonzero()[0])
    s = int(r["rowptr"][row])
    col = r["col"].clone()
    j = s + 100
    while col[j] == col[j + 1]:
        j += 1
    col[[j, j + 1]] = col[[j + 1, j]]
    assert row_mismatch(r["rowptr"], col, r["rowptr"], r["col"]) == [row]
    assert row_mismatch(r["rowptr"], col, r["rowptr"], r["col"], unsorted=[row]) == [], "a permutation within an unsorted row"
    col[s] = col[s] + 1
    assert row_mismatch(r["rowptr"], col, r["rowptr"], r["col"], unsorted=[row]) == [row]


# ------------------------------------------------------------------------------------------------
# the builds
# ------------------------------------------------------------------------------------------------
GRAPH_NAMES = list(G.GRAPHS)


@pytest.mark.parametrize("name", GRAPH_NAMES)
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("by_source", [False, True])
def test_csr_build(K, name, mode, by_source):
    ei, _ = graph(name)
    n = G.GRAPHS[name].n
    got = K.csr_build(ei, n, by_source, mode, True)
    unsorted = check_csr(got, ref_csr(ei, n, by_source, mode), _tot(ei, n), f"{name} mode {mode} by_source {by_source}")
    if name == "large" and not by_source:
        lens = got[0][1:] - got[0][:-1]
        tot = _tot(ei, n)
        tiers = {G.tier(x, tot) for x in lens.unique().tolist()}
        assert "hub1" in tiers and "hub16" in tiers
        assert len(unsorted) == (1 if mode == 0 else 0), unsorted       # mode 1 drops the hub's three loops: 2^26 - 1 fits


@pytest.mark.parametrize("name", GRAPH_NAMES)
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("by_source", [False, True])
def test_csr_build_weighted(K, name, mode, by_source):
    ei, w = graph(name)
    n = G.GRAPHS[name].n
    got = K.csr_build_weighted(ei, w, n, by_source, mode, True)
    check_weighted(got, ref_csr(ei, n, by_source, mode, w=w), w, _tot(ei, n), f"{name} mode {mode} by_source {by_source}")
    if mode == 1 and not by_source:
        # rows with three duplicated loops: the added loop carries the last one's edge position and weight
        rowptr, col, eid = got[0], got[1], got[2]
        rows = torch.repeat_interleave(torch.arange(n, device=DEV), rowptr[1:] - rowptr[:-1])
        loop = col.long() == rows
        src_loops = (ei[0] == ei[1])
        cnt = torch.bincount(ei[0][src_loops], minlength=n)
        assert int((cnt >= 3).sum()) > 0
        assert int(loop.sum()) == n and bool((eid[loop][cnt >= 3] >= 0).all())


def _shards(n):
    return [(0, n // 3), (n // 3, n - 1), (n - 1, n)]


@pytest.mark.parametrize("name", ["small", "medium", "large"])
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("by_source", [False, True])
def test_row_shard_and_rotated_builds(K, name, mode, by_source):
    ei, _ = graph(name)
    n = G.GRAPHS[name].n
    tot = _tot(ei, n)
    for rows in _shards(n):
        got = K.csr_build(ei, n, by_source, mode, True, rows=rows)
        check_csr(got, ref_csr(ei, n, by_source, mode, rows=rows), ei.shape[1] + rows[1] - rows[0], f"{name} rows {rows}")
    for rot in ((n // 3, n), (n - 1, n + 7)):
        got = K.csr_build(ei, n, by_source, mode, True, col_rot=rot)
        check_csr(got, ref_csr(ei, n, by_source, mode, col_rot=rot), tot, f"{name} col_rot {rot}")
    rows, rot = (n // 4, n // 2 + 1), (n // 2, n + 3)
    got = K.csr_build(ei, n, by_source, mode, True, rows=rows, col_rot=rot)
    check_csr(got, ref_csr(ei, n, by_source, mode, rows=rows, col_rot=rot), ei.shape[1] + rows[1] - rows[0],
              f"{name} rows {rows} col_rot {rot}")


@pytest.mark.parametrize("name", ["small", "medium"])
def test_csr_row_splits(K, name):
    """Split counts on the rotated CSR at 0, on both sides of the rank-block edges and at mod."""
    ei, _ = graph(name)
    n = G.GRAPHS[name].n
    mod = n + 5
    rp, col, _ = K.csr_build(ei, n, col_rot=(n // 3, mod))
    b = mod // 4
    thr = [0, 1, b - 1, b, b + 1, 2 * b, 3 * b, mod - 1, mod]
    got = K.csr_row_splits(rp, col, thr)
    rows = torch.repeat_interleave(torch.arange(n, device=DEV), rp[1:] - rp[:-1])
    for t, x in enumerate(thr):
        want = torch.zeros(n, dtype=torch.int64, device=DEV).index_add_(0, rows, (col.long() < x).long())
        assert torch.equal(got[t].long(), want), (name, x)
    assert bool((got[0] == 0).all()) and torch.equal(got[-1].long(), rp[1:] - rp[:-1])


@pytest.mark.parametrize("name", ["small", "medium"])
def test_to_undirected(K, name):
    ei, _ = graph(name)
    n = G.GRAPHS[name].n
    got = K.to_undirected(ei, n)
    want = torch.from_numpy(np_ref.to_undirected(ei.cpu().numpy(), n))
    assert torch.equal(got.cpu(), want)
    # the run rows reach to_undirected's rows with 31 to 65 equal columns, across its 32-entry passes
    und_rp = ref_csr(torch.cat([ei, ei.flip(0)], 1), n)
    rows = torch.repeat_interleave(torch.arange(n, device=DEV), und_rp["rowptr"][1:] - und_rp["rowptr"][:-1])
    c = und_rp["col"].long()
    runs = torch.unique_consecutive(rows * n + c, return_counts=True)[1]
    assert {31, 32, 33, 64, 65} <= set(runs.tolist())


@pytest.mark.parametrize("name", ["medium", "many"])
def test_remove_self_loops_and_subgraph(K, name):
    ei, _ = graph(name)
    n = G.GRAPHS[name].n
    if name == "many":
        assert ei.shape[1] > 4_194_304, "the flag scans make two block-sum passes"
    got = K.remove_self_loops(ei)
    assert torch.equal(got, ei[:, ei[0] != ei[1]])
    assert np.array_equal(got.cpu().numpy(), np_ref.remove_self_loops(ei.cpu().numpy()))
    g = torch.Generator(device=DEV).manual_seed(5)
    for frac in (0.6, 1.0):
        subset = torch.randperm(n, generator=g, device=DEV)[:int(frac * n)]
        assert torch.equal(K.subgraph(ei, n, subset), ref_subgraph(ei, n, subset)), frac


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("frac", [1.0, 0.5])
def test_csr_subset(K, mode, frac):
    """Subsets of the medium graph whose induced rows fall in every tier (a permutation of all nodes keeps every row; half the
    nodes plus every special row), against the subgraph's edge list built by the reference; mode 0 with the transposed half."""
    name = "medium"
    ei, _ = graph(name)
    spec = G.GRAPHS[name]
    n = spec.n
    g = torch.Generator(device=DEV).manual_seed(7)
    perm = torch.randperm(n, generator=g, device=DEV)
    if frac < 1.0:
        special = torch.tensor([r for r, _ in spec.special_rows()], device=DEV)
        keep = torch.zeros(n, dtype=torch.bool, device=DEV)
        keep[perm[: int(frac * n)]] = True
        keep[special] = True
        perm = perm[keep[perm]]
    b = perm.numel()
    sub_ei = ref_subgraph(ei, n, perm)
    node_map = torch.full((n,), -1, dtype=torch.int32, device=DEV)
    rp, col, _ = K.csr_build(ei, n, False, mode, False)
    want = ref_csr(sub_ei, b, False, mode)
    capacity = int((rp[perm + 1] - rp[perm]).sum())       # the default bound; the sort scratch is sized by it
    if mode == 0:
        rp_t, col_t, _ = K.csr_build(ei, n, True, 0, False)
        capacity = min(capacity, int((rp_t[perm + 1] - rp_t[perm]).sum()))
        got = K.csr_subset(rp, col, n, perm, node_map, transposed=(rp_t, col_t))
        want_t = ref_csr(sub_ei, b, True, 0)
        check_csr((got[4], got[5], None), want_t, capacity + b, f"subset {frac} transposed")
    else:
        got = K.csr_subset(rp, col, n, perm, node_map)
    tot = capacity + b
    check_csr(got[:3], want, tot, f"subset {frac} mode {mode}")
    assert bool((node_map == -1).all()), "node_map restored"
    lens = got[0][1:] - got[0][:-1]
    tiers = {G.tier(x, tot) for x in lens.unique().tolist()}
    assert {"warp1", "warp2", "warp_smem", "block_smem", "hub16"} <= tiers, tiers
    if frac == 1.0 and mode == 0:
        assert "hub1" in tiers


def test_run_to_run_bit_identity(K):
    ei, w = graph("medium")
    n = G.GRAPHS["medium"].n
    for mode in (0, 1):
        a, b = K.csr_build(ei, n, False, mode), K.csr_build(ei, n, False, mode)
        assert all(torch.equal(x, y) for x, y in zip(a, b)), mode
        a, b = K.csr_build_weighted(ei, w, n, False, mode), K.csr_build_weighted(ei, w, n, False, mode)
        assert all(torch.equal(x, y) for x, y in zip(a, b)), mode
    assert torch.equal(K.to_undirected(ei, n), K.to_undirected(ei, n))


def test_edge_symmetry(K):
    ei, _ = graph("medium")
    n = G.GRAPHS["medium"].n
    und = K.to_undirected(ei, n)
    und = und[:, torch.randperm(und.shape[1], generator=torch.Generator(device=DEV).manual_seed(3), device=DEV)].contiguous()
    assert K.edge_symmetry(und, n)
    k = int((und[0] != und[1]).nonzero()[0])
    moved = und.clone()
    moved[1, k] = (moved[1, k] + 1) % n
    assert not K.edge_symmetry(moved, n), "one edge moved"
    assert not K.edge_symmetry(torch.cat([und, und[:, k:k + 1]], 1), n), "one edge doubled"
    lo, hi = torch.minimum(und[0], und[1]), torch.maximum(und[0], und[1])
    w = ((lo * 31 + hi * 17) % 16 + 1).float() / 4           # symmetric: w(r, c) == w(c, r)
    assert K.edge_symmetry_weighted(und, w, n)
    w2 = w.clone()
    w2[k] = torch.nextafter(w2[k], torch.tensor(100.0, device=DEV))
    assert not K.edge_symmetry_weighted(und, w2, n), "one weight one ulp off"
    assert not K.edge_symmetry_weighted(moved, w, n)


# ------------------------------------------------------------------------------------------------
# fill windows: the same builds with SGF_CSR_FILL_WINDOW_MB = 1 (past the 12-window cap) and 0 (one launch), in a child process
# ------------------------------------------------------------------------------------------------
def _window_builds(K, name):
    """The builds whose fill is windowed, each checked against the reference as it is made: plain (both orientations, both
    modes), weighted (both modes), a row shard and rotated.  -> {build: outputs on the host} of the medium graph."""
    ei, w = graph(name)
    n = G.GRAPHS[name].n
    cases = [(f"plain-{int(s)}-{m}", dict(by_source=s, mode=m)) for s in (False, True) for m in (0, 1)
             if not (name == "large" and m == 1)]
    cases += [(f"weighted-{m}", dict(mode=m, w=w)) for m in (0, 1)]
    cases += [("shard", dict(rows=(n // 5, n - n // 7))), ("rot", dict(col_rot=(n // 3, n + 1)))]
    saved = {}
    for key, kw in cases:
        want = ref_csr(ei, n, **kw)
        tot = ei.shape[1] + want["rowptr"].numel() - 1
        if "w" in kw:
            got = K.csr_build_weighted(ei, w, n, False, kw["mode"])
            check_weighted(got, want, w, tot, f"{name} {key}")
        else:
            got = K.csr_build(ei, n, kw.get("by_source", False), kw.get("mode", 0), rows=kw.get("rows"), col_rot=kw.get("col_rot"))
            check_csr(got, want, tot, f"{name} {key}")
        if name == "medium":
            saved[key] = [t.cpu() if t is not None else None for t in got]
        del got, want
    return saved


def window_child(out_dir):
    """Run in a child process with SGF_CSR_FILL_WINDOW_MB set: every windowed build against the reference; the medium graph's
    outputs are saved for the parent to compare with its default-window builds."""
    from sgformer_b200 import kernels as K
    for name in ("medium", "large"):
        saved = _window_builds(K, name)
        if name == "medium":
            torch.save(saved, os.path.join(out_dir, "medium.pt"))
        print(f"{name}: the windowed builds equal the reference")
    print(f"child peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


@pytest.mark.parametrize("window_mb", [1, 0])
def test_fill_windows_in_a_child_process(K, window_mb):
    spec = G.GRAPHS["medium"]
    nnz = spec.nnz()
    if window_mb == 1:
        assert G.fill_windows(nnz, spec.n, 4, 1)["windows"] == G.MAX_FILL_WINDOWS
    torch.cuda.empty_cache()
    with tempfile.TemporaryDirectory() as d:
        env = dict(os.environ, SGF_CSR_FILL_WINDOW_MB=str(window_mb))
        code = (f"import sys; sys.path[:0] = [{TESTS!r}, {ROOT!r}]; import test_gpu_csr_sweep as T; T.window_child({d!r})")
        r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0, f"child exit {r.returncode}\n{r.stdout[-3000:]}\n{r.stderr[-6000:]}"
        print(r.stdout)
        saved = torch.load(os.path.join(d, "medium.pt"))
    builds = _window_builds(K, "medium")
    assert builds.keys() == saved.keys()
    for key, got in builds.items():
        for a, b in zip(got, saved[key]):
            assert (a is None) == (b is None) and (a is None or torch.equal(a, b)), f"{key}: windowed build differs"


# ------------------------------------------------------------------------------------------------
# out-of-range node ids
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("row", [0, 1])
@pytest.mark.parametrize("bad", ["-1", "n"])
def test_out_of_range_ids_are_refused(K, row, bad):
    ei, w = graph("small")
    n = G.GRAPHS["small"].n
    e = ei.clone()
    e[row, e.shape[1] // 2] = -1 if bad == "-1" else n
    msg = (r"\[-1, \d+\]" if bad == "-1" else rf"\[\d+, {n}\]") + rf", outside \[0, n={n}\)"
    for by_source in (False, True):
        for mode in (0, 1):
            with pytest.raises(ValueError, match=msg):
                K.csr_build(e, n, by_source, mode)
            with pytest.raises(ValueError, match=msg):
                K.csr_build_weighted(e, w, n, by_source, mode)
    with pytest.raises(ValueError, match=msg):
        K.csr_build(e, n, rows=(0, n // 2))
    with pytest.raises(ValueError, match=msg):
        K.to_undirected(e, n)
    K.csr_build(ei, n)          # the unmodified list still builds


# ------------------------------------------------------------------------------------------------
def test_peak_device_memory(mem0):
    """The module keeps its device memory under 12 GiB above what it found (the GPU is shared)."""
    _CACHE.clear()
    peak = torch.cuda.max_memory_allocated() - mem0
    p = torch.cuda.get_device_properties(torch.cuda.current_device())
    print(f"test_gpu_csr_sweep: peak device memory {peak / 2 ** 30:.2f} GiB above the module's start, {p.name}, "
          f"{p.multi_processor_count} SMs")
    assert peak < PEAK_BUDGET
