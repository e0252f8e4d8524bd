"""Kernel-level parity on the H100: every C-ABI kernel against the oracle / its documented semantics.

Integer work (CSR build, subgraph) is compared bit-exactly with the numpy / C oracle; floating-point kernels against
fp64 numpy (SpMM, attention contractions) or the torch-CPU statement of the kernel contract (tests/kernel_emu.py,
itself pinned to the reference through tests/test_schedule_emulated.py)."""
import ctypes
import os

import numpy as np
import pytest
import torch

import kernel_emu as emu
from oracle import np_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def K():
    from sgformer_b200 import kernels
    return kernels


def rand_graph(n, e, seed, directed=False, isolated=0, dup=0, hub=0):
    g = torch.Generator().manual_seed(seed)
    hi = max(n - isolated, 1)
    src = torch.randint(0, hi, (e,), generator=g)
    dst = torch.randint(0, hi, (e,), generator=g)
    if hub:
        dst[:hub] = 3 % hi  # one node with a huge in-degree
    ei = torch.stack([src, dst])
    if not directed:
        ei = torch.cat([ei, ei.flip(0)], 1)
    if dup:
        ei = torch.cat([ei, ei[:, :dup]], 1)
    return ei[:, torch.randperm(ei.shape[1], generator=g)].contiguous()


def _close(a, b, rtol, atol, what):
    a = torch.as_tensor(a).detach().cpu().double()
    b = torch.as_tensor(b).detach().cpu().double()
    assert a.shape == b.shape, f"{what}: shape {tuple(a.shape)} vs {tuple(b.shape)}"
    err = (a - b).abs().max().item() if a.numel() else 0.0
    ref = b.abs().max().item() if b.numel() else 0.0
    assert np.isfinite(err) and err <= atol + rtol * ref, f"{what}: max err {err:.3e} (ref max {ref:.3e})"


def _close_gated(a, b, rtol, atol, what, max_bad=3e-5):
    """Like _close but tolerates a vanishing fraction of outliers: a ReLU gate whose pre-activation is ~0 (exact ties
    of bf16-quantised inputs) may flip between two correct fp32 evaluation orders and change single elements."""
    a = torch.as_tensor(a).detach().cpu().double()
    b = torch.as_tensor(b).detach().cpu().double()
    assert a.shape == b.shape, f"{what}: shape {tuple(a.shape)} vs {tuple(b.shape)}"
    bad = ((a - b).abs() > atol + rtol * b.abs().max()).double().mean().item()
    assert bad <= max_bad, f"{what}: {bad:.2e} of the elements differ"


# ------------------------------------------------------------------------------------------------
# K5 / K9: integers, bit-exact
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [
    dict(n=1, e=0), dict(n=7, e=0), dict(n=50, e=200), dict(n=300, e=3000, directed=True, isolated=11, dup=57),
    dict(n=2000, e=60000), dict(n=500, e=9000, directed=True, hub=3000), dict(n=1000, e=300, directed=True, hub=280),
    dict(n=40000, e=400000), dict(n=1500, e=70000, directed=True, dup=5000),
])
@pytest.mark.parametrize("by_source", [False, True])
def test_csr_build_bit_exact(K, case, by_source):
    c = dict(case)
    n, e = c.pop("n"), c.pop("e")
    ei = rand_graph(n, e, 1, **c) if e else torch.zeros((2, 0), dtype=torch.int64)
    rowptr, col, dinv = K.csr_build(ei.to(DEV), n, by_source, 0, True)
    eio = ei.flip(0) if by_source else ei
    rp, cl, dv = np_ref.gcn_csr(eio.numpy(), n)
    assert np.array_equal(rowptr.cpu().numpy(), rp), "rowptr differs"
    assert np.array_equal(col.cpu().numpy(), cl), "col differs"
    if not by_source:
        assert np.array_equal(dinv.cpu().numpy(), dv), "dinv differs (bitwise)"


def test_edge_symmetry(K):
    """sgf_edge_symmetry: multiset equality of the edge list and its transpose (decides whether the backward SpMM reuses the CSR)."""
    n = 3000
    und = rand_graph(n, 40000, 3)
    assert K.edge_symmetry(und.to(DEV), n)
    perm = torch.randperm(und.shape[1], generator=torch.Generator().manual_seed(0))
    assert K.edge_symmetry(und[:, perm].contiguous().to(DEV), n), "order must not matter"
    d = rand_graph(n, 40000, 3, directed=True)
    assert not K.edge_symmetry(d.to(DEV), n)
    k = int((und[0] != und[1]).nonzero()[0])
    one_more = torch.cat([und, und[:, k:k + 1]], 1)     # (r,c) twice, (c,r) once: same SET, different multiset
    assert not K.edge_symmetry(one_more.to(DEV), n)
    loops = torch.cat([und, torch.arange(10).repeat(2, 1)], 1)
    assert K.edge_symmetry(loops.to(DEV), n)
    assert K.edge_symmetry(torch.zeros((2, 0), dtype=torch.int64, device=DEV), n)


def test_csr_build_matches_c_oracle(K):
    """The C restatement (oracle/csr_ref.c, built by __graft_entry__.build) against the CUDA build."""
    so = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_build", "libcsr_ref.so")
    if not os.path.exists(so):
        pytest.skip("oracle/_build/libcsr_ref.so not built")
    lib = ctypes.CDLL(so)
    n = 777
    ei = rand_graph(n, 5000, 9, directed=True, dup=100, isolated=5)
    nnz = ei.shape[1]
    rp = np.zeros(n + 1, dtype=np.int64)
    cl = np.zeros(nnz, dtype=np.int32)
    ein = np.ascontiguousarray(ei.numpy())
    rc = lib.sgf_oracle_csr_build(ein.ctypes.data_as(ctypes.c_void_p), ctypes.c_int64(nnz), ctypes.c_int64(n), 0,
                                  rp.ctypes.data_as(ctypes.c_void_p), cl.ctypes.data_as(ctypes.c_void_p), None)
    assert rc == 0
    rowptr, col, _ = K.csr_build(ei.to(DEV), n)
    assert np.array_equal(rowptr.cpu().numpy(), rp) and np.array_equal(col.cpu().numpy(), cl)


def test_csr_build_pyg_self_loops(K):
    n = 400
    ei = rand_graph(n, 3000, 4, directed=True, dup=30)
    ei[1, :20] = ei[0, :20]  # some explicit self loops
    rowptr, col, dinv = K.csr_build(ei.to(DEV), n, False, 1, True)
    rp, cl, dv = emu.csr_build(ei, n, False, 1, True)
    assert torch.equal(rowptr.cpu(), rp) and torch.equal(col.cpu(), cl)
    _close(dinv, dv, 1e-7, 0, "dinv")


def test_subgraph_bit_exact(K):
    n = 5000
    ei = rand_graph(n, 40000, 2)
    g = torch.Generator().manual_seed(0)
    subset = torch.randperm(n, generator=g)[:1500]
    out = K.subgraph(ei.to(DEV), n, subset.to(DEV))
    mask = torch.zeros(n, dtype=torch.bool)
    mask[subset] = True
    keep = mask[ei[0]] & mask[ei[1]]
    relabel = torch.zeros(n, dtype=torch.long)
    relabel[subset] = torch.arange(subset.numel())
    assert torch.equal(out.cpu(), relabel[ei[:, keep]])
    empty = K.subgraph(ei.to(DEV), n, torch.zeros(0, dtype=torch.long, device=DEV))
    assert empty.shape == (2, 0)


@pytest.mark.parametrize("case", [dict(n=300, e=2000), dict(n=5000, e=60000, dup=500), dict(n=50, e=0), dict(n=7, e=40, dup=10),
                                  dict(n=20000, e=150000, hub=5000), dict(n=1000, e=5000, isolated=300, directed=True)])
def test_graph_preprocessing_bit_exact(K, case):
    """K10: to_undirected / remove_self_loops / add_self_loops == torch_geometric semantics (oracle/np_ref.py), bit for bit,
    including duplicates, self loops, isolated nodes, a hub row beyond the shared-memory sort tier and the empty graph."""
    from oracle import np_ref
    c = dict(case)
    n, e = c.pop("n"), c.pop("e")
    ei = rand_graph(n, e, 5, directed=True, **{k: v for k, v in c.items() if k != "directed"}) if e else torch.zeros((2, 0), dtype=torch.int64)
    if e:
        ei[1, : max(1, e // 50)] = ei[0, : max(1, e // 50)]      # explicit self loops
    d = ei.to(DEV)
    und = K.to_undirected(d, n)
    assert torch.equal(und.cpu(), torch.from_numpy(np_ref.to_undirected(ei.numpy(), n)))
    nsl = K.remove_self_loops(d)
    assert torch.equal(nsl.cpu(), torch.from_numpy(np_ref.remove_self_loops(ei.numpy())))
    asl = K.add_self_loops(d, n)
    assert torch.equal(asl.cpu(), torch.from_numpy(np_ref.add_self_loops(ei.numpy(), n)))
    # the reference's sequence (large/main.py:75-79) through the PyG-shaped wrappers
    from sgformer_b200 import pyg_utils as U
    x = U.to_undirected(d, num_nodes=n) if e else d
    x, _ = U.remove_self_loops(x)
    x, _ = U.add_self_loops(x, num_nodes=n)
    ref = np_ref.add_self_loops(np_ref.remove_self_loops(np_ref.to_undirected(ei.numpy(), n) if e else ei.numpy()), n)
    assert torch.equal(x.cpu(), torch.from_numpy(ref))


@pytest.mark.parametrize("rows,c,m", [(1000, 47, 300), (5000, 2, 5000), (257, 172, 100), (64, 7, 0)])
def test_eval_acc_matches_reference_semantics(K, rows, c, m):
    """K11 == eval_acc of the reference (oracle/np_ref.eval_acc restates large/data_utils.py:210-220) and the NLL of
    log_softmax on the split; ties resolve to the first maximum."""
    from oracle import np_ref
    g = torch.Generator().manual_seed(rows + c)
    logits = torch.randn(rows, c, generator=g)
    logits[::7, 1 % c] = logits[::7].max(dim=1).values        # exact ties with the row maximum (first index must win)
    labels = torch.randint(0, c, (rows, 1), generator=g)
    idx = torch.randperm(rows, generator=g)[:m]
    padded = torch.zeros(rows, c + 3)
    padded[:, :c] = logits
    for lg in (logits.to(DEV), padded.to(DEV)[:, :c]):           # contiguous and strided logits
        acc, loss = K.eval_acc(lg, labels.to(DEV), idx.to(DEV), want_loss=True)
        if m == 0:
            assert acc != acc and loss is None
            continue
        assert acc == np_ref.eval_acc(labels[idx].numpy(), logits[idx].numpy())
        ref_loss = torch.nn.functional.nll_loss(torch.log_softmax(logits.double(), 1)[idx], labels.squeeze(1)[idx]).item()
        assert abs(loss - ref_loss) <= 1e-5 * max(1.0, abs(ref_loss))
    acc_all, _ = K.eval_acc(logits.to(DEV), labels.to(DEV))
    assert acc_all == np_ref.eval_acc(labels.numpy(), logits.numpy())


def test_eval_and_graph_prep_match_reference_fixtures(K):
    """K10 / K11 against tests/golden/{graph_prep,evaluate}.pt (the reference's own evaluate()/eval_acc; PyG-semantics preprocessing)."""
    from fixture_checks import check_evaluate_fixture, check_graph_prep_fixture
    dev = lambda t: t.to(DEV)      # noqa: E731
    check_evaluate_fixture(lambda lg, lb, idx, want: K.eval_acc(lg, lb, idx, want_loss=want), to_dev=dev)
    check_graph_prep_fixture(K.to_undirected, K.remove_self_loops, K.add_self_loops, to_dev=dev)


def test_csr_subset_matches_subgraph_then_build(K):
    """K9 on the CSR == PyG-semantics subgraph (sgf_subgraph) followed by a CSR build, bit-exactly; node_map is restored."""
    from sgformer_b200.graph import Graph
    from sgformer_b200.synth import make_graph
    n = 20000
    ei = make_graph(n, 150000, seed=2).to(DEV)
    full = Graph(ei, n)
    g = torch.Generator().manual_seed(1)
    for b in (1, 777, 5000):
        idx = torch.randperm(n, generator=g)[:b].to(DEV)
        sub = full.subset(idx)
        ei_sub = K.subgraph(ei, n, idx)
        rp, cl, dv = K.csr_build(ei_sub, b)
        assert torch.equal(sub.rowptr, rp) and torch.equal(sub.col, cl) and torch.equal(sub.dinv, dv)
        assert int((full._node_map != -1).sum()) == 0
    x = torch.randn(n, 24, device=DEV)
    idx = torch.randperm(n, generator=g)[:300].to(DEV)
    a, b_ = K.pack_operand(x, row_index=idx), K.pack_operand(x[idx].contiguous())
    assert torch.equal(a.data, b_.data)


def test_csr_subset_capacity_is_never_overrun(K):
    """A too-small nnz capacity truncates the batch structure instead of writing past out_col, and is reported."""
    from sgformer_b200.graph import Graph
    from sgformer_b200.minibatch import RandomPartitionSampler
    from sgformer_b200.synth import make_graph
    n = 6000
    ei = make_graph(n, 60000, seed=5).to(DEV)
    full = Graph(ei, n)
    idx = torch.randperm(n, generator=torch.Generator().manual_seed(0))[:3000].to(DEV)
    exact = full.subset(idx)
    nnz = int(exact.rowptr[-1])
    assert int(exact.nnz_needed) == nnz
    cap = nnz // 3
    node_map = full._node_map
    rp, cl, dv, needed = K.csr_subset(full.rowptr, full.col, n, idx, node_map, cap + 64)    # buffer has 64 guard entries
    guard = torch.full((64,), -7, dtype=torch.int32, device=DEV)
    cl[cap:] = guard
    rp, cl2, dv, needed = K.csr_subset(full.rowptr, full.col, n, idx, node_map, cap)
    assert int(needed) == nnz and int(rp[-1]) == cap and int(rp.max()) == cap
    assert bool((rp[1:] >= rp[:-1]).all())
    first = int((exact.rowptr <= cap).sum()) - 1             # rows that fit entirely are untouched
    assert torch.equal(rp[:first + 1], exact.rowptr[:first + 1])
    assert torch.equal(cl2[:int(rp[first])], exact.col[:int(rp[first])])
    assert int((node_map != -1).sum()) == 0
    sampler = RandomPartitionSampler(full, torch.randn(n, 8, device=DEV), None, 3000, capacity=cap)
    with pytest.raises(RuntimeError, match="capacity"):
        for _ in sampler:
            pass


# ------------------------------------------------------------------------------------------------
# K6/K7: SpMM
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,h", [(torch.float32, 4), (torch.float32, 64), (torch.float32, 100), (torch.float32, 256),
                                     (torch.bfloat16, 8), (torch.bfloat16, 64), (torch.bfloat16, 96),
                                     (torch.bfloat16, 128), (torch.bfloat16, 256), (torch.bfloat16, 512)])
def test_spmm_matches_scipy(K, dtype, h):
    n = 3000
    ei = rand_graph(n, 40000, 5, directed=True, dup=200, isolated=17, hub=700)
    rowptr, col, dinv = K.csr_build(ei.to(DEV), n)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(n, h, generator=g)
    xd = x.to(DEV).to(dtype)
    xs = K.axpby(xd, None, 1.0, 0.0, row_scale=dinv)
    y = K.spmm(rowptr, col, dinv, xs)
    ref = np_ref.spmm_fp64(ei.numpy(), n, xd.float().cpu().numpy())
    tol = 1e-5 if dtype == torch.float32 else 1.5e-2
    _close(y.float(), ref, tol, tol * 1e-2, f"spmm {dtype} h={h}")
    # linearity (size-independent property): A(x + 2x') = Ax + 2Ax'
    if dtype == torch.float32:
        x2 = torch.randn(n, h, generator=g).to(DEV)
        lhs = K.spmm(rowptr, col, None, K.axpby(xd, x2, 1.0, 2.0))
        rhs = K.axpby(K.spmm(rowptr, col, None, xd), K.spmm(rowptr, col, None, x2), 1.0, 2.0)
        _close(lhs, rhs, 1e-5, 1e-5, "spmm linearity")


@pytest.mark.parametrize("dtype,h", [(torch.float32, 64), (torch.bfloat16, 256), (torch.bfloat16, 64)])
def test_spmm_hub_rows_segmented_path(K, dtype, h):
    """Power-law graphs: rows longer than kernels.HEAVY_ROW go through the segmented (deterministic) path."""
    from sgformer_b200.synth import make_rmat_graph
    n = 30000
    ei = make_rmat_graph(n, 600000, seed=1)
    rowptr, col, dinv = K.csr_build(ei.to(DEV), n)
    plan = K.heavy_rows(rowptr)
    lens = (rowptr[1:] - rowptr[:-1])
    assert plan is not None and plan.rows.numel() == int((lens > K.HEAVY_ROW).sum()) and int(lens.max()) > 4 * K.HEAVY_ROW
    assert int(plan.seg_len.sum()) == int(lens[plan.rows].sum())
    x = torch.randn(n, h, generator=torch.Generator().manual_seed(3)).to(DEV).to(dtype)
    xs = K.axpby(x, None, 1.0, 0.0, row_scale=dinv)
    y = K.spmm(rowptr, col, dinv, xs, heavy=plan)
    ref = np_ref.spmm_fp64(ei.numpy(), n, x.float().cpu().numpy())
    tol = 1e-5 if dtype == torch.float32 else 1.5e-2
    _close(y.float(), ref, tol, tol * 1e-2, "spmm with hub rows")
    y2 = K.spmm(rowptr, col, dinv, xs, heavy=plan)
    assert torch.equal(y, y2), "segmented path must be deterministic"
    y_plain = K.spmm(rowptr, col, dinv, xs)      # single-warp path on the same rows
    _close(y.float(), y_plain.float(), tol, tol * 1e-2, "segmented vs plain")


# ------------------------------------------------------------------------------------------------
# row kernels vs the kernel contract
# ------------------------------------------------------------------------------------------------
def _acts(n, h, dtype, seed, k=1):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, h, generator=g).to(dtype) for _ in range(k)]


@pytest.mark.parametrize("dtype,h,n", [(torch.float32, 32, 1000), (torch.bfloat16, 64, 777), (torch.bfloat16, 256, 2500),
                                       (torch.float32, 256, 300), (torch.bfloat16, 16, 5), (torch.bfloat16, 96, 1234)])
def test_row_kernels(K, dtype, h, n):
    tol = 2e-5 if dtype == torch.float32 else 2e-2
    x, r, dy, z, res, mix = _acts(n, h, dtype, 3, 6)
    g = torch.Generator().manual_seed(8)
    gamma, beta, zb = 1 + 0.1 * torch.randn(h, generator=g), 0.1 * torch.randn(h, generator=g), 0.2 * torch.randn(h, generator=g)
    w = torch.rand(n, generator=g)
    D = lambda t: None if t is None else t.to(DEV)

    s, q = K.colstats(D(x), D(w))
    se, qe = emu.colstats(x, w)
    _close(s, se, tol, tol * n ** 0.5, "colstats sum")
    _close(q, qe, tol, tol, "colstats sumsq")

    for use_ln, use_relu, rr in [(True, True, r), (True, False, None), (False, True, r)]:
        y, st = K.ln_fwd(D(x), D(rr), 0.7, 0.3, D(gamma), D(beta), use_ln, use_relu, 0.0, 1)
        ye, ste = emu.ln_fwd(x, rr, 0.7, 0.3, gamma, beta, use_ln, use_relu, 0.0, 1)
        _close(y.float(), ye.float(), tol, tol, f"ln_fwd ln={use_ln}")
        if use_ln:
            _close(st, ste, 1e-4, 1e-5, "ln stats")
        dg, db = torch.zeros(h, device=DEV), torch.zeros(h, device=DEV)
        dge, dbe = torch.zeros(h), torch.zeros(h)
        dx, dr = K.ln_bwd(D(dy), D(x), D(rr), 0.7, 0.3, D(gamma), D(beta), st, use_ln, use_relu, 0.0, 1, 0.5, rr is not None, dg, db)
        dxe, dre = emu.ln_bwd(dy, x, rr, 0.7, 0.3, gamma, beta, ste, use_ln, use_relu, 0.0, 1, 0.5, rr is not None, dge, dbe)
        _close_gated(dx.float(), dxe.float(), tol, tol, "ln_bwd dx")
        if rr is not None:
            _close_gated(dr.float(), dre.float(), tol, tol, "ln_bwd dr")
        if use_ln:
            _close(dg, dge, tol, tol * n ** 0.5, "ln dgamma")
            _close(db, dbe, tol, tol * n ** 0.5, "ln dbeta")

    rs = torch.rand(n, generator=g) + 0.5
    for use_bn, use_relu, training in [(True, True, True), (True, False, False), (False, True, True)]:
        rm, rv = 0.1 * torch.randn(h, generator=g), 1 + 0.2 * torch.rand(h, generator=g)
        rmd, rvd = D(rm.clone()), D(rv.clone())
        if use_bn and training:
            s, q = K.colstats(D(z))
            mean, rstd = K.bn_finalize(s, q, n, h, D(zb), rmd, rvd, DEV)
            se, qe = emu.colstats(z)
            me, re_ = emu.bn_finalize(se, qe, n, h, zb, rm, rv, "cpu")
            _close(rmd, rm, 1e-4, 1e-5, "running mean")
            _close(rvd, rv, 1e-3, 1e-4, "running var")
        elif use_bn:
            mean, rstd = K.bn_finalize(None, None, n, h, None, rmd, rvd, DEV)
            me, re_ = emu.bn_finalize(None, None, n, h, None, rm, rv, "cpu")
        else:
            mean = rstd = me = re_ = None
        if use_bn:
            _close(mean, me, 1e-3, 1e-4, "bn mean")
            _close(rstd, re_, 2e-3, 1e-4, "bn rstd")
            me, re_ = mean.cpu(), rstd.cpu()  # identical statistics downstream
        y, ys = K.bn_fwd(D(z), D(res), D(mix), mean, rstd, D(gamma), D(beta), D(zb), use_bn, use_relu, 0.0, 1, 0.6, D(rs), True, True)
        ye, yse = emu.bn_fwd(z, res, mix, me, re_, gamma, beta, zb, use_bn, use_relu, 0.0, 1, 0.6, rs, True, True)
        _close(y.float(), ye.float(), tol, tol, f"bn_fwd y bn={use_bn}")
        _close(ys.float(), yse.float(), tol, tol, "bn_fwd y_scaled")
        dres = D(res.clone())
        dz, sums, cs = K.bn_bwd(D(dy), D(x), D(rs), D(z), mean, rstd, D(gamma), D(beta), D(zb), use_bn, use_relu, training, 0.0, 1,
                                0.8, dres=dres, dres_accumulate=True, want_dz_colsum=True, out_row_scale=D(rs))
        drese = res.clone()
        dze, sumse, cse = emu.bn_bwd(dy, x, rs, z, me, re_, gamma, beta, zb, use_bn, use_relu, training, 0.0, 1, 0.8, dres=drese,
                                     dres_accumulate=True, want_dz_colsum=True, out_row_scale=rs)
        _close_gated(dz.float(), dze.float(), tol, tol, f"bn_bwd dz bn={use_bn} train={training}")
        _close(dres.float(), drese.float(), tol, tol, "bn_bwd dres")
        _close(cs, cse, tol, tol * n ** 0.5, "bn_bwd dz colsum")
        if sums is not None:
            _close(sums, sumse, tol, tol * n ** 0.5, "bn_bwd sums")

    out = K.axpby(D(x), D(r), 0.25, -1.5, out_dtype=torch.float32, row_scale=D(rs))
    _close(out, emu.axpby(x, r, 0.25, -1.5, torch.float32, rs), tol, tol, "axpby")
    if h % 4 == 0:
        _close(K.head_mean(D(x), 4, h // 4).float(), emu.head_mean(x, 4, h // 4).float(), tol, tol, "head_mean")
    den = torch.rand(n, generator=g) + 1.0
    gnum, gden = K.attn_bwd_prep(D(dy), D(x), D(den), 0.5)
    gne, gde = emu.attn_bwd_prep(dy, x, den, 0.5)
    _close(gnum.float(), gne.float(), tol, tol, "attn_bwd_prep gnum")
    _close(gden, gde, tol, tol, "attn_bwd_prep gden")


def test_dropout_statistics_and_consistency(K):
    """Dropout cannot match torch's Philox stream (SURVEY §7.7): check rate, scaling and fwd/bwd mask agreement."""
    n, h, p = 4096, 128, 0.3
    x = torch.ones(n, h, device=DEV)
    y, _ = K.ln_fwd(x, None, 1.0, 0.0, None, None, False, False, p, 1234)
    kept = (y > 0).float().mean().item()
    assert abs(kept - (1 - p)) < 0.01
    _close(y[y > 0], torch.full_like(y[y > 0], 1 / (1 - p)), 1e-4, 0, "dropout scale")
    dx, _ = K.ln_bwd(x, x, None, 1.0, 0.0, None, None, None, False, False, p, 1234, 1.0, False, None, None)
    assert torch.equal(dx > 0, y > 0), "forward / backward masks differ"
    y2, _ = K.ln_fwd(x, None, 1.0, 0.0, None, None, False, False, p, 1235)
    assert not torch.equal(y2 > 0, y > 0)
    z = torch.ones(n, h, device=DEV)
    yb, _ = K.bn_fwd(z, None, None, None, None, None, None, None, False, False, p, 77, 1.0, None, True, False)
    dz, _, _ = K.bn_bwd(z, None, None, z, None, None, None, None, None, False, False, True, p, 77, 1.0)
    assert abs((yb > 0).float().mean().item() - (1 - p)) < 0.01 and torch.equal(dz > 0, yb > 0)


def test_dropout_epoch_under_graph_replay(K):
    """A captured step freezes the host seed; the device epoch (sgf_advance_dropout_epoch inside the graph) must give every
    replay fresh masks while the backward of the same replay recomputes the forward's mask (ADVICE r1: dropout seed)."""
    n, h, p = 2048, 64, 0.4
    x = torch.ones(n, h, device=DEV)
    K.dropout_epoch()                       # registers the word
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        K.advance_dropout_epoch()           # warm-up outside the capture
        K.ln_fwd(x, None, 1.0, 0.0, None, None, False, False, p, 99)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        K.advance_dropout_epoch()
        y, _ = K.ln_fwd(x, None, 1.0, 0.0, None, None, False, False, p, 99)
        dx, _ = K.ln_bwd(x, x, None, 1.0, 0.0, None, None, None, False, False, p, 99, 1.0, False, None, None)
    masks = []
    for _ in range(3):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(dx > 0, y > 0), "forward / backward masks of one replay differ"
        assert abs((y > 0).float().mean().item() - (1 - p)) < 0.02
        masks.append((y > 0).clone())
    assert not torch.equal(masks[0], masks[1]) and not torch.equal(masks[1], masks[2])
    assert abs((masks[0] & masks[1]).float().mean().item() - (1 - p) ** 2) < 0.02, "masks of consecutive replays are correlated"


def test_softmax_nll_matches_torch(K):
    from sgformer_b200.loss import nll_loss_from_logits
    g = torch.Generator().manual_seed(4)
    for n, c in [(1000, 47), (333, 2), (5000, 172), (64, 7)]:
        x = (torch.randn(n, c, generator=g) * 3).to(DEV).requires_grad_(True)
        y = torch.randint(0, c, (n,), generator=g).to(DEV)
        mask = (torch.rand(n, generator=g) < 0.5).to(DEV)
        for m in (None, mask):
            xr = x.detach().clone().requires_grad_(True)
            ref = torch.nn.functional.nll_loss(torch.log_softmax(xr if m is None else xr[m], 1), y if m is None else y[m])
            ref.backward()
            x.grad = None
            loss = nll_loss_from_logits(x, y, m)
            (loss * 2.0).backward()
            _close(loss, ref, 1e-5, 1e-6, f"loss n={n} c={c}")
            _close(x.grad, 2.0 * xr.grad, 1e-4, 1e-7, "dlogits")


def test_pack_operand(K):
    g = torch.Generator().manual_seed(2)
    src = torch.randn(130, 47, generator=g)
    for transpose in (False, True):
        for planes in (1, 3):
            cs = torch.zeros(47, device=DEV)
            op = K.pack_operand(src.to(DEV), transpose, planes, colsum=cs)
            want = src.t() if transpose else src
            data = op.data.float().cpu()
            rec = sum(data[:, i * op.kp:i * op.kp + op.k] for i in range(planes))
            _close(rec, want, 1e-6 if planes == 3 else 8e-3, 1e-7 if planes == 3 else 1e-3, f"pack t={transpose} p={planes}")
            assert torch.count_nonzero(data[:, op.k:op.kp]) == 0, "K padding must be zero"
            _close(cs, src.sum(0), 1e-5, 1e-5, "pack colsum")


# ------------------------------------------------------------------------------------------------
# wgmma GEMMs
# ------------------------------------------------------------------------------------------------
def _ops(K, a, b, planes):
    """CUDA + emulated operands for fp32 sources a [rows,k], b [n,k]."""
    return (K.pack_operand(a.to(DEV), False, planes), K.pack_operand(b.to(DEV), False, planes),
            emu.pack_operand(a, False, planes), emu.pack_operand(b, False, planes))


@pytest.mark.parametrize("rows,k,n_out", [(1, 16, 16), (127, 64, 32), (128, 100, 47), (1000, 256, 256), (300, 256, 768),
                                          (5000, 128, 64), (129, 1433, 64), (2000, 64, 172)])
@pytest.mark.parametrize("planes", [1, 3])
def test_gemm_nt_affine(K, rows, k, n_out, planes):
    g = torch.Generator().manual_seed(rows + k)
    a, b = torch.randn(rows, k, generator=g), torch.randn(n_out, k, generator=g) / k ** 0.5
    bias, aux = torch.randn(n_out, generator=g), torch.randn(rows, n_out, generator=g)
    rs, r1r, r1c = torch.rand(rows, generator=g), torch.randn(rows, generator=g), torch.randn(n_out, generator=g)
    ad, bd = torch.tensor([0.5]), torch.tensor([-2.0])
    A, B, Ae, Be = _ops(K, a, b, planes)
    tol = 2e-5 if planes == 3 else 1e-2
    for out_dtype in (torch.float32, torch.bfloat16):
        if out_dtype == torch.bfloat16 and n_out % 8:
            continue
        out = K.alloc_act(rows, n_out, out_dtype, DEV)
        K.gemm_nt([A], [B], [(0, 0, 0, 0, k)], n_out, out)
        oe = emu.gemm_nt([Ae], [Be], [(0, 0, 0, 0, k)], n_out, torch.zeros(rows, n_out))
        t = tol if out_dtype == torch.float32 else max(tol, 1e-2)
        _close(out.float(), oe, t, t, f"plain {out_dtype}")
    out = torch.full((rows, n_out), 0.25, device=DEV)
    K.gemm_nt([A], [B], [(0, 0, 0, 0, k)], n_out, out, bias=bias.to(DEV), aux=aux.to(DEV), row_scale=rs.to(DEV), alpha=1.5,
              beta=0.5, alpha_dev=ad.to(DEV), beta_dev=bd.to(DEV), relu=True, accumulate=True, r1_row=r1r.to(DEV), r1_col=r1c.to(DEV))
    oe = emu.gemm_nt([Ae], [Be], [(0, 0, 0, 0, k)], n_out, torch.full((rows, n_out), 0.25), bias=bias, aux=aux, row_scale=rs,
                     alpha=1.5, beta=0.5, alpha_dev=ad, beta_dev=bd, relu=True, accumulate=True, r1_row=r1r, r1_col=r1c)
    _close(out, oe, tol, tol, "full epilogue")


@pytest.mark.parametrize("rows,k,n_out,dtype", [(1000, 64, 64, torch.bfloat16), (130, 256, 256, torch.bfloat16),
                                                 (4097, 256, 768, torch.bfloat16), (777, 128, 96, torch.float32),
                                                 (3000, 256, 256, torch.float32), (5, 32, 16, torch.bfloat16)])
def test_gemm_nt_fused_column_stats(K, monkeypatch, rows, k, n_out, dtype):
    """Column sums / sums of squares of the STORED output from the GEMM epilogue == a colstats pass over the output."""
    g = torch.Generator().manual_seed(rows)
    a, b = torch.randn(rows, k, generator=g), torch.randn(n_out, k, generator=g) / k ** 0.5
    bias = torch.randn(n_out, generator=g)
    planes = 1 if dtype == torch.bfloat16 else 3
    A, B = K.pack_operand(a.to(DEV), False, planes), K.pack_operand(b.to(DEV), False, planes)
    out = K.alloc_act(rows, n_out, dtype, DEV)
    cs, cq = torch.zeros(n_out, device=DEV), torch.zeros(n_out, device=DEV)
    monkeypatch.setattr(K, "FUSE_GEMM_STATS", True)     # the fused path is opt-in (see kernels.FUSE_GEMM_STATS)
    K.gemm_nt([A], [B], [(0, 0, 0, 0, k)], n_out, out, bias=bias.to(DEV), col_sum=cs, col_sumsq=cq)
    s_ref, q_ref = K.colstats(out)
    _close(cs, s_ref, 1e-5, 1e-3, "fused column sums")
    _close(cq, q_ref, 1e-5, 1e-3, "fused column sums of squares")
    _close(cs, out.float().sum(0), 1e-4, 1e-2, "vs torch sum")


@pytest.mark.parametrize("rows,k,n_out", [(200_000, 64, 600), (160_001, 128, 256), (4100, 256, 768), (3000, 512, 256), (130, 256, 48)])
def test_gemm_nt_schedules_agree(K, rows, k, n_out):
    """Resident-B (weights parked in shared memory, row tiles visited in chunks with the n-block loop outside) and the
    streaming schedule issue the same MMAs per tile: outputs must be bit-identical, including the prefetched bf16 addend
    (aux / accumulate) of the epilogue.  200 k rows = more than 8 row tiles per CTA, i.e. several chunks per CTA."""
    g = torch.Generator().manual_seed(rows + n_out)
    a = torch.randn(rows, k, generator=g).to(DEV)
    b = (torch.randn(n_out, k, generator=g) / k ** 0.5).to(DEV)
    bias = torch.randn(n_out, generator=g).to(DEV)
    aux = torch.randn(rows, n_out, generator=g).to(DEV).to(torch.bfloat16)
    A, B = K.pack_operand(a, False, 1), K.pack_operand(b, False, 1)
    outs = {}
    for sched in (1, 2):
        o1 = K.alloc_act(rows, n_out, torch.bfloat16, DEV)
        K.gemm_nt([A], [B], [(0, 0, 0, 0, k)], n_out, o1, bias=bias, schedule=sched)
        o2 = K.alloc_act(rows, n_out, torch.bfloat16, DEV)
        K.gemm_nt([A], [B], [(0, 0, 0, 0, k)], n_out, o2, aux=aux, beta=0.5, alpha=2.0, schedule=sched)
        o3 = aux.clone()
        K.gemm_nt([A], [B], [(0, 0, 0, 0, k)], n_out, o3, accumulate=True, relu=True, schedule=sched)
        outs[sched] = (o1, o2, o3)
    for x, y, what in zip(outs[1], outs[2], ("bias", "aux", "accumulate")):
        assert torch.equal(x, y), f"schedules differ ({what}): max diff {(x.float() - y.float()).abs().max().item()}"
    ref = a.to(torch.bfloat16).float() @ b.to(torch.bfloat16).float().t()
    _close(outs[2][0].float(), ref + bias, 2e-2, 2e-2, "resident vs matmul")
    _close(outs[2][1].float(), 2.0 * ref + 0.5 * aux.float(), 3e-2, 2e-2, "resident aux vs matmul")
    _close(outs[2][2].float(), torch.relu(ref) + aux.float(), 2e-2, 2e-2, "resident accumulate vs matmul")


@pytest.mark.parametrize("planes", [1, 3])
@pytest.mark.parametrize("h", [16, 32, 64, 256])
def test_gemm_nt_concat_segments(K, planes, h):
    """[y || x0] . W^T as two K segments of one B source (GraphConvLayer use_init, large/ours.py:37-38)."""
    rows = 700
    g = torch.Generator().manual_seed(h)
    y, x0, w = torch.randn(rows, h, generator=g), torch.randn(rows, h, generator=g), torch.randn(h, 2 * h, generator=g) / h ** 0.5
    Y, W, Ye, We = _ops(K, y, w, planes)
    X0, X0e = K.pack_operand(x0.to(DEV), False, planes), emu.pack_operand(x0, False, planes)
    out = torch.empty(rows, h, device=DEV)
    pairs = [(0, 0, 0, 0, h), (1, 0, 0, h, h)]
    K.gemm_nt([Y, X0], [W], pairs, h, out)
    oe = emu.gemm_nt([Ye, X0e], [We], pairs, h, torch.zeros(rows, h))
    tol = 2e-5 if planes == 3 else 1e-2
    _close(out, oe, tol, tol, "concat segments")
    _close(out, torch.cat([y, x0], 1) @ w.t(), 5e-5 if planes == 3 else 2e-2, 5e-5 if planes == 3 else 2e-2, "vs fp32 matmul")


@pytest.mark.parametrize("rows,m,d", [(64, 16, 16), (1000, 64, 64), (777, 128, 128), (3000, 256, 256), (130, 32, 64)])
@pytest.mark.parametrize("planes", [1, 3])
def test_gemm_nt_attention_apply(K, rows, m, d, planes):
    g = torch.Generator().manual_seed(m)
    q, v = torch.randn(rows, m, generator=g), torch.randn(rows, d, generator=g)
    s_raw, z_raw = torch.randn(m, d, generator=g) * 3, torch.randn(m, generator=g) * 3
    nq2v, nk2v = torch.rand(m, generator=g) * rows, torch.rand(m, generator=g) * rows
    bmat, btail, scal = K.attn_prepare_fwd(s_raw.to(DEV), z_raw.to(DEV), nq2v.to(DEV), nk2v.to(DEV), planes)
    bme, bte, sce = emu.attn_prepare_fwd(s_raw, z_raw, nq2v, nk2v, planes)
    _close(scal[:3], sce[:3], 1e-5, 0, "scal")
    Q, Qe = K.pack_operand(q.to(DEV), False, planes), emu.pack_operand(q, False, planes)
    out, den = torch.empty(rows, d, device=DEV), torch.empty(rows, device=DEV)
    K.gemm_nt([Q], [bmat], [(0, 0, 0, 0, m)], d, out, epi=1, aux=v.to(DEV), tail=btail, nf=float(rows), den_out=den)
    oe, de = torch.zeros(rows, d), torch.zeros(rows)
    emu.gemm_nt([Qe], [bme], [(0, 0, 0, 0, m)], d, oe, epi=1, aux=v, tail=bte, nf=float(rows), den_out=de)
    tol = 2e-5 if planes == 3 else 2e-3
    _close(den, de, tol, tol, "den")
    _close(out, oe, tol, tol, "attention apply")


@pytest.mark.parametrize("rows,m,n", [(1, 16, 16), (63, 32, 47), (64, 64, 64), (1000, 128, 128), (20000, 256, 256),
                                      (5000, 256, 100), (4097, 47, 256), (300, 768, 256), (300, 64, 1433)])
@pytest.mark.parametrize("planes", [1, 3])
def test_gemm_tn(K, rows, m, n, planes):
    g = torch.Generator().manual_seed(rows + m)
    a, b = torch.randn(rows, m, generator=g), torch.randn(rows, n, generator=g)
    A, B = K.pack_operand(a.to(DEV), False, planes), K.pack_operand(b.to(DEV), False, planes)
    Ae, Be = emu.pack_operand(a, False, planes), emu.pack_operand(b, False, planes)
    tol = 2e-5 if planes == 3 else 1e-2
    out = torch.empty(m, n, device=DEV)
    K.gemm_tn(A, B, out)
    _close(out, emu.gemm_tn(Ae, Be, torch.zeros(m, n)), tol, tol * rows ** 0.5, "tn")
    outt = torch.full((n, m), 2.0, device=DEV)
    K.gemm_tn(A, B, outt, transpose_out=True, alpha=0.5, beta=-1.0, alpha_dev=torch.tensor([3.0], device=DEV))
    oe = emu.gemm_tn(Ae, Be, torch.full((n, m), 2.0), transpose_out=True, alpha=0.5, beta=-1.0, alpha_dev=torch.tensor([3.0]))
    _close(outt, oe, tol, tol * rows ** 0.5, "tn transposed/scaled")
    # determinism of the two-stage reduction
    out2 = torch.empty(m, n, device=DEV)
    K.gemm_tn(A, B, out2)
    assert torch.equal(out, out2), "gemm_tn must be run-to-run deterministic"


def test_gemm_on_bf16_views(K):
    """Operands that are column slices of a wider activation buffer (q/k/v inside the fused qkv buffer)."""
    g = torch.Generator().manual_seed(0)
    rows, h = 900, 64
    qkv = torch.randn(rows, 3 * h, generator=g).to(torch.bfloat16).to(DEV)
    k_, v_ = qkv[:, h:2 * h], qkv[:, 2 * h:]
    out = torch.empty(h, h, device=DEV)
    K.gemm_tn(K.as_operand(k_, 1), K.as_operand(v_, 1), out)
    _close(out, k_.float().t() @ v_.float(), 1e-3, 1e-2, "tn on views")
    w = torch.randn(h, h, generator=g)
    o2 = torch.empty(rows, h, device=DEV)
    K.gemm_nt([K.as_operand(k_, 1)], [K.pack_operand(w.to(DEV), False, 1)], [(0, 0, 0, 0, h)], h, o2)
    _close(o2, k_.float().cpu() @ w.bfloat16().float().t(), 1e-3, 1e-2, "nt on views")


def test_attention_partials_vs_fp64(K):
    """S' = k^T v, z', norms against the fp64 einsum oracle with *relative* tolerances (SURVEY.md §4)."""
    from sgformer_b200 import engine as E
    g = torch.Generator().manual_seed(5)
    for n, hd, m in [(16, 1, 8), (257, 2, 32), (4000, 1, 256)]:
        q, k, v = (torch.randn(n, hd * m, generator=g) for _ in range(3))
        ref = np_ref.attention_fp64(q.reshape(n, hd, m).numpy(), k.reshape(n, hd, m).numpy(), v.reshape(n, hd, m).numpy())
        tape = E.Tape()
        o = E.attention_forward(q.to(DEV), k.to(DEV), v.to(DEV), hd, E.FP32, tape)
        for i in range(hd):
            _close(tape["s"][i], ref["S"][i], 2e-5, 1e-4, f"S' head {i}")
        _close(tape["z"].reshape(hd, m), ref["z"], 2e-5, 1e-4, "z'")
        _close(o.reshape(n, hd, m), ref["out"], 1e-5, 1e-5, "attention out")
        o_b = E.attention_forward(q.to(DEV).bfloat16(), k.to(DEV).bfloat16(), v.to(DEV).bfloat16(), hd, E.BF16, None)
        _close(o_b.float().reshape(n, hd, m), ref["out"], 1e-2, 1e-2, "attention out bf16")


# ------------------------------------------------------------------------------------------------
# Gram-form attention: row prologue, h x h algebra, apply epilogue, and the whole layer against fp64
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,h,n", [(torch.float32, 32, 1000), (torch.bfloat16, 64, 777), (torch.bfloat16, 256, 2500),
                                       (torch.float32, 256, 300), (torch.bfloat16, 16, 5)])
def test_ln_bwd_attn(K, dtype, h, n):
    tol = 2e-5 if dtype == torch.float32 else 2e-2
    o, r, dy, xa = _acts(n, h, dtype, 11, 4)
    g = torch.Generator().manual_seed(3)
    gamma, beta = 1 + 0.1 * torch.randn(h, generator=g), 0.1 * torch.randn(h, generator=g)
    den = torch.rand(n, generator=g) + 0.5
    D = lambda t: None if t is None else t.to(DEV)
    for use_ln, use_relu, rr, xx in [(True, False, r, r), (True, True, None, xa), (False, True, r, xa), (False, False, r, r)]:
        _, ste = emu.ln_fwd(o, rr, 0.5, 0.5, gamma, beta, use_ln, use_relu, 0.0, 1)
        st = D(ste)
        dg, db = torch.zeros(h, device=DEV), torch.zeros(h, device=DEV)
        dge, dbe = torch.zeros(h), torch.zeros(h)
        rd = D(rr)
        xd = rd if xx is rr else D(xx)          # the residual IS the layer input: same device tensor (aliasing path)
        gnum, gden, dr, cs, pg, sg = K.ln_bwd_attn(D(dy), D(o), rd, xd, 0.5, 0.5, D(gamma), D(beta), st, use_ln, use_relu, 0.0, 1,
                                                   0.7, rr is not None, dg, db, D(den))
        gne, gde, dre, cse, pge, sge = emu.ln_bwd_attn(dy, o, rr, xx, 0.5, 0.5, gamma, beta, ste, use_ln, use_relu, 0.0, 1, 0.7,
                                                       rr is not None, dge, dbe, den)
        _close_gated(gnum.float(), gne.float(), tol, tol, f"gnum ln={use_ln}")
        _close(gden, gde, tol * 4, tol * 4, "gden")
        if rr is not None:
            _close_gated(dr.float(), dre.float(), tol, tol, "dr")
        _close(cs, cse, tol, tol * n ** 0.5, "cs")
        _close(pg, pge, tol * 4, tol * 4 * n ** 0.5, "pg")
        _close(sg, sge, tol * 4, tol * 4 * n ** 0.5, "sg")
        if use_ln:
            _close(dg, dge, tol, tol * n ** 0.5, "dgamma")
            _close(db, dbe, tol, tol * n ** 0.5, "dbeta")


@pytest.mark.parametrize("h,m,d,n", [(16, 16, 16, 40), (64, 64, 64, 5000), (256, 256, 256, 170000), (100, 100, 100, 900), (8, 8, 8, 3)])
def test_attn_gram_prepare_vs_fp64(K, h, m, d, n):
    """sgf_attn_gram_prepare_fwd/_bwd (fp32 SIMT) against the same algebra in fp64 (tests/test_gram_attention_math.py pins it
    to the reference)."""
    g = torch.Generator().manual_seed(h + n)
    x = torch.randn(min(n, 4000), h, generator=g, dtype=torch.float64).clamp_min(-0.5)       # non-zero mean like relu outputs
    G = (x.t() @ x) * (n / x.shape[0])
    s = x.sum(0) * (n / x.shape[0])
    ws = [torch.randn(m, h, generator=g, dtype=torch.float64) / h ** 0.5 for _ in range(2)] + \
         [torch.randn(d, h, generator=g, dtype=torch.float64) / h ** 0.5]
    bs = [0.1 * torch.randn(k, generator=g, dtype=torch.float64) for k in (m, m, d)]
    ref = emu.attn_gram_prepare_fwd(G, s, ws[0], bs[0], ws[1], bs[1], ws[2], bs[2], n)
    f = lambda t: t.float().to(DEV).contiguous()
    st = K.attn_gram_prepare_fwd(f(G), f(s), f(ws[0]), f(bs[0]), f(ws[1]), f(bs[1]), f(ws[2]), f(bs[2]), n)
    for name in ("kx", "qx", "vx", "z1", "q1", "v1", "S", "Bt", "bt"):
        _close(getattr(st, name), ref[name], 2e-5, 0, name)
    _close(st.tail[0], ref.tail[0], 5e-5, 0, "ct")
    assert float(st.tail[1:].abs().max()) == 0.0
    for slot in (emu.SC_NQ2, emu.SC_NK2, emu.SC_ALPHA, emu.SC_BETA, emu.SC_DEN, emu.SC_N):
        _close(st.sc[slot], ref.sc[slot], 2e-5, 0, f"sc[{slot}]")
    # backward with random upstream contractions of the right magnitude
    P = torch.randn(h, d, generator=g, dtype=torch.float64) * n ** 0.5
    pg, cs = torch.randn(h, generator=g, dtype=torch.float64) * n ** 0.5, torch.randn(d, generator=g, dtype=torch.float64) * n ** 0.5
    sg = torch.randn(1, generator=g, dtype=torch.float64) * n ** 0.5
    refb = emu.attn_gram_prepare_bwd(ref, P, pg, cs, sg)
    got = K.attn_gram_prepare_bwd(st, f(P), f(pg), f(cs), f(sg))
    for name, a, b in zip(("dWq", "dbq", "dWk", "dbk", "dWv", "dbv", "bcat", "a4"), got, refb):
        # relative to the largest entry: the q/k gradients are differences of O(1/N) terms
        _close(a, b, 2e-4, 0, name)


@pytest.mark.parametrize("rows,h,d", [(64, 16, 16), (1000, 64, 64), (3000, 256, 256), (130, 32, 32), (5000, 100, 100)])
@pytest.mark.parametrize("planes", [1, 3])
def test_gemm_nt_attention_gram_epilogue(K, rows, h, d, planes):
    g = torch.Generator().manual_seed(d)
    x = torch.randn(rows, h, generator=g)
    bt_m, tail = torch.randn(d, h, generator=g) / h ** 0.5, torch.zeros(16, h)
    tail[0] = 0.01 * torch.randn(h, generator=g)
    bias, dconst = torch.randn(d, generator=g), torch.tensor([1.25])
    X, Xe = K.pack_operand(x.to(DEV), False, planes), emu.pack_operand(x, False, planes)
    B, T = K.pack_operand(bt_m.to(DEV), False, planes), K.pack_operand(tail.to(DEV), False, planes)
    Be, Te = emu.pack_operand(bt_m, False, planes), emu.pack_operand(tail, False, planes)
    for dt in ([torch.float32, torch.bfloat16] if planes == 1 else [torch.float32]):
        out = K.alloc_act(rows, d, dt, DEV)
        den = torch.empty(rows, device=DEV)
        K.gemm_nt([X], [B], [(0, 0, 0, 0, h)], d, out, epi=2, bias=bias.to(DEV), tail=T, nf_dev=dconst.to(DEV), den_out=den)
        oe, de = torch.zeros(rows, d), torch.zeros(rows)
        emu.gemm_nt([Xe], [Be], [(0, 0, 0, 0, h)], d, oe, epi=2, bias=bias, tail=Te, nf_dev=dconst, den_out=de)
        tol = 2e-5 if planes == 3 else (2e-3 if dt == torch.float32 else 1e-2)
        _close(den, de, tol, tol, "den")
        _close(out.float(), oe, tol, tol, f"gram apply {dt}")


@pytest.mark.parametrize("n,h,use_weight,residual", [(16, 8, True, True), (257, 32, True, False), (4000, 256, True, True),
                                                      (1500, 64, False, True), (30000, 128, True, True)])
def test_gram_attention_layer_vs_fp64(K, n, h, use_weight, residual):
    """Whole single-head TransConv layer (projections + full_attention_conv + residual + LayerNorm) forward and backward
    on the device against fp64 autograd of the reference formula; attention term checked with RELATIVE tolerances at small N."""
    from sgformer_b200 import engine as E
    g = torch.Generator().manual_seed(n)
    x = torch.randn(n, h, generator=g).clamp_min(-0.3)
    P64, P = {}, {}
    lp = "convs.0."
    for nm in ("Wq", "Wk") + (("Wv",) if use_weight else ()):
        P64[lp + nm + ".weight"] = (torch.randn(h, h, generator=g, dtype=torch.float64) / h ** 0.5).requires_grad_(True)
        P64[lp + nm + ".bias"] = (0.1 * torch.randn(h, generator=g, dtype=torch.float64)).requires_grad_(True)
    gamma = (1 + 0.1 * torch.randn(h, generator=g, dtype=torch.float64)).requires_grad_(True)
    beta = (0.1 * torch.randn(h, generator=g, dtype=torch.float64)).requires_grad_(True)
    for k_, v in P64.items():
        P[k_] = v.detach().float().to(DEV)
    x64 = x.double().requires_grad_(True)
    q = x64 @ P64[lp + "Wq.weight"].t() + P64[lp + "Wq.bias"]
    k = x64 @ P64[lp + "Wk.weight"].t() + P64[lp + "Wk.bias"]
    v = x64 @ P64[lp + "Wv.weight"].t() + P64[lp + "Wv.bias"] if use_weight else x64
    qs, ks = q / torch.norm(q), k / torch.norm(k)
    o64 = (qs @ (ks.t() @ v) + n * v) / (qs @ ks.sum(0) + n)[:, None]
    ca, cb = (0.5, 0.5) if residual else (1.0, 0.0)
    u = ca * o64 + (cb * x64 if residual else 0.0)
    y64 = torch.nn.functional.layer_norm(u, (h,), gamma, beta, 1e-5)
    w = torch.randn(n, h, generator=g, dtype=torch.float64)
    (y64 * w).sum().backward()

    for prec, tol_o, tol_g in ((E.FP32, 1e-4, 3e-3), (E.BF16, 1e-2, 6e-2)):
        xa = x.to(DEV).to(prec.act_dtype)
        K.operand_memo_begin()
        tape = E.Tape()
        o = E.attention_gram_forward(P, lp, xa, use_weight, prec, tape)
        _close(o.float(), o64.detach(), tol_o, tol_o, f"{prec.name} attention output")
        if prec is E.FP32:
            # attention term alone (out - v), relative: invisible behind N*v at the output (SURVEY.md §7 hard part 1)
            att = o.double().cpu() - v.detach()
            att64 = (o64 - v).detach()
            if n <= 300:
                _close(att, att64, 2e-3, 0, "attention term (relative)")
            _close(tape["st"].S, (k.t() @ v).detach(), 5e-5, 0, "S' = k^T v")
            _close(tape["st"].z1, k.sum(0).detach(), 5e-5, 0, "z' = k^T 1")
            _close(tape["st"].sc[K.SC_NQ2], (q * q).sum().detach(), 5e-5, 0, "||q||^2")
            _close(tape["st"].sc[K.SC_NK2], (k * k).sum().detach(), 5e-5, 0, "||k||^2")
        y, stt = K.ln_fwd(o, xa if residual else None, ca, cb, gamma.detach().float().to(DEV), beta.detach().float().to(DEV), True,
                          False, 0.0, 1)
        _close(y.float(), y64.detach(), tol_o * 3, tol_o * 3, f"{prec.name} layer output")
        dg, db = torch.zeros(h, device=DEV), torch.zeros(h, device=DEV)
        dy = w.float().to(DEV).to(prec.act_dtype)
        gnum, gden, dr, cs, pg, sg = K.ln_bwd_attn(dy, o, xa if residual else None, xa, ca, cb, gamma.detach().float().to(DEV),
                                                   beta.detach().float().to(DEV), stt, True, False, 0.0, 1, 1.0, residual, dg, db,
                                                   tape["den"])
        grads = {}
        dprev = dr if dr is not None else K.new_like(xa)
        E.attention_gram_backward(P, lp, tape, xa, gnum, gden, cs, pg, sg, use_weight, prec, dprev, dr is not None, grads)
        K.operand_memo_clear()
        _close(dprev.float(), x64.grad, tol_g, tol_g * 0.1, f"{prec.name} dx")
        _close(dg, gamma.grad, tol_g, tol_g, "dgamma")
        _close(db, beta.grad, tol_g, tol_g, "dbeta")
        if use_weight:
            _close(grads[lp + "Wv.weight"], P64[lp + "Wv.weight"].grad, tol_g, 0, f"{prec.name} dWv")
            _close(grads[lp + "Wv.bias"], P64[lp + "Wv.bias"].grad, tol_g, 0, f"{prec.name} dbv")
        if prec is E.FP32 and n <= 300:      # q/k gradients are O(1/N) relative: only pinned where the attention term is visible
            for nm in ("Wq.weight", "Wq.bias", "Wk.weight", "Wk.bias"):
                _close(grads[lp + nm], P64[lp + nm].grad, 2e-2, 0, f"fp32 d{nm}")


@pytest.mark.parametrize("rows,h", [(1, 16), (63, 64), (64, 64), (1000, 128), (20000, 256), (5000, 100), (4097, 200), (300000, 256),
                                    (777, 8)])
@pytest.mark.parametrize("planes", [1, 3])
def test_gram_kernel(K, monkeypatch, rows, h, planes):
    """sgf_gram (X^T X with one operand load, upper block triangle mirrored, X^T 1 as an MMA column) against fp64, and against
    the generic node-contracting GEMM path; deterministic."""
    g = torch.Generator().manual_seed(rows + h)
    x = (torch.randn(rows, h, generator=g) + 0.3)
    xd = x.to(DEV)
    X = K.pack_operand(xd, False, planes)
    xe = emu.pack_operand(x, False, planes).data.double()
    G, s = K.gram(X, xd)
    tol = 2e-5 if planes == 3 else 1e-2
    _close(G, xe.t() @ xe, tol, tol * rows ** 0.5, "G = X^T X")
    _close(s, xe.sum(0), tol, tol * rows ** 0.5, "s = X^T 1")
    _close(G, G.t(), 1e-6, 0, "G symmetric")
    G2, s2 = K.gram(X, xd)
    assert torch.equal(G, G2) and torch.equal(s, s2), "sgf_gram must be run-to-run deterministic"
    monkeypatch.setattr(K, "GRAM_KERNEL", False)
    Gl, sl = K.gram(X, xd)          # colstats of the fp32 rows: the bf16 plane rounds each element by <= 2^-9
    _close(G, Gl, tol, tol * rows ** 0.5, "dedicated kernel vs gemm_tn path")
    _close(s, sl, tol, tol * rows ** 0.5, "s vs colstats path")


@pytest.mark.parametrize("dtype,h", [(torch.bfloat16, 256), (torch.bfloat16, 64), (torch.float32, 128), (torch.float32, 100)])
def test_spmm_range_phases_equal_the_whole(K, dtype, h):
    """Rotated CSR + sgf_csr_row_splits + sgf_spmm_range: running the slot-group phases one after the other (fp32 partials carried
    in place) gives the plain SpMM of the same rows; splits are exact."""
    n, world, rank = 9001, 4, 1
    block = (n + world - 1) // world
    r0, r1 = rank * block, min(n, (rank + 1) * block)
    ei = rand_graph(n, 60000, 7)
    rp, cl, dinv = K.csr_build(ei.to(DEV), n, rows=(r0, r1), col_rot=(r0, world * block))
    rpe, cle, dve = emu.csr_build(ei, n, rows=(r0, r1), col_rot=(r0, world * block))
    assert torch.equal(rp.cpu(), rpe) and torch.equal(cl.cpu(), cle), "rotated CSR differs from its definition"
    thr = (block, 2 * block, 3 * block)
    sp = K.csr_row_splits(rp, cl, thr)
    assert torch.equal(sp.cpu(), emu.csr_row_splits(rpe, cle, thr))
    x = torch.randn(world * block, h, generator=torch.Generator().manual_seed(3)).to(dtype).to(DEV)
    whole = K.spmm(rp, cl, dinv, x)
    part = torch.empty((r1 - r0, h), dtype=torch.float32, device=DEV)
    K.spmm_range(rp, cl, dinv, x, None, sp[0], None, part)
    K.spmm_range(rp, cl, dinv, x, sp[0], sp[1], part, part)
    K.spmm_range(rp, cl, dinv, x, sp[1], sp[2], part, part)
    out = K.spmm_range(rp, cl, dinv, x, sp[2], None, part, None)
    tol = 1e-6 if dtype == torch.float32 else 1e-2
    _close(out.float(), whole.float(), tol, tol, "phased SpMM vs single launch")
    ref = emu.spmm(rpe, cle, dve, x.cpu())
    _close(out.float(), ref.float(), 2e-5 if dtype == torch.float32 else 2e-2, 1e-5, "phased SpMM vs contract")


def test_cross_block_reductions_are_deterministic(K):
    """Column sums and the loss reduced across thread blocks are bit-identical from run to run (blocks add in a fixed order,
    no float atomics), so two runs of a training step compute the same."""
    g = torch.Generator().manual_seed(11)
    rows = 300_000
    x = torch.randn(rows, 256, generator=g).to(DEV)
    logits = torch.randn(rows, 47, generator=g).to(DEV)
    y = torch.randint(0, 47, (rows,), generator=g).to(DEV)
    for xx in (x, x.to(torch.bfloat16)):
        a, b = K.colstats(xx), K.colstats(xx)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), "colstats"
    l1, l2 = K.softmax_nll(logits, y, None, 1.0 / rows)[0], K.softmax_nll(logits, y, None, 1.0 / rows)[0]
    assert torch.equal(l1, l2), "softmax_nll loss"
    c1, c2 = torch.zeros(256, device=DEV), torch.zeros(256, device=DEV)
    K.pack_operand(x, False, 1, colsum=c1)
    K.pack_operand(x, False, 1, colsum=c2)
    assert torch.equal(c1, c2), "pack_operand column sums"
    _close(c1, x.double().sum(0).float(), 1e-5, 1e-3, "pack_operand column sums vs fp64")
    xt = x[:5000].t().contiguous()                  # [256, 5000]: the column sums of the source are the row sums of x[:5000]
    ct1, ct2 = torch.zeros(5000, device=DEV), torch.zeros(5000, device=DEV)
    K.pack_operand(xt, True, 1, colsum=ct1)
    K.pack_operand(xt, True, 1, colsum=ct2)
    assert torch.equal(ct1, ct2), "transposed pack_operand column sums"
    _close(ct1, x[:5000].double().sum(1).float(), 1e-5, 1e-3, "transposed pack_operand column sums vs fp64")
