"""Size-independent properties at BASELINE.json's full shapes (where the CPU oracle would take minutes): the CSR invariants,
A.1 = degree (exact), linearity and the adjoint identity of the SpMM, conservation laws of the linear attention, and the
induced-subgraph / CSR-subset consistency, on the ogbn-products- and Pokec-shaped synthetic graphs."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def products():
    from sgformer_b200.graph import Graph
    from sgformer_b200.synth import SHAPES, make_graph
    n, d, e, c, h, layers, use_init = SHAPES["products"]
    ei = make_graph(n, e, seed=0, device=DEV)
    return n, ei, Graph(ei, n)


def test_csr_invariants_products_shape(products):
    n, ei, g = products
    rowptr, col = g.rowptr, g.col
    assert rowptr[0].item() == 0 and rowptr[-1].item() == ei.shape[1] == col.numel()      # nnz conserved
    lens = rowptr[1:] - rowptr[:-1]
    assert bool((lens >= 1).all())                                                         # every node has its self loop
    assert torch.equal(lens, torch.bincount(ei[1], minlength=n))                           # in-degree over `col` (bit-exact)
    # sortedness inside rows: a position may decrease only where a new row starts
    dec = (col[1:] < col[:-1]).nonzero().flatten() + 1
    starts = torch.zeros(col.numel() + 1, dtype=torch.bool, device=DEV)
    starts[rowptr] = True
    assert bool(starts[dec].all())
    assert int(col.min()) >= 0 and int(col.max()) < n
    assert torch.equal(g.dinv, (1.0 / lens.float()).sqrt())                                # same op order as the reference
    rp_t, col_t = g.transpose()
    assert rp_t is g.rowptr                                                                # symmetric edge set detected
    # checksum of checksums: sum of column ids per row, summed over rows == sum over the edge list
    assert int(col.sum(dtype=torch.int64)) == int(ei[0].sum())


def test_spmm_properties_products_shape(products):
    from sgformer_b200 import kernels as K
    n, ei, g = products
    ones = torch.ones(n, 8, device=DEV)
    deg = K.spmm(g.rowptr, g.col, None, ones, heavy=g.heavy)
    assert torch.equal(deg[:, 0], (g.rowptr[1:] - g.rowptr[:-1]).float())                 # A.1 = degree, exact in fp32
    gen = torch.Generator(device=DEV).manual_seed(0)
    x = torch.randn(n, 64, generator=gen, device=DEV)
    y = torch.randn(n, 64, generator=gen, device=DEV)
    ax, ay = K.spmm(g.rowptr, g.col, None, x), K.spmm(g.rowptr, g.col, None, y)
    lin = K.spmm(g.rowptr, g.col, None, K.axpby(x, y, 1.0, 2.0))
    err = (lin - (ax + 2 * ay)).abs().max().item() / ax.abs().max().item()
    assert err < 1e-5, f"linearity: {err:.2e}"
    # adjoint identity on the symmetric graph: <A x, y> == <x, A y>
    lhs, rhs = (ax.double() * y.double()).sum().item(), (x.double() * ay.double()).sum().item()
    assert abs(lhs - rhs) <= 1e-6 * max(abs(lhs), 1.0) + 1e-3, f"adjoint: {lhs} vs {rhs}"
    # bf16 path at h=256 (the benchmarked configuration) against the fp32 path on the same (bf16-rounded) input
    xb = torch.randn(n, 256, generator=gen, device=DEV).to(torch.bfloat16)
    yb = K.spmm(g.rowptr, g.col, g.dinv, xb)
    yf = K.spmm(g.rowptr, g.col, g.dinv, xb.float())
    rel = (yb.float() - yf).abs().max().item() / yf.abs().max().item()
    assert rel < 8e-3, f"bf16 vs fp32 SpMM: {rel:.2e}"


def _spmm_ref_int(ei, n, xi):
    """Exact y[r] = sum of xi[c] over the edges (c -> r) of the edge list, in int32 (edge chunks; |y| <= degree)."""
    out = torch.zeros_like(xi)
    for i in range(0, ei.shape[1], 1 << 19):
        out.index_add_(0, ei[1, i:i + (1 << 19)], xi.index_select(0, ei[0, i:i + (1 << 19)]))
    return out


def _check_spmm_exact(K, rowptr, col, dinv, heavy, ei, n):
    """Integer features make every row sum exact in fp32, whatever the order: the SpMM must equal the edge-list sum bit for bit
    (bf16 outputs after round-to-nearest-even).  With the row scale dinv the kernel rounds the exact sum times dinv once (fp32),
    which is what fp64 rounds to as well (a 24-bit integer times a 24-bit fp32 is exact in fp64)."""
    gen = torch.Generator(device=DEV).manual_seed(5)
    for dtype, h, lo in ((torch.bfloat16, 256, -1), (torch.float32, 64, -2)):
        xi = torch.randint(lo, -lo + 1, (n, h), generator=gen, device=DEV, dtype=torch.int32)
        ref = _spmm_ref_int(ei, n, xi).float()                  # exact: |sum| <= max degree < 2^24
        x = xi.to(dtype)
        del xi
        y = K.spmm(rowptr, col, None, x, heavy=heavy)
        want = ref.to(dtype)                                    # bf16: round-to-nearest-even of the exact sum
        assert torch.equal(y, want), f"{dtype} h={h}: {int((y != want).sum())} elements differ"
        del y, want
        y = K.spmm(rowptr, col, dinv, x, heavy=heavy)
        for i in range(0, n, 1 << 18):
            want = (ref[i:i + (1 << 18)].double() * dinv[i:i + (1 << 18)].double()[:, None]).float().to(dtype)
            got = y[i:i + (1 << 18)]
            assert torch.equal(got, want), f"{dtype} h={h} with dinv, rows from {i}: {int((got != want).sum())} elements differ"
        del x, y, ref


def test_spmm_exact_products_shape(products):
    """The products SpMM against an independent exact reference (the int32 sum over the edge list): which columns each row
    gathers, not only how many (A.1 = degree) or that it is linear."""
    from sgformer_b200 import kernels as K
    n, ei, g = products
    _check_spmm_exact(K, g.rowptr, g.col, g.dinv, g.heavy, ei, n)


def test_spmm_heavy_rows_exact_products_size():
    """The segmented hub-row path (heavy=) on a power-law graph of the products size, exactly; the single-warp path on the
    same rows too."""
    from sgformer_b200 import kernels as K
    from sgformer_b200.graph import Graph
    from sgformer_b200.synth import SHAPES, make_rmat_graph
    n, _, e = SHAPES["products"][:3]
    ei = make_rmat_graph(n, e, seed=1, device=DEV)
    g = Graph(ei, n)
    lens = g.rowptr[1:] - g.rowptr[:-1]
    assert g.heavy is not None and int(lens.max()) > 8 * K.HEAVY_ROW
    assert bool(((g.heavy.seg_len > 0) & (g.heavy.seg_len <= K.HEAVY_ROW)).all())
    assert bool((lens[g.heavy.rows] % K.HEAVY_ROW != 0).any()), "some hub row must end in a short segment"
    _check_spmm_exact(K, g.rowptr, g.col, g.dinv, g.heavy, ei, n)
    _check_spmm_exact(K, g.rowptr, g.col, g.dinv, None, ei, n)


def test_attention_conservation_laws_pokec_shape():
    """With v = 1 every output is exactly 1 (num = q~.z + N = den); in general the output stays within O(N^-1.5) of v."""
    from sgformer_b200 import engine as E
    n, h = 1632803, 64
    gen = torch.Generator(device=DEV).manual_seed(1)
    q = torch.randn(n, h, generator=gen, device=DEV)
    k = torch.randn(n, h, generator=gen, device=DEV)
    v1 = torch.ones(n, h, device=DEV)
    o = E.attention_forward(q, k, v1, 1, E.FP32, None)
    assert (o - 1).abs().max().item() < 1e-5
    v = torch.randn(n, h, generator=gen, device=DEV)
    tape = E.Tape()
    o = E.attention_forward(q, k, v, 1, E.FP32, tape)
    # the attention term is O(N^-1.5) of the residual term (SURVEY.md TL;DR 3): outputs stay within 1e-4 of v ...
    assert (o - v).abs().max().item() < 1e-3
    # ... while the pass-1 partial is checked against a chunked fp64 reduction
    s_ref = torch.zeros(h, h, dtype=torch.float64, device=DEV)
    for i in range(0, n, 1 << 18):
        s_ref += k[i:i + (1 << 18)].double().t() @ v[i:i + (1 << 18)].double()
    rel = (tape["s"][0].double() - s_ref).abs().max().item() / s_ref.abs().max().item()
    assert rel < 1e-4, f"S' = k^T v at N = 1.6 M: {rel:.2e}"
    assert torch.isfinite(o).all()


def test_subgraph_consistency_products_shape(products):
    from sgformer_b200 import kernels as K
    n, ei, g = products
    idx = torch.randperm(n, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))[:100000]
    sub = g.subset(idx)
    ei_sub = K.subgraph(ei, n, idx)
    rp, cl, dv = K.csr_build(ei_sub, idx.numel())
    assert torch.equal(sub.rowptr, rp) and torch.equal(sub.col, cl) and torch.equal(sub.dinv, dv)
    # idempotence: the subset of all nodes in natural order is the graph itself
    full = g.subset(torch.arange(n, device=DEV))
    assert torch.equal(full.rowptr, g.rowptr) and torch.equal(full.col, g.col) and torch.equal(full.dinv, g.dinv)
