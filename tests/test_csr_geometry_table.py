"""The graph table of tests/csr_geometry.py reaches what tests/test_gpu_csr_sweep.py is for, on a 132-SM and a 114-SM H100: rows
on both sides of every row-sort tier edge for both key widths, queues long enough that the block-sort loops stride, the capped
scratch, scans of two and of three or more block-sum passes, fill windows past their cap, and grids that grid-stride at least
three times with a ragged tail.  The constants are read from csrc/csr.cu, so a changed tier constant fails here.  No GPU needed."""
import os
import re

import pytest

import csr_geometry as G

SMS = [132, 114]
CSR_CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sgformer_b200", "csrc", "csr.cu")


@pytest.fixture(scope="module")
def src():
    with open(CSR_CU) as f:
        return f.read()


@pytest.fixture(scope="module")
def table():
    """name -> (spec, lengths, nnz, nnz + n)"""
    out = {}
    for name, spec in G.GRAPHS.items():
        lens = spec.lengths()
        nnz = int(lens.sum())
        out[name] = (spec, lens, nnz, nnz + spec.n)
    return out


def _const(src, name):
    m = re.search(r"constexpr\s+(?:int|int64_t)\s+" + name + r"\s*=\s*([^;]+);", src)
    assert m, f"{name} not found in csr.cu"
    expr = m.group(1).replace("(int64_t)", "")
    assert re.fullmatch(r"[0-9 <()]+", expr), expr
    return eval(expr)       # a literal or a literal shift


def test_constants_match_the_source(src):
    for name, value in (("kScanBlock", G.SCAN_BLOCK), ("kScanItems", G.SCAN_ITEMS), ("kWarpSortMax", G.WARP_SORT_MAX),
                        ("kSortSmemMax", G.SORT_SMEM_MAX), ("kHubBlocks", G.HUB_BLOCKS), ("kHubScratchMax", G.HUB_SCRATCH_MAX),
                        ("kMaxFillWindows", G.MAX_FILL_WINDOWS)):
        assert _const(src, name) == value, name
    assert re.search(r'getenv\("SGF_CSR_FILL_WINDOW_MB"\);\s*return \(int64_t\)\(e \? std::atoi\(e\) : (\d+)\) << 20;', src).group(1) \
        == str(G.FILL_WINDOW_MB)
    assert re.search(r"static inline int grid_for\(int64_t work, int block, int per_sm = (\d+)\)", src).group(1) == str(G.GRID_PER_SM)
    # the three queue launches of sort_long_rows and the tier limits they pass
    launches = re.findall(r"csr_sort_rows_block_kernel<<<([^,]+), (\d+), 0, st>>>\(rowptr, col, w\.long_rows, w\.n_long, scratch, "
                          r"([^,]+), ([^,]+), ([^)]+)\)", src)
    assert launches == [("num_sms() * %d" % G.SMEM_SORT_BLOCKS_PER_SM, "256", "0", "0", "kSortSmemMax"),
                        ("kHubBlocks", "1024", "share", "kSortSmemMax", "share"),
                        ("1", "1024", "w.scratch_elems", "share", "w.scratch_elems")], launches
    assert "int64_t share = w.scratch_elems / kHubBlocks;" in src
    assert "int64_t p2 = kSortSmemMax * kHubBlocks;\n    while (p2 < tot && p2 < kHubScratchMax) p2 <<= 1;" in src
    # the warp sort's register paths and its queue edge
    assert "if (len <= 32) {" in src and "if (len <= 64) {" in src and "if (len64 > kWarpSortMax) {" in src
    # every grid-stride launch goes through grid_for with 256 threads (the caps below), except the sort queue / scan launches
    grids = re.findall(r"<<<grid_for\(([^,]+), (\d+)\), (\d+), 0,", src)
    assert len(grids) == src.count("<<<grid_for(") > 30
    for work, block, threads in grids:
        assert block == threads == str(G.BLOCK), (work, block, threads)


def test_geometry_functions():
    assert G.scratch_elems(0) == 32768 and G.share(32768) == 2048 and G.share(32769) == 4096
    assert G.scratch_elems(1 << 30) == 1 << 26 and G.share(1 << 30) == 1 << 22
    tot = 1 << 20
    assert [G.tier(x, tot) for x in (1, 2, 32, 33, 64, 65, 256, 257, 2048, 2049, 1 << 16, (1 << 16) + 1, 1 << 20, (1 << 20) + 1)] \
        == ["none", "warp1", "warp1", "warp2", "warp2", "warp_smem", "warp_smem", "block_smem", "block_smem", "hub16", "hub16",
            "hub1", "hub1", "unsorted"]
    assert G.block_sum_passes(4_194_304) == 1 and G.block_sum_passes(4_194_305) == 2
    assert G.fill_windows(0, 10, 4)["windows"] == 1 and G.fill_windows(100, 0, 4, 0)["windows"] == 1
    assert G.warp_cap(132) == 8448 and G.edge_cap(132) == 270336


@pytest.mark.parametrize("key_bytes", G.KEY_BYTES)
def test_rows_on_both_sides_of_every_tier_edge(table, key_bytes):
    """Per graph: the row lengths on both sides of 1/2, 32/33, 64/65, 256/257, 2048/2049 and share/share + 1, and the tier each
    lands in.  The weighted build sorts the same rows, with the same key counts, as int64 keys."""
    edges = [(1, 2), (32, 33), (64, 65), (256, 257), (2048, 2049)]
    seen = set()
    for name, (spec, lens, nnz, tot) in table.items():
        present = set(lens.unique().tolist())
        sh = G.share(tot)
        assert G.scratch_elems(tot) * key_bytes <= (1 << 26) * key_bytes
        if name == "many":
            continue
        for a, b in edges + [(sh, sh + 1)]:
            assert a in present and b in present, (name, key_bytes, a, b)
            assert G.tier(a, tot) != G.tier(b, tot), (name, a, b)
        seen |= {G.tier(x, tot) for x in present}
    assert seen == set(G.TIERS), sorted(set(G.TIERS) - seen)


def test_small_medium_and_large_regimes(table):
    _, _, _, tot = table["small"]
    assert tot <= 32768 and G.share(tot) == G.SORT_SMEM_MAX, "small: the 16-block tier is empty"
    _, lens, _, tot = table["medium"]
    assert 32768 < tot <= G.HUB_SCRATCH_MAX and G.share(tot) > G.SORT_SMEM_MAX
    _, lens, nnz, tot = table["large"]
    n = G.GRAPHS["large"].n
    assert tot > G.HUB_SCRATCH_MAX and G.scratch_elems(tot) == 1 << 26 and G.share(tot) == 1 << 22
    assert G.tier((1 << 22) + 1, tot) == "hub1" and G.tier((1 << 26) + 1, tot) == "unsorted"
    assert int((lens == (1 << 22) + 1).sum()) == 1 and int((lens == (1 << 26) + 1).sum()) == 1
    assert n > 4_194_304 and G.block_sum_passes(n) == 2
    assert G.fill_windows(nnz, n, 4)["launches"] >= 3 and G.fill_windows(nnz, n, 8)["launches"] >= 3


@pytest.mark.parametrize("sms", SMS)
def test_block_sort_queues_stride(table, sms):
    _, lens, _, tot = table["medium"]
    tiers = [G.tier(x, tot) for x in lens.tolist()]
    assert tiers.count("block_smem") > 3 * sms * G.SMEM_SORT_BLOCKS_PER_SM
    assert tiers.count("hub16") > 3 * G.HUB_BLOCKS


def test_scan_depths(table):
    spec = G.GRAPHS["many"]
    _, _, nnz, _ = table["many"]
    assert spec.n >= 12_000_000 and G.block_sum_passes(spec.n) >= 3 and G.block_sum_last_pass_partial(spec.n)
    assert spec.n % (G.SCAN_BLOCK * G.SCAN_ITEMS) != 0, "the last scan block is partial"
    assert nnz > 4_194_304 and G.block_sum_passes(nnz) >= 2, "remove_self_loops / subgraph flag scans of two passes or more"
    _, _, nnz, _ = table["medium"]
    assert G.block_sum_passes(2 * nnz) >= 2, "to_undirected's doubled rows"


def test_fill_windows_reach_the_cap(table):
    """The default window splits the large graph's builds; a 1 MiB window makes more than 12 windows of the medium and
    large graphs for both entry widths, so the cap applies; 0 MiB is one launch."""
    for name in ("medium", "large"):
        spec, _, nnz, _ = table[name]
        for eb in G.KEY_BYTES:
            w = G.fill_windows(nnz, spec.n, eb, 1)
            assert w["want"] > G.MAX_FILL_WINDOWS and w["windows"] == w["launches"] == G.MAX_FILL_WINDOWS, (name, eb, w)
            assert G.fill_windows(nnz, spec.n, eb, 0)["launches"] == 1
            # a row shard of the middle half still splits
            assert G.fill_windows(nnz, spec.n // 2, eb, 1)["windows"] > 1
    spec, _, nnz, _ = table["large"]
    assert G.fill_windows(nnz, spec.n, 4)["windows"] == 3


@pytest.mark.parametrize("sms", SMS)
def test_grids_stride_three_times_with_a_ragged_tail(table, sms):
    for name in ("medium", "large", "many"):
        spec, _, nnz, _ = table[name]
        for work, cap in ((spec.n, G.warp_cap(sms)), (nnz, G.edge_cap(sms)), (nnz + spec.n, G.edge_cap(sms))):
            lo, hi = G.iterations(work, cap)
            assert lo >= 3 and hi == lo + 1, (name, sms, work, cap)
