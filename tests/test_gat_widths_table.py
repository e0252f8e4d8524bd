"""CPU checks of tests/gat_widths.py: the shape table reaches every GAT kernel instantiation, `geometry` is gat_geom with the
header's limits, the engine accepts every shape, and the vectorised dropout replays agree with the scalar ones."""
import numpy as np
import pytest
import torch

import gat_widths as W


def _pairs(mean=None):
    return {(dt, W.geometry(dt, h, c)[2]) for dt, h, c, m in W.SHAPES if mean is None or m == mean}


def test_shapes_cover_every_instantiation():
    """gat_logits / gat_fwd / gat_bwd_dst / gat_bwd_src are built for CPL 1-4 in fp32 and bf16: 8 (dtype, CPL) pairs, each run
    by a concatenating and a head-mean shape."""
    want = {(dt, cpl) for dt in ("fp32", "bf16") for cpl in (1, 2, 3, 4)}
    assert all(W.geometry(dt, h, c) is not None for dt, h, c, _ in W.SHAPES)
    assert _pairs() == want, sorted(want - _pairs())
    assert _pairs(False) == want, f"no concat shape for {sorted(want - _pairs(False))}"
    assert _pairs(True) == want, f"no head-mean shape for {sorted(want - _pairs(True))}"
    assert len(set(W.SHAPES)) == len(W.SHAPES)


def test_elu_widths_cover_every_row_kernel_instantiation():
    """The ELU checks of bn_fwd / bn_bwd / bn_bwd_sums run the row kernels at CPL 1-4 in fp32 and bf16, and at the recipe's
    hidden width (8 x 64 = 512) in both."""
    want = {(dt, cpl) for dt in ("fp32", "bf16") for cpl in (1, 2, 3, 4)}
    assert all(W.row_geometry(dt, h) is not None for dt, h in W.ELU_WIDTHS)
    got = {(dt, W.row_geometry(dt, h)[2]) for dt, h in W.ELU_WIDTHS}
    assert got == want, f"no ELU width for {sorted(want - got)}"
    assert {("fp32", 512), ("bf16", 512)} <= set(W.ELU_WIDTHS)
    assert W.row_geometry("bf16", 512) == (64, 32, 2) and W.row_geometry("fp32", 256) == (64, 32, 2)
    assert W.row_geometry("fp32", 300) == (75, 32, 3) and W.row_geometry("bf16", 200) == (25, 32, 1)
    assert W.row_geometry("fp32", 6) is None and W.row_geometry("fp32", 516) is None


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_shapes_reach_the_edges_of_the_geometry(dtype):
    geo = [(h, c, W.geometry(dtype, h, c)) for dt, h, c, _ in W.SHAPES if dt == dtype]
    # a partial last chunk per lane: some lanes own one chunk fewer than CPL
    assert any(cpl >= 2 and chunks % lpr for _, _, (chunks, lpr, cpl) in geo)
    # idle lanes in a row group: fewer chunks than lanes
    assert any(lpr < 32 and chunks < lpr for _, _, (chunks, lpr, cpl) in geo)
    # 32 rows per warp (lpr 1) or a single chunk, and the full row at the recipe's width
    assert any(chunks == 1 for _, _, (chunks, _, _) in geo)
    assert any(h == 8 and c == 64 for h, c, _ in geo)
    # odd head counts: heads that straddle a lane's chunks
    assert any(h % 2 for h, _, _ in geo)


def test_geometry_restates_gat_geom():
    from sgformer_b200 import kernels as K
    assert W.max_heads() == K.GAT_MAX_HEADS == 8
    assert W.geometry("fp32", 8, 64) == (128, 32, 4)
    assert W.geometry("bf16", 8, 64) == (64, 32, 2)
    assert W.geometry("fp32", 3, 8) == (6, 8, 1)
    assert W.geometry("bf16", 3, 8) == (3, 4, 1)
    assert W.geometry("bf16", 5, 104) == (65, 32, 3)
    assert W.geometry("fp32", 1, 4) == (1, 1, 1)
    for bad in (("fp32", 9, 4), ("fp32", 0, 4), ("fp32", 2, 6), ("bf16", 2, 4), ("fp16", 1, 8), ("fp32", 8, 72)):
        assert W.geometry(*bad) is None, bad
    # the kernels' CPL <= 4 is the engine's H*C limit (512 fp32 / 1024 bf16)
    for dt, vn, hc_max in (("fp32", 4, 512), ("bf16", 8, 1024)):
        for h in range(1, 9):
            for c in range(vn, 1100, vn):
                assert (W.geometry(dt, h, c) is not None) == (h * c <= hc_max), (dt, h, c)


def test_engine_accepts_every_shape():
    from sgformer_b200 import engine as E
    for dt, h, c, mean in W.SHAPES:
        P = {"l.lin_src.weight": torch.zeros(h * c, 16), "l.att_src": torch.zeros(1, h, c), "l.att_dst": torch.zeros(1, h, c),
             "l.bias": torch.zeros(c if mean else h * c)}
        cp, w, a_s, a_d, b = E._gat_layer(P, "l.", h, c, mean, E.precision(dt), 0)
        assert cp == c and w.shape == (h * c, 16) and a_s.shape == (h * c,), (dt, h, c, mean)


def _runs_graph():
    """A multigraph with runs of 70, 33 and 32 identical edges among distinct ones, in shuffled order."""
    g = torch.Generator().manual_seed(3)
    src = [torch.arange(20), torch.full((70,), 50), torch.full((33,), 5), torch.full((32,), 150), torch.randint(0, 400, (300,), generator=g)]
    dst = [torch.full((20,), 100), torch.full((70,), 100), torch.full((33,), 400), torch.full((32,), 200), torch.randint(0, 400, (300,), generator=g)]
    ei = torch.stack([torch.cat(src), torch.cat(dst)])
    return ei[:, torch.randperm(ei.shape[1], generator=g)]


@pytest.mark.parametrize("p", [0.5, 0.3])
def test_edge_keep_matches_the_scalar_replay(p):
    from test_gpu_gat import _edge_keep
    from oracle import gat_oracle as G
    n, heads, seed = 401, 3, (0xC0FFEE + 5 * 0xD1B54A32D192ED03) & W.M64
    ei = G.gat_edges(_runs_graph(), n)
    got, ref = W.edge_keep(seed, n, ei, heads, p), _edge_keep(seed, n, ei, heads, p)
    assert torch.equal(got == 0, ref == 0)
    torch.testing.assert_close(got, ref, rtol=1e-7, atol=0)
    rank = W.duplicate_rank(ei[0].numpy(), ei[1].numpy(), n)
    assert rank.max() == 69 and np.sum(rank == 31) == 3 and np.sum(rank == 32) == 2     # runs of 70, 33 and 32
    assert 0.3 * p < float((got == 0).double().mean()) < 2 * p


def test_dense_keep_matches_the_scalar_hash():
    seed, rows, cols, p = 987654321, 3, 7, 0.4
    m = W.dense_keep(seed, rows, cols, p)
    thr = W.keep_threshold(p)
    for r in range(rows):
        for c in range(cols):
            x = (seed + (r * cols + c) * W.GOLDEN) & W.M64
            x ^= x >> 33; x = (x * 0xff51afd7ed558ccd) & W.M64
            x ^= x >> 33; x = (x * 0xc4ceb9fe1a85ec53) & W.M64
            x ^= x >> 33
            assert bool(m[r, c]) == ((x & 0xFFFF) >= thr), (r, c)


def test_check_elementwise_names_the_tensor():
    ref = torch.tensor([[1.0, -2.0], [3.0, 0.5]], dtype=torch.float64)
    S = ref.abs() + 1
    assert W.check_elementwise("out", ref.float(), ref, S, 8, False) == []
    bad = ref.clone()
    bad[1, 0] *= 1 + 1e-5
    lines = W.check_elementwise("out", bad, ref, S, 8, False)
    assert len(lines) == 1 and lines[0].startswith("out:") and "(1, 0)" in lines[0]
    # a bf16-stored output may be off by one bf16 ulp of |ref| on top
    assert W.check_elementwise("dxp", ref.bfloat16().float() * (1 + 2 ** -9), ref, S, 8, True) == []
    assert W.check_elementwise("dxp", bad, ref, S, 8, True) == []
    assert W.check_elementwise("lse", torch.full_like(ref, float("nan")), ref, S, 8, False)[0].startswith("lse:")
