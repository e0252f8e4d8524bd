"""The streamed-tile heights of the fused attention kernels without a GPU: tests/attn_tiles.py against the library's own choice
(sgf_attn_softmax_tile_rows calls the `pick_bs` the launches use and makes no CUDA call), the table's reach over every legal
shape, and the refusal of every shape whose backward has no tile."""
import functools

import pytest
import torch

from attn_tiles import KINDS, TABLE, combos
from sgformer_b200 import engine as E
from sgformer_b200 import kernels as K

DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16}


@pytest.fixture(scope="module", autouse=True)
def _library():
    import __graft_entry__ as g
    g.build()


@pytest.mark.parametrize("t", TABLE, ids=str)
def test_table_matches_the_library(t):
    assert K.attn_softmax_tile_rows(t.heads, t.m, t.d, DTYPES[t.dtype], t.shared_v, t.shared_g) == t.rows
    assert K.attn_softmax_fits(t.heads, t.m, t.d, DTYPES[t.dtype], t.shared_v, t.shared_g)
    if t.mode == "gat":         # the scaled mode takes per-head v only, and q/k blocks padded as the GAT layers pad them
        assert not t.shared_v and t.m == E.gat_attn_pad(t.dk, E.precision(t.dtype))


@functools.lru_cache(maxsize=None)
def _sweep():
    """Every legal shape: heads 1..16; m and d in steps of 16 bytes up to 1 KB; shared and per-head v and g.
    -> {(dtype, heads, m, d, shared_v, shared_g): (fwd, bwd_q, bwd_kv)}"""
    out = {}
    for name, dt in DTYPES.items():
        step = 16 // dt.itemsize
        widths = range(step, 1024 // dt.itemsize + 1, step)
        for heads in range(1, 17):
            for m in widths:
                if K.attn_softmax_tile_rows(heads, m, step, dt, True, True) is None:
                    break           # the q row is past the limit, and stays so for every wider m
                for d in widths:
                    for sv in (False, True):
                        for sg in (False, True):
                            rows = K.attn_softmax_tile_rows(heads, m, d, dt, sv, sg)
                            if rows is not None:
                                out[(name, heads, m, d, sv, sg)] = rows
    return out


def test_table_reaches_every_height_any_shape_reaches():
    reach = set()
    for (name, heads, m, d, sv, sg), rows in _sweep().items():
        modes = ("softmax",) if sv else ("softmax", "gat")         # the scaled mode refuses a shared v
        reach |= {(name, mode, kind, bs) for mode in modes for kind, bs in zip(KINDS, rows) if bs}
    table = set().union(*(combos(t) for t in TABLE))
    assert reach - table == set(), f"heights no table row runs: {sorted(reach - table)}"
    assert table <= reach
    # fwd at 64 / 32, bwd_q and bwd_kv at 64 / 32 / 16, in two dtypes and two modes
    assert len(reach) == 32, sorted(reach)


def test_table_covers_gradient_and_value_layouts():
    for name in DTYPES:
        for mode in ("softmax", "gat"):
            rows = [t for t in TABLE if t.dtype == name and t.mode == mode]
            assert any(t.shared_g and t.heads > 1 for t in rows) and any(not t.shared_g and t.heads > 1 for t in rows), (name, mode)
            assert mode == "gat" or any(t.shared_v for t in rows), (name, mode)


def test_every_shape_without_a_backward_tile_is_refused():
    zero = [(key, rows) for key, rows in _sweep().items() if 0 in rows]
    assert zero, "no legal shape lacks a tile: the refusal below checks nothing"
    for (name, heads, m, d, sv, sg), rows in zero:
        assert rows[0] != 0, "the forward always has a tile"
        assert not K.attn_softmax_fits(heads, m, d, DTYPES[name], sv, False)
        assert not K.attn_softmax_fits(heads, m, d, DTYPES[name], sv, sg)


@pytest.mark.parametrize("prec,heads,m,d", [("fp32", 2, 128, 256), ("fp32", 4, 64, 256), ("fp32", 8, 32, 128),
                                            ("bf16", 2, 256, 512), ("bf16", 4, 128, 512), ("bf16", 8, 64, 256)])
def test_shared_v_with_per_head_gradient_has_no_backward_tile(prec, heads, m, d):
    """A one-head v [N, 1, D] with a gradient block per head (softmax_attention's backward): the gradient rows are heads x d
    wide, and no streamed tile of bwd_q / bwd_kv fits beside them.  The head mean's shared gradient leaves room."""
    dt = DTYPES[prec]
    rows = K.attn_softmax_tile_rows(heads, m, d, dt, True, False)
    assert rows[0] != 0 and rows[1:] == (0, 0)
    assert K.attn_softmax_fits(heads, m, d, dt, True, True)
    what = f"softmax attention with {heads} heads of width {m} and value width {d}"
    with pytest.raises(ValueError, match=r"backward \(bwd_q / bwd_kv\) has no streamed tile"):
        E.check_attn_softmax(what, heads, m, d, E.precision(prec), True, False)
    E.check_attn_softmax(what, heads, m, d, E.precision(prec), True, True)
    E.check_attn_softmax(what, heads, m, d, E.precision(prec), True, None)      # no backward follows: the forward runs


@pytest.mark.parametrize("heads,m,d,shared_v", [(4, 128, 16, True), (2, 16, 256, False), (1, 6, 16, True), (1, 16, 6, True)])
def test_widths_the_kernels_refuse(heads, m, d, shared_v):
    """fp32: past the 1 KB row limit, or a head width that is not a multiple of 16 bytes."""
    assert K.attn_softmax_tile_rows(heads, m, d, torch.float32, shared_v, False) is None
    assert not K.attn_softmax_fits(heads, m, d, torch.float32, shared_v, True)
    with pytest.raises(ValueError, match="at most 1024 bytes"):
        E.check_attn_softmax("attention", heads, m, d, E.FP32, shared_v, None)
