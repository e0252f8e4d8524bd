"""The width table and work plans of tests/spmm_geometry.py reach what tests/test_gpu_spmm_sweep.py is for, on a 132-SM and a
114-SM H100: every (dtype, lanes per row, chunks per lane) class of the CSR gather kernels, a partial last pass at every
chunks-per-lane count above one, and grids that grid-stride at least three times.  No GPU needed."""
import pytest

import spmm_geometry as G
from sgformer_b200 import engine as E

PREC = {G.F32: E.FP32, G.B16: E.BF16}
SMS = [132, 114]


def _admitted(dtype, h) -> bool:
    try:
        E.check_width(h, PREC[dtype], "hidden")
        return True
    except ValueError:
        return False


def _admitted_widths(dtype):
    return [h for h in range(1, 2 * G.MAX_ROW_BYTES) if _admitted(dtype, h)]


def test_every_class_is_in_the_table():
    for dtype in (G.F32, G.B16):
        want = {G.klass(dtype, h) for h in _admitted_widths(dtype)}
        have = {G.klass(dtype, h) for h in G.WIDTHS[dtype]}
        assert have == want, (G.name(dtype), sorted(want - have))
        lprs = {lpr for _, lpr, _ in want}
        assert lprs == {1, 2, 4, 8, 16, 32} and {cpl for _, _, cpl in want} == {1, 2, 3, 4}
        for cpl in (2, 3, 4):
            partial = [h for h in G.WIDTHS[dtype] if G.geom(dtype, h)["cpl"] == cpl and G.geom(dtype, h)["partial"]]
            assert partial, f"{G.name(dtype)}: no partial last pass at cpl {cpl}"
            assert any(G.geom(dtype, h)["last_live"] == 1 for h in G.WIDTHS[dtype] if G.geom(dtype, h)["cpl"] >= 2)
        assert any(G.geom(dtype, h)["idle"] > 0 and G.geom(dtype, h)["cpl"] == 1 for h in G.WIDTHS[dtype]), "idle lanes, one pass"
    for dtype, h in G.FLOAT_WIDTHS + G.EDGE_GRAD_WIDTHS:
        assert h in G.WIDTHS[dtype]
    assert {G.klass(d, h)[1:] for d, h in G.FLOAT_WIDTHS} >= {(1, 1), (4, 1), (32, 1), (32, 2), (32, 3), (32, 4)}


def test_admitted_widths_fall_in_table_classes():
    for dtype in (G.F32, G.B16):
        classes = {G.klass(dtype, h) for h in G.WIDTHS[dtype]}
        widths = _admitted_widths(dtype)
        assert widths[0] == G.vn(dtype) and widths[-1] == G.MAX_ROW_BYTES // (4 if dtype == G.F32 else 2)
        for h in widths:
            assert G.klass(dtype, h) in classes, (G.name(dtype), h)
            assert h <= G.edge_grad_max_width(dtype), "the edge-weight gradient takes every width the layers admit"


def test_refused_widths_are_exactly_those_check_width_refuses():
    for dtype in (G.F32, G.B16):
        for h in range(1, 2 * G.MAX_ROW_BYTES):
            assert G.launch_refuses(dtype, h) == (not _admitted(dtype, h)), (G.name(dtype), h)
            assert G.launch_refuses(dtype, h) == (h % G.vn(dtype) != 0 or h > G.edge_grad_max_width(dtype)), (G.name(dtype), h)
    for dtype, h in G.REFUSED:
        assert G.launch_refuses(dtype, h) and not _admitted(dtype, h)
    assert {h % G.vn(d) != 0 for d, h in G.REFUSED} == {True, False}, "one refused for its width, one for its alignment"
    for dtype, h in G.WIDTH_LIST:
        assert not G.launch_refuses(dtype, h)


@pytest.mark.parametrize("sms", SMS)
def test_plans_exceed_their_caps(sms):
    assert G.row_cap(132) == 33792 and G.edge_grad_cap(132) == 8448
    for cap in (G.row_cap(sms), G.edge_grad_cap(sms)):
        for kind in G.PLANS:
            n = G.plan(cap, kind)
            lo, hi = G.iterations(n, cap)
            assert lo >= 3, (cap, kind)
            if kind == "exact":
                assert n % cap == 0 and lo == hi == 3
            else:
                assert hi == lo + 1 and (n % cap) % G.WARPS_PER_CTA != 0, "the tail must end inside a CTA"
    sp = G.segment_plan(sms)
    assert sp["row_len"] > G.HEAVY_ROW and sp["row_len"] % G.HEAVY_ROW != 0, "hub rows end in a short segment"
    assert -(-sp["row_len"] // G.HEAVY_ROW) == G.SEG_PER_ROW
    lo, hi = G.iterations(sp["n_seg"], G.row_cap(sms))
    assert lo >= 3 and hi == lo + 1, sp
    for dtype, h in ((G.F32, 512), (G.B16, 1024)):
        fp = G.finalize_plan(dtype, h, sms)
        assert min(fp["lens"]) > G.HEAVY_ROW
        lo, _ = G.iterations(fp["n_heavy"] * h, G.finalize_cap(sms))
        assert lo >= 3, (G.name(dtype), fp["n_heavy"])
