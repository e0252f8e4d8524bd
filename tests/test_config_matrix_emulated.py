"""The schedule-switch table of tests/config_matrix.py on the CPU: every case, scaled down (n <= 300, h in {16, 20, 24, 32}), through
the fused schedule and through each branch alone with the kernels replaced by their emulation (tests/kernel_emu.py), against the
fp64 oracle with the per-tensor bounds of `check`; the pairwise coverage of the table; and the planted errors, which `check` must
report against the tensor they corrupt.  tests/test_gpu_config_matrix.py runs the same table on the device at full width."""
import pytest
import torch

import config_matrix as M
import kernel_emu
from sgformer_b200 import engine as E
from sgformer_b200 import functional as Fn

SMALL = [M.small_view(c) for c in M.CASES]
IDS = [c.name for c in SMALL]


@pytest.fixture(autouse=True)
def emulated_kernels(monkeypatch):
    monkeypatch.setattr(E, "K", kernel_emu)
    monkeypatch.setattr(Fn, "K", kernel_emu)
    yield


def _graph(c):
    return kernel_emu.EmuGraph(M.inputs(c)["ei"], c.n, 1 if c.variant == "medium" else 0) if c.ug else None


def _check(c, stage, training=True):
    got = M.run_stage(c, stage, E.FP32, _graph(c), training=training)
    return M.check(c, got, M.oracle_run(c, torch.float64, stage, training), M.oracle_run(c, torch.float32, stage, training), "fp32")


def test_table_covers_every_pair_of_switch_values():
    assert len(M.CASES) <= 36
    assert M.uncovered_pairs() == []
    # the coverage test itself must notice a missing case
    assert M.uncovered_pairs([c for c in M.CASES if not (c.agg == "cat" and c.variant == "medium")])


def test_table_shapes():
    """None of the row counts is a multiple of 128; at least four hub graphs; the recipes' widths and one fp32-only width."""
    assert all(c.n % 128 for c in M.CASES)
    assert {c.h for c in M.CASES} == {64, 96, 100, 256} and sum(c.h == 100 for c in M.CASES) == 2
    assert all(M.small_view(c).h % 8 for c in M.CASES if c.h == 100)     # the CPU leg keeps the width off a multiple of 8
    assert {c.d for c in M.CASES} == {65, 100, 128, 602, 1433} and {c.c for c in M.CASES} == {2, 7, 40, 47}
    assert {c.n for c in M.CASES} == {129, 1000, 3001, 8200, 20011}
    hubs = [c for c in M.CASES if c.hub]
    assert len(hubs) >= 4 and any(not c.sym for c in hubs)
    ei = M.make_edges(hubs[0])
    assert torch.bincount(ei[1]).max() > 1024 and torch.bincount(ei[0]).max() > 1024
    c = M.BY_NAME["pokec"]
    ei = M.make_edges(c)
    deg = torch.bincount(ei[1], minlength=c.n) + torch.bincount(ei[0], minlength=c.n)
    assert (deg == 0).sum() >= c.n // 16 and (ei[0] == ei[1]).any()
    assert torch.unique(ei, dim=1).shape[1] < ei.shape[1]


@pytest.mark.parametrize("c", SMALL, ids=IDS)
def test_fused_schedule(c):
    problems = _check(c, "model")
    assert not problems, "\n".join(problems)


@pytest.mark.parametrize("stage", ["trans", "graph", "head"])
@pytest.mark.parametrize("c", SMALL, ids=IDS)
def test_stage_alone(c, stage):
    if not M.stage_applies(c, stage):
        pytest.skip("no graph branch in this case")
    problems = _check(c, stage)
    assert not problems, "\n".join(problems)


@pytest.mark.parametrize("name", M.EVAL_CASES)
def test_eval_mode_backward(name):
    """Backward of an eval-mode forward: the BatchNorm backward runs on the running statistics."""
    c = M.small_view(M.BY_NAME[name])
    problems = _check(c, "model", training=False)
    assert not problems, "\n".join(problems)


@pytest.mark.parametrize("plant", list(M.PLANTED))
def test_checker_reports_planted_error(plant, monkeypatch):
    case, make, expect = M.PLANTED[plant]
    c = M.PLANT_CASES[case]._replace(n=257, h=32, d=5)
    problems = _check(c, "model")
    assert not problems, "unperturbed run must be clean:\n" + "\n".join(problems)
    graph = _graph(c)
    attr, wrapper = make(kernel_emu, graph)
    monkeypatch.setattr(kernel_emu, attr, wrapper)
    got = M.run_stage(c, "model", E.FP32, graph)
    problems = M.check(c, got, M.oracle_run(c, torch.float64), M.oracle_run(c, torch.float32), "fp32")
    named = {p.split(":")[0] for p in problems}
    assert set(expect) <= named, f"{plant}: expected {expect} among {sorted(named)}"


def test_misaligned_column_blocks_are_packed_apart():
    """A block of B that would start off a 16-byte boundary (a multiple of 8 bf16 columns) becomes an operand of its own."""
    w = torch.randn(12, 40)
    ops, at = E._b_blocks(w, [20, 20], E.FP32)
    assert at == [(0, 0), (1, 0)] and [o.k for o in ops] == [20, 20] and torch.equal(ops[1].data, w[:, 20:])
    ops, at = E._b_blocks(w, [16, 24], E.FP32)
    assert at == [(0, 0), (0, 16)] and len(ops) == 1
