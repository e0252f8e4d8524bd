"""Every schedule switch of the SGFormer encoder on the H100 at the widths the reference's recipes use (tests/config_matrix.py:
h in {64, 96, 100, 256}, n up to 20 011, hub rows, directed graphs), fp32 and bf16:

* the drop-in modules against an fp64 run of the oracle — eval logits, train logits, every parameter gradient and the input
  gradient each on its own scale (`config_matrix.check`), the BatchNorm buffers after the step, and for three cases the backward
  of an eval-mode forward;
* each branch alone (functional.TransConvFn / GraphBranchFn / HeadFn) with a seeded upstream gradient against fp64 autograd of the
  oracle's stage: here no other branch's gradient can hide an error, and the attention's Wq / Wk gradients get a bound at real N;
* planted errors: one entry point of sgformer_b200.kernels wrapped so that a valid launch returns a subtly wrong result, which
  `check` must report against the tensor it corrupts;
* run-to-run determinism of the gradients for one case per variant.

SGF_CONFIG_MATRIX_REPORT=<file> appends one JSON line per (case, precision, tensor) with the measured error, the fp32 oracle's own
error and the bound: the calibration of config_matrix.FLOOR (DESIGN.md §6)."""
import pytest
import torch

import config_matrix as M
from test_gpu_model import build_model, run

pytestmark = pytest.mark.gpu
DEV = "cuda"
IDS = [c.name for c in M.CASES]
STAGE_CASES = [c for c in M.CASES if c.h in (64, 100, 256)]


def _graph(c):
    from sgformer_b200.graph import Graph
    return Graph(M.inputs(c)["ei"].to(DEV), c.n, 1 if c.variant == "medium" else 0) if c.ug else None


def _prec(precision):
    from sgformer_b200 import engine as E
    return E.precision(precision)


def _module_step(c, precision, training=True):
    """One forward/backward of the drop-in module -> (eval logits, what check() takes)."""
    inp = M.inputs(c)
    ocfg = inp["ocfg"]
    model = build_model(ocfg).to(DEV).set_precision(precision)
    model.load_state_dict(inp["sd"])
    x, ei = inp["x"].to(DEV), inp["ei"].to(DEV)
    model.eval()
    with torch.no_grad():
        out_eval = run(model, ocfg, x, ei)
    model.train(training)
    xg = x.clone().requires_grad_(True)
    out = run(model, ocfg, xg, ei)
    (out * inp["lw"].to(DEV)).sum().backward()
    grads = {k: p.grad for k, p in model.named_parameters() if p.grad is not None}
    grads["__x__"] = xg.grad
    stats = {k: v for k, v in model.state_dict().items() if "running" in k or k.endswith("num_batches_tracked")}
    return out_eval, dict(out=out, grads=grads, stats=stats if training else {})


def _refs(c, stage="model", training=True):
    return M.oracle_run(c, torch.float64, stage, training), M.oracle_run(c, torch.float32, stage, training)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("c", M.CASES, ids=IDS)
def test_module_matches_fp64_oracle(c, precision):
    if not M.supports(c, precision):
        pytest.skip("bf16 rows move in 8-element chunks: h must be a multiple of 8")
    out_eval, got = _module_step(c, precision)
    ref64, ref32 = _refs(c)
    problems = M.check(c, got, ref64, ref32, precision, M.REPORT)
    ref_eval = M.oracle_run(c, torch.float64, "model", False)["out"]
    tol = M.LOGIT_TOL[precision]
    err = (out_eval.cpu().double() - ref_eval).abs().max().item()
    if not err <= tol + tol * ref_eval.abs().max().item():
        problems.append(f"eval out: max err {err:.3e}")
    assert not problems, "\n".join(problems)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", M.EVAL_CASES)
def test_module_eval_mode_backward(name, precision):
    """Backward of an eval-mode forward: the BatchNorm backward and its affine gradients run on the running statistics."""
    c = M.BY_NAME[name]
    _, got = _module_step(c, precision, training=False)
    problems = M.check(c, got, *_refs(c, "model", False), precision, M.REPORT)
    assert not problems, "\n".join(problems)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("stage", ["trans", "graph", "head"])
@pytest.mark.parametrize("c", STAGE_CASES, ids=[c.name for c in STAGE_CASES])
def test_stage_alone_matches_fp64_oracle(c, stage, precision):
    if not M.stage_applies(c, stage):
        pytest.skip("no graph branch in this case")
    if not M.supports(c, precision):
        pytest.skip("bf16 rows move in 8-element chunks: h must be a multiple of 8")
    got = M.run_stage(c, stage, _prec(precision), _graph(c) if stage == "graph" else None, DEV)
    problems = M.check(c._replace(name=f"{c.name}/{stage}"), got, *_refs(c, stage), precision, M.REPORT)
    assert not problems, "\n".join(problems)


def test_query_key_gradients_are_bounded_at_recipe_sizes():
    """The table puts a Wq / Wk gradient under check() at n >= 8200 for h = 64 and h = 256, one head and two."""
    big = [c for c in M.CASES if c.tl > 0 and c.n >= 8200]
    assert {(c.h, c.heads) for c in big} >= {(64, 1), (256, 1), (256, 2)}
    assert M.FLOOR["qk"]["fp32"] <= 1e-3 and M.FLOOR["qk_bias"]["fp32"] <= 1e-3 and M.FLOOR["qk"]["bf16"] <= 0.4


def test_gemm_nt_refuses_a_misaligned_k_offset():
    """A K offset off a 16-byte boundary is an error at the call, not a barrier wait that never completes on the device."""
    from sgformer_b200 import kernels as K
    a = K.pack_operand(torch.randn(64, 40, device=DEV), False, 3)
    b = K.pack_operand(torch.randn(16, 40, device=DEV), False, 3)
    with pytest.raises(ValueError, match="multiples of 8"):
        K.gemm_nt([a], [b], [(0, 0, 0, 20, 20)], 16, torch.empty(64, 16, device=DEV))


@pytest.mark.parametrize("plant", list(M.PLANTED))
def test_checker_reports_planted_error(plant, monkeypatch):
    from sgformer_b200 import kernels as K
    case, make, expect = M.PLANTED[plant]
    c = M.PLANT_CASES[case]
    graph = _graph(c)
    ref64, ref32 = _refs(c)
    problems = M.check(c, M.run_stage(c, "model", _prec("fp32"), graph, DEV), ref64, ref32, "fp32")
    assert not problems, "unperturbed run must be clean:\n" + "\n".join(problems)
    attr, wrapper = make(K, graph)
    monkeypatch.setattr(K, attr, wrapper)
    problems = M.check(c, M.run_stage(c, "model", _prec("fp32"), graph, DEV), ref64, ref32, "fp32")
    named = {p.split(":")[0] for p in problems}
    assert set(expect) <= named, f"{plant}: expected {expect} among {sorted(named)}"


@pytest.mark.parametrize("name", ["pokec", "papers100M", "deezer"])
def test_gradients_are_bit_identical_run_to_run(name):
    c = M.BY_NAME[name]
    _, a = _module_step(c, "fp32")
    _, b = _module_step(c, "fp32")
    assert torch.equal(a["out"], b["out"])
    for k, g in a["grads"].items():
        assert torch.equal(g, b["grads"][k]), f"{k} differs between two runs"
