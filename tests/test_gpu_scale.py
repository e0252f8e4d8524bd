"""Bit-exact checks of the node-contracting GEMMs (`gemm_tn`, `gram`) and of every `gemm_nt` epilogue instantiation at the
row counts where their code paths switch on, up to the ogbn-products row count (2,449,029).

Floating-point sums of small integers are exact.  The operands are integers in {-1, 0, 1} at the products row count and in
{-2, ..., 2} below it; alpha, beta and row scales are powers of two, bias and r1 small integers.  Every product and every
partial sum is then an integer (or a power-of-two multiple of one) below 2^22, so each kernel's fp32 result has exactly one
correct value, whatever the summation order, and a bf16 output must equal round-to-nearest-even of it.  A dropped, doubled
or misplaced node block, a lost flush partial, a wrong slice remainder or a wrong epilogue term fails `torch.equal` instead
of hiding inside a tolerance.  The fp64 references are computed on the device in row chunks of 2^18.

The flush geometry of `gemm_tn` / `gram` (csrc/gemm_tc.cu: `tn_splits`, the per-CTA node slice, FLUSH_KB) is restated
here so that the generated row counts provably reach each case; `test_flush_geometry_covers_every_case` checks that
without a GPU."""
import pytest
import torch

DEV = "cuda"
CHUNK = 1 << 18                  # rows per fp64 reference step
PRODUCTS_ROWS = 2_449_029        # ogbn-products (sgformer_b200/synth.py SHAPES)
EXACT_LIMIT = 1 << 22            # every exact sum below stays under this

# ------------------------------------------------------------------------------------------------
# flush geometry of gemm_tn / gram (host only)
# ------------------------------------------------------------------------------------------------
BKN = 64          # node rows per block (tn::BKN, gramk::BKN)
FLUSH_KB = 16     # a CTA flushes its accumulators every FLUSH_KB node blocks, except after its last block
CATEGORIES = ("no_flush", "flush_16k", "flush_16k_plus_1", "flush_rem", "ragged", "products")


def tn_splits(kb_total: int, m_blocks: int, sms: int) -> int:
    """Node slices per 128-feature block of A: one wave of CTAs over all blocks (gemm_tc.cu tn_splits)."""
    cap = max(sms // m_blocks, 1)
    return max(kb_total, 1) if kb_total < cap else cap


def node_slices(rows: int, m_blocks: int, sms: int):
    """-> (per, rem, grid): CTA y owns per + (y < rem) consecutive node blocks."""
    kb = -(-rows // BKN)
    g = tn_splits(kb, m_blocks, sms)
    return kb // g, kb % g, g


def categories_of(rows: int, m_blocks: int, sms: int) -> set:
    per, rem, _ = node_slices(rows, m_blocks, sms)
    lens = {per, per + 1} if rem else {per}
    cats = set()
    if max(lens) < FLUSH_KB:
        cats.add("no_flush")                       # no mid-loop flush at all
    if not rem and per >= FLUSH_KB and per % FLUSH_KB == 0:
        cats.add("flush_16k")                      # the last block of every slice skips the mid-loop flush
    if any(n > FLUSH_KB and n % FLUSH_KB == 1 for n in lens):
        cats.add("flush_16k_plus_1")               # one block left after the last mid-loop flush
    if rem and (min(lens) - 1) // FLUSH_KB >= 2:
        cats.add("flush_rem")                      # several flushes, slices of unequal length
    if rows % BKN:
        cats.add("ragged")                         # partial last node block
    if rows == PRODUCTS_ROWS:
        cats.add("products")
    return cats


def row_counts(m_blocks: int, sms: int) -> dict:
    """One row count per category for a product with `m_blocks` 128-feature blocks on a GPU with `sms` SMs."""
    g = max(sms // m_blocks, 1)
    return {
        "no_flush": (10 * g + 1) * BKN,                   # slices of 10 and 11 blocks
        "flush_16k": 2 * FLUSH_KB * g * BKN,              # every slice 32 blocks: one mid-loop flush, the second skipped
        "flush_16k_plus_1": (FLUSH_KB + 1) * g * BKN,     # every slice 17 blocks
        "flush_rem": (50 * g + g // 3) * BKN,             # slices of 50 and 51 blocks: three mid-loop flushes each
        "ragged": (20 * g + 7) * BKN - 23,                # last block 41 rows long
        "products": PRODUCTS_ROWS,                        # 38,267 blocks, the last one 5 rows long
    }


@pytest.mark.parametrize("sms", [132, 114])       # H100 SXM, H100 PCIe
def test_flush_geometry_covers_every_case(sms):
    assert -(-PRODUCTS_ROWS // BKN) == 38_267 and PRODUCTS_ROWS - 38_266 * BKN == 5
    for m_blocks in (1, 2):
        rc = row_counts(m_blocks, sms)
        assert set(rc) == set(CATEGORIES)
        for cat, rows in rc.items():
            assert cat in categories_of(rows, m_blocks, sms), f"{rows} rows, m_blocks={m_blocks}, {sms} SMs: not {cat}"
            # {-2..2} operands below the products row count, {-1, 0, 1} at it: every exact sum stays under 2^22
            assert rows * (1 if cat == "products" else 4) < EXACT_LIMIT
        # the products row count itself flushes several times over unequal slices
        assert {"flush_rem", "ragged"} <= categories_of(PRODUCTS_ROWS, m_blocks, sms)
    assert node_slices(PRODUCTS_ROWS, 2, 132) == (579, 53, 66)
    assert node_slices(PRODUCTS_ROWS, 1, 132) == (289, 119, 132)


# ------------------------------------------------------------------------------------------------
# fixtures and references
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def K():
    from sgformer_b200 import kernels
    return kernels


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ints(rows, cols, lo, hi, seed, dtype=torch.bfloat16):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randint(lo, hi + 1, (rows, cols), generator=g, device=DEV, dtype=torch.int8).to(dtype)


@pytest.fixture(scope="module")
def mem0():
    """Device memory held when this module starts; test_peak_device_memory reports the module's peak above it."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    return torch.cuda.memory_allocated()


@pytest.fixture(scope="module")
def big(mem0):
    """Two [products rows, 256] bf16 operands in {-1, 0, 1}: |sum over all rows| <= 2,449,029 < 2^22."""
    return _ints(PRODUCTS_ROWS, 256, -1, 1, 1), _ints(PRODUCTS_ROWS, 256, -1, 1, 2)


@pytest.fixture(scope="module")
def small(mem0, sms):
    """Two bf16 operands in {-2, ..., 2} covering every generated row count below the products one (rows * 4 < 2^22)."""
    rows = max(r for mb in (1, 2) for c, r in row_counts(mb, sms).items() if c != "products")
    assert rows * 4 < EXACT_LIMIT
    return _ints(rows, 256, -2, 2, 3), _ints(rows, 256, -2, 2, 4)


def _operands(big, small, rows):
    x, y = big if rows == PRODUCTS_ROWS else small
    return x[:rows], y[:rows]


def ref_tn(a_cols, b_cols):
    """fp64 sum_p a_p^T b_p over row chunks; a_cols / b_cols: equally long lists of [rows, m] / [rows, n] device views."""
    rows = a_cols[0].shape[0]
    out = torch.zeros(a_cols[0].shape[1], b_cols[0].shape[1], dtype=torch.float64, device=DEV)
    for i in range(0, rows, CHUNK):
        for a, b in zip(a_cols, b_cols):
            out += a[i:i + CHUNK].double().t() @ b[i:i + CHUNK].double()
    return out


def _equal(got, want, what):
    if not torch.equal(got, want):
        bad = (got != want)
        i = bad.nonzero()[0].tolist()
        pytest.fail(f"{what}: {int(bad.sum())} of {got.numel()} elements differ; first at {i}: {got[tuple(i)].item()} "
                    f"vs {want[tuple(i)].item()}")


# ------------------------------------------------------------------------------------------------
# gemm_tn
# ------------------------------------------------------------------------------------------------
TN_SHAPES = [(256, 256), (256, 100), (47, 256), (256, 47), (128, 16), (129, 200)]


@pytest.mark.gpu
@pytest.mark.parametrize("cat", CATEGORIES)
@pytest.mark.parametrize("m,n", TN_SHAPES)
def test_gemm_tn_exact(K, sms, big, small, m, n, cat):
    """Single-plane bf16 gemm_tn == the exact integer A^T B at every flush geometry; a second run is bit-identical."""
    rows = row_counts((m + 127) // 128, sms)[cat]
    x, y = _operands(big, small, rows)
    a, b = x[:, :m], y[:, :n]
    A, B = K.operand_from_bf16(a), K.operand_from_bf16(b)
    out = torch.empty(m, n, device=DEV)
    K.gemm_tn(A, B, out)
    _equal(out, ref_tn([a], [b]).float(), f"gemm_tn {rows} rows, m={m} n={n}")
    out2 = torch.empty(m, n, device=DEV)
    K.gemm_tn(A, B, out2)
    assert torch.equal(out, out2), "gemm_tn must be run-to-run deterministic"


@pytest.mark.gpu
@pytest.mark.parametrize("cat", ["flush_rem", "ragged", "products"])
def test_gemm_tn_epilogue_exact(K, sms, big, small, cat):
    """transpose_out, beta = 1 accumulation into an integer output and a device alpha: out^T = 0.25 * 2 * A^T B + C."""
    m, n = 256, 100
    rows = row_counts(2, sms)[cat]
    x, y = _operands(big, small, rows)
    a, b = x[:, :m], y[:, :n]
    c = _ints(n, m, -8, 8, 5, torch.float32)
    out = c.clone()
    K.gemm_tn(K.operand_from_bf16(a), K.operand_from_bf16(b), out, transpose_out=True, alpha=0.25, beta=1.0,
              alpha_dev=torch.tensor([2.0], device=DEV))
    _equal(out, (0.5 * ref_tn([a], [b]).t() + c.double()).float(), f"gemm_tn transposed, {rows} rows")


@pytest.mark.gpu
@pytest.mark.parametrize("cat", ["flush_16k_plus_1", "products"])
def test_gemm_tn_into_column_slices(K, sms, big, small, cat):
    """The GraphConv use_init weight gradient: dw[:, :h] = dz^T y and dw[:, h:] = dz^T x0 into one [h, 2h] tensor."""
    h = 256
    rows = row_counts(2, sms)[cat]
    x, y = _operands(big, small, rows)
    dz, yy, x0 = x, y, x.flip(1)          # x0: a third operand that differs from both
    dw = torch.full((h, 2 * h), 7.0, device=DEV)
    dz_op = K.operand_from_bf16(dz)
    K.gemm_tn(dz_op, K.operand_from_bf16(yy), dw[:, :h])
    x0c = x0.contiguous()
    K.gemm_tn(dz_op, K.operand_from_bf16(x0c), dw[:, h:])
    _equal(dw[:, :h], ref_tn([dz], [yy]).float(), "dw[:, :h]")
    _equal(dw[:, h:], ref_tn([dz], [x0c]).float(), "dw[:, h:]")


@pytest.mark.gpu
@pytest.mark.parametrize("cat", ["no_flush", "flush_16k", "flush_rem", "ragged"])
@pytest.mark.parametrize("m,n", [(256, 100), (47, 256)])
def test_gemm_tn_three_planes_exact(K, sms, m, n, cat):
    """bf16x3 operands: the six plane pairs of kernels._PAIRS3 accumulate in one launch.  Each plane holds its own integers in
    {-1, 0, 1} (as if a bf16x3 split had produced them), so a pair read from the wrong plane, a missing or a doubled pair
    changes the exact result: sum over the six pairs of A_pa^T B_pb (|.| <= 6 rows < 2^22)."""
    from sgformer_b200.kernels import _PAIRS3, Operand
    rows = row_counts((m + 127) // 128, sms)[cat]
    assert 6 * rows < EXACT_LIMIT
    kpa, kpb = -(-m // 64) * 64, -(-n // 64) * 64
    ad, bd = _ints(rows, 3 * kpa, -1, 1, 6), _ints(rows, 3 * kpb, -1, 1, 7)
    for p in range(3):                    # zero K padding, as sgf_pack_operand leaves it
        ad[:, p * kpa + m:(p + 1) * kpa] = 0
        bd[:, p * kpb + n:(p + 1) * kpb] = 0
    A, B = Operand(ad, rows, m, kpa, 3), Operand(bd, rows, n, kpb, 3)
    out = torch.empty(m, n, device=DEV)
    K.gemm_tn(A, B, out)
    ref = ref_tn([ad[:, pa * kpa:pa * kpa + m] for pa, _ in _PAIRS3], [bd[:, pb * kpb:pb * kpb + n] for _, pb in _PAIRS3])
    _equal(out, ref.float(), f"gemm_tn bf16x3 {rows} rows, m={m} n={n}")


@pytest.mark.gpu
def test_gemm_tn_three_planes_fp32_bound(K, sms):
    """bf16x3 products of full fp32 values (24 significant bits, in [1, 2)) at the arxiv row count, against fp64.

    Bound, per output element, as a multiple of S = sum |a||b| (= the result here, as all values are positive):
      * splitting: a - (hi + mid + lo) and the three dropped plane pairs (1,2), (2,1), (2,2) cost at most 5 * 2^-24 |a||b|
        per product (each bf16 rounding keeps 8 significant bits);
      * accumulation: a product passes through at most D fp32 additions, each off by at most 2^-23 relative (allowing for
        truncation): D = 2 * 6 * 4 * FLUSH_KB (two roundings per wgmma k-step, six pairs, four k-steps per node block, FLUSH_KB
        blocks between flushes) + the flushes of a slice + the slices summed by the reduction + 1 for alpha.
    |err| <= (5 * 2^-24 + D * 2^-23) * S, about 1.2e-4 S.  A missing middle plane would cost about 2^-9 S."""
    rows, m, n = 169_343, 256, 256
    g = torch.Generator(device=DEV).manual_seed(8)
    a = 1.0 + torch.rand(rows, m, generator=g, device=DEV)
    b = 1.0 + torch.rand(rows, n, generator=g, device=DEV)
    out = torch.empty(m, n, device=DEV)
    K.gemm_tn(K.pack_operand(a, False, 3), K.pack_operand(b, False, 3), out)
    ref, s = ref_tn([a], [b]), ref_tn([a.abs()], [b.abs()])
    per, rem, grid = node_slices(rows, 2, sms)
    d = 2 * 6 * 4 * FLUSH_KB + (per + 1) // FLUSH_KB + grid + 1
    bound = (5 * 2.0 ** -24 + d * 2.0 ** -23) * s
    err = (out.double() - ref).abs()
    assert bool((err <= bound).all()), f"max err / S = {(err / s).max().item():.3e}, bound {(bound / s).max().item():.3e}"


# ------------------------------------------------------------------------------------------------
# gram
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cat", CATEGORIES)
@pytest.mark.parametrize("h", [16, 64, 100, 128, 200, 256])
def test_gram_exact(K, sms, big, small, h, cat):
    """sgf_gram: G = X^T X (both triangles: the lower block triangle is mirrored) and s = X^T 1, exactly, at every flush
    geometry of both warpgroup layouts (m_blocks 1 for h <= 128, 2 above)."""
    rows = row_counts(2 if h > 128 else 1, sms)[cat]
    x, _ = _operands(big, small, rows)
    xv = x[:, :h]
    G, s = K.gram(K.operand_from_bf16(xv), xv)
    _equal(G, ref_tn([xv], [xv]).float(), f"G, {rows} rows, h={h}")
    s_ref = torch.zeros(h, dtype=torch.float64, device=DEV)
    for i in range(0, rows, CHUNK):
        s_ref += xv[i:i + CHUNK].double().sum(0)
    _equal(s, s_ref.float(), f"s, {rows} rows, h={h}")


# ------------------------------------------------------------------------------------------------
# gemm_nt: every compiled epilogue instantiation
# ------------------------------------------------------------------------------------------------
# Host geometry of sgf_gemm_nt (gemm_tc.cu), restated to decide which kernel a call runs.
NT_BK, NT_RES_BYTES, NT_RES_MAX_KB = 64, (256 + 16) * 256 * 2, 16


def nt_blocks(n_out: int, total_kb: int, has_tail: bool, schedule: int):
    """-> (n_blocks, bn_main) of one sgf_gemm_nt call (schedule 0 auto, 1 streaming B, 2 resident B)."""
    n16 = -(-n_out // 16) * 16
    n_blocks = -(-n16 // 256)
    if has_tail and n16 + 16 > 256:
        one = schedule != 1 and n16 <= 256 and total_kb <= NT_RES_MAX_KB and \
            (-(-n16 // 64) * 64 + 16) * NT_BK * 2 * total_kb <= NT_RES_BYTES
        if not one:
            n_blocks = 2
    bn = n16 if n_blocks == 1 else (n16 // n_blocks + 63) // 64 * 64
    n_blocks = -(-n16 // bn)
    if schedule == 2 and not has_tail:
        bn_pad = -(-bn // 64) * 64
        while bn_pad * NT_BK * 2 * total_kb > NT_RES_BYTES and bn > 64:
            bn = bn_pad = bn_pad - 64
            n_blocks = -(-n16 // bn)
    return n_blocks, bn


def fast_ok(out, n_out, total_kb, schedule, bias=None, aux=None, r1_col=None, tail=None):
    """Whether sgf_gemm_nt runs a feature-specialised kernel rather than F_GENERIC (gemm_tc.cu `fast_ok`); no column statistics."""
    es = out.element_size()
    tma_store = out.data_ptr() % 16 == 0 and (out.stride(0) * es) % 16 == 0
    al16 = (bias is None or bias.data_ptr() % 16 == 0) and (r1_col is None or r1_col.data_ptr() % 16 == 0) and \
        (aux is None or (aux.dtype == torch.bfloat16 and aux.data_ptr() % 16 == 0 and (aux.stride(0) * 2) % 16 == 0))
    nb, bn = nt_blocks(n_out, total_kb, tail is not None, schedule)
    return tma_store and out.dtype == torch.bfloat16 and n_out % 32 == 0 and al16 and nb * bn == n_out


# feature set -> keyword arguments of K.gemm_nt (strings name the tensors the test prepares), with the engine.py call sites
# that reach each set in the bf16 step:
#   0               stem / head / GCN input gradients, the first dx0 of the GraphConv backward (gconv_backward)
#   BIAS            input Linear fcs.0 (_stem_forward, gconv_forward), GraphConv layer without use_init
#   BIAS|RELU       no engine call site (kernel API)
#   ROWSCALE        dys = (dz W) . dinv (gconv_backward), GCN forward x W^T . dinv (gcn_forward)
#   ACCUM           dx0 += dz W_x0 (gconv_backward), TransConv dprev += dqkv W (trans_backward)
#   AUX             dv of the attention backward without accumulation (attention_backward)
#   AUX|ACCUM       dv with accumulation (attention_backward)
#   AUX|BIAS        dk (attention_backward)
#   AUX|R1          dq (attention_backward)
#   AUX|ATTN        attention apply (attention_forward)
#   BIAS|ATTN       Gram-form attention apply (attention_gram_forward)
#   BIAS|R1         Gram-form attention dx (attention_gram_backward, accumulate=False)
#   BIAS|R1|ACCUM   Gram-form attention dx (attention_gram_backward, accumulate=True)
#   GENERIC         fp32 outputs (head logits), unaligned or ragged widths, BIAS|ROWSCALE (_difformer_v_scaled)
#   BIAS_use_init   GraphConv use_init forward [y || x0] . W^T (gconv_forward): two A sources, K = 512
NT_CASES = {
    "0": dict(),
    "BIAS": dict(bias="bias"),
    "BIAS|RELU": dict(bias="bias", relu=True),
    "ROWSCALE": dict(row_scale="rs"),
    "ACCUM": dict(accumulate=True),
    "AUX": dict(aux="aux", alpha=2.0, beta=0.5),
    "AUX|ACCUM": dict(aux="aux", alpha_dev="half", beta=4.0, accumulate=True),
    "AUX|BIAS": dict(aux="aux", alpha_dev="half", beta=1.0, beta_dev="minus2", bias="bias"),
    "AUX|R1": dict(aux="aux", alpha_dev="two", beta=1.0, beta_dev="quarter", r1_row="r1r", r1_col="r1c"),
    "AUX|ATTN": dict(epi=1, aux="aux", tail="tail", nf=300.0, den_out="den"),
    "BIAS|ATTN": dict(epi=2, bias="bias", tail="tail", nf_dev="nf300", den_out="den"),
    "BIAS|R1": dict(bias="bias", r1_row="r1r", r1_col="r1c"),
    "BIAS|R1|ACCUM": dict(bias="bias", r1_row="r1r", r1_col="r1c", accumulate=True),
    "GENERIC": dict(out_dtype=torch.float32, bias="bias", aux="aux", row_scale="rs", alpha=0.5, beta=2.0, alpha_dev="two",
                    beta_dev="minus2", relu=True, accumulate=True, r1_row="r1r", r1_col="r1c"),
    "BIAS_use_init": dict(bias="bias", use_init=True),
}
NT_ROWS = {"products": PRODUCTS_ROWS, "partial_tile": 77_777}      # 2,449,029 = 19,132 tiles of 128 + 5 rows; 77,777 = 607 + 81


def _nt_expect(kw, t, acc, r0, r1):
    """fp64 epilogue of rows [r0, r1) on the exact product acc, as the kernel states it (gemm_tc.cu gemm_nt_kernel)."""
    if kw.get("epi"):
        num = acc.clone()
        if "aux" in kw:
            num += kw["nf"] * t["aux"][r0:r1].double()
        if "bias" in kw:
            num += t["bias"].double()
        return num, (kw["nf"] if "nf" in kw else float(t[kw["nf_dev"]]))
    alpha = kw.get("alpha", 1.0) * (float(t[kw["alpha_dev"]]) if "alpha_dev" in kw else 1.0)
    beta = kw.get("beta", 0.0) * (float(t[kw["beta_dev"]]) if "beta_dev" in kw else 1.0)
    x = acc * alpha
    if "aux" in kw:
        x += beta * t["aux"][r0:r1].double()
    if "bias" in kw:
        x += t["bias"].double()
    if "r1_row" in kw:
        x += t["r1r"][r0:r1, None].double() * t["r1c"].double()
    if kw.get("relu"):
        x.clamp_(min=0.0)
    if "row_scale" in kw:
        x *= t["rs"][r0:r1, None].double()
    if kw.get("accumulate"):
        x += t["old"][r0:r1].double()
    return x, None


@pytest.mark.gpu
@pytest.mark.parametrize("schedule", [1, 2])
@pytest.mark.parametrize("rows_kind", list(NT_ROWS))
@pytest.mark.parametrize("feat", list(NT_CASES))
def test_gemm_nt_epilogue_exact(K, big, small, feat, rows_kind, schedule):
    """Each feature set sgf_gemm_nt compiles a kernel for (and F_GENERIC) against the fp64 epilogue of the exact product,
    under the streaming and the resident-B schedule.  The operands satisfy `fast_ok` for every specialised set (asserted), so
    the specialised kernel is the one that runs.  Affine epilogues are exact; the two ATTN sets divide, and are compared
    with fp64 to within one bf16 ulp (their denominators, written to den_out, are exact)."""
    kw = dict(NT_CASES[feat])
    rows = NT_ROWS[rows_kind]
    x, y = _operands(big, small, rows)
    n_out, k = 256, 256
    g = torch.Generator(device=DEV).manual_seed(rows + len(feat))
    w = _ints(n_out, 2 * k, -2, 2, 9)
    t = dict(bias=_ints(1, n_out, -4, 4, 10, torch.float32)[0], aux=y, r1r=_ints(1, rows, -2, 2, 11, torch.float32)[0],
             r1c=_ints(1, n_out, -3, 3, 12, torch.float32)[0],
             rs=torch.pow(2.0, torch.randint(-2, 3, (rows,), generator=g, device=DEV).float()),
             half=torch.tensor([0.5], device=DEV), two=torch.tensor([2.0], device=DEV),
             quarter=torch.tensor([0.25], device=DEV), minus2=torch.tensor([-2.0], device=DEV),
             nf300=torch.tensor([300.0], device=DEV), den=torch.empty(rows, device=DEV))
    tail = torch.zeros(16, k, dtype=torch.bfloat16, device=DEV)
    tail[0] = _ints(1, k, 0, 1, 13)[0]                           # den = A . tail_0 + 300 lies in [44, 556]
    t["tail"] = tail
    out_dtype = kw.pop("out_dtype", torch.bfloat16)
    use_init = kw.pop("use_init", False)
    if use_init:                                                 # [y || x0] . W^T: two A sources, K = 512
        A, pairs, wk = [K.operand_from_bf16(x), K.operand_from_bf16(y)], [(0, 0, 0, 0, k), (1, 0, 0, k, k)], w
    else:
        A, pairs, wk = [K.operand_from_bf16(x)], [(0, 0, 0, 0, k)], w[:, :k].contiguous()
    total_kb = sum(-(-p[4] // NT_BK) for p in pairs)
    out = K.alloc_act(rows, n_out, out_dtype, DEV)
    if kw.get("accumulate"):
        out.copy_(y)                                             # integers: exact in bf16 and fp32
        t["old"] = y
    args = {name: (t[v] if isinstance(v, str) else v) for name, v in kw.items()}
    if "tail" in args:
        args["tail"] = K.operand_from_bf16(tail)
    specialised = fast_ok(out, n_out, total_kb, schedule, bias=args.get("bias"), aux=args.get("aux"),
                          r1_col=args.get("r1_col"), tail=args.get("tail"))
    assert specialised == (feat != "GENERIC"), f"{feat}: fast_ok = {specialised}"
    K.gemm_nt(A, [K.operand_from_bf16(wk)], pairs, n_out, out, schedule=schedule, **args)

    wd = wk.double()
    for r0 in range(0, rows, CHUNK):
        r1 = min(rows, r0 + CHUNK)
        if use_init:
            acc = x[r0:r1].double() @ wd[:, :k].t() + y[r0:r1].double() @ wd[:, k:].t()
        else:
            acc = x[r0:r1].double() @ wd.t()
        want, nf = _nt_expect(kw, t, acc, r0, r1)
        got = out[r0:r1]
        if nf is None:
            _equal(got, want.to(out_dtype) if out_dtype == torch.float32 else want.float().to(out_dtype),
                   f"{feat} rows [{r0}, {r1})")
            continue
        den = x[r0:r1].double() @ tail[0].double() + nf
        _equal(t["den"][r0:r1], den.float(), f"{feat} den_out rows [{r0}, {r1})")
        ref = want / den[:, None]
        ulp = torch.pow(2.0, torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -100))) - 7)
        err = (got.double() - ref).abs()
        assert bool((err <= ulp).all()), f"{feat} rows [{r0}, {r1}): max error {(err / ulp).max().item():.2f} bf16 ulp"


@pytest.mark.gpu
def test_peak_device_memory(mem0):
    """The module keeps its device memory under 16 GiB above what it found (the GPU is shared)."""
    peak = torch.cuda.max_memory_allocated() - mem0
    print(f"test_gpu_scale: peak device memory {peak / 2 ** 30:.2f} GiB above the module's start")
    assert peak < 16 * 2 ** 30
