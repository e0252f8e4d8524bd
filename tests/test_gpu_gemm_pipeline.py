"""The wgmma GEMMs with their MMAs kept in flight across k-blocks, the red.add flush of gemm_tn / gram and the deeper A ring of
gemm_nt's resident-B schedule, checked bit for bit:

* gemm_tn and gram against their per-slice, per-flush-window sums restated in fp64 (integer operands: every partial is an
  exact integer, so any lost, doubled or misplaced window, flush or slice changes the result), at row counts where a flush falls
  on the last block of a slice and at the products row count;
* gemm_nt's accumulate, addend and fp32-head epilogues (the resident schedule with 4 and 8 ring stages) against exact integer
  products at the products row count;
* two replays of a CUDA-graph-captured products-shaped forward + backward give byte-identical logits and gradients.
"""
import pytest
import torch

from tests.test_gpu_scale import BKN, FLUSH_KB, PRODUCTS_ROWS, node_slices, row_counts

DEV = "cuda"


def _ints(rows, cols, lo, hi, seed, dtype=torch.bfloat16):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randint(lo, hi + 1, (rows, cols), generator=g, device=DEV, dtype=torch.int8).to(dtype)


@pytest.fixture(scope="module")
def K():
    from sgformer_b200 import kernels
    return kernels


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def ops():
    """[products rows, 256] bf16 operands in {-1, 0, 1}: every sum below stays under 2^22 in magnitude."""
    return _ints(PRODUCTS_ROWS, 256, -1, 1, 11), _ints(PRODUCTS_ROWS, 256, -1, 1, 12)


def restated_tn(a, b, m_blocks, sms):
    """sum over slices (in slice order) of the sum over flush windows (in window order) of the window's a^T b, as the kernel
    splits the node range: slices of `per` or `per + 1` node blocks, a flush every FLUSH_KB blocks of a slice."""
    rows = a.shape[0]
    per, rem, grid = node_slices(rows, m_blocks, sms)
    kb_total = -(-rows // BKN)
    out = torch.zeros(a.shape[1], b.shape[1], dtype=torch.float64, device=DEV)
    kb = 0
    for y in range(grid):
        n = per + (1 if y < rem else 0)
        part = torch.zeros_like(out)
        for w0 in range(0, n, FLUSH_KB):
            r0, r1 = (kb + w0) * BKN, min((kb + min(n, w0 + FLUSH_KB)) * BKN, rows)
            part += a[r0:r1].double().t() @ b[r0:r1].double()
        out += part
        kb += n
    assert kb == kb_total
    return out


def _cats(m_blocks, sms):
    rc = row_counts(m_blocks, sms)
    return {"flush_on_last_block": rc["flush_16k"], "products": PRODUCTS_ROWS}


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["flush_on_last_block", "products"])
@pytest.mark.parametrize("m,n", [(256, 256), (256, 100), (47, 256)])
def test_gemm_tn_restated_order(K, sms, ops, m, n, where):
    rows = _cats((m + 127) // 128, sms)[where]
    a, b = ops[0][:rows, :m], ops[1][:rows, :n]
    out = torch.empty(m, n, device=DEV)
    K.gemm_tn(K.operand_from_bf16(a), K.operand_from_bf16(b), out)
    want = restated_tn(a, b, (m + 127) // 128, sms).float()
    assert torch.equal(out, want), f"{int((out != want).sum())} of {out.numel()} elements differ"


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["flush_on_last_block", "products"])
def test_gram_restated_order(K, sms, ops, where):
    rows = _cats(2, sms)[where]
    x = ops[0][:rows]
    G, s = K.gram(K.operand_from_bf16(x), x)
    want = restated_tn(x, x, 2, sms)
    assert torch.equal(G, want.float())
    ones = torch.ones(rows, 1, dtype=torch.bfloat16, device=DEV)
    assert torch.equal(s, restated_tn(x, ones, 2, sms)[:, 0].float())


@pytest.mark.gpu
def test_gemm_nt_resident_ring_epilogues_exact(K, ops):
    """Resident-B gemm_nt at the products row count: accumulate and addend (4 ring stages beside a 256-wide B), the fp32 47-class
    head (8 stages beside a 64-wide B).  Integer operands, |result| <= 256 + 8: exact in bf16 and fp32."""
    x, v = ops
    rows, h = PRODUCTS_ROWS, 256
    w = _ints(h, h, -1, 1, 13).float()
    w[:, 128:] = 0                                         # |x . w| <= 128
    W = K.pack_operand(w, False, 1)
    X = K.operand_from_bf16(x)
    exact = (x.float() @ w.t())                            # exact: integers below 2^24
    old = _ints(rows, h, -8, 8, 14)
    out = K.alloc_act(rows, h, torch.bfloat16, DEV)
    out.copy_(old)
    K.gemm_nt([X], [W], [(0, 0, 0, 0, h)], h, out, accumulate=True)
    assert torch.equal(out.float(), exact + old.float()), "accumulate"
    out2 = K.alloc_act(rows, h, torch.bfloat16, DEV)
    K.gemm_nt([X], [W], [(0, 0, 0, 0, h)], h, out2, aux=v, beta=1.0)
    assert torch.equal(out2.float(), exact + v.float()), "aux"
    w47 = _ints(47, h, -1, 1, 15).float()
    bias = _ints(1, 47, -4, 4, 16, torch.float32)[0]
    out47 = torch.empty(rows, 47, device=DEV)
    K.gemm_nt([X], [K.pack_operand(w47, False, 1)], [(0, 0, 0, 0, h)], 47, out47, bias=bias)
    assert torch.equal(out47, x.float() @ w47.t() + bias), "fp32 head"


@pytest.mark.gpu
def test_captured_products_step_replays_bit_identical():
    """Forward + loss + backward of the products-shaped model (bench.py's configuration, no dropout) captured in a CUDA graph:
    two replays write byte-identical logits and gradients."""
    from sgformer_b200 import large as L
    from sgformer_b200.loss import nll_loss_from_logits
    from sgformer_b200.synth import make_graph
    n, d, e, c, h = PRODUCTS_ROWS, 100, 61_859_140, 47, 256
    torch.manual_seed(1234)
    ei = make_graph(n, e, seed=100, device=DEV)
    g = torch.Generator(device=DEV).manual_seed(7)
    x = torch.randn(n, d, generator=g, device=DEV)
    y = torch.randint(0, c, (n,), generator=g, device=DEV)
    model = L.SGFormer(d, h, c, trans_num_layers=1, trans_num_heads=1, trans_dropout=0.0, trans_use_bn=True,
                       trans_use_residual=True, trans_use_weight=True, trans_use_act=False, gnn_num_layers=3, gnn_dropout=0.0,
                       gnn_use_weight=True, gnn_use_init=True, gnn_use_bn=True, gnn_use_residual=True, gnn_use_act=True,
                       use_graph=True, graph_weight=0.5, aggregate="add").to(DEV).set_precision("bf16")
    model.train()
    last = {}

    def step():
        model.zero_grad(set_to_none=True)
        out = model(x, ei)
        nll_loss_from_logits(out, y, None, float(n)).backward()
        last["out"] = out.detach()

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    cg = torch.cuda.CUDAGraph()
    with torch.cuda.graph(cg):
        step()
    params = [p for p in model.parameters() if p.grad is not None]
    assert params
    cg.replay()
    torch.cuda.synchronize()
    first = [last["out"].clone()] + [p.grad.clone() for p in params]
    cg.replay()
    torch.cuda.synchronize()
    second = [last["out"]] + [p.grad for p in params]
    for i, (a, b) in enumerate(zip(first, second)):
        assert torch.equal(a, b), f"tensor {i} differs between replays"
