"""Functional (autograd-free) Python wrappers over the C-ABI kernels.

Every function takes CUDA torch tensors, validates layout, and launches on torch's current stream.
Nothing here touches CPU tensors: a non-CUDA tensor raises — there is no fallback path.
"""
from __future__ import annotations

import ctypes as C
import os
import threading
from dataclasses import dataclass
from typing import Optional, Sequence, Tuple

import torch

from . import _lib
from ._lib import BF16, EPI_AFFINE, EPI_ATTN_APPLY, EPI_ATTN_GRAM, F32, AttnGramArgs, GemmNtArgs, GemmTnArgs, check

Tensor = torch.Tensor
_tls = threading.local()


def lib():
    return _lib.load()


def _use(t: Tensor):
    if not t.is_cuda:
        raise RuntimeError("sgformer_b200 kernels need CUDA tensors (no CPU fallback); got device " + str(t.device))
    idx = t.device.index if t.device.index is not None else torch.cuda.current_device()
    if getattr(_tls, "dev", None) != idx:
        check(lib().sgf_set_device(idx), "sgf_set_device")
        _tls.dev = idx


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _p(t: Optional[Tensor]):
    return None if t is None else t.data_ptr()


def dcode(t_or_dtype) -> int:
    dt = t_or_dtype.dtype if isinstance(t_or_dtype, torch.Tensor) else t_or_dtype
    if dt == torch.float32:
        return F32
    if dt == torch.bfloat16:
        return BF16
    raise TypeError(f"unsupported dtype {dt}")


def _mat(t: Tensor, name: str):
    if t.dim() != 2 or t.stride(1) != 1:
        raise ValueError(f"{name}: expected a row-major 2-D tensor, got shape {tuple(t.shape)} stride {t.stride()}")
    return t.shape[0], t.shape[1], t.stride(0)


def _f32vec(t: Optional[Tensor], n: int, name: str):
    if t is None:
        return None
    if t.dtype != torch.float32 or not t.is_contiguous() or t.numel() < n:
        raise ValueError(f"{name}: expected contiguous fp32 with >= {n} elements")
    return t


def ceil_to(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def alloc_act(rows: int, h: int, dtype, device) -> Tensor:
    """[rows, h] activation whose pitch keeps rows 16-byte aligned."""
    mult = 8 if dtype == torch.bfloat16 else 4
    hp = ceil_to(h, mult)
    buf = torch.empty((rows, hp), dtype=dtype, device=device)
    return buf[:, :h] if hp != h else buf


def _out_like(out: Optional[Tensor], x: Tensor, name: str) -> Tensor:
    """`out` checked to have x's shape, dtype and pitch (an output the caller placed, e.g. a column block), or new_like(x)."""
    if out is None:
        return new_like(x)
    if out.shape != x.shape or out.dtype != x.dtype or out.device != x.device or _mat(out, name)[2] != x.stride(0):
        raise ValueError(f"{name}: expected {tuple(x.shape)} {x.dtype} with pitch {x.stride(0)}, got {tuple(out.shape)} {out.dtype} "
                         f"with pitch {out.stride(0)}")
    return out


def new_like(x: Tensor) -> Tensor:
    """Uninitialised activation with the same shape and pitch as the 2-D row-major tensor x."""
    rows, h, ld = _mat(x, "x")
    if ld == h:
        return torch.empty((rows, h), dtype=x.dtype, device=x.device)
    return torch.empty((rows, ld), dtype=x.dtype, device=x.device)[:, :h]


# ------------------------------------------------------------------------------------------------
# graph structure
# ------------------------------------------------------------------------------------------------
def csr_build(edge_index: Tensor, n: int, by_source: bool = False, self_loop_mode: int = 0, want_dinv: bool = True,
              rows: Optional[Tuple[int, int]] = None, col_rot: Optional[Tuple[int, int]] = None):
    """-> (rowptr int64 [n_rows+1], col int32 [nnz'], dinv fp32 [n_rows] | None).  See sgf_csr_build(_rect).
    `rows=(r0, r1)` builds only that row range of the n x n pattern (row shard; column ids stay global).
    `col_rot=(rot, mod)` stores the column ids rotated, (col - rot) mod `mod`, and sorts the rows by them (sgf_csr_build_rot)."""
    _use(edge_index)
    if edge_index.dtype != torch.int64 or edge_index.dim() != 2 or edge_index.shape[0] != 2:
        raise ValueError("edge_index must be int64 [2, nnz]")
    ei = edge_index.contiguous()
    nnz = ei.shape[1]
    dev = ei.device
    r0, r1 = rows if rows is not None else (0, n)
    n_cols, n = n, r1 - r0
    cap = nnz + (n if self_loop_mode == 1 else 0)
    rowptr = torch.empty(n + 1, dtype=torch.int64, device=dev)
    col = torch.empty(max(cap, 1), dtype=torch.int32, device=dev)
    dinv = torch.empty(max(n, 1), dtype=torch.float32, device=dev) if (want_dinv and not by_source) else None
    nbytes = C.c_size_t(0)
    check(lib().sgf_csr_build_ws_bytes(nnz, n, C.byref(nbytes)), "sgf_csr_build_ws_bytes")
    ws = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=dev)
    rot, mod = col_rot if col_rot is not None else (0, 0)
    check(lib().sgf_csr_build_rot(_p(ei), nnz, r0, r1, n_cols, int(by_source), self_loop_mode, rot, mod, _p(rowptr), _p(col),
                                  _p(dinv), _p(ws), nbytes.value, _stream()), "sgf_csr_build_rot")
    if self_loop_mode == 1 or rows is not None:
        total = int(rowptr[n].item())
        col = col[:total]
    else:
        col = col[:nnz]
    return rowptr, col, (dinv[:n] if dinv is not None else None)


def edge_weight_vec(edge_weight: Tensor, nnz: int) -> Tensor:
    """edge_weight as contiguous fp32 [nnz] (other floating dtypes are cast, as the drivers pass fp32)."""
    _use(edge_weight)
    if edge_weight.dim() != 1 or edge_weight.numel() != nnz or not edge_weight.dtype.is_floating_point:
        raise ValueError(f"edge_weight must be a floating [nnz={nnz}] vector (multi-dimensional edge_attr is not supported); "
                         f"got {edge_weight.dtype} {tuple(edge_weight.shape)}")
    return edge_weight.detach().to(torch.float32).contiguous()


def csr_build_weighted(edge_index: Tensor, edge_weight: Tensor, n: int, by_source: bool = False, self_loop_mode: int = 0,
                       want_dinv: bool = True):
    """-> (rowptr int64 [n+1], col int32 [nnz'], eid int64 [nnz'], val fp32 [nnz'], dinv fp32 [n] | None): the weighted CSR of
    sgf_csr_build_weighted (rows sorted by (col, eid); self_loop_mode 1: the added loop carries the weight of the node's last self
    loop; dinv = weighted deg^-1/2 in mode 1, the count-based one in mode 0)."""
    _use(edge_index)
    if edge_index.dtype != torch.int64 or edge_index.dim() != 2 or edge_index.shape[0] != 2:
        raise ValueError("edge_index must be int64 [2, nnz]")
    ei = edge_index.contiguous()
    nnz = ei.shape[1]
    w = edge_weight_vec(edge_weight, nnz)
    dev = ei.device
    cap = max(nnz + (n if self_loop_mode == 1 else 0), 1)
    rowptr = torch.empty(n + 1, dtype=torch.int64, device=dev)
    col = torch.empty(cap, dtype=torch.int32, device=dev)
    eid = torch.empty(cap, dtype=torch.int64, device=dev)
    val = torch.empty(cap, dtype=torch.float32, device=dev)
    dinv = torch.empty(max(n, 1), dtype=torch.float32, device=dev) if want_dinv else None
    nbytes = C.c_size_t(0)
    check(lib().sgf_csr_build_weighted_ws_bytes(nnz, n, C.byref(nbytes)), "sgf_csr_build_weighted_ws_bytes")
    ws = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=dev)
    check(lib().sgf_csr_build_weighted(_p(ei), _p(w), nnz, n, int(by_source), self_loop_mode, _p(rowptr), _p(col), _p(eid), _p(val),
                                       _p(dinv), _p(ws), nbytes.value, _stream()), "sgf_csr_build_weighted")
    total = int(rowptr[n].item()) if self_loop_mode == 1 else nnz      # mode 1: existing self loops dropped (one device sync)
    return rowptr, col[:total], eid[:total], val[:total], (dinv[:n] if dinv is not None else None)


def edge_symmetry_weighted(edge_index: Tensor, edge_weight: Tensor, n: int) -> bool:
    """Multiset equality of {(r,c,w)} and {(c,r,w)} (edge_symmetry with the weights' bit patterns hashed along)."""
    ei = _edge_index(edge_index)
    w = edge_weight_vec(edge_weight, ei.shape[1])
    out = torch.empty(2, dtype=torch.int64, device=ei.device)
    check(lib().sgf_edge_symmetry_weighted(_p(ei), _p(w), ei.shape[1], n, _p(out), _stream()), "sgf_edge_symmetry_weighted")
    a, b = out.tolist()
    return a == b


def edge_weight_grad(rowptr: Tensor, col: Tensor, eid: Tensor, a: Tensor, b: Tensor, out: Tensor, y: Optional[Tensor] = None,
                     u: Optional[Tensor] = None, dinv: Optional[Tensor] = None, edge_index: Optional[Tensor] = None,
                     loops: bool = False):
    """out[eid[j]] += <a_c, b_r> (+ the degree term -1/2 dinv_c (<a_c, y_c> + <b_c, u_c>) when y is given) for every CSR entry
    j = (c, r); `loops` (self_loop_mode 1): the added loop's share goes to every self-loop edge of edge_index (sgf_edge_weight_grad)."""
    _use(a)
    n = rowptr.numel() - 1
    _, h, lda = _mat(a, "a")
    _, hb, ldb = _mat(b, "b")
    if hb != h or b.dtype != a.dtype or out.dtype != torch.float32 or not out.is_contiguous():
        raise ValueError("edge_weight_grad: operand shape/dtype mismatch")
    ldy = ldu = 0
    if y is not None:
        _, _, ldy = _mat(y, "y")
        _, _, ldu = _mat(u, "u")
        if y.dtype != a.dtype or u.dtype != a.dtype:
            raise ValueError("edge_weight_grad: y / u dtype mismatch")
    loop_grad = torch.empty(max(n, 1), dtype=torch.float32, device=a.device) if loops else None
    ei = _edge_index(edge_index) if loops else None
    check(lib().sgf_edge_weight_grad(_p(rowptr), _p(col), _p(eid), n, h, dcode(a), _p(a), lda, _p(b), ldb, _p(y), ldy, _p(u), ldu,
                                     _p(_f32vec(dinv, n, "dinv")), _p(ei), out.numel(), _p(loop_grad), _p(out), _stream()),
          "sgf_edge_weight_grad")
    return out


def subgraph(edge_index: Tensor, n: int, subset: Tensor) -> Tensor:
    """Induced subgraph with relabelling; returns int64 [2, nnz_sub] in input edge order (PyG `subgraph` semantics)."""
    _use(edge_index)
    ei = edge_index.contiguous()
    subset = subset.contiguous().to(torch.int64)
    nnz = ei.shape[1]
    dev = ei.device
    node_map = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    out = torch.empty((2, max(nnz, 1)), dtype=torch.int64, device=dev)
    count = torch.zeros(1, dtype=torch.int64, device=dev)
    nbytes = C.c_size_t(0)
    check(lib().sgf_subgraph_ws_bytes(nnz, n, C.byref(nbytes)), "sgf_subgraph_ws_bytes")
    ws = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=dev)
    check(lib().sgf_subgraph(_p(ei), nnz, n, _p(subset), subset.numel(), _p(node_map), _p(out), _p(count), _p(ws),
                             nbytes.value, _stream()), "sgf_subgraph")
    k = int(count.item())
    return out[:, :k]


def _edge_index(edge_index: Tensor) -> Tensor:
    _use(edge_index)
    if edge_index.dtype != torch.int64 or edge_index.dim() != 2 or edge_index.shape[0] != 2:
        raise TypeError("edge_index must be int64 [2, nnz]")
    return edge_index.contiguous()


def edge_symmetry(edge_index: Tensor, n: int) -> bool:
    """Multiset equality of {(r,c)} and {(c,r)} (order-independent 64-bit hash sums, one pass, one device sync)."""
    ei = _edge_index(edge_index)
    out = torch.empty(2, dtype=torch.int64, device=ei.device)
    check(lib().sgf_edge_symmetry(_p(ei), ei.shape[1], n, _p(out), _stream()), "sgf_edge_symmetry")
    a, b = out.tolist()
    return a == b


def to_undirected(edge_index: Tensor, n: int) -> Tensor:
    """K10: PyG to_undirected = every edge in both directions, sorted by (row, col), duplicates removed (bit-exact)."""
    ei = _edge_index(edge_index)
    nnz, dev = ei.shape[1], ei.device
    out = torch.empty((2, max(2 * nnz, 1)), dtype=torch.int64, device=dev)
    count = torch.zeros(1, dtype=torch.int64, device=dev)
    nbytes = C.c_size_t(0)
    check(lib().sgf_to_undirected_ws_bytes(nnz, n, C.byref(nbytes)), "sgf_to_undirected_ws_bytes")
    ws = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=dev)
    check(lib().sgf_to_undirected(_p(ei), nnz, n, _p(out), _p(count), _p(ws), nbytes.value, _stream()), "sgf_to_undirected")
    return out[:, :int(count.item())]


def remove_self_loops(edge_index: Tensor) -> Tensor:
    """K10: PyG remove_self_loops (order-preserving)."""
    ei = _edge_index(edge_index)
    nnz, dev = ei.shape[1], ei.device
    out = torch.empty((2, max(nnz, 1)), dtype=torch.int64, device=dev)
    count = torch.zeros(1, dtype=torch.int64, device=dev)
    nbytes = C.c_size_t(0)
    check(lib().sgf_remove_self_loops_ws_bytes(nnz, C.byref(nbytes)), "sgf_remove_self_loops_ws_bytes")
    ws = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=dev)
    check(lib().sgf_remove_self_loops(_p(ei), nnz, _p(out), _p(count), _p(ws), nbytes.value, _stream()), "sgf_remove_self_loops")
    return out[:, :int(count.item())]


def add_self_loops(edge_index: Tensor, n: int) -> Tensor:
    """K10: PyG add_self_loops(edge_index, num_nodes=n): [edge_index | (i, i) for i < n]."""
    ei = _edge_index(edge_index)
    nnz = ei.shape[1]
    out = torch.empty((2, nnz + n), dtype=torch.int64, device=ei.device)
    check(lib().sgf_add_self_loops(_p(ei), nnz, n, _p(out), _stream()), "sgf_add_self_loops")
    return out


# bench.py sets this to a list to collect (start, end) CUDA events around every SpMM launch (roofline measurement)
spmm_events = None


def csr_subset(rowptr: Tensor, col: Tensor, n: int, subset: Tensor, node_map: Tensor, capacity: Optional[int] = None):
    """Induced-subgraph CSR of `subset` from the full CSR.  -> (rowptr int64 [b+1], col int32 [nnz_b], dinv fp32 [b], needed).
    `capacity` bounds the output nnz (default: a device sync to read the exact sum of the subset rows' lengths); the kernels
    never write past it, and `needed` (device int64 [1]) holds the nnz the untruncated result requires: needed > capacity
    means the batch was truncated (checked without a per-batch sync by RandomPartitionSampler.check)."""
    _use(rowptr)
    subset = subset.contiguous().to(torch.int64)
    b = subset.numel()
    dev = rowptr.device
    trim = capacity is None
    if capacity is None:
        capacity = int((rowptr[subset + 1] - rowptr[subset]).sum().item()) if b else 0
    out_rowptr = torch.empty(b + 1, dtype=torch.int64, device=dev)
    out_col = torch.empty(max(capacity, 1), dtype=torch.int32, device=dev)
    dinv = torch.empty(max(b, 1), dtype=torch.float32, device=dev)
    needed = torch.empty(1, dtype=torch.int64, device=dev)
    nbytes = C.c_size_t(0)
    check(lib().sgf_csr_subset_ws_bytes(b, capacity, C.byref(nbytes)), "sgf_csr_subset_ws_bytes")
    ws = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=dev)
    check(lib().sgf_csr_subset(_p(rowptr), _p(col), n, _p(subset), b, _p(node_map), _p(out_rowptr), _p(out_col), capacity,
                               _p(dinv), _p(needed), _p(ws), nbytes.value, _stream()), "sgf_csr_subset")
    if trim:    # exact-size result (one more device sync); with a caller-provided capacity the tail of `col` is unused
        out_col = out_col[:int(out_rowptr[b].item())]
    return out_rowptr, out_col, dinv[:b], needed


HEAVY_ROW = 1024      # rows longer than this are processed in segments of HEAVY_ROW entries (hub rows of power-law graphs)


@dataclass
class HeavyRows:
    """Segment plan for the rows longer than HEAVY_ROW (built once per CSR by `heavy_rows`)."""
    rows: Tensor       # int64 [nh]
    seg_ptr: Tensor    # int64 [nh+1]
    seg_start: Tensor  # int64 [ns]
    seg_len: Tensor    # int32 [ns]


def heavy_rows(rowptr: Tensor) -> Optional[HeavyRows]:
    """Plan for the hub rows of a CSR, or None when no row exceeds HEAVY_ROW (one device sync; graph-build time)."""
    lens = rowptr[1:] - rowptr[:-1]
    rows = (lens > HEAVY_ROW).nonzero().flatten()
    if rows.numel() == 0:
        return None
    nseg = (lens[rows] + HEAVY_ROW - 1) // HEAVY_ROW
    seg_ptr = torch.zeros(rows.numel() + 1, dtype=torch.int64, device=rowptr.device)
    seg_ptr[1:] = torch.cumsum(nseg, 0)
    owner = torch.repeat_interleave(torch.arange(rows.numel(), device=rowptr.device), nseg)
    k = torch.arange(owner.numel(), device=rowptr.device) - seg_ptr[owner]
    seg_start = rowptr[rows][owner] + k * HEAVY_ROW
    seg_len = torch.minimum(rowptr[rows + 1][owner] - seg_start, torch.full_like(seg_start, HEAVY_ROW)).to(torch.int32)
    return HeavyRows(rows.contiguous(), seg_ptr, seg_start.contiguous(), seg_len.contiguous())


def spmm(rowptr: Tensor, col: Tensor, row_scale: Optional[Tensor], x: Tensor, out: Optional[Tensor] = None,
         heavy: Optional[HeavyRows] = None, val: Optional[Tensor] = None) -> Tensor:
    """y = row_scale (.) A x over the CSR (rowptr, col); `val` (fp32 [nnz]): the weighted CSR's values (sgf_spmm_weighted)."""
    if val is not None:
        return _spmm_weighted(rowptr, col, val, row_scale, x, out, heavy)
    _use(x)
    n = rowptr.numel() - 1
    rows, h, ldx = _mat(x, "x")
    if out is None:
        out = alloc_act(n, h, x.dtype, x.device)
    _, ho, ldy = _mat(out, "out")
    if ho != h or out.dtype != x.dtype:
        raise ValueError("spmm: out shape/dtype mismatch")
    ev = spmm_events
    if ev is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    rs = _f32vec(row_scale, n, "row_scale")
    check(lib().sgf_spmm(_p(rowptr), _p(col), _p(rs), _p(x), ldx, _p(out), ldy, n, h, dcode(x),
                         HEAVY_ROW if heavy is not None else 0, _stream()), "sgf_spmm")
    if heavy is not None:
        ns = heavy.seg_start.numel()
        partial = torch.empty((ns, h), dtype=torch.float32, device=x.device)
        check(lib().sgf_spmm_heavy(_p(col), _p(rs), _p(x), ldx, _p(out), ldy, h, dcode(x), _p(heavy.seg_start),
                                   _p(heavy.seg_len), ns, _p(partial), _p(heavy.rows), _p(heavy.seg_ptr), heavy.rows.numel(),
                                   _stream()), "sgf_spmm_heavy")
    if ev is not None:
        e1.record()
        ev.append((e0, e1))
    return out


def spmm_sum(rowptr: Tensor, col: Tensor, x: Tensor, out: Optional[Tensor] = None, heavy: Optional[HeavyRows] = None) -> Tensor:
    """y = A x over the CSR (rowptr, col) as built: the plain neighbour sum of GCNConv(normalize=False) (sgf_spmm_sum)."""
    _use(x)
    n = rowptr.numel() - 1
    rows, h, ldx = _mat(x, "x")
    if out is None:
        out = alloc_act(n, h, x.dtype, x.device)
    _, ho, ldy = _mat(out, "out")
    if ho != h or out.dtype != x.dtype:
        raise ValueError("spmm_sum: out shape/dtype mismatch")
    ev = spmm_events
    if ev is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    check(lib().sgf_spmm_sum(_p(rowptr), _p(col), _p(x), ldx, _p(out), ldy, n, h, dcode(x), HEAVY_ROW if heavy is not None else 0,
                             _stream()), "sgf_spmm_sum")
    if heavy is not None:
        ns = heavy.seg_start.numel()
        partial = torch.empty((ns, h), dtype=torch.float32, device=x.device)
        check(lib().sgf_spmm_heavy_sum(_p(col), _p(x), ldx, _p(out), ldy, h, dcode(x), _p(heavy.seg_start), _p(heavy.seg_len), ns,
                                       _p(partial), _p(heavy.rows), _p(heavy.seg_ptr), heavy.rows.numel(), _stream()),
              "sgf_spmm_heavy_sum")
    if ev is not None:
        e1.record()
        ev.append((e0, e1))
    return out


def _spmm_weighted(rowptr: Tensor, col: Tensor, val: Tensor, row_scale: Optional[Tensor], x: Tensor, out: Optional[Tensor],
                   heavy: Optional[HeavyRows]) -> Tensor:
    _use(x)
    n = rowptr.numel() - 1
    rows, h, ldx = _mat(x, "x")
    if val.dtype != torch.float32 or not val.is_contiguous() or val.numel() != col.numel():
        raise ValueError("spmm: val must be contiguous fp32 with one value per column id")
    if out is None:
        out = alloc_act(n, h, x.dtype, x.device)
    _, ho, ldy = _mat(out, "out")
    if ho != h or out.dtype != x.dtype:
        raise ValueError("spmm: out shape/dtype mismatch")
    ev = spmm_events
    if ev is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    rs = _f32vec(row_scale, n, "row_scale")
    check(lib().sgf_spmm_weighted(_p(rowptr), _p(col), _p(val), _p(rs), _p(x), ldx, _p(out), ldy, n, h, dcode(x),
                                  HEAVY_ROW if heavy is not None else 0, _stream()), "sgf_spmm_weighted")
    if heavy is not None:
        ns = heavy.seg_start.numel()
        partial = torch.empty((ns, h), dtype=torch.float32, device=x.device)
        check(lib().sgf_spmm_heavy_weighted(_p(col), _p(val), _p(rs), _p(x), ldx, _p(out), ldy, h, dcode(x), _p(heavy.seg_start),
                                            _p(heavy.seg_len), ns, _p(partial), _p(heavy.rows), _p(heavy.seg_ptr),
                                            heavy.rows.numel(), _stream()), "sgf_spmm_heavy_weighted")
    if ev is not None:
        e1.record()
        ev.append((e0, e1))
    return out


def spmm_flagged(rowptr: Tensor, col: Tensor, row_scale: Optional[Tensor], x: Tensor, flags: Tensor, slot_rows: int,
                 heavy: Optional[HeavyRows] = None) -> Tensor:
    """Row-sharded SpMM over the gathered operand x [n_slots*slot_rows, h] whose slots s > 0 are still being pushed by the
    peers: the kernel consumes slot s once flags[s] != 0 (sgf_spmm_flagged).  col holds rotated ids (csr_build(col_rot=...))."""
    _use(x)
    n = rowptr.numel() - 1
    rows, h, ldx = _mat(x, "x")
    n_slots = flags.numel()
    if flags.dtype not in (torch.int32, torch.uint32) or not flags.is_contiguous() or rows != n_slots * slot_rows:
        raise ValueError("spmm_flagged: flags must be contiguous int32 [n_slots] and x must hold n_slots*slot_rows rows")
    out = alloc_act(n, h, x.dtype, x.device)
    _, _, ldy = _mat(out, "out")
    ev = spmm_events
    if ev is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    rs = _f32vec(row_scale, n, "row_scale")
    check(lib().sgf_spmm_flagged(_p(rowptr), _p(col), _p(rs), _p(x), ldx, _p(out), ldy, n, h, dcode(x),
                                 HEAVY_ROW if heavy is not None else 0, _p(flags), slot_rows, n_slots, _stream()), "sgf_spmm_flagged")
    if heavy is not None:
        # hub rows touch every slot: wait for all of them, then the segmented path on the complete operand
        check(lib().sgf_wait_flags(_p(flags[1:]), n_slots - 1, _stream()), "sgf_wait_flags")
        ns = heavy.seg_start.numel()
        partial = torch.empty((ns, h), dtype=torch.float32, device=x.device)
        check(lib().sgf_spmm_heavy(_p(col), _p(rs), _p(x), ldx, _p(out), ldy, h, dcode(x), _p(heavy.seg_start),
                                   _p(heavy.seg_len), ns, _p(partial), _p(heavy.rows), _p(heavy.seg_ptr), heavy.rows.numel(),
                                   _stream()), "sgf_spmm_heavy")
    if ev is not None:
        e1.record()
        ev.append((e0, e1))
    return out


def csr_row_splits(rowptr: Tensor, col: Tensor, thresholds: Sequence[int]) -> Tensor:
    """int32 [len(thresholds), n_rows]: per row the number of entries with column id < threshold (rows sorted by column)."""
    _use(rowptr)
    n = rowptr.numel() - 1
    thr = torch.tensor(list(thresholds), dtype=torch.int32, device=rowptr.device)
    out = torch.empty((len(thresholds), max(n, 1)), dtype=torch.int32, device=rowptr.device)
    check(lib().sgf_csr_row_splits(_p(rowptr), _p(col), n, _p(thr), len(thresholds), _p(out), _stream()), "sgf_csr_row_splits")
    return out[:, :n]


def spmm_range(rowptr: Tensor, col: Tensor, row_scale: Optional[Tensor], x: Tensor, lo: Optional[Tensor], hi: Optional[Tensor],
               part_in: Optional[Tensor], part_out: Optional[Tensor]) -> Optional[Tensor]:
    """One phase of a phased SpMM (sgf_spmm_range): entries [lo, hi) of every row, plus part_in, into part_out (fp32 partials;
    returns None) or, when part_out is None, scaled into a new activation that is returned."""
    _use(x)
    n = rowptr.numel() - 1
    _, h, ldx = _mat(x, "x")
    ev = spmm_events
    if ev is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    out = alloc_act(n, h, x.dtype, x.device) if part_out is None else None
    ldp = (part_in if part_in is not None else part_out).stride(0) if (part_in is not None or part_out is not None) else 0
    for t in (lo, hi):
        if t is not None and (t.dtype != torch.int32 or not t.is_contiguous() or t.numel() < n):
            raise ValueError("spmm_range: lo / hi must be contiguous int32 [n_rows]")
    for t in (part_in, part_out):
        if t is not None and (t.dtype != torch.float32 or t.stride(1) != 1 or t.shape[0] < n or t.shape[1] != h):
            raise ValueError("spmm_range: partials must be fp32 [n_rows, h]")
    rs = _f32vec(row_scale, n, "row_scale") if part_out is None else None
    check(lib().sgf_spmm_range(_p(rowptr), _p(col), _p(rs), _p(x), ldx, _p(out), out.stride(0) if out is not None else 0, n, h,
                               dcode(x), _p(lo), _p(hi), _p(part_in), _p(part_out), ldp, _stream()), "sgf_spmm_range")
    if ev is not None:
        e1.record()
        ev.append((e0, e1))
    return out


def memcpy_async(dst: Tensor, src: Tensor):
    """Stream-ordered raw copy src -> dst (same byte size, both contiguous) on the current stream; dst may be the mapping of a
    peer GPU's symmetric buffer (sgf_memcpy_async: copy engine over NVLink, no cross-device stream synchronisation)."""
    nb = src.numel() * src.element_size()
    if not (dst.is_contiguous() and src.is_contiguous()) or dst.numel() * dst.element_size() != nb:
        raise ValueError("memcpy_async: contiguous tensors of equal byte size expected")
    check(lib().sgf_memcpy_async(_p(dst), _p(src), nb, _stream()), "sgf_memcpy_async")


def wait_flags(flags: Tensor):
    """Returns (on the current stream) once every entry of the int32 vector `flags` is non-zero."""
    if flags.numel():
        check(lib().sgf_wait_flags(_p(flags), flags.numel(), _stream()), "sgf_wait_flags")


_epoch = None


def dropout_epoch(create: bool = True):
    """The device word the dropout kernels add to their seed (sgf_set_dropout_epoch); created and registered on first use."""
    global _epoch
    if _epoch is None and create:
        _epoch = torch.zeros(1, dtype=torch.int64, device="cuda")
        check(lib().sgf_set_dropout_epoch(_p(_epoch)), "sgf_set_dropout_epoch")
    return _epoch


def advance_dropout_epoch():
    """*epoch += 1 on the current stream: call once at the top of a training step that is captured in a CUDA graph, so that
    every replay draws fresh dropout masks (the host seed is frozen into the graph)."""
    check(lib().sgf_advance_dropout_epoch(_p(dropout_epoch()), _stream()), "sgf_advance_dropout_epoch")


def signal(flag: Tensor, value: int = 1):
    """flag[0] = value (release, system scope) on the current stream; `flag` may be a view of a peer GPU's symmetric memory."""
    check(lib().sgf_signal(_p(flag), value, _stream()), "sgf_signal")


# ------------------------------------------------------------------------------------------------
# tensor-core operands
# ------------------------------------------------------------------------------------------------
@dataclass
class Operand:
    """bf16 matrix [rows, k] laid out for TMA: `planes` (1 or 3) copies side by side along K, each `kp` wide."""
    data: Tensor
    rows: int
    k: int
    kp: int
    planes: int

    @property
    def ld(self) -> int:
        return self.data.stride(0)

    @property
    def cols(self) -> int:
        return self.kp * self.planes if self.planes > 1 else self.k


# plane pairs of the bf16x3 product, smallest terms first
_PAIRS3 = [(0, 2), (2, 0), (1, 1), (0, 1), (1, 0), (0, 0)]


def operand_from_bf16(x: Tensor) -> Operand:
    rows, k, ld = _mat(x, "operand")
    if x.dtype != torch.bfloat16 or ld % 8 != 0 or x.data_ptr() % 16 != 0:
        raise ValueError("bf16 operand must be 16-byte aligned with a pitch multiple of 8")
    return Operand(x, rows, k, k, 1)


_red_bytes = {}


def _red_ws(width: int, dev):
    """Workspace of a launcher that sums across thread blocks in a fixed order (sgf_reduce_ws_bytes) -> (ptr, bytes); one per
    call, so that calls on different streams never share it."""
    if width not in _red_bytes:
        n = C.c_size_t(0)
        check(lib().sgf_reduce_ws_bytes(width, C.byref(n)), "sgf_reduce_ws_bytes")
        _red_bytes[width] = n.value
    ws = torch.empty(_red_bytes[width], dtype=torch.uint8, device=dev)
    return ws, _red_bytes[width]


def pack_operand(src: Tensor, transpose: bool = False, planes: int = 1, colsum: Optional[Tensor] = None,
                 row_index: Optional[Tensor] = None) -> Operand:
    """fp32 [r, c] -> bf16 Operand ([c, r] if transpose).  planes=3: bf16x3 split (fp32-accurate products).
    row_index (int64 [b]): gather rows src[row_index] while packing (mini-batch features)."""
    _use(src)
    if src.dtype != torch.float32:
        raise TypeError("pack_operand expects fp32")
    r, c, ld = _mat(src, "src")
    if row_index is not None:
        if row_index.dtype != torch.int64 or transpose:
            raise ValueError("row_index must be int64 and cannot be combined with transpose")
        row_index = row_index.contiguous()
        r = row_index.numel()
    rows_out, cols_out = (c, r) if transpose else (r, c)
    kp = ceil_to(cols_out, 64) if planes == 3 else ceil_to(cols_out, 8)
    dst = torch.empty((rows_out, kp * planes), dtype=torch.bfloat16, device=src.device)
    ws, nws = _red_ws(c, src.device) if colsum is not None else (None, 0)
    check(lib().sgf_pack_operand(_p(src), ld, r, c, int(transpose), _p(dst), dst.stride(0), kp, kp if planes == 3 else 0,
                                 _p(colsum), _p(row_index), _p(ws), nws, _stream()), "sgf_pack_operand")
    return Operand(dst, rows_out, cols_out, kp, planes)


# fp32 activations that feed several GEMMs of one step (q, k, v, the layer inputs, x0: forward product + weight gradient) are
# packed into bf16x3 planes once: memo keyed by the tensor's storage, alive from the start of a forward to the end of its backward
_operand_memo: Optional[dict] = None


def operand_memo_begin():
    global _operand_memo
    _operand_memo = {}


def operand_memo_clear():
    global _operand_memo
    _operand_memo = None


def as_operand(x: Tensor, planes: int, memo: bool = False) -> Operand:
    """Activation -> operand: bf16 activations are used in place (planes=1); fp32 activations are packed.
    memo=True (forward activations that are never written again) reuses the packed planes within the step."""
    if x.dtype == torch.bfloat16:
        if planes != 1:
            raise ValueError("bf16 activations only form single-plane operands")
        return operand_from_bf16(x)
    if memo and _operand_memo is not None:
        key = (x.data_ptr(), tuple(x.shape), x.stride(), planes)
        hit = _operand_memo.get(key)
        if hit is not None:
            return hit[1]
        op = pack_operand(x, False, planes)
        _operand_memo[key] = (x, op)          # holding x keeps its address from being reused while the entry lives
        return op
    return pack_operand(x, False, planes)


def gemm_nt(A: Sequence[Operand], B: Sequence[Operand], pairs: Sequence[Tuple[int, int, int, int, int]], n_out: int,
            out: Tensor, *, epi: int = EPI_AFFINE, bias: Optional[Tensor] = None, aux: Optional[Tensor] = None,
            row_scale: Optional[Tensor] = None, alpha: float = 1.0, beta: float = 0.0,
            alpha_dev: Optional[Tensor] = None, beta_dev: Optional[Tensor] = None, relu: bool = False,
            accumulate: bool = False, tail: Optional[Operand] = None, nf: float = 0.0, den_out: Optional[Tensor] = None,
            r1_row: Optional[Tensor] = None, r1_col: Optional[Tensor] = None, col_sum: Optional[Tensor] = None,
            col_sumsq: Optional[Tensor] = None, schedule: Optional[int] = None, nf_dev: Optional[Tensor] = None) -> Tensor:
    """out[rows, n_out] = epilogue(sum over `pairs` (ai, a_k0, bi, b_k0, klen) of A[ai][:, a_k0:+klen] . B[bi][:, b_k0:+klen]^T).

    Logical K offsets; 3-plane operands expand every pair into the six bf16x3 partial products."""
    _use(out)
    rows = A[0].rows
    args = GemmNtArgs()
    if len(A) > _lib.SGF_MAX_SRC or len(B) > _lib.SGF_MAX_SRC:
        raise ValueError("too many GEMM sources")
    planes = A[0].planes
    for o in list(A) + list(B) + ([tail] if tail is not None else []):
        if o.planes != planes:
            raise ValueError("all operands of one GEMM must use the same plane count")
    for i, a in enumerate(A):
        if a.rows != rows:
            raise ValueError("A operands must have equal row counts")
        args.a[i], args.lda[i], args.a_cols[i] = a.data.data_ptr(), a.ld, a.cols
    for i, b in enumerate(B):
        if b.rows != n_out:
            raise ValueError(f"B operand {i} has {b.rows} rows, expected n_out={n_out}")
        args.b[i], args.ldb[i], args.b_cols[i] = b.data.data_ptr(), b.ld, b.cols
    args.n_a, args.n_b = len(A), len(B)
    segs = []
    combos = _PAIRS3 if planes == 3 else [(0, 0)]
    for (ai, ak, bi, bk, klen) in pairs:
        if ak % 8 or bk % 8:       # a TMA load starts on a 16-byte boundary; elsewhere its barrier never completes
            raise ValueError(f"gemm_nt: K offsets must be multiples of 8 columns, got {ak} / {bk}")
        for (pa, pb) in combos:
            segs.append((ai, pa * A[ai].kp + ak, bi, pb * B[bi].kp + bk, klen))
    if len(segs) > _lib.SGF_MAX_SEG:
        raise ValueError("too many GEMM segments")
    args.n_seg = len(segs)
    for s, (ai, ak, bi, bk, klen) in enumerate(segs):
        args.seg_a[s], args.seg_akoff[s], args.seg_b[s], args.seg_bkoff[s], args.seg_klen[s] = ai, ak, bi, bk, klen
    if tail is not None:
        if planes != 1 and len(pairs) != 1:
            raise ValueError("tail with multi-plane operands needs a single pair")
        args.b_tail, args.ldb_tail = tail.data.data_ptr(), tail.ld
    args.rows, args.n_out, args.epi = rows, n_out, epi
    orows, ocols, ldo = _mat(out, "out")
    if orows != rows or ocols != n_out:
        raise ValueError(f"out is {tuple(out.shape)}, expected ({rows}, {n_out})")
    args.out, args.ldo, args.out_dtype = out.data_ptr(), ldo, dcode(out)
    args.bias = _p(_f32vec(bias, n_out, "bias"))
    if aux is not None:
        ar, ac, lda_ = _mat(aux, "aux")
        if ar != rows or ac != n_out:
            raise ValueError("aux shape mismatch")
        args.aux, args.ld_aux, args.aux_dtype = aux.data_ptr(), lda_, dcode(aux)
    args.row_scale = _p(_f32vec(row_scale, rows, "row_scale"))
    args.alpha, args.beta = alpha, beta
    args.alpha_dev, args.beta_dev = _p(alpha_dev), _p(beta_dev)
    args.relu, args.accumulate = int(relu), int(accumulate)
    args.nf, args.den_out = nf, _p(_f32vec(den_out, rows, "den_out"))
    args.nf_dev = _p(_f32vec(nf_dev, 1, "nf_dev"))
    args.r1_row, args.r1_col = _p(_f32vec(r1_row, rows, "r1_row")), _p(_f32vec(r1_col, n_out, "r1_col"))
    fused_stats = (col_sum is not None or col_sumsq is not None) and stats_fusable(out)
    if fused_stats:
        args.col_sum, args.col_sumsq = _p(_f32vec(col_sum, n_out, "col_sum")), _p(_f32vec(col_sumsq, n_out, "col_sumsq"))
    args.schedule = GEMM_NT_SCHEDULE if schedule is None else schedule
    check(lib().sgf_gemm_nt(C.byref(args), _stream()), "sgf_gemm_nt")
    if (col_sum is not None or col_sumsq is not None) and not fused_stats:
        s_, q_ = colstats(out, want_sum=col_sum is not None, want_sumsq=col_sumsq is not None)   # unaligned output: extra pass
        if col_sum is not None:
            col_sum.add_(s_)
        if col_sumsq is not None:
            col_sumsq.add_(q_)
    return out


# 0 auto / 1 stream B through the TMA ring / 2 B resident in shared memory (include/sgformer_b200.h: sgf_gemm_nt_args.schedule)
GEMM_NT_SCHEDULE = int(os.environ.get("SGF_GEMM_NT_SCHEDULE", "0"))

# Accumulating the statistics in the GEMM epilogue costs epilogue issue slots that can exceed the separate colstats pass it
# saves, so the fused path is opt-in.
FUSE_GEMM_STATS = os.environ.get("SGF_FUSED_STATS", "0") == "1"


def stats_fusable(out: Tensor) -> bool:
    """Whether sgf_gemm_nt accumulates the column statistics of `out` in its epilogue (TMA-store path, n_out <= 1024)."""
    return FUSE_GEMM_STATS and out.data_ptr() % 16 == 0 and (out.stride(0) * out.element_size()) % 16 == 0 and \
        out.shape[1] <= 1024


def _tn_once(a: Tensor, lda: int, m: int, b: Tensor, ldb: int, n: int, rows: int, out: Tensor, transpose_out: bool,
             alpha: float, beta: float, alpha_dev: Optional[Tensor], pairs: Sequence[Tuple[int, int]] = ()):
    nbytes = C.c_size_t(0)
    check(lib().sgf_gemm_tn_ws_bytes(m, n, rows, C.byref(nbytes)), "sgf_gemm_tn_ws_bytes")
    ws = torch.empty(max(nbytes.value, 4), dtype=torch.uint8, device=out.device)
    args = GemmTnArgs()
    args.a, args.lda, args.m = a.data_ptr(), lda, m
    args.b, args.ldb, args.n = b.data_ptr(), ldb, n
    args.rows = rows
    args.out, args.ldo, args.transpose_out = out.data_ptr(), out.stride(0), int(transpose_out)
    args.alpha, args.beta, args.alpha_dev = alpha, beta, _p(alpha_dev)
    args.ws, args.ws_bytes = ws.data_ptr(), nbytes.value
    args.n_pairs = len(pairs)
    for i, (ao, bo) in enumerate(pairs):
        args.a_off[i], args.b_off[i] = ao, bo
    check(lib().sgf_gemm_tn(C.byref(args), _stream()), "sgf_gemm_tn")


def gemm_tn(A: Operand, B: Operand, out: Tensor, *, transpose_out: bool = False, alpha: float = 1.0, beta: float = 0.0,
            alpha_dev: Optional[Tensor] = None) -> Tensor:
    """out[m, n] (fp32; [n, m] if transpose_out) = alpha * A^T B (+ beta*out), A: [rows, m], B: [rows, n].
    Blocks of 256 features per call; 3-plane operands accumulate the six bf16x3 partial products."""
    _use(out)
    if A.rows != B.rows or A.planes != B.planes:
        raise ValueError("gemm_tn operand mismatch")
    if out.dtype != torch.float32 or out.stride(-1) != 1:
        raise ValueError("gemm_tn output must be fp32 row-major")
    exp = (B.k, A.k) if transpose_out else (A.k, B.k)
    if tuple(out.shape) != exp:
        raise ValueError(f"gemm_tn out is {tuple(out.shape)}, expected {exp}")
    # bf16x3: the six partial products of a block accumulate inside ONE launch (plane column offsets, smallest terms first)
    pairs = [(pa * A.kp, pb * B.kp) for pa, pb in _PAIRS3] if A.planes == 3 else []
    for m0 in range(0, A.k, 256):
        m = min(256, A.k - m0)
        for n0 in range(0, B.k, 256):
            n = min(256, B.k - n0)
            sub = out[n0:n0 + n, m0:m0 + m] if transpose_out else out[m0:m0 + m, n0:n0 + n]
            _tn_once(A.data[:, m0:], A.ld, m, B.data[:, n0:], B.ld, n, A.rows, sub, transpose_out, alpha, beta, alpha_dev, pairs)
    return out


# ------------------------------------------------------------------------------------------------
# row-streaming kernels
# ------------------------------------------------------------------------------------------------
def colstats(x: Tensor, w: Optional[Tensor] = None, want_sum: bool = True, want_sumsq: bool = True,
             sum_out: Optional[Tensor] = None):
    """-> (column sums | None, column sums of squares | None).  sum_out (fp32 [h]): the sums are added to it instead."""
    _use(x)
    rows, h, ld = _mat(x, "x")
    s = sum_out if sum_out is not None else (torch.zeros(h, dtype=torch.float32, device=x.device) if want_sum else None)
    q = torch.zeros(h, dtype=torch.float32, device=x.device) if want_sumsq else None
    wv = _f32vec(w, rows, "w")
    blk = 2048 // x.element_size()      # the row kernels cover at most 2 KB of a row per launch
    for c0 in range(0, h, blk):
        c1 = min(h, c0 + blk)
        ws, nws = _red_ws(c1 - c0, x.device)
        check(lib().sgf_colstats(_p(x[:, c0:c1]), ld, rows, c1 - c0, dcode(x), _p(wv), _p(s[c0:c1] if s is not None else None),
                                 _p(q[c0:c1] if q is not None else None), _p(ws), nws, _stream()), "sgf_colstats")
    return s, q


def _same_ld(ld: int, *ts: Optional[Tensor]):
    for t in ts:
        if t is not None and (t.dim() != 2 or t.stride(1) != 1 or t.stride(0) != ld):
            raise ValueError("row kernels need all activations with the same pitch")


def ln_fwd(x: Tensor, r: Optional[Tensor], a: float, b: float, gamma: Optional[Tensor], beta: Optional[Tensor],
           use_ln: bool, use_relu: bool, p: float, seed: int, want_stats: bool = True):
    _use(x)
    rows, h, ld = _mat(x, "x")
    y = new_like(x)
    _same_ld(ld, r, y)
    stats = torch.empty((rows, 2), dtype=torch.float32, device=x.device) if (use_ln and want_stats) else None
    check(lib().sgf_ln_fwd(_p(x), _p(r), ld, rows, h, dcode(x), a, b, _p(gamma), _p(beta), int(use_ln), int(use_relu), p,
                           seed, _p(y), _p(stats), _stream()), "sgf_ln_fwd")
    return y, stats


def ln_bwd(dy: Tensor, x: Tensor, r: Optional[Tensor], a: float, b: float, gamma, beta, stats, use_ln: bool,
           use_relu: bool, p: float, seed: int, gscale: float, want_dr: bool, dgamma: Optional[Tensor],
           dbeta: Optional[Tensor]):
    _use(x)
    rows, h, ld = _mat(x, "x")
    dx = new_like(x)
    dr = new_like(x) if want_dr else None
    _same_ld(ld, dy, r, dx, dr)
    ws, nws = _red_ws(h, x.device)
    check(lib().sgf_ln_bwd(_p(dy), _p(x), _p(r), ld, rows, h, dcode(x), a, b, _p(gamma), _p(beta), _p(stats), int(use_ln),
                           int(use_relu), p, seed, gscale, _p(dx), _p(dr), _p(dgamma), _p(dbeta), _p(ws), nws, _stream()),
          "sgf_ln_bwd")
    return dx, dr


def ln_bwd_attn(dy: Tensor, o: Tensor, r: Optional[Tensor], xa: Tensor, a: float, b: float, gamma, beta, stats, use_ln: bool,
                use_relu: bool, p: float, seed: int, gscale: float, want_dr: bool, dgamma: Optional[Tensor],
                dbeta: Optional[Tensor], den: Tensor):
    """LayerNorm backward of y = dropout(relu?(LN?(a*o + b*r))) fused with the row prologue of the Gram-form attention
    backward (sgf_ln_bwd_attn).  -> (gnum' [rows,h], gden' fp32 [rows], dr | None, cs [h], pg [h], sg [1])."""
    _use(o)
    rows, h, ld = _mat(o, "o")
    gnum = new_like(o)
    dr = new_like(o) if want_dr else None
    _same_ld(ld, dy, r, xa, gnum, dr)
    dev = o.device
    gden = torch.empty(rows, dtype=torch.float32, device=dev)
    acc = torch.zeros(2 * h + 1, dtype=torch.float32, device=dev)
    cs, pg, sg = acc[:h], acc[h:2 * h], acc[2 * h:]
    ws, nws = _red_ws(h, dev)
    check(lib().sgf_ln_bwd_attn(_p(dy), _p(o), _p(r), _p(xa), ld, rows, h, dcode(o), a, b, _p(gamma), _p(beta), _p(stats),
                                int(use_ln), int(use_relu), p, seed, gscale, _p(_f32vec(den, rows, "den")), _p(gnum), _p(gden),
                                _p(dr), _p(dgamma), _p(dbeta), _p(cs), _p(pg), _p(sg), _p(ws), nws, _stream()),
          "sgf_ln_bwd_attn")
    return gnum, gden, dr, cs, pg, sg


def ln_fwd_graph(x: Tensor, r: Optional[Tensor], gy: Tensor, a: float, b: float, c: float, gamma: Optional[Tensor],
                 beta: Optional[Tensor], use_ln: bool, use_relu: bool, p: float, seed: int, want_stats: bool = True):
    """ln_fwd of u = a*x + b*r + c*gy (sgf_ln_fwd_graph): the row pass of a DIFFormer layer."""
    _use(x)
    rows, h, ld = _mat(x, "x")
    y = new_like(x)
    _same_ld(ld, r, gy, y)
    stats = torch.empty((rows, 2), dtype=torch.float32, device=x.device) if (use_ln and want_stats) else None
    check(lib().sgf_ln_fwd_graph(_p(x), _p(r), _p(gy), ld, rows, h, dcode(x), a, b, c, _p(gamma), _p(beta), int(use_ln),
                                 int(use_relu), p, seed, _p(y), _p(stats), _stream()), "sgf_ln_fwd_graph")
    return y, stats


def ln_bwd_attn_graph(dy: Tensor, o: Tensor, r: Optional[Tensor], xa: Tensor, gy: Tensor, a: float, b: float, c: float, gamma, beta, stats,
                      use_ln: bool, p: float, seed: int, gscale: float, want_dr: bool, dgamma: Optional[Tensor],
                      dbeta: Optional[Tensor], den: Tensor, dinv: Tensor):
    """ln_bwd_attn for u = a*o + b*r + c*gy, also writing ys = dinv (.) (c*du) (sgf_ln_bwd_attn_graph).
    -> (gnum' [rows,h], gden' fp32 [rows], dr | None, ys [rows,h], cs [h], pg [h], sg [1])."""
    _use(o)
    rows, h, ld = _mat(o, "o")
    gnum = new_like(o)
    ys = new_like(o)
    dr = new_like(o) if want_dr else None
    _same_ld(ld, dy, r, xa, gy, gnum, dr, ys)
    dev = o.device
    gden = torch.empty(rows, dtype=torch.float32, device=dev)
    acc = torch.zeros(2 * h + 1, dtype=torch.float32, device=dev)
    cs, pg, sg = acc[:h], acc[h:2 * h], acc[2 * h:]
    ws, nws = _red_ws(h, dev)
    check(lib().sgf_ln_bwd_attn_graph(_p(dy), _p(o), _p(r), _p(xa), _p(gy), ld, rows, h, dcode(o), a, b, c, _p(gamma), _p(beta), _p(stats),
                                      int(use_ln), p, seed, gscale, _p(_f32vec(den, rows, "den")), _p(_f32vec(dinv, rows, "dinv")),
                                      _p(gnum), _p(gden), _p(dr), _p(ys), _p(dgamma), _p(dbeta), _p(cs), _p(pg), _p(sg), _p(ws),
                                      nws, _stream()), "sgf_ln_bwd_attn_graph")
    return gnum, gden, dr, ys, cs, pg, sg


def bn_finalize(sum_: Optional[Tensor], sumsq: Optional[Tensor], rows: int, h: int, zbias: Optional[Tensor],
                running_mean: Optional[Tensor], running_var: Optional[Tensor], device, eps: float = 1e-5,
                momentum: float = 0.1):
    mean = torch.empty(h, dtype=torch.float32, device=device)
    rstd = torch.empty(h, dtype=torch.float32, device=device)
    _use(mean)
    check(lib().sgf_bn_finalize(_p(sum_), _p(sumsq), rows, h, eps, momentum, _p(zbias), _p(mean), _p(rstd),
                                _p(running_mean), _p(running_var), _stream()), "sgf_bn_finalize")
    return mean, rstd


def bn_fwd(z: Tensor, res: Optional[Tensor], mix: Optional[Tensor], mean, rstd, gamma, beta, zbias, use_bn: bool,
           use_relu: bool, p: float, seed: int, gw: float, row_scale: Optional[Tensor], want_y: bool, want_scaled: bool,
           ys_out: Optional[Tensor] = None, y_out: Optional[Tensor] = None):
    """y_out (z's shape, dtype and pitch): y is written there (a column block of a wider activation)."""
    _use(z)
    rows, h, ld = _mat(z, "z")
    y = _out_like(y_out, z, "y_out") if want_y else None
    ys = (ys_out if (ys_out is not None and ys_out.stride(0) == ld) else new_like(z)) if want_scaled else None
    _same_ld(ld, res, mix, y, ys)
    check(lib().sgf_bn_fwd(_p(z), _p(res), _p(mix), ld, rows, h, dcode(z), _p(mean), _p(rstd), _p(gamma), _p(beta),
                           _p(zbias), int(use_bn), int(use_relu), p, seed, gw, _p(row_scale), _p(y), _p(ys), _stream()),
          "sgf_bn_fwd")
    return y, ys


def bn_bwd(dy: Optional[Tensor], dy2: Optional[Tensor], row_scale2: Optional[Tensor], z: Tensor, mean, rstd, gamma, beta,
           zbias, use_bn: bool, use_relu: bool, training: bool, p: float, seed: int, gscale: float,
           dres: Optional[Tensor] = None, dres_accumulate: bool = False, want_dz_colsum: bool = False,
           out_row_scale: Optional[Tensor] = None, reduce_fn=None, stat_rows: int = 0, dz_out: Optional[Tensor] = None):
    """-> (dz, sums [2h] or None (dbeta, dgamma), dz_colsum [h] or None).
    `reduce_fn(sums)` runs between the two phases (the row-sharded all-reduce of the BatchNorm sums); `stat_rows` is then
    the global row count.  dz_out (z's shape, dtype and pitch): dz is written there."""
    _use(z)
    rows, h, ld = _mat(z, "z")
    dz = _out_like(dz_out, z, "dz_out")
    _same_ld(ld, dy, dy2, dz, dres)
    sums = None
    if use_bn and training:
        sums = bn_bwd_sums(dy, dy2, row_scale2, z, mean, rstd, gamma, beta, zbias, use_bn, use_relu, p, seed, gscale)
        if reduce_fn is not None:
            reduce_fn(sums)
    colsum = torch.zeros(h, dtype=torch.float32, device=z.device) if want_dz_colsum else None
    ws, nws = _red_ws(h, z.device)
    check(lib().sgf_bn_bwd_apply(_p(dy), _p(dy2), _p(row_scale2), _p(z), ld, rows, h, dcode(z), _p(mean), _p(rstd),
                                 _p(gamma), _p(beta), _p(zbias), int(use_bn), int(use_relu), int(training), p, seed,
                                 gscale, int(stat_rows), _p(sums), _p(dz), _p(dres), int(dres_accumulate), _p(colsum),
                                 _p(out_row_scale), _p(ws), nws, _stream()), "sgf_bn_bwd_apply")
    return dz, sums, colsum


def bn_bwd_sums(dy, dy2, row_scale2, z: Tensor, mean, rstd, gamma, beta, zbias, use_bn: bool, use_relu: bool, p: float,
                seed: int, gscale: float) -> Tensor:
    """Phase 1 alone: fp32 [2h] = (sum g, sum g*xhat)."""
    _use(z)
    rows, h, ld = _mat(z, "z")
    _same_ld(ld, dy, dy2)
    sums = torch.zeros(2 * h, dtype=torch.float32, device=z.device)
    ws, nws = _red_ws(h, z.device)
    check(lib().sgf_bn_bwd_reduce(_p(dy), _p(dy2), _p(row_scale2), _p(z), ld, rows, h, dcode(z), _p(mean), _p(rstd),
                                  _p(gamma), _p(beta), _p(zbias), int(use_bn), int(use_relu), p, seed, gscale, _p(sums),
                                  _p(ws), nws, _stream()), "sgf_bn_bwd_reduce")
    return sums


JK_MAX, JK_CAT = 1, 2      # jk_mode of sgf_bn_fwd_jk / sgf_bn_bwd_*_jk
_JK_MODES = {"max": JK_MAX, "cat": JK_CAT}


def _jk_args(mode: str, buf: Tensor, idx: Optional[Tensor], layer: int, z: Tensor, name: str):
    """(mode code, buf, pitch, idx) of a JK call, checked: `buf` has z's rows and width and the activation dtype; `idx` (max) is
    uint8 with buf's pitch in bytes."""
    code = _JK_MODES[mode]
    rows, h, ld = _mat(buf, name)
    if rows != z.shape[0] or h != z.shape[1] or buf.dtype != z.dtype or buf.device != z.device:
        raise ValueError(f"{name}: expected {tuple(z.shape)} {z.dtype}, got {tuple(buf.shape)} {buf.dtype}")
    if not 0 <= layer <= 255:
        raise ValueError(f"JK layer index {layer} out of range 0..255")
    if code == JK_MAX:
        if idx is None or idx.dtype != torch.uint8 or _mat(idx, "jk_idx")[2] != ld or idx.shape[0] != rows or idx.shape[1] < h:
            raise ValueError("jk_idx: expected uint8 [rows, >= h] with the JK buffer's pitch")
    return code, ld


def bn_fwd_jk(z: Tensor, mean, rstd, gamma, beta, zbias, use_bn: bool, use_relu: bool, p: float, seed: int, want_y: bool,
              mode: str, jk: Tensor, jk_idx: Optional[Tensor], layer: int) -> Optional[Tensor]:
    """bn_fwd of GCN layer `layer` that also folds its pre-dropout activation into the jumping knowledge (include/sgformer_b200.h:
    sgf_bn_fwd_jk): the running max / layer index (mode 'max'), or column block `jk` of the concatenation (mode 'cat')."""
    _use(z)
    rows, h, ld = _mat(z, "z")
    code, ld_jk = _jk_args(mode, jk, jk_idx, layer, z, "jk")
    y = new_like(z) if want_y else None
    check(lib().sgf_bn_fwd_jk(_p(z), ld, rows, h, dcode(z), _p(mean), _p(rstd), _p(gamma), _p(beta), _p(zbias), int(use_bn),
                              int(use_relu), p, seed, _p(y), code, _p(jk), ld_jk, _p(jk_idx), layer, _stream()), "sgf_bn_fwd_jk")
    return y


def bn_bwd_jk(dy: Optional[Tensor], z: Tensor, mean, rstd, gamma, beta, zbias, use_bn: bool, use_relu: bool, training: bool,
              p: float, seed: int, mode: str, jk_g: Tensor, jk_idx: Optional[Tensor], layer: int, want_dz_colsum: bool = False,
              out_row_scale: Optional[Tensor] = None):
    """bn_bwd whose upstream gradient is dropout(dy) + the JK gradient of layer `layer` (sgf_bn_bwd_*_jk) -> (dz, sums [2h] or None,
    dz_colsum or None).  Eval mode with BatchNorm returns the sums too (the affine gradients need them)."""
    _use(z)
    rows, h, ld = _mat(z, "z")
    code, ld_jk = _jk_args(mode, jk_g, jk_idx, layer, z, "jk_g")
    _same_ld(ld, dy)
    dz = new_like(z)
    sums = None
    if use_bn:
        sums = torch.zeros(2 * h, dtype=torch.float32, device=z.device)
        ws, nws = _red_ws(h, z.device)
        check(lib().sgf_bn_bwd_reduce_jk(_p(dy), _p(z), ld, rows, h, dcode(z), _p(mean), _p(rstd), _p(gamma), _p(beta), _p(zbias),
                                         int(use_bn), int(use_relu), p, seed, _p(sums), code, _p(jk_g), ld_jk, _p(jk_idx), layer,
                                         _p(ws), nws, _stream()), "sgf_bn_bwd_reduce_jk")
    colsum = torch.zeros(h, dtype=torch.float32, device=z.device) if want_dz_colsum else None
    ws, nws = _red_ws(h, z.device)
    check(lib().sgf_bn_bwd_apply_jk(_p(dy), _p(z), ld, rows, h, dcode(z), _p(mean), _p(rstd), _p(gamma), _p(beta), _p(zbias),
                                    int(use_bn), int(use_relu), int(training), p, seed, _p(sums), _p(dz), _p(colsum),
                                    _p(out_row_scale), code, _p(jk_g), ld_jk, _p(jk_idx), layer, _p(ws), nws, _stream()),
          "sgf_bn_bwd_apply_jk")
    return dz, sums, colsum


def axpby(x: Tensor, y: Optional[Tensor], a: float, b: float, out_dtype=None, row_scale: Optional[Tensor] = None,
          out: Optional[Tensor] = None) -> Tensor:
    _use(x)
    rows, h, ldx = _mat(x, "x")
    out_dtype = out_dtype or x.dtype
    if out is None:
        out = alloc_act(rows, h, out_dtype, x.device)
    ldy = y.stride(0) if y is not None else 0
    check(lib().sgf_axpby(_p(x), ldx, dcode(x), _p(y), ldy, dcode(y) if y is not None else dcode(x), a, b, _p(row_scale),
                          _p(out), out.stride(0), dcode(out), rows, h, _stream()), "sgf_axpby")
    return out


def _heads_fit(x: Tensor, heads: int, d: int, name: str):
    """Kernels that take a head count read `heads` blocks of d columns from every row of x: refuse a narrower x (the kernel
    would read past the end of the row, or of the allocation)."""
    rows, cols, ld = _mat(x, name)
    if heads < 1 or d < 1 or cols < heads * d:
        raise ValueError(f"{name}: {cols} columns, but {heads} heads of width {d} need {heads * d}")
    return rows, cols, ld


def head_mean(x: Tensor, heads: int, d: int) -> Tensor:
    """x [N, >= heads*d] -> [N, d]: the mean of the heads' column blocks."""
    _use(x)
    rows, _, ld = _heads_fit(x, heads, d, "x")
    out = alloc_act(rows, d, x.dtype, x.device)
    check(lib().sgf_head_mean(_p(x), ld, rows, heads, d, dcode(x), _p(out), out.stride(0), _stream()), "sgf_head_mean")
    return out


# ------------------------------------------------------------------------------------------------
# GAT edge softmax (csrc/gat.cu)
# ------------------------------------------------------------------------------------------------
ACT_ELU = 2          # `use_relu` code of bn_fwd / bn_bwd for ELU (GAT's F.elu)
GAT_MAX_HEADS = 8    # SGF_GAT_MAX_HEADS


def gat_logits(xp: Tensor, heads: int, c: int, att_src: Tensor, att_dst: Tensor) -> Tuple[Tensor, Tensor]:
    """xp [N, heads*c] -> (a_src, a_dst) fp32 [N, heads]."""
    _use(xp)
    n, _, ld = _heads_fit(xp, heads, c, "xp")
    a_src = torch.empty((n, heads), dtype=torch.float32, device=xp.device)
    a_dst = torch.empty((n, heads), dtype=torch.float32, device=xp.device)
    check(lib().sgf_gat_logits(_p(xp), ld, n, heads, c, dcode(xp), _p(_f32vec(att_src, heads * c, "att_src")),
                               _p(_f32vec(att_dst, heads * c, "att_dst")), _p(a_src), _p(a_dst), _stream()), "sgf_gat_logits")
    return a_src, a_dst


def gat_fwd(rowptr: Tensor, col: Tensor, xp: Tensor, a_src: Tensor, a_dst: Tensor, heads: int, c: int, mean: bool,
            bias: Optional[Tensor], p: float, seed: int, out: Optional[Tensor] = None) -> Tuple[Tensor, Tensor]:
    """-> (out [N, c] if mean else [N, heads*c] in xp's dtype, lse fp32 [N, heads]).  See sgf_gat_fwd.
    out: written in place when given (a column block of a wider activation)."""
    _use(xp)
    n, _, ld = _heads_fit(xp, heads, c, "xp")
    width = c if mean else heads * c
    if out is None:
        out = alloc_act(n, width, xp.dtype, xp.device)
    elif tuple(out.shape) != (n, width) or out.dtype != xp.dtype or out.device != xp.device:
        raise ValueError(f"gat_fwd: out must be [{n}, {width}] {xp.dtype}, got {tuple(out.shape)} {out.dtype}")
    _mat(out, "out")
    lse = torch.empty((n, heads), dtype=torch.float32, device=xp.device)
    check(lib().sgf_gat_fwd(_p(rowptr), _p(col), _p(xp), ld, _p(a_src), _p(a_dst), n, heads, c, dcode(xp), int(mean),
                            _p(_f32vec(bias, out.shape[1], "bias")), _p(out), out.stride(0), _p(lse), p, seed, _stream()),
          "sgf_gat_fwd")
    return out, lse


def gat_bwd(rowptr: Tensor, col: Tensor, rowptr_t: Tensor, col_t: Tensor, xp: Tensor, a_src: Tensor, a_dst: Tensor, lse: Tensor,
            g: Tensor, att_src: Tensor, att_dst: Tensor, heads: int, c: int, mean: bool, p: float, seed: int,
            dxp_out: Optional[Tensor] = None):
    """g = dL/dout -> (dxp [N, heads*c] in xp's dtype, da_src fp32 [heads, N], da_dst fp32 [heads, N]).  See sgf_gat_bwd.
    dxp_out (xp's shape and dtype, any 16-byte pitch): dxp is written there."""
    _use(xp)
    n, _, ld = _heads_fit(xp, heads, c, "xp")
    _, _, ldg = _heads_fit(g, 1 if mean else heads, c, "g")
    if g.dtype != xp.dtype:
        raise TypeError("gat_bwd: g and xp must share the activation dtype")
    dev = xp.device
    r_ws = torch.empty((n, heads), dtype=torch.float32, device=dev)
    da_src = torch.empty((heads, n), dtype=torch.float32, device=dev)
    da_dst = torch.empty((heads, n), dtype=torch.float32, device=dev)
    dxp = new_like(xp) if dxp_out is None else dxp_out
    if dxp.shape != xp.shape or dxp.dtype != xp.dtype or dxp.device != xp.device:
        raise ValueError(f"gat_bwd: dxp_out must be {tuple(xp.shape)} {xp.dtype}, got {tuple(dxp.shape)} {dxp.dtype}")
    _mat(dxp, "dxp_out")
    check(lib().sgf_gat_bwd(_p(rowptr), _p(col), _p(rowptr_t), _p(col_t), _p(xp), ld, _p(a_src), _p(a_dst), _p(lse), _p(g), ldg,
                            _p(_f32vec(att_src, heads * c, "att_src")), _p(_f32vec(att_dst, heads * c, "att_dst")), n, heads, c,
                            dcode(xp), int(mean), p, seed, _p(r_ws), _p(da_src), _p(da_dst), _p(dxp), dxp.stride(0), _stream()),
          "sgf_gat_bwd")
    return dxp, da_src, da_dst


def dense_dropout(x: Tensor, p: float, seed: int) -> Tensor:
    """fp32 [rows, cols] -> dropout(x) (sgf_dense_dropout; the same (p, seed) applied to a gradient is its backward)."""
    _use(x)
    rows, cols, ld = _mat(x, "x")
    if x.dtype != torch.float32:
        raise TypeError("dense_dropout expects fp32")
    y = alloc_act(rows, cols, torch.float32, x.device)
    check(lib().sgf_dense_dropout(_p(x), ld, rows, cols, p, seed, _p(y), y.stride(0), _stream()), "sgf_dense_dropout")
    return y


# ------------------------------------------------------------------------------------------------
# attention glue
# ------------------------------------------------------------------------------------------------
def attn_prepare_fwd(s_raw: Tensor, z_raw: Tensor, nq2v: Tensor, nk2v: Tensor, planes: int):
    """-> (bmat Operand [d, m], btail Operand [16, m], scal fp32 [4])."""
    _use(s_raw)
    m, d = s_raw.shape
    kp = ceil_to(m, 64) if planes == 3 else ceil_to(m, 8)
    bmat = torch.empty((d, kp * planes), dtype=torch.bfloat16, device=s_raw.device)
    btail = torch.empty((16, kp * planes), dtype=torch.bfloat16, device=s_raw.device)
    if kp != m:
        bmat.zero_()
        btail.zero_()
    scal = torch.empty(4, dtype=torch.float32, device=s_raw.device)
    check(lib().sgf_attn_prepare_fwd(_p(s_raw), _p(z_raw), _p(nq2v), nq2v.numel(), _p(nk2v), nk2v.numel(), m, d, _p(bmat),
                                     bmat.stride(0), _p(btail), btail.stride(0), kp if planes == 3 else 0, _p(scal),
                                     _stream()), "sgf_attn_prepare_fwd")
    return Operand(bmat, d, m, kp, planes), Operand(btail, 16, m, kp, planes), scal


def attn_bwd_prep(g: Tensor, o: Tensor, den: Tensor, gscale: float):
    _use(g)
    rows, d, ld = _mat(g, "g")
    _, _, ld_o = _mat(o, "o")
    gnum = alloc_act(rows, d, g.dtype, g.device)
    gden = torch.empty(rows, dtype=torch.float32, device=g.device)
    check(lib().sgf_attn_bwd_prep(_p(g), ld, _p(o), ld_o, _p(den), rows, d, dcode(g), gscale, _p(gnum), gnum.stride(0),
                                  _p(gden), _stream()), "sgf_attn_bwd_prep")
    return gnum, gden


def attn_prepare_bwd(s_raw: Tensor, z_raw: Tensor, ds_raw: Tensor, dz_raw: Tensor, scal_fwd: Tensor, planes: int,
                     scal_bwd: Tensor):
    _use(s_raw)
    m, d = s_raw.shape
    kpd = ceil_to(d, 64) if planes == 3 else ceil_to(d, 8)
    kpm = ceil_to(m, 64) if planes == 3 else ceil_to(m, 8)
    dev = s_raw.device
    b_dq = torch.zeros((m, kpd * planes), dtype=torch.bfloat16, device=dev)
    b_dk = torch.zeros((m, kpd * planes), dtype=torch.bfloat16, device=dev)
    b_dv = torch.zeros((d, kpm * planes), dtype=torch.bfloat16, device=dev)
    r1_col = torch.empty(m, dtype=torch.float32, device=dev)
    dk_bias = torch.empty(m, dtype=torch.float32, device=dev)
    check(lib().sgf_attn_prepare_bwd(_p(s_raw), _p(z_raw), _p(ds_raw), _p(dz_raw), _p(scal_fwd), m, d, _p(b_dq),
                                     b_dq.stride(0), _p(b_dv), b_dv.stride(0), _p(b_dk), b_dk.stride(0),
                                     kpd if planes == 3 else 0, kpm if planes == 3 else 0, _p(r1_col), _p(dk_bias),
                                     _p(scal_bwd), _stream()), "sgf_attn_prepare_bwd")
    return (Operand(b_dq, m, d, kpd, planes), Operand(b_dv, d, m, kpm, planes), Operand(b_dk, m, d, kpd, planes), r1_col,
            dk_bias)


def attn_combine_scal(scal_bwd_all: Tensor, heads: int, scal_fwd: Tensor):
    _use(scal_bwd_all)
    if heads < 1 or scal_bwd_all.dim() != 2 or scal_bwd_all.shape[0] < heads or scal_bwd_all.shape[1] < 4:
        raise ValueError(f"attn_combine_scal: scal_bwd_all {tuple(scal_bwd_all.shape)} holds fewer than {heads} rows of 4 scalars")
    check(lib().sgf_attn_combine_scal(_p(scal_bwd_all), heads, scal_bwd_all.stride(0), _p(scal_fwd), _stream()),
          "sgf_attn_combine_scal")


# ------------------------------------------------------------------------------------------------
# Gram-form linear attention (engine.attention_gram_forward / _backward)
# ------------------------------------------------------------------------------------------------
# slots of the device scalar vector `sc` (include/sgformer_b200.h: sgf_attn_gram_args.sc)
SC_NQ2, SC_NK2, SC_ALPHA, SC_BETA, SC_DEN, SC_N, SC_IP, SC_C, SC_CQ, SC_CK, SC_SG = 0, 1, 2, 3, 4, 5, 8, 9, 10, 11, 12


GRAM_KERNEL = os.environ.get("SGF_GRAM_KERNEL", "1") == "1"


def gram(xop: Operand, x: Tensor):
    """Pass 1 of the Gram-form attention: G = x^T x (fp32 [h,h]) and s = x^T 1 (fp32 [h]) of the layer input.
    h <= 256: sgf_gram (one load per tile, upper block triangle, X^T 1 as an extra MMA column); wider layers: the generic
    node-contracting GEMM + a column-sum pass."""
    h = xop.k
    dev = x.device
    if h <= 256 and GRAM_KERNEL:
        _use(xop.data)
        G = torch.empty((h, h), dtype=torch.float32, device=dev)
        s = torch.empty(h, dtype=torch.float32, device=dev)
        nbytes = C.c_size_t(0)
        check(lib().sgf_gram_ws_bytes(h, xop.planes, xop.rows, C.byref(nbytes)), "sgf_gram_ws_bytes")
        ws = torch.empty(max(nbytes.value, 4), dtype=torch.uint8, device=dev)
        check(lib().sgf_gram(_p(xop.data), xop.ld, xop.rows, h, xop.planes, xop.kp if xop.planes == 3 else 0, _p(G), h, _p(s), _p(ws),
                             nbytes.value, _stream()), "sgf_gram")
        return G, s
    G = torch.empty((h, h), dtype=torch.float32, device=dev)
    gemm_tn(xop, xop, G)
    s, _ = colstats(x, want_sumsq=False)
    return G, s


class GramState:
    """fp32 device tensors written by sgf_attn_gram_prepare_fwd and re-read by its backward (h x h algebra on the weights)."""
    __slots__ = ("wq", "bq", "wk", "bk", "wv", "bv", "G", "s", "kx", "qx", "vx", "z1", "q1", "v1", "S", "Bt", "tail", "bt", "sc",
                 "n", "h", "m", "d", "ws", "vsum")


def _w2(t: Tensor, name: str) -> Tensor:
    if t.dtype != torch.float32 or t.dim() != 2 or t.stride(1) != 1:
        raise ValueError(f"{name}: expected an fp32 row-major matrix")
    return t


def _gram_args(st: GramState) -> AttnGramArgs:
    a = AttnGramArgs()
    a.h, a.m, a.d, a.n_nodes = st.h, st.m, st.d, st.n
    a.wq, a.bq, a.wk, a.bk, a.wv, a.bv = (_p(t) for t in (st.wq, st.bq, st.wk, st.bk, st.wv, st.bv))
    a.ld_wq, a.ld_wk, a.ld_wv = st.wq.stride(0), st.wk.stride(0), st.wv.stride(0)
    a.G, a.s = _p(st.G), _p(st.s)
    for f in ("kx", "qx", "vx", "z1", "q1", "v1", "S", "Bt", "tail", "bt", "sc"):
        setattr(a, f, _p(getattr(st, f)))
    a.ws, a.ws_floats = _p(st.ws), st.ws.numel()
    return a


def attn_gram_prepare_fwd(G: Tensor, s: Tensor, wq: Tensor, bq: Tensor, wk: Tensor, bk: Tensor, wv: Tensor, bv: Tensor,
                          n: int, vsum: bool = False) -> GramState:
    """h x h algebra between the two passes (sgf_attn_gram_prepare_fwd): from G = x^T x, s = x^T 1 and the projection weights
    -> Bt [d,h], tail [16,h] (row 0 = ct), bt [d], sc[SC_DEN] such that out = (x Bt^T + bt)/(x ct + sc[SC_DEN]).
    vsum=True: DIFFormer's numerator (column sum of v instead of N v; sgf_attn_gram_prepare_fwd_vsum)."""
    _use(G)
    st = GramState()
    st.vsum = bool(vsum)
    st.wq, st.wk, st.wv = _w2(wq, "Wq"), _w2(wk, "Wk"), _w2(wv, "Wv")
    st.bq, st.bk, st.bv = (t.contiguous() for t in (bq, bk, bv))
    st.m, st.h = wq.shape
    st.d = wv.shape[0]
    st.n = int(n)
    if wk.shape != wq.shape or wv.shape[1] != st.h or tuple(G.shape) != (st.h, st.h) or not G.is_contiguous():
        raise ValueError("attn_gram_prepare_fwd: shape mismatch")
    st.G, st.s = G, s
    dev = G.device
    h, m, d = st.h, st.m, st.d
    # one allocation for the saved fp32 state
    sizes = dict(kx=m * h, qx=m * h, vx=d * h, z1=m, q1=m, v1=d, S=m * d, Bt=d * h, tail=16 * h, bt=d, sc=16)
    buf = torch.zeros(sum(ceil_to(v, 4) for v in sizes.values()), dtype=torch.float32, device=dev)
    o = 0
    shapes = dict(kx=(m, h), qx=(m, h), vx=(d, h), S=(m, d), Bt=(d, h), tail=(16, h))
    for k_, v in sizes.items():
        t = buf[o:o + v]
        setattr(st, k_, t.view(shapes[k_]) if k_ in shapes else t)
        o += ceil_to(v, 4)
    nws = C.c_int64(0)
    check(lib().sgf_attn_gram_ws_floats(h, m, d, C.byref(nws)), "sgf_attn_gram_ws_floats")
    st.ws = torch.empty(max(nws.value, 1), dtype=torch.float32, device=dev)
    if st.vsum:
        check(lib().sgf_attn_gram_prepare_fwd_vsum(C.byref(_gram_args(st)), _stream()), "sgf_attn_gram_prepare_fwd_vsum")
    else:
        check(lib().sgf_attn_gram_prepare_fwd(C.byref(_gram_args(st)), _stream()), "sgf_attn_gram_prepare_fwd")
    return st


def attn_gram_prepare_fwd_vsum(G: Tensor, s: Tensor, wq: Tensor, bq: Tensor, wk: Tensor, bk: Tensor, wv: Tensor, bv: Tensor,
                               n: int) -> GramState:
    """attn_gram_prepare_fwd in value-sum mode (DIFFormer); attn_gram_prepare_bwd then runs the matching backward."""
    return attn_gram_prepare_fwd(G, s, wq, bq, wk, bk, wv, bv, n, vsum=True)


def attn_gram_prepare_bwd(st: GramState, P: Tensor, pg: Tensor, cs: Tensor, sg: Tensor):
    """-> (dWq, dbq, dWk, dbk, dWv, dbv, bcat fp32 [h, d+h], a4 fp32 [h]); see sgf_attn_gram_prepare_bwd."""
    _use(P)
    h, m, d = st.h, st.m, st.d
    dev = P.device
    if tuple(P.shape) != (h, d) or not P.is_contiguous():
        raise ValueError("attn_gram_prepare_bwd: P must be contiguous fp32 [h, d]")
    sizes = dict(dwq=m * h, dbq=m, dwk=m * h, dbk=m, dwv=d * h, dbv=d, bcat=h * (d + h), a4=h)
    buf = torch.empty(sum(ceil_to(v, 4) for v in sizes.values()), dtype=torch.float32, device=dev)
    out, o = {}, 0
    shapes = dict(dwq=(m, h), dwk=(m, h), dwv=(d, h), bcat=(h, d + h))
    for k_, v in sizes.items():
        t = buf[o:o + v]
        out[k_] = t.view(shapes[k_]) if k_ in shapes else t
        o += ceil_to(v, 4)
    a = _gram_args(st)
    a.P, a.pg, a.cs, a.sg = _p(P), _p(_f32vec(pg, h, "pg")), _p(_f32vec(cs, d, "cs")), _p(_f32vec(sg, 1, "sg"))
    for k_ in sizes:
        setattr(a, k_, _p(out[k_]))
    if st.vsum:
        check(lib().sgf_attn_gram_prepare_bwd_vsum(C.byref(a), _stream()), "sgf_attn_gram_prepare_bwd_vsum")
    else:
        check(lib().sgf_attn_gram_prepare_bwd(C.byref(a), _stream()), "sgf_attn_gram_prepare_bwd")
    return out["dwq"], out["dbq"], out["dwk"], out["dbk"], out["dwv"], out["dbv"], out["bcat"], out["a4"]


def softmax_nll(logits: Tensor, labels: Tensor, mask: Optional[Tensor], scale: float, want_grad: bool = True):
    """-> (loss fp32 [1], dlogits fp32 [rows, c] | None).  See sgf_softmax_nll."""
    _use(logits)
    if logits.dtype != torch.float32 or labels.dtype != torch.int64:
        raise TypeError("softmax_nll expects fp32 logits and int64 labels")
    rows, c, ld = _mat(logits, "logits")
    labels = labels.reshape(-1).contiguous()
    if labels.numel() != rows:
        raise ValueError("labels / logits row mismatch")
    m = None
    if mask is not None:
        m = mask.reshape(-1).to(torch.uint8).contiguous()
    loss = torch.zeros(1, dtype=torch.float32, device=logits.device)
    d = torch.empty((rows, c), dtype=torch.float32, device=logits.device) if want_grad else None
    ws, nws = _red_ws(1, logits.device)
    check(lib().sgf_softmax_nll(_p(logits), ld, _p(labels), _p(m), rows, c, scale, _p(loss), _p(d), c, _p(ws), nws,
                                _stream()), "sgf_softmax_nll")
    return loss, d


def eval_acc(logits: Tensor, labels: Tensor, idx: Optional[Tensor] = None, want_loss: bool = False):
    """K11: (accuracy, mean NLL of log_softmax | None) over the rows `idx` (all rows if None), computed on the device.
    labels: int64 [rows] or [rows, 1] for ALL rows of `logits` (indexed by idx inside the kernel)."""
    _use(logits)
    if logits.dtype != torch.float32:
        raise TypeError("eval_acc expects fp32 logits")
    rows, c, ld = _mat(logits, "logits")
    labels = labels.reshape(-1).contiguous()
    if labels.dtype != torch.int64 or labels.numel() != rows:
        raise ValueError("eval_acc: labels must be int64 with one entry per logits row")
    if idx is not None:
        idx = idx.reshape(-1).to(device=logits.device, dtype=torch.int64).contiguous()
    m = rows if idx is None else idx.numel()
    correct = torch.empty(1, dtype=torch.int64, device=logits.device)
    nll = torch.empty(1, dtype=torch.float64, device=logits.device) if want_loss else None
    check(lib().sgf_eval_acc(_p(logits), ld, _p(labels), _p(idx), m, rows, c, _p(correct), _p(nll), _stream()), "sgf_eval_acc")
    acc = float(correct.item()) / m if m else float("nan")
    return acc, (float(nll.item()) / m if want_loss and m else None)


def launch_count() -> int:
    return int(lib().sgf_launch_count())
