"""Graph structure cache: CSR of the GCN aggregation pattern (+ lazily its transpose) built once per edge list.

The reference rebuilds degree -> edge weights -> sort -> CSR inside every GraphConvLayer.forward
(reference large/ours.py:26-33); it is graph-constant, so it is hoisted here and keyed on the edge_index tensor."""
from __future__ import annotations

from collections import OrderedDict
from typing import Optional, Tuple

import torch

from . import kernels as K

Tensor = torch.Tensor


class Graph:
    """rowptr int64 [n_rows+1], col int32 [nnz] (rows = edge targets, sorted columns, duplicates kept), dinv fp32 [n_rows].
    self_loop_mode 0: large/100M GraphConv; 1: PyG gcn_norm (medium GCN).
    `rows=(r0, r1)`: row shard of the global pattern (column ids stay global) for row-sharded multi-GPU runs.
    `edge_weight` (fp32 [nnz]): weighted graph (DESIGN.md §4.10): `val` fp32 / `eid` int64 per entry (value and source edge
    position; rows sorted by (col, eid)), `dinv` of the weighted degree in mode 1 (the count-based one in mode 0), and after
    transpose() `val_t` / `eid_t` of the transposed CSR.  Unweighted graphs have val = eid = None."""

    def __init__(self, edge_index: Tensor, n: int, self_loop_mode: int = 0, rows: Optional[Tuple[int, int]] = None,
                 col_rot: Optional[Tuple[int, int]] = None, edge_weight: Optional[Tensor] = None):
        if not edge_index.is_cuda:
            raise RuntimeError("Graph needs a CUDA edge_index (no CPU fallback)")
        self.n = int(n)
        self.rows = rows
        self.col_rot = col_rot          # (rot, mod): column ids stored as (col - rot) mod `mod` (row shards with pushed operands)
        self.self_loop_mode = self_loop_mode
        self.edge_index = edge_index
        self.edge_weight = edge_weight
        self.val = self.eid = self.val_t = self.eid_t = None
        if edge_weight is not None:
            if rows is not None or col_rot is not None:
                raise NotImplementedError("Graph: row sharding of a weighted graph is not supported")
            self.rowptr, self.col, self.eid, self.val, self.dinv = K.csr_build_weighted(edge_index, edge_weight, self.n, False,
                                                                                       self_loop_mode, True)
        else:
            self.rowptr, self.col, self.dinv = K.csr_build(edge_index, self.n, False, self_loop_mode, True, rows=rows,
                                                           col_rot=col_rot)
        self.heavy = K.heavy_rows(self.rowptr)      # segment plan for hub rows (None on graphs without them)
        self.heavy_t = None
        self._t: Optional[Tuple[Tensor, Tensor]] = None

    def pattern(self) -> "Graph":
        """The unweighted Graph of the same edge list and self-loop mode (the last conv of a weighted models.GCN runs on it)."""
        if self.val is None:
            return self
        if getattr(self, "_pattern", None) is None:
            self._pattern = get_graph(self.edge_index, self.n, self.self_loop_mode)
        return self._pattern

    @property
    def nnz(self) -> int:
        return int(self.rowptr[-1].item())

    @classmethod
    def _from_parts(cls, n, rowptr, col, dinv, transpose_same: bool):
        g = cls.__new__(cls)
        g.n, g.rows, g.self_loop_mode, g.edge_index, g.col_rot = int(n), None, 0, None, None
        g.edge_weight = g.val = g.eid = g.val_t = g.eid_t = None
        g.rowptr, g.col, g.dinv = rowptr, col, dinv
        g.heavy = g.heavy_t = None       # batch subgraphs: no per-batch sync for a hub plan
        g._t = (rowptr, col) if transpose_same else None
        return g

    def subset(self, idx: Tensor, capacity: Optional[int] = None) -> "Graph":
        """Induced subgraph of the nodes `idx` (int64, local id = position in idx), built from this CSR in
        O(sum of the selected rows' lengths) — the mini-batch structure of large/main-batch.py:136-139 without the per-batch
        O(E) PyG `subgraph` mask and without a CSR rebuild.  Requires a symmetric edge set for the backward (checked once)."""
        if self.rows is not None:
            raise ValueError("subset() needs the full (unsharded) graph")
        if self.val is not None:
            raise NotImplementedError("Graph.subset of a weighted graph is not supported")
        if not hasattr(self, "_node_map"):
            self._node_map = torch.full((max(self.n, 1),), -1, dtype=torch.int32, device=self.rowptr.device)
            self._symmetric = self.transpose()[0] is self.rowptr
            if not self._symmetric:
                raise NotImplementedError("Graph.subset: directed graphs need the transposed subset as well")
        rp, cl, dv, needed = K.csr_subset(self.rowptr, self.col, self.n, idx, self._node_map, capacity)
        g = Graph._from_parts(idx.numel(), rp, cl, dv, True)
        g.nnz_needed, g.capacity = needed, capacity      # device int64 [1]: > capacity means the batch structure was truncated
        return g

    def row_splits(self, thresholds: Tuple[int, ...], transposed: bool = False) -> Tensor:
        """int32 [len(thresholds), n_rows]: per row the number of entries whose (rotated) column id is below each threshold - the
        phase boundaries of a row-sharded SpMM (dist.Comm._spmm_phased); cached."""
        rp, cl = self.transpose() if transposed else (self.rowptr, self.col)
        same = rp is self.rowptr
        key = (tuple(thresholds), transposed and not same)
        cache = self.__dict__.setdefault("_splits", {})
        if key not in cache:
            cache[key] = K.csr_row_splits(rp, cl, thresholds)
        return cache[key]

    def transpose(self) -> Tuple[Tensor, Tensor]:
        """CSR of the transposed pattern (rows = edge sources) for the backward SpMM; shares storage when the edge
        list is symmetric (the usual case after to_undirected).  Weighted graphs share it only when the weighted multiset
        {(r, c, w)} is symmetric; `val_t` / `eid_t` hold the transpose's values and edge positions."""
        if self._t is None and self.val is not None:
            if K.edge_symmetry_weighted(self.edge_index, self.edge_weight, self.n):
                self._t = (self.rowptr, self.col)
                self.val_t, self.eid_t, self.heavy_t = self.val, self.eid, self.heavy
            else:
                rp, cl, self.eid_t, self.val_t, _ = K.csr_build_weighted(self.edge_index, self.edge_weight, self.n, True,
                                                                          self.self_loop_mode, False)
                self._t = (rp, cl)
                self.heavy_t = K.heavy_rows(rp)
        if self._t is None:
            if K.edge_symmetry(self.edge_index, self.n):
                self._t = (self.rowptr, self.col)      # also true per row shard: rows r0..r1 of A^T == rows of A
                self.heavy_t = self.heavy
            else:
                rp, cl, _ = K.csr_build(self.edge_index, self.n, True, self.self_loop_mode, False, rows=self.rows,
                                        col_rot=self.col_rot)
                self._t = (rp, cl)
                self.heavy_t = K.heavy_rows(rp)
        return self._t


_CACHE: "OrderedDict[tuple, Graph]" = OrderedDict()
_CACHE_MAX = 4


def get_graph(edge_index: Tensor, n: int, self_loop_mode: int = 0, rows: Optional[Tuple[int, int]] = None,
              col_rot: Optional[Tuple[int, int]] = None, edge_weight: Optional[Tensor] = None) -> Graph:
    """Cached Graph for this edge_index tensor (identity: storage pointer, shape, version) and, for a weighted graph, this
    edge_weight tensor (same identity)."""
    wkey = None if edge_weight is None else (edge_weight.data_ptr(), tuple(edge_weight.shape), edge_weight._version,
                                             edge_weight.dtype)
    key = (edge_index.data_ptr(), tuple(edge_index.shape), edge_index._version, edge_index.device.index, int(n),
           self_loop_mode, rows, col_rot, wkey)
    g = _CACHE.get(key)
    if g is not None and g.edge_index is edge_index and g.edge_weight is edge_weight:
        _CACHE.move_to_end(key)
        return g
    g = Graph(edge_index, n, self_loop_mode, rows, col_rot, edge_weight)
    _CACHE[key] = g
    while len(_CACHE) > _CACHE_MAX:
        _CACHE.popitem(last=False)
    return g


def clear_cache():
    _CACHE.clear()
