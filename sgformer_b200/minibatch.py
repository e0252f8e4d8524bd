"""Mini-batch path of the reference (large/main-batch.py:130-151: `randperm(n)` -> slices of `batch_size` ->
`subgraph(idx_i, edge_index, relabel_nodes=True)` on the CPU -> model on the GPU) kept entirely on the device:
the graph's CSR is built once, every batch structure comes from `Graph.subset` (K9 on the CSR) and the batch features
are gathered while they are packed into the tensor-core operand format."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Iterator, Optional

import torch

from .graph import Graph

Tensor = torch.Tensor


@dataclass
class MiniBatch:
    idx: Tensor        # int64 [b] global node ids (local id = position)
    features: Tensor   # fp32 [b, d_in]
    graph: Graph       # induced subgraph, local ids
    labels: Optional[Tensor] = None


class RandomPartitionSampler:
    """One epoch = a random permutation of the nodes cut into consecutive batches (large/main-batch.py:134-136).
    Everything stays in HBM; `capacity` (max induced nnz per batch) avoids a device sync per batch when given."""

    def __init__(self, graph: Graph, x: Tensor, y: Optional[Tensor], batch_size: int, capacity: Optional[int] = None,
                 generator: Optional[torch.Generator] = None):
        if not x.is_cuda:
            raise RuntimeError("RandomPartitionSampler keeps the graph and features on the GPU (no CPU fallback)")
        self.graph, self.x, self.y, self.batch_size = graph, x, y, int(batch_size)
        self.capacity, self.generator = capacity, generator
        self.n = graph.n
        self._max_needed = None      # device int64 [1]: largest induced nnz any batch needed (overflow check without per-batch syncs)

    def __len__(self) -> int:
        return (self.n + self.batch_size - 1) // self.batch_size

    def batch(self, idx: Tensor) -> MiniBatch:
        g = self.graph.subset(idx, self.capacity)
        if self.capacity is not None:
            # a directed graph's batch has a transposed half with its own induced nnz; a symmetric one shares it
            needed = g.nnz_needed if g.nnz_needed_t is g.nnz_needed else torch.maximum(g.nnz_needed, g.nnz_needed_t)
            self._max_needed = needed.clone() if self._max_needed is None else torch.maximum(self._max_needed, needed)
        return MiniBatch(idx, self.x.index_select(0, idx), g, None if self.y is None else self.y.index_select(0, idx))

    def __iter__(self) -> Iterator[MiniBatch]:
        perm = torch.randperm(self.n, device=self.x.device, generator=self.generator)
        for i in range(len(self)):
            yield self.batch(perm[i * self.batch_size:(i + 1) * self.batch_size])
        self.check()

    def check(self):
        """Raise if a batch's induced subgraph did not fit `capacity` (its structure was truncated, never overrun).  One device
        sync: called at the end of every epoch, and by the user after a partial epoch."""
        if self._max_needed is not None and int(self._max_needed.item()) > self.capacity:
            raise RuntimeError(f"RandomPartitionSampler: a batch needed {int(self._max_needed.item())} induced edges but capacity is "
                               f"{self.capacity}; rerun with a larger capacity (or capacity=None for exact sizing)")
