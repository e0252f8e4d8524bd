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
    graph: Graph       # induced subgraph (RandomPartitionSampler) or sampled edges (NeighborSampler), local ids
    labels: Optional[Tensor] = None
    num_seeds: Optional[int] = None    # NeighborSampler: the batch's seeds are its first num_seeds nodes


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


class NeighborSampler:
    """PyG NeighborLoader(data, num_neighbors, batch_size, input_nodes, shuffle) of 100M/nb-sample.py:125-150 on the device
    (replace=False, disjoint=False; DESIGN.md §4.15).  `graph` is the parent Graph in self_loop_mode 0 (rows = edge targets):
    every node of hop t's frontier draws min(k_t, deg) distinct entries of its row (k_t = -1: all of them, at most `capacity`),
    the seeds are local ids 0..B-1 and the other nodes follow in order of first appearance by (hop, frontier position, entry
    position); the batch's edges are the drawn entries only (source -> target), so `mb.graph` equals
    Graph(mb.graph.edge_index, b, 0).  Every draw is a pure function of (seed, hop, node, draw index) with one 64-bit seed per
    batch drawn from `generator` (a CPU torch.Generator, default the global one) on the host: the same generator state replays
    the same batches.  The kernels need no host sync; yielding a batch reads its node and edge counts back once, because the
    batch's tensors are shaped by them.  NeighborLoader's `num_workers` / `persistent_workers` are accepted and ignored: there are
    no host workers."""

    def __init__(self, graph: Graph, x: Tensor, y: Optional[Tensor], num_neighbors, batch_size: int,
                 input_nodes: Optional[Tensor] = None, shuffle: bool = False, generator: Optional[torch.Generator] = None,
                 capacity: Optional[int] = None, num_workers: int = 0, persistent_workers: bool = False):
        from . import kernels as K
        if not x.is_cuda:
            raise RuntimeError("NeighborSampler keeps the graph and features on the GPU (no CPU fallback)")
        if graph.rows is not None:
            raise ValueError("NeighborSampler needs the full (unsharded) graph")
        if graph.val is not None:
            raise NotImplementedError("NeighborSampler of a weighted graph is not supported")
        if graph.self_loop_mode != 0:
            raise ValueError(f"NeighborSampler needs a parent Graph in self_loop_mode 0 (rows = edge targets, edges as given); "
                             f"got self_loop_mode {graph.self_loop_mode}")
        if generator is not None and generator.device.type != "cpu":
            raise ValueError("NeighborSampler draws its seeds on the host: pass a CPU torch.Generator")
        self.graph, self.x, self.y = graph, x, y
        self.batch_size, self.shuffle, self.capacity = int(batch_size), bool(shuffle), capacity
        self.generator = generator if generator is not None else torch.default_generator
        self.plan = K.neighbor_sample_plan(self.batch_size, num_neighbors, capacity)
        dev = graph.rowptr.device
        if input_nodes is None:
            input_nodes = torch.arange(graph.n, device=dev)
        if input_nodes.dtype == torch.bool:
            input_nodes = input_nodes.nonzero().flatten()
        self.input_nodes = input_nodes.to(device=dev, dtype=torch.int64).contiguous()
        if self.input_nodes.numel():        # once per sampler: the seeds must be distinct node ids
            lo, hi = torch.stack(torch.aminmax(self.input_nodes)).tolist()
            if lo < 0 or hi >= graph.n or torch.unique(self.input_nodes).numel() != self.input_nodes.numel():
                raise ValueError(f"input_nodes must hold distinct node ids in [0, {graph.n})")
        if getattr(graph, "_sample_map", None) is None:
            graph._sample_map = torch.full((max(graph.n, 1),), -1, dtype=torch.int32, device=dev)
        self._need = torch.zeros(1, dtype=torch.int64, device=dev)     # largest row a k = -1 hop met (overflow check)

    def __len__(self) -> int:
        return (self.input_nodes.numel() + self.batch_size - 1) // self.batch_size

    def draw_seed(self) -> int:
        """The next batch's 64-bit sampling seed from the generator (host only)."""
        return int(torch.randint(0, 2 ** 63 - 1, (1,), generator=self.generator).item())

    def batch(self, seed_idx: Tensor, seed: Optional[int] = None) -> MiniBatch:
        """The batch of the seeds `seed_idx` (global ids, at most batch_size); `seed` defaults to draw_seed()."""
        from . import kernels as K
        seed = self.draw_seed() if seed is None else int(seed)
        seeds = seed_idx.to(device=self.graph.rowptr.device, dtype=torch.int64).contiguous()
        idx, ei, counts, rp, cl, dv, rp_t, cl_t = K.neighbor_sample(self.graph.rowptr, self.graph.col, self.graph._sample_map, seeds,
                                                                    self.plan, seed, self._need)
        b, e = counts.tolist()
        g = Graph._from_parts(b, rp[:b + 1], cl[:e], dv[:b], False, 0)
        g._t = (rp_t[:b + 1], cl_t[:e])
        g.edge_index = ei[:, :e]
        idx = idx[:b]
        return MiniBatch(idx, self.x.index_select(0, idx), g, None if self.y is None else self.y.index_select(0, idx),
                         num_seeds=seeds.numel())

    def __iter__(self) -> Iterator[MiniBatch]:
        nodes = self.input_nodes
        if self.shuffle:
            nodes = nodes[torch.randperm(nodes.numel(), generator=self.generator).to(nodes.device)]
        for i in range(len(self)):
            yield self.batch(nodes[i * self.batch_size:(i + 1) * self.batch_size])
        self.check()

    def check(self):
        """Raise if a k = -1 hop met a row longer than `capacity` (that row was cut to its first `capacity` entries, never
        overrun).  One device sync: called at the end of every epoch, and by the user after a partial epoch."""
        need = int(self._need.item())
        if self.capacity is not None and need > self.capacity:
            raise RuntimeError(f"NeighborSampler: a row of {need} entries was sampled with k = -1 but capacity is {self.capacity}; "
                               f"rerun with capacity >= {need}")
