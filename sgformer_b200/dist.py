"""Row-sharded execution across GPUs (SURVEY.md §8e): nodes are split into contiguous row blocks, parameters are
replicated, and the schedule exchanges only

  C1  {G = x^T x, s = x^T 1} (Gram-form attention; {S', z', ||q||^2, ||k||^2} on the multi-head path)   one all-reduce per layer
  C2  {P = x^T gnum', x^T gden', column sums} (resp. {dS', dz'})                                          its backward
  C3  BatchNorm column sums (forward and backward)      2h floats each
  C4  the pre-scaled SpMM operand rows                  every rank needs the operand rows its CSR block references
  C5  parameter gradients                               one flattened all-reduce per step

through torch.distributed (NCCL over NVLink on GPUs; gloo in the CPU tests).  `Comm(None)` is the single-GPU no-op.

C4 — the halo exchange.  On the reference's graphs (uniform random, mean degree 40-50, P <= 8 row blocks) every remote row is
referenced by some local row, so the halo of a rank IS the other ranks' blocks; what can be won is overlap, not volume.  Three modes
(`SGF_C4_MODE`, default `push` on CUDA when symmetric memory can be set up, else `allgather`):

  push       fused compute + exchange.  Every rank owns a symmetric buffer [world*block, h] per SpMM of the step.  The producer of the
             operand writes its block straight into slot 0; the rank then PUSHES the block into slot (rank - r) mod world of every peer
             r with copy-engine peer copies over NVLink (a side stream: no SMs, no NCCL kernels) and raises the peer's arrival flag
             with a second, 4-byte copy-engine write behind it (a flag KERNEL cannot be used: it is not scheduled while the
             consumer's SpMM occupies the SMs spinning on that very flag).
             The CSR shard stores ROTATED column ids (`sgf_csr_build_rot`): a row's neighbours are sorted by arrival slot.  The SpMM
             runs in PHASES over groups of slots (`sgf_spmm_range` + per-row split offsets): the phase of the local slot starts at
             once and hides the transfer, every later phase is launched behind a tiny `sgf_wait_flags` on the slots it reads and
             carries the rows' fp32 partial sums forward.  (A single kernel that waits inside each row, `sgf_spmm_flagged`,
             is correct but overlaps nothing: every warp stalls in its FIRST row until the last slot has landed - measured
             5.7 ms vs 4.9 ms of pure gather at 2 GPUs; kept as SGF_C4_MODE=push-flagged.)  The consumer lowers its flags after the
             SpMM; the step's collectives (C1 / C3 / C5) order the reuse of a buffer between steps, and a schedule that has none
             between two uses of a buffer gets a 4-byte all-reduce as a fence (`Comm._fence_reuse`).
  rotated    the same rotated layout filled by one all-gather (CPU tests of the layout; no overlap).
  allgather  r1 behaviour: blocking all-gather of the blocks in rank order, plain SpMM.
"""
from __future__ import annotations

import os
from typing import Optional, Tuple

import torch
import torch.distributed as dist

Tensor = torch.Tensor

# Column chunks of the all-gather / SpMM pipeline of the `allgather` mode (1 = one blocking all-gather per SpMM).  More chunks do
# not overlap: NCCL's all-gather kernels need SMs that the HBM-bound SpMM grid already fills; hence the copy-engine `push` mode.
C4_CHUNKS = int(os.environ.get("SGF_C4_CHUNKS", "1"))
C4_MIN_CHUNK_BYTES = 256      # gathered rows stay >= two full 128-byte lines per neighbour
C4_MODE = os.environ.get("SGF_C4_MODE", "auto")
MAX_PUSH_BUFFERS = 16         # SpMMs per step that get their own symmetric buffer (2 * GNN layers)


def partition(n: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous row block of `rank`: [r0, r1) with block = ceil(n / world)."""
    block = (n + world - 1) // world
    r0 = min(n, rank * block)
    return r0, min(n, r0 + block)


class _PushState:
    """Symmetric operand buffers + arrival flags of the `push` mode (one set per (h, dtype))."""

    def __init__(self, comm: "Comm", h: int, dtype, device):
        import torch.distributed._symmetric_memory as symm
        self.symm = symm
        self.comm, self.h, self.dtype, self.device = comm, h, dtype, device
        self.group = comm.group if comm.group is not None else dist.group.WORLD
        self.bufs = {}                       # k -> (local [world*block, h], [peer views of their buffers])
        w = comm.world
        self.flags = symm.empty((MAX_PUSH_BUFFERS, w), dtype=torch.int32, device=device)
        self.flags.zero_()
        hdl = symm.rendezvous(self.flags, self.group)
        self.peer_flags = [hdl.get_buffer(r, (MAX_PUSH_BUFFERS, w), torch.int32) for r in range(w)]
        self.side = torch.cuda.Stream(device=device, priority=-1)
        # First peer copy NOW, while every GPU is quiescent (any lazy driver-side set-up of the peer mapping happens here, not while a
        # flagged SpMM spins on this very rank's push).
        from . import kernels as K
        K._use(self.flags)
        self.fence = torch.zeros(1, dtype=torch.float32, device=device)
        self.one = torch.ones(1, dtype=torch.int32, device=device)     # source of the arrival flags (copied by the copy engine)
        for r in range(w):
            if r != comm.rank:
                K.memcpy_async(self.peer_flags[r][MAX_PUSH_BUFFERS - 1, comm.rank:comm.rank + 1], self.flags[0, 0:1])
        torch.cuda.synchronize(device)
        dist.barrier(group=self.group)       # every rank's flags are zero (the warm-up wrote zeros) before anybody signals

    def buffer(self, k: int):
        if k not in self.bufs:
            w, b = self.comm.world, self.comm.block
            t = self.symm.empty((w * b, self.h), dtype=self.dtype, device=self.device)
            hdl = self.symm.rendezvous(t, self.group)          # collective: the schedule reaches it in the same order on all ranks
            peers = [hdl.get_buffer(r, (w * b, self.h), self.dtype) for r in range(w)]
            self.bufs[k] = (t, peers)
        return self.bufs[k]


class Comm:
    def __init__(self, group=None, n_global: Optional[int] = None, c4_mode: Optional[str] = None):
        self.group = group
        self.active = group is not None or (dist.is_available() and dist.is_initialized() and n_global is not None)
        if self.active:
            self.world = dist.get_world_size(group)
            self.rank = dist.get_rank(group)
        else:
            self.world, self.rank = 1, 0
        self.n_global = n_global
        if self.active and n_global is None:
            raise ValueError("Comm needs the global node count")
        self.block = (n_global + self.world - 1) // self.world if n_global is not None else None
        self.rows = partition(n_global, self.world, self.rank) if n_global is not None else None
        mode = c4_mode or C4_MODE
        if mode == "auto":
            mode = "push" if (self.active and self.world > 1 and dist.get_backend(group) == "nccl") else "allgather"
        if not self.active or self.world == 1:
            mode = "allgather"
        if mode not in ("push", "push-flagged", "rotated", "allgather"):
            raise ValueError(f"unknown C4 mode {mode!r}")
        self.c4_mode = mode
        # slot groups of the phased SpMM: every slot its own phase up to 4 GPUs, else the local slot + 3 groups of remote slots
        # (each phase boundary costs one fp32 write + read of the partial sums, each group delays its slots to the last arrival)
        self._groups_forced = int(os.environ.get("SGF_C4_GROUPS", "0"))
        ng = self._groups_forced or min(self.world, 4)
        ng = max(1, min(ng, self.world))
        if ng == 1:
            self.groups = [(0, self.world)]
        else:
            rest, k = self.world - 1, ng - 1
            cuts = [1 + (rest * i) // k for i in range(k + 1)]
            self.groups = [(0, 1)] + [(cuts[i], cuts[i + 1]) for i in range(k) if cuts[i + 1] > cuts[i]]
        self._push = {}            # (h, dtype) -> _PushState
        self._spmm_calls = 0       # position of the next SpMM inside the current step (selects the symmetric buffer)
        self._coll_seq = 0         # collectives issued through this Comm so far
        self._last_use = {}        # symmetric buffer k -> _coll_seq after its last use (see _fence_reuse)
        self._push_failed = False

    # column-id rotation the CSR shard of this rank must be built with (None: global ids)
    @property
    def col_rot(self) -> Optional[Tuple[int, int]]:
        if self.c4_mode in ("push", "push-flagged", "rotated") and self.active and self.world > 1:
            return (self.rank * self.block, self.world * self.block)
        return None

    def begin_step(self):
        """Called at the start of every sharded forward: SpMM k of this step uses symmetric buffer k."""
        self._spmm_calls = 0

    def _fence_reuse(self, st, k: int):
        """Symmetric buffer k may be overwritten by a peer's push of the NEXT use as soon as that peer gets there, so a collective
        that every rank joins only after finishing its previous read of buffer k has to lie between two uses.  The step's own
        all-reduces (C1 Gram, C3 BatchNorm) normally are that collective; a schedule without any (no attention layer, eval mode,
        one GCN layer) gets an explicit 4-byte all-reduce here.  Every rank runs the same schedule, so all take the same branch."""
        if self._last_use.get(k) == self._coll_seq:
            dist.all_reduce(st.fence, group=self.group)
            self._coll_seq += 1

    # -- small reductions (C1, C2, C3, C5) ----------------------------------------------------------
    def allreduce_(self, *tensors: Tensor):
        """In-place sum over ranks; several small fp32 tensors travel as one flat buffer."""
        if not self.active or self.world == 1:
            return
        ts = [t for t in tensors if t is not None]
        self._coll_seq += 1
        if len(ts) == 1 and ts[0].is_contiguous():
            dist.all_reduce(ts[0], group=self.group)
            return
        flat = torch.cat([t.reshape(-1).float() for t in ts])
        dist.all_reduce(flat, group=self.group)
        o = 0
        for t in ts:
            k = t.numel()
            t.copy_(flat[o:o + k].view_as(t))
            o += k

    # -- C4 -----------------------------------------------------------------------------------------
    def allgather_rows(self, x_local: Tensor) -> Tensor:
        """[n_local, h] row block -> [n_global, h] (blocks of ceil(N/P) rows; the last block may be short)."""
        if not self.active or self.world == 1:
            return x_local
        n_loc, h = x_local.shape
        xl = x_local
        if n_loc != self.block or not xl.is_contiguous():
            pad = torch.zeros((self.block, h), dtype=x_local.dtype, device=x_local.device)
            pad[:n_loc] = x_local
            xl = pad
        out = torch.empty((self.world * self.block, h), dtype=x_local.dtype, device=x_local.device)
        dist.all_gather_into_tensor(out, xl, group=self.group)
        return out[:self.n_global]

    def c4_chunks(self, h: int, elem_size: int) -> int:
        """Column chunks of the all-gather pipeline (C4_CHUNKS, reduced until the chunk rows are >= C4_MIN_CHUNK_BYTES)."""
        if not self.active or self.world == 1:
            return 1
        want = C4_CHUNKS
        while want > 1 and (h % want != 0 or (h // want) * elem_size < C4_MIN_CHUNK_BYTES):
            want -= 1
        return want

    def _push_state(self, h: int, dtype, device) -> Optional[_PushState]:
        key = (h, dtype)
        if key not in self._push and not self._push_failed:
            try:
                self._push[key] = _PushState(self, h, dtype, device)
            except Exception as exc:      # no symmetric memory on this system: every rank takes the all-gather route
                import warnings
                warnings.warn(f"sgformer_b200: symmetric memory unavailable ({type(exc).__name__}: {exc}); C4 falls back to "
                              f"the rotated all-gather (no overlap)")
                self._push_failed = True
        return self._push.get(key)

    def operand_out(self, n_local: int, h: int, dtype, device) -> Optional[Tensor]:
        """Where the producer of the NEXT SpMM operand should write its [n_local, h] block so that it needs no staging copy:
        slot 0 of that SpMM's symmetric buffer (push mode), else None (the caller allocates)."""
        esize = 2 if dtype == torch.bfloat16 else 4
        if self.c4_mode not in ("push", "push-flagged") or not self.active or self.world == 1 or (h * esize) % 16 != 0 or device.type != "cuda":
            return None
        st = self._push_state(h, dtype, device)
        if st is None or self._spmm_calls >= MAX_PUSH_BUFFERS:
            return None
        buf, _ = st.buffer(self._spmm_calls)
        return buf[:n_local]

    def _rotated_gather(self, x_local: Tensor) -> Tensor:
        """all-gather into the rotated slot order (slot s = block of rank (rank + s) mod world)."""
        full = self.allgather_rows(x_local)
        w, b = self.world, self.block
        if full.shape[0] != w * b:
            pad = torch.zeros((w * b, full.shape[1]), dtype=full.dtype, device=full.device)
            pad[:full.shape[0]] = full
            full = pad
        return torch.roll(full, shifts=-self.rank * b, dims=0)

    def _spmm_phased(self, Kmod, graph, transposed: bool, rowptr, col, row_scale, buf: Tensor, wait) -> Tensor:
        """SpMM over the rotated operand buffer in slot-group phases; wait(s0, s1) (or None) blocks the stream until slots
        [s0, s1) have landed.  fp32 partial sums travel from phase to phase in place."""
        groups = self.groups
        if len(groups) == 1:
            if wait is not None:
                wait(1, self.world)
            return Kmod.spmm(rowptr, col, row_scale, buf)
        thr = tuple(g[0] * self.block for g in groups[1:])
        sp = graph.row_splits(thr, transposed)            # int32 [G-1, n_rows], cached on the graph
        n_rows, h = rowptr.numel() - 1, buf.shape[1]
        part = torch.empty((n_rows, h), dtype=torch.float32, device=buf.device)
        out = None
        for gi, (s0, s1) in enumerate(groups):
            if wait is not None and gi > 0:
                wait(s0, s1)
            last = gi == len(groups) - 1
            out = Kmod.spmm_range(rowptr, col, row_scale, buf, sp[gi - 1] if gi > 0 else None, None if last else sp[gi],
                                  part if gi > 0 else None, None if last else part)
        return out

    def spmm_gathered(self, Kmod, graph, transposed: bool, row_scale: Optional[Tensor], x_local: Tensor) -> Tensor:
        """C4 + SpMM: y[rows of this rank] = scale * A[rows, :] @ (operand rows of every rank); A = `graph` (its transpose when
        `transposed`), `Kmod` = the kernels module.  The CSR shard must have been built with this Comm's `col_rot`."""
        rowptr, col = graph.transpose() if transposed else (graph.rowptr, graph.col)
        heavy = graph.heavy_t if transposed else graph.heavy
        spmm = Kmod.spmm
        if not self.active or self.world == 1:
            return spmm(rowptr, col, row_scale, x_local, heavy=heavy)
        k = self._spmm_calls
        self._spmm_calls += 1
        n_loc, h = x_local.shape
        if self.c4_mode in ("push", "push-flagged"):
            st = self._push_state(h, x_local.dtype, x_local.device) if (k < MAX_PUSH_BUFFERS and x_local.is_cuda) else None
            if st is not None:
                return self._spmm_pushed(st, k, Kmod, graph, transposed, rowptr, col, row_scale, x_local, heavy)
        if self.c4_mode in ("push", "push-flagged", "rotated"):
            buf = self._rotated_gather(x_local)
            if heavy is not None:
                return spmm(rowptr, col, row_scale, buf, heavy=heavy)
            return self._spmm_phased(Kmod, graph, transposed, rowptr, col, row_scale, buf, None)
        nch = self.c4_chunks(h, x_local.element_size())
        if nch == 1:
            return spmm(rowptr, col, row_scale, self.allgather_rows(x_local), heavy=heavy)
        hc = h // nch
        dev, dt = x_local.device, x_local.dtype
        pending = []
        for c in range(nch):
            xc = torch.zeros((self.block, hc), dtype=dt, device=dev) if n_loc != self.block else \
                torch.empty((self.block, hc), dtype=dt, device=dev)
            xc[:n_loc].copy_(x_local[:, c * hc:(c + 1) * hc])
            gc = torch.empty((self.world * self.block, hc), dtype=dt, device=dev)
            pending.append((dist.all_gather_into_tensor(gc, xc, group=self.group, async_op=True), gc, xc))
        n_rows = rowptr.numel() - 1
        # same pitch rule as kernels.alloc_act (rows 16-byte aligned); chunk offsets are multiples of 256 bytes
        out = torch.empty((n_rows, h), dtype=dt, device=dev)
        for c, (work, gc, _) in enumerate(pending):
            work.wait()
            spmm(rowptr, col, row_scale, gc[:self.n_global], out=out[:, c * hc:(c + 1) * hc], heavy=heavy)
        return out

    def _spmm_pushed(self, st: _PushState, k: int, Kmod, graph, transposed, rowptr, col, row_scale, x_local: Tensor, heavy) -> Tensor:
        K = Kmod
        w, b, rank = self.world, self.block, self.rank
        buf, peers = st.buffer(k)
        self._fence_reuse(st, k)
        n_loc = x_local.shape[0]
        own = buf[:n_loc]
        if x_local.data_ptr() != own.data_ptr():
            own.copy_(x_local)                       # the producer did not write in place (operand_out was not used)
        main = torch.cuda.current_stream(st.device)
        ready = torch.cuda.Event()
        ready.record(main)
        with torch.cuda.stream(st.side):
            st.side.wait_event(ready)
            for s in range(1, w):                    # my block is slot s of rank (rank - s): nearest consumer position first
                r = (rank - s) % w
                K.memcpy_async(peers[r][s * b:s * b + n_loc], own)               # copy-engine peer copy over NVLink
                # ... and the arrival flag behind it, ALSO by the copy engine: a 1-thread flag kernel of another stream is never
                # scheduled while a consumer kernel holds the SMs spinning on that flag (tests/push_debug2.py
                # stages S1/P2 trap, S2/P1 pass), whereas stream-ordered copy-engine writes need no SM
                K.memcpy_async(st.peer_flags[r][k, s:s + 1], st.one)
            done = torch.cuda.Event()
            done.record(st.side)
        flags = st.flags[k]
        # phased vs in-row waiting: the phases pay one fp32 write + read of the partial sums per boundary and shorter per-row
        # gathers, the in-row wait overlaps nothing
        rowbytes = x_local.shape[1] * x_local.element_size()
        phased = self._groups_forced > 1 or (self._groups_forced == 0 and ((w >= 4 and rowbytes >= 512) or w >= 8))
        if self.c4_mode == "push-flagged" or heavy is not None or not phased:
            if heavy is not None:
                K.wait_flags(flags[1:])
                y = K.spmm(rowptr, col, row_scale, buf, heavy=heavy)
            else:
                y = K.spmm_flagged(rowptr, col, row_scale, buf, flags, b)
        else:
            y = self._spmm_phased(K, graph, transposed, rowptr, col, row_scale, buf, lambda s0, s1: K.wait_flags(flags[s0:s1]))
        # every peer's signal of THIS use has been seen before the flags are lowered for the next step (a slot no row references
        # would otherwise leave a late signal behind); the step's collectives (C1 / C5) order the reuse of the buffer itself
        K.wait_flags(flags[1:])
        flags.zero_()
        main.wait_event(done)
        self._last_use[k] = self._coll_seq
        return y


SINGLE = Comm(None)
