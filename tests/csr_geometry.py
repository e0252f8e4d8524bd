"""The launch geometry of the graph-structure kernels (csrc/csr.cu), restated in plain Python, and the table of graphs
tests/test_gpu_csr_sweep.py builds.

Row sort (sort_rows / sort_long_rows).  A row of `len` entries takes one of these paths (p2 = next_pow2(len)):
  len <= 1                     nothing to sort
  len <= 32                    warp bitonic, one register per lane
  len <= 64                    warp bitonic, two registers per lane
  len <= kWarpSortMax (256)    warp bitonic in per-warp shared memory
  p2 <= kSortSmemMax (2048)    queued; num_sms x 4 blocks sort it in shared memory
  p2 <= share                  queued; kHubBlocks (16) blocks sort it in their share of the global scratch
  p2 <= scratch                queued; one block sorts it in the whole scratch
  longer                       left in fill order (the documented limit: only > 2^26 entries in one row)
The scratch holds max(kSortSmemMax x kHubBlocks, next_pow2(nnz + n)) keys, capped at kHubScratchMax = 2^26, and share is a
sixteenth of it: with nnz + n <= 32768 the 16-block tier is empty, above 2^26 the cap applies.  The weighted build sorts int64
keys through the same tiers with the same key counts (its scratch is twice as many bytes).

Scan (launch_scan): scan_local_kernel scans kScanBlock x kScanItems = 4096 entries per block; scan_block_sums_kernel, one block,
scans the block sums kScanBlock = 1024 at a time, so it loops once per 1024 x 4096 = 4 194 304 scanned entries.

Fill windows (for_fill_windows): the fill runs one launch per row window of SGF_CSR_FILL_WINDOW_MB (128) MiB of entries, at most
kMaxFillWindows (12); past 12 x the window the windows grow.  0 MiB: one launch.

Grids (grid_for): every grid-stride launch is capped at num_sms x 8 blocks of 256 threads: 8 448 warps for the warp-per-row
kernels and 270 336 threads for the edge loops on 132 SMs."""
from dataclasses import dataclass

import torch

SCAN_BLOCK = 1024               # kScanBlock
SCAN_ITEMS = 4                  # kScanItems
WARP_SORT_MAX = 256             # kWarpSortMax
SORT_SMEM_MAX = 2048            # kSortSmemMax
HUB_BLOCKS = 16                 # kHubBlocks
HUB_SCRATCH_MAX = 1 << 26       # kHubScratchMax
MAX_FILL_WINDOWS = 12           # kMaxFillWindows
FILL_WINDOW_MB = 128            # default of SGF_CSR_FILL_WINDOW_MB
SMEM_SORT_BLOCKS_PER_SM = 4     # csr_sort_rows_block_kernel<<<num_sms() * 4, ...>>> of sort_long_rows
GRID_PER_SM = 8                 # grid_for's per_sm
BLOCK = 256                     # threads of every grid_for launch
KEY_BYTES = (4, 8)              # int32 column ids; int64 (col << 32 | eid + 1) keys of the weighted build

TIERS = ("none", "warp1", "warp2", "warp_smem", "block_smem", "hub16", "hub1", "unsorted")


def next_pow2(x: int) -> int:
    p = 1
    while p < x:
        p <<= 1
    return p


def scratch_elems(nnz_plus_n: int) -> int:
    """Keys of the hub-row sort scratch (carve_ws)."""
    p = SORT_SMEM_MAX * HUB_BLOCKS
    while p < nnz_plus_n and p < HUB_SCRATCH_MAX:
        p <<= 1
    return p


def share(nnz_plus_n: int) -> int:
    """Keys of one of the 16 blocks' shares of the scratch."""
    return scratch_elems(nnz_plus_n) // HUB_BLOCKS


def tier(length: int, nnz_plus_n: int) -> str:
    if length <= 1:
        return "none"
    if length <= 32:
        return "warp1"
    if length <= 64:
        return "warp2"
    if length <= WARP_SORT_MAX:
        return "warp_smem"
    p2 = next_pow2(length)
    if p2 <= SORT_SMEM_MAX:
        return "block_smem"
    if p2 <= share(nnz_plus_n):
        return "hub16"
    if p2 <= scratch_elems(nnz_plus_n):
        return "hub1"
    return "unsorted"


def scan_blocks(n: int) -> int:
    """Blocks of scan_local_kernel over n entries."""
    return max(1, -(-n // (SCAN_BLOCK * SCAN_ITEMS)))


def block_sum_passes(n: int) -> int:
    """Iterations of scan_block_sums_kernel's loop over the block sums of an n-entry scan."""
    return -(-scan_blocks(n) // SCAN_BLOCK)


def block_sum_last_pass_partial(n: int) -> bool:
    return scan_blocks(n) % SCAN_BLOCK != 0


def fill_windows(nnz: int, n: int, entry_bytes: int, window_mib: int = FILL_WINDOW_MB) -> dict:
    """for_fill_windows: the window count before and after the cap, rows per window and the launches made."""
    win = window_mib << 20
    want = -(-(nnz + n) * entry_bytes // win) if win > 0 else 1
    nwin = min(want, MAX_FILL_WINDOWS)
    if nwin < 1 or n == 0:
        nwin = 1
    rows_per = -(-n // nwin)
    launches = 1 if nwin == 1 else sum(1 for w in range(nwin) if w * rows_per < n)
    return dict(want=want, windows=nwin, rows_per=rows_per, launches=launches)


def warp_cap(sms: int) -> int:
    """Warps of a capped warp-per-row grid (row sort, row_unique_*, subset count / fill)."""
    return sms * GRID_PER_SM * BLOCK // 32


def edge_cap(sms: int) -> int:
    """Threads of a capped edge / entry loop (count, fill, flags, scatter, unpack, symmetry hashes)."""
    return sms * GRID_PER_SM * BLOCK


def iterations(work: int, cap: int):
    """(fewest, most) iterations a warp / thread of the capped grid runs."""
    return work // cap, -(-work // cap)


# ------------------------------------------------------------------------------------------------
# the graphs of the device sweep
# ------------------------------------------------------------------------------------------------
# Rows are edge targets (sgf_csr_build, by_source = 0, self_loop_mode 0).  A graph's in-degrees are exact: every row gets a
# background length from `bg_cycle` (row r: bg_cycle[r % len(bg_cycle)]), and the rows listed in `special` (length, count) get
# exactly that length instead.  Sources are drawn at random by the device test.
BOUNDARY_LENS = (1, 2, 31, 32, 33, 64, 65, 256, 257, 2048, 2049)
RUN_LENS = (31, 32, 33, 64, 65)         # one row of each of these lengths holds a single repeated source (to_undirected runs)


@dataclass(frozen=True)
class GraphSpec:
    name: str
    n: int
    bg_cycle: tuple
    special: tuple                      # ((length, count), ...)

    def special_rows(self):
        """[(row id, length)]: spread over the id range, two specials never adjacent."""
        lens = [length for length, count in self.special for _ in range(count)]
        step = self.n // (len(lens) + 1)
        assert step >= 2, self.name
        return [((k + 1) * step + 1, length) for k, length in enumerate(lens)]

    def lengths(self) -> torch.Tensor:
        cyc = torch.tensor(self.bg_cycle, dtype=torch.int64)
        lens = cyc[torch.arange(self.n) % cyc.numel()]
        for r, length in self.special_rows():
            lens[r] = length
        return lens

    def nnz(self) -> int:
        return int(self.lengths().sum())


def _smem_rows(count):      # rows of the block-shared-memory tier, lengths spread over (256, 2048]
    return tuple((257 + 7 * (i % 61), 1) for i in range(count))


def _hub16_rows(count):     # rows of the 16-block tier below the 2^18 share of "medium": (2048, 4096 + ...]
    return tuple((2049 + 97 * (i % 53), 1) for i in range(count))


GRAPHS = {
    # nnz + n <= 32768: share = 2048, the 16-block tier is empty and 2049 goes to the single block
    "small": GraphSpec("small", 4003, (0, 1, 2, 3, 4), tuple((length, 2) for length in BOUNDARY_LENS)),
    # share = 2^18: every tier, queues of more than 3 x (132 x 4) and 3 x 16 rows, warp and edge grids past three caps
    "medium": GraphSpec("medium", 250_003, tuple(range(13)),
                        tuple((length, 2) for length in BOUNDARY_LENS) + _smem_rows(1700) + _hub16_rows(60)
                        + ((4 * 2048 + 1, 1), ((1 << 18), 1), ((1 << 18) + 1, 1))),
    # nnz + n > 2^26: the capped scratch (share = 2^22), a row past it, two block-sum passes, three default fill windows
    "large": GraphSpec("large", 5_000_000, (0, 1, 2),
                       tuple((length, 1) for length in BOUNDARY_LENS)
                       + (((1 << 22), 1), ((1 << 22) + 1, 1), ((1 << 26) + 1, 1))),
    # 12.5 M rows, 5 M edges: a row scan of three block-sum passes, the last one partial; edge-list scans of two
    "many": GraphSpec("many", 12_500_000, (1, 1, 0, 0, 0), ((2, 1), (33, 1))),
}
