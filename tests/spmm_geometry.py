"""The launch geometry of the CSR gather kernels (csrc/spmm.cu, csrc/edge_weight.cu), restated in plain Python.

A feature row of h values is moved in 16-byte chunks of VN values (VN = 4 fp32, 8 bf16): chunks = h / VN.  Each neighbour row
is gathered by `lpr` = min(32, next_pow2(chunks)) lanes, and each lane handles `cpl` = ceil(chunks / lpr) chunks, in `cpl`
passes of lpr chunks; `cpl` is instantiated for 1 to 4.  When chunks is not a multiple of lpr the last pass is partial: only
`last_live` lanes of a group hold a chunk in it, the other `idle` lanes load nothing.

Grids (one warp per row, segment or edge-gradient row; 8 warps per CTA):
  rows, segments, phased ranges  SMs x kMinBlocks (4) x 8 CTAs          = row_cap warps (33,792 on 132 SMs)
  hub-row finalize               SMs x 32 blocks x 256 threads          = finalize_cap threads (one per output value)
  edge-weight gradient           SMs x 8 CTAs                           = edge_grad_cap warps (8,448 on 132 SMs)
Past its cap a launch grid-strides.  The plans below pick work counts past three caps, so every warp (thread) of the capped grid
runs at least three iterations:
  ragged  3 x cap + tail, the tail ending inside a CTA (tail % 8 != 0: the last CTA has live and idle warps);
  exact   3 x cap: every warp's last iteration lands on the `r < n` boundary."""
import torch

F32, B16 = torch.float32, torch.bfloat16
WARPS_PER_CTA = 8
MIN_BLOCKS = 4                  # kMinBlocks of csrc/spmm.cu
MAX_CPL = 4                     # cpl instantiations of launch_spmm / launch_heavy / launch_range
HEAVY_ROW = 1024                # kernels.HEAVY_ROW: longer rows take the segmented path
MAX_ROW_BYTES = 2048            # 128 chunks of 16 bytes: the widest row of the SpMM and of the edge-weight gradient


def vn(dtype) -> int:
    return 8 if dtype == B16 else 4


def name(dtype) -> str:
    return "bf16" if dtype == B16 else "fp32"


def geom(dtype, h: int) -> dict:
    """chunks, lanes per neighbour row, chunks per lane, live lanes of the last pass and lanes idle in it."""
    assert h % vn(dtype) == 0
    chunks = h // vn(dtype)
    lpr = 1
    while lpr < chunks and lpr < 32:
        lpr *= 2
    cpl = -(-chunks // lpr)
    last_live = chunks - lpr * (cpl - 1)
    return dict(chunks=chunks, lpr=lpr, cpl=cpl, last_live=last_live, idle=lpr - last_live, partial=last_live < lpr)


def launch_refuses(dtype, h: int) -> bool:
    """launch_spmm / launch_heavy / launch_range return an error: h not a multiple of VN (SGF_ERR_ARG) or wider than 4 chunks
    per lane (SGF_ERR_UNSUPPORTED)."""
    return h % vn(dtype) != 0 or geom(dtype, h)["cpl"] > MAX_CPL


def klass(dtype, h: int):
    g = geom(dtype, h)
    return dtype, g["lpr"], g["cpl"]


def row_cap(sms: int) -> int:
    """Warps of the capped row / segment / range grid."""
    return sms * MIN_BLOCKS * 8 * WARPS_PER_CTA


def finalize_cap(sms: int) -> int:
    """Threads of the capped hub-row finalize grid (its block count is capped like the row grid's)."""
    return sms * MIN_BLOCKS * 8 * 256


def edge_grad_cap(sms: int) -> int:
    """Warps of the capped edge-weight gradient grid (grid_for in csrc/edge_weight.cu)."""
    return sms * 8 * WARPS_PER_CTA


def edge_grad_max_width(dtype) -> int:
    """The widest row sgf_edge_weight_grad takes: 2 KB of a_c spread over 32 lanes."""
    return MAX_ROW_BYTES // (4 if dtype == F32 else 2)


def plan(cap: int, kind: str) -> int:
    tail = cap // 2 + 3
    return {"ragged": 3 * cap + tail, "exact": 3 * cap}[kind]


PLANS = ("ragged", "exact")


def iterations(work: int, cap: int):
    """(fewest, most) iterations a warp / thread of the capped grid runs."""
    return work // cap, -(-work // cap)


# hub rows past the segment cap: `rows` hub rows of SEG_PER_ROW segments each (the last one short), so n_seg > 3 x row_cap
SEG_PER_ROW = 1000
SEG_ROW_LEN = SEG_PER_ROW * HEAVY_ROW - 100


def segment_plan(sms: int) -> dict:
    rows = -(-plan(row_cap(sms), "ragged") // SEG_PER_ROW)
    return dict(rows=rows, row_len=SEG_ROW_LEN, n_seg=rows * SEG_PER_ROW)


def finalize_plan(dtype, h: int, sms: int) -> dict:
    """Hub rows of 2 segments each (lengths 1025 + 256 k, k < 4), enough of them that n_heavy x h > 3 x finalize_cap."""
    n_heavy = 3 * -(-finalize_cap(sms) // h) + 5
    return dict(n_heavy=n_heavy, lens=[HEAVY_ROW + 1 + 256 * (i % 4) for i in range(n_heavy)])


# one or more widths for every (dtype, lpr, cpl) class; partial last passes at every cpl >= 2
WIDTHS = {
    F32: [4, 8, 12, 16, 32, 64, 100, 128, 132, 256, 300, 384, 388, 512],
    B16: [8, 16, 24, 64, 96, 128, 200, 256, 264, 512, 520, 768, 776, 1024],
}
WIDTH_LIST = [(d, h) for d in (F32, B16) for h in WIDTHS[d]]
WIDTH_IDS = [f"{name(d)}-h{h}" for d, h in WIDTH_LIST]

# the widths the launches refuse: one wider than 4 chunks per lane and one not a multiple of VN per dtype
REFUSED = [(F32, 516), (F32, 6), (B16, 1032), (B16, 12)]

# a few widths per (lpr, cpl) class for the float-input checks
FLOAT_WIDTHS = [(F32, 4), (F32, 12), (F32, 100), (F32, 132), (F32, 300), (F32, 512), (B16, 8), (B16, 96), (B16, 264), (B16, 520),
                (B16, 776), (B16, 1024)]

# edge-weight gradient widths, up to the widest each dtype admits
EDGE_GRAD_WIDTHS = [(F32, 4), (F32, 32), (F32, 100), (F32, 512), (B16, 8), (B16, 256), (B16, 520), (B16, 768), (B16, 1024)]
