"""The GAT kernels' row geometries at the widths the reference runs, and the host tools that check them element by element.

`csrc/gat.cu` cuts a feature row of H*C elements into 16-byte chunks (4 fp32 / 8 bf16 values), lets lpr lanes cover one row
(lpr = the next power of two >= chunks, at most 32) and gives each lane CPL = ceil(chunks / lpr) of them; every kernel is built
for CPL 1-4 in both dtypes.  `SHAPES` is a table of (dtype, H, C, mean) that runs every (dtype, CPL) instantiation in concat and
head-mean form, with partial last chunks, idle lanes and odd head counts (tests/test_gat_widths_table.py asserts that);
`geometry` restates `gat_geom`.  `edge_keep` / `dense_keep` restate the attention- and input-dropout hashes in vectorised numpy,
and `check_elementwise` is the per-element bound of tests/test_gpu_gat_widths.py:

    |got - ref| <= k * 2^-24 * S   (+ one bf16 ulp of |ref| for an output stored in bf16)

where S is the reference's own sum with every term replaced by its absolute value."""
import os
import re

import numpy as np
import torch

from dropout_mask import EPOCH_MUL, GOLDEN, M64, _fmix64, keep_scale, keep_threshold

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS32 = 2.0 ** -24
K_CAP = 4096        # largest k of a bound: one dropped or doubled edge stays visible on rows of up to ~4 000 entries

# (dtype, H, C, mean).  Beside each: chunks of 16 bytes, lanes per row (lpr), chunks per lane (CPL).
SHAPES = [
    ("fp32", 1, 4, False),      # 1 chunk, lpr 1: 32 rows per warp
    ("fp32", 3, 8, False),      # 6 chunks on 8 lanes: 2 idle
    ("fp32", 8, 16, False),     # 32, CPL 1 full
    ("fp32", 8, 16, True),      # the same, head mean
    ("fp32", 5, 32, False),     # 40, CPL 2 partial
    ("fp32", 2, 128, True),     # 64, CPL 2 full
    ("fp32", 6, 64, False),     # 96, CPL 3
    ("fp32", 6, 64, True),      # the same, head mean
    ("fp32", 7, 72, False),     # 126, CPL 4 partial
    ("fp32", 8, 64, False),     # 128, CPL 4: the reference's recipe (--hidden_channels 64, --gat_heads 8)
    ("fp32", 8, 64, True),      # the recipe's head mean
    ("fp32", 1, 512, False),    # one head over all four chunks of every lane
    ("bf16", 1, 8, False),      # 1 chunk
    ("bf16", 3, 8, True),       # 3 chunks on 4 lanes
    ("bf16", 8, 32, False),     # 32, CPL 1 full
    ("bf16", 8, 64, False),     # 64, CPL 2: the recipe
    ("bf16", 8, 64, True),      # the recipe's head mean
    ("bf16", 5, 104, False),    # 65: only lane 0 has a third chunk
    ("bf16", 6, 128, False),    # 96, CPL 3
    ("bf16", 6, 128, True),     # the same, head mean
    ("bf16", 7, 136, False),    # 119, CPL 4 partial
    ("bf16", 8, 128, True),     # 128, CPL 4 full
]


def shape_id(s) -> str:
    dt, h, c, mean = s
    return f"{dt}-H{h}-C{c}" + ("-mean" if mean else "")


def max_heads() -> int:
    """SGF_GAT_MAX_HEADS of include/sgformer_b200.h."""
    with open(os.path.join(ROOT, "include", "sgformer_b200.h")) as f:
        return int(re.search(r"#define\s+SGF_GAT_MAX_HEADS\s+(\d+)", f.read()).group(1))


def geometry(dtype: str, H: int, C: int):
    """gat_geom of csrc/gat.cu -> (chunks, lpr, cpl), or None where the kernels refuse the shape."""
    vn = 8 if dtype == "bf16" else 4
    if dtype not in ("fp32", "bf16") or H < 1 or H > max_heads() or C <= 0 or C % vn:
        return None
    return _lanes(H * C // vn)


def row_geometry(dtype: str, h: int):
    """make_geom of csrc/rowops.cu (the BatchNorm / activation / dropout row kernels at width h) -> (chunks, lpr, cpl), or None."""
    vn = 8 if dtype == "bf16" else 4
    if dtype not in ("fp32", "bf16") or h <= 0 or h % vn:
        return None
    return _lanes(h // vn)


# (dtype, h) of the ELU checks of bn_fwd / bn_bwd / bn_bwd_sums: CPL 1-4 in both dtypes (tests/test_gat_widths_table.py asserts
# it); bf16 h = 512 is the recipe's hidden layer (8 heads x 64, CPL 2), fp32 h = 512 the same in fp32 (CPL 4).
ELU_WIDTHS = [("fp32", h) for h in (12, 100, 256, 300, 512)] + [("bf16", h) for h in (24, 200, 512, 768, 1024)]


def _lanes(chunks: int):
    lpr_log2 = 0
    while (1 << lpr_log2) < chunks and lpr_log2 < 5:
        lpr_log2 += 1
    lpr = 1 << lpr_log2
    cpl = (chunks + lpr - 1) // lpr
    return (chunks, lpr, cpl) if cpl <= 4 else None


def _hash(seed: int, idx: np.ndarray) -> np.ndarray:
    with np.errstate(over="ignore"):
        return _fmix64(np.uint64(seed & M64) + idx * np.uint64(GOLDEN))


def duplicate_rank(src: np.ndarray, dst: np.ndarray, n: int) -> np.ndarray:
    """Position of each edge among the identical edges (src, dst) before it, in the given order."""
    key = dst.astype(np.int64) * n + src.astype(np.int64)
    order = np.argsort(key, kind="stable")
    ks = key[order]
    start = np.r_[0, np.flatnonzero(ks[1:] != ks[:-1]) + 1]
    run = np.zeros(len(ks), dtype=np.int64)
    run[start] = start
    np.maximum.accumulate(run, out=run)
    rank = np.empty(len(ks), dtype=np.int64)
    rank[order] = np.arange(len(ks)) - run
    return rank


def edge_keep(seed: int, n: int, ei_gat, heads: int, p: float, rank=None) -> torch.Tensor:
    """fp64 [E, heads]: the attention-dropout factor gat_keep draws for every edge of `ei_gat` ([2, E], source row 0, target
    row 1; duplicate ranks in the given order unless `rank` is passed) under `seed` (the epoch already added), at the kernels'
    fp32 scale 65536 / (65536 - thr16)."""
    ei = torch.as_tensor(ei_gat).cpu().numpy().astype(np.int64)
    src, dst = ei[0], ei[1]
    r = duplicate_rank(src, dst, n) if rank is None else np.asarray(rank, dtype=np.int64)
    key = (dst.astype(np.uint64) << np.uint64(32)) | src.astype(np.uint64)
    thr = keep_threshold(p)
    out = np.empty((len(src), heads), dtype=np.float64)
    with np.errstate(over="ignore"):
        base = np.uint64(seed & M64) + key * np.uint64(GOLDEN)
        for h in range(heads):
            salt = ((r.astype(np.uint64) << np.uint64(8)) | np.uint64(h)) * np.uint64(EPOCH_MUL)
            x = _fmix64(base + salt)
            out[:, h] = np.where((x & np.uint64(0xFFFF)) >= np.uint64(thr), keep_scale(p), 0.0)
    return torch.from_numpy(out)


def dense_keep(seed: int, rows: int, cols: int, p: float) -> torch.Tensor:
    """bool [rows, cols]: the elements sgf_dense_dropout keeps under `seed` (the epoch already added); element (r, c) hashes
    index r * cols + c."""
    x = _hash(seed, np.arange(rows * cols, dtype=np.uint64))
    return torch.from_numpy(((x & np.uint64(0xFFFF)) >= np.uint64(keep_threshold(p))).reshape(rows, cols))


def with_epoch(seed: int, epoch: int) -> int:
    return (int(seed) + int(epoch) * EPOCH_MUL) & M64


def bf16_ulp(t: torch.Tensor) -> torch.Tensor:
    """One bf16 ulp of |t| (8 significant bits); 0 where t == 0."""
    m, e = torch.frexp(t.abs())
    return torch.where(m == 0, torch.zeros_like(t), torch.ldexp(torch.ones_like(t), e - 8))


def ratio(got: torch.Tensor, ref: torch.Tensor, S: torch.Tensor, bf16_out: bool) -> torch.Tensor:
    """Per element: (|got - ref| - one bf16 ulp of |ref| if bf16_out) / (2^-24 S), in fp64; inf where got is not finite or S is 0
    with a difference."""
    got, ref, S = got.detach().double(), ref.detach().double().to(got.device), S.detach().double().to(got.device)
    d = (got - ref).abs()
    if bf16_out:
        d = (d - bf16_ulp(ref)).clamp_min(0)
    r = torch.where(d == 0, torch.zeros_like(d), d / (EPS32 * S))
    return torch.where(torch.isfinite(got), r, torch.full_like(r, float("inf")))


def check_elementwise(name: str, got, ref, S, k: float, bf16_out: bool) -> list:
    """|got - ref| <= k 2^-24 S (+ one bf16 ulp of |ref|) per element.  Returns one line per violated tensor, starting with
    `name`: how many elements broke the bound and the worst of them."""
    assert k <= K_CAP, f"{name}: k = {k} above {K_CAP}"
    got = got.detach()
    if tuple(got.shape) != tuple(ref.shape):
        return [f"{name}: shape {tuple(got.shape)} vs {tuple(ref.shape)}"]
    r = ratio(got, ref, S, bf16_out)
    bad = ~(r <= k)
    if not bool(bad.any()):
        return []
    worst = int(torch.argmax(torch.where(bad, r.nan_to_num(float("inf")), torch.zeros_like(r))))
    idx = np.unravel_index(worst, tuple(r.shape))
    g, rf, s = got.double().reshape(-1)[worst].item(), ref.double().reshape(-1)[worst].item(), S.double().reshape(-1)[worst].item()
    return [f"{name}: {int(bad.sum())} of {r.numel()} elements above k={k} (worst at {tuple(int(i) for i in idx)}: got {g:.9g}, "
            f"ref {rf:.9g}, |err| {abs(g - rf):.3e} = {r.reshape(-1)[worst].item():.1f} x 2^-24 S, S {s:.3e})"]
