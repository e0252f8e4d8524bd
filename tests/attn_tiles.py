"""Geometry table of the fused attention kernels' streamed tiles (csrc/attn_softmax.cu).

fwd_kernel, bwd_q_kernel and bwd_kv_kernel are templates over the height BS of the tile that streams through shared memory
(64, 32 or 16 rows); `pick_bs` takes, per launch, the largest height whose double buffer fits next to the resident tiles, so
BS follows the row widths of q/k, v and g.  Each height is its own code path: double-buffer offsets, tile count, the inner
16-row loop and the mask of the last, partial tile.  Every row below names a shape and the heights the library picks for it
(sgf_attn_softmax_tile_rows); together the rows reach every (dtype, mode, kernel, height) that any legal shape reaches.

Row fields: dtype, mode ("softmax": the Frobenius-normalised scores of SGFormerSOFT; "gat": the scaled scores of SGFormerGAT),
heads, m (each head's q/k width; in "gat" mode the key width dk padded as engine.gat_attn_pad pads it), d (v's width per head),
shared_v (one [N, d] v for every head), shared_g (the backward's gradient is one [N, d] block for every head, as the head mean
gives it; else one block per head), dk (the unpadded key width in "gat" mode, else m), and the expected heights."""
from typing import NamedTuple

from sgformer_b200 import engine as E

KINDS = ("fwd", "bwd_q", "bwd_kv")


class Tile(NamedTuple):
    dtype: str
    mode: str
    heads: int
    m: int
    d: int
    shared_v: bool
    shared_g: bool
    dk: int
    rows: tuple          # expected (fwd, bwd_q, bwd_kv) heights

    def __str__(self):
        v = "v1" if self.shared_v else "vH"
        g = "g1" if self.shared_g else "gH"
        return f"{self.dtype}-{self.mode}-h{self.heads}-m{self.m}-dk{self.dk}-d{self.d}-{v}-{g}"


def _soft(dtype, heads, m, d, shared_v, shared_g, rows):
    return Tile(dtype, "softmax", heads, m, d, shared_v, shared_g, m, rows)


def _gat(dtype, heads, dk, d, shared_g, rows):
    return Tile(dtype, "gat", heads, E.gat_attn_pad(dk, E.precision(dtype)), d, False, shared_g, dk, rows)


T, F = True, False
TABLE = [
    # softmax mode, fp32
    _soft("fp32", 2, 64, 64, F, T, (64, 64, 64)),
    _soft("fp32", 2, 64, 64, F, F, (64, 64, 64)),
    _soft("fp32", 1, 256, 256, F, F, (32, 16, 16)),
    _soft("fp32", 2, 128, 128, F, T, (32, 16, 16)),
    _soft("fp32", 2, 128, 128, F, F, (32, 16, 16)),
    _soft("fp32", 2, 120, 120, F, F, (32, 16, 16)),      # 120 columns pad to 128 in shared memory
    _soft("fp32", 8, 32, 32, F, T, (64, 32, 32)),
    _soft("fp32", 2, 32, 64, T, T, (64, 64, 64)),
    _soft("fp32", 4, 64, 64, T, F, (32, 32, 32)),
    _soft("fp32", 2, 64, 128, T, F, (64, 32, 32)),
    _soft("fp32", 2, 128, 256, T, T, (32, 16, 16)),      # with per-head g this shape has no backward tile
    # softmax mode, bf16
    _soft("bf16", 2, 64, 64, F, F, (64, 64, 64)),
    _soft("bf16", 2, 64, 64, T, T, (64, 64, 64)),
    _soft("bf16", 4, 128, 128, F, T, (32, 32, 32)),
    _soft("bf16", 2, 256, 256, F, T, (32, 16, 16)),
    _soft("bf16", 1, 512, 512, F, F, (32, 16, 16)),
    _soft("bf16", 2, 16, 512, T, F, (64, 32, 32)),
    _soft("bf16", 8, 64, 64, T, F, (64, 32, 32)),
    _soft("bf16", 4, 128, 256, T, T, (32, 32, 32)),
    _soft("bf16", 2, 256, 512, T, T, (32, 16, 16)),
    # gat (scaled) mode, fp32: v is always per head
    _gat("fp32", 1, 5, 32, F, (64, 64, 64)),
    _gat("fp32", 3, 21, 64, F, (64, 64, 64)),
    _gat("fp32", 4, 61, 64, T, (32, 32, 32)),
    _gat("fp32", 2, 118, 64, F, (32, 32, 32)),
    _gat("fp32", 2, 128, 128, T, (32, 16, 16)),
    _gat("fp32", 2, 125, 128, F, (32, 16, 16)),
    # gat (scaled) mode, bf16
    _gat("bf16", 3, 5, 16, F, (64, 64, 64)),
    _gat("bf16", 2, 64, 64, T, (64, 64, 64)),
    _gat("bf16", 4, 128, 128, T, (32, 32, 32)),
    _gat("bf16", 4, 117, 128, F, (32, 16, 16)),
    _gat("bf16", 2, 250, 256, T, (32, 16, 16)),
    _gat("bf16", 1, 509, 512, F, (32, 16, 16)),
]


def combos(t: Tile):
    """The (dtype, mode, kernel, height) instantiations a row runs."""
    return {(t.dtype, t.mode, kind, bs) for kind, bs in zip(KINDS, t.rows)}
