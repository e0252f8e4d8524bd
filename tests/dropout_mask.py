"""Host restatement of the dropout mask the row kernels apply, and the tools that replay it in the oracles.

The kernels draw no mask tensor: every element's keep bit is a pure function of (seed, epoch, row, column, h, p)
(csrc/common.cuh dropout_chunk, csrc/rowops.cu Lane::dropout and SeedArg), so the backward recomputes the forward's mask.
Restated bit for bit:

    s   = seed + epoch * 0xD1B54A32D192ED03                 (mod 2^64; epoch = the registered device word, else 0)
    i   = r * (h/4) + c/4                                    (fp32 and bf16 chunks both reduce to this hash index)
    x   = fmix64(s + i * 0x9E3779B97F4A7C15)                 (mod 2^64)
    u   = (x >> (16 * (c % 4))) & 0xFFFF
    thr = uint32(float32(p) * 65536 + 0.5)                   keep iff u >= thr, kept values scaled by 65536 / (65536 - thr)

`keep_mask` / `keep_scale` compute it in numpy.  `DropoutRecorder` wraps the forward dropout kernels of a kernels module
(the CUDA one, or the CPU emulation) and records (seed, p, rows, h, epoch) per call; `MaskReplayer` stands in for the
oracles' `_dropout(x, p, training)` and applies recorded or stored masks in call order, so a model run on the kernels can
be compared value for value with the fp64 oracle under the same masks."""
from __future__ import annotations

import sys
from dataclasses import dataclass
from typing import List, Optional

import numpy as np
import torch

M64 = (1 << 64) - 1
EPOCH_MUL = 0xD1B54A32D192ED03
GOLDEN = 0x9E3779B97F4A7C15


def _fmix64(x: np.ndarray) -> np.ndarray:
    x = x ^ (x >> np.uint64(33))
    x = x * np.uint64(0xFF51AFD7ED558CCD)
    x = x ^ (x >> np.uint64(33))
    x = x * np.uint64(0xC4CEB9FE1A85EC53)
    return x ^ (x >> np.uint64(33))


def keep_threshold(p: float) -> int:
    """thr16 of the kernels: uint32(float32(p) * 65536.f + 0.5f), evaluated in fp32."""
    return int(np.float32(np.float32(p) * np.float32(65536.0) + np.float32(0.5)))


def keep_scale(p: float) -> float:
    """The kernels' fp32 scale of a kept element, 65536.f / (65536.f - thr16)."""
    return float(np.float32(65536.0) / (np.float32(65536.0) - np.float32(keep_threshold(p))))


def keep_mask(seed: int, rows: int, h: int, p: float, epoch: int = 0) -> np.ndarray:
    """bool [rows, h]: the elements the kernels keep for this (seed, epoch, p) at row width h (h % 4 == 0)."""
    assert h % 4 == 0, h
    s = np.uint64((int(seed) + int(epoch) * EPOCH_MUL) & M64)
    g = h // 4
    idx = np.arange(rows * g, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = _fmix64(s + idx * np.uint64(GOLDEN))
    shifts = np.arange(4, dtype=np.uint64) * np.uint64(16)
    u = (x[:, None] >> shifts[None, :]) & np.uint64(0xFFFF)          # [rows*g, 4]: element c = 4*j + k of hash j
    return (u >= np.uint64(keep_threshold(p))).reshape(rows, h)


def current_epoch() -> int:
    """The device epoch word the kernels add to their seeds, or 0 when none is registered.  sgf_set_dropout_epoch is
    process-global: once a test registers the word, every later dropout kernel call uses it."""
    K = sys.modules.get("sgformer_b200.kernels")
    ep = getattr(K, "_epoch", None) if K is not None else None
    return int(ep.item()) & M64 if ep is not None else 0


@dataclass
class DropCall:
    seed: int
    p: float
    rows: int
    h: int
    epoch: int
    fn: str

    def mask(self) -> np.ndarray:
        return keep_mask(self.seed, self.rows, self.h, self.p, self.epoch)


class DropoutRecorder:
    """Wraps the forward dropout kernels `ln_fwd`, `ln_fwd_graph` and `bn_fwd` of the kernels module `K` (engine.py calls them
    as `K.<name>`) and records every call with p > 0, in call order."""

    FORWARD = {"ln_fwd": (8, 9), "ln_fwd_graph": (10, 11), "bn_fwd": (10, 11)}     # positional index of (p, seed)

    def __init__(self, monkeypatch, K):
        self.calls: List[DropCall] = []
        for name, (ip, iseed) in self.FORWARD.items():
            fn = getattr(K, name, None)
            if fn is not None:
                monkeypatch.setattr(K, name, self._wrap(name, fn, ip, iseed))

    def _wrap(self, name, fn, ip, iseed):
        def wrapped(*args, **kw):
            p, seed = float(args[ip]), int(args[iseed])
            if p > 0.0:
                rows, h = args[0].shape
                self.calls.append(DropCall(seed, p, rows, h, current_epoch(), name))
            return fn(*args, **kw)
        return wrapped

    def masks(self):
        return [(c.p, c.mask()) for c in self.calls]


class MaskReplayer:
    """Drop-in for the oracles' `_dropout(x, p, training)`: every call with p > 0 in training takes the next (p, mask) of the
    queue, checks that p and the shape match, and returns x * mask * scale.  scale='kernel' uses the kernels' fp32 scale,
    scale='ref' the reference's 1/(1-p).  `finish()` asserts that every mask was used."""

    def __init__(self, masks, scale: str = "kernel"):
        assert scale in ("kernel", "ref")
        self.queue = list(masks)
        self.scale = scale
        self.used = 0

    def __call__(self, x: torch.Tensor, p: float, training: bool) -> torch.Tensor:
        if not training or p == 0.0:
            return x
        assert self.queue, f"oracle dropout call {self.used} (p={p}, shape {tuple(x.shape)}) has no recorded mask"
        mp, m = self.queue.pop(0)
        assert abs(float(mp) - float(p)) < 1e-12, f"dropout call {self.used}: p {p} vs recorded {mp}"
        m = torch.as_tensor(np.asarray(m))
        assert tuple(m.shape) == tuple(x.shape), f"dropout call {self.used}: shape {tuple(x.shape)} vs recorded {tuple(m.shape)}"
        self.used += 1
        sc = keep_scale(p) if self.scale == "kernel" else 1.0 / (1.0 - p)
        return x * (m.to(x.dtype) * sc)

    def finish(self):
        assert not self.queue, f"{len(self.queue)} recorded dropout masks were not used by the oracle"


def pack_mask(m: np.ndarray) -> dict:
    """bool [rows, h] -> bit-packed storage (tests/golden/dropout.pt)."""
    m = np.asarray(m, dtype=bool)
    return dict(shape=list(m.shape), bits=torch.from_numpy(np.packbits(m.reshape(-1)).copy()))


def unpack_mask(d: dict) -> np.ndarray:
    shape = tuple(d["shape"])
    n = int(np.prod(shape))
    return np.unpackbits(d["bits"].numpy())[:n].astype(bool).reshape(shape)


def apply_kernel_dropout(t: torch.Tensor, seed: int, p: float, epoch: Optional[int] = None) -> torch.Tensor:
    """t * mask * scale with the kernels' mask for a [rows, h] tensor (emulation / fp64 references)."""
    if p <= 0.0:
        return t
    rows, h = t.shape
    m = torch.from_numpy(keep_mask(seed, rows, h, p, current_epoch() if epoch is None else epoch)).to(t.device)
    return t * (m.to(t.dtype) * keep_scale(p))
