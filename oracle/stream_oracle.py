"""fp64 restatement of live conversion's host-visible rules (``ns2vc_b200.stream``): the SOLA join of one tick and the per-slot
input window under ``push`` and ``reset``.  numpy only."""
from __future__ import annotations

import numpy as np


def sola_ratios(seg: np.ndarray, tail: np.ndarray, Nc: int, Ns: int) -> np.ndarray:
    """num(k) / den(k) for k in [0, Ns] in fp64: the correlation of seg[k : k + Nc] with the tail over the segment's energy."""
    s = np.asarray(seg, dtype=np.float64)
    t = np.asarray(tail, dtype=np.float64)[:Nc]
    win = np.lib.stride_tricks.sliding_window_view(s[:Nc + Ns], Nc)            # [Ns + 1, Nc]
    num = (win * t).sum(axis=1)                 # one summation per row, so equal rows give equal sums (exact ties stay ties)
    den = np.sqrt((win * win).sum(axis=1) + 1e-8)
    return num / den


def sola_at(seg: np.ndarray, tail: np.ndarray, fade_in: np.ndarray, Nb: int, Nc: int, k: int):
    """The emitted block and the next tail for offset k, in fp64."""
    s = np.asarray(seg, dtype=np.float64)
    t = np.asarray(tail, dtype=np.float64)
    f = np.asarray(fade_in, dtype=np.float64)
    out = s[k:k + Nb].copy()
    out[:Nc] = s[k:k + Nc] * f + t[:Nc] * (1.0 - f)
    return out, s[k + Nb:k + Nb + Nc].copy()


def sola(seg: np.ndarray, tail: np.ndarray, fade_in: np.ndarray, Nb: int, Nc: int, Ns: int):
    """-> (out [Nb], new_tail [Nc], k): k = argmax of ``sola_ratios``, the lowest k on ties."""
    k = int(np.argmax(sola_ratios(seg, tail, Nc, Ns)))
    out, new_tail = sola_at(seg, tail, fade_in, Nb, Nc, k)
    return out, new_tail, k


class WindowRing:
    """The per-slot input windows [B, W_in] float32: ``push`` shifts every window left by one block and appends it, ``reset``
    zeroes one slot."""

    def __init__(self, B: int, W_in: int):
        self.window = np.zeros((B, W_in), dtype=np.float32)

    def push(self, block: np.ndarray) -> np.ndarray:
        n = block.shape[1]
        self.window = np.concatenate([self.window[:, n:], np.asarray(block, dtype=np.float32)], axis=1)
        return self.window

    def reset(self, slot: int) -> None:
        self.window[slot] = 0.0
