"""The silence slicer's framewise RMS as librosa 0.10 computes it (``librosa.feature.rms(y=y, frame_length=win,
hop_length=hop)``, center=True, pad_mode="constant"), restated as its numpy op sequence so that nothing here needs librosa:

* ``np.pad`` of win // 2 zeros at both ends;
* ``util.frame``: an ``as_strided`` window view [..., n_f, win] moved to [win, n_f] and taken every hop frames, so
  n_f = 1 + (N + 2 (win // 2) - win) // hop;
* ``np.mean(util.abs2(frame), axis=-2)`` in float32 (``abs2`` of a real array is its square), then ``np.sqrt``.

The squared frame array is F-contiguous, so numpy reduces each frame with its pairwise float32 sum; the CUDA kernel
(``csrc/slicer.cu``) restates that association and is checked against this module bit for bit.

``slicer_params`` is ``Slicer.__init__``'s arithmetic (reference ``inference/slicer.py:18-24``), Python's ``round`` included.
"""
from __future__ import annotations

from typing import Dict

import numpy as np
from numpy.lib.stride_tricks import as_strided


def frame(y: np.ndarray, frame_length: int, hop_length: int) -> np.ndarray:
    """librosa 0.10 ``util.frame(y, frame_length, hop_length)`` of a 1-D array (axis -1): [frame_length, n_frames]."""
    if y.shape[-1] < frame_length:
        raise ValueError(f"input is too short (n={y.shape[-1]}) for frame_length={frame_length}")
    xw = as_strided(y, shape=(y.shape[-1] - frame_length + 1, frame_length), strides=(y.strides[-1], y.strides[-1]), writeable=False)
    xw = np.moveaxis(xw, -1, -2)
    return xw[:, ::hop_length]


def rms(y: np.ndarray, frame_length: int, hop_length: int) -> np.ndarray:
    """librosa 0.10 ``feature.rms(y=y, frame_length=frame_length, hop_length=hop_length)`` of 1-D float32 y: float32 [1, n_f]."""
    if y.ndim != 1 or y.dtype != np.float32:
        raise ValueError(f"expected 1-D float32 samples, got {y.dtype} {y.shape}")
    y = np.pad(y, (frame_length // 2, frame_length // 2), mode="constant")
    x = frame(y, frame_length, hop_length)
    power = np.mean(np.square(x), axis=-2, keepdims=True)
    return np.sqrt(power)


def slicer_params(sr: int, threshold: float = -40.0, min_length: int = 5000, min_interval: int = 300, hop_size: int = 20,
                  max_sil_kept: int = 5000) -> Dict[str, float]:
    """``Slicer(sr, threshold, min_length, min_interval, hop_size, max_sil_kept)``'s attributes: the linear threshold, hop and
    win in samples, and min_length / min_interval / max_sil_kept in frames."""
    mi = sr * min_interval / 1000
    hop = round(sr * hop_size / 1000)
    return dict(threshold=10 ** (threshold / 20.0), hop=hop, win=min(round(mi), 4 * hop), min_length=round(sr * min_length / 1000 / hop),
                min_interval=round(mi / hop), max_sil_kept=round(sr * max_sil_kept / 1000 / hop))
