"""Feature-side helpers of the CLI / dataset path in front of the condition encoders (SURVEY.md §8(f) rank 4):

* ``repeat_expand_2d`` - the nearest-frame stretch of the ContentVec features [h, t_src] to the f0 frame count
  (reference ``utils.py:482-496``, called from ``inference/infer_tool.py:166`` and ``dataset.py:37, 85``).

  The reference walks the target frames in a Python loop and copies one column per iteration (on a CUDA tensor: one tiny kernel per
  frame - about a thousand launches per slice, the same order as this package's whole first-call overhead for a new shape).  Here the
  SAME walk runs on the host over the same fp32 boundary table and produces an index vector; the copy is one gather.  Bit-identical
  output (``tests/test_frontend.py``, against outputs recorded from the reference's own function).

  Drop-in: ``utils.repeat_expand_2d = ns2vc_b200.frontend.repeat_expand_2d`` after ``import utils``.

* ``resample`` / ``log_mel_spectrogram`` - the prompt mel ``refer`` [B, 100, S] that ``Pre_model.infer`` takes, computed on the GPU
  for a ragged batch of waveforms: torchaudio ``Resample(sr, 24000)`` then ``MelSpectrogram(24000, n_fft=1024, hop_length=256,
  n_mels=100, center=True, power=1)`` then ``log(clip(., 1e-7))`` per utterance (reference ``inference/infer_tool.py:170-181``,
  ``preprocess.py:27-31, 49-59``).  Kernels in ``csrc/frontend.cu``; accuracy against an fp64 restatement of the recipe in
  ``tests/test_frontend_mel.py``.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, List, Optional, Tuple

import torch

from . import _lib

MEL_SAMPLE_RATE = 24000
N_FFT = 1024
HOP = 256
N_MELS = 100


def repeat_expand_index(src_len: int, target_len: int) -> List[int]:
    """Source column of every target column, exactly as the reference's walk chooses it: boundaries ``temp[j] = j * target_len /
    src_len`` in fp32 (int64 arange times int, true-divided: torch promotes to the default float dtype), the cursor advances by at
    most ONE column per target frame (so a down-stretch lags, like the reference)."""
    if src_len < 1 or target_len < 0:
        raise ValueError(f"repeat_expand: bad lengths {src_len} -> {target_len}")
    temp = (torch.arange(src_len + 1) * target_len / src_len).tolist()      # the reference's own expression (utils.py:487), fp32 values
    idx, pos = [], 0
    for i in range(target_len):
        if not (i < temp[pos + 1]):
            pos += 1
        idx.append(pos)
    return idx


def repeat_expand_2d(content: torch.Tensor, target_len: int) -> torch.Tensor:
    """content [h, t_src] -> float32 [h, target_len] on content's device (reference utils.py:482-496)."""
    if content.dim() != 2:
        raise ValueError(f"content must be [h, t], got {tuple(content.shape)}")
    idx = torch.tensor(repeat_expand_index(content.shape[-1], int(target_len)), dtype=torch.int64, device=content.device)
    return content.to(torch.float).index_select(1, idx)


# ---------------------------------------------------------------------------------------------------------------------------------
# prompt mel
# ---------------------------------------------------------------------------------------------------------------------------------
_resamplers: Dict[Tuple[int, int, int], C.c_void_p] = {}
_mels: Dict[int, C.c_void_p] = {}


def resample_out_length(orig_freq: int, new_freq: int, n: int) -> int:
    """torchaudio's output length of ``Resample(orig_freq, new_freq)`` for n input samples: ``ceil(fp32(new * n / orig))`` over the
    gcd-reduced ratio, the quotient taken in fp64 - not the exact integer ceiling (they first differ at 368 891 samples for
    44.1 -> 24 kHz)."""
    r = _lib.lib().ns2vc_resample_out_length(int(orig_freq), int(new_freq), int(n))
    if r < 0:
        raise ValueError(f"resample: bad arguments {orig_freq} -> {new_freq} Hz, n={n}")
    return r


def resample_check(orig_freq: int, new_freq: int) -> None:
    """Raises ValueError, on the host and before any device work, unless ``resample`` accepts the rate pair: both rates
    positive, and a reduced ratio whose input window per CTA fits in 48 KB of shared memory (46:1 is the first refused)."""
    if _lib.lib().ns2vc_resample_check(int(orig_freq), int(new_freq)) != 0:
        raise ValueError((_lib.lib().ns2vc_last_error() or b"").decode("utf-8", "replace"))


def _rows(wav: torch.Tensor, lengths: Optional[torch.Tensor]):
    """[B, N] or [N] float32 (+ optional int64 [B] lengths) -> (2-D view, was 1-D, host lengths)."""
    if wav.dim() not in (1, 2):
        raise ValueError(f"wav must be [B, N] or [N], got {tuple(wav.shape)}")
    if wav.dtype != torch.float32:
        raise TypeError(f"wav must be float32, got {wav.dtype}")
    squeeze = wav.dim() == 1
    x = wav.unsqueeze(0) if squeeze else wav
    B, N = x.shape
    if B < 1:
        raise ValueError("wav holds no rows")
    if lengths is None:
        host = [N] * B
    else:
        if lengths.dim() != 1 or lengths.shape[0] != B or lengths.dtype.is_floating_point:
            raise ValueError(f"lengths must be an integer tensor [{B}], got {lengths.dtype} {tuple(lengths.shape)}")
        host = [int(v) for v in lengths.tolist()]
        if min(host) < 0 or max(host) > N:
            raise ValueError(f"lengths must lie in [0, {N}], got [{min(host)}, {max(host)}]")
    return x, squeeze, host


def _on_device(x: torch.Tensor, what: str) -> torch.device:
    if x.device.type != "cuda":
        raise RuntimeError(f"ns2vc_b200.frontend.{what} has no CPU path: move the waveform to an H100 ('cuda')")
    return x.device


def _dev_lengths(lengths: Optional[torch.Tensor], dev: torch.device) -> Optional[torch.Tensor]:
    return None if lengths is None else lengths.to(device=dev, dtype=torch.int64).contiguous()


def _resampler(dev: torch.device, orig_freq: int, new_freq: int) -> C.c_void_p:
    key = (dev.index, int(orig_freq), int(new_freq))
    h = _resamplers.get(key)
    if h is None:
        h = C.c_void_p()
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().ns2vc_resampler_create(int(orig_freq), int(new_freq), C.byref(h)))
        _resamplers[key] = h
    return h


def mel_tables() -> Tuple[torch.Tensor, torch.Tensor]:
    """The recipe's fp32 tables as torch computes them: the periodic Hann window [1024] and the HTK filterbank [513, 100] in
    torchaudio ``melscale_fbanks``' operation order (0 .. 12 kHz, norm=None).  torch's vectorised cosf / powf round some entries
    1 ulp apart from the C library's, and quiet mel bands notice that, so the kernel takes these rather than its own."""
    window = torch.hann_window(N_FFT, dtype=torch.float32)
    all_freqs = torch.linspace(0, MEL_SAMPLE_RATE // 2, N_FFT // 2 + 1)
    m_pts = torch.linspace(0.0, 2595.0 * math.log10(1.0 + (MEL_SAMPLE_RATE / 2) / 700.0), N_MELS + 2)
    f_pts = 700.0 * (10.0 ** (m_pts / 2595.0) - 1.0)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts.unsqueeze(0) - all_freqs.unsqueeze(1)
    fb = torch.max(torch.zeros(1), torch.min((-1.0 * slopes[:, :-2]) / f_diff[:-1], slopes[:, 2:] / f_diff[1:]))
    return window.contiguous(), fb.contiguous()


def _mel(dev: torch.device) -> C.c_void_p:
    h = _mels.get(dev.index)
    if h is None:
        h = C.c_void_p()
        window, fb = mel_tables()
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().ns2vc_mel_create(window.data_ptr(), fb.data_ptr(), C.byref(h)))
        _mels[dev.index] = h
    return h


def _resample_rows(x: torch.Tensor, dlen: Optional[torch.Tensor], orig_freq: int, new_freq: int, n_out: int) -> torch.Tensor:
    dev = x.device
    if x.stride(-1) != 1:
        x = x.contiguous()
    B, N = x.shape
    y = torch.empty((B, n_out), dtype=torch.float32, device=dev)
    h = _resampler(dev, orig_freq, new_freq)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().ns2vc_resample(h, x.data_ptr(), x.stride(0), N, None if dlen is None else dlen.data_ptr(), y.data_ptr(),
                                             n_out, n_out, B, torch.cuda.current_stream(dev).cuda_stream))
    return y


def resample(wav: torch.Tensor, orig_freq: int, new_freq: int,
             lengths: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """wav CUDA float32 [B, N] (or [N]), lengths int64 [B] (default all N) -> (y [B, N_out], out_lengths int64 [B]).

    Row b equals ``torchaudio.transforms.Resample(orig_freq, new_freq)(wav[b, :lengths[b]])`` (sinc_interp_hann,
    lowpass_filter_width 6, rolloff 0.99) up to fp32 summation order; samples at or past ``out_lengths[b]`` are exactly 0.
    ``N_out = resample_out_length(orig_freq, new_freq, N)``.  orig_freq == new_freq gives a copy.

    A NaN input sample makes NaN exactly the outputs whose nonzero taps cover it; the others are unchanged.  torchaudio also
    multiplies the exact-zero taps at each phase's ends, so there a NaN reaches a few samples further; downstream the
    utterance is NaN either way."""
    if int(orig_freq) <= 0 or int(new_freq) <= 0:
        raise ValueError(f"resample: bad rates {orig_freq} -> {new_freq}")
    x, squeeze, host = _rows(wav, lengths)
    dev = _on_device(x, "resample")
    n_out = resample_out_length(orig_freq, new_freq, x.shape[1])
    y = _resample_rows(x, _dev_lengths(lengths, dev), orig_freq, new_freq, n_out)
    out_len = torch.tensor([resample_out_length(orig_freq, new_freq, n) for n in host], dtype=torch.int64, device=dev)
    return (y[0] if squeeze else y), out_len


def log_mel_spectrogram(wav: torch.Tensor, sample_rate: int = MEL_SAMPLE_RATE,
                        lengths: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """The prompt mel of reference ``inference/infer_tool.py:170-181`` per utterance of a ragged batch.

    wav CUDA float32 [B, N] (or [N]) at ``sample_rate``, lengths int64 [B] (default all N) -> (mel [B, 100, S] (or [100, S]),
    frame_lengths int64 [B]): ``Resample(sample_rate, 24000)`` when the rate differs, then ``MelSpectrogram(24000, n_fft=1024,
    hop_length=256, n_mels=100, center=True, power=1)`` of ``wav[b, :lengths[b]]`` with the reflect padding at that row's own
    ends, then ``log(max(., 1e-7))``.  ``frame_lengths[b] = 1 + len24k[b] // 256``; frames past it are exactly 0 (the layout of
    the reference's collate, dataset.py:151-173), ``S = 1 + N24k // 256``.  A 24 kHz row of 512 samples or fewer raises
    ValueError, as torch's reflect padding does.

    The clip keeps NaN, as ``torch.clip`` does: a NaN 24 kHz sample makes NaN every band of exactly the frames whose
    reflect-padded window holds it (mirrored positions near both ends included), and +-Inf makes those frames non-finite in
    every band with a nonzero weight; every other frame is unchanged.  A NaN prompt mel then fails its conversion with the
    reference's AssertionError (model.py:404) rather than passing as silence."""
    sr = int(sample_rate)
    if sr <= 0:
        raise ValueError(f"log_mel_spectrogram: bad sample rate {sample_rate}")
    x, squeeze, host = _rows(wav, lengths)
    N = x.shape[1]
    n24 = resample_out_length(sr, MEL_SAMPLE_RATE, N)
    len24 = [resample_out_length(sr, MEL_SAMPLE_RATE, n) for n in host]
    if min(len24) <= N_FFT // 2:
        raise ValueError(f"log_mel_spectrogram: {min(len24)} samples at 24 kHz; the reflect padding needs more than {N_FFT // 2}")
    dev = _on_device(x, "log_mel_spectrogram")
    dlen = _dev_lengths(lengths, dev)
    if sr != MEL_SAMPLE_RATE:
        x = _resample_rows(x, dlen, sr, MEL_SAMPLE_RATE, n24)
        dlen = None if lengths is None else torch.tensor(len24, dtype=torch.int64, device=dev)
    elif x.stride(-1) != 1:
        x = x.contiguous()
    B = x.shape[0]
    S = 1 + n24 // HOP
    mel = torch.empty((B, N_MELS, S), dtype=torch.float32, device=dev)
    h = _mel(dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().ns2vc_log_mel(h, x.data_ptr(), x.stride(0), n24, None if dlen is None else dlen.data_ptr(), mel.data_ptr(),
                                            S, B, torch.cuda.current_stream(dev).cuda_stream))
    frames = torch.tensor([1 + n // HOP for n in len24], dtype=torch.int64, device=dev)
    return (mel[0] if squeeze else mel), frames
