"""Test-side restatement of the prompt-mel recipe (reference inference/infer_tool.py:170-181) with plain torch ops, no torchaudio:

    Resample(sr, 24000)                      sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99: pad + conv1d(stride=orig)
    MelSpectrogram(24000, n_fft=1024, hop_length=256, n_mels=100, center=True, power=1)
                                             torch.stft with reflect centring and the periodic Hann window, |.|, HTK filterbank
    log(clip(., 1e-7))

``dtype`` is the arithmetic: float64 gives the reference values, float32 the recipe as torchaudio runs it, so the difference of the
two is the recipe's own rounding error.  The window and the filterbank are the recipe's fp32 tables in both cases (a float64
``MelSpectrogram(...).double()`` keeps their fp32 values); the sinc table is built in fp64 and rounded to ``dtype``, as torchaudio's
``Resample(..., dtype=...)`` does.  oracle/make_golden_mel.py checks the float64 path against torchaudio's own float64 run.
"""
from __future__ import annotations

import math
from typing import List, Optional, Tuple

import torch
import torch.nn.functional as F

SR = 24000
N_FFT = 1024
HOP = 256
N_MELS = 100
F_MAX = 12000.0


def sinc_kernel(orig: int, new: int, dtype: torch.dtype) -> Tuple[torch.Tensor, int]:
    """Phase table [new, 1, 2*width + orig] of the gcd-reduced ratio orig:new, and width."""
    base = min(orig, new) * 0.99
    width = math.ceil(6 * orig / base)
    idx = torch.arange(-width, width + orig, dtype=torch.float64)[None, None] / orig
    t = torch.arange(0, -new, -1, dtype=dtype)[:, None, None] / new + idx     # float32: the phase offsets are fp32 values
    t = (t * base).clamp(-6, 6)
    window = torch.cos(t * math.pi / 6 / 2) ** 2
    t = t * math.pi
    k = torch.where(t == 0, torch.tensor(1.0, dtype=torch.float64), t.sin() / t)
    return (k * (window * (base / orig))).to(dtype), width


def out_length(orig_freq: int, new_freq: int, n: int) -> int:
    """ceil of the fp64 quotient rounded to fp32 (torch.as_tensor of a Python float), over the gcd-reduced ratio."""
    if orig_freq == new_freq:
        return n
    g = math.gcd(orig_freq, new_freq)
    return int(torch.ceil(torch.as_tensor((new_freq // g) * n / (orig_freq // g), dtype=torch.float32)))


def resample(x: torch.Tensor, orig_freq: int, new_freq: int, dtype: torch.dtype = torch.float64) -> torch.Tensor:
    """One utterance x [N] -> [out_length(N)] in dtype."""
    x = x.to(dtype)
    if orig_freq == new_freq:
        return x.clone()
    g = math.gcd(orig_freq, new_freq)
    orig, new = orig_freq // g, new_freq // g
    kernel, width = sinc_kernel(orig, new, dtype)
    kernel = kernel.to(x.device)
    xp = F.pad(x[None, None], (width, width + orig))
    y = F.conv1d(xp, kernel, stride=orig).transpose(1, 2).reshape(-1)
    return y[:out_length(orig_freq, new_freq, x.shape[-1])]


def hann_window() -> torch.Tensor:
    return torch.hann_window(N_FFT, dtype=torch.float32)


def mel_filterbank() -> torch.Tensor:
    """[513, 100] fp32: HTK mel scale, 0 .. 12 kHz, norm=None, in torchaudio melscale_fbanks' fp32 operation order."""
    all_freqs = torch.linspace(0, SR // 2, N_FFT // 2 + 1)
    m_max = 2595.0 * math.log10(1.0 + (F_MAX / 700.0))
    m_pts = torch.linspace(0.0, m_max, N_MELS + 2)
    f_pts = 700.0 * (10.0 ** (m_pts / 2595.0) - 1.0)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts.unsqueeze(0) - all_freqs.unsqueeze(1)
    down = (-1.0 * slopes[:, :-2]) / f_diff[:-1]
    up = slopes[:, 2:] / f_diff[1:]
    return torch.max(torch.zeros(1), torch.min(down, up))


def stft_magnitude(x24: torch.Tensor, window: Optional[torch.Tensor] = None, dtype: torch.dtype = torch.float64) -> torch.Tensor:
    """|STFT| [513, 1 + N // 256] of one 24 kHz utterance [N] (N > 512): reflect centring, ``window`` [1024] (default the
    periodic Hann window), in dtype."""
    w = hann_window() if window is None else window
    return torch.stft(x24.to(dtype), N_FFT, HOP, window=w.to(dtype), center=True, pad_mode="reflect", return_complex=True).abs()


def mel_project(spec: torch.Tensor, fb: Optional[torch.Tensor] = None) -> torch.Tensor:
    """[513, frames] magnitudes -> [100, frames] through ``fb`` [513, 100] (default the HTK filterbank), in spec's dtype."""
    fb = mel_filterbank() if fb is None else fb
    return torch.matmul(spec.transpose(-1, -2), fb.to(spec.dtype)).transpose(-1, -2)


def log_clip(mel: torch.Tensor) -> torch.Tensor:
    """log(clip(., 1e-7)): torch.clip keeps NaN"""
    return torch.log(torch.clip(mel, min=1e-7))


def log_mel_24k(x24: torch.Tensor, dtype: torch.dtype = torch.float64, window: Optional[torch.Tensor] = None,
                fb: Optional[torch.Tensor] = None) -> torch.Tensor:
    """One 24 kHz utterance [N] (N > 512) -> log-mel [100, 1 + N // 256] in dtype, with the recipe's tables unless given."""
    return log_clip(mel_project(stft_magnitude(x24, window, dtype), fb))


def log_mel(x: torch.Tensor, sample_rate: int, dtype: torch.dtype = torch.float64) -> torch.Tensor:
    """The whole recipe for one utterance x [N] at sample_rate."""
    return log_mel_24k(resample(x, sample_rate, SR, dtype), dtype)


def log_mel_batch(wav: torch.Tensor, sample_rate: int, lengths: Optional[List[int]] = None,
                  dtype: torch.dtype = torch.float64) -> Tuple[torch.Tensor, torch.Tensor]:
    """wav [B, N] with per-row lengths -> ([B, 100, 1 + N24 // 256] with zero frames past each row's length, frame lengths [B]),
    every row computed on its own (the reference's per-utterance recipe and its collate's zero padding)."""
    B, N = wav.shape
    lengths = [N] * B if lengths is None else [int(v) for v in lengths]
    S = 1 + out_length(sample_rate, SR, N) // HOP
    out = torch.zeros((B, N_MELS, S), dtype=dtype)
    frames = []
    for b in range(B):
        m = log_mel(wav[b, :lengths[b]], sample_rate, dtype)
        out[b, :, :m.shape[-1]] = m
        frames.append(m.shape[-1])
    return out, torch.tensor(frames, dtype=torch.int64)
