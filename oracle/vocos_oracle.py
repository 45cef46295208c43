"""TEST INFRASTRUCTURE ONLY — functional ATen restatement of ``Vocos.decode`` for the mel configuration (no AdaLayerNorm,
ISTFT padding "same"), written from the package's published architecture:

  vocos/models.py      VocosBackbone   embed Conv1d(k=7, pad 3) -> LayerNorm(eps 1e-6) -> ConvNeXtBlocks -> final LayerNorm
  vocos/modules.py     ConvNeXtBlock   x + gamma * pwconv2(gelu(pwconv1(LayerNorm(dwconv(x)))))   (depthwise k=7, pad 3)
  vocos/heads.py       ISTFTHead       Linear(dim, n_fft + 2) -> mag, p = chunk(2) -> clip(exp(mag), max=100) * (cos p + i sin p)
  vocos/spectral_ops.py ISTFT          irfft(n_fft, norm="backward") * window, overlap-add (F.fold) at hop, trimmed by
                                       (n_fft - hop) / 2 on both ends, divided by the overlap-added window^2

The ``vocos`` package is not available here, so this restatement is NOT pinned against it; its ISTFT is pinned independently
by a round trip through ``torch.stft`` (tests/test_vocoder.py).  Everything runs in the dtype of the input (fp32 or fp64) on
the input's device.  Activations are token-major [B, T, C] between the stages, as the GPU engine's taps are.
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence

import torch
import torch.nn.functional as F

EPS = 1e-6


def _w(sd: Dict[str, torch.Tensor], k: str, like: torch.Tensor) -> torch.Tensor:
    return sd[k].to(like.device, like.dtype)


def embed_norm(sd, mel: torch.Tensor) -> torch.Tensor:
    """mel [B, C_in, T] -> backbone.norm(embed(mel)) [B, T, dim]."""
    x = F.conv1d(mel, _w(sd, "backbone.embed.weight", mel), _w(sd, "backbone.embed.bias", mel), padding=3)
    x = x.transpose(1, 2)
    return F.layer_norm(x, (x.shape[-1],), _w(sd, "backbone.norm.weight", x), _w(sd, "backbone.norm.bias", x), EPS)


def convnext_block(sd, i: int, x: torch.Tensor) -> torch.Tensor:
    """backbone.convnext.i on token-major x [B, T, dim]."""
    p = f"backbone.convnext.{i}"
    D = x.shape[-1]
    h = F.conv1d(x.transpose(1, 2), _w(sd, p + ".dwconv.weight", x), _w(sd, p + ".dwconv.bias", x), padding=3, groups=D).transpose(1, 2)
    h = F.layer_norm(h, (D,), _w(sd, p + ".norm.weight", x), _w(sd, p + ".norm.bias", x), EPS)
    h = F.gelu(F.linear(h, _w(sd, p + ".pwconv1.weight", x), _w(sd, p + ".pwconv1.bias", x)))
    h = F.linear(h, _w(sd, p + ".pwconv2.weight", x), _w(sd, p + ".pwconv2.bias", x))
    return x + _w(sd, p + ".gamma", x) * h


def final_norm(sd, x: torch.Tensor) -> torch.Tensor:
    return F.layer_norm(x, (x.shape[-1],), _w(sd, "backbone.final_layer_norm.weight", x), _w(sd, "backbone.final_layer_norm.bias", x), EPS)


def head_linear(sd, x: torch.Tensor) -> torch.Tensor:
    """head.out: [B, T, dim] -> [B, T, n_fft + 2] (log-magnitudes, then phases)."""
    return F.linear(x, _w(sd, "head.out.weight", x), _w(sd, "head.out.bias", x))


def istft_same(S: torch.Tensor, window: torch.Tensor, hop: int) -> torch.Tensor:
    """ISTFT(padding="same") of a one-sided spectrum S [B, n_fft / 2 + 1, T] -> [B, T * hop]."""
    n_fft = window.numel()
    pad = (n_fft - hop) // 2
    T = S.shape[-1]
    frames = torch.fft.irfft(S, n_fft, dim=1, norm="backward") * window[None, :, None]
    out = (T - 1) * hop + n_fft
    y = F.fold(frames, output_size=(1, out), kernel_size=(1, n_fft), stride=(1, hop))[:, 0, 0, pad:-pad]
    env = F.fold(window.square().expand(1, T, -1).transpose(1, 2), output_size=(1, out), kernel_size=(1, n_fft),
                 stride=(1, hop)).squeeze()[pad:-pad]
    assert (env > 1e-11).all()
    return y / env


def head_istft(h: torch.Tensor, window: torch.Tensor, hop: int) -> torch.Tensor:
    """The rest of ISTFTHead.forward: h [B, T, n_fft + 2] -> audio [B, T * hop]."""
    mag, p = h.transpose(1, 2).chunk(2, dim=1)
    mag = torch.clip(torch.exp(mag), max=1e2)
    S = mag * (torch.cos(p) + 1j * torch.sin(p))
    return istft_same(S, window.to(h.device, h.dtype), hop)


def decode_stages(sd, mel: torch.Tensor, hop: int = 256) -> Dict[str, torch.Tensor]:
    """Every stage of ``decode`` on mel [B, C_in, T], keyed like the engine's taps, plus ``"audio"``."""
    out = {}
    x = out["backbone.norm"] = embed_norm(sd, mel)
    i = 0
    while f"backbone.convnext.{i}.gamma" in sd:
        x = out[f"backbone.convnext.{i}"] = convnext_block(sd, i, x)
        i += 1
    x = out["backbone.final_layer_norm"] = final_norm(sd, x)
    h = out["head.out"] = head_linear(sd, x)
    out["audio"] = head_istft(h, sd["head.istft.window"], hop)
    return out


def decode(sd, mel: torch.Tensor, hop: int = 256, lengths: Optional[Sequence[int]] = None, dtype=torch.float64) -> torch.Tensor:
    """``Vocos.decode(mel)`` in ``dtype``; with ``lengths`` each row b is decoded alone on mel[b, :, :lengths[b]] and zero-padded
    to T * hop samples."""
    mel = mel.to(dtype)
    if lengths is None:
        return decode_stages(sd, mel, hop)["audio"]
    B, _, T = mel.shape
    audio = mel.new_zeros((B, T * hop))
    for b, L in enumerate(int(v) for v in lengths):
        audio[b, :L * hop] = decode_stages(sd, mel[b:b + 1, :, :L], hop)["audio"][0]
    return audio
