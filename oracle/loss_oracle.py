"""CPU restatement of the training objective, ``NaturalSpeech2.forward`` (reference model.py:706-734) in eval mode, over
``pre_model_oracle`` and ``unet_oracle``: mask, ``q_sample``, the padded-batch denoiser call and the SNR-weighted MSE.  fp32
reproduces the reference's own arithmetic; fp64 is the yardstick for the device path's error."""
from __future__ import annotations

from typing import Dict, Optional

import torch

from oracle import pre_model_oracle, unet_oracle


def loss_buffers(timesteps: int = 1000, min_snr_gamma: Optional[float] = None) -> Dict[str, torch.Tensor]:
    """model.py:456-498: fp64 schedule, each buffer cast to fp32 by ``register_buffer``."""
    scale = 1000 / timesteps
    betas = torch.linspace(scale * 0.0001, scale * 0.02, timesteps, dtype=torch.float64)
    alphas_cumprod = torch.cumprod(1. - betas, dim=0)
    snr = alphas_cumprod / (1 - alphas_cumprod)
    clipped = snr.clone()
    if min_snr_gamma is not None:
        clipped.clamp_(max=min_snr_gamma)
    return {"sqrt_alphas_cumprod": torch.sqrt(alphas_cumprod).to(torch.float32),
            "sqrt_one_minus_alphas_cumprod": torch.sqrt(1. - alphas_cumprod).to(torch.float32),
            "loss_weight": clipped.to(torch.float32)}


def extract(a: torch.Tensor, t: torch.Tensor, ndim: int) -> torch.Tensor:
    """model.py:422-425"""
    return a.gather(-1, t).reshape(t.shape[0], *((1,) * (ndim - 1)))


@torch.no_grad()
def diffusion_loss(sd_pre, sd_unet, ucfg, c_padded, refer_padded, spec_padded, lengths, refer_lengths, t, noise,
                   dtype: torch.dtype = torch.float32, min_snr_gamma: Optional[float] = None, n_layers=(6, 6)) -> Dict[str, torch.Tensor]:
    """Steps 1-7 of ``forward`` for given ``t`` [B] and unmasked ``noise`` [B, C, T].  The schedule buffers keep their fp32
    values in both precisions (they are part of the number); everything else runs in ``dtype``."""
    cast = lambda v: v.to(dtype)
    sd_pre = {k: cast(v) for k, v in sd_pre.items()}
    sd_unet = {k: cast(v) for k, v in sd_unet.items()}
    buf = {k: cast(v) for k, v in loss_buffers(1000, min_snr_gamma).items()}
    spec = cast(spec_padded)
    x_mask = unet_oracle.sequence_mask(lengths, spec.shape[2]).unsqueeze(1).to(dtype)
    x_start = spec * x_mask
    content, refer = pre_model_oracle.pre_model_infer(sd_pre, cast(c_padded), cast(refer_padded), lengths, refer_lengths, *n_layers)
    noise = cast(noise) * x_mask
    x = extract(buf["sqrt_alphas_cumprod"], t, 3) * x_start + extract(buf["sqrt_one_minus_alphas_cumprod"], t, 3) * noise
    model_out = unet_oracle.denoiser_forward(sd_unet, ucfg, x, content, refer, refer_lengths, t)
    # model.py:723-726: `reduce(loss, 'b ... -> b (...)', 'mean')` only flattens to [B, C*T] (no axis is reduced), and the
    # [B, 1, 1] weights then broadcast it to [B, B, C*T]; the mean of that is mean_b(weight) * mean_b(row MSE)
    sq = ((model_out - x_start) ** 2).reshape(x.shape[0], -1)
    w = buf["loss_weight"].gather(-1, t)
    loss = (sq * w.reshape(-1, 1, 1)).mean()
    loss_row = sq.mean(dim=1)
    return {"x_start": x_start, "x": x, "model_out": model_out, "loss_row": loss_row, "loss_weighted": loss_row * w, "loss": loss}
