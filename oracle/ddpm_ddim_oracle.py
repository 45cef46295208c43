"""ORACLE (test infrastructure only - never imported by the product path).

Plain-loop CPU restatements of ``NaturalSpeech2.p_sample_loop`` and ``ddim_sample`` with any eta (reference model.py:535-603), the
noise supplied by the caller in the reference's draw order.  ``sampler_oracle.ddim_sample`` covers eta = 0 without noise.
"""
from __future__ import annotations

from typing import Callable, Iterator

import torch

from .sampler_oracle import OracleDDPM


def p_sample_loop(x_start_fn: Callable, x: torch.Tensor, noises: Iterator[torch.Tensor], timesteps: int = 1000) -> torch.Tensor:
    """t = timesteps-1 .. 0; one noise tensor is taken per step with t > 0 (model.py:539)."""
    ddpm = OracleDDPM(timesteps)
    for t in reversed(range(timesteps)):
        x = ddpm.p_sample(x_start_fn, x, t, next(noises) if t > 0 else None)
    return x


def ddim_sample(x_start_fn: Callable, alphas_cumprod: torch.Tensor, x: torch.Tensor, total_timesteps: int, sampling_timesteps: int,
                eta: float, noises: Iterator[torch.Tensor]) -> torch.Tensor:
    """model.py:570-601: one noise tensor per pair except the last, also at eta = 0."""
    times = torch.linspace(-1, total_timesteps - 1, steps=sampling_timesteps + 1)
    times = list(reversed(times.int().tolist()))
    ac = alphas_cumprod.to(torch.float32)
    sqrt_recip = torch.sqrt(1.0 / alphas_cumprod).to(torch.float32)
    sqrt_recipm1 = torch.sqrt(1.0 / alphas_cumprod - 1).to(torch.float32)
    B = x.shape[0]
    for time, time_next in zip(times[:-1], times[1:]):
        bt = torch.full((B,), time, dtype=torch.long)
        x0 = x_start_fn(x, bt)
        pred_noise = (sqrt_recip[bt][:, None, None] * x - x0) / sqrt_recipm1[bt][:, None, None]
        if time_next < 0:
            x = x0
            continue
        alpha, alpha_next = ac[time], ac[time_next]
        sigma = eta * ((1 - alpha / alpha_next) * (1 - alpha_next) / (1 - alpha)).sqrt()
        c = (1 - alpha_next - sigma ** 2).sqrt()
        x = x0 * alpha_next.sqrt() + c * pred_noise + sigma * next(noises)
    return x
