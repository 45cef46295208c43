"""Public convenience API: host tensors in, sampled latents out (what bench.py's ``e2e`` leg times).

``sample_latents`` is the batched equivalent of the sampling block of ``NaturalSpeech2.sample``
(reference model.py:620-686) after ``pre_model.infer``: it takes the condition tensors in the
reference's own layouts (content [T,B,C], prompt [S,B,C], lengths) and returns the mel latents
[B,100,T].  Inputs may live on the host (pinned memory recommended); they are copied to the device,
sampled with the fused loop, and the result is returned on the requested device.
"""
from __future__ import annotations

from typing import Optional

import torch

from .fused import get_session
from .schedule import NoiseScheduleVP
from .synth import linear_betas
from .unet import UNet1DConditionModel

_SCHEDULES = {}


def default_schedule(timesteps: int = 1000) -> NoiseScheduleVP:
    """NoiseScheduleVP('discrete', betas=NaturalSpeech2.betas) (reference model.py:426-433, 622)."""
    if timesteps not in _SCHEDULES:
        _SCHEDULES[timesteps] = NoiseScheduleVP("discrete", betas=linear_betas(timesteps))
    return _SCHEDULES[timesteps]


def sequence_mask(lengths: torch.Tensor, max_length: int) -> torch.Tensor:
    """reference modules/commons.py:149-153"""
    x = torch.arange(max_length, dtype=lengths.dtype, device=lengths.device)
    return x.unsqueeze(0) < lengths.unsqueeze(1)


@torch.no_grad()
def sample_latents(unet: UNet1DConditionModel, x_T: torch.Tensor, content_TBC: torch.Tensor, prompt_SBC: torch.Tensor,
                   prompt_lengths: Optional[torch.Tensor], steps: Optional[int] = None, method: str = "dpmsolver",
                   device: Optional[torch.device] = None, out_device: Optional[torch.device] = None,
                   noise_schedule: Optional[NoiseScheduleVP] = None, skip_type: str = "time_uniform", eta: float = 0.0,
                   noise: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``method``: ``"dpmsolver"`` / ``"unipc"`` (``steps`` solver steps, default 50), ``"ddim"`` (``steps`` = the reference's
    ``sampling_timesteps``, default 100 as in ``sample()``; ``eta`` = ``ddim_sampling_eta``) or ``"ddpm"`` (``p_sample_loop``: every
    timestep 999 .. 0; ``steps`` may be left unset or be 1000).  DDPM / DDIM draw their noise with ``torch.randn_like`` on the
    device's default generator, in the reference's order, unless ``noise`` [N, B, 100, T] (one tensor per step) is given."""
    if method not in ("dpmsolver", "unipc", "ddpm", "ddim"):
        raise ValueError(f"unknown method {method!r} (dpmsolver | unipc | ddpm | ddim)")
    if method in ("ddpm", "ddim"):
        if noise_schedule is not None:
            raise ValueError(f"method {method!r} uses NaturalSpeech2's own schedule buffers; noise_schedule applies to dpmsolver / unipc")
        if method == "ddpm" and steps not in (None, 1000):
            raise ValueError("method 'ddpm' runs every one of the 1000 timesteps (p_sample_loop); use 'ddim' for fewer steps")
    elif noise is not None or eta != 0.0:
        raise ValueError("eta and noise apply to the ddpm / ddim methods")
    if steps is None:
        steps = 100 if method == "ddim" else 50
    dev = torch.device(device) if device is not None else next(unet.parameters()).device
    if dev.type != "cuda":
        raise RuntimeError("sample_latents needs the model on a CUDA device (no CPU path)")
    ns = noise_schedule or default_schedule()
    nb = True
    x = x_T.to(dev, torch.float32, non_blocking=nb)
    content = content_TBC.to(dev, torch.float32, non_blocking=nb).permute(1, 2, 0)
    prompt = prompt_SBC.to(dev, torch.float32, non_blocking=nb).permute(1, 0, 2)
    mask = None
    if prompt_lengths is not None:
        mask = sequence_mask(prompt_lengths.to(dev, non_blocking=nb), prompt_SBC.shape[0])
    sess = get_session(unet, content, prompt, mask)
    if method == "ddpm":
        out = sess.sample_ddpm(x, noise=noise)
        return out.to(out_device) if out_device is not None else out
    if method == "ddim":
        out = sess.sample_ddim(x, steps, eta=eta, noise=noise)
        return out.to(out_device) if out_device is not None else out
    t_T, t_0 = ns.T, 1.0 / ns.total_N
    if skip_type != "time_uniform":
        raise ValueError("sample_latents supports skip_type='time_uniform' (the reference's setting)")
    ts = torch.linspace(t_T, t_0, steps + 1)
    if method == "dpmsolver":
        out = sess.sample_dpmpp_2m(x, ns, ts)
    else:
        out = sess.sample_unipc(x, ns, ts, variant="bh2")
    if out_device is not None:
        out = out.to(out_device)
    return out


@torch.no_grad()
def sample_from_features(pre_model, unet: UNet1DConditionModel, x_T: torch.Tensor, c_padded: torch.Tensor, refer_padded: torch.Tensor,
                         lengths: torch.Tensor, refer_lengths: torch.Tensor, steps: Optional[int] = None, method: str = "dpmsolver",
                         device: Optional[torch.device] = None, out_device: Optional[torch.device] = None, eta: float = 0.0,
                         noise: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The device part of ``NaturalSpeech2.sample`` before the vocoder (reference model.py:606-686): ``pre_model.infer`` (condition
    encoders) followed by the sampling run.  c_padded [B, 256, T] (ContentVec features), refer_padded [B, 100, S] (mel prompt),
    lengths / refer_lengths [B]; host tensors are copied to the device.  Returns the mel latents [B, 100, T].  ``steps``, ``method``,
    ``eta`` and ``noise`` as for ``sample_latents``."""
    dev = torch.device(device) if device is not None else next(unet.parameters()).device
    data = (c_padded.to(dev, torch.float32, non_blocking=True), refer_padded.to(dev, torch.float32, non_blocking=True), None, None, None,
            lengths.to(dev, non_blocking=True), refer_lengths.to(dev, non_blocking=True), None)
    content, prompt = pre_model.infer(data)
    return sample_latents(unet, x_T, content, prompt, data[6], steps=steps, method=method, device=dev, out_device=out_device, eta=eta,
                          noise=noise)
