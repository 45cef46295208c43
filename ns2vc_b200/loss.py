"""The training objective of ``NaturalSpeech2.forward`` (reference model.py:706-734) evaluated under ``no_grad``: the number the
reference's training step minimises, for comparing checkpoints on held-out batches and for seeing where in the noise schedule a
checkpoint is weak.  No gradients: training itself keeps the reference's modules.

One call evaluates K timesteps per batch.  The condition encoders and the denoiser's step-invariant conditioning run once; the K
noisy inputs come from one ``q_sample`` launch, the K predictions from K denoiser forwards on one session, and every loss from
one deterministic reduction (``csrc/loss.cu``).  Eval mode only: ``Pre_model.forward`` is ``Pre_model.infer`` without dropout.

The loss of a row is the mean over all ``C x T`` elements of the PADDED row, as in the reference (past a row's length the target
is 0 and the prediction is whatever the network emits there).  Inputs must be finite: the length mask is a 0/1 factor, as in the
reference, so a non-finite value past a length turns the row into NaN.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional, Tuple

import torch

from . import _lib, coefs
from .api import sequence_mask
from .fused import check_lengths, get_session
from .unet import UNet1DConditionModel

_BUFFERS = {}


def _loss_buffers(timesteps: int, dev: torch.device) -> dict:
    key = (timesteps, str(dev))
    if key not in _BUFFERS:
        _BUFFERS[key] = {k: v.to(dev) for k, v in coefs.loss_buffers(timesteps).items()}
    return _BUFFERS[key]


@dataclass
class DiffusionLoss:
    """``loss`` [K] (0-d for one timestep per row): mean over the batch of ``loss_weighted``; ``loss_row`` [K, B]: the unweighted
    per-row MSE; ``loss_weighted`` [K, B]: times ``loss_weight[t]``; ``t`` [K, B]; ``x`` / ``model_out`` [K, B, C, T]: the noisy
    input and the predicted x_start; ``target`` [B, C, T]: the masked x_start.  The leading K is dropped when ``t`` was [B] or
    None."""
    loss: torch.Tensor
    loss_row: torch.Tensor
    loss_weighted: torch.Tensor
    t: torch.Tensor
    x: torch.Tensor
    model_out: torch.Tensor
    target: torch.Tensor


def draw_t_noise(x_start: torch.Tensor, t: Optional[torch.Tensor], noise: Optional[torch.Tensor],
                 timesteps: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """The reference's draws on ``x_start``'s device's default generator, in its order (model.py:714-716): ``torch.randint(0,
    timesteps, (B,))`` when ``t`` is None, then ``torch.randn_like(x_start)`` when ``noise`` is None: once for a [B] ``t``, once
    per k in k order for a [K, B] ``t``.  Returns (t, noise) as given or drawn."""
    if t is None:
        t = torch.randint(0, timesteps, (x_start.shape[0],), device=x_start.device).long()
    if noise is None:
        noise = torch.randn_like(x_start) if t.dim() == 1 else torch.stack([torch.randn_like(x_start) for _ in range(t.shape[0])])
    return t, noise


def q_sample(spec: torch.Tensor, noise: torch.Tensor, lengths: torch.Tensor, t: torch.Tensor, timesteps: int = 1000,
             want_noise: bool = False):
    """spec [B, C, T], noise [B, C, T] or [K, B, C, T], lengths [B] and t [K, B] int64, on one CUDA device ->
    (x_start [B, C, T], x [K, B, C, T]) and, with ``want_noise``, the masked noise: the reference's ``spec * x_mask``,
    ``q_sample(x_start, t, randn * x_mask)`` bit for bit."""
    K, B = t.shape
    _, Cl, T = spec.shape
    dev = spec.device
    buf = _loss_buffers(timesteps, dev)
    x_start = torch.empty_like(spec)
    x = torch.empty((K, B, Cl, T), dtype=torch.float32, device=dev)
    noise_m = torch.empty_like(noise) if want_noise else None
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().ns2vc_q_sample(
            spec.data_ptr(), noise.data_ptr(), int(noise.dim() == 4), lengths.data_ptr(), t.data_ptr(),
            buf["sqrt_alphas_cumprod"].data_ptr(), buf["sqrt_one_minus_alphas_cumprod"].data_ptr(), timesteps, x_start.data_ptr(),
            noise_m.data_ptr() if want_noise else None, x.data_ptr(), K, B, Cl, T, torch.cuda.current_stream(dev).cuda_stream))
    return (x_start, x, noise_m) if want_noise else (x_start, x)


def mse_rows(out: torch.Tensor, target: torch.Tensor, t: torch.Tensor, timesteps: int = 1000, min_snr_gamma: Optional[float] = None,
             ws: Optional[torch.Tensor] = None):
    """out [K, B, C, T], target [B, C, T] or [K, B, C, T], t [K, B] int64 on one CUDA device -> (loss_row [K, B],
    loss_weighted [K, B], loss [K]); deterministic (see ``ns2vc_mse_rows``).  ``ws``: scratch to reuse (uint8, 8-byte aligned)."""
    K, B, Cl, T = out.shape
    dev = out.device
    L = _lib.lib()
    need = C.c_size_t()
    _lib.check(L.ns2vc_mse_workspace_bytes(K, B, Cl, T, C.byref(need)))
    if ws is None:
        ws = torch.empty(need.value, dtype=torch.uint8, device=dev)
    elif ws.numel() < need.value:
        raise ValueError(f"workspace of {ws.numel()} bytes, {need.value} needed")
    loss_row = torch.empty((K, B), dtype=torch.float32, device=dev)
    loss_weighted = torch.empty((K, B), dtype=torch.float32, device=dev)
    loss = torch.empty((K,), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(L.ns2vc_mse_rows(out.data_ptr(), target.data_ptr(), int(target.dim() == 4), t.data_ptr(),
                                    _loss_buffers(timesteps, dev)["loss_weight"].data_ptr(), timesteps,
                                    float(min_snr_gamma) if min_snr_gamma is not None else 0.0, loss_row.data_ptr(),
                                    loss_weighted.data_ptr(), loss.data_ptr(), K, B, Cl, T, ws.data_ptr(),
                                    torch.cuda.current_stream(dev).cuda_stream))
    return loss_row, loss_weighted, loss


def _check_args(unet, data, t, noise, timesteps, min_snr_gamma):
    """Host-side argument checks; returns (B, C, T, S)."""
    if len(data) != 8:
        raise ValueError("data must be the reference's 8-tuple (c_padded, refer_padded, f0_padded, spec_padded, wav_padded, lengths, "
                         "refer_lengths, uv_padded)")
    c_padded, refer_padded, _f0, spec_padded, _wav, lengths, refer_lengths, _uv = data
    Cl = unet.latent_channels
    if unet.cfg.out_channels != Cl:
        raise ValueError("the x_start objective needs a denoiser with out_channels equal to its latent channels")
    if spec_padded.dim() != 3 or spec_padded.shape[1] != Cl:
        raise ValueError(f"spec_padded must be [B, {Cl}, T], got {tuple(spec_padded.shape)}")
    B, _, T = spec_padded.shape
    if c_padded.dim() != 3 or c_padded.shape[0] != B or c_padded.shape[2] != T:
        raise ValueError(f"c_padded must be [{B}, C, {T}] like spec_padded, got {tuple(c_padded.shape)}")
    if refer_padded.dim() != 3 or refer_padded.shape[0] != B:
        raise ValueError(f"refer_padded must be [{B}, C, S], got {tuple(refer_padded.shape)}")
    S = refer_padded.shape[2]
    check_lengths(lengths, B, T, "lengths")
    check_lengths(refer_lengths, B, S, "refer_lengths")
    if int(timesteps) < 1:
        raise ValueError("timesteps must be >= 1")
    if min_snr_gamma is not None and not float(min_snr_gamma) > 0:
        raise ValueError("min_snr_gamma must be positive")
    if t is not None:
        if not torch.is_tensor(t) or t.dtype != torch.int64 or t.dim() not in (1, 2) or t.shape[-1] != B or t.numel() == 0:
            raise ValueError(f"t must be an int64 tensor [{B}] or [K, {B}]")
        if int(t.min()) < 0 or int(t.max()) >= timesteps:
            raise ValueError(f"t must lie in [0, {timesteps})")
    if noise is not None:
        ok = [(B, Cl, T)]
        if t is not None and t.dim() == 2:
            ok.append((t.shape[0], B, Cl, T))
        if not torch.is_tensor(noise) or tuple(noise.shape) not in ok:
            raise ValueError(f"noise must have one of the shapes {ok}, got {tuple(noise.shape) if torch.is_tensor(noise) else noise!r}")
    return B, Cl, T, S


@torch.no_grad()
def diffusion_loss(pre_model, unet: UNet1DConditionModel, data, t: Optional[torch.Tensor] = None, noise: Optional[torch.Tensor] = None,
                   timesteps: int = 1000, min_snr_gamma: Optional[float] = None) -> DiffusionLoss:
    """``NaturalSpeech2.forward(data, vocos)`` (reference model.py:706-734) without gradients, with ``pre_model`` / ``unet`` this
    package's ``Pre_model`` / ``UNet1DConditionModel`` in eval mode on a CUDA device.  ``data`` is the reference's 8-tuple (the
    output of ``TextAudioCollate``); only ``c_padded`` [B, 256, T], ``refer_padded`` [B, 100, S], ``spec_padded`` [B, 100, T],
    ``lengths`` [B] and ``refer_lengths`` [B] are read.

    ``t``: None (drawn as the reference draws it), int64 [B], or [K, B] for K timesteps per row behind one run of the encoders.
    ``noise``: None (``torch.randn_like``, once per k), [B, C, T] (shared by every k) or [K, B, C, T]; it is masked by the
    lengths as in the reference.  With both None, the call consumes the device's default generator exactly as the reference's
    ``forward`` does (``randint`` then ``randn_like``), so after the same ``torch.manual_seed`` it evaluates the same draws.
    ``min_snr_gamma``: the clamp of ``min_snr_loss_weight=True`` (the reference's default is no clamp)."""
    B, Cl, T, S = _check_args(unet, data, t, noise, timesteps, min_snr_gamma)
    dev = next(unet.parameters()).device
    if dev.type != "cuda":
        raise RuntimeError("diffusion_loss needs the models on a CUDA device (no CPU path)")
    c_padded, refer_padded, _f0, spec_padded, _wav, lengths, refer_lengths, _uv = data
    f32 = lambda v: v.to(dev, torch.float32, non_blocking=True).contiguous()
    spec = f32(spec_padded)
    len_c = lengths.to(dev, torch.int64, non_blocking=True).contiguous()
    len_r = refer_lengths.to(dev, torch.int64, non_blocking=True).contiguous()
    content, prompt = pre_model.infer((f32(c_padded), f32(refer_padded), None, None, None, len_c, len_r, None))
    t, noise = draw_t_noise(spec, t.to(dev) if t is not None else None, f32(noise) if noise is not None else None, timesteps)
    single = t.dim() == 1
    t2 = (t[None] if single else t).contiguous()
    x_start, x = q_sample(spec, noise, len_c, t2, timesteps)
    sess = get_session(unet, content.permute(1, 2, 0), prompt.permute(1, 0, 2), sequence_mask(len_r, S))
    model_out = sess.eval_x_start(x, t2, torch.empty_like(x))
    loss_row, loss_weighted, loss = mse_rows(model_out, x_start, t2, timesteps, min_snr_gamma)
    if single:
        loss, loss_row, loss_weighted, x, model_out = loss[0], loss_row[0], loss_weighted[0], x[0], model_out[0]
    return DiffusionLoss(loss=loss, loss_row=loss_row, loss_weighted=loss_weighted, t=t, x=x, model_out=model_out, target=x_start)


def loss_profile(pre_model, unet: UNet1DConditionModel, data, t_grid=range(0, 1000, 50), noise: Optional[torch.Tensor] = None,
                 timesteps: int = 1000, min_snr_gamma: Optional[float] = None) -> DiffusionLoss:
    """The objective at a grid of timesteps, every row of the batch at the same ``t_k``: ``loss`` [K] is the curve that shows
    where in the noise schedule a checkpoint is weak, ``loss_row`` [K, B] its unweighted per-row MSE.  ``noise`` as for
    ``diffusion_loss`` (one [B, C, T] tensor makes the K points differ in ``t`` only)."""
    grid = [int(v) for v in t_grid]
    if not grid:
        raise ValueError("t_grid is empty")
    B = data[3].shape[0]
    t = torch.tensor(grid, dtype=torch.int64)[:, None].expand(len(grid), B).contiguous()
    return diffusion_loss(pre_model, unet, data, t=t, noise=noise, timesteps=timesteps, min_snr_gamma=min_snr_gamma)
