"""The training objective of ``NaturalSpeech2.forward`` (reference model.py:706-734) evaluated under ``no_grad``: the number the
reference's training step minimises, for comparing checkpoints on held-out batches and for seeing where in the noise schedule a
checkpoint is weak.  No gradients: training itself keeps the reference's modules.

One call evaluates K timesteps per batch.  The condition encoders and the denoiser's step-invariant conditioning run once; the K
noisy inputs come from one ``q_sample`` launch, the K predictions from K denoiser forwards on one session, and every loss from
one deterministic reduction (``csrc/loss.cu``).  Eval mode only: ``Pre_model.forward`` is ``Pre_model.infer`` without dropout.

The loss of a row is the mean over all ``C x T`` elements of the PADDED row, as in the reference (past a row's length the target
is 0 and the prediction is whatever the network emits there).  Inputs must be finite: the length mask is a 0/1 factor, as in the
reference, so a non-finite value past a length turns the row into NaN.

``utterance_losses`` is the per-utterance reading: each utterance's loss is what ``forward`` returns for that utterance alone as an
unpadded B = 1 batch, whatever batch it is evaluated in.  It runs ragged batches (the ragged encoders, the ragged denoiser program
and a reduction over each row's own length), on one GPU or over the ranks of a process group.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

from . import _lib, coefs, shard
from .api import batch_plan, pad_batch, sequence_mask
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


def mse_rows_ragged(out: torch.Tensor, target: torch.Tensor, lengths, t: torch.Tensor, timesteps: int = 1000,
                    min_snr_gamma: Optional[float] = None, ws: Optional[torch.Tensor] = None):
    """The per-utterance reduction of a ragged batch: out [K, B, C, T], target [B, C, T] or [K, B, C, T] and t [K, B] int64 on one
    CUDA device, ``lengths`` B host ints (or a tensor) in [1, T] -> (loss_row [K, B], loss_weighted [K, B]): the mean of
    (out - target)^2 over row b's own C x T_b elements and that times ``loss_weight[t]``.  Nothing past a length is read, and a row's
    bits depend on (C, T_b) only (see ``ns2vc_mse_rows_ragged``).  ``ws``: scratch to reuse (uint8, 8-byte aligned)."""
    if out.dim() != 4:
        raise ValueError(f"out must be [K, B, C, T], got {tuple(out.shape)}")
    K, B, Cl, T = out.shape
    if tuple(target.shape) not in ((B, Cl, T), (K, B, Cl, T)):
        raise ValueError(f"target must be [{B}, {Cl}, {T}] or [{K}, {B}, {Cl}, {T}], got {tuple(target.shape)}")
    if not torch.is_tensor(t) or t.dtype != torch.int64 or tuple(t.shape) != (K, B):
        raise ValueError(f"t must be an int64 tensor [{K}, {B}]")
    lens = check_lengths(lengths, B, T, "lengths")
    for name, v in (("out", out), ("target", target), ("t", t)):
        if not v.is_cuda or not v.is_contiguous():
            raise ValueError(f"{name} must be a contiguous CUDA tensor (no CPU path)")
    if out.dtype != torch.float32 or target.dtype != torch.float32 or target.device != out.device or t.device != out.device:
        raise ValueError("out and target must be fp32, and out, target and t on one device")
    dev = out.device
    L = _lib.lib()
    need = C.c_size_t()
    _lib.check(L.ns2vc_mse_ragged_workspace_bytes(K, B, Cl, T, C.byref(need)))
    if ws is None:
        ws = torch.empty(need.value, dtype=torch.uint8, device=dev)
    elif ws.numel() < need.value:
        raise ValueError(f"workspace of {ws.numel()} bytes, {need.value} needed")
    len_d = torch.tensor(lens, dtype=torch.int64).to(dev, non_blocking=True)
    loss_row = torch.empty((K, B), dtype=torch.float32, device=dev)
    loss_weighted = torch.empty((K, B), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(L.ns2vc_mse_rows_ragged(out.data_ptr(), target.data_ptr(), int(target.dim() == 4), len_d.data_ptr(), t.data_ptr(),
                                           _loss_buffers(timesteps, dev)["loss_weight"].data_ptr(), timesteps,
                                           float(min_snr_gamma) if min_snr_gamma is not None else 0.0, loss_row.data_ptr(),
                                           loss_weighted.data_ptr(), K, B, Cl, T, ws.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
    return loss_row, loss_weighted


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


# ------------------------------------------------------------------------------------------------ per-utterance (ragged) objective
HOP = 256                # mel hop of 24 kHz audio: the cost rows of shard.plan_batches count 24 kHz samples (convert.frame_plan)


@dataclass
class UtteranceLosses:
    """``loss``: each utterance's ``loss_weight[t] * mse``, [N] (or [K, N] for a ``t_grid`` of K timesteps); ``mse``: the
    unweighted mean over the utterance's own 100 x T_i elements, same shape; ``t``: the timesteps, same shape, int64.  On the
    models' device, in input order."""
    loss: torch.Tensor
    mse: torch.Tensor
    t: torch.Tensor


@torch.no_grad()
def batch_utterance_losses(pre_model, unet: UNet1DConditionModel, c_padded: torch.Tensor, refer_padded: torch.Tensor,
                           spec_padded: torch.Tensor, lengths, refer_lengths, t: torch.Tensor, noise: torch.Tensor,
                           timesteps: int = 1000, min_snr_gamma: Optional[float] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """One ragged batch: c_padded [B, 256, T], refer_padded [B, 100, S], spec_padded [B, 100, T] fp32, t [K, B] int64 and noise
    [B, 100, T] (shared by every k) or [K, B, 100, T], all on the models' device; lengths / refer_lengths: B host ints.  Returns
    (mse [K, B], loss [K, B]); row b is utterance b's objective alone, and values past its lengths are never read.

    ``Pre_model.infer(per_utterance=True)`` -> ``q_sample`` (masked by ``lengths``) -> the ragged session's
    ``eval_x_start_ragged`` -> ``mse_rows_ragged``."""
    dev = spec_padded.device
    B, _, T = spec_padded.shape
    S = refer_padded.shape[2]
    tl = torch.tensor(check_lengths(lengths, B, T, "lengths"), dtype=torch.int64)
    sl = torch.tensor(check_lengths(refer_lengths, B, S, "refer_lengths"), dtype=torch.int64)
    content, prompt = pre_model.infer((c_padded, refer_padded, None, None, None, tl, sl, None), per_utterance=True)
    x_start, x = q_sample(spec_padded, noise, tl.to(dev, non_blocking=True), t, timesteps)
    sess = get_session(unet, content.permute(1, 2, 0), prompt.permute(1, 0, 2), None, content_lengths=tl, prompt_lengths=sl)
    model_out = sess.eval_x_start_ragged(x, t, torch.empty_like(x))
    mse, loss = mse_rows_ragged(model_out, x_start, tl, t, timesteps, min_snr_gamma)
    return mse, loss


def _check_items(unet, items, t, t_grid, noise, max_batch, timesteps, min_snr_gamma) -> Tuple[List[int], List[int], Optional[List[int]]]:
    """Host-side argument checks of ``utterance_losses``; returns (T_i, S_i, the grid or None)."""
    if len(items) == 0:
        raise ValueError("items is empty")
    Cl = unet.latent_channels
    if unet.cfg.out_channels != Cl:
        raise ValueError("the x_start objective needs a denoiser with out_channels equal to its latent channels")
    tl, sl = [], []
    for i, it in enumerate(items):
        if not isinstance(it, (tuple, list)) or len(it) != 3 or not all(torch.is_tensor(v) for v in it):
            raise ValueError(f"utterance {i}: expected a (c [C, T_i], spec [{Cl}, T_i], refer [C, S_i]) tuple of tensors")
        c, spec, refer = it
        if spec.dim() != 2 or spec.shape[0] != Cl or c.dim() != 2 or c.shape[1] != spec.shape[1] or refer.dim() != 2:
            raise ValueError(f"utterance {i}: expected c [C, T_i], spec [{Cl}, T_i] and refer [C, S_i], got {tuple(c.shape)}, "
                             f"{tuple(spec.shape)}, {tuple(refer.shape)}")
        if spec.shape[1] < 1 or refer.shape[1] < 1:
            raise ValueError(f"utterance {i}: T_i = {spec.shape[1]} and S_i = {refer.shape[1]} must be >= 1")
        if c.shape[0] != items[0][0].shape[0] or refer.shape[0] != items[0][2].shape[0]:
            raise ValueError(f"utterance {i}: channel counts differ from utterance 0's")
        tl.append(int(spec.shape[1]))
        sl.append(int(refer.shape[1]))
    N = len(items)
    if int(max_batch) < 1:
        raise ValueError("max_batch must be >= 1")
    if int(timesteps) < 1:
        raise ValueError("timesteps must be >= 1")
    if min_snr_gamma is not None and not float(min_snr_gamma) > 0:
        raise ValueError("min_snr_gamma must be positive")
    if t is not None and t_grid is not None:
        raise ValueError("pass t (one timestep per utterance) or t_grid (the same K timesteps for every utterance), not both")
    if t is not None:
        if not torch.is_tensor(t) or t.dtype != torch.int64 or tuple(t.shape) != (N,):
            raise ValueError(f"t must be an int64 tensor [{N}]")
        if int(t.min()) < 0 or int(t.max()) >= timesteps:
            raise ValueError(f"t must lie in [0, {timesteps})")
    grid = None
    if t_grid is not None:
        grid = [int(v) for v in t_grid]
        if not grid:
            raise ValueError("t_grid is empty")
        if min(grid) < 0 or max(grid) >= timesteps:
            raise ValueError(f"t_grid must lie in [0, {timesteps})")
        if len(grid) * min(int(max_batch), N) > 65535:
            raise ValueError(f"t_grid of {len(grid)} points times max_batch rows exceeds 65535 evaluations per batch")
    if noise is not None:
        if len(noise) != N:
            raise ValueError(f"{len(noise)} noise tensors for {N} utterances")
        for i, (nz, T) in enumerate(zip(noise, tl)):
            if not torch.is_tensor(nz) or tuple(nz.shape) != (Cl, T):
                raise ValueError(f"noise {i}: expected [{Cl}, {T}], got {tuple(nz.shape) if torch.is_tensor(nz) else nz!r}")
    return tl, sl, grid


@torch.no_grad()
def utterance_losses(pre_model, unet: UNet1DConditionModel, items: Sequence[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]],
                     t: Optional[torch.Tensor] = None, t_grid=None, noise: Optional[Sequence[torch.Tensor]] = None, max_batch: int = 8,
                     group: Optional[dist.ProcessGroup] = None, timesteps: int = 1000,
                     min_snr_gamma: Optional[float] = None) -> UtteranceLosses:
    """Each utterance's own training objective: for ``items[i] = (c [256, T_i], spec [100, T_i], refer [100, S_i])`` the number
    ``NaturalSpeech2.forward`` (reference model.py:706-734) returns for the unpadded B = 1 batch ``(c[None], refer[None], ...,
    spec[None], lengths=[T_i], refer_lengths=[S_i])``: ``loss_weight[t] * mean((model_out - spec)^2)`` over its 100 x T_i
    elements.  Unlike ``diffusion_loss`` on a padded batch, the value does not depend on the batch the utterance is evaluated in,
    so it compares checkpoints on a held-out set, profiles the schedule per utterance, or ranks a corpus by fit.

    ``t``: int64 [N], one timestep per utterance; ``t_grid``: K timesteps evaluated for every utterance with one noise tensor per
    utterance shared by the grid (results [K, N]); neither: one drawn timestep each.  ``noise``: one [100, T_i] per utterance, or
    None.  Default draws, per utterance in input order on the device's default generator: ``torch.randint(0, timesteps, (1,))``
    when ``t`` and ``t_grid`` are None, then ``torch.randn_like(spec_i[None])`` when ``noise`` is None - the draws of the loop
    ``for i: diffusion_loss(pre_model, unet, unpadded_batch_i)``, so after the same ``torch.manual_seed`` both give the same
    values and leave the generator in the same state, whatever ``max_batch`` and ``group``.

    The utterances run in ragged batches of at most ``max_batch`` (``api.batch_plan``, longest first): ``batch_utterance_losses``.
    With a process ``group`` of more than one rank (one process per GPU, every rank making the same call with its models on its
    own device), the batches are shared out by ``shard.plan_batches``, run by ``shard.run_sharded`` and all-gathered once; every
    rank draws the defaults for all utterances, so every rank returns the one-GPU result and ends with the same generator state."""
    tl, sl, grid = _check_items(unet, items, t, t_grid, noise, max_batch, timesteps, min_snr_gamma)
    dev = next(unet.parameters()).device
    if dev.type != "cuda":
        raise RuntimeError("utterance_losses needs the models on a CUDA device (no CPU path)")
    N, Cl = len(items), unet.latent_channels
    sharded = group is not None and dist.get_world_size(group) > 1
    if sharded and (t is None and grid is None or noise is None):
        shard.check_generator(torch.cuda.default_generators[dev.index], group, dev)
    # the default draws, utterance by utterance in input order (every rank draws all of them)
    t_u = [None] * N if t is None else list(t.to(dev))
    noise_u = [None] * N if noise is None else list(noise)
    for i in range(N):
        if t is None and grid is None:
            t_u[i] = torch.randint(0, timesteps, (1,), device=dev).long()[0]
        if noise is None:
            noise_u[i] = torch.randn((1, Cl, tl[i]), device=dev)[0]
    if grid is not None:
        t_all = torch.tensor(grid, dtype=torch.int64, device=dev)[:, None].expand(len(grid), N).contiguous()
    else:
        t_all = torch.stack(t_u)[None].contiguous()
    K = t_all.shape[0]

    def work(idx: List[int]) -> List[torch.Tensor]:
        spec, c, refer, _, _ = pad_batch([(items[i][1], items[i][0].t(), items[i][2].t()) for i in idx], range(len(idx)))
        f32 = lambda v: v.to(dev, torch.float32, non_blocking=True).contiguous()
        nz = torch.zeros((len(idx), Cl, max(tl[i] for i in idx)), dtype=torch.float32, device=dev)
        for j, i in enumerate(idx):
            nz[j, :, :tl[i]] = noise_u[i]
        mse, loss = batch_utterance_losses(pre_model, unet, f32(c.permute(1, 2, 0)), f32(refer.permute(1, 2, 0)), f32(spec),
                                           [tl[i] for i in idx], [sl[i] for i in idx], t_all[:, idx].contiguous(), nz, timesteps,
                                           min_snr_gamma)
        both = torch.stack([mse, loss])                                      # [2, K, B]
        return [both[:, :, j] for j in range(len(idx))]

    if sharded:
        world = dist.get_world_size(group)
        plan = shard.plan_batches([dict(n24=T * HOP, T=T) for T in tl], sl, world, int(max_batch))
        rows = shard.run_sharded(work, plan, [(2, K)] * N, group, dev)
    else:
        rows: List[Optional[torch.Tensor]] = [None] * N
        for idx in batch_plan(tl, int(max_batch)):
            for i, r in zip(idx, work(idx)):
                rows[i] = r
    both = torch.stack([r.to(dev) for r in rows], dim=-1)                   # [2, K, N]
    if grid is None:
        return UtteranceLosses(loss=both[1, 0], mse=both[0, 0], t=t_all[0])
    return UtteranceLosses(loss=both[1], mse=both[0], t=t_all)
