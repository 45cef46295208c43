"""Drop-in ``NaturalSpeech2.p_sample_loop`` / ``ddim_sample`` (reference model.py:544-603) that take the fused DDPM / DDIM loops
(``ns2vc_b200.install_diffusion()`` puts them on the reference's class).

Each runs ``self.pre_model.infer`` and draws ``img`` as the reference does, then evaluates the first step through the object's
own ``model_predictions`` while recording the denoiser calls.  If that was exactly one call of our UNet on ``cat([img, content])``
at the step's timestep, with its output returned unchanged as x_start, and the object's schedule buffers are the ones the
fused path computes, the rest of the run is ``DenoiserSession.sample_ddpm`` / ``sample_ddim`` (the first output is reused, so
no extra denoiser call).  Otherwise the reference's own loop continues from step 1.  ``NS2VC_B200_FUSED=0`` forces that loop.
"""
from __future__ import annotations

import torch

from . import coefs
from .fused import _diffusion_buffers, _fast_path_enabled, _session_from_record
from .unet import UNet1DConditionModel, trace_calls

_BUFFER_NAMES = ("alphas_cumprod", "sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod", "posterior_mean_coef1",
                 "posterior_mean_coef2", "posterior_log_variance_clipped")


def _buffers_match(model) -> bool:
    """The fused loops use NaturalSpeech2's buffers for 1000 linear-beta timesteps (coefs.diffusion_buffers)."""
    if getattr(model, "num_timesteps", None) != 1000:
        return False
    ours = _diffusion_buffers(1000)
    for name in _BUFFER_NAMES:
        b = getattr(model, name, None)
        if not torch.is_tensor(b) or b.dtype != torch.float32 or not torch.equal(b.detach().cpu(), ours[name]):
            return False
    return True


def _loss_gamma(model):
    """(True, gamma) when the model's ``q_sample`` / ``loss_weight`` buffers are the ones ``coefs.loss_buffers`` computes; gamma is
    the clamp its ``loss_weight`` was built with (``min_snr_loss_weight=True``) or None.  A clamped weight table's maximum is
    the clamp itself: the SNR at t = 0 is ~1e4."""
    lw = getattr(model, "loss_weight", None)
    if not torch.is_tensor(lw) or lw.dtype != torch.float32 or lw.shape != (1000,):
        return False, None
    plain = coefs.loss_buffers(1000)
    gamma = None if torch.equal(lw.detach().cpu(), plain["loss_weight"]) else float(lw.max())
    ours = plain if gamma is None else coefs.loss_buffers(1000, gamma)
    for name, v in ours.items():
        b = getattr(model, name, None)
        if not torch.is_tensor(b) or b.dtype != torch.float32 or not torch.equal(b.detach().cpu(), v):
            return False, None
    return True, gamma


def validation_loss(self, data, t=None, noise=None):
    """``NaturalSpeech2.forward(data, vocos)`` (reference model.py:706-734) under ``no_grad`` through ``loss.diffusion_loss``: the
    same 7-tuple ``(loss, loss_diff, 0, 0, 0, model_out, target)``, with ``t`` / ``noise`` drawn as ``forward`` draws them unless
    given ([K, B] ``t`` gives [K] losses).  ``forward`` itself is untouched: training keeps the reference's modules.  Raises when
    the object's modules or schedule buffers are not the ones the device path computes with."""
    from .loss import diffusion_loss
    from .pre_model import Pre_model
    unet = getattr(self.diff_model, "unet", None)
    if not isinstance(self.pre_model, Pre_model) or not isinstance(unet, UNet1DConditionModel):
        raise TypeError("validation_loss needs ns2vc_b200's Pre_model and UNet1DConditionModel in the model (install() and "
                        "install_pre_model() before it is constructed)")
    ok, gamma = _loss_gamma(self)
    if not (ok and _buffers_match(self)):
        raise ValueError("validation_loss supports NaturalSpeech2's 1000-step linear-beta schedule buffers; this model's differ")
    r = diffusion_loss(self.pre_model, unet, data, t=t, noise=noise, timesteps=1000, min_snr_gamma=gamma)
    return r.loss, r.loss, 0, 0, 0, r.model_out, r.target


def _our_call(recs, x: torch.Tensor, x_start: torch.Tensor, time: int):
    """The call record if the first model_predictions was one call of our UNet on cat([x, content]) at ``time`` whose output is
    x_start itself, else None (same test as fused._trace_first_call, for the reference's x_start parameterisation)."""
    if len(recs) != 1 or not x.is_cuda or x.dtype != torch.float32 or x.dim() != 3:
        return None
    r = recs[0]
    u = r.unet
    if not isinstance(u, UNet1DConditionModel):
        return None
    Cl = u.latent_channels
    if u.cfg.out_channels != Cl or x.shape[1] != Cl or r.sample.shape[1] != u.cfg.in_channels or tuple(r.sample.shape[::2]) != tuple(x.shape[::2]):
        return None
    if not torch.equal(r.sample[:, :Cl], x) or not torch.equal(r.timesteps, torch.full_like(r.timesteps, float(time))):
        return None
    if not torch.is_tensor(x_start) or x_start.shape != r.output.shape or not torch.equal(x_start, r.output):
        return None
    return r


def _first_step(model, img, time, cond):
    bt = torch.full((img.shape[0],), time, device=img.device, dtype=torch.long)
    with trace_calls() as recs:
        preds = model.model_predictions(img, bt, cond)
    rec = None
    if _fast_path_enabled():
        rec = _our_call(recs, img, preds.pred_x_start, time)
        if rec is not None and not _buffers_match(model):
            rec = None
    return bt, preds, rec


@torch.no_grad()
def p_sample_loop(self, content, refer, lengths, refer_lengths, f0, uv, auto_predict_f0=True):
    """Reference model.py:544-561 (no progress bar)."""
    data = (content, refer, f0, 0, 0, lengths, refer_lengths, uv)
    content, refer = self.pre_model.infer(data)
    shape = (content.shape[1], self.dim, content.shape[0])
    img = torch.randn(shape, device=refer.device)
    cond = (content, refer, lengths, refer_lengths)
    ts = list(reversed(range(0, self.num_timesteps)))
    bt, preds, rec = _first_step(self, img, ts[0], cond)
    if rec is not None:
        return _session_from_record(rec).sample_ddpm(img, ts, first_out=rec.output)
    # the reference's p_sample (:535-542) for the step already evaluated, then its loop
    model_mean, _, model_log_variance = self.q_posterior(x_start=preds.pred_x_start, x_t=img, t=bt)
    noise = torch.randn_like(img) if ts[0] > 0 else 0.
    img = model_mean + (0.5 * model_log_variance).exp() * noise
    for t in ts[1:]:
        img, _ = self.p_sample(img, t, cond)
    return img


@torch.no_grad()
def ddim_sample(self, content, refer, lengths, refer_lengths, f0, uv, auto_predict_f0=True):
    """Reference model.py:563-603 (no progress bar)."""
    data = (content, refer, f0, 0, 0, lengths, refer_lengths, uv)
    content, refer = self.pre_model.infer(data, auto_predict_f0=auto_predict_f0)
    shape = (content.shape[1], self.dim, content.shape[0])
    batch, device, total_timesteps, sampling_timesteps, eta = shape[0], refer.device, self.num_timesteps, self.sampling_timesteps, self.ddim_sampling_eta
    time_pairs = coefs.ddim_time_pairs(total_timesteps, sampling_timesteps)
    img = torch.randn(shape, device=device)
    cond = (content, refer, lengths, refer_lengths)
    _bt, preds, rec = _first_step(self, img, time_pairs[0][0], cond)
    if rec is not None:
        return _session_from_record(rec).sample_ddim(img, sampling_timesteps, eta=eta, first_out=rec.output)
    for k, (time, time_next) in enumerate(time_pairs):
        if k > 0:
            time_cond = torch.full((batch,), time, device=device, dtype=torch.long)
            preds = self.model_predictions(img, time_cond, cond)
        pred_noise, x_start = preds.pred_noise, preds.pred_x_start
        if time_next < 0:
            img = x_start
            continue
        alpha = self.alphas_cumprod[time]
        alpha_next = self.alphas_cumprod[time_next]
        sigma = eta * ((1 - alpha / alpha_next) * (1 - alpha_next) / (1 - alpha)).sqrt()
        c = (1 - alpha_next - sigma ** 2).sqrt()
        noise = torch.randn_like(img)
        img = x_start * alpha_next.sqrt() + c * pred_noise + sigma * noise
    return img
