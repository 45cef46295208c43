"""Public convenience API: host tensors in, sampled latents out (what bench.py's ``e2e`` leg times), and latents to waveforms.

``sample_latents`` is the batched equivalent of the sampling block of ``NaturalSpeech2.sample``
(reference model.py:620-686) after ``pre_model.infer``: it takes the condition tensors in the
reference's own layouts (content [T,B,C], prompt [S,B,C], lengths) and returns the mel latents
[B,100,T].  Inputs may live on the host (pinned memory recommended); they are copied to the device,
sampled with the fused loop, and the result is returned on the requested device.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import torch

from .fused import check_lengths, get_session
from .noise import check_seeds
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
                   noise: Optional[torch.Tensor] = None, content_lengths: Optional[torch.Tensor] = None,
                   noise_seeds: Optional[Sequence[int]] = None) -> torch.Tensor:
    """``method``: ``"dpmsolver"`` / ``"unipc"`` (``steps`` solver steps, default 50), ``"ddim"`` (``steps`` = the reference's
    ``sampling_timesteps``, default 100 as in ``sample()``; ``eta`` = ``ddim_sampling_eta``) or ``"ddpm"`` (``p_sample_loop``: every
    timestep 999 .. 0; ``steps`` may be left unset or be 1000).  DDPM / DDIM draw their noise with ``torch.randn_like`` on the
    device's default generator, in the reference's order, unless ``noise`` [N, B, 100, T] (one tensor per step) is given, or
    ``noise_seeds`` (one int in [0, 2**63) per utterance): row b's noise is then drawn on the GPU from its own seed
    (``ns2vc_b200.noise``), the same bits whatever batch the utterance runs in.

    ``content_lengths`` [B] (opt-in): sample a ragged batch.  Row b of the result is then utterance b sampled alone on
    x_T[b, :, :T_b], content[:T_b, b], prompt[:S_b, b] with S_b = ``prompt_lengths[b]`` (S when None), and its frames >= T_b
    are 0; values past the lengths are never read.  Without it the batch keeps the reference's padded semantics, in which
    ``prompt_lengths`` is the cross-attention mask and every row sees the whole padded T.  See ``DenoiserSession`` for the
    DDPM / DDIM noise of a ragged batch."""
    if content_lengths is not None:
        content_lengths = check_lengths(content_lengths, x_T.shape[0], x_T.shape[2], "content_lengths")
        if prompt_lengths is not None:
            prompt_lengths = check_lengths(prompt_lengths, x_T.shape[0], prompt_SBC.shape[0], "prompt_lengths")
    if method not in ("dpmsolver", "unipc", "ddpm", "ddim"):
        raise ValueError(f"unknown method {method!r} (dpmsolver | unipc | ddpm | ddim)")
    if method in ("ddpm", "ddim"):
        if noise_schedule is not None:
            raise ValueError(f"method {method!r} uses NaturalSpeech2's own schedule buffers; noise_schedule applies to dpmsolver / unipc")
        if method == "ddpm" and steps not in (None, 1000):
            raise ValueError("method 'ddpm' runs every one of the 1000 timesteps (p_sample_loop); use 'ddim' for fewer steps")
        if noise_seeds is not None:
            if noise is not None:
                raise ValueError("noise and noise_seeds are mutually exclusive")
            if not 0.0 <= eta <= 1.0:
                raise ValueError(f"eta must lie in [0, 1], got {eta}")
            noise_seeds = check_seeds(noise_seeds, x_T.shape[0], "noise_seeds")
    elif noise is not None or eta != 0.0 or noise_seeds is not None:
        raise ValueError("eta, noise and noise_seeds apply to the ddpm / ddim methods")
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
    if content_lengths is not None:
        sess = get_session(unet, content, prompt, None, content_lengths=content_lengths, prompt_lengths=prompt_lengths)
    else:
        if prompt_lengths is not None:
            mask = sequence_mask(prompt_lengths.to(dev, non_blocking=nb), prompt_SBC.shape[0])
        sess = get_session(unet, content, prompt, mask)
    if method == "ddpm":
        out = sess.sample_ddpm(x, noise=noise, seeds=noise_seeds)
        return out.to(out_device) if out_device is not None else out
    if method == "ddim":
        out = sess.sample_ddim(x, steps, eta=eta, noise=noise, seeds=noise_seeds)
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
                         noise: Optional[torch.Tensor] = None, per_utterance: bool = False) -> torch.Tensor:
    """The device part of ``NaturalSpeech2.sample`` before the vocoder (reference model.py:606-686): ``pre_model.infer`` (condition
    encoders) followed by the sampling run.  c_padded [B, 256, T] (ContentVec features), refer_padded [B, 100, S] (mel prompt),
    lengths / refer_lengths [B]; host tensors are copied to the device.  Returns the mel latents [B, 100, T].  ``steps``, ``method``,
    ``eta`` and ``noise`` as for ``sample_latents``.  ``per_utterance=True`` samples the encoders' output as ragged utterances
    (``sample_latents(content_lengths=lengths, prompt_lengths=refer_lengths)``): row b of the sampling equals ``sample_latents`` on
    row b of ``pre_model.infer``'s output alone.  The encoders themselves run on the padded batch as the reference runs them,
    so their row b need not equal utterance b encoded alone; for that, encode with ``pre_model.infer(data, per_utterance=True)``
    and sample with ``sample_latents(content_lengths=...)`` (or convert whole waveforms with ``convert_utterances``).
    The default keeps the padded semantics."""
    dev = torch.device(device) if device is not None else next(unet.parameters()).device
    data = (c_padded.to(dev, torch.float32, non_blocking=True), refer_padded.to(dev, torch.float32, non_blocking=True), None, None, None,
            lengths.to(dev, non_blocking=True), refer_lengths.to(dev, non_blocking=True), None)
    content, prompt = pre_model.infer(data)
    return sample_latents(unet, x_T, content, prompt, data[6], steps=steps, method=method, device=dev, out_device=out_device, eta=eta,
                          noise=noise, content_lengths=lengths if per_utterance else None)


Utterance = Tuple[torch.Tensor, torch.Tensor, torch.Tensor]


def batch_plan(lengths: Sequence[int], max_batch: int) -> List[List[int]]:
    """Indices of the utterances grouped into batches of at most ``max_batch``, longest first (so each batch pads to a
    length close to its rows').  Ties keep the input order."""
    if max_batch < 1:
        raise ValueError("max_batch must be >= 1")
    order = sorted(range(len(lengths)), key=lambda i: -int(lengths[i]))
    return [order[i:i + max_batch] for i in range(0, len(order), max_batch)]


def pad_batch(items: Sequence[Utterance], idx: Sequence[int]):
    """Pads utterances ``items[i]`` (x_T [Cl, T_b], content [T_b, Cc], prompt [S_b, D]) for i in ``idx`` into one ragged batch:
    x_T [B, Cl, T], content [T, B, Cc], prompt [S, B, D] (zeros past each length), content lengths [B], prompt lengths [B]."""
    xs, cs, ps = [items[i][0] for i in idx], [items[i][1] for i in idx], [items[i][2] for i in idx]
    tl = torch.tensor([x.shape[-1] for x in xs], dtype=torch.int64)
    sl = torch.tensor([p.shape[0] for p in ps], dtype=torch.int64)
    T, S, B = int(tl.max()), int(sl.max()), len(idx)
    x = xs[0].new_zeros((B, xs[0].shape[0], T))
    c = cs[0].new_zeros((T, B, cs[0].shape[1]))
    p = ps[0].new_zeros((S, B, ps[0].shape[1]))
    for j in range(B):
        x[j, :, :xs[j].shape[-1]] = xs[j]
        c[:cs[j].shape[0], j] = cs[j]
        p[:ps[j].shape[0], j] = ps[j]
    return x, c, p, tl, sl


@torch.no_grad()
def sample_utterances(unet: UNet1DConditionModel, items: Sequence[Utterance], steps: Optional[int] = None, method: str = "dpmsolver",
                      max_batch: int = 8, device: Optional[torch.device] = None, out_device: Optional[torch.device] = None,
                      noise_schedule: Optional[NoiseScheduleVP] = None, eta: float = 0.0,
                      noise_seeds: Optional[Sequence[int]] = None) -> List[torch.Tensor]:
    """Samples a list of utterances of different lengths, ``(x_T [100, T_b], content [T_b, C], prompt [S_b, C])`` each, in
    ragged batches of at most ``max_batch`` (longest first) and returns their latents [100, T_b] in input order.  Each result
    equals ``sample_latents`` on that utterance alone.  DDPM / DDIM with ``noise_seeds`` (one per utterance): equal bit for bit
    to ``sample_latents(noise_seeds=[seed])`` on that utterance alone; without seeds their noise comes from the default
    generator, drawn over each padded batch, so a result then depends on the batch it ran in.
    The slices of one file (the reference CLI's ``infer.py`` loop) go in as one call."""
    for k, (x, c, p) in enumerate(items):
        if x.dim() != 2 or c.dim() != 2 or p.dim() != 2 or x.shape[1] != c.shape[0]:
            raise ValueError(f"utterance {k}: expected x_T [C, T_b], content [T_b, C] and prompt [S_b, C], got "
                             f"{tuple(x.shape)}, {tuple(c.shape)}, {tuple(p.shape)}")
        if x.shape[1] < 1 or p.shape[0] < 1:
            raise ValueError(f"utterance {k}: empty content or prompt")
    if noise_seeds is not None:
        noise_seeds = check_seeds(noise_seeds, len(items), "noise_seeds")
    out: List[Optional[torch.Tensor]] = [None] * len(items)
    for idx in batch_plan([x.shape[1] for x, _, _ in items], max_batch):
        x, c, p, tl, sl = pad_batch(items, idx)
        lat = sample_latents(unet, x, c, p, sl, steps=steps, method=method, device=device, out_device=out_device,
                             noise_schedule=noise_schedule, eta=eta, content_lengths=tl,
                             noise_seeds=[noise_seeds[i] for i in idx] if noise_seeds is not None else None)
        for j, i in enumerate(idx):
            out[i] = lat[j, :, :int(tl[j])]
    return out


@torch.no_grad()
def decode_utterances(vocoder, latents: Sequence[torch.Tensor], max_batch: int = 8) -> List[torch.Tensor]:
    """Decodes a list of mel latents [C, T_b] of different lengths (what ``sample_utterances`` returns) with a
    ``vocoder.Vocos`` in ragged batches of at most ``max_batch`` (longest first) and returns the waveforms [T_b * hop_length]
    in input order.  Each equals ``vocoder.decode`` of that latent alone."""
    C = vocoder.cfg["input_channels"]
    for k, x in enumerate(latents):
        if x.dim() != 2 or x.shape[0] != C or x.shape[1] < 1:
            raise ValueError(f"latent {k}: expected [{C}, T_b] with T_b >= 1, got {tuple(x.shape)}")
    dev = next(vocoder.parameters()).device
    hop = vocoder.hop_length
    out: List[Optional[torch.Tensor]] = [None] * len(latents)
    for idx in batch_plan([x.shape[1] for x in latents], max_batch):
        tl = [int(latents[i].shape[1]) for i in idx]
        mel = torch.zeros((len(idx), C, max(tl)), dtype=torch.float32, device=dev)
        for j, i in enumerate(idx):
            mel[j, :, :tl[j]] = latents[i]
        audio = vocoder.decode(mel, torch.tensor(tl, dtype=torch.int64))
        for j, i in enumerate(idx):
            out[i] = audio[j, :tl[j] * hop]
    return out


@torch.no_grad()
def encode_voices(pre_model, mels: Sequence[torch.Tensor], max_batch: int = 8) -> list:
    """Encodes target voices once for reuse: each prompt mel [100, S_v] of ``mels`` goes through ``pre_model.encode_voices`` in
    ragged batches of at most ``max_batch`` (longest first), and one ``pre_model.Voice`` per mel is returned in input order.
    The conversion entry points take a ``Voice`` wherever they take a prompt mel, and skip the voice's encoders."""
    from .pre_model import REF_DIM
    for k, m in enumerate(mels):
        if not isinstance(m, torch.Tensor) or m.dim() != 2 or m.shape[0] != REF_DIM or m.shape[1] < 1:
            raise ValueError(f"mel {k}: expected a mel [{REF_DIM}, S_v] with S_v >= 1, got {tuple(getattr(m, 'shape', ()))}")
    dev = next(pre_model.parameters()).device
    out: list = [None] * len(mels)
    for idx in batch_plan([int(m.shape[1]) for m in mels], max_batch):
        sl = [int(mels[i].shape[1]) for i in idx]
        refer = torch.zeros((len(idx), REF_DIM, max(sl)), dtype=torch.float32, device=dev)
        for j, i in enumerate(idx):
            refer[j, :, :sl[j]] = mels[i]
        for i, v in zip(idx, pre_model.encode_voices(refer, torch.tensor(sl, dtype=torch.int64))):
            out[i] = v
    return out


def content_utterances(model, wavs16k: Sequence[torch.Tensor], target_frames: Optional[Sequence[int]] = None,
                       max_batch: int = 8) -> List[torch.Tensor]:
    """Content units of a list of 1-D 16 kHz waveforms of different lengths with a ``content.ContentVec``, in ragged batches of
    at most ``max_batch`` (longest first).  Returns [final_dim, T_b] per waveform in input order (each equals
    ``get_hubert_content`` of that waveform alone), or, with ``target_frames``, [final_dim, target_frames[b]] through
    ``frontend.repeat_expand_2d``: the ``c`` that ``Svc.get_unit_f0_code`` builds (its target is the f0 length, N24 // 256)."""
    from .content import MIN_SAMPLES
    from .frontend import repeat_expand_2d
    for k, w in enumerate(wavs16k):
        if w.dim() != 1 or w.shape[0] < MIN_SAMPLES:
            raise ValueError(f"waveform {k}: expected a 1-D tensor of at least {MIN_SAMPLES} samples, got {tuple(w.shape)}")
    if target_frames is not None and len(target_frames) != len(wavs16k):
        raise ValueError(f"target_frames has {len(target_frames)} entries for {len(wavs16k)} waveforms")
    dev = next(model.parameters()).device
    out: List[Optional[torch.Tensor]] = [None] * len(wavs16k)
    for idx in batch_plan([int(w.shape[0]) for w in wavs16k], max_batch):
        nl = [int(wavs16k[i].shape[0]) for i in idx]
        wav = torch.zeros((len(idx), max(nl)), dtype=torch.float32, device=dev)
        for j, i in enumerate(idx):
            wav[j, :nl[j]] = wavs16k[i]
        with torch.no_grad():
            units, frames = model.extract(wav, torch.tensor(nl, dtype=torch.int64))
        fl = frames.tolist()
        for j, i in enumerate(idx):
            c = units[j, :fl[j]].t()
            out[i] = c if target_frames is None else repeat_expand_2d(c, int(target_frames[i]))
    return out


def __getattr__(name):
    # waveform-to-waveform conversion lives in convert.py, live conversion in stream.py and serving in serve.py; they build on this module
    if name in ("convert_utterances", "convert_slices", "convert_files"):
        from . import convert
        return getattr(convert, name)
    if name in ("diffusion_loss", "loss_profile", "utterance_losses"):     # the training objective under no_grad lives in loss.py
        from . import loss
        return getattr(loss, name)
    if name in ("preprocess_utterances", "dataset_item"):   # a corpus to the reference's training files lives in preprocess.py
        from . import preprocess
        return getattr(preprocess, name)
    if name == "StreamConverter":
        from . import stream
        return stream.StreamConverter
    if name == "ConversionServer":                          # requests served as they arrive (continuous batching)
        from . import serve
        return serve.ConversionServer
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
