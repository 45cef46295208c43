"""Waveform-to-waveform conversion of a file's voice slices in ragged batches: the device part of ``Svc.infer``
(reference ``inference/infer_tool.py:141-206``) and the slicing loop of the CLI (``infer.py:99-141``) around it.

Per utterance the chain is ``Svc.get_unit_f0_code`` + ``NaturalSpeech2.sample``:

1. resample the input to 24 kHz (``frontend.resample``): N24 samples;
2. T = N24 // 256, the frame count of ``compute_f0_parselmouth`` (``utils.py:159-160``).  f0 itself is not read by the model
   (``model.py:349-375``) and the transposition only scales f0, so neither enters here;
3. resample 24 -> 16 kHz, ContentVec units (``content.ContentVec.extract``), stretched to T frames (``repeat_expand_2d``);
4. the condition encoders (``Pre_model.infer(per_utterance=True)``), as its two halves: the prompt mel's ``Pre_model.encode_voices``
   and the units' ``Pre_model.infer_content``, so that a prompt given as an encoded ``Voice`` is not encoded again;
5. UniPC (30 steps, what ``Svc.infer`` runs) or DPM-Solver++ (40 steps) from x_T ~ N(0, 1) [1, 100, T];
6. the vocoder (``Vocos.decode``): T * 256 samples at 24 kHz.

Every stage runs on a ragged batch in which row b equals utterance b run alone, so a file's slices convert together and each
result equals that slice's own conversion.  Every length is computed on the host from the input sizes.

``convert_files`` is the whole CLI: a list of files, each cut at its silences by ``slicer.cut_batch``, against a list of
reference voices, with every voice sub-slice of every (file, voice) pair in shared ragged batches.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch
import torch.distributed as dist

from . import frontend, noise, shard
from .api import batch_plan, encode_voices, sample_latents
from .content import MIN_SAMPLES, num_frames
from .pre_model import Voice

TARGET_SR = 24000        # config data.sampling_rate: the rate of the converted audio
HOP = 256                # config data.hop_length
CONTENT_SR = 16000       # ContentVec's input rate (infer_tool.py:162)
LATENT_CH = 100
DEFAULT_STEPS = {"unipc": 30, "dpmsolver": 40}       # model.py:654-686 / :620-653


def frame_plan(n: int, sr: int) -> Dict[str, int]:
    """Host lengths of one utterance of n samples at ``sr``: 24 kHz samples ``n24``, frames ``T`` (= the f0 length), 16 kHz samples
    ``n16`` and ContentVec frames ``units`` (stretched to T afterwards)."""
    n24 = frontend.resample_out_length(sr, TARGET_SR, n)
    n16 = frontend.resample_out_length(TARGET_SR, CONTENT_SR, n24)
    return dict(n24=n24, T=n24 // HOP, n16=n16, units=num_frames(n16))


def _check_method(method: str, steps: Optional[int], seeded: bool = False) -> int:
    """The step count of ``method``.  DDPM and DDIM are accepted only for seeded rows (``seeded``: each row draws its noise
    from its own seed, so a row equals its own conversion): DDPM runs all 1000 timesteps (``steps`` None or 1000), DDIM
    ``steps`` pairs (default 100, ``sample()``'s ``sampling_timesteps``)."""
    if method in ("ddpm", "ddim") and seeded:
        if method == "ddpm":
            if steps not in (None, 1000):
                raise ValueError("method 'ddpm' runs every one of the 1000 timesteps (p_sample_loop); use 'ddim' for fewer steps")
            return 1000
        steps = 100 if steps is None else int(steps)
        if steps < 1:
            raise ValueError(f"steps must be >= 1, got {steps}")
        return steps
    if method in ("ddpm", "ddim"):
        raise ValueError(f"method {method!r}: its per-step noise of a ragged batch is drawn over the padded tensor, so a slice would "
                         "not equal its own conversion; use 'unipc' or 'dpmsolver'")
    if method not in DEFAULT_STEPS:
        raise ValueError(f"unknown method {method!r} (unipc | dpmsolver)")
    return DEFAULT_STEPS[method] if steps is None else int(steps)


def prompt_frames(p) -> int:
    """S_b of a prompt: a mel [100, S_b] or a ``Voice``."""
    return p.S_v if isinstance(p, Voice) else int(p.shape[1])


def check_voices(pre_model, prompts, dev: torch.device) -> None:
    """ValueError unless every ``Voice`` among ``prompts`` was encoded by ``pre_model`` on ``dev``."""
    for k, p in enumerate(prompts):
        if isinstance(p, Voice):
            pre_model.check_voice(p, dev, f"prompt {k}")


class FrontCache:
    """What the encoders computed during one conversion call, keyed by the identity of its input tensors: the units and
    stretched units of each waveform, and the ``Voice`` of each prompt mel.  Rows that repeat a waveform or a mel object share
    them.  The call holds every input it was given, so no identity is reused while the cache lives."""

    def __init__(self) -> None:
        self.units: Dict[int, Tuple[torch.Tensor, torch.Tensor]] = {}
        self.voices: Dict[int, Voice] = {}


def _check_seeds(noise_seeds, eta: float, method: str, n: int) -> Optional[List[int]]:
    """The seeds as n ints (or None), after the checks of ``eta``: in [0, 1], and 0 unless the method is DDIM."""
    if not 0.0 <= float(eta) <= 1.0:
        raise ValueError(f"eta must lie in [0, 1], got {eta}")
    if eta != 0.0 and method != "ddim":
        raise ValueError("eta applies to the ddim method")
    return None if noise_seeds is None else noise.check_seeds(noise_seeds, n, "noise_seeds")


def _check_inputs(wavs: Sequence[torch.Tensor], sr: int, prompt, x_T) -> List[Dict[str, int]]:
    if len(wavs) == 0:
        raise ValueError("wavs is empty")
    if int(sr) <= 0:
        raise ValueError(f"bad sample rate {sr}")
    plans = []
    for k, w in enumerate(wavs):
        if not isinstance(w, torch.Tensor) or w.dim() != 1:
            raise ValueError(f"waveform {k}: expected a 1-D (mono) tensor, got {tuple(getattr(w, 'shape', ()))}")
        p = frame_plan(int(w.shape[0]), sr)
        if p["T"] < 1 or p["n16"] < MIN_SAMPLES:
            raise ValueError(f"waveform {k}: {w.shape[0]} samples at {sr} Hz are too short ({p['n24']} at 24 kHz, {p['n16']} at 16 kHz; "
                             f"one frame needs {HOP} and {MIN_SAMPLES})")
        plans.append(p)
    prompts = list(prompt) if isinstance(prompt, (list, tuple)) else [prompt] * len(wavs)
    if len(prompts) != len(wavs):
        raise ValueError(f"{len(prompts)} prompts for {len(wavs)} waveforms")
    for k, p in enumerate(prompts):
        if isinstance(p, Voice):
            continue
        if not isinstance(p, torch.Tensor) or p.dim() != 2 or p.shape[0] != LATENT_CH or p.shape[1] < 1:
            raise ValueError(f"prompt {k}: expected a mel [{LATENT_CH}, S] or a Voice, got {tuple(getattr(p, 'shape', ()))}")
    if x_T is not None:
        if len(x_T) != len(wavs):
            raise ValueError(f"{len(x_T)} x_T tensors for {len(wavs)} waveforms")
        for k, (x, p) in enumerate(zip(x_T, plans)):
            if tuple(x.shape) not in ((1, LATENT_CH, p["T"]), (LATENT_CH, p["T"])):
                raise ValueError(f"x_T {k}: expected [1, {LATENT_CH}, {p['T']}], got {tuple(x.shape)}")
    return plans


@torch.no_grad()
def convert_batch(content_model, pre_model, unet, vocoder, wavs: Sequence[torch.Tensor], sr: int, prompts: Sequence,
                  x_T: Optional[Sequence[torch.Tensor]], method: str = "unipc", steps: Optional[int] = None,
                  cache: Optional[FrontCache] = None, noise_seeds: Optional[Sequence[int]] = None,
                  eta: float = 0.0) -> Dict[str, List[torch.Tensor]]:
    """Converts ``wavs`` (1-D, at ``sr``) as ONE ragged batch, each with its prompt (a mel [100, S_b] or a ``Voice``) and x_T
    [1, 100, T_b], and returns every stage per utterance, unpadded: ``units`` [D, units_b], ``c`` [D, T_b] (stretched), ``content``
    [T_b, C], ``prompt`` [S_b, C] (the encoders' outputs), ``latent`` [100, T_b] and ``audio`` [T_b * 256].  ``cache``: see
    ``encode_front``.

    ``noise_seeds`` (one int in [0, 2**63) per waveform): each row's x_T, when ``x_T`` is None, is ``noise.x_T`` of its seed, and
    ``ddpm`` / ``ddim`` (``eta``: the reference's ``ddim_sampling_eta``) are accepted, each row drawing its step noise from its
    seed; a row then equals that waveform converted alone with its seed, bit for bit."""
    steps = _check_method(method, steps, seeded=noise_seeds is not None)
    noise_seeds = _check_seeds(noise_seeds, eta, method, len(wavs))
    if x_T is None and noise_seeds is None:
        raise ValueError("x_T is required without noise_seeds")
    plans = _check_inputs(wavs, sr, list(prompts), None if x_T is None else list(x_T))
    dev = next(unet.parameters()).device
    check_voices(pre_model, prompts, dev)
    B = len(wavs)
    front = encode_front(content_model, pre_model, wavs, sr, prompts, plans, dev, cache)
    tl, content, prompt = front["tl"], front["content"], front["prompt"]
    sl = [prompt_frames(p) for p in prompts]
    T = max(tl)
    tl_h, sl_h = torch.tensor(tl, dtype=torch.int64), torch.tensor(sl, dtype=torch.int64)
    if x_T is None:
        x = noise.x_T(noise_seeds, LATENT_CH, tl, dev)
    else:
        x = torch.zeros((B, LATENT_CH, T), dtype=torch.float32, device=dev)
        for j, xt in enumerate(x_T):
            x[j, :, :tl[j]] = xt.reshape(LATENT_CH, tl[j]).to(dev, torch.float32)
    seeded = method in ("ddpm", "ddim")
    lat = sample_latents(unet, x, content, prompt, sl_h, steps=None if method == "ddpm" else steps, method=method, device=dev,
                         content_lengths=tl_h, eta=eta, noise_seeds=noise_seeds if seeded else None)
    audio = vocoder.decode(lat, tl_h)
    return dict(units=front["units"], c=front["c"], content=[content[:tl[j], j] for j in range(B)],
                prompt=[prompt[:sl[j], j] for j in range(B)], latent=[lat[j, :, :tl[j]] for j in range(B)],
                audio=[audio[j, :tl[j] * HOP] for j in range(B)])


def _first_rows(xs: Sequence, known: Dict[int, object]) -> List[int]:
    """The first row of each distinct object of ``xs`` (by identity) that ``known`` does not hold yet."""
    first: Dict[int, int] = {}
    for j, x in enumerate(xs):
        if id(x) not in known and id(x) not in first:
            first[id(x)] = j
    return list(first.values())


@torch.no_grad()
def encode_front(content_model, pre_model, wavs: Sequence[torch.Tensor], sr: int, prompts: Sequence,
                 plans: Sequence[Dict[str, int]], dev: torch.device, cache: Optional[FrontCache] = None) -> Dict[str, object]:
    """The encoders in front of the sampler, on ``wavs`` (checked by ``_check_inputs``, which gave ``plans``) as ONE ragged batch:
    resampling, ContentVec and ``repeat_expand_2d`` once per distinct waveform, ``Pre_model.encode_voices`` once per distinct
    prompt mel (a ``Voice`` is used as it is), then ``Pre_model.infer_content`` on every row.  Waveforms and mels are matched by
    tensor identity, within the call and with what ``cache`` (a ``FrontCache``, which this call extends) already holds.  Each
    row equals ``Pre_model.infer(per_utterance=True)`` on it.  Returns ``units`` and ``c`` per utterance, the frame counts
    ``tl``, and the encoders' padded outputs ``content`` [T, B, C] and ``prompt`` [S, B, C]."""
    cache = FrontCache() if cache is None else cache
    B = len(wavs)
    tl = [p["T"] for p in plans]
    todo = _first_rows(wavs, cache.units)
    if todo:
        n = [int(wavs[j].shape[0]) for j in todo]
        n24, n16, nu = ([plans[j][k] for j in todo] for k in ("n24", "n16", "units"))
        wav = torch.zeros((len(todo), max(n)), dtype=torch.float32, device=dev)
        for i, j in enumerate(todo):
            wav[i, :n[i]] = wavs[j].to(dev, torch.float32)
        w24, _ = frontend.resample(wav, sr, TARGET_SR, torch.tensor(n, dtype=torch.int64))
        w16, _ = frontend.resample(w24, TARGET_SR, CONTENT_SR, torch.tensor(n24, dtype=torch.int64))
        units_all, _ = content_model.extract(w16, torch.tensor(n16, dtype=torch.int64))
        for i, j in enumerate(todo):
            u = units_all[i, :nu[i]].t()
            cache.units[id(wavs[j])] = (u, frontend.repeat_expand_2d(u, tl[j]))
    mels = [p for p in prompts if not isinstance(p, Voice)]
    todo = _first_rows(mels, cache.voices)
    for j, v in zip(todo, encode_voices(pre_model, [mels[j] for j in todo], max_batch=max(len(todo), 1))):
        cache.voices[id(mels[j])] = v
    voices = [p if isinstance(p, Voice) else cache.voices[id(p)] for p in prompts]
    units = [cache.units[id(w)][0] for w in wavs]
    cs = [cache.units[id(w)][1] for w in wavs]
    T, S = max(tl), max(v.S_v for v in voices)
    c = torch.zeros((B, cs[0].shape[0], T), dtype=torch.float32, device=dev)
    for j in range(B):
        c[j, :, :tl[j]] = cs[j]
    content = pre_model.infer_content(c, torch.tensor(tl, dtype=torch.int64), voices)
    prompt = torch.zeros((S, B, voices[0].prompt.shape[1]), dtype=torch.float32, device=dev)
    for j, v in enumerate(voices):
        prompt[:v.S_v, j] = v.prompt
    return dict(units=units, c=cs, tl=tl, content=content, prompt=prompt)


@torch.no_grad()
def convert_utterances(content_model, pre_model, unet, vocoder, wavs: Sequence[torch.Tensor], sr: int,
                       prompt: Union[torch.Tensor, Voice, Sequence], method: str = "unipc", steps: Optional[int] = None,
                       max_batch: int = 8, x_T: Optional[Sequence[torch.Tensor]] = None,
                       group: Optional[dist.ProcessGroup] = None, noise_seeds: Optional[Sequence[int]] = None,
                       eta: float = 0.0) -> List[torch.Tensor]:
    """Converts 1-D float32 waveforms at ``sr`` with one prompt (or one per waveform) and returns one 24 kHz waveform
    [T_b * 256] per input, in input order, T_b = resample_out_length(sr, 24000, len) // 256.  The waveforms run in ragged
    batches of at most ``max_batch`` (longest first); each result equals that waveform converted alone.

    A prompt is a mel [100, S] or a ``Voice`` from ``api.encode_voices``.  Each distinct mel (by tensor identity) is encoded
    once per call, and each distinct waveform object goes through ContentVec once per call, whichever batches it lands in.

    ``x_T`` (one [1, 100, T_b] per waveform) defaults to ``torch.randn((1, 100, T_b), device=dev)`` drawn per waveform in input
    order before any batching: the shape and order in which ``Svc.infer`` draws it once per slice (``model.py:633-635``), so after
    the same ``torch.manual_seed`` each waveform gets the reference CLI's x_T.

    With a process ``group`` of more than one rank (one process per GPU, each with its models on its own device, every rank
    making the same call) the waveforms are shared out by ``shard.plan_batches`` and every rank returns the full list; see
    ``_convert_sharded``.

    ``noise_seeds`` (one int in [0, 2**63) per waveform) and ``eta``: as for ``convert_batch``.  With seeds, ``ddpm`` and ``ddim``
    are accepted and an x_T not given comes from each waveform's seed (no draw on the default generator, on any rank); each
    result equals that waveform converted alone with its seed, bit for bit."""
    steps = _check_method(method, steps, seeded=noise_seeds is not None)
    noise_seeds = _check_seeds(noise_seeds, eta, method, len(wavs))
    plans = _check_inputs(wavs, sr, prompt, x_T)
    prompts = list(prompt) if isinstance(prompt, (list, tuple)) else [prompt] * len(wavs)
    dev = next(unet.parameters()).device
    check_voices(pre_model, prompts, dev)
    if group is not None and dist.get_world_size(group) > 1:
        return _convert_sharded(content_model, pre_model, unet, vocoder, wavs, sr, prompts, plans, method, steps, max_batch, x_T, group, dev,
                                noise_seeds, eta)
    if x_T is None and noise_seeds is None:
        x_T = [torch.randn((1, LATENT_CH, p["T"]), device=dev) for p in plans]
    out: List[Optional[torch.Tensor]] = [None] * len(wavs)
    cache = FrontCache()
    for idx in batch_plan([int(w.shape[0]) for w in wavs], max_batch):
        r = convert_batch(content_model, pre_model, unet, vocoder, [wavs[i] for i in idx], sr, [prompts[i] for i in idx],
                          None if x_T is None else [x_T[i] for i in idx], method, steps, cache,
                          None if noise_seeds is None else [noise_seeds[i] for i in idx], eta)
        for j, i in enumerate(idx):
            out[i] = r["audio"][j]
    return out


def _convert_sharded(content_model, pre_model, unet, vocoder, wavs, sr, prompts, plans, method, steps, max_batch, x_T, group,
                     dev, noise_seeds=None, eta=0.0) -> List[torch.Tensor]:
    """``convert_utterances`` over the ranks of ``group``: each rank runs its batches of ``shard.plan_batches`` through
    ``convert_batch`` and ``shard.run_sharded`` gathers the audio of all ranks (one status exchange, one all-gather).

    The default x_T: every rank draws all of them, in input order on its own device, and keeps its own, so each waveform gets
    the x_T of the one-GPU call and every rank's generator ends where that call leaves it.  The ranks' CUDA generators must
    therefore start equal, which one all-gather of their seed and offset checks first.  With ``noise_seeds`` each rank draws only
    its own rows' x_T, from their seeds, and the generators are neither read nor checked."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    plan = shard.plan_batches(plans, [prompt_frames(p) for p in prompts], world, max_batch)
    if x_T is None and noise_seeds is None:
        shard.check_generator(torch.cuda.default_generators[dev.index], group, dev)
        mine = {i for b in plan[rank] for i in b}
        x_T = [x if i in mine else None for i, x in enumerate([torch.randn((1, LATENT_CH, p["T"]), device=dev) for p in plans])]
    cache = FrontCache()
    return shard.run_sharded(lambda idx: convert_batch(content_model, pre_model, unet, vocoder, [wavs[i] for i in idx], sr,
                                                       [prompts[i] for i in idx], None if x_T is None else [x_T[i] for i in idx],
                                                       method, steps, cache,
                                                       None if noise_seeds is None else [noise_seeds[i] for i in idx], eta)["audio"],
                             plan, [p["T"] * HOP for p in plans], group, dev)


# ------------------------------------------------------------------------------------------------------------ slicing (infer.py)
def pad_array(arr: np.ndarray, target_length: int) -> np.ndarray:
    """Centres ``arr`` in zeros up to ``target_length`` (longer arrays are returned as they are)."""
    if arr.shape[0] >= target_length:
        return arr
    w = target_length - arr.shape[0]
    return np.pad(arr, (w // 2, w - w // 2), "constant", constant_values=(0, 0))


def split_list_by_n(x, n: int, pre: int = 0) -> list:
    """Pieces of n samples, each but the first starting ``pre`` samples early (the cross-fade overlap)."""
    return [x[i - pre if i - pre >= 0 else i: i + n] for i in range(0, len(x), n)]


def _plan_slices(audio_data, audio_sr: int, pad_seconds: float, clip_seconds: float, linear_gradient: float):
    """The voice sub-slices to convert, padded with ``pad_seconds`` of zeros at the input rate, in the CLI's order."""
    per_size, lg_size = int(clip_seconds * audio_sr), int(linear_gradient * audio_sr)
    pad_len = int(audio_sr * pad_seconds)
    subs = []
    for slice_tag, data in audio_data:
        if slice_tag:
            continue
        for dat in (split_list_by_n(data, per_size, lg_size) if per_size != 0 else [data]):
            subs.append(np.concatenate([np.zeros([pad_len]), dat, np.zeros([pad_len])]))
    return subs


def stitch(audio_data, audio_sr: int, converted: Sequence[np.ndarray], pad_seconds: float = 0.5, clip_seconds: float = 0,
           linear_gradient: float = 0, linear_gradient_retain: float = 0.75) -> np.ndarray:
    """Assembles a file from the conversions of its voice sub-slices (``converted``, 24 kHz, in ``_plan_slices`` order) as
    ``infer.py:99-141`` does: silence as zeros, the ``pad_seconds`` trim, ``pad_array`` to each piece's length and the linear
    cross-fade between the pieces of a forced split.  float64."""
    per_size = int(clip_seconds * audio_sr)
    lg_size = int(linear_gradient * audio_sr)
    lg_size_r = int(lg_size * linear_gradient_retain)
    lg_size_c_l = (lg_size - lg_size_r) // 2
    lg_size_c_r = lg_size - lg_size_r - lg_size_c_l
    lg = np.linspace(0, 1, lg_size_r) if lg_size != 0 else 0
    lgr = linear_gradient_retain
    trim = int(TARGET_SR * pad_seconds)
    chunks: List[np.ndarray] = []
    it = iter(converted)

    def flat() -> np.ndarray:
        a = np.concatenate(chunks) if chunks else np.zeros(0)
        chunks[:] = [a]
        return a

    for slice_tag, data in audio_data:
        length = int(np.ceil(len(data) / audio_sr * TARGET_SR))
        if slice_tag:
            chunks.append(pad_array(np.zeros(length), length))
            continue
        for k, dat in enumerate(split_list_by_n(data, per_size, lg_size) if per_size != 0 else [data]):
            per_length = int(np.ceil(len(dat) / audio_sr * TARGET_SR)) if clip_seconds != 0 else length
            _audio = pad_array(np.asarray(next(it))[trim:-trim], per_length)
            if lg_size != 0 and k != 0:
                audio = flat()
                lg1 = audio[-(lg_size_r + lg_size_c_r):-lg_size_c_r] if lgr != 1 else audio[-lg_size:]
                lg2 = _audio[lg_size_c_l:lg_size_c_l + lg_size_r] if lgr != 1 else _audio[0:lg_size]
                lg_pre = lg1 * (1 - lg) + lg2 * lg
                chunks[:] = [audio[0:-(lg_size_r + lg_size_c_r)] if lgr != 1 else audio[0:-lg_size], lg_pre]
                _audio = _audio[lg_size_c_l + lg_size_r:] if lgr != 1 else _audio[lg_size:]
            chunks.append(_audio)
    return flat().astype(np.float64)


@torch.no_grad()
def convert_slices(content_model, pre_model, unet, vocoder, audio_data, audio_sr: int, prompt: Union[torch.Tensor, Voice], pad_seconds: float = 0.5,
                   clip_seconds: float = 0, linear_gradient: float = 0, linear_gradient_retain: float = 0.75, method: str = "unipc",
                   steps: Optional[int] = None, max_batch: int = 8, x_T: Optional[Sequence[torch.Tensor]] = None,
                   group: Optional[dist.ProcessGroup] = None) -> np.ndarray:
    """Converts one file given as ``slicer.chunks2audio``'s list of (is_silence, samples) at ``audio_sr`` with one prompt mel
    [100, S] (or a ``Voice``) and returns the float64 24 kHz array ``infer.py`` writes for it.  Every voice sub-slice goes through one
    ``convert_utterances`` call (``x_T``, if given, holds one tensor per sub-slice in order); stitching is ``stitch``.  With a
    ``group`` of more than one rank, the sub-slices are shared out over its ranks and every rank returns the stitched file."""
    _check_method(method, steps)
    if int(TARGET_SR * pad_seconds) <= 0:
        raise ValueError(f"pad_seconds={pad_seconds} trims no sample at {TARGET_SR} Hz, and the reference's [0:-0] trim would leave "
                         "every slice empty")
    subs = _plan_slices(audio_data, audio_sr, pad_seconds, clip_seconds, linear_gradient)
    converted = []
    if subs:
        outs = convert_utterances(content_model, pre_model, unet, vocoder, [torch.from_numpy(s.astype(np.float32)) for s in subs],
                                  audio_sr, prompt, method=method, steps=steps, max_batch=max_batch, x_T=x_T, group=group)
        converted = [o.cpu().numpy() for o in outs]
    return stitch(audio_data, audio_sr, converted, pad_seconds, clip_seconds, linear_gradient, linear_gradient_retain)


# ------------------------------------------------------------------------------------------------------------ the CLI (infer.py)
def voice_mels(voices: Sequence[Tuple[object, int]], dev: torch.device) -> List[torch.Tensor]:
    """The prompt mel [100, S_v] of each reference recording ``(wav, sr)``: ``frontend.log_mel_spectrogram`` in one ragged
    batch per rate.  A 2-D wav [channels, N] gives its channel 0, the channel ``model.py:610-611`` keeps."""
    from .slicer import _mono
    wavs, srs = [], []
    for k, v in enumerate(voices):
        if not isinstance(v, (tuple, list)) or len(v) != 2:
            raise ValueError(f"voice {k}: expected a (wav, sr) pair")
        w = torch.as_tensor(v[0])
        wavs.append(_mono(w[0] if w.dim() == 2 else w, f"voice {k}"))
        srs.append(int(v[1]))
    out: List[Optional[torch.Tensor]] = [None] * len(wavs)
    for sr in dict.fromkeys(srs):
        idx = [i for i, s in enumerate(srs) if s == sr]
        n = [int(wavs[i].shape[0]) for i in idx]
        x = torch.zeros((len(idx), max(n)), dtype=torch.float32, device=dev)
        for j, i in enumerate(idx):
            x[j, :n[j]] = wavs[i].to(dev)
        mel, frames = frontend.log_mel_spectrogram(x, sr, torch.tensor(n, dtype=torch.int64))
        for j, (i, s) in enumerate(zip(idx, frames.tolist())):
            out[i] = mel[j, :, :s]
    return out


def _files_x_T(sub_T: Sequence[Sequence[int]], n_voices: int, dev) -> List[List[List[torch.Tensor]]]:
    """x_T[f][v][k] = ``torch.randn((1, 100, sub_T[f][k]), device=dev)`` drawn in the CLI's nested order: file, then voice, then
    sub-slice (``infer.py:77, 92, 99-122``; ``Svc.infer`` draws once per call)."""
    return [[[torch.randn((1, LATENT_CH, T), device=dev) for T in Ts] for _ in range(n_voices)] for Ts in sub_T]


@torch.no_grad()
def convert_files(content_model, pre_model, unet, vocoder, files: Sequence[Tuple[object, int]], voices: Sequence[Tuple[object, int]],
                  slice_db: float = -40, pad_seconds: float = 0.5, clip_seconds: float = 0, linear_gradient: float = 0,
                  linear_gradient_retain: float = 0.75, method: str = "unipc", steps: Optional[int] = None, max_batch: int = 8,
                  x_T: Optional[Sequence[Sequence[Sequence[torch.Tensor]]]] = None,
                  group: Optional[dist.ProcessGroup] = None) -> List[List[np.ndarray]]:
    """The reference CLI (``infer.py:58-145``): every file of ``files`` converted with every voice of ``voices``.  Returns
    ``out[f][v]``, the float64 24 kHz array ``infer.py`` writes for file f and voice v.

    ``files`` are ``(wav, sr)`` pairs of 1-D float32 samples (as ``librosa.load(sr=None)`` returns them); each is cut at its
    silences by ``slicer.cut_batch`` (``slice_db``, min_len 5000 ms, as ``infer.py:83`` calls ``slicer.cut``; one RMS launch for
    all files) and split into voice sub-slices as ``convert_slices`` does.  ``voices`` are ``(wav, sr)`` reference recordings
    (1-D, or [channels, N] of which channel 0 is used); their prompt mels come from ``voice_mels`` and are encoded once, by
    ``api.encode_voices``.  Every (file, voice, sub-slice) item of one input rate goes through ONE ``convert_utterances`` call,
    so the slices of different files and voices share ragged batches (files at several rates take one call per rate); the V
    items of one sub-slice share its ContentVec units, which each rank computes once, for the sub-slices of its own batches.
    Each file is stitched per voice by ``stitch``.

    ``x_T`` (``x_T[f][v]``: one [1, 100, T] per voice sub-slice of file f) defaults to ``torch.randn((1, 100, T))`` per item drawn
    in the CLI's order - file, then voice, then sub-slice - before any conversion, so after the same ``torch.manual_seed`` every
    slice starts from the reference CLI's noise.  ``group`` is passed to ``convert_utterances``; every rank draws every x_T,
    after ``shard.check_generator`` has checked that the ranks' generators agree."""
    from . import slicer
    _check_method(method, steps)
    if int(TARGET_SR * pad_seconds) <= 0:
        raise ValueError(f"pad_seconds={pad_seconds} trims no sample at {TARGET_SR} Hz, and the reference's [0:-0] trim would leave "
                         "every slice empty")
    if len(files) == 0 or len(voices) == 0:
        raise ValueError(f"{len(files)} files and {len(voices)} voices: give at least one of each")
    for k, f in enumerate(files):
        if not isinstance(f, (tuple, list)) or len(f) != 2:
            raise ValueError(f"file {k}: expected a (wav, sr) pair")
        slicer._mono(f[0], f"file {k}")
    dev = next(unet.parameters()).device
    wavs, srs = [f[0] for f in files], [int(f[1]) for f in files]
    chunks = slicer.cut_batch(wavs, srs, slice_db, 5000, device=dev)
    audio_data = [slicer.chunks2audio(w, c) for w, c in zip(wavs, chunks)]
    subs = [_plan_slices(a, sr, pad_seconds, clip_seconds, linear_gradient) for a, sr in zip(audio_data, srs)]
    sub_T = [[frame_plan(len(s), sr)["T"] for s in ss] for ss, sr in zip(subs, srs)]
    encoded = encode_voices(pre_model, voice_mels(voices, dev), max_batch=max_batch)
    V = len(voices)
    if x_T is None:
        if group is not None and dist.get_world_size(group) > 1:
            shard.check_generator(torch.cuda.default_generators[dev.index], group, dev)
        x_T = _files_x_T(sub_T, V, dev)
    elif len(x_T) != len(files) or any(len(xf) != V or any(len(xv) != len(ss) for xv in xf) for xf, ss in zip(x_T, subs)):
        raise ValueError("x_T must hold x_T[f][v], one tensor per voice sub-slice of file f, for every file and voice")
    converted: Dict[Tuple[int, int], List[np.ndarray]] = {(f, v): [] for f in range(len(files)) for v in range(V)}
    sources = [[torch.from_numpy(s.astype(np.float32)) for s in ss] for ss in subs]     # one tensor per sub-slice: its V items share it
    for sr in dict.fromkeys(srs):
        items = [(f, v, k) for f in range(len(files)) if srs[f] == sr for v in range(V) for k in range(len(subs[f]))]
        if not items:
            continue
        outs = convert_utterances(content_model, pre_model, unet, vocoder, [sources[f][k] for f, _, k in items], sr,
                                  [encoded[v] for _, v, _ in items], method=method, steps=steps, max_batch=max_batch,
                                  x_T=[x_T[f][v][k] for f, v, k in items], group=group)
        for (f, v, _), o in zip(items, outs):
            converted[(f, v)].append(o.cpu().numpy())
    return [[stitch(audio_data[f], srs[f], converted[(f, v)], pad_seconds, clip_seconds, linear_gradient, linear_gradient_retain)
             for v in range(V)] for f in range(len(files))]
