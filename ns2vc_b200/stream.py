"""Live conversion: waveform streams converted in real time, one block per tick, several streams per tick.

Each stream (a *slot*) keeps a fixed input window of ``context_frames + block_frames`` output frames.  A tick (``push``) slides
every window by one block, converts all windows as one ragged batch with ``convert.convert_batch`` (so slot b of a tick equals
its window converted alone), and joins the end of each converted window to the last tick's output by SOLA (synchronized
overlap-add, ``csrc/stream.cu``): the offset in a short search range where the new audio best matches the tail kept from the
last tick, a cross-fade there, one block emitted, the next tail kept.  Every tick has the same shape, so the sampler session of
that shape is reused (and replays its captured graph) from tick to tick.

Sizes are in 24 kHz output frames of ``HOP = 256`` samples; see ``stream_plan``.
"""
from __future__ import annotations

import math
import operator
from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib, convert
from .api import encode_voices
from .content import MIN_SAMPLES
from .convert import HOP, LATENT_CH, TARGET_SR
from .pre_model import Voice

# (2 Nc + Ns) fp32 samples staged in shared memory by the SOLA kernel
SOLA_MAX_SAMPLES = 47 * 1024 // 4


def _frame_step(sr: int) -> int:
    """The smallest number of frames whose input samples at ``sr`` are a whole number: frames * 256 * sr / 24000."""
    return TARGET_SR // math.gcd(HOP * sr, TARGET_SR)


def _nearest(v: int, q: int) -> str:
    lo = v // q * q
    return " or ".join(str(c) for c in (lo, lo + q) if c >= q)


def stream_plan(sr: int, block_frames: int = 45, context_frames: int = 150, crossfade: int = 1024, search: int = 512) -> Dict[str, int]:
    """The fixed geometry of a live-conversion session at input rate ``sr``: window ``T`` frames, ``Nb`` samples emitted per tick,
    cross-fade ``Nc`` and search ``Ns`` samples (24 kHz), and ``block_in`` / ``context_in`` / ``W_in`` input samples per block,
    context and window.  ``seg = Nb + Nc + Ns`` is the end of each converted window that SOLA reads.  Raises ValueError when a
    block or the context is not a whole number of input samples (naming the nearest valid frame counts), when the context is
    shorter than the cross-fade plus the search, or the block shorter than the cross-fade."""
    sr, bf, cf, Nc, Ns = (int(v) for v in (sr, block_frames, context_frames, crossfade, search))
    if sr <= 0:
        raise ValueError(f"bad sample rate {sr}")
    if bf < 1 or cf < 1:
        raise ValueError(f"block_frames and context_frames must be >= 1, got {bf} and {cf}")
    if Nc < 2 or Ns < 0:
        raise ValueError(f"crossfade must be >= 2 and search >= 0 samples, got {Nc} and {Ns}")
    q = _frame_step(sr)
    for name, v in (("block_frames", bf), ("context_frames", cf)):
        if v % q:
            raise ValueError(f"{name}={v}: {v} frames are {v * HOP * sr / TARGET_SR:g} samples at {sr} Hz, not a whole number; "
                             f"use a multiple of {q}, e.g. {_nearest(v, q)}")
    Nb = bf * HOP
    if cf * HOP < Nc + Ns:
        raise ValueError(f"context_frames={cf} ({cf * HOP} samples) is shorter than crossfade + search = {Nc + Ns} samples")
    if Nb < Nc:
        raise ValueError(f"block_frames={bf} ({Nb} samples) is shorter than the crossfade of {Nc} samples")
    if 2 * Nc + Ns > SOLA_MAX_SAMPLES:
        raise ValueError(f"2 * crossfade + search = {2 * Nc + Ns} samples exceed the SOLA kernel's {SOLA_MAX_SAMPLES}")
    T = cf + bf
    block_in, context_in = bf * HOP * sr // TARGET_SR, cf * HOP * sr // TARGET_SR
    W_in = block_in + context_in
    fp = convert.frame_plan(W_in, sr)
    assert fp["T"] == T, (fp, T)
    if fp["n16"] < MIN_SAMPLES:
        raise ValueError(f"a window of {T} frames is {fp['n16']} samples at 16 kHz; ContentVec needs {MIN_SAMPLES}")
    return dict(sr=sr, block_frames=bf, context_frames=cf, T=T, Nb=Nb, Nc=Nc, Ns=Ns, seg=Nb + Nc + Ns, block_in=block_in,
                context_in=context_in, W_in=W_in)


def fade_in_table(Nc: int) -> np.ndarray:
    """sin^2(pi/2 * i / (Nc - 1)), i < Nc, computed in fp64 and rounded once to fp32."""
    i = np.arange(Nc, dtype=np.float64)
    return (np.sin(np.pi / 2 * (i / (Nc - 1))) ** 2).astype(np.float32)


def _check_prompt(p, what: str) -> None:
    if isinstance(p, Voice):
        return
    if not isinstance(p, torch.Tensor) or p.dim() != 2 or p.shape[0] != LATENT_CH or p.shape[1] < 1:
        raise ValueError(f"{what}: expected a mel [{LATENT_CH}, S], got {tuple(getattr(p, 'shape', ()))}")


def sola(seg: torch.Tensor, tail: torch.Tensor, fade_in: torch.Tensor, Nb: int, Nc: int, Ns: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """The SOLA join of one tick on the GPU (``ns2vc_stream_sola``).  seg [B, >= Nb + Nc + Ns] (unit inner stride; its first
    Nb + Nc + Ns samples are read), tail [B, Nc] contiguous (replaced in place by the next tail), fade_in [Nc], all CUDA float32
    -> (out [B, Nb], offsets [B] int32): the emitted block and the chosen offset of each row."""
    B = seg.shape[0]
    for name, t in (("seg", seg), ("tail", tail), ("fade_in", fade_in)):
        if t.device.type != "cuda" or t.dtype != torch.float32:
            raise ValueError(f"sola: {name} must be CUDA float32, got {t.dtype} on {t.device}")
    if seg.dim() != 2 or seg.shape[1] < Nb + Nc + Ns or seg.stride(1) != 1:
        raise ValueError(f"sola: seg must be [B, >= {Nb + Nc + Ns}] with unit inner stride, got {tuple(seg.shape)} / {seg.stride()}")
    if tuple(tail.shape) != (B, Nc) or not tail.is_contiguous() or tuple(fade_in.shape) != (Nc,) or not fade_in.is_contiguous():
        raise ValueError(f"sola: expected a contiguous tail [{B}, {Nc}] and fade_in [{Nc}], got {tuple(tail.shape)} and {tuple(fade_in.shape)}")
    dev = seg.device
    out = torch.empty((B, Nb), dtype=torch.float32, device=dev)
    offsets = torch.empty((B,), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().ns2vc_stream_sola(seg.data_ptr(), seg.stride(0), tail.data_ptr(), fade_in.data_ptr(), out.data_ptr(),
                                                offsets.data_ptr(), B, Nb, Nc, Ns, torch.cuda.current_stream(dev).cuda_stream))
    return out, offsets


class StreamConverter:
    """Converts ``len(prompts)`` live streams at input rate ``sr`` in ticks of ``block_frames`` output frames (0.48 s by default),
    stream b with the target voice of ``prompts[b]`` (a mel [100, S_b] or a ``Voice``).  Geometry as ``stream_plan``; ``method``
    / ``steps`` as ``convert.convert_utterances`` (UniPC-30 by default, or DPM-Solver++).  Every window and SOLA tail starts as
    zeros.  Each prompt mel is encoded once (``api.encode_voices``, at the first tick after it is given), so a tick runs only
    the content side of the condition encoders.

    Attributes after each ``push``: ``seg`` [B, Nb + Nc + Ns] (the end of each converted window that SOLA joined) and
    ``offsets`` [B] int32 (the chosen SOLA offsets)."""

    def __init__(self, content_model, pre_model, unet, vocoder, prompts: Sequence[torch.Tensor], sr: int, block_frames: int = 45,
                 context_frames: int = 150, crossfade: int = 1024, search: int = 512, method: str = "unipc",
                 steps: Optional[int] = None):
        self.steps = convert._check_method(method, steps)
        self.method = method
        self.plan = stream_plan(sr, block_frames, context_frames, crossfade, search)
        prompts = list(prompts)
        if not prompts:
            raise ValueError("prompts is empty: give one prompt mel per stream")
        for k, p in enumerate(prompts):
            _check_prompt(p, f"prompt {k}")
        self.models = (content_model, pre_model, unet, vocoder)
        self.sr = self.plan["sr"]
        self.device = next(unet.parameters()).device
        self.prompts = [p if isinstance(p, Voice) else p.to(self.device, torch.float32) for p in prompts]
        self.voices = [p if isinstance(p, Voice) else None for p in self.prompts]     # None: encoded at the next tick
        self.B = len(prompts)
        self.window = torch.zeros((self.B, self.plan["W_in"]), dtype=torch.float32, device=self.device)
        self.tail = torch.zeros((self.B, self.plan["Nc"]), dtype=torch.float32, device=self.device)
        self.fade_in = torch.from_numpy(fade_in_table(self.plan["Nc"])).to(self.device)
        self.seg: Optional[torch.Tensor] = None
        self.offsets = torch.zeros((self.B,), dtype=torch.int32, device=self.device)

    @torch.no_grad()
    def push(self, block: torch.Tensor, x_T: Optional[Sequence[torch.Tensor]] = None) -> torch.Tensor:
        """One tick: ``block`` [B, block_in] float32 input samples (one block per stream, on any device) -> the next [B, Nb]
        24 kHz output samples of every stream, on ``block``'s device.  ``x_T`` (B tensors [1, 100, T]) defaults to
        ``torch.randn((1, 100, T), device=dev)`` drawn once per stream in stream order, the draw ``convert_utterances`` makes per
        utterance.  A NaN in the sampler raises its AssertionError here."""
        p = self.plan
        B, T = self.B, p["T"]
        if not isinstance(block, torch.Tensor) or tuple(block.shape) != (B, p["block_in"]):
            raise ValueError(f"block: expected [{B}, {p['block_in']}] ({p['block_frames']} frames at {self.sr} Hz for {B} streams), "
                             f"got {tuple(getattr(block, 'shape', ()))}")
        if x_T is not None:
            if len(x_T) != B:
                raise ValueError(f"{len(x_T)} x_T tensors for {B} streams")
            for k, x in enumerate(x_T):
                if tuple(x.shape) not in ((1, LATENT_CH, T), (LATENT_CH, T)):
                    raise ValueError(f"x_T {k}: expected [1, {LATENT_CH}, {T}], got {tuple(x.shape)}")
        dev = self.device
        self.window = torch.cat((self.window[:, p["block_in"]:], block.to(dev, torch.float32)), dim=1)
        if x_T is None:
            x_T = [torch.randn((1, LATENT_CH, T), device=dev) for _ in range(B)]
        todo = [b for b, v in enumerate(self.voices) if v is None]
        for b, v in zip(todo, encode_voices(self.models[1], [self.prompts[b] for b in todo], max_batch=max(len(todo), 1))):
            self.voices[b] = v
        r = convert.convert_batch(*self.models, list(self.window.unbind(0)), self.sr, self.voices, x_T, self.method, self.steps)
        audio = torch.stack(r["audio"])
        self.seg = audio[:, T * HOP - p["seg"]:]
        out, self.offsets = sola(self.seg, self.tail, self.fade_in, p["Nb"], p["Nc"], p["Ns"])
        return out.to(block.device)

    def reset(self, slot: int, prompt: Optional[torch.Tensor] = None) -> None:
        """Starts stream ``slot`` again from silence: zeroes its window and SOLA tail and, if given, replaces its prompt (a mel
        [100, S] or a ``Voice``; a prompt longer than the others makes the next tick run a new shape)."""
        slot = operator.index(slot)
        if not 0 <= slot < self.B:
            raise IndexError(f"slot {slot} out of range for {self.B} streams")
        if prompt is not None:
            _check_prompt(prompt, "prompt")
            self.prompts[slot] = prompt if isinstance(prompt, Voice) else prompt.to(self.device, torch.float32)
            self.voices[slot] = prompt if isinstance(prompt, Voice) else None
        self.window[slot].zero_()
        self.tail[slot].zero_()
