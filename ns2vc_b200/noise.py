"""Seeded sampler noise: each utterance's DDPM / DDIM noise and x_T drawn from its own 64-bit seed on the GPU.

The normal at (seed, step, c, t) is a pure function of those four values (Philox4x32-10 keyed by the seed, counter
(t >> 2, c, step, 0), Box-Muller; ``csrc/philox.cuh``), so an utterance's noise is the same whatever batch, slot, padding or
rank it runs in.  Step k of a run draws at step index k; ``XT_STEP`` is reserved for the utterance's x_T.  ``normal_rows`` is
the exact tensor the seeded step kernels draw in-register, so a seeded run equals the injected-noise path fed with it.
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch

from . import _lib

MAX_SEED = 1 << 63                  # seeds are ints in [0, 2**63): an int64 on the device
XT_STEP = 0xFFFFFFFF


def check_seeds(seeds, B: int, name: str = "seeds") -> list:
    """The seeds as a list of B ints in [0, 2**63); ValueError otherwise."""
    vals = [int(s) for s in (seeds.tolist() if isinstance(seeds, torch.Tensor) else seeds)]
    if len(vals) != B:
        raise ValueError(f"{name} must have {B} entries (one per utterance), got {len(vals)}")
    bad = [s for s in vals if not 0 <= s < MAX_SEED]
    if bad:
        raise ValueError(f"{name} must lie in [0, 2**63), got {bad}")
    return vals


def normal_rows(seeds: Sequence[int], C: int, lengths: Optional[Sequence[int]] = None, step: int = 0,
                device: Optional[torch.device] = None, T: Optional[int] = None) -> torch.Tensor:
    """[B, C, T] fp32 on ``device`` (default: the current CUDA device): row b holds the normals at (seeds[b], step, c, t) for
    t < lengths[b] and zeros past it.  T defaults to max(lengths); without lengths every row is T long."""
    if lengths is None and T is None:
        raise ValueError("normal_rows needs lengths or T")
    seeds = check_seeds(seeds, len(seeds))
    B = len(seeds)
    lens = [int(v) for v in lengths] if lengths is not None else None
    T = int(T) if T is not None else max(lens)
    if lens is not None and (len(lens) != B or any(not 1 <= v <= T for v in lens)):
        raise ValueError(f"lengths must be {B} values in [1, {T}], got {lens}")
    if not 0 <= int(step) <= XT_STEP:
        raise ValueError(f"step must lie in [0, 2**32), got {step}")
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    out = torch.empty((B, int(C), T), dtype=torch.float32, device=dev)
    sd = torch.tensor(seeds, dtype=torch.int64).to(dev)
    ln = torch.tensor(lens, dtype=torch.int64).to(dev) if lens is not None else None
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().ns2vc_noise_normal_rows(sd.data_ptr(), int(step), int(C), T, ln.data_ptr() if ln is not None else None,
                                                      out.data_ptr(), B, torch.cuda.current_stream(dev).cuda_stream))
    return out


def x_T(seeds: Sequence[int], C: int, lengths: Sequence[int], device: Optional[torch.device] = None,
        T: Optional[int] = None) -> torch.Tensor:
    """Each utterance's x_T [B, C, T]: ``normal_rows`` at the reserved step ``XT_STEP``."""
    return normal_rows(seeds, C, lengths, XT_STEP, device, T)
