"""Diagnostics for the parity tests: run a forward and collect the engine's per-op activations."""
from __future__ import annotations

import ctypes as C
from typing import Any, Callable, Dict, Optional, Tuple

import torch

from . import _lib
from .arch import level_lengths


def run_with_taps(unet, device: torch.device, B: int, T: int, run: Callable[[], Any]) -> Tuple[Any, Dict[str, torch.Tensor]]:
    """Sets every tap of the engine's ACTIVE program (B, T: its batch and frame count), calls ``run()``, clears the taps.
    ``run`` must execute that program (the module call of the same shape, or ``DenoiserSession.forward`` of the session that
    prepared it) without building another one first.  Returns (run's result, {op name: activation [B,C,T_level]}) —
    activations converted from the engine's token-major layout to the reference's channel-major layout; fresh zeroed
    buffers, so a tap the program does not write reads 0."""
    Tl = level_lengths(T, len(unet.cfg.block_out_channels))
    res, bufs = unet._collect_taps(device, B, run, rows=lambda level: Tl[level])
    return res, {k: v.permute(0, 2, 1).contiguous() for k, v in bufs.items()}


def forward_with_taps(unet, sample: torch.Tensor, timestep, ehs: torch.Tensor,
                      mask: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
    """Module call (the padded program) with taps: (output [B,Cout,T], {op name: activation [B,C,T_level]})."""
    with torch.no_grad():
        unet(sample, timestep, ehs, encoder_attention_mask=mask)      # builds the program for this shape
    B, _, T = sample.shape
    return run_with_taps(unet, sample.device, B, T, lambda: unet(sample, timestep, ehs, encoder_attention_mask=mask).sample)


def session_forward_with_taps(sess, x: torch.Tensor, t: torch.Tensor) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
    """``DenoiserSession.forward`` (its padded or ragged program) with taps: (output [B,Cout,T], taps as above)."""
    out = torch.empty((sess.B, sess.Co, sess.T), dtype=torch.float32, device=sess.dev)
    sess.forward(x, t, out)                                            # builds and prepares the session's program
    return run_with_taps(sess.unet, sess.dev, sess.B, sess.T, lambda: (sess.forward(x, t, out), out)[1])


def profile_forward(unet, steps_fn, device, dump_csv: Optional[str] = None) -> Dict[str, Tuple[float, int]]:
    """Run ``steps_fn()`` with per-launch CUDA-event timing on; returns {kind: (total ms, launches)}."""
    L = _lib.lib()
    h = unet.engine(device)
    _lib.check(L.ns2vc_unet_profile_reset(h))
    _lib.check(L.ns2vc_unet_set_profiling(h, 1))
    try:
        steps_fn()
        torch.cuda.synchronize(device)
    finally:
        _lib.check(L.ns2vc_unet_set_profiling(h, 0))
    out = {}
    for k in range(L.ns2vc_profile_num_kinds()):
        ms, n = C.c_double(), C.c_longlong()
        _lib.check(L.ns2vc_unet_profile_read(h, k, C.byref(ms), C.byref(n)))
        if n.value:
            out[L.ns2vc_profile_kind_name(k).decode()] = (ms.value, n.value)
    if dump_csv:
        _lib.check(L.ns2vc_unet_profile_dump(h, dump_csv.encode()))
    _lib.check(L.ns2vc_unet_profile_reset(h))
    return out
