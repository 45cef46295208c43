"""The reference CLI's silence slicer (``inference/slicer.py``) without librosa: a file is cut at its silences into voice and
silence chunks before conversion (``infer.py:83-84``).

* ``rms_frames`` - the framewise RMS that ``Slicer.slice`` takes from ``librosa.feature.rms`` (librosa 0.10: centre padding with
  zeros, numpy's pairwise float32 mean of each squared frame, sqrt), computed on the GPU for a ragged batch of files, each at
  its own rate, bit for bit (``csrc/slicer.cu``, checked against ``oracle/slicer_oracle.py``).
* ``cut`` / ``cut_batch`` - ``slicer.cut``'s chunk dict: the RMS on the GPU (one launch and one device-to-host copy of the
  frames per call), then the reference's decision logic on the host, restated line for line with its quirks: a file of at
  most ``min_length`` samples (a frame count) is returned whole, ``argmin`` takes the first minimum, and the trailing-silence
  tag ends at ``total_frames + 1``.  ``rms < threshold`` compares in float32, as NumPy >= 2 does (NEP 50).
* ``chunks2audio`` - the (is_silence, samples) list that ``convert.convert_slices`` takes.

Inputs are 1-D float32 mono, as ``librosa.load(path, sr=None)`` returns them; a caller with several channels mixes them first.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _lib

MIN_INTERVAL_MS = 300      # Slicer defaults that slicer.cut keeps (slicer.py:6-13)
HOP_MS = 20
MAX_SIL_KEPT_MS = 5000

Chunks = Dict[str, Dict[str, object]]
Wave = Union[np.ndarray, torch.Tensor]


def hop_win(sr: int) -> Tuple[int, int]:
    """The slicer's RMS hop and window in samples at ``sr``: round(sr * 20 / 1000) and min(round(sr * 300 / 1000), 4 hop)."""
    sr = int(sr)
    if sr <= 0:
        raise ValueError(f"bad sample rate {sr}")
    hop = round(sr * HOP_MS / 1000)
    if hop < 1:
        raise ValueError(f"sample rate {sr} Hz gives a hop of {hop} samples")
    return hop, min(round(sr * MIN_INTERVAL_MS / 1000), 4 * hop)


def slicer_params(sr: int, db_thresh: float = -30, min_len: int = 5000) -> Dict[str, float]:
    """``Slicer(sr, threshold=db_thresh, min_length=min_len)``'s attributes (slicer.py:14-24): the linear ``threshold``, ``hop``
    and ``win`` in samples, ``min_length``, ``min_interval`` and ``max_sil_kept`` in frames.  Python's ``round`` halves to even
    (11025 Hz gives hop 220)."""
    hop, win = hop_win(sr)
    if not min_len >= MIN_INTERVAL_MS:
        raise ValueError(f"min_len={min_len} ms: the slicer needs min_len >= min_interval ({MIN_INTERVAL_MS} ms)")
    sr = int(sr)
    return dict(threshold=10 ** (db_thresh / 20.), hop=hop, win=win, min_length=round(sr * min_len / 1000 / hop),
                min_interval=round(sr * MIN_INTERVAL_MS / 1000 / hop), max_sil_kept=round(sr * MAX_SIL_KEPT_MS / 1000 / hop))


def num_frames(n: int, hop: int, win: int) -> int:
    """librosa's RMS frame count for n samples: 1 + (n + 2 (win // 2) - win) // hop."""
    r = _lib.lib().ns2vc_slice_rms_frames(int(n), int(hop), int(win))
    if r < 0:
        raise ValueError(_lib.lib().ns2vc_last_error().decode())
    return r


def _mono(wav: Wave, what: str) -> Wave:
    if not isinstance(wav, (np.ndarray, torch.Tensor)):
        raise ValueError(f"{what}: expected a 1-D float32 array, got {type(wav).__name__}")
    if wav.ndim != 1:
        raise ValueError(f"{what}: expected 1-D mono samples, got shape {tuple(wav.shape)}; mix the channels first")
    if wav.dtype not in (np.float32, torch.float32):
        raise ValueError(f"{what}: expected float32 samples, got {wav.dtype}")
    return wav


def rms_frames(wavs: torch.Tensor, lengths: Optional[torch.Tensor], sr: Union[int, Sequence[int]]) -> Tuple[torch.Tensor, List[int]]:
    """wavs CUDA float32 [B, N] (or [N]), lengths int64 [B] (default all N), sr one rate or one per row -> (rms [B, F] float32 on
    the device, frame counts [B]).  Row b equals ``librosa.feature.rms(y=wavs[b, :lengths[b]], frame_length=win_b,
    hop_length=hop_b)[0]`` bit for bit, with the slicer's hop and win at rate sr[b]; frames past its count are 0 and samples
    past its length are never read.  F is the largest count."""
    if not isinstance(wavs, torch.Tensor) or wavs.dim() not in (1, 2) or wavs.dtype != torch.float32:
        raise ValueError(f"wavs must be a float32 tensor [B, N] or [N], got {getattr(wavs, 'dtype', type(wavs))} "
                         f"{tuple(getattr(wavs, 'shape', ()))}")
    if wavs.device.type != "cuda":
        raise RuntimeError("slicer.rms_frames has no CPU path: move the waveforms to an H100 ('cuda')")
    x = wavs.unsqueeze(0) if wavs.dim() == 1 else wavs
    if x.stride(-1) != 1:
        x = x.contiguous()
    B, N = x.shape
    if B < 1:
        raise ValueError("wavs holds no rows")
    srs = [int(sr)] * B if isinstance(sr, (int, np.integer)) else [int(s) for s in sr]
    if len(srs) != B:
        raise ValueError(f"{len(srs)} sample rates for {B} rows")
    host = [N] * B if lengths is None else [int(v) for v in lengths.tolist()]
    if len(host) != B or min(host) < 0 or max(host) > N:
        raise ValueError(f"lengths must be {B} values in [0, {N}], got {host}")
    hw = [hop_win(s) for s in srs]
    frames = [num_frames(n, h, w) for n, (h, w) in zip(host, hw)]
    dev = x.device
    F = max(frames)
    rms = torch.empty((B, F), dtype=torch.float32, device=dev)
    dlen = torch.tensor(host, dtype=torch.int64).to(dev)
    dhw = torch.tensor(hw, dtype=torch.int32).to(dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().ns2vc_slice_rms(x.data_ptr(), x.stride(0), dlen.data_ptr(), dhw.data_ptr(), rms.data_ptr(), F, B,
                                              torch.cuda.current_stream(dev).cuda_stream))
    return rms, frames


def slice_from_rms(rms_list: np.ndarray, n: int, p: Dict[str, float]) -> Chunks:
    """``Slicer.slice`` (slicer.py:33-117) of a file of n samples, given its float32 rms frames and ``slicer_params``."""
    hop = p["hop"]
    if n <= p["min_length"]:           # the reference compares samples against a frame count
        return {"0": {"slice": False, "split_time": f"0,{n}"}}
    silent = (rms_list < np.float32(p["threshold"])).tolist()
    min_interval, min_length, max_sil_kept = p["min_interval"], p["min_length"], p["max_sil_kept"]
    sil_tags = []
    silence_start = None
    clip_start = 0
    for i in range(len(silent)):
        if silent[i]:
            if silence_start is None:
                silence_start = i
            continue
        if silence_start is None:
            continue
        is_leading_silence = silence_start == 0 and i > max_sil_kept
        need_slice_middle = i - silence_start >= min_interval and i - clip_start >= min_length
        if not is_leading_silence and not need_slice_middle:
            silence_start = None
            continue
        if i - silence_start <= max_sil_kept:
            pos = int(rms_list[silence_start: i + 1].argmin()) + silence_start
            if silence_start == 0:
                sil_tags.append((0, pos))
            else:
                sil_tags.append((pos, pos))
            clip_start = pos
        elif i - silence_start <= max_sil_kept * 2:
            pos = int(rms_list[i - max_sil_kept: silence_start + max_sil_kept + 1].argmin())
            pos += i - max_sil_kept
            pos_l = int(rms_list[silence_start: silence_start + max_sil_kept + 1].argmin()) + silence_start
            pos_r = int(rms_list[i - max_sil_kept: i + 1].argmin()) + i - max_sil_kept
            if silence_start == 0:
                sil_tags.append((0, pos_r))
                clip_start = pos_r
            else:
                sil_tags.append((min(pos_l, pos), max(pos_r, pos)))
                clip_start = max(pos_r, pos)
        else:
            pos_l = int(rms_list[silence_start: silence_start + max_sil_kept + 1].argmin()) + silence_start
            pos_r = int(rms_list[i - max_sil_kept: i + 1].argmin()) + i - max_sil_kept
            if silence_start == 0:
                sil_tags.append((0, pos_r))
            else:
                sil_tags.append((pos_l, pos_r))
            clip_start = pos_r
        silence_start = None
    total_frames = len(silent)
    if silence_start is not None and total_frames - silence_start >= min_interval:
        silence_end = min(total_frames, silence_start + max_sil_kept)
        pos = int(rms_list[silence_start: silence_end + 1].argmin()) + silence_start
        sil_tags.append((pos, total_frames + 1))
    if len(sil_tags) == 0:
        return {"0": {"slice": False, "split_time": f"0,{n}"}}
    chunks = []
    if sil_tags[0][0]:
        chunks.append({"slice": False, "split_time": f"0,{min(n, sil_tags[0][0] * hop)}"})
    for i in range(0, len(sil_tags)):
        if i:
            chunks.append({"slice": False, "split_time": f"{sil_tags[i - 1][1] * hop},{min(n, sil_tags[i][0] * hop)}"})
        chunks.append({"slice": True, "split_time": f"{sil_tags[i][0] * hop},{min(n, sil_tags[i][1] * hop)}"})
    if sil_tags[-1][1] * hop < n:
        chunks.append({"slice": False, "split_time": f"{sil_tags[-1][1] * hop},{n}"})
    return {str(i): c for i, c in enumerate(chunks)}


def cut_batch(wavs: Sequence[Wave], srs: Union[int, Sequence[int]], db_thresh: float = -30, min_len: int = 5000,
              device: Union[str, torch.device] = "cuda") -> List[Chunks]:
    """``slicer.cut`` of several files: 1-D float32 samples (numpy or torch) at ``srs`` (one rate or one per file) -> one chunk
    dict per file, each equal to the reference's on the same samples.  One RMS launch on ``device`` covers every file."""
    wavs = [_mono(w, f"file {k}") for k, w in enumerate(wavs)]
    if not wavs:
        raise ValueError("wavs is empty")
    srs = [int(srs)] * len(wavs) if isinstance(srs, (int, np.integer)) else [int(s) for s in srs]
    if len(srs) != len(wavs):
        raise ValueError(f"{len(srs)} sample rates for {len(wavs)} files")
    params = [slicer_params(s, db_thresh, min_len) for s in srs]
    n = [int(w.shape[0]) for w in wavs]
    dev = torch.device(device)
    x = torch.zeros((len(wavs), max(max(n), 1)), dtype=torch.float32, device=dev)
    for j, w in enumerate(wavs):
        x[j, :n[j]] = torch.as_tensor(w).to(dev)
    rms, frames = rms_frames(x, torch.tensor(n, dtype=torch.int64), srs)
    host = rms.cpu().numpy()
    return [slice_from_rms(host[j, :frames[j]], n[j], params[j]) for j in range(len(wavs))]


def cut(wav: Wave, sr: int, db_thresh: float = -30, min_len: int = 5000, device: Union[str, torch.device] = "cuda") -> Chunks:
    """``slicer.cut`` (slicer.py:120-128) on 1-D float32 samples at ``sr`` instead of a file path."""
    return cut_batch([wav], [sr], db_thresh, min_len, device)[0]


def chunks2audio(wav: Wave, chunks: Chunks) -> List[Tuple[bool, np.ndarray]]:
    """``slicer.chunks2audio`` (slicer.py:131-142) on 1-D float32 samples: [(is_silence, float32 samples), ...] in chunk order,
    leaving out chunks whose split_time starts where it ends.  The list goes straight to ``convert.convert_slices``."""
    wav = _mono(wav, "wav")
    audio = wav.cpu().numpy() if isinstance(wav, torch.Tensor) else wav
    result = []
    for v in dict(chunks).values():
        tag = v["split_time"].split(",")
        if tag[0] != tag[1]:
            result.append((v["slice"], audio[int(tag[0]):int(tag[1])]))
    return result
