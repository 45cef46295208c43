"""Corpus preprocessing on the GPU: the reference's ``preprocess.py`` (``process_one``, ``preprocess.py:26-60``), which turns a
corpus of audio files into the training data ``NS2VCDataset`` reads (``dataset.py:73-92``).

Per file, ``process_one`` does:

1. ``wav`` [C, N] at ``sr``; if C > 1, ``wav.mean(dim=0, keepdim=True)``;
2. ``wav16k = Resample(sr, 16000)(wav)`` and ``wav24k = Resample(sr, 24000)(wav)``, both from the ORIGINAL rate (inference,
   ``convert.encode_front``, reaches 16 kHz through 24 kHz instead, so ``convert.frame_plan`` is not this plan);
3. writes ``wav24k`` as a float32 WAV at 24 kHz under ``filename.replace(in_dir, in_dir + "_processed")`` with ``.mp3`` /
   ``.flac`` renamed to ``.wav``;
4. ``<name>.soft.pt``: ``get_hubert_content(hmodel, wav16k[0])``, the ContentVec units [1, 256, U];
5. ``<name>.f0.npy``: WORLD's DIO + StoneMask f0, rounded to 0.1 Hz and ``resize_f0``'d to ``N24 // 256`` frames;
6. ``<name>`` with ``.wav`` -> ``.spec.pt``: ``log(clip(MelSpectrogram(24000, 1024, 256, 100, center, power=1)(wav24k), 1e-7))``
   [1, 100, N24 // 256 + 1].

``preprocess_utterances`` runs steps 1, 2, 4 and 6 for a list of ``(wav, sr)`` items in ragged batches on the GPU (one batch per
rate group at a time; every stage takes per-row lengths, so each record equals its file processed alone); ``save`` writes the
four files of steps 3-6, with f0 computed on the host (WORLD is third-party code); ``dataset_item`` restates the loader's
alignment.  Finding and decoding the files (wav, mp3, flac) stays with the caller, as for ``convert.convert_files``.
"""
from __future__ import annotations

import math
import os
import struct
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist

from . import frontend, shard
from .api import batch_plan
from .content import CONV_LAYERS, MIN_SAMPLES, num_frames

TARGET_SR = 24000        # config data.sampling_rate: the rate of wav24k, the mel and f0
HOP = 256                # config data.hop_length
CONTENT_SR = 16000       # ContentVec's input rate
N_MELS = frontend.N_MELS

Record = Dict[str, object]


def length_plan(n: int, sr: int) -> Dict[str, int]:
    """Host lengths of one file of n samples at ``sr``: ``n16`` / ``n24`` samples resampled from ``sr`` directly, ContentVec
    frames ``units`` (of the 16 kHz signal), ``frames = n24 // 256`` (the f0 length, and the loader's ``lmin``) and the mel's
    ``spec = frames + 1`` frames (center=True)."""
    n16 = frontend.resample_out_length(sr, CONTENT_SR, n)
    n24 = frontend.resample_out_length(sr, TARGET_SR, n)
    return dict(n=int(n), n16=n16, n24=n24, units=num_frames(n16), frames=n24 // HOP, spec=n24 // HOP + 1)


def content_flops(n16: int, cfg: Dict[str, int]) -> int:
    """Algorithmic FLOPs of ``ContentVec.extract`` (configuration ``cfg``) on one row of ``n16`` samples at 16 kHz: the seven
    convs, the three projections, the positional conv and the transformer layers with their attention.  The cost of a batch
    when ``preprocess_utterances`` shares batches over ranks: the encoder is most of the work, the resamplers and the mel a
    few percent."""
    n, cin, flops = int(n16), 1, 0
    for k, s in CONV_LAYERS:
        n = 0 if n < k else (n - k) // s + 1
        flops += 2 * k * cin * cfg["conv_dim"] * n
        cin = cfg["conv_dim"]
    D, F = cfg["embed_dim"], cfg["ffn_dim"]
    flops += 2 * n * (cfg["conv_dim"] * D + D * (D // cfg["pos_conv_groups"]) * cfg["pos_conv_kernel"] + D * cfg["final_dim"])
    return flops + cfg["num_layers"] * (2 * n * (4 * D * D + 2 * D * F) + 4 * n * n * D)


def _check_items(items: Sequence[Tuple[torch.Tensor, int]]) -> List[Dict[str, int]]:
    """Host-side argument checks of ``preprocess_utterances``; returns each item's ``length_plan`` with its rate."""
    if len(items) == 0:
        raise ValueError("items is empty")
    plans = []
    for k, it in enumerate(items):
        if not isinstance(it, (tuple, list)) or len(it) != 2:
            raise ValueError(f"item {k}: expected a (wav, sr) pair")
        wav, sr = it
        if not torch.is_tensor(wav) or wav.dim() not in (1, 2) or not wav.dtype.is_floating_point:
            raise ValueError(f"item {k}: expected a floating-point wav [N] or [channels, N], got "
                             f"{tuple(wav.shape) if torch.is_tensor(wav) else type(wav).__name__}"
                             f"{' ' + str(wav.dtype) if torch.is_tensor(wav) else ''}")
        if wav.dim() == 2 and wav.shape[0] < 1:
            raise ValueError(f"item {k}: wav has no channels")
        if isinstance(sr, bool) or not isinstance(sr, (int, np.integer)) or int(sr) <= 0:
            raise ValueError(f"item {k}: bad sample rate {sr!r} (a positive integer in Hz)")
        sr = int(sr)
        for new in (CONTENT_SR, TARGET_SR):
            try:
                frontend.resample_check(sr, new)
            except ValueError as e:
                raise ValueError(f"item {k}: {sr} -> {new} Hz cannot be resampled here: {e}") from None
        p = length_plan(int(wav.shape[-1]), sr)
        if p["n16"] < MIN_SAMPLES:
            raise ValueError(f"item {k}: {p['n']} samples at {sr} Hz give {p['n16']} at 16 kHz; ContentVec needs at least {MIN_SAMPLES}")
        if p["frames"] < 1 or p["n24"] <= frontend.N_FFT // 2:
            raise ValueError(f"item {k}: {p['n']} samples at {sr} Hz give {p['n24']} at 24 kHz, zero frames of {HOP}")
        p["sr"] = sr
        plans.append(p)
    return plans


def _mono(wav: torch.Tensor, dev: torch.device) -> torch.Tensor:
    """Step 1 on the device: [N] as it is, [C, N] averaged over its channels (``wav.mean(dim=0)`` of the fp32 samples)."""
    x = wav.to(dev, torch.float32)
    return x if x.dim() == 1 else x.mean(dim=0)


@torch.no_grad()
def _run_batch(content_model, items, plans: Sequence[Dict[str, int]], idx: Sequence[int], dev: torch.device) -> List[Record]:
    """One ragged batch of items of one rate: mono mix, both resamples from that rate, one ContentVec run over the 16 kHz rows
    and one log-mel over the 24 kHz rows; every stage takes the rows' own lengths."""
    sr = plans[idx[0]]["sr"]
    n = [plans[i]["n"] for i in idx]
    n16, n24 = [plans[i]["n16"] for i in idx], [plans[i]["n24"] for i in idx]
    x = torch.zeros((len(idx), max(n)), dtype=torch.float32, device=dev)
    for j, i in enumerate(idx):
        x[j, :n[j]] = _mono(items[i][0], dev)
    lens = torch.tensor(n, dtype=torch.int64)
    w16, _ = frontend.resample(x, sr, CONTENT_SR, lens)
    w24, _ = frontend.resample(x, sr, TARGET_SR, lens)
    units, _ = content_model.extract(w16, torch.tensor(n16, dtype=torch.int64))
    mel, _ = frontend.log_mel_spectrogram(w24, TARGET_SR, torch.tensor(n24, dtype=torch.int64))
    out = []
    for j, i in enumerate(idx):
        p = plans[i]
        out.append(dict(wav24k=w24[j, None, :p["n24"]].clone(), soft=units[j, :p["units"]].t()[None].contiguous(),
                        spec=mel[j, None, :, :p["spec"]].clone(), frames=p["frames"]))
    return out


def _sizes(p: Dict[str, int], D: int) -> Tuple[int, int, int]:
    return p["n24"], D * p["units"], N_MELS * p["spec"]


def _pack(r: Record) -> torch.Tensor:
    return torch.cat([r["wav24k"].reshape(-1), r["soft"].reshape(-1), r["spec"].reshape(-1)])


def _unpack(flat: torch.Tensor, p: Dict[str, int], D: int) -> Record:
    a, b, c = _sizes(p, D)
    return dict(wav24k=flat[:a].view(1, a).clone(), soft=flat[a:a + b].view(1, D, p["units"]).clone(),
                spec=flat[a + b:a + b + c].view(1, N_MELS, p["spec"]).clone(), frames=p["frames"])


@torch.no_grad()
def preprocess_utterances(content_model, items: Sequence[Tuple[torch.Tensor, int]], max_batch: int = 8,
                          group: Optional[dist.ProcessGroup] = None) -> List[Record]:
    """Steps 1, 2, 4 and 6 of the reference's ``process_one`` for each ``(wav, sr)`` item: ``wav`` a float CPU or CUDA tensor
    [N] or [channels, N] (channels are averaged), ``sr`` its integer rate.  Returns one record per item, in input order, on
    the content model's device: ``wav24k`` [1, N24] (``Resample(sr, 24000)``), ``soft`` [1, final_dim, U] (ContentVec units of
    ``Resample(sr, 16000)``, U = ``content.num_frames(N16)``), ``spec`` [1, 100, N24 // 256 + 1] (the log-mel of ``wav24k``)
    and ``frames`` = N24 // 256.  Each record equals that file processed alone.

    Every argument is checked on the host before any device work: a bad rank, dtype or rate, a rate that ``frontend.resample``
    refuses to or from, fewer than ``content.MIN_SAMPLES`` samples at 16 kHz or no frame at 24 kHz raise ValueError naming the
    item.  Items are grouped by rate (one resampler pair per rate) and run in longest-first ragged batches of at most
    ``max_batch`` rows (``api.batch_plan``) per group.

    With a process ``group`` of more than one rank (one process per GPU, every rank making the same call with its model on its
    own device), whole batches go to ranks by ``shard.assign_batches`` at the content encoder's cost (``content_flops``), run
    under ``shard.run_sharded`` and are all-gathered once; every rank returns the one-GPU result."""
    if int(max_batch) < 1:
        raise ValueError("max_batch must be >= 1")
    plans = _check_items(items)
    dev = next(content_model.parameters()).device
    if dev.type != "cuda":
        raise RuntimeError("preprocess_utterances needs the content model on a CUDA device (no CPU path)")
    world = dist.get_world_size(group) if group is not None else 1
    cap = min(int(max_batch), max(1, math.ceil(len(items) / world)))
    batches: List[List[int]] = []
    for sr in dict.fromkeys(p["sr"] for p in plans):
        idx = [i for i, p in enumerate(plans) if p["sr"] == sr]
        batches += [[idx[j] for j in b] for b in batch_plan([plans[i]["n"] for i in idx], cap)]
    if world == 1:
        out: List[Optional[Record]] = [None] * len(items)
        for b in batches:
            for i, r in zip(b, _run_batch(content_model, items, plans, b, dev)):
                out[i] = r
        return out
    D = content_model.cfg["final_dim"]
    cost = [len(b) * content_flops(max(plans[i]["n16"] for i in b), content_model.cfg) for b in batches]
    plan = shard.assign_batches(batches, cost, world)
    flat = shard.run_sharded(lambda b: [_pack(r) for r in _run_batch(content_model, items, plans, b, dev)], plan,
                             [sum(_sizes(p, D)) for p in plans], group, dev)
    return [_unpack(f.to(dev), p, D) for f, p in zip(flat, plans)]


# ------------------------------------------------------------------------------------------------------------- the loader's view
def dataset_item(record: Record) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """``NS2VCDataset.get_audio``'s alignment (``dataset.py:73-92``) on a record: ``c = repeat_expand_2d(soft[0], frames)``
    (the f0 length), every stream cut to ``lmin = min(c, spec)`` frames (= ``frames``), with the loader's two asserts (c and
    spec within 3 frames, the audio within 3 hops of ``lmin * 256``).  Returns ``(c [256, lmin], spec [100, lmin],
    audio [1, lmin * 256])``.

    ``(c, spec)`` with a prompt mel ``refer`` [100, S] is exactly an item of ``loss.utterance_losses``, so held-out raw audio
    is scored straight from its records::

        recs = preprocess_utterances(cv, [(wav, sr), ...])
        items = [(c, spec, refer) for c, spec, _ in map(dataset_item, recs)]
        utterance_losses(pre_model, unet, items, ...)
    """
    frames = int(record["frames"])
    c = frontend.repeat_expand_2d(record["soft"][0], frames)
    spec = record["spec"][0]
    audio = record["wav24k"]
    lmin = min(c.shape[-1], spec.shape[-1])
    assert abs(c.shape[-1] - spec.shape[-1]) < 3, (c.shape[-1], spec.shape[-1])
    assert abs(audio.shape[1] - lmin * HOP) < 3 * HOP, (audio.shape[1], lmin)
    return c[:, :lmin], spec[:, :lmin], audio[:, :lmin * HOP]


# ------------------------------------------------------------------------------------------------------------------ the files
def output_paths(filename: str, in_dir: str) -> Dict[str, str]:
    """The four names ``process_one`` writes for ``filename``, with its string replacements as they are (each ``replace``
    acts on every occurrence, so a directory named ``x.wav`` becomes ``x.spec.pt`` in the spec's path, as in the reference)."""
    if not in_dir:
        raise ValueError("in_dir is empty: str.replace('', ...) would insert '_processed' between every character")
    wav = filename.replace(in_dir, in_dir + "_processed").replace(".mp3", ".wav").replace(".flac", ".wav")
    return dict(wav=wav, soft=wav + ".soft.pt", f0=wav + ".f0.npy", spec=wav.replace(".wav", ".spec.pt"))


def resize_f0(x, target_len: int) -> np.ndarray:
    """Reference ``utils.resize_f0`` (``utils.py:175-180``): values below 0.001 (unvoiced) become NaN, linear interpolation
    to ``target_len`` points, NaN back to 0."""
    source = np.array(x, dtype=np.float64)
    source[source < 0.001] = np.nan
    target = np.interp(np.arange(0, len(source) * target_len, len(source)) / target_len, np.arange(0, len(source)), source)
    return np.nan_to_num(target)


def compute_f0_dio(wav_numpy: np.ndarray, sampling_rate: int = TARGET_SR, hop_length: int = HOP) -> np.ndarray:
    """The f0 of reference ``utils.compute_f0_dio`` (``utils.py:182-195``) before its ``resize_f0``: pyworld's ``dio``
    (f0_ceil 800 Hz, one frame per hop) refined by ``stonemask``, rounded to 0.1 Hz.  Runs on the host."""
    import pyworld
    x = wav_numpy.astype(np.double)
    f0, t = pyworld.dio(x, fs=sampling_rate, f0_ceil=800, frame_period=1000 * hop_length / sampling_rate)
    f0 = pyworld.stonemask(x, f0, t, sampling_rate)
    for index, pitch in enumerate(f0):
        f0[index] = round(pitch, 1)
    return f0


def _default_f0_fn() -> Callable[[np.ndarray], np.ndarray]:
    try:
        import pyworld  # noqa: F401
    except ImportError as e:
        raise ImportError("save's default f0_fn is WORLD's DIO, which needs the pyworld package: install pyworld or pass "
                          "f0_fn") from e
    return compute_f0_dio


def write_wav_float32(path: str, samples: np.ndarray, sample_rate: int = TARGET_SR) -> None:
    """A mono IEEE-float (format 3) 32-bit WAV: RIFF header, an 18-byte fmt chunk, the fact chunk non-PCM data carries, data."""
    data = np.ascontiguousarray(samples, dtype="<f4").reshape(-1).tobytes()
    n = len(data) // 4
    fmt = struct.pack("<HHIIHHH", 3, 1, int(sample_rate), int(sample_rate) * 4, 4, 32, 0)
    body = (b"WAVE" + b"fmt " + struct.pack("<I", len(fmt)) + fmt + b"fact" + struct.pack("<II", 4, n)
            + b"data" + struct.pack("<I", len(data)) + data)
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", len(body)) + body)


def save(record: Record, filename: str, in_dir: str, f0_fn: Optional[Callable[[np.ndarray], np.ndarray]] = None) -> Dict[str, str]:
    """Writes a record as ``process_one`` writes file ``filename`` of the corpus under ``in_dir`` (``output_paths``), and returns
    the four paths: the 24 kHz mono float32 WAV, ``.soft.pt`` ([1, 256, U] fp32), ``.f0.npy`` (``resize_f0(f0_fn(wav24k),
    frames)``, float64) and ``.spec.pt`` ([1, 100, frames + 1] fp32); the directory is created if needed.

    ``f0_fn(wav24k [N24] float32 numpy) -> f0`` runs on the host and defaults to ``compute_f0_dio``; without pyworld that
    default raises ImportError before anything is written, and so does an f0 that does not resize to ``frames`` entries."""
    fn = f0_fn if f0_fn is not None else _default_f0_fn()
    paths = output_paths(filename, in_dir)
    wav = record["wav24k"].detach().to("cpu", torch.float32).reshape(-1).numpy()
    frames = int(record["frames"])
    f0_raw = np.asarray(fn(wav))
    if f0_raw.ndim != 1 or f0_raw.shape[0] < 1:
        raise ValueError(f"f0_fn returned an array of shape {f0_raw.shape}; expected a non-empty 1-D f0")
    f0 = resize_f0(f0_raw, frames)
    if f0.shape != (frames,):
        raise ValueError(f"f0 of {f0.shape} for {frames} frames")
    d = os.path.dirname(paths["wav"])
    if d:
        os.makedirs(d, exist_ok=True)
    write_wav_float32(paths["wav"], wav)
    torch.save(record["soft"].detach().to("cpu", torch.float32).contiguous().clone(), paths["soft"])
    np.save(paths["f0"], f0)
    torch.save(record["spec"].detach().to("cpu", torch.float32).contiguous().clone(), paths["spec"])
    return paths
