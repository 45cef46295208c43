"""Throughput of corpus preprocessing (``preprocess.preprocess_utterances``: mono mix, both resamples, ContentVec units and the
log-mel of each file) on a synthetic corpus, with ContentVec's full configuration and synthetic ``trained_like`` weights.

    python scripts/preprocess_bench.py [--iters 3] [--warmup 1] [--out results/preprocess_bench.json]

The corpus: 64 files of 1-15 s (uniform, seed 0) at 16 / 22.05 / 44.1 / 48 kHz in turn, every fourth one stereo.  Reported:
audio-seconds per second at ``max_batch`` 1 and 8, and the same corpus through the reference's per-file path as a stand-in:
torchaudio's ``Resample`` and ``MelSpectrogram`` on the CPU, as ``process_one`` runs them, and the content oracle
(``oracle/content_oracle.py``, eager fp32 on the GPU, TF32 off) in place of fairseq's HubertModel, which is absent: NOT
fairseq.  f0 (pyworld's DIO on the host) is left out of every number, and so are file decoding and writing.

Timing: CUDA events after ``--warmup`` untimed passes, the mean of ``--iters`` passes over the whole corpus (the stand-in runs
once).  Prints the card's name and power limit with the numbers.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ns2vc_b200 import preprocess  # noqa: E402
from ns2vc_b200.content import ContentVec  # noqa: E402
from ns2vc_b200.synth import make_contentvec_state_dict  # noqa: E402
from scripts.ragged_bench import card  # noqa: E402

RATES = (16000, 22050, 44100, 48000)


def corpus(n_files: int = 64, seed: int = 0):
    g = torch.Generator().manual_seed(seed)
    items = []
    for k in range(n_files):
        sr = RATES[k % len(RATES)]
        n = int(float(1 + 14 * torch.rand(1, generator=g)) * sr)
        ch = 2 if k % 4 == 3 else 1
        x = 0.1 * torch.randn((ch, n), generator=g)
        items.append((x[0] if ch == 1 else x, sr))
    return items


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3 / iters


def stand_in(items, sd, heads):
    """process_one's arithmetic per file: CPU torchaudio resamples and mel, the content oracle in eager fp32 on the GPU"""
    import torchaudio.transforms as T
    from oracle import content_oracle
    sd = {k: v.cuda() for k, v in sd.items()}
    mel = T.MelSpectrogram(sample_rate=24000, n_fft=1024, hop_length=256, n_mels=100, center=True, power=1)
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for x, sr in items:
            wav = x[None] if x.dim() == 1 else x.mean(dim=0, keepdim=True)
            w16, w24 = T.Resample(sr, 16000)(wav), T.Resample(sr, 24000)(wav)
            soft = content_oracle.extract(sd, w16.cuda(), heads, dtype=torch.float32).transpose(1, 2).cpu()
            spec = torch.log(torch.clip(mel(w24), min=1e-7))
        torch.cuda.synchronize()
        return time.perf_counter() - t0, soft.shape, spec.shape
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("preprocess_bench needs a CUDA device")
    torch.set_grad_enabled(False)
    sd = make_contentvec_state_dict(0, "trained_like")
    m = ContentVec.from_state_dict(sd).cuda().eval()
    items = corpus()
    audio_s = sum(x.shape[-1] / sr for x, sr in items)
    res = {"card": card(), "files": len(items), "audio_seconds": round(audio_s, 1), "f0": "not included (host pyworld)",
           "preprocess_utterances": {}, "stand_in_torchaudio_cpu_plus_oracle_fp32": "not measured"}
    print("card", res["card"], "corpus", len(items), "files,", res["audio_seconds"], "s", flush=True)
    for mb in (1, 8):
        sec = timed(lambda: preprocess.preprocess_utterances(m, items, max_batch=mb), args.iters, args.warmup)
        row = {"s": round(sec, 3), "audio_seconds_per_second": round(audio_s / sec, 1)}
        res["preprocess_utterances"][f"max_batch={mb}"] = row
        print("preprocess_utterances", mb, row, flush=True)
    try:
        sec, _, _ = stand_in(items, sd, 12)
        res["stand_in_torchaudio_cpu_plus_oracle_fp32"] = {
            "what": "torchaudio CPU Resample x2 + MelSpectrogram, content oracle eager fp32 on the GPU, per file (NOT fairseq)",
            "cpu_threads": torch.get_num_threads(), "s": round(sec, 3), "audio_seconds_per_second": round(audio_s / sec, 1)}
        print("stand-in", res["stand_in_torchaudio_cpu_plus_oracle_fp32"], flush=True)
    except ImportError as e:
        res["stand_in_torchaudio_cpu_plus_oracle_fp32"] = f"not measured: {e}"
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
