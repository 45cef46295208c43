"""Time ``frontend.log_mel_spectrogram`` on the GPU (CUDA events, after warm-up) and the reference's host recipe next to it
(torchaudio on the CPU, one prompt at a time with a fresh Resample per call, as inference/infer_tool.py:170-181 runs it).

    python scripts/frontend_bench.py [--iters 50] [--out results/frontend_bench.json]

Prints the card's name and power limit with the numbers.  Shapes: B = 1, 8, 64 prompts of 3 s and 10 s at 24 and 44.1 kHz
(ragged: lengths uniform in [0.6, 1] of the row).  Needs a CUDA device; torchaudio is optional (host column left out without it).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ns2vc_b200 import frontend  # noqa: E402


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable: {e}"


def gpu_ms(wav, sr, lens, iters):
    for _ in range(5):
        frontend.log_mel_spectrogram(wav, sr, lens)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        frontend.log_mel_spectrogram(wav, sr, lens)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def host_ms(wav, sr, lens, reps=3):
    import torchaudio
    best = float("inf")
    for _ in range(reps):
        t0 = time.perf_counter()
        for i in range(wav.shape[0]):
            x = wav[i:i + 1, :int(lens[i])]
            x24 = torchaudio.transforms.Resample(sr, 24000)(x)
            spec = torchaudio.transforms.MelSpectrogram(sample_rate=24000, n_fft=1024, hop_length=256, n_mels=100, center=True, power=1)(x24)
            torch.log(torch.clip(spec, min=1e-7))
        best = min(best, time.perf_counter() - t0)
    return best * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "frontend_bench needs a CUDA device"
    try:
        import torchaudio  # noqa: F401
        have_ta = True
    except ImportError:
        have_ta = False
    info = card()
    print(f"card: {info}; torch threads {torch.get_num_threads()}")
    rows = []
    for sr in (24000, 44100):
        for sec in (3, 10):
            for B in (1, 8, 64):
                g = torch.Generator().manual_seed(B * 100 + sec)
                N = sr * sec
                wav = torch.randn((B, N), generator=g) * 0.1
                lens = (N * (0.6 + 0.4 * torch.rand(B, generator=g))).long()
                lens[0] = N
                wg, lg = wav.cuda(), lens.cuda()
                ms = gpu_ms(wg, sr, lg, args.iters)
                r = dict(sr=sr, seconds=sec, B=B, gpu_ms=round(ms, 4))
                if have_ta and B <= 8:
                    r["host_ms"] = round(host_ms(wav, sr, lens), 3)
                rows.append(r)
                print(json.dumps(r), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
