"""Throughput of the vocoder (``vocoder.Vocos.decode``, vocos-mel-24khz shapes with synthetic ``trained_like`` weights).

    python scripts/vocoder_bench.py [--iters 20] [--warmup 3] [--out results/vocoder_bench.json]

(a) ``decode`` at B=1, T=256 / 1024 and B=8, T=1024: ms per call and audio-seconds per second (frames x 256 / 24 kHz).
(b) the 16-slice list of scripts/ragged_bench.py (lengths uniform in [150, 1000] frames, seed 0): one ``decode`` per slice at
    B = 1 against ``api.decode_utterances(max_batch=8)``.
(c) the same inputs through ``oracle/vocos_oracle.py``'s fp32 path run eagerly on the GPU, a stand-in for the ``vocos``
    package's eager PyTorch (not the package itself): its TF32 flags and the worst err/tol of our output against it
    (rtol 1e-3, atol 1e-4 rms) are recorded, and the same err/tol with cuDNN's TF32 turned off.

Timing: CUDA events around the timed calls after ``--warmup`` untimed passes, the mean of ``--iters`` calls.  Work per frame
from shapes: embed 2 x 100 x 7 x 512, eight blocks 2 x (7 + 2 x 1536) x 512, head 2 x 512 x 1026 multiply-adds (about 27 MFLOP).
Prints the card's name and power limit with the numbers.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ns2vc_b200 import api  # noqa: E402
from ns2vc_b200.synth import make_vocos_state_dict  # noqa: E402
from ns2vc_b200.vocoder import Vocos  # noqa: E402
from oracle import vocos_oracle  # noqa: E402
from scripts.ragged_bench import card  # noqa: E402

FRAME_SECONDS = 256 / 24000
FLOP_PER_FRAME = 2 * (100 * 7 * 512 + 8 * (7 * 512 + 2 * 1536 * 512) + 512 * 1026)


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b) / 1e3 / iters


def worst_ratio(ours, theirs):
    """worst |ours - theirs| / (1e-3 |theirs| + 1e-4 rms(theirs)) over a list of waveforms"""
    return max(((a - r).abs() / (1e-3 * r.abs() + 1e-4 * r.pow(2).mean().sqrt())).max().item() for a, r in zip(ours, theirs))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vocoder_bench needs a CUDA device")
    sd = make_vocos_state_dict(0, "trained_like")
    m = Vocos.from_state_dict(sd).cuda().eval()
    res = {"card": card(), "decode": {}, "slices": {}, "oracle_fp32_eager": {}}
    torch.set_grad_enabled(False)
    g = torch.Generator().manual_seed(1)
    for B, T in ((1, 256), (1, 1024), (8, 1024)):
        mel = torch.randn((B, 100, T), generator=g).cuda()
        _, sec = timed(lambda: m.decode(mel), args.iters, args.warmup)
        row = {"ms": round(sec * 1e3, 3), "audio_seconds_per_second": round(B * T * FRAME_SECONDS / sec, 1),
               "tflops": round(B * T * FLOP_PER_FRAME / sec / 1e12, 1), "launches": m.launch_count()}
        res["decode"][f"B={B},T={T}"] = row
        print("decode", B, T, row, flush=True)

    gs = torch.Generator().manual_seed(0)
    lengths = torch.randint(150, 1001, (16,), generator=gs).tolist()
    latents = [torch.randn((100, t), generator=gs).cuda() for t in lengths]
    audio_s = sum(lengths) * FRAME_SECONDS
    modes = [("B=1", lambda: [m.decode(x[None])[0] for x in latents]),
             ("decode_utterances(max_batch=8)", lambda: api.decode_utterances(m, latents, max_batch=8))]
    ref = None
    for name, fn in modes:
        out, sec = timed(fn, max(1, args.iters // 4), args.warmup)
        row = {"ms": round(sec * 1e3, 3), "audio_seconds_per_second": round(audio_s / sec, 1)}
        if ref is None:
            ref = out
        else:
            row["speedup_vs_B1"] = round(res["slices"]["B=1"]["ms"] / row["ms"], 2)
            row["bit_identical_to_B1"] = sum(int(torch.equal(a, r)) for a, r in zip(out, ref))
        res["slices"][name] = row
        print("slices", name, row, flush=True)

    sd_dev = {k: v.cuda() for k, v in sd.items()}
    flags = {"matmul.allow_tf32": torch.backends.cuda.matmul.allow_tf32, "cudnn.allow_tf32": torch.backends.cudnn.allow_tf32}
    mel8 = torch.randn((8, 100, 1024), generator=g).cuda()
    for name, fn in (("B=1", lambda: [vocos_oracle.decode(sd_dev, x[None], dtype=torch.float32)[0] for x in latents]),
                     ("B=8,T=1024", lambda: vocos_oracle.decode(sd_dev, mel8, dtype=torch.float32))):
        out, sec = timed(fn, max(1, args.iters // 4), 1)
        row = {"ms": round(sec * 1e3, 3)}
        if name == "B=1":
            row["audio_seconds_per_second"] = round(audio_s / sec, 1)
            row["ours_vs_it_worst_err_over_tol"] = round(worst_ratio(ref, out), 3)
            # the default flags let cuDNN run the fp32 convs in TF32; the same comparison with TF32 off (untimed)
            cudnn_tf32 = torch.backends.cudnn.allow_tf32
            torch.backends.cudnn.allow_tf32 = False
            row["ours_vs_it_tf32_off_worst_err_over_tol"] = round(worst_ratio(ref, fn()), 3)
            torch.backends.cudnn.allow_tf32 = cudnn_tf32
        else:
            row["audio_seconds_per_second"] = round(8 * 1024 * FRAME_SECONDS / sec, 1)
        res["oracle_fp32_eager"][name] = row
        print("oracle fp32 eager", name, row, flush=True)
    res["oracle_fp32_eager"]["tf32_flags"] = flags
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
