"""The silence slicer and the whole-CLI call on the GPU against what they replace.

    python scripts/slicer_bench.py [--files 8] [--minutes 10] [--steps 30] [--reps 3] [--out results/slicer_bench.json]

1. ``slicer.cut_batch`` over ``--files`` files of ``--minutes`` minutes at 44.1 kHz (voice-like bursts between silences,
   seeded), against the numpy restatement of librosa's RMS (``oracle/slicer_oracle.py``) plus the same host decision logic on
   the host cores: wall time of the whole call (host samples in, chunk dicts out), and CUDA events around ``rms_frames`` alone
   with the samples already on the device.  The chunk dicts of both paths are compared.
2. ``convert.convert_files`` with 2 files x 3 voices (20 s and 13 s files at 44.1 kHz with silences, 3 s voices) against one
   ``convert.convert_slices`` call per (file, voice) pair with the same x_T: audio-seconds per second (input seconds of every
   pair over wall time), and the padding fraction of the ragged batches (padded frames over all frames the denoiser ran).
   Full-size models with synthetic weights, UniPC-``--steps``.  Modes alternate over ``--reps`` timed passes after one warm-up
   pass each; the outputs of the two modes are compared (bit for bit, and ||a - b|| / ||b|| per pair).

Reported with the card's name and power limit.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from convert_bench import PRE_CFG, card  # noqa: E402
from ns2vc_b200 import api, convert, slicer  # noqa: E402
from ns2vc_b200.arch import ns2vc_denoiser_config  # noqa: E402
from ns2vc_b200.content import ContentVec  # noqa: E402
from ns2vc_b200.pre_model import Pre_model  # noqa: E402
from ns2vc_b200.synth import make_contentvec_state_dict, make_pre_state_dict, make_state_dict, make_vocos_state_dict  # noqa: E402
from ns2vc_b200.unet import UNet1DConditionModel  # noqa: E402
from ns2vc_b200.vocoder import Vocos  # noqa: E402
from oracle import slicer_oracle  # noqa: E402

SR = 44100


def bursts(g: np.random.Generator, seconds: float, sr: int = SR) -> np.ndarray:
    """Voice-like bursts of 0.5-8 s (tone plus noise) separated by 0.1-2 s of low noise, float32."""
    out, n = [], int(seconds * sr)
    total = 0
    while total < n:
        v, s = int(g.uniform(0.5, 8.0) * sr), int(g.uniform(0.1, 2.0) * sr)
        t = np.arange(v) / sr
        out.append(0.3 * np.sin(2 * np.pi * g.uniform(100, 300) * t) + 0.05 * g.standard_normal(v))
        out.append(1e-4 * g.standard_normal(s))
        total += v + s
    return np.concatenate(out)[:n].astype(np.float32)


def padding_fraction(T_lists, max_batch):
    """Padded frames over all frames the denoiser runs, for each list of frame counts batched by ``api.batch_plan``."""
    pad = tot = 0
    for T in T_lists:
        for idx in api.batch_plan(T, max_batch):
            m = max(T[i] for i in idx)
            pad += sum(m - T[i] for i in idx)
            tot += m * len(idx)
    return pad / tot if tot else 0.0


def bench_cut(args, res):
    g = np.random.default_rng(args.seed)
    files = [bursts(g, args.minutes * 60) for _ in range(args.files)]
    srs = [SR] * len(files)
    slicer.cut_batch(files[:1], srs[:1], -40)                  # warm-up: library load, first launch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    got = slicer.cut_batch(files, srs, -40)
    gpu_s = time.perf_counter() - t0
    hop, win = slicer.hop_win(SR)
    p = slicer.slicer_params(SR, -40, 5000)
    t0 = time.perf_counter()
    want = [slicer.slice_from_rms(slicer_oracle.rms(y, win, hop)[0], len(y), p) for y in files]
    cpu_s = time.perf_counter() - t0
    n = [len(y) for y in files]
    x = torch.zeros((len(files), max(n)), device="cuda")
    for j, y in enumerate(files):
        x[j, :n[j]] = torch.from_numpy(y).cuda()
    lengths = torch.tensor(n)
    slicer.rms_frames(x, lengths, SR)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(args.reps):
        slicer.rms_frames(x, lengths, SR)
    e.record()
    torch.cuda.synchronize()
    audio_s = sum(n) / SR
    res["cut_batch"] = dict(files=args.files, minutes=args.minutes, audio_seconds=audio_s, gpu_call_s=gpu_s, cpu_numpy_s=cpu_s,
                            speedup=cpu_s / gpu_s, rms_frames_ms=s.elapsed_time(e) / args.reps, chunks_equal=got == want,
                            host_cores=os.cpu_count())
    print(json.dumps(res["cut_batch"]), flush=True)


def bench_convert(args, res):
    dev = torch.device("cuda")
    cfg = ns2vc_denoiser_config()
    unet = UNet1DConditionModel(in_channels=cfg.in_channels, out_channels=cfg.out_channels, block_out_channels=cfg.block_out_channels,
                                layers_per_block=list(cfg.layers_per_block), norm_num_groups=cfg.norm_num_groups,
                                cross_attention_dim=cfg.cross_attention_dim, attention_head_dim=cfg.num_heads,
                                addition_embed_type=cfg.addition_embed_type, addition_embed_type_num_heads=cfg.addition_embed_type_num_heads,
                                resnet_time_scale_shift=cfg.resnet_time_scale_shift)
    unet.load_state_dict(make_state_dict(cfg, 0))
    unet = unet.to(dev).eval()
    cv = ContentVec.from_state_dict(make_contentvec_state_dict(0, "trained_like")).to(dev)
    pre = Pre_model(PRE_CFG)
    pre.load_state_dict(make_pre_state_dict(PRE_CFG, 0))
    pre = pre.to(dev).eval()
    voc = Vocos.from_state_dict(make_vocos_state_dict(0, "trained_like")).to(dev)
    models = (cv, pre, unet, voc)
    g = np.random.default_rng(args.seed + 1)
    files = [(bursts(g, 20.0), SR), (bursts(g, 13.0), SR)]
    voices = [(bursts(g, 3.0), SR) for _ in range(3)]
    audio_data = [slicer.chunks2audio(w, c) for (w, _), c in zip(files, slicer.cut_batch([w for w, _ in files], SR, -40))]
    subs = [convert._plan_slices(a, SR, 0.5, 0, 0) for a in audio_data]
    sub_T = [[convert.frame_plan(len(s), SR)["T"] for s in ss] for ss in subs]
    mels = convert.voice_mels(voices, dev)
    torch.manual_seed(args.seed)
    x_T = convert._files_x_T(sub_T, len(voices), dev)

    def files_mode():
        return convert.convert_files(*models, files, voices, steps=args.steps, max_batch=args.max_batch, x_T=x_T)

    def pairs_mode():
        return [[convert.convert_slices(*models, audio_data[f], SR, mels[v], steps=args.steps, max_batch=args.max_batch, x_T=x_T[f][v])
                 for v in range(len(voices))] for f in range(len(files))]

    modes = dict(convert_files=files_mode, per_pair=pairs_mode)
    outs, times = {}, {k: [] for k in modes}
    for k, fn in modes.items():
        outs[k] = fn()
    torch.cuda.synchronize()
    for _ in range(args.reps):
        for k, fn in modes.items():
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
    audio_s = len(voices) * sum(len(w) for w, _ in files) / SR
    all_items = [T for Ts in sub_T for _ in voices for T in Ts]
    res["convert_files"] = dict(
        files=len(files), voices=len(voices), sub_slices=[len(s) for s in subs], steps=args.steps, max_batch=args.max_batch,
        audio_seconds=audio_s, bit_identical=all(np.array_equal(a, b) for ra, rb in zip(outs["convert_files"], outs["per_pair"])
                                                 for a, b in zip(ra, rb)),
        max_rel_diff=max(float(np.linalg.norm(a - b) / np.linalg.norm(b)) for ra, rb in zip(outs["convert_files"], outs["per_pair"])
                         for a, b in zip(ra, rb)),
        **{f"{k}_s": min(v) for k, v in times.items()}, **{f"{k}_audio_s_per_s": audio_s / min(v) for k, v in times.items()},
        padding_convert_files=padding_fraction([all_items], args.max_batch),
        padding_per_pair=padding_fraction([Ts for Ts in sub_T for _ in voices], args.max_batch), spread={k: v for k, v in times.items()})
    print(json.dumps(res["convert_files"]), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=8)
    ap.add_argument("--minutes", type=float, default=10.0)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--max-batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--skip-convert", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("slicer_bench needs a CUDA device")
    res = dict(card=card(), torch=torch.__version__)
    print(res["card"], flush=True)
    bench_cut(args, res)
    if not args.skip_convert:
        bench_convert(args, res)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
