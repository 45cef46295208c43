"""Throughput of waveform-to-waveform conversion: one file's slices converted one by one at B = 1, stage by stage (the reference
CLI's structure, infer.py:99-141), against ``convert.convert_utterances`` over ragged batches.

    python scripts/convert_bench.py [--slices 16] [--steps 30] [--max-batch 8] [--warmup 2] [--out results/convert_bench.json]

The slices are the lengths of ``scripts/ragged_bench.py`` (``--slices`` draws from [150, 1000] frames, seeded) turned into
44.1 kHz input lengths, each a synthetic voice-like signal, with one 3 s prompt mel.  Full-size models with synthetic weights:
ContentVec, the shipped condition encoders, the 66 M-parameter denoiser and the vocos-mel-24khz vocoder shapes; UniPC-30.
Both modes use the same x_T per slice.  CUDA events around the whole list after ``--warmup`` passes of each mode; the time per
stage is the sum of CUDA events around each stage call.  Reported: audio-seconds per second, the time per stage, the padding
fraction of the batched runs (padded frames over all frames the denoiser ran) and the worst batched-vs-alone audio error
||batched - alone|| / ||alone||, with the card's name and power limit.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
from collections import defaultdict

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ns2vc_b200 import api, convert, frontend  # noqa: E402
from ns2vc_b200.arch import ns2vc_denoiser_config  # noqa: E402
from ns2vc_b200.content import ContentVec  # noqa: E402
from ns2vc_b200.pre_model import Pre_model  # noqa: E402
from ns2vc_b200.synth import make_contentvec_state_dict, make_pre_state_dict, make_state_dict, make_vocos_state_dict  # noqa: E402
from ns2vc_b200.unet import UNet1DConditionModel  # noqa: E402
from ns2vc_b200.vocoder import Vocos  # noqa: E402

SR = 44100
PRE_CFG = {"phoneme_encoder": dict(in_channels=256, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2),
           "prompt_encoder": dict(in_channels=100, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2)}


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable: {e}"


class StageTimer:
    """CUDA events around every call of the wrapped stage functions; ``totals()`` synchronises and sums them per stage."""

    def __init__(self):
        self.events = defaultdict(list)

    def wrap(self, name, fn):
        def run(*a, **kw):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            out = fn(*a, **kw)
            e.record()
            self.events[name].append((s, e))
            return out
        return run

    def totals(self):
        torch.cuda.synchronize()
        out = {k: sum(s.elapsed_time(e) for s, e in v) / 1e3 for k, v in self.events.items()}
        self.events.clear()
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slices", type=int, default=16)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--max-batch", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("convert_bench needs a CUDA device")
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

    g = torch.Generator().manual_seed(args.seed)
    frames = torch.randint(150, 1001, (args.slices,), generator=g).tolist()
    wavs = []
    for t in frames:
        n = int(t * 256 * SR / 24000) + 100
        tt = torch.arange(n) / SR
        f0 = 100 + 200 * torch.rand(1, generator=g)
        wavs.append((0.3 * torch.sin(2 * torch.pi * f0 * tt) * (1 + 0.5 * torch.sin(2 * torch.pi * 3 * tt))
                     + 0.02 * torch.randn(n, generator=g)).float())
    pw = (0.2 * torch.randn(3 * 24000, generator=g)).float().to(dev)
    prompt = frontend.log_mel_spectrogram(pw, 24000)[0]
    plans = [convert.frame_plan(len(w), SR) for w in wavs]
    tl = [p["T"] for p in plans]
    x_T = [torch.randn((1, 100, t), generator=g).to(dev) for t in tl]
    wavs = [w.to(dev) for w in wavs]
    audio_s = sum(t * 256 for t in tl) / 24000

    timer = StageTimer()
    frontend.resample = timer.wrap("resample", frontend.resample)
    cv.extract = timer.wrap("content", cv.extract)
    pre.encode_voices = timer.wrap("encoders", pre.encode_voices)
    pre.infer_content = timer.wrap("encoders", pre.infer_content)
    convert.sample_latents = timer.wrap("sampler", convert.sample_latents)
    voc.decode = timer.wrap("vocoder", voc.decode)

    def one_by_one():
        return [convert.convert_batch(*models, [w], SR, [prompt], [x], "unipc", args.steps)["audio"][0] for w, x in zip(wavs, x_T)]

    def batched():
        return convert.convert_utterances(*models, wavs, SR, prompt, steps=args.steps, max_batch=args.max_batch, x_T=x_T)

    res = {}
    outs = {}
    for name, fn in (("one_by_one", one_by_one), ("batched", batched)):
        for _ in range(args.warmup):
            fn()
        timer.totals()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        outs[name] = fn()
        b.record()
        torch.cuda.synchronize()
        sec = a.elapsed_time(b) / 1e3
        res[name] = dict(seconds=sec, audio_s_per_s=audio_s / sec, stages_s=timer.totals())
    padded = sum(len(idx) * max(tl[i] for i in idx) for idx in api.batch_plan([len(w) for w in wavs], args.max_batch))
    worst = max(((a.double() - b.double()).norm() / b.double().norm()).item() for a, b in zip(outs["batched"], outs["one_by_one"]))
    report = dict(card=card(), slices=args.slices, frames=frames, audio_seconds=audio_s, steps=args.steps, method="unipc",
                  max_batch=args.max_batch, padding_fraction=1 - sum(tl) / padded, worst_batched_vs_alone=worst,
                  speedup=res["one_by_one"]["seconds"] / res["batched"]["seconds"], **res)
    print(json.dumps(report))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
