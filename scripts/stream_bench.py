"""Tick time of live conversion (``stream.StreamConverter``): B streams in one session against B separate one-stream sessions
ticked one after another.

    python scripts/stream_bench.py [--batches 1 2 4 8] [--steps 30 10] [--warmup 3] [--ticks 10] [--runs 2] [--out FILE]

Full-size models with synthetic weights as in ``scripts/convert_bench.py`` (ContentVec, the shipped condition encoders, the
66 M-parameter denoiser, the vocos-mel-24khz vocoder shapes), the default geometry (0.48 s blocks, 1.6 s of context), a 16 kHz
voice-like input per stream, one 3 s prompt mel per stream, UniPC.  The first ``--warmup`` ticks of every session are not
timed: the sampler session of the tick's shape captures its graph on the third.  A tick's time is a host clock around ``push``
with the input block on the host, so it includes the host-to-device copy of the block and the device-to-host copy of the
output; the time per stage is the sum of CUDA events around each stage call.  The real-time factor is tick time / block
duration: below 1 keeps up with live input.  Each measurement is taken ``--runs`` times in the same process for the spread.
Reported with the card's name and power limit.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ns2vc_b200 import convert, frontend, stream  # noqa: E402
from ns2vc_b200.arch import ns2vc_denoiser_config  # noqa: E402
from ns2vc_b200.content import ContentVec  # noqa: E402
from ns2vc_b200.pre_model import Pre_model  # noqa: E402
from ns2vc_b200.synth import make_contentvec_state_dict, make_pre_state_dict, make_state_dict, make_vocos_state_dict  # noqa: E402
from ns2vc_b200.unet import UNet1DConditionModel  # noqa: E402
from ns2vc_b200.vocoder import Vocos  # noqa: E402
from convert_bench import PRE_CFG, StageTimer, card  # noqa: E402

SR = 16000


def voice(g: torch.Generator, n: int) -> torch.Tensor:
    t = torch.arange(n) / SR
    f0 = 100 + 200 * torch.rand(1, generator=g)
    return (0.3 * torch.sin(2 * torch.pi * f0 * t) * (1 + 0.5 * torch.sin(2 * torch.pi * 3 * t)) + 0.02 * torch.randn(n, generator=g)).float()


def run_ticks(sessions, blocks, warmup, timer):
    """Ticks every session in turn once per tick (one session: a batched tick; B sessions: the one-by-one baseline); returns the
    host seconds of each timed tick and the stage totals over the timed ticks."""
    times = []
    for i, blk in enumerate(blocks):
        if i == warmup:
            timer.totals()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for s, b in zip(sessions, blk):
            s.push(b)
        t1 = time.perf_counter()
        if i >= warmup:
            times.append(t1 - t0)
    return times, timer.totals()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 2, 4, 8])
    ap.add_argument("--steps", type=int, nargs="+", default=[30, 10])
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ticks", type=int, default=10)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stream_bench needs a CUDA device")
    if args.warmup < 3:
        raise SystemExit("--warmup must be >= 3: the sampler captures its graph on a shape's third tick")
    dev = torch.device("cuda")
    gpu = card()
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

    plan = stream.stream_plan(SR)
    block_s = plan["Nb"] / convert.TARGET_SR
    g = torch.Generator().manual_seed(args.seed)
    Bmax = max(args.batches)
    prompts = [frontend.log_mel_spectrogram((0.2 * torch.randn(3 * 24000, generator=g)).float().to(dev), 24000)[0] for _ in range(Bmax)]
    n_ticks = args.warmup + args.ticks
    inp = torch.stack([voice(g, n_ticks * plan["block_in"]) for _ in range(Bmax)])        # host [Bmax, n_ticks * block_in]

    timer = StageTimer()
    frontend.resample = timer.wrap("resample", frontend.resample)
    cv.extract = timer.wrap("content", cv.extract)
    pre.infer = timer.wrap("encoders", pre.infer)
    convert.sample_latents = timer.wrap("sampler", convert.sample_latents)
    voc.decode = timer.wrap("vocoder", voc.decode)
    stream.sola = timer.wrap("sola", stream.sola)

    rows = []
    for steps in args.steps:
        for B in args.batches:
            for mode in ("batched", "one_by_one"):
                for run in range(args.runs):
                    if mode == "batched":
                        sessions = [stream.StreamConverter(*models, prompts[:B], SR, steps=steps)]
                        blocks = [[inp[:B, i * plan["block_in"]:(i + 1) * plan["block_in"]]] for i in range(n_ticks)]
                    else:
                        sessions = [stream.StreamConverter(*models, [prompts[j]], SR, steps=steps) for j in range(B)]
                        blocks = [[inp[j:j + 1, i * plan["block_in"]:(i + 1) * plan["block_in"]] for j in range(B)]
                                  for i in range(n_ticks)]
                    times, stages = run_ticks(sessions, blocks, args.warmup, timer)
                    med = statistics.median(times)
                    row = dict(steps=steps, B=B, mode=mode, run=run, tick_ms_median=1e3 * med, tick_ms_min=1e3 * min(times),
                               tick_ms_max=1e3 * max(times), rtf=med / block_s,
                               stages_ms_per_tick={k: 1e3 * v / len(times) for k, v in stages.items()})
                    rows.append(row)
                    print(json.dumps(row), flush=True)

    def real_time(steps, B):
        return all(r["rtf"] < 1.0 for r in rows if r["steps"] == steps and r["mode"] == "batched" and r["B"] == B)
    realtime = {steps: max([B for B in args.batches if real_time(steps, B)], default=None) for steps in args.steps}
    report = dict(card=gpu, sr=SR, plan=plan, block_seconds=block_s, warmup=args.warmup, ticks=args.ticks, runs=args.runs,
                  largest_real_time_B=realtime, rows=rows)
    print(json.dumps(dict(card=gpu, largest_real_time_B=realtime)))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
