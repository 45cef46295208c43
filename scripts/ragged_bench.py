"""Throughput of one file's slices sampled one by one at B = 1 (the reference CLI's loop, infer.py:99-126) against the same
slices sampled as ragged batches with ``api.sample_utterances``.

    python scripts/ragged_bench.py [--slices 16] [--steps 40] [--batches 8,16] [--warmup 3] [--out results/ragged_bench.json]

The slices are ``--slices`` lengths drawn uniformly from [150, 1000] frames (seeded) sharing one 256-frame prompt, as the slices
of one file do; the 66 M-parameter denoiser with synthetic weights, 40-step DPM-Solver++.  Two measurements, CUDA events around
the whole list:

- ``warm``: every mode samples through ``DenoiserSession`` objects the bench holds (one per B = 1 slice, one per ragged batch of
  ``api.batch_plan``), device-resident inputs, after ``--warmup`` passes, so every session replays its captured graph.
- ``api``: the public calls as a caller makes them, host tensors in and out, one pass after the same warm-up: ``sample_latents``
  per slice against ``sample_utterances``.  The module's session cache holds 8 shapes, so with more than 8 slices every B = 1
  call builds a new session and runs eagerly; that is what the one-by-one loop costs a caller.

Reported: utterance-seconds of audio per second (frames x 256 / 24 kHz over wall time) and the padding fraction of the batched
runs (padded frames over all frames the denoiser ran).  Each batched result is checked against its B = 1 result (rtol 1e-3 /
atol 1e-4).  Prints the card's name and power limit with the numbers.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ns2vc_b200 import api  # noqa: E402
from ns2vc_b200.arch import ns2vc_denoiser_config  # noqa: E402
from ns2vc_b200.fused import DenoiserSession  # noqa: E402
from ns2vc_b200.synth import make_state_dict  # noqa: E402
from ns2vc_b200.unet import UNet1DConditionModel  # noqa: E402

FRAME_SECONDS = 256 / 24000          # mel hop / sample rate


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable: {e}"


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slices", type=int, default=16)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--batches", default="8,16")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ragged_bench needs a CUDA device")
    cfg = ns2vc_denoiser_config()
    m = UNet1DConditionModel(in_channels=cfg.in_channels, out_channels=cfg.out_channels, block_out_channels=cfg.block_out_channels,
                             layers_per_block=list(cfg.layers_per_block), norm_num_groups=cfg.norm_num_groups,
                             cross_attention_dim=cfg.cross_attention_dim, attention_head_dim=cfg.num_heads,
                             addition_embed_type=cfg.addition_embed_type,
                             addition_embed_type_num_heads=cfg.addition_embed_type_num_heads,
                             resnet_time_scale_shift=cfg.resnet_time_scale_shift)
    m.load_state_dict(make_state_dict(cfg, 0))
    m = m.to("cuda").eval()
    g = torch.Generator().manual_seed(args.seed)
    lengths = torch.randint(150, 1001, (args.slices,), generator=g).tolist()
    prompt = torch.randn((256, cfg.cross_attention_dim), generator=g)
    items = [(torch.randn((100, t), generator=g), torch.randn((t, cfg.in_channels - 100), generator=g), prompt) for t in lengths]
    audio_s = sum(lengths) * FRAME_SECONDS

    ns = api.default_schedule()
    ts = torch.linspace(ns.T, 1.0 / ns.total_N, args.steps + 1)
    batches = [int(v) for v in args.batches.split(",")]

    # ---- warm: sessions held by the bench, device-resident inputs, captured graphs
    dev_items = [(x.cuda(), c.cuda(), p.cuda()) for x, c, p in items]
    singles = [(DenoiserSession(m, c.t()[None].contiguous(), p[None].contiguous(), None), x[None].contiguous()) for x, c, p in dev_items]

    def warm_b1():
        return [s.sample_dpmpp_2m(x, ns, ts)[0] for s, x in singles]

    def warm_batched(mb):
        held = []
        for idx in api.batch_plan(lengths, mb):
            x, c, p, tl, sl = api.pad_batch(dev_items, idx)
            held.append((idx, tl, DenoiserSession(m, c.permute(1, 2, 0).contiguous(), p.permute(1, 0, 2).contiguous(), None,
                                                   content_lengths=tl, prompt_lengths=sl), x.contiguous()))

        def run():
            out = [None] * len(items)
            for idx, tl, s, x in held:
                lat = s.sample_dpmpp_2m(x, ns, ts)
                for j, i in enumerate(idx):
                    out[i] = lat[j, :, :int(tl[j])]
            return out
        return run

    def api_b1():
        return [api.sample_latents(m, x[None], c[:, None], p[:, None], None, steps=args.steps)[0] for x, c, p in items]

    res = {"card": card(), "slices": lengths, "steps": args.steps, "audio_seconds": round(audio_s, 3), "warm": {}, "api": {}}
    for kind, modes in (("warm", [("B=1", warm_b1)] + [(f"max_batch={mb}", warm_batched(mb)) for mb in batches]),
                        ("api", [("B=1", api_b1)] + [(f"max_batch={mb}", lambda mb=mb: api.sample_utterances(m, items, steps=args.steps,
                                                                                                            max_batch=mb))
                                                     for mb in batches])):
        ref = None
        for name, fn in modes:
            for _ in range(args.warmup):
                fn()
            out, sec = timed(fn)
            out = [o.cpu() for o in out]
            row = {"seconds": round(sec, 4), "audio_seconds_per_second": round(audio_s / sec, 2)}
            if ref is None:
                ref = out
            else:
                worst = max(((o - r).abs() / (1e-4 + 1e-3 * r.abs())).max().item() for o, r in zip(out, ref))
                assert worst <= 1.0, f"{kind} {name}: batched result disagrees with B=1 (worst err/tol {worst:.2f})"
                mb = int(name.split("=")[1])
                ran = sum(len(idx) * max(lengths[i] for i in idx) for idx in api.batch_plan(lengths, mb))
                row.update({"padding_fraction": round(1 - sum(lengths) / ran, 4), "worst_err_over_tol_vs_B1": round(worst, 3),
                            "speedup_vs_B1": round(res[kind]["B=1"]["seconds"] / sec, 2)})
            res[kind][name] = row
            print(kind, name, row, flush=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
