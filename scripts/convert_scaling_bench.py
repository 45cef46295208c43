"""Scaling of waveform-to-waveform conversion over GPUs: ``convert.convert_utterances(..., group=dist.group.WORLD)``, one
process per GPU.

    torchrun --nproc_per_node N scripts/convert_scaling_bench.py [--repeat 4] [--steps 30] [--max-batch 8] [--warmup 3]
                                                                 [--iters 2] [--out results/convert_scaling_N.json]

The utterances are the 16 slice lengths of ``scripts/ragged_bench.py`` (seeded, [150, 1000] frames) as 44.1 kHz input, ``--repeat``
times over (97 s of audio each time), each a synthetic voice-like signal, with one 3 s prompt mel.  Full-size models with
synthetic weights (ContentVec, the shipped condition encoders, the 66 M-parameter denoiser, vocos-mel-24khz shapes), UniPC-30.
Every rank builds the same inputs and x_T.  After ``--warmup`` calls (so every sampler session replays its captured graph),
each of ``--iters`` timed calls is bracketed by CUDA events on every rank; the call's time is the slowest rank's.

Reported per timed call: audio-seconds per second, each rank's busy time (the sum of CUDA-event spans around its
``convert_batch`` calls), the imbalance max/min busy over ranks with work, and each rank's gather time (CUDA events around
``shard.gather_ragged``: pack, all-gather, unpack).  Rank 0 then converts the same list alone (``group=None``) and reports the
worst ||sharded - alone|| / ||alone|| over the utterances, divided by the 1e-4 tolerance of ``tests/test_shard_convert.py``.
The card's name, power limit and SM clock limit are read in the same run.  Needs CUDA devices.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ns2vc_b200 import convert, frontend, shard  # noqa: E402
from ns2vc_b200.arch import ns2vc_denoiser_config  # noqa: E402
from ns2vc_b200.content import ContentVec  # noqa: E402
from ns2vc_b200.pre_model import Pre_model  # noqa: E402
from ns2vc_b200.synth import make_contentvec_state_dict, make_pre_state_dict, make_state_dict, make_vocos_state_dict  # noqa: E402
from ns2vc_b200.unet import UNet1DConditionModel  # noqa: E402
from ns2vc_b200.vocoder import Vocos  # noqa: E402

SR = 44100
TOL = 1e-4
PRE_CFG = {"phoneme_encoder": dict(in_channels=256, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2),
           "prompt_encoder": dict(in_channels=100, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2)}


def card(index: int) -> str:
    try:
        return subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable: {e}"


def timed_calls(name, fn, spans):
    """Wraps ``fn`` so that each call appends a pair of CUDA events around it to ``spans[name]``."""
    def run(*a, **kw):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        out = fn(*a, **kw)
        e.record()
        spans[name].append((s, e))
        return out
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=4)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--max-batch", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("convert_scaling_bench needs CUDA devices")
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    torch.cuda.set_device(dev)
    group = None
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
        group = dist.group.WORLD

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
    frames = torch.randint(150, 1001, (16,), generator=g).tolist() * args.repeat
    wavs = []
    for t in frames:
        n = int(t * 256 * SR / 24000) + 100
        tt = torch.arange(n) / SR
        f0 = 100 + 200 * torch.rand(1, generator=g)
        wavs.append((0.3 * torch.sin(2 * torch.pi * f0 * tt) * (1 + 0.5 * torch.sin(2 * torch.pi * 3 * tt))
                     + 0.02 * torch.randn(n, generator=g)).float().to(dev))
    pw = (0.2 * torch.randn(3 * 24000, generator=g)).float().to(dev)
    prompt = frontend.log_mel_spectrogram(pw, 24000)[0]
    plans = [convert.frame_plan(len(w), SR) for w in wavs]
    x_T = [torch.randn((1, 100, p["T"]), generator=g).to(dev) for p in plans]
    audio_s = sum(p["T"] * 256 for p in plans) / 24000

    spans = {"busy": [], "gather": []}
    convert.convert_batch = timed_calls("busy", convert.convert_batch, spans)
    shard.gather_ragged = timed_calls("gather", shard.gather_ragged, spans)

    def run(grp):
        return convert.convert_utterances(*models, wavs, SR, prompt, steps=args.steps, max_batch=args.max_batch, x_T=x_T, group=grp)

    for _ in range(args.warmup):
        run(group)
    calls = []
    for _ in range(args.iters):
        torch.cuda.synchronize(dev)
        if world > 1:
            dist.barrier()
        for v in spans.values():
            v.clear()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = run(group)
        e1.record()
        torch.cuda.synchronize(dev)
        mine = torch.tensor([e0.elapsed_time(e1), sum(s.elapsed_time(e) for s, e in spans["busy"]),
                             sum(s.elapsed_time(e) for s, e in spans["gather"])], dtype=torch.float64, device=dev)
        every = torch.empty((world, 3), dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_gather_into_tensor(every, mine[None], group=group)
        else:
            every.copy_(mine[None])
        every = every.cpu()
        busy = every[:, 1].tolist()
        worked = [b for b in busy if b > 0]
        calls.append(dict(seconds=every[:, 0].max().item() / 1e3, audio_s_per_s=audio_s / (every[:, 0].max().item() / 1e3),
                          busy_ms=busy, imbalance=max(worked) / min(worked), gather_ms=every[:, 2].tolist()))
    report = None
    if rank == 0:
        alone = run(None) if world > 1 else out
        worst = max(((a.double() - b.double()).norm() / b.double().norm()).item() for a, b in zip(out, alone))
        plan = shard.plan_batches(plans, [prompt.shape[1]] * len(plans), world, args.max_batch)
        report = dict(card=card(dev.index), gpus=world, utterances=len(wavs), audio_seconds=audio_s, steps=args.steps, method="unipc",
                      max_batch=args.max_batch, batches_per_rank=[len(b) for b in plan], calls=calls,
                      worst_err_over_tol=worst / TOL, tol=TOL)
        print(json.dumps(report))
        if args.out:
            os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
            with open(args.out, "w") as f:
                json.dump(report, f, indent=1)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
