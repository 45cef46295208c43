"""Throughput of each utterance's own training objective: 64 utterances scored one by one with ``diffusion_loss`` on unpadded B = 1
batches (what a caller without the ragged path writes) against one ``utterance_losses(max_batch=8)`` call.

    python scripts/utterance_loss_bench.py [--n 64] [--max-batch 8] [--warmup 2] [--reps 3] [--out results/utterance_loss_bench.json]

The utterances take the slice lengths of ``scripts/ragged_bench.py`` (seeded uniform in [150, 1000] frames, here ``--n`` of them)
with prompt lengths uniform in [50, 300] frames; full-size synthetic models (66 M-parameter denoiser, the shipped encoders); one
drawn timestep per utterance, passed explicitly so both ways evaluate the same ``t`` and noise.  CUDA events around each whole
pass, after ``--warmup`` passes of both; the two ways alternate ``--reps`` times and the median is reported.  Reported:
utterances per second, denoiser / encoder launches per pass (each engine's launch count per call times the calls), and the
padding fraction of the ragged batches (padded frames over all frames the denoiser ran).  The two ways are checked to agree
(rtol 1e-3).  Prints the card's name, power limit and SM clocks with the numbers.  Needs a CUDA device.
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
from ns2vc_b200.loss import diffusion_loss, utterance_losses  # noqa: E402
from ns2vc_b200.pre_model import Pre_model  # noqa: E402
from ns2vc_b200.synth import make_pre_state_dict, make_state_dict  # noqa: E402
from ns2vc_b200.unet import UNet1DConditionModel  # noqa: E402

PRE_CFG = {"phoneme_encoder": dict(in_channels=256, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2),
           "prompt_encoder": dict(in_channels=100, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2)}


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
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


@torch.no_grad()
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=64)
    ap.add_argument("--max-batch", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("utterance_loss_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    unet = UNet1DConditionModel(in_channels=356, out_channels=100, block_out_channels=(128, 256, 384, 512), norm_num_groups=8,
                                cross_attention_dim=256, attention_head_dim=8, addition_embed_type="text", resnet_time_scale_shift="scale_shift")
    unet.load_state_dict(make_state_dict(ns2vc_denoiser_config(), seed=0))
    pre = Pre_model(PRE_CFG)
    pre.load_state_dict(make_pre_state_dict(PRE_CFG, seed=0))
    unet, pre = unet.to(dev).eval(), pre.to(dev).eval()
    g = torch.Generator().manual_seed(args.seed)
    lengths = torch.randint(150, 1001, (args.n,), generator=g).tolist()          # scripts/ragged_bench.py's slice lengths
    prompts = torch.randint(50, 301, (args.n,), generator=g).tolist()
    items = [(torch.randn(256, T, generator=g), torch.randn(100, T, generator=g), torch.randn(100, S, generator=g))
             for T, S in zip(lengths, prompts)]
    t = torch.randint(0, 1000, (args.n,), generator=g)
    noise = [torch.randn(100, T, generator=g) for T in lengths]
    dev_items = [tuple(v.to(dev) for v in it) for it in items]
    dev_noise = [nz.to(dev) for nz in noise]

    def one_by_one():
        out = []
        for i, (c, spec, refer) in enumerate(dev_items):
            data = (c[None], refer[None], None, spec[None], None, torch.tensor([lengths[i]]), torch.tensor([prompts[i]]), None)
            out.append(diffusion_loss(pre, unet, data, t=t[i:i + 1], noise=dev_noise[i][None]).loss)
        return torch.stack(out)

    def ragged():
        return utterance_losses(pre, unet, dev_items, t=t, noise=dev_noise, max_batch=args.max_batch).loss

    res = {"card": card(), "n": args.n, "max_batch": args.max_batch, "lengths": lengths, "prompt_lengths": prompts}
    print(res["card"], flush=True)
    for _ in range(args.warmup):
        a, b = one_by_one(), ragged()
    worst = ((b - a).abs() / a.abs()).max().item()
    assert worst <= 1e-3, f"ragged and one-by-one disagree (rel {worst:.2e})"
    t_one, t_rag = [], []
    for _ in range(args.reps):
        t_one.append(timed(one_by_one)[1])
        t_rag.append(timed(ragged)[1])
    med = lambda v: sorted(v)[len(v) // 2]
    # launches per pass: each engine's launches of its last call (that mode's program) times the calls of the pass
    counts = {}
    for name, fn in (("one_by_one", one_by_one), ("ragged", ragged)):
        fn()
        counts[name] = (unet.launch_count(), pre.launch_count())
    batches = api.batch_plan(lengths, args.max_batch)
    ran = sum(len(b) * max(lengths[i] for i in b) for b in batches)
    calls = {"one_by_one": args.n, "ragged": len(batches)}
    res.update({k: {"seconds": med(v), "seconds_runs": v, "utterances_per_second": args.n / med(v), "calls": calls[k],
                    "denoiser_launches": counts[k][0] * calls[k], "encoder_launches": counts[k][1] * calls[k]}
                for k, v in (("one_by_one", t_one), ("ragged", t_rag))})
    res["ragged"]["padding_fraction"] = 1 - sum(lengths) / ran
    res.update({
        "speedup": med(t_one) / med(t_rag),
        "worst_rel_ragged_vs_one_by_one": worst,
        "card_after": card(),
    })
    for k in ("one_by_one", "ragged"):
        print(k, {n: (round(v, 4) if isinstance(v, float) else v) for n, v in res[k].items() if n != "seconds_runs"}, flush=True)
    print(json.dumps({k: v for k, v in res.items() if k not in ("lengths", "prompt_lengths")}))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
