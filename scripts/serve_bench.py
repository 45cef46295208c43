"""Requests that arrive at random times, served three ways: ``serve.ConversionServer`` (continuous batching), static batching
(whenever the previous call has returned, ``convert_utterances`` on everything queued, ``max_batch=slots``) and one by one.

    python scripts/serve_bench.py [--requests 48] [--slots 8] [--steps 30] [--loads 0.3,0.6,0.9] [--out results/serve_bench.json]

The requests have the frame counts of ``scripts/ragged_bench.py`` (uniform in [150, 1000], seeded) as 44.1 kHz waveforms, one 3 s
prompt mel, and seeded Poisson arrivals.  Full-size models with synthetic weights (ContentVec, the shipped condition encoders, the
66 M-parameter denoiser, the vocos-mel-24khz vocoder shapes); UniPC with ``--steps`` steps; the server's geometry is ``--slots`` x
1024 frames x 512 prompt frames.  The arrival rates are ``--loads`` times what static batching sustains, measured first as
``slots`` over the time of one ``convert_utterances`` call on ``slots`` requests.  Every mode gets the same trace and x_T and runs
one warm-up trace first.

Reported per load and mode: latency from arrival to audio ready (p50, p95, max; host clock after a device synchronise, every
finished result included) and audio-seconds per second over the trace (first arrival to last result).  Also the server's
admission cost per admitted group (encoders + prepare + time table, CUDA events) and a full-occupancy tick against one ragged
``forward_film`` of the same geometry (CUDA events over ``--reps`` calls each).  Prints the card's name and power limit with the
numbers.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ns2vc_b200 import convert, frontend, serve  # noqa: E402
from ns2vc_b200.arch import ns2vc_denoiser_config  # noqa: E402
from ns2vc_b200.content import ContentVec  # noqa: E402
from ns2vc_b200.pre_model import Pre_model  # noqa: E402
from ns2vc_b200.synth import make_contentvec_state_dict, make_pre_state_dict, make_state_dict, make_vocos_state_dict  # noqa: E402
from ns2vc_b200.unet import UNet1DConditionModel  # noqa: E402
from ns2vc_b200.vocoder import Vocos  # noqa: E402

SR = 44100
MAX_FRAMES, MAX_PROMPT = 1024, 512
PRE_CFG = {"phoneme_encoder": dict(in_channels=256, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2),
           "prompt_encoder": dict(in_channels=100, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2)}


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable: {e}"


def models(dev):
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
    return cv, pre, unet, voc


def make_requests(n, g, dev):
    """n (wav on the device, x_T on the device, frames) with frame counts uniform in [150, 1000]."""
    out = []
    for t in torch.randint(150, 1001, (n,), generator=g).tolist():
        ns = int(t * 256 * SR / 24000) + 100
        tt = torch.arange(ns) / SR
        f0 = 100 + 200 * torch.rand(1, generator=g)
        w = (0.3 * torch.sin(2 * torch.pi * f0 * tt) * (1 + 0.5 * torch.sin(2 * torch.pi * 3 * tt)) + 0.02 * torch.randn(ns, generator=g)).float()
        T = convert.frame_plan(ns, SR)["T"]
        out.append((w.to(dev), torch.randn((1, 100, T), generator=g).to(dev), T))
    return out


def wait_until(t0, t):
    while time.perf_counter() - t0 < t:
        time.sleep(min(1e-3, max(0.0, t - (time.perf_counter() - t0))))


def run_server(srv, reqs, arrivals):
    """Feeds the arrivals to the server and ticks while anything is queued or running.  Returns the finish time of each request."""
    t0 = time.perf_counter()
    finish, ticket_of, nxt = {}, {}, 0
    while len(finish) < len(reqs):
        now = time.perf_counter() - t0
        while nxt < len(reqs) and arrivals[nxt] <= now:
            w, x, _ = reqs[nxt]
            ticket_of[srv.submit(w, SR, PROMPT[0], x_T=x)] = nxt
            nxt += 1
        if srv.table.idle:
            wait_until(t0, arrivals[nxt])
            continue
        done = srv.tick()
        torch.cuda.synchronize()
        now = time.perf_counter() - t0
        for tk in done:
            finish[ticket_of[tk]] = now
    return finish


def run_calls(models_, reqs, arrivals, max_batch, one_by_one):
    """Static batching (every queued request in one ``convert_utterances`` call) or one request per call."""
    t0 = time.perf_counter()
    finish, queue, nxt = {}, [], 0
    while len(finish) < len(reqs):
        now = time.perf_counter() - t0
        while nxt < len(reqs) and arrivals[nxt] <= now:
            queue.append(nxt)
            nxt += 1
        if not queue:
            wait_until(t0, arrivals[nxt])
            continue
        take = queue[:1] if one_by_one else queue[:]
        del queue[:len(take)]
        convert.convert_utterances(*models_, [reqs[i][0] for i in take], SR, PROMPT[0], max_batch=max_batch,
                                   x_T=[reqs[i][1] for i in take], steps=STEPS[0])
        torch.cuda.synchronize()
        now = time.perf_counter() - t0
        for i in take:
            finish[i] = now
    return finish


PROMPT, STEPS = [None], [None]


def summary(reqs, arrivals, finish):
    lat = np.array([finish[i] - arrivals[i] for i in range(len(reqs))])
    audio_s = sum(T * 256 for _, _, T in reqs) / 24000
    span = max(finish.values()) - arrivals[0]
    return {"latency_s": {"p50": round(float(np.percentile(lat, 50)), 4), "p95": round(float(np.percentile(lat, 95)), 4),
                          "max": round(float(lat.max()), 4)},
            "audio_seconds_per_second": round(audio_s / span, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=48)
    ap.add_argument("--slots", type=int, default=8)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--loads", default="0.3,0.6,0.9")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("serve_bench needs a CUDA device")
    dev = torch.device("cuda")
    ms = models(dev)
    g = torch.Generator().manual_seed(args.seed)
    pw = (0.2 * torch.randn(3 * 24000, generator=g)).float().to(dev)
    PROMPT[0] = frontend.log_mel_spectrogram(pw, 24000)[0]
    STEPS[0] = args.steps
    B = args.slots
    res = {"card": card(), "slots": B, "max_frames": MAX_FRAMES, "max_prompt_frames": MAX_PROMPT, "steps": args.steps,
           "requests": args.requests, "loads": {}}
    print("card:", res["card"], flush=True)

    # what static batching sustains: one full call of `slots` requests, after two warm-up calls
    cap_reqs = make_requests(B, g, dev)
    for _ in range(3):
        torch.cuda.synchronize()
        t = time.perf_counter()
        convert.convert_utterances(*ms, [w for w, _, _ in cap_reqs], SR, PROMPT[0], max_batch=B, x_T=[x for _, x, _ in cap_reqs], steps=args.steps)
        torch.cuda.synchronize()
        t = time.perf_counter() - t
    cap = B / t
    res["static_capacity_requests_per_s"] = round(cap, 3)
    print(f"static batching sustains {cap:.2f} requests/s ({t:.3f} s per call of {B})", flush=True)

    srv = serve.ConversionServer(*ms, slots=B, max_frames=MAX_FRAMES, max_prompt_frames=MAX_PROMPT, method="unipc", steps=args.steps)
    warm = make_requests(B + 2, g, dev)
    warm_arr = [0.0] * len(warm)
    run_server(srv, warm, warm_arr)
    run_calls(ms, warm, warm_arr, B, False)
    run_calls(ms, warm, warm_arr, B, True)

    reqs = make_requests(args.requests, g, dev)
    for load in [float(v) for v in args.loads.split(",")]:
        rate = load * cap
        rng = np.random.default_rng(args.seed + int(load * 1000))
        arrivals = np.cumsum(rng.exponential(1.0 / rate, len(reqs))).tolist()
        arrivals = [a - arrivals[0] for a in arrivals]
        row = {"rate_requests_per_s": round(rate, 3)}
        srv.admission_events = []
        row["server"] = summary(reqs, arrivals, run_server(srv, reqs, arrivals))
        adm = [s.elapsed_time(e) for s, e in srv.admission_events]
        srv.admission_events = None
        row["server"]["admission_ms"] = {"groups": len(adm), "mean": round(float(np.mean(adm)), 3), "max": round(float(np.max(adm)), 3)}
        row["static"] = summary(reqs, arrivals, run_calls(ms, reqs, arrivals, B, False))
        row["one_by_one"] = summary(reqs, arrivals, run_calls(ms, reqs, arrivals, B, True))
        res["loads"][str(load)] = row
        print(f"load {load}:", json.dumps(row), flush=True)

    # a full-occupancy tick against one ragged forward_film of the same geometry
    full = serve.ConversionServer(*ms, slots=B, max_frames=MAX_FRAMES, max_prompt_frames=MAX_PROMPT, method="unipc", steps=args.reps + 10)
    for w, x, _ in make_requests(B, g, dev):
        full.submit(w, SR, PROMPT[0], x_T=x)
    for _ in range(5):                                   # admission, eager ticks, capture
        full.tick()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(args.reps):
        full.tick()
    b.record()
    torch.cuda.synchronize()
    tick_ms = a.elapsed_time(b) / args.reps
    sess, out = full._sess, torch.empty_like(full._x)
    for _ in range(3):
        sess.forward(full._x, None, out, film_rows=full._film)
    torch.cuda.synchronize()
    a.record()
    for _ in range(args.reps):
        sess.forward(full._x, None, out, film_rows=full._film)
    b.record()
    torch.cuda.synchronize()
    fwd_ms = a.elapsed_time(b) / args.reps
    res["full_tick_ms"] = round(tick_ms, 3)
    res["forward_film_ms"] = round(fwd_ms, 3)
    print(f"full-occupancy tick {tick_ms:.3f} ms (captured graph) vs one ragged forward_film {fwd_ms:.3f} ms (eager) at "
          f"B={B}, T={MAX_FRAMES}, S={MAX_PROMPT}", flush=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
