"""Requests with two sampler settings, half UniPC-10 and half DPM-Solver++-40, arriving at random times, served three ways:

    (a) mixed:  one ``serve.ConversionServer`` of ``--slots`` slots, each request with its own method and steps;
    (b) split:  two single-method servers of ``--slots / 2`` slots each on the same GPU, each with its own copy of the models,
                ticked alternately from one host loop;
    (c) slow:   one server of ``--slots`` slots running every request at DPM-Solver++-40.

    python scripts/serve_mixed_bench.py [--requests 48] [--slots 8] [--loads 0.5,0.8] [--out results/serve_mixed_bench.json]

Requests, prompt, models and geometry are those of ``scripts/serve_bench.py`` (full-size synthetic models, ``--slots`` x 1024
frames x 512 prompt frames; frame counts uniform in [150, 1000]); each request's class is a seeded coin flip.  The arrival rate
is ``--loads`` times what (a) sustains at full occupancy, ``slots / (mean steps x tick)`` with the tick measured first.  Every
mode gets the same trace and x_T and runs a warm-up trace first (every schedule resident and every tick captured).

Reported per load, mode and class: latency from arrival to audio ready (p50, p95, max; host clock after a device synchronise)
and requests/s (the class's requests over first arrival to the class's last result).  Also a full-occupancy mixed tick (half
the slots on each method) against full-occupancy UniPC-only and DPM-Solver++-only ticks on the same requests, CUDA events over
``--reps`` ticks, alternated ``--rounds`` times.  Prints the card's name and power limit with the numbers.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import serve_bench as sb  # noqa: E402
from ns2vc_b200 import frontend, serve  # noqa: E402

CLASSES = (("unipc", 10), ("dpmsolver", 40))


def server(ms, slots, method="unipc", steps=10):
    return serve.ConversionServer(*ms, slots=slots, max_frames=sb.MAX_FRAMES, max_prompt_frames=sb.MAX_PROMPT, method=method,
                                  steps=steps)


def run(servers, route, reqs, cls, arrivals):
    """Feeds the arrivals to ``servers`` (request i goes to ``servers[route(i)]`` with the settings ``route`` gives) and ticks every
    busy server once per loop, in order, until every request finished.  Returns the finish time of each request."""
    t0 = time.perf_counter()
    finish, owner, nxt = {}, {}, 0
    while len(finish) < len(reqs):
        now = time.perf_counter() - t0
        while nxt < len(reqs) and arrivals[nxt] <= now:
            w, x, _ = reqs[nxt]
            j, method, steps = route(cls[nxt])
            owner[(j, servers[j].submit(w, sb.SR, sb.PROMPT[0], x_T=x, method=method, steps=steps))] = nxt
            nxt += 1
        busy = [j for j, s in enumerate(servers) if not s.table.idle]
        if not busy:
            sb.wait_until(t0, arrivals[nxt])
            continue
        done = [(j, tk) for j in busy for tk in servers[j].tick()]
        torch.cuda.synchronize()
        now = time.perf_counter() - t0
        for key in done:
            finish[owner.pop(key)] = now
    return finish


def summary(cls, arrivals, finish):
    out = {}
    for c, (method, steps) in enumerate(CLASSES):
        idx = [i for i in range(len(cls)) if cls[i] == c]
        lat = np.array([finish[i] - arrivals[i] for i in idx])
        span = max(finish[i] for i in idx) - arrivals[0]
        out[f"{method}-{steps}"] = {"requests": len(idx), "p50": round(float(np.percentile(lat, 50)), 4),
                                    "p95": round(float(np.percentile(lat, 95)), 4), "max": round(float(lat.max()), 4),
                                    "requests_per_s": round(len(idx) / span, 2)}
    out["all_requests_per_s"] = round(len(cls) / (max(finish.values()) - arrivals[0]), 2)
    return out


def full_tick_ms(srv, reqs, settings, reps):
    """Fills every slot of ``srv`` with ``reqs``, slot b with ``settings[b % len(settings)]`` (steps long enough to stay for the
    whole measurement), and returns a function that gives the mean time of ``reps`` more ticks."""
    for b, (w, x, _) in enumerate(reqs):
        m, s = settings[b % len(settings)]
        srv.submit(w, sb.SR, sb.PROMPT[0], x_T=x, method=m, steps=s)
    for _ in range(5):                                   # admission, eager ticks, capture
        srv.tick()
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed():
        torch.cuda.synchronize()
        a.record()
        for _ in range(reps):
            srv.tick()
        e.record()
        torch.cuda.synchronize()
        return a.elapsed_time(e) / reps
    return timed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=48)
    ap.add_argument("--slots", type=int, default=8)
    ap.add_argument("--loads", default="0.5,0.8")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("serve_mixed_bench needs a CUDA device")
    if args.slots < 2 or args.slots % 2:
        raise SystemExit("--slots must be even (the split setup gives each method half)")
    dev = torch.device("cuda")
    ms = sb.models(dev)
    g = torch.Generator().manual_seed(args.seed)
    pw = (0.2 * torch.randn(3 * 24000, generator=g)).float().to(dev)
    sb.PROMPT[0] = frontend.log_mel_spectrogram(pw, 24000)[0]
    B = args.slots
    res = {"card": sb.card(), "slots": B, "max_frames": sb.MAX_FRAMES, "max_prompt_frames": sb.MAX_PROMPT,
           "classes": [f"{m}-{s}" for m, s in CLASSES], "requests": args.requests, "loads": {}}
    print("card:", res["card"], flush=True)

    # full-occupancy ticks on the same requests (the ragged attention's cost depends on the lengths): mixed (alternate slots on
    # each method) against single-method, alternated
    long = args.reps * (args.rounds + 1) + 10
    full = sb.make_requests(B, g, dev)
    mixed = full_tick_ms(server(ms, B), full, [("unipc", long), ("dpmsolver", long)], args.reps)
    single = {m: full_tick_ms(server(ms, B), full, [(m, long)], args.reps) for m in ("unipc", "dpmsolver")}
    tm, ts = [], {m: [] for m in single}
    for _ in range(args.rounds):
        tm.append(mixed())
        for m, f in single.items():
            ts[m].append(f())
    res["full_tick_ms"] = {"mixed": [round(v, 3) for v in tm], **{m: [round(v, 3) for v in t] for m, t in ts.items()}}
    print(f"full-occupancy tick (ms): {res['full_tick_ms']} at B={B}, T={sb.MAX_FRAMES}, S={sb.MAX_PROMPT}", flush=True)
    tick = float(np.mean(tm))
    mean_steps = float(np.mean([s for _, s in CLASSES]))
    cap = B / (mean_steps * tick * 1e-3)
    res["mixed_capacity_requests_per_s"] = round(cap, 2)

    modes = {
        "mixed": ([server(ms, B)], lambda c: (0,) + CLASSES[c]),
        # two deployments: each server with its own models, so each keeps its own workspace and conditioning
        "split": ([server(ms, B // 2, *CLASSES[0]), server(sb.models(dev), B // 2, *CLASSES[1])], lambda c: (c,) + CLASSES[c]),
        "slow": ([server(ms, B, *CLASSES[1])], lambda c: (0,) + CLASSES[1]),
    }
    warm = sb.make_requests(2 * B, g, dev)
    warm_cls = [i % 2 for i in range(len(warm))]
    for servers, route in modes.values():
        run(servers, route, warm, warm_cls, [0.0] * len(warm))

    reqs = sb.make_requests(args.requests, g, dev)
    cls = torch.randint(0, 2, (len(reqs),), generator=g).tolist()
    for load in [float(v) for v in args.loads.split(",")]:
        rate = load * cap
        rng = np.random.default_rng(args.seed + int(load * 1000))
        arrivals = np.cumsum(rng.exponential(1.0 / rate, len(reqs))).tolist()
        arrivals = [a - arrivals[0] for a in arrivals]
        row = {"rate_requests_per_s": round(rate, 3)}
        for name, (servers, route) in modes.items():
            row[name] = summary(cls, arrivals, run(servers, route, reqs, cls, arrivals))
        res["loads"][str(load)] = row
        print(f"load {load}:", json.dumps(row), flush=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
