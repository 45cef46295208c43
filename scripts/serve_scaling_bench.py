"""What a server admission costs, re-preparing every slot against only the rows it changes, and what that does to latency.

    python scripts/serve_scaling_bench.py [--slots 8] [--steps 30] [--reps 20] [--requests 32] [--load 0.8] [--out results/x.json]

Full-size models with synthetic weights, as ``scripts/serve_bench.py`` builds them; the server's geometry is ``--slots`` x 1024
frames x 512 prompt frames, UniPC with ``--steps`` steps.

1. Admission split.  With every slot occupied and prepared, 1, 4 and ``slots`` newcomers are admitted into the first slots.  The
   three parts of an admission are timed with CUDA events: the encoders (``convert.encode_front`` on the newcomers), the
   conditioning (``prepare`` of every slot against ``prepare_rows`` of the newcomers' rows) and the FiLM table (``time_table``
   of steps x slots rows against ``time_table_rows``).  Full and row-scoped calls alternate, ``--reps`` times each, after
   warm-up; mean, min and max are reported.
2. Latency under arrivals.  ``--requests`` requests (frame counts uniform in [150, 1000], seeded) arrive as a seeded Poisson
   process at ``--load`` times the rate one tick per step sustains at full occupancy (slots / (steps x tick time)).  The same
   trace is served twice in alternation, by a server whose admissions re-prepare every slot and by one that re-prepares
   only the changed rows; latency from arrival to audio (p50, p95, max), sustained requests/s and the admission cost per
   admitted group are reported for each.

Under ``torchrun --nproc_per_node W`` (W > 1) only part 2 runs, on a server spread over the W ranks (``group=``, row-scoped
admission, ``slots`` per rank) with the arrival rate scaled by W; rank 0 prints and writes the result.  A run without torchrun
reports world sizes 2, 4 and 8 as not measured, with the number of GPUs the machine has.  Prints the card's name and power
limit with the numbers.  Needs a CUDA device.
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
from serve_bench import MAX_FRAMES, MAX_PROMPT, SR, card, make_requests, models, wait_until  # noqa: E402

from ns2vc_b200 import convert, frontend, serve  # noqa: E402


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    return a, b


def stats(pairs):
    torch.cuda.synchronize()
    v = np.array([a.elapsed_time(b) for a, b in pairs])
    return {"mean": round(float(v.mean()), 3), "min": round(float(v.min()), 3), "max": round(float(v.max()), 3)}


def full_server(ms, prompt, slots, steps, reqs):
    srv = serve.ConversionServer(*ms, slots=slots, max_frames=MAX_FRAMES, max_prompt_frames=MAX_PROMPT, method="unipc", steps=steps)
    for w, x, _ in reqs:
        srv.submit(w, SR, prompt, x_T=x)
    for _ in range(4):                                   # the first (full) admission, eager ticks, the capture
        srv.tick()
    torch.cuda.synchronize()
    return srv


def admission_split(ms, prompt, srv, reqs, counts, reps):
    """{n: {part: {full / rows: stats}}} for n newcomers into slots 0..n-1 of a full, prepared server."""
    cm, pm, _, _ = ms
    sess, dev = srv._sess, torch.device("cuda")
    out = {}
    for n in counts:
        rows = list(range(n))
        wavs = [reqs[i][0] for i in rows]
        plans = [convert._check_inputs([w], SR, [prompt], None)[0] for w in wavs]
        enc, prep, film = [], {"full": [], "rows": []}, {"full": [], "rows": []}
        for r in range(reps + 3):
            e = timed(lambda: convert.encode_front(cm, pm, wavs, SR, [prompt] * n, plans, dev))
            p_full = timed(sess.prepare)
            f_full = timed(lambda: sess.time_table(srv._tvals, srv._film_table))
            p_rows = timed(lambda: sess.prepare_rows(rows))
            f_rows = timed(lambda: sess.time_table_rows(srv._tvals, srv._film_table, rows))
            if r >= 3:
                enc.append(e)
                prep["full"].append(p_full)
                prep["rows"].append(p_rows)
                film["full"].append(f_full)
                film["rows"].append(f_rows)
        out[n] = {"encoders": stats(enc), "prepare": {k: stats(v) for k, v in prep.items()},
                  "film_table": {k: stats(v) for k, v in film.items()}}
        print(f"{n} newcomer(s) into {srv.B} slots:", json.dumps(out[n]), flush=True)
    return out


def run_trace(srv, reqs, arrivals, prompt):
    t0 = time.perf_counter()
    finish, ticket_of, nxt = {}, {}, 0
    srv.admission_events = []
    while len(finish) < len(reqs):
        now = time.perf_counter() - t0
        while nxt < len(reqs) and arrivals[nxt] <= now:
            w, x, _ = reqs[nxt]
            ticket_of[srv.submit(w, SR, prompt, x_T=x)] = nxt
            nxt += 1
        if srv.table.idle:
            wait_until(t0, arrivals[nxt])
            continue
        done = srv.tick()
        torch.cuda.synchronize()
        now = time.perf_counter() - t0
        for tk in done:
            finish[ticket_of[tk]] = now
    lat = np.array([finish[i] - arrivals[i] for i in range(len(reqs))])
    adm = dict(stats(srv.admission_events), groups=len(srv.admission_events))
    srv.admission_events = None
    return {"latency_s": {"p50": round(float(np.percentile(lat, 50)), 4), "p95": round(float(np.percentile(lat, 95)), 4),
                          "max": round(float(lat.max()), 4)},
            "requests_per_s": round(len(reqs) / (max(finish.values()) - arrivals[0]), 3),
            "admission_ms": adm}


def tick_ms(ms, prompt, slots, steps, g, dev):
    """One full-occupancy tick of a one-GPU server (captured graph, CUDA events over 10 ticks)."""
    srv = full_server(ms, prompt, slots, steps, make_requests(slots, g, dev))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(10):
        srv.tick()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 10


def run_group(args, world):
    """Part 2 on ``world`` ranks: every rank ticks in lockstep, rank 0 submits on the arrival clock."""
    import torch.distributed as dist
    rank = int(os.environ["RANK"])
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", rank)))
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    try:
        ms = models(dev)
        g = torch.Generator().manual_seed(args.seed)
        prompt = frontend.log_mel_spectrogram((0.2 * torch.randn(3 * 24000, generator=g)).float().to(dev), 24000)[0]
        B = args.slots
        t = torch.tensor([tick_ms(ms, prompt, B, args.steps, g, dev)], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        rate = args.load * world * B / (args.steps * t.item() / 1e3)
        srv = serve.ConversionServer(*ms, slots=B, max_frames=MAX_FRAMES, max_prompt_frames=MAX_PROMPT, method="unipc",
                                     steps=args.steps, group=dist.group.WORLD)
        reqs = make_requests(args.requests, g, dev)
        rng = np.random.default_rng(args.seed)
        arrivals = np.cumsum(rng.exponential(1.0 / rate, len(reqs))).tolist()
        arrivals = [a - arrivals[0] for a in arrivals]
        rows = []
        for r in range(args.rounds + 1):                  # round 0 warms up
            t0, base = time.perf_counter(), srv.served
            finish, ticket_of, nxt = {}, {}, 0
            while srv.served - base < len(reqs):
                if rank == 0:
                    now = time.perf_counter() - t0
                    if nxt < len(reqs) and not srv._pending and all(tab.occupied == 0 for tab in srv.tables):
                        wait_until(t0, arrivals[nxt])
                        now = time.perf_counter() - t0
                    while nxt < len(reqs) and arrivals[nxt] <= now:
                        w, x, _ = reqs[nxt]
                        ticket_of[srv.submit(w, SR, prompt, x_T=x)] = nxt
                        nxt += 1
                done = srv.tick()
                if rank == 0:
                    now = time.perf_counter() - t0
                    for tk in done:
                        finish[ticket_of[tk]] = now
            if rank == 0 and r > 0:
                lat = np.array([finish[i] - arrivals[i] for i in range(len(reqs))])
                rows.append({"latency_s": {"p50": round(float(np.percentile(lat, 50)), 4), "p95": round(float(np.percentile(lat, 95)), 4),
                                           "max": round(float(lat.max()), 4)},
                             "requests_per_s": round(len(reqs) / (max(finish.values()) - arrivals[0]), 3)})
                print(f"world {world}, round {r}:", json.dumps(rows[-1]), flush=True)
        if rank == 0:
            res = {"card": card(), "world": world, "slots_per_rank": B, "steps": args.steps,
                   "rate_requests_per_s": round(rate, 3), "rounds": rows}
            print(json.dumps(res))
            if args.out:
                os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
                with open(args.out, "w") as f:
                    json.dump(res, f, indent=1)
    finally:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=8)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--requests", type=int, default=32)
    ap.add_argument("--load", type=float, default=0.8)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("serve_scaling_bench needs a CUDA device")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1:
        run_group(args, world)
        return
    dev = torch.device("cuda")
    res = {"card": card(), "slots": args.slots, "max_frames": MAX_FRAMES, "max_prompt_frames": MAX_PROMPT, "steps": args.steps}
    print("card:", res["card"], flush=True)
    ms = models(dev)
    g = torch.Generator().manual_seed(args.seed)
    prompt = frontend.log_mel_spectrogram((0.2 * torch.randn(3 * 24000, generator=g)).float().to(dev), 24000)[0]
    B = args.slots

    srv = full_server(ms, prompt, B, args.steps, make_requests(B, g, dev))
    res["admission_split_ms"] = admission_split(ms, prompt, srv, make_requests(B, g, dev), sorted({1, min(4, B), B}), args.reps)

    # one tick at full occupancy: the rate the server sustains when every slot is busy
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(10):
        srv.tick()
    b.record()
    torch.cuda.synchronize()
    tick_ms = a.elapsed_time(b) / 10
    cap = B / (args.steps * tick_ms / 1e3)
    res["full_tick_ms"] = round(tick_ms, 3)
    print(f"full-occupancy tick {tick_ms:.3f} ms: at most {cap:.2f} requests/s", flush=True)
    del srv

    servers = {mode: serve.ConversionServer(*ms, slots=B, max_frames=MAX_FRAMES, max_prompt_frames=MAX_PROMPT, method="unipc",
                                            steps=args.steps) for mode in ("full", "rows")}
    servers["full"]._prepare_rows = lambda rows, s=servers["full"]: s._prepare_all()   # every admission re-prepares every slot
    warm = make_requests(B + 2, g, dev)
    for s in servers.values():
        run_trace(s, warm, [0.0] * len(warm), prompt)
    reqs = make_requests(args.requests, g, dev)
    rate = args.load * cap
    rng = np.random.default_rng(args.seed)
    arrivals = np.cumsum(rng.exponential(1.0 / rate, len(reqs))).tolist()
    arrivals = [t - arrivals[0] for t in arrivals]
    world = {"1": {"rate_requests_per_s": round(rate, 3), "full": [], "rows": []}}
    for r in range(args.rounds):
        for mode in ("full", "rows"):
            row = run_trace(servers[mode], reqs, arrivals, prompt)
            world["1"][mode].append(row)
            print(f"world 1, round {r}, {mode} admission:", json.dumps(row), flush=True)
    n_gpu = torch.cuda.device_count()
    for w in (2, 4, 8):
        world[str(w)] = (f"not measured: this machine has {n_gpu} GPU(s)" if n_gpu < w else
                         f"run under torchrun --nproc_per_node {w}")
    res["latency_under_arrivals"] = world
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
