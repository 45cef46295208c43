"""``serve.ConversionServer(..., group=...)`` on several ranks.

CPU: the placement function, the header round trip, a 3-rank gloo run of the header / payload / gather protocol with a stub
for the device work (an idle rank, a request placed on each rank, a request with a NaN prompt), a failing rank that makes
every rank raise, ``submit`` on a rank other than 0 and servers built with different arguments.  GPU: two ranks (NCCL on two
GPUs, else gloo with both ranks on cuda:0) serve the six utterances of ``tests/test_convert.py`` with ``slots=2`` per rank at
staggered ticks, for UniPC and DPM-Solver++; every latent and waveform must equal ``convert_batch`` of that request alone bit
for bit, the default draws must equal ``convert_utterances``, a NaN prompt must fail only its own request and an exception
injected on rank 1 must raise on both ranks."""
import os

import pytest
import torch
import torch.distributed as dist

from ns2vc_b200 import convert, serve
from test_shard_convert import _run

SR = 44100


# ----------------------------------------------------------------------------------------------------------------- CPU
def test_place_requests():
    assert serve.place_requests([2, 2, 2], 4) == [0, 1, 2, 0]
    assert serve.place_requests([0, 3, 1], 5) == [1, 1, 1, 2]          # never more than a rank's free slots
    assert serve.place_requests([1, 0, 2], 2) == [2, 0]
    assert serve.place_requests([0, 0], 3) == [] and serve.place_requests([4], 0) == [] and serve.place_requests([], 2) == []
    g = torch.Generator().manual_seed(0)
    for _ in range(200):
        free = torch.randint(0, 5, (int(torch.randint(1, 9, (1,), generator=g)),), generator=g).tolist()
        n = int(torch.randint(0, 30, (1,), generator=g))
        out = serve.place_requests(free, n)
        assert out == serve.place_requests(free, n), "deterministic"
        assert len(out) == min(n, sum(free))
        assert all(out.count(r) <= f for r, f in enumerate(free))
        left = list(free)
        for r in out:                                                   # each pick: the most free slots, the lowest rank on ties
            assert left[r] == max(left) and r == left.index(max(left))
            left[r] -= 1


def test_header_round_trip():
    adm = [(0, 1, 0, 20000, 44100, 42, 30), (5, 0, 3, 123457, 16000, 1000, 512)]
    for a, idle, cap in ((adm, False, 4), ([], True, 3), ([], False, 1), (adm[:1], False, 1)):
        h = serve.pack_header(a, idle, cap)
        assert h.dtype == torch.int64 and h.numel() == 2 + serve.HEADER_FIELDS * cap
        assert serve.unpack_header(h) == (a, idle)
    with pytest.raises(ValueError):
        serve.pack_header(adm, False, 1)
    with pytest.raises(ValueError):
        serve.pack_header([(1, 2, 3)], False, 2)


class _Stub(serve.ConversionServer):
    """The server's protocol with the device work replaced: a tick records the newcomers, and a retired request's result is
    its ticket (audio) and its own x_T (latent), so the test sees what each rank received."""
    fail_at = None

    def _step(self, new):
        if self.fail_at is not None and self.ticks == self.fail_at:
            raise RuntimeError("injected failure")
        self.seen = getattr(self, "seen", []) + [(self.ticks, s, tk) for s, tk in new]

    def _collect(self, done):
        out = []
        for _, tk in done:
            q = self._requests.pop(tk)
            flag = int(bool(q["prompt"].isnan().any()))
            out.append((flag, q["x_T"].reshape(100, q["T"]).float(), torch.full((q["T"] * 256,), float(tk)) + q["wav"][0]))
        return out


def _requests():
    g = torch.Generator().manual_seed(4)
    out = []
    for i, n in enumerate((20000, 15000, 18000, 21000)):
        w = torch.randn(n, generator=g)
        p = torch.randn((100, 20 + i), generator=g)
        if i == 2:
            p[3, 4] = float("nan")
        out.append((w, p, torch.randn((1, 100, convert.frame_plan(n, SR)["T"]), generator=g)))
    return out


def _protocol_worker(rank, world):
    srv = _Stub(None, None, None, None, slots=1, max_frames=100, max_prompt_frames=40, steps=3, group=dist.group.WORLD)
    reqs = _requests()
    res, lat = {}, {}
    if rank == 0:
        for w, p, x in reqs[:2]:                     # tick 0: ranks 0 and 1; rank 2 idle
            srv.submit(w, SR, p, x_T=x)
    res.update(srv.tick())
    lat.update(srv.last_latents)
    if rank == 0:
        for w, p, x in reqs[2:]:                     # tick 1: rank 2 (the only free slot); the next waits for tick 3 (rank 0)
            srv.submit(w, SR, p, x_T=x)
    while not srv._idle:
        res.update(srv.tick())
        lat.update(srv.last_latents)
    assert srv.drain() == {} and srv.tick() == {}    # idle: nothing happens
    ok = True
    if rank == 0:
        for tk, (w, p, x) in enumerate(reqs):
            if tk == 2:
                ok &= isinstance(res[tk], AssertionError) and "model.py:404" in str(res[tk])
                continue
            T = x.shape[2]
            ok &= torch.equal(res[tk], torch.full((T * 256,), float(tk)) + w[0])
        ok &= len(res) == 4 and torch.equal(lat[3], reqs[3][2][0])
    else:
        ok &= res == {}
    return ok, srv.ticks, getattr(srv, "seen", [])


def test_protocol_three_ranks():
    out = _run(_protocol_worker, 3)
    assert all(ok for ok, _, _ in out), out
    assert len({t for _, t, _ in out}) == 1, "drain() returned in different ticks"
    assert [s for _, _, s in out] == [[(0, 0, 0), (3, 0, 3)], [(0, 0, 1)], [(1, 0, 2)]]


def _failing_worker(rank, world):
    srv = _Stub(None, None, None, None, slots=1, max_frames=100, max_prompt_frames=40, steps=3, group=dist.group.WORLD)
    srv.fail_at = 1 if rank == 1 else None
    if rank == 0:
        for w, p, x in _requests()[:3]:
            srv.submit(w, SR, p, x_T=x)
    try:
        srv.drain()
    except RuntimeError as e:
        return str(e)
    return "no error"


def test_a_failing_rank_makes_every_rank_raise():
    msgs = _run(_failing_worker, 3)
    for r, m in enumerate(msgs):
        assert m.startswith("server tick 1 failed on rank(s) [1]"), f"rank {r}: {m}"
    assert "injected failure" in msgs[1]


def _argument_worker(rank, world):
    out = []
    srv = _Stub(None, None, None, None, slots=1, max_frames=100, max_prompt_frames=40, steps=3, group=dist.group.WORLD)
    w, p, x = _requests()[0]
    try:
        srv.submit(w, SR, p, x_T=x)
        out.append("no error")
    except RuntimeError as e:
        out.append(str(e))
    bad = _Stub(None, None, None, None, slots=1, max_frames=100, max_prompt_frames=40, steps=3 + (rank == 2), group=dist.group.WORLD)
    try:
        bad.tick()
        out.append("no error")
    except ValueError as e:
        out.append(str(e))
    return out


def test_argument_errors_on_several_ranks():
    out = _run(_argument_worker, 3)
    assert out[0][0] == "no error"
    for r in (1, 2):
        assert out[r][0] == f"submit() on rank {r}: only rank 0 of the server's group takes requests"
    for r in range(3):
        assert out[r][1].startswith("the ranks built their servers with different arguments"), out[r][1]


# ----------------------------------------------------------------------------------------------------------------- GPU
STEPS, SLOTS = 8, 2
ARRIVALS = {0: [0, 1, 2], 1: [3], 4: [4], 6: [5]}       # tick -> requests submitted just before it


def _serve(srv, wavs, prompts, xs, rank):
    """Serves the six requests on ARRIVALS; rank 0 returns ({request: audio or exception}, {request: latent})."""
    req, res, lat = {}, {}, {}
    while True:
        if rank == 0:
            for i in ARRIVALS.get(srv.ticks, ()):
                req[srv.submit(wavs[i], SR, prompts[i], x_T=None if xs is None else xs[i])] = i
        done = srv.tick()
        res.update({req[tk]: (v.cpu() if isinstance(v, torch.Tensor) else v) for tk, v in done.items()})
        lat.update({req[tk]: v.cpu() for tk, v in srv.last_latents.items()})
        if srv.ticks > max(ARRIVALS) and srv._idle:
            return res, lat


def _gpu_worker(rank, world, out_dir):
    from test_shard_convert import _chain
    dev = torch.device("cuda", torch.cuda.current_device())
    models, wavs, prompt = _chain(dev)
    g = torch.Generator().manual_seed(5)
    xs = [torch.randn((1, 100, convert.frame_plan(len(w), SR)["T"]), generator=g) for w in wavs]
    kw = dict(slots=SLOTS, max_frames=400, max_prompt_frames=80, steps=STEPS, group=dist.group.WORLD)
    out = {"backend": str(dist.get_backend())}
    for method in ("unipc", "dpmsolver"):
        res, lat = _serve(serve.ConversionServer(*models, method=method, **kw), wavs, [prompt] * 6, xs, rank)
        if rank == 0:
            out[method + "_res"] = res
            bad = []
            for i in range(6):
                r = convert.convert_batch(*models, [wavs[i]], SR, [prompt], [xs[i]], method, STEPS)
                if not (torch.equal(lat[i], r["latent"][0].cpu()) and torch.equal(res[i], r["audio"][0].cpu())):
                    bad.append(i)
            out[method] = bad
        else:
            out[method] = res == {} and lat == {}
    # default draws on rank 0 after a seed, against convert_utterances of the list
    torch.manual_seed(1234)
    res, _ = _serve(serve.ConversionServer(*models, **kw), wavs, [prompt] * 6, None, rank)
    if rank == 0:
        torch.manual_seed(1234)
        want = convert.convert_utterances(*models, wavs, SR, prompt, steps=STEPS, max_batch=SLOTS)
        out["draws"] = [i for i in range(6) if not torch.equal(res[i], want[i].cpu())]
    # a NaN prompt fails only its own request
    bad_prompt = prompt.clone()
    bad_prompt[7, 11] = float("nan")
    prompts = [prompt] * 6
    prompts[2] = bad_prompt
    res, lat = _serve(serve.ConversionServer(*models, method="unipc", **kw), wavs, prompts, xs, rank)
    if rank == 0:
        clean = out.pop("unipc_res")
        same = [i for i in range(6) if i != 2 and torch.equal(res[i], clean[i])]
        out["nan"] = (isinstance(res[2], AssertionError) and "model.py:404" in str(res[2]), 2 not in lat, same)
        out.pop("dpmsolver_res")
    # an exception injected on rank 1 raises on both ranks
    srv = serve.ConversionServer(*models, method="unipc", **kw)
    if rank == 1:
        def boom():
            raise RuntimeError("injected on rank 1")
        srv._run_tick = boom
    try:
        _serve(srv, wavs, [prompt] * 6, xs, rank)
        out["raise"] = "no error"
    except RuntimeError as e:
        out["raise"] = str(e)
    path = os.path.join(out_dir, f"rank{rank}.pt")
    torch.save(out, path)
    return path


@pytest.mark.gpu
def test_two_ranks_serve_each_request_as_converted_alone(tmp_path):
    backend = "nccl" if torch.cuda.device_count() >= 2 else "gloo"
    paths = _run(_gpu_worker, 2, str(tmp_path), backend=backend, timeout=900)
    assert all(p.endswith(".pt") for p in paths), paths
    r0, r1 = [torch.load(p, weights_only=False) for p in paths]
    print(f"2 ranks over {r0['backend']}: {r0}")
    for method in ("unipc", "dpmsolver"):
        assert r0[method] == [], f"{method}: requests {r0[method]} differ from convert_batch alone"
        assert r1[method] is True, f"{method}: rank 1 returned results"
    assert r0["draws"] == [], f"default draws of requests {r0['draws']} differ from convert_utterances"
    assert r0["nan"] == (True, True, [0, 1, 3, 4, 5]), r0["nan"]
    for r in (r0, r1):
        assert r["raise"].startswith("server tick 0 failed on rank(s) [1]"), r["raise"]
