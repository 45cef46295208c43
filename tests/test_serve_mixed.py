"""Per-request sampler settings in ``serve.ConversionServer``: DPM-Solver++ and UniPC rows at their own step counts in one tick.

CPU: per-request retirement ticks in ``serve.SlotTable``, the per-request argument errors of ``submit``, and a 3-rank gloo run
of the header / payload / settings protocol with a stub for the device work, in which every rank must see each newcomer's
(method, steps) and hold the same mirrored slot tables.  GPU: ``ns2vc_sampler_step_rows`` on rows of both methods and of
several schedules against the scalar step kernels bit for bit (empty rows exactly 0, NaN flags per row, poison in the planes a
row's method does not read changes nothing), and a server whose six requests each bring their own method and step count, one
GPU and two ranks over gloo, every result bit-identical to ``convert_batch`` of that request alone."""
import ctypes as C
import os

import pytest
import torch
import torch.distributed as dist

from ns2vc_b200 import _lib, api, coefs, convert, serve
from test_convert import SR
from test_serve import MAX_FRAMES, MAX_PROMPT, SLOTS, chain  # noqa: F401  (chain: the shared fixture)
from test_serve_group import _requests, _Stub
from test_shard_convert import _run


# ----------------------------------------------------------------------------------------------------------------- CPU
def test_slot_table_retires_each_request_after_its_own_steps():
    tab = serve.SlotTable(2, 5)
    for tk, steps in ((0, 3), (1, None), (2, 1), (3, 7)):
        tab.enqueue(tk, steps)
    assert tab.admit(0) == [(0, 0), (1, 1)] and tab.last == [2, 4]
    assert tab.retire(1) == [] and tab.retire(2) == [(0, 0)]
    assert tab.admit(3) == [(0, 2)] and tab.last == [3, 4]
    assert tab.retire(3) == [(0, 2)] and tab.retire(4) == [(1, 1)]
    assert tab.admit(5) == [(0, 3)] and tab.last == [11, None] and tab.retire(11) == [(0, 3)] and tab.idle
    for bad in (0, -2):
        with pytest.raises(ValueError, match="steps must be >= 1"):
            tab.enqueue(9, bad)
    assert tab.idle, "a refused request must not be queued"
    g = torch.Generator().manual_seed(1)
    for slots in (1, 3, 8):
        tab = serve.SlotTable(slots, 4)
        steps, admitted, retired, nxt = {}, {}, {}, 0
        for tick in range(300):
            for _ in range(int(torch.poisson(torch.tensor(0.1 * slots), generator=g))) if tick < 200 else ():
                steps[nxt] = int(torch.randint(1, 12, (1,), generator=g))
                tab.enqueue(nxt, steps[nxt])
                nxt += 1
            for s, t in tab.admit(tick):
                admitted[t] = (s, tick)
            assert not (tab.queue and tab.free_slots())
            for s, t in tab.retire(tick):
                retired[t] = tick
        assert tab.idle and len(retired) == nxt
        assert sorted(admitted, key=lambda t: (admitted[t][1], admitted[t][0])) == sorted(admitted), "admission is not FIFO"
        for t, (s, a) in admitted.items():
            assert retired[t] == a + steps[t] - 1, "a request must retire after exactly its own steps"


def test_per_request_argument_errors():
    w, mel = torch.zeros(20000), torch.zeros(100, 30)
    x = torch.zeros(1, 100, convert.frame_plan(20000, SR)["T"])
    srv = serve.ConversionServer(None, None, None, None, slots=2, max_frames=100, max_prompt_frames=40)
    for method in ("ddpm", "ddim"):
        with pytest.raises(ValueError, match="per-step noise") as e:
            srv.submit(w, SR, mel, x_T=x, method=method)
        with pytest.raises(ValueError) as e2:
            convert._check_method(method, None)
        assert str(e.value) == str(e2.value), "the server refuses DDPM / DDIM per request as convert_utterances does"
    with pytest.raises(ValueError, match="unknown method 'euler'"):
        srv.submit(w, SR, mel, x_T=x, method="euler")
    for steps in (0, -1):
        with pytest.raises(ValueError, match="steps must be >= 1"):
            srv.submit(w, SR, mel, x_T=x, steps=steps)
        with pytest.raises(ValueError, match="steps must be >= 1"):
            srv.submit(w, SR, mel, x_T=x, method="dpmsolver", steps=steps)
    assert srv.table.idle and srv._next_ticket == 0, "a refused request takes no ticket"
    tks = [srv.submit(w, SR, mel, x_T=x, method=m, steps=s) for m, s in ((None, None), ("dpmsolver", None), ("dpmsolver", 12),
                                                                           (None, 3))]
    assert tks == [0, 1, 2, 3] and list(srv.table.queue) == tks
    got = [(srv._requests[t]["method"], srv._requests[t]["steps"]) for t in tks]
    assert got == [("unipc", 30), ("dpmsolver", 30), ("dpmsolver", 12), ("unipc", 3)], got
    assert [srv.table._steps[t] for t in tks] == [30, 30, 12, 3]


class _MixedStub(_Stub):
    """``test_serve_group._Stub`` that also records each newcomer's (method, steps) as this rank received them and, after
    every tick, this rank's mirror of every rank's slot table."""

    def _step(self, new):
        self.seen = getattr(self, "seen", []) + [(self.ticks, s, tk, self._requests[tk]["method"], self._requests[tk]["steps"])
                                                 for s, tk in new]

    def tick(self):
        out = super().tick()
        self.mirror = getattr(self, "mirror", []) + [[(list(t.ticket), list(t.last)) for t in self.tables]]
        return out


SETTINGS = [("dpmsolver", 2), (None, None), ("unipc", 5), ("dpmsolver", 1)]       # the server's own: unipc, 3 steps


def _mixed_protocol_worker(rank, world):
    srv = _MixedStub(None, None, None, None, slots=1, max_frames=100, max_prompt_frames=40, steps=3, group=dist.group.WORLD)
    reqs = _requests()
    res, when = {}, {}

    def tick():
        t = srv.ticks
        for tk, v in srv.tick().items():
            res[tk], when[tk] = v, t

    if rank == 0:
        for (w, p, x), (m, s) in list(zip(reqs, SETTINGS))[:2]:     # tick 0: ranks 0 and 1; rank 2 idle
            srv.submit(w, SR, p, x_T=x, method=m, steps=s)
    tick()
    if rank == 0:
        for (w, p, x), (m, s) in list(zip(reqs, SETTINGS))[2:]:     # tick 1: rank 2; the last waits for rank 0's slot
            srv.submit(w, SR, p, x_T=x, method=m, steps=s)
    while not srv._idle:
        tick()
    ok = True
    if rank == 0:
        ok &= isinstance(res[2], AssertionError) and len(res) == 4
        for tk in (0, 1, 3):
            ok &= torch.equal(res[tk], torch.full((reqs[tk][2].shape[2] * 256,), float(tk)) + reqs[tk][0][0])
    else:
        ok &= res == {}
    return ok, when, getattr(srv, "seen", []), srv.mirror


def test_settings_reach_every_rank_and_retirements_agree():
    out = _run(_mixed_protocol_worker, 3)
    assert all(ok for ok, _, _, _ in out), out
    # request 0: rank 0 at tick 0, 2 steps; 1: rank 1 at tick 0, the default 3; 2: rank 2 at tick 1, 5; 3: rank 0 at tick 2, 1
    assert out[0][1] == {0: 1, 1: 2, 3: 2, 2: 5}, out[0][1]
    assert [s for _, _, s, _ in out] == [[(0, 0, 0, "dpmsolver", 2), (2, 0, 3, "dpmsolver", 1)], [(0, 0, 1, "unipc", 3)],
                                         [(1, 0, 2, "unipc", 5)]]
    assert out[0][3] == out[1][3] == out[2][3], "the ranks' mirrored slot tables differ"
    assert out[0][3][0] == [([0], [1]), ([1], [2]), ([None], [None])]


# ----------------------------------------------------------------------------------------------------------------- GPU
DPM, UNIPC = 0, 1                         # NS2VC_ROW_DPM, NS2VC_ROW_UNIPC


def _table(method, n):
    ns = api.default_schedule()
    ts = torch.linspace(ns.T, 1.0 / ns.total_N, n + 1)
    return coefs.dpmpp_2m_table(ns, ts, True) if method == DPM else coefs.unipc_bh2_table(ns, ts, "bh2")


# (method, steps): DPM-Solver++ at 6 steps ends on a lower-order step, at 10 it does not (lower_order_final applies below 10)
SCHEDULES = [(DPM, 6), (DPM, 10), (UNIPC, 4), (UNIPC, 8)]


def _rows():
    """Rows at k = 0, 1, a middle step, the step before the last and the last of every schedule, plus three empty rows, shuffled."""
    rows = [(m, n, k) for m, n in SCHEDULES for k in sorted({0, 1, n // 2, n - 2, n - 1})] + [(None, None, -1)] * 3
    perm = torch.randperm(len(rows), generator=torch.Generator().manual_seed(2)).tolist()
    return [rows[i] for i in perm]


PLANES = ("x_in", "o", "m0", "m1", "x_prev")
OUTS = ("m_new", "x_t", "x_new")


def _unused(m, st):
    """The input planes a row's step does not read."""
    if m == DPM:
        return ("m1", "x_prev") + (("m0",) if st.order < 2 else ())
    return {0: ("x_prev", "m0", "m1"), 1: ("m1",), 2: ()}[st.corr_order]


class _Mixed:
    def __init__(self):
        self.L = _lib.lib()
        self.tabs = {m: [] for m in (DPM, UNIPC)}
        self.base = {}
        for m, n in SCHEDULES:
            self.base[(m, n)] = len(self.tabs[m])
            self.tabs[m] += _table(m, n)
        self.dev = {m: coefs.c_table(self.tabs[m], "cuda")[0] for m in (DPM, UNIPC)}
        self.rows = _rows()
        self.B, self.Cl, self.T = len(self.rows), 100, 97
        g = torch.Generator(device="cuda").manual_seed(7)
        self.ins = {p: torch.randn((self.B, self.Cl, self.T), device="cuda", generator=g) for p in PLANES}

    def struct(self, b):
        m, n, k = self.rows[b]
        return self.tabs[m][self.base[(m, n)] + k]

    def run(self, ins, nan=None):
        B = self.B
        k = torch.tensor([r[2] for r in self.rows], dtype=torch.int32, device="cuda")
        tag = torch.tensor([r[0] if r[0] is not None else 1 - (b % 2) for b, r in enumerate(self.rows)], dtype=torch.int32, device="cuda")
        base = torch.tensor([self.base[(m, n)] if m is not None else 0 for m, n, _ in self.rows], dtype=torch.int32, device="cuda")
        outs = {p: torch.full((B, self.Cl, self.T), 7.0, device="cuda") for p in OUTS}
        _lib.check(self.L.ns2vc_sampler_step_rows(
            ins["x_in"].data_ptr(), ins["o"].data_ptr(), ins["m0"].data_ptr(), ins["m1"].data_ptr(), ins["x_prev"].data_ptr(),
            self.dev[DPM].data_ptr(), self.dev[UNIPC].data_ptr(), tag.data_ptr(), base.data_ptr(), k.data_ptr(),
            outs["m_new"].data_ptr(), outs["x_t"].data_ptr(), outs["x_new"].data_ptr(), self.Cl * self.T, B,
            nan.data_ptr() if nan is not None else None, None))
        torch.cuda.synchronize()
        return k, outs

    def scalar(self, b):
        """Row b through the scalar step of its method: {m_new, x_t, x_new}, x_t left at 7 where the step does not write it."""
        m, _, _ = self.rows[b]
        st, n = self.struct(b), self.Cl * self.T
        c = coefs.c_struct(st)
        i = {p: self.ins[p][b] for p in PLANES}
        ref = {p: torch.full((self.Cl, self.T), 7.0, device="cuda") for p in OUTS}
        if m == DPM:
            _lib.check(self.L.ns2vc_dpm_step(i["x_in"].data_ptr(), i["o"].data_ptr(), i["m0"].data_ptr(), C.byref(c),
                                             ref["m_new"].data_ptr(), ref["x_new"].data_ptr(), n, None, None))
        else:
            _lib.check(self.L.ns2vc_unipc_step(i["x_prev"].data_ptr(), i["x_in"].data_ptr(), i["o"].data_ptr(), i["m0"].data_ptr(),
                                               i["m1"].data_ptr(), C.byref(c), ref["m_new"].data_ptr(), ref["x_t"].data_ptr(),
                                               ref["x_new"].data_ptr(), n, None, None))
            if st.corr_order == 0:               # the scalar step leaves x_t alone there; the row step writes x_eval
                ref["x_t"] = i["x_in"].clone()
        torch.cuda.synchronize()
        return ref


@pytest.mark.gpu
def test_mixed_rows_equal_the_scalar_steps_bit_for_bit():
    mx = _Mixed()
    rows = mx.rows
    kinds = {(m, mx.struct(b).order if m == DPM else (mx.struct(b).corr_order, mx.struct(b).pred_order))
             for b, (m, _, k) in enumerate(rows) if k >= 0}
    assert {(DPM, 1), (DPM, 2), (UNIPC, (0, 1)), (UNIPC, (1, 2)), (UNIPC, (2, 2)), (UNIPC, (2, 1))} <= kinds, kinds
    nan = torch.zeros(mx.B, dtype=torch.int32, device="cuda")
    k, outs = mx.run(mx.ins, nan)
    assert k.tolist() == [r[2] + 1 if r[2] >= 0 else -1 for r in rows], "occupied rows advance by one step, empty rows stay empty"
    assert nan.tolist() == [0] * mx.B
    for b, (m, n, kb) in enumerate(rows):
        if kb < 0:
            for p in OUTS:
                assert torch.count_nonzero(outs[p][b]) == 0, f"empty row {b}: {p} is not exactly 0"
            continue
        ref = mx.scalar(b)
        name = ("DPM-Solver++" if m == DPM else "UniPC") + f"-{n} step {kb}"
        for p in OUTS:
            assert torch.equal(outs[p][b], ref[p]), f"row {b} ({name}): {p} differs from the scalar step"

    # NaN in the input of one DPM row, one UniPC row and one empty row: only the two occupied rows' flags
    d = next(b for b, r in enumerate(rows) if r[0] == DPM)
    u = next(b for b, r in enumerate(rows) if r[0] == UNIPC)
    e = next(b for b, r in enumerate(rows) if r[2] < 0)
    for hit in ([d], [u], [d, u, e]):
        ins = {p: v.clone() for p, v in mx.ins.items()}
        for b in hit:
            ins["x_in"][b, 3, 5] = float("nan")
        nan.zero_()
        mx.run(ins, nan)
        assert nan.nonzero().flatten().tolist() == sorted(b for b in hit if b != e), (hit, nan.tolist())

    # NaN in every plane a row's method and step do not read (and everywhere in the empty rows) changes nothing
    ins = {p: v.clone() for p, v in mx.ins.items()}
    for b, (m, _, kb) in enumerate(rows):
        for p in (PLANES if kb < 0 else _unused(m, mx.struct(b))):
            ins[p][b].fill_(float("nan"))
    nan.zero_()
    _, poisoned = mx.run(ins, nan)
    assert nan.tolist() == [0] * mx.B
    for p in OUTS:
        assert torch.equal(poisoned[p], outs[p]), f"{p}: NaN in unread planes changed the step"


def test_mixed_rows_argument_errors():
    """Refused on the host before any launch, so the pointers are never dereferenced."""
    L, p = _lib.lib(), 256
    with pytest.raises(_lib.Ns2vcError, match="no coefficient table"):
        _lib.check(L.ns2vc_sampler_step_rows(p, p, p, p, p, None, None, p, p, p, p, p, p, 4, 1, None, None))
    for j in range(13):
        if j in (5, 6):                                      # the two tables: one of them may be NULL
            continue
        args = [p] * 13
        args[j] = None
        with pytest.raises(_lib.Ns2vcError, match="null argument"):
            _lib.check(L.ns2vc_sampler_step_rows(*args, 4, 1, None, None))
    for B, n in ((0, 4), (65536, 4), (1, 0)):
        with pytest.raises(_lib.Ns2vcError, match="bad row batch"):
            _lib.check(L.ns2vc_sampler_step_rows(*([p] * 13), n, B, None, None))


# the six utterances' settings; the server's own is DPM-Solver++ at 5 steps
REQ = [("unipc", 8), ("dpmsolver", 6), ("unipc", 4), ("dpmsolver", 10), ("unipc", 8), (None, None)]
SERVER = dict(method="dpmsolver", steps=5)
OWN = [(m or SERVER["method"], s or SERVER["steps"]) for m, s in REQ]
ARRIVALS = {0: [0, 1, 2], 2: [3], 5: [4], 9: [5]}        # tick -> requests submitted just before it


def _serve_script(srv, wavs, prompt, xs, submit=True):
    """Serves the six requests on ARRIVALS with their own settings (``submit``: this rank takes requests).  Returns
    ({request: audio}, {request: latent}, {request: (admission tick, retirement tick)})."""
    req, res, lat, span = {}, {}, {}, {}
    while True:
        if submit:
            for i in ARRIVALS.get(srv.ticks, ()):
                m, s = REQ[i]
                req[srv.submit(wavs[i], SR, prompt, x_T=None if xs is None else xs[i], method=m, steps=s)] = i
                span[i] = srv.ticks
        t = srv.ticks
        done = srv.tick()
        for tk, v in done.items():
            res[req[tk]] = v.cpu() if isinstance(v, torch.Tensor) else v
            span[req[tk]] = (span[req[tk]], t)
        lat.update({req[tk]: v.cpu() for tk, v in srv.last_latents.items()})
        idle = srv._idle if srv.world > 1 else srv.table.idle
        if srv.ticks > max(ARRIVALS) and idle:
            return res, lat, span


def _alone(models, wavs, prompt, x, i):
    m, s = OWN[i]
    r = convert.convert_batch(*models, [wavs[i]], SR, [prompt], [x], m, s)
    return r["latent"][0].cpu(), r["audio"][0].cpu()


@pytest.mark.gpu
def test_each_request_with_its_own_sampler_equals_its_own_conversion(chain):
    models, wavs, prompt, xs = chain
    srv = serve.ConversionServer(*models, slots=SLOTS, max_frames=MAX_FRAMES, max_prompt_frames=MAX_PROMPT, **SERVER)
    res, lat, span = _serve_script(srv, wavs, prompt, xs)
    for i, (a, r) in span.items():
        assert r - a + 1 == OWN[i][1], f"request {i} ({OWN[i]}) ran ticks {a}..{r}"
    assert len(srv._sched) == 5 and srv._tvals.shape[0] == 10, "every schedule stays resident; the FiLM table fits the longest"
    bad = []
    for i in range(len(wavs)):
        la, aa = _alone(models, wavs, prompt, xs[i], i)
        if not (torch.equal(lat[i], la) and torch.equal(res[i], aa)):
            bad.append(f"request {i} {OWN[i]}: max|latent diff| {(lat[i] - la).abs().max().item():.3e}")
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
def test_default_draws_with_per_request_settings_match_convert_utterances(chain):
    models, wavs, prompt, _ = chain
    torch.manual_seed(1234)
    srv = serve.ConversionServer(*models, slots=SLOTS, max_frames=MAX_FRAMES, max_prompt_frames=MAX_PROMPT, **SERVER)
    tickets = [srv.submit(w, SR, prompt, method=m, steps=s) for w, (m, s) in zip(wavs, REQ)]
    got = srv.drain()
    bad = []
    for setting in sorted(set(OWN)):
        torch.manual_seed(1234)
        want = convert.convert_utterances(*models, wavs, SR, prompt, method=setting[0], steps=setting[1], max_batch=SLOTS)
        for i, tk in enumerate(tickets):
            if OWN[i] == setting and not torch.equal(got[tk], want[i]):
                bad.append(f"request {i} {setting}")
    assert not bad, bad


def _gpu_worker(rank, world, out_dir):
    from test_shard_convert import _chain
    dev = torch.device("cuda", torch.cuda.current_device())
    models, wavs, prompt = _chain(dev)
    g = torch.Generator().manual_seed(5)
    xs = [torch.randn((1, 100, convert.frame_plan(len(w), SR)["T"]), generator=g) for w in wavs]
    kw = dict(slots=2, max_frames=400, max_prompt_frames=80, **SERVER)
    res, lat, span = _serve_script(serve.ConversionServer(*models, group=dist.group.WORLD, **kw), wavs, prompt, xs, submit=rank == 0)
    out = {"rank": rank}
    if rank == 0:
        one_kw = dict(kw, slots=2 * world)                  # as many slots as the two ranks together: the same admission ticks
        one, one_lat, one_span = _serve_script(serve.ConversionServer(*models, **one_kw), wavs, prompt, xs)
        out["one_gpu"] = [i for i in range(6) if not (torch.equal(res[i], one[i]) and torch.equal(lat[i], one_lat[i]))]
        out["alone"] = []
        for i in range(6):
            la, aa = _alone(models, wavs, prompt, xs[i], i)
            if not (torch.equal(lat[i], la) and torch.equal(res[i], aa)):
                out["alone"].append(i)
        out["span"] = span == one_span
    else:
        out["empty"] = res == {} and lat == {}
    path = os.path.join(out_dir, f"rank{rank}.pt")
    torch.save(out, path)
    return path


@pytest.mark.gpu
def test_two_ranks_with_per_request_settings_equal_one_gpu(tmp_path):
    paths = _run(_gpu_worker, 2, str(tmp_path), backend="gloo", timeout=900)
    r0, r1 = [torch.load(p, weights_only=False) for p in paths]
    print(f"2 ranks over gloo: {r0}")
    assert r0["one_gpu"] == [], f"requests {r0['one_gpu']} differ from the one-GPU server"
    assert r0["alone"] == [], f"requests {r0['alone']} differ from convert_batch alone"
    assert r0["span"] is True, "the ranks retired requests at other ticks than one GPU"
    assert r1["empty"] is True
