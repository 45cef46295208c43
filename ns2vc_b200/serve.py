"""Conversion requests served as they arrive (continuous batching): the rows of one ragged denoiser batch at their own sampler steps.

A ``ConversionServer`` owns a fixed set of *slots*, the rows of one ragged program of geometry B = slots, T = max_frames,
S = max_prompt_frames.  It advances one *tick* at a time: one denoiser forward plus one sampler step for every occupied slot,
each slot at its own step index.  Requests wait in a FIFO queue; at the start of a tick the queued ones are *admitted* into the
free slots, and a request *retires* at the end of its ``steps``-th tick, leaving its slot free for the next one.  A request thus
waits at most one tick for a slot (plus its own admission), never for another request's whole run.

Each request brings its own sampler: DPM-Solver++ or UniPC at its own step count, rows of both methods side by side in one tick.
The coefficient structs of every schedule in use sit in one device table per method, each slot holds its schedule's base in
that table and its method tag, and its FiLM rows hold its own model times; a schedule not yet resident grows the tables and
re-captures the tick once.

Each request's result equals ``convert.convert_batch`` of that request alone with the same x_T, because every stage keeps row b
equal to utterance b run alone: the encoders run on the newcomers as one ragged batch, ``ns2vc_unet_prepare_cond_ragged`` keeps its
lengths in device tables, the FiLM rows are per row, and the row step kernel (``ns2vc_sampler_step_rows_seeded``) does the scalar step's
arithmetic with each row's own method and coefficient struct.

An admission re-prepares only the rows it changes: the newcomers' slots and the slots freed since the last admission, which
go back to length 1 and zero inputs (``ns2vc_unet_prepare_cond_rows`` and ``ns2vc_unet_time_table_rows`` write those rows
exactly as the full prepare and FiLM table would, and nothing else).  The residents' conditioning and FiLM rows stay as they
are, so an admission costs in proportion to its newcomers, not to the slot count.  Every slot is prepared again after the
weights are re-packed or when another caller has used the module's shared workspace.

A tick costs one forward of the whole slots x max_frames geometry whatever the occupancy (the ragged GEMMs compute padded rows),
so for a list known in advance ``convert.convert_utterances`` (longest-first batches) remains the faster call: the server buys
latency under arrivals, not peak throughput.

A seeded request (``submit(..., seed=)``) may also use DDPM or DDIM: its row draws its step noise in the row step kernel from its
own seed (``ns2vc_b200.noise``), so its audio is the same whatever else is in flight, and its x_T defaults to its seed's reserved
stream.  Unseeded DDPM / DDIM requests are refused as ``convert_utterances`` refuses them.  A DDPM request (1000 steps) grows the
FiLM table to 1000 x slots rows of ``ns2vc_unet_film_width`` floats each (see DESIGN.md §5 for its size at the real config).
"""
from __future__ import annotations

import collections
import os
import struct
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

from . import _lib, coefs, convert, noise, shard
from .api import default_schedule
from .convert import HOP, LATENT_CH
from .fused import DenoiserSession, _diffusion_buffers, _step_table, schedule_signature
from .pre_model import Voice

NAN_MESSAGE = "NaN in the denoiser input during the fused sampling run (reference model.py:404)"


class SlotTable:
    """The host bookkeeping of a server: the FIFO queue of tickets, the ticket in each slot and the tick at whose end it retires.
    No device state; every decision is made from tick numbers alone, so finding the finished rows needs no device sync.
    ``steps`` is the step count of a request enqueued without its own."""

    def __init__(self, slots: int, steps: int):
        self.slots, self.steps = int(slots), int(steps)
        self.queue: collections.deque = collections.deque()
        self.ticket: List[Optional[int]] = [None] * self.slots
        self.last: List[Optional[int]] = [None] * self.slots
        self._steps: Dict[int, int] = {}                    # queued ticket -> its step count

    def enqueue(self, ticket: int, steps: Optional[int] = None) -> None:
        steps = self.steps if steps is None else int(steps)
        if steps < 1:
            raise ValueError(f"steps must be >= 1, got {steps}")
        self.queue.append(ticket)
        self._steps[ticket] = steps

    def free_slots(self) -> List[int]:
        return [s for s in range(self.slots) if self.ticket[s] is None]

    def admit(self, tick: int) -> List[Tuple[int, int]]:
        """(slot, ticket) of the requests admitted at the start of ``tick``: the oldest queued ones, into the free slots in
        ascending order.  Each will run ticks ``tick .. tick + steps_b - 1``, steps_b its own step count."""
        out = []
        for s in self.free_slots():
            if not self.queue:
                break
            t = self.queue.popleft()
            self.ticket[s], self.last[s] = t, tick + self._steps.pop(t) - 1
            out.append((s, t))
        return out

    def retire(self, tick: int) -> List[Tuple[int, int]]:
        """(slot, ticket) of the requests whose last tick is ``tick``; their slots are free from the next tick on."""
        out = [(s, self.ticket[s]) for s in range(self.slots) if self.ticket[s] is not None and self.last[s] == tick]
        for s, _ in out:
            self.ticket[s] = self.last[s] = None
        return out

    @property
    def occupied(self) -> int:
        return sum(t is not None for t in self.ticket)

    @property
    def idle(self) -> bool:
        return not self.queue and self.occupied == 0


HEADER_FIELDS = 7          # per admission: ticket, rank, slot, samples, sr, T_b, S_b
_METHODS = ("dpmsolver", "unipc", "ddpm", "ddim")    # a row's method tag (NS2VC_ROW_DPM, _UNIPC, _DDPM, _DDIM) and its name
_METHOD_CODE = {m: i for i, m in enumerate(_METHODS)}
_KIND = {"dpmsolver": "dpm", "unipc": "unipc", "ddpm": "ddpm", "ddim": "ddim"}   # the sampler tables' name of each method
SETTINGS_FIELDS = 6        # per admission: method, steps, prompt is a Voice, seeded, seed, eta (its float64 bits)


def _eta_bits(eta: float) -> int:
    return struct.unpack("<q", struct.pack("<d", float(eta)))[0]


def _eta_of(bits: int) -> float:
    return struct.unpack("<d", struct.pack("<q", int(bits)))[0]


def place_requests(free: Sequence[int], n: int) -> List[int]:
    """The rank of each of the first queued requests, in FIFO order, on a server spread over several ranks: each goes to the
    rank with the most free slots (the lowest rank on ties), which then has one fewer.  Stops when no rank has a free slot, so
    the result has at most ``min(n, sum(free))`` entries."""
    free = [int(f) for f in free]
    out: List[int] = []
    for _ in range(int(n)):
        r = max(range(len(free)), key=lambda r: (free[r], -r)) if free else 0
        if not free or free[r] <= 0:
            break
        out.append(r)
        free[r] -= 1
    return out


def pack_header(admissions: Sequence[Sequence[int]], idle: bool, capacity: int) -> torch.Tensor:
    """One tick's int64 header: [count, idle, then HEADER_FIELDS values per admission], padded to ``capacity`` admissions so
    that every rank receives a tensor of one known size."""
    if len(admissions) > capacity:
        raise ValueError(f"{len(admissions)} admissions in a header for {capacity}")
    h = torch.zeros(2 + HEADER_FIELDS * capacity, dtype=torch.int64)
    h[0], h[1] = len(admissions), int(bool(idle))
    for i, a in enumerate(admissions):
        if len(a) != HEADER_FIELDS:
            raise ValueError(f"an admission has {len(a)} fields, not {HEADER_FIELDS}")
        h[2 + HEADER_FIELDS * i:2 + HEADER_FIELDS * (i + 1)] = torch.tensor([int(v) for v in a], dtype=torch.int64)
    return h


def unpack_header(h: torch.Tensor) -> Tuple[List[Tuple[int, ...]], bool]:
    """(admissions, idle) of ``pack_header``'s tensor."""
    v = h.cpu().tolist()
    n = int(v[0])
    return [tuple(v[2 + HEADER_FIELDS * i:2 + HEADER_FIELDS * (i + 1)]) for i in range(n)], bool(v[1])


class ConversionServer:
    """Waveform-to-waveform conversion of requests that arrive at any time; the caller owns the loop::

        srv = ConversionServer(content_model, pre_model, unet, vocoder, slots=8, max_frames=1024, max_prompt_frames=512)
        ticket = srv.submit(wav, sr, prompt_mel)       # FIFO order
        done = srv.tick()                              # {ticket: audio [T_b * 256]} of the requests that finished in this tick
        done = srv.drain()                             # tick until the queue and the slots are empty

    ``method`` is ``"unipc"`` (30 steps by default) or ``"dpmsolver"`` (40), as for ``convert_utterances``: the sampler of a
    request submitted without its own (``submit(..., method=, steps=)``).  A request whose
    denoiser input held a NaN comes back as an ``AssertionError`` (the reference's per-call guard, model.py:404) in place of its
    audio; the others carry on.  ``last_latents`` holds the latents [100, T_b] of the requests that finished in the last tick.

    The tick is captured as one CUDA graph on its ``DenoiserSession.CAPTURE_AFTER``-th run and replayed from then on
    (``NS2VC_GRAPH=0``: eager).  It holds the FiLM-row gather, the forward, the row step and the sampler's buffer rotation as
    stream-ordered device copies (see ``_body``).

    With a process ``group`` of more than one rank (one process per GPU, each rank with its models on its own device, every
    rank constructing the server with the same arguments), ``slots`` are per rank.  Rank 0 is the front: only it may
    ``submit``, and it places each newcomer, FIFO, on the rank with the most free slots (``place_requests``).  Every rank calls
    ``tick()`` and ``drain()`` in lockstep and mirrors the whole placement, so each knows every retirement tick.  Per tick, one
    int64 header broadcast from rank 0 carries the admissions and a global idle flag; when something is admitted, one float32
    broadcast carries the newcomers' wav | prompt | x_T and one int64 broadcast their (method, steps, prompt kind).  A prompt
    travels as its mel, or, for a ``Voice``, as its encoded spk | prompt rows, which the admitting rank uses without encoding.  Each rank admits and ticks its own slots, the ranks exchange one status
    flag (an exception on any rank raises a RuntimeError on every rank), and on ticks where something retires one ragged gather
    (``shard.gather_ragged``) brings each result's NaN flag, latent and audio to rank 0.  Rank 0 returns the results and holds
    ``last_latents``; the other ranks return {}.  The default x_T is drawn on rank 0 at ``submit``, as on one GPU, so every
    result equals the one-GPU server's.  Waveforms and prompts travel as float32.  ``group=None`` or a world of 1 is the
    one-GPU server."""

    def __init__(self, content_model, pre_model, unet, vocoder, slots: int = 8, max_frames: int = 1024, max_prompt_frames: int = 512,
                 method: str = "unipc", steps: Optional[int] = None, group: Optional[dist.ProcessGroup] = None):
        self.steps = convert._check_method(method, steps)
        if self.steps < 1:
            raise ValueError(f"steps must be >= 1, got {self.steps}")
        for name, v in (("slots", slots), ("max_frames", max_frames), ("max_prompt_frames", max_prompt_frames)):
            if int(v) < 1:
                raise ValueError(f"{name} must be >= 1, got {v}")
        self.models = (content_model, pre_model, unet, vocoder)
        self.method, self.kind = method, ("dpm" if method == "dpmsolver" else "unipc")
        self.B, self.T, self.S = int(slots), int(max_frames), int(max_prompt_frames)
        self.table = SlotTable(self.B, self.steps)
        self.ticks = 0                                      # ticks run so far (the index of the next one)
        self.last_latents: Dict[int, torch.Tensor] = {}
        self.admission_events: Optional[list] = None        # set to [] to record (start, end) CUDA events around each admission
        self._requests: Dict[int, dict] = {}
        self._next_ticket = 0
        self._sess: Optional[DenoiserSession] = None        # device state: allocated by the first tick
        self._freed: set = set()                            # slots retired since the last admission (their rows still hold the request)
        self.group = group
        self.world = dist.get_world_size(group) if group is not None else 1
        self.rank = dist.get_rank(group) if self.world > 1 else 0
        if self.world > 1:
            self.tables = [SlotTable(self.B, self.steps) for _ in range(self.world)]   # every rank's slots, mirrored on every rank
            self.table = self.tables[self.rank]
            self._pending: collections.deque = collections.deque()                     # rank 0: tickets not yet placed
            self._frames: Dict[int, int] = {}                                          # T_b of every placed request
            self._checked = False
            self._idle = True
            self.served = 0                                                            # requests retired on any rank so far

    # ------------------------------------------------------------------------------------------------ requests
    def submit(self, wav: torch.Tensor, sr: int, prompt_mel, x_T: Optional[torch.Tensor] = None,
               method: Optional[str] = None, steps: Optional[int] = None, seed: Optional[int] = None, eta: float = 0.0) -> int:
        """Queues one 1-D waveform at ``sr`` with its prompt and returns its ticket (increasing, FIFO).  The prompt is a mel
        [100, S_b], encoded at admission, or a ``Voice`` of this server's ``pre_model`` (``api.encode_voices``), used as it is;
        S_b may not exceed ``max_prompt_frames``.  ``x_T``
        ([1, 100, T_b] or [100, T_b]) defaults to ``torch.randn((1, 100, T_b))`` on the model's device, drawn here: requests
        submitted in list order get the draws ``convert_utterances`` makes for that list.  On several ranks only rank 0 submits.

        ``method`` (``"unipc"`` or ``"dpmsolver"``) and ``steps`` are this request's sampler; ``None`` takes the server's
        ``method`` / ``steps``.  The result equals ``convert_batch`` of the request alone with that method and step count.

        ``seed`` (an int in [0, 2**63)): the request's x_T, when not given, is ``noise.x_T`` of its seed, and ``method`` may also be
        ``"ddpm"`` (1000 steps) or ``"ddim"`` (``steps`` pairs, default 100; ``eta``: the reference's ``ddim_sampling_eta``), whose
        step noise the row draws from its seed.  The result then equals ``convert_batch(..., noise_seeds=[seed], eta=eta)`` of the
        request alone, bit for bit, whatever else is in flight."""
        if self.world > 1 and self.rank != 0:
            raise RuntimeError(f"submit() on rank {self.rank}: only rank 0 of the server's group takes requests")
        method = self.method if method is None else method
        if steps is None and method not in ("ddpm", "ddim"):
            steps = self.steps
        steps = convert._check_method(method, steps, seeded=seed is not None)
        if steps < 1:
            raise ValueError(f"steps must be >= 1, got {steps}")
        seeds = convert._check_seeds(None if seed is None else [seed], eta, method, 1)
        eta = float(eta)
        plan = convert._check_inputs([wav], sr, [prompt_mel], None if x_T is None else [x_T])[0]
        if isinstance(prompt_mel, Voice):
            self.models[1].check_voice(prompt_mel, self._device(), "prompt")
        if plan["T"] > self.T:
            raise ValueError(f"the waveform is {plan['T']} frames, more than max_frames={self.T}")
        S_b = convert.prompt_frames(prompt_mel)
        if S_b > self.S:
            raise ValueError(f"the prompt is {S_b} frames, more than max_prompt_frames={self.S}")
        if x_T is None:
            x_T = noise.x_T(seeds, LATENT_CH, [plan["T"]], self._device()) if seeds is not None \
                else torch.randn((1, LATENT_CH, plan["T"]), device=self._device())
        ticket = self._next_ticket
        self._next_ticket += 1
        self._requests[ticket] = dict(wav=wav, sr=int(sr), prompt=prompt_mel, x_T=x_T, plan=plan, T=plan["T"], S=S_b, method=method,
                                      steps=steps, seed=None if seeds is None else seeds[0], eta=eta)
        if self.world > 1:
            self._pending.append(ticket)
        else:
            self.table.enqueue(ticket, steps)
        return ticket

    @torch.no_grad()
    def tick(self) -> Dict[int, object]:
        """Admits queued requests into the free slots, runs one tick and returns {ticket: audio [T_b * 256]} (or an
        ``AssertionError``) for the requests that finished in it.  Does nothing when the queue and the slots are empty."""
        if self.world > 1:
            return self._tick_group()
        if self.table.idle:
            return {}
        t = self.ticks
        self._step(self.table.admit(t))
        self.ticks += 1
        return self._retire(t)

    def drain(self) -> Dict[int, object]:
        """Ticks until the queue and the slots are empty (on several ranks: everywhere, and every rank returns in the same
        tick); returns every result."""
        out: Dict[int, object] = {}
        if self.world > 1:
            while True:
                out.update(self.tick())
                if self._idle:
                    return out
        while not self.table.idle:
            out.update(self.tick())
        return out

    def _step(self, new: List[Tuple[int, int]]):
        """The device work of one tick on this server's slots: the admission of ``new`` (slot, ticket), then the tick."""
        stale = self._setup()
        stale = self._resident([self._setting(self._requests[tk]) for _, tk in new]) or stale
        if new:
            self._admit(new, full=stale or not self._owns_cond())
        elif stale:
            self._prepare_all()
        elif not self._owns_cond():
            self._sess.prepare()                            # another caller used the module's shared workspace since the last tick
        self._run_tick()

    # ------------------------------------------------------------------------------------------------ several ranks
    def _coll_device(self) -> Optional[torch.device]:
        return self._device() if "nccl" in str(dist.get_backend(self.group)) else None

    def _broadcast(self, t: torch.Tensor) -> torch.Tensor:
        dev = self._coll_device()
        t = t.to(dev) if dev is not None else t.cpu()
        dist.broadcast(t, src=dist.get_global_rank(self.group, 0), group=self.group)
        return t.cpu()

    def _check_group_args(self):
        """Raises ValueError on every rank unless every rank built the server with the same arguments (one all-gather)."""
        key = torch.tensor([self.B, self.T, self.S, self.steps, int(self.kind == "dpm")], dtype=torch.int64)
        keys = shard._all_gather(key, self.group, self._coll_device()).view(self.world, -1).cpu()
        self._checked = True
        if not bool((keys == keys[0]).all()):
            raise ValueError("the ranks built their servers with different arguments (slots, max_frames, max_prompt_frames, steps, "
                             f"dpmsolver per rank: {keys.tolist()})")

    def _header(self, t: int) -> torch.Tensor:
        """Rank 0: places the queued requests and packs the tick's header."""
        free = {r: tab.free_slots() for r, tab in enumerate(self.tables)}
        adm = []
        for r in place_requests([len(free[r]) for r in range(self.world)], len(self._pending)):
            tk = self._pending.popleft()
            q = self._requests[tk]
            adm.append((tk, r, free[r].pop(0), q["wav"].numel(), q["sr"], q["T"], q["S"]))
        idle = not adm and all(tab.occupied == 0 for tab in self.tables)
        return pack_header(adm, idle, self.world * self.B)

    def _payload(self, adm, voiced: Sequence[bool]) -> List[Tuple[torch.Tensor, object, torch.Tensor]]:
        """Every newcomer's (wav, prompt, x_T [1, 100, T_b]) as sent by rank 0 in one float32 broadcast.  The prompt is its mel
        [100, S_b], or (``voiced``) its ``Voice``, sent as its spk | prompt rows and rebuilt on this rank's device with this
        rank's ``pre_model``."""
        pm = self.models[1]
        ph, ro = pm.voice_widths() if any(voiced) else (0, 0)
        sizes = [(n, ph + Sb * ro if v else LATENT_CH * Sb, LATENT_CH * Tb) for (_, _, _, n, _, Tb, Sb), v in zip(adm, voiced)]
        if self.rank == 0:
            parts = []
            for tk, *_ in adm:
                q = self._requests[tk]
                p = q["prompt"]
                prompt = [p.spk, p.prompt.reshape(-1)] if isinstance(p, Voice) else [p.reshape(-1)]
                parts += [q["wav"].reshape(-1)] + prompt + [q["x_T"].reshape(-1)]
            dev = self._coll_device()
            flat = torch.cat([p.to(dev if dev is not None else "cpu", torch.float32) for p in parts])
        else:
            flat = torch.empty(sum(sum(z) for z in sizes), dtype=torch.float32)
        flat = self._broadcast(flat)
        out, off = [], 0
        for (n, np_, nx), (_, _, _, _, _, Tb, Sb), v in zip(sizes, adm, voiced):
            p = flat[off + n:off + n + np_]
            if v:
                dev = self._device()
                p = Voice(p[:ph].to(dev), p[ph:].view(Sb, ro).to(dev), pm)
            else:
                p = p.view(LATENT_CH, Sb)
            out.append((flat[off:off + n], p, flat[off + n + np_:off + n + np_ + nx].view(1, LATENT_CH, Tb)))
            off += n + np_ + nx
        return out

    def _settings(self, adm) -> List[Tuple[str, int, bool, Optional[int], float]]:
        """Every newcomer's (method, steps, whether its prompt is a ``Voice``, seed or None, eta) as sent by rank 0 in one int64
        broadcast (eta as its float64 bits): each rank needs them to mirror the retirements, and the newcomer's rank to run its
        schedule, draw its noise and read its prompt."""
        F = SETTINGS_FIELDS
        if self.rank == 0:
            vals = []
            for tk, *_ in adm:
                q = self._requests[tk]
                vals += [_METHOD_CODE[q["method"]], q["steps"], int(isinstance(q["prompt"], Voice)), int(q["seed"] is not None),
                         q["seed"] or 0, _eta_bits(q["eta"])]
            flat = torch.tensor(vals, dtype=torch.int64)
        else:
            flat = torch.zeros(F * len(adm), dtype=torch.int64)
        v = self._broadcast(flat).tolist()
        return [(_METHODS[v[F * i]], int(v[F * i + 1]), bool(v[F * i + 2]), int(v[F * i + 4]) if v[F * i + 3] else None,
                 _eta_of(v[F * i + 5])) for i in range(len(adm))]

    def _tick_group(self) -> Dict[int, object]:
        if not self._checked:
            self._check_group_args()
        t = self.ticks
        hdr = self._header(t) if self.rank == 0 else torch.zeros(2 + HEADER_FIELDS * self.world * self.B, dtype=torch.int64)
        adm, self._idle = unpack_header(self._broadcast(hdr))
        self.last_latents = {}
        if self._idle:
            return {}
        settings = self._settings(adm) if adm else []
        payload = self._payload(adm, [v for _, _, v, _, _ in settings]) if adm else []
        for (tk, r, slot, _, sr, Tb, Sb), (wav, prompt, x_T), (method, steps, _, seed, eta) in zip(adm, payload, settings):
            self.tables[r].enqueue(tk, steps)
            self._frames[tk] = Tb
            if r == self.rank and self.rank != 0:
                plan = convert._check_inputs([wav], sr, [prompt], [x_T])[0]
                self._requests[tk] = dict(wav=wav, sr=sr, prompt=prompt, x_T=x_T, plan=plan, T=Tb, S=Sb, method=method, steps=steps,
                                          seed=seed, eta=eta)
            elif r != self.rank:
                self._requests.pop(tk, None)               # (rank 0: placed elsewhere)
        news = [tab.admit(t) for tab in self.tables]
        placed = sorted((r, s, tk) for r, new in enumerate(news) for s, tk in new)
        if placed != sorted((r, s, tk) for tk, r, s, *_ in adm):
            raise RuntimeError(f"rank {self.rank}: the mirrored placement {placed} differs from rank 0's")
        err: Optional[Exception] = None
        local: List[torch.Tensor] = []
        dones: List[List[Tuple[int, int]]] = [[] for _ in range(self.world)]
        try:
            if self.table.occupied:
                self._step(news[self.rank])
            dones = [tab.retire(t) for tab in self.tables]   # (after the step: an admission zeroes the slots it sees free)
            for flag, lat, audio in self._collect(dones[self.rank]):
                local.append(torch.cat([torch.tensor([float(flag)], device=lat.device), lat.reshape(-1), audio.reshape(-1)]))
        except Exception as e:                              # noqa: BLE001 (re-raised below on every rank)
            err = e
        failed = shard._all_gather(torch.tensor([err is not None], dtype=torch.int32), self.group,
                                   self._coll_device()).nonzero().flatten().tolist()
        if failed:
            mine = f"; rank {self.rank} raised {type(err).__name__}: {err}" if err is not None else ""
            raise RuntimeError(f"server tick {t} failed on rank(s) {failed}{mine}") from err
        self.ticks += 1
        if not any(dones):
            return {}
        order = [tk for done in dones for _, tk in done]
        index = {tk: i for i, tk in enumerate(order)}
        plan = [[[index[tk] for _, tk in done]] if done else [] for done in dones]
        sizes = [1 + (LATENT_CH + HOP) * self._frames[tk] for tk in order]
        got = shard.gather_ragged(local, plan, sizes, self.group, self._coll_device())
        frames = [self._frames.pop(tk) for tk in order]
        self.served += len(order)
        if self.rank != 0:
            return {}
        out: Dict[int, object] = {}
        for tk, Tb, v in zip(order, frames, got):
            if v[0].item() != 0:
                out[tk] = AssertionError(NAN_MESSAGE)
                continue
            self.last_latents[tk] = v[1:1 + LATENT_CH * Tb].view(LATENT_CH, Tb)
            out[tk] = v[1 + LATENT_CH * Tb:]
        return dict(sorted(out.items()))

    # ------------------------------------------------------------------------------------------------ device state
    @property
    def _unet(self):
        return self.models[2]

    def _device(self) -> torch.device:
        return next(self._unet.parameters()).device

    def _owns_cond(self) -> bool:
        """True while the module's shared workspace holds this server's prepared conditioning."""
        return self._sess._prepared and self._unet.__dict__.get("_cond_owner") is self._sess

    def _setup(self) -> bool:
        """Allocates the device state on the first call.  True when the weights were re-packed since the last tick: the captured
        tick, the prepared conditioning and the FiLM table are then stale."""
        sess = self._sess
        if sess is not None:
            wsig = sess._wsig
            sess._sync_engine()
            if sess._wsig == wsig:
                return False
            self._graph, self._runs = None, 0
            return True
        unet = self._unet
        dev = self._device()
        B, T, S = self.B, self.T, self.S
        f32 = dict(dtype=torch.float32, device=dev)
        Cc = unet.cfg.in_channels - unet.latent_channels
        content = torch.zeros((B, Cc, T), **f32) if Cc > 0 else None
        prompt = torch.zeros((B, S, unet.cfg.cross_attention_dim), **f32)
        sess = DenoiserSession(unet, content, prompt, None, T=T, content_lengths=[1] * B, prompt_lengths=[1] * B)
        if sess.Cl != sess.Co:
            raise ValueError("the server needs out_channels == latent channels (x_start parameterisation)")
        self._sess, self._L = sess, _lib.lib()
        self._clen, self._plen = [1] * B, [1] * B
        self._fw = int(self._L.ns2vc_unet_film_width(sess.h))
        self._sched: Dict[Tuple[str, int, float], dict] = {}  # (method, steps, eta) -> its tag, its base in its method's table, its t column
        self._tab: Dict[str, list] = {k: [] for k in ("dpm", "unipc", "ddpm", "ddim")}   # the step records of every resident schedule
        self._coef: Dict[str, Optional[torch.Tensor]] = {k: None for k in self._tab}
        self._tvals = torch.zeros((0, B), **f32)           # [K, B]: the model time of slot b's request at its step k
        self._film = torch.empty((B, self._fw), **f32)
        self._rowbase = torch.arange(B, dtype=torch.int64, device=dev)
        self._k = torch.full((B,), -1, dtype=torch.int32, device=dev)
        self._tag, self._base = [0] * B, [0] * B            # each slot's method tag and schedule base (host copies)
        self._row_tag = torch.zeros((B,), dtype=torch.int32, device=dev)
        self._row_base = torch.zeros((B,), dtype=torch.int32, device=dev)
        self._nan = torch.zeros((B,), dtype=torch.int32, device=dev)
        self._seeds = torch.zeros((B,), dtype=torch.int64, device=dev)   # each slot's noise seed (read by DDPM / DDIM rows only)
        shape = (B, sess.Cl, T)
        self._buf = {n: torch.zeros(shape, **f32) for n in ("x_in", "m0", "m1", "x_prev", "m_new", "x_t", "x_new", "out")}
        self._x = self._buf["x_in"]                         # the denoiser input; after a request's last tick, its latent
        self._resident([(self.method, self.steps, 0.0)])
        self._tvals.copy_(self._sched[(self.method, self.steps, 0.0)]["t"][:, None].expand(self.steps, B))
        return False

    @staticmethod
    def _setting(q: dict) -> Tuple[str, int, float]:
        """A request's schedule key (method, steps, eta)."""
        return q["method"], q["steps"], q["eta"]

    def _resident(self, settings: Sequence[Tuple[str, int, float]]) -> bool:
        """Makes every (method, steps, eta) schedule of ``settings`` resident.  The tables only grow: a schedule not yet resident
        appends its coefficient structs to its method's table (the residents keep their bases), re-allocates that table and,
        when it is the longest yet, the FiLM table, and drops the captured tick.  True when that happened: the FiLM rows of
        every slot must then be written again (``_prepare_all``)."""
        new = [st for st in dict.fromkeys(settings) if st not in self._sched]
        if not new:
            return False
        ns, dev, B = default_schedule(), self._device(), self.B
        for method, steps, eta in new:
            kind = _KIND[method]
            if kind == "ddpm":
                tab = coefs.ddpm_table(_diffusion_buffers(), range(steps - 1, -1, -1))
            elif kind == "ddim":
                buf = _diffusion_buffers()
                tab = coefs.ddim_table(buf, buf["betas"].shape[0], steps, eta)
            else:
                ts = torch.linspace(ns.T, 1.0 / ns.total_N, steps + 1)
                extra = True if kind == "dpm" else "bh2"   # lower_order_final / variant, as sample_latents runs them
                tab = _step_table(kind, ns, ts, extra, (kind, tuple(float(v) for v in ts), extra, schedule_signature(ns)))
            self._sched[(method, steps, eta)] = dict(tag=_METHOD_CODE[method], base=len(self._tab[kind]),
                                                     t=coefs.t_inputs(tab, 1, "cpu")[:, 0])
            self._tab[kind] = self._tab[kind] + list(tab)
            self._coef[kind] = coefs.c_table(self._tab[kind], dev)[0]
        K = max(steps for _, steps, _ in self._sched)
        if K > self._tvals.shape[0]:
            tv = torch.zeros((K, B), dtype=torch.float32, device=dev)
            tv[:self._tvals.shape[0]] = self._tvals
            self._tvals = tv
            L, h = self._L, self._sess.h
            self._film_table = torch.empty(int(L.ns2vc_unet_time_table_floats(h, K * B)), dtype=torch.float32, device=dev)
            self._film_rows = self._film_table[:K * B * self._fw].view(K * B, self._fw)
        self._graph, self._runs = None, 0
        return True

    def _admit(self, new: List[Tuple[int, int]], full: bool):
        """Encodes the newcomers as one ragged batch per input rate and writes them into their slots.  Then prepares the rows
        of the newcomers and of the slots freed since the last admission (``full``: every slot)."""
        cm, pm, _, _ = self.models
        sess, dev = self._sess, self._device()
        ev = None
        if self.admission_events is not None:
            ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            ev[0].record()
        by_rate: Dict[int, List[Tuple[int, int]]] = {}
        for s, tk in new:
            by_rate.setdefault(self._requests[tk]["sr"], []).append((s, tk))
        for sr, group in by_rate.items():
            reqs = [self._requests[tk] for _, tk in group]
            front = convert.encode_front(cm, pm, [r["wav"] for r in reqs], sr, [r["prompt"] for r in reqs], [r["plan"] for r in reqs], dev)
            for j, ((s, _), r) in enumerate(zip(group, reqs)):
                Tb, Sb = r["T"], r["S"]
                if sess.content is not None:
                    sess.content[s].zero_()
                    sess.content[s, :, :Tb] = front["content"][:Tb, j].t()
                sess.prompt[s].zero_()
                sess.prompt[s, :Sb] = front["prompt"][:Sb, j]
                for b in self._buf.values():
                    b[s].zero_()
                self._x[s, :, :Tb] = r["x_T"].reshape(LATENT_CH, Tb).to(dev, torch.float32)
                self._clen[s], self._plen[s] = Tb, Sb
                sched = self._sched[self._setting(r)]
                self._seeds[s] = r["seed"] or 0
                self._tvals[:r["steps"], s] = sched["t"].to(dev)          # the FiLM rows (k, s) hold this request's own times
                self._tag[s], self._base[s] = sched["tag"], sched["base"]
        occupied = {s for s in range(self.B) if self.table.ticket[s] is not None}
        for s in range(self.B):
            if s not in occupied:                           # empty slots: length 1, zero inputs
                if sess.content is not None:
                    sess.content[s].zero_()
                sess.prompt[s].zero_()
                for b in self._buf.values():
                    b[s].zero_()
                self._clen[s], self._plen[s] = 1, 1
        slots = torch.tensor([s for s, _ in new], dtype=torch.int64, device=dev)
        self._row_tag.copy_(torch.tensor(self._tag, dtype=torch.int32))
        self._row_base.copy_(torch.tensor(self._base, dtype=torch.int32))
        self._k.index_fill_(0, slots, 0)
        self._nan.index_fill_(0, slots, 0)
        if full:
            self._prepare_all()
        else:
            self._prepare_rows(sorted({s for s, _ in new} | (self._freed - occupied)))
        self._freed.clear()
        if ev is not None:
            ev[1].record()
            self.admission_events.append(ev)

    def _prepare_all(self):
        """The conditioning of every slot (ns2vc_unet_prepare_cond_ragged) and the FiLM rows of all steps x slots."""
        sess = self._sess
        sess.clen.copy_(torch.tensor(self._clen, dtype=torch.int64))
        sess.plen.copy_(torch.tensor(self._plen, dtype=torch.int64))
        sess.prepare()
        sess.time_table(self._tvals, self._film_table)

    def _prepare_rows(self, rows: List[int]):
        """The conditioning and the FiLM rows (every step) of the listed slots only; the other slots' stay as they are."""
        sess = self._sess
        sess.clen.copy_(torch.tensor(self._clen, dtype=torch.int64))
        sess.plen.copy_(torch.tensor(self._plen, dtype=torch.int64))
        sess.prepare_rows(rows)
        sess.time_table_rows(self._tvals, self._film_table, rows)

    def _body(self):
        """One tick: the FiLM row (k_b, b) of every slot, the forward, the row step of every slot with its own method and
        schedule (``ns2vc_sampler_step_rows_seeded``; DDPM / DDIM rows draw their noise from their seeds), then the rotation of the sampler's buffers: m1 <- m0 <- m_new, x_prev <- x_t,
        x_in <- x_new, the same for both methods (a DPM-Solver++ row never reads m1 or x_prev).  The rotation is four device
        copies inside the one captured graph rather than a cycle of graphs over rotating pointers: UniPC's 3-deep history and
        2-deep state would need lcm(3, 2) = 6 captures of the whole forward, and the copies move 4 x slots x 100 x max_frames
        floats, small next to one forward."""
        sess, L, b = self._sess, self._L, self._buf
        idx = self._k.clamp(min=0).to(torch.int64) * self.B + self._rowbase       # empty slots read step 0's row (their output is discarded)
        torch.index_select(self._film_rows, 0, idx, out=self._film)
        sess.forward(b["x_in"], None, b["out"], film_rows=self._film)
        n, stream = sess.Cl * self.T, sess._stream()
        dpm, unipc, ddpm, ddim = (self._coef[k].data_ptr() if self._coef[k] is not None else None
                                  for k in ("dpm", "unipc", "ddpm", "ddim"))
        with torch.cuda.device(sess.dev):
            _lib.check(L.ns2vc_sampler_step_rows_seeded(
                b["x_in"].data_ptr(), b["out"].data_ptr(), b["m0"].data_ptr(), b["m1"].data_ptr(), b["x_prev"].data_ptr(), dpm, unipc,
                ddpm, ddim, self._seeds.data_ptr(), self.T, self._row_tag.data_ptr(), self._row_base.data_ptr(), self._k.data_ptr(),
                b["m_new"].data_ptr(), b["x_t"].data_ptr(), b["x_new"].data_ptr(), n, self.B, self._nan.data_ptr(), stream))
        b["m1"].copy_(b["m0"])
        b["m0"].copy_(b["m_new"])
        b["x_prev"].copy_(b["x_t"])
        b["x_in"].copy_(b["x_new"])

    def _run_tick(self):
        self._runs += 1
        if os.environ.get("NS2VC_GRAPH", "1") == "0" or (self._graph is None and self._runs < DenoiserSession.CAPTURE_AFTER):
            self._body()
            return
        if self._graph is None:
            torch.cuda.synchronize(self._sess.dev)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._body()
            self._graph = g
        self._graph.replay()

    def _retire(self, t: int) -> Dict[int, object]:
        done = self.table.retire(t)
        self.last_latents = {}
        if not done:
            return {}
        out: Dict[int, object] = {}
        for (_, tk), (flag, lat, audio) in zip(done, self._collect(done)):
            if flag != 0:
                out[tk] = AssertionError(NAN_MESSAGE)
            else:
                out[tk] = audio
                self.last_latents[tk] = lat
        return dict(sorted(out.items()))

    def _collect(self, done: List[Tuple[int, int]]) -> List[Tuple[int, torch.Tensor, torch.Tensor]]:
        """(NaN flag, latent [100, T_b], audio [T_b * 256]) of each retired (slot, ticket), in order; a flagged request's
        latent and audio are zeros.  Frees the slots and forgets the requests."""
        if not done:
            return []
        dev = self._device()
        slots = torch.tensor([s for s, _ in done], dtype=torch.int64, device=dev)
        flags = self._nan.index_select(0, slots).tolist()
        self._k.index_fill_(0, slots, -1)
        self._freed.update(s for s, _ in done)
        res: Dict[int, Tuple[torch.Tensor, torch.Tensor]] = {}
        ok = [(s, tk) for (s, tk), f in zip(done, flags) if f == 0]
        if ok:
            tl = [self._requests[tk]["T"] for _, tk in ok]
            rows = torch.tensor([s for s, _ in ok], dtype=torch.int64, device=dev)
            lat = self._x.index_select(0, rows)[:, :, :max(tl)].contiguous()
            audio = self.models[3].decode(lat, torch.tensor(tl, dtype=torch.int64))
            for j, (_, tk) in enumerate(ok):
                res[tk] = (lat[j, :, :tl[j]], audio[j, :tl[j] * HOP])
        out = []
        for (_, tk), f in zip(done, flags):
            Tb = self._requests[tk]["T"]
            lat, audio = res.get(tk, (torch.zeros((LATENT_CH, Tb), device=dev), torch.zeros(Tb * HOP, device=dev)))
            out.append((int(f), lat, audio))
        for _, tk in done:
            del self._requests[tk]
        return out
