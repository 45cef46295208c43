"""Fused sampling loops: UNet forward (C-ABI) + one fused sampler-step kernel per step.

``DenoiserSession`` is the explicit fast API (device-resident x, content, prompt):
conditioning prepared once per utterance batch, per-step scalars precomputed on the host
(``coefs.py``), no host synchronisation inside the loop (the reference syncs every step on
``assert torch.isnan(x).any() == False``, model.py:404).

``try_fused_dpm`` / ``try_fused_unipc`` let the drop-in ``DPM_Solver`` / ``UniPC`` classes
take this path when the model closure they were given turns out to wrap our UNet (detected by
tracing the first model call), so ``model.py:621-686`` benefits unchanged.
"""
from __future__ import annotations

import collections
import ctypes as C
import hashlib
import os
from typing import Optional, Sequence

import torch

from . import _lib, coefs, noise as seeded_noise
from .unet import UNet1DConditionModel, trace_calls


def schedule_signature(ns) -> tuple:
    """Content key of a noise schedule.  The reference builds a NEW NoiseScheduleVP inside every ``sample()``
    (model.py:621-622, 655-656), so object identity is useless as a cache key (and a recycled ``id()`` could
    alias a different beta table); two schedules with the same knots share tables and captured graphs."""
    if getattr(ns, "schedule", None) == "discrete":
        la = ns.log_alpha_array.detach().to("cpu", torch.float32).contiguous()
        return ("discrete", int(ns.total_N), hashlib.sha1(la.numpy().tobytes()).hexdigest())
    return (str(getattr(ns, "schedule", "?")), float(getattr(ns, "beta_0", 0.0)), float(getattr(ns, "beta_1", 0.0)), int(getattr(ns, "total_N", 0)))


_TABLES = collections.OrderedDict()     # per-step scalars do not depend on the shape: shared by every session (the CLI: a new shape per slice)


def _step_table(kind, ns, ts, extra, key):
    tab = _TABLES.get(key)
    if tab is None:
        tab = coefs.dpmpp_2m_table(ns, ts, extra) if kind == "dpm" else coefs.unipc_bh2_table(ns, ts, extra)
        _TABLES[key] = tab
        while len(_TABLES) > 16:
            _TABLES.popitem(last=False)
    else:
        _TABLES.move_to_end(key)
    return tab


class DenoiserSession:
    """One utterance-batch shape (B, T, S) on one GPU: UNet engine, static input buffers, prepared
    conditioning and the whole sampling loop captured as one CUDA graph.

    The C calls are stream-ordered and allocation-free, so the N-step loop (prepare_cond + the timestep
    table of all N evaluation times + N x (UNet forward + fused sampler step), every kernel linked to its
    predecessor by programmatic dependent launch) is captured once per (sampler, time grid, schedule) and
    replayed; new inputs are copied into the static buffers.  ``NS2VC_GRAPH=0`` disables the capture.

    The reference asserts ``not isnan(x)`` on the host before every denoiser call (model.py:404: one
    device->host sync per step).  Here the sampler-step kernel accumulates a device flag and the host checks
    it ONCE after the run, raising the same ``AssertionError``.

    Ragged batches: with ``content_lengths`` [B] (and optionally ``prompt_lengths`` [B], default S; no ``prompt_mask``)
    the session runs the engine's ragged program, for every sampling method.  Row b of a result is then utterance b
    sampled alone on x_T[b, :, :T_b], content[b, :, :T_b], prompt[b, :S_b]; its frames >= T_b are exactly 0 and input
    values past the lengths are never read.  x_T's padding is zeroed on entry and the denoiser output is zero there, so
    the DPM-Solver++ / UniPC state stays zero in the padding.  DDPM / DDIM noise is by default ``randn_like`` over the padded
    [B, C, T] tensor (the default generator advances as for one padded call, not as for B separate runs): a row then equals its
    B = 1 run when the caller injects the per-row noise (``noise``).  With ``seeds`` (one per row) each row draws its own noise
    in the step kernel from its seed (``ns2vc_b200.noise``), and row b equals utterance b run alone with seeds[b], bit for bit."""

    MAX_GRAPHS = 4                                           # LRU bound of captured loops per session
    CAPTURE_AFTER = 3                                        # the loop is captured on its third run, replayed from the fourth

    def __init__(self, unet: UNet1DConditionModel, content_BCT: Optional[torch.Tensor], prompt_BSC: torch.Tensor,
                 prompt_mask: Optional[torch.Tensor], T: Optional[int] = None, content_lengths=None, prompt_lengths=None):
        if not prompt_BSC.is_cuda:
            raise RuntimeError("DenoiserSession needs CUDA tensors (no CPU path)")
        self.unet = unet
        self.dev = prompt_BSC.device
        self.B, self.S = prompt_BSC.shape[0], prompt_BSC.shape[1]
        self.Cc = unet.cfg.in_channels - unet.latent_channels
        if self.Cc > 0:
            if content_BCT is None or content_BCT.shape[1] != self.Cc:
                raise ValueError(f"content must be [B, {self.Cc}, T]")
            self.T = content_BCT.shape[2]
        else:
            if T is None:
                raise ValueError("T is required when the model has no content channels")
            self.T = T
        f32 = dict(dtype=torch.float32, device=self.dev)
        self.content = torch.empty((self.B, self.Cc, self.T), **f32) if self.Cc > 0 else None
        self.prompt = torch.empty((self.B, self.S, unet.cfg.cross_attention_dim), **f32)
        self.mask = torch.empty((self.B, self.S), dtype=torch.uint8, device=self.dev) if prompt_mask is not None else None
        self.ragged = content_lengths is not None
        if self.ragged:
            if prompt_mask is not None:
                raise ValueError("a ragged session takes prompt_lengths, not a prompt mask")
            self.clen = torch.empty((self.B,), dtype=torch.int64, device=self.dev)
            self.plen = torch.empty((self.B,), dtype=torch.int64, device=self.dev)
            self.keep = torch.empty((self.B, 1, self.T), dtype=torch.bool, device=self.dev)   # frame t < T_b
        elif prompt_lengths is not None:
            raise ValueError("prompt_lengths applies to ragged sessions (content_lengths); pass a prompt mask instead")
        self.L = _lib.lib()
        self.h = unet.engine(self.dev)
        self.Cl, self.Co = unet.latent_channels, unet.cfg.out_channels
        self.x_in = torch.empty((self.B, self.Cl, self.T), **f32)
        self.first_out = torch.empty((self.B, self.Co, self.T), **f32)   # step-0 model output handed in by the drop-in samplers
        self.nan_flag = torch.zeros((1,), dtype=torch.int32, device=self.dev)
        self.ws = unet.workspace(self.B, self.T, self.S, self.dev)     # the module's shared grow-only scratch buffer
        self._graphs = collections.OrderedDict()
        self._chains = collections.OrderedDict()             # DDPM / DDIM runs: device coefficient + time tables
        self._chunk_graphs = collections.OrderedDict()       # captured DDPM / DDIM chunks, by (kind, noise draws)
        self._chunk = None                                   # their static windows (allocated on the first such run)
        self._wsig = unet._wsig
        self.set_cond(content_BCT, prompt_BSC, prompt_mask, content_lengths, prompt_lengths)

    def set_cond(self, content_BCT, prompt_BSC, prompt_mask, content_lengths=None, prompt_lengths=None):
        """Copy a new utterance batch (same shapes; for a ragged session, new lengths) into the static buffers."""
        if (content_lengths is not None) != self.ragged:
            raise ValueError("content_lengths must be given exactly when the session is ragged")
        if self.ragged:
            cl = check_lengths(content_lengths, self.B, self.T, "content_lengths")
            pl = check_lengths(prompt_lengths, self.B, self.S, "prompt_lengths") if prompt_lengths is not None else [self.S] * self.B
            self.clen.copy_(torch.tensor(cl, dtype=torch.int64), non_blocking=False)
            self.plen.copy_(torch.tensor(pl, dtype=torch.int64), non_blocking=False)
            self.keep.copy_(torch.arange(self.T, device=self.dev)[None, None, :] < self.clen[:, None, None])
        if self.content is not None:
            self.content.copy_(content_BCT, non_blocking=True)
        self.prompt.copy_(prompt_BSC, non_blocking=True)
        if (prompt_mask is None) != (self.mask is None):
            raise ValueError("mask presence must not change within a session")
        if self.mask is not None:
            self.mask.copy_(prompt_mask.to(torch.bool), non_blocking=True)
        self._prepared = False

    def _stream(self):
        return torch.cuda.current_stream(self.dev).cuda_stream

    def prepare(self):
        if self.ragged:
            with torch.cuda.device(self.dev):
                _lib.check(self.L.ns2vc_unet_prepare_cond_ragged(
                    self.h, self.content.data_ptr() if self.content is not None else None,
                    (self.Cc * self.T) if self.content is not None else 0, self.prompt.data_ptr(), self.clen.data_ptr(),
                    self.plen.data_ptr(), self.B, self.T, self.S, self.ws.data_ptr(), self._stream()))
            self._prepared = True
            self.unet.__dict__["_cond_owner"] = self
            return
        with torch.cuda.device(self.dev):
            _lib.check(self.L.ns2vc_unet_prepare_cond(
                self.h, self.content.data_ptr() if self.content is not None else None,
                (self.Cc * self.T) if self.content is not None else 0, self.prompt.data_ptr(),
                self.mask.data_ptr() if self.mask is not None else None, self.B, self.T, self.S, self.ws.data_ptr(), self._stream()))
        self._prepared = True
        self.unet.__dict__["_cond_owner"] = self                 # the shared workspace holds THIS session's conditioning now

    def forward(self, x: torch.Tensor, t: torch.Tensor, out: torch.Tensor, film_rows: Optional[torch.Tensor] = None):
        """x [B,Cl,T] fp32 contiguous, t [B] fp32 (or B precomputed FiLM rows), out [B,Co,T] fp32 — all on the session device."""
        if not self._prepared or self.unet.__dict__.get("_cond_owner") is not self:
            self.prepare()
        with torch.cuda.device(self.dev):
            if film_rows is not None:
                _lib.check(self.L.ns2vc_unet_forward_film(self.h, x.data_ptr(), self.Cl * self.T, film_rows.data_ptr(), out.data_ptr(),
                                                          self.B, self.T, self.S, self.ws.data_ptr(), self._stream()))
            else:
                _lib.check(self.L.ns2vc_unet_forward(self.h, x.data_ptr(), self.Cl * self.T, t.data_ptr(), out.data_ptr(),
                                                     self.B, self.T, self.S, self.ws.data_ptr(), self._stream()))

    def prepare_rows(self, rows: Sequence[int]):
        """Ragged sessions: the conditioning of the listed rows only (``ns2vc_unet_prepare_cond_rows``), from the static buffers
        and length tensors as they stand now; every other row keeps what the last ``prepare()`` wrote.  Needs that prepare()
        to be this session's and the last one on the module's workspace."""
        if not self.ragged:
            raise ValueError("prepare_rows needs a ragged session")
        if not self._prepared or self.unet.__dict__.get("_cond_owner") is not self:
            raise RuntimeError("prepare_rows() needs this session's prepare() first")
        rows = [int(r) for r in rows]
        with torch.cuda.device(self.dev):
            _lib.check(self.L.ns2vc_unet_prepare_cond_rows(
                self.h, self.content.data_ptr() if self.content is not None else None,
                (self.Cc * self.T) if self.content is not None else 0, self.prompt.data_ptr(), self.clen.data_ptr(),
                self.plen.data_ptr(), (C.c_int * len(rows))(*rows), len(rows), self.B, self.T, self.S, self.ws.data_ptr(),
                self._stream()))

    def time_table(self, tvals: torch.Tensor, table: torch.Tensor):
        """FiLM rows of every evaluation time of a run (tvals [steps, B] fp32) into ``table`` (needs prepare())."""
        with torch.cuda.device(self.dev):
            _lib.check(self.L.ns2vc_unet_time_table(self.h, tvals.data_ptr(), tvals.numel(), table.data_ptr(), self.B, self.T, self.S,
                                                    self.ws.data_ptr(), self._stream()))

    def time_table_rows(self, tvals: torch.Tensor, table: torch.Tensor, rows: Sequence[int]):
        """``time_table`` for the listed rows only: FiLM rows k * B + b for b in ``rows`` and every step k; the others are
        left as they are."""
        rows = [int(r) for r in rows]
        with torch.cuda.device(self.dev):
            _lib.check(self.L.ns2vc_unet_time_table_rows(self.h, tvals.data_ptr(), tvals.numel() // self.B, (C.c_int * len(rows))(*rows),
                                                         len(rows), table.data_ptr(), self.B, self.T, self.S, self.ws.data_ptr(),
                                                         self._stream()))

    # ------------------------------------------------------------------ loop bodies (eager or under capture)
    def _film(self, ent, k):
        fw = ent["film_width"]
        return ent["table"][k * self.B * fw:(k + 1) * self.B * fw]

    def _body_dpm(self, ent, use_first):
        x = self.x_in.clone()
        n = x.numel()
        x_next, out = torch.empty_like(x), torch.empty_like(x)
        m_a, m_b = torch.empty_like(x), torch.empty_like(x)
        stream = self._stream()
        for k, st in enumerate(ent["steps"]):
            if k == 0 and use_first:
                out.copy_(self.first_out)
            else:
                self.forward(x, ent["tvals"][k], out, film_rows=self._film(ent, k))
            c = coefs.c_struct(st)
            with torch.cuda.device(self.dev):
                _lib.check(self.L.ns2vc_dpm_step(x.data_ptr(), out.data_ptr(), m_b.data_ptr(), C.byref(c), m_a.data_ptr(),
                                                 x_next.data_ptr(), n, self.nan_flag.data_ptr(), stream))
            x, x_next = x_next, x
            m_a, m_b = m_b, m_a
        return x

    def _body_unipc(self, ent, use_first):
        x_prev = self.x_in                                 # x at the previous time point (corrector base); never written
        x_eval = x_prev                                    # where the model is evaluated
        n = x_prev.numel()
        out = torch.empty_like(x_prev)
        m0 = m1 = None
        stream = self._stream()
        for k, st in enumerate(ent["steps"]):
            if k == 0 and use_first:
                out.copy_(self.first_out)
            else:
                self.forward(x_eval, ent["tvals"][k], out, film_rows=self._film(ent, k))
            m_t = torch.empty_like(x_prev)
            x_t = torch.empty_like(x_prev) if st.corr_order > 0 else None
            x_pred = torch.empty_like(x_prev)
            c = coefs.c_struct(st)
            with torch.cuda.device(self.dev):
                _lib.check(self.L.ns2vc_unipc_step(
                    x_prev.data_ptr(), x_eval.data_ptr(), out.data_ptr(), m0.data_ptr() if m0 is not None else None,
                    m1.data_ptr() if m1 is not None else None, C.byref(c), m_t.data_ptr(),
                    x_t.data_ptr() if x_t is not None else None, x_pred.data_ptr(), n, self.nan_flag.data_ptr(), stream))
            # history m1 <- m0 <- m_t ; corrector base <- corrected x_t (x_eval itself at k = 0)
            m1, m0 = m0, m_t
            x_prev = x_t if x_t is not None else x_eval
            x_eval = x_pred
        return x_eval

    def _loop(self, kind, ent, use_first):
        """prepare_cond + timestep table + the N-step loop; returns the final latents (a fresh tensor)."""
        self.nan_flag.zero_()
        self.prepare()
        self.time_table(ent["tvals"], ent["table"])
        res = self._body_dpm(ent, use_first) if kind == "dpm" else self._body_unipc(ent, use_first)
        return res.clone()

    def _unpad(self, x: torch.Tensor) -> torch.Tensor:
        """Ragged sessions: zero every frame past its utterance's length (in place; NaN-safe)."""
        if self.ragged:
            x.masked_fill_(~self.keep, 0.0)
        return x

    def _check_nan(self, flags=None):
        if int((self.nan_flag if flags is None else flags).max().item()) != 0:
            # same exception type as the reference's per-call guard (model.py:404)
            raise AssertionError("NaN in the denoiser input during the fused sampling run (reference model.py:404)")

    def _sync_engine(self):
        if self.unet._wsig != self._wsig:                  # weights were re-packed: captured graphs are stale
            self._graphs.clear()
            self._chunk_graphs.clear()
            for ent in self._chains.values():
                ent["graphs"].clear()
            self.h = self.unet.engine(self.dev)
            self._wsig = self.unet._wsig
            self._prepared = False

    def _run(self, kind, x_T, ns, ts, first_out, extra):
        assert self.Cl == self.Co, "x_start parameterisation needs out_channels == latent channels"
        self._sync_engine()
        self._unpad(self.x_in.copy_(x_T, non_blocking=True))
        use_first = first_out is not None
        if use_first:
            self.first_out.copy_(first_out, non_blocking=True)
        key = (kind, tuple(float(v) for v in ts), extra, schedule_signature(ns), use_first)
        use_graph = os.environ.get("NS2VC_GRAPH", "1") != "0"
        ent = self._graphs.get(key)
        if ent is None:
            steps = _step_table(kind, ns, ts, extra, key[:4])
            tvals = coefs.t_inputs(steps, self.B, self.dev)
            nrows = tvals.numel()
            table = torch.empty(int(self.L.ns2vc_unet_time_table_floats(self.h, nrows)), dtype=torch.float32, device=self.dev)
            ent = {"steps": steps, "tvals": tvals, "table": table, "film_width": int(self.L.ns2vc_unet_film_width(self.h)),
                   "graph": None, "out": None, "runs": 0}
            self._graphs[key] = ent
            while len(self._graphs) > self.MAX_GRAPHS:     # LRU: the oldest captured loop (graph + tables) is dropped
                self._graphs.popitem(last=False)
        else:
            self._graphs.move_to_end(key)
        ent["runs"] += 1
        if not use_graph:
            res = self._loop(kind, ent, use_first)
        elif ent["graph"] is None and ent["runs"] < self.CAPTURE_AFTER:
            # eager: the first run builds the launch program and sets kernel attributes; a shape / schedule seen only once or
            # twice (the CLI: every slice a new length) never pays for a capture (~0.1-1 s for 6 000+ kernel nodes)
            res = self._loop(kind, ent, use_first)
        else:
            if ent["graph"] is None:
                torch.cuda.synchronize(self.dev)
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    ent["out"] = self._loop(kind, ent, use_first)
                ent["graph"] = g
            ent["graph"].replay()
            self._prepared = True
            self.unet.__dict__["_cond_owner"] = self
            res = ent["out"].clone()
        self._check_nan()
        return self._unpad(res)

    # ------------------------------------------------------------------ public samplers
    def sample_dpmpp_2m(self, x_T: torch.Tensor, ns, ts: torch.Tensor, lower_order_final: bool = True,
                        first_out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """DPM-Solver++ multistep order 2 over time points ``ts`` (N+1 values), x_start model.
        Equivalent to reference DPM_Solver.sample(method='multistep', order=2) (dpm_solver.py:1171-1213).
        ``first_out``: the model output at ts[0] if the caller already evaluated it (saves one forward)."""
        return self._run("dpm", x_T, ns, ts, first_out, bool(lower_order_final))

    def sample_unipc(self, x_T: torch.Tensor, ns, ts: torch.Tensor, variant: str = "bh2",
                     first_out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """UniPC multistep order 2, data prediction, lower_order_final (uni_pc.py:606-658)."""
        return self._run("unipc", x_T, ns, ts, first_out, variant)

    # ------------------------------------------------------------------ DDPM / DDIM: chunked replay
    # A 1000-step DDPM run as one graph would hold ~1000 x 205 nodes and its FiLM table 1000 x B rows, so these runs go in chunks
    # of CHUNK steps.  One chunk = the FiLM rows of its CHUNK x B evaluation times (read from a static time window) + per step
    # (UNet forward + noise draw + step kernel reading its scalars from a static coefficient window); x stays in one static
    # buffer (the step kernels update it in place).  Before each chunk the host refills both windows with stream-ordered D2D
    # copies from the run's full device tables, so one captured chunk is replayed for every full chunk of every run of that
    # sampler, plus one capture for the final chunk (a different noise-draw pattern and, usually, length).
    CHUNK = 50                                               # steps per chunk: the node count of a 50-step DPM-Solver graph

    def _chunk_buffers(self):
        if self._chunk is None:
            f32 = dict(dtype=torch.float32, device=self.dev)
            K, B = self.CHUNK, self.B
            self._chunk = {
                "tvals": torch.empty((K * B,), **f32),
                "coef": torch.empty((K * 32,), dtype=torch.uint8, device=self.dev),
                "table": torch.empty(int(self.L.ns2vc_unet_time_table_floats(self.h, K * B)), **f32),
                "film_width": int(self.L.ns2vc_unet_film_width(self.h)),
                "x": torch.empty((B, self.Cl, self.T), **f32),
                "x0": torch.empty((B, self.Co, self.T), **f32),
                "noise": torch.empty((B, self.Cl, self.T), **f32),
                # seeded runs: the row step's per-row operands (k advanced by the kernel) and NaN flags
                "seeds": torch.empty((B,), dtype=torch.int64, device=self.dev),
                "method": torch.empty((B,), dtype=torch.int32, device=self.dev),
                "base": torch.zeros((B,), dtype=torch.int32, device=self.dev),
                "k": torch.empty((B,), dtype=torch.int32, device=self.dev),
                "nan_rows": torch.empty((B,), dtype=torch.int32, device=self.dev),
            }
        return self._chunk

    def _chain_step(self, kind, coef_ptr, noise_ptr):
        cb = self._chunk
        x = cb["x"]
        fn = self.L.ns2vc_ddpm_step if kind == "ddpm" else self.L.ns2vc_ddim_step
        with torch.cuda.device(self.dev):
            _lib.check(fn(x.data_ptr(), cb["x0"].data_ptr(), noise_ptr, coef_ptr, x.data_ptr(), x.numel(), self.nan_flag.data_ptr(),
                          self._stream()))

    def _seeded_step(self, kind, ent):
        """One step of a seeded run: the row kernel with every row at step k (on the device) of the run's full table."""
        cb = self._chunk
        x = cb["x"]
        tab = ent["coef"].data_ptr()
        with torch.cuda.device(self.dev):
            _lib.check(self.L.ns2vc_sampler_step_rows_seeded(
                x.data_ptr(), cb["x0"].data_ptr(), None, None, None, None, None, tab if kind == "ddpm" else None,
                tab if kind == "ddim" else None, cb["seeds"].data_ptr(), self.T, cb["method"].data_ptr(), cb["base"].data_ptr(),
                cb["k"].data_ptr(), None, None, x.data_ptr(), self.Cl * self.T, self.B, cb["nan_rows"].data_ptr(), self._stream()))

    def _seeded_body(self, kind, ent, L):
        """L steps of a seeded run from the time window; the steps' structs and noise follow the device counter k."""
        cb = self._chunk
        B, fw = self.B, cb["film_width"]
        self.time_table(cb["tvals"][:L * B], cb["table"])
        for k in range(L):
            self.forward(cb["x"], None, cb["x0"], film_rows=cb["table"][k * B * fw:(k + 1) * B * fw])
            self._seeded_step(kind, ent)

    def _chunk_body(self, kind, draws, noise, j, csize):
        """Steps j .. j+len(draws)-1 of a run, scalars and times from the windows.  noise: the injected [N, B, C, T] tensor or
        None (draw ``randn_like(x)`` on the default generator where ``draws`` says the reference draws)."""
        cb = self._chunk
        L, B, fw = len(draws), self.B, cb["film_width"]
        self.time_table(cb["tvals"][:L * B], cb["table"])
        for k in range(L):
            self.forward(cb["x"], None, cb["x0"], film_rows=cb["table"][k * B * fw:(k + 1) * B * fw])
            if noise is not None:
                nz = noise[j + k].data_ptr()
            elif draws[k]:
                nz = cb["noise"].normal_().data_ptr()      # = torch.randn_like(x): empty_like(x).normal_()
            else:
                nz = None
            self._chain_step(kind, cb["coef"].data_ptr() + k * csize, nz)

    def _chain(self, kind, x_T, key, make_steps, first_out, noise, seeds=None):
        assert self.Cl == self.Co, "x_start parameterisation needs out_channels == latent channels"
        if seeds is not None:
            if noise is not None:
                raise ValueError("seeds and noise are mutually exclusive: seeded rows draw their own noise")
            seeds = seeded_noise.check_seeds(seeds, self.B)
        self._sync_engine()
        ent = self._chains.get(key)
        if ent is None:
            steps = make_steps()
            draws = tuple(s.add_noise for s in steps) if kind == "ddpm" else tuple(not s.last for s in steps)
            coef, csize = coefs.c_table(steps, self.dev)
            ent = {"n": len(steps), "draws": draws, "csize": csize, "coef": coef,
                   "tvals": coefs.t_inputs(steps, self.B, self.dev).reshape(-1), "runs": 0, "seeded_runs": 0, "graphs": {}}
            self._chains[key] = ent
            while len(self._chains) > self.MAX_GRAPHS:
                self._chains.popitem(last=False)
        else:
            self._chains.move_to_end(key)
        N, B, csize = ent["n"], self.B, ent["csize"]
        if noise is not None:
            if tuple(noise.shape) != (N, B, self.Cl, self.T):
                raise ValueError(f"noise must be [{N}, {B}, {self.Cl}, {self.T}] (one tensor per step), got {tuple(noise.shape)}")
            noise = noise.to(self.dev, torch.float32).contiguous()
        runs = "seeded_runs" if seeds is not None else "runs"    # (counted apart: each path's first runs are eager)
        if noise is None:
            ent[runs] += 1
        use_graph = noise is None and os.environ.get("NS2VC_GRAPH", "1") != "0" and ent[runs] >= self.CAPTURE_AFTER
        cb = self._chunk_buffers()
        self._unpad(cb["x"].copy_(x_T, non_blocking=True))
        if seeds is not None:
            return self._seeded_chain(kind, ent, first_out, seeds, use_graph)
        self.nan_flag.zero_()
        self.prepare()
        j = 0
        if first_out is not None:                          # step 0 was evaluated by the caller: its update runs on its own
            cb["x0"].copy_(first_out, non_blocking=True)
            nz = noise[0].data_ptr() if noise is not None else (cb["noise"].normal_().data_ptr() if ent["draws"][0] else None)
            self._chain_step(kind, ent["coef"].data_ptr(), nz)
            j = 1
        while j < N:
            L = min(self.CHUNK, N - j)
            cb["tvals"][:L * B].copy_(ent["tvals"][j * B:(j + L) * B], non_blocking=True)
            cb["coef"][:L * csize].copy_(ent["coef"][j * csize:(j + L) * csize], non_blocking=True)
            draws = ent["draws"][j:j + L]
            if not use_graph:
                self._chunk_body(kind, draws, noise, j, csize)
            else:
                gkey = (kind, draws)
                g = self._chunk_graphs.get(gkey)
                if g is None:
                    torch.cuda.synchronize(self.dev)
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g):
                        self._chunk_body(kind, draws, None, j, csize)
                    self._chunk_graphs[gkey] = g
                    while len(self._chunk_graphs) > 2 * self.MAX_GRAPHS:
                        self._chunk_graphs.popitem(last=False)
                else:
                    self._chunk_graphs.move_to_end(gkey)
                g.replay()
            j += L
        res = cb["x"].clone()
        self._check_nan()
        return self._unpad(res)

    def _seeded_chain(self, kind, ent, first_out, seeds, use_graph):
        """A seeded run (x_T already in the static x): every step is the row kernel over the run's full coefficient table, its
        struct and noise picked by the device counter k, so one captured chunk of L steps serves every chunk of that length of
        this run's schedule.  Those captures bake the table's pointer and live in the run's own entry (dropped with it)."""
        cb = self._chunk
        N, B = ent["n"], self.B
        cb["seeds"].copy_(torch.tensor(seeds, dtype=torch.int64), non_blocking=False)
        cb["method"].fill_(_lib.ROW_DDPM if kind == "ddpm" else _lib.ROW_DDIM)
        cb["k"].zero_()
        cb["nan_rows"].zero_()
        self.prepare()
        j = 0
        if first_out is not None:
            cb["x0"].copy_(first_out, non_blocking=True)
            self._seeded_step(kind, ent)
            j = 1
        while j < N:
            L = min(self.CHUNK, N - j)
            cb["tvals"][:L * B].copy_(ent["tvals"][j * B:(j + L) * B], non_blocking=True)
            if not use_graph:
                self._seeded_body(kind, ent, L)
            else:
                g = ent["graphs"].get(L)
                if g is None:
                    torch.cuda.synchronize(self.dev)
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g):
                        self._seeded_body(kind, ent, L)
                    ent["graphs"][L] = g
                g.replay()
            j += L
        res = cb["x"].clone()
        self._check_nan(cb["nan_rows"])
        return self._unpad(res)

    def sample_ddpm(self, x_T: torch.Tensor, timesteps=None, noise: Optional[torch.Tensor] = None,
                    first_out: Optional[torch.Tensor] = None, seeds=None) -> torch.Tensor:
        """DDPM ancestral sampling, one ``p_sample`` (reference model.py:535-542) per integer t of ``timesteps`` (descending;
        default 999 .. 0: ``p_sample_loop``, :544-561).  Noise: ``torch.randn_like(x)`` on the device's default generator for every
        step with t > 0, in the reference's order, or the injected ``noise`` [N, B, C, T] (row k for step k; the run is then
        eager), or with ``seeds`` ([B] ints in [0, 2**63)) row b's step-k noise ``noise.normal_rows(seeds[b], step=k)`` drawn in
        the step kernel (captured and replayed like the default path).  ``first_out``: the model output at timesteps[0] if the
        caller already evaluated it."""
        buf = _diffusion_buffers()
        total = buf["betas"].shape[0]
        ts = tuple(range(total - 1, -1, -1)) if timesteps is None else tuple(int(t) for t in timesteps)
        if not ts or any(not 0 <= t < total for t in ts):
            raise ValueError(f"timesteps must be a non-empty list of integers in [0, {total})")
        return self._chain("ddpm", x_T, ("ddpm", ts), lambda: coefs.ddpm_table(buf, ts), first_out, noise, seeds)

    def sample_ddim(self, x_T: torch.Tensor, sampling_timesteps: int, eta: float = 0.0, noise: Optional[torch.Tensor] = None,
                    first_out: Optional[torch.Tensor] = None, seeds=None) -> torch.Tensor:
        """DDIM (reference ``ddim_sample``, model.py:563-603) over ``sampling_timesteps`` pairs with ``ddim_sampling_eta = eta``.
        Noise: ``torch.randn_like(x)`` once per pair except the last (also at eta = 0, as the reference draws it), or the
        injected ``noise`` [N, B, C, T], or drawn per row from ``seeds`` as for ``sample_ddpm`` (eta must then lie in [0, 1])."""
        buf = _diffusion_buffers()
        total = buf["betas"].shape[0]
        S, eta = int(sampling_timesteps), float(eta)
        if S < 1:
            raise ValueError("sampling_timesteps must be >= 1")
        if seeds is not None and not 0.0 <= eta <= 1.0:
            raise ValueError(f"eta must lie in [0, 1], got {eta}")
        return self._chain("ddim", x_T, ("ddim", S, eta), lambda: coefs.ddim_table(buf, total, S, eta), first_out, noise, seeds)


    # ------------------------------------------------------------------ training objective: K evaluations behind one prepare
    def eval_x_start(self, x_KBCT: torch.Tensor, t_KB: torch.Tensor, out_KBCT: torch.Tensor) -> torch.Tensor:
        """The denoiser's x_start prediction of K noisy batches on this session's conditioning: ``out[k] = denoiser(x[k], t[k])``
        with x [K, B, Cl, T] fp32 and t [K, B] (integer timesteps, any dtype) on the session device.  ``prepare()`` runs once
        and the FiLM rows of all K * B times come from one ``time_table`` launch per CHUNK evaluations; each evaluation is the
        ``forward`` the samplers run.  Eager (no CUDA graph).  Padded sessions only: ``NaturalSpeech2.forward`` averages its
        loss over the padded rows."""
        if self.ragged:
            raise ValueError("eval_x_start runs the padded program (the reference's objective averages over padded rows)")
        return self._eval_k(x_KBCT, t_KB, out_KBCT)

    def eval_x_start_ragged(self, x_KBCT: torch.Tensor, t_KB: torch.Tensor, out_KBCT: torch.Tensor) -> torch.Tensor:
        """``eval_x_start`` on a ragged session: ``out[k, b, :, :T_b]`` is the prediction for utterance b alone at ``t[k, b]``, from
        ``x[k, b, :, :T_b]`` (values past T_b are never read; ``out`` past T_b is left unspecified).  The same one ``prepare()``
        and one ``time_table`` per CHUNK evaluations, the forwards of the ragged program."""
        if not self.ragged:
            raise ValueError("eval_x_start_ragged needs a ragged session (get_session(..., content_lengths=...))")
        return self._eval_k(x_KBCT, t_KB, out_KBCT)

    def _eval_k(self, x_KBCT: torch.Tensor, t_KB: torch.Tensor, out_KBCT: torch.Tensor) -> torch.Tensor:
        K = x_KBCT.shape[0]
        if tuple(x_KBCT.shape) != (K, self.B, self.Cl, self.T) or tuple(t_KB.shape) != (K, self.B) \
                or tuple(out_KBCT.shape) != (K, self.B, self.Co, self.T):
            raise ValueError(f"expected x [K, {self.B}, {self.Cl}, {self.T}], t [K, {self.B}] and out [K, {self.B}, {self.Co}, {self.T}], "
                             f"got {tuple(x_KBCT.shape)}, {tuple(t_KB.shape)}, {tuple(out_KBCT.shape)}")
        for v in (x_KBCT, out_KBCT):
            if v.dtype != torch.float32 or not v.is_contiguous() or v.device != self.dev:
                raise ValueError("x and out must be contiguous fp32 tensors on the session device")
        self._sync_engine()
        self.prepare()
        tvals = t_KB.to(self.dev, torch.float32).contiguous()
        fw = int(self.L.ns2vc_unet_film_width(self.h))
        n = min(K, self.CHUNK)
        table = torch.empty(int(self.L.ns2vc_unet_time_table_floats(self.h, n * self.B)), dtype=torch.float32, device=self.dev)
        for j in range(0, K, self.CHUNK):
            L = min(self.CHUNK, K - j)
            self.time_table(tvals[j:j + L], table)
            for k in range(L):
                self.forward(x_KBCT[j + k], None, out_KBCT[j + k], film_rows=table[k * self.B * fw:(k + 1) * self.B * fw])
        return out_KBCT


def check_lengths(lengths, B: int, limit: int, name: str) -> list:
    """Per-utterance lengths as a list of B ints in [1, limit]; ValueError otherwise."""
    vals = [int(v) for v in (lengths.tolist() if isinstance(lengths, torch.Tensor) else lengths)]
    if len(vals) != B:
        raise ValueError(f"{name} must have {B} entries, got {len(vals)}")
    bad = [v for v in vals if not 1 <= v <= limit]
    if bad:
        raise ValueError(f"{name} must lie in [1, {limit}], got {bad}")
    return vals


_BUFFERS = {}


def _diffusion_buffers(timesteps: int = 1000) -> dict:
    if timesteps not in _BUFFERS:
        _BUFFERS[timesteps] = coefs.diffusion_buffers(timesteps)
    return _BUFFERS[timesteps]


def get_session(unet: UNet1DConditionModel, content_BCT, prompt_BSC, prompt_mask, T=None, content_lengths=None,
                prompt_lengths=None) -> DenoiserSession:
    """Session cache per (B, T, S, mask?, ragged?) on the module: captured graphs and static buffers are reused
    across utterance batches of the same shape (a ragged session across any lengths)."""
    B, S = prompt_BSC.shape[0], prompt_BSC.shape[1]
    Tn = content_BCT.shape[2] if content_BCT is not None else T
    ragged = content_lengths is not None
    key = (B, Tn, S, prompt_mask is not None, str(prompt_BSC.device)) + (("ragged",) if ragged else ())
    cache = unet.__dict__.setdefault("_sessions", {})
    sess = cache.get(key)
    if sess is None or sess.h != unet.engine(prompt_BSC.device):
        while len(cache) >= 8:                               # bounded: oldest shape first (dicts keep insertion order)
            cache.pop(next(iter(cache)))
        sess = DenoiserSession(unet, content_BCT, prompt_BSC, prompt_mask, T=T, content_lengths=content_lengths,
                               prompt_lengths=prompt_lengths)
        cache = unet.__dict__.setdefault("_sessions", {})     # (the workspace may have grown and dropped the old sessions)
        cache[key] = sess
    else:
        sess.set_cond(content_BCT, prompt_BSC, prompt_mask, content_lengths, prompt_lengths)
    return sess


def _fast_path_enabled() -> bool:
    return os.environ.get("NS2VC_B200_FUSED", "1") != "0"


def _trace_first_call(solver, x: torch.Tensor, t0: torch.Tensor):
    """Run the solver's first model evaluation through the user's closure while recording which
    denoiser calls it makes.  Returns (record, noise) if the closure is exactly one call of our
    UNet whose output is returned unchanged (x_start model, no guidance), else (None, noise)."""
    wrapped = getattr(solver, "_wrapped", None)
    from .schedule import WrappedModel
    with trace_calls() as recs:
        noise = solver.model(x, t0)
    if not isinstance(wrapped, WrappedModel) or wrapped.model_type != "x_start" or wrapped.guidance_type != "uncond":
        return None, noise
    if len(recs) != 1:
        return None, noise
    r = recs[0]
    u = r.unet
    Cl = u.latent_channels
    if u.cfg.out_channels != Cl or r.sample.shape[1] != u.cfg.in_channels or tuple(r.sample.shape[::2]) != tuple(x.shape[::2]):
        return None, noise
    if x.shape[1] != Cl or x.dtype != torch.float32:
        return None, noise
    if not torch.equal(r.sample[:, :Cl], x):
        return None, noise
    # the closure must hand back the UNet output itself: noise == (x - alpha*out)/sigma
    ns = wrapped.noise_schedule
    tt = t0.expand(x.shape[0])
    a, s = ns.marginal_alpha(tt), ns.marginal_std(tt)
    expect = (x - a[:, None, None] * r.output) / s[:, None, None]
    if not torch.equal(expect, noise):
        return None, noise
    return r, noise


def _session_from_record(r) -> DenoiserSession:
    u = r.unet
    Cl = u.latent_channels
    content = r.sample[:, Cl:] if r.sample.shape[1] > Cl else None
    return get_session(u, content, r.ehs, r.mask, T=r.sample.shape[2])


def _try_fused(solver, x, steps, skip_type, t_T, t_0, kind):
    """(latents, None) when the fused path ran; (None, first_noise) when the closure is not ours — first_noise is the
    model output of the solver's first evaluation (already paid for by the trace), or None if nothing was evaluated."""
    if not (_fast_path_enabled() and x.is_cuda and skip_type in ("time_uniform", "time_quadratic", "logSNR")):
        return None, None
    ns = solver.noise_schedule
    ts = solver.get_time_steps(skip_type=skip_type, t_T=t_T, t_0=t_0, N=steps, device="cpu")
    with torch.no_grad():
        rec, noise = _trace_first_call(solver, x, ts[0].to(x.device))
        if rec is None:
            return None, noise
        sess = _session_from_record(rec)
        if kind == "dpm":
            return sess.sample_dpmpp_2m(x, ns, ts, lower_order_final=True, first_out=rec.output), None
        return sess.sample_unipc(x, ns, ts, variant=solver.variant, first_out=rec.output), None


def try_fused_dpm(solver, x, steps, skip_type, t_T, t_0):
    return _try_fused(solver, x, steps, skip_type, t_T, t_0, "dpm")


def try_fused_unipc(solver, x, steps, skip_type, t_T, t_0):
    return _try_fused(solver, x, steps, skip_type, t_T, t_0, "unipc")
