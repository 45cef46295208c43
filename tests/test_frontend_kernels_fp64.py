"""The prompt-mel front end's two launches, resample_kernel and log_mel_kernel (csrc/frontend.cu), each on its own input through
the C ABI (ns2vc_resampler_create / ns2vc_resample / ns2vc_resample_table, ns2vc_mel_create / ns2vc_log_mel), at every rate
ratio the resampler accepts and with caller windows and filterbanks.  The log-mel gets 24 kHz fp32 rows of its own, not the
resampler's output, so an error in one launch cannot hide in the other.

Resampler, two truths, each row alone (oracle/kernel_oracle.py):
  * A: the fp64 convolution on the handle's own fp32 table, read back with ns2vc_resample_table.  Bound: one rounding to fp32
    and the fp64 sums, 2^-24 |y| + 2 taps 2^-53 sum |w||x| (resample_terms_a).  It notices fp32 accumulation and any tap or
    phase slip.
  * B: mel_oracle.resample in fp64 on the fp64 table.  Bound: the parity rule plus the table's rounding, 2^-24 sum |w||x|.
Log-mel: the fp64 STFT -> |.| -> projection -> log(max(., 1e-7)) on the kernel's own fp32 input and tables, each row alone.
Bound: the interval of log_mel_terms (the fp32 radix-2 FFT and split step, the fmaf projection, logf's ulp, mapped through the
clip as an interval, so clipped entries are exact), and the parity rule.  Each case prints its worst ratio; the module prints
the worst of each family, and for information the log-mel's error over the fp32 recipe's error on the same entries.

No bound is vacuous (the CPU tier): a tap shifted by one input sample, phase p read as p + 1, the width off by one and fp32
accumulation (against truth A) move the resampler's reference, and reflecting about L, a frame start off by one, the symmetric
Hann window, a band shifted by one bin, power 2, a clip at 1e-6 and one window tap scaled by 1 + 2^-10 move the log-mel's, by
>= 16 x the bound in every case that has the feature.

Exact properties of both launches: everything at or past each row's length is 0; a ragged row equals the row launched alone;
a second launch is bit-identical; NaN from a row's length to the batch stride changes no bit; lengths and frame counts follow
the fp32 rules; the identity ratio copies.  NaN reach: a NaN input sample makes NaN exactly the outputs whose nonzero taps
cover it (resampler) or every band of exactly the frames whose reflect-padded window holds it (log-mel; +-Inf: non-finite in
every band with a weight), every other output bit-identical.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, List

import pytest
import torch

from conftest import REPO  # noqa: F401  (puts the repository on sys.path)
from ns2vc_b200 import _lib, frontend
from oracle import kernel_oracle as ko
from oracle import mel_oracle
from test_frontend_mel import DIVERGENT

F64 = torch.float64
SENSITIVITY = 16.0
WORST: Dict[str, float] = {}


def gpu(f):
    """a GPU case: marked `gpu`, skipped where there is no CUDA device"""
    return pytest.mark.gpu(pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")(f))


def record(family: str, r: float) -> None:
    WORST[family] = max(WORST.get(family, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    for fam, r in sorted(WORST.items()):
        print(f"\n[front-end kernel checks] {fam}: worst ratio {r:.3g}")


@pytest.fixture(scope="module")
def speech(gold):
    """the fixture's int16 speech (the reference's 1.wav and 2.wav), one float row"""
    fx = gold("frontend_mel.pt")
    return torch.cat([fx["cases"][k]["pcm_int16"].float() / 32768.0 for k in ("1.wav", "2.wav")])


def stream() -> int:
    return torch.cuda.current_stream().cuda_stream


# ---------------------------------------------------------------------------------------------------------------------------
# signals
# ---------------------------------------------------------------------------------------------------------------------------
def signal(kind: str, n: int, g: torch.Generator, speech: torch.Tensor, fc: float = 0.25) -> torch.Tensor:
    """n samples of `kind`; frequencies in cycles per sample, fc the resampler's cutoff"""
    t = torch.arange(n, dtype=F64)
    if kind == "noise":
        v = 0.3 * torch.randn(n, generator=g, dtype=F64)
    elif kind == "speech":
        reps = n // speech.numel() + 1
        v = speech.to(F64).repeat(reps)[:n]
    elif kind.startswith("dc"):                                        # DC of 10^2 / 10^4 x the AC amplitude 1e-3
        v = float(kind[2:]) * 1e-3 + 1e-3 * torch.randn(n, generator=g, dtype=F64)
    elif kind == "square":                                            # full scale, period 37
        v = torch.where((t // 37) % 2 == 0, 1.0, -1.0).to(F64)
    elif kind == "impulse":
        v = torch.zeros(n, dtype=F64)
        if n:
            v[n // 2] = 0.9
    elif kind == "silence":
        v = torch.zeros(n, dtype=F64)
    elif kind == "chirp":                                             # 0.9 fc .. min(1.1 fc, 0.5) across the row
        f0, f1 = 0.9 * fc, min(1.1 * fc, 0.5)
        v = 0.5 * torch.sin(2 * math.pi * (f0 * t + (f1 - f0) * t * t / (2 * max(n, 1))))
    elif kind == "stopband":                                          # tones between the cutoff and the input's Nyquist
        f = [min(fc * 1.3, 0.49), min(fc * 1.7, 0.495), 0.45 if fc < 0.3 else 0.4985]
        v = sum(0.3 * torch.cos(2 * math.pi * fi * t + k) for k, fi in enumerate(f))
    else:
        raise ValueError(kind)
    return v.float()


# ---------------------------------------------------------------------------------------------------------------------------
# resampler
# ---------------------------------------------------------------------------------------------------------------------------
RATIOS = [(1, 1), (2, 1), (4, 1), (8, 1), (1, 2), (1, 3), (147, 80), (147, 160), (2, 3), (441, 160), (147, 320), (80, 441),
          (45, 1), (2991, 112)]
RES_SIGNALS = ["noise", "speech", "dc1e2", "dc1e4", "square", "impulse", "silence", "chirp", "stopband"]
EDGE_OUT = [255, 256, 257, 511, 512, 513]


def handle_info(orig: int, nw: int):
    """(phases, taps, width, fp32 table [nw, taps]) of the handle; the identity's one unit tap"""
    if orig == nw:
        return 1, 1, 0, torch.ones(1, 1)
    P, T, W = C.c_int(), C.c_int(), C.c_int()
    L = _lib.lib()
    _lib.check(L.ns2vc_resample_table(orig, nw, C.byref(P), C.byref(T), C.byref(W), None))
    buf = torch.empty(P.value * T.value)
    _lib.check(L.ns2vc_resample_table(orig, nw, None, None, None, buf.data_ptr()))
    return P.value, T.value, W.value, buf.view(P.value, T.value)


def n_for_out(orig: int, nw: int, target: int) -> int:
    """the fewest input samples that give `target` outputs"""
    n = max(0, target * orig // nw - 2)
    while ko.resample_out_len(orig, nw, n) < target:
        n += 1
    return n


class RCase:
    def __init__(self, name, orig, nw, lens, N, signals, seed):
        self.name, self.orig, self.nw, self.lens, self.N, self.signals, self.seed = name, orig, nw, lens, N, signals, seed

    @property
    def fc(self) -> float:
        return 0.99 * min(self.orig, self.nw) / (2 * self.orig)


def res_cases() -> List[RCase]:
    out = []
    for i, (o, n) in enumerate(RATIOS):
        width = ko.resample_width(o, n)                                 # no library call while collecting
        top = EDGE_OUT[i % len(EDGE_OUT)]
        edge = sorted({0, 1, max(width - 1, 0), width, width + 1} | {n_for_out(o, n, t) for t in EDGE_OUT if t <= top})
        N = n_for_out(o, n, top)
        lens = [v for v in edge if v <= N]
        sig = [RES_SIGNALS[(k + i) % len(RES_SIGNALS)] for k in range(len(lens))]
        out.append(RCase(f"r{o}_{n}_edges_out{top}", o, n, lens, N, sig, 100 + i))
        N2 = n_for_out(o, n, 700)
        out.append(RCase(f"r{o}_{n}_signals", o, n, [N2 - 3 * k for k in range(len(RES_SIGNALS))], N2, RES_SIGNALS, 200 + i))
    for k, (o, n, N) in enumerate(DIVERGENT):                      # the fp32 length rule differs from the exact ceiling here
        g = math.gcd(o, n)
        out.append(RCase(f"r{o}_{n}_divergent{N}", o // g, n // g, [N, N - 1, 1000], N, ["speech", "noise", "stopband"], 300 + k))
    out.append(RCase("r147_80_2p22", 147, 80, [1 << 22], 1 << 22, ["speech"], 400))
    return out


RES_CASES = res_cases()


def build_res(c: RCase, speech: torch.Tensor) -> torch.Tensor:
    g = torch.Generator().manual_seed(c.seed)
    wav = torch.zeros(len(c.lens), c.N)
    for b, (n, s) in enumerate(zip(c.lens, c.signals)):
        wav[b, :n] = signal(s, n, g, speech, c.fc)
    return wav


def res_n_out(c: RCase) -> int:
    return ko.resample_out_len(c.orig, c.nw, c.N)


def truth_a(c: RCase, wav: torch.Tensor, b: int, table: torch.Tensor, width: int, dev, **defect) -> torch.Tensor:
    return ko.resample_rows(wav[b].to(dev), c.lens[b], table.to(dev), c.orig, c.nw, width, res_n_out(c), **defect)


def truth_b(c: RCase, wav: torch.Tensor, b: int, dev, dt=F64) -> torch.Tensor:
    out = torch.zeros(res_n_out(c), dtype=dt, device=dev)
    y = mel_oracle.resample(wav[b, :c.lens[b]].to(dev), c.orig, c.nw, dt)
    out[:y.numel()] = y[:out.numel()]
    return out


def res_bounds(c: RCase, wav: torch.Tensor, b: int, dev):
    """(truth A, bound A, truth B, bound B) of row b"""
    _, taps, width, table = handle_info(c.orig, c.nw)
    ya = truth_a(c, wav, b, table, width, dev)
    absum = ko.resample_abs_sum(wav[b].to(dev), c.lens[b], table.to(dev), c.orig, c.nw, width, res_n_out(c))
    yb = truth_b(c, wav, b, dev)
    e32 = float((truth_b(c, wav, b, dev, torch.float32).to(F64) - yb).abs().max()) if yb.numel() else 0.0
    return ya, ko.resample_terms_a(ya, absum, taps), yb, ko.parity_tol(yb, e32) + ko.resample_terms_b(absum)


def moved(defect: torch.Tensor, ref: torch.Tensor, tol: torch.Tensor) -> float:
    return ko.ratio(defect - ref, tol) if ref.numel() else 0.0


@pytest.mark.parametrize("c", [c for c in RES_CASES if c.N < (1 << 20)], ids=lambda c: c.name)
def test_resample_reference_is_sensitive(c, speech):
    """CPU: truth B is mel_oracle's recipe on the fp64 table, and each defect moves truth A by >= 16 x bound A (fp32
    accumulation) or bound B (the slips) wherever the case has the feature: outputs at all (every defect), more than one
    phase (p + 1), an output whose sum cancels 6 bits or more (fp32 accumulation)"""
    wav = build_res(c, speech)
    P, taps, width, table = handle_info(c.orig, c.nw)
    assert width == ko.resample_width(c.orig, c.nw)
    if c.orig != c.nw:
        assert torch.equal(ko.sinc_table64(c.orig, c.nw, width).float(), table)
    s = {"shift": 0.0, "phase": 0.0, "width": 0.0, "fp32acc": 0.0}
    old_caught = set()
    any_out = cancels = False
    for b in range(len(c.lens)):
        ya, ta, yb, tb = res_bounds(c, wav, b, "cpu")
        if c.orig != c.nw:                                             # truth B is this convolution on mel_oracle's fp64 table
            t64 = mel_oracle.sinc_kernel(c.orig, c.nw, F64)[0].reshape(P, taps)
            assert moved(ko.resample_rows(wav[b], c.lens[b], t64, c.orig, c.nw, width, res_n_out(c)), yb, tb) < 1e-3
        if not (ya != 0).any():
            continue
        any_out = True
        absum = ko.resample_abs_sum(wav[b], c.lens[b], table, c.orig, c.nw, width, res_n_out(c))
        cancels |= bool((absum > 64 * ya.abs()).any())                  # a sum that cancels 6 bits or more
        old = 4 * float((truth_b(c, wav, b, "cpu", torch.float32).to(F64) - yb).abs().max())   # test_frontend_mel's bound
        for k, kw in (("shift", dict(shift=1)), ("phase", dict(phase_plus_one=True)), ("width", dict(width_delta=1)),
                      ("fp32acc", dict(fp32_acc=True))):
            if k == "phase" and P == 1 or k == "width" and c.orig == c.nw:
                continue
            d = truth_a(c, wav, b, table, width, "cpu", **kw)
            s[k] = max(s[k], moved(d, ya, ta) if k == "fp32acc" else moved(d, yb, tb))
            if float((d - yb).abs().max()) > old:
                old_caught.add(k)
    if not any_out:
        return
    assert s["shift"] >= SENSITIVITY, s
    assert P == 1 or s["phase"] >= SENSITIVITY, s
    assert c.orig == c.nw or s["width"] >= SENSITIVITY, s
    assert not cancels or s["fp32acc"] >= SENSITIVITY, s
    print(f"{c.name}: defect / bound {', '.join(f'{k} {v:.3g}' for k, v in s.items())}; missed by 4 e_ref: {sorted(set(s) - old_caught)}")


def test_resampler_refuses_a_window_past_48kb():
    """46:1 stages 12380 floats per 256 outputs; 45:1 (12111) and 2991:112 (exactly 12288) are accepted (their creation is
    covered on the GPU), and the host check comes before any allocation"""
    h = C.c_void_p()
    with pytest.raises(_lib.Ns2vcError, match="46:1, whose 12380-sample input window per 256 outputs exceeds 12288"):
        _lib.check(_lib.lib().ns2vc_resampler_create(46000, 1000, C.byref(h)))
    for o, n, win in ((45, 1, 12111), (2991, 112, 12288), (46, 1, 12380)):
        _, taps, _, _ = handle_info(o, n)
        assert (255 // n + 1) * o + taps == win


def test_length_rules():
    L = _lib.lib()
    for o, n in RATIOS:
        for N in list(range(0, 40)) + [n_for_out(o, n, t) + d for t in EDGE_OUT for d in (-1, 0, 1)] + [1 << 22]:
            N = max(N, 0)
            assert L.ns2vc_resample_out_length(o, n, N) == ko.resample_out_len(o, n, N) == mel_oracle.out_length(o, n, N), (o, n, N)
    for N in (513, 767, 768, 769, 1791, 1792, 2049, 4097):
        assert ko.log_mel_frames(N, 1 << 30) == 1 + N // 256 == mel_oracle.log_mel_24k(torch.zeros(N)).shape[-1]
    assert ko.log_mel_frames(4097, 14) == 14


def launch_res(c: RCase, wav: torch.Tensor, dev, poison=False, only=None, nan_at=None, h=None) -> torch.Tensor:
    bsel = list(range(len(c.lens))) if only is None else [only]
    B, slack = len(bsel), 5
    x = torch.zeros(B, c.N + slack, device=dev)
    x[:, :c.N] = wav[bsel].to(dev)
    if poison:                                                       # from the row's length to the batch stride: never read
        for i, b in enumerate(bsel):
            x[i, c.lens[b]:] = float("nan")
    if nan_at is not None:
        x[nan_at] = float("nan")
    lens = torch.tensor([c.lens[b] for b in bsel], dtype=torch.int64, device=dev)
    n_out = res_n_out(c)
    y = torch.full((B, n_out + 3), float("nan"), device=dev)
    L = _lib.lib()
    own = h is None
    if own:
        h = C.c_void_p()
        _lib.check(L.ns2vc_resampler_create(c.orig, c.nw, C.byref(h)))
    try:
        _lib.check(L.ns2vc_resample(h, x.data_ptr(), c.N + slack, c.N, lens.data_ptr(), y.data_ptr(), n_out + 3, n_out, B, stream()))
        torch.cuda.synchronize()
    finally:
        if own:
            L.ns2vc_resampler_destroy(h)
    assert y[:, n_out:].isnan().all(), "wrote past n_out"
    return y[:, :n_out]


def nan_reach_res(c: RCase, b: int, i: int, dev) -> torch.Tensor:
    """outputs of row b whose nonzero taps (the handle's trimmed range) cover input sample i"""
    _, _, width, table = handle_info(c.orig, c.nw)
    lo, hi = ko.resample_trim(table)
    n_out = res_n_out(c)
    L_out = min(ko.resample_out_len(c.orig, c.nw, c.lens[b]), n_out)
    j = torch.arange(n_out)
    off = i - ((j // c.nw) * c.orig - width)
    p = j % c.nw
    return ((off >= lo[p]) & (off <= hi[p]) & (j < L_out)).to(dev)


@gpu
@pytest.mark.parametrize("c", RES_CASES, ids=lambda c: c.name)
def test_resample_kernel(c, speech):
    dev = torch.device("cuda")
    wav = build_res(c, speech)
    y = launch_res(c, wav, dev)
    n_out = res_n_out(c)
    wa = wb = 0.0
    for b, n in enumerate(c.lens):
        L_out = min(ko.resample_out_len(c.orig, c.nw, n), n_out)
        assert L_out == min(frontend.resample_out_length(c.orig, c.nw, n), n_out)
        assert (y[b, L_out:] == 0).all(), f"{c.name} row {b}: not 0 past its {L_out} outputs"
        if c.orig == c.nw:
            assert torch.equal(y[b, :n], wav[b, :n].to(dev)), f"{c.name} row {b}: the identity is not a copy"
        ya, ta, yb, tb = res_bounds(c, wav, b, dev)
        ra, rb = ko.ratio(y[b].to(F64) - ya, ta), ko.ratio(y[b].to(F64) - yb, tb)
        assert ra <= 1.0, f"{c.name} row {b} ({c.signals[b]}, {n} samples): {ra:.3f} of bound A"
        assert rb <= 1.0, f"{c.name} row {b} ({c.signals[b]}, {n} samples): {rb:.3f} of bound B"
        wa, wb = max(wa, ra), max(wb, rb)
    # NaN from each row's length to the stride changes no bit, and so this second launch is bit-identical
    assert torch.equal(launch_res(c, wav, dev, poison=True), y)
    if len(c.lens) > 1:                                              # each ragged row equals that row launched alone
        for b in range(len(c.lens)):
            assert torch.equal(launch_res(c, wav, dev, only=b)[0], y[b]), f"{c.name}: row {b} differs alone"
    if c.name.endswith("_signals"):                                  # NaN reach: a NaN sample near each end and in the middle
        b = 0
        n = c.lens[b]
        for i in (0, min(3, n - 1), n // 2, n - 1):
            got = launch_res(c, wav, dev, nan_at=(b, i))
            hit = nan_reach_res(c, b, i, dev)
            assert torch.equal(got[b].isnan(), hit), f"{c.name}: a NaN at sample {i} reaches other outputs"
            assert torch.equal(got[b][~hit], y[b][~hit]) and torch.equal(got[1:], y[1:])
    record("resample (truth A)", wa)
    record("resample (truth B)", wb)
    print(f"{c.name}: worst ratio {wa:.3f} of bound A, {wb:.3f} of bound B")


@gpu
def test_resample_refusals_on_the_device():
    with pytest.raises(_lib.Ns2vcError, match="exceeds 12288"):
        frontend.resample(torch.zeros(5000, device="cuda"), 46, 1)
    for o, n in ((45, 1), (2991, 112)):                              # the largest accepted windows are created
        h = C.c_void_p()
        _lib.check(_lib.lib().ns2vc_resampler_create(o, n, C.byref(h)))
        _lib.lib().ns2vc_resampler_destroy(h)


# ---------------------------------------------------------------------------------------------------------------------------
# log-mel
# ---------------------------------------------------------------------------------------------------------------------------
MEL_SIGNALS = ["speech", "silence", "dc1e2", "dc1e4", "square", "tone_bin", "tone_between", "tone_6k", "tone_12k", "noise1e-6",
               "from16k", "click", "noise"]
EDGE_LENS = [513, 514, 767, 768, 769, 1791, 1792, 2047, 2048, 2049, 3839, 3840, 4095, 4096, 4097]
CLICK_AT = 2048                                                    # frame 8's centre tap (512); the scaled-tap defect's tap


def mel_signal(kind: str, n: int, g: torch.Generator, speech: torch.Tensor) -> torch.Tensor:
    t = torch.arange(n, dtype=F64)
    if kind.startswith("tone"):
        k = {"tone_bin": 100.0, "tone_between": 100.5, "tone_6k": 256.0, "tone_12k": 512.0}[kind]
        return (0.5 * torch.cos(2 * math.pi * k / 1024 * t + (0.0 if kind == "tone_12k" else 0.3))).float()
    if kind == "noise1e-6":
        return (1e-6 * torch.randn(n, generator=g, dtype=F64)).float()
    if kind == "from16k":                                          # the recipe's fp32 resampler: top bands hold its rounding
        x16 = 0.3 * torch.randn(n * 2 // 3 + 2, generator=g)
        return mel_oracle.resample(x16, 16000, 24000, torch.float32)[:n].contiguous()
    if kind == "click":
        v = torch.zeros(n)
        v[min(CLICK_AT, n - 1)] = 0.8
        return v
    return signal(kind, n, g, speech)


def mel_tables(kind: str):
    """(window, fb) fp32 as the kernel receives them, and whether to pass them (False: the C defaults)"""
    window, fb = frontend.mel_tables()
    if kind == "shipped":
        return window, fb, True
    if kind == "default":
        i = torch.arange(1024, dtype=F64)
        cfb = torch.empty(513 * 100)
        _lib.check(_lib.lib().ns2vc_mel_filterbank(cfb.data_ptr()))
        return (0.5 - 0.5 * torch.cos(2 * math.pi * i / 1024)).float(), cfb.view(513, 100), False
    if kind == "asym":                                             # positive, not symmetric
        m = torch.arange(1024, dtype=F64)
        return (0.6 - 0.4 * torch.cos(2 * math.pi * m / 1024) + 0.3 * m / 1024).float(), fb, True
    if kind == "odd_fb":                                           # an all-zero band, a band over all 513 bins, zeros inside a band
        fb = fb.clone()
        fb[:, 10] = 0
        fb[:, 50] = (0.01 + 0.002 * torch.arange(513) / 513).float()
        nz = (fb[:, 80] != 0).nonzero().flatten()
        fb[nz[1:-1:3], 80] = 0
        return window, fb, True
    raise ValueError(kind)


class MCase:
    def __init__(self, name, tables, lens, N, S, signals, seed):
        self.name, self.tables, self.lens, self.N, self.S, self.signals, self.seed = name, tables, lens, N, S, signals, seed


def mel_cases() -> List[MCase]:
    out = []
    for i, tab in enumerate(("shipped", "default", "asym", "odd_fb")):
        sig = [MEL_SIGNALS[(k + 4 * i) % len(MEL_SIGNALS)] for k in range(len(EDGE_LENS))]
        N = EDGE_LENS[-1] + 11
        out.append(MCase(f"{tab}_edges", tab, EDGE_LENS, N, 1 + N // 256, sig, 10 + i))
        n2 = 6000
        out.append(MCase(f"{tab}_signals", tab, [n2 - 37 * k for k in range(len(MEL_SIGNALS))], n2, 1 + n2 // 256, MEL_SIGNALS, 20 + i))
    out.append(MCase("shipped_S_short", "shipped", [4097, 2049, 1000], 4097, 1 + 4097 // 256 - 3, ["speech", "noise", "square"], 30))
    out.append(MCase("shipped_2p22", "shipped", [1 << 22], 1 << 22, 1 + (1 << 22) // 256, ["speech"], 31))
    return out


MEL_CASES = mel_cases()


def build_mel(c: MCase, speech: torch.Tensor) -> torch.Tensor:
    g = torch.Generator().manual_seed(c.seed)
    wav = torch.zeros(len(c.lens), c.N)
    for b, (n, s) in enumerate(zip(c.lens, c.signals)):
        wav[b, :n] = mel_signal(s, n, g, speech)
    return wav


def mel_truth(c: MCase, wav, b: int, dev):
    window, fb, _ = mel_tables(c.tables)
    return ko.log_mel_terms(wav[b].to(dev), c.lens[b], window.to(dev), fb.to(dev), c.S)


LOG_CLIP = math.log(ko.MEL_CLIP)


@pytest.mark.parametrize("c", [c for c in MEL_CASES if c.N < (1 << 20)], ids=lambda c: c.name)
def test_log_mel_reference_is_sensitive(c, speech):
    """CPU: kernel_oracle.log_mel_rows is mel_oracle's stages on the same tables, and each defect moves it by >= 16 x the
    interval wherever the case has the feature: any unclipped entry (a frame start off by one, a band shifted by a bin, power
    2), the Hann window (the symmetric one), entries between 1e-7 and 1e-6 (a clip at 1e-6), rows whose last frame reflects
    past the end (about L), and the click row (its frame's centre tap scaled by 1 + 2^-10)"""
    wav = build_mel(c, speech)
    window, fb, _ = mel_tables(c.tables)
    defects = {"frame_offset": dict(frame_offset=1), "band_shift": dict(band_shift=1), "power2": dict(power=2),
               "symmetric": dict(symmetric_window=True), "clip1e-6": dict(clip=1e-6), "about_L": dict(reflect_about_L=True),
               "tap_scale": dict(tap_scale=(512, 1 + 2.0 ** -10))}
    s = {k: 0.0 for k in defects}
    need = {"frame_offset", "band_shift", "power2", "about_L"}
    old_caught = set()
    for b, n in enumerate(c.lens):
        ref, lo, hi = mel_truth(c, wav, b, "cpu")
        F = ko.log_mel_frames(n, c.S)
        want = mel_oracle.log_mel_24k(wav[b, :n], F64, window, fb)[:, :F]
        assert torch.allclose(ref[:, :F], torch.clamp(want, min=LOG_CLIP), rtol=0, atol=1e-9)
        e32 = (mel_oracle.log_mel_24k(wav[b, :n], torch.float32, window, fb)[:, :F].to(F64) - want).abs().max()
        for k, kw in defects.items():
            d = ko.log_mel_rows(wav[b], n, window, fb, c.S, **kw)
            s[k] = max(s[k], float(ko.interval_ratio(d, ref, lo, hi).max()))
            if float((d[:, :F] - ref[:, :F]).abs().max()) > 3 * float(e32):
                old_caught.add(k)
        if c.tables in ("shipped", "default"):
            need.add("symmetric")
        if ((ref[:, :F] > LOG_CLIP + 1e-9) & (ref[:, :F] < math.log(1e-6))).any():
            need.add("clip1e-6")
        if c.signals[b] == "click" and n > CLICK_AT + 512:
            need.add("tap_scale")
    for k in need:
        assert s[k] >= SENSITIVITY, f"{c.name}: {k} moves the result by only {s[k]:.2f} x the interval ({s})"
    print(f"{c.name}: defect / interval {', '.join(f'{k} {v:.3g}' for k, v in s.items())}; missed by 3 e_ref: {sorted(set(s) - old_caught)}")


def test_oracle_stages_equal_the_recipe(gold):
    """mel_oracle's stages with the shipped tables are its recipe, and reproduce torchaudio's fp64 pins of the fixture"""
    fx = gold("frontend_mel.pt")
    window, fb = frontend.mel_tables()
    for name, cs in fx["cases"].items():
        x24 = mel_oracle.resample(cs["pcm_int16"].float() / 32768.0, cs["sr"], 24000, F64)
        a = mel_oracle.log_mel_24k(x24, F64, window, fb)
        assert torch.equal(a, mel_oracle.log_mel_24k(x24, F64)), name
        fr = __import__("oracle.make_golden_mel", fromlist=["pin_frames"]).pin_frames(cs["frames"])
        assert (a[:, fr] - cs["pin_mel_f64"].double()).abs().max() <= 1e-12, name
        ref = ko.log_mel_rows(x24.float(), x24.numel(), window, fb, cs["frames"])   # on the fp32-rounded row
        assert torch.allclose(ref, torch.clamp(mel_oracle.log_mel_24k(x24.float(), F64, window, fb), min=LOG_CLIP), rtol=0, atol=1e-9)


def test_log_mel_interval_in_loud_bands(gold):
    """CPU: how wide the interval is where the log-mel is >= 0, on the fixture's speech (1.wav, 2.wav at 24 kHz, resampled by
    the fp32 recipe).  Printed as quantiles of the half-width, with the share of loud entries above 1e-4 and above the parity
    rule; asserted at the levels the node-by-node FFT bound reaches, so a looser bound fails here"""
    fx = gold("frontend_mel.pt")
    window, fb = frontend.mel_tables()
    for name in ("1.wav", "2.wav"):
        cs = fx["cases"][name]
        x24 = mel_oracle.resample(cs["pcm_int16"].float() / 32768.0, cs["sr"], 24000, torch.float32)
        L = x24.numel()
        ref, lo, hi = ko.log_mel_terms(x24, L, window, fb, 1 + L // 256)
        loud = ref >= 0
        hw = torch.maximum(hi - ref, ref - lo)[loud]
        q50, q90, q99 = torch.quantile(hw, torch.tensor([0.5, 0.9, 0.99], dtype=F64)).tolist()
        above, wider = float((hw > 1e-4).double().mean()), float((hw > ko.rule_tol(ref)[loud]).double().mean())
        print(f"{name}: {int(loud.sum())} loud entries, half-width median {q50:.2e}, 90 % {q90:.2e}, 99 % {q99:.2e}, max "
              f"{float(hw.max()):.2e}; {100 * above:.1f} % above 1e-4, {100 * wider:.1f} % wider than the parity rule")
        assert q50 <= 6e-5 and q90 <= 5e-4 and float(hw.max()) <= 3e-3 and wider <= 0.1, name


class MelHandle:
    def __init__(self, c: MCase):
        window, fb, pass_tables = mel_tables(c.tables)
        self.h = C.c_void_p()
        _lib.check(_lib.lib().ns2vc_mel_create(window.data_ptr() if pass_tables else None, fb.data_ptr() if pass_tables else None,
                                               C.byref(self.h)))

    def __del__(self):
        _lib.lib().ns2vc_mel_destroy(self.h)


def launch_mel(c: MCase, wav: torch.Tensor, dev, h: MelHandle, poison=False, only=None, nan_at=None, value=float("nan")):
    bsel = list(range(len(c.lens))) if only is None else [only]
    B, slack = len(bsel), 7
    x = torch.zeros(B, c.N + slack, device=dev)
    x[:, :c.N] = wav[bsel].to(dev)
    if poison:
        for i, b in enumerate(bsel):
            x[i, c.lens[b]:] = float("nan")
    if nan_at is not None:
        x[nan_at] = value
    lens = torch.tensor([c.lens[b] for b in bsel], dtype=torch.int64, device=dev)
    mel = torch.full((B, 100, c.S), float("nan"), device=dev)
    _lib.check(_lib.lib().ns2vc_log_mel(h.h, x.data_ptr(), c.N + slack, c.N, lens.data_ptr(), mel.data_ptr(), c.S, B, stream()))
    torch.cuda.synchronize()
    return mel


def frames_holding(n: int, F: int, i: int, dev) -> torch.Tensor:
    """[F] frames whose reflect-padded window holds sample i of a row of n samples"""
    return (ko._reflect_index(n, F, device=dev) == i).any(-1)


@gpu
@pytest.mark.parametrize("c", MEL_CASES, ids=lambda c: c.name)
def test_log_mel_kernel(c, speech):
    dev = torch.device("cuda")
    wav = build_mel(c, speech)
    h = MelHandle(c)
    mel = launch_mel(c, wav, dev, h)
    window, fb, _ = mel_tables(c.tables)
    worst = rule = vs32 = 0.0
    clip_vals = set()
    for b, n in enumerate(c.lens):
        F = ko.log_mel_frames(n, c.S)
        assert (mel[b, :, F:] == 0).all(), f"{c.name} row {b}: not 0 past its {F} frames"
        ref, lo, hi = mel_truth(c, wav, b, dev)
        got = mel[b].to(F64)
        # an entry whose whole interval is clipped must be logf(1e-7f) exactly: one value, within logf's ulp of log(1e-7f)
        clipped = (hi == lo) & (ref == LOG_CLIP)
        clip_vals |= set(got[clipped].tolist())
        if c.signals[b] == "silence":
            assert clipped[:, :F].all()
        r = float(ko.interval_ratio(torch.where(clipped, ref, got), ref, lo, hi).max())
        assert r <= 1.0, f"{c.name} row {b} ({c.signals[b]}, {n} samples): {r:.3f} of the interval"
        w32 = mel_oracle.log_mel_24k(wav[b, :n].to(dev), torch.float32, window.to(dev), fb.to(dev))[:, :F].to(F64)
        want = ref[:, :F]
        rr = ko.ratio(got[:, :F] - want, ko.parity_tol(want, float((w32 - want).abs().max())))
        assert rr <= 1.0, f"{c.name} row {b}: {rr:.3f} of the parity rule"
        loud = want >= 0
        if loud.any():
            e32 = float((w32 - want)[loud].abs().max())
            vs32 = max(vs32, float((got[:, :F] - want)[loud].abs().max()) / max(e32, 1e-30))
        worst, rule = max(worst, r), max(rule, rr)
    assert len(clip_vals) <= 1 and all(abs(v - LOG_CLIP) <= 2.0 ** -23 * abs(LOG_CLIP) for v in clip_vals), clip_vals
    # NaN from each row's length to the stride changes no bit, and so this second launch is bit-identical
    assert torch.equal(launch_mel(c, wav, dev, h, poison=True), mel)
    if len(c.lens) > 1:
        for b in (0, 1, len(c.lens) - 1):
            assert torch.equal(launch_mel(c, wav, dev, h, only=b)[0], mel[b]), f"{c.name}: row {b} differs alone"
    if c.name == "shipped_signals":                                  # NaN / Inf reach, mirrored positions near both ends included
        b = 0
        n, F = c.lens[b], ko.log_mel_frames(c.lens[b], c.S)
        for i, v in ((0, float("nan")), (5, float("nan")), (300, float("nan")), (n // 2, float("inf")), (n - 3, float("nan")),
                     (n - 1, float("-inf"))):
            got = launch_mel(c, wav, dev, h, nan_at=(b, i), value=v)
            hit = frames_holding(n, F, i, dev)
            bad = got[b, :, :F]
            if math.isnan(v):
                assert bad[:, hit].isnan().all() and not bad[:, ~hit].isnan().any(), f"a NaN at sample {i}"
            else:
                assert not bad[:, hit].isfinite().any() and bad[:, ~hit].isfinite().all(), f"{v} at sample {i}"
            assert torch.equal(bad[:, ~hit], mel[b, :, :F][:, ~hit]) and torch.equal(got[1:], mel[1:])
    record("log_mel (interval)", worst)
    record("log_mel (rule)", rule)
    print(f"{c.name}: worst ratio {worst:.3f} of the interval, {rule:.3f} of the rule; loud entries' error {vs32:.3g} x the "
          f"fp32 recipe's")
    record("log_mel loud error / fp32 recipe's (information)", vs32)
