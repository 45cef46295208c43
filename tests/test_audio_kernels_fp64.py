"""The content encoder's first conv (cv_gn_stats + cv_conv0) and positional conv (cv_pos_windows, one gemm_tc per group,
cv_add), and the vocoder's ISTFT (voc_istft_kernel) launch by launch, through the test-only C entry points of
csrc/kernel_check.cu (ns2vc_check_cv_conv0, _cv_pos_conv, _istft), which run the engines' own launchers, weight packer, GEMM
builder and twiddle tables, at every configuration the engines accept: conv_dim 128 .. 1024, positional-conv group widths
4 .. 64 and kernels 16 .. 128, n_fft 64 .. 2048 at three row pitches.  Every case asserts the instantiation it launched.

Truth: the pinned oracles' stages in fp64 on the kernel's own fp32 inputs (content_oracle.conv_layer / pos_conv,
vocos_oracle.head_istft), each row alone on its own samples or frames.  Rule: the model-level parity rule per row,
1e-3 |ref| + 1e-4 rms(ref) floored at 2 e32 (e32 = max |fp32 - fp64| of the same operation on the same row), plus the design's
error terms, derived in oracle/kernel_oracle.py:
  * conv 0: the fp32 conv and the fp32 mean subtraction, (10 sum |w||x| + |mean|) 2^-24 rstd |gamma|, which under a DC offset
    is the design's cancellation, the fp64 one-pass statistics, and the 2^-17 of the bf16 hi/lo output (conv0_terms);
  * positional conv: the 3xBF16 product of the split windows and weights and the fp32 accumulation (pos_conv_terms);
  * ISTFT: none.  Its fp32 radix-2 transform stays inside the rule alone up to n_fft = 2048, so its bound is the rule.
Each case prints its ratio to the bound and to the rule alone; the module prints the worst of each family.

No bound is vacuous (the CPU tier): GroupNorm statistics over the padded frames, the unbiased variance and a dropped eps
(seen on the silent and impulse rows), a window tap shifted by one and SamePad's dropped frame kept, and an envelope over
frames past the row's length, a reversed window and the clip applied before exp each move the fp64 reference by >= 16 x the
bound in every case that has the feature.

Exact properties: outputs at or past each row's length are exactly 0 (past L_b the positional conv's output is x itself); a
ragged row equals the same row launched alone; NaN where nothing may be read (wav samples past N_b, ISTFT frames past L_b and
columns >= n_fft + 2 inside ld, x rows past L_b for the windows) changes no bit; the windows are the split of the shifted frames;
one NaN log-magnitude makes NaN exactly the samples whose frames include it; a second launch is bit-identical.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, List, Sequence

import pytest
import torch

from conftest import REPO  # noqa: F401  (puts the repository on sys.path)
from ns2vc_b200 import _lib
from oracle import content_oracle as co
from oracle import kernel_oracle as ko
from oracle import vocos_oracle as vo

F64 = torch.float64
SENSITIVITY = 16.0
WORST: Dict[str, float] = {}


def gpu(f):
    """a GPU case: marked `gpu`, skipped where there is no CUDA device"""
    return pytest.mark.gpu(pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")(f))


class Split(C.Structure):
    _fields_ = [("hi", C.c_void_p), ("lo", C.c_void_p), ("T", C.c_int), ("C", C.c_int), ("ld", C.c_int), ("bpitch", C.c_longlong)]


class Conv0Args(C.Structure):
    _fields_ = [("wav", C.c_void_p), ("bstride", C.c_longlong), ("lengths", C.c_void_p), ("B", C.c_int), ("N", C.c_int), ("C0", C.c_int),
                ("w0", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p), ("eps", C.c_float), ("stats", C.c_void_p),
                ("out", Split), ("rows", C.c_int)]


class PosConvArgs(C.Structure):
    _fields_ = [("x", C.c_void_p), ("B", C.c_int), ("T", C.c_int), ("D", C.c_int), ("G", C.c_int), ("K", C.c_int), ("frames", C.c_void_p),
                ("w", C.c_void_p), ("bias", C.c_void_p), ("keep", C.c_void_p), ("win_hi", C.c_void_p), ("win_lo", C.c_void_p),
                ("out", C.c_void_p), ("windows_only", C.c_int)]


class IstftArgs(C.Structure):
    _fields_ = [("h", C.c_void_p), ("ld", C.c_int), ("len", C.c_void_p), ("B", C.c_int), ("T", C.c_int), ("n_fft", C.c_int),
                ("window", C.c_void_p), ("audio", C.c_void_p)]


def stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def call(fn, args) -> str:
    desc = C.create_string_buffer(128)
    _lib.check(fn(C.cast(C.byref(args), C.c_void_p), desc, 128, stream()))
    torch.cuda.synchronize()
    return desc.value.decode()


def record(family: str, r: float) -> None:
    WORST[family] = max(WORST.get(family, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    for fam, r in sorted(WORST.items()):
        print(f"\n[audio kernel checks] {fam}: worst ratio {r:.3g}")


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def row_bound(ref: torch.Tensor, ref32: torch.Tensor, extra: torch.Tensor) -> torch.Tensor:
    """the parity rule of one row (floored at 2 e32 of that row) plus the design's terms"""
    e32 = float((ref32.to(F64) - ref).abs().max()) if ref.numel() else 0.0
    return ko.parity_tol(ref, e32) + extra


def rule_of(ref: torch.Tensor, ref32: torch.Tensor) -> torch.Tensor:
    e32 = float((ref32.to(F64) - ref).abs().max()) if ref.numel() else 0.0
    return ko.parity_tol(ref, e32)


def moved(defect: torch.Tensor, ref: torch.Tensor, tol: torch.Tensor) -> float:
    return float(((defect - ref).abs() / tol).max()) if ref.numel() else 0.0


# ---------------------------------------------------------------------------------------------------------------------------
# conv 0: cv_gn_stats + cv_conv0
# ---------------------------------------------------------------------------------------------------------------------------
SIGNALS = ["noise", "dc1e2", "dc1e3", "dc1e4", "silent", "impulse", "square"]
# <= 0 and 399 clamp to 400; 400 / 404 give T0 = 79, 405 80, 410 81, 480 95, 485 96, 490 97 (the 16-frame CTA edges); N = 1000
# gives T0 = 199, odd, so rows[0] = 200 carries the pad row
CONV0_LENS = [-5, 399, 400, 404, 405, 410, 480, 485, 490, 1000]
CONV0_N = 1000


class Conv0Case:
    def __init__(self, name, C0, lens, N, signals, seed):
        self.name, self.C0, self.lens, self.N, self.signals, self.seed = name, C0, lens, N, signals, seed

    @property
    def samples(self) -> List[int]:
        return [min(max(n, 400), self.N) for n in self.lens]


def conv0_cases() -> List[Conv0Case]:
    out = []
    for C0 in (128, 256, 512, 768, 1024):
        for k, rot in enumerate((0, 3)):
            sig = [SIGNALS[(i + rot + C0 // 128) % len(SIGNALS)] for i in range(len(CONV0_LENS))]
            out.append(Conv0Case(f"C{C0}_mix{k}", C0, CONV0_LENS, CONV0_N, sig, C0 + k))
    out.append(Conv0Case("C512_30s", 512, [480000], 480000, ["noise"], 5))
    out.append(Conv0Case("C128_2p22_dc1e2", 128, [1 << 22], 1 << 22, ["dc1e2"], 6))
    return out


CONV0_CASES = conv0_cases()


def build_conv0(c: Conv0Case) -> Dict:
    g = torch.Generator().manual_seed(c.seed)
    B = len(c.lens)
    wav = torch.zeros(B, c.N)
    for b, (n, s) in enumerate(zip(c.samples, c.signals)):
        ac = 0.1 * torch.randn(n, generator=g)
        if s == "noise":
            v = ac
        elif s.startswith("dc"):
            v = ac + float(s[2:]) * 0.1                                  # a DC offset of 10^2 .. 10^4 x the AC amplitude
        elif s == "silent":
            v = torch.zeros(n)
        elif s == "impulse":                                            # one sample: two frames of each channel are nonzero
            v = torch.zeros(n)
            v[n // 2 + 3] = 0.05
        else:                                                           # full-scale square wave, period 37 samples
            v = torch.where((torch.arange(n) // 37) % 2 == 0, torch.ones(n), -torch.ones(n))
        wav[b, :n] = v
    w0 = torch.randn(c.C0, 1, 10, generator=g) / math.sqrt(10)
    gamma = 1 + 0.3 * torch.randn(c.C0, generator=g)
    beta = torch.randn(c.C0, generator=g)                               # |beta| ~ 1: outputs near GELU's zero occur
    return dict(wav=wav, w0=w0, gamma=gamma, beta=beta)


def conv0_sd(d, dt, dev):
    return {"feature_extractor.conv_layers.0.0.weight": d["w0"].to(dev, dt), "feature_extractor.conv_layers.0.2.weight": d["gamma"].to(dev, dt),
            "feature_extractor.conv_layers.0.2.bias": d["beta"].to(dev, dt)}


def conv0_truth(c: Conv0Case, d, b: int, dev, dt=F64) -> torch.Tensor:
    """the oracle's conv-0 stage of row b alone: [T0_b, C0]"""
    return co.conv_layer(conv0_sd(d, dt, dev), 0, d["wav"][b, :c.samples[b]].to(dev, dt))


def conv0_rows_of(c: Conv0Case) -> int:
    T0 = (c.N - 10) // 5 + 1
    return T0 + (T0 & 1)


@pytest.mark.parametrize("c", [c for c in CONV0_CASES if len(c.lens) > 1], ids=lambda c: c.name)
def test_conv0_reference_is_sensitive(c):
    """CPU: kernel_oracle.conv0_rows is the oracle's conv-0 stage, and the bound notices GroupNorm over the padded frames
    (ragged rows with signal), the unbiased variance (every case) and a dropped eps (the silent and impulse rows)"""
    d = build_conv0(c)
    worst = {"padded": 0.0, "unbiased": 0.0, "eps": 0.0}
    has = {"padded": False}
    for b, n in enumerate(c.samples):
        ref = conv0_truth(c, d, b, "cpu")
        args = (d["wav"][b].to(F64), n, d["w0"].to(F64), d["gamma"].to(F64), d["beta"].to(F64), 1e-5)
        if c.signals[b] == "silent":                                 # variance 0: GELU(beta) exactly
            assert torch.equal(ref, torch.nn.functional.gelu(d["beta"].to(F64)).expand_as(ref))
        tol = row_bound(ref, conv0_truth(c, d, b, "cpu", torch.float32), ko.conv0_terms(*args))
        # the same operation as the oracle's, to fp64 rounding (which a DC offset of 10^4 std magnifies 10^8 times)
        assert moved(ko.conv0_rows(*args), ref, tol) < 1e-3
        if n < c.N and c.signals[b] != "silent":
            has["padded"] = True
            worst["padded"] = max(worst["padded"], moved(ko.conv0_rows(*args, padded_stats=True), ref, tol))
        worst["unbiased"] = max(worst["unbiased"], moved(ko.conv0_rows(*args, unbiased=True), ref, tol))
        if c.signals[b] in ("silent", "impulse"):
            bad = ko.conv0_rows(*args, use_eps=False)
            if c.signals[b] == "silent":                             # 0 / 0: every output NaN
                assert torch.isnan(bad).all()
            else:
                worst["eps"] = max(worst["eps"], moved(bad, ref, tol))
    assert worst["unbiased"] >= SENSITIVITY, f"{c.name}: the unbiased variance moves the result by only {worst['unbiased']:.1f} x"
    assert not has["padded"] or worst["padded"] >= SENSITIVITY, f"{c.name}: padded statistics move it by only {worst['padded']:.1f} x"
    assert "impulse" not in c.signals or worst["eps"] >= SENSITIVITY, f"{c.name}: a dropped eps moves it by only {worst['eps']:.1f} x"


def launch_conv0(c: Conv0Case, d, dev, poison=False, only=None):
    bsel = list(range(len(c.lens))) if only is None else [only]
    B, slack = len(bsel), 3
    wav = torch.zeros(B, c.N + slack, device=dev)
    wav[:, :c.N] = d["wav"][bsel].to(dev)
    if poison:                                                       # samples past N_b (and the stride's slack) are never read
        for i, b in enumerate(bsel):
            wav[i, c.samples[b]:] = float("nan")
    lens = torch.tensor([c.lens[b] for b in bsel], dtype=torch.int64, device=dev)
    rows = conv0_rows_of(c)
    hi = torch.full((B * rows, c.C0), 0x7fc0, dtype=torch.int16, device=dev)   # bf16 NaN: every element must be written
    lo = hi.clone()
    stats = torch.full((B, c.C0, 2), float("nan"), device=dev)
    w0, gm, bt = d["w0"].to(dev), d["gamma"].to(dev), d["beta"].to(dev)
    a = Conv0Args(wav.data_ptr(), c.N + slack, lens.data_ptr(), B, c.N, c.C0, w0.data_ptr(), gm.data_ptr(), bt.data_ptr(), 1e-5,
                  stats.data_ptr(), Split(hi.data_ptr(), lo.data_ptr(), rows, c.C0, c.C0, 0), rows)
    desc = call(_lib.lib().ns2vc_check_cv_conv0, a)
    assert desc == f"cv_gn_stats+cv_conv0<{c.C0 // 2}>", desc
    return hi.reshape(B, rows, c.C0), lo.reshape(B, rows, c.C0), stats


@gpu
@pytest.mark.parametrize("c", CONV0_CASES, ids=lambda c: c.name)
def test_cv_conv0(c):
    dev = torch.device("cuda")
    d = build_conv0(c)
    hi, lo, stats = launch_conv0(c, d, dev)
    got = hi.view(torch.bfloat16).to(F64) + lo.view(torch.bfloat16).to(F64)
    worst = rule = 0.0
    for b, n in enumerate(c.samples):
        T0 = (n - 10) // 5 + 1
        assert (hi[b, T0:] == 0).all() and (lo[b, T0:] == 0).all(), f"{c.name}: row {b} is not 0 past its {T0} frames"
        ref = conv0_truth(c, d, b, dev)
        ref32 = conv0_truth(c, d, b, dev, torch.float32)
        wav_b = d["wav"][b].to(dev)
        extra = ko.conv0_terms(wav_b, n, d["w0"].to(dev), d["gamma"].to(dev), d["beta"].to(dev), 1e-5)
        err = got[b, :T0] - ref
        r = ko.ratio(err, row_bound(ref, ref32, extra))
        assert r <= 1.0, f"{c.name} row {b} ({c.signals[b]}, {n} samples): {r:.3f} of the bound (max |err| {float(err.abs().max()):.3e})"
        worst, rule = max(worst, r), max(rule, ko.ratio(err, rule_of(ref, ref32)))
        # the statistics against fp64 sums of the kernel's own fp32 conv, to their fp32 rounding and the fp64 one-pass sums
        y32 = ko.conv0_fp32(wav_b, n, d["w0"].to(dev))
        mean, var, mean_tol, var_err = ko.conv0_stats_tol(y32)
        eps = float(torch.tensor(1e-5, dtype=torch.float32))         # the kernel's eps argument
        rstd = 1.0 / torch.sqrt(var + eps)
        rstd_tol = rstd * (ko.U32 + var_err / (2 * (var + eps)))
        st = stats[b].to(F64)
        assert ((st[:, 0] - mean).abs() <= mean_tol).all(), f"{c.name} row {b}: mean off by {float(((st[:, 0] - mean).abs() / mean_tol).max()):.2f} x"
        assert ((st[:, 1] - rstd).abs() <= rstd_tol).all(), f"{c.name} row {b}: rstd off by {float(((st[:, 1] - rstd).abs() / rstd_tol).max()):.2f} x"
    # NaN past N_b changes no bit, and so this second launch is bit-identical to the first
    hi_p, lo_p, stats_p = launch_conv0(c, d, dev, poison=True)
    assert torch.equal(hi_p, hi) and torch.equal(lo_p, lo) and torch.equal(stats_p, stats)
    if len(c.lens) > 1 and c.name.endswith("mix0"):                 # each ragged row equals that row launched alone
        for b in range(len(c.lens)):
            ah, al, ast = launch_conv0(c, d, dev, only=b)
            assert torch.equal(ah[0], hi[b]) and torch.equal(al[0], lo[b]) and torch.equal(ast[0], stats[b]), f"{c.name}: row {b} differs alone"
    record("cv_conv0", worst)
    record("cv_conv0 (rule alone)", rule)
    print(f"{c.name}: worst ratio {worst:.3f} (rule alone {rule:.3f})")


# ---------------------------------------------------------------------------------------------------------------------------
# positional conv: cv_pos_windows, one gemm_tc per group, cv_add
# ---------------------------------------------------------------------------------------------------------------------------
POS_CASES = [  # (D, G, K, T): group widths 4, 8, 32, 48, 64; K 16 .. 128; T 1 .. 1049
    (128, 32, 16, 1), (128, 32, 16, 65), (256, 32, 32, 2), (256, 32, 32, 129), (384, 8, 48, 15), (384, 8, 48, 1049),
    (512, 16, 32, 63), (512, 8, 64, 64), (768, 16, 128, 65), (1024, 16, 128, 129), (1024, 16, 128, 1049),
]


def pos_id(p) -> str:
    D, G, K, T = p
    return f"D{D}_gw{D // G}_K{K}_T{T}"


def pos_lens(K: int, T: int) -> List[int]:
    """1, K/2 - 1, K/2, K/2 + 1, T - 1, T within [1, T] (rows shorter than K/2: every tap of some outputs is outside the row)"""
    return sorted({min(max(v, 1), T) for v in (1, K // 2 - 1, K // 2, K // 2 + 1, T - 1, T)})


def build_pos(p) -> Dict:
    D, G, K, T = p
    g = torch.Generator().manual_seed(D * 7 + K + T)
    L = pos_lens(K, T)
    B, gw = len(L), D // G
    x = torch.randn(B, T, D, generator=g)
    x = x + 30 * torch.rand(1, 1, D, generator=g) * torch.sign(torch.randn(1, 1, D, generator=g))   # channel means up to 30 std
    W = torch.randn(D, gw, K, generator=g) / math.sqrt(gw * K) * 3
    bias = 0.5 * torch.randn(D, generator=g)
    return dict(x=x, W=W, bias=bias, L=L)


def pos_truth(p, d, dev, dt=F64) -> torch.Tensor:
    """the oracle's positional-conv stage of each row alone (weight norm given as the per-tap norms of the fp32 folded weight,
    so it folds back to that weight), rows past L_b equal to x"""
    W = d["W"].to(dev, dt)
    sd = {"encoder.pos_conv.0.weight_g": W.pow(2).sum(dim=(0, 1), keepdim=True).sqrt(), "encoder.pos_conv.0.weight_v": W,
          "encoder.pos_conv.0.bias": d["bias"].to(dev, dt)}
    x = d["x"].to(dev, dt)
    out = x.clone()
    for b, n in enumerate(d["L"]):
        out[b, :n] = co.pos_conv(sd, x[b, :n])
    return out


@pytest.mark.parametrize("p", POS_CASES, ids=pos_id)
def test_pos_conv_reference_is_sensitive(p):
    """CPU: kernel_oracle.pos_conv_rows is the oracle's stage, and the bound notices a tap shifted by one and SamePad's
    dropped frame kept (every row shorter than T)"""
    D, G, K, T = p
    d = build_pos(p)
    ref = pos_truth(p, d, "cpu")
    x64, W64 = d["x"].to(F64), d["W"].to(F64)
    assert torch.allclose(ko.pos_conv_rows(x64, W64, d["bias"].to(F64), d["L"]), ref, rtol=1e-10, atol=1e-10)
    ref32 = pos_truth(p, d, "cpu", torch.float32)
    extra = ko.pos_conv_terms(d["x"], d["W"], d["bias"], d["L"])
    shifted = ko.pos_conv_rows(x64, W64, d["bias"].to(F64), d["L"], shift=1)
    kept = ko.pos_conv_rows(x64, W64, d["bias"].to(F64), d["L"], keep_last=True)
    s_shift = s_kept = 0.0
    for b, n in enumerate(d["L"]):
        tol = row_bound(ref[b], ref32[b], extra[b])
        s_shift = max(s_shift, moved(shifted[b], ref[b], tol))
        if n < T:
            s_kept = max(s_kept, moved(kept[b], ref[b], tol))
    assert s_shift >= SENSITIVITY, f"a shifted tap moves the result by only {s_shift:.1f} x the bound"
    assert T == 1 or s_kept >= SENSITIVITY, f"the kept SamePad frame moves the result by only {s_kept:.1f} x the bound"


def launch_pos(p, d, dev, windows_only=False, poison=False, only=None):
    D, G, K, T = p
    bsel = list(range(len(d["L"]))) if only is None else [only]
    B = len(bsel)
    x = d["x"][bsel].to(dev).contiguous()
    if poison:
        for i, b in enumerate(bsel):
            x[i, d["L"][b]:] = float("nan")
    frames = torch.tensor([d["L"][b] for b in bsel], dtype=torch.int64, device=dev)
    keep = (torch.arange(T, device=dev)[None, :] < frames[:, None]).float()
    W, bias = d["W"].to(dev), d["bias"].to(dev)
    win_hi = torch.full((B, G, T + K, 1024), 0x7fc0, dtype=torch.int16, device=dev)
    win_lo = win_hi.clone()
    out = torch.full((B, T, D), float("nan"), device=dev)
    a = PosConvArgs(x.data_ptr(), B, T, D, G, K, frames.data_ptr(), W.data_ptr(), bias.data_ptr(), keep.data_ptr(), win_hi.data_ptr(),
                    win_lo.data_ptr(), out.data_ptr(), int(windows_only))
    desc = call(_lib.lib().ns2vc_check_cv_pos_conv, a)
    if windows_only:
        assert desc == "cv_pos_windows", desc
    else:
        assert desc.startswith(f"cv_pos_windows+{G}xgemm_tc<") and desc.endswith(",LNF=0,XF=0,ENC=0,RAG=0,VOC=1>+cv_add"), desc
    return win_hi, win_lo, out


def expected_windows(p, d, dev):
    """win[b, g, r, q * 64 + i] = x[b, r - K/2 + q, g gw + i] for q < 16, i < gw, inside the row's own frames; else 0"""
    D, G, K, T = p
    gw, B = D // G, len(d["L"])
    x = d["x"].to(dev)
    xp = torch.zeros(B, T + 2 * K + 16, D, device=dev)
    for b, n in enumerate(d["L"]):
        xp[b, K // 2:K // 2 + n] = x[b, :n]
    idx = torch.arange(T + K, device=dev)[:, None] + torch.arange(16, device=dev)[None, :]          # row r + q of xp
    w = xp[:, idx].reshape(B, T + K, 16, G, gw).permute(0, 3, 1, 2, 4)
    w = torch.nn.functional.pad(w, (0, 64 - gw)).reshape(B, G, T + K, 1024)
    return ko.split(w)


@gpu
@pytest.mark.parametrize("p", POS_CASES, ids=pos_id)
def test_cv_pos_conv(p):
    D, G, K, T = p
    dev = torch.device("cuda")
    d = build_pos(p)
    # the windows alone: the split of the shifted frames, bit for bit, and NaN in x past L_b changes no bit
    wh, wl, _ = launch_pos(p, d, dev, windows_only=True)
    eh, el = expected_windows(p, d, dev)
    assert torch.equal(wh.view(torch.bfloat16), eh) and torch.equal(wl.view(torch.bfloat16), el), "windows are not the split of the frames"
    ph, pl, _ = launch_pos(p, d, dev, windows_only=True, poison=True)
    assert torch.equal(ph, wh) and torch.equal(pl, wl)
    _, _, out = launch_pos(p, d, dev)
    ref = pos_truth(p, d, dev)
    ref32 = pos_truth(p, d, dev, torch.float32)
    extra = ko.pos_conv_terms(d["x"].to(dev), d["W"].to(dev), d["bias"].to(dev), d["L"])
    x = d["x"].to(dev)
    worst = rule = 0.0
    for b, n in enumerate(d["L"]):
        assert torch.equal(out[b, n:], x[b, n:]), f"row {b}: past its {n} frames the output is not x"
        err = out[b].to(F64) - ref[b]
        r = ko.ratio(err, row_bound(ref[b], ref32[b], extra[b]))
        assert r <= 1.0, f"{pos_id(p)} row {b} (L = {n}): {r:.3f} of the bound (max |err| {float(err.abs().max()):.3e})"
        worst, rule = max(worst, r), max(rule, ko.ratio(err, rule_of(ref[b], ref32[b])))
    _, _, out2 = launch_pos(p, d, dev)                               # a second launch is bit-identical
    assert torch.equal(out2, out)
    for b in (0, len(d["L"]) // 2):                                  # a ragged row equals the row launched alone
        _, _, alone = launch_pos(p, d, dev, only=b)
        assert torch.equal(alone[0], out[b]), f"row {b} differs alone"
    record(f"pos conv gw={D // G}", worst)
    record("pos conv (rule alone)", rule)
    print(f"{pos_id(p)}: worst ratio {worst:.3f} (rule alone {rule:.3f})")


# ---------------------------------------------------------------------------------------------------------------------------
# ISTFT: voc_istft_kernel
# ---------------------------------------------------------------------------------------------------------------------------
ISTFT_T = [1, 2, 3, 12, 13, 14, 25, 26, 27, 300, 1001]               # T + 1 on and around the 13-hop CTA edge
ISTFT_NFFT = [64, 128, 256, 512, 1024, 2048]
MAG_REGIMES = ["normal", "ln100", "big", "m80"]


def istft_cases() -> List[tuple]:
    """(n_fft, T, ld kind): every T at two n_fft, every n_fft at the three pitches"""
    out = []
    for i, n in enumerate(ISTFT_NFFT):
        for j in range(4):
            T = ISTFT_T[(i * 4 + j) % len(ISTFT_T)]
            out.append((n, T, (i + j) % 3))
    return out


ISTFT_CASES = istft_cases()


def istft_id(c) -> str:
    n, T, k = c
    return f"n{n}_T{T}_ld{['tight', 'pad4', 'wide'][k]}"


def istft_ld(n: int, kind: int) -> int:
    return [n + 2, (n + 2 + 3) // 4 * 4, n + 64][kind]


def istft_lens(T: int) -> List[int]:
    return sorted({min(max(v, 1), T) for v in (1, 2, 3, 4, 5, 13, 14, T - 1, T)})


def build_istft(c) -> Dict:
    n, T, kind = c
    g = torch.Generator().manual_seed(n + 31 * T + kind)
    L = istft_lens(T)
    B, nb = len(L), n // 2 + 1
    mag = torch.randn(B, T, nb, generator=g)
    for b in range(B):
        reg = MAG_REGIMES[b % len(MAG_REGIMES)]
        if reg == "ln100":                                          # within 1e-6 of ln 100: both sides of the clip
            mag[b] = math.log(100.0) + 1e-6 * (2 * torch.rand(T, nb, generator=g) - 1)
        elif reg == "big":                                          # 50, 88.7 (exp just below fp32 overflow), 100 (overflows)
            mag[b] = torch.tensor([50.0, 88.7, 100.0])[torch.randint(0, 3, (T, nb), generator=g)] + torch.where(
                torch.rand(T, nb, generator=g) < 0.5, torch.zeros(T, nb), mag[b])
        elif reg == "m80":
            mag[b] = -80.0 + mag[b]
    phase = (2 * torch.rand(B, T, nb, generator=g) - 1) * math.pi
    phase[1::2] *= 1e4 / math.pi                                     # |p| up to 1e4 on every other row
    h = torch.cat([mag, phase], -1)
    m = torch.arange(n, dtype=F64)
    window = (0.6 - 0.4 * torch.cos(2 * math.pi * m / n) + 0.3 * m / n).float()   # positive, not symmetric
    return dict(h=h, window=window, L=L)


def istft_truth(c, d, dev, dt=F64) -> torch.Tensor:
    """the oracle's ISTFT head of each row alone on its first L_b frames, zero past L_b hop samples"""
    n, T, _ = c
    hop = n // 4
    out = torch.zeros(len(d["L"]), T * hop, dtype=dt, device=dev)
    for b, L in enumerate(d["L"]):
        out[b, :L * hop] = vo.head_istft(d["h"][b:b + 1, :L].to(dev, dt), d["window"].to(dev, dt), hop)[0]
    return out


@pytest.mark.parametrize("c", ISTFT_CASES, ids=istft_id)
def test_istft_reference_is_sensitive(c):
    """CPU: kernel_oracle.istft_rows is the oracle's head, and the bound notices an envelope over frames past L_b (rows with
    L_b < T), a reversed window (every row) and the clip applied before exp (the rows with log-magnitudes of 50 .. 100)"""
    n, T, _ = c
    hop = n // 4
    d = build_istft(c)
    h64, w64 = d["h"].to(F64), d["window"].to(F64)
    ref = istft_truth(c, d, "cpu")
    assert torch.allclose(ko.istft_rows(h64, w64, hop, d["L"]), ref, rtol=1e-9, atol=1e-9 * float(ref.abs().max()))
    ref32 = istft_truth(c, d, "cpu", torch.float32)
    bad = {k: ko.istft_rows(h64, w64, hop, d["L"], **{k: True}) for k in ("env_all_frames", "reverse_window", "clip_first")}
    s = {k: 0.0 for k in bad}
    for b, L in enumerate(d["L"]):
        tol = rule_of(ref[b], ref32[b])
        s["reverse_window"] = max(s["reverse_window"], moved(bad["reverse_window"][b], ref[b], tol))
        if L < T:
            s["env_all_frames"] = max(s["env_all_frames"], moved(bad["env_all_frames"][b], ref[b], tol))
        if MAG_REGIMES[b % len(MAG_REGIMES)] == "big":
            s["clip_first"] = max(s["clip_first"], moved(bad["clip_first"][b], ref[b], tol))
    assert s["reverse_window"] >= SENSITIVITY, s
    assert T == 1 or s["env_all_frames"] >= SENSITIVITY, s
    assert len(d["L"]) < 3 or s["clip_first"] >= SENSITIVITY, s


def launch_istft(c, d, dev, poison=False, only=None, nan_at=None):
    n, T, kind = c
    ld = istft_ld(n, kind)
    bsel = list(range(len(d["L"]))) if only is None else [only]
    B = len(bsel)
    h = torch.zeros(B, T, ld, device=dev)
    h[..., :n + 2] = d["h"][bsel].to(dev)
    if poison:                                                       # frames past L_b and columns >= n_fft + 2 are never read
        h[..., n + 2:] = float("nan")
        for i, b in enumerate(bsel):
            h[i, d["L"][b]:] = float("nan")
    if nan_at is not None:
        h[nan_at] = float("nan")
    lens = torch.tensor([d["L"][b] for b in bsel], dtype=torch.int64, device=dev)
    win = d["window"].to(dev)
    audio = torch.full((B, T * (n // 4)), float("nan"), device=dev)
    a = IstftArgs(h.data_ptr(), ld, lens.data_ptr(), B, T, n, win.data_ptr(), audio.data_ptr())
    desc = call(_lib.lib().ns2vc_check_istft, a)
    log2m = int(math.log2(n)) - 1
    assert desc == f"voc_istft<log2m={log2m},smem={16 * n * 4}>", desc
    return audio


@gpu
@pytest.mark.parametrize("c", ISTFT_CASES, ids=istft_id)
def test_istft(c):
    n, T, kind = c
    hop = n // 4
    dev = torch.device("cuda")
    d = build_istft(c)
    audio = launch_istft(c, d, dev)
    ref = istft_truth(c, d, dev)
    ref32 = istft_truth(c, d, dev, torch.float32)
    rule = 0.0
    for b, L in enumerate(d["L"]):
        assert (audio[b, L * hop:] == 0).all(), f"row {b}: samples past {L} frames are not 0"
        err = audio[b].to(F64) - ref[b]
        r = ko.ratio(err, rule_of(ref[b], ref32[b]))
        assert r <= 1.0, f"{istft_id(c)} row {b} (L = {L}, {MAG_REGIMES[b % 4]}): {r:.3f} of the rule (max |err| {float(err.abs().max()):.3e})"
        rule = max(rule, r)
    # NaN where nothing is read changes no bit, and so this second launch is bit-identical to the first
    assert torch.equal(launch_istft(c, d, dev, poison=True), audio)
    for b in (0, len(d["L"]) - 1):                                   # a ragged row equals the row launched alone
        assert torch.equal(launch_istft(c, d, dev, only=b)[0], audio[b]), f"row {b} differs alone"
    # one NaN log-magnitude: NaN exactly where its frame overlaps the row's samples, every other sample unchanged
    b = len(d["L"]) - 1
    L = d["L"][b]
    f = L // 2
    nan_audio = launch_istft(c, d, dev, nan_at=(b, f, 3))
    pad = (n - hop) // 2
    hit = torch.zeros(T * hop, dtype=torch.bool, device=dev)
    hit[max(f * hop - pad, 0):min(f * hop + n - pad, L * hop)] = True
    assert torch.isnan(nan_audio[b][hit]).all() and not torch.isnan(nan_audio[b][~hit]).any()
    assert torch.equal(nan_audio[b][~hit], audio[b][~hit])
    others = [i for i in range(len(d["L"])) if i != b]
    assert torch.equal(nan_audio[others], audio[others])
    record(f"voc_istft n_fft={n} (rule alone)", rule)
    print(f"{istft_id(c)}: worst ratio {rule:.3f} (the rule alone)")
