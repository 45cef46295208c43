"""The stride-2 convolutions' row-pair GEMM views launch by launch: the denoiser's Downsample1D (down_conv: one GEMM over the
block input's raw split seen as row pairs, or two prep launches decimating it) and the content encoder's convs 1-6
(cv_conv_gemm: one GEMM over the previous level's split seen as row pairs), through the test-only C entry points
ns2vc_check_down_conv / ns2vc_check_cv_conv (csrc/kernel_check.cu), which run the engines' own host code.  Each case is
compared with three references (the machinery of tests/test_kernels_fp64.py and oracle/kernel_oracle.py):

* the emulation: gemm_emulate on the de-interleaved operand (even rows x[2t], odd rows x[2t+1]; for the content convs row
  2t+2 as tap 2), so the views must pick exactly the right rows and channels; |gpu - emu| <= tol_emu;
* the truth in fp64 from the input, under the parity rule 1e-3 |ref| + 1e-4 rms(ref): F.conv1d(x, W, b, stride=2, padding=1)
  for the denoiser, gelu(F.conv1d(x, W, stride=2)) times the keep mask for the content convs (no bias, no padding);
* a dense copy: the denoiser's launch with the prep path forced (prep_split decimation into dense even / odd splits), the
  content conv's GEMM over an explicit dense im2col copy of its operand; both must be bit-identical, since the TMA unit loads
  the same bf16 values in the same k-order.

No bound is vacuous: for every case the emulation is evaluated again with one defect injected - each of the three split
products dropped, the odd rows shifted by one row (x[2t+2]), the even rows read at 2t+1 and (content, k = 3) tap 2 read at
row 2t+1 - and each must move it by >= 16 x tol_emu somewhere.

Exact properties: rows at or past each entry's output frames are exactly 0 in the fp32 output and the split; the split is the
split of the fp32 output; entry b of a batch equals that entry launched alone, bit for bit; NaN where nothing valid reads
(channels past C inside the denoiser's ld; a content level's pad row and rows past an entry's frames) changes no valid
output bit; a second launch is bit-identical; the description names the instantiation the engine picks.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, List, Optional

import pytest
import torch
import torch.nn.functional as F

import test_kernels_fp64 as kf
from conftest import REPO  # noqa: F401  (puts the repository on sys.path)
from ns2vc_b200 import _lib
from oracle import kernel_oracle as ko
from test_content import batch_full
from test_kernels_fp64 import SENSITIVITY, _no_tf32, call, stream  # noqa: F401  (_no_tf32: autouse fixture)

F64 = torch.float64
gpu = pytest.mark.gpu
FAM = "strided "
NAN16 = 0x7fc0                                               # bf16 NaN: every valid output element must be written


class DownArgs(C.Structure):
    _fields_ = [("B", C.c_int), ("Tin", C.c_int), ("C", C.c_int), ("x", C.c_void_p), ("in_hi", C.c_void_p), ("in_lo", C.c_void_p),
                ("ld", C.c_int), ("w", C.c_void_p), ("bias", C.c_void_p), ("row_len", C.c_void_p), ("len_shift", C.c_int),
                ("out", C.c_void_p), ("out_hi", C.c_void_p), ("out_lo", C.c_void_p), ("force_prep", C.c_int)]


class CvConvArgs(C.Structure):
    _fields_ = [("B", C.c_int), ("rows_in", C.c_int), ("rows_out", C.c_int), ("C0", C.c_int), ("l", C.c_int), ("in_hi", C.c_void_p),
                ("in_lo", C.c_void_p), ("w", C.c_void_p), ("keep", C.c_void_p), ("out", C.c_void_p), ("out_hi", C.c_void_p),
                ("out_lo", C.c_void_p)]


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    for fam, w in sorted(kf.WORST.items()):
        if fam.startswith(FAM):
            print(f"\n[kernel checks] {fam}: " + ", ".join(f"{k}={v:.3g}" for k, v in sorted(w.items())))


def pad8(c: int) -> int:
    return (c + 7) // 8 * 8


def width64(c: int) -> int:
    return 64 * ((c + 63) // 64)


def rows_at(x: torch.Tensor, r: int, n: int) -> torch.Tensor:
    """rows r + 2t (t < n) of x [B, T, C], zero past its T rows"""
    need = r + 2 * n
    if need > x.shape[1]:
        x = F.pad(x, (0, 0, 0, need - x.shape[1]))
    return x[:, r:need:2]


def emulate(Ah: torch.Tensor, Al: torch.Tensor, W: torch.Tensor, ep: Dict, drop: Optional[int] = None):
    """ko.gemm_emulate on the given operand split, in row chunks (its running-magnitude term is [B, rows, N, K / 16])"""
    B, T, K = Ah.shape
    step = max(1, int(3e7 // (B * W.shape[0] * max(K // 16, 1))))
    emus, bounds = [], []
    for t0 in range(0, T, step):
        sl = slice(t0, t0 + step)
        e = {k: (v[:, sl] if k in ("rowmask", "row_valid") else v) for k, v in ep.items()}
        emu, bound = ko.gemm_emulate(None, W, e, drop, a_split=(Ah[:, sl], Al[:, sl]))
        emus.append(emu)
        bounds.append(bound)
    return torch.cat(emus, 1), (torch.cat(bounds, 1) if drop is None else None)


def sensitivities(operand, hi64, lo64, W, ep, emu, bound, defects: Dict[str, Dict]) -> Dict[str, float]:
    """max |defect - emu| / tol_emu of each dropped product and each operand defect (keyword arguments of `operand`)"""
    Ah, Al = operand(hi64), operand(lo64)
    s = {f"drop{i}": ko.ratio(emulate(Ah, Al, W, ep, drop=i)[0] - emu, bound) for i in range(3)}
    for name, kw in defects.items():
        s[name] = ko.ratio(emulate(operand(hi64, **kw), operand(lo64, **kw), W, ep)[0] - emu, bound)
    return s


def assert_sensitive(name: str, s: Dict[str, float]) -> float:
    weak = {k: round(v, 2) for k, v in s.items() if v < SENSITIVITY}
    assert not weak, f"{name}: defects that move the emulation by less than {SENSITIVITY} x tol_emu: {weak}"
    return min(s.values())


def bits(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.int32) if t.dtype == torch.float32 else t


# ---------------------------------------------------------------------------------------------------------------------------
# Denoiser: Downsample1D (down_conv)
# ---------------------------------------------------------------------------------------------------------------------------
class DownCase:
    def __init__(self, C: int, Tin: int, B: int = 3, T0: Optional[int] = None, lens: Optional[List[int]] = None, shift: int = 0):
        self.C, self.Tin, self.B, self.lens, self.shift = C, Tin, B, lens, shift
        self.T0 = T0
        self.name = f"C{C}_Tin{Tin}_B{B}" + (f"_rag_shift{shift}" if lens else "")

    @property
    def TL(self) -> int:
        return (self.Tin + 1) // 2

    def valid_in(self, b: int) -> int:
        return self.Tin if self.lens is None else ((self.lens[b] - 1) >> (self.shift - 1)) + 1

    def valid_out(self, b: int) -> int:
        return self.TL if self.lens is None else ((self.lens[b] - 1) >> self.shift) + 1


def level_len(T: int, level: int) -> int:
    for _ in range(level):
        T = (T - 1) // 2 + 1
    return T


def down_cases() -> List[DownCase]:
    out = [DownCase(C, Tin) for C in (128, 256, 384, 32, 64) for Tin in (1, 2, 3, 4, 5, 127, 128, 129, 1025, 2049)]
    out += [DownCase(100, Tin) for Tin in (3, 128, 129)]      # ld = 104 > C: NaN in the pad channels must not be read
    # ragged: level-0 lengths whose rows at the input level (shift - 1) are odd, even and 1, and the longest entry
    for C, shift, T0, lens in ((128, 1, 255, [255, 200, 37, 1]), (256, 2, 1000, [999, 74, 128, 1]), (384, 3, 2049, [2049, 397, 132, 1]),
                               (64, 2, 257, [257, 2, 8, 129])):
        out.append(DownCase(C, level_len(T0, shift - 1), B=len(lens), T0=T0, lens=lens, shift=shift))
    return out


DOWN_CASES = down_cases()


def build_down(c: DownCase, dev) -> Dict:
    g = torch.Generator().manual_seed(7 * c.C + c.Tin + 1000 * c.shift)
    x = torch.randn(c.B, c.Tin, c.C, generator=g)
    for b in range(c.B):                                      # producers store zeros past each entry's rows
        x[b, c.valid_in(b):] = 0.0
    W = torch.randn(c.C, c.C, 3, generator=g) / math.sqrt(3 * c.C)
    bias = 0.1 * torch.randn(c.C, generator=g)
    d = dict(x=x.to(dev), W=W.to(dev), bias=bias.to(dev))
    W64 = width64(c.C)
    Wf = torch.zeros(c.C, 3 * W64, device=dev)                # tap j at k-block j nkb(C): O[t-1], E[t], O[t]
    for j in range(3):
        Wf[:, j * W64:j * W64 + c.C] = d["W"][:, :, j]
    d["Wf"] = Wf
    ep = dict(n_valid=c.C, bias=d["bias"])
    if c.lens is not None:
        ep["row_valid"] = torch.arange(c.TL, device=dev)[None, :] < torch.tensor([c.valid_out(b) for b in range(c.B)], device=dev)[:, None]
    d["ep"] = ep
    return d


def down_operand(x: torch.Tensor, C: int, even: int = 0, odd: int = 1) -> torch.Tensor:
    """[B, TL, 3 width64(C)]: O[t-1] | E[t] | O[t] with E[t] = x[2t + even], O[t] = x[2t + odd], zero past Tin"""
    TL = (x.shape[1] + 1) // 2
    xw = F.pad(x[..., :C], (0, width64(C) - C))
    E, O = rows_at(xw, even, TL), rows_at(xw, odd, TL)
    return torch.cat([F.pad(O, (0, 0, 1, 0))[:, :TL], E, O], -1)


def down_truth(c: DownCase, d: Dict) -> torch.Tensor:
    y = F.conv1d(d["x"].to(F64).transpose(1, 2), d["W"].to(F64), d["bias"].to(F64), stride=2, padding=1).transpose(1, 2)
    if "row_valid" in d["ep"]:
        y = torch.where(d["ep"]["row_valid"][..., None], y, torch.zeros((), dtype=F64, device=y.device))
    return y


def launch_down(c: DownCase, d: Dict, force_prep=False, only=None, poison=False) -> Dict:
    dev = d["x"].device
    bsel = list(range(c.B)) if only is None else [only]
    B, ld = len(bsel), pad8(c.C)
    x = d["x"][bsel].contiguous()
    xs = torch.zeros(B, c.Tin, ld, device=dev)
    xs[..., :c.C] = x
    if poison:
        xs[..., c.C:] = float("nan")
    hi, lo = ko.split(xs)
    out = torch.full((B, c.TL, c.C), float("nan"), device=dev)
    ohi = torch.full((B, c.TL, ld), NAN16, dtype=torch.int16, device=dev)
    olo = ohi.clone()
    rl = None
    if c.lens is not None:
        rl = torch.tensor([c.lens[b] for b in bsel], dtype=torch.int32, device=dev)
    a = DownArgs(B, c.Tin, c.C, x.data_ptr(), hi.data_ptr(), lo.data_ptr(), ld, d["W"].data_ptr(), d["bias"].data_ptr(),
                 None if rl is None else rl.data_ptr(), c.shift, out.data_ptr(), ohi.data_ptr(), olo.data_ptr(), int(force_prep))
    desc = call(_lib.lib().ns2vc_check_down_conv, a)
    torch.cuda.synchronize()
    return dict(f32=out, hi=ohi, lo=olo, desc=desc, in_hi=hi, in_lo=lo)


def down_refs(c: DownCase, d: Dict, hi: torch.Tensor, lo: torch.Tensor):
    hi64, lo64 = hi.to(F64), lo.to(F64)
    operand = lambda s, **kw: down_operand(s, c.C, **kw)   # noqa: E731
    emu, bound = emulate(operand(hi64), operand(lo64), d["Wf"], d["ep"])
    defects = {"even_at_2t+1": dict(even=1)}
    if c.Tin >= 2:                                            # (Tin = 1 has no odd row to shift)
        defects["odd_shifted"] = dict(odd=2)
    s = sensitivities(operand, hi64, lo64, d["Wf"], d["ep"], emu, bound, defects)
    return emu, bound, s


@gpu
@pytest.mark.parametrize("c", DOWN_CASES, ids=lambda c: c.name)
def test_down_conv(c: DownCase):
    dev = torch.device("cuda")
    d = build_down(c, dev)
    got = launch_down(c, d)
    rag = int(c.lens is not None)
    gemm = f"gemm_tc<64,LNF=0,XF=0,ENC=0,RAG={rag},VOC=0>"
    assert got["desc"] == ("2xprep_split<RAG=0>+" if c.Tin == 1 else "") + gemm, got["desc"]
    emu, bound, s = down_refs(c, d, got["in_hi"], got["in_lo"])
    sens = assert_sensitive(c.name, s)
    g64 = got["f32"].to(F64)
    r_emu = ko.ratio(g64 - emu, bound)
    assert r_emu <= 1.0, f"{c.name}: |gpu - emu| reaches {r_emu:.2f} x tol_emu"
    r_truth = ko.rule_ratio(got["f32"], down_truth(c, d))
    assert r_truth <= 1.0, f"{c.name}: vs the fp64 conv {r_truth:.3f} of the rule"
    # the split output is the split of the fp32 output; rows past each entry's own rows are exact zeros
    hb, lb = ko.split(got["f32"])
    assert torch.equal(got["hi"][..., :c.C], hb.view(torch.int16)) and torch.equal(got["lo"][..., :c.C], lb.view(torch.int16)), \
        f"{c.name}: split output is not the split of the fp32 output"
    for b in range(c.B):
        n = c.valid_out(b)
        assert (got["f32"][b, n:] == 0).all() and (got["hi"][b, n:, :c.C] == 0).all() and (got["lo"][b, n:, :c.C] == 0).all(), \
            f"{c.name}: entry {b} is not 0 past its {n} rows"
    # the dense copy: prep-path decimation, bit for bit
    prep = launch_down(c, d, force_prep=True)
    assert prep["desc"] == "2xprep_split<RAG=0>+" + gemm, prep["desc"]
    for k in ("f32", "hi", "lo"):
        assert torch.equal(bits(prep[k]), bits(got[k])), f"{c.name}: the row-pair views differ from the prep path ({k})"
    # a second launch (with NaN in the pad channels inside ld, where there are any) is bit-identical
    again = launch_down(c, d, poison=pad8(c.C) > c.C)
    for k in ("f32", "hi", "lo"):
        assert torch.equal(bits(again[k]), bits(got[k])), f"{c.name}: a second launch differs ({k})"
    # each entry equals that entry launched alone (B = 1), which catches a batch pitch that is not Tin rows
    for b in range(c.B):
        alone = launch_down(c, d, only=b)
        for k in ("f32", "hi", "lo"):
            assert torch.equal(bits(alone[k][0]), bits(got[k][b])), f"{c.name}: entry {b} differs from its launch alone ({k})"
    fam = FAM + ("down_conv ragged" if rag else f"down_conv C={c.C}")
    kf.record(fam, emu_ratio=r_emu, truth_ratio=r_truth, sens_margin=sens)
    print(f"{c.name}: emu {r_emu:.3f}, truth {r_truth:.3f}, weakest defect {sens:.0f} x")


# ---------------------------------------------------------------------------------------------------------------------------
# Content encoder: convs 1-6 (cv_conv_gemm)
# ---------------------------------------------------------------------------------------------------------------------------
def conv_k(l: int) -> int:
    return 3 if l <= 4 else 2


def conv_frames(n: int, l: int) -> int:
    k, s = (10, 5) if l == 0 else (conv_k(l), 2)
    return 0 if n < k else (n - k) // s + 1


def rows_of(T: int, l: int) -> int:
    """the engine's rows per entry of level l: padded to even so that the next conv's pairs stay inside the entry (the last
    level has no next conv)"""
    return T + (T & 1) if l < 6 else T


def cv_operand(x: torch.Tensor, rows_out: int, k: int, first: int = 0, second: int = 1, third: int = 2) -> torch.Tensor:
    """[B, rows_out, k C0]: x[2t + first] | x[2t + second] (| x[2t + third]), zero past the input's rows"""
    parts = [rows_at(x, first, rows_out), rows_at(x, second, rows_out)]
    if k == 3:
        parts.append(rows_at(x, third, rows_out))
    return torch.cat(parts, -1)


class CvLevel:
    """one launch of conv l over B entries of frames_in[b] input frames (the rows of the longest, padded)"""

    def __init__(self, C0: int, l: int, frames_in: List[int]):
        self.C0, self.l, self.frames_in = C0, l, frames_in
        self.k = conv_k(l)
        self.rows_in = rows_of(max(frames_in), l - 1)
        self.rows_out = rows_of(conv_frames(max(frames_in), l), l)
        self.frames_out = [conv_frames(n, l) for n in frames_in]

    @property
    def B(self) -> int:
        return len(self.frames_in)

    def keep(self, dev) -> torch.Tensor:
        return (torch.arange(self.rows_out, device=dev)[None, :] < torch.tensor(self.frames_out, device=dev)[:, None]).float()


def cv_weights(C0: int, l: int, dev) -> Dict:
    g = torch.Generator().manual_seed(C0 + l)
    k = conv_k(l)
    W = (torch.randn(C0, C0, k, generator=g) / math.sqrt(k * C0) * 2).to(dev)
    return dict(W=W, Wf=W.permute(0, 2, 1).reshape(C0, k * C0).contiguous())


def cv_input(lv: CvLevel, seed: int, dev) -> torch.Tensor:
    """a split level [B, rows_in, C0] (int16 hi | lo): GELU-like values, exact zeros past each entry's frames"""
    g = torch.Generator().manual_seed(seed)
    x = ko.gelu_erf(torch.randn(lv.B, lv.rows_in, lv.C0, generator=g).double()).float()
    for b, n in enumerate(lv.frames_in):
        x[b, n:] = 0.0
    hi, lo = ko.split(x.to(dev))
    return torch.stack([hi.view(torch.int16), lo.view(torch.int16)])


def launch_cv(lv: CvLevel, wd: Dict, xin: torch.Tensor, split_out: bool, keep=None, out=None):
    """one conv-l launch on the split xin [2, B, rows_in, C0]; returns the fp32 output or the split [2, B, rows_out, C0]"""
    dev = xin.device
    keep = lv.keep(dev) if keep is None else keep
    if out is None:
        out = (torch.full((2, lv.B, lv.rows_out, lv.C0), NAN16, dtype=torch.int16, device=dev) if split_out
               else torch.full((lv.B, lv.rows_out, lv.C0), float("nan"), device=dev))
    a = CvConvArgs(lv.B, lv.rows_in, lv.rows_out, lv.C0, lv.l, xin[0].data_ptr(), xin[1].data_ptr(), wd["W"].data_ptr(), keep.data_ptr())
    if split_out:
        a.out_hi, a.out_lo = out[0].data_ptr(), out[1].data_ptr()
    else:
        a.out = out.data_ptr()
    desc = call(_lib.lib().ns2vc_check_cv_conv, a)
    torch.cuda.synchronize()
    assert desc == "gemm_tc<64,LNF=0,XF=0,ENC=0,RAG=0,VOC=1>", desc
    return out


def split_value(s: torch.Tensor) -> torch.Tensor:
    return s[0].view(torch.bfloat16).to(F64) + s[1].view(torch.bfloat16).to(F64)


def cv_refs(lv: CvLevel, wd: Dict, xin: torch.Tensor, sens: bool):
    """(emulation, tol_emu, truth, sensitivities) of one launch on the split xin"""
    dev = xin.device
    hi64, lo64 = xin[0].view(torch.bfloat16).to(F64), xin[1].view(torch.bfloat16).to(F64)
    ep = dict(n_valid=lv.C0, gelu=True, rowmask=lv.keep(dev))
    operand = lambda s, **kw: cv_operand(s, lv.rows_out, lv.k, **kw)   # noqa: E731
    emu, bound = emulate(operand(hi64), operand(lo64), wd["Wf"], ep)
    x = F.pad(hi64 + lo64, (0, 0, 0, max(0, 2 * lv.rows_out + 2 - lv.rows_in)))
    y = F.conv1d(x.transpose(1, 2), wd["W"].to(F64), stride=2).transpose(1, 2)[:, :lv.rows_out]
    y = F.pad(y, (0, 0, 0, lv.rows_out - y.shape[1]))
    truth = ko.gelu_erf(y) * ep["rowmask"].to(F64)[..., None]
    s = None
    if sens:
        defects = {"odd_shifted": dict(second=2), "even_at_2t+1": dict(first=1)}
        if lv.k == 3:
            defects["tap2_at_2t+1"] = dict(third=1)
        s = sensitivities(operand, hi64, lo64, wd["Wf"], ep, emu, bound, defects)
    return emu, bound, truth, s


def check_cv_level(name: str, lv: CvLevel, wd: Dict, xin: torch.Tensor, f32: torch.Tensor, split: Optional[torch.Tensor], sens: bool):
    """the references, the exact zeros past each entry's frames and the split's consistency with the fp32 output"""
    emu, bound, truth, s = cv_refs(lv, wd, xin, sens)
    r_emu = ko.ratio(f32.to(F64) - emu, bound)
    assert r_emu <= 1.0, f"{name}: |gpu - emu| reaches {r_emu:.2f} x tol_emu"
    r_truth = ko.rule_ratio(f32, truth)
    assert r_truth <= 1.0, f"{name}: vs the fp64 conv {r_truth:.3f} of the rule"
    for b, n in enumerate(lv.frames_out):
        assert (f32[b, n:] == 0).all(), f"{name}: entry {b} is not 0 past its {n} frames"
    if split is not None:
        hb, lb = ko.split(f32)
        assert torch.equal(split[0], hb.view(torch.int16)) and torch.equal(split[1], lb.view(torch.int16)), \
            f"{name}: split output is not the split of the fp32 output"
    return r_emu, r_truth, (assert_sensitive(name, s) if sens else math.inf)


def launch_cv_dense(lv: CvLevel, wd: Dict, xin: torch.Tensor) -> torch.Tensor:
    """the same GEMM (ns2vc_check_gemm, weights packed as one [C0, k C0] tap) over an explicit dense im2col copy of the operand"""
    dev = xin.device
    K = lv.k * lv.C0
    Ah = cv_operand(xin[0].view(torch.bfloat16), lv.rows_out, lv.k).contiguous()
    Al = cv_operand(xin[1].view(torch.bfloat16), lv.rows_out, lv.k).contiguous()
    nkb = K // 64
    wh = torch.zeros(nkb * lv.C0 * 64, dtype=torch.bfloat16, device=dev)
    wl = torch.zeros_like(wh)
    _lib.check(_lib.lib().ns2vc_check_pack_b(wd["Wf"].data_ptr(), lv.C0, K, 1, 0, 0, K, 0, 0, 0, None, wh.data_ptr(), wl.data_ptr(),
                                             lv.C0, nkb, stream()))
    keep = lv.keep(dev)
    out = torch.full((lv.B, lv.rows_out, lv.C0), float("nan"), device=dev)
    a = kf.GemmArgs()
    a.B, a.T_out, a.nsrc, a.nseg = lv.B, lv.rows_out, 1, 1
    a.src[0] = kf.Split(Ah.data_ptr(), Al.data_ptr(), lv.rows_out, K, K, 0)
    a.seg[0] = (C.c_int * 4)(0, 0, K, 0)
    a.w_hi, a.w_lo, a.N, a.n_valid, a.nkb_w = wh.data_ptr(), wl.data_ptr(), lv.C0, lv.C0, nkb
    a.flags = kf.EPI_GELU | kf.EPI_ROWMASK | kf.EPI_OUT_F32
    a.out, a.out_ld, a.rowmask, a.f16_col0, a.ksplit = out.data_ptr(), lv.C0, keep.data_ptr(), -1, 1
    desc = call(_lib.lib().ns2vc_check_gemm, a)
    torch.cuda.synchronize()
    assert desc == "gemm_tc<64,LNF=0,XF=0,ENC=0,RAG=0,VOC=1>", desc
    return out


def cv_counts(l: int) -> List[int]:
    """input frame counts: the smallest that give 1 and 2 output frames, and every residue mod 4"""
    k = conv_k(l)
    return [k, k + 2, 100, 101, 102, 103]


CV_CASES = [(C0, l) for C0 in (512, 128) for l in range(1, 7)]


@gpu
@pytest.mark.parametrize("C0,l", CV_CASES, ids=[f"C{C0}_l{l}" for C0, l in CV_CASES])
def test_cv_conv(C0: int, l: int):
    dev = torch.device("cuda")
    wd = cv_weights(C0, l, dev)
    worst = dict(emu=0.0, truth=0.0, sens=math.inf)

    def run(name, lv, seed, sens=True):
        xin = cv_input(lv, seed, dev)
        f32 = launch_cv(lv, wd, xin, split_out=False)
        split = launch_cv(lv, wd, xin, split_out=True)
        r = check_cv_level(name, lv, wd, xin, f32, split, sens)
        for k, v in zip(("emu", "truth"), r[:2]):
            worst[k] = max(worst[k], v)
        worst["sens"] = min(worst["sens"], r[2])
        return xin, f32, split

    for n in cv_counts(l):                                  # B = 1 at each count
        run(f"C{C0}_l{l}_T{n}", CvLevel(C0, l, [n]), 10 * l + n)
    # B = 3 whose counts differ in parity: the dense copy, NaN where nothing valid reads, a repeat, each entry alone
    lv = CvLevel(C0, l, [103, 100, 37])
    name = f"C{C0}_l{l}_B3"
    xin, f32, split = run(name, lv, 5 * l)
    assert torch.equal(bits(launch_cv_dense(lv, wd, xin)), bits(f32)), f"{name}: the row-pair view differs from the dense copy"
    assert torch.equal(bits(launch_cv(lv, wd, xin, split_out=False)), bits(f32)), f"{name}: a second launch differs"
    poisoned = xin.clone()
    for b, n in enumerate(lv.frames_in):                    # the pad row and the rows past each entry's frames
        poisoned[:, b, n:] = NAN16
    pf32, psplit = launch_cv(lv, wd, poisoned, split_out=False), launch_cv(lv, wd, poisoned, split_out=True)
    for b, n in enumerate(lv.frames_out):
        assert torch.equal(bits(pf32[b, :n]), bits(f32[b, :n])) and torch.equal(psplit[:, b, :n], split[:, b, :n]), \
            f"{name}: NaN past entry {b}'s input frames changes a valid output"
    for b, n in enumerate(lv.frames_in):
        alone = CvLevel(C0, l, [n])
        xa = xin[:, b:b + 1, :alone.rows_in].contiguous()
        fa = launch_cv(alone, wd, xa, split_out=False)
        m = min(alone.rows_out, lv.rows_out)
        assert torch.equal(bits(fa[0, :m]), bits(f32[b, :m])), f"{name}: entry {b} differs from its launch alone"
    kf.record(FAM + f"cv_conv C0={C0} k={conv_k(l)}", emu_ratio=worst["emu"], truth_ratio=worst["truth"], sens_margin=worst["sens"])
    print(f"C{C0}_l{l}: emu {worst['emu']:.3f}, truth {worst['truth']:.3f}, weakest defect {worst['sens']:.0f} x")


def chain_frames(samples: List[int]) -> List[List[int]]:
    """frames per level (0 .. 6) of each entry"""
    out, cur = [], [conv_frames(n, 0) for n in samples]
    out.append(cur)
    for l in range(1, 7):
        cur = [conv_frames(n, l) for n in cur]
        out.append(cur)
    return out


CHAIN_CASES = {"batch_full": batch_full()[1], "N400": [400], "N401": [401]}


@gpu
@pytest.mark.parametrize("which", list(CHAIN_CASES))
def test_cv_conv_chain(which: str):
    """levels 1 -> 6 on the engine's two shared splits (levels 0, 2, 4 in one, 1, 3, 5 in the other), each level reading the
    previous level's GPU output and checked against fp64 on that input"""
    dev = torch.device("cuda")
    C0 = 512
    samples = CHAIN_CASES[which]
    B = len(samples)
    fr = chain_frames(samples)
    rows = [rows_of(max(fr[l]), l) for l in range(7)]
    bufs = [torch.zeros(2, B * rows[0] * C0, dtype=torch.int16, device=dev), torch.zeros(2, B * rows[1] * C0, dtype=torch.int16, device=dev)]
    # level 0 (cv_conv0's output): GELU-like values, zero past each entry's frames
    g = torch.Generator().manual_seed(B)
    x0 = ko.gelu_erf(torch.randn(B, rows[0], C0, generator=g).double()).float()
    for b, n in enumerate(fr[0]):
        x0[b, n:] = 0.0
    h0, l0 = ko.split(x0.to(dev))
    bufs[0][0].copy_(h0.view(torch.int16).reshape(-1))
    bufs[0][1].copy_(l0.view(torch.int16).reshape(-1))
    worst = dict(emu=0.0, truth=0.0)
    for l in range(1, 7):
        lv = CvLevel(C0, l, fr[l - 1])
        assert (lv.rows_in, lv.rows_out, lv.frames_out) == (rows[l - 1], rows[l], fr[l])
        src = bufs[(l - 1) % 2][:, :B * rows[l - 1] * C0].view(2, B, rows[l - 1], C0)
        wd = cv_weights(C0, l, dev)
        f32 = launch_cv(lv, wd, src, split_out=False)
        split = None
        if l < 6:
            split = bufs[l % 2][:, :B * rows[l] * C0].view(2, B, rows[l], C0)
            launch_cv(lv, wd, src, split_out=True, out=split)
        r = check_cv_level(f"{which} level {l}", lv, wd, src, f32, split, sens=False)
        worst["emu"], worst["truth"] = max(worst["emu"], r[0]), max(worst["truth"], r[1])
    kf.record(FAM + "cv_conv chain", emu_ratio=worst["emu"], truth_ratio=worst["truth"])
    print(f"{which} (frames {fr[6]}): emu {worst['emu']:.3f}, truth {worst['truth']:.3f}")


# ---------------------------------------------------------------------------------------------------------------------------
# Argument errors
# ---------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("field,value,match", [
    ("x", None, "check_down_conv: null argument"), ("Tin", 0, "check_down_conv: bad sizes"), ("ld", 36, "input ld=36"),
    ("out", None, "check_down_conv: no output"), ("len_shift", 0, "ragged output level 0")])
def test_down_conv_argument_errors(field, value, match):
    dev = torch.device("cuda")
    c = DownCase(32, 4, B=1)
    d = build_down(c, dev)
    hi, lo = ko.split(d["x"])
    out = torch.zeros(1, 2, 32, device=dev)
    rl = torch.tensor([4], dtype=torch.int32, device=dev)
    a = DownArgs(1, 4, 32, d["x"].data_ptr(), hi.data_ptr(), lo.data_ptr(), 32, d["W"].data_ptr(), d["bias"].data_ptr(), rl.data_ptr(), 1,
                 out.data_ptr(), None, None, 0)
    setattr(a, field, value)
    with pytest.raises(_lib.Ns2vcError, match=match):
        call(_lib.lib().ns2vc_check_down_conv, a)


@gpu
@pytest.mark.parametrize("field,value,match", [
    ("w", None, "check_cv_conv: null argument"), ("l", 7, "conv index 7"), ("l", 0, "conv index 0"), ("C0", 192, "C0=192"),
    ("rows_out", 0, "check_cv_conv: bad sizes"), ("rows_in", 9, "rows_in=9 is odd"), ("out_hi", "both", "exactly one output")])
def test_cv_conv_argument_errors(field, value, match):
    dev = torch.device("cuda")
    lv = CvLevel(128, 1, [9])
    wd = cv_weights(128, 1, dev)
    xin = cv_input(lv, 0, dev)
    keep = lv.keep(dev)
    out = torch.zeros(2, 1, lv.rows_out, 128, dtype=torch.int16, device=dev)
    a = CvConvArgs(1, lv.rows_in, lv.rows_out, 128, 1, xin[0].data_ptr(), xin[1].data_ptr(), wd["W"].data_ptr(), keep.data_ptr(),
                   out.data_ptr(), None, None)
    if value == "both":
        a.out_hi, a.out_lo = out[0].data_ptr(), out[1].data_ptr()
    else:
        setattr(a, field, value)
    with pytest.raises(_lib.Ns2vcError, match=match):
        call(_lib.lib().ns2vc_check_cv_conv, a)
