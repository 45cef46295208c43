"""The GroupNorm prep, the LayerNorm kernels, the small linear of the timestep path, the AttentionPooling pieces and the
[B, C, T] -> split conversion launch by launch, through the test-only C entry points of csrc/kernel_check.cu (ns2vc_check_prep,
_ln, _voc_norm, _small_linear, _pool, _nct_split), which run the engines' own descriptor code (set_group_norm, linear_op) and
launchers.  Every case asserts the instantiation it launched.

Truth: the operation in fp64 on the kernel's actual fp32 input (oracle/kernel_oracle.py).  Rule: the parity rule of the
model-level files, 1e-3 |ref| + 1e-4 rms(ref) floored at 2 e32 (e32 = max |fp32 - fp64| of the same operation on the same input),
plus the error terms the design carries, each named where it is added:
  * the GroupNorm's uncentred fp32 affine and its bf16 hi/lo output (kernel_oracle.affine_terms);
  * the one-pass variance q / n - mean^2 from given fp64 sums adds nothing measurable.  What the producers' sums can add: each
    column is summed in fp32 over partials of p = 32 rows, then in fp64, and a partial of p terms is within (p - 1) 2^-24 of
    the sum of their magnitudes, so with S1 = sum |x|, S2 = sum x^2 over a group of n elements
        |d mean| <= (p - 1) 2^-24 S1 / n,   |d var| <= (p - 1) 2^-24 (S2 / n + 2 |mean| S1 / n) (+ d mean^2),
    i.e. ~ 3 (p - 1) 2^-24 (1 + r^2) of var for r = |group mean| / group std: the r^2 term, not the fp64 finish, limits how
    far a group may sit from zero.  The constant-group cases pass sums of squares understated within that bound, so the
    variance comes out below -eps and only the clamp at 0 keeps the group finite.
No bound is vacuous: dropping the FiLM 1+, reading the second source's statistics from the first, or counting one row fewer in
a ragged group moves the fp64 result by >= 16 x the bound somewhere in every case that has that feature.

Exact properties: rows past a length and channels past C are exactly 0; NaN past the lengths or in channels >= C inside ld
changes no bit; a ragged entry equals the same entry launched alone at B = 1; the prep's raw split is the split of its
untransformed input; tokens copied by the class-token kernel are the input rows.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import math
from typing import Dict, List, Optional

import pytest
import torch

from conftest import REPO  # noqa: F401  (puts the repository on sys.path)
from ns2vc_b200 import _lib
from oracle import kernel_oracle as ko
from oracle import unet_oracle

F64 = torch.float64


def gpu(f):
    """a GPU case: marked `gpu`, skipped where there is no CUDA device"""
    return pytest.mark.gpu(pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")(f))


SENSITIVITY = 16.0
WORST: Dict[str, float] = {}


class Split(C.Structure):
    _fields_ = [("hi", C.c_void_p), ("lo", C.c_void_p), ("T", C.c_int), ("C", C.c_int), ("ld", C.c_int), ("bpitch", C.c_longlong)]


class PrepArgs(C.Structure):
    _fields_ = [("src1", C.c_void_p), ("ld1", C.c_int), ("C1", C.c_int), ("src2", C.c_void_p), ("ld2", C.c_int), ("C2", C.c_int),
                ("B", C.c_int), ("T_src", C.c_int), ("T_dst", C.c_int), ("row_mul", C.c_int), ("row_add", C.c_int),
                ("rowmap", C.c_void_p), ("mode", C.c_int), ("scale", C.c_void_p), ("shift", C.c_void_p), ("stats1", C.c_void_p),
                ("stats2", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p), ("G", C.c_int), ("eps", C.c_float),
                ("film", C.c_void_p), ("film_ld", C.c_int), ("out", Split), ("raw", Split), ("row_len", C.c_void_p),
                ("len_shift", C.c_int)]


class LnArgs(C.Structure):
    _fields_ = [("kind", C.c_int), ("x", C.c_void_p), ("ld", C.c_int), ("M", C.c_int), ("C", C.c_int), ("eps", C.c_float),
                ("gamma", C.c_void_p), ("beta", C.c_void_p), ("keep", C.c_void_p), ("y", C.c_void_p), ("y_ld", C.c_int),
                ("split", Split)]


class VocNormArgs(C.Structure):
    _fields_ = [("x", C.c_void_p), ("B", C.c_int), ("T", C.c_int), ("C", C.c_int), ("dw", C.c_void_p), ("gamma", C.c_void_p),
                ("beta", C.c_void_p), ("eps", C.c_float), ("len", C.c_void_p), ("out", C.c_void_p), ("split", Split)]


class LinArgs(C.Structure):
    _fields_ = [("x", C.c_void_p), ("x_ld", C.c_int), ("M", C.c_int), ("K", C.c_int), ("W", C.c_void_p), ("bias", C.c_void_p),
                ("N", C.c_int), ("add", C.c_void_p), ("add_ld", C.c_int), ("add_rows", C.c_int), ("out", C.c_void_p),
                ("out_ld", C.c_int), ("in_mode", C.c_int), ("flip_sin_to_cos", C.c_int), ("freq_shift", C.c_float),
                ("out_silu", C.c_int)]


class PoolArgs(C.Structure):
    _fields_ = [("x", C.c_void_p), ("pos", C.c_void_p), ("B", C.c_int), ("S", C.c_int), ("C", C.c_int), ("tokens", C.c_void_p),
                ("q", C.c_void_p), ("kv", C.c_void_p), ("heads", C.c_int), ("wide", C.c_int), ("out", C.c_void_p),
                ("lens", C.c_void_p)]


class NctArgs(C.Structure):
    _fields_ = [("x", C.c_void_p), ("bstride", C.c_longlong), ("B", C.c_int), ("C", C.c_int), ("T", C.c_int), ("out", Split),
                ("row_len", C.c_void_p)]


def stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def call(fn, args) -> str:
    desc = C.create_string_buffer(96)
    _lib.check(fn(C.cast(C.byref(args), C.c_void_p), desc, 96, stream()))
    torch.cuda.synchronize()
    return desc.value.decode()


def record(family: str, r: float) -> None:
    WORST[family] = max(WORST.get(family, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    for fam, r in sorted(WORST.items()):
        print(f"\n[norm kernel checks] {fam}: worst ratio {r:.3g}")


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def split_buf(T: int, C_: int, ld: int, rows: int, dev) -> Dict:
    hi = torch.full((rows, ld), 0x7fc0, dtype=torch.int16, device=dev)       # bf16 NaN: every element must be written
    lo = hi.clone()
    return dict(hi=hi, lo=lo, s=Split(hi.data_ptr(), lo.data_ptr(), T, C_, ld, 0))


def joined(buf: Dict) -> torch.Tensor:
    return buf["hi"].view(torch.bfloat16).to(F64) + buf["lo"].view(torch.bfloat16).to(F64)


def check(name: str, got: torch.Tensor, ref: torch.Tensor, e32: float, extra: Optional[torch.Tensor] = None) -> float:
    tol = ko.parity_tol(ref, e32)
    if extra is not None:
        tol = tol + extra
    r = ko.ratio(got.to(F64) - ref, tol)
    assert r <= 1.0, f"{name}: {r:.3f} of the bound (max |err| {float((got.to(F64) - ref).abs().max()):.3e})"
    return r


def sensitive(name: str, defect: torch.Tensor, ref: torch.Tensor, e32: float, extra: Optional[torch.Tensor] = None) -> None:
    tol = ko.parity_tol(ref, e32) + (extra if extra is not None else 0)
    s = float(((defect - ref).abs() / tol).max())
    assert s >= SENSITIVITY, f"{name}: the defect moves the result by only {s:.1f} x the bound"


def rows_of(L: List[int], shift: int) -> List[int]:
    return [((l - 1) >> shift) + 1 for l in L]


# ---------------------------------------------------------------------------------------------------------------------------
# GroupNorm prep (prep_split_kernel)
# ---------------------------------------------------------------------------------------------------------------------------
class GN:
    def __init__(self, name, B, T, C1, C2=0, G=8, film=None, r=0.0, lens=None, shift=0, silu=True, const_group=False, ld_pad=0):
        self.name, self.B, self.T, self.C1, self.C2, self.G = name, B, T, C1, C2, G
        self.film, self.r, self.lens, self.shift, self.silu, self.const_group, self.ld_pad = film, r, lens, shift, silu, const_group, ld_pad


GN_CASES = [
    GN("G1_C2_T1", 1, 1, 2, G=1),
    GN("G8_C16_T2_film_m1", 2, 2, 16, film="m1"),
    GN("G32_C64_T63_r4", 2, 63, 64, G=32, r=4.0),
    GN("G32_C2048cap_C1024_T64", 1, 64, 1024, G=32),
    GN("G4_C100_T65_scalar_ld", 2, 65, 100, G=4, ld_pad=3),
    GN("G8_C512_T127_r30_bigfilm", 2, 127, 512, film="big", r=30.0),
    GN("G8_C128_T128_r100", 1, 128, 128, r=100.0),
    GN("G8_C72_T129_const", 2, 129, 72, const_group=True),
    GN("seam_C40_24_G8_T65", 2, 65, 40, 24, G=8, film="plain"),             # C/G = 8: group 5 straddles the seam at 40
    GN("seam_C96_160_G8_T63_r4", 3, 63, 96, 160, G=8, r=4.0, film="m1"),      # C/G = 32: group 2 straddles the seam at 96
    GN("rag_G8_C64_T129_s0", 3, 129, 64, lens=[129, 64, 1], shift=0, film="plain"),
    GN("rag_G32_C128_T33_s2", 3, 33, 128, G=32, lens=[129, 127, 2], shift=2, r=30.0),
    GN("rag_seam_C64_64_T65_s1", 2, 65, 64, 64, lens=[129, 3], shift=1, film="big"),
    GN("rag_G1_C8_T64_s3_r100", 2, 64, 8, G=1, lens=[505, 9], shift=3, r=100.0),
]


def build_gn(c: GN, dev):
    g = torch.Generator().manual_seed(sum(map(ord, c.name)))
    rn = lambda *s: torch.randn(*s, generator=g)
    Cg = c.C1 + c.C2
    rows = rows_of(c.lens, c.shift) if c.lens else [c.T] * c.B
    x = rn(c.B, c.T, Cg)
    if c.r:                                                   # group means r x the group std
        x = x + c.r * torch.sign(rn(c.B, 1, c.G)).repeat_interleave(Cg // c.G, -1)
    if c.const_group:                                        # group 0 of every entry constant: variance 0 (the clamp)
        x[:, :, :Cg // c.G] = 2.0
    for b in range(c.B):
        x[b, rows[b]:] = 0.0                                 # producers store zeros past the rows
    gamma, beta = 1.0 + 0.2 * rn(Cg), 0.1 * rn(Cg)
    film = None
    if c.film == "m1":
        film = torch.cat([-1.0 + 0.01 * rn(c.B, Cg), 0.1 * rn(c.B, Cg)], -1)
    elif c.film == "big":
        film = torch.cat([30.0 * rn(c.B, Cg), rn(c.B, Cg)], -1)
    elif c.film == "plain":
        film = torch.cat([0.3 * rn(c.B, Cg), 0.3 * rn(c.B, Cg)], -1)
    x64 = x.to(F64)
    st = torch.stack([x64.sum(1), (x64 * x64).sum(1)])        # [2, B, C]: the fp64 sums over the valid rows
    if c.const_group:
        # sums of squares 2e-5 per element low, as fp32 partial sums may leave them (module docstring: up to 31 * 2^-24 *
        # (S2 / n + 2 |mean| S1 / n) = 2.2e-5 at mean 2): the one-pass variance is -2e-5 < -eps
        st[1, :, :Cg // c.G] -= 2e-5 * torch.tensor(rows, dtype=F64)[:, None]
        bound = 31 * 2.0 ** -24 * (4.0 + 2 * 2.0 * 2.0)
        assert 2e-5 <= bound
    return dict(x=x, gamma=gamma, beta=beta, film=film, rows=rows, st1=st[:, :, :c.C1].contiguous(), st2=st[:, :, c.C1:].contiguous())


def gn_refs(c: GN, d, dt=F64, **defect):
    x = d["x"].to(dt)
    film = d["film"].to(dt) if d["film"] is not None else None
    return ko.group_norm_rows(x, c.G, d["gamma"].to(dt), d["beta"].to(dt), 1e-5, d["rows"], film, c.silu, **defect)


def gn_extra(c: GN, d):
    film = d["film"].to(F64) if d["film"] is not None else None
    e = ko.affine_terms(d["x"].to(F64), c.G, d["gamma"].to(F64), d["beta"].to(F64), d["rows"], film, 1e-5)
    if c.silu:
        e = e * 1.1                                          # SiLU's slope is below 1.1
    return e


def launch_prep(c: GN, d, dev, poison=False, only=None, raw=False):
    bsel = slice(None) if only is None else slice(only, only + 1)
    B = c.B if only is None else 1
    x = d["x"][bsel].to(dev)
    ld1, ld2 = c.C1 + c.ld_pad, c.C2 + c.ld_pad
    s1 = torch.zeros(B, c.T, ld1, device=dev)
    s1[..., :c.C1] = x[..., :c.C1]
    s2 = torch.zeros(B, c.T, max(ld2, 1), device=dev)
    s2[..., :c.C2] = x[..., c.C1:]
    if poison:
        s1[..., c.C1:] = float("nan")
        s2[..., c.C2:] = float("nan")
        if c.lens:
            for i, b in enumerate(range(c.B)[bsel]):
                s1[i, d["rows"][b]:] = float("nan")
                s2[i, d["rows"][b]:] = float("nan")
    Cg = c.C1 + c.C2
    ld = (Cg + 7) // 8 * 8
    out = split_buf(c.T, Cg, ld, B * c.T, dev)
    rawb = split_buf(c.T, Cg, ld, B * c.T, dev) if raw else None
    st1, st2 = d["st1"][:, bsel].contiguous().to(dev), d["st2"][:, bsel].contiguous().to(dev)
    gamma, beta = d["gamma"].to(dev), d["beta"].to(dev)
    film = d["film"][bsel].contiguous().to(dev) if d["film"] is not None else None
    a = PrepArgs()
    a.src1, a.ld1, a.C1 = s1.data_ptr(), ld1, c.C1
    if c.C2:
        a.src2, a.ld2, a.C2, a.stats2 = s2.data_ptr(), ld2, c.C2, st2.data_ptr()
    a.B, a.T_src, a.T_dst, a.row_mul = B, c.T, c.T, 1
    a.mode = 2 if c.silu else 1
    a.stats1, a.gamma, a.beta, a.G, a.eps = st1.data_ptr(), gamma.data_ptr(), beta.data_ptr(), c.G, 1e-5
    if film is not None:
        a.film, a.film_ld = film.data_ptr(), 2 * Cg
    a.out = out["s"]
    if raw:
        a.raw = rawb["s"]
    if c.lens:
        rl = torch.tensor(c.lens, dtype=torch.int32, device=dev)[bsel].contiguous()
        a.row_len, a.len_shift = rl.data_ptr(), c.shift
    desc = call(_lib.lib().ns2vc_check_prep, a)
    assert desc == f"prep_split<RAG={1 if c.lens else 0}>", desc
    return out, rawb


@pytest.mark.parametrize("c", GN_CASES, ids=lambda c: c.name)
def test_group_norm_reference_is_sensitive(c):
    """CPU: the fp64 reference equals F.group_norm per entry, and its bound notices each defect the case can show"""
    d = build_gn(c, "cpu")
    ref = gn_refs(c, d)
    e32 = float((gn_refs(c, d, torch.float32).to(F64) - ref).abs().max())
    extra = gn_extra(c, d)
    for b in range(c.B):                                     # the reference against torch's GroupNorm of the unpadded entry
        n = d["rows"][b]
        want = torch.nn.functional.group_norm(d["x"][b, :n].T[None].to(F64), c.G, d["gamma"].to(F64), d["beta"].to(F64), 1e-5)[0].T
        if d["film"] is not None:
            f = d["film"][b].to(F64)
            want = want * (1 + f[:c.C1 + c.C2]) + f[c.C1 + c.C2:]
        want = want * torch.sigmoid(want) if c.silu else want
        assert torch.allclose(ref[b, :n], want, rtol=1e-12, atol=1e-12)
    if d["film"] is not None:
        sensitive(c.name + " FiLM without 1+", gn_refs(c, d, one_plus=False), ref, e32, extra)
    if c.C2:                                                 # the second source's statistics read from the first source's
        bad = seam_defect(c, d)
        sensitive(c.name + " sum2 read as sum1", bad, ref, e32, extra)
    if c.lens and any(r > 1 for r in d["rows"]):
        sensitive(c.name + " one row fewer in the count", gn_refs(c, d, count=[max(r - 1, 1) for r in d["rows"]]), ref, e32, extra)


def seam_defect(c: GN, d) -> torch.Tensor:
    """the GroupNorm whose channels past the seam take their statistics (sums) from the first source's channels instead"""
    st = torch.cat([d["st1"], d["st1"][:, :, :c.C2] if c.C2 <= c.C1 else torch.cat([d["st1"], d["st2"][:, :, c.C1:]], -1)], -1)
    Cg, cpg = c.C1 + c.C2, (c.C1 + c.C2) // c.G
    x = d["x"].to(F64)
    out = torch.zeros_like(x)
    film = d["film"].to(F64) if d["film"] is not None else None
    for b in range(c.B):
        n = d["rows"][b]
        s, q = st[0, b].reshape(c.G, cpg).sum(-1), st[1, b].reshape(c.G, cpg).sum(-1)
        mean = s / (n * cpg)
        var = (q / (n * cpg) - mean * mean).clamp_min(0)
        m, rs = mean.repeat_interleave(cpg), (1.0 / torch.sqrt(var + 1e-5)).repeat_interleave(cpg)
        y = (x[b, :n] - m) * rs * d["gamma"].to(F64) + d["beta"].to(F64)
        if film is not None:
            y = y * (1 + film[b, :Cg]) + film[b, Cg:]
        out[b, :n] = y * torch.sigmoid(y) if c.silu else y
    return out


@gpu
@pytest.mark.parametrize("c", GN_CASES, ids=lambda c: c.name)
def test_group_norm_prep(c):
    dev = torch.device("cuda")
    d = build_gn(c, "cpu")
    ref = gn_refs(c, d)
    e32 = float((gn_refs(c, d, torch.float32).to(F64) - ref).abs().max())
    extra = gn_extra(c, d)
    out, raw = launch_prep(c, d, dev, raw=True)
    Cg = c.C1 + c.C2
    ld = out["hi"].shape[1]
    got = joined(out).reshape(c.B, c.T, ld).cpu()
    assert (out["hi"].reshape(c.B, c.T, ld)[..., Cg:] == 0).all() and (out["lo"].reshape(c.B, c.T, ld)[..., Cg:] == 0).all()
    for b in range(c.B):                                     # rows past the length: exact zeros
        assert (got[b, d["rows"][b]:] == 0).all()
    r = check(c.name, got[..., :Cg], ref, e32, extra)
    record("prep GroupNorm", r)
    # the raw split is the split of the untransformed input
    rh, rl = ko.split(d["x"].to(dev))
    assert torch.equal(raw["hi"].reshape(c.B, c.T, ld)[..., :Cg].view(torch.bfloat16), rh)
    assert torch.equal(raw["lo"].reshape(c.B, c.T, ld)[..., :Cg].view(torch.bfloat16), rl)
    # NaN past the lengths and in channels >= C inside ld: no bit changes
    out_p, _ = launch_prep(c, d, dev, poison=True)
    assert torch.equal(out_p["hi"], out["hi"]) and torch.equal(out_p["lo"], out["lo"])
    if c.lens:                                               # each ragged entry equals that entry launched alone
        for b in range(c.B):
            alone, _ = launch_prep(c, d, dev, only=b)
            assert torch.equal(alone["hi"], out["hi"][b * c.T:(b + 1) * c.T]), f"{c.name}: entry {b} differs from B = 1"
            assert torch.equal(alone["lo"], out["lo"][b * c.T:(b + 1) * c.T])
    print(f"{c.name}: worst ratio {r:.3f}")


@gpu
@pytest.mark.parametrize("kind", ["stride2_even", "stride2_odd", "upsample", "upsample_rag"])
def test_prep_row_remap(kind):
    """The raw prep's row remaps: the stride-2 decimation of the downsample convs and the nearest-upsample table, including the
    ragged rule (each entry's own lengths at levels shift + 1 and shift), bit-exact against the split of the gathered rows"""
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(7)
    C_ = 72
    lens = None
    if kind.startswith("stride2"):
        B, T_src = 2, 33
        add = 0 if kind == "stride2_even" else 1
        T_dst = (T_src + 1 - add) // 2
        idx = [[t * 2 + add for t in range(T_dst)]] * B
        rowmap = None
    else:
        # 4189 = 2 * 2095 - 1 rows from 2095: the fp32 nearest rule is not t >> 1 at t = 4187 (the padded table of 2095 -> 4190 is)
        B, T_src, T_dst = 2, 2095, 4190
        rowmap = torch.tensor([t >> 1 for t in range(T_dst)], dtype=torch.int32, device=dev)
        if kind == "upsample_rag":
            lens, shift = [4189, 2000], 0
            idx = []
            for L in lens:
                t_in, t_out = rows_of([L], 1)[0], rows_of([L], 0)[0]
                src = torch.nn.functional.interpolate(torch.arange(t_in, dtype=torch.float32)[None, None], size=t_out, mode="nearest")
                idx.append([int(v) for v in src[0, 0]] + [-1] * (T_dst - t_out))
            assert idx[0][4187] == 2094
        else:
            idx = [[t >> 1 for t in range(T_dst)]] * B
    x = torch.randn(B, T_src, C_, generator=g).to(dev)
    out = split_buf(T_dst, C_, C_, B * T_dst, dev)
    a = PrepArgs()
    a.src1, a.ld1, a.C1, a.B, a.T_src, a.T_dst, a.mode = x.data_ptr(), C_, C_, B, T_src, T_dst, 0
    if rowmap is None:
        a.row_mul, a.row_add = 2, add
    else:
        a.rowmap, a.row_mul = rowmap.data_ptr(), 1
    a.out = out["s"]
    if lens:
        rl = torch.tensor(lens, dtype=torch.int32, device=dev)
        a.row_len, a.len_shift = rl.data_ptr(), 0
    desc = call(_lib.lib().ns2vc_check_prep, a)
    assert desc == f"prep_split<RAG={1 if lens else 0}>"
    want = torch.zeros(B, T_dst, C_, device=dev)
    for b in range(B):
        for t, s in enumerate(idx[b]):
            if 0 <= s < T_src:
                want[b, t] = x[b, s]
    wh, wl = ko.split(want)
    assert torch.equal(out["hi"].reshape(B, T_dst, C_).view(torch.bfloat16), wh)
    assert torch.equal(out["lo"].reshape(B, T_dst, C_).view(torch.bfloat16), wl)


# ---------------------------------------------------------------------------------------------------------------------------
# LayerNorm: ln_split / ln_apply / ln_mask, voc_norm
# ---------------------------------------------------------------------------------------------------------------------------
LN_CASES = [(36, 37, 13), (100, 100, 50), (256, 256, 9), (1020, 1020, 17), (1024, 1024, 8)]


@gpu
@pytest.mark.parametrize("kind", [0, 1, 2, 3], ids=["ln_split", "ln_apply", "ln_mask", "ln_split_nokeep"])
@pytest.mark.parametrize("C_,ld,M", LN_CASES, ids=[f"C{c}_ld{l}_M{m}" for c, l, m in LN_CASES])
@pytest.mark.parametrize("r", [0.0, 30.0, 1000.0])
def test_layer_norm(kind, C_, ld, M, r):
    """kind 0 / 1 / 2: ln_split with keep factors, ln_apply, ln_mask; 3: ln_split without keep (the denoiser's launches)"""
    names = ["ln_split<KEEP=1>", "ln_apply", "ln_mask", "ln_split<KEEP=0>"]
    split_out, masked = kind in (0, 3), kind in (0, 2)
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(C_ * 7 + M + int(r) + kind)
    x = torch.randn(M, ld, generator=g) + r * torch.sign(torch.randn(M, 1, generator=g))
    xin = x.clone()
    xin[:, C_:] = float("nan")                               # channels >= C inside ld are never read
    base = torch.randn(C_ + 1, generator=g)
    gamma, beta = (1 + 0.2 * base[1:]), 0.1 * base[:-1]
    gamma_d = torch.cat([torch.zeros(1), gamma]).to(dev)[1:] if C_ == 256 else gamma.to(dev)   # C = 256: misaligned gamma
    keep = (torch.rand(M, generator=g) < 0.7).float()
    keep[0] = 0.0
    a = LnArgs()
    xd, bd, kd = xin.to(dev), beta.to(dev), keep.to(dev)
    a.kind, a.x, a.ld, a.M, a.C, a.eps, a.gamma, a.beta = kind % 3, xd.data_ptr(), ld, M, C_, 1e-5, gamma_d.data_ptr(), bd.data_ptr()
    if masked:
        a.keep = kd.data_ptr()
    sld = (C_ + 7) // 8 * 8
    if split_out:
        out = split_buf(M, C_, sld, M, dev)
        a.split = out["s"]
    else:
        y = torch.full((M, C_ + 1), float("nan"), device=dev)
        a.y, a.y_ld = y.data_ptr(), C_ + 1
    desc = call(_lib.lib().ns2vc_check_ln, a)
    assert desc == names[kind]
    ref = ko.layer_norm_rows(x[:, :C_].to(F64), gamma.to(F64), beta.to(F64), 1e-5)
    r32 = ko.layer_norm_rows(x[:, :C_], gamma, beta, 1e-5).to(F64)
    if masked:
        ref, r32 = ref * keep.to(F64)[:, None], r32 * keep.to(F64)[:, None]
    e32 = float((r32 - ref).abs().max())
    got = joined(out).reshape(M, sld).cpu()[:, :C_] if split_out else y[:, :C_].cpu()
    if split_out:
        assert (out["hi"][:, C_:] == 0).all() and (out["lo"][:, C_:] == 0).all()
    if kind == 0:
        assert (out["hi"][keep.to(dev) == 0] == 0).all() and (out["lo"][keep.to(dev) == 0] == 0).all()
    if not split_out:
        assert torch.isnan(y[:, C_]).all()                   # nothing written past C
    # the bf16 hi/lo split of the output: 2^-17 |y|
    extra = 2.0 ** -17 * ref.abs() if split_out else None
    ratio = check(f"{desc} C={C_} r={r}", got, ref, e32, extra)
    record(f"LayerNorm {names[kind]}", ratio)
    print(f"{desc} C={C_} ld={ld} M={M} r={r}: ratio {ratio:.3f} (e32 {e32:.2e})")


@gpu
@pytest.mark.parametrize("dw", [False, True], ids=["plain", "dw"])
@pytest.mark.parametrize("C_", [128, 512, 768, 1024])
def test_voc_norm(C_, dw):
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(C_ + dw)
    worst = rule = 0.0
    for eps in (1e-6, 1e-5):
        for T in (1, 2, 15, 16, 17, 33):
            for L in sorted({1, max(T - 1, 1), T}):
                for r in (0.0, 30.0, 1000.0):
                    B = 2
                    # row means of r x the row std: on x itself, or (DW) on the depthwise output through the conv bias
                    x = torch.randn(B, T, C_, generator=g)
                    if not dw:
                        x = x + r * torch.sign(torch.randn(B, T, 1, generator=g))
                    Ls = [L, T]
                    gamma, beta = 1 + 0.2 * torch.randn(C_, generator=g), 0.1 * torch.randn(C_, generator=g)
                    dwt = torch.randn(C_, 8, generator=g) / 3 if dw else None
                    if dw:
                        dwt[:, 7] = r + 0.1 * torch.randn(C_, generator=g)
                    xin = x.clone()
                    xin[0, L:] = float("nan")                # rows past the length are never read (taps included)
                    xd, gd, bd = xin.to(dev), gamma.to(dev), beta.to(dev)
                    dwd = dwt.to(dev) if dw else None
                    ln = torch.tensor(Ls, dtype=torch.int64, device=dev)
                    out = torch.full((B, T, C_), float("nan"), device=dev)
                    sp = split_buf(T, C_, C_, B * T, dev)
                    a = VocNormArgs(xd.data_ptr(), B, T, C_, dwd.data_ptr() if dw else None, gd.data_ptr(), bd.data_ptr(), eps,
                                    ln.data_ptr(), out.data_ptr(), sp["s"])
                    desc = call(_lib.lib().ns2vc_check_voc_norm, a)
                    assert desc == f"voc_norm<DW={int(dw)}>"

                    def ref_of(dt):
                        xx = x.to(dt)
                        h = ko.depthwise7(xx, dwt.to(dt), Ls) if dw else xx
                        y = ko.layer_norm_rows(h, gamma.to(dt), beta.to(dt), eps)
                        for b in range(B):
                            y[b, Ls[b]:] = 0
                        return y.to(F64)
                    ref = ref_of(F64)
                    e32 = float((ref_of(torch.float32) - ref).abs().max())
                    for b in range(B):
                        assert (out[b, Ls[b]:] == 0).all()
                    # split output = the split of the same launch's fp32 output
                    h_, l_ = ko.split(out.reshape(B * T, C_))
                    assert torch.equal(sp["hi"].view(torch.bfloat16), h_) and torch.equal(sp["lo"].view(torch.bfloat16), l_)
                    # the fp32 row mean: the two passes keep the variance from cancelling, but the mean itself is an fp32 sum of
                    # C values (four per thread, a warp tree, then the warps in order): within (log2 C + 8) 2^-24 of mean |h|,
                    # and every output of the row moves by that times rstd |gamma|
                    h64 = ko.depthwise7(x.to(F64), dwt.to(F64), Ls) if dw else x.to(F64)
                    rstd = 1.0 / torch.sqrt(h64.var(-1, unbiased=False, keepdim=True) + eps)
                    mean_t = (math.log2(C_) + 8) * 2.0 ** -24 * h64.abs().mean(-1, keepdim=True) * rstd * gamma.to(F64).abs()
                    for b in range(B):
                        mean_t[b, Ls[b]:] = 0
                    name = f"voc_norm C={C_} T={T} L={L} eps={eps} r={r}"
                    worst = max(worst, check(name, out.cpu(), ref, e32, mean_t))
                    rule = max(rule, ko.ratio(out.cpu().to(F64) - ref, ko.parity_tol(ref, e32)))
    record(f"voc_norm<DW={int(dw)}>", worst)
    record(f"voc_norm<DW={int(dw)}> (rule alone)", rule)
    print(f"voc_norm C={C_} DW={int(dw)}: worst ratio {worst:.3f} (rule alone {rule:.3f})")


# ---------------------------------------------------------------------------------------------------------------------------
# Timestep path: small_linear
# ---------------------------------------------------------------------------------------------------------------------------
def dpm_t_inputs(steps: int = 10) -> list:
    """the model-input times t_input = (t - 1/N) N of a time-uniform DPM-Solver++ grid of the sampler (N = 1000 steps)"""
    from ns2vc_b200.dpm_solver import time_grid
    from ns2vc_b200.schedule import NoiseScheduleVP
    from ns2vc_b200.synth import linear_betas
    ns = NoiseScheduleVP("discrete", betas=linear_betas(1000))
    grid = time_grid(ns, "time_uniform", ns.T, 1.0 / ns.total_N, steps, "cpu").double()
    return ((grid - 1.0 / ns.total_N) * ns.total_N).tolist()


DPM_T = dpm_t_inputs()
LIN_CASES = [  # (name, M, K, N, in_mode, flip, shift, out_silu, add_rows, misalign)
    ("sin_M1_K128_flip", 1, 128, 512, 2, 1, 0.0, 1, 0, False),
    ("sin_M8_K512_noflip_shift1", 8, 512, 256, 2, 0, 1.0, 1, 0, False),
    ("sin_M9_K101_odd", 9, 101, 64, 2, 1, 1.0, 0, 0, False),
    ("raw_M50x4_K512_add4", 200, 512, 384, 0, 0, 0.0, 0, 4, False),
    ("silu_M9_K100_scalarW", 9, 100, 130, 1, 0, 0.0, 0, 0, False),
    ("silu_M8_K512_misalignedW", 8, 512, 96, 1, 0, 0.0, 1, 3, True),
]


def lin_inputs(case, gen):
    name, M, K, N, mode, flip, shift, osilu, add_rows, mis = case
    if mode == 2:
        ts = [0.0, 1.0, 17.5, 999.0, 1000.0] + DPM_T
        x = torch.tensor((ts * ((M + len(ts) - 1) // len(ts)))[:M]).float()[:, None]
    else:
        x = torch.randn(M, K, generator=gen)
    W = torch.randn(N, K, generator=gen) / math.sqrt(K)
    bias = 0.1 * torch.randn(N, generator=gen)
    add = torch.randn(add_rows, N, generator=gen) if add_rows else None
    return x, W, bias, add


def lin_ref(case, x, W, bias, add, dt):
    name, M, K, N, mode, flip, shift, osilu, add_rows, mis = case
    if mode == 2:
        xin = ko.sinusoid(x[:, 0].to(dt), K, bool(flip), shift)
    else:
        xin = x.to(dt)
        if mode == 1:
            xin = xin * torch.sigmoid(xin)
    return ko.small_linear(xin, W, bias, add, add_rows, bool(osilu)).to(F64)


def test_sinusoid_matches_oracle_embedding():
    """CPU: the fp64 sinusoid is the oracle's timestep_embedding (fp32) to fp32 accuracy, for both flips, shifts and odd K"""
    t = torch.tensor([0.0, 1.0, 17.5, 999.0, 1000.0] + DPM_T)
    for K in (100, 101, 128, 512):
        for flip in (True, False):
            for sh in (0.0, 1.0):
                ref = ko.sinusoid(t.to(F64), K, flip, sh)
                want = unet_oracle.timestep_embedding(t, K, flip, sh).to(F64)
                assert (ref - want).abs().max() < 2e-4, (K, flip, sh)
                # the flip is visible: swapping the halves moves the result
                assert (ko.sinusoid(t.to(F64), K, not flip, sh) - ref).abs().max() > 0.5


def test_layer_norm_and_pool_references_match_torch():
    """CPU: the LayerNorm and pooling references against F.layer_norm and the oracle's AttentionPooling in fp64"""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(5, 100, generator=g, dtype=F64)
    gm, bt = torch.randn(100, generator=g, dtype=F64), torch.randn(100, generator=g, dtype=F64)
    assert torch.equal(ko.layer_norm_rows(x, gm, bt, 1e-5), torch.nn.functional.layer_norm(x, (100,), gm, bt, 1e-5))
    B, S, Cc, H = 2, 6, 16, 4
    xs = torch.randn(B, S, Cc, generator=g, dtype=F64)
    pos = torch.randn(Cc, generator=g, dtype=F64)
    sd = {"p.norm1.weight": torch.ones(Cc, dtype=F64), "p.norm1.bias": torch.zeros(Cc, dtype=F64), "p.pool.positional_embedding": pos,
          "p.pool.q_proj.weight": torch.eye(Cc, dtype=F64), "p.pool.q_proj.bias": torch.zeros(Cc, dtype=F64),
          "p.pool.k_proj.weight": torch.eye(Cc, dtype=F64), "p.pool.k_proj.bias": torch.zeros(Cc, dtype=F64),
          "p.pool.v_proj.weight": torch.eye(Cc, dtype=F64), "p.pool.v_proj.bias": torch.zeros(Cc, dtype=F64),
          "p.proj.weight": torch.eye(Cc, dtype=F64), "p.proj.bias": torch.zeros(Cc, dtype=F64),
          "p.norm2.weight": torch.ones(Cc, dtype=F64), "p.norm2.bias": torch.zeros(Cc, dtype=F64)}
    want = unet_oracle.text_time_embedding(sd, "p", xs, H)
    xn = torch.nn.functional.layer_norm(xs, (Cc,), None, None, 1e-5)
    tok = torch.cat([xn.mean(1, keepdim=True) + pos, xn], 1)
    pooled = ko.pool_attend(tok[:, 0], torch.cat([tok, tok], -1), H, [S + 1] * B)
    got = torch.nn.functional.layer_norm(pooled, (Cc,), None, None, 1e-5)
    assert torch.allclose(got, want, rtol=1e-10, atol=1e-10)


@gpu
@pytest.mark.parametrize("case", LIN_CASES, ids=lambda c: c[0])
def test_small_linear(case):
    dev = torch.device("cuda")
    name, M, K, N, mode, flip, shift, osilu, add_rows, mis = case
    gen = torch.Generator().manual_seed(sum(map(ord, name)))
    x, W, bias, add = lin_inputs(case, gen)
    Wd = torch.zeros(N * K + 1, device=dev)
    Wv = Wd[1:].view(N, K) if mis else Wd[:N * K].view(N, K)   # misaligned: every row starts 4 bytes past a 16-byte boundary
    Wv.copy_(W.to(dev))
    xd, bd = x.to(dev).contiguous(), bias.to(dev)
    ad = add.to(dev) if add is not None else None
    out = torch.full((M, N), float("nan"), device=dev)
    a = LinArgs(xd.data_ptr(), 1 if mode == 2 else K, M, K, Wv.data_ptr(), bd.data_ptr(), N, ad.data_ptr() if ad is not None else None,
                N, add_rows, out.data_ptr(), N, mode, flip, shift, osilu)
    assert call(_lib.lib().ns2vc_check_small_linear, a) == "small_linear"
    ref = lin_ref(case, x, W, bias, add, F64)
    e32 = float((lin_ref(case, x, W, bias, add, torch.float32) - ref).abs().max())
    r = check(name, out.cpu(), ref, e32)
    tol = ko.parity_tol(ref, e32)
    if mode == 2:                                            # the flip is visible to the bound
        bad = lin_ref((name, M, K, N, mode, 1 - flip, shift, osilu, add_rows, mis), x, W, bias, add, F64)
        assert float(((bad - ref).abs() / tol).max()) >= SENSITIVITY
    if add is not None:                                      # so is the added row
        assert float(((lin_ref(case, x, W, bias, None, F64) - ref).abs() / tol).max()) >= SENSITIVITY
    record("small_linear", r)
    print(f"{name}: ratio {r:.3f} (e32 {e32:.2e})")


# ---------------------------------------------------------------------------------------------------------------------------
# AttentionPooling: pool_class_token + pool_attend / pool_attend_wide
# ---------------------------------------------------------------------------------------------------------------------------
POOL_CASES = [(dph, S, wide) for dph, wide in ((1, 0), (7, 0), (16, 0), (7, 1), (100, 1)) for S in (1, 2, 31, 32, 33, 1100)]


@gpu
@pytest.mark.parametrize("dph,S,wide", POOL_CASES, ids=[f"dph{d}_S{s}_{'wide' if w else 'narrow'}" for d, s, w in POOL_CASES])
def test_pool(dph, S, wide):
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(dph * 10007 + S + wide)
    heads = 1 if dph == 100 else 4
    C_ = heads * dph
    B = 3
    for lens in (None, [1, S, max(S // 2, 1)]):
        x = torch.randn(B, S, C_, generator=g)
        pos = torch.randn(C_, generator=g)
        q = torch.randn(B, C_, generator=g)
        kv = torch.randn(B, S + 1, 2 * C_, generator=g)
        kv[..., :C_] *= 8.0 / math.sqrt(max(1, dph)) ** 0.5 * dph ** 0.25   # scores of std ~ 8
        keys = [S + 1] * B if lens is None else [l + 1 for l in lens]
        rows = [S] * B if lens is None else lens
        xin, kvin = x.clone(), kv.clone()
        for b in range(B):
            xin[b, rows[b]:] = float("nan")
            kvin[b, keys[b]:] = float("nan")
        xd, pd, qd, kvd = xin.to(dev), pos.to(dev), q.to(dev), kvin.to(dev)
        tok = torch.full((B, S + 1, C_), float("nan"), device=dev)
        out = torch.full((B, C_), float("nan"), device=dev)
        ld = torch.tensor(lens, dtype=torch.int32, device=dev) if lens else None
        a = PoolArgs(xd.data_ptr(), pd.data_ptr(), B, S, C_, tok.data_ptr(), qd.data_ptr(), kvd.data_ptr(), heads, wide, out.data_ptr(),
                     ld.data_ptr() if lens else None)
        desc = call(_lib.lib().ns2vc_check_pool, a)
        assert desc == f"pool_class_token+{'pool_attend_wide' if wide else 'pool_attend'}<RAG={int(bool(lens))}>"
        cls_ref = torch.stack([x[b, :rows[b]].to(F64).mean(0) for b in range(B)]) + pos.to(F64)
        cls32 = torch.stack([x[b, :rows[b]].mean(0) for b in range(B)]) + pos
        r1 = check(f"class token S={S}", tok[:, 0].cpu(), cls_ref, float((cls32.to(F64) - cls_ref).abs().max()))
        for b in range(B):                                   # copied rows are the input rows
            assert torch.equal(tok[b, 1:rows[b] + 1], xd[b, :rows[b]])
        ref = ko.pool_attend(q.to(F64), kv.to(F64), heads, keys)
        e32 = float((ko.pool_attend(q, kv, heads, keys).to(F64) - ref).abs().max())
        r2 = check(f"pool dph={dph} S={S} rag={bool(lens)}", out.cpu(), ref, e32)
        if S > 1:                                            # pooling over the padded S is visible to the bound
            bad = ko.pool_attend(q.to(F64), kv.to(F64), heads, [S + 1] * B)
            if lens:
                assert float(((bad - ref).abs() / ko.parity_tol(ref, e32)).max()) >= SENSITIVITY
        if lens:                                             # a ragged entry equals that entry alone at B = 1
            for b in range(B):
                o1 = torch.full((1, C_), float("nan"), device=dev)
                t1 = torch.full((1, S + 1, C_), float("nan"), device=dev)
                a1 = PoolArgs(xd[b:b + 1].data_ptr(), pd.data_ptr(), 1, S, C_, t1.data_ptr(), qd[b:b + 1].data_ptr(),
                              kvd[b:b + 1].data_ptr(), heads, wide, o1.data_ptr(), ld[b:b + 1].data_ptr())
                call(_lib.lib().ns2vc_check_pool, a1)
                assert torch.equal(o1, out[b:b + 1]) and torch.equal(t1[:, 0], tok[b:b + 1, 0])
        record("pool_attend_wide" if wide else "pool_attend", r2)
        record("pool_class_token", r1)


# ---------------------------------------------------------------------------------------------------------------------------
# nct_to_split
# ---------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("rag", [False, True])
def test_nct_split(rag):
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(11)
    B, C_, T, ld = 3, 100, 67, 104
    buf = torch.randn(B, C_ * T + 13, generator=g)           # [B, C, T] entries at a batch stride of C T + 13
    xv = buf[:, :C_ * T].reshape(B, C_, T).clone()
    lens = [T, 1, 40]
    if rag:
        for b in range(B):
            buf[b, :C_ * T].view(C_, T)[:, lens[b]:] = float("nan")
    bd = buf.to(dev)
    out = split_buf(T, C_, ld, B * T, dev)
    rl = torch.tensor(lens, dtype=torch.int32, device=dev)
    a = NctArgs(bd.data_ptr(), C_ * T + 13, B, C_, T, out["s"], rl.data_ptr() if rag else None)
    assert call(_lib.lib().ns2vc_check_nct_split, a) == f"nct_to_split<RAG={int(rag)}>"
    want = torch.zeros(B, T, ld)
    want[..., :C_] = xv.transpose(1, 2)
    if rag:
        for b in range(B):
            want[b, lens[b]:] = 0
    wh, wl = ko.split(want.to(dev))
    assert torch.equal(out["hi"].view(torch.bfloat16).reshape(B, T, ld), wh)
    assert torch.equal(out["lo"].view(torch.bfloat16).reshape(B, T, ld), wl)


# ---------------------------------------------------------------------------------------------------------------------------
# The product's GroupNorm path: a producing gemm_tc with EPI_STATS (its own fp32-partial / fp64-atomic sums), consumed by the
# prep kernel and by a panel-mode gemm_tc whose prologue finishes the same sums (prep_affine over the 256 transform threads)
# ---------------------------------------------------------------------------------------------------------------------------
class Chain:
    def __init__(self, name, B, T, Cn, G, r, lens=None, shift=0, film=None):
        self.name, self.B, self.T, self.C, self.G, self.r, self.lens, self.shift, self.film = name, B, T, Cn, G, r, lens, shift, film


CHAIN_CASES = [
    Chain("G32_C64_T129_r0", 2, 129, 64, 32, 0.0),
    Chain("rag_G8_C128_T65_r30_film", 3, 65, 128, 8, 30.0, lens=[65, 2, 63], film="plain"),
    Chain("rag_G1_C64_T128_r100_bigfilm", 2, 128, 64, 1, 100.0, lens=[128, 1], film="big"),
    Chain("G8_C256_T127_r4_film_m1", 2, 127, 256, 8, 4.0, film="m1"),
    Chain("rag_G32_C512_T64_s1_r30", 2, 64, 512, 32, 30.0, lens=[127, 3], shift=1),
    Chain("G8_C64_T63_r100", 3, 63, 64, 8, 100.0),
]


def pack(W: torch.Tensor, dev) -> Dict:
    import test_kernels_fp64 as tk
    N = tk.pad128(W.shape[0])
    nkb = W.shape[1] // 64
    wh = torch.zeros(nkb * N * 64, dtype=torch.bfloat16, device=dev)
    wl = torch.zeros_like(wh)
    _lib.check(_lib.lib().ns2vc_check_pack_b(W.data_ptr(), W.shape[0], W.shape[1], 1, 0, 0, W.shape[1], 0, 0, 0, None, wh.data_ptr(),
                                             wl.data_ptr(), N, nkb, stream()))
    return dict(hi=wh, lo=wl, N=N, nkb=nkb, W=W)


def run_chain(c: Chain, dev):
    import test_kernels_fp64 as tk
    g = torch.Generator().manual_seed(sum(map(ord, c.name)))
    rn = lambda *s: torch.randn(*s, generator=g)
    B, T, Cn = c.B, c.T, c.C
    rows = rows_of(c.lens, c.shift) if c.lens else [T] * B
    rl = torch.tensor(c.lens, dtype=torch.int32, device=dev) if c.lens else None
    # producer: x = A W1^T + bias1 over 64 input channels; bias1 puts each group's mean at r x its std (~1)
    A = rn(B, T, 64).to(dev)
    ah, al = ko.split(A)
    W1 = (rn(Cn, 64) / 8).to(dev)
    b1 = (c.r * torch.sign(rn(c.G)).repeat_interleave(Cn // c.G) + 0.1 * rn(Cn)).to(dev)
    p1 = pack(W1, dev)
    ld = (Cn + 7) // 8 * 8
    x32 = torch.full((B * T, Cn), float("nan"), device=dev)
    xs = split_buf(T, Cn, ld, B * T, dev)
    st = torch.zeros(2, B, Cn, dtype=F64, device=dev)
    a = tk.GemmArgs()
    a.B, a.T_out, a.nsrc = B, T, 1
    a.src[0] = tk.Split(ah.data_ptr(), al.data_ptr(), T, 64, 64, 0)
    a.seg[0] = (C.c_int * 4)(0, 0, 64, 0)
    a.nseg = 1
    a.w_hi, a.w_lo, a.N, a.n_valid, a.nkb_w = p1["hi"].data_ptr(), p1["lo"].data_ptr(), p1["N"], Cn, 1
    a.flags = tk.EPI_BIAS | tk.EPI_OUT_F32 | tk.EPI_OUT_SPLIT | tk.EPI_STATS
    a.bias, a.out, a.out_ld = b1.data_ptr(), x32.data_ptr(), Cn
    a.out_hi, a.out_lo, a.out_split_ld, a.f16_col0 = xs["hi"].data_ptr(), xs["lo"].data_ptr(), ld, -1
    a.stat_sum, a.stat_sq = st[0].data_ptr(), st[1].data_ptr()
    if rl is not None:
        a.row_len, a.len_shift = rl.data_ptr(), c.shift
    a.ksplit = 1
    d1 = tk.call(_lib.lib().ns2vc_check_gemm, a)
    torch.cuda.synchronize()
    assert "XF=0" in d1 and f"RAG={int(rl is not None)}" in d1, d1
    gamma, beta = (1 + 0.2 * rn(Cn)).to(dev), (0.1 * rn(Cn)).to(dev)
    film = None
    if c.film == "plain":
        film = torch.cat([0.3 * rn(B, Cn), 0.3 * rn(B, Cn)], -1).to(dev)
    elif c.film == "big":
        film = torch.cat([30.0 * rn(B, Cn), rn(B, Cn)], -1).to(dev)
    elif c.film == "m1":
        film = torch.cat([-1.0 + 0.01 * rn(B, Cn), 0.1 * rn(B, Cn)], -1).to(dev)
    # consumer 1: the prep kernel from the producer's sums
    out = split_buf(T, Cn, ld, B * T, dev)
    pa = PrepArgs()
    pa.src1, pa.ld1, pa.C1, pa.B, pa.T_src, pa.T_dst, pa.row_mul, pa.mode = x32.data_ptr(), Cn, Cn, B, T, T, 1, 2
    pa.stats1, pa.gamma, pa.beta, pa.G, pa.eps = st.data_ptr(), gamma.data_ptr(), beta.data_ptr(), c.G, 1e-5
    if film is not None:
        pa.film, pa.film_ld = film.data_ptr(), 2 * Cn
    pa.out = out["s"]
    if rl is not None:
        pa.row_len, pa.len_shift = rl.data_ptr(), c.shift
    assert call(_lib.lib().ns2vc_check_prep, pa) == f"prep_split<RAG={int(rl is not None)}>"
    # consumer 2: a k = 3 panel-mode conv over the producer's raw split, GroupNorm(+FiLM)+SiLU in its prologue
    ncb = (Cn + 63) // 64
    W2 = (rn(64, 3 * ncb * 64) / math.sqrt(3 * Cn)).to(dev)
    b2 = (0.1 * rn(64)).to(dev)
    p2 = pack(W2, dev)
    y2 = torch.full((B * T, 64), float("nan"), device=dev)
    a2 = tk.GemmArgs()
    a2.B, a2.T_out, a2.nsrc = B, T, 1
    a2.src[0] = tk.Split(xs["hi"].data_ptr(), xs["lo"].data_ptr(), T, Cn, ld, 0)
    a2.xseg[0] = (C.c_int * 8)(0, 0, Cn, 3, 0, ncb, 1, 0)
    a2.nxs = 1
    a2.w_hi, a2.w_lo, a2.N, a2.n_valid, a2.nkb_w = p2["hi"].data_ptr(), p2["lo"].data_ptr(), p2["N"], 64, 3 * ncb
    a2.flags, a2.bias, a2.out, a2.out_ld, a2.f16_col0, a2.ksplit = tk.EPI_BIAS | tk.EPI_OUT_F32, b2.data_ptr(), y2.data_ptr(), 64, -1, 1
    if rl is not None:
        a2.row_len, a2.len_shift = rl.data_ptr(), c.shift
    a2.pre_mode = 2
    a2.gn_stats1, a2.gn_C1, a2.gn_G, a2.gn_eps, a2.gn_gamma, a2.gn_beta = st.data_ptr(), Cn, c.G, 1e-5, gamma.data_ptr(), beta.data_ptr()
    if film is not None:
        a2.gn_film, a2.gn_film_ld = film.data_ptr(), 2 * Cn
    d2 = tk.call(_lib.lib().ns2vc_check_gemm, a2)
    torch.cuda.synchronize()
    assert "XF=1" in d2 and f"RAG={int(rl is not None)}" in d2, d2
    return dict(rows=rows, x=x32.reshape(B, T, Cn).cpu(), st=st.cpu(), prep=joined(out).reshape(B, T, ld)[..., :Cn].cpu(),
                conv=y2.reshape(B, T, 64).cpu(), gamma=gamma.cpu(), beta=beta.cpu(), film=film.cpu() if film is not None else None,
                W2=W2.cpu(), b2=b2.cpu(), ncb=ncb, out=out)


def chain_refs(c: Chain, d, dt=F64, **defect):
    x = d["x"].to(dt)
    film = d["film"].to(dt) if d["film"] is not None else None
    return ko.group_norm_rows(x, c.G, d["gamma"].to(dt), d["beta"].to(dt), 1e-5, d["rows"], film, True, **defect)


def chain_conv(c: Chain, d, y: torch.Tensor) -> torch.Tensor:
    """k = 3 conv (zero padding) of the normalised [B, T, C] y with W2 (tap-major k-blocks), + b2, in y's dtype"""
    cols = [ko.gather(y, c.T, c.C, 0, 64 * d["ncb"], t, c.T) for t in (-1, 0, 1)]
    out = torch.cat(cols, -1) @ d["W2"].to(y.dtype).T + d["b2"].to(y.dtype)
    for b in range(c.B):
        out[b, d["rows"][b]:] = 0
    return out


@gpu
@pytest.mark.parametrize("c", CHAIN_CASES, ids=lambda c: c.name)
def test_group_norm_from_producer_sums(c):
    """EPI_STATS -> prep and EPI_STATS -> panel-mode conv, against fp64 on the producer's own fp32 output.  Bound: the rule
    (floored at 2 e32) plus the named design terms: the producers' fp32 partial sums (kernel_oracle.one_pass_variance_term), the
    uncentred affine and the hi/lo output (affine_terms), and for the panel the hi/lo split of its raw input, 2^-17 |x| rstd
    |gamma (1 + s)|, carried through SiLU (slope < 1.1) and |W2|.  The ratio to the rule alone is printed and recorded."""
    dev = torch.device("cuda")
    d = run_chain(c, dev)
    x64 = d["x"].to(F64)
    for b in range(c.B):                                     # the producer's sums are those of its fp32 output to the partials' rounding
        assert (d["x"][b, d["rows"][b]:] == 0).all()
    film = d["film"].to(F64) if d["film"] is not None else None
    g64 = d["gamma"].to(F64)
    ref = chain_refs(c, d)
    e32 = float((chain_refs(c, d, torch.float32).to(F64) - ref).abs().max())
    var_t = ko.one_pass_variance_term(x64, c.G, g64, d["rows"], film, 1e-5)
    aff_t = ko.affine_terms(x64, c.G, g64, d["beta"].to(F64), d["rows"], film, 1e-5)
    extra = 1.1 * (var_t + aff_t)
    r_prep = check(c.name + " prep", d["prep"], ref, e32, extra)
    rule_prep = ko.ratio(d["prep"].to(F64) - ref, ko.parity_tol(ref, e32))
    for b in range(c.B):
        assert (d["prep"][b, d["rows"][b]:] == 0).all()
    # panel: the raw input as hi + lo (2^-17 |x|), normalised: |x| rstd |gamma (1 + s)| per unit; then re-split (2^-17 |y|)
    panel_t = torch.zeros_like(x64)
    for b in range(c.B):
        n = d["rows"][b]
        gq = x64[b, :n].T.reshape(c.G, -1)
        rstd = 1.0 / torch.sqrt(gq.var(-1, unbiased=False, keepdim=True) + 1e-5)
        fs = (1 + film[b, :c.C]).abs() if film is not None else 1.0
        panel_t[b, :n] = 2.0 ** -17 * x64[b, :n].abs() * rstd.expand_as(gq).reshape(c.C, n).T * g64.abs() * fs
    gn_err = extra + 1.1 * panel_t + 2.0 ** -17 * ref.abs()
    cref = chain_conv(c, d, ref)
    cols_abs = torch.cat([ko.gather(ref.abs(), c.T, c.C, 0, 64 * d["ncb"], t, c.T) for t in (-1, 0, 1)], -1)
    cols_err = torch.cat([ko.gather(gn_err, c.T, c.C, 0, 64 * d["ncb"], t, c.T) for t in (-1, 0, 1)], -1)
    Wabs = d["W2"].to(F64).abs()
    conv_extra = cols_err @ Wabs.T + 64 * 2.0 ** -24 * (cols_abs @ Wabs.T)
    conv_e32 = float((chain_conv(c, d, chain_refs(c, d, torch.float32)).to(F64) - cref).abs().max())
    r_conv = check(c.name + " panel conv", d["conv"], cref, conv_e32, conv_extra)
    rule_conv = ko.ratio(d["conv"].to(F64) - cref, ko.parity_tol(cref, conv_e32))
    # the bound notices the defects the product could have
    if film is not None:
        sensitive(c.name + " FiLM without 1+", chain_refs(c, d, one_plus=False), ref, e32, extra)
    if c.lens and any(r > 1 for r in d["rows"]):
        sensitive(c.name + " one row fewer", chain_refs(c, d, count=[max(r - 1, 1) for r in d["rows"]]), ref, e32, extra)
    record("chain EPI_STATS -> prep", r_prep)
    record("chain EPI_STATS -> prep (rule alone)", rule_prep)
    record("chain EPI_STATS -> panel gemm_tc", r_conv)
    record("chain EPI_STATS -> panel gemm_tc (rule alone)", rule_conv)
    print(f"{c.name}: prep {r_prep:.3f} (rule alone {rule_prep:.3f}), panel conv {r_conv:.3f} (rule alone {rule_conv:.3f})")


# ---------------------------------------------------------------------------------------------------------------------------
# The whole timestep path: ns2vc_unet_time_table runs the engine's time_path_ops chain (sinusoid -> linear_1 -> SiLU ->
# linear_2 (+ aug_emb of the prompt, row m reading entry m % B) -> every resnet's time_emb_proj of SiLU(emb)) over steps x B rows
# ---------------------------------------------------------------------------------------------------------------------------
def time_path_truth(sd, cfg, t: torch.Tensor, prompt: torch.Tensor, dt) -> torch.Tensor:
    """FiLM rows [steps * B, film_width] of t [steps, B] in dtype dt: unet_oracle's embeddings (the sinusoid of kernel_oracle in
    fp64, unet_oracle.timestep_embedding in fp32) -> text_time_embedding -> the resnets' time_emb_proj, step-major rows"""
    from ns2vc_b200.arch import build_plan
    s = {k: v.to(dt) for k, v in sd.items()}
    K, B = t.shape
    tt = t.reshape(-1)
    if dt == F64:
        temb = ko.sinusoid(tt.to(F64), cfg.block_out_channels[0], cfg.flip_sin_to_cos, cfg.freq_shift)
    else:
        temb = unet_oracle.timestep_embedding(tt, cfg.block_out_channels[0], cfg.flip_sin_to_cos, cfg.freq_shift).to(dt)
    emb = torch.nn.functional.linear(temb, s["time_embedding.linear_1.weight"], s["time_embedding.linear_1.bias"])
    emb = torch.nn.functional.linear(torch.nn.functional.silu(emb), s["time_embedding.linear_2.weight"], s["time_embedding.linear_2.bias"])
    aug = unet_oracle.text_time_embedding(s, "add_embedding", prompt.to(dt), cfg.addition_embed_type_num_heads)
    emb = emb + aug.repeat(K, 1)
    return torch.cat([torch.nn.functional.linear(torch.nn.functional.silu(emb), s[op.prefix + ".time_emb_proj.weight"],
                                                 s[op.prefix + ".time_emb_proj.bias"])
                      for op in build_plan(cfg) if op.kind == "resnet"], dim=1).to(F64)


@gpu
@pytest.mark.parametrize("which", ["tiny", "full"])
def test_time_path_against_fp64(which):
    from conftest import tiny_config
    from ns2vc_b200.arch import ns2vc_denoiser_config
    from ns2vc_b200.fused import DenoiserSession
    from ns2vc_b200.synth import make_state_dict
    from ns2vc_b200.unet import UNet1DConditionModel
    cfg = tiny_config() if which == "tiny" else ns2vc_denoiser_config()
    m = UNet1DConditionModel(in_channels=cfg.in_channels, out_channels=cfg.out_channels, block_out_channels=cfg.block_out_channels,
                             layers_per_block=list(cfg.layers_per_block), norm_num_groups=cfg.norm_num_groups,
                             cross_attention_dim=cfg.cross_attention_dim, attention_head_dim=cfg.num_heads,
                             addition_embed_type=cfg.addition_embed_type, addition_embed_type_num_heads=cfg.addition_embed_type_num_heads,
                             resnet_time_scale_shift=cfg.resnet_time_scale_shift)
    sd = make_state_dict(cfg, 0)
    m.load_state_dict(sd)
    m = m.cuda().eval()
    g = torch.Generator().manual_seed(5)
    B, T, S = 3, 40, 13
    Cc = cfg.in_channels - cfg.out_channels
    content = torch.randn(B, Cc, T, generator=g).cuda()
    prompt = torch.randn(B, S, cfg.cross_attention_dim, generator=g)
    sess = DenoiserSession(m, content, prompt.cuda(), None)
    sess.prepare()
    t_in = DPM_T + [0.0, 1.0, 17.5, 999.0, 1000.0]
    tv = torch.tensor(t_in, dtype=torch.float32)
    tv = torch.stack([tv.roll(b) for b in range(B)], 1).contiguous()            # [steps, B]: each entry its own order
    L = _lib.lib()
    table = torch.empty(int(L.ns2vc_unet_time_table_floats(sess.h, tv.numel())), dtype=torch.float32, device="cuda")
    sess.time_table(tv.cuda(), table)
    torch.cuda.synchronize()
    fw = int(L.ns2vc_unet_film_width(sess.h))
    got = table[:tv.numel() * fw].view(tv.numel(), fw).cpu()
    ref = time_path_truth(sd, cfg, tv, prompt, F64)
    e32 = float((time_path_truth(sd, cfg, tv, prompt, torch.float32) - ref).abs().max())
    r = check(f"time path {which}", got, ref, e32)
    tol = ko.parity_tol(ref, e32)
    # the bound sees a wrong flip and a wrong aug row
    cfg_f = dataclasses.replace(cfg, flip_sin_to_cos=not cfg.flip_sin_to_cos)
    assert float(((time_path_truth(sd, cfg_f, tv, prompt, F64) - ref).abs() / tol).max()) >= SENSITIVITY
    assert float(((time_path_truth(sd, cfg, tv, prompt.roll(1, 0), F64) - ref).abs() / tol).max()) >= SENSITIVITY
    record(f"time path ({which} config)", r)
    print(f"time path {which}: {tv.numel()} rows x {fw}: ratio {r:.3f} (e32 {e32:.2e})")
