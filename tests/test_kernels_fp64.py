"""The wgmma GEMM (gemm_tc_kernel) and the flash attention (attn_v2_kernel, attn_tc_kernel) launch by launch, through the
test-only C entry points ns2vc_check_gemm / ns2vc_check_attention / ns2vc_check_pack_b (csrc/kernel_check.cu), which run the
engines' own host code and launchers.  Each case is compared with two references (oracle/kernel_oracle.py):

* the emulation: the documented roundings (bf16 hi/lo operands, the 3-term product, the epilogue; fp16 or bf16 hi/lo softmax
  weights, online softmax tile by tile) in fp64.  |gpu - emu| <= tol_emu elementwise, where tol_emu is an fp32-accumulation
  level bound: for the GEMM 16 * 2^-24 * (|A| |W|) per output plus 2 ulps of the running accumulator for each of the three
  MMAs of every 16-wide k-step (the tensor cores add each MMA's products to the fp32 accumulator with truncation, so the error
  grows with the number of k-steps: 1.5 x the first term alone at K = 4096), carried through the epilogue's slope, plus a few
  fp32 roundings of the epilogue's values; for the attention 16 * 2^-24 * (weighted |v| + |out|), plus ln2 * the weighted score error
  (16 * 2^-24 * (|q| |k| * scale + |s|)) on |v| and |out|, plus two fp16 ulps of the largest weight * |v| for fp16 weights
  whose rounding flips between the kernel's fp32 exponentials and the emulation's fp64 ones (2^-16 of the weight * |v| for a
  bf16 hi/lo weight near a rounding boundary of its hi or lo half);
* the truth: the operation in fp64 from the fp32 inputs, under the project's parity rule 1e-3 |ref| + 1e-4 rms(ref).  Where the
  precision design itself does not meet that rule in one launch, the case adds the design's own error terms and the test
  prints the rule's ratio: fp16 softmax weights (2^-12 relative per weight, which averages out only over many keys and mild
  scores: 2.2 - 2.9 x the rule on random values), scores of std 8 (3 * 2^-17 of |q| |k| per score: 1.07 x), and a folded
  LayerNorm over rows whose mean is 30 x their std (the 3xBF16 product sees the uncentred row: 3.5 - 4 x).

No bound may be vacuous: for every case the emulation is evaluated again with one defect injected - each of the three split
products dropped (GEMM; attention cases whose score std is >= 2), the key mask moved by one key (attention) - and the largest
|defect - emu| / tol_emu must be >= 16.

Exact properties: rows past row_len / a zero row mask are exactly 0; NaN in the rows and channels of the sources the contract
says are never read (rows past src.T inside the batch pitch, channels >= src.C inside ld, key tiles past key_len) changes
nothing bitwise and a second launch is bit-identical; a split output is bit-consistent with the same launch's fp32 output; the
column and row statistics (EPI_STATS / EPI_ROWSTATS) equal fp64 sums of the kernel's own fp32 output within the fp32 rounding of
its 32-element partial sums (the kernel adds them in fp32 before its fp64 atomics, so they are not fp64-exact); ragged rows equal
the same entry run alone, bit for bit.  A ksplit = 2 launch adds the partner's fp32 partial tile at the end: it is checked
against the references, and it is not bit-identical to ksplit = 1 (the test prints which).

The fp16-weight attention cases run only when NS2VC_ATTN_P selects fp16 weights (the default) and are skipped otherwise.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess
import sys
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import pytest
import torch

from conftest import REPO
from ns2vc_b200 import _lib
from oracle import kernel_oracle as ko

F64 = torch.float64
gpu = pytest.mark.gpu

EPI_BIAS, EPI_RESIDUAL, EPI_GEGLU, EPI_OUT_NCT, EPI_ROWBIAS, EPI_OUT_F32, EPI_OUT_SPLIT, EPI_STATS = 1, 2, 4, 8, 16, 32, 64, 128
EPI_LNFOLD, EPI_ROWSTATS, EPI_RELU, EPI_ROWMASK, EPI_GELU = 256, 512, 1024, 2048, 4096
SENSITIVITY = 16.0
WORST: Dict[str, Dict[str, float]] = {}        # family -> worst ratios, printed at the end of the module


class Split(C.Structure):
    _fields_ = [("hi", C.c_void_p), ("lo", C.c_void_p), ("T", C.c_int), ("C", C.c_int), ("ld", C.c_int), ("bpitch", C.c_longlong)]


class GemmArgs(C.Structure):
    _fields_ = [("B", C.c_int), ("T_out", C.c_int), ("nsrc", C.c_int), ("src", Split * 4), ("nseg", C.c_int), ("seg", (C.c_int * 4) * 8),
                ("nxs", C.c_int), ("xseg", (C.c_int * 8) * 4), ("w_hi", C.c_void_p), ("w_lo", C.c_void_p), ("N", C.c_int),
                ("n_valid", C.c_int), ("nkb_w", C.c_int), ("flags", C.c_int), ("bias", C.c_void_p), ("rowbias", C.c_void_p),
                ("rowbias_ld", C.c_int), ("res", C.c_void_p), ("res_ld", C.c_int), ("out", C.c_void_p), ("out_ld", C.c_int),
                ("out_hi", C.c_void_p), ("out_lo", C.c_void_p), ("out_split_ld", C.c_int), ("f16_col0", C.c_int),
                ("ln_stats", C.c_void_p), ("ln_g", C.c_void_p), ("ln_C", C.c_int), ("ln_eps", C.c_float), ("row_stats", C.c_void_p),
                ("stat_sum", C.c_void_p), ("stat_sq", C.c_void_p), ("rowmask", C.c_void_p), ("row_len", C.c_void_p),
                ("len_shift", C.c_int), ("pre_scale", C.c_void_p), ("pre_shift", C.c_void_p), ("pre_mode", C.c_int), ("pre_C", C.c_int),
                ("ksplit", C.c_int), ("gn_stats1", C.c_void_p), ("gn_stats2", C.c_void_p), ("gn_C1", C.c_int), ("gn_C2", C.c_int),
                ("gn_G", C.c_int), ("gn_eps", C.c_float), ("gn_gamma", C.c_void_p), ("gn_beta", C.c_void_p), ("gn_film", C.c_void_p),
                ("gn_film_ld", C.c_int), ("bn", C.c_int), ("tma_out", C.c_int)]


class AttnArgs(C.Structure):
    _fields_ = [("B", C.c_int), ("H", C.c_int), ("Tq", C.c_int), ("Tk", C.c_int), ("dh", C.c_int), ("scale", C.c_float), ("v2", C.c_int),
                ("q", C.c_void_p), ("q_ld", C.c_int), ("k", C.c_void_p), ("k_ld", C.c_int), ("v", C.c_void_p), ("v_ld", C.c_int),
                ("qs", Split), ("ks", Split), ("vs", Split), ("q_c0", C.c_int), ("k_c0", C.c_int), ("v_c0", C.c_int),
                ("p_split", C.c_int), ("key_len", C.c_void_p), ("key_shift", C.c_int), ("bias", C.c_void_p), ("out", C.c_void_p),
                ("out_ld", C.c_int), ("out_hi", C.c_void_p), ("out_lo", C.c_void_p), ("out_split_ld", C.c_int), ("pb", C.c_int)]


def ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def call(fn, args) -> str:
    desc = C.create_string_buffer(96)
    _lib.check(fn(C.cast(C.byref(args), C.c_void_p), desc, 96, stream()))
    return desc.value.decode()


def record(family: str, **ratios: float) -> None:
    w = WORST.setdefault(family, {})
    for k, v in ratios.items():
        w[k] = max(w.get(k, 0.0), v) if not k.startswith("sens") else min(w.get(k, math.inf), v)


@pytest.fixture(autouse=True)
def _no_tf32():
    """The fp64 references' matmuls stay fp64 / true fp32 while a test of this module runs; the flags are restored after it"""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    for fam, w in sorted(WORST.items()):
        print(f"\n[kernel checks] {fam}: " + ", ".join(f"{k}={v:.3g}" for k, v in sorted(w.items())))


# ---------------------------------------------------------------------------------------------------------------------------
# GEMM cases
# ---------------------------------------------------------------------------------------------------------------------------
@dataclass
class GCase:
    name: str
    B: int
    T: int
    srcs: List[Tuple[int, int, int]]                 # (C, ld, rows of padding past T inside the batch pitch)
    segs: List[Tuple[int, int, int, int]] = field(default_factory=list)      # plain: (src, c0, nch, tap)
    xsegs: List[Tuple[int, int, int, int, int]] = field(default_factory=list)  # panel: (src, nch, ntap, xf, aff_c0)
    n_valid: int = 128
    kind: str = "plain"                              # plain | lnf | geglu | geglu_lnf | enc | voc
    flags: int = EPI_BIAS | EPI_OUT_F32
    out_ld: Optional[int] = None
    res_ld: Optional[int] = None
    f16_col0: int = -1
    row_len: Optional[List[int]] = None              # level-0 lengths (ragged), with len_shift
    len_shift: int = 0
    ksplit: int = 1
    silu: bool = True
    shift: float = 0.0                               # panel affine shift offset (5: the padding must stay zero after it)
    rowmask: bool = False
    mean_over_std: float = 0.0                       # lnf: |row mean| / row std
    rule: bool = True                                # False: truth within the rule plus the design's own error terms
    seed: int = 0


def k3(src, C):
    return [(src, 0, C, t) for t in (-1, 0, 1)]


GEMM_CASES = [
    GCase("plain_k3_B3_T129_C100_nv100_res_f16col", 3, 129, [(100, 112, 3)], k3(0, 100), n_valid=100,
          flags=EPI_BIAS | EPI_RESIDUAL | EPI_OUT_F32 | EPI_OUT_SPLIT, out_ld=100, res_ld=101, f16_col0=64),
    GCase("plain_2src_B1_T1_C576_C36_c0", 1, 1, [(576, 584, 0), (36, 48, 2)], [(0, 0, 576, 0), (1, 0, 36, 0), (0, 64, 100, -1)],
          flags=EPI_OUT_F32 | EPI_ROWSTATS),
    GCase("plain_7seg_B1_T257_nct", 1, 257, [(64, 64, 1)], [(0, 0, 64, t) for t in range(-3, 4)], n_valid=100,
          flags=EPI_BIAS | EPI_OUT_NCT),
    GCase("plain_8seg_B3_T2_C36_stats", 3, 2, [(36, 40, 1)], [(0, 0, 36, t) for t in range(-3, 5)], flags=EPI_BIAS | EPI_OUT_F32 | EPI_STATS),
    GCase("plain_nkb64_B1_T1025", 1, 1025, [(4096, 4096, 0)], [(0, 0, 4096, 0)], flags=EPI_OUT_F32 | EPI_OUT_SPLIT, seed=5),
    GCase("head_nv1026_B3_T255_odd_ld", 3, 255, [(128, 128, 0)], [(0, 0, 128, 0)], n_valid=1026, flags=EPI_BIAS | EPI_OUT_F32,
          out_ld=1027),
    GCase("lnf_B3_T255_C576_mean30", 3, 255, [(576, 576, 0)], [(0, 0, 576, 0)], n_valid=200, kind="lnf",
          flags=EPI_BIAS | EPI_OUT_F32 | EPI_OUT_SPLIT, mean_over_std=30.0, rule=False),
    GCase("lnf_B1_T1_C128_mean4", 1, 1, [(128, 128, 0)], [(0, 0, 128, 0)], n_valid=128, kind="lnf", flags=EPI_BIAS | EPI_OUT_F32,
          mean_over_std=4.0),
    GCase("geglu_B3_T127_C128", 3, 127, [(128, 128, 0)], [(0, 0, 128, 0)], n_valid=128, kind="geglu", flags=EPI_OUT_F32 | EPI_OUT_SPLIT),
    GCase("geglu_lnf_B1_T257_C100_mean1", 1, 257, [(100, 104, 0)], [(0, 0, 100, 0)], n_valid=64, kind="geglu_lnf",
          flags=EPI_OUT_F32 | EPI_OUT_SPLIT, mean_over_std=1.0),
    GCase("enc_relu_mask_res_B3_T129", 3, 129, [(100, 104, 0)], k3(0, 100), kind="enc",
          flags=EPI_BIAS | EPI_RESIDUAL | EPI_RELU | EPI_ROWMASK | EPI_OUT_F32, rowmask=True),
    GCase("voc_gelu_B1_T1025", 1, 1025, [(128, 128, 0)], [(0, 0, 128, 0)], kind="voc", flags=EPI_BIAS | EPI_GELU | EPI_OUT_F32),
    GCase("voc_gelu_mask_B3_T127", 3, 127, [(128, 128, 0)], [(0, 0, 128, 0)], kind="voc",
          flags=EPI_BIAS | EPI_GELU | EPI_ROWMASK | EPI_OUT_F32, rowmask=True),
    GCase("rag_k3_B3_T255_shift2", 3, 255, [(128, 128, 0)], k3(0, 128), flags=EPI_BIAS | EPI_OUT_F32, row_len=[1017, 509, 1],
          len_shift=2),
    GCase("xf_k3_ks1_B3_T129_shift5", 3, 129, [(100, 104, 2)], xsegs=[(0, 100, 3, 1, 0)], flags=EPI_BIAS | EPI_OUT_F32 | EPI_STATS,
          shift=5.0),
    GCase("xf_k3_ks2_9panels_B1_T128", 1, 128, [(576, 576, 1)], xsegs=[(0, 576, 3, 1, 0)], ksplit=2, shift=5.0, silu=False),
    GCase("xf_ks2_11panels_B1_T257", 1, 257, [(576, 576, 0), (128, 136, 0)], xsegs=[(0, 576, 3, 1, 0), (1, 128, 1, 0, 0)],
          ksplit=2, shift=5.0),
    GCase("xf_rag_k3_B3_T257_shift1", 3, 257, [(128, 128, 0)], xsegs=[(0, 128, 3, 1, 0)], row_len=[513, 255, 257], len_shift=1,
          shift=5.0),
    GCase("xf_rag_ks2_B1_T129_shift3", 1, 129, [(576, 576, 0)], xsegs=[(0, 576, 3, 1, 0)], row_len=[1025], len_shift=3, ksplit=2,
          shift=5.0),
]


def pad128(n):
    return (n + 127) // 128 * 128


def valid_rows(case: GCase, dev) -> torch.Tensor:
    if case.row_len is None:
        return torch.full((case.B,), case.T, dtype=torch.long, device=dev)
    return torch.tensor([min(case.T, ((L - 1) >> case.len_shift) + 1) for L in case.row_len], device=dev)


def build_gemm(case: GCase, dev) -> Dict:
    """Inputs of a case (fp32, on dev) and the pieces both references and the launch need."""
    g = torch.Generator().manual_seed(1000 + case.seed + sum(map(ord, case.name)))
    rn = lambda *s: torch.randn(*s, generator=g)
    B, T = case.B, case.T
    rows_valid = valid_rows(case, "cpu")
    srcs = []
    for C_, ld, extra in case.srcs:
        x = rn(B, T + extra, ld)
        if case.kind in ("lnf", "geglu_lnf"):
            x = x + case.mean_over_std * torch.sign(rn(B, T + extra, 1))
        x[:, :, C_:] = 0.0
        x[:, T:, :] = 0.0
        if case.row_len is not None:                   # producers store zeros past each entry's rows
            for b in range(B):
                x[b, int(rows_valid[b]):] = 0.0
        srcs.append(dict(x=x.to(dev), T=T, C=C_, ld=ld, extra=extra))
    d = dict(srcs=srcs, rows_valid=rows_valid.to(dev))
    # the implicit GEMM's operand, its K layout and the panel transform
    if case.xsegs:
        Cs = sum(srcs[s]["C"] for s, _, _, xf, _ in case.xsegs if xf)
        scale = (0.5 + rn(B, max(Cs, 1)).abs()).to(dev)
        shift = (case.shift + 0.3 * rn(B, max(Cs, 1))).to(dev)
        d.update(scale=scale, shift=shift)
        segs_plain, kb, xargs = [], 0, []
        for si, nch, ntap, xf, aff_c0 in case.xsegs:
            ncb = (nch + 63) // 64
            kb_tap0, stride = kb, (ncb if ntap == 3 else 0)
            xargs.append([si, 0, nch, ntap, kb_tap0, stride, xf, aff_c0])
            kb += ncb * ntap
        d["xargs"] = xargs
        d["nkb"] = kb
    else:
        d["nkb"] = sum((nch + 63) // 64 for _, _, nch, _ in case.segs)
    K = 64 * d["nkb"]
    n_rows = 2 * case.n_valid if case.kind.startswith("geglu") else case.n_valid
    W = (rn(n_rows, K) / math.sqrt(K)).to(dev)
    d.update(W=W, K=K, n_rows=n_rows, N=pad128(n_rows))
    ep = dict(n_valid=case.n_valid, geglu=case.kind.startswith("geglu"), gelu=case.kind == "voc", relu=bool(case.flags & EPI_RELU))
    if case.flags & (EPI_BIAS | EPI_GEGLU) or ep["geglu"]:
        ep["bias"] = (0.1 * rn(n_rows)).to(dev)
    if case.flags & EPI_RESIDUAL:
        d["res_ld"] = case.res_ld or case.n_valid
        d["res_buf"] = rn(B * T, d["res_ld"]).to(dev)
        ep["res"] = d["res_buf"][:, :case.n_valid].reshape(B, T, case.n_valid)
    if case.rowmask:
        ep["rowmask"] = (torch.rand(B, T, generator=g) < 0.7).float().to(dev)
    if case.row_len is not None:
        ep["row_valid"] = torch.arange(T, device=dev)[None, :] < d["rows_valid"][:, None]
    if case.kind in ("lnf", "geglu_lnf"):
        x = srcs[0]["x"][:, :T, :srcs[0]["C"]].to(F64)
        s1, s2 = x.sum(-1), (x * x).sum(-1)
        gamma = (1.0 + 0.2 * rn(srcs[0]["C"])).to(dev)
        Wg = W[:, :srcs[0]["C"]].to(F64) * gamma.to(F64)
        ep.update(lnf=True, ln_g=Wg.sum(-1).float(), ln_stats=torch.stack([s1, s2], -1).reshape(B * T, 2).contiguous(),
                  ln_C=srcs[0]["C"])
        mean = s1 / srcs[0]["C"]
        var = (s2 / srcs[0]["C"] - mean * mean).clamp_min(0)
        ep["ln_mu"], ep["ln_rstd"] = mean, 1.0 / torch.sqrt(var + 1e-5)
        d["gamma"] = gamma
        d["gamma_k"] = torch.nn.functional.pad(gamma, (0, K - gamma.shape[0]), value=1.0)   # cscale of every packed channel
    d["ep"] = ep
    return d


def gemm_operands(case: GCase, d: Dict, exact: bool):
    """[B, T, K] operand (fp64) in the packed K order; panel mode applies the affine first (truth: exact, emulation: fp32)."""
    srcs = d["srcs"]
    if not case.xsegs:
        return ko.im2col([dict(x=s["x"].to(F64), T=s["T"], C=s["C"]) for s in srcs], case.segs, case.T)
    cols, aff = [], 0
    for (si, nch, ntap, xf, aff_c0), xa in zip(case.xsegs, d["xargs"]):
        s = srcs[si]
        x = s["x"][:, :case.T, :s["C"]]
        if xf:
            y = ko.affine_rows(x, d["scale"][:, aff_c0:aff_c0 + s["C"]], d["shift"][:, aff_c0:aff_c0 + s["C"]], case.silu,
                               d["rows_valid"], exact)
        else:
            y = x.to(F64)
        if not exact:                                  # the kernel re-splits the transformed panel: y = hi + lo
            h, l = ko.split_f64(y.float())
            y = h + l
        width = 64 * ((nch + 63) // 64)
        taps = (-1, 0, 1) if ntap == 3 else (0,)
        for t in taps:                                 # tap j's k-blocks sit at kb_tap0 + j * ncb: tap-major per segment
            cols.append(ko.gather(y, case.T, s["C"], 0, width, t, case.T))
    return torch.cat(cols, -1)


def references(case: GCase, d: Dict, drop=None):
    W = d["W"] if "gamma" not in d else (d["W"][:, :d["ep"]["ln_C"]] * d["gamma"]).float()
    if "gamma" in d:
        W = torch.nn.functional.pad(W, (0, d["K"] - W.shape[1]))
    if case.xsegs:
        A_emu = gemm_operands(case, d, exact=False)
        emu, bound = ko.gemm_emulate(A_emu, W, d["ep"], drop, a_split=ko.split_f64(A_emu.float()))
    else:
        A = gemm_operands(case, d, exact=True)
        emu, bound = ko.gemm_emulate(A.float(), W, d["ep"], drop)
    if drop is not None:
        return emu
    extra = None
    if "gamma" in d:                                   # truth: LayerNorm(x) W^T + bias in fp64
        x = d["srcs"][0]["x"][:, :case.T, :d["ep"]["ln_C"]].to(F64)
        xn = (x - d["ep"]["ln_mu"][..., None]) * d["ep"]["ln_rstd"][..., None] * d["gamma"].to(F64)
        A_t = torch.nn.functional.pad(xn, (0, d["K"] - xn.shape[-1]))
        ep_t = dict(d["ep"], lnf=False)
        truth = ko.gemm_truth(A_t, d["W"], ep_t)
        if not case.rule:                              # the split of the UNCENTRED row: 3 * 2^-17 of |x| |gamma W|, times rstd
            Wg = (d["W"][:, :x.shape[-1]].to(F64) * d["gamma"].to(F64)).abs()
            extra = 3 * 2.0 ** -17 * d["ep"]["ln_rstd"][..., None] * (x.abs() @ Wg.T)[..., :case.n_valid]
    else:
        truth = ko.gemm_truth(gemm_operands(case, d, exact=True), d["W"], d["ep"])
    return emu, bound, truth, extra


def gemm_emu_checks(case: GCase, d: Dict):
    emu, bound, truth, extra = references(case, d)
    sens = min(ko.ratio(references(case, d, drop=i) - emu, bound) for i in range(3))
    return emu, bound, truth, extra, sens


def truth_check(name: str, got: torch.Tensor, truth: torch.Tensor, extra: Optional[torch.Tensor]) -> float:
    """the parity rule, or (where the design's own error terms exceed it: `extra`) the rule plus those terms; returns the
    rule's ratio"""
    r_rule = ko.rule_ratio(got, truth)
    if extra is None:
        assert r_rule <= 1.0, f"{name}: vs truth {r_rule:.3f} of the rule"
    else:
        r = ko.ratio(got.to(F64) - truth, ko.rule_tol(truth) + extra)
        assert r <= 1.0, f"{name}: vs truth {r:.3f} of the rule plus the design's error terms (rule alone: {r_rule:.3f})"
    return r_rule


@pytest.mark.parametrize("case", GEMM_CASES, ids=lambda c: c.name)
def test_gemm_emulation_meets_truth(case):
    """The precision design alone (no kernel): the documented roundings stay inside the parity rule, and the bound is sensitive."""
    d = build_gemm(case, "cpu")
    emu, bound, truth, extra, sens = gemm_emu_checks(case, d)
    truth_check(case.name + " emulation", emu, truth, extra)
    assert sens >= SENSITIVITY, f"{case.name}: a dropped product moves the result by only {sens:.1f} x tol_emu"


def launch_gemm(case: GCase, d: Dict, poison: bool, ksplit: Optional[int] = None, only: Optional[int] = None):
    """One launch; returns the outputs.  poison: NaN in the never-read rows / channels of the sources.  only: run batch entry
    `only` alone (its own rows, B = 1)."""
    dev = d["W"].device
    B = case.B if only is None else 1
    bsel = slice(None) if only is None else slice(only, only + 1)
    args = GemmArgs()
    args.B, args.T_out = B, case.T
    keep = []
    for i, s in enumerate(d["srcs"]):
        x = s["x"][bsel].clone()
        if poison:
            x[:, :, s["C"]:] = float("nan")
            x[:, case.T:, :] = float("nan")
        hi, lo = ko.split(x)
        keep += [hi, lo]
        args.src[i] = Split(hi.data_ptr(), lo.data_ptr(), case.T, s["C"], s["ld"], (case.T + s["extra"]) * s["ld"] if s["extra"] else 0)
    args.nsrc = len(d["srcs"])
    for i, sg in enumerate(case.segs):
        args.seg[i] = (C.c_int * 4)(*sg)
    args.nseg = len(case.segs)
    for i, xa in enumerate(d.get("xargs", [])):
        args.xseg[i] = (C.c_int * 8)(*xa)
    args.nxs = len(case.xsegs)
    wh = torch.zeros(d["nkb"] * d["N"] * 64, dtype=torch.bfloat16, device=dev)
    wl = torch.zeros_like(wh)
    _lib.check(_lib.lib().ns2vc_check_pack_b(d["W"].data_ptr(), d["n_rows"], d["K"], 1, 0, 0, d["K"], 0, 0,
                                             case.n_valid if case.kind.startswith("geglu") else 0, ptr(d.get("gamma_k")),
                                             wh.data_ptr(), wl.data_ptr(), d["N"], d["nkb"], stream()))
    args.w_hi, args.w_lo, args.N, args.n_valid, args.nkb_w = wh.data_ptr(), wl.data_ptr(), d["N"], case.n_valid, d["nkb"]
    flags = case.flags | (EPI_GEGLU if case.kind.startswith("geglu") else 0) | (EPI_LNFOLD if "lnf" in case.kind else 0)
    args.flags = flags
    ep = d["ep"]
    M = B * case.T
    out = {}
    if "bias" in ep:
        args.bias = ep["bias"].data_ptr()
    if flags & EPI_RESIDUAL:
        res = d["res_buf"].reshape(case.B, case.T, -1)[bsel].contiguous()
        keep.append(res)
        args.res, args.res_ld = res.data_ptr(), d["res_ld"]
    out_ld = case.out_ld or case.n_valid
    if flags & EPI_OUT_NCT:
        out["nct"] = torch.full((B, case.n_valid, case.T), float("nan"), device=dev)
        args.out = out["nct"].data_ptr()
    if flags & EPI_OUT_F32:
        out["f32"] = torch.full((M, out_ld), float("nan"), device=dev)
        args.out, args.out_ld = out["f32"].data_ptr(), out_ld
    if flags & EPI_OUT_SPLIT:
        sld = (case.n_valid + 7) // 8 * 8
        out["hi"] = torch.zeros(M, sld, dtype=torch.int16, device=dev)
        out["lo"] = torch.zeros_like(out["hi"])
        args.out_hi, args.out_lo, args.out_split_ld = out["hi"].data_ptr(), out["lo"].data_ptr(), sld
    args.f16_col0 = case.f16_col0
    if ep.get("lnf"):
        lns = ep["ln_stats"].reshape(case.B, case.T, 2)[bsel].reshape(M, 2).contiguous()
        keep.append(lns)
        args.ln_stats, args.ln_g, args.ln_C, args.ln_eps = lns.data_ptr(), ep["ln_g"].data_ptr(), ep["ln_C"], 1e-5
    if flags & EPI_ROWSTATS:
        out["row_stats"] = torch.zeros(M, 2, dtype=F64, device=dev)
        args.row_stats = out["row_stats"].data_ptr()
    if flags & EPI_STATS:
        out["stat_sum"] = torch.zeros(B, case.n_valid, dtype=F64, device=dev)
        out["stat_sq"] = torch.zeros_like(out["stat_sum"])
        args.stat_sum, args.stat_sq = out["stat_sum"].data_ptr(), out["stat_sq"].data_ptr()
    if "rowmask" in ep:
        rm = ep["rowmask"][bsel].contiguous()
        keep.append(rm)
        args.rowmask = rm.data_ptr()
    if case.row_len is not None:
        rl = torch.tensor(case.row_len, dtype=torch.int32, device=dev)[bsel].contiguous()
        keep.append(rl)
        args.row_len, args.len_shift = rl.data_ptr(), case.len_shift
    if case.xsegs:
        sc, sh = d["scale"][bsel].contiguous(), d["shift"][bsel].contiguous()
        keep += [sc, sh]
        args.pre_scale, args.pre_shift, args.pre_mode, args.pre_C = sc.data_ptr(), sh.data_ptr(), 2 if case.silu else 1, sc.shape[1]
    args.ksplit = ksplit or case.ksplit
    desc = call(_lib.lib().ns2vc_check_gemm, args)
    torch.cuda.synchronize()
    out["desc"] = desc
    return out


def logical(case: GCase, out: Dict, B: int) -> torch.Tensor:
    if "nct" in out:
        return out["nct"].transpose(1, 2)
    return out["f32"][:, :case.n_valid].reshape(B, case.T, case.n_valid)


EXPECT_DESC = {"plain": "gemm_tc<64,LNF=0,XF=0,ENC=0,RAG={rag},VOC=0>", "lnf": "gemm_tc<64,LNF=1,XF=0,ENC=0,RAG=0,VOC=0>",
               "geglu": "gemm_tc<128,LNF=0,XF=0,ENC=0,RAG=0,VOC=0>", "geglu_lnf": "gemm_tc<128,LNF=1,XF=0,ENC=0,RAG=0,VOC=0>",
               "enc": "gemm_tc<64,LNF=0,XF=0,ENC=1,RAG=0,VOC=0>", "voc": "gemm_tc<64,LNF=0,XF=0,ENC=0,RAG=0,VOC=1>"}


@gpu
@pytest.mark.parametrize("case", GEMM_CASES, ids=lambda c: c.name)
def test_gemm_kernel(case):
    dev = torch.device("cuda")
    d = build_gemm(case, dev)
    emu, bound, truth, extra, sens = gemm_emu_checks(case, d)
    assert sens >= SENSITIVITY, f"{case.name}: tol_emu is not sensitive to a dropped product ({sens:.1f})"
    clean = launch_gemm(case, d, poison=False)
    got_o = launch_gemm(case, d, poison=True)
    want = EXPECT_DESC[case.kind].format(rag=int(case.row_len is not None))
    if case.xsegs:
        want = f"gemm_tc<64,LNF=0,XF=1,ENC=0,RAG={int(case.row_len is not None)},VOC=0>"
    assert got_o["desc"] == want, (case.name, got_o["desc"])
    got = logical(case, got_o, case.B)
    # never-read NaN changes nothing, and two launches agree bit for bit (statistics: fp64 atomics in any order)
    for k in ("f32", "nct", "hi", "lo"):
        if k in got_o:
            assert torch.equal(got_o[k].view(torch.int32 if got_o[k].dtype == torch.float32 else got_o[k].dtype),
                               clean[k].view(torch.int32 if clean[k].dtype == torch.float32 else clean[k].dtype)), f"{case.name}: {k} differs"
    g64 = got.to(F64)
    r_emu = ko.ratio(g64 - emu, bound)
    assert r_emu <= 1.0, f"{case.name}: |gpu - emu| reaches {r_emu:.2f} x tol_emu"
    r_truth = truth_check(case.name, got, truth, extra)
    fam = got_o["desc"]
    record(fam, emu_ratio=r_emu, truth_ratio=r_truth, sens_margin=sens)
    # exact zeros: rows past row_len / zero row mask; columns past n_valid untouched (fp32 output)
    if case.row_len is not None:
        assert (got[~d["ep"]["row_valid"]] == 0).all(), f"{case.name}: rows past row_len not zero"
    if "rowmask" in d["ep"]:
        assert (got[d["ep"]["rowmask"] == 0] == 0).all(), f"{case.name}: masked rows not zero"
    if "f32" in got_o and got_o["f32"].shape[1] > case.n_valid:
        assert got_o["f32"][:, case.n_valid:].isnan().all(), f"{case.name}: columns past n_valid written"
    # split output bit-consistent with the fp32 output of the same launch
    if "hi" in got_o and "f32" in got_o:
        v = got_o["f32"][:, :case.n_valid]
        f16 = torch.arange(case.n_valid, device=dev) >= (case.f16_col0 if case.f16_col0 >= 0 else 1 << 30)
        hb, lb = ko.split(v, torch.bfloat16)
        hf, lf = ko.split(v, torch.float16)
        want_hi = torch.where(f16, hf.view(torch.int16), hb.view(torch.int16))
        want_lo = torch.where(f16, lf.view(torch.int16), lb.view(torch.int16))
        assert torch.equal(got_o["hi"][:, :case.n_valid], want_hi) and torch.equal(got_o["lo"][:, :case.n_valid], want_lo), \
            f"{case.name}: split output is not the split of the fp32 output"
    # statistics of the kernel's own fp32 output: fp32 partial sums of 32 values, then fp64
    u = 2.0 ** -24
    if "row_stats" in got_o:
        v = g64.reshape(-1, case.n_valid)
        for j, f in enumerate((lambda z: z, lambda z: z * z)):
            ref, mag = f(v).sum(-1), f(v).abs().sum(-1)
            assert ((got_o["row_stats"][:, j] - ref).abs() <= 33 * u * mag + 1e-12 * ref.abs()).all(), f"{case.name}: row statistics"
    if "stat_sum" in got_o:
        for key, f in (("stat_sum", lambda z: z), ("stat_sq", lambda z: z * z)):
            ref, mag = f(g64).sum(1), f(g64).abs().sum(1)
            assert ((got_o[key] - ref).abs() <= 33 * u * mag + 1e-12 * ref.abs()).all(), f"{case.name}: {key}"
    # ragged rows equal the entry run alone
    if case.row_len is not None and case.ksplit == 1:
        for b in range(case.B):
            alone = logical(case, launch_gemm(case, d, poison=False, only=b), 1)[0]
            assert torch.equal(alone.view(torch.int32), got[b].view(torch.int32)), f"{case.name}: entry {b} differs from its run alone"
    # split-K: the same tile with one CTA is checked against the references too; bit-identity is not part of the design
    if case.ksplit == 2:
        one = logical(case, launch_gemm(case, d, poison=False, ksplit=1), case.B)
        r1 = ko.ratio(one.to(F64) - emu, bound)
        assert r1 <= 1.0, f"{case.name}: ksplit = 1 reaches {r1:.2f} x tol_emu"
        print(f"{case.name}: ksplit 2 vs 1 bit-identical: {torch.equal(one.view(torch.int32), got.view(torch.int32))}")


@gpu
def test_gemm_invalid_combinations_are_errors():
    case = next(c for c in GEMM_CASES if c.name.startswith("xf_k3_ks1"))
    d = build_gemm(case, torch.device("cuda"))
    with pytest.raises(_lib.Ns2vcError, match="ksplit must be 1 or 2"):
        launch_gemm(case, d, poison=False, ksplit=3)
    bad = GCase("bad", 1, 16, [(64, 64, 0)], [(0, 0, 64, 0)], kind="voc", flags=EPI_GELU | EPI_RELU | EPI_OUT_F32)
    with pytest.raises(_lib.Ns2vcError, match="GELU epilogue"):
        launch_gemm(bad, build_gemm(bad, torch.device("cuda")), poison=False)
    rag_lnf = GCase("bad2", 1, 16, [(64, 64, 0)], [(0, 0, 64, 0)], kind="lnf", row_len=[16], flags=EPI_BIAS | EPI_OUT_F32)
    with pytest.raises(_lib.Ns2vcError, match="ragged row masks"):
        launch_gemm(rag_lnf, build_gemm(rag_lnf, torch.device("cuda")), poison=False)


@gpu
@pytest.mark.parametrize("variant", ["k3_tap1", "geglu_half64", "cscale_cin0"])
def test_pack_b_layout(variant):
    """Unswizzled packed images equal bf16(w) and bf16(w - bf16(w)) at their documented places."""
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(7)
    if variant == "k3_tap1":
        n_rows, cin, ktaps, tap, cin0, ncin, geglu, cs = 100, 100, 3, 1, 0, 100, 0, None
    elif variant == "geglu_half64":
        n_rows, cin, ktaps, tap, cin0, ncin, geglu, cs = 256, 64, 1, 0, 0, 64, 128, None
    else:
        n_rows, cin, ktaps, tap, cin0, ncin, geglu, cs = 128, 200, 1, 0, 72, 100, 0, torch.randn(200, generator=g)
    w = torch.randn(n_rows, cin, ktaps, generator=g)
    Npad, nkb, kb0, n_dst0 = pad128(n_rows + 5), 4, 1, 5
    wh = torch.zeros(nkb * Npad * 64, dtype=torch.bfloat16, device=dev)
    wl = torch.zeros_like(wh)
    w_dev, cs_dev = w.to(dev).contiguous(), None if cs is None else cs.to(dev)     # (alive until the packing has run)
    _lib.check(_lib.lib().ns2vc_check_pack_b(w_dev.data_ptr(), n_rows, cin, ktaps, tap, cin0, ncin, n_dst0, kb0, geglu, ptr(cs_dev),
                                             wh.data_ptr(), wl.data_ptr(), Npad, nkb, stream()))
    torch.cuda.synchronize()
    # unswizzle: element (kb, n, kk) at ((kb * Npad + n) * 64 + (((kk >> 3) ^ (n & 7)) << 3) + (kk & 7))
    kb, n, kk = torch.meshgrid(torch.arange(nkb), torch.arange(Npad), torch.arange(64), indexing="ij")
    idx = ((kb * Npad + n) * 64 + ((((kk >> 3) ^ (n & 7)) << 3) + (kk & 7))).reshape(-1)
    Hi, Lo = wh.cpu()[idx].reshape(nkb, Npad, 64), wl.cpu()[idx].reshape(nkb, Npad, 64)
    src = w[:, :, tap].clone()
    if cs is not None:
        src = src * cs
    src = src[:, cin0:cin0 + ncin]
    if geglu:
        blocks = [torch.cat([src[64 * j:64 * j + 64], src[geglu + 64 * j:geglu + 64 * j + 64]]) for j in range(geglu // 64)]
        src = torch.cat(blocks)
    want = torch.zeros(nkb, Npad, 64)
    nk = (ncin + 63) // 64
    full = torch.zeros(n_rows, nk * 64)
    full[:, :ncin] = src
    want[kb0:kb0 + nk, n_dst0:n_dst0 + n_rows] = full.reshape(n_rows, nk, 64).transpose(0, 1)
    hi, lo = ko.split(want)
    assert torch.equal(Hi.view(torch.int16), hi.view(torch.int16)) and torch.equal(Lo.view(torch.int16), lo.view(torch.int16)), variant


# ---------------------------------------------------------------------------------------------------------------------------
# Attention cases
# ---------------------------------------------------------------------------------------------------------------------------
@dataclass
class ACase:
    name: str
    dh: int
    Tq: int
    Tk: int
    B: int = 2
    H: int = 2
    mode: str = "f16"                 # f16 | split (v2), v1
    bias: str = "none"                # none | mask10000 | neginf (trailing keys) | random
    key_len: Optional[List[int]] = None
    key_shift: int = 0
    std: float = 1.0                  # score std (log-space of softmax, natural units)
    v_rms: float = 1.0
    fused: bool = False               # q | k | v in one split buffer (Tq == Tk)
    odd_out_ld: bool = False
    q_ld_pad: int = 0                 # v1: q row pitch dh*H + pad (unaligned: the scalar load path)
    sharp: bool = False               # the truth check adds the design's score-rounding term (fp16 weights: always)
    seed: int = 0


ATTN_CASES = [
    ACase("v2_dh16_Tq129_Tk768_mask10000_std4_f16", 16, 129, 768, bias="mask10000", std=4.0),
    ACase("v2_dh32_Tq1000_Tk1024_std8_f16", 32, 1000, 1024, B=1, std=8.0),
    ACase("v2_dh48_T257_fused_neginf_split_oddld", 48, 257, 257, bias="neginf", mode="split", fused=True, odd_out_ld=True, std=4.0),
    ACase("v2_dh64_Tq128_Tk256_keylen_f16_vrms1e-3", 64, 128, 256, B=4, key_len=[256, 1, 65, 128], v_rms=1e-3),
    ACase("v2_dh64_Tq127_Tk1024_keylen_shift3_split", 64, 127, 1024, B=3, key_len=[8192, 513, 1017], key_shift=3, mode="split", std=4.0),
    ACase("v2_dh16_Tq1_Tk1_split_vrms1e4", 16, 1, 1, mode="split", v_rms=1e4),
    ACase("v2_dh32_Tq2_Tk63_random_bias_f16", 32, 2, 63, bias="random"),
    ACase("v2_dh48_Tq128_Tk65_f16_vrms1e4_std2", 48, 128, 65, v_rms=1e4, std=2.0),
    ACase("v2_dh16_Tq255_Tk767_keylen_shift1_f16", 16, 255, 767, B=2, key_len=[1533, 127], key_shift=1, std=2.0),
    ACase("v1_dh8_Tq129_Tk769_mask10000", 8, 129, 769, mode="v1", bias="mask10000", std=4.0),
    ACase("v1_dh24_Tq127_Tk1025_mask10000_qld_unaligned", 24, 127, 1025, mode="v1", bias="mask10000", q_ld_pad=1, std=2.0),
    ACase("v1_dh40_Tq1_Tk1100_random_bias", 40, 1, 1100, mode="v1", bias="random"),
    ACase("v1_dh64_Tq128_Tk64_nobias_std8", 64, 128, 64, mode="v1", std=8.0, sharp=True),
    # the models' mild scores over few keys: many bf16 hi/lo weights near a rounding boundary of their lo half, where the
    # kernel's weight and the emulation's may split apart (the programs' launches found it: tests/test_program_launches_fp64.py)
    ACase("v2_dh64_Tq256_Tk9_std0.05_split", 64, 256, 9, B=1, H=8, mode="split", std=0.05),
    ACase("v1_dh16_Tq256_Tk11_std0.1", 16, 256, 11, B=1, H=8, mode="v1", std=0.1),
]


def eff_keys(case: ACase) -> List[int]:
    if case.key_len is None:
        return [case.Tk] * case.B
    return [min(case.Tk, ((L - 1) >> case.key_shift) + 1) for L in case.key_len]


def build_attn(case: ACase, dev):
    g = torch.Generator().manual_seed(2000 + case.seed + sum(map(ord, case.name)))
    rn = lambda *s: torch.randn(*s, generator=g)
    B, H, dh = case.B, case.H, case.dh
    a = math.sqrt(case.std)                           # q . k / sqrt(dh) with q, k ~ N(0, a^2): std a^2
    u = rn(dh)
    u = u / u.norm()
    q = a * rn(B, H, case.Tq, dh) + 2 * a * u
    k = a * rn(B, H, case.Tk, dh)
    nk = eff_keys(case)
    for b in range(B):                               # the largest score in the last valid tile: the running max moves late
        last = nk[b] - 1 - (100 if case.bias == "mask10000" and case.Tk > 200 else 0)
        last = max(last, 0)
        k[b, :, last] = 3 * case.std * math.sqrt(dh) / (2 * a) * u
    v = case.v_rms * rn(B, H, case.Tk, dh)
    bias = None
    if case.bias == "mask10000":
        bias = torch.zeros(B, case.Tk)
        bias[:, max(1, case.Tk - 100):] = -10000.0
    elif case.bias == "neginf":
        bias = torch.zeros(B, case.Tk)
        bias[0, case.Tk - 37:] = float("-inf")
        bias[-1, case.Tk // 2:] = float("-inf")
    elif case.bias == "random":
        bias = 2.0 * rn(B, case.Tk)
    t = lambda x: None if x is None else x.to(dev)
    return dict(q=t(q), k=t(k), v=t(v), bias=t(bias), nkeys=nk, scale=1.0 / math.sqrt(dh))


def attn_refs(case: ACase, d: Dict, drop=None, mask_defect=False):
    nk, bias = list(d["nkeys"]), d["bias"]
    if mask_defect:
        if bias is not None and (bias < -1000).any():   # the first masked key unmasked
            bias = bias.clone()
            for b in range(bias.shape[0]):
                idx = (bias[b] < -1000).nonzero()
                if len(idx):
                    bias[b, idx[0, 0]] = 0.0
        else:
            nk = [n - 1 if n > 1 else n + 1 for n in nk]
    q, k, v = d["q"], d["k"], d["v"]
    if mask_defect and max(nk) > k.shape[2]:          # one key past the end: the zeros the kernel's tail tile holds
        k = torch.nn.functional.pad(k, (0, 0, 0, 1))
        v = torch.nn.functional.pad(v, (0, 0, 0, 1))
        if bias is not None:
            bias = torch.nn.functional.pad(bias, (0, 1))
    return ko.attention_emulate(q, k, v, d["scale"], bias, nk, case.mode, drop)


def attn_sensitivity(case: ACase, d: Dict, emu, bound) -> float:
    devs = [attn_refs(case, d, mask_defect=True)[0]]
    if case.std >= 2:
        devs += [attn_refs(case, d, drop=i)[0] for i in range(3)]
    return min(ko.ratio(x - emu, bound) for x in devs)


def attn_truth(case: ACase, d: Dict):
    truth = ko.attention_truth(d["q"], d["k"], d["v"], d["scale"], d["bias"], d["nkeys"])
    extra = None
    if case.mode == "f16" or case.sharp:
        extra = ko.attention_design_terms(d["q"], d["k"], d["v"], d["scale"], d["bias"], d["nkeys"], truth, case.mode == "f16")
    return truth, extra


@pytest.mark.parametrize("case", ATTN_CASES, ids=lambda c: c.name)
def test_attention_emulation_meets_truth(case):
    d = build_attn(case, "cpu")
    emu, bound = attn_refs(case, d)
    truth, extra = attn_truth(case, d)
    truth_check(case.name + " emulation", emu, truth, extra)
    sens = attn_sensitivity(case, d, emu, bound)
    assert sens >= SENSITIVITY, f"{case.name}: a defect moves the result by only {sens:.1f} x tol_emu"


def _split_tokens(x: torch.Tensor, dt) -> torch.Tensor:
    """[B, H, T, dh] fp32 -> token-major [B, T, H dh] 16-bit hi, lo (as int16 views)"""
    B, H, T, dh = x.shape
    hi, lo = ko.split(x.permute(0, 2, 1, 3).reshape(B, T, H * dh), dt)
    return hi.view(torch.int16), lo.view(torch.int16)


def launch_attn(case: ACase, d: Dict, poison: bool):
    dev = d["q"].device
    B, H, dh, Tq, Tk = case.B, case.H, case.dh, case.Tq, case.Tk
    HD = H * dh
    args = AttnArgs()
    args.B, args.H, args.Tq, args.Tk, args.dh, args.scale = B, H, Tq, Tk, dh, d["scale"]
    keep = []
    nk = d["nkeys"]
    if case.mode == "v1":
        args.v2 = 0
        qld = HD + case.q_ld_pad
        qb = torch.zeros(B, Tq, qld, device=dev)
        qb[..., :HD] = d["q"].permute(0, 2, 1, 3).reshape(B, Tq, HD)
        kv = torch.cat([d["k"], d["v"]], 1).permute(0, 2, 1, 3).reshape(B, Tk, 2 * HD).contiguous()   # one [k | v] cache
        if poison:
            qb[..., HD:] = float("nan")
        keep += [qb, kv]
        args.q, args.q_ld, args.k, args.k_ld, args.v, args.v_ld = qb.data_ptr(), qld, kv.data_ptr(), 2 * HD, kv.data_ptr() + 4 * HD, 2 * HD
    else:
        args.v2 = 1
        vdt = torch.float16 if case.mode == "f16" else torch.bfloat16
        parts = [_split_tokens(d["q"], torch.bfloat16), _split_tokens(d["k"], torch.bfloat16), _split_tokens(d["v"], vdt)]
        if case.fused:
            ld = 3 * HD + 8
            hi = torch.zeros(B, Tq, ld, dtype=torch.int16, device=dev)
            lo = torch.zeros_like(hi)
            for i, (h, l) in enumerate(parts):
                hi[..., i * HD:(i + 1) * HD], lo[..., i * HD:(i + 1) * HD] = h, l
            if poison:                                # channels >= C inside ld: NaN
                hi[..., 3 * HD:], lo[..., 3 * HD:] = 0x7fc0, 0x7fc0
            keep += [hi, lo]
            sp = Split(hi.data_ptr(), lo.data_ptr(), Tq, 3 * HD, ld, 0)
            args.qs = args.ks = args.vs = sp
            args.q_c0, args.k_c0, args.v_c0 = 0, HD, 2 * HD
        else:
            sps = []
            for i, (h, l) in enumerate(parts):
                T_ = Tq if i == 0 else Tk
                ld = HD + 8
                hb = torch.zeros(B, T_, ld, dtype=torch.int16, device=dev)
                lb = torch.zeros_like(hb)
                hb[..., :HD], lb[..., :HD] = h, l
                if poison:
                    hb[..., HD:], lb[..., HD:] = 0x7fc0, 0x7fc0
                    if i > 0 and case.key_len is not None:
                        for b in range(B):                     # keys past the entry's count: NaN in tiles never loaded,
                            n = nk[b]                          # NaN K / large finite V inside the last loaded tile
                            tail = min(Tk, (n + 63) // 64 * 64)
                            if i == 1:
                                hb[b, n:], lb[b, n:] = 0x7fc0, 0x7fc0
                            else:
                                big = 0x7bff if case.mode == "f16" else 0x7149     # 65504 (fp16) / 1e30 (bf16)
                                hb[b, n:tail], lb[b, n:tail] = big, 0
                                hb[b, tail:], lb[b, tail:] = 0x7fc0, 0x7fc0
                keep += [hb, lb]
                sps.append(Split(hb.data_ptr(), lb.data_ptr(), T_, HD, ld, 0))
            args.qs, args.ks, args.vs = sps
        args.p_split = 1 if case.mode == "split" else 0
        if case.key_len is not None:
            kl = torch.tensor(case.key_len, dtype=torch.int32, device=dev)
            keep.append(kl)
            args.key_len, args.key_shift = kl.data_ptr(), case.key_shift
    if d["bias"] is not None:
        args.bias = d["bias"].data_ptr()
    out_ld = HD + (1 if case.odd_out_ld else 0)
    out = torch.full((B, Tq, out_ld), float("nan"), device=dev)
    sld = HD + (1 if case.odd_out_ld else 0)
    hi_o = torch.zeros(B, Tq, sld, dtype=torch.int16, device=dev)
    lo_o = torch.zeros_like(hi_o)
    args.out, args.out_ld = out.data_ptr(), out_ld
    args.out_hi, args.out_lo, args.out_split_ld = hi_o.data_ptr(), lo_o.data_ptr(), sld
    desc = call(_lib.lib().ns2vc_check_attention, args)
    torch.cuda.synchronize()
    return dict(out=out, hi=hi_o, lo=lo_o, desc=desc)


def fp16_p_selected() -> bool:
    return not os.environ.get("NS2VC_ATTN_P", "").startswith("s")


def expected_attn_desc(case: ACase) -> str:
    if case.mode == "v1":
        return f"attn_tc<{16 * ((case.dh + 15) // 16)}>"
    pb = {16: 32, 32: 64}.get(case.dh, 128)
    return (f"attn_v2<{case.dh},PB={pb},BIAS={int(case.bias != 'none')},PF16={int(case.mode == 'f16')},"
            f"RAGK={int(case.key_len is not None)}>")


@gpu
@pytest.mark.parametrize("case", ATTN_CASES, ids=lambda c: c.name)
def test_attention_kernel(case):
    if case.mode == "f16" and not fp16_p_selected():
        pytest.skip("NS2VC_ATTN_P selects bf16 hi/lo softmax weights: the fp16-weight kernel is not launched")
    dev = torch.device("cuda")
    d = build_attn(case, dev)
    emu, bound = attn_refs(case, d)
    sens = attn_sensitivity(case, d, emu, bound)
    assert sens >= SENSITIVITY, f"{case.name}: tol_emu is not sensitive ({sens:.1f})"
    truth, extra = attn_truth(case, d)
    clean = launch_attn(case, d, poison=False)
    res = launch_attn(case, d, poison=True)
    assert res["desc"] == expected_attn_desc(case), (case.name, res["desc"])
    for key in ("out", "hi", "lo"):
        assert torch.equal(res[key].view(torch.int32) if key == "out" else res[key],
                           clean[key].view(torch.int32) if key == "out" else clean[key]), f"{case.name}: never-read NaN changed {key}"
    B, H, dh, HD = case.B, case.H, case.dh, case.H * case.dh
    out = res["out"][..., :HD]
    if case.odd_out_ld:
        assert res["out"][..., HD:].isnan().all(), f"{case.name}: wrote past the heads"
    got = out.reshape(B, case.Tq, H, dh).permute(0, 2, 1, 3).to(F64)
    r_emu = ko.ratio(got - emu, bound)
    assert r_emu <= 1.0, f"{case.name}: |gpu - emu| reaches {r_emu:.2f} x tol_emu"
    r_truth = truth_check(case.name, got, truth, extra)
    hb, lb = ko.split(out, torch.bfloat16)
    assert torch.equal(res["hi"][..., :HD], hb.view(torch.int16)) and torch.equal(res["lo"][..., :HD], lb.view(torch.int16)), \
        f"{case.name}: split output is not the split of the fp32 output"
    record(res["desc"].split("<")[0] + ("_f16" if case.mode == "f16" else "_split" if case.mode == "split" else ""),
           emu_ratio=r_emu, truth_ratio=r_truth, sens_margin=sens)


@gpu
def test_attention_invalid_combinations_are_errors():
    case = ACase("bad", 16, 64, 769, B=1, H=1, bias="mask10000")
    d = build_attn(case, torch.device("cuda"))
    with pytest.raises(_lib.Ns2vcError, match="staged-bias capacity"):
        launch_attn(case, d, poison=False)
    case2 = ACase("bad2", 16, 64, 64, B=1, H=1, bias="random", key_len=[64])
    with pytest.raises(_lib.Ns2vcError, match="per-entry key counts take no additive bias"):
        launch_attn(case2, build_attn(case2, torch.device("cuda")), poison=False)


_TWO_DEVICES = r"""
import sys, torch
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + '/tests')
import test_kernels_fp64 as t
front = []
for dev in (0, 1):
    with torch.cuda.device(dev):
        gc = t.GEMM_CASES[0]
        t.launch_gemm(gc, t.build_gemm(gc, torch.device('cuda', dev)), poison=False)
        ac = t.ATTN_CASES[5]
        t.launch_attn(ac, t.build_attn(ac, torch.device('cuda', dev)), poison=False)
        ac = t.ATTN_CASES[12]
        t.launch_attn(ac, t.build_attn(ac, torch.device('cuda', dev)), poison=False)
        a = __import__('test_audio_kernels_fp64'); a.launch_istft((2048, 2, 0), a.build_istft((2048, 2, 0)), torch.device('cuda', dev))
        f = __import__('test_frontend_kernels_fp64'); sp = torch.randn(4000, generator=torch.Generator().manual_seed(0))
        rc = f.RES_CASES[13]; front.append(f.launch_res(rc, f.build_res(rc, sp), torch.device('cuda', dev)).cpu())
        mc = f.MEL_CASES[1]; front.append(f.launch_mel(mc, f.build_mel(mc, sp), torch.device('cuda', dev), f.MelHandle(mc)).cpu())
# each handle reads the tables of its own device: device 1's front-end outputs equal device 0's bit for bit
assert torch.equal(front[0], front[2]) and torch.equal(front[1], front[3])
print('ok')
"""


@gpu
def test_launchers_on_two_devices_in_one_process():
    """The launchers set each kernel's dynamic shared-memory attribute once per process; CUDA keeps it per device.  The front
    end's resampler and log-mel handles keep their tables on the device they were created on."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    r = subprocess.run([sys.executable, "-c", _TWO_DEVICES, REPO], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout + r.stderr
