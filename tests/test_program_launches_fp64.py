"""Every wgmma GEMM and flash-attention launch of the engines' real programs, each on the input the earlier launches left in
memory, against the references of tests/test_kernels_fp64.py.

The hand cases of test_kernels_fp64.py build their descriptors themselves, at the shapes and edges the models never reach.
Here the descriptors are the ones the engines' builders chose: an observer on the run loops (ns2vc_check_set_launch_hook)
stops before and after every launch of one ordinary engine call, with the stream synchronised, and hands over the launch's
record as bound to the call's arguments (the flat ns2vc_check_gemm_args / ns2vc_check_attn_args and the instantiation string).
Before a GEMM or attention launch the test copies out what it reads (the source splits, the residual, row bias, LayerNorm
statistics, GroupNorm sums, FiLM rows, q / k / v and the key counts, and the statistics buffers it accumulates into); after
it, what it wrote (fp32 output, the hi / lo split with its fp16 columns, the column and row statistics).  Then:

* emulation: ko.gemm_emulate / ko.attention_emulate on the launch's own split operands and its packed weight split (read
  from the launch's weight pointers and unswizzled as pack_oracle.unswizzle does), |gpu - emu| <= tol_emu elementwise.  A
  panel GroupNorm is emulated as the kernel computes it (mean and rstd from the producers' fp64 sums, the per-channel affine
  in fp32, one rounding of the fma, one of the SiLU, re-split) and tol_emu adds 8 * 2^-24 (|x a| + |b| + |beta (1 + s)|) of
  each panel element carried by |W| (rsqrtf and the order of the affine's fp32 products are not bit-faithful).  The running
  accumulator term of tol_emu follows the panel loop's order of K (segments, then channel blocks, then taps).  A split-only
  output is compared as hi + lo, with 2^-16 |emu| more (the split's own rounding, 2^-24 more for fp16 columns).  Column and
  row statistics (what the launch added to its buffers) equal fp64 sums of the launch's own fp32 output within 33 * 2^-24 of
  the sum of magnitudes (fp32 partial sums of 32 values; 2^-16 more of it when the output is read back from its split);
* truth: the launch's operation in fp64 on its fp32 inputs (hi + lo of every split, the packed weights' hi + lo, the
  GroupNorm from the same sums in fp64) under the parity rule 1e-3 |ref| + 1e-4 rms(ref).  Where the design's own terms
  exceed the rule, the rule plus those terms, as truth_check does: the attention's fp16 weights and score rounding
  (ko.attention_design_terms), and for a folded LayerNorm the fp32 accumulation of its uncentred rows (tol_emu).  The truth
  operand of a folded LayerNorm is the launch's own split, so there the truth differs from the emulation only by the dropped
  lo x lo product, and the check adds little to the emulation's: its rule ratio is printed for information (it reaches 46 x
  the rule under the ln_offset weights);
* exact zeros in rows past a ragged row's length and in rows the row mask drops.

Not vacuous: for every instantiation signature, the emulation of its first launch in each program is rerun with each of the
three split products dropped, and each drop must move it by more than tol_emu.  Nothing is skipped: after each engine call the
launches the observer saw (tap copies aside) equal the engine's own launch count of that run (<engine>_launch_count, kept by
the run loop whether or not an observer is set), and every GEMM and attention launch seen is checked.  The observed call's
output is bit-identical to an unobserved call on the same inputs.  Each program prints a table: signature, launches, worst
ratios.

Programs stepped through: the denoiser's prepare_cond, forward and forward_film (on the rows of ns2vc_unet_time_table, the
forward the sampling loops replay) at shapes A-D of test_numerics_fp64.py under their weight regimes, the same three for the
ragged program R1 and for the tiny configuration; the condition encoders' infer and per-utterance infer under the synthetic
and sharp weights of test_pre_model_ragged.py; ContentVec's extract and Vocos' decode under each of their regimes.  Not
stepped through: the denoiser's prepare_cond_rows, the condition encoders' encode_voices / infer_content programs, and the
graph-captured sampling loops (which replay the forward_film program above).
"""
from __future__ import annotations

import ctypes as C
from collections import defaultdict
from typing import Dict, Optional

import pytest
import torch

from ns2vc_b200 import _lib
from ns2vc_b200.synth import CONTENTVEC_REGIMES, VOCOS_REGIMES
from oracle import kernel_oracle as ko
from oracle import pack_oracle as po
from test_kernels_fp64 import (EPI_BIAS, EPI_GEGLU, EPI_GELU, EPI_LNFOLD, EPI_OUT_F32, EPI_OUT_NCT, EPI_OUT_SPLIT, EPI_RELU,
                               EPI_RESIDUAL, EPI_ROWBIAS, EPI_ROWMASK, EPI_ROWSTATS, EPI_STATS, AttnArgs, GemmArgs, Split,
                               truth_check)
from test_numerics_fp64 import CASES as DENOISER_CASES     # shapes A-D of the block-level tests and their weight regimes

F64 = torch.float64
U = 2.0 ** -24
GEMM, ATTN = 0, 1                                   # Launch::Kind (ns2vc_profile_kind_name numbering)
TAP_KINDS = (11, 26)                                # TAP, CV_SPLIT_TAP: the tap copies, which no launch count includes
HOOK = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(GemmArgs), C.POINTER(AttnArgs), C.c_char_p)
PER_ROW = ("res", "rowmask", "row_valid", "ln_mu", "ln_rstd")   # epilogue tensors indexed [b, t]


# ----------------------------------------------------------------------------------------------------------- device memory
class _Dev:
    def __init__(self, p: int, n: int, typestr: str):
        self.__cuda_array_interface__ = dict(shape=(n,), typestr=typestr, data=(p, False), version=3, strides=None)


_TYPESTR = {torch.float32: "<f4", torch.float64: "<f8", torch.int16: "<i2", torch.int32: "<i4"}


def read(p: int, n: int, dtype) -> torch.Tensor:
    """a copy of n elements of device memory at p"""
    return torch.as_tensor(_Dev(p, n, _TYPESTR[dtype]), device="cuda").clone()


def read_rows(p: int, B: int, T: int, ld: int, bpitch: int, C_: int, dtype=torch.int16) -> torch.Tensor:
    """[B, T, C_] of a token-major buffer (row pitch ld, batch pitch bpitch elements; 0: T * ld)"""
    bp = bpitch or T * ld
    flat = read(p, (B - 1) * bp + (T - 1) * ld + C_, dtype)
    return flat.as_strided((B, T, C_), (bp, ld, 1)).clone()


def split_value(hi: torch.Tensor, lo: torch.Tensor, dt=torch.bfloat16):
    """(hi, lo) in fp64 of an int16-viewed 16-bit pair"""
    return hi.view(dt).to(F64), lo.view(dt).to(F64)


def src_split(s: Split, B: int):
    hi = read_rows(s.hi, B, s.T, s.ld, s.bpitch, s.C)
    lo = read_rows(s.lo, B, s.T, s.ld, s.bpitch, s.C)
    return split_value(hi, lo)


# ----------------------------------------------------------------------------------------------------------- GEMM
def packed_weights(a: GemmArgs):
    """(W hi, W lo) fp64 [rows, K] in the epilogue's order: GEGLU value rows then gate rows (the packing interleaves 64 | 64)"""
    n = a.N * a.nkb_w * 64
    hi = po.unswizzle(read(a.w_hi, n, torch.int16).view(torch.bfloat16), a.N, a.nkb_w).to(F64)
    lo = po.unswizzle(read(a.w_lo, n, torch.int16).view(torch.bfloat16), a.N, a.nkb_w).to(F64)
    nv = a.n_valid
    if a.flags & EPI_GEGLU:
        order = torch.cat([torch.arange(128 * j, 128 * j + 64) for j in range(a.N // 128)] +
                          [torch.arange(128 * j + 64, 128 * j + 128) for j in range(a.N // 128)])
        sel = torch.cat([order[:a.N // 2][:nv], order[a.N // 2:][:nv]]).to(hi.device)
        return hi[sel], lo[sel]
    return hi[:nv], lo[:nv]


def gn_affine(a: GemmArgs, rows_valid: torch.Tensor):
    """The panel GroupNorm's per-(entry, channel) affine from the producers' sums: (a32, b32) as the kernel forms them in fp32,
    (a64, b64) in fp64, and |beta (1 + s)| (for the bound)"""
    B, C1, C2, G = a.B, a.gn_C1, a.gn_C2, a.gn_G
    Cg = C1 + C2
    st1 = read(a.gn_stats1, 2 * B * C1, F64).reshape(2, B, C1)
    st = st1 if not C2 else torch.cat([st1, read(a.gn_stats2, 2 * B * C2, F64).reshape(2, B, C2)], -1)
    cpg = Cg // G
    n = (rows_valid.to(F64) if a.row_len else torch.full((B,), float(a.T_out), dtype=F64, device=st.device)) * cpg
    s = st[0].reshape(B, G, cpg).sum(-1) / n[:, None]
    var = (st[1].reshape(B, G, cpg).sum(-1) / n[:, None] - s * s).clamp_min(0)
    gamma, beta = read(a.gn_gamma, Cg, torch.float32), read(a.gn_beta, Cg, torch.float32)
    if a.gn_film:
        film = read(a.gn_film, (B - 1) * a.gn_film_ld + 2 * Cg, torch.float32).as_strided((B, 2 * Cg), (a.gn_film_ld, 1))
        fs32, fb32 = 1.0 + film[:, :Cg], film[:, Cg:2 * Cg]
    else:
        fs32, fb32 = torch.ones(B, Cg, device=st.device), torch.zeros(B, Cg, device=st.device)
    rep = lambda t: t.repeat_interleave(cpg, -1)
    # fp32, as prep_affine
    mean32, rstd32 = rep(s.float()), rep((1.0 / torch.sqrt(var.float().to(F64) + a.gn_eps)).float())
    ga = gamma * rstd32
    be = beta - mean32 * ga
    a32, b32 = ga * fs32, be * fs32 + fb32
    # fp64
    rstd = rep(1.0 / torch.sqrt(var + a.gn_eps))
    g64 = gamma.to(F64) * rstd
    a64 = g64 * fs32.to(F64)
    b64 = (beta.to(F64) - rep(s) * g64) * fs32.to(F64) + fb32.to(F64)
    return (a32, b32), (a64, b64), (beta.to(F64) * fs32.to(F64)).abs()


def panel_affine(a: GemmArgs, rows_valid: torch.Tensor):
    """the affine of a panel-mode launch: the given scale / shift, or the GroupNorm of its sums (see gn_affine)"""
    if a.gn_stats1:
        return gn_affine(a, rows_valid)
    sc = read(a.pre_scale, a.B * a.pre_C, torch.float32).reshape(a.B, a.pre_C)
    sh = read(a.pre_shift, a.B * a.pre_C, torch.float32).reshape(a.B, a.pre_C)
    return (sc, sh), (sc.to(F64), sh.to(F64)), sh.to(F64).abs()


def gemm_operands(a: GemmArgs, rows_valid: torch.Tensor, srcs, aff):
    """The launch's A operand in the packed K order [B, T_out, 64 nkb_w] from its sources srcs [(hi, lo) fp64 [B, T, C]] and
    (panel mode) its affine `aff` (panel_affine): (hi, lo) as the kernel multiplies them (panel segments: the emulated fp32
    transform, re-split), the fp64 truth operand, and the panel transform's rounding allowance (None without panels)"""
    B, T = a.B, a.T_out
    K = 64 * a.nkb_w
    dev = srcs[0][0].device
    Ah, Al, At, Ad = (torch.zeros(B, T, K, dtype=F64, device=dev) for _ in range(4))
    g = lambda x, s, c0, width, tap: ko.gather(x, s.T, s.C, c0, width, tap, T)
    if a.nxs == 0:
        k = 0
        for i in range(a.nseg):
            si, c0, width, tap = list(a.seg[i])
            s, (h, l) = a.src[si], srcs[si]
            Ah[..., k:k + width], Al[..., k:k + width] = g(h, s, c0, width, tap), g(l, s, c0, width, tap)
            At[..., k:k + width] = Ah[..., k:k + width] + Al[..., k:k + width]
            k += width
        assert k == K
        return (Ah, Al), At, None
    for i in range(a.nxs):
        si, c0, width, ntap, kb0, kbs, xf, aff_c0 = list(a.xseg[i])
        s, (h, l) = a.src[si], srcs[si]
        x = (h + l)[:, :, c0:c0 + width]
        C_ = min(width, s.C - c0)
        x = torch.nn.functional.pad(x[..., :C_], (0, width - C_))
        silu = a.pre_mode == 2
        if xf:
            (a32, b32), (a64, b64), bfs = aff
            cols = slice(aff_c0, aff_c0 + C_)
            pad = lambda t: torch.nn.functional.pad(t[:, cols], (0, width - C_))
            y = ko.affine_rows(x, pad(a32), pad(b32), silu, rows_valid, exact=False)
            yt = ko.affine_rows(x, pad(a64), pad(b64), silu, rows_valid, exact=True)
            slope = 1.1 if silu else 1.0
            keep = (torch.arange(x.shape[1], device=dev)[None, :] < rows_valid[:, None])[..., None]
            dy = 8 * U * slope * ((x * pad(a32).to(F64)[:, None]).abs() + pad(b32).to(F64)[:, None].abs() + pad(bfs)[:, None]) * keep
            yh, yl = ko.split_f64(y.float())
        else:
            keep = (torch.arange(T, device=dev)[None, :] < rows_valid[:, None])[..., None]
            yh, yl = h[:, :, c0:c0 + width], l[:, :, c0:c0 + width]
            yh, yl = (torch.nn.functional.pad(t[..., :C_], (0, width - C_)) * keep for t in (yh, yl))
            yt, dy = yh + yl, torch.zeros_like(yh)
        tap_rows = (-1, 0, 1) if ntap == 3 else (0,)
        for j, tap in enumerate(tap_rows):
            k0 = 64 * (kb0 + j * kbs)
            full = lambda t: ko.gather(t, s.T, width, 0, width, tap, T)
            Ah[..., k0:k0 + width], Al[..., k0:k0 + width] = full(yh), full(yl)
            At[..., k0:k0 + width], Ad[..., k0:k0 + width] = full(yt), full(dy)
    return (Ah, Al), At, Ad


def panel_order(a: GemmArgs) -> torch.Tensor:
    """the packed K columns in the panel loop's order: panel segments in turn, their channel blocks in turn, the taps of each"""
    cols = []
    for i in range(a.nxs):
        _, _, width, ntap, kb0, kbs, _, _ = list(a.xseg[i])
        for cb in range(width // 64):
            for j in range(ntap):
                k0 = 64 * (kb0 + j * kbs + cb)
                cols.append(torch.arange(k0, k0 + 64))
    return torch.cat(cols)


def gemm_epilogue_inputs(a: GemmArgs, rows_valid: torch.Tensor) -> Dict:
    B, T, n = a.B, a.T_out, a.n_valid
    f = a.flags
    ep = dict(n_valid=n, geglu=bool(f & EPI_GEGLU), gelu=bool(f & EPI_GELU), relu=bool(f & EPI_RELU))
    if f & (EPI_BIAS | EPI_GEGLU):
        ep["bias"] = read(a.bias, 2 * n if f & EPI_GEGLU else n, torch.float32)
    res = None
    if f & EPI_RESIDUAL:
        res = read_rows(a.res, 1, B * T, a.res_ld, 0, n, torch.float32).reshape(B, T, n).to(F64)
    if f & EPI_ROWBIAS:                                # a per-entry bias row: part of what the epilogue adds to the sum
        rb = read(a.rowbias, (B - 1) * a.rowbias_ld + n, torch.float32).as_strided((B, n), (a.rowbias_ld, 1)).to(F64)
        res = (0 if res is None else res) + rb[:, None, :].expand(B, T, n)
    if res is not None:
        ep["res"] = res
    if f & EPI_ROWMASK:
        ep["rowmask"] = read(a.rowmask, B * T, torch.float32).reshape(B, T)
    if a.row_len:
        ep["row_valid"] = torch.arange(T, device=rows_valid.device)[None, :] < rows_valid[:, None]
    if f & EPI_LNFOLD:
        st = read(a.ln_stats, 2 * B * T, F64).reshape(B, T, 2)
        mean = st[..., 0] / a.ln_C
        var = (st[..., 1] / a.ln_C - mean * mean).clamp_min(0)
        ep.update(lnf=True, ln_mu=mean, ln_rstd=1.0 / torch.sqrt(var + a.ln_eps),
                  ln_g=read(a.ln_g, 2 * n if f & EPI_GEGLU else n, torch.float32))
    return ep


def rows_of(ep: Dict, b: int) -> Dict:
    return {k: (v[b:b + 1] if k in PER_ROW and torch.is_tensor(v) else v) for k, v in ep.items()}


def emulate(A2, W2, ep, drop=None):
    """ko.gemm_emulate entry by entry (its running-magnitude term is [rows, N, K / 16])"""
    outs, bounds = [], []
    for b in range(A2[0].shape[0]):
        o, bd = ko.gemm_emulate(None, None, rows_of(ep, b), drop, a_split=(A2[0][b:b + 1], A2[1][b:b + 1]), w_split=W2)
        outs.append(o)
        bounds.append(bd)
    return torch.cat(outs), (None if drop is not None else torch.cat(bounds))


def valid_rows(B: int, T: int, row_len: int, shift: int, dev) -> torch.Tensor:
    if not row_len:
        return torch.full((B,), T, dtype=torch.long, device=dev)
    L = read(row_len, B, torch.int32).long()
    return torch.clamp(((L - 1) >> shift) + 1, max=T)


class GemmLaunch:
    """One GEMM launch: its inputs before, its outputs after, the comparison"""

    def __init__(self, a: GemmArgs, desc: str):
        self.a, self.desc = a, desc
        dev = torch.device("cuda")
        B, T, n = a.B, a.T_out, a.n_valid
        self.rv = valid_rows(B, T, a.row_len, a.len_shift, dev)
        srcs = [src_split(a.src[i], B) for i in range(a.nsrc)]
        self.A2, self.At, self.Ad = gemm_operands(a, self.rv, srcs, panel_affine(a, self.rv) if a.nxs else None)
        self.W2 = packed_weights(a)
        if a.nxs:                                      # K in the order the panel loop accumulates it (the running-magnitude term)
            k = panel_order(a).to(self.At.device)
            self.A2, self.At, self.Ad = (self.A2[0][..., k], self.A2[1][..., k]), self.At[..., k], self.Ad[..., k]
            self.W2 = (self.W2[0][:, k], self.W2[1][:, k])
        self.ep = gemm_epilogue_inputs(a, self.rv)
        self.stats0 = {}
        if a.flags & EPI_STATS:
            self.stats0 = dict(sum=read(a.stat_sum, B * n, F64), sq=read(a.stat_sq, B * n, F64))
        if a.flags & EPI_ROWSTATS:
            self.stats0["row"] = read(a.row_stats, 2 * B * T, F64)

    def outputs(self):
        a, B, T, n = self.a, self.a.B, self.a.T_out, self.a.n_valid
        out = {}
        if a.flags & EPI_OUT_NCT:
            out["f32"] = read(a.out, B * n * T, torch.float32).reshape(B, n, T).transpose(1, 2)
        elif a.flags & EPI_OUT_F32:
            out["f32"] = read_rows(a.out, 1, B * T, a.out_ld, 0, n, torch.float32).reshape(B, T, n)
        if a.flags & EPI_OUT_SPLIT:
            hi = read_rows(a.out_hi, 1, B * T, a.out_split_ld, 0, n).reshape(B, T, n)
            lo = read_rows(a.out_lo, 1, B * T, a.out_split_ld, 0, n).reshape(B, T, n)
            f16 = torch.arange(n, device=hi.device) >= (a.f16_col0 if a.f16_col0 >= 0 else 1 << 30)
            hb, lb = split_value(hi, lo)
            hf, lf = split_value(hi, lo, torch.float16)
            out["split"] = torch.where(f16, hf + lf, hb + lb)
            out["hi"], out["lo"], out["f16"] = hi, lo, f16
        return out

    def check(self, name: str, ratios: Dict):
        a, ep = self.a, self.ep
        B, T, n = a.B, a.T_out, a.n_valid
        out = self.outputs()
        emu, bound = emulate(self.A2, self.W2, ep)
        if self.Ad is not None:                        # the panel transform's fp32 rounding, carried by |W|
            bound = bound + self.slope(self.Ad @ (self.W2[0] + self.W2[1]).abs().T)
        truth = ko.gemm_truth(self.At, self.W2[0] + self.W2[1], ep)
        extra = bound if a.flags & EPI_LNFOLD else None
        if "f32" in out:
            got = out["f32"].to(F64)
            r_emu = ko.ratio(got - emu, bound)
            if "split" in out:                         # the split is the split of the fp32 value, column by column
                v = out["f32"]
                hb, lb = ko.split(v, torch.bfloat16)
                hf, lf = ko.split(v, torch.float16)
                f16 = out["f16"]
                want_hi = torch.where(f16, hf.view(torch.int16), hb.view(torch.int16))
                want_lo = torch.where(f16, lf.view(torch.int16), lb.view(torch.int16))
                assert torch.equal(out["hi"], want_hi) and torch.equal(out["lo"], want_lo), f"{name}: split is not the split of the fp32 output"
        else:
            got = out["split"]
            tol_split = 2.0 ** -16 * emu.abs() + torch.where(out["f16"], U, 0.0)
            r_emu = ko.ratio(got - emu, bound + tol_split)
        assert r_emu <= 1.0, f"{name}: |gpu - emu| reaches {r_emu:.2f} x tol_emu"
        r_truth = truth_check(name, got, truth, extra)
        if "row_valid" in ep:
            assert (got[~ep["row_valid"]] == 0).all(), f"{name}: rows past the row length are not zero"
        if "rowmask" in ep:
            assert (got[ep["rowmask"] == 0] == 0).all(), f"{name}: rows the mask drops are not zero"
        # statistics: what the launch added, against fp64 sums of its own output
        slack = 33 * U + (0 if "f32" in out else 2.0 ** -16)
        if a.flags & EPI_STATS:
            for key, fn in (("sum", lambda z: z), ("sq", lambda z: z * z)):
                ptr_ = a.stat_sum if key == "sum" else a.stat_sq
                added = (read(ptr_, B * n, F64) - self.stats0[key]).reshape(B, n)
                ref, mag = fn(got).sum(1), fn(got).abs().sum(1)
                assert ((added - ref).abs() <= slack * mag + 1e-12 * ref.abs() + 1e-300).all(), f"{name}: column {key}"
        if a.flags & EPI_ROWSTATS:
            added = (read(a.row_stats, 2 * B * T, F64) - self.stats0["row"]).reshape(B, T, 2)
            for j, fn in enumerate((lambda z: z, lambda z: z * z)):
                ref, mag = fn(got).sum(-1), fn(got).abs().sum(-1)
                assert ((added[..., j] - ref).abs() <= slack * mag + 1e-12 * ref.abs() + 1e-300).all(), f"{name}: row statistics"
        ratios["emu"] = max(ratios.get("emu", 0.0), r_emu)
        ratios["truth"] = max(ratios.get("truth", 0.0), r_truth)
        return emu, bound

    def slope(self, d: torch.Tensor) -> torch.Tensor:
        """an accumulator allowance carried through the epilogue's slope (LayerNorm fold: rstd; GELU: |gelu'| <= 1.13; row
        mask)"""
        ep = self.ep
        if ep.get("lnf"):
            d = d * ep["ln_rstd"][..., None]
        n = ep["n_valid"]
        assert not ep.get("geglu"), "a GEGLU launch over panels"
        if ep.get("gelu"):
            d = d * 1.2
        if ep.get("rowmask") is not None:
            d = d * ep["rowmask"].to(F64).abs()[..., None]
        return d[..., :n]

    def sensitivity(self, emu, bound) -> float:
        return min(ko.ratio(emulate(self.A2, self.W2, self.ep, drop=i)[0] - emu, bound) for i in range(3))


# ----------------------------------------------------------------------------------------------------------- attention
def heads(x: torch.Tensor, H: int, dh: int) -> torch.Tensor:
    B, T, _ = x.shape
    return x[..., :H * dh].reshape(B, T, H, dh).permute(0, 2, 1, 3)


def span(p: Optional[int], n_elems: int, elem_bytes: int):
    return None if not p else (p, p + n_elems * elem_bytes)


def split_spans(s: Split, B: int):
    n = (B - 1) * (s.bpitch or s.T * s.ld) + (s.T - 1) * s.ld + s.C
    return [span(s.hi, n, 2), span(s.lo, n, 2)]


def assert_disjoint(name: str, reads, writes):
    """no byte a launch writes is one it reads: other CTAs may still be reading it"""
    for w in filter(None, writes):
        for r in filter(None, reads):
            assert w[1] <= r[0] or r[1] <= w[0], f"{name}: output [{w[0]:#x}, {w[1]:#x}) overlaps input [{r[0]:#x}, {r[1]:#x})"


class AttnLaunch:
    def __init__(self, a: AttnArgs, desc: str):
        self.a, self.desc = a, desc
        B, H, dh = a.B, a.H, a.dh
        HD = H * dh
        if a.v2:
            reads = split_spans(a.qs, B) + split_spans(a.ks, B) + split_spans(a.vs, B)
        else:
            reads = [span(a.q, (B * a.Tq - 1) * a.q_ld + HD, 4), span(a.k, (B * a.Tk - 1) * a.k_ld + HD, 4),
                     span(a.v, (B * a.Tk - 1) * a.v_ld + HD, 4)]
        writes = [span(a.out, (B * a.Tq - 1) * a.out_ld + HD, 4), span(a.out_hi, (B * a.Tq - 1) * a.out_split_ld + HD, 2),
                  span(a.out_lo, (B * a.Tq - 1) * a.out_split_ld + HD, 2)]
        assert_disjoint(f"attention {desc}", reads, writes)
        if a.v2:
            pf16 = "PF16=1" in desc
            self.mode = "f16" if pf16 else "split"

            def part(s: Split, c0: int, T: int, dt):
                hi = read_rows(s.hi, B, T, s.ld, s.bpitch, c0 + HD)[..., c0:]
                lo = read_rows(s.lo, B, T, s.ld, s.bpitch, c0 + HD)[..., c0:]
                return [heads(t, H, dh) for t in split_value(hi, lo, dt)]
            qp, kp = part(a.qs, a.q_c0, a.Tq, torch.bfloat16), part(a.ks, a.k_c0, a.Tk, torch.bfloat16)
            vp = part(a.vs, a.v_c0, a.Tk, torch.float16 if pf16 else torch.bfloat16)
            self.splits = tuple(qp + kp + vp)                # the operands as the launch reads them
            self.q, self.k, self.v = ((h + l).float() for h, l in (qp, kp, vp))
        else:
            self.splits = None
            self.mode = "v1"
            rd = lambda p, ld, T: heads(read_rows(p, B, T, ld, 0, HD, torch.float32), H, dh)
            self.q, self.k, self.v = rd(a.q, a.q_ld, a.Tq), rd(a.k, a.k_ld, a.Tk), rd(a.v, a.v_ld, a.Tk)
        self.bias = read(a.bias, B * a.Tk, torch.float32).reshape(B, a.Tk) if a.bias else None
        if a.key_len:
            L = read(a.key_len, B, torch.int32).long()
            self.nkeys = [min(a.Tk, int(((x - 1) >> a.key_shift) + 1)) for x in L.tolist()]
        else:
            self.nkeys = [a.Tk] * B

    def check(self, name: str, ratios: Dict):
        a = self.a
        B, H, dh = a.B, a.H, a.dh
        HD = H * dh
        emu, bound = ko.attention_emulate(self.q, self.k, self.v, a.scale, self.bias, self.nkeys, self.mode, splits=self.splits)
        if a.out:
            got = heads(read_rows(a.out, B, a.Tq, a.out_ld, 0, HD, torch.float32), H, dh).to(F64)
            r_emu = ko.ratio(got - emu, bound)
            if a.out_hi:
                v = read_rows(a.out, B, a.Tq, a.out_ld, 0, HD, torch.float32)
                hb, lb = ko.split(v, torch.bfloat16)
                hi = read_rows(a.out_hi, B, a.Tq, a.out_split_ld, 0, HD)
                lo = read_rows(a.out_lo, B, a.Tq, a.out_split_ld, 0, HD)
                assert torch.equal(hi, hb.view(torch.int16)) and torch.equal(lo, lb.view(torch.int16)), f"{name}: split output"
        else:
            h, l = split_value(read_rows(a.out_hi, B, a.Tq, a.out_split_ld, 0, HD), read_rows(a.out_lo, B, a.Tq, a.out_split_ld, 0, HD))
            got = heads(h + l, H, dh)
            r_emu = ko.ratio(got - emu, bound + 2.0 ** -16 * emu.abs())
        assert r_emu <= 1.0, f"{name}: |gpu - emu| reaches {r_emu:.2f} x tol_emu"
        truth = ko.attention_truth(self.q, self.k, self.v, a.scale, self.bias, self.nkeys)
        extra = ko.attention_design_terms(self.q, self.k, self.v, a.scale, self.bias, self.nkeys, truth, self.mode == "f16")
        r_truth = truth_check(name, got, truth, extra)
        ratios["emu"] = max(ratios.get("emu", 0.0), r_emu)
        ratios["truth"] = max(ratios.get("truth", 0.0), r_truth)
        return emu, bound

    def sensitivity(self, emu, bound) -> float:
        a = self.a
        return min(ko.ratio(ko.attention_emulate(self.q, self.k, self.v, a.scale, self.bias, self.nkeys, self.mode, drop=i,
                                                 splits=self.splits)[0] - emu, bound) for i in range(3))


# ----------------------------------------------------------------------------------------------------------- the observer
class Observer:
    """Checks every GEMM and attention launch of the runs made while it is installed on engine `kind`'s handle `h`."""

    def __init__(self, kind: int, h: int, program: str):
        self.kind, self.h, self.program = kind, h, program
        self.pending = None
        self.error: Optional[BaseException] = None
        self.launched = defaultdict(int)              # launch kind -> launches the program ran
        self.counted = 0                              # launches the engine's launch count includes (not the tap copies)
        self.table: Dict[str, Dict] = {}              # signature -> {n, emu, truth, sens}
        self.cb = HOOK(self._hook)

    def _hook(self, user, index, phase, kind, gp, ap, desc):
        try:
            d = desc.decode()
            if phase == 0:
                self.launched[kind] += 1
                self.counted += kind not in TAP_KINDS
                if kind == GEMM:
                    self.pending = GemmLaunch(gp.contents, d)
                elif kind == ATTN:
                    self.pending = AttnLaunch(ap.contents, d)
                return 0
            if kind in (GEMM, ATTN):
                L, self.pending = self.pending, None
                row = self.table.setdefault(d, dict(n=0))
                emu, bound = L.check(f"{self.program} launch {index} {d}", row)
                row["n"] += 1
                if "sens" not in row:
                    row["sens"] = L.sensitivity(emu, bound)
            return 0
        except BaseException as e:                    # the C side ends the run; the test raises this
            if self.error is None:
                self.error = e
            return 1

    def __enter__(self):
        _lib.check(_lib.lib().ns2vc_check_set_launch_hook(self.kind, self.h, C.cast(self.cb, C.c_void_p), None))
        return self

    def __exit__(self, *exc):
        _lib.lib().ns2vc_check_set_launch_hook(self.kind, self.h, None, None)

    def run(self, fn):
        """calls fn() with the observer installed; raises the first failed check"""
        with self:
            try:
                res = fn()
            except _lib.Ns2vcError:
                if self.error is None:
                    raise
                res = None
        if self.error is not None:
            raise self.error
        return res

    def report(self):
        checked = sum(r["n"] for r in self.table.values())
        ran = self.launched[GEMM] + self.launched[ATTN]
        print(f"\n[{self.program}] {ran} GEMM / attention launches of {sum(self.launched.values())}, {checked} checked")
        for sig, r in sorted(self.table.items()):
            print(f"  {sig:48s} launches {r['n']:4d}  emu {r['emu']:.3f}  truth {r['truth']:.3f}  sens {r['sens']:.3g}")
        assert ran > 0
        for sig, r in self.table.items():
            assert r["sens"] > 1.0, f"{self.program} {sig}: a dropped split product moves the emulation by only {r['sens']:.2f} x tol_emu"


def observed(m, kind: int, program: str, steps):
    """Runs `steps` (callables of one engine run each, returning their output or None) unobserved, then observed: every GEMM
    and attention launch is checked; after each step the launches the observer saw (tap copies aside) equal the engine's own
    launch count of that run; every step's output is bit-identical to the unobserved one's."""
    torch.cuda.synchronize()
    ref = [f() for f in steps]
    torch.cuda.synchronize()
    ob = Observer(kind, m.engine(torch.device("cuda", torch.cuda.current_device())), program)
    got = []
    for f in steps:
        n0 = ob.counted
        got.append(ob.run(f))
        torch.cuda.synchronize()
        assert ob.counted - n0 == m.launch_count(), f"{program}: the observer saw {ob.counted - n0} launches of {m.launch_count()}"
    for r, g in zip(ref, got):
        r = () if r is None else r if isinstance(r, (tuple, list)) else (r,)
        g = () if g is None else g if isinstance(g, (tuple, list)) else (g,)
        for x, y in zip(r, g):
            assert torch.equal(x.view(torch.int32), y.view(torch.int32)), f"{program}: the observed call's output differs from the unobserved one"
    ob.report()


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


# ----------------------------------------------------------------------------------------------------------- programs
def unet_module(cfg, sd=None):
    """UNet1DConditionModel of an arch.UNetConfig, with `sd` loaded (on the GPU when given)"""
    from ns2vc_b200.unet import UNet1DConditionModel
    m = UNet1DConditionModel(in_channels=cfg.in_channels, out_channels=cfg.out_channels, block_out_channels=cfg.block_out_channels,
                             layers_per_block=list(cfg.layers_per_block), norm_num_groups=cfg.norm_num_groups,
                             cross_attention_dim=cfg.cross_attention_dim, attention_head_dim=cfg.num_heads,
                             addition_embed_type=cfg.addition_embed_type, resnet_time_scale_shift=cfg.resnet_time_scale_shift,
                             addition_embed_type_num_heads=cfg.addition_embed_type_num_heads)
    if sd is None:
        return m
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


def session_steps(m, sess, x, t):
    """prepare_cond, forward, and forward_film on the rows of ns2vc_unet_time_table (the forward the sampling loops replay)"""
    L = _lib.lib()
    out = torch.empty((sess.B, sess.Co, sess.T), device="cuda")
    table = torch.empty(L.ns2vc_unet_time_table_floats(m.engine(x.device), sess.B), device="cuda")

    def forward_film():
        sess.time_table(t, table)                      # (small linears outside the run loop: no GEMM or attention)
        sess.forward(x, t, out, film_rows=table)
        return out.clone()
    return [sess.prepare, lambda: (sess.forward(x, t, out), out.clone())[1], forward_film]


@pytest.mark.gpu
@pytest.mark.parametrize("shape,regime", DENOISER_CASES, ids=[f"{s}_{r}" for s, r in DENOISER_CASES])
def test_denoiser_launches(shape, regime):
    import test_numerics_fp64 as tn
    from ns2vc_b200.fused import DenoiserSession
    m = unet_module(tn.CFG, tn.regime_state_dict(regime))
    x, t, ehs, mask = (v.cuda() for v in tn.case_inputs(shape))
    Cl = m.latent_channels
    sess = DenoiserSession(m, x[:, Cl:].contiguous(), ehs, mask)
    with torch.no_grad():
        observed(m, 0, f"denoiser {shape} {regime}", session_steps(m, sess, x[:, :Cl].contiguous(), t))


@pytest.mark.gpu
def test_denoiser_ragged_launches():
    import test_numerics_fp64 as tn
    m = unet_module(tn.CFG, tn.regime_state_dict("synthetic"))
    x, _, _, t = tn.ragged_inputs("R1")
    with torch.no_grad():
        observed(m, 0, "denoiser R1 ragged", session_steps(m, tn.ragged_session(m, "R1"), x[:, :m.latent_channels].contiguous().cuda(),
                                                           t.cuda()))


@pytest.mark.gpu
def test_tiny_denoiser_launches():
    from conftest import tiny_config, tiny_inputs
    from ns2vc_b200.fused import DenoiserSession
    from ns2vc_b200.synth import make_state_dict
    cfg = tiny_config()
    m = unet_module(cfg, make_state_dict(cfg, 0))
    inp = tiny_inputs()
    sess = DenoiserSession(m, inp["content"].permute(1, 2, 0).contiguous().cuda(), inp["prompt"].permute(1, 0, 2).contiguous().cuda(),
                           None)
    with torch.no_grad():
        observed(m, 0, "tiny denoiser", session_steps(m, sess, inp["x"].cuda(), torch.tensor([17.5, 941.25], device="cuda")))


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["synthetic", "sharp"])
def test_condition_encoder_launches(regime):
    import test_pre_model_ragged as tr
    from test_numerics_fp64 import pre_inputs
    m, _ = tr.model(regime)
    c, refer, lengths, refer_lengths = pre_inputs()
    data = (c.cuda(), refer.cuda(), None, None, None, lengths.cuda(), refer_lengths.cuda(), None)
    with torch.no_grad():
        observed(m, 1, f"condition encoders {regime}", [lambda: tuple(v.clone() for v in m.infer(data))])
        observed(m, 1, f"condition encoders {regime} per utterance",
                 [lambda: tuple(v.clone() for v in m.infer(data, per_utterance=True))])


@pytest.mark.gpu
@pytest.mark.parametrize("regime", CONTENTVEC_REGIMES)
def test_content_encoder_launches(regime):
    import test_content as tc
    m, _, _ = tc.model(regime)
    wav, lens = tc.batch_full()
    wav, L = wav.cuda(), torch.tensor(lens).cuda()
    with torch.no_grad():
        observed(m, 2, f"content encoder {regime}", [lambda: tuple(v.clone() for v in m.extract(wav, L))])


@pytest.mark.gpu
@pytest.mark.parametrize("regime", VOCOS_REGIMES)
def test_vocoder_launches(regime):
    import test_vocoder as tv
    m, _ = tv.model(regime)
    mel = tv.mel_of(4, 1024, 0)
    L = torch.tensor([1024, 700, 65, 1])
    with torch.no_grad():
        observed(m, 3, f"vocoder {regime}", [lambda: m.decode(mel, L).clone()])


# ----------------------------------------------------------------------------------------------------------- CPU tier
def test_flat_record_decodes_to_the_segments_operand():
    """The decoder from a flat record to the operand equals ko.im2col / the panel transform of the same segments, with two
    normalised panel sources, the second at aff_c0 != 0.  The expected operand is built from the same ko.affine_rows /
    ko.gather the decoder calls, so this checks the layout the record describes (segment order, kb0 and the tap stride,
    aff_c0, ragged rows), not the transform itself."""
    g = torch.Generator().manual_seed(5)
    B, T = 2, 37
    Cs = [64, 128]
    srcs = []
    for C_ in Cs:
        h, l = ko.split(torch.randn(B, T, C_, generator=g))
        srcs.append((h.to(F64), l.to(F64)))
    a = GemmArgs()
    a.B, a.T_out, a.nsrc = B, T, 2
    for i in range(2):
        a.src[i] = Split(None, None, T, Cs[i], Cs[i] + 8, 0)
    segs = [(0, 0, 64, -1), (1, 64, 64, 0), (0, 0, 64, 1), (1, 0, 128, 2)]
    a.nseg = len(segs)
    for i, sg in enumerate(segs):
        a.seg[i] = (C.c_int * 4)(*sg)
    a.nkb_w = 5
    rv = torch.full((B,), T)
    (Ah, Al), At, Ad = gemm_operands(a, rv, srcs, None)
    hl = [dict(x=h + l, T=T, C=C_) for (h, l), C_ in zip(srcs, Cs)]
    assert Ad is None and torch.equal(At, ko.im2col(hl, segs, T)) and torch.equal(Ah + Al, At)
    # panel mode: source 0 (k = 3) normalised with the affine's channels [0, 64), source 1 (1x1) with [64, 192); one entry
    # ragged at 30 rows
    a.nseg, a.nxs, a.nkb_w, a.pre_mode = 0, 2, 5, 2
    a.xseg[0] = (C.c_int * 8)(0, 0, 64, 3, 0, 1, 1, 0)
    a.xseg[1] = (C.c_int * 8)(1, 0, 128, 1, 3, 0, 1, 64)
    sc, sh = 0.5 + torch.rand(B, 192, generator=g), torch.randn(B, 192, generator=g)
    rv = torch.tensor([T, 30])
    (Ah, Al), At, Ad = gemm_operands(a, rv, srcs, ((sc, sh), (sc.to(F64), sh.to(F64)), sh.to(F64).abs()))
    want_h, want_l, want_t = [], [], []
    for si, aff0, taps in ((0, 0, (-1, 0, 1)), (1, 64, (0,))):
        x, C_ = hl[si]["x"], Cs[si]
        y = ko.affine_rows(x, sc[:, aff0:aff0 + C_], sh[:, aff0:aff0 + C_], True, rv, exact=False)
        yt = ko.affine_rows(x, sc[:, aff0:aff0 + C_], sh[:, aff0:aff0 + C_], True, rv, exact=True)
        yh, yl = ko.split_f64(y.float())
        for t in taps:
            want_h.append(ko.gather(yh, T, C_, 0, C_, t, T))
            want_l.append(ko.gather(yl, T, C_, 0, C_, t, T))
            want_t.append(ko.gather(yt, T, C_, 0, C_, t, T))
    assert torch.equal(Ah, torch.cat(want_h, -1)) and torch.equal(Al, torch.cat(want_l, -1)) and torch.equal(At, torch.cat(want_t, -1))
    assert (Ad >= 0).all() and (Ad[1, 31:] == 0).all() and (Ad[:, 1:29] > 0).all()


def test_hook_refuses_bad_engine_kind_and_null_handle():
    from conftest import tiny_config
    L = _lib.lib()
    m = unet_module(tiny_config())
    h = C.c_void_p()
    _lib.check(L.ns2vc_unet_create(C.byref(m._c_cfg()), C.byref(h)))
    try:
        cb = HOOK(lambda *a: 0)
        assert L.ns2vc_check_set_launch_hook(7, h.value, C.cast(cb, C.c_void_p), None) < 0
        assert "engine kind 7" in L.ns2vc_last_error().decode()
        assert L.ns2vc_check_set_launch_hook(0, None, C.cast(cb, C.c_void_p), None) < 0
        assert "null handle" in L.ns2vc_last_error().decode()
        assert L.ns2vc_check_set_launch_hook(0, h.value, C.cast(cb, C.c_void_p), None) == 0
        assert L.ns2vc_check_set_launch_hook(0, h.value, None, None) == 0
    finally:
        L.ns2vc_unet_destroy(h.value)
