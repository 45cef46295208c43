"""Two references for single launches of the wgmma GEMM (csrc/gemm_tc.cu) and the flash attention (csrc/attention_v2.cu,
csrc/attention.cu on csrc/flash_mma.cuh), used by tests/test_kernels_fp64.py.

* truth:     the operation in fp64 from the fp32 inputs;
* emulation: the same operation with exactly the roundings the kernels document, evaluated in fp64 - operands as bf16 (or fp16)
  hi/lo splits, the 3-term product hi*hi + lo*hi + hi*lo, the folded-LayerNorm epilogue from the given row sums, the online softmax
  tile by tile over 64-key tiles with fp16 P (l summing the rounded weights) or bf16 hi/lo P.

The emulation takes a `drop` argument (the index of a split product to leave out) and the attention a key-mask defect, so a test
can show that its tolerance would notice each of those defects.  Everything runs on the device of its inputs."""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence, Tuple

import torch

F64 = torch.float64
LOG2E = 1.4426950408889634
KEYS = 64                         # keys per tile of the flash kernels


def split(x: torch.Tensor, dt: torch.dtype = torch.bfloat16) -> Tuple[torch.Tensor, torch.Tensor]:
    """fp32 x -> (hi, lo) in `dt`: hi = rn(x), lo = rn(x - hi) (the fp32 difference is exact)."""
    x = x.float()
    hi = x.to(dt)
    return hi, (x - hi.float()).to(dt)


def split_f64(x: torch.Tensor, dt: torch.dtype = torch.bfloat16) -> Tuple[torch.Tensor, torch.Tensor]:
    hi, lo = split(x, dt)
    return hi.to(F64), lo.to(F64)


def product3(ah, al, wh, wl, drop: Optional[int] = None) -> torch.Tensor:
    """ah/al [..., K] x wh/wl [N, K]^T: Ah Wh + Al Wh + Ah Wl (term `drop` left out)"""
    terms = [(ah, wh), (al, wh), (ah, wl)]
    out = 0
    for i, (a, w) in enumerate(terms):
        if i != drop:
            out = out + a @ w.transpose(-1, -2)
    return out


def gelu_erf(x: torch.Tensor) -> torch.Tensor:
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_erf_slope(x: torch.Tensor) -> torch.Tensor:
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


# ---------------------------------------------------------------------------------------------------------------------------
# GEMM
# ---------------------------------------------------------------------------------------------------------------------------
def gather(x: torch.Tensor, T_src: int, C_src: int, c0: int, width: int, tap: int, T_out: int) -> torch.Tensor:
    """Rows t + tap (t < T_out) and channels [c0, c0 + width) of a token-major [B, >= T_src, >= C_src] source, zero outside
    [0, T_src) x [0, C_src): one segment of the implicit GEMM as the TMA unit reads it."""
    B = x.shape[0]
    out = torch.zeros(B, T_out, width, dtype=x.dtype, device=x.device)
    t_lo, t_hi = max(0, -tap), min(T_out, T_src - tap)
    c_hi = min(width, C_src - c0)
    if t_hi > t_lo and c_hi > 0:
        out[:, t_lo:t_hi, :c_hi] = x[:, t_lo + tap:t_hi + tap, c0:c0 + c_hi]
    return out


def im2col(srcs: Sequence[Dict], segs: Sequence[Tuple[int, int, int, int]], T_out: int) -> torch.Tensor:
    """[B, T_out, K] operand of the segments (src, c0, nch, tap); each segment is 64 * ceil(nch / 64) wide."""
    cols = []
    for si, c0, nch, tap in segs:
        s = srcs[si]
        cols.append(gather(s["x"], s["T"], s["C"], c0, 64 * ((nch + 63) // 64), tap, T_out))
    return torch.cat(cols, -1)


def affine_rows(x: torch.Tensor, scale: torch.Tensor, shift: torch.Tensor, silu: bool, T_valid: torch.Tensor,
                exact: bool) -> torch.Tensor:
    """Panel-mode transform of a raw [B, T, C] source: y = x * scale[b] + shift[b] (then SiLU), rows t >= T_valid[b] zero.
    exact: in fp64 (truth); else rounded to fp32 after the affine and after SiLU, as the kernel's fp32 registers."""
    y = x.to(F64) * scale[:, None, :].to(F64) + shift[:, None, :].to(F64)
    if not exact:
        y = y.float().to(F64)
    if silu:
        y = y * torch.sigmoid(y)
        if not exact:
            y = y.float().to(F64)
    keep = torch.arange(x.shape[1], device=x.device)[None, :] < T_valid[:, None]
    return torch.where(keep[..., None], y, torch.zeros((), dtype=F64, device=x.device))


def gemm_epilogue(acc: torch.Tensor, ep: Dict) -> torch.Tensor:
    """The wgmma kernel's epilogue on a [B, T, n] fp64 accumulator (GEGLU: [B, T, 2n], value | gate), in fp64."""
    if ep.get("lnf"):
        mu, rstd, g = ep["ln_mu"][..., None], ep["ln_rstd"][..., None], ep["ln_g"].to(F64)
        acc = rstd * (acc - mu * g)
    n = ep["n_valid"]
    if ep.get("geglu"):
        b = ep["bias"].to(F64)
        v = (acc[..., :n] + b[:n]) * gelu_erf(acc[..., n:] + b[n:])
    else:
        v = acc[..., :n]
        if ep.get("bias") is not None:
            v = v + ep["bias"].to(F64)[:n]
    if ep.get("res") is not None:
        v = v + ep["res"].to(F64)
    if ep.get("gelu"):
        v = gelu_erf(v)
    if ep.get("relu"):
        v = v.clamp_min(0.0)
    if ep.get("rowmask") is not None:
        v = v * ep["rowmask"].to(F64)[..., None]
    if ep.get("row_valid") is not None:
        v = torch.where(ep["row_valid"][..., None], v, torch.zeros((), dtype=F64, device=v.device))
    return v


def running_magnitude(a: torch.Tensor, w: torch.Tensor, step: int = 16) -> torch.Tensor:
    """sum over the 16-wide k-steps of |the accumulator after the step|: a [..., K], w [N, K] -> [..., N]"""
    K = a.shape[-1]
    blocks = torch.einsum("...ks,nks->...nk", a.reshape(*a.shape[:-1], K // step, step), w.reshape(w.shape[0], K // step, step))
    return blocks.cumsum(-1).abs().sum(-1)


def gemm_bound(absacc: torch.Tensor, run: torch.Tensor, acc: torch.Tensor, ep: Dict) -> torch.Tensor:
    """fp32-accumulation-level bound of |kernel - emulation| per output, on the accumulator: 16 * 2^-24 * (|A| |W|) for the
    sums inside one MMA, plus 2 ulps (2^-22) of the running accumulator for each of the three MMAs of a 16-wide k-step (`run`:
    the sum of the accumulator's magnitudes after each step); carried through the epilogue by its slope, plus a few fp32
    roundings of the epilogue's own values."""
    u = 2.0 ** -24
    e = 16 * u * absacc + 3 * 4 * u * run
    n = ep["n_valid"]
    if ep.get("lnf"):
        mu, rstd, g = ep["ln_mu"][..., None], ep["ln_rstd"][..., None], ep["ln_g"].to(F64)
        centred = acc - mu * g
        e = rstd * (e + 4 * u * (acc.abs() + (mu * g).abs())) + 4 * u * (rstd * centred).abs()
        acc = rstd * centred
    if ep.get("geglu"):
        b = ep["bias"].to(F64)
        v, gt = acc[..., :n] + b[:n], acc[..., n:] + b[n:]
        out = v * gelu_erf(gt)
        err = gelu_erf(gt).abs() * (e[..., :n] + 2 * u * v.abs()) + v.abs() * (gelu_erf_slope(gt).abs() * (e[..., n:] + 2 * u * gt.abs())
                                                                                + 4e-7 * (1 + gt.abs()))
        return err + 4 * u * out.abs()
    v = acc[..., :n]
    err = e[..., :n] + 2 * u * v.abs()
    if ep.get("bias") is not None:
        v = v + ep["bias"].to(F64)[:n]
    if ep.get("res") is not None:
        v = v + ep["res"].to(F64)
    err = err + 2 * u * v.abs()
    if ep.get("gelu"):
        err = gelu_erf_slope(v).abs() * err + 4e-7 * (1 + v.abs()) + 4 * u * gelu_erf(v).abs()
    if ep.get("rowmask") is not None:
        err = err * ep["rowmask"].to(F64).abs()[..., None]
    return err


def gemm_truth(A: torch.Tensor, W: torch.Tensor, ep: Dict) -> torch.Tensor:
    """A [B, T, K] (fp64 from fp32 values), W [N, K] fp32: the epilogue of A W^T in fp64."""
    return gemm_epilogue(A.to(F64) @ W.to(F64).T, ep)


def gemm_emulate(A: torch.Tensor, W: torch.Tensor, ep: Dict, drop: Optional[int] = None, a_split: Optional[Tuple] = None):
    """(emulation, bound): A as bf16 hi/lo (or the given split pair), W fp32 as bf16 hi/lo, 3-term product, epilogue."""
    ah, al = a_split if a_split is not None else split_f64(A)
    wh, wl = split_f64(W)
    acc = product3(ah, al, wh, wl, drop)
    if drop is not None:
        return gemm_epilogue(acc, ep), None
    absacc = (ah + al).abs() @ (wh + wl).abs().T
    return gemm_epilogue(acc, ep), gemm_bound(absacc, running_magnitude(ah + al, wh + wl), acc, ep)


# ---------------------------------------------------------------------------------------------------------------------------
# Attention
# ---------------------------------------------------------------------------------------------------------------------------
def attention_truth(q, k, v, scale: float, bias: Optional[torch.Tensor], nkeys: Sequence[int]) -> torch.Tensor:
    """q [B, H, Tq, dh], k / v [B, H, Tk, dh], bias [B, Tk] or None; entry b attends over its first nkeys[b] keys."""
    s = (q.to(F64) @ k.to(F64).transpose(-1, -2)) * scale
    if bias is not None:
        s = s + bias.to(F64)[:, None, None, :]
    Tk = k.shape[2]
    valid = torch.arange(Tk, device=q.device)[None, :] < torch.tensor(list(nkeys), device=q.device)[:, None]
    s = s.masked_fill(~valid[:, None, None, :], float("-inf"))
    return torch.softmax(s, -1) @ v.to(F64)


def attention_design_terms(q, k, v, scale: float, bias, nkeys, out: torch.Tensor, fp16_p: bool) -> torch.Tensor:
    """The precision design's own error terms of one launch against the truth, per output: a 3xBF16 score is exact to
    3 * 2^-17 of |q| |k| * scale (moving weight j by ln2 times that), and an fp16 weight is exact to 2^-12 relative."""
    s = (q.to(F64) @ k.to(F64).transpose(-1, -2)) * scale
    if bias is not None:
        s = s + bias.to(F64)[:, None, None, :]
    Tk = k.shape[2]
    valid = torch.arange(Tk, device=q.device)[None, :] < torch.tensor(list(nkeys), device=q.device)[:, None]
    P = torch.softmax(s.masked_fill(~valid[:, None, None, :], float("-inf")), -1)
    ds = 3 * 2.0 ** -17 * (q.to(F64).abs() @ k.to(F64).abs().transpose(-1, -2)) * scale
    absv, absout = v.to(F64).abs(), out.to(F64).abs()
    terms = math.log(2.0) * ((P * ds) @ absv + (P * ds).sum(-1, keepdim=True) * absout)
    if fp16_p:
        terms = terms + 2.0 ** -12 * (P @ absv + absout)
    return terms


def attention_emulate(q, k, v, scale: float, bias: Optional[torch.Tensor], nkeys: Sequence[int], mode: str,
                      drop: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """(emulation, bound) of one flash launch.  mode: "f16" (v2, fp16 P, V as fp16 hi/lo), "split" (v2, bf16 hi/lo P and V),
    "v1" (attn_tc_kernel: q pre-scaled in fp32 before its split, bf16 hi/lo P and V).  q/k/v fp32 [B, H, T, dh]."""
    dev = q.device
    B, H, Tq, dh = q.shape
    Tk = k.shape[2]
    qs32 = torch.tensor(scale, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32)
    if mode == "v1":
        qh, ql = split_f64(q.float() * qs32.to(dev))
        qs = 1.0
    else:
        qh, ql = split_f64(q)
        qs = float(qs32)
    kh, kl = split_f64(k)
    vdt = torch.float16 if mode == "f16" else torch.bfloat16
    vh, vl = split_f64(v, vdt)
    raw = product3(qh, ql, kh, kl, drop)                      # [B, H, Tq, Tk]
    s = raw * qs
    if bias is not None:
        s = s + (bias.float() * torch.tensor(LOG2E, dtype=torch.float32)).to(F64)[:, None, None, :]
    valid = torch.arange(Tk, device=dev)[None, :] < torch.tensor(list(nkeys), device=dev)[:, None]
    s = s.masked_fill(~valid[:, None, None, :], float("-inf")).float().to(F64)    # fp32 scores
    # score error of the kernel against this emulation (log2 units): fp32 accumulation of the 3-term product and the scaling
    u = 2.0 ** -24
    score_mag = ((qh + ql).abs() @ (kh + kl).abs().transpose(-1, -2)) * abs(qs)
    ds = 16 * u * (score_mag + s.abs().nan_to_num(0.0, posinf=0.0, neginf=0.0)) + 4 * u
    absv = (vh + vl).abs()
    m = torch.full((B, H, Tq, 1), float("-inf"), dtype=F64, device=dev)
    l = torch.zeros((B, H, Tq, 1), dtype=F64, device=dev)
    o = torch.zeros((B, H, Tq, dh), dtype=F64, device=dev)
    # fp16 weights within the kernel's error of a rounding midpoint may round the other way there: one fp16 ulp each
    flip_o = torch.zeros((B, H, Tq, dh), dtype=F64, device=dev)
    flip_l = torch.zeros((B, H, Tq, 1), dtype=F64, device=dev)
    for j0 in range(0, Tk, KEYS):
        st = s[..., j0:j0 + KEYS]
        mn = torch.maximum(m, st.amax(-1, keepdim=True))
        corr = torch.where(mn == float("-inf"), torch.zeros_like(mn), torch.exp2(m - mn))
        l, o, flip_o, flip_l = l * corr, o * corr, flip_o * corr, flip_l * corr
        p = torch.exp2(st - mn).float()                        # the kernel's fp32 weights
        vj_h, vj_l = vh[..., j0:j0 + KEYS, :], vl[..., j0:j0 + KEYS, :]
        if mode == "f16":
            p64 = p.to(F64)
            p16 = p.to(torch.float16).to(F64)
            l = l + p16.sum(-1, keepdim=True)
            o = o + p16 @ (vj_h + vj_l)
            ulp = torch.where(p64 >= 2.0 ** -14, 2.0 ** (torch.floor(torch.log2(p64.clamp_min(2.0 ** -14))) - 10),
                              torch.full_like(p64, 2.0 ** -24))
            err_p = p64 * (4 * u + math.log(2.0) * ds[..., j0:j0 + KEYS])
            near = ((ulp / 2 - (p64 - p16).abs()) <= err_p) & (p64 > 0)
            fu = torch.where(near, ulp, torch.zeros_like(ulp))
            flip_o = flip_o + fu @ absv[..., j0:j0 + KEYS, :]
            flip_l = flip_l + fu.sum(-1, keepdim=True)
        else:
            ph, pl = split_f64(p)
            l = l + p.to(F64).sum(-1, keepdim=True)
            o = o + ph @ vj_h + pl @ vj_h + ph @ vj_l
        m = mn
    out = o / l
    # bound: fp32 accumulation of the weighted |v|, the score errors (a score error ds moves a weight by p ln2 ds), the flips
    p_all = torch.exp2(s - m).nan_to_num(0.0)                 # final-max weights (<= 1)
    wv = (p_all @ absv) / l                                   # weighted |v|
    wdv = (p_all * ds) @ absv / l + ((p_all * ds).sum(-1, keepdim=True) / l) * out.abs()
    bound = 16 * u * (wv + out.abs()) + math.log(2.0) * wdv + (flip_o + flip_l * out.abs()) / l
    return out, bound


def rms(x: torch.Tensor) -> float:
    return float(x.double().pow(2).mean().sqrt())


def rule_tol(ref: torch.Tensor, rtol: float = 1e-3, atol_rms: float = 1e-4) -> torch.Tensor:
    """the project's parity rule: rtol |ref| + atol_rms rms(ref)"""
    return rtol * ref.abs() + atol_rms * rms(ref)


def ratio(err: torch.Tensor, bound: torch.Tensor) -> float:
    """max err / bound elementwise, 0 where err is 0 (a bound of 0 is met only exactly)"""
    err = err.to(F64).abs()
    return float(torch.where(err == 0, torch.zeros_like(err), err / bound).max())


def rule_ratio(got: torch.Tensor, ref: torch.Tensor) -> float:
    """max |got - ref| / rule_tol(ref) (<= 1 passes)"""
    return ratio(got.to(F64) - ref, rule_tol(ref))
