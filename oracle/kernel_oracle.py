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


def gemm_emulate(A: torch.Tensor, W: torch.Tensor, ep: Dict, drop: Optional[int] = None, a_split: Optional[Tuple] = None,
                 w_split: Optional[Tuple] = None):
    """(emulation, bound): A as bf16 hi/lo (or the given split pair), W fp32 as bf16 hi/lo (or the given packed pair), 3-term
    product, epilogue."""
    ah, al = a_split if a_split is not None else split_f64(A)
    wh, wl = w_split if w_split is not None else split_f64(W)
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
                      drop: Optional[int] = None, splits: Optional[Tuple] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """(emulation, bound) of one flash launch.  mode: "f16" (v2, fp16 P, V as fp16 hi/lo), "split" (v2, bf16 hi/lo P and V),
    "v1" (attn_tc_kernel: q pre-scaled in fp32 before its split, bf16 hi/lo P and V).  q/k/v fp32 [B, H, T, dh].  splits (v2):
    the launch's own (qh, ql, kh, kl, vh, vl) in fp64 instead of the splits of q / k / v (a producer's split of x need not be
    the split of fp32(hi + lo): where lo is half an ulp of hi, round-to-even may split the sum the other way)."""
    dev = q.device
    B, H, Tq, dh = q.shape
    Tk = k.shape[2]
    qs32 = torch.tensor(scale, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32)
    vdt = torch.float16 if mode == "f16" else torch.bfloat16
    if splits is not None:
        qh, ql, kh, kl, vh, vl = splits
        qs = float(qs32)
    else:
        if mode == "v1":
            qh, ql = split_f64(q.float() * qs32.to(dev))
            qs = 1.0
        else:
            qh, ql = split_f64(q)
            qs = float(qs32)
        kh, kl = split_f64(k)
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
    # A weight within the kernel's error of a rounding boundary of its 16-bit form may round the other way there: one fp16 ulp
    # of an fp16 weight (numerator and row sum), 2^-16 p of a bf16 hi/lo weight near a boundary of its hi or lo half
    # (numerator only: the row sum adds the fp32 weights)
    flip_o = torch.zeros((B, H, Tq, dh), dtype=F64, device=dev)
    flip_l = torch.zeros((B, H, Tq, 1), dtype=F64, device=dev)
    for j0 in range(0, Tk, KEYS):
        st = s[..., j0:j0 + KEYS]
        mn = torch.maximum(m, st.amax(-1, keepdim=True))
        corr = torch.where(mn == float("-inf"), torch.zeros_like(mn), torch.exp2(m - mn))
        l, o, flip_o, flip_l = l * corr, o * corr, flip_o * corr, flip_l * corr
        p = torch.exp2(st - mn).float()                        # the kernel's fp32 weights
        vj_h, vj_l = vh[..., j0:j0 + KEYS, :], vl[..., j0:j0 + KEYS, :]
        p64 = p.to(F64)
        err_p = p64 * (4 * u + math.log(2.0) * ds[..., j0:j0 + KEYS])
        if mode == "f16":
            p16 = p.to(torch.float16).to(F64)
            l = l + p16.sum(-1, keepdim=True)
            o = o + p16 @ (vj_h + vj_l)
            ulp = torch.where(p64 >= 2.0 ** -14, 2.0 ** (torch.floor(torch.log2(p64.clamp_min(2.0 ** -14))) - 10),
                              torch.full_like(p64, 2.0 ** -24))
            near = ((ulp / 2 - (p64 - p16).abs()) <= err_p) & (p64 > 0)
            fu = torch.where(near, ulp, torch.zeros_like(ulp))
            flip_l = flip_l + fu.sum(-1, keepdim=True)
        else:
            ph, pl = split_f64(p)
            l = l + p64.sum(-1, keepdim=True)
            o = o + ph @ vj_h + pl @ vj_h + ph @ vj_l
            ulp_of = lambda x: 2.0 ** (torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -140))) - 7)
            r = p64 - ph
            near_hi = (ulp_of(p64) / 2 - r.abs()) <= err_p
            near_lo = (r != 0) & ((ulp_of(r) / 2 - (r - pl).abs()) <= err_p)
            fu = torch.where((near_hi | near_lo) & (p64 > 0), 2.0 ** -16 * p64, torch.zeros_like(p64))
        flip_o = flip_o + fu @ absv[..., j0:j0 + KEYS, :]
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


# ---------------------------------------------------------------------------------------------------------------------------
# GroupNorm / LayerNorm / timestep / pooling launches (tests/test_norm_kernels_fp64.py).  Each reference is the operation in
# the dtype of its arguments: fp64 on the kernel's fp32 input is the truth, fp32 gives e32 (the floor of the parity rule).
# ---------------------------------------------------------------------------------------------------------------------------
def parity_tol(ref: torch.Tensor, e32: float) -> torch.Tensor:
    """the parity rule of the model-level files: max(1e-3 |ref| + 1e-4 rms(ref), 2 e32), e32 = max |fp32 - fp64| of the same
    operation on the same input"""
    return torch.clamp(rule_tol(ref), min=2 * e32)


def group_norm_rows(x: torch.Tensor, G: int, gamma, beta, eps: float, rows: Sequence[int], film: Optional[torch.Tensor] = None,
                    silu: bool = False, one_plus: bool = True, count: Optional[Sequence[int]] = None) -> torch.Tensor:
    """GroupNorm of token-major x [B, T, C] over each entry's first rows[b] rows (nn.GroupNorm on the unpadded entry), then
    x * (1 + scale) + shift of film [B, >= 2C] (scale | shift), then SiLU; rows past rows[b] are 0.  In x's dtype.
    one_plus=False (FiLM scale without 1+) and count (the rows the statistics are divided by) are defects for the sensitivity checks."""
    B, T, C = x.shape
    out = torch.zeros_like(x)
    for b in range(B):
        n = int(rows[b])
        xb = x[b, :n].T[None]                                          # [1, C, n]
        if count is None:
            y = torch.nn.functional.group_norm(xb, G, gamma.to(x.dtype), beta.to(x.dtype), eps)[0].T
        else:
            g = xb.reshape(G, -1)
            k = int(count[b]) * (C // G)
            mean = g.sum(-1, keepdim=True) / k
            var = (g * g).sum(-1, keepdim=True) / k - mean * mean
            y = ((g - mean) / torch.sqrt(var.clamp_min(0) + eps)).reshape(C, n).T * gamma.to(x.dtype) + beta.to(x.dtype)
        if film is not None:
            s, sh = film[b, :C].to(x.dtype), film[b, C:2 * C].to(x.dtype)
            y = y * ((1 + s) if one_plus else s) + sh
        if silu:
            y = y * torch.sigmoid(y)
        out[b, :n] = y
    return out


def one_pass_variance_term(x: torch.Tensor, G: int, gamma, rows: Sequence[int], film: Optional[torch.Tensor], eps: float,
                           partial: int = 32) -> torch.Tensor:
    """Bound of what the producers' statistics add to a GroupNorm output, per element.  The producing GEMM epilogue (EPI_STATS)
    sums each column in fp32 over `partial` rows, then adds the partial sums in fp64: a partial of p terms is within
    (p - 1) 2^-24 of the sum of their magnitudes (the standard summation bound), so with S1 = sum |x| and S2 = sum x^2 over a
    group of n elements
        |d mean| <= (p - 1) 2^-24 S1 / n,      |d q / n| <= (p - 1) 2^-24 S2 / n,
    and the one-pass variance q / n - mean^2 is off by |d var| <= (p - 1) 2^-24 (S2 / n + 2 |mean| S1 / n) + d mean^2.  Relative
    to var that is ~ 3 (p - 1) 2^-24 (1 + r^2) for r = |mean| / std (a worst case; random roundings give ~ 2^-24 r^2 sqrt(p / n)).
    An output y = (x - mean) rstd gamma (1 + s) then moves by
        |gamma (1 + s)| rstd (|d mean| + |x - mean| |d var| / (2 (var + eps))).
    Rows past rows[b] get 0 (the kernels store exact zeros there)."""
    B, T, C = x.shape
    u = (partial - 1) * 2.0 ** -24
    out = torch.zeros_like(x)
    for b in range(B):
        n = int(rows[b])
        g = x[b, :n].T.reshape(G, -1)
        k = g.shape[1]
        mean = g.sum(-1, keepdim=True) / k
        var = ((g - mean) ** 2).sum(-1, keepdim=True) / k
        s1, s2 = g.abs().sum(-1, keepdim=True) / k, (g * g).sum(-1, keepdim=True) / k
        dmean = u * s1
        dvar = u * (s2 + 2 * mean.abs() * s1) + dmean * dmean
        e = ((dmean + (g - mean).abs() * dvar / (2 * (var + eps))) / torch.sqrt(var + eps)).reshape(C, n).T * gamma.abs()
        if film is not None:
            e = e * (1 + film[b, :C]).abs()
        out[b, :n] = e
    return out


def affine_terms(x: torch.Tensor, G: int, gamma, beta, rows: Sequence[int], film: Optional[torch.Tensor], eps: float) -> torch.Tensor:
    """The kernel's fp32 uncentred affine y = fma(x, a, b) with a = gamma rstd (1 + s), b = (beta - mean gamma rstd)(1 + s) + shift:
    a few roundings of |x a| and |b|, which for a group offset r carry r |gamma (1 + s)| of the output - 8 * 2^-24 of those, plus
    2^-17 |y| of the bf16 hi/lo split of the output."""
    B, T, C = x.shape
    out = torch.zeros_like(x)
    for b in range(B):
        n = int(rows[b])
        g = x[b, :n].T.reshape(G, -1)
        k = g.shape[1]
        mean = g.sum(-1, keepdim=True) / k
        var = ((g - mean) ** 2).sum(-1, keepdim=True) / k
        a = (1.0 / torch.sqrt(var + eps)).expand(G, k).reshape(C, n).T * gamma
        m = mean.expand(G, k).reshape(C, n).T
        fs = (1 + film[b, :C]) if film is not None else 1.0
        fb = film[b, C:2 * C] if film is not None else 0.0
        bb = (beta - m * a) * fs + fb
        y = x[b, :n] * a * fs + bb
        out[b, :n] = 8 * 2.0 ** -24 * ((x[b, :n] * a * fs).abs() + bb.abs() + (beta * fs).abs()) + 2.0 ** -17 * y.abs()
    return out


def layer_norm_rows(x: torch.Tensor, gamma, beta, eps: float) -> torch.Tensor:
    """LayerNorm over the last dim in x's dtype"""
    return torch.nn.functional.layer_norm(x, (x.shape[-1],), gamma.to(x.dtype), beta.to(x.dtype), eps)


def depthwise7(x: torch.Tensor, dw: torch.Tensor, L: Sequence[int]) -> torch.Tensor:
    """ConvNeXt's depthwise conv (k = 7, padding 3) of token-major x [B, T, C] with dw [C, 8] (taps, bias), rows >= L[b] of the
    input read as 0"""
    B, T, C = x.shape
    xm = x.clone()
    for b in range(B):
        xm[b, int(L[b]):] = 0
    w = dw[:, :7].to(x.dtype)[:, None, :]
    return torch.nn.functional.conv1d(xm.transpose(1, 2), w, dw[:, 7].to(x.dtype), padding=3, groups=C).transpose(1, 2)


def sinusoid(t: torch.Tensor, K: int, flip: bool, freq_shift: float) -> torch.Tensor:
    """the timestep embedding of embeddings.py:24-64 in t's dtype: [sin | cos] (flipped: [cos | sin]) of t * 10^(-4 i / (half -
    shift)), zero-padded to an odd K"""
    half = K // 2
    ex = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=t.dtype, device=t.device) / (half - freq_shift))
    arg = t[:, None] * ex[None, :]
    emb = torch.cat([torch.cos(arg), torch.sin(arg)] if flip else [torch.sin(arg), torch.cos(arg)], -1)
    return torch.nn.functional.pad(emb, (0, K - 2 * half))


def small_linear(xin: torch.Tensor, W, bias, add: Optional[torch.Tensor], add_rows: int, out_silu: bool) -> torch.Tensor:
    """xin [M, K] (already through the input mode) @ W^T + bias (+ add row m % add_rows, or m) (then SiLU), in xin's dtype"""
    y = xin @ W.to(xin.dtype).T
    if bias is not None:
        y = y + bias.to(xin.dtype)
    if add is not None:
        idx = torch.arange(xin.shape[0], device=xin.device)
        y = y + add.to(xin.dtype)[idx % add_rows if add_rows > 0 else idx]
    return y * torch.sigmoid(y) if out_silu else y


def pool_attend(q: torch.Tensor, kv: torch.Tensor, heads: int, keys: Sequence[int]) -> torch.Tensor:
    """AttentionPooling's attention (embeddings.py:521-546): q [B, C], kv [B, S1, 2C]; entry b over its first keys[b] rows; both
    q and k scaled by dph^-1/4; in q's dtype"""
    B, C = q.shape
    dph = C // heads
    s4 = 1.0 / math.sqrt(math.sqrt(dph))
    out = torch.zeros_like(q)
    for b in range(B):
        n = int(keys[b])
        qh = (q[b] * s4).reshape(heads, dph)
        k = (kv[b, :n, :C] * s4).reshape(n, heads, dph)
        v = kv[b, :n, C:].reshape(n, heads, dph)
        w = torch.softmax(torch.einsum("hd,nhd->hn", qh, k), -1)
        out[b] = torch.einsum("hn,nhd->hd", w, v).reshape(C)
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# The content encoder's first conv and positional conv, the vocoder's ISTFT (tests/test_audio_kernels_fp64.py).  The truth of
# each is the pinned oracle's stage (content_oracle.conv_layer / pos_conv, vocos_oracle.head_istft); these restate the same
# operations with a switch per defect, so the tests can show each bound would notice it, and derive the design's error terms.
# ---------------------------------------------------------------------------------------------------------------------------
U32 = 2.0 ** -24


def conv0_rows(wav: torch.Tensor, n: int, w0: torch.Tensor, gamma, beta, eps: float, padded_stats: bool = False,
               unbiased: bool = False, use_eps: bool = True) -> torch.Tensor:
    """conv 0 (k 10, s 5) -> GroupNorm(C0, C0) -> erf-GELU of one row's first n samples of wav [>= n], [T0, C0] in wav's dtype.
    Defects: padded_stats (the statistics over the frames of the whole zero-padded wav instead of the row's own), unbiased
    (variance over T0 - 1), use_eps=False (eps dropped)."""
    x = wav.clone()
    x[n:] = 0
    T0 = (n - 10) // 5 + 1
    y = torch.nn.functional.conv1d(x[None, None], w0.to(x.dtype), stride=5)[0]          # [C0, frames of the whole wav]
    ys = y if padded_stats else y[:, :T0]
    mean = ys.mean(-1, keepdim=True)
    var = ys.var(-1, unbiased=unbiased, keepdim=True)
    z = (y[:, :T0] - mean) / torch.sqrt(var + (eps if use_eps else 0.0)) * gamma.to(x.dtype)[:, None] + beta.to(x.dtype)[:, None]
    return gelu_erf(z).T


def conv0_fp32(wav: torch.Tensor, n: int, w0: torch.Tensor) -> torch.Tensor:
    """The kernel's fp32 conv 0 of a row, emulated: y = fmaf(w[j], x[5t + j], y) for j = 0 .. 9, each step rounded to fp32 once
    (the fp64 sum of an exact fp64 product and an fp32 value, then rounded: the same value but for a double rounding in 2^-29 of
    the steps).  [C0, T0] as fp64."""
    T0 = (n - 10) // 5 + 1
    x = wav[:5 * (T0 - 1) + 10].to(F64)
    cols = torch.stack([x[j:j + 5 * (T0 - 1) + 1:5] for j in range(10)])                # [10, T0]
    w = w0.reshape(w0.shape[0], 10).to(F64)
    y = torch.zeros(w.shape[0], T0, dtype=F64, device=x.device)
    for j in range(10):
        y = (w[:, j:j + 1] * cols[j][None] + y).float().to(F64)
    return y


def conv0_stats_tol(y32: torch.Tensor) -> tuple:
    """What the kernel's stored (mean, 1 / std) may differ from the fp64 statistics of its own fp32 conv y32 [C0, T0]: the fp32
    rounding of each (2^-24 relative), and the one-pass fp64 sums (32 time lanes of T0 / 32 frames, then the lanes in order:
    (T0 / 32 + 32) 2^-53 of sum |y| and sum y^2, which the variance q / T0 - mean^2 carries relative to mean^2 + var).
    Returns (mean, var, mean_tol, var_err), each [C0]: var_err bounds the fp64 sums' error in the variance."""
    T0 = y32.shape[1]
    mean = y32.mean(-1)
    var = y32.var(-1, unbiased=False)
    n_add = T0 / 32 + 34
    mean_tol = U32 * mean.abs() + n_add * 2.0 ** -53 * y32.abs().mean(-1)
    return mean, var, mean_tol, n_add * 2.0 ** -52 * (mean * mean + var)


def conv0_terms(wav: torch.Tensor, n: int, w0: torch.Tensor, gamma, beta, eps: float) -> torch.Tensor:
    """The design's error terms of cv_gn_stats + cv_conv0 against the fp64 truth, per output of one row ([T0, C0]):
      * the fp32 conv, ten fmaf in tap order: d = 10 2^-24 sum_j |w_j| |x_5t+j|, at the output and in each statistic;
      * the fp32 mean and the fp32 subtraction y - mean: 2^-24 (|mean| + |y - mean|);
      * rstd: its fp32 rounding, the conv's error in the variance (2 std max d + max d^2) and the fp64 one-pass sums
        (conv0_stats_tol), relative to var + eps;
    all times rstd |gamma|, then the affine's two fp32 roundings, GELU's slope (< 1.13) and erff / its products (4 2^-24 of
    |z| + |GELU(z)|), and 2^-17 |out| of the bf16 hi/lo split.  Under a DC offset the first two are
    (10 sum |w||x| + |mean|) 2^-24 rstd |gamma|: the cancellation the design accepts."""
    T0 = (n - 10) // 5 + 1
    x = wav[:5 * (T0 - 1) + 10].to(F64)
    y = torch.nn.functional.conv1d(x[None, None], w0.to(F64), stride=5)[0]                # [C0, T0]
    d = 10 * U32 * torch.nn.functional.conv1d(x.abs()[None, None], w0.to(F64).abs(), stride=5)[0]
    mean = y.mean(-1, keepdim=True)
    var = y.var(-1, unbiased=False, keepdim=True)
    dmax = d.amax(-1, keepdim=True)
    _, _, _, var_sum = conv0_stats_tol(y)
    rstd = 1.0 / torch.sqrt(var + eps)
    drel = U32 + (2 * torch.sqrt(var) * dmax + dmax * dmax + var_sum[:, None]) / (2 * (var + eps))
    g = gamma.to(F64).abs()[:, None]
    yh = (y - mean) * rstd
    z = yh * gamma.to(F64)[:, None] + beta.to(F64)[:, None]
    dz = g * rstd * (d + dmax + U32 * (mean.abs() + (y - mean).abs())) + g * yh.abs() * drel + 2 * U32 * ((g * yh).abs() + z.abs())
    out = gelu_erf(z)
    return (1.13 * dz + 4 * U32 * (z.abs() + out.abs()) + 2.0 ** -17 * out.abs()).T


def pos_conv_rows(x: torch.Tensor, W: torch.Tensor, bias, L: Sequence[int], shift: int = 0, keep_last: bool = False) -> torch.Tensor:
    """x + GELU(SamePad(pos_conv(x))) of token-major x [B, T, D] (W [D, D / G, K], bias [D]), row b on its first L[b] frames,
    rows at or past L[b] equal to x.  In x's dtype.  Defects: shift (every tap reads one frame later), keep_last (SamePad's
    dropped frame kept: row L[b] gets a conv output too)."""
    B, T, D = x.shape
    K, gw = W.shape[-1], W.shape[1]
    out = x.clone()
    for b in range(B):
        n = int(L[b])
        xb = torch.zeros(n + K + 2, D, dtype=x.dtype, device=x.device)
        xb[:n] = x[b, :n]
        # output t reads x[t - K / 2 + j + shift], j < K: pad K / 2 - shift in front
        front = K // 2 - shift
        xp = torch.cat([torch.zeros(front, D, dtype=x.dtype, device=x.device), xb], 0).T[None]
        y = torch.nn.functional.conv1d(xp, W.to(x.dtype), bias.to(x.dtype), groups=D // gw)[0].T
        m = min(n + (1 if keep_last else 0), T)
        out[b, :m] = x[b, :m] + gelu_erf(y[:m])
    return out


def pos_conv_terms(x: torch.Tensor, W: torch.Tensor, bias, L: Sequence[int]) -> torch.Tensor:
    """The design's error terms of the positional conv per output: the 3xBF16 product of the split windows and split weights
    (each split exact to 2^-17 relative, the lo x lo product left out: 3 2^-18 of sum |w||x|), the fp32 accumulation over the
    4 K k-steps of 16 (worst case (4 K + 16) 2^-24 of sum |w||x|), carried through GELU's slope with the epilogue's
    polynomial erf (4e-7 (1 + |v|)) and its roundings, and the fp32 residual add (2^-24 |out|).  Rows past L[b]: 0 (exact)."""
    B, T, D = x.shape
    K, gw = W.shape[-1], W.shape[1]
    out = torch.zeros_like(x, dtype=F64)
    for b in range(B):
        n = int(L[b])
        xp = torch.nn.functional.pad(x[b, :n].to(F64).T[None], (K // 2, K // 2))
        v = torch.nn.functional.conv1d(xp, W.to(F64), bias.to(F64), groups=D // gw)[0].T[:n]
        a = torch.nn.functional.conv1d(xp.abs(), W.to(F64).abs(), groups=D // gw)[0].T[:n]
        e = (3 * 2.0 ** -18 + (4 * K + 16) * U32) * a + 2 * U32 * v.abs()
        e = gelu_erf_slope(v).abs() * e + 4e-7 * (1 + v.abs()) + 4 * U32 * gelu_erf(v).abs()
        out[b, :n] = e + U32 * (x[b, :n].to(F64) + gelu_erf(v)).abs()
    return out


def istft_rows(h: torch.Tensor, window: torch.Tensor, hop: int, L: Sequence[int], env_all_frames: bool = False,
               reverse_window: bool = False, clip_first: bool = False) -> torch.Tensor:
    """The ISTFT head of h [B, T, >= n_fft + 2] (log-magnitudes, then phases), row b alone on its first L[b] frames, zero past
    L[b] hop samples: [B, T hop] in h's dtype.  Defects: env_all_frames (the envelope counts all T frames), reverse_window,
    clip_first (clip(h, max=100) before exp instead of clip(exp(h), max=100))."""
    B, T, _ = h.shape
    n = window.numel()
    nb, pad = n // 2 + 1, (n - hop) // 2
    w = window.to(h.dtype).flip(0) if reverse_window else window.to(h.dtype)
    out = torch.zeros(B, T * hop, dtype=h.dtype, device=h.device)
    for b in range(B):
        Lb = int(L[b])
        lm, p = h[b, :Lb, :nb], h[b, :Lb, nb:2 * nb]
        mag = torch.exp(torch.clip(lm, max=100.0)) if clip_first else torch.clip(torch.exp(lm), max=1e2)
        S = mag * (torch.cos(p) + 1j * torch.sin(p))
        frames = torch.fft.irfft(S, n, dim=-1) * w                                        # [Lb, n]
        Le = T if env_all_frames else Lb
        y = torch.nn.functional.fold(frames.T[None], (1, (Lb - 1) * hop + n), (1, n), stride=(1, hop))[0, 0, 0]
        env = torch.nn.functional.fold((w * w)[None, :, None].expand(1, n, Le), (1, (Le - 1) * hop + n), (1, n), stride=(1, hop))[0, 0, 0]
        out[b, :Lb * hop] = y[pad:pad + Lb * hop] / env[pad:pad + Lb * hop]
    return out



# ---------------------------------------------------------------------------------------------------------------------------
# Prompt-mel front end: resample_kernel and log_mel_kernel (csrc/frontend.cu), tests/test_frontend_kernels_fp64.py.  Each
# reference takes one row alone, in fp64 on the kernel's own fp32 input and fp32 tables, with a switch per defect so the tests
# can show each bound would notice it.
# ---------------------------------------------------------------------------------------------------------------------------
U53 = 2.0 ** -53
MEL_CLIP = float(torch.tensor(1e-7, dtype=torch.float32))          # the kernel's 1e-7f; torch.clip(fp32, 1e-7) clips at it too


def resample_trim(table: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(first, last) nonzero tap of each phase of a [nw, taps] table: the range the kernel's loop runs over"""
    nz = table != 0
    taps = table.shape[1]
    idx = torch.arange(taps, device=table.device)
    lo = torch.where(nz, idx, taps).amin(1)
    hi = torch.where(nz, idx, -1).amax(1)
    return lo, hi


def resample_width(orig: int, nw: int) -> int:
    """lowpass width of the reduced ratio orig:nw, ceil(6 orig / (0.99 min(orig, nw))) as the host computes it; 0 for the
    identity"""
    return 0 if orig == nw else math.ceil(6.0 * orig / (min(orig, nw) * 0.99))


def sinc_table64(orig: int, nw: int, width: int) -> torch.Tensor:
    """torchaudio's phase table of the reduced ratio orig:nw built for lowpass width `width` (fp32 phase offsets, the rest in
    fp64, not rounded): [nw, 2 width + orig] fp64.  At the ratio's own width it is the fp64 value of the handle's table."""
    base = min(orig, nw) * 0.99
    idx = torch.arange(-width, width + orig, dtype=F64)[None] / orig
    t = (torch.arange(0, -nw, -1, dtype=torch.float32)[:, None] / nw).to(F64) + idx
    t = (t * base).clamp(-6, 6)
    window = torch.cos(t * math.pi / 6 / 2) ** 2
    t = t * math.pi
    k = torch.where(t == 0, torch.ones((), dtype=F64), t.sin() / t)
    return k * (window * (base / orig))


def resample_out_len(orig: int, nw: int, n: int) -> int:
    """ceil(fp32(nw n / orig)), the fp64 quotient rounded to fp32 (torchaudio's length rule); n for the identity"""
    if orig == nw:
        return n
    return int(math.ceil(float(torch.tensor(nw * n / orig, dtype=torch.float32))))


def _resample_windows(x: torch.Tensor, L: int, orig: int, width: int, taps: int, K: int, shift: int = 0) -> torch.Tensor:
    """[K, taps] fp64: window k holds x[k orig - width + shift + i], i < taps, zero outside [0, L)"""
    front = width + 1
    xp = torch.zeros(front + (K - 1) * orig + taps + 2, dtype=F64, device=x.device)
    n = max(0, min(L, xp.numel() - front))
    xp[front:front + n] = x[:n].to(F64)
    return xp[1 + shift:].unfold(0, taps, orig)[:K]


def resample_rows(x: torch.Tensor, L: int, table: torch.Tensor, orig: int, nw: int, width: int, n_out: int, shift: int = 0,
                  phase_plus_one: bool = False, width_delta: int = 0, fp32_acc: bool = False) -> torch.Tensor:
    """One row of resample_kernel: output j < L_out (the length rule at the row's L) is sum_i table[j mod nw][i] x[(j div nw) orig
    - width + i] over the row's first L samples, later outputs 0.  [n_out] fp64.  table [nw, taps] (fp32 values: truth A; the
    fp64 table: truth B's arithmetic).  Defects: shift (every tap reads one input sample later), phase_plus_one (phase p reads
    table row p + 1), width_delta (a table built for width + delta applied at the handle's width), fp32_acc (the sum in fp32,
    one fmaf per tap in tap order)."""
    if width_delta:
        table = sinc_table64(orig, nw, width + width_delta)
    if phase_plus_one:
        table = table.roll(-1, 0)
    taps = table.shape[1]
    L_out = min(resample_out_len(orig, nw, L), n_out)
    out = torch.zeros(n_out, dtype=F64, device=x.device)
    if L_out <= 0:
        return out
    K = (L_out + nw - 1) // nw
    win = _resample_windows(x, L, orig, width, taps, K, shift)
    w = table.to(F64)
    if fp32_acc:
        acc = torch.zeros(K, nw, dtype=F64, device=x.device)
        for i in range(taps):
            acc = (win[:, i:i + 1] * w[None, :, i] + acc).float().to(F64)
        y = acc
    else:
        y = win @ w.T
    out[:L_out] = y.reshape(-1)[:L_out]
    return out


def resample_abs_sum(x: torch.Tensor, L: int, table: torch.Tensor, orig: int, nw: int, width: int, n_out: int) -> torch.Tensor:
    """sum_i |table[p][i]| |x[...]| of each output, the scale of every rounding of the convolution: [n_out] fp64"""
    return resample_rows(x.abs(), L, table.abs(), orig, nw, width, n_out)


def resample_terms_a(y: torch.Tensor, absum: torch.Tensor, taps: int) -> torch.Tensor:
    """The kernel's error against truth A (the fp64 convolution on its own fp32 table), per output: it multiplies and adds in
    fp64 (each fma rounds at 2^-53 of a partial sum no larger than sum |w||x|: taps 2^-53 sum |w||x|) and rounds once to fp32
    (2^-24 |y|, and 2^-150 below fp32's normal range).  The fp64 reference's own summation adds the same taps 2^-53 sum |w||x|
    again."""
    return U32 * y.abs() + 2 * taps * U53 * absum + 2.0 ** -150


def resample_terms_b(absum: torch.Tensor) -> torch.Tensor:
    """What truth B (the recipe in fp64 on the fp64 table) adds to the parity rule: the table's rounding to fp32, 2^-24 of each
    |w|, so 2^-24 sum |w||x|"""
    return U32 * absum


def _reflect_index(L: int, F: int, frame_offset: int = 0, about_L: bool = False, device=None) -> torch.Tensor:
    """[F, 1024] sample index of tap t of frame f: 256 f + t - 512 reflected about sample 0 and about sample L - 1 (center=True,
    pad_mode='reflect'), clamped into the row as the kernel does.  Defects: frame_offset (frames start that many samples
    later), about_L (the right end reflected about L instead of L - 1)."""
    p = torch.arange(F, device=device)[:, None] * 256 + torch.arange(1024, device=device)[None, :] - 512 + frame_offset
    s = p.abs()
    s = torch.where(s >= L, (2 * L if about_L else 2 * (L - 1)) - s, s)
    return s.clamp(0, L - 1)


def log_mel_frames(L: int, S: int) -> int:
    """frames log_mel_kernel computes for a row of L samples in a launch of S frames"""
    return min(1 + L // 256, S)


def mel_band_bins(fb: torch.Tensor) -> torch.Tensor:
    """[100] bins from each band's first to its last nonzero weight (the kernel's loop length; 0 for an all-zero band)"""
    lo, hi = resample_trim(fb.T)
    return (hi - lo + 1).clamp_min(0)


def log_mel_rows(x: torch.Tensor, L: int, window: torch.Tensor, fb: torch.Tensor, S: int, reflect_about_L: bool = False,
                 frame_offset: int = 0, symmetric_window: bool = False, band_shift: int = 0, power: int = 1,
                 clip: float = MEL_CLIP, tap_scale: Optional[Tuple[int, float]] = None, magnitudes: bool = False):
    """One row of log_mel_kernel: log(max(fb^T |rfft(window * frame)|, clip)) of the reflect-padded frames of x[:L], [100, S] fp64
    with frames past log_mel_frames(L, S) 0.  window [1024] and fb [513, 100] are the kernel's fp32 tables.  magnitudes=True
    also returns (|X| [F, 513], the windowed frames [F, 1024]).  Defects: reflect_about_L, frame_offset, symmetric_window (the
    symmetric Hann window in place of `window`), band_shift (every band one bin higher), power, clip, tap_scale (i, s):
    window tap i times s."""
    F = log_mel_frames(L, S)
    dev = x.device
    w = (torch.hann_window(1024, periodic=False, dtype=torch.float32) if symmetric_window else window).to(dev, F64).clone()
    if tap_scale is not None:
        w[tap_scale[0]] *= tap_scale[1]
    fr = x[:L].to(F64)[_reflect_index(L, F, frame_offset, reflect_about_L, dev)] * w                  # [F, 1024]
    mag = torch.fft.rfft(fr, dim=-1).abs()                                                              # [F, 513]
    fbd = fb.to(dev, F64)
    if band_shift:
        fbd = fbd.roll(band_shift, 0)
    mel = (mag ** power) @ fbd                                                                          # [F, 100]
    out = torch.zeros(100, S, dtype=F64, device=dev)
    out[:, :F] = torch.log(torch.clip(mel, min=clip)).T
    if magnitudes:
        return out, mag, fr
    return out


def _twiddles(n: int, count: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """(exact exp(-2 pi i k / n), the kernel's fp32 table of it) for k < count, complex128"""
    k = torch.arange(count, dtype=F64)
    ex = torch.complex(torch.cos(2 * math.pi * k / n), -torch.sin(2 * math.pi * k / n))
    return ex, torch.complex(ex.real.float().to(F64), ex.imag.float().to(F64))


def _l1(z: torch.Tensor) -> torch.Tensor:
    return z.real.abs() + z.imag.abs()


def _cmul_error(c: torch.Tensor, ex: torch.Tensor, t32: torch.Tensor) -> torch.Tensor:
    """What the kernel's fp32 complex product c x t32 (cmul: two products and a sum per part, or one of them fused) adds to
    the exact c x ex, given c exactly: the twiddle's own rounding |c| |t32 - ex|, 2^-24 of every product that is not exact (a
    factor 0 or +-1 is exact) and 2^-24 of each part of the result."""
    tr, ti = t32.real, t32.imag
    inexact_r = ((tr != 0) & (tr.abs() != 1)).to(F64)
    inexact_i = ((ti != 0) & (ti.abs() != 1)).to(F64)
    prods = (c.real.abs() + c.imag.abs()) * (tr.abs() * inexact_r + ti.abs() * inexact_i)
    return c.abs() * (t32 - ex).abs() + U32 * prods + U32 * _l1(c * ex)


def fft_magnitude_bound(fr: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """|rfft| [F, 513] of windowed frames fr [F, 1024] (fp64 products of the kernel's fp32 samples and window) and, per bin,
    a bound on how far log_mel_kernel's fp32 magnitude may lie from it.

    The bound follows the kernel's own passes in fp64, carrying per node an error bound E next to the exact node value:
      * z[q] = x[2q] w[2q] + i x[2q+1] w[2q+1], rounded to fp32: E = 2^-24 (|Re z| + |Im z|), stored bit-reversed;
      * each radix-2 stage (half = 1 .. 256): a, c -> a +- c W, W the fp32 twiddle.  E(c W) = E(c) (1 + u) + _cmul_error, and
        each output adds E(a) + E(c W) + 2^-24 of its parts (the fp32 add), times (1 + 2u) for the second-order terms;
      * the split step: Xe = (Z_k + conj Z_(512-k)) / 2 and Xo = (Z_k - conj Z_(512-k)) / 2i (the halving is exact), the
        product with the fp32 tw1024 and the sum / difference, each bounded the same way;
      * |X| = sqrtf(ar^2 + ai^2): two squares, a sum and the root, 3 2^-24 |X|.
    Every rounding is charged at the magnitude of the value it rounds, node by node, not at the frame's sum |x w|: a bin that
    is weak within a loud frame gets a bound of its own size wherever the passes leading to it carry little."""
    u = U32
    F, dev = fr.shape[0], fr.device
    z = torch.complex(fr[:, 0::2], fr[:, 1::2])                                                         # [F, 512]
    brev = torch.tensor([int(f"{i:09b}"[::-1], 2) for i in range(512)], device=dev)
    Z, E = z[:, brev], u * _l1(z)[:, brev]
    ex512, t512 = (t.to(dev) for t in _twiddles(512, 256))
    half = 1
    while half < 512:
        tws = 256 // half
        Zr, Er = Z.reshape(F, 512 // (2 * half), 2, half), E.reshape(F, 512 // (2 * half), 2, half)
        a, c, Ea, Ec = Zr[:, :, 0], Zr[:, :, 1], Er[:, :, 0], Er[:, :, 1]
        idx = torch.arange(half, device=dev) * tws
        ct = c * ex512[idx]
        Ect = Ec * (1 + u) + _cmul_error(c, ex512[idx], t512[idx])
        o0, o1 = a + ct, a - ct
        E0 = (Ea + Ect + u * _l1(o0)) * (1 + 2 * u)
        E1 = (Ea + Ect + u * _l1(o1)) * (1 + 2 * u)
        Z = torch.stack([o0, o1], 2).reshape(F, 512)
        E = torch.stack([E0, E1], 2).reshape(F, 512)
        half *= 2
    k = torch.arange(257, device=dev)
    n = (512 - k) % 512
    zk, zn, Ek, En = Z[:, k], Z[:, n], E[:, k], E[:, n]
    xe, xo = (zk + zn.conj()) / 2, (zk - zn.conj()) / 2j
    Exe, Exo = 0.5 * (Ek + En) + u * _l1(xe), 0.5 * (Ek + En) + u * _l1(xo)
    ex1024, t1024 = (t.to(dev) for t in _twiddles(1024, 257))
    wx = ex1024 * xo
    Ewx = Exo * (1 + u) + _cmul_error(xo, ex1024, t1024)
    Xk, Xn = xe + wx, xe - wx
    Bk = (Exe + Ewx + u * _l1(Xk)) * (1 + 2 * u) + 3 * u * Xk.abs()
    Bn = (Exe + Ewx + u * _l1(Xn)) * (1 + 2 * u) + 3 * u * Xn.abs()
    mag = torch.zeros(F, 513, dtype=F64, device=dev)
    bound = torch.zeros(F, 513, dtype=F64, device=dev)
    mag[:, :257], bound[:, :257] = Xk.abs(), Bk
    mag[:, 512 - k], bound[:, 512 - k] = Xn.abs(), Bn                                                   # bins 256 .. 512
    bound[:, 256] = torch.maximum(Bk[:, 256], Bn[:, 256])                                               # written twice
    return mag, bound


def log_mel_terms(x: torch.Tensor, L: int, window: torch.Tensor, fb: torch.Tensor, S: int):
    """The fp64 truth of log_mel_kernel on one row and the interval its fp32 output must lie in: (ref, lo, hi), each [100, S].

    Magnitude per bin: fft_magnitude_bound, the kernel's FFT, split step and |.| followed node by node.  Band m: sum fb x the
    magnitude bound, plus the fmaf chain over its n_m bins from the first to the last nonzero weight, n_m 2^-24 sum fb M.  The
    interval [mel - d, mel + d] maps through log(max(., 1e-7f)), so an entry whose whole interval is clipped is exact, and then
    widens by logf's 1 ulp (2^-23 |log|)."""
    ref, _, fr = log_mel_rows(x, L, window, fb, S, magnitudes=True)
    F = fr.shape[0]
    mag, dM = fft_magnitude_bound(fr)
    fbd = fb.to(x.device, F64)
    mel = mag @ fbd
    d = dM @ fbd + mel_band_bins(fb).to(x.device, F64)[None, :] * U32 * ((mag + dM) @ fbd)
    lo_m, hi_m = (mel - d).clamp_min(MEL_CLIP), (mel + d).clamp_min(MEL_CLIP)
    lo, hi = ref.clone(), ref.clone()
    lo_l, hi_l = torch.log(lo_m), torch.log(hi_m)
    clipped = hi_m <= MEL_CLIP
    lo_l = torch.where(clipped, lo_l, lo_l - 2.0 ** -23 * lo_l.abs())
    hi_l = torch.where(clipped, hi_l, hi_l + 2.0 ** -23 * hi_l.abs())
    lo[:, :F], hi[:, :F] = lo_l.T, hi_l.T
    return ref, lo, hi


def interval_ratio(got: torch.Tensor, ref: torch.Tensor, lo: torch.Tensor, hi: torch.Tensor) -> torch.Tensor:
    """|got - ref| over the side of [lo, hi] it lies towards, elementwise (0 where got == ref, inf past a zero-width side)"""
    e = got.to(F64) - ref
    side = torch.where(e > 0, hi - ref, ref - lo)
    return torch.where(e == 0, torch.zeros_like(e), e.abs() / side)
