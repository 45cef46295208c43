"""Host-side per-step sampler coefficients for the fused CUDA sampler steps.

Nothing in DPM-Solver++ / UniPC depends on the data except the element-wise tensor updates
(SURVEY.md Appendix A), so every scalar of every step is computed once, on the CPU, with the
same fp32 torch ops in the same order as the reference evaluates them per step
(``sampler/dpm_solver.py:796-852, 547-580, 271-298, 433-442``; ``sampler/uni_pc.py:471-588``).
The reference spends ~165 micro-kernels per step on this (SURVEY §2.3 K17).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List, Tuple

import torch

from . import _lib
from .schedule import NoiseScheduleVP


def _f(x) -> float:
    return float(x.reshape(-1)[0].item()) if torch.is_tensor(x) else float(x)


@dataclass
class DpmStep:
    t_input: float      # model time fed to the UNet (fractional, reference dpm_solver.py:278)
    alpha_s: float
    sigma_s: float
    c_x: float = 0.0
    c_m: float = 0.0
    c_d: float = 0.0
    inv_r0: float = 0.0
    order: int = 0


def model_input_time(ns: NoiseScheduleVP, t: torch.Tensor) -> torch.Tensor:
    if ns.schedule == "discrete":
        return (t - 1.0 / ns.total_N) * ns.total_N
    return t


def dpmpp_2m_table(ns: NoiseScheduleVP, ts: torch.Tensor, lower_order_final: bool = True, order: int = 2) -> List[DpmStep]:
    """ts: the N+1 CPU time points (fp32).  Entry k = evaluate the model at ts[k] (x0 round trip
    with alpha/sigma at ts[k]) then advance x to ts[k+1] with DPM-Solver++ order 1 (k=0) or 2."""
    ts = ts.detach().to("cpu", torch.float32)
    N = ts.shape[0] - 1
    out: List[DpmStep] = []
    for k in range(N):
        s, t = ts[k], ts[k + 1]
        te = s.expand(1)
        st = DpmStep(t_input=_f(model_input_time(ns, te)), alpha_s=_f(ns.marginal_alpha(te)), sigma_s=_f(ns.marginal_std(te)))
        step = k + 1
        max_order = order
        if step < max_order:
            k_order = step
        elif lower_order_final and N < 10:
            k_order = min(max_order, N + 1 - step)
        else:
            k_order = max_order
        lam_s, lam_t = ns.marginal_lambda(s), ns.marginal_lambda(t)
        h = lam_t - lam_s
        sigma_s, sigma_t = ns.marginal_std(s), ns.marginal_std(t)
        alpha_t = torch.exp(ns.marginal_log_mean_coeff(t))
        phi_1 = torch.expm1(-h)
        st.c_x = _f(sigma_t / sigma_s)
        st.c_m = _f(alpha_t * phi_1)
        st.order = k_order
        if k_order == 2:
            h_0 = lam_s - ns.marginal_lambda(ts[k - 1])
            r0 = h_0 / h
            st.inv_r0 = _f(1.0 / r0)
            st.c_d = _f(0.5 * (alpha_t * phi_1))
        out.append(st)
    return out


@dataclass
class UniPcStep:
    t_input: float
    alpha_t: float
    sigma_t: float
    c_x: float = 0.0
    c_m: float = 0.0
    ab: float = 0.0
    rk: float = 1.0
    rho0: float = 0.0
    rho1: float = 0.0
    corr_order: int = 0
    n_c_x: float = 0.0
    n_c_m: float = 0.0
    nab: float = 0.0
    nrk: float = 1.0
    pred_order: int = 0


def _unipc_scalars(ns: NoiseScheduleVP, t_hist: List[torch.Tensor], t: torch.Tensor, order: int, variant: str = "bh2"):
    """Scalars of one multistep_uni_pc_bh_update (data prediction) from history times to t."""
    t = t.view(-1)
    t0 = t_hist[-1]
    lam0, lam_t = ns.marginal_lambda(t0), ns.marginal_lambda(t)
    sg0, sg_t = ns.marginal_std(t0), ns.marginal_std(t)
    alpha_t = torch.exp(ns.marginal_log_mean_coeff(t))
    h = lam_t - lam0
    rks = []
    for i in range(1, order):
        lam_i = ns.marginal_lambda(t_hist[-(i + 1)])
        rks.append((lam_i - lam0) / h)
    rk_first = rks[0] if rks else None
    rks.append(1.0)
    rks = torch.tensor(rks)
    hh = -h
    h_phi_1 = torch.expm1(hh)
    B_h = hh if variant == "bh1" else torch.expm1(hh)
    R, b = [], []
    h_phi_k = h_phi_1 / hh - 1
    fact = 1
    for i in range(1, order + 1):
        R.append(torch.pow(rks, i - 1))
        b.append(h_phi_k * fact / B_h)
        fact *= (i + 1)
        h_phi_k = h_phi_k / hh - 1 / fact
    R = torch.stack(R)
    b = torch.cat(b)
    rhos_c = torch.tensor([0.5]) if order == 1 else torch.linalg.solve(R, b)
    return dict(c_x=_f(sg_t / sg0), c_m=_f(alpha_t * h_phi_1), ab=_f(alpha_t * B_h),
                rk=_f(rk_first) if rk_first is not None else 1.0, rhos_c=[float(v) for v in rhos_c])


def unipc_bh2_table(ns: NoiseScheduleVP, ts: torch.Tensor, variant: str = "bh2") -> List[UniPcStep]:
    """Entry k (k = 0..N-1) = evaluate the model at ts[k] (at x_pred_k; x_pred_0 = x_T), run the
    corrector at ts[k] (k >= 1) and the predictor to ts[k+1].  Order 2, lower_order_final=True:
    the predictor to the final point ts[N] is first order and is the returned sample."""
    ts = ts.detach().to("cpu", torch.float32)
    N = ts.shape[0] - 1
    out: List[UniPcStep] = []
    for k in range(N):
        te = ts[k].expand(1)
        st = UniPcStep(t_input=_f(model_input_time(ns, te)), alpha_t=_f(ns.marginal_alpha(te)), sigma_t=_f(ns.marginal_std(te)))
        # corrector at ts[k] from history ending at ts[k-1]
        if k >= 1:
            order = 1 if k == 1 else 2
            hist = [ts[k - 1]] if k == 1 else [ts[k - 2], ts[k - 1]]
            sc = _unipc_scalars(ns, hist, ts[k], order, variant)
            st.c_x, st.c_m, st.ab, st.rk = sc["c_x"], sc["c_m"], sc["ab"], sc["rk"]
            if order == 1:
                st.rho0, st.rho1 = 0.0, sc["rhos_c"][0]
            else:
                st.rho0, st.rho1 = sc["rhos_c"][0], sc["rhos_c"][1]
            st.corr_order = order
        # predictor from ts[k] to ts[k+1]; history after this step's evaluation ends at ts[k]
        step = k + 1
        p_order = 1 if step < 2 else min(2, N + 1 - step)
        hist = [ts[k]] if p_order == 1 else [ts[k - 1], ts[k]]
        sp = _unipc_scalars(ns, hist, ts[k + 1], p_order, variant)
        st.n_c_x, st.n_c_m, st.nab, st.nrk = sp["c_x"], sp["c_m"], sp["ab"], sp["rk"]
        st.pred_order = p_order
        out.append(st)
    return out


# ---------------------------------------------------------------------------------------------------------- DDPM / DDIM
def diffusion_buffers(timesteps: int = 1000) -> dict:
    """The schedule buffers of ``NaturalSpeech2.__init__`` (reference model.py:456-498): computed in fp64 from the linear beta
    schedule, then each cast to fp32 as ``register_buffer`` does."""
    scale = 1000 / timesteps
    betas = torch.linspace(scale * 0.0001, scale * 0.02, timesteps, dtype=torch.float64)
    alphas = 1. - betas
    alphas_cumprod = torch.cumprod(alphas, dim=0)
    alphas_cumprod_prev = torch.nn.functional.pad(alphas_cumprod[:-1], (1, 0), value=1.)
    posterior_variance = betas * (1. - alphas_cumprod_prev) / (1. - alphas_cumprod)
    f32 = lambda v: v.to(torch.float32)
    return {
        "betas": f32(betas),
        "alphas_cumprod": f32(alphas_cumprod),
        "sqrt_recip_alphas_cumprod": f32(torch.sqrt(1. / alphas_cumprod)),
        "sqrt_recipm1_alphas_cumprod": f32(torch.sqrt(1. / alphas_cumprod - 1)),
        "posterior_log_variance_clipped": f32(torch.log(posterior_variance.clamp(min=1e-20))),
        "posterior_mean_coef1": f32(betas * torch.sqrt(alphas_cumprod_prev) / (1. - alphas_cumprod)),
        "posterior_mean_coef2": f32((1. - alphas_cumprod_prev) * torch.sqrt(alphas) / (1. - alphas_cumprod)),
    }


def loss_buffers(timesteps: int = 1000, min_snr_gamma=None) -> dict:
    """The schedule buffers ``NaturalSpeech2.forward`` reads (reference model.py:461-498), fp64 then cast to fp32 as
    ``register_buffer`` does: ``sqrt_alphas_cumprod`` and ``sqrt_one_minus_alphas_cumprod`` (``q_sample``) and ``loss_weight``,
    the SNR ``alphas_cumprod / (1 - alphas_cumprod)``, clamped to ``min_snr_gamma`` when given (``min_snr_loss_weight=True``)."""
    scale = 1000 / timesteps
    betas = torch.linspace(scale * 0.0001, scale * 0.02, timesteps, dtype=torch.float64)
    alphas_cumprod = torch.cumprod(1. - betas, dim=0)
    snr = alphas_cumprod / (1 - alphas_cumprod)
    if min_snr_gamma is not None:
        snr = snr.clamp(max=min_snr_gamma)
    f32 = lambda v: v.to(torch.float32)
    return {
        "sqrt_alphas_cumprod": f32(torch.sqrt(alphas_cumprod)),
        "sqrt_one_minus_alphas_cumprod": f32(torch.sqrt(1. - alphas_cumprod)),
        "loss_weight": f32(snr),
    }


@dataclass
class DdpmStep:
    t_input: float      # model time: the integer timestep t
    c_x0: float         # posterior_mean_coef1[t]
    c_x: float          # posterior_mean_coef2[t]
    c_noise: float      # (0.5 * posterior_log_variance_clipped[t]).exp()
    add_noise: bool     # t > 0


def ddpm_table(buffers: dict, timesteps: List[int]) -> List[DdpmStep]:
    """One p_sample step (reference model.py:535-542) per integer t of a descending list (999 .. 0 for ``p_sample_loop``).
    The scalars are the fp32 buffer entries and the reference's fp32 ops on them (one-element CPU tensors: the reference's
    [B, 1, 1] extracts take the same scalar path)."""
    c1, c2, lv = buffers["posterior_mean_coef1"], buffers["posterior_mean_coef2"], buffers["posterior_log_variance_clipped"]
    out = []
    for t in timesteps:
        t = int(t)
        out.append(DdpmStep(t_input=float(t), c_x0=_f(c1[t]), c_x=_f(c2[t]), c_noise=_f((0.5 * lv[t:t + 1]).exp()), add_noise=t > 0))
    return out


def ddim_time_pairs(total: int, sampling_timesteps: int) -> List[tuple]:
    """(time, time_next) pairs of ``ddim_sample`` (reference model.py:570-572): an fp32 linspace truncated by ``.int()``, which
    differs from exact integer arithmetic for some counts (26, 52, 60, ...)."""
    times = torch.linspace(-1, total - 1, steps=sampling_timesteps + 1)
    times = list(reversed(times.int().tolist()))
    return list(zip(times[:-1], times[1:]))


@dataclass
class DdimStep:
    t_input: float
    time: int
    time_next: int
    alpha: float = 0.0
    alpha_next: float = 0.0
    sqrt_recip: float = 0.0       # sqrt_recip_alphas_cumprod[time]
    sqrt_recipm1: float = 0.0     # sqrt_recipm1_alphas_cumprod[time]
    sqrt_alpha_next: float = 0.0
    c: float = 0.0
    sigma: float = 0.0
    last: bool = False            # time_next < 0: the step returns x0


def ddim_table(buffers: dict, total: int, sampling_timesteps: int, eta: float = 0.0) -> List[DdimStep]:
    """The scalars of every ``ddim_sample`` pair (reference model.py:579-601), fp32 torch scalars in the reference's op order."""
    ac, sr, srm1 = buffers["alphas_cumprod"], buffers["sqrt_recip_alphas_cumprod"], buffers["sqrt_recipm1_alphas_cumprod"]
    out = []
    for time, time_next in ddim_time_pairs(total, sampling_timesteps):
        st = DdimStep(t_input=float(time), time=time, time_next=time_next, sqrt_recip=_f(sr[time]), sqrt_recipm1=_f(srm1[time]))
        if time_next < 0:
            st.last = True
        else:
            alpha, alpha_next = ac[time], ac[time_next]
            sigma = eta * ((1 - alpha / alpha_next) * (1 - alpha_next) / (1 - alpha)).sqrt()
            c = (1 - alpha_next - sigma ** 2).sqrt()
            st.alpha, st.alpha_next, st.sqrt_alpha_next = _f(alpha), _f(alpha_next), _f(alpha_next.sqrt())
            st.c, st.sigma = _f(c), _f(sigma)
        out.append(st)
    return out


# ---------------------------------------------------------------------------------------------------------- C-ABI structs
_C_STRUCTS = {DpmStep: _lib.DpmCoef, UniPcStep: _lib.UniPcCoef, DdpmStep: _lib.DdpmCoef, DdimStep: _lib.DdimCoef}


def c_struct(step):
    """The step's coefficient struct of the C-ABI (``ns2vc_dpm_coef``, ``ns2vc_unipc_coef``, ``ns2vc_ddpm_coef`` or
    ``ns2vc_ddim_coef``), every field taken by name from the step record."""
    cls = _C_STRUCTS[type(step)]
    return cls(**{name: int(getattr(step, name)) if ctype is C.c_int else getattr(step, name) for name, ctype in cls._fields_})


def c_table(steps, device) -> Tuple[torch.Tensor, int]:
    """The steps' structs back to back in a device byte table (the row steps and the DDPM / DDIM steps read their struct from
    device memory), and the size of one struct in bytes."""
    arr = (_C_STRUCTS[type(steps[0])] * len(steps))(*[c_struct(s) for s in steps])
    return torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(device), C.sizeof(arr) // len(steps)


def t_inputs(steps, B: int, device) -> torch.Tensor:
    """The model time of every step for each of B rows: [steps, B] fp32 on ``device``, the step-major rows of the FiLM table."""
    return torch.tensor([[s.t_input] * B for s in steps], dtype=torch.float32).to(device)
