"""Drop-in sampler classes (generic Python path) against fixtures produced by the reference's own
DPM_Solver / UniPC classes; the host-side coefficient tables of the fused CUDA sampler against
the same classes through a Python emulation of the fused kernels' arithmetic; and the C-ABI structs
built from those tables.  CPU only."""
import ctypes as C

import pytest
import torch

from ns2vc_b200 import _lib, coefs
from ns2vc_b200 import dpm_solver as our_dpm
from ns2vc_b200 import uni_pc as our_upc
from ns2vc_b200.schedule import NoiseScheduleVP, interpolate_fn
from ns2vc_b200.synth import linear_betas


def toy(x, t, **kw):
    return torch.tanh(x) * 0.7 + 0.1 * torch.sin(t / 100.0)[:, None, None]


def test_schedule_bit_exact(gold):
    g = gold("schedule.pt")
    ns = NoiseScheduleVP("discrete", betas=linear_betas(1000))
    assert ns.total_N == 1000
    for steps in (10, 30, 50):
        e = g[steps]
        la = torch.stack([ns.marginal_log_mean_coeff(t) for t in e["ts"]]).reshape(-1)
        sg = torch.stack([ns.marginal_std(t) for t in e["ts"]]).reshape(-1)
        lm = torch.stack([ns.marginal_lambda(t) for t in e["ts"]]).reshape(-1)
        assert torch.equal(la, e["log_alpha"]) and torch.equal(sg, e["sigma"]) and torch.equal(lm, e["lam"])
        # vectorised query gives the same values as per-scalar queries
        assert torch.equal(ns.marginal_lambda(e["ts"]), e["lam"])
    assert torch.equal(ns.inverse_lambda(g["inverse_lambda"]["lam"]), g["inverse_lambda"]["t"])


def test_interpolate_extrapolates():
    xp = torch.tensor([[0.0, 1.0, 3.0]])
    yp = torch.tensor([[0.0, 2.0, 2.0]])
    x = torch.tensor([[-1.0], [0.0], [0.5], [1.0], [2.0], [3.0], [5.0]])
    assert torch.allclose(interpolate_fn(x, xp, yp).reshape(-1), torch.tensor([-2.0, 0.0, 1.0, 2.0, 2.0, 2.0, 2.0]))


def _dpm_cases(g):
    for key in g["out"]:
        if key.startswith("dpm|"):
            _, algo, method, order, steps, skip, stype = key.split("|")
            yield key, algo, method, int(order), int(steps), skip, stype


def test_dpm_solver_matches_reference(gold):
    """Kept modes (multistep, order <= 2, dpmsolver++, 'dpmsolver' solver type) are bit-equal to the reference's own class on
    every time grid; every other mode of the reference class is rejected loudly (SURVEY.md 8b)."""
    g = gold("toy_samplers.pt")
    ns = NoiseScheduleVP("discrete", betas=linear_betas(1000))
    kept = rejected = 0
    for key, algo, method, order, steps, skip, stype in _dpm_cases(g):
        supported = algo == "dpmsolver++" and method == "multistep" and order <= 2 and stype == "dpmsolver"
        fn = our_dpm.model_wrapper(toy, ns, model_type="x_start")
        if not supported:
            with pytest.raises(NotImplementedError):
                our_dpm.DPM_Solver(fn, ns, algorithm_type=algo).sample(
                    g["xT"], steps=steps, order=order, skip_type=skip, method=method, solver_type=stype)
            rejected += 1
            continue
        out = our_dpm.DPM_Solver(fn, ns, algorithm_type=algo).sample(
            g["xT"], steps=steps, order=order, skip_type=skip, method=method, solver_type=stype)
        assert torch.equal(out, g["out"][key]) if skip == "time_uniform" else torch.allclose(out, g["out"][key], rtol=1e-6, atol=1e-6), key
        kept += 1
    assert kept >= 3 and kept + rejected == 24, (kept, rejected)


def test_unipc_matches_reference(gold):
    g = gold("toy_samplers.pt")
    ns = our_upc.NoiseScheduleVP("discrete", betas=linear_betas(1000))
    kept = rejected = 0
    for key in g["out"]:
        if not key.startswith("unipc|"):
            continue
        _, variant, order, steps, algo = key.split("|")
        supported = algo == "data_prediction" and variant in ("bh1", "bh2") and int(order) == 2
        fn = our_upc.model_wrapper(toy, ns, model_type="x_start")
        if not supported:
            with pytest.raises(NotImplementedError):
                our_upc.UniPC(fn, ns, algorithm_type=algo, variant=variant).sample(
                    g["xT"], steps=int(steps), order=int(order), skip_type="time_uniform", method="multistep")
            rejected += 1
            continue
        out = our_upc.UniPC(fn, ns, algorithm_type=algo, variant=variant).sample(
            g["xT"], steps=int(steps), order=int(order), skip_type="time_uniform", method="multistep")
        assert torch.allclose(out, g["out"][key], rtol=1e-6, atol=1e-6), key
        kept += 1
    assert kept >= 2 and kept + rejected == 18, (kept, rejected)


# ---- Python emulation of the fused kernels (sampler.cu dpm_step_kernel / unipc_step_kernel) ----
def _rt(x, o, a, s):
    noise = (x - a * o) / s
    return (x - s * noise) / a


def _emulate_dpm(table, x, B):
    f = lambda v: torch.tensor(v, dtype=torch.float32)
    m_prev = None
    for st in table:
        out = toy(x, torch.full((B,), st.t_input, dtype=torch.float32))
        m0 = _rt(x, out, f(st.alpha_s), f(st.sigma_s))
        r = f(st.c_x) * x - f(st.c_m) * m0
        if st.order == 2:
            d1 = f(st.inv_r0) * (m0 - m_prev)
            r = r - f(st.c_d) * d1
        x, m_prev = r, m0
    return x


@pytest.mark.parametrize("steps", [6, 12, 50])
def test_dpm_coef_table_bit_exact(steps):
    ns = NoiseScheduleVP("discrete", betas=linear_betas(1000))
    xT = torch.randn((2, 5, 33), generator=torch.Generator().manual_seed(5))
    ts = torch.linspace(1.0, 1e-3, steps + 1)
    table = coefs.dpmpp_2m_table(ns, ts)
    assert len(table) == steps and table[0].order == 1
    fn = our_dpm.model_wrapper(toy, ns, model_type="x_start")
    ref = our_dpm.DPM_Solver(fn, ns, algorithm_type="dpmsolver++").sample(xT, steps=steps, order=2, skip_type="time_uniform", method="multistep")
    assert torch.equal(_emulate_dpm(table, xT, 2), ref)


def _emulate_unipc(table, x, B):
    f = lambda v: torch.tensor(v, dtype=torch.float32)
    x_prev, x_eval, m0, m1 = x, x, None, None
    for st in table:
        out = toy(x_eval, torch.full((B,), st.t_input, dtype=torch.float32))
        mt = _rt(x_eval, out, f(st.alpha_t), f(st.sigma_t))
        xt = x_eval
        if st.corr_order > 0:
            xbar = f(st.c_x) * x_prev - f(st.c_m) * m0
            d1t = mt - m0
            if st.corr_order == 2:
                inner = f(st.rho0) * ((m1 - m0) / f(st.rk)) + f(st.rho1) * d1t
            else:
                inner = f(st.rho1) * d1t
            xt = xbar - f(st.ab) * inner
        nbar = f(st.n_c_x) * xt - f(st.n_c_m) * mt
        xpred = nbar
        if st.pred_order == 2:
            xpred = nbar - f(st.nab) * (f(0.5) * ((m0 - mt) / f(st.nrk)))
        m1, m0 = m0, mt
        x_prev, x_eval = xt, xpred
    return x_eval


@pytest.mark.parametrize("steps,variant", [(8, "bh2"), (30, "bh2"), (5, "bh1")])
def test_unipc_coef_table_bit_exact(steps, variant):
    ns = our_upc.NoiseScheduleVP("discrete", betas=linear_betas(1000))
    xT = torch.randn((1, 5, 33), generator=torch.Generator().manual_seed(6))
    ts = torch.linspace(1.0, 1e-3, steps + 1)
    table = coefs.unipc_bh2_table(ns, ts, variant)
    fn = our_upc.model_wrapper(toy, ns, model_type="x_start")
    ref = our_upc.UniPC(fn, ns, variant=variant).sample(xT, steps=steps, order=2, skip_type="time_uniform", method="multistep")
    assert torch.equal(_emulate_unipc(table, xT, 1), ref)


# ---- the C-ABI structs of the step records ----
def _positional(st):
    """The struct of a step record with its fields written out in the order of include/ns2vc_b200.h."""
    if isinstance(st, coefs.DpmStep):
        return _lib.DpmCoef(st.alpha_s, st.sigma_s, st.c_x, st.c_m, st.c_d, st.inv_r0, st.order)
    if isinstance(st, coefs.UniPcStep):
        return _lib.UniPcCoef(st.alpha_t, st.sigma_t, st.c_x, st.c_m, st.ab, st.rk, st.rho0, st.rho1, st.corr_order,
                              st.n_c_x, st.n_c_m, st.nab, st.nrk, st.pred_order)
    if isinstance(st, coefs.DdpmStep):
        return _lib.DdpmCoef(st.c_x0, st.c_x, st.c_noise, int(st.add_noise))
    return _lib.DdimCoef(st.sqrt_recip, st.sqrt_recipm1, st.sqrt_alpha_next, st.c, st.sigma, int(st.last))


def test_c_structs_fill_every_field_by_name():
    ns = NoiseScheduleVP("discrete", betas=linear_betas(1000))
    buf = coefs.diffusion_buffers(1000)
    tables = []
    for steps in (6, 20):                      # lower-order final steps at 6, none at 20
        ts = torch.linspace(1.0, 1e-3, steps + 1)
        tables += [coefs.dpmpp_2m_table(ns, ts), coefs.unipc_bh2_table(ns, ts)]
    tables += [coefs.ddpm_table(buf, range(999, -1, -1)), coefs.ddpm_table(buf, range(999, -1, -111))]
    tables += [coefs.ddim_table(buf, 1000, 6, 0.0), coefs.ddim_table(buf, 1000, 50, 0.5)]
    for tab in tables:
        want = [bytes(_positional(s)) for s in tab]
        assert [bytes(coefs.c_struct(s)) for s in tab] == want, type(tab[0]).__name__
        table, size = coefs.c_table(tab, "cpu")
        assert size == len(want[0]) and table.numpy().tobytes() == b"".join(want)
