"""DDPM (``p_sample_loop``) and DDIM (``ddim_sample``) on the fused device loop (reference model.py:456-603).

CPU: the schedule buffers and per-step scalars are bit-equal to the reference's; the oracle reproduces the short DDIM case of
tests/golden/ddpm_ddim.pt (written by the unmodified reference, oracle/make_golden_ddpm_ddim.py); ``install_diffusion`` patches the
two methods.  GPU: the step kernels are bit-exact, the session and the API reproduce the fixtures, the captured chunks are
bit-identical to the eager loop and leave the default generator where the reference's call sequence does."""
import inspect
import sys
import types
from fractions import Fraction

import pytest
import torch

from conftest import tiny_config, tiny_inputs
from ns2vc_b200 import coefs
from ns2vc_b200.arch import ns2vc_denoiser_config
from ns2vc_b200.synth import make_inputs, make_pre_inputs, make_pre_state_dict, make_state_dict, state_dict_checksum
from oracle import sampler_oracle

RTOL, ATOL = 1e-3, 1e-4
PRE_CFG = {"phoneme_encoder": dict(in_channels=256, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2),
           "prompt_encoder": dict(in_channels=100, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2)}


def close(a, b, rtol=RTOL, atol=ATOL):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    err = (a - b).abs()
    worst = (err / (atol + rtol * b.abs())).max().item()
    return worst <= 1.0, f"max_abs={err.max().item():.3e} worst err/tol={worst:.2f}"


def fixture_noise(k, n_steps, draws):
    """x_T and the per-step noise of a ddpm_ddim.pt case: every patched randn / randn_like call drew from one CPU generator, x_T
    first.  Rows of steps that draw nothing are zeros (not read)."""
    shape = (k["B"], 100, k["T"])
    g = torch.Generator().manual_seed(k["noise_seed"])
    xT = torch.randn(shape, generator=g)
    noise = torch.zeros((n_steps,) + shape)
    for i, d in enumerate(draws):
        if d:
            noise[i] = torch.randn(shape, generator=g)
    assert 1 + sum(draws) == k["n_draws"]
    return xT, noise


def case_draws(k):
    if k["method"] == "ddpm":
        return [t > 0 for t in range(999, -1, -1)]
    return [tn >= 0 for _t, tn in coefs.ddim_time_pairs(1000, k["steps"])]


# ------------------------------------------------------------------------------------------------------------------- CPU
def test_product_buffers_are_the_references(gold):
    b = coefs.diffusion_buffers(1000)
    ref = gold("ddpm_ddim.pt")["buffers"]
    for name, v in ref.items():
        assert v.dtype == torch.float32 and torch.equal(b[name], v), name
    for name, v in gold("p_sample.pt")["buffers"].items():
        assert torch.equal(b[name], v), name
    assert torch.equal(b["alphas_cumprod"], gold("ddim.pt")["alphas_cumprod"])
    o = sampler_oracle.OracleDDPM(1000)
    assert torch.equal(b["betas"], o.betas) and torch.equal(b["posterior_mean_coef1"], o.coef1)
    assert torch.equal(b["posterior_mean_coef2"], o.coef2) and torch.equal(b["posterior_log_variance_clipped"], o.log_var)


def test_ddpm_table_is_the_references_scalars(gold):
    buf = gold("ddpm_ddim.pt")["buffers"]
    ts = list(range(999, -1, -1))
    tab = coefs.ddpm_table(coefs.diffusion_buffers(1000), ts)
    for t, st in zip(ts, tab):
        bt = torch.full((2,), t, dtype=torch.long)                       # extract(): [B, 1, 1] gathers (model.py:414-417)
        lv = buf["posterior_log_variance_clipped"].gather(-1, bt).reshape(2, 1, 1)
        assert st.t_input == float(t) and st.add_noise == (t > 0)
        assert st.c_x0 == buf["posterior_mean_coef1"][t].item() and st.c_x == buf["posterior_mean_coef2"][t].item()
        assert st.c_noise == (0.5 * lv).exp()[0, 0, 0].item(), t
    assert [s.t_input for s in coefs.ddpm_table(coefs.diffusion_buffers(1000), range(999, 989, -1))] == [float(t) for t in range(999, 989, -1)]


@pytest.mark.parametrize("eta", [0.0, 0.5])
def test_ddim_table_is_the_references_scalars(gold, eta):
    buf = gold("ddpm_ddim.pt")["buffers"]
    ac = buf["alphas_cumprod"]
    for S in (1, 6, 10, 26, 52, 60, 100, 333, 1000):
        times = torch.linspace(-1, 999, steps=S + 1)                     # model.py:570-572
        times = list(reversed(times.int().tolist()))
        pairs = list(zip(times[:-1], times[1:]))
        tab = coefs.ddim_table(coefs.diffusion_buffers(1000), 1000, S, eta)
        assert [(s.time, s.time_next) for s in tab] == pairs
        for (time, time_next), st in zip(pairs, tab):
            assert st.t_input == float(time) and st.last == (time_next < 0)
            assert st.sqrt_recip == buf["sqrt_recip_alphas_cumprod"][time].item()
            assert st.sqrt_recipm1 == buf["sqrt_recipm1_alphas_cumprod"][time].item()
            if time_next < 0:
                continue
            alpha, alpha_next = ac[time], ac[time_next]
            sigma = eta * ((1 - alpha / alpha_next) * (1 - alpha_next) / (1 - alpha)).sqrt()
            c = (1 - alpha_next - sigma ** 2).sqrt()
            assert (st.alpha, st.alpha_next, st.sqrt_alpha_next) == (alpha.item(), alpha_next.item(), alpha_next.sqrt().item())
            assert (st.sigma, st.c) == (sigma.item(), c.item()), (S, time)
    # the fp32 linspace truncates differently from exact arithmetic at these counts: the pairs must come from the linspace
    for S in (26, 52):
        exact = [int(Fraction(-S + k * 1000, S)) for k in range(S + 1)]  # -1 + k * 1000 / S, truncated toward zero
        assert torch.linspace(-1, 999, steps=S + 1).int().tolist() != exact, S


def test_oracle_reproduces_the_short_ddim_case(gold):
    from oracle import ddpm_ddim_oracle, pre_model_oracle as po, unet_oracle
    g = gold("ddpm_ddim.pt")
    sd_u, sd_p = make_state_dict(ns2vc_denoiser_config(), seed=0), make_pre_state_dict(PRE_CFG, seed=0)
    assert state_dict_checksum(sd_u) == g["unet_checksum"] and state_dict_checksum(sd_p) == g["pre_checksum"]
    k = g["cases"]["ddim_eta"]
    assert k["eta"] == 0.5
    xT, noise = fixture_noise(k, k["steps"], case_draws(k))
    pin = make_pre_inputs(k["B"], k["T"], k["S"], ragged=True, seed=k["seed"])
    with torch.no_grad():
        content, prompt = po.pre_model_infer(sd_p, pin["c"], pin["refer"], pin["lengths"], pin["refer_lengths"], 6, 6)
        fn = lambda x, t: unet_oracle.denoiser_forward(sd_u, ns2vc_denoiser_config(), x, content, prompt, pin["refer_lengths"], t)
        got = ddpm_ddim_oracle.ddim_sample(fn, g["buffers"]["alphas_cumprod"], xT, 1000, k["steps"], k["eta"], iter(noise))
    assert (got - k["mel"]).abs().max().item() <= 2e-5


class _StubNaturalSpeech2:
    """The two methods with the reference's signatures (model.py:544, 563)."""

    def p_sample_loop(self, content, refer, lengths, refer_lengths, f0, uv, auto_predict_f0=True):
        raise AssertionError("not patched")

    def ddim_sample(self, content, refer, lengths, refer_lengths, f0, uv, auto_predict_f0=True):
        raise AssertionError("not patched")


def test_install_diffusion_replaces_both_methods(monkeypatch):
    import ns2vc_b200
    from ns2vc_b200 import diffusion
    monkeypatch.delitem(sys.modules, "model", raising=False)
    with pytest.raises(RuntimeError):
        ns2vc_b200.install_diffusion()                       # model.py not imported yet
    cls = type("NaturalSpeech2", (_StubNaturalSpeech2,), {})
    mod = types.ModuleType("model")
    mod.NaturalSpeech2 = cls
    monkeypatch.setitem(sys.modules, "model", mod)
    ns2vc_b200.install_diffusion()
    assert cls.p_sample_loop is diffusion.p_sample_loop and cls.ddim_sample is diffusion.ddim_sample
    for name in ("p_sample_loop", "ddim_sample"):
        assert inspect.signature(getattr(cls, name)) == inspect.signature(getattr(_StubNaturalSpeech2, name)), name


# ------------------------------------------------------------------------------------------------------------------- GPU
def make_unet(cfg, seed=0):
    from ns2vc_b200.unet import UNet1DConditionModel
    m = UNet1DConditionModel(in_channels=cfg.in_channels, out_channels=cfg.out_channels, block_out_channels=cfg.block_out_channels,
                             layers_per_block=list(cfg.layers_per_block), norm_num_groups=cfg.norm_num_groups,
                             cross_attention_dim=cfg.cross_attention_dim, attention_head_dim=cfg.num_heads,
                             addition_embed_type=cfg.addition_embed_type, addition_embed_type_num_heads=cfg.addition_embed_type_num_heads,
                             resnet_time_scale_shift=cfg.resnet_time_scale_shift)
    sd = make_state_dict(cfg, seed)
    m.load_state_dict(sd, strict=True)
    return m.to("cuda").eval(), sd


@pytest.fixture(scope="module")
def full_model():
    return make_unet(ns2vc_denoiser_config())


def session(m, inp):
    from ns2vc_b200.fused import DenoiserSession
    from oracle import unet_oracle
    content = inp["content"].permute(1, 2, 0).contiguous().cuda()
    prompt = inp["prompt"].permute(1, 0, 2).contiguous().cuda()
    mask = unet_oracle.sequence_mask(inp["refer_lengths"], inp["prompt"].shape[0]).cuda()
    return DenoiserSession(m, content, prompt, mask)


def closure(m, inp):
    """Diffusion_Encoder.forward (model.py:403-415) around the drop-in UNet's generic forward."""
    from oracle import unet_oracle
    content, prompt, plen = inp["content"].cuda(), inp["prompt"].cuda(), inp["refer_lengths"].cuda()

    def fn(x, t):
        assert torch.isnan(x).any() == False  # noqa: E712
        p = prompt.permute(1, 0, 2)
        xin = torch.cat([x, content.permute(1, 2, 0)], dim=1)
        return m(xin, t, p, encoder_attention_mask=unet_oracle.sequence_mask(plen, p.size(1)).to(torch.bool)).sample
    return fn


@pytest.mark.gpu
def test_step_kernels_bit_exact():
    from ns2vc_b200 import _lib
    L = _lib.lib()
    g = torch.Generator(device="cuda").manual_seed(3)
    x, x0, nz = (torch.randn(3, 100, 257, device="cuda", generator=g) for _ in range(3))   # n = 77 100: not a multiple of 256
    x0[0, 0, :8] = 0.0
    x[0, 0, :8] = -0.0
    buf = coefs.diffusion_buffers(1000)
    dbuf = {k: v.cuda() for k, v in buf.items()}
    for t in (999, 500, 1, 0):
        st = coefs.ddpm_table(buf, [t])[0]
        cdev, _ = coefs.c_table([st], "cuda")
        out = torch.full_like(x, float("nan"))
        _lib.check(L.ns2vc_ddpm_step(x.data_ptr(), x0.data_ptr(), nz.data_ptr(), cdev.data_ptr(), out.data_ptr(), x.numel(), None, None))
        inplace = x.clone()
        _lib.check(L.ns2vc_ddpm_step(inplace.data_ptr(), x0.data_ptr(), nz.data_ptr(), cdev.data_ptr(), inplace.data_ptr(), x.numel(), None, None))
        bt = torch.full((3,), t, dtype=torch.long, device="cuda")
        ext = lambda a: a.gather(-1, bt).reshape(3, 1, 1)
        mean = ext(dbuf["posterior_mean_coef1"]) * x0 + ext(dbuf["posterior_mean_coef2"]) * x
        want = mean + torch.tensor(st.c_noise, device="cuda") * (nz if t > 0 else 0.)
        torch.cuda.synchronize()
        assert torch.equal(out, want) and torch.equal(out.signbit(), want.signbit()), t
        assert torch.equal(inplace, out)
    for S, eta in ((6, 0.0), (10, 0.5), (1000, 0.5)):
        tab = coefs.ddim_table(buf, 1000, S, eta)
        for st in (tab[0], tab[len(tab) // 2], tab[-2], tab[-1]):
            cdev, _ = coefs.c_table([st], "cuda")
            out = torch.full_like(x, float("nan"))
            _lib.check(L.ns2vc_ddim_step(x.data_ptr(), x0.data_ptr(), nz.data_ptr(), cdev.data_ptr(), out.data_ptr(), x.numel(), None, None))
            bt = torch.full((3,), st.time, dtype=torch.long, device="cuda")
            ext = lambda a: a.gather(-1, bt).reshape(3, 1, 1)
            pred_noise = (ext(dbuf["sqrt_recip_alphas_cumprod"]) * x - x0) / ext(dbuf["sqrt_recipm1_alphas_cumprod"])
            if st.last:
                want = x0
            else:
                f = lambda v: torch.tensor(v, dtype=torch.float32, device="cuda")
                want = x0 * f(st.sqrt_alpha_next) + f(st.c) * pred_noise + f(st.sigma) * nz
            torch.cuda.synchronize()
            assert torch.equal(out, want) and torch.equal(out.signbit(), want.signbit()), (S, eta, st.time)
    # the NaN guard reads the step's input
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    xn = x.clone()
    xn[2, 99, 256] = float("nan")
    _lib.check(L.ns2vc_ddim_step(xn.data_ptr(), x0.data_ptr(), nz.data_ptr(), cdev.data_ptr(), out.data_ptr(), x.numel(), flag.data_ptr(), None))
    assert flag.item() == 1


@pytest.mark.gpu
def test_fused_ddpm_with_injected_noise_reproduces_the_p_sample_fixtures(gold, full_model):
    from oracle.make_golden_cfg1 import cfg1_config
    g = gold("cfg1_p_sample.pt")
    m, _ = make_unet(cfg1_config())
    inp = make_inputs(1, 128, 64, seed=g["seed_inputs"])
    noise = torch.stack([torch.randn(inp["x"].shape, generator=torch.Generator().manual_seed(g["noise_seed0"] + i)) for i in range(10)])
    sess = session(m, inp)
    for n in (10, 4):                                        # ten steps t = 999 .. 990, and the first four of them
        out = sess.sample_ddpm(inp["x"].cuda(), range(999, 999 - n, -1), noise=noise[:n].cuda())
        ok, msg = close(out, g["xs"][n - 1])
        assert ok, f"cfg1 {n} steps: {msg}"
    g = gold("p_sample.pt")
    m, _ = full_model
    inp = make_inputs(1, 64, 32, seed=30)
    noise = torch.stack([torch.randn(inp["x"].shape, generator=torch.Generator().manual_seed(100 + i)) for i in range(3)])
    out = session(m, inp).sample_ddpm(inp["x"].cuda(), [999, 998, 997], noise=noise)
    ok, msg = close(out, g["xs"][2])
    assert ok, msg


@pytest.mark.gpu
def test_fused_ddim_reproduces_the_ddim_fixture(gold, full_model):
    g = gold("ddim.pt")
    m, _ = full_model
    inp = make_inputs(2, 72, 24, ragged=True, seed=g["seed_inputs"])
    sess = session(m, inp)
    for i in range(4):                                       # eager, eager, capture, replay
        out = sess.sample_ddim(inp["x"].cuda(), g["steps"])
        ok, msg = close(out, g["out"])
        assert ok, f"call {i}: {msg}"


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["ddpm", "ddim", "ddim_eta"])
def test_api_reproduces_the_reference_sample(gold, case):
    from ns2vc_b200 import api
    from ns2vc_b200.pre_model import Pre_model
    from ns2vc_b200.unet import UNet1DConditionModel
    g = gold("ddpm_ddim.pt")
    k = g["cases"][case]
    unet = UNet1DConditionModel(in_channels=356, out_channels=100, block_out_channels=(128, 256, 384, 512), norm_num_groups=8,
                                cross_attention_dim=256, attention_head_dim=8, addition_embed_type="text", resnet_time_scale_shift="scale_shift")
    unet.load_state_dict(make_state_dict(ns2vc_denoiser_config(), seed=0))
    pre = Pre_model(PRE_CFG)
    pre.load_state_dict(make_pre_state_dict(PRE_CFG, seed=0))
    unet, pre = unet.cuda().eval(), pre.cuda().eval()
    draws = case_draws(k)
    xT, noise = fixture_noise(k, len(draws), draws)
    pin = make_pre_inputs(k["B"], k["T"], k["S"], ragged=True, seed=k["seed"])
    steps = None if k["method"] == "ddpm" else k["steps"]
    mel = api.sample_from_features(pre, unet, xT, pin["c"], pin["refer"], pin["lengths"], pin["refer_lengths"], steps=steps,
                                   method=k["method"], eta=k["eta"], noise=noise, device="cuda").cpu()
    ok, msg = close(mel, k["mel"])
    print(f"[api {case}: {len(draws)} steps] {msg}")
    assert ok, f"{case} ({len(draws)} steps): {msg}"


@pytest.mark.gpu
def test_captured_chunks_are_bit_identical_to_the_eager_loop(monkeypatch):
    """180 DDPM steps t = 179 .. 0: three full chunks of 50 and a final one of 30 (its last step draws no noise)."""
    m, _ = make_unet(tiny_config())
    inp = tiny_inputs()
    sess = session(m, inp)
    x = inp["x"].cuda()
    ts = range(179, -1, -1)

    def run():
        torch.cuda.manual_seed(11)
        out = sess.sample_ddpm(x, ts)
        return out, torch.cuda.get_rng_state()
    monkeypatch.setenv("NS2VC_GRAPH", "0")
    eager, rng = run()
    monkeypatch.delenv("NS2VC_GRAPH")
    assert not sess._chunk_graphs
    for i in range(3):                                       # eager (2nd run), capture (3rd), replay (4th)
        out, r = run()
        assert torch.equal(out, eager), f"run {i + 2}"
        assert torch.equal(r, rng), f"run {i + 2}: generator state"
    assert len(sess._chunk_graphs) == 2                      # the full chunk (replayed three times per run) and the final chunk
    assert torch.isfinite(eager).all()


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["ddpm", "ddim"])
def test_default_generator_run_follows_the_reference_call_sequence(method):
    """The reference's loops written out with the drop-in UNet's generic forward and torch.randn_like (model.py:535-601): same
    latents within tolerance and the same generator state afterwards, eager and captured."""
    m, _ = make_unet(tiny_config())
    inp = tiny_inputs()
    sess = session(m, inp)
    fn = closure(m, inp)
    buf = {k: v.cuda() for k, v in coefs.diffusion_buffers(1000).items()}
    x = inp["x"].cuda()
    B = x.shape[0]
    ext = lambda a, bt: a.gather(-1, bt).reshape(B, 1, 1)
    ts = list(range(59, -1, -1))
    S, eta = 12, 0.5

    @torch.no_grad()
    def reference():
        img = x
        if method == "ddpm":
            for t in ts:
                bt = torch.full((B,), t, device="cuda", dtype=torch.long)
                x0 = fn(img, bt)
                mean = ext(buf["posterior_mean_coef1"], bt) * x0 + ext(buf["posterior_mean_coef2"], bt) * img
                noise = torch.randn_like(img) if t > 0 else 0.
                img = mean + (0.5 * ext(buf["posterior_log_variance_clipped"], bt)).exp() * noise
            return img
        for time, time_next in coefs.ddim_time_pairs(1000, S):
            bt = torch.full((B,), time, device="cuda", dtype=torch.long)
            x0 = fn(img, bt)
            pred_noise = (ext(buf["sqrt_recip_alphas_cumprod"], bt) * img - x0) / ext(buf["sqrt_recipm1_alphas_cumprod"], bt)
            if time_next < 0:
                img = x0
                continue
            alpha, alpha_next = buf["alphas_cumprod"][time], buf["alphas_cumprod"][time_next]
            sigma = eta * ((1 - alpha / alpha_next) * (1 - alpha_next) / (1 - alpha)).sqrt()
            c = (1 - alpha_next - sigma ** 2).sqrt()
            img = x0 * alpha_next.sqrt() + c * pred_noise + sigma * torch.randn_like(img)
        return img

    torch.cuda.manual_seed(21)
    want = reference()
    want_rng = torch.cuda.get_rng_state()
    for i in range(4):                                       # eager, eager, capture, replay
        torch.cuda.manual_seed(21)
        got = sess.sample_ddpm(x, ts) if method == "ddpm" else sess.sample_ddim(x, S, eta=eta)
        assert torch.equal(torch.cuda.get_rng_state(), want_rng), f"run {i}: generator state"
        ok, msg = close(got, want)
        assert ok, f"run {i}: {msg}"


class _RefNaturalSpeech2:
    """The parts of NaturalSpeech2 the two loops use (model.py:403-415, 456-542), restated around our Pre_model and UNet."""

    def __init__(self, pre, unet, sampling_timesteps, eta):
        self.pre_model, self.unet, self.dim, self.num_timesteps = pre, unet, 100, 1000
        self.sampling_timesteps, self.ddim_sampling_eta = sampling_timesteps, eta
        for k, v in coefs.diffusion_buffers(1000).items():
            setattr(self, k, v.cuda())
        self.calls = 0

    def diff_model(self, x, data, t):                        # Diffusion_Encoder.forward
        self.calls += 1
        assert torch.isnan(x).any() == False                 # noqa: E712
        contentvec, prompt, _cl, prompt_lengths = data
        prompt = prompt.permute(1, 0, 2)
        x = torch.cat([x, contentvec.permute(1, 2, 0)], dim=1)
        mask = (torch.arange(prompt.size(1), device=x.device).unsqueeze(0) < prompt_lengths.unsqueeze(1)).to(torch.bool)
        return self.unet(x, t, prompt, encoder_attention_mask=mask).sample

    def model_predictions(self, x, t, data=None):
        from collections import namedtuple
        x_start = self.diff_model(x, data, t)
        t = t.type(torch.int64)
        ext = lambda a: a.gather(-1, t).reshape(t.shape[0], 1, 1)
        pred_noise = (ext(self.sqrt_recip_alphas_cumprod) * x - x_start) / ext(self.sqrt_recipm1_alphas_cumprod)
        return namedtuple("ModelPrediction", ["pred_noise", "pred_x_start"])(pred_noise, x_start)

    def q_posterior(self, x_start, x_t, t):
        ext = lambda a: a.gather(-1, t).reshape(t.shape[0], 1, 1)
        mean = ext(self.posterior_mean_coef1) * x_start + ext(self.posterior_mean_coef2) * x_t
        return mean, None, ext(self.posterior_log_variance_clipped)

    def p_sample(self, x, t, data):
        bt = torch.full((x.shape[0],), t, device=x.device, dtype=torch.long)
        preds = self.model_predictions(x, bt, data)
        mean, _, logvar = self.q_posterior(preds.pred_x_start, x, bt)
        noise = torch.randn_like(x) if t > 0 else 0.
        return mean + (0.5 * logvar).exp() * noise, preds.pred_x_start

    p_sample_loop = _StubNaturalSpeech2.p_sample_loop
    ddim_sample = _StubNaturalSpeech2.ddim_sample


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["ddpm", "ddim"])
def test_install_diffusion_methods_take_the_fused_path(monkeypatch, full_model, method):
    import ns2vc_b200
    from ns2vc_b200 import api
    from ns2vc_b200.pre_model import Pre_model
    unet, _ = full_model
    pre = Pre_model(PRE_CFG)
    pre.load_state_dict(make_pre_state_dict(PRE_CFG, seed=0))
    pre = pre.cuda().eval()
    cls = type("NaturalSpeech2", (_RefNaturalSpeech2,), {})
    ns2vc_b200.install_diffusion(types.SimpleNamespace(NaturalSpeech2=cls))
    model = cls(pre, unet, sampling_timesteps=20, eta=0.5)
    pin = {k: v.cuda() for k, v in make_pre_inputs(1, 40, 24, ragged=True, seed=5).items()}
    fn = model.p_sample_loop if method == "ddpm" else model.ddim_sample
    with torch.no_grad():
        torch.cuda.manual_seed(8)
        got = fn(pin["c"], pin["refer"], pin["lengths"], pin["refer_lengths"], None, None)
        rng = torch.cuda.get_rng_state()
        assert model.calls == 1                              # the traced first step; the rest ran on the session
        torch.cuda.manual_seed(8)
        xT = torch.randn((1, 100, 40), device="cuda")
        want = api.sample_from_features(pre, unet, xT, pin["c"], pin["refer"], pin["lengths"], pin["refer_lengths"], method=method,
                                        steps=None if method == "ddpm" else 20, eta=0.0 if method == "ddpm" else 0.5)
        assert torch.equal(torch.cuda.get_rng_state(), rng)
        ok, msg = close(got, want)
        assert ok, msg
        # NS2VC_B200_FUSED=0: the reference's loop, one denoiser call per step, same generator use
        monkeypatch.setenv("NS2VC_B200_FUSED", "0")
        torch.cuda.manual_seed(8)
        slow = fn(pin["c"], pin["refer"], pin["lengths"], pin["refer_lengths"], None, None)
        assert model.calls == 1 + (1000 if method == "ddpm" else 20)
        assert torch.equal(torch.cuda.get_rng_state(), rng)
        ok, msg = close(got, slow)
        assert ok, "fused vs generic: " + msg


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["ddpm", "ddim"])
def test_nan_in_x_T_raises_after_the_run(method):
    m, _ = make_unet(tiny_config())
    inp = tiny_inputs()
    sess = session(m, inp)
    run = (lambda x: sess.sample_ddpm(x, range(59, -1, -1))) if method == "ddpm" else (lambda x: sess.sample_ddim(x, 10))
    x = inp["x"].cuda().clone()
    assert torch.isfinite(run(x)).all()
    x[1, 3, 5] = float("nan")
    for _ in range(4):                                       # eager, eager, capture, replay
        with pytest.raises(AssertionError):
            run(x)
    assert torch.isfinite(run(inp["x"].cuda())).all()


@pytest.mark.gpu
def test_chunk_table_stays_chunk_sized_for_1000_steps():
    from ns2vc_b200 import _lib
    from ns2vc_b200.fused import DenoiserSession
    m, _ = make_unet(tiny_config())
    inp = tiny_inputs()
    sess = session(m, inp)
    out = sess.sample_ddpm(inp["x"].cuda())
    assert torch.isfinite(out).all()
    B, K = inp["x"].shape[0], DenoiserSession.CHUNK
    assert K == 50
    assert sess._chunk["table"].numel() == int(_lib.lib().ns2vc_unet_time_table_floats(sess.h, K * B))
    assert sess._chunk["tvals"].numel() == K * B
    ent = next(iter(sess._chains.values()))
    assert ent["n"] == 1000 and ent["tvals"].numel() == 1000 * B
