"""Parity of the CUDA path against the oracle / reference fixtures.  All tests call through the
C-ABI (via the drop-in Python modules).  Tolerance for floating-point results is the north-star's
rtol=1e-3 / atol=1e-4 (fp32 outputs vs the reference's CPU fp32 path); element-wise sampler kernels
and index/mask ops are bit-exact."""
import ctypes as C
import os

import pytest
import torch

from conftest import tiny_config, tiny_inputs
from ns2vc_b200 import _lib, coefs, dpm_solver as our_dpm, uni_pc as our_upc
from ns2vc_b200.arch import ns2vc_denoiser_config
from ns2vc_b200.debug import forward_with_taps
from ns2vc_b200.fused import DenoiserSession
from ns2vc_b200.schedule import NoiseScheduleVP
from ns2vc_b200.synth import linear_betas, make_inputs, make_state_dict
from ns2vc_b200.unet import UNet1DConditionModel
from oracle import sampler_oracle, unet_oracle

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-3, 1e-4


def close(a, b, rtol=RTOL, atol=ATOL):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    err = (a - b).abs()
    viol = (err > atol + rtol * b.abs()).float().mean().item()
    return viol == 0.0, f"max_abs={err.max().item():.3e} violations={viol:.3%} ref_rms={b.pow(2).mean().sqrt().item():.3e}"


def make_unet(cfg, seed=0, backend=None):
    kw = dict(in_channels=cfg.in_channels, out_channels=cfg.out_channels, block_out_channels=cfg.block_out_channels,
              layers_per_block=list(cfg.layers_per_block), norm_num_groups=cfg.norm_num_groups, cross_attention_dim=cfg.cross_attention_dim,
              attention_head_dim=cfg.num_heads, addition_embed_type=cfg.addition_embed_type,
              addition_embed_type_num_heads=cfg.addition_embed_type_num_heads, resnet_time_scale_shift=cfg.resnet_time_scale_shift)
    m = UNet1DConditionModel(**kw)
    sd = make_state_dict(cfg, seed)
    m.load_state_dict(sd, strict=True)
    m = m.to("cuda").eval()
    old = os.environ.get("NS2VC_GEMM_BACKEND")
    if backend:
        os.environ["NS2VC_GEMM_BACKEND"] = backend
    else:
        os.environ.pop("NS2VC_GEMM_BACKEND", None)
    try:
        m.engine(torch.device("cuda", 0))          # the backend is fixed when the engine is created
    finally:
        if old is None:
            os.environ.pop("NS2VC_GEMM_BACKEND", None)
        else:
            os.environ["NS2VC_GEMM_BACKEND"] = old
    return m, sd


@pytest.fixture(scope="module")
def full_model():
    return make_unet(ns2vc_denoiser_config())


def unet_inputs(inp, dev="cuda"):
    x = torch.cat([inp["x"], inp["content"].permute(1, 2, 0)], 1).to(dev)
    ehs = inp["prompt"].permute(1, 0, 2).contiguous().to(dev)
    mask = unet_oracle.sequence_mask(inp["refer_lengths"], inp["prompt"].shape[0]).to(dev)
    return x, ehs, mask


def test_native_library_is_the_in_tree_build():
    assert os.path.isfile(_lib.LIB_PATH) and "ns2vc_b200/_C" in _lib.LIB_PATH
    assert torch.cuda.get_device_capability(0) == (9, 0), "these kernels are sm_90a only"


@pytest.mark.parametrize("backend", ["simt", "tc"])
def test_tiny_forward_every_op(gold, backend):
    """Every op output of the tiny UNet against the reference's activations: localises any defect."""
    g = gold("tiny_forward.pt")
    m, _ = make_unet(tiny_config(), backend=None if backend == "tc" else "simt")
    x, ehs, mask = unet_inputs(tiny_inputs())
    out, taps = forward_with_taps(m, x, g["t"].cuda(), ehs, mask)
    bad = []
    for name, ref in g["taps"].items():
        if name in ("emb", "aug_emb"):
            continue
        assert name in taps, f"engine has no tap {name}"
        ok, msg = close(taps[name], ref, atol=2e-4)     # intermediate activations: diagnostic tolerance
        if not ok:
            bad.append(f"{name}: {msg}")
    assert not bad, "first failing ops:\n" + "\n".join(bad[:8])
    ok, msg = close(out, g["out"])
    assert ok, msg
    # integer timesteps, no mask (p_sample-style call)
    with torch.no_grad():
        out2 = m(x, torch.tensor([999, 0], device="cuda"), ehs).sample
    ok, msg = close(out2, g["out_nomask"])
    assert ok, msg


def test_full_forward_matches_reference_fixture(gold, full_model):
    g = gold("full_forward.pt")
    m, _ = full_model
    x, ehs, mask = unet_inputs(make_inputs(2, 131, 48, ragged=True, seed=20))
    with torch.no_grad():
        out = m(x, g["t"].cuda(), ehs, encoder_attention_mask=mask).sample
    ok, msg = close(out, g["out"])
    assert ok, msg


@pytest.mark.parametrize("B,T,S", [(2, 1024, 256), (1, 1000, 100), (1, 1023, 7), (3, 8, 1), (1, 2048, 300), (1, 136, 1100)])
def test_full_forward_vs_oracle_shapes(full_model, B, T, S):
    """config-2 sequence length, lengths that are not multiples of 8 (forced-size upsample), T=8 minimum, the cfg3
    length (T=2048: several persistent-GEMM tiles per CTA, 32 key tiles per attention row) and a prompt longer than
    the staged-bias capacity of the TMA-fed attention kernel (S=1100: the whole model falls back to the v1 kernel)."""
    m, sd = full_model
    inp = make_inputs(B, T, S, ragged=True, seed=40 + T)
    x, ehs, mask = unet_inputs(inp)
    t = torch.linspace(3.5, 990.25, B)
    with torch.no_grad():
        out = m(x, t.cuda(), ehs, encoder_attention_mask=mask).sample
        ref = unet_oracle.denoiser_forward(sd, ns2vc_denoiser_config(), inp["x"], inp["content"], inp["prompt"], inp["refer_lengths"], t)
    ok, msg = close(out, ref)
    assert ok, msg


def test_forward_is_deterministic_and_batch_independent(full_model):
    m, _ = full_model
    inp = make_inputs(8, 1024, 256, seed=77)
    x, ehs, mask = unet_inputs(inp)
    t = torch.full((8,), 421.5, device="cuda")
    with torch.no_grad():
        a = m(x, t, ehs, encoder_attention_mask=mask).sample
        b = m(x, t, ehs, encoder_attention_mask=mask).sample
        assert torch.equal(a, b)
        x2 = x.clone()
        x2[0] = torch.randn_like(x2[0])
        c = m(x2, t, ehs, encoder_attention_mask=mask).sample
    assert torch.equal(a[1:], c[1:]), "samples of a batch must not influence each other"
    assert not torch.equal(a[0], c[0])
    assert torch.isfinite(a).all()


def test_return_to_a_cached_program_reproduces_it(full_model):
    """Shape A, then a smaller shape B, then A again on one module and one shared workspace: the return to A reactivates A's
    cached program, whose conditioning must be prepared again because B has run in the same workspace since."""
    m, _ = full_model
    dev = torch.device("cuda", 0)
    shapes = {"A": (2, 256, 64), "B": (1, 128, 32)}
    inps = {k: make_inputs(*v, ragged=True, seed=90 + i) for i, (k, v) in enumerate(shapes.items())}
    pool = m.workspace(*shapes["A"], dev).data_ptr()
    ns = NoiseScheduleVP("discrete", betas=linear_betas(1000))

    def forward(k):
        x, ehs, mask = unet_inputs(inps[k])
        t = torch.linspace(11.5, 870.25, x.shape[0], device="cuda")
        with torch.no_grad():
            return m(x, t, ehs, encoder_attention_mask=mask).sample.clone()

    def dpm10(k):
        return _session(m, inps[k]).sample_dpmpp_2m(inps[k]["x"].cuda(), ns, torch.linspace(1.0, 1e-3, 11)).clone()

    a0 = forward("A")
    forward("B")
    assert torch.equal(forward("A"), a0)
    s0 = dpm10("A")
    dpm10("B")
    assert torch.equal(dpm10("A"), s0)
    assert torch.isfinite(a0).all() and torch.isfinite(s0).all()
    assert m.workspace(*shapes["B"], dev).data_ptr() == pool, "both shapes must run in the same workspace"


# ------------------------------------------------------------------ sampler kernels: bit-exact
def _rt(x, o, a, s):
    noise = (x - a * o) / s
    return (x - s * noise) / a


def test_dpm_step_kernel_bit_exact():
    L = _lib.lib()
    g = torch.Generator(device="cuda").manual_seed(1)
    x, o, mp = (torch.randn(3, 100, 257, device="cuda", generator=g) for _ in range(3))
    f = lambda v: torch.tensor(v, dtype=torch.float32, device="cuda")
    for order in (0, 1, 2):
        c = _lib.DpmCoef(0.37, 0.929, 0.9571, -0.0123, -0.00615, 1.0231, order)
        mc, xn = torch.empty_like(x), torch.zeros_like(x)
        _lib.check(L.ns2vc_dpm_step(x.data_ptr(), o.data_ptr(), mp.data_ptr(), C.byref(c), mc.data_ptr(), xn.data_ptr(), x.numel(), None, None))
        torch.cuda.synchronize()
        m0 = _rt(x, o, f(c.alpha_s), f(c.sigma_s))
        assert torch.equal(mc, m0)
        if order >= 1:
            r = f(c.c_x) * x - f(c.c_m) * m0
            if order == 2:
                r = r - f(c.c_d) * (f(c.inv_r0) * (m0 - mp))
            assert torch.equal(xn, r)


def test_unipc_step_kernel_bit_exact():
    L = _lib.lib()
    g = torch.Generator(device="cuda").manual_seed(2)
    xp, xe, o, m0, m1 = (torch.randn(2, 100, 131, device="cuda", generator=g) for _ in range(5))
    f = lambda v: torch.tensor(v, dtype=torch.float32, device="cuda")
    for corr, pred in ((0, 1), (1, 2), (2, 2), (2, 1)):
        c = _lib.UniPcCoef(0.41, 0.912, 0.961, -0.0131, -0.0127, -1.07, 0.4931, 0.5069, corr, 0.957, -0.0141, -0.0139, -0.97, pred)
        mt, xt, xq = torch.empty_like(xp), torch.empty_like(xp), torch.empty_like(xp)
        _lib.check(L.ns2vc_unipc_step(xp.data_ptr(), xe.data_ptr(), o.data_ptr(), m0.data_ptr(), m1.data_ptr(), C.byref(c),
                                      mt.data_ptr(), xt.data_ptr(), xq.data_ptr(), xp.numel(), None, None))
        torch.cuda.synchronize()
        mt_ref = _rt(xe, o, f(c.alpha_t), f(c.sigma_t))
        assert torch.equal(mt, mt_ref)
        xt_ref = xe
        if corr:
            xbar = f(c.c_x) * xp - f(c.c_m) * m0
            inner = f(c.rho1) * (mt_ref - m0)
            if corr == 2:
                inner = f(c.rho0) * ((m1 - m0) / f(c.rk)) + f(c.rho1) * (mt_ref - m0)
            xt_ref = xbar - f(c.ab) * inner
            assert torch.equal(xt, xt_ref)
        nbar = f(c.n_c_x) * xt_ref - f(c.n_c_m) * mt_ref
        if pred == 2:
            nbar = nbar - f(c.nab) * (f(0.5) * ((m0 - mt_ref) / f(c.nrk)))
        assert torch.equal(xq, nbar)


# ------------------------------------------------------------------ full sampling loops
def _session(m, inp):
    content = inp["content"].permute(1, 2, 0).contiguous().cuda()
    prompt = inp["prompt"].permute(1, 0, 2).contiguous().cuda()
    mask = unet_oracle.sequence_mask(inp["refer_lengths"], inp["prompt"].shape[0]).cuda()
    return DenoiserSession(m, content, prompt, mask)


def test_fused_samplers_tiny_vs_reference_fixture(gold):
    g = gold("tiny_samplers.pt")
    m, _ = make_unet(tiny_config())
    inp = tiny_inputs()
    ns = NoiseScheduleVP("discrete", betas=linear_betas(1000))
    sess = _session(m, inp)
    outs = []
    for i in range(4):          # calls 1-2 eager, the 3rd captures the CUDA graph, the 4th replays it
        out = sess.sample_dpmpp_2m(inp["x"].cuda(), ns, torch.linspace(1.0, 1e-3, 13))
        ok, msg = close(out, g["dpmpp2m_12"])
        assert ok, f"call {i}: {msg}"
        outs.append(out)
    assert torch.equal(outs[2], outs[3]), "graph replay must reproduce the captured run"
    # new inputs through the same captured graph
    x2 = torch.randn_like(outs[0])
    a = sess.sample_dpmpp_2m(x2, ns, torch.linspace(1.0, 1e-3, 13))
    assert not torch.allclose(a, outs[2])
    for i in range(4):
        out = sess.sample_unipc(inp["x"].cuda(), ns, torch.linspace(1.0, 1e-3, 9))
        ok, msg = close(out, g["unipc_bh2_8"])
        assert ok, f"unipc call {i}: {msg}"


def test_fused_dpm_50_steps_full_model_vs_oracle(full_model):
    """The metric path (50-step DPM-Solver++ 2M) end to end, small T so the CPU oracle stays fast."""
    m, sd = full_model
    cfg = ns2vc_denoiser_config()
    inp = make_inputs(2, 64, 32, ragged=True, seed=3)
    ns = NoiseScheduleVP("discrete", betas=linear_betas(1000))
    sess = _session(m, inp)
    out = sess.sample_dpmpp_2m(inp["x"].cuda(), ns, torch.linspace(1.0, 1e-3, 51))
    sch = sampler_oracle.OracleSchedule(linear_betas(1000))
    fn = lambda x, t: unet_oracle.denoiser_forward(sd, cfg, x, inp["content"], inp["prompt"], inp["refer_lengths"], t)
    with torch.no_grad():
        ref = sampler_oracle.dpmpp_2m(fn, sch, inp["x"], 50)
    ok, msg = close(out, ref)
    assert ok, msg


def test_fused_unipc_30_steps_full_model_vs_oracle(full_model):
    """cfg3's sampler (UniPC bh2, the reference's default 30 steps, model.py:655-686) on the full architecture."""
    m, sd = full_model
    cfg = ns2vc_denoiser_config()
    inp = make_inputs(2, 72, 24, ragged=True, seed=11)
    ns = NoiseScheduleVP("discrete", betas=linear_betas(1000))
    sess = _session(m, inp)
    out = sess.sample_unipc(inp["x"].cuda(), ns, torch.linspace(1.0, 1e-3, 31))
    sch = sampler_oracle.OracleSchedule(linear_betas(1000))
    fn = lambda x, t: unet_oracle.denoiser_forward(sd, cfg, x, inp["content"], inp["prompt"], inp["refer_lengths"], t)
    with torch.no_grad():
        ref = sampler_oracle.unipc_bh(fn, sch, inp["x"], 30)
    ok, msg = close(out, ref)
    assert ok, msg


def _closure(m, inp):
    """Same call chain as NaturalSpeech2.sample_fun -> Diffusion_Encoder.forward (model.py:520, 403-415)."""
    content, prompt, plen = inp["content"].cuda(), inp["prompt"].cuda(), inp["refer_lengths"].cuda()

    def fn(x, t, **kw):
        assert torch.isnan(x).any() == False  # noqa: E712
        p = prompt.permute(1, 0, 2)
        c = content.permute(1, 2, 0)
        xin = torch.cat([x, c], dim=1)
        mask = unet_oracle.sequence_mask(plen, p.size(1)).to(torch.bool)
        return m(xin, t, p, encoder_attention_mask=mask).sample
    return fn


def test_dropin_sampler_classes_take_the_fused_path(gold, monkeypatch):
    """model.py:621-652 / 655-686 style usage with our classes: fused path == explicit session, and the
    generic Python path (NS2VC_B200_FUSED=0) agrees with both."""
    g = gold("tiny_samplers.pt")
    m, _ = make_unet(tiny_config())
    inp = tiny_inputs()
    betas = linear_betas(1000).cuda()
    x0 = inp["x"].cuda()
    with torch.no_grad():
        ns = our_dpm.NoiseScheduleVP("discrete", betas=betas)
        mf = our_dpm.model_wrapper(_closure(m, inp), ns, model_type="x_start", model_kwargs={})
        fast = our_dpm.DPM_Solver(mf, ns, algorithm_type="dpmsolver++").sample(x0, steps=12, order=2, skip_type="time_uniform", method="multistep")
        monkeypatch.setenv("NS2VC_B200_FUSED", "0")
        slow = our_dpm.DPM_Solver(mf, ns, algorithm_type="dpmsolver++").sample(x0, steps=12, order=2, skip_type="time_uniform", method="multistep")
        monkeypatch.delenv("NS2VC_B200_FUSED")
    ok, msg = close(fast, g["dpmpp2m_12"])
    assert ok, "fused: " + msg
    ok, msg = close(slow, g["dpmpp2m_12"])
    assert ok, "generic: " + msg
    ok, msg = close(fast, slow)
    assert ok, "fused vs generic: " + msg
    with torch.no_grad():
        ns = our_upc.NoiseScheduleVP("discrete", betas=betas)
        mf = our_upc.model_wrapper(_closure(m, inp), ns, model_type="x_start", model_kwargs={})
        fast = our_upc.UniPC(mf, ns, variant="bh2").sample(x0, steps=8, order=2, skip_type="time_uniform", method="multistep")
    ok, msg = close(fast, g["unipc_bh2_8"])
    assert ok, "unipc fused: " + msg


def test_p_sample_chain_through_generic_forward(gold, full_model):
    """DDPM p_sample (model.py:535-542) with injected noise: integer timesteps through UNet.forward."""
    g = gold("p_sample.pt")
    m, _ = full_model
    inp = make_inputs(1, 64, 32, seed=30)
    fn = _closure(m, inp)
    ddpm = sampler_oracle.OracleDDPM(1000)
    x = inp["x"].cuda()
    with torch.no_grad():
        for i, t in enumerate((999, 998, 997)):
            noise = torch.randn(x.shape, generator=torch.Generator().manual_seed(100 + i)).cuda()
            bt = torch.full((1,), t, dtype=torch.long, device="cuda")
            x0 = fn(x, bt)
            mean = ddpm.coef1.cuda()[bt][:, None, None] * x0 + ddpm.coef2.cuda()[bt][:, None, None] * x
            x = mean + (0.5 * ddpm.log_var.cuda()[bt][:, None, None]).exp() * noise
            ok, msg = close(x, g["xs"][i])
            assert ok, f"step {i}: {msg}"


def test_weights_repack_after_update(full_model):
    """load_state_dict / optimizer-style in-place updates must reach the packed tensor-core weights."""
    cfg = tiny_config()
    m, sd = make_unet(cfg)
    x, ehs, mask = unet_inputs(tiny_inputs())
    t = torch.tensor([10.0, 20.0], device="cuda")
    with torch.no_grad():
        a = m(x, t, ehs, encoder_attention_mask=mask).sample
        sd2 = make_state_dict(cfg, seed=1)
        m.load_state_dict(sd2)
        b = m(x, t, ehs, encoder_attention_mask=mask).sample
    ref = unet_oracle.unet_forward(sd2, cfg, x.cpu(), t.cpu(), ehs.cpu(), mask.cpu())
    ok, msg = close(b, ref)
    assert ok, msg
    assert not torch.allclose(a, b)


# ------------------------------------------------------------------ BASELINE cfg1 / DDIM through the generic forward
def test_cfg1_one_layer_unet_ten_p_sample_steps(gold):
    """BASELINE.json configs[0] exactly: layers_per_block=1, B=1, C=100, T=128, S=64, DDPM p_sample t = 999 .. 990
    (model.py:535-542) with injected noise; every intermediate latent against the reference's own run."""
    from oracle.make_golden_cfg1 import cfg1_config
    g = gold("cfg1_p_sample.pt")
    m, _ = make_unet(cfg1_config())
    inp = make_inputs(1, 128, 64, seed=g["seed_inputs"])
    fn = _closure(m, inp)
    ddpm = sampler_oracle.OracleDDPM(1000)
    x = inp["x"].cuda()
    with torch.no_grad():
        for i, t in enumerate(range(999, 989, -1)):
            noise = torch.randn(x.shape, generator=torch.Generator().manual_seed(g["noise_seed0"] + i)).cuda()
            bt = torch.full((1,), t, dtype=torch.long, device="cuda")
            x0 = fn(x, bt)
            mean = ddpm.coef1.cuda()[bt][:, None, None] * x0 + ddpm.coef2.cuda()[bt][:, None, None] * x
            x = mean + (0.5 * ddpm.log_var.cuda()[bt][:, None, None]).exp() * noise
            ok, msg = close(x, g["xs"][i])
            assert ok, f"step {i}: {msg}"


def test_ddim_sample_through_generic_forward(gold, full_model):
    """NaturalSpeech2.ddim_sample (model.py:563-603; 6 steps, eta 0): integer timesteps through UNet.forward, fixture from the
    reference's own ddim_sample."""
    g = gold("ddim.pt")
    m, _ = full_model
    inp = make_inputs(2, 72, 24, ragged=True, seed=g["seed_inputs"])
    fn = _closure(m, inp)
    with torch.no_grad():
        out = sampler_oracle.ddim_sample(lambda x, t: fn(x.cuda(), t.cuda()).cpu(), g["alphas_cumprod"], inp["x"], 1000, g["steps"])
    ok, msg = close(out, g["out"])
    assert ok, msg


# ------------------------------------------------------------------ small pieces that used to be checked only through the outputs
def test_mask_bias_bit_exact():
    L = _lib.lib()
    g = torch.Generator().manual_seed(7)
    mask = (torch.rand(3, 257, generator=g) > 0.4)
    m8 = mask.to(torch.uint8).cuda()
    bias = torch.empty(mask.shape, dtype=torch.float32, device="cuda")
    _lib.check(L.ns2vc_mask_bias(m8.data_ptr(), m8.numel(), bias.data_ptr(), None))
    torch.cuda.synchronize()
    want = (1 - mask.to(torch.float32)) * -10000.0          # reference unet_1d_condition.py:817
    assert torch.equal(bias.cpu(), want)


def test_timestep_table_matches_reference_embeddings(gold):
    """emb = time_embedding(t) + add_embedding(prompt) of the tiny fixture (taps 'emb', 'aug_emb' recorded from the reference's
    forward hooks) pushed through every resnet's time_emb_proj: the rows ns2vc_unet_time_table() produces."""
    from ns2vc_b200.arch import build_plan
    g = gold("tiny_forward.pt")
    cfg = tiny_config()
    m, sd = make_unet(cfg)
    inp = tiny_inputs()
    sess = _session(m, inp)
    sess.prepare()
    L = _lib.lib()
    B = 2
    tv = g["t"].to(torch.float32).cuda().contiguous()
    table = torch.empty(int(L.ns2vc_unet_time_table_floats(sess.h, B)), dtype=torch.float32, device="cuda")
    sess.time_table(tv.view(1, B), table)
    torch.cuda.synchronize()
    fw = int(L.ns2vc_unet_film_width(sess.h))
    film = table[:B * fw].view(B, fw).cpu()
    emb = g["taps"]["emb"]
    want = torch.cat([torch.nn.functional.linear(torch.nn.functional.silu(emb), sd[op.prefix + ".time_emb_proj.weight"], sd[op.prefix + ".time_emb_proj.bias"])
                      for op in build_plan(cfg) if op.kind == "resnet"], dim=1)
    assert film.shape == want.shape
    ok, msg = close(film, want, rtol=1e-4, atol=1e-5)
    assert ok, msg


# ------------------------------------------------------------------ drop-in semantics of the fused path
def test_fresh_schedule_objects_share_one_graph_and_other_betas_do_not(gold):
    """model.py:621-622 builds a NEW NoiseScheduleVP in every sample(): the captured loop must be found by schedule CONTENT
    (replayed, same result), and a different beta table must neither hit that entry nor reuse its coefficients."""
    g = gold("tiny_samplers.pt")
    m, _ = make_unet(tiny_config())
    inp = tiny_inputs()
    x0 = inp["x"].cuda()

    def run(betas):
        ns = our_dpm.NoiseScheduleVP("discrete", betas=betas)          # fresh object every call, as the reference does
        mf = our_dpm.model_wrapper(_closure(m, inp), ns, model_type="x_start", model_kwargs={})
        return our_dpm.DPM_Solver(mf, ns, algorithm_type="dpmsolver++").sample(x0, steps=12, order=2, skip_type="time_uniform", method="multistep")
    with torch.no_grad():
        outs = [run(linear_betas(1000).cuda()) for _ in range(4)]
    sessions = list(m.__dict__["_sessions"].values())
    assert len(sessions) == 1
    ents = list(sessions[0]._graphs.values())
    assert len(ents) == 1 and ents[0]["graph"] is not None and ents[0]["runs"] == 4, "calls with fresh schedule objects must find (and end up replaying) ONE captured loop"
    for o in outs:
        ok, msg = close(o, g["dpmpp2m_12"])
        assert ok, msg
    assert torch.equal(outs[2], outs[3])
    # a different schedule: own entry, own coefficients; must agree with the generic Python loop for THAT schedule
    betas2 = torch.linspace(2e-4, 0.03, 1000, dtype=torch.float64).to(torch.float32).cuda()
    with torch.no_grad():
        o2 = run(betas2)
        os.environ["NS2VC_B200_FUSED"] = "0"
        try:
            o2_generic = run(betas2)
        finally:
            os.environ.pop("NS2VC_B200_FUSED")
    assert len(sessions[0]._graphs) == 2
    assert not torch.allclose(o2, outs[0], atol=1e-3)
    ok, msg = close(o2, o2_generic)
    assert ok, "second schedule, fused vs generic: " + msg
    assert len(sessions[0]._graphs) <= sessions[0].MAX_GRAPHS


def test_nan_input_raises_like_the_reference():
    """model.py:404 asserts on NaN in the denoiser input every call; the fused loop checks a device flag once per run."""
    m, _ = make_unet(tiny_config())
    inp = tiny_inputs()
    ns = NoiseScheduleVP("discrete", betas=linear_betas(1000))
    sess = _session(m, inp)
    x = inp["x"].cuda().clone()
    ok = sess.sample_dpmpp_2m(x, ns, torch.linspace(1.0, 1e-3, 11))
    assert torch.isfinite(ok).all()
    x[1, 3, 5] = float("nan")
    for _ in range(4):                                   # eager, eager, capture, replay
        with pytest.raises(AssertionError):
            sess.sample_dpmpp_2m(x, ns, torch.linspace(1.0, 1e-3, 11))
    assert torch.isfinite(sess.sample_dpmpp_2m(inp["x"].cuda(), ns, torch.linspace(1.0, 1e-3, 11))).all()


# ------------------------------------------------------------------ the benchmark shapes end to end
def test_fused_dpm_50_steps_T1024_vs_oracle(full_model):
    """cfg2's sequence length and prompt length (B=1): 50-step DPM-Solver++(2M) against the CPU oracle loop."""
    m, sd = full_model
    cfg = ns2vc_denoiser_config()
    inp = make_inputs(1, 1024, 256, seed=51)
    ns = NoiseScheduleVP("discrete", betas=linear_betas(1000))
    sess = _session(m, inp)
    out = sess.sample_dpmpp_2m(inp["x"].cuda(), ns, torch.linspace(1.0, 1e-3, 51))
    sch = sampler_oracle.OracleSchedule(linear_betas(1000))
    fn = lambda x, t: unet_oracle.denoiser_forward(sd, cfg, x, inp["content"], inp["prompt"], inp["refer_lengths"], t)
    with torch.no_grad():
        ref = sampler_oracle.dpmpp_2m(fn, sch, inp["x"], 50)
    ok, msg = close(out, ref)
    assert ok, msg


def test_fused_unipc_30_steps_T2048_vs_oracle(full_model):
    """cfg3's sequence length (B=1, T=2048, S=256): UniPC bh2, the reference's default 30 steps."""
    m, sd = full_model
    cfg = ns2vc_denoiser_config()
    inp = make_inputs(1, 2048, 256, seed=52)
    ns = NoiseScheduleVP("discrete", betas=linear_betas(1000))
    sess = _session(m, inp)
    out = sess.sample_unipc(inp["x"].cuda(), ns, torch.linspace(1.0, 1e-3, 31))
    sch = sampler_oracle.OracleSchedule(linear_betas(1000))
    fn = lambda x, t: unet_oracle.denoiser_forward(sd, cfg, x, inp["content"], inp["prompt"], inp["refer_lengths"], t)
    with torch.no_grad():
        ref = sampler_oracle.unipc_bh(fn, sch, inp["x"], 30)
    ok, msg = close(out, ref)
    assert ok, msg


# ------------------------------------------------------------------ numerics under stress
@pytest.mark.parametrize("gain,offset", [(3.0, 0.0), (1.0, 30.0), (3.0, 30.0)])
def test_forward_with_large_gain_weights_and_offset_activations(gain, offset):
    """3xBF16 GEMMs, folded LayerNorms (rstd * (x W' - mean g): cancellation grows with |row mean| / std) and the fp16-P / fp16-V
    attention under weights of `gain` x the synthetic scale and a per-channel offset on the residual stream (the proj_in bias of
    every transformer, so LayerNorm rows have |mean| >> std).  Reports err / tol; must stay inside the contract."""
    cfg = ns2vc_denoiser_config()
    sd = make_state_dict(cfg, 0)
    for k in sd:
        if k.endswith(".weight") and sd[k].dim() >= 2 and ".norm" not in k:
            sd[k] = sd[k] * gain ** 0.25                       # four-ish contractions deep per block: keeps activations finite
        if offset and k.endswith("proj_in.bias"):
            sd[k] = sd[k] + offset
    m, _ = make_unet(cfg)
    m.load_state_dict(sd)
    inp = make_inputs(2, 200, 40, ragged=True, seed=61)
    x, ehs, mask = unet_inputs(inp)
    t = torch.tensor([731.0, 12.5], device="cuda")
    with torch.no_grad():
        out = m(x, t, ehs, encoder_attention_mask=mask).sample.cpu()
        ref = unet_oracle.unet_forward(sd, cfg, x.cpu(), t.cpu(), ehs.cpu(), mask.cpu())
    err = (out - ref).abs()
    ratio = (err / (ATOL + RTOL * ref.abs())).max().item()
    print(f"gain {gain} offset {offset}: max|err| {err.max().item():.3e}, ref rms {ref.pow(2).mean().sqrt().item():.3e}, worst err/tol {ratio:.2f}")
    assert ratio <= 1.0, f"worst err/tol {ratio:.2f}"


# ------------------------------------------------------------------ every documented switch keeps parity
@pytest.mark.parametrize("env", ["NS2VC_ATTN_P=split", "NS2VC_PDL=0", "NS2VC_GRAPH=0"])
def test_diagnostic_switches_keep_parity(env):
    """The environment switches of README.md (A/B paths and numerical fallbacks) are read once per process / engine, so each one is
    exercised in a child process on the per-op tap test, the reference full-config fixture and the tiny sampler fixtures."""
    import subprocess
    import sys
    k, v = env.split("=")
    child_env = dict(os.environ, **{k: v})
    sel = "tiny_forward_every_op and tc or full_forward_matches_reference_fixture or fused_samplers_tiny_vs_reference_fixture"
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "-m", "gpu", "-p", "no:cacheprovider", "-k", sel],
                       env=child_env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and " passed" in r.stdout, f"{env}:\n{r.stdout[-1500:]}\n{r.stderr[-500:]}"
