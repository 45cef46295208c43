"""The training objective under no_grad: ``loss.diffusion_loss`` / ``loss_profile`` / ``NaturalSpeech2.validation_loss`` against
``NaturalSpeech2.forward`` (reference model.py:706-734).

CPU: the oracle reproduces tests/golden/train_loss.pt (written by the unmodified reference, oracle/make_golden_loss.py), the three
schedule buffers are the reference's, argument errors, and the order of the default draws.  GPU: ``q_sample`` is bit-identical to
the torch expression, the reduction is deterministic and accurate, the whole call reproduces the fixture, K timesteps in one call
equal K calls, the default draws consume the generator as the reference does, and the samplers' session state is untouched."""
import types

import pytest
import torch

from ns2vc_b200 import coefs
from ns2vc_b200.arch import ns2vc_denoiser_config
from ns2vc_b200.synth import make_pre_state_dict, make_state_dict, state_dict_checksum

RTOL, ATOL = 1e-3, 1e-4
LOSS_RTOL = 5e-5                                             # observed on an H100: loss 5.2e-7, rows 4.1e-6 at worst
PRE_CFG = {"phoneme_encoder": dict(in_channels=256, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2),
           "prompt_encoder": dict(in_channels=100, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2)}


def case_data(k, device="cpu"):
    mv = lambda v: v.to(device)
    return (mv(k["c"]), mv(k["refer"]), None, mv(k["spec"]), None, mv(k["lengths"]), mv(k["refer_lengths"]), None)


def bits(x):
    return x.contiguous().view(torch.int32)


def torch_q_sample(spec, noise, lengths, t, buf):
    """model.py:710-718 for one [B] t: (x_start, masked noise, x)."""
    B, _, T = spec.shape
    x_mask = (torch.arange(T, device=spec.device)[None, :] < lengths[:, None]).unsqueeze(1).to(spec.dtype)
    x_start = spec * x_mask
    noise = noise * x_mask
    ext = lambda a: a.gather(-1, t).reshape(B, 1, 1)
    return x_start, noise, ext(buf["sqrt_alphas_cumprod"]) * x_start + ext(buf["sqrt_one_minus_alphas_cumprod"]) * noise


# ------------------------------------------------------------------------------------------------------------------- CPU
def test_loss_buffers_are_the_references(gold):
    g = gold("train_loss.pt")
    for gamma, key in ((None, "buffers"), (5, "buffers_min_snr_5")):
        ours = coefs.loss_buffers(1000, gamma)
        assert set(ours) == set(g[key])
        for name, v in g[key].items():
            assert v.dtype == torch.float32 and torch.equal(ours[name], v), (key, name)
    assert g["buffers_min_snr_5"]["loss_weight"].max().item() == 5.0
    lw = g["buffers"]["loss_weight"]
    assert lw[0] > 9e3 and lw[999] < 5e-5


@pytest.mark.parametrize("case", ["drawn", "edges"])
def test_oracle_reproduces_the_reference_forward(gold, case):
    from oracle import loss_oracle
    g = gold("train_loss.pt")
    sd_u, sd_p = make_state_dict(ns2vc_denoiser_config(), seed=0), make_pre_state_dict(PRE_CFG, seed=0)
    assert state_dict_checksum(sd_u) == g["unet_checksum"] and state_dict_checksum(sd_p) == g["pre_checksum"]
    k = g["cases"][case]
    assert (k["lengths"] < k["spec"].shape[2]).any() and (k["refer_lengths"] < k["refer"].shape[2]).any()
    if case == "edges":
        assert 0 in k["t"].tolist() and 999 in k["t"].tolist()
    o = loss_oracle.diffusion_loss(sd_p, sd_u, ns2vc_denoiser_config(), k["c"], k["refer"], k["spec"], k["lengths"], k["refer_lengths"],
                                   k["t"], k["noise"])
    assert torch.equal(o["x"], k["x"]) and torch.equal(o["x_start"], k["target"])
    assert (o["model_out"] - k["model_out"]).abs().max().item() <= 2e-5
    assert abs(o["loss"].item() - k["loss"].item()) <= 1e-6 * abs(k["loss"].item())
    # the number forward() returns is mean_b(weight) * mean_b(row MSE), not the mean of the products (see loss_oracle)
    w = g["buffers"]["loss_weight"][k["t"]]
    assert abs((w.double().mean() * k["loss_row64"].mean()).item() - k["loss"].item()) <= 1e-5 * abs(k["loss"].item())
    assert abs((w.double() * k["loss_row64"]).mean().item() - k["loss"].item()) > 1e-3 * abs(k["loss"].item())


def _cpu_models():
    """A denoiser left on the CPU (20 latent + 16 content channels) and a stand-in for the encoders, which are never reached."""
    from ns2vc_b200.unet import UNet1DConditionModel
    unet = UNet1DConditionModel(in_channels=36, out_channels=20, block_out_channels=(32, 64, 64, 96), norm_num_groups=8,
                                cross_attention_dim=16, attention_head_dim=8)
    return types.SimpleNamespace(infer=None), unet


def test_argument_errors():
    from ns2vc_b200 import api
    from ns2vc_b200.loss import diffusion_loss, loss_profile
    assert api.diffusion_loss is diffusion_loss and api.loss_profile is loss_profile
    pre, unet = _cpu_models()
    B, T, S = 2, 12, 6
    c, refer, spec = torch.zeros(B, 16, T), torch.zeros(B, 20, S), torch.zeros(B, 20, T)
    ln, rl = torch.tensor([12, 5]), torch.tensor([6, 3])
    data = (c, refer, None, spec, None, ln, rl, None)
    with pytest.raises(RuntimeError, match="no CPU path"):
        diffusion_loss(pre, unet, data)
    bad = [
        (data[:7], {}),                                                            # not the 8-tuple
        ((c, refer, None, torch.zeros(B, 19, T), None, ln, rl, None), {}),         # spec channels
        ((torch.zeros(B, 16, T + 1), refer, None, spec, None, ln, rl, None), {}),  # c_padded frames
        ((c, refer, None, spec, None, torch.tensor([12, 0]), rl, None), {}),       # lengths outside [1, T]
        ((c, refer, None, spec, None, torch.tensor([13, 5]), rl, None), {}),
        ((c, refer, None, spec, None, ln, torch.tensor([7, 3]), None), {}),        # refer_lengths outside [1, S]
        (data, dict(t=torch.tensor([0, 1000]))),                                   # t outside [0, timesteps)
        (data, dict(t=torch.tensor([-1, 5]))),
        (data, dict(t=torch.tensor([0, 10]), timesteps=10)),
        (data, dict(t=torch.tensor([0, 1], dtype=torch.int32))),                   # dtype
        (data, dict(t=torch.zeros(3, 3, dtype=torch.int64))),                      # [K, B] with the wrong B
        (data, dict(noise=torch.zeros(B, 20, T + 1))),
        (data, dict(t=torch.tensor([0, 1]), noise=torch.zeros(2, B, 20, T))),      # per-k noise needs a [K, B] t
        (data, dict(t=torch.zeros(3, B, dtype=torch.int64), noise=torch.zeros(2, B, 20, T))),
        (data, dict(min_snr_gamma=0.0)),
    ]
    for d, kw in bad:
        with pytest.raises(ValueError):
            diffusion_loss(pre, unet, d, **kw)
    with pytest.raises(ValueError, match="empty"):
        loss_profile(pre, unet, data, t_grid=[])
    with pytest.raises(ValueError):
        loss_profile(pre, unet, data, t_grid=[0, 1000])


def test_default_draws_follow_the_reference_order():
    """randint, then randn_like (model.py:714-716), on the generator of the tensor's device; [K, B]: one randn_like per k."""
    from ns2vc_b200.loss import draw_t_noise
    x = torch.zeros(3, 5, 7)
    torch.manual_seed(4)
    t, noise = draw_t_noise(x, None, None, 1000)
    torch.manual_seed(4)
    want_t = torch.randint(0, 1000, (3,)).long()
    want_noise = torch.randn_like(x)
    assert t.dtype == torch.int64 and torch.equal(t, want_t) and torch.equal(noise, want_noise)
    tk = torch.zeros(4, 3, dtype=torch.int64)
    torch.manual_seed(5)
    t2, noise2 = draw_t_noise(x, tk, None, 1000)
    torch.manual_seed(5)
    assert t2 is tk and torch.equal(noise2, torch.stack([torch.randn_like(x) for _ in range(4)]))
    state = torch.get_rng_state()
    t3, noise3 = draw_t_noise(x, tk, noise2, 1000)                   # nothing to draw
    assert noise3 is noise2 and torch.equal(torch.get_rng_state(), state)


def test_install_diffusion_binds_validation_loss_and_keeps_forward():
    import ns2vc_b200
    from ns2vc_b200 import diffusion

    def forward(self, data, vocos):
        raise AssertionError("the reference's own forward")
    cls = type("NaturalSpeech2", (), {"forward": forward})
    ns2vc_b200.install_diffusion(types.SimpleNamespace(NaturalSpeech2=cls))
    assert cls.validation_loss is diffusion.validation_loss and cls.forward is forward
    model = cls()
    model.pre_model, model.diff_model = object(), types.SimpleNamespace(unet=object())
    with pytest.raises(TypeError):
        model.validation_loss(None)
    # the schedule check: the reference's buffers pass (with and without the min-SNR clamp), anything else does not
    for gamma in (None, 5):
        m = types.SimpleNamespace(**coefs.loss_buffers(1000, gamma))
        assert diffusion._loss_gamma(m) == (True, None if gamma is None else 5.0)
    m = types.SimpleNamespace(**coefs.loss_buffers(1000))
    m.sqrt_alphas_cumprod = m.sqrt_alphas_cumprod.clone()
    m.sqrt_alphas_cumprod[3] += 1e-3
    assert diffusion._loss_gamma(m) == (False, None)


# ------------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def models():
    from ns2vc_b200.pre_model import Pre_model
    from ns2vc_b200.unet import UNet1DConditionModel
    unet = UNet1DConditionModel(in_channels=356, out_channels=100, block_out_channels=(128, 256, 384, 512), norm_num_groups=8,
                                cross_attention_dim=256, attention_head_dim=8, addition_embed_type="text", resnet_time_scale_shift="scale_shift")
    unet.load_state_dict(make_state_dict(ns2vc_denoiser_config(), seed=0))
    pre = Pre_model(PRE_CFG)
    pre.load_state_dict(make_pre_state_dict(PRE_CFG, seed=0))
    return pre.cuda().eval(), unet.cuda().eval()


@pytest.mark.gpu
def test_q_sample_is_bit_identical_to_the_torch_expression():
    from ns2vc_b200.loss import q_sample
    g = torch.Generator(device="cuda").manual_seed(1)
    B, C, T, K = 5, 100, 203, 3                                     # T is not a multiple of 4
    spec = torch.randn(B, C, T, device="cuda", generator=g)
    spec[0, 0, :4] = -0.0
    lengths = torch.tensor([1, T, 77, T, 130], device="cuda")
    buf = {k: v.cuda() for k, v in coefs.loss_buffers(1000).items()}
    t = torch.tensor([[0, 999, 500, 1, 998], [37, 37, 37, 37, 37], [999, 0, 250, 750, 3]], device="cuda")
    noise = torch.randn(K, B, C, T, device="cuda", generator=g)
    for tt, nz in ((t[:1], noise[0]), (t, noise[0]), (t, noise)):   # [B] t; [K, B] t with shared and with per-k noise
        x_start, x, noise_m = q_sample(spec, nz.contiguous(), lengths, tt.contiguous(), want_noise=True)
        assert noise_m.shape == nz.shape
        for k in range(tt.shape[0]):
            nk = nz[k] if nz.dim() == 4 else nz
            want_xs, want_nm, want_x = torch_q_sample(spec, nk, lengths, tt[k], buf)
            assert torch.equal(bits(x_start), bits(want_xs))
            assert torch.equal(bits(noise_m[k] if nz.dim() == 4 else noise_m), bits(want_nm)), k
            assert torch.equal(bits(x[k]), bits(want_x)), k
        assert not x_start[0, :, 1:].any() and not x[:, 0, :, 1:].any()
    x_start2, x2 = q_sample(spec, noise, lengths, t)                # without the masked-noise output
    assert torch.equal(bits(x2), bits(x)) and torch.equal(bits(x_start2), bits(x_start))


@pytest.mark.gpu
@pytest.mark.parametrize("gamma", [None, 5.0])
def test_mse_rows_is_accurate_and_deterministic(gamma):
    from ns2vc_b200.loss import mse_rows
    g = torch.Generator(device="cuda").manual_seed(2)
    K, B, C, T = 3, 4, 100, 203                                     # C * T = 20 300: three chunks, the last one partial
    out = torch.randn(K, B, C, T, device="cuda", generator=g) * 3
    target = torch.randn(B, C, T, device="cuda", generator=g)
    t = torch.tensor([[0, 999, 500, 37], [10, 10, 10, 10], [999, 998, 1, 0]], device="cuda")
    w = coefs.loss_buffers(1000, gamma)["loss_weight"].cuda().double()[t]
    rows64 = (out.double() - target.double()[None]).pow(2).reshape(K, B, -1).mean(-1)
    want_loss = w.mean(-1) * rows64.mean(-1)                        # forward()'s broadcast: mean_b(w) * mean_b(row)
    rel = lambda a, b: ((a.double() - b).abs() / b.abs()).max().item()
    first = mse_rows(out, target, t, min_snr_gamma=gamma)
    assert rel(first[0], rows64) <= 1e-6 and rel(first[1], rows64 * w) <= 1e-6 and rel(first[2], want_loss) <= 1e-6
    assert rel(first[2][1], (rows64 * w).mean(-1)[1]) <= 1e-6      # the same t in every row: also the mean of the products
    again = mse_rows(out, target, t, min_snr_gamma=gamma)
    ws = torch.full((1 << 16,), 0xFF, dtype=torch.uint8, device="cuda")
    dirty = mse_rows(out, target, t, min_snr_gamma=gamma, ws=ws)
    per_k = mse_rows(out, target[None].expand(K, -1, -1, -1).contiguous(), t, min_snr_gamma=gamma)
    for a, b, c, d in zip(first, again, dirty, per_k):
        assert torch.equal(bits(a), bits(b)) and torch.equal(bits(a), bits(c)) and torch.equal(bits(a), bits(d))


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["drawn", "edges"])
def test_diffusion_loss_reproduces_the_reference_forward(gold, models, case):
    from ns2vc_b200.loss import diffusion_loss
    pre, unet = models
    k = gold("train_loss.pt")["cases"][case]
    r = diffusion_loss(pre, unet, case_data(k), t=k["t"], noise=k["noise"])
    assert r.loss.dim() == 0 and r.loss_row.shape == (4,) and r.model_out.shape == k["model_out"].shape
    assert torch.equal(bits(r.target.cpu()), bits(k["target"])) and torch.equal(bits(r.x.cpu()), bits(k["x"]))
    err = (r.model_out.cpu() - k["model_out"]).abs()
    worst = (err / (ATOL + RTOL * k["model_out"].abs())).max().item()
    e_loss = abs(r.loss.item() - k["loss"].item()) / abs(k["loss"].item())
    e_row = ((r.loss_row.cpu().double() - k["loss_row64"]).abs() / k["loss_row64"]).max().item()
    print(f"[loss {case}] model_out max|err| {err.max().item():.2e} worst err/tol {worst:.2f}; loss rel {e_loss:.2e}; rows rel {e_row:.2e}")
    assert worst <= 1.0 and e_loss <= LOSS_RTOL and e_row <= LOSS_RTOL
    w = coefs.loss_buffers(1000)["loss_weight"][k["t"]]
    assert torch.allclose(r.loss_weighted.cpu(), r.loss_row.cpu() * w, rtol=1e-6, atol=0)
    # the clamp only changes the weights
    r5 = diffusion_loss(pre, unet, case_data(k, "cuda"), t=k["t"].cuda(), noise=k["noise"].cuda(), min_snr_gamma=5.0)
    assert torch.equal(bits(r5.model_out), bits(r.model_out)) and torch.equal(bits(r5.loss_row), bits(r.loss_row))
    assert torch.allclose(r5.loss_weighted.cpu(), r.loss_row.cpu() * w.clamp(max=5.0), rtol=1e-6, atol=0)


@pytest.mark.gpu
def test_k_timesteps_in_one_call_equal_k_calls(gold, models):
    from ns2vc_b200.loss import diffusion_loss, loss_profile
    pre, unet = models
    k = gold("train_loss.pt")["cases"]["edges"]
    data = case_data(k, "cuda")
    K, B = 5, 4
    t = torch.tensor([[0, 999, 500, 37], [999, 0, 1, 998], [3, 3, 3, 3], [640, 120, 877, 412], [0, 0, 999, 999]])
    noise = torch.randn((K,) + tuple(k["spec"].shape), generator=torch.Generator().manual_seed(7))
    many = diffusion_loss(pre, unet, data, t=t, noise=noise)
    assert many.loss.shape == (K,) and many.loss_row.shape == (K, B) and many.model_out.shape == (K,) + tuple(k["spec"].shape)
    for j in range(K):
        one = diffusion_loss(pre, unet, data, t=t[j], noise=noise[j])
        for name in ("loss", "loss_row", "loss_weighted", "x", "model_out"):
            assert torch.equal(bits(getattr(many, name)[j]), bits(getattr(one, name))), (j, name)
        assert torch.equal(bits(many.target), bits(one.target))
    shared = diffusion_loss(pre, unet, data, t=t, noise=noise[2])
    assert torch.equal(bits(shared.model_out[2]), bits(many.model_out[2]))
    # the profile: every row at the same t_k
    grid = [0, 3, 500, 999]
    prof = loss_profile(pre, unet, data, t_grid=grid, noise=noise[2])
    assert prof.t.tolist() == [[v] * B for v in grid] and prof.loss.shape == (4,)
    assert torch.equal(bits(prof.model_out[1]), bits(many.model_out[2]))
    assert torch.allclose(prof.loss, prof.loss_weighted.mean(-1), rtol=1e-6, atol=0)
    assert torch.isfinite(prof.loss).all()


@pytest.mark.gpu
def test_default_draws_use_the_generator_as_the_reference_does(gold, models):
    from ns2vc_b200.loss import diffusion_loss
    pre, unet = models
    k = gold("train_loss.pt")["cases"]["drawn"]
    data = case_data(k, "cuda")
    torch.manual_seed(31)
    r = diffusion_loss(pre, unet, data)
    rng = torch.cuda.get_rng_state()
    torch.manual_seed(31)
    t = torch.randint(0, 1000, (4,), device="cuda").long()
    noise = torch.randn_like(data[3])
    assert torch.equal(torch.cuda.get_rng_state(), rng)
    assert torch.equal(r.t, t)
    buf = {n: v.cuda() for n, v in coefs.loss_buffers(1000).items()}
    _, _, want_x = torch_q_sample(data[3], noise, data[5], t, buf)
    assert torch.equal(bits(r.x), bits(want_x))
    explicit = diffusion_loss(pre, unet, data, t=t, noise=noise)
    assert torch.equal(bits(explicit.model_out), bits(r.model_out)) and torch.equal(bits(explicit.loss), bits(r.loss))


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["dpmsolver", "ddim"])
def test_samplers_are_undisturbed_by_a_loss_evaluation(gold, models, method):
    """Sampler, loss, the same sampler again on one unet and one session shape: bit-identical samples (four sampler runs, so the
    captured loop is replayed around a loss evaluation as well)."""
    from ns2vc_b200 import api
    from ns2vc_b200.loss import diffusion_loss
    pre, unet = models
    k = gold("train_loss.pt")["cases"]["drawn"]
    data = case_data(k, "cuda")
    xT = torch.randn(tuple(k["spec"].shape), generator=torch.Generator().manual_seed(3)).cuda()

    def sample():
        torch.manual_seed(9)
        return api.sample_from_features(pre, unet, xT, data[0], data[1], data[5], data[6], steps=6, method=method, eta=0.5 if method == "ddim" else 0.0)
    first = sample()
    for i in range(4):
        r = diffusion_loss(pre, unet, data, t=k["t"].cuda(), noise=k["noise"].cuda())
        assert torch.isfinite(r.loss)
        assert torch.equal(bits(sample()), bits(first)), f"run {i}"


class _NaturalSpeech2:
    """The attributes ``validation_loss`` reads of the reference's NaturalSpeech2 (model.py:451-498)."""

    def __init__(self, pre, unet, gamma=None):
        self.pre_model, self.diff_model, self.num_timesteps = pre, types.SimpleNamespace(unet=unet), 1000
        for n, v in {**coefs.diffusion_buffers(1000), **coefs.loss_buffers(1000, gamma)}.items():
            setattr(self, n, v.cuda())

    def forward(self, data, vocos):
        raise AssertionError("validation_loss must not call forward")


@pytest.mark.gpu
def test_validation_loss_returns_the_references_tuple(gold, models):
    import ns2vc_b200
    from ns2vc_b200.loss import diffusion_loss
    pre, unet = models
    cls = type("NaturalSpeech2", (_NaturalSpeech2,), {})
    ns2vc_b200.install_diffusion(types.SimpleNamespace(NaturalSpeech2=cls))
    k = gold("train_loss.pt")["cases"]["edges"]
    data = case_data(k, "cuda")
    out = cls(pre, unet).validation_loss(data, t=k["t"], noise=k["noise"])
    assert len(out) == 7
    loss, loss_diff, loss_f0, lf0, lf0_pred, model_out, target = out
    assert loss is loss_diff and loss.dim() == 0 and (loss_f0, lf0, lf0_pred) == (0, 0, 0)
    assert model_out.shape == k["model_out"].shape and torch.equal(bits(target.cpu()), bits(k["target"]))
    assert abs(loss.item() - k["loss"].item()) <= LOSS_RTOL * abs(k["loss"].item())
    # a model built with min_snr_loss_weight=True evaluates with its clamp
    clamped = cls(pre, unet, gamma=5).validation_loss(data, t=k["t"], noise=k["noise"])[0]
    assert torch.equal(bits(clamped), bits(diffusion_loss(pre, unet, data, t=k["t"], noise=k["noise"], min_snr_gamma=5.0).loss))
    assert clamped.item() < loss.item()
    torch.manual_seed(2)
    drawn = cls(pre, unet).validation_loss(data)
    assert torch.isfinite(drawn[0])
    broken = cls(pre, unet)
    broken.sqrt_alphas_cumprod = broken.sqrt_alphas_cumprod * 1.001
    with pytest.raises(ValueError, match="schedule"):
        broken.validation_loss(data)
