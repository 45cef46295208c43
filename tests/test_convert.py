"""Waveform-to-waveform conversion (``convert.convert_utterances`` / ``convert_slices``).

CPU: the CLI's stitching (``infer.py:99-141``) and the host length bookkeeping against ``oracle/convert_oracle.py``, and the
argument errors.  GPU, with small models chained consistently (ContentVec 32-dim units, 32-wide encoders of 2 layers, a tiny
UNet with 32-dim cross-attention, a 2-layer 128-wide Vocos): every stage of each slice of a ragged batch against the same slice
converted alone, the whole chain against the fp64 oracle chain, the x_T draws, and ``convert_slices`` end to end."""
import numpy as np
import pytest
import torch

from ns2vc_b200 import api, convert
from oracle import convert_oracle

SR = 44100


# ----------------------------------------------------------------------------------------------------------------- CPU
def _fake_convert(dat):
    """A stand-in for one slice's conversion: float32 24 kHz audio of the slice's length, its values a function of the input."""
    T = convert_oracle.lengths(len(dat), SR)["T"]
    g = np.random.default_rng(int(abs(dat).sum() * 1e3) % (2 ** 32) + len(dat))
    return g.standard_normal(T * 256).astype(np.float32)


def _audio_data(seed=0):
    g = np.random.default_rng(seed)
    spans = [(True, 0.21), (False, 1.37), (True, 0.05), (False, 2.61), (False, 0.4), (True, 0.33), (False, 0.93)]
    return [(tag, np.zeros(int(s * SR)) if tag else g.standard_normal(int(s * SR)) * 0.1) for tag, s in spans]


@pytest.mark.parametrize("clip,lg,lgr", [(0, 0, 0.75), (0.8, 0, 0.75), (1.0, 0.2, 0.75), (1.0, 0.2, 1), (1.2, 0.3, 0.5)])
def test_stitching_equals_the_cli_loop(clip, lg, lgr):
    audio_data = _audio_data()
    seen = []

    def conv(dat):
        seen.append(dat)
        return _fake_convert(dat)

    want = convert_oracle.cli_loop(audio_data, SR, conv, 0.5, clip, lg, lgr)
    subs = convert._plan_slices(audio_data, SR, 0.5, clip, lg)
    assert len(subs) == len(seen) and all(np.array_equal(a, b) and a.dtype == b.dtype for a, b in zip(subs, seen))
    got = convert.stitch(audio_data, SR, [_fake_convert(s) for s in subs], 0.5, clip, lg, lgr)
    assert got.dtype == np.float64 and got.shape == want.shape
    assert np.array_equal(got.view(np.int64), want.view(np.int64)), f"stitching differs at {np.flatnonzero(got != want)[:5]}"


def test_host_lengths_equal_the_oracle():
    for sr in (44100, 48000, 24000, 16000, 22050):
        for n in (7000, 13230, 44100, 44101, 176400, 368891 * 2, 1000003):
            assert convert.frame_plan(n, sr) == convert_oracle.lengths(n, sr), (sr, n)


def test_argument_errors():
    w = [torch.zeros(20000)]
    mel = torch.zeros(100, 30)
    for method in ("ddpm", "ddim", "euler"):
        with pytest.raises(ValueError):
            convert.convert_utterances(None, None, None, None, w, SR, mel, method=method)
    with pytest.raises(ValueError, match="empty"):
        convert.convert_utterances(None, None, None, None, [], SR, mel)
    with pytest.raises(ValueError, match="mono"):
        convert.convert_utterances(None, None, None, None, [torch.zeros(2, 20000)], SR, mel)
    with pytest.raises(ValueError, match="too short"):
        convert.convert_utterances(None, None, None, None, [torch.zeros(300)], SR, mel)
    with pytest.raises(ValueError, match="x_T"):
        convert.convert_utterances(None, None, None, None, w, SR, mel, x_T=[torch.zeros(1, 100, 3)])
    with pytest.raises(ValueError, match="trims no sample"):
        convert.convert_slices(None, None, None, None, _audio_data(), SR, mel, pad_seconds=0.00001)
    assert api.convert_utterances is convert.convert_utterances and api.convert_slices is convert.convert_slices


# ----------------------------------------------------------------------------------------------------------------- GPU
DURATIONS = (1.3, 0.3, 4.0, 2.2, 0.75, 3.1)      # seconds at 44.1 kHz; max_batch 4 splits them 4 + 2
PRE_CFG = {"phoneme_encoder": dict(in_channels=32, hidden_channels=32, out_channels=32, n_layers=2),
           "prompt_encoder": dict(in_channels=100, hidden_channels=32, out_channels=32, n_layers=2)}


@pytest.fixture(scope="module")
def chain():
    from ns2vc_b200.arch import UNetConfig
    from ns2vc_b200.content import ContentVec
    from ns2vc_b200.pre_model import Pre_model
    from ns2vc_b200.synth import CONTENTVEC_SMALL, linear_betas, make_contentvec_state_dict, make_pre_state_dict, make_vocos_state_dict
    from ns2vc_b200.vocoder import Vocos
    from test_gpu_parity import make_unet
    cv_sd = make_contentvec_state_dict(0, "trained_like", **CONTENTVEC_SMALL)
    cv = ContentVec.from_state_dict(cv_sd, num_heads=CONTENTVEC_SMALL["num_heads"]).to("cuda")
    pre_sd = make_pre_state_dict(PRE_CFG, 0)
    pre = Pre_model(PRE_CFG)
    pre.load_state_dict(pre_sd)
    pre = pre.to("cuda").eval()
    ucfg = UNetConfig(in_channels=132, out_channels=100, block_out_channels=(32, 64, 64, 96), norm_num_groups=8, cross_attention_dim=32,
                      num_heads=8, addition_embed_type="text", addition_embed_type_num_heads=4, resnet_time_scale_shift="scale_shift")
    unet, unet_sd = make_unet(ucfg)
    voc_sd = make_vocos_state_dict(0, "trained_like", dim=128, intermediate_dim=384, num_layers=2)
    voc = Vocos.from_state_dict(voc_sd).to("cuda")
    g = torch.Generator().manual_seed(3)
    wavs = []
    for d in DURATIONS:
        n = int(d * SR)
        t = torch.arange(n) / SR
        wavs.append((0.3 * torch.sin(2 * torch.pi * (110 + 300 * torch.rand(1, generator=g)) * t) + 0.05 * torch.randn(n, generator=g)).float())
    prompt = (torch.randn((100, 70), generator=g) - 4.0).float()
    models = dict(cv_sd=cv_sd, cv_heads=CONTENTVEC_SMALL["num_heads"], pre_sd=pre_sd, pre_layers=(2, 2), unet_sd=unet_sd, unet_cfg=ucfg,
                  voc_sd=voc_sd, betas=linear_betas(1000))
    return (cv, pre, unet, voc), wavs, prompt, models


def _x_T(wavs, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn((1, 100, convert.frame_plan(len(w), SR)["T"]), generator=g) for w in wavs]


def _close(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    err = (a - b).abs()
    return bool((err <= 1e-4 + 1e-3 * b.abs()).all()), err.max().item()


@pytest.mark.gpu
def test_every_stage_of_each_slice_matches_the_slice_alone(chain):
    models, wavs, prompt, _ = chain
    xs = _x_T(wavs, 1)
    steps = 8
    batched = {}
    for idx in api.batch_plan([len(w) for w in wavs], 4):
        r = convert.convert_batch(*models, [wavs[i] for i in idx], SR, [prompt] * len(idx), [xs[i] for i in idx], "unipc", steps)
        for j, i in enumerate(idx):
            batched[i] = {k: v[j] for k, v in r.items()}
    outs = convert.convert_utterances(*models, wavs, SR, prompt, steps=steps, max_batch=4, x_T=xs)
    bad = []
    for i, w in enumerate(wavs):
        alone = {k: v[0] for k, v in convert.convert_batch(*models, [w], SR, [prompt], [xs[i]], "unipc", steps).items()}
        got = batched[i]
        tag = f"slice {i} ({DURATIONS[i]} s, T_b={alone['latent'].shape[1]})"
        assert torch.equal(outs[i], got["audio"]), f"{tag}: convert_utterances differs from its batch"
        for k in ("units", "c", "content", "prompt", "latent"):
            ok, mx = _close(got[k], alone[k])
            if not ok:
                bad.append(f"{tag} {k}: max|diff| {mx:.3e}")
        a, b = got["audio"].double().cpu(), alone["audio"].double().cpu()
        rel = ((a - b).norm() / b.norm()).item()
        et = ((a - b).abs() / (1e-3 * b.abs() + 1e-4 * b.pow(2).mean().sqrt())).max().item()
        same = {k: torch.equal(got[k], alone[k]) for k in got}
        print(f"{tag}: audio ||diff||/||alone|| {rel:.2e}, elementwise err/tol {et:.3f}; bit-identical {[k for k, v in same.items() if v]}")
        if rel > 1e-4:
            bad.append(f"{tag} audio: ||diff||/||alone|| {rel:.2e}")
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
def test_chain_matches_the_fp64_oracle_of_each_slice(chain):
    models, wavs, prompt, om = chain
    xs = _x_T(wavs, 2)
    steps = 3
    outs = convert.convert_batch(*models, wavs, SR, [prompt] * len(wavs), xs, "unipc", steps)
    bad = []
    for i, w in enumerate(wavs):
        with torch.no_grad():
            ref = convert_oracle.convert_one(om, w, SR, prompt, xs[i], "unipc", steps, torch.float64)
            r32 = convert_oracle.convert_one(om, w, SR, prompt, xs[i], "unipc", steps, torch.float32)
        for k in ("units", "content", "prompt", "latent", "audio"):
            got, want = outs[k][i].double().cpu(), ref[k]
            if k == "units":
                want = want[:, :got.shape[1]]
            e32 = (r32[k].double() - want).abs().max().item()
            tol = torch.clamp(1e-3 * want.abs() + 1e-4 * want.pow(2).mean().sqrt(), min=2 * e32)
            r = ((got - want).abs() / tol).max().item()
            print(f"slice {i} ({DURATIONS[i]} s) {k:8s} err/tol {r:.3f}  fp32 oracle max {e32:.2e}")
            if r > 1.0:
                bad.append(f"slice {i} ({DURATIONS[i]} s) {k}: err/tol {r:.3f}")
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
def test_default_x_T_is_drawn_per_slice_in_input_order(chain):
    models, wavs, prompt, _ = chain
    torch.manual_seed(1234)
    got = convert.convert_utterances(*models, wavs, SR, prompt, steps=4, max_batch=4)
    torch.manual_seed(1234)
    xs = [torch.randn((1, 100, convert.frame_plan(len(w), SR)["T"]), device="cuda") for w in wavs]
    want = convert.convert_utterances(*models, wavs, SR, prompt, steps=4, max_batch=4, x_T=xs)
    for i in range(len(wavs)):
        assert torch.equal(got[i], want[i]), f"slice {i}: the default x_T is not the reference CLI's draw"


@pytest.mark.gpu
def test_convert_slices_end_to_end(chain):
    models, _, prompt, _ = chain
    audio_data = _audio_data(5)
    subs = convert._plan_slices(audio_data, SR, 0.5, 1.0, 0.2)
    xs = _x_T([s for s in subs], 3)
    per = convert.convert_utterances(*models, [torch.from_numpy(s.astype(np.float32)) for s in subs], SR, prompt, steps=4, max_batch=4, x_T=xs)
    it = iter(per)
    want = convert_oracle.cli_loop(audio_data, SR, lambda dat: next(it).cpu().numpy(), 0.5, 1.0, 0.2, 0.75)
    got = convert.convert_slices(*models, audio_data, SR, prompt, pad_seconds=0.5, clip_seconds=1.0, linear_gradient=0.2, steps=4,
                                 max_batch=4, x_T=xs)
    assert got.dtype == np.float64 and got.shape == want.shape
    assert np.array_equal(got, want), f"max|diff| {np.abs(got - want).max():.3e}"
