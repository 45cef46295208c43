"""Prompt-mel front end (``ns2vc_b200.frontend.resample`` / ``log_mel_spectrogram``, kernels in csrc/frontend.cu) against the
reference's recipe (inference/infer_tool.py:170-181) as recorded by oracle/make_golden_mel.py (tests/golden/frontend_mel.pt:
torchaudio in fp32 and fp64 on the reference's dataset/1/1.wav, dataset/2/2.wav and seeded synthetic signals).  The fixture
keeps the inputs, lengths, the recipe's own errors and torchaudio's values at pinned frames / samples; the full fp64 and fp32
outputs are rebuilt here by oracle/mel_oracle.py, which those pinned values tie to torchaudio's runs.

Accuracy bounds are multiples of the recipe's own fp32 error ``e_ref`` = max |torchaudio fp32 - torchaudio fp64| on the same input."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from ns2vc_b200 import _lib, frontend
from oracle import mel_oracle
from oracle.make_golden_mel import dense_rows as dense, pin_frames, pin_samples

DIVERGENT = [(44100, 24000, 368891), (22050, 24000, 122632), (44100, 16000, 368891)]   # fp32 rule != exact ceiling here


@pytest.fixture(scope="module")
def fx(gold):
    return gold("frontend_mel.pt")


def case_wav(c):
    return c["pcm_int16"].float() / 32768.0




# ------------------------------------------------------------------------------------------------------------------ CPU tier
def test_phase_tables_bitwise_equal_torchaudio(fx):
    """The host-built fp32 phase tables equal torchaudio's bit for bit (same fp64 formula, same fp32 phase offsets)."""
    L = _lib.lib()
    for key, t in fx["tables"].items():
        o, n = map(int, key.split("_"))
        P, T, W = C.c_int(), C.c_int(), C.c_int()
        _lib.check(L.ns2vc_resample_table(o, n, C.byref(P), C.byref(T), C.byref(W), None))
        kernel = dense(t["kernel"])
        assert (P.value, T.value, W.value) == (*kernel.shape, t["width"]), key
        buf = torch.empty(P.value * T.value)
        _lib.check(L.ns2vc_resample_table(o, n, None, None, None, buf.data_ptr()))
        assert torch.equal(buf.view(P.value, T.value).view(torch.int32), kernel.view(torch.int32)), key
        assert torch.equal(mel_oracle.sinc_kernel(o // math.gcd(o, n), n // math.gcd(o, n), torch.float32)[0].reshape(P.value, T.value),
                           kernel), key
    assert L.ns2vc_resample_table(24000, 24000, None, None, None, None) != 0


def test_filterbank_matches_melscale_fbanks(fx):
    """Same band supports as torchaudio's melscale_fbanks; each weight within 2 ulp of the mel points it is built from: torch's
    vectorised powf may round a mel point's frequency 1 ulp apart from the C library's, and a weight near a triangle's edge is
    a difference of nearby frequencies over the band width, so its ulp distance is not bounded by its own magnitude."""
    fb = torch.empty(513 * 100)
    _lib.check(_lib.lib().ns2vc_mel_filterbank(fb.data_ptr()))
    fb, ref = fb.view(513, 100), dense(fx["fbanks_t"]).t()
    assert torch.equal(fb != 0, ref != 0)
    m_max = 2595.0 * math.log10(1.0 + 12000.0 / 700.0)
    f_pts = (700.0 * (10.0 ** (torch.linspace(0.0, m_max, 102) / 2595.0) - 1.0)).numpy()
    ulp = np.spacing(f_pts)
    width = np.minimum(f_pts[1:-1] - f_pts[:-2], f_pts[2:] - f_pts[1:-1])                  # per band
    tol = 2 * np.maximum(ulp[2:], ulp[1:-1]) / width + 2 * np.spacing(np.abs(ref.numpy()))
    assert ((fb - ref).abs().numpy() <= tol).all(), (fb - ref).abs().max().item()
    # the tables the GPU path runs with are torch's own, as in the recipe
    window, fbt = frontend.mel_tables()
    assert torch.equal(window, torch.hann_window(1024)) and torch.equal(window, mel_oracle.hann_window())
    assert torch.equal(fbt, mel_oracle.mel_filterbank()) and torch.equal(fbt != 0, ref != 0)
    assert ((fbt - ref).abs().numpy() <= tol).all()


def test_out_length_is_torchaudios_fp32_rule():
    L = _lib.lib()
    for o, n, N in DIVERGENT:
        g = math.gcd(o, n)
        exact = -(-(n // g) * N // (o // g))
        assert L.ns2vc_resample_out_length(o, n, N) == exact - 1 == mel_oracle.out_length(o, n, N)
    for o, n in [(44100, 24000), (22050, 24000), (16000, 24000), (48000, 24000), (44100, 16000), (8000, 24000), (24000, 24000)]:
        for N in list(range(0, 700)) + [1023, 1024, 12345, 65536, 99999, 368890, 368891, 368892, 1 << 22]:
            assert L.ns2vc_resample_out_length(o, n, N) == mel_oracle.out_length(o, n, N), (o, n, N)
    assert L.ns2vc_resample_out_length(0, 24000, 5) == -1


def test_out_length_equals_torchaudio_output():
    ta = pytest.importorskip("torchaudio")
    L = _lib.lib()
    for o, n, N in DIVERGENT + [(44100, 24000, 1), (44100, 24000, 146), (22050, 24000, 513), (16000, 24000, 342), (48000, 24000, 1025),
                                (44100, 16000, 4410), (44100, 16000, 368890)]:
        assert L.ns2vc_resample_out_length(o, n, N) == ta.transforms.Resample(o, n)(torch.zeros(1, N)).shape[-1], (o, n, N)


def test_frame_counts_and_lengths(fx):
    for name, c in fx["cases"].items():
        assert c["pcm_int16"].shape == (c["n"],), name
        assert frontend.resample_out_length(c["sr"], 24000, c["n"]) == c["len24"], name
        assert c["frames"] == 1 + c["len24"] // 256, name


def test_oracle_equals_fixture(fx):
    """The fp64 oracle reproduces torchaudio's fp64 run (1e-12) and the fp32 oracle its fp32 run (same ops; within a quarter of the
    recipe's own fp32 error, so a different CPU FFT path cannot make it a different comparator) at every pinned value."""
    for name, c in fx["cases"].items():
        x = case_wav(c)
        fr, sm = pin_frames(c["frames"]), pin_samples(c["len24"])
        for dt, tol_r, tol_m in ((torch.float64, 1e-12, 1e-12), (torch.float32, 0.25 * c["e_ref_resample"], 0.25 * c["e_ref"])):
            tag = "f64" if dt == torch.float64 else "f32"
            r = mel_oracle.resample(x, c["sr"], 24000, dt)
            m = mel_oracle.log_mel(x, c["sr"], dt)
            assert r.shape == (c["len24"],) and m.shape == (100, c["frames"]), name
            assert (r[sm].double() - c[f"pin_wav24_{tag}"].double()).abs().max().item() <= tol_r, (name, tag)
            assert (m[:, fr].double() - c[f"pin_mel_{tag}"].double()).abs().max().item() <= tol_m, (name, tag)


def test_cpu_input_raises_and_short_input_is_rejected():
    with pytest.raises(RuntimeError, match="no CPU path"):
        frontend.log_mel_spectrogram(torch.zeros(2, 4000))
    with pytest.raises(RuntimeError, match="no CPU path"):
        frontend.resample(torch.zeros(4000), 44100, 24000)
    with pytest.raises(ValueError):
        frontend.log_mel_spectrogram(torch.zeros(512))                                   # reflect padding needs > 512 samples
    with pytest.raises(ValueError):
        frontend.log_mel_spectrogram(torch.zeros(2, 4000), lengths=torch.tensor([4000, 512]))
    with pytest.raises(ValueError):
        frontend.log_mel_spectrogram(torch.zeros(940), 44100)                            # 512 samples at 24 kHz
    with pytest.raises(ValueError):
        frontend.resample(torch.zeros(2, 10), 44100, 24000, lengths=torch.tensor([11, 3]))
    with pytest.raises(TypeError):
        frontend.resample(torch.zeros(10, dtype=torch.float64), 44100, 24000)


# ------------------------------------------------------------------------------------------------------------------ GPU tier
def padded_batch(x: torch.Tensor, pad: int = 777):
    """x [N] as row 1 of a 2-row batch of length N + pad: row 0 is full-length noise, so row 1's tail must be ignored."""
    N = x.shape[0]
    g = torch.Generator().manual_seed(N)
    w = torch.randn((2, N + pad), generator=g) * 0.3
    w[1, :N] = x
    return w, torch.tensor([N + pad, N])


@pytest.mark.gpu
def test_resampler_on_fixture_cases(fx):
    for name, c in fx["cases"].items():
        w, lens = padded_batch(case_wav(c))
        y, out_len = frontend.resample(w.cuda(), c["sr"], 24000, lens.cuda())
        y, out_len = y.cpu(), out_len.cpu()
        assert out_len[1].item() == c["len24"], name
        assert torch.all(y[1, c["len24"]:] == 0), name
        err = (y[1, :c["len24"]].double() - mel_oracle.resample(case_wav(c), c["sr"], 24000, torch.float64)).abs().max().item()
        assert err <= 4 * c["e_ref_resample"], (name, err, c["e_ref_resample"])


@pytest.mark.gpu
def test_resample_same_rate_is_a_copy():
    w = torch.randn(3, 1000).cuda()
    y, n = frontend.resample(w, 24000, 24000, torch.tensor([1000, 10, 0]).cuda())
    assert n.tolist() == [1000, 10, 0]
    assert torch.equal(y[0], w[0]) and torch.equal(y[1, :10], w[1, :10]) and torch.all(y[1, 10:] == 0) and torch.all(y[2] == 0)


@pytest.mark.gpu
def test_log_mel_on_fixture_cases(fx):
    for name, c in fx["cases"].items():
        w, lens = padded_batch(case_wav(c), pad=int(c["sr"] * 0.05))
        mel, frames = frontend.log_mel_spectrogram(w.cuda(), c["sr"], lens.cuda())
        mel, frames = mel.cpu(), frames.cpu()
        F = c["frames"]
        assert frames[1].item() == F, name
        assert torch.all(mel[1, :, F:] == 0), name
        err = (mel[1, :, :F].double() - mel_oracle.log_mel(case_wav(c), c["sr"], torch.float64)).abs().max().item()
        assert err <= 3 * c["e_ref"], (name, err, c["e_ref"])
        # alone, unbatched
        one, f1 = frontend.log_mel_spectrogram(case_wav(c).cuda(), c["sr"])
        assert one.shape == (100, F) and f1.tolist() == [F]
        assert torch.equal(one.cpu(), mel[1, :, :F]), name


@pytest.mark.gpu
@pytest.mark.parametrize("sr", [24000, 44100])
def test_random_ragged_batches(sr):
    g = torch.Generator().manual_seed(sr)
    for B in (1, 3, 8):
        N = int(torch.randint(sr // 10, sr // 2, (1,), generator=g))
        lens = torch.randint(int(0.03 * sr), N + 1, (B,), generator=g)
        lens[0] = N
        w = torch.randn((B, N), generator=g) * torch.linspace(0.01, 0.8, N) ** 2
        mel, frames = frontend.log_mel_spectrogram(w.cuda(), sr, lens.cuda())
        want, want_frames = mel_oracle.log_mel_batch(w, sr, lens.tolist(), torch.float64)
        got32, _ = mel_oracle.log_mel_batch(w, sr, lens.tolist(), torch.float32)
        e_ref = (got32.double() - want).abs().max().item()
        mel = mel.cpu()
        assert torch.equal(frames.cpu(), want_frames) and mel.shape == want.shape
        err = (mel.double() - want).abs().max().item()
        assert err <= 3 * e_ref, (B, err, e_ref)
        for b in range(B):
            F = int(want_frames[b])
            assert torch.all(mel[b, :, F:] == 0)
            one, _ = frontend.log_mel_spectrogram(w[b, :lens[b]].contiguous().cuda(), sr)
            assert torch.equal(one.cpu(), mel[b, :, :F]), (B, b)


@pytest.mark.gpu
def test_downstream_prompt_encoder(fx):
    """Our GPU mel of 2.wav and the reference's fp32 mel through the oracle encoders: the prompt output agrees to the encoders'
    own tolerance."""
    from ns2vc_b200.synth import make_pre_state_dict
    from oracle import pre_model_oracle
    c = fx["cases"]["2.wav"]
    mel, _ = frontend.log_mel_spectrogram(case_wav(c)[None].cuda(), c["sr"])
    cfg = {"phoneme_encoder": dict(in_channels=256, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2),
           "prompt_encoder": dict(in_channels=100, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2)}
    sd = make_pre_state_dict(cfg, 0)
    S = c["frames"]
    cc = torch.randn((1, 256, 40), generator=torch.Generator().manual_seed(0))
    lens, rlens = torch.tensor([40]), torch.tensor([S])
    with torch.no_grad():
        _, ours = pre_model_oracle.pre_model_infer(sd, cc, mel.cpu(), lens, rlens, 6, 6)
        ref32 = mel_oracle.log_mel(case_wav(c), c["sr"], torch.float32)      # the reference's fp32 recipe (same ops as torchaudio)
        _, ref = pre_model_oracle.pre_model_infer(sd, cc, ref32[None], lens, rlens, 6, 6)
    worst = ((ours - ref).abs() / (1e-4 + 1e-3 * ref.abs())).max().item()
    assert worst <= 1.0, worst
