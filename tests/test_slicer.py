"""The silence slicer (``slicer.py``, ``csrc/slicer.cu``) and the whole-CLI call ``convert.convert_files``.

CPU: the numpy restatement of librosa 0.10's ``feature.rms`` (``oracle/slicer_oracle.py``) against the fixture that the
reference's own ``Slicer`` wrote (``oracle/make_golden_slicer.py``), the host decision logic on the fixture's rms frames,
``chunks2audio``, argument errors and the order of ``convert_files``' default x_T draws.  GPU: the RMS kernel bit for bit
against the oracle (every fixture signal, and a ragged batch of mixed rates with NaN past each length), ``cut`` / ``cut_batch``
against the fixture's chunk dicts, and ``convert_files`` against one ``convert_slices`` call per (file, voice) pair."""
import numpy as np
import pytest
import torch

from ns2vc_b200 import api, convert, frontend, slicer
from oracle import slicer_oracle
from oracle.make_golden_slicer import samples
from test_convert import _audio_data, chain  # noqa: F401  (chain: the small conversion chain, a module-scoped fixture)

RATES = (16000, 22050, 44100, 48000, 11025)


@pytest.fixture(scope="module")
def cases(gold):
    return gold("slicer.pt")


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


# ----------------------------------------------------------------------------------------------------------------- CPU
def test_oracle_rms_equals_golden(cases):
    assert {c["sr"] for c in cases} == set(RATES)
    for c in cases:
        got = slicer_oracle.rms(samples(c), c["win"], c["hop"])[0]
        assert np.array_equal(_bits(got), _bits(c["rms"].numpy())), c["name"]


def test_slicer_params_equal_the_reference_arithmetic(cases):
    assert slicer.hop_win(11025) == (220, 880)          # round(220.5) halves to even
    for c in cases:
        p = slicer.slicer_params(c["sr"], c["db"], c["min_len"])
        assert p == slicer_oracle.slicer_params(c["sr"], c["db"], c["min_len"]), c["name"]
        assert (p["hop"], p["win"]) == (c["hop"], c["win"])
        assert slicer.num_frames(c["n"], c["hop"], c["win"]) == c["rms"].shape[0]


def test_host_decision_logic_on_golden_rms_equals_golden_chunks(cases):
    for c in cases:
        p = slicer.slicer_params(c["sr"], c["db"], c["min_len"])
        assert slicer.slice_from_rms(c["rms"].numpy(), c["n"], p) == c["chunks"], c["name"]


def test_chunks2audio_equals_the_reference(cases):
    for c in cases:
        y = samples(c)
        for wav in (y, torch.from_numpy(y)):
            got = slicer.chunks2audio(wav, c["chunks"])
            assert [t for t, _ in got] == [t for t, _, _ in c["chunks2audio"]], c["name"]
            for (_, a), (_, s, e) in zip(got, c["chunks2audio"]):
                assert a.dtype == np.float32 and np.array_equal(a, y[s:e]), c["name"]


def test_argument_errors():
    y = np.zeros(20000, np.float32)
    with pytest.raises(ValueError, match="mono"):
        slicer.cut(np.zeros((2, 20000), np.float32), 44100)
    with pytest.raises(ValueError, match="mono"):
        slicer.chunks2audio(np.zeros((1, 20000), np.float32), {"0": {"slice": False, "split_time": "0,20000"}})
    with pytest.raises(ValueError, match="float32"):
        slicer.cut(np.zeros(20000), 44100)
    with pytest.raises(ValueError, match="min_len"):
        slicer.cut(y, 44100, min_len=200)
    with pytest.raises(ValueError, match="sample rate"):
        slicer.cut_batch([y, y], [44100])
    with pytest.raises(ValueError, match="hop"):
        slicer.hop_win(20)
    with pytest.raises(ValueError, match="bad arguments"):
        slicer.num_frames(100, 0, 880)
    with pytest.raises(ValueError, match="bad arguments"):
        slicer.num_frames(100, 220, 1 << 20)
    with pytest.raises(ValueError, match="no rows|float32"):
        slicer.rms_frames(torch.zeros(3, 4, 5), None, 44100)
    files, voices = [(y, 44100)], [(y, 44100)]
    with pytest.raises(ValueError, match="ddpm"):
        convert.convert_files(None, None, None, None, files, voices, method="ddpm")
    with pytest.raises(ValueError, match="at least one"):
        convert.convert_files(None, None, None, None, [], voices)
    with pytest.raises(ValueError, match="mono"):
        convert.convert_files(None, None, None, None, [(np.zeros((2, 100), np.float32), 44100)], voices)
    with pytest.raises(ValueError, match="trims no sample"):
        convert.convert_files(None, None, None, None, files, voices, pad_seconds=0.00001)
    assert api.convert_files is convert.convert_files


def test_convert_files_draws_x_T_file_then_voice_then_sub_slice():
    srs = (44100, 16000)
    sub_T = []
    for seed, sr in zip((1, 2), srs):
        subs = convert._plan_slices(_audio_data(seed), sr, 0.5, 1.0, 0.2)
        sub_T.append([convert.frame_plan(len(s), sr)["T"] for s in subs])
    assert len(sub_T[0]) > 1 and sub_T[0] != sub_T[1]
    torch.manual_seed(11)
    got = convert._files_x_T(sub_T, 3, "cpu")
    after = torch.get_rng_state()
    torch.manual_seed(11)
    for f, Ts in enumerate(sub_T):            # infer.py:77 (files), :92 (voices), :99-122 (sub-slices)
        for v in range(3):
            for k, T in enumerate(Ts):
                want = torch.randn((1, 100, T))
                assert torch.equal(got[f][v][k], want), f"file {f} voice {v} sub-slice {k}"
    assert torch.equal(torch.get_rng_state(), after)


# ----------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_rms_frames_bit_identical_to_the_oracle_on_every_golden_signal(cases):
    for c in cases:
        y = samples(c)
        x = torch.full((c["n"] + 777,), float("nan"), device="cuda")
        x[:c["n"]] = torch.from_numpy(y).cuda()
        rms, frames = slicer.rms_frames(x, torch.tensor([c["n"]]), c["sr"])
        want = slicer_oracle.rms(y, c["win"], c["hop"])[0]
        assert frames == [want.shape[0]] and rms.shape == (1, want.shape[0]), c["name"]
        got = rms[0].cpu().numpy()
        bad = np.flatnonzero(_bits(got) != _bits(want))
        assert bad.size == 0, f"{c['name']}: {bad.size} frames differ, first {bad[:5]}"


@pytest.mark.gpu
def test_rms_frames_ragged_batch_of_mixed_rates_with_nan_past_the_lengths(cases):
    g = np.random.default_rng(4)
    rows = [(samples(c), c["sr"]) for c in cases]
    for k, sr in enumerate(RATES * 2):
        n = int(sr * g.uniform(0.01, 2.5)) if k else 5
        rows.append(((g.standard_normal(n) * g.uniform(1e-3, 0.8)).astype(np.float32), sr))
    N = max(len(y) for y, _ in rows) + 100
    x = torch.full((len(rows), N), float("nan"))
    for j, (y, _) in enumerate(rows):
        x[j, :len(y)] = torch.from_numpy(y)
    lengths = torch.tensor([len(y) for y, _ in rows])
    rms, frames = slicer.rms_frames(x.cuda(), lengths.cuda(), [sr for _, sr in rows])
    rms = rms.cpu().numpy()
    for j, (y, sr) in enumerate(rows):
        hop, win = slicer.hop_win(sr)
        want = slicer_oracle.rms(y, win, hop)[0]
        assert frames[j] == want.shape[0]
        bad = np.flatnonzero(_bits(rms[j, :frames[j]]) != _bits(want))
        assert bad.size == 0, f"row {j} ({sr} Hz, {len(y)} samples): {bad.size} frames differ, first {bad[:5]}"
        assert not rms[j, frames[j]:].any(), f"row {j}: frames past its count are not 0"


@pytest.mark.gpu
def test_cut_and_cut_batch_equal_the_golden_chunks(cases):
    for c in cases:
        assert slicer.cut(samples(c), c["sr"], c["db"], c["min_len"]) == c["chunks"], c["name"]
    for db, min_len in {(c["db"], c["min_len"]) for c in cases}:
        group = [c for c in cases if (c["db"], c["min_len"]) == (db, min_len)]
        got = slicer.cut_batch([torch.from_numpy(samples(c)) for c in group], [c["sr"] for c in group], db, min_len)
        assert got == [c["chunks"] for c in group], (db, min_len)


def _file(sr, spans, seed):
    """Tone-plus-noise voice and digital-zero silence, [(is_voice, seconds), ...] at sr."""
    g = torch.Generator().manual_seed(seed)
    parts = []
    for voiced, s in spans:
        n = int(s * sr)
        t = torch.arange(n) / sr
        parts.append(0.3 * torch.sin(2 * torch.pi * (120 + 200 * torch.rand(1, generator=g)) * t) + 0.05 * torch.randn(n, generator=g)
                     if voiced else torch.zeros(n))
    return torch.cat(parts).float().numpy()


@pytest.mark.gpu
def test_convert_files_equals_convert_slices_per_pair_with_cli_noise(chain):
    models = chain[0]
    files = [(_file(44100, [(False, 0.4), (True, 5.3), (False, 0.6), (True, 1.2)], 1), 44100),
             (_file(16000, [(True, 2.1), (False, 0.5)], 2), 16000)]
    voice0 = _file(24000, [(True, 1.5)], 3)
    voices = [(np.stack([voice0, voice0[::-1].copy()]), 24000), (_file(44100, [(True, 0.9)], 4), 44100)]
    kw = dict(pad_seconds=0.5, clip_seconds=2.0, linear_gradient=0.2)
    audio_data = [slicer.chunks2audio(w, slicer.cut(w, sr, -40)) for w, sr in files]
    assert len(audio_data[0]) >= 2 and audio_data[1][-1][0], "the test files should hold silences the slicer cuts"
    subs = [convert._plan_slices(a, sr, kw["pad_seconds"], kw["clip_seconds"], kw["linear_gradient"]) for a, (_, sr) in zip(audio_data, files)]
    mels = [frontend.log_mel_spectrogram(torch.from_numpy(voice0).cuda(), 24000)[0],
            frontend.log_mel_spectrogram(torch.from_numpy(voices[1][0]).cuda(), 44100)[0]]
    torch.manual_seed(77)
    xs = [[[torch.randn((1, 100, convert.frame_plan(len(s), sr)["T"]), device="cuda") for s in ss] for _ in voices]
          for ss, (_, sr) in zip(subs, files)]
    want_state = torch.cuda.get_rng_state()
    torch.manual_seed(77)
    out = convert.convert_files(*models, files, voices, steps=4, max_batch=4, **kw)
    assert torch.equal(torch.cuda.get_rng_state(), want_state), "the generator did not end where the CLI's draws leave it"
    for f, ((_, sr), a) in enumerate(zip(files, audio_data)):
        for v in range(len(voices)):
            want = convert.convert_slices(*models, a, sr, mels[v], steps=4, max_batch=4, x_T=xs[f][v], **kw)
            got = out[f][v]
            assert got.dtype == np.float64 and got.shape == want.shape, (f, v, got.shape, want.shape)
            assert np.array_equal(got, want), f"file {f} voice {v}: max|diff| {np.abs(got - want).max():.3e}"
    again = convert.convert_files(*models, files, voices, steps=4, max_batch=4, x_T=xs, **kw)
    assert all(np.array_equal(again[f][v], out[f][v]) for f in range(2) for v in range(2))

