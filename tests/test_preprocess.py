"""Corpus preprocessing (``preprocess.preprocess_utterances`` / ``dataset_item`` / ``save``) against the reference's
``process_one`` as recorded by oracle/make_golden_preprocess.py (tests/golden/preprocess.pt: torchaudio's transforms and the
content oracle on the CPU, at a small seeded ContentVec configuration with 256 output channels).

CPU: the host length plans, the output names and ``resize_f0`` against the fixture, argument errors raised before any device
work, and the default f0's ImportError without pyworld.  GPU: every record against the fixture (the resampler within 4 and the
log-mel within 3 times the recipe's own fp32 error, as tests/test_frontend_mel.py bounds them; the units within the elementwise
tolerance of tests/test_content.py), batch independence at max_batch 1, 3 and 8 in shuffled order, a save / load round trip
through the loader's alignment, the training objective on records against the fixture's tensors, and two ranks."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist

from ns2vc_b200 import frontend, preprocess
from ns2vc_b200.content import ContentVec
from ns2vc_b200.synth import make_contentvec_state_dict, state_dict_checksum
from oracle import content_oracle, mel_oracle

RTOL, ATOL_RMS = 1e-3, 1e-4          # tests/test_content.py's elementwise bound on the units
BATCH_RTOL = 1e-3                    # tests/test_utterance_loss.py: one utterance's objective under different batch partners


@pytest.fixture(scope="module")
def fx(gold):
    return gold("preprocess.pt")


def mono_input(it):
    """The fixture's input as the caller passes it: 1-D when mono, [2, N] when stereo."""
    x = it["pcm_int16"].float() / 32768.0
    return x[0] if x.shape[0] == 1 else x


def fx_items(fx):
    return [(mono_input(it), it["sr"]) for it in fx["items"]]


def mixed64(it):
    """process_one's fp32 mono mix, in fp64 for the oracles"""
    x = it["pcm_int16"].float() / 32768.0
    return (x.mean(dim=0) if x.shape[0] > 1 else x[0]).double()


# ------------------------------------------------------------------------------------------------------------------ CPU tier
def test_length_plans_match_the_fixture(fx):
    for k, it in enumerate(fx["items"]):
        p = preprocess.length_plan(it["pcm_int16"].shape[-1], it["sr"])
        assert p["n16"] == it["wav16k"].shape[-1] and p["n24"] == it["wav24k"].shape[-1], k
        assert p["units"] == it["soft"].shape[-1] and p["frames"] == it["frames"] and p["spec"] == it["spec"].shape[-1], k
    assert fx["items"][5]["wav16k"].shape[-1] == 400                          # the shortest accepted input
    assert preprocess.length_plan(1099, 44100)["n16"] == 399


def test_output_names_and_resize_f0_match_the_reference(fx):
    for c in fx["names"]:
        got = preprocess.output_paths(c["filename"], c["in_dir"])
        assert got == {k: c[k] for k in ("wav", "soft", "f0", "spec")}, c["filename"]
    assert any(".flac" in c["filename"] for c in fx["names"]) and any(".wav/" in c["filename"] for c in fx["names"])
    with pytest.raises(ValueError, match="in_dir is empty"):
        preprocess.output_paths("a.wav", "")
    for c in fx["resize_f0"]:
        got = preprocess.resize_f0(c["f0"], c["target_len"])
        assert got.shape == (c["target_len"],) and np.array_equal(got, c["resized"]), (len(c["f0"]), c["target_len"])


def test_argument_errors_come_before_any_device_work():
    ok = torch.zeros(8000)
    cases = [([], "items is empty"),
             ([(ok, 16000), (torch.zeros(2, 3, 800), 16000)], "item 1: expected a floating-point wav"),
             ([(torch.zeros(8000, dtype=torch.int16), 16000)], "item 0: expected a floating-point wav"),
             ([(torch.zeros(0, 8000), 16000)], "item 0: wav has no channels"),
             ([(ok, 0)], "item 0: bad sample rate"),
             ([(ok, 16000.5)], "item 0: bad sample rate"),
             ([(ok, True)], "item 0: bad sample rate"),
             ([(ok, 16000), ok], "item 1: expected a \\(wav, sr\\) pair"),
             ([(ok, 16000), (ok, 16000), (torch.zeros(399), 16000)], "item 2: 399 samples at 16000 Hz give 399 at 16 kHz"),
             ([(torch.zeros(1099), 44100)], "item 0: 1099 samples"),
             ([(ok, 736000)], "item 0: 736000 -> 16000 Hz cannot be resampled here: .*46:1")]
    for items, msg in cases:
        with pytest.raises(ValueError, match=msg):
            preprocess.preprocess_utterances(None, items)        # no model: nothing past the host checks may run
    with pytest.raises(ValueError, match="max_batch"):
        preprocess.preprocess_utterances(None, [(ok, 16000)], max_batch=0)


def test_default_f0_needs_pyworld(fx, tmp_path, monkeypatch):
    monkeypatch.setitem(sys.modules, "pyworld", None)             # import pyworld raises ImportError
    it = fx["items"][0]
    rec = dict(wav24k=it["wav24k"], soft=it["soft"], spec=it["spec"], frames=it["frames"])
    in_dir = str(tmp_path / "corpus")
    with pytest.raises(ImportError, match="pyworld"):
        preprocess.save(rec, os.path.join(in_dir, "spk", "a.wav"), in_dir)
    assert not any(tmp_path.iterdir()), "nothing may be written before the ImportError"


def test_f0_of_the_wrong_shape_writes_nothing(fx, tmp_path):
    it = fx["items"][0]
    rec = dict(wav24k=it["wav24k"], soft=it["soft"], spec=it["spec"], frames=it["frames"])
    in_dir = str(tmp_path / "corpus")
    with pytest.raises(ValueError, match="f0_fn returned"):
        preprocess.save(rec, os.path.join(in_dir, "a.wav"), in_dir, f0_fn=lambda w: np.zeros((2, 3)))
    assert not any(tmp_path.iterdir())


def stub_f0(wav24k: np.ndarray) -> np.ndarray:
    """DIO's frame count for the signal (one per hop, plus one), voiced at 150 Hz with unvoiced ends"""
    n = wav24k.shape[0] // 256 + 1
    f0 = np.full(n, 150.0)
    f0[:2] = 0
    f0[-1] = 0
    return f0


def round_trip(rec, tmp_path, name):
    """save, then NS2VCDataset.get_audio (dataset.py:73-92) restated on the files; returns (paths, get_audio's c, spec, audio)"""
    import scipy.io.wavfile
    in_dir = str(tmp_path / "corpus")
    paths = preprocess.save(rec, os.path.join(in_dir, "spk", name), in_dir, f0_fn=stub_f0)
    assert paths == preprocess.output_paths(os.path.join(in_dir, "spk", name), in_dir)
    assert all(os.path.exists(p) for p in paths.values()) and "corpus_processed" in paths["wav"]
    sr, data = scipy.io.wavfile.read(paths["wav"])
    assert sr == 24000 and data.dtype == np.float32 and data.ndim == 1
    audio = torch.from_numpy(data)[None]
    assert torch.equal(audio, rec["wav24k"].cpu())
    soft, spec = torch.load(paths["soft"]), torch.load(paths["spec"])
    assert soft.dtype == spec.dtype == torch.float32
    assert torch.equal(soft, rec["soft"].cpu()) and torch.equal(spec, rec["spec"].cpu())
    f0 = np.load(paths["f0"])
    assert f0.shape == (rec["frames"],) and f0.dtype == np.float64
    spec = spec.squeeze(0)
    c = frontend.repeat_expand_2d(soft.squeeze(0), f0.shape[0])
    lmin = min(c.size(-1), spec.size(-1))
    assert abs(c.size(-1) - spec.size(-1)) < 3
    assert abs(audio.shape[1] - lmin * 256) < 3 * 256
    return c[:, :lmin], spec[:, :lmin], audio[:, :lmin * 256]


def test_round_trip_of_fixture_records(fx, tmp_path):
    for k, it in enumerate(fx["items"]):
        rec = dict(wav24k=it["wav24k"], soft=it["soft"], spec=it["spec"], frames=it["frames"])
        got = round_trip(rec, tmp_path, f"{k}.flac")
        for a, b in zip(got, preprocess.dataset_item(rec)):
            assert torch.equal(a, b), k


# ------------------------------------------------------------------------------------------------------------------ GPU tier
@pytest.fixture(scope="module")
def cv(fx):
    sd = make_contentvec_state_dict(fx["cv_seed"], fx["cv_regime"], **fx["cv_cfg"])
    assert state_dict_checksum(sd) == fx["cv_checksum"], "regenerated ContentVec weights differ from the fixture's"
    return ContentVec.from_state_dict(sd, num_heads=fx["cv_cfg"]["num_heads"]).cuda().eval(), sd


def soft_ratio(got, ref, e32):
    """worst |got - ref| / max(1e-3 |ref| + 1e-4 rms(ref), 2 e32) (tests/test_content.py's bound)"""
    got, ref = got.double().cpu(), ref.double().cpu()
    tol = torch.clamp(RTOL * ref.abs() + ATOL_RMS * ref.pow(2).mean().sqrt(), min=2 * e32)
    return ((got - ref).abs() / tol).max().item()


@pytest.fixture(scope="module")
def records(fx, cv):
    return preprocess.preprocess_utterances(cv[0], fx_items(fx), max_batch=8)


@pytest.mark.gpu
def test_records_match_the_reference(fx, cv, records):
    _, sd = cv
    heads = fx["cv_cfg"]["num_heads"]
    for k, (it, r) in enumerate(zip(fx["items"], records)):
        sr, x = it["sr"], mixed64(it)
        assert r["frames"] == it["frames"], k
        assert r["wav24k"].shape == it["wav24k"].shape and r["spec"].shape == it["spec"].shape and r["soft"].shape == it["soft"].shape, k
        assert r["wav24k"].is_cuda and r["wav24k"].dtype == r["soft"].dtype == r["spec"].dtype == torch.float32
        if sr == 24000:
            assert torch.equal(r["wav24k"].cpu(), it["wav24k"]), k
        else:
            err = (r["wav24k"][0].cpu().double() - mel_oracle.resample(x, sr, 24000)).abs().max().item()
            assert err <= 4 * it["e_ref_24k"], (k, err, it["e_ref_24k"])
        err = (r["spec"][0].cpu().double() - mel_oracle.log_mel(x, sr)).abs().max().item()
        assert err <= 3 * it["e_ref_mel"], (k, err, it["e_ref_mel"])
        w16 = x if sr == 16000 else mel_oracle.resample(x, sr, 16000)
        soft64 = content_oracle.extract(sd, w16[None], heads)[0].t()
        worst = soft_ratio(r["soft"][0], soft64, it["e_ref_soft"])
        print(f"item {k} ({sr} Hz): units err/tol {worst:.3f}")
        assert worst <= 1.0, k


@pytest.mark.gpu
@pytest.mark.parametrize("max_batch", [1, 3, 8])
def test_records_do_not_depend_on_the_batch(fx, cv, max_batch):
    items = fx_items(fx)
    alone = [preprocess.preprocess_utterances(cv[0], [i], max_batch=1)[0] for i in items]
    perm = torch.randperm(len(items), generator=torch.Generator().manual_seed(max_batch)).tolist()
    got = preprocess.preprocess_utterances(cv[0], [items[i] for i in perm], max_batch=max_batch)
    identical = 0
    for j, i in enumerate(perm):
        a, b = got[j], alone[i]
        assert a["frames"] == b["frames"]
        assert torch.equal(a["wav24k"], b["wav24k"]) and torch.equal(a["spec"], b["spec"]), (max_batch, i)
        assert soft_ratio(a["soft"], b["soft"], fx["items"][i]["e_ref_soft"]) <= 1.0, (max_batch, i)
        identical += torch.equal(a["soft"], b["soft"])
    print(f"max_batch {max_batch}: units bit-identical to the item alone for {identical} of {len(items)}")


@pytest.mark.gpu
def test_save_round_trip_through_the_loader(records, tmp_path):
    for k, rec in enumerate(records):
        got = round_trip(rec, tmp_path, f"{k}.mp3" if k % 2 else f"{k}.wav")
        want = preprocess.dataset_item(rec)
        assert want[0].shape == (256, rec["frames"]) and want[1].shape == (100, rec["frames"])
        for a, b in zip(got, want):
            assert torch.equal(a, b.cpu()), k


@pytest.mark.gpu
def test_scoring_records_equals_scoring_the_reference_tensors(fx, records):
    from ns2vc_b200.arch import ns2vc_denoiser_config
    from ns2vc_b200.loss import utterance_losses
    from ns2vc_b200.pre_model import Pre_model
    from ns2vc_b200.synth import make_pre_state_dict, make_state_dict
    from ns2vc_b200.unet import UNet1DConditionModel
    from test_utterance_loss import PRE_CFG
    unet = UNet1DConditionModel(in_channels=356, out_channels=100, block_out_channels=(128, 256, 384, 512), norm_num_groups=8,
                                cross_attention_dim=256, attention_head_dim=8, addition_embed_type="text", resnet_time_scale_shift="scale_shift")
    unet.load_state_dict(make_state_dict(ns2vc_denoiser_config(), seed=0))
    pre = Pre_model(PRE_CFG)
    pre.load_state_dict(make_pre_state_dict(PRE_CFG, seed=0))
    pre, unet = pre.cuda().eval(), unet.cuda().eval()
    refer = fx["items"][6]["spec"][0]                                           # one prompt mel for every utterance
    ours = [(c, spec, refer.cuda()) for c, spec, _ in map(preprocess.dataset_item, records)]
    theirs = []
    for it in fx["items"]:
        F = it["frames"]
        theirs.append((frontend.repeat_expand_2d(it["soft"][0], F)[:, :F], it["spec"][0, :, :F], refer))
    g = torch.Generator().manual_seed(4)
    t = torch.tensor([0, 10, 100, 250, 500, 750, 900, 999])
    noise = [torch.randn(100, it["frames"], generator=g) for it in fx["items"]]
    a = utterance_losses(pre, unet, ours, t=t, noise=noise, max_batch=8)
    b = utterance_losses(pre, unet, theirs, t=t, noise=noise, max_batch=8)
    rel = lambda u, v: ((u.double().cpu() - v.double().cpu()).abs() / v.double().cpu().abs()).max().item()
    print(f"loss rel {rel(a.loss, b.loss):.2e}, mse rel {rel(a.mse, b.mse):.2e}")
    assert rel(a.loss, b.loss) <= BATCH_RTOL and rel(a.mse, b.mse) <= BATCH_RTOL


def _shard_worker(rank, world, out_dir):
    from conftest import GOLD
    fx = torch.load(os.path.join(GOLD, "preprocess.pt"), weights_only=False)
    sd = make_contentvec_state_dict(fx["cv_seed"], fx["cv_regime"], **fx["cv_cfg"])
    dev = torch.device("cuda", torch.cuda.current_device())
    m = ContentVec.from_state_dict(sd, num_heads=fx["cv_cfg"]["num_heads"]).to(dev).eval()
    recs = preprocess.preprocess_utterances(m, fx_items(fx), max_batch=3, group=dist.group.WORLD)
    path = os.path.join(out_dir, f"rank{rank}.pt")
    torch.save(dict(backend=str(dist.get_backend()), records=[{k: (v.cpu() if torch.is_tensor(v) else v) for k, v in r.items()}
                                                              for r in recs]), path)
    return path


@pytest.mark.gpu
def test_two_ranks_return_the_one_gpu_records(fx, cv, tmp_path):
    from test_shard_convert import _run
    one = preprocess.preprocess_utterances(cv[0], fx_items(fx), max_batch=3)
    backend = "nccl" if torch.cuda.device_count() >= 2 else "gloo"
    paths = _run(_shard_worker, 2, str(tmp_path), backend=backend, timeout=600)
    assert all(isinstance(p, str) and p.endswith(".pt") for p in paths), paths
    for r, p in enumerate(paths):
        res = torch.load(p, weights_only=False)
        print(f"rank {r} over {res['backend']}")
        assert len(res["records"]) == len(one)
        for k, (a, b) in enumerate(zip(res["records"], one)):
            assert a["frames"] == b["frames"], (r, k)
            for key in ("wav24k", "soft", "spec"):
                assert torch.equal(a[key], b[key].cpu()), (r, k, key)
