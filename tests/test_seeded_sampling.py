"""Seeded DDPM and DDIM on the fused device loop: each row's step noise drawn in the step kernel from its own seed.

GPU, on a ragged batch of rows T_b = 37, 64, 128, 250: the seeded run equals the injected-noise path fed with ``noise.normal_rows``
bit for bit (which ties it to the fixtures test_ddpm_ddim.py pins against the reference), its captured replay equals the eager
run bit for bit, each row equals that utterance sampled alone (B = 1, unpadded) with its seed, and ``sample_utterances`` with
seeds equals ``sample_latents`` on each utterance alone.  A NaN in x_T raises the reference's AssertionError."""
import pytest
import torch

from conftest import tiny_config
from ns2vc_b200 import api, coefs, noise
from ns2vc_b200.synth import make_inputs
from test_ddpm_ddim import make_unet

LENGTHS = [37, 64, 128, 250]
PROMPTS = [11, 5, 11, 8]
SEEDS = [1, 2, 1 << 40, (1 << 63) - 1]
CASES = [("ddpm", 20, 0.0), ("ddim", 10, 0.0), ("ddim", 10, 0.5), ("ddim", 10, 1.0)]
DDPM_TS = list(range(999, 0, -53)) + [0]                     # a 20-step timesteps list ending at t = 0 (no noise there)


@pytest.fixture(scope="module")
def tiny():
    m, _ = make_unet(tiny_config())
    inp = make_inputs(len(LENGTHS), max(LENGTHS), max(PROMPTS), latent_ch=20, content_ch=16, seed=31)
    x = noise.x_T(SEEDS, 20, LENGTHS)
    return m, x, inp["content"].cuda(), inp["prompt"].cuda()


def _session(m, content_TBC, prompt_SBC, lengths, prompts):
    from ns2vc_b200.fused import get_session
    return get_session(m, content_TBC.permute(1, 2, 0).contiguous(), prompt_SBC.permute(1, 0, 2).contiguous(), None,
                       content_lengths=lengths, prompt_lengths=prompts)


def _run(sess, method, S, eta, x, **kw):
    if method == "ddpm":
        return sess.sample_ddpm(x, DDPM_TS if S == 20 else None, **kw)
    return sess.sample_ddim(x, S, eta=eta, **kw)


def _n_steps(method, S):
    return len(DDPM_TS) if (method, S) == ("ddpm", 20) else (1000 if method == "ddpm" else S)


def _close(a, b):
    err = (a.double() - b.double()).abs()
    return bool((err <= 1e-4 + 1e-3 * b.double().abs()).all()), err.max().item()


@pytest.mark.gpu
def test_x_T_is_the_reserved_step():
    x = noise.x_T([5, 6], 20, [37, 64])
    assert torch.equal(x, noise.normal_rows([5, 6], 20, [37, 64], step=noise.XT_STEP))
    assert torch.equal(x[0, :, :37], noise.x_T([5], 20, [37])[0]) and not x[0, :, 37:].any()


@pytest.mark.gpu
@pytest.mark.parametrize("method,S,eta", CASES + [("ddpm", 1000, 0.0)])
def test_seeded_rows_equal_injected_noise_replay_and_each_row_alone(tiny, monkeypatch, method, S, eta):
    m, x, content, prompt = tiny
    sess = _session(m, content, prompt, LENGTHS, PROMPTS)
    N, T = _n_steps(method, S), max(LENGTHS)
    monkeypatch.setenv("NS2VC_GRAPH", "0")
    eager = _run(sess, method, S, eta, x, seeds=SEEDS)
    nz = torch.stack([noise.normal_rows(SEEDS, 20, LENGTHS, step=k) for k in range(N)])
    injected = _run(sess, method, S, eta, x, noise=nz)
    del nz
    assert torch.equal(eager, injected), f"seeded run differs from the injected normal_rows, max {(eager - injected).abs().max():.3e}"
    monkeypatch.delenv("NS2VC_GRAPH")
    for i in range(4):                                       # eager, eager, capture + replay, replay
        got = _run(sess, method, S, eta, x, seeds=SEEDS)
        assert torch.equal(got, eager), f"run {i}: the captured replay differs from the eager run"
    ent = sess._chains[(method, tuple(DDPM_TS) if S == 20 else tuple(range(999, -1, -1)))] if method == "ddpm" \
        else sess._chains[("ddim", S, eta)]
    assert ent["graphs"], "the seeded chunks were not captured"
    assert sess._chunk["table"].numel() == int(sess.L.ns2vc_unet_time_table_floats(sess.h, sess.CHUNK * sess.B))
    assert torch.isfinite(eager).all()
    bitwise = []
    for b, (Tb, Sb) in enumerate(zip(LENGTHS, PROMPTS)):
        assert not eager[b, :, Tb:].any()
        alone_sess = _session(m, content[:Tb, b:b + 1], prompt[:Sb, b:b + 1], [Tb], [Sb])
        alone = _run(alone_sess, method, S, eta, x[b:b + 1, :, :Tb].contiguous(), seeds=[SEEDS[b]])
        ok, mx = _close(eager[b, :, :Tb], alone[0])
        assert ok, f"row {b} (T_b={Tb}): max|diff| {mx:.3e}"
        bitwise.append(torch.equal(eager[b, :, :Tb], alone[0]))
    print(f"[{method} {N} steps eta={eta}] rows bit-identical to their B = 1 runs: {bitwise}")
    assert all(bitwise), f"rows not bit-identical to their B = 1 runs: {bitwise}"


@pytest.mark.gpu
def test_sample_utterances_with_seeds_equals_each_utterance_alone(tiny):
    m, x, content, prompt = tiny
    items = [(x[b, :, :Tb].cpu(), content[:Tb, b].cpu(), prompt[:Sb, b].cpu()) for b, (Tb, Sb) in enumerate(zip(LENGTHS, PROMPTS))]
    for method, steps in (("ddim", 10), ("ddpm", None)):
        got = api.sample_utterances(m, items, steps=steps, method=method, max_batch=3, eta=0.5 if method == "ddim" else 0.0,
                                    noise_seeds=SEEDS)
        for k, (xt, ct, pt) in enumerate(items):
            alone = api.sample_latents(m, xt[None], ct[:, None], pt[:, None], None, steps=steps, method=method,
                                       eta=0.5 if method == "ddim" else 0.0, noise_seeds=[SEEDS[k]],
                                       content_lengths=torch.tensor([xt.shape[1]]))[0]
            assert torch.equal(got[k], alone), f"{method} utterance {k}"


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["ddpm", "ddim"])
def test_nan_in_x_T_raises_on_the_seeded_path(tiny, method):
    m, x, content, prompt = tiny
    sess = _session(m, content, prompt, LENGTHS, PROMPTS)
    run = (lambda v: sess.sample_ddpm(v, range(59, -1, -1), seeds=SEEDS)) if method == "ddpm" \
        else (lambda v: sess.sample_ddim(v, 10, seeds=SEEDS))
    assert torch.isfinite(run(x)).all()
    bad = x.clone()
    bad[1, 3, 5] = float("nan")
    for _ in range(4):                                       # eager, eager, capture, replay
        with pytest.raises(AssertionError):
            run(bad)
    assert torch.isfinite(run(x)).all()
    with pytest.raises(ValueError):
        sess.sample_ddim(x, 10, seeds=SEEDS, noise=torch.zeros(10, 4, 20, max(LENGTHS), device="cuda"))
    for bad_seeds in (SEEDS[:3], [1, 2, 3, -1], [1, 2, 3, 1 << 63]):
        with pytest.raises(ValueError):
            sess.sample_ddpm(x, range(9, -1, -1), seeds=bad_seeds)
    with pytest.raises(ValueError):
        sess.sample_ddim(x, 10, eta=1.5, seeds=SEEDS)


@pytest.mark.gpu
def test_seeded_runs_are_counted_apart_from_default_runs(tiny):
    """After two default runs of a schedule, the first seeded runs of it are still eager: each path captures on its own third run."""
    m, x, content, prompt = tiny
    sess = _session(m, content, prompt, LENGTHS, PROMPTS)
    for _ in range(2):
        sess.sample_ddim(x, 6)
    ent = sess._chains[("ddim", 6, 0.0)]
    first = sess.sample_ddim(x, 6, seeds=SEEDS)
    assert not ent["graphs"], "the first seeded run was captured"
    for _ in range(3):
        assert torch.equal(sess.sample_ddim(x, 6, seeds=SEEDS), first)
    assert ent["graphs"] and ent["runs"] == 2 and ent["seeded_runs"] == 4
