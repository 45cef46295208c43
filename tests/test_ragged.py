"""Ragged utterance batches: per-utterance content lengths T_b <= T and prompt lengths S_b <= S in one denoiser run.

The contract: row b of a ragged run equals utterance b run alone (x_T[b, :, :T_b], content[:T_b], prompt[:S_b], no mask) and
its frames >= T_b are exactly 0.  Tolerance rtol 1e-3 / atol 1e-4 against the fp32 oracle; our own B = 1 runs are compared
at the same tolerance and the tests report whether they are bit-identical."""
import pytest
import torch

from ns2vc_b200 import api
from ns2vc_b200.arch import ns2vc_denoiser_config
from ns2vc_b200.synth import make_inputs
from oracle import unet_oracle

RTOL, ATOL = 1e-3, 1e-4


def close(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    err = (a - b).abs()
    viol = (err > ATOL + RTOL * b.abs()).float().mean().item()
    return viol == 0.0, f"max_abs={err.max().item():.3e} violations={viol:.3%}"


# ----------------------------------------------------------------------------------------------------------------- CPU
def _utterances(lengths, prompts, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn((5, t), generator=g), torch.randn((t, 3), generator=g), torch.randn((s, 4), generator=g))
            for t, s in zip(lengths, prompts)]


def test_batch_plan_pad_unpad_round_trip_is_exact():
    lengths, prompts = [150, 1000, 377, 377, 64, 999, 512], [40, 40, 12, 40, 1, 33, 40]
    items = _utterances(lengths, prompts)
    plan = api.batch_plan(lengths, 3)
    assert sorted(i for idx in plan for i in idx) == list(range(len(items)))
    assert all(len(idx) <= 3 for idx in plan)
    assert [lengths[i] for idx in plan for i in idx] == sorted(lengths, reverse=True)
    for idx in plan:
        x, c, p, tl, sl = api.pad_batch(items, idx)
        assert x.shape == (len(idx), 5, max(lengths[i] for i in idx)) and c.shape[:2] == (x.shape[2], len(idx))
        assert p.shape[:2] == (max(prompts[i] for i in idx), len(idx))
        for j, i in enumerate(idx):
            xt, ct, pt = items[i]
            assert int(tl[j]) == xt.shape[1] and int(sl[j]) == pt.shape[0]
            assert torch.equal(x[j, :, :tl[j]], xt) and torch.equal(c[:tl[j], j], ct) and torch.equal(p[:sl[j], j], pt)
            assert not x[j, :, tl[j]:].any() and not c[tl[j]:, j].any() and not p[sl[j]:, j].any()


def test_lengths_out_of_range_raise():
    from ns2vc_b200.fused import check_lengths
    assert check_lengths(torch.tensor([3, 1, 8]), 3, 8, "n") == [3, 1, 8]
    for bad in ([0, 4], [9, 4], [4]):
        with pytest.raises(ValueError):
            check_lengths(bad, 2, 8, "content_lengths")
    x, c, p = torch.zeros(2, 100, 8), torch.zeros(8, 2, 256), torch.zeros(5, 2, 256)
    for cl, pl in (([9, 8], None), ([0, 8], None), ([8, 8], [6, 5]), ([8, 8], [0, 5])):
        with pytest.raises(ValueError):
            api.sample_latents(None, x, c, p, None if pl is None else torch.tensor(pl), content_lengths=torch.tensor(cl))
    with pytest.raises(ValueError):
        api.batch_plan([3, 4], 0)


# ----------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def full():
    from test_gpu_parity import make_unet
    cfg = ns2vc_denoiser_config()
    m, sd = make_unet(cfg)
    return m, sd, cfg


def _session(m, content_BCT, prompt_BSC, **kw):
    from ns2vc_b200.fused import DenoiserSession
    return DenoiserSession(m, content_BCT.contiguous().cuda(), prompt_BSC.contiguous().cuda(), None, **kw)


def _forward(sess, x, t):
    out = torch.empty((x.shape[0], 100, x.shape[2]), device="cuda")
    sess.forward(x.contiguous().cuda(), t.cuda(), out)
    torch.cuda.synchronize()
    return out.cpu()


FWD_T, FWD_S = [1024, 777, 513, 64], [256, 200, 31, 256]     # odd lengths at every level (513 -> 257 -> 129 -> 65), one T_b = T


@pytest.mark.gpu
def test_ragged_forward_matches_each_utterance_alone(full):
    m, sd, cfg = full
    B, T, S = 4, 1024, 256
    inp = make_inputs(B, T, S, seed=21)
    x, content, prompt = inp["x"], inp["content"].permute(1, 2, 0), inp["prompt"].permute(1, 0, 2)
    t = torch.tensor([900.5, 450.25, 10.0, 0.5])
    out = _forward(_session(m, content, prompt, content_lengths=FWD_T, prompt_lengths=FWD_S), x, t)
    bad, bitwise = [], []
    for b, (Tb, Sb) in enumerate(zip(FWD_T, FWD_S)):
        assert not out[b, :, Tb:].any(), f"row {b}: padded output frames are not 0"
        xin = torch.cat([x[b:b + 1, :, :Tb], content[b:b + 1, :, :Tb]], 1)
        with torch.no_grad():
            ref = unet_oracle.unet_forward(sd, cfg, xin, t[b:b + 1], prompt[b:b + 1, :Sb], None)
        ok, msg = close(out[b:b + 1, :, :Tb], ref)
        if not ok:
            bad.append(f"row {b} (T_b={Tb}, S_b={Sb}) vs oracle: {msg}")
        own = _forward(_session(m, content[b:b + 1, :, :Tb], prompt[b:b + 1, :Sb]), x[b:b + 1, :, :Tb], t[b:b + 1])
        ok, msg = close(out[b:b + 1, :, :Tb], own)
        if not ok:
            bad.append(f"row {b} vs our B=1 forward: {msg}")
        bitwise.append(torch.equal(out[b:b + 1, :, :Tb], own))
    print(f"ragged rows bit-identical to our B=1 forward: {bitwise}")
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
def test_values_past_the_lengths_are_never_read(full):
    m, _, _ = full
    B, T, S = 4, 1024, 256
    inp = make_inputs(B, T, S, seed=22)
    x, content, prompt = inp["x"], inp["content"].permute(1, 2, 0).contiguous(), inp["prompt"].permute(1, 0, 2).contiguous()
    t = torch.tensor([700.0, 300.5, 50.0, 999.0])
    clean = _forward(_session(m, content, prompt, content_lengths=FWD_T, prompt_lengths=FWD_S), x, t)
    xg, cg, pg = x.clone(), content.clone(), prompt.clone()
    for b, (Tb, Sb) in enumerate(zip(FWD_T, FWD_S)):
        xg[b, :, Tb:] = float("nan")
        cg[b, :, Tb:] = 1e30
        pg[b, Sb:] = float("nan")
    dirty = _forward(_session(m, cg, pg, content_lengths=FWD_T, prompt_lengths=FWD_S), xg, t)
    assert torch.equal(clean, dirty), f"max diff {(clean - dirty).abs().nan_to_num(float('inf')).max().item():.3e}"


@pytest.mark.gpu
@pytest.mark.parametrize("T,S,rows", [
    (4189, 256, [(4189, 256), (4188, 256)]),       # padded table 2095 -> 4189 maps row 4187 to 2094; the 4188-frame row alone: 2093
    (4190, 1100, [(4190, 1100), (4189, 300)]),     # the reverse (2x table vs 2095 -> 4189); S > 1024: the fp32 attention kernel
])
def test_long_rows_upsample_with_their_own_nearest_rule(full, T, S, rows):
    """In fp32 the nearest-upsample index of (t_in, 2 t_in - 1) is not always i >> 1 (t_in >= 2095): each row must use the
    table of its own lengths, not the padded batch's."""
    m, _, _ = full
    B = len(rows)
    inp = make_inputs(B, T, S, seed=24)
    x, content, prompt = inp["x"], inp["content"].permute(1, 2, 0), inp["prompt"].permute(1, 0, 2)
    t = torch.tensor([600.5, 20.0])
    out = _forward(_session(m, content, prompt, content_lengths=[r[0] for r in rows], prompt_lengths=[r[1] for r in rows]), x, t)
    for b, (Tb, Sb) in enumerate(rows):
        assert not out[b, :, Tb:].any()
        own = _forward(_session(m, content[b:b + 1, :, :Tb], prompt[b:b + 1, :Sb]), x[b:b + 1, :, :Tb], t[b:b + 1])
        ok, msg = close(out[b:b + 1, :, :Tb], own)
        assert ok, f"T={T} row {b} (T_b={Tb}, S_b={Sb}) vs our B=1 forward: {msg}"


SMP_T, SMP_S = [300, 211, 97], [64, 40, 17]


def _sampler_inputs():
    inp = make_inputs(3, 300, 64, seed=23)
    return inp["x"], inp["content"].permute(1, 2, 0).contiguous(), inp["prompt"].permute(1, 0, 2).contiguous()


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["dpm", "unipc", "ddim"])
def test_ragged_samplers_match_each_utterance_alone(full, method):
    m, _, _ = full
    ns = api.default_schedule()
    ts = torch.linspace(ns.T, 1.0 / ns.total_N, 21)
    x, content, prompt = _sampler_inputs()
    noise = torch.randn((10, 3, 100, 300), generator=torch.Generator().manual_seed(5))

    def run(sess, xT, nz=None):
        xT = xT.contiguous().cuda()
        if method == "dpm":
            r = sess.sample_dpmpp_2m(xT, ns, ts)
        elif method == "unipc":
            r = sess.sample_unipc(xT, ns, ts)
        else:
            r = sess.sample_ddim(xT, 10, eta=0.5, noise=nz.cuda())
        torch.cuda.synchronize()
        return r.cpu()

    got = run(_session(m, content, prompt, content_lengths=SMP_T, prompt_lengths=SMP_S), x, noise)
    bad = []
    for b, (Tb, Sb) in enumerate(zip(SMP_T, SMP_S)):
        assert not got[b, :, Tb:].any(), f"row {b}: padded frames are not 0"
        alone = run(_session(m, content[b:b + 1, :, :Tb], prompt[b:b + 1, :Sb]), x[b:b + 1, :, :Tb], noise[:, b:b + 1, :, :Tb])
        ok, msg = close(got[b:b + 1, :, :Tb], alone)
        if not ok:
            bad.append(f"{method} row {b}: {msg}")
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
def test_ragged_graph_replay_and_padded_session_unchanged(full):
    m, _, _ = full
    ns = api.default_schedule()
    ts = torch.linspace(ns.T, 1.0 / ns.total_N, 11)
    x, content, prompt = _sampler_inputs()
    xc = x.cuda()
    padded = _session(m, content, prompt)
    p0 = padded.sample_dpmpp_2m(xc, ns, ts).cpu()
    rag = _session(m, content, prompt, content_lengths=SMP_T, prompt_lengths=SMP_S)
    runs = [rag.sample_dpmpp_2m(xc, ns, ts).cpu() for _ in range(4)]     # eager, eager, capture + replay, replay
    assert torch.equal(runs[0], runs[2]) and torch.equal(runs[0], runs[3]), "captured replay differs from the eager run"
    # the same graph serves new lengths: its replay equals an eager run of a fresh session at those lengths
    new_T, new_S = [150, 211, 300], [10, 64, 64]
    rag.set_cond(content.cuda(), prompt.cuda(), None, new_T, new_S)
    other = rag.sample_dpmpp_2m(xc, ns, ts).cpu()
    fresh = _session(m, content, prompt, content_lengths=new_T, prompt_lengths=new_S).sample_dpmpp_2m(xc, ns, ts).cpu()
    assert torch.equal(other, fresh), "the replay with new lengths differs from a fresh session at those lengths"
    assert not other[0, :, 150:].any() and not torch.equal(other[:, :, :97], runs[0][:, :, :97])
    p1 = padded.sample_dpmpp_2m(xc, ns, ts).cpu()
    assert torch.equal(p0, p1), "the padded run changed after a ragged run on the same module"


@pytest.mark.gpu
def test_sample_from_features_per_utterance(full):
    """per_utterance=True: the encoders run on the padded batch as the reference runs them, and each row of the sampling equals
    sample_latents on that row of the encoders' output alone."""
    from test_pre_model_gpu import FULL, inputs, make
    m, _, _ = full
    pre, _ = make(FULL, seed=1)
    c, refer, lengths, _ = inputs(3, 240, 64, 256, seed=12, dl=71)
    refer_lengths = torch.full((3,), 64, dtype=torch.int64)
    x = torch.randn((3, 100, 240), generator=torch.Generator().manual_seed(8))
    got = api.sample_from_features(pre, m, x, c, refer, lengths, refer_lengths, steps=8, per_utterance=True).cpu()
    from test_pre_model_gpu import data_of
    content, prompt = pre.infer(data_of(c, refer, lengths, refer_lengths))
    for b in range(3):
        Tb = int(lengths[b])
        assert not got[b, :, Tb:].any()
        alone = api.sample_latents(m, x[b:b + 1, :, :Tb], content[:Tb, b:b + 1], prompt[:, b:b + 1], None, steps=8).cpu()
        ok, msg = close(got[b:b + 1, :, :Tb], alone)
        assert ok, f"row {b} (T_b={Tb}): {msg}"


@pytest.mark.gpu
def test_sample_utterances_equals_each_utterance_alone(full):
    m, _, _ = full
    g = torch.Generator().manual_seed(7)
    items = [(torch.randn((100, t), generator=g), torch.randn((t, 256), generator=g), torch.randn((48, 256), generator=g))
             for t in (150, 333, 97, 260)]
    got = api.sample_utterances(m, items, steps=8, max_batch=3)
    for k, (xt, ct, pt) in enumerate(items):
        assert got[k].shape == xt.shape
        alone = api.sample_latents(m, xt[None], ct[:, None], pt[:, None], None, steps=8)[0]
        ok, msg = close(got[k], alone)
        assert ok, f"utterance {k}: {msg}"
