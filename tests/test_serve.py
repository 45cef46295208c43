"""Continuous batching (``serve.ConversionServer``) and its per-row sampler step kernels.

CPU: the argument errors (with ``None`` models, raised before anything touches a device) and the slot bookkeeping of
``serve.SlotTable``.  GPU, with the small chained models of ``test_convert.py``: the row step kernels bit for bit against the
scalar ones, each served request against that request converted alone (latent and audio), the default x_T draws, slot hygiene
(NaN in every buffer a request must not read, and another caller taking the shared workspace between ticks, leave every result
bit-identical) and a request with a NaN prompt failing alone."""
import ctypes as C

import pytest
import torch

from ns2vc_b200 import _lib, api, coefs, convert, serve
from test_convert import DURATIONS, PRE_CFG, SR, _close

STEPS = 8
SLOTS = 4
MAX_FRAMES = 400                     # the longest of DURATIONS is 375 frames
MAX_PROMPT = 80


# ----------------------------------------------------------------------------------------------------------------- CPU
def test_argument_errors():
    w, mel = torch.zeros(20000), torch.zeros(100, 30)
    for method in ("ddpm", "ddim", "euler"):
        with pytest.raises(ValueError):
            serve.ConversionServer(None, None, None, None, method=method)
    for kw in (dict(slots=0), dict(max_frames=0), dict(max_prompt_frames=0), dict(steps=0)):
        with pytest.raises(ValueError):
            serve.ConversionServer(None, None, None, None, **kw)
    srv = serve.ConversionServer(None, None, None, None, slots=2, max_frames=100, max_prompt_frames=40)
    with pytest.raises(ValueError, match="max_frames=100"):
        srv.submit(torch.zeros(int(1.5 * SR)), SR, mel)                        # 140 frames
    with pytest.raises(ValueError, match="max_prompt_frames=40"):
        srv.submit(w, SR, torch.zeros(100, 41))
    with pytest.raises(ValueError, match="mono"):
        srv.submit(torch.zeros(2, 20000), SR, mel)
    with pytest.raises(ValueError, match="too short"):
        srv.submit(torch.zeros(300), SR, mel)
    with pytest.raises(ValueError, match="x_T"):
        srv.submit(w, SR, mel, x_T=torch.zeros(1, 100, 3))
    with pytest.raises(ValueError, match="prompt"):
        srv.submit(w, SR, torch.zeros(80, 30))
    with pytest.raises(ValueError, match="sample rate"):
        srv.submit(w, 0, mel)
    assert srv.table.idle and srv.tick() == {} and srv.ticks == 0              # nothing was queued; no device touched
    T = convert.frame_plan(20000, SR)["T"]
    assert [srv.submit(w, SR, mel, x_T=torch.zeros(1, 100, T)) for _ in range(3)] == [0, 1, 2]
    assert list(srv.table.queue) == [0, 1, 2]
    assert api.ConversionServer is serve.ConversionServer


def test_slot_bookkeeping():
    g = torch.Generator().manual_seed(0)
    for slots, steps in ((1, 1), (3, 5), (4, 8)):
        tab = serve.SlotTable(slots, steps)
        admitted, retired, nxt = {}, {}, 0
        for tick in range(200):
            for _ in range(int(torch.poisson(torch.tensor(0.6 * slots / steps), generator=g))) if tick < 150 else ():
                tab.enqueue(nxt)
                nxt += 1
            free_before = tab.free_slots()
            new = tab.admit(tick)
            for s, t in new:
                admitted[t] = (s, tick)
                assert s in free_before
            assert not (tab.queue and tab.free_slots()), "a request waits while a slot is free (freed slots are reused at the next tick)"
            assert tab.occupied <= slots
            for s, t in tab.retire(tick):
                retired[t] = tick
        assert tab.idle and len(admitted) == len(retired) == nxt
        order = sorted(admitted, key=lambda t: (admitted[t][1], admitted[t][0]))
        assert order == sorted(admitted), "admission is not FIFO"
        for t, (s, a) in admitted.items():
            assert retired[t] == a + steps - 1, "a request must retire after exactly `steps` ticks"
        for t, (s, a) in admitted.items():     # no slot holds two requests at once
            assert not any(s2 == s and a2 < a <= retired[u] for u, (s2, a2) in admitted.items() if u != t)
    tab = serve.SlotTable(2, 3)
    for t in range(4):
        tab.enqueue(t)
    assert tab.admit(0) == [(0, 0), (1, 1)] and tab.admit(1) == [] and tab.retire(1) == []
    assert tab.retire(2) == [(0, 0), (1, 1)] and tab.admit(3) == [(0, 2), (1, 3)]


# ----------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def chain():
    from ns2vc_b200.arch import UNetConfig
    from ns2vc_b200.content import ContentVec
    from ns2vc_b200.pre_model import Pre_model
    from ns2vc_b200.synth import CONTENTVEC_SMALL, make_contentvec_state_dict, make_pre_state_dict, make_vocos_state_dict
    from ns2vc_b200.vocoder import Vocos
    from test_gpu_parity import make_unet
    cv = ContentVec.from_state_dict(make_contentvec_state_dict(0, "trained_like", **CONTENTVEC_SMALL),
                                    num_heads=CONTENTVEC_SMALL["num_heads"]).to("cuda")
    pre = Pre_model(PRE_CFG)
    pre.load_state_dict(make_pre_state_dict(PRE_CFG, 0))
    pre = pre.to("cuda").eval()
    ucfg = UNetConfig(in_channels=132, out_channels=100, block_out_channels=(32, 64, 64, 96), norm_num_groups=8, cross_attention_dim=32,
                      num_heads=8, addition_embed_type="text", addition_embed_type_num_heads=4, resnet_time_scale_shift="scale_shift")
    unet, _ = make_unet(ucfg)
    voc = Vocos.from_state_dict(make_vocos_state_dict(0, "trained_like", dim=128, intermediate_dim=384, num_layers=2)).to("cuda")
    g = torch.Generator().manual_seed(3)
    wavs = []
    for d in DURATIONS:
        n = int(d * SR)
        t = torch.arange(n) / SR
        wavs.append((0.3 * torch.sin(2 * torch.pi * (110 + 300 * torch.rand(1, generator=g)) * t) + 0.05 * torch.randn(n, generator=g)).float())
    prompt = (torch.randn((100, 70), generator=g) - 4.0).float()
    xs = [torch.randn((1, 100, convert.frame_plan(len(w), SR)["T"]), generator=g) for w in wavs]
    return (cv, pre, unet, voc), wavs, prompt, xs


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["dpm", "unipc"])
def test_row_steps_equal_the_scalar_steps_bit_for_bit(kind):
    L = _lib.lib()
    ns = api.default_schedule()
    ts = torch.linspace(ns.T, 1.0 / ns.total_N, STEPS + 1)
    steps = coefs.dpmpp_2m_table(ns, ts, True) if kind == "dpm" else coefs.unipc_bh2_table(ns, ts, "bh2")
    dev_coef, _ = coefs.c_table(steps, "cuda")
    ks = [0, 3, STEPS - 1, -1]                 # first step, a middle step, the lower-order final step, an empty row
    B, Cl, T = len(ks), 100, 97
    n = Cl * T
    g = torch.Generator(device="cuda").manual_seed(5)
    ins = {name: torch.randn((B, Cl, T), device="cuda", generator=g) for name in
           (("x", "o", "mp") if kind == "dpm" else ("xp", "xe", "o", "m0", "m1"))}
    outs_names = ("mc", "xn") if kind == "dpm" else ("mt", "xt", "xq")

    def run_rows(nan):
        k = torch.tensor(ks, dtype=torch.int32, device="cuda")
        outs = {name: torch.full((B, Cl, T), 7.0, device="cuda") for name in outs_names}
        if kind == "dpm":
            _lib.check(L.ns2vc_dpm_step_rows(ins["x"].data_ptr(), ins["o"].data_ptr(), ins["mp"].data_ptr(), dev_coef.data_ptr(), k.data_ptr(),
                                             outs["mc"].data_ptr(), outs["xn"].data_ptr(), n, B, nan.data_ptr(), None))
        else:
            _lib.check(L.ns2vc_unipc_step_rows(ins["xp"].data_ptr(), ins["xe"].data_ptr(), ins["o"].data_ptr(), ins["m0"].data_ptr(),
                                               ins["m1"].data_ptr(), dev_coef.data_ptr(), k.data_ptr(), outs["mt"].data_ptr(),
                                               outs["xt"].data_ptr(), outs["xq"].data_ptr(), n, B, nan.data_ptr(), None))
        torch.cuda.synchronize()
        return k, outs

    nan = torch.zeros(B, dtype=torch.int32, device="cuda")
    k, outs = run_rows(nan)
    assert k.tolist() == [v + 1 if v >= 0 else -1 for v in ks], "occupied rows advance by one step, empty rows stay empty"
    assert nan.tolist() == [0] * B
    for b, kb in enumerate(ks):
        if kb < 0:
            for name in outs_names:
                assert torch.count_nonzero(outs[name][b]) == 0, f"empty row: {name} is not exactly 0"
            continue
        ref = {name: torch.full((Cl, T), 7.0, device="cuda") for name in outs_names}
        c = coefs.c_struct(steps[kb])
        if kind == "dpm":
            _lib.check(L.ns2vc_dpm_step(ins["x"][b].data_ptr(), ins["o"][b].data_ptr(), ins["mp"][b].data_ptr(), C.byref(c),
                                        ref["mc"].data_ptr(), ref["xn"].data_ptr(), n, None, None))
        else:
            _lib.check(L.ns2vc_unipc_step(ins["xp"][b].data_ptr(), ins["xe"][b].data_ptr(), ins["o"][b].data_ptr(), ins["m0"][b].data_ptr(),
                                          ins["m1"][b].data_ptr(), C.byref(c), ref["mt"].data_ptr(), ref["xt"].data_ptr(), ref["xq"].data_ptr(),
                                          n, None, None))
            if c.corr_order == 0:                 # the scalar step leaves x_t alone there; the row step writes x_eval
                ref["xt"] = ins["xe"][b]
        torch.cuda.synchronize()
        for name in outs_names:
            assert torch.equal(outs[name][b], ref[name]), f"row {b} (step {kb}): {name} differs from the scalar step"
    # a NaN in one occupied row's input raises that row's flag only; one in the empty row raises nothing
    xin = ins["x" if kind == "dpm" else "xe"]
    xin[1, 5, 7] = float("nan")
    xin[3, 0, 0] = float("nan")
    nan.zero_()
    run_rows(nan)
    assert nan.tolist() == [0, 1, 0, 0]


def _script(models, wavs, prompt, xs, method, between=None, prompts=None):
    """Serves the six requests on a script: three before tick 0, one before tick 2, two more after the first retirement.
    ``between(srv)`` runs after every tick.  Returns ({request: audio or exception}, {request: latent}, the slot of each)."""
    srv = serve.ConversionServer(*models, slots=SLOTS, max_frames=MAX_FRAMES, max_prompt_frames=MAX_PROMPT, method=method, steps=STEPS)
    prompts = prompts or [prompt] * len(wavs)
    req, res, lat, slot_of = {}, {}, {}, {}

    def submit(i):
        req[srv.submit(wavs[i], SR, prompts[i], x_T=xs[i])] = i

    for i in (0, 1, 2):
        submit(i)
    while len(res) < len(wavs):
        if srv.ticks == 2:
            submit(3)
        t = srv.ticks
        done = srv.tick()
        assert srv.table.occupied <= SLOTS
        for s, tk in enumerate(srv.table.ticket):
            if tk is not None:
                slot_of.setdefault(req[tk], (s, srv.table.last[s] - STEPS + 1))
        for tk, v in done.items():
            res[req[tk]] = v
            assert t == slot_of[req[tk]][1] + STEPS - 1, "a request must retire after exactly `steps` ticks"
        lat.update({req[tk]: v for tk, v in srv.last_latents.items()})
        if done and 4 not in req.values():
            submit(4)
            submit(5)
        if between is not None:
            between(srv)
    assert srv.table.idle
    return res, lat, slot_of


_ALONE = {}


def _alone(models, wavs, prompt, xs, method, i):
    key = (method, i)
    if key not in _ALONE:
        r = convert.convert_batch(*models, [wavs[i]], SR, [prompt], [xs[i]], method, STEPS)
        _ALONE[key] = (r["latent"][0], r["audio"][0])
    return _ALONE[key]


def _check_parity(models, wavs, prompt, xs, method, res, lat, skip=()):
    bad = []
    for i in range(len(wavs)):
        if i in skip:
            continue
        la, aa = _alone(models, wavs, prompt, xs, method, i)
        tag = f"{method} request {i} ({DURATIONS[i]} s, T_b={la.shape[1]})"
        ok, mx = _close(lat[i], la)
        a, b = lat[i].double().cpu(), la.double().cpu()
        et = ((a - b).abs() / (1e-4 + 1e-3 * b.abs())).max().item()
        ga, gb = res[i].double().cpu(), aa.double().cpu()
        rel = ((ga - gb).norm() / gb.norm()).item()
        print(f"{tag}: latent err/tol {et:.3f} (max|diff| {mx:.2e}), audio ||diff||/||alone|| {rel:.2e} (tol 1e-4)")
        if not ok:
            bad.append(f"{tag} latent: max|diff| {mx:.3e}")
        if rel > 1e-4:
            bad.append(f"{tag} audio: ||diff||/||alone|| {rel:.2e}")
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["unipc", "dpmsolver"])
def test_each_request_equals_its_own_conversion(chain, method):
    models, wavs, prompt, xs = chain
    res, lat, slot_of = _script(models, wavs, prompt, xs, method)
    assert slot_of == {0: (0, 0), 1: (1, 0), 2: (2, 0), 3: (3, 2), 4: (0, STEPS), 5: (1, STEPS)}, slot_of
    _check_parity(models, wavs, prompt, xs, method, res, lat)


@pytest.mark.gpu
def test_default_x_T_draws_match_convert_utterances(chain):
    models, wavs, prompt, _ = chain
    torch.manual_seed(1234)
    srv = serve.ConversionServer(*models, slots=SLOTS, max_frames=MAX_FRAMES, max_prompt_frames=MAX_PROMPT, steps=STEPS)
    tickets = [srv.submit(w, SR, prompt) for w in wavs]
    got = srv.drain()
    torch.manual_seed(1234)
    want = convert.convert_utterances(*models, wavs, SR, prompt, steps=STEPS, max_batch=SLOTS)
    bad = []
    for i, tk in enumerate(tickets):
        a, b = got[tk].double().cpu(), want[i].double().cpu()
        rel = ((a - b).norm() / b.norm()).item()
        print(f"request {i}: audio ||diff||/||convert_utterances|| {rel:.2e} (tol 1e-4)")
        if a.shape != b.shape or rel > 1e-4:
            bad.append(f"request {i}: {rel:.2e}")
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["unipc", "dpmsolver"])
def test_slot_hygiene_bit_for_bit(chain, method):
    models, wavs, prompt, xs = chain
    clean, clean_lat, _ = _script(models, wavs, prompt, xs, method)
    nan = float("nan")

    def poison(srv):
        """NaN into every buffer of a free slot, and into the conditioning inputs of every occupied slot past its lengths."""
        sess = srv._sess
        for s in range(srv.B):
            if srv.table.ticket[s] is None:
                sess.content[s].fill_(nan)
                sess.prompt[s].fill_(nan)
                for b in srv._buf.values():
                    b[s].fill_(nan)
            else:
                sess.content[s, :, srv._clen[s]:].fill_(nan)
                sess.prompt[s, srv._plen[s]:].fill_(nan)

    dirty, dirty_lat, _ = _script(models, wavs, prompt, xs, method, between=poison)
    for i in range(len(wavs)):
        assert torch.equal(dirty_lat[i], clean_lat[i]) and torch.equal(dirty[i], clean[i]), f"request {i}: NaN in unread buffers changed it"

    def interleave(srv):
        if srv.ticks == 5:                 # another caller takes the module's shared workspace between ticks 4 and 5
            convert.convert_utterances(*models, [wavs[1], wavs[4]], SR, prompt, method=method, steps=4, x_T=[xs[1], xs[4]])

    inter, inter_lat, _ = _script(models, wavs, prompt, xs, method, between=interleave)
    for i in range(len(wavs)):
        assert torch.equal(inter_lat[i], clean_lat[i]) and torch.equal(inter[i], clean[i]), f"request {i}: the interleaved call changed it"


@pytest.mark.gpu
def test_a_nan_prompt_fails_only_its_own_request(chain):
    models, wavs, prompt, xs = chain
    bad_prompt = prompt.clone()
    bad_prompt[7, 11] = float("nan")
    prompts = [prompt] * len(wavs)
    prompts[2] = bad_prompt
    res, lat, _ = _script(models, wavs, prompt, xs, "unipc", prompts=prompts)
    assert isinstance(res[2], AssertionError) and "model.py:404" in str(res[2])
    assert 2 not in lat
    _check_parity(models, wavs, prompt, xs, "unipc", res, lat, skip=(2,))


@pytest.mark.gpu
def test_a_nan_voice_sample_fails_only_its_own_request(chain):
    """One NaN sample in a voice recording reaches its prompt mel (torch.clip keeps NaN) and so fails that request with the
    reference's AssertionError, as a NaN prompt does; the requests with the clean voice are bit-identical to a run without it."""
    models, wavs, _, xs = chain
    g = torch.Generator().manual_seed(11)
    voice = (0.2 * torch.randn(11000, generator=g)).float()                   # 16 kHz: 16500 samples, 65 frames at 24 kHz
    bad_voice = voice.clone()
    bad_voice[5000] = float("nan")
    clean, bad = convert.voice_mels([(voice, 16000), (bad_voice, 16000)], torch.device("cuda"))
    hit = bad.isnan().any(0)
    assert bad.isnan()[:, hit].all() and 0 < int(hit.sum()) < 8 and torch.equal(bad[:, ~hit], clean[:, ~hit])
    prompts = [clean.cpu()] * len(wavs)
    ref, ref_lat, _ = _script(models, wavs, clean.cpu(), xs, "unipc", prompts=prompts)
    prompts[2] = bad.cpu()
    res, lat, _ = _script(models, wavs, clean.cpu(), xs, "unipc", prompts=prompts)
    assert isinstance(res[2], AssertionError) and "model.py:404" in str(res[2])
    assert 2 not in lat
    for i in range(len(wavs)):
        if i != 2:
            assert torch.equal(lat[i], ref_lat[i]) and torch.equal(res[i], ref[i]), f"request {i} changed"
