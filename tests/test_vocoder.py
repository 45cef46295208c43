"""Vocoder (`Vocos.decode`, vocos-mel-24khz configuration) on the GPU against the functional oracle ``oracle/vocos_oracle.py``.

The ``vocos`` package is absent, so the oracle is a restatement from the published architecture; its ISTFT is pinned here
independently of its authorship by a round trip through ``torch.stft``.

GPU contract, per stage (ref = the oracle's fp64 output of that stage on the GPU's OWN input for it, taken from the engine's
taps; e32 = max |fp32 - fp64| of the same stage on the same input):
    |gpu - ref| <= max(1e-3 |ref| + 1e-4 rms(ref), 2 e32)   elementwise
The stages are backbone.norm (embed + LayerNorm from the mel), each ConvNeXt block, final_layer_norm, head.out and the head's
ISTFT (the audio).  A ragged row is judged on its own slice: the oracle decodes it alone.  The whole chain is also compared
end to end with the fp64 oracle, normwise.  The oracle runs on the GPU with TF32 off (its fp64 path is the truth; its fp32
path only sizes e32).
"""
import types

import pytest
import torch
import torch.nn.functional as F

from ns2vc_b200 import api
from ns2vc_b200.synth import VOCOS_REGIMES, make_vocos_state_dict
from ns2vc_b200.vocoder import Vocos, vocos_param_shapes
from oracle import vocos_oracle as vo

RTOL, ATOL_RMS = 1e-3, 1e-4
HOP, NFFT = 256, 1024
SMALL = dict(input_channels=100, dim=128, intermediate_dim=384, num_layers=2, n_fft=NFFT)


# ----------------------------------------------------------------------------------------------------------------- CPU
def round_trip_spectrum(T, B=2, dtype=torch.float64, seed=0):
    """y [B, T * 256] and its STFT (zero-padded by 384 per side, no centring) as head output [B, T, 1026]: log|S| | angle S."""
    g = torch.Generator().manual_seed(seed)
    y = (0.1 * torch.randn((B, T * HOP), generator=g, dtype=torch.float64)).to(dtype)
    win = torch.hann_window(NFFT, dtype=dtype)
    S = torch.stft(F.pad(y, (384, 384)), NFFT, HOP, window=win, center=False, return_complex=True)
    assert S.shape[-1] == T and S.abs().max() < 100
    return y, torch.cat([S.abs().log(), S.angle()], 1).transpose(1, 2).contiguous(), win


@pytest.mark.parametrize("T", [1, 2, 7, 300])
def test_oracle_istft_round_trip(T):
    for dtype, bound in ((torch.float64, 1e-12), (torch.float32, 1e-5)):
        y, h, win = round_trip_spectrum(T, dtype=dtype)
        got = vo.head_istft(h, win, HOP)
        assert got.shape == y.shape
        rel = ((got - y).abs().max() / y.pow(2).mean().sqrt()).item()
        assert rel <= bound, (dtype, rel)


def test_oracle_precisions_agree_and_lengths_decode_rows_alone():
    sd = make_vocos_state_dict(0, "trained_like", **SMALL)
    mel = torch.randn((3, 100, 40), generator=torch.Generator().manual_seed(1))
    a64, a32 = vo.decode(sd, mel, HOP), vo.decode(sd, mel, HOP, dtype=torch.float32)
    assert ((a32.double() - a64).abs().max() / a64.pow(2).mean().sqrt()).item() < 1e-4
    lens = [40, 17, 1]
    rag = vo.decode(sd, mel, HOP, lengths=lens)
    for b, L in enumerate(lens):
        assert torch.equal(rag[b, :L * HOP], vo.decode(sd, mel[b:b + 1, :, :L], HOP)[0])
        assert not rag[b, L * HOP:].any()


def test_registry_matches_state_dict_order():
    import ctypes as C
    from ns2vc_b200 import _lib
    m = Vocos()
    L = _lib.lib()
    h = C.c_void_p()
    _lib.check(L.ns2vc_voc_create(C.byref(m._c_cfg()), C.byref(h)))
    try:
        got = []
        for i in range(L.ns2vc_voc_num_weights(h)):
            name, shp, nd = C.c_char_p(), (C.c_int64 * 4)(), C.c_int()
            _lib.check(L.ns2vc_voc_weight_info(h, i, C.byref(name), shp, C.byref(nd)))
            got.append((name.value.decode(), tuple(shp[k] for k in range(nd.value))))
    finally:
        L.ns2vc_voc_destroy(h)
    assert got == [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    assert got == list(vocos_param_shapes().items())
    for bad in (dict(n_fft=1000, hop_length=250), dict(dim=100), dict(intermediate_dim=100)):
        cfg = _lib.VocCfg(**{**dict(input_channels=100, dim=512, intermediate_dim=1536, num_layers=8, n_fft=1024, hop_length=256), **bad})
        assert L.ns2vc_voc_create(C.byref(cfg), C.byref(h)) != 0


def _stub(sd, padding="same"):
    full = {"feature_extractor.mel_spec.spectrogram.window": torch.hann_window(NFFT),
            "feature_extractor.mel_spec.mel_scale.fb": torch.zeros(513, 100), **sd}
    return types.SimpleNamespace(state_dict=lambda: dict(full),
                                 head=types.SimpleNamespace(istft=types.SimpleNamespace(hop_length=HOP, padding=padding)))


def test_from_vocos_loads_and_rejects_loudly():
    sd = make_vocos_state_dict(3, "trained_like", **SMALL)
    m = Vocos.from_vocos(_stub(sd))
    assert m.cfg == dict(SMALL, hop_length=HOP)
    assert list(m.state_dict()) == list(sd) and all(torch.equal(m.state_dict()[k], v) for k, v in sd.items())
    assert m.to("cpu") is m
    cases = {
        "backbone.convnext.1.pwconv2.bias": lambda d: d.pop("backbone.convnext.1.pwconv2.bias"),
        "backbone.extra.weight": lambda d: d.__setitem__("backbone.extra.weight", torch.zeros(3)),
        "backbone.norm.scale.weight": lambda d: d.__setitem__("backbone.norm.scale.weight", torch.zeros(4, 128)),
        "backbone.convnext.1.pwconv1.weight": lambda d: d.__setitem__("backbone.convnext.1.pwconv1.weight", torch.zeros(384, 127)),
    }
    for key, edit in cases.items():
        d = dict(sd)
        edit(d)
        with pytest.raises(ValueError, match=key.replace(".", r"\.")):
            Vocos.from_vocos(_stub(d))
    with pytest.raises(ValueError, match="padding"):
        Vocos.from_vocos(_stub(sd, padding="center"))
    with torch.no_grad(), pytest.raises(RuntimeError, match="no CPU path"):
        m.decode(torch.zeros(1, 100, 4))
    with pytest.raises(ValueError):
        api.decode_utterances(m, [torch.zeros(80, 5)])


# ----------------------------------------------------------------------------------------------------------------- GPU
_models = {}


def model(regime, small=False):
    key = (regime, small)
    if key not in _models:
        sd = make_vocos_state_dict(0, regime, **(SMALL if small else {}))
        _models[key] = (Vocos.from_state_dict(sd).cuda().eval(), {k: v.cuda() for k, v in sd.items()})
    return _models[key]


def ratio(got, ref64, ref32):
    """worst elementwise err / tol of the module docstring's rule"""
    got, ref = got.double(), ref64.double()
    e32 = (ref32.double() - ref).abs().max()
    tol = torch.clamp(RTOL * ref.abs() + ATOL_RMS * ref.pow(2).mean().sqrt(), min=2 * e32.item())
    return ((got - ref).abs() / tol).max().item()


def stage_ratios(sd, taps, mel, lengths):
    """{stage: worst err/tol over the rows}, each row's stage re-run by the oracle on the GPU's input for it, on the row's slice"""
    stages = [k for k in taps if k != "audio"]
    worst = {}
    for b, L in enumerate(lengths):
        def sl(name):
            return taps[name][b:b + 1, :L]
        for s, name in enumerate(stages):
            if name == "backbone.norm":
                fn, inp = (lambda x: vo.embed_norm(sd, x)), mel[b:b + 1, :, :L]
            elif name.startswith("backbone.convnext."):
                i = int(name.rsplit(".", 1)[1])
                fn, inp = (lambda x, i=i: vo.convnext_block(sd, i, x)), sl(stages[s - 1])
            elif name == "backbone.final_layer_norm":
                fn, inp = (lambda x: vo.final_norm(sd, x)), sl(stages[s - 1])
            else:
                fn, inp = (lambda x: vo.head_linear(sd, x)), sl("backbone.final_layer_norm")
            r = ratio(sl(name), fn(inp.double()), fn(inp.float()))
            worst[name] = max(worst.get(name, 0.0), r)
        h = sl("head.out")
        win = sd["head.istft.window"].cuda()
        r = ratio(taps["audio"][b:b + 1, :L * HOP], vo.head_istft(h.double(), win, HOP), vo.head_istft(h.float(), win, HOP))
        worst["audio"] = max(worst.get("audio", 0.0), r)
        assert not taps["audio"][b, L * HOP:].any(), f"row {b}: samples past its length are not 0"
    return worst


@pytest.fixture(autouse=False)
def no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def mel_of(B, T, seed):
    return torch.randn((B, 100, T), generator=torch.Generator().manual_seed(seed)).cuda()


def run_case(regime, B, T, lengths=None, seed=0):
    m, sd = model(regime)
    mel = mel_of(B, T, seed)
    lens = lengths or [T] * B
    with torch.no_grad():
        taps = m.taps(mel, None if lengths is None else torch.tensor(lengths))
        worst = stage_ratios(sd, taps, mel, lens)
        ref = vo.decode(sd, mel, HOP, lengths=lens)
    e2e = ((taps["audio"].double() - ref).norm() / ref.norm()).item()
    print(f"\n{regime} B={B} T={T}: worst err/tol per stage {max(worst.values()):.3f} "
          f"({max(worst, key=worst.get)}; audio {worst['audio']:.3f}), end-to-end ||err||/||ref|| {e2e:.2e}, launches {m.launch_count()}")
    bad = {k: round(v, 3) for k, v in worst.items() if v > 1.0}
    assert not bad, bad
    assert e2e <= 1e-3
    return m, mel, taps


@pytest.mark.gpu
@pytest.mark.parametrize("regime", VOCOS_REGIMES)
def test_regimes(regime, no_tf32):
    run_case(regime, 4, 1024)


@pytest.mark.gpu
@pytest.mark.parametrize("B,T", [(1, 1), (1, 2), (1, 3), (1, 64), (1, 1023), (8, 1024), (2, 4096)])
def test_shapes(B, T, no_tf32):
    run_case("init", B, T)


@pytest.mark.gpu
def test_ragged_rows_decode_alone(no_tf32):
    lengths = [1, 2, 7, 300, 1000, 1024]
    m, mel, taps = run_case("trained_like", 6, 1024, lengths, seed=5)
    with torch.no_grad():
        audio = taps["audio"]
        poisoned = mel.clone()
        for b, L in enumerate(lengths):
            poisoned[b, :, L:] = float("nan") if b % 2 else 1e30
        assert torch.equal(m.decode(poisoned, torch.tensor(lengths)), audio)
        same = [torch.equal(m.decode(mel[b:b + 1, :, :L])[0], audio[b, :L * HOP]) for b, L in enumerate(lengths)]
    print(f"rows bit-identical to their B = 1 decode: {same}")


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 2, 7, 300])
def test_istft_stage_alone(T, no_tf32):
    m, sd = model("init", small=True)
    y, h, _ = round_trip_spectrum(T, B=2, dtype=torch.float64, seed=T)
    h32 = h.float()
    win = sd["head.istft.window"].cpu()
    lens = [T, max(1, T // 2)]
    with torch.no_grad():
        got = m.istft(h32.cuda(), torch.tensor(lens)).cpu()
    for b, L in enumerate(lens):
        hb = h32[b:b + 1, :L]
        r = ratio(got[b:b + 1, :L * HOP], vo.head_istft(hb.double(), win, HOP), vo.head_istft(hb, win, HOP))
        assert r <= 1.0, (b, r)
        assert not got[b, L * HOP:].any()
    assert ((got[0].double() - y[0]).abs().max() / y[0].pow(2).mean().sqrt()).item() < 1e-5


@pytest.mark.gpu
def test_graph_replay_with_new_lengths():
    m, _ = model("trained_like")
    mel = mel_of(3, 512, 7)
    lens = torch.tensor([512, 300, 1], device="cuda")
    with torch.no_grad():
        m.decode(mel, lens)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = m.decode(mel, lens)
        for new in ([512, 300, 1], [17, 512, 256]):
            lens.copy_(torch.tensor(new))
            g.replay()
            torch.cuda.synchronize()
            assert torch.equal(out, m.decode(mel, torch.tensor(new))), new


@pytest.mark.gpu
def test_decode_utterances_in_input_order():
    m, _ = model("trained_like")
    g = torch.Generator().manual_seed(0)
    lengths = torch.randint(150, 1001, (16,), generator=g).tolist()
    latents = [torch.randn((100, t), generator=g).cuda() for t in lengths]
    with torch.no_grad():
        out = api.decode_utterances(m, latents, max_batch=8)
        same = 0
        for x, a in zip(latents, out):
            alone = m.decode(x[None])[0]
            assert a.shape == alone.shape == (x.shape[1] * HOP,)
            assert ratio(a, alone, alone) <= 1.0
            same += int(torch.equal(a, alone))
    print(f"decode_utterances: {same}/16 bit-identical to their B = 1 decode")
