"""Content encoder (ContentVec / fairseq HubertModel units, ``utils.get_hubert_content``) on the GPU against the functional
oracle ``oracle/content_oracle.py``.

fairseq and the ContentVec checkpoint are absent.  The oracle is pinned on the CPU against transformers' ``HubertModel`` (a port
of fairseq's) when transformers is importable; the parameter names are pinned only by the strict loader.

GPU contract, per stage (ref = the oracle's fp64 output of that stage on the GPU's OWN input for it, taken from the engine's
taps, for each row on its own frames; e32 = max |fp32 - fp64| of the same stage on the same input):
    |gpu - ref| <= max(1e-3 |ref| + 1e-4 rms(ref), 2 e32)   elementwise
The stages are the seven convs, layer_norm, post_extract_proj, the positional conv with its residual, encoder.layer_norm, each
layer's two post-LN blocks, and final_proj.  The oracle runs on the GPU with TF32 off.
"""
import ctypes as C
import math
import types

import pytest
import torch

from ns2vc_b200 import api
from ns2vc_b200.content import CONTENTVEC, ContentVec, contentvec_param_shapes, get_hubert_content, num_frames
from ns2vc_b200.synth import CONTENTVEC_REGIMES, CONTENTVEC_SMALL, make_contentvec_state_dict
from oracle import content_oracle as co

RTOL, ATOL_RMS = 1e-3, 1e-4
SR = 16000


def white(n, seed):
    return 0.1 * torch.randn(n, generator=torch.Generator().manual_seed(seed))


def chirp(n):
    """A chirp with a DC offset and 0.5 s of exact zeros at each end (what the reference's slicer feeds)"""
    t = torch.arange(n, dtype=torch.float64) / SR
    x = 0.3 * torch.sin(2 * math.pi * (100 + 2000 * t / max(t[-1].item(), 1e-9)) * t) + 0.05
    z = min(SR // 2, n // 4)
    x[:z] = 0
    x[n - z:] = 0
    return x.float()


def level_frames(n):
    out = []
    for k, s in co.CONV_LAYERS:
        n = 0 if n < k else (n - k) // s + 1
        out.append(n)
    return out


# ----------------------------------------------------------------------------------------------------------------- CPU
def test_frame_count_rule():
    # the reference's own fixtures: dataset/1/1.wav resampled to 21 163 samples -> 65 frames, dataset/2/2.wav to 17 750 -> 55
    assert num_frames(21163) == 65 and num_frames(17750) == 55
    for n, t in {399: 0, 400: 1, 401: 1, 719: 1, 720: 2, 16000: 49, 16079: 49, 16080: 50, 16319: 50, 16320: 50}.items():
        assert num_frames(n) == t == co.num_frames(n), n


def test_oracle_precisions_agree_and_rows_are_alone():
    sd = make_contentvec_state_dict(0, "trained_like", **CONTENTVEC_SMALL)
    wav = torch.stack([white(9600, 1), chirp(9600), white(9600, 2)])
    a64 = co.extract(sd, wav, 2)
    a32 = co.extract(sd, wav, 2, dtype=torch.float32)
    assert ((a32.double() - a64).abs().max() / a64.pow(2).mean().sqrt()).item() < 1e-4
    lens = [9600, 6400, 400]
    rag = co.extract(sd, wav, 2, lengths=lens)
    for b, n in enumerate(lens):
        T = num_frames(n)
        assert torch.equal(rag[b, :T], co.extract(sd, wav[b:b + 1, :n], 2)[0])
        assert not rag[b, T:].any()


def test_weight_norm_key_forms_fold_alike():
    sd = make_contentvec_state_dict(0, "trained_like", **CONTENTVEC_SMALL)
    p = "encoder.pos_conv.0."
    alt = {(k.replace("weight_g", "parametrizations.weight.original0").replace("weight_v", "parametrizations.weight.original1")
            if k.startswith(p) else k): v for k, v in sd.items()}
    assert torch.equal(co.pos_conv_weight(sd), co.pos_conv_weight(alt))
    m1, m2 = ContentVec.from_state_dict(sd, num_heads=2), ContentVec.from_state_dict(alt, num_heads=2)
    assert all(torch.equal(m1.state_dict()[k], m2.state_dict()[k]) for k in m1.state_dict())


def test_registry_matches_fairseq_order():
    from ns2vc_b200 import _lib
    m = ContentVec()
    keys = [f"feature_extractor.conv_layers.{l}.0.weight" for l in range(7)]
    keys.insert(1, "feature_extractor.conv_layers.0.2.weight")
    keys.insert(2, "feature_extractor.conv_layers.0.2.bias")
    keys += ["post_extract_proj.weight", "post_extract_proj.bias", "encoder.pos_conv.0.bias", "encoder.pos_conv.0.weight_g",
             "encoder.pos_conv.0.weight_v"]
    for i in range(12):
        for sub in ("self_attn.k_proj", "self_attn.v_proj", "self_attn.q_proj", "self_attn.out_proj", "self_attn_layer_norm", "fc1", "fc2",
                    "final_layer_norm"):
            keys += [f"encoder.layers.{i}.{sub}.weight", f"encoder.layers.{i}.{sub}.bias"]
    keys += ["encoder.layer_norm.weight", "encoder.layer_norm.bias", "layer_norm.weight", "layer_norm.bias", "final_proj.weight",
             "final_proj.bias"]
    assert list(m.state_dict()) == keys == list(contentvec_param_shapes())
    L = _lib.lib()
    h = C.c_void_p()
    _lib.check(L.ns2vc_cv_create(C.byref(m._c_cfg()), C.byref(h)))
    try:
        got = []
        for i in range(L.ns2vc_cv_num_weights(h)):
            name, shp, nd = C.c_char_p(), (C.c_int64 * 4)(), C.c_int()
            _lib.check(L.ns2vc_cv_weight_info(h, i, C.byref(name), shp, C.byref(nd)))
            got.append((name.value.decode(), tuple(shp[k] for k in range(nd.value))))
    finally:
        L.ns2vc_cv_destroy(h)
    assert got == [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    for n in (400, 401, 16000, 16320, 336000):
        assert L.ns2vc_cv_num_frames(n) == num_frames(n)
    for bad in (dict(num_heads=10), dict(conv_dim=96), dict(embed_dim=800, num_heads=10), dict(pos_conv_groups=8),
                dict(pos_conv_kernel=100), dict(ffn_dim=100)):
        cfg = _lib.CvCfg(**{**CONTENTVEC, **bad})
        assert L.ns2vc_cv_create(C.byref(cfg), C.byref(h)) != 0, bad


def _fairseq_stub(sd, layer_norm_first=False):
    full = {"mask_emb": torch.zeros(sd["post_extract_proj.weight"].shape[0]), "label_embs_concat": torch.zeros(504, 32), **sd}
    layers = [types.SimpleNamespace(self_attn=types.SimpleNamespace(num_heads=2))]
    return types.SimpleNamespace(state_dict=lambda: dict(full),
                                 encoder=types.SimpleNamespace(layer_norm_first=layer_norm_first, layers=layers))


def test_loader_rejects_loudly():
    sd = make_contentvec_state_dict(3, "trained_like", **CONTENTVEC_SMALL)
    m = ContentVec.from_fairseq(_fairseq_stub(sd))
    assert m.cfg == CONTENTVEC_SMALL
    assert list(m.state_dict()) == list(sd) and all(torch.equal(m.state_dict()[k], v) for k, v in sd.items())
    cases = {
        "encoder.layers.1.fc2.bias": lambda d: d.pop("encoder.layers.1.fc2.bias"),
        "encoder.extra.weight": lambda d: d.__setitem__("encoder.extra.weight", torch.zeros(3)),
        "encoder.layers.0.fc1.weight": lambda d: d.__setitem__("encoder.layers.0.fc1.weight", torch.zeros(256, 127)),
        "feature_extractor.conv_layers.1.2.1.weight": lambda d: d.__setitem__("feature_extractor.conv_layers.1.2.1.weight", torch.ones(128)),
        "feature_extractor.conv_layers.2.0.bias": lambda d: d.__setitem__("feature_extractor.conv_layers.2.0.bias", torch.zeros(128)),
    }
    for key, edit in cases.items():
        d = dict(sd)
        edit(d)
        with pytest.raises(ValueError, match=key.replace(".", r"\.")):
            ContentVec.from_fairseq(_fairseq_stub(d))
    with pytest.raises(ValueError, match="layer_norm_first"):
        ContentVec.from_fairseq(_fairseq_stub(sd, layer_norm_first=True))
    with torch.no_grad(), pytest.raises(RuntimeError, match="no CPU path"):
        m.extract(torch.zeros(1, 800))
    with pytest.raises(ValueError):
        api.content_utterances(m, [torch.zeros(399)])


def test_oracle_against_golden_fixture():
    """tests/golden/content_tiny.pt (oracle/make_golden_content.py): transformers' eager HubertModel, each row alone"""
    import os
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "content_tiny.pt"))
    c, sd, wav, lens = g["cfg"], g["state_dict"], g["wav"], g["lengths"].tolist()
    got = co.extract(sd, wav, c["num_heads"], lens, dtype=torch.float32)
    assert got.shape == g["units"].shape
    assert ((got - g["units"]).abs().max() / g["units"].abs().max()).item() <= 1e-5
    got64 = co.extract(sd, wav, c["num_heads"], lens)
    assert ((got64 - g["units"].double()).abs().max() / g["units"].abs().max()).item() <= 1e-5
    for b, n in enumerate(lens):                                 # the stage before final_proj, too
        st = co.stages(sd, wav[b, :n], c["num_heads"], torch.float32)
        last = st[f"encoder.layers.{c['num_layers'] - 1}"]
        assert ((last - g["last_hidden_state"][b, :last.shape[0]]).abs().max() / g["last_hidden_state"].abs().max()).item() <= 1e-5


def _transformers_hubert(sd, cfg):
    transformers = pytest.importorskip("transformers")
    hc = transformers.HubertConfig(
        hidden_size=cfg["embed_dim"], num_hidden_layers=cfg["num_layers"], num_attention_heads=cfg["num_heads"],
        intermediate_size=cfg["ffn_dim"], conv_dim=(cfg["conv_dim"],) * 7, conv_stride=(5, 2, 2, 2, 2, 2, 2),
        conv_kernel=(10, 3, 3, 3, 3, 2, 2), num_conv_pos_embeddings=cfg["pos_conv_kernel"],
        num_conv_pos_embedding_groups=cfg["pos_conv_groups"], feat_extract_norm="group", conv_bias=False, do_stable_layer_norm=False,
        hidden_act="gelu", feat_extract_activation="gelu", feat_proj_layer_norm=True, layer_norm_eps=1e-5, hidden_dropout=0.0,
        attention_dropout=0.0, activation_dropout=0.0, feat_proj_dropout=0.0, layerdrop=0.0, apply_spec_augment=False)
    model = transformers.HubertModel(hc).eval()
    own = model.state_dict()
    ren = {}
    for k in sd:
        t = k
        if k.startswith("feature_extractor.conv_layers."):
            t = k.replace(".0.2.", ".0.layer_norm.").replace(".0.weight", ".conv.weight") if ".2." in k else k.replace(".0.weight", ".conv.weight")
        elif k.startswith("layer_norm."):
            t = "feature_projection." + k
        elif k.startswith("post_extract_proj."):
            t = k.replace("post_extract_proj", "feature_projection.projection")
        elif k.startswith("encoder.pos_conv.0."):
            leaf = k.rsplit(".", 1)[1]
            pre = "encoder.pos_conv_embed.conv."
            if leaf != "bias" and pre + leaf not in own:
                leaf = {"weight_g": "parametrizations.weight.original0", "weight_v": "parametrizations.weight.original1"}[leaf]
            t = pre + leaf
        elif k.startswith("encoder.layers."):
            t = (k.replace("self_attn_layer_norm", "layer_norm").replace("self_attn.", "attention.")
                 .replace(".fc1.", ".feed_forward.intermediate_dense.").replace(".fc2.", ".feed_forward.output_dense."))
        elif k.startswith("final_proj."):
            continue
        ren[t] = sd[k]
    missing, unexpected = model.load_state_dict(ren, strict=False)
    assert not unexpected and set(missing) <= {"masked_spec_embed"}, (missing, unexpected)
    return model


@pytest.mark.parametrize("full", [False, True])
def test_oracle_against_transformers_hubert(full):
    cfg = CONTENTVEC if full else CONTENTVEC_SMALL
    sd = make_contentvec_state_dict(7, "trained_like", **cfg)
    model = _transformers_hubert(sd, cfg)
    n = SR if full else 9600
    wav = torch.stack([white(n, 5), chirp(n)])
    with torch.no_grad():
        hs = model(wav).last_hidden_state
        got = torch.nn.functional.linear(hs, sd["final_proj.weight"], sd["final_proj.bias"])
    want = co.extract(sd, wav, cfg["num_heads"], dtype=torch.float32)
    rel = ((got - want).abs().max() / want.abs().max()).item()
    assert rel <= 1e-5, rel


# ----------------------------------------------------------------------------------------------------------------- GPU
_models = {}


def model(regime, small=False):
    key = (regime, small)
    if key not in _models:
        sd = make_contentvec_state_dict(0, regime, **(CONTENTVEC_SMALL if small else {}))
        heads = (CONTENTVEC_SMALL if small else CONTENTVEC)["num_heads"]
        _models[key] = (ContentVec.from_state_dict(sd, num_heads=heads).cuda().eval(), {k: v.cuda() for k, v in sd.items()}, heads)
    return _models[key]


def ratio(got, ref64, ref32):
    got, ref = got.double(), ref64.double()
    e32 = (ref32.double() - ref).abs().max()
    tol = torch.clamp(RTOL * ref.abs() + ATOL_RMS * ref.pow(2).mean().sqrt(), min=2 * e32.item())
    return ((got - ref).abs() / tol).max().item()


@pytest.fixture(autouse=True)
def _no_tf32():
    """The oracle's matmuls and convs in true fp32 / fp64 while a test of this module runs; the flags are restored after it"""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def stage_ratios(sd, heads, taps, wav, lengths):
    """{(stage, row): worst err/tol}; asserts exact zeros past each row's frames at every tap"""
    names = co.stage_names(sum(1 for k in sd if k.endswith(".fc1.weight")))
    worst = {}
    for b, n in enumerate(lengths):
        lf = level_frames(n)
        prev = wav[b, :n]
        for s in names:
            t = taps[s][b]
            T = lf[int(s.rsplit(".", 1)[1])] if s.startswith("feature_extractor.conv_layers.") else lf[-1]
            assert not t[T:].any(), f"{s}, row {b} (N = {n}): nonzero past its {T} frames"
            fn = co.stage_fn(sd, s, heads)
            r64, r32 = fn(prev.double()), fn(prev.float())
            worst[(s, b)] = ratio(t[:T], r64, r32)
            prev = t[:T]
    return worst


def batch_full():
    lens = [10 * SR, int(3.2 * SR), 401, 400]
    N = max(lens)
    wav = torch.zeros((4, N))
    wav[0] = white(N, 11)
    wav[1, :lens[1]] = chirp(lens[1])
    wav[2, :401] = white(401, 12)
    wav[3, :400] = chirp(400) + white(400, 13)
    return wav, lens


@pytest.mark.gpu
@pytest.mark.parametrize("regime", CONTENTVEC_REGIMES)
def test_stages_against_fp64(regime):
    m, sd, heads = model(regime)
    wav, lens = batch_full()
    wav = wav.cuda()
    taps = m.taps(wav, torch.tensor(lens))
    assert taps["frames"].tolist() == [num_frames(n) for n in lens]
    worst = stage_ratios(sd, heads, taps, wav, lens)
    bad = {k: v for k, v in worst.items() if v > 1.0}
    print(f"{regime}: worst err/tol {max(worst.values()):.3f} at {max(worst, key=worst.get)}")
    assert not bad, f"{regime}: stages over tolerance (stage, row): {bad}"


@pytest.mark.gpu
def test_long_row_attends_over_every_key():
    m, sd, heads = model("trained_like")
    n = 21 * SR
    wav = torch.stack([white(n, 21), torch.zeros(n)]).cuda()
    wav[1, :5 * SR] = white(5 * SR, 22).cuda()
    lens = [n, 5 * SR]
    taps = m.taps(wav, torch.tensor(lens))
    assert num_frames(n) == 1049
    worst = stage_ratios(sd, heads, taps, wav, lens)
    assert max(worst.values()) <= 1.0, {k: v for k, v in worst.items() if v > 1.0}


@pytest.mark.gpu
@torch.no_grad()
def test_padding_values_and_workspace_are_never_read():
    m, sd, heads = model("trained_like")
    wav, lens = batch_full()
    wav = wav.cuda()
    lt = torch.tensor(lens)
    u0, f0 = m.extract(wav, lt)
    poisoned = wav.clone()
    for b, n in enumerate(lens):
        poisoned[b, n:] = float("nan") if b % 2 else 1e30
    u1, f1 = m.extract(poisoned, lt)
    assert torch.equal(u0, u1) and torch.equal(f0, f1)
    ref = m.taps(wav, lt)
    m._ws = torch.full_like(m._ws, 255)
    got = m.taps(wav, lt)
    for k in ref:
        assert torch.equal(ref[k], got[k]), k


@pytest.mark.gpu
@torch.no_grad()
def test_rows_match_their_own_runs():
    m, sd, heads = model("trained_like")
    wav, lens = batch_full()
    wav = wav.cuda()
    units, frames = m.extract(wav, torch.tensor(lens))
    identical = []
    for b, n in enumerate(lens):
        alone, _ = m.extract(wav[b:b + 1, :n])
        T = num_frames(n)
        ref64 = co.extract(sd, wav[b:b + 1, :n], heads)[0]
        ref32 = co.extract(sd, wav[b:b + 1, :n], heads, dtype=torch.float32)[0]
        assert ratio(units[b, :T], ref64, ref32) <= 1.0 and ratio(alone[0], ref64, ref32) <= 1.0, b
        identical.append(torch.equal(units[b, :T], alone[0]))
    print(f"rows bit-identical to their B = 1 runs: {identical}")


@pytest.mark.gpu
@torch.no_grad()
def test_graph_replay_with_new_lengths():
    m, sd, heads = model("trained_like", small=True)
    N = 24000
    wav = torch.stack([white(N, 31), chirp(N), white(N, 32)]).cuda()
    lens = torch.tensor([N, 9000, 4000], device="cuda")
    m.extract(wav, lens)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        units, frames = m.extract(wav, lens)
    lens.copy_(torch.tensor([12345, N, 400]))
    g.replay()
    torch.cuda.synchronize()
    m2 = ContentVec.from_state_dict(sd, num_heads=heads).cuda()
    want, wf = m2.extract(wav, torch.tensor([12345, N, 400]))
    assert torch.equal(units, want) and torch.equal(frames, wf)
    assert m.launch_count() > 0


@pytest.mark.gpu
@torch.no_grad()
def test_drop_in_and_content_utterances():
    m, sd, heads = model("trained_like", small=True)
    wavs = [chirp(12000), white(5000, 41), white(400, 42), white(20000, 43)]
    c = get_hubert_content(m, torch.stack([wavs[0], wavs[0] * 0.5], 1).cuda())
    assert c.shape == (1, 32, num_frames(12000)) and c.is_cuda
    ref64 = co.extract(sd, (wavs[0] * 0.75)[None].cuda(), heads)[0]
    ref32 = co.extract(sd, (wavs[0] * 0.75)[None].cuda(), heads, dtype=torch.float32)[0]
    assert ratio(c[0].t(), ref64, ref32) <= 1.0
    got = api.content_utterances(m, wavs, max_batch=2)
    for w, u in zip(wavs, got):
        alone, _ = m.extract(w[None].cuda())
        assert u.shape == (32, num_frames(w.shape[0]))
        r64 = co.extract(sd, w[None].cuda(), heads)[0]
        r32 = co.extract(sd, w[None].cuda(), heads, dtype=torch.float32)[0]
        assert ratio(u.t(), r64, r32) <= 1.0
    tgt = [80, 30, 3, 100]
    exp = api.content_utterances(m, wavs, target_frames=tgt, max_batch=8)
    from ns2vc_b200.frontend import repeat_expand_2d
    for u, e, t in zip(got, exp, tgt):
        assert e.shape == (32, t) and torch.equal(e, repeat_expand_2d(u, t))
