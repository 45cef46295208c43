"""Reusable voice encodings: ``Pre_model.encode_voices`` / ``infer_content`` (C-ABI ``ns2vc_pre_encode_voices_ragged`` /
``ns2vc_pre_infer_content_ragged``), ``api.encode_voices`` and the ``Voice`` prompts of the conversion entry points.

CPU: the new entry points are exported and bound, and a ``Voice`` from another ``Pre_model``, on another device, over
``max_prompt_frames`` or a malformed mel raises ValueError.  GPU, every comparison ``torch.equal``: the two halves against
``ns2vc_pre_infer_ragged`` row by row and their launch counts; ``convert_utterances``, ``convert_files``, ``StreamConverter``
and ``ConversionServer`` (one GPU and two ranks) with voices against the same chain restated with the fused encoders
(``Pre_model.infer(per_utterance=True)`` + ``sample_latents`` + ``Vocos.decode``)."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist

from ns2vc_b200 import _lib, api, convert, frontend, serve, stream
from ns2vc_b200.pre_model import Pre_model, Voice

SR = 44100
SMALL = {"phoneme_encoder": dict(in_channels=32, hidden_channels=32, out_channels=32, n_layers=2),
         "prompt_encoder": dict(in_channels=100, hidden_channels=32, out_channels=32, n_layers=2)}


# ----------------------------------------------------------------------------------------------------------------- CPU
def test_entry_points_are_exported_and_bound():
    L = _lib.lib()
    for name in ("ns2vc_pre_encode_voices_ragged", "ns2vc_pre_infer_content_ragged"):
        fn = getattr(L, name)
        assert fn.restype is not None and len(fn.argtypes) == 9, name


def _voice(m, S=5, device="cpu"):
    return Voice(torch.zeros(32, device=device), torch.zeros((S, 32), device=device), m)


def test_voice_argument_errors():
    m, other = Pre_model(SMALL), Pre_model(SMALL)
    c, lengths = torch.zeros(1, 32, 4), torch.tensor([4])
    with pytest.raises(ValueError, match="another Pre_model"):
        m.infer_content(c, lengths, [_voice(other)])
    with pytest.raises(ValueError, match="lives on meta"):
        m.infer_content(c, lengths, [_voice(m, device="meta")])
    with pytest.raises(ValueError, match="expected a Voice"):
        m.infer_content(c, lengths, [torch.zeros(100, 5)])
    with pytest.raises(ValueError, match="spk"):
        m.infer_content(c, lengths, [Voice(torch.zeros(31), torch.zeros(5, 32), m)])
    w = [torch.zeros(20000)]
    with pytest.raises(ValueError, match="another Pre_model"):
        convert.convert_utterances(None, m, torch.nn.Linear(1, 1), None, w, SR, _voice(other))
    with pytest.raises(ValueError, match="prompt 1: expected a mel"):
        convert.convert_utterances(None, m, None, None, w * 2, SR, [_voice(m), torch.zeros(100)])
    for bad in (torch.zeros(99, 5), torch.zeros(100, 0), torch.zeros(100, 5, 1), "mel"):
        with pytest.raises(ValueError, match="mel 1"):
            api.encode_voices(m, [torch.zeros(100, 5), bad])
    with pytest.raises(ValueError, match="prompt"):
        stream.StreamConverter(None, m, torch.nn.Linear(1, 1), None, [_voice(m), torch.zeros(99, 3)], 16000)


def test_server_checks_voices():
    m, other = Pre_model(SMALL), Pre_model(SMALL)
    srv = serve.ConversionServer(None, m, torch.nn.Linear(1, 1), None, slots=2, max_frames=400, max_prompt_frames=8)
    wav = torch.zeros(20000)
    with pytest.raises(ValueError, match="max_prompt_frames"):
        srv.submit(wav, SR, _voice(m, S=9))
    with pytest.raises(ValueError, match="another Pre_model"):
        srv.submit(wav, SR, _voice(other))
    with pytest.raises(ValueError, match="lives on meta"):
        srv.submit(wav, SR, _voice(m, device="meta"))
    assert srv.submit(wav, SR, _voice(m, S=8)) == 0


# ----------------------------------------------------------------------------------------------------------------- GPU
_pre = {}


def _shipped():
    """The shipped condition encoders (6 + 6 layers, 512 / 256 wide) with seed-0 synthetic weights, on cuda."""
    if not _pre:
        from ns2vc_b200.synth import make_pre_state_dict
        from test_numerics_fp64 import PRE_FULL
        m = Pre_model(PRE_FULL)
        m.load_state_dict(make_pre_state_dict(PRE_FULL, 0))
        _pre["m"] = m.to("cuda").eval()
    return _pre["m"]


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 3, 8])
def test_voice_and_content_halves_equal_the_ragged_program(B):
    m = _shipped()
    g = torch.Generator().manual_seed(B)
    S, T = 37, 53
    refer_lengths = torch.tensor(([1, S, 11, 2, 29, 36, 5, 17])[:B])
    lengths = torch.tensor(([T, 1, 40, 53, 2, 7, 52, 30])[:B])
    c = torch.randn((B, m.cfg["phoneme_encoder"]["in_channels"], T), generator=g).cuda()
    refer = (torch.randn((B, 100, S), generator=g) - 4).cuda()
    content_f, prompt_f = m.infer((c, refer, None, None, None, lengths, refer_lengths, None), per_utterance=True)
    n_fused = m.launch_count()
    voices = m.encode_voices(refer, refer_lengths)
    n_voice = m.launch_count()
    content = m.infer_content(c, lengths, voices)
    n_content = m.launch_count()
    torch.cuda.synchronize()
    for b, v in enumerate(voices):
        Sb = int(refer_lengths[b])
        assert v.S_v == Sb and v.pre_model is m and v.device == c.device
        assert torch.equal(v.prompt, prompt_f[:Sb, b]), f"row {b} (S_b={Sb}): prompt differs from ns2vc_pre_infer_ragged"
    assert torch.equal(content, content_f), "content differs from ns2vc_pre_infer_ragged"
    # Each encoder is 6 + 6 L launches (SEQMASK, ENC_INPUT, pre LN, pre GEMM, per layer 4 GEMMs + attention + LN2, out GEMM,
    # LN_MASK).  The voice half adds NCT2TOK, ref_enc's 7 launches and spk_proj; each half has its own statistics memset.
    L_phone, L_prompt = 6, 6
    assert n_content == 1 + 6 + 6 * L_phone, n_content
    assert n_voice == 1 + 6 + 6 * L_prompt + 1 + 7 + 1, n_voice
    assert n_voice + n_content == n_fused + 1, (n_voice, n_content, n_fused)


# ---- the small chain of tests/test_convert.py, restated with the fused encoders
@torch.no_grad()
def _restated_batch(models, wavs, sr, mels, xs, steps, method="unipc"):
    """convert_batch as it ran before voices could be reused: the fused ragged encoders on every row."""
    cv, pre, unet, voc = models
    dev = next(unet.parameters()).device
    plans = [convert.frame_plan(int(w.shape[0]), sr) for w in wavs]
    B, n = len(wavs), [int(w.shape[0]) for w in wavs]
    tl, sl = [p["T"] for p in plans], [int(p.shape[1]) for p in mels]
    T, S = max(tl), max(sl)
    wav = torch.zeros((B, max(n)), device=dev)
    for j, w in enumerate(wavs):
        wav[j, :n[j]] = w.to(dev)
    w24, _ = frontend.resample(wav, sr, convert.TARGET_SR, torch.tensor(n))
    w16, _ = frontend.resample(w24, convert.TARGET_SR, convert.CONTENT_SR, torch.tensor([p["n24"] for p in plans]))
    units, _ = cv.extract(w16, torch.tensor([p["n16"] for p in plans]))
    c = torch.zeros((B, units.shape[2], T), device=dev)
    refer = torch.zeros((B, 100, S), device=dev)
    for j in range(B):
        c[j, :, :tl[j]] = frontend.repeat_expand_2d(units[j, :plans[j]["units"]].t(), tl[j])
        refer[j, :, :sl[j]] = mels[j].to(dev)
    tl_h, sl_h = torch.tensor(tl), torch.tensor(sl)
    content, prompt = pre.infer((c, refer, None, None, None, tl_h, sl_h, None), per_utterance=True)
    x = torch.zeros((B, 100, T), device=dev)
    for j in range(B):
        x[j, :, :tl[j]] = xs[j].reshape(100, tl[j]).to(dev)
    lat = api.sample_latents(unet, x, content, prompt, sl_h, steps=steps, method=method, device=dev, content_lengths=tl_h)
    audio = voc.decode(lat, tl_h)
    return [audio[j, :tl[j] * convert.HOP] for j in range(B)], [lat[j, :, :tl[j]] for j in range(B)]


def _restated(models, wavs, sr, mels, xs, steps, max_batch):
    out = [None] * len(wavs)
    for idx in api.batch_plan([int(w.shape[0]) for w in wavs], max_batch):
        audio, _ = _restated_batch(models, [wavs[i] for i in idx], sr, [mels[i] for i in idx], [xs[i] for i in idx], steps)
        for j, i in enumerate(idx):
            out[i] = audio[j]
    return out


@pytest.fixture(scope="module")
def small():
    from test_shard_convert import _chain
    models, wavs, prompt = _chain(torch.device("cuda"))
    g = torch.Generator().manual_seed(11)
    mels = [prompt, (torch.randn((100, 23), generator=g) - 4).float(), (torch.randn((100, 1), generator=g) - 4).float()]
    return models, wavs, mels


def _x_T(wavs, seed, sr=SR):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn((1, 100, convert.frame_plan(len(w), sr)["T"]), generator=g) for w in wavs]


class _Counter:
    """Wraps ``obj.name`` and adds the first dim of its first argument to ``rows`` on every call."""

    def __init__(self, obj, name):
        self.obj, self.name, self.rows, self.fn = obj, name, 0, getattr(obj, name)

        def call(x, *a, **k):
            self.rows += int(x.shape[0])
            return self.fn(x, *a, **k)
        setattr(obj, name, call)

    def restore(self):
        delattr(self.obj, self.name)


@pytest.mark.gpu
def test_convert_utterances_with_voices(small):
    models, wavs, mels = small
    pre = models[1]
    xs = _x_T(wavs, 4)
    steps, mb = 4, 4
    voices = api.encode_voices(pre, mels)
    mixed_mels = [mels[i % 3] for i in range(len(wavs))]
    mixed = [voices[i % 3] if i % 2 else mels[i % 3] for i in range(len(wavs))]
    cases = {"one Voice": (voices[1], [mels[1]] * len(wavs)), "one shared mel": (mels[0], [mels[0]] * len(wavs)),
             "mels and Voices": (mixed, mixed_mels)}
    for tag, (prompt, want_mels) in cases.items():
        enc = _Counter(pre, "encode_voices")
        try:
            got = convert.convert_utterances(*models, wavs, SR, prompt, steps=steps, max_batch=mb, x_T=xs)
        finally:
            enc.restore()
        want = _restated(models, wavs, SR, want_mels, xs, steps, mb)
        bad = [i for i in range(len(wavs)) if not torch.equal(got[i], want[i])]
        assert not bad, f"{tag}: waveforms {bad} differ from the fused-encoder chain"
        n_mels = {"one Voice": 0, "one shared mel": 1, "mels and Voices": 3}[tag]
        assert enc.rows == n_mels, f"{tag}: the voice encoder saw {enc.rows} rows, want {n_mels} (one per distinct mel)"


@pytest.mark.gpu
def test_convert_files_encodes_each_voice_and_each_sub_slice_once(small):
    from ns2vc_b200 import slicer
    models, wavs, mels = small
    cv, pre = models[0], models[1]
    files = [(wavs[2].numpy(), SR), (torch.cat([wavs[0], torch.zeros(SR), wavs[5]]).numpy(), SR)]
    vsr = 24000
    voices = [(torch.from_numpy(np.random.default_rng(k).standard_normal(int(vsr * d)).astype(np.float32) * 0.1), vsr)
              for k, d in enumerate((1.1, 0.6, 1.7))]
    dev = torch.device("cuda")
    steps, mb, clip = 3, 4, 1.5
    chunks = slicer.cut_batch([f[0] for f in files], [SR, SR], -40, 5000, device=dev)
    audio_data = [slicer.chunks2audio(f[0], c) for f, c in zip(files, chunks)]
    subs = [convert._plan_slices(a, SR, 0.5, clip, 0) for a in audio_data]
    n_subs = sum(len(s) for s in subs)
    x_T = [[_x_T(ss, 20 + 3 * f + v) for v in range(3)] for f, ss in enumerate(subs)]
    ext, enc = _Counter(cv, "extract"), _Counter(pre, "encode_voices")
    try:
        got = convert.convert_files(*models, files, voices, clip_seconds=clip, steps=steps, max_batch=mb, x_T=x_T)
    finally:
        ext.restore()
        enc.restore()
    assert ext.rows == n_subs, f"ContentVec saw {ext.rows} rows for {n_subs} distinct sub-slices"
    assert enc.rows == 3, f"the voice encoder saw {enc.rows} rows for 3 voices"
    mel = convert.voice_mels(voices, dev)
    items = [(f, v, k) for f in range(2) for v in range(3) for k in range(len(subs[f]))]
    outs = _restated(models, [torch.from_numpy(subs[f][k].astype(np.float32)) for f, _, k in items], SR, [mel[v] for _, v, _ in items],
                     [x_T[f][v][k] for f, v, k in items], steps, mb)
    per = {(f, v): [] for f in range(2) for v in range(3)}
    for (f, v, _), o in zip(items, outs):
        per[(f, v)].append(o.cpu().numpy())
    for f in range(2):
        for v in range(3):
            want = convert.stitch(audio_data[f], SR, per[(f, v)], 0.5, clip, 0, 0.75)
            assert np.array_equal(got[f][v], want), f"file {f}, voice {v} differs from the fused-encoder chain"


@pytest.mark.gpu
def test_stream_ticks_equal_the_fused_encoders(small):
    models, _, mels = small
    sr, B = 16000, 3
    prompts = [mels[0], api.encode_voices(models[1], [mels[1]])[0], mels[2]]
    sess = stream.StreamConverter(*models, prompts, sr, steps=3)
    tick_mels = [mels[0], mels[1], mels[2]]
    g = torch.Generator().manual_seed(9)
    T = sess.plan["T"]
    bad = []
    for t in range(4):
        if t == 2:
            new = (torch.randn((100, 31), generator=g) - 4).float()
            sess.reset(1, new)
            tick_mels[1] = new
        block = 0.1 * torch.randn((B, sess.plan["block_in"]), generator=g)
        xs = [torch.randn((1, 100, T), generator=g) for _ in range(B)]
        window = torch.cat((sess.window[:, sess.plan["block_in"]:], block.cuda()), dim=1)
        want, _ = _restated_batch(models, list(window.unbind(0)), sr, tick_mels, xs, 3)
        sess.push(block, x_T=xs)
        seg = torch.stack(want)[:, T * convert.HOP - sess.plan["seg"]:]
        if not torch.equal(sess.seg, seg):
            bad.append(t)
    assert not bad, f"ticks {bad} differ from the tick restated with the fused encoders"


SERVE_KW = dict(slots=2, max_frames=400, max_prompt_frames=80, steps=4)


def _serve_all(srv, wavs, prompts, xs):
    tickets = {srv.submit(w, SR, p, x_T=x): i for i, (w, p, x) in enumerate(zip(wavs, prompts, xs))}
    res = srv.drain()
    return {tickets[tk]: v for tk, v in res.items()}


@pytest.mark.gpu
def test_server_voice_requests_equal_mel_requests(small):
    models, wavs, mels = small
    xs = _x_T(wavs, 6)
    voices = api.encode_voices(models[1], mels)
    by_mel = _serve_all(serve.ConversionServer(*models, **SERVE_KW), wavs, [mels[i % 3] for i in range(6)], xs)
    enc = _Counter(models[1], "encode_voices")
    try:
        by_voice = _serve_all(serve.ConversionServer(*models, **SERVE_KW), wavs, [voices[i % 3] for i in range(6)], xs)
    finally:
        enc.restore()
    assert enc.rows == 0, "admission encoded a Voice request's prompt"
    bad = [i for i in range(6) if not torch.equal(by_voice[i], by_mel[i])]
    assert not bad, f"Voice requests {bad} differ from the same requests with mels"


def _group_worker(rank, world, out_dir):
    from test_shard_convert import _chain
    dev = torch.device("cuda", torch.cuda.current_device())
    models, wavs, prompt = _chain(dev)
    g = torch.Generator().manual_seed(13)
    mels = [prompt, (torch.randn((100, 23), generator=g) - 4).float()]
    xs = _x_T(wavs, 7)
    voices = api.encode_voices(models[1], mels)
    prompts = [voices[i % 2] if i % 3 else mels[i % 2] for i in range(6)]
    out = {}
    if rank == 0:
        out["one"] = _serve_all(serve.ConversionServer(*models, **SERVE_KW), wavs, prompts, xs)
    srv = serve.ConversionServer(*models, group=dist.group.WORLD, **SERVE_KW)
    enc = _Counter(models[1], "encode_voices")
    tickets = {}
    while True:
        if rank == 0 and not tickets:
            tickets = {srv.submit(w, SR, p, x_T=x): i for i, (w, p, x) in enumerate(zip(wavs, prompts, xs))}
        done = srv.tick()
        out.setdefault("two", {}).update({tickets[tk]: v.cpu() for tk, v in done.items()})
        if srv._idle:
            break
    enc.restore()
    out["encoded_rows"] = enc.rows
    if rank == 0:
        out["one"] = {i: v.cpu() for i, v in out["one"].items()}
    path = os.path.join(out_dir, f"rank{rank}.pt")
    torch.save(out, path)
    return path


@pytest.mark.gpu
def test_server_voice_requests_on_two_ranks_equal_one_gpu(tmp_path):
    from test_shard_convert import _run
    backend = "nccl" if torch.cuda.device_count() >= 2 else "gloo"
    paths = _run(_group_worker, 2, str(tmp_path), backend=backend, timeout=900)
    r0, r1 = [torch.load(p, weights_only=False) for p in paths]
    assert sorted(r0["two"]) == list(range(6)) and r1["two"] == {}
    bad = [i for i in range(6) if not torch.equal(r0["two"][i], r0["one"][i])]
    assert not bad, f"requests {bad} differ between two ranks and one GPU"
    # the mel requests (0 and 3) are encoded where they are admitted; the four Voice requests nowhere
    assert r0["encoded_rows"] + r1["encoded_rows"] == 2, (r0["encoded_rows"], r1["encoded_rows"])
