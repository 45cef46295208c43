"""Live conversion (``stream.StreamConverter``): sliding-window ticks joined by SOLA.

CPU: the session geometry (``stream_plan``), the fp64 SOLA oracle on planted shifts and a silent tail, and the argument errors.
GPU: the SOLA kernel alone against the oracle on six kinds of rows and three geometries; then whole sessions on the small
chain of ``test_convert.py`` (3 streams with different prompts, at 44.1 and 16 kHz, one stream reset with a longer prompt):
every tick's converted window of every stream against ``convert.convert_batch`` of that window alone, the emitted block and
tail against the oracle SOLA of the session's own segment and previous tail, the windows against the host ring model bit for
bit, and the default x_T draws."""
import numpy as np
import pytest
import torch

from ns2vc_b200 import api, convert, stream
from oracle import stream_oracle
from test_convert import chain  # noqa: F401  (the module-scoped fixture of small chained models)

RATES = (16000, 22050, 24000, 32000, 44100, 48000)


# ----------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("sr", RATES)
def test_plan_accepts_the_defaults_at_common_rates(sr):
    p = stream.stream_plan(sr)
    assert (p["T"], p["Nb"], p["Nc"], p["Ns"], p["seg"]) == (195, 45 * 256, 1024, 512, 45 * 256 + 1024 + 512)
    assert p["block_in"] * 24000 == 45 * 256 * sr and p["context_in"] * 24000 == 150 * 256 * sr
    assert p["W_in"] == p["block_in"] + p["context_in"]
    assert convert.frame_plan(p["W_in"], sr)["T"] == p["T"]


def test_plan_rejects_bad_geometry():
    with pytest.raises(ValueError, match="block_frames=48.*45 or 50"):
        stream.stream_plan(44100, block_frames=48)
    with pytest.raises(ValueError, match="context_frames=7"):
        stream.stream_plan(44100, context_frames=7)
    with pytest.raises(ValueError, match="shorter than crossfade"):
        stream.stream_plan(16000, context_frames=3)                # 768 samples < 1024 + 512
    with pytest.raises(ValueError, match="shorter than crossfade"):
        stream.stream_plan(24000, context_frames=5, crossfade=1024, search=512)
    with pytest.raises(ValueError, match="shorter than the crossfade"):
        stream.stream_plan(24000, block_frames=3)                  # 768 samples < 1024
    with pytest.raises(ValueError):
        stream.stream_plan(0)


def _planted(rng, k0, Nb, Nc, Ns):
    """A previous tick's tail taken from one signal and a segment of the same signal continued, shifted so that seg[k0 + i] is
    tail[i]."""
    y = rng.standard_normal(Nb + 2 * Nc + 2 * Ns + 10).astype(np.float32)
    P = Ns + 5
    tail = y[P:P + Nc].copy()
    seg = y[P - k0:P - k0 + Nb + Nc + Ns].copy()
    return seg, tail, y, P


@pytest.mark.parametrize("k0", [0, 1, 137, 512])
def test_oracle_finds_a_planted_shift(k0):
    p = stream.stream_plan(16000)
    Nb, Nc, Ns = p["Nb"], p["Nc"], p["Ns"]
    seg, tail, y, P = _planted(np.random.default_rng(k0), k0, Nb, Nc, Ns)
    out, new_tail, k = stream_oracle.sola(seg, tail, stream.fade_in_table(Nc), Nb, Nc, Ns)
    assert k == k0
    assert np.allclose(out, y[P:P + Nb], rtol=0, atol=1e-6)          # the cross-fade of a signal with itself is the signal
    assert np.array_equal(new_tail, y[P + Nb:P + Nb + Nc].astype(np.float64))


def test_oracle_takes_offset_zero_after_silence():
    rng = np.random.default_rng(3)
    seg = rng.standard_normal(11520 + 1024 + 512)
    _, _, k = stream_oracle.sola(seg, np.zeros(1024), stream.fade_in_table(1024), 11520, 1024, 512)
    assert k == 0


def test_fade_in_table():
    f = stream.fade_in_table(1024)
    assert f.dtype == np.float32 and f[0] == 0.0 and f[-1] == 1.0
    i = np.arange(1024, dtype=np.float64)
    assert np.array_equal(f, (np.sin(np.pi / 2 * (i / 1023)) ** 2).astype(np.float32))


def test_argument_errors():
    dummy = torch.nn.Linear(1, 1)                        # stands in for the models: only the denoiser's device is read here
    mel = torch.zeros(100, 30)
    for method in ("ddpm", "ddim", "euler"):
        with pytest.raises(ValueError) as got:
            stream.StreamConverter(None, None, dummy, None, [mel], 16000, method=method)
        with pytest.raises(ValueError) as want:
            convert._check_method(method, None)
        assert str(got.value) == str(want.value)
    with pytest.raises(ValueError, match="empty"):
        stream.StreamConverter(None, None, dummy, None, [], 16000)
    with pytest.raises(ValueError, match="prompt 1"):
        stream.StreamConverter(None, None, dummy, None, [mel, torch.zeros(80, 30)], 16000)
    with pytest.raises(ValueError, match="block_frames=46"):
        stream.StreamConverter(None, None, dummy, None, [mel], 44100, block_frames=46)
    s = stream.StreamConverter(None, None, dummy, None, [mel, mel], 16000)
    assert s.plan["block_in"] == 7680 and tuple(s.window.shape) == (2, s.plan["W_in"]) and tuple(s.tail.shape) == (2, 1024)
    for bad in (torch.zeros(2, 7679), torch.zeros(1, 7680), torch.zeros(2 * 7680), torch.zeros(2, 1, 7680)):
        with pytest.raises(ValueError, match="block"):
            s.push(bad)
    with pytest.raises(ValueError, match="x_T"):
        s.push(torch.zeros(2, 7680), x_T=[torch.zeros(1, 100, 195)])
    with pytest.raises(ValueError, match="x_T 1"):
        s.push(torch.zeros(2, 7680), x_T=[torch.zeros(1, 100, 195), torch.zeros(1, 100, 194)])
    assert not s.window.any()                            # a rejected push leaves the windows alone
    for slot in (2, -1, 5):
        with pytest.raises(IndexError):
            s.reset(slot)
    with pytest.raises(TypeError):
        s.reset(0.5)
    with pytest.raises(ValueError, match="prompt"):
        s.reset(0, torch.zeros(100, 0))
    s.reset(1, torch.ones(100, 40))
    assert tuple(s.prompts[1].shape) == (100, 40)
    assert api.StreamConverter is stream.StreamConverter


# ----------------------------------------------------------------------------------------------------------------- GPU
def check_sola(seg, prev_tail, fade, out, new_tail, k_gpu, Nb, Nc, Ns, ties=(), tag=""):
    """The SOLA of each row against the fp64 oracle on the same inputs.  k must be the oracle's, or within 1e-9 relative of the
    oracle's maximum ratio (printed); rows in ``ties`` have equal ratios everywhere and must take k = 0.  out and the new tail
    must equal the oracle at the GPU's k within 1e-6 (|seg| + |tail|).  Returns the failures."""
    seg, prev_tail = np.asarray(seg, np.float64), np.asarray(prev_tail, np.float64)
    out, new_tail = np.asarray(out, np.float64), np.asarray(new_tail, np.float64)
    bad = []
    for b in range(seg.shape[0]):
        kg = int(k_gpu[b])
        name = f"{tag} row {b}"
        if not 0 <= kg <= Ns:
            bad.append(f"{name}: k {kg} outside [0, {Ns}]")
            continue
        r = stream_oracle.sola_ratios(seg[b], prev_tail[b], Nc, Ns)
        ko = int(np.argmax(r))
        if b in ties and kg != 0:
            bad.append(f"{name}: equal ratios everywhere, k {kg} instead of the lowest (0)")
        if kg != ko:
            near = r[kg] >= r[ko] - 1e-9 * abs(r[ko])
            print(f"{name}: GPU k {kg} vs oracle k {ko}, ratios {r[kg]!r} / {r[ko]!r} ({'within' if near else 'NOT within'} 1e-9)")
            if not near:
                bad.append(f"{name}: k {kg} vs oracle {ko}, ratio {r[kg]:.9g} vs max {r[ko]:.9g}")
        o, t = stream_oracle.sola_at(seg[b], prev_tail[b], fade, Nb, Nc, kg)
        tail_pad = np.zeros(Nb)
        tail_pad[:Nc] = np.abs(prev_tail[b, :Nc])
        tol_o = 1e-6 * (np.abs(seg[b, kg:kg + Nb]) + tail_pad)
        tol_t = 1e-6 * np.abs(seg[b, kg + Nb:kg + Nb + Nc])
        eo, et = np.abs(out[b] - o) - tol_o, np.abs(new_tail[b] - t) - tol_t
        if (eo > 0).any() or (et > 0).any():
            bad.append(f"{name} (k {kg}): out exceeds its bound at {np.flatnonzero(eo > 0)[:5]}, tail at {np.flatnonzero(et > 0)[:5]}")
    return bad


@pytest.mark.gpu
@pytest.mark.parametrize("Nb,Nc,Ns", [(11520, 1024, 512), (1000, 777, 301), (700, 333, 0)])
def test_sola_kernel_matches_the_oracle(Nb, Nc, Ns):
    rng = np.random.default_rng(Nb + Nc + Ns)
    L = Nb + Nc + Ns
    B = 6
    seg = np.zeros((B, L), np.float32)
    tail = np.zeros((B, Nc), np.float32)
    seg[0], tail[0] = rng.standard_normal(L), rng.standard_normal(Nc)                     # random
    k1, k4 = min(137, Ns), Ns
    seg[1], tail[1] = _planted(rng, k1, Nb, Nc, Ns)[:2]                                   # planted shifts
    seg[4], tail[4] = _planted(rng, k4, Nb, Nc, Ns)[:2]
    seg[2] = rng.standard_normal(L)                                                       # silent tail
    seg[3], tail[3] = 0.3, rng.standard_normal(Nc)                                       # constant segment: equal ratios
    seg[5], tail[5] = (0.5 * rng.standard_normal(L)).cumsum() / 30, rng.standard_normal(Nc) * 0.01 # smooth, small tail
    fade = stream.fade_in_table(Nc)
    # seg rows inside a wider buffer: the kernel takes a batch stride
    buf = torch.zeros((B, L + 37), dtype=torch.float32)
    buf[:, 5:5 + L] = torch.from_numpy(seg)
    dbuf = buf.cuda()
    dtail = torch.from_numpy(tail).cuda()
    out, k = stream.sola(dbuf[:, 5:], dtail, torch.from_numpy(fade).cuda(), Nb, Nc, Ns)
    torch.cuda.synchronize()
    k = k.cpu().numpy()
    print(f"Nb={Nb} Nc={Nc} Ns={Ns}: GPU k {k.tolist()}")
    assert k[1] == k1 and k[4] == k4, "a planted shift was not found"
    bad = check_sola(seg, tail, fade, out.cpu().numpy(), dtail.cpu().numpy(), k, Nb, Nc, Ns, ties=(2, 3), tag=f"({Nb}, {Nc}, {Ns})")
    assert not bad, "\n".join(bad)
    assert torch.equal(dbuf.cpu(), buf), "the kernel wrote into seg"


def _voice(rng, n, sr):
    t = np.arange(n) / sr
    f0 = 110 + 200 * rng.random()
    return (0.3 * np.sin(2 * np.pi * f0 * t) * (1 + 0.5 * np.sin(2 * np.pi * 3 * t)) + 0.05 * rng.standard_normal(n)).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("sr", [44100, 16000])
def test_each_tick_equals_each_window_converted_alone(chain, sr):  # noqa: F811
    models, _, _, _ = chain
    g = torch.Generator().manual_seed(sr)
    prompts = [(torch.randn((100, s), generator=g) - 4.0).float() for s in (70, 50, 90)]
    new_prompt = (torch.randn((100, 120), generator=g) - 4.0).float()
    steps, ticks = 4, 6
    sess = stream.StreamConverter(*models, prompts, sr, steps=steps)
    p = sess.plan
    B, T, Nb, Nc, Ns = 3, p["T"], p["Nb"], p["Nc"], p["Ns"]
    rng = np.random.default_rng(sr)
    audio_in = np.stack([_voice(rng, ticks * p["block_in"], sr) for _ in range(B)])
    ring = stream_oracle.WindowRing(B, p["W_in"])
    fade = sess.fade_in.cpu().numpy()
    bad = []
    for tick in range(ticks):
        if tick == 2:
            sess.reset(1, new_prompt)
            ring.reset(1)
            prompts[1] = new_prompt
        block = torch.from_numpy(audio_in[:, tick * p["block_in"]:(tick + 1) * p["block_in"]].copy())
        xs = [torch.randn((1, 100, T), generator=g) for _ in range(B)]
        prev_tail = sess.tail.cpu().numpy().copy()
        out = sess.push(block, x_T=xs)
        assert out.device.type == "cpu" and tuple(out.shape) == (B, Nb)
        assert np.array_equal(sess.window.cpu().numpy(), ring.push(block.numpy())), f"tick {tick}: window differs from the ring model"
        seg = sess.seg.cpu()
        for j in range(B):
            alone = convert.convert_batch(*models, [sess.window[j]], sr, [prompts[j]], [xs[j]], "unipc", steps)["audio"][0]
            want = alone[T * 256 - p["seg"]:].double().cpu()
            rel = ((seg[j].double() - want).norm() / want.norm()).item()
            print(f"sr {sr} tick {tick} slot {j}: seg ||diff||/||alone|| {rel:.2e}, bit-identical {torch.equal(seg[j], want.float())}, "
                  f"k {int(sess.offsets[j])}")
            if not rel <= 1e-4:
                bad.append(f"tick {tick} slot {j}: ||diff||/||alone|| {rel:.2e}")
        bad += check_sola(seg.numpy(), prev_tail, fade, out.numpy(), sess.tail.cpu().numpy(), sess.offsets.cpu().numpy(), Nb, Nc, Ns,
                          tag=f"sr {sr} tick {tick}")
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
def test_default_x_T_is_drawn_per_slot_in_order(chain):  # noqa: F811
    models, _, prompt, _ = chain
    prompts = [prompt, prompt[:, :40]]
    sr = 16000
    a = stream.StreamConverter(*models, prompts, sr, steps=3)
    b = stream.StreamConverter(*models, prompts, sr, steps=3)
    rng = np.random.default_rng(1)
    for tick in range(2):
        block = torch.from_numpy(np.stack([_voice(rng, a.plan["block_in"], sr) for _ in range(2)])).cuda()
        torch.manual_seed(100 + tick)
        got = a.push(block)
        torch.manual_seed(100 + tick)
        xs = [torch.randn((1, 100, a.plan["T"]), device="cuda") for _ in range(2)]
        want = b.push(block, x_T=xs)
        assert got.device == block.device
        assert torch.equal(got, want) and torch.equal(a.seg, b.seg), f"tick {tick}: the default x_T is not per-slot randn in slot order"
