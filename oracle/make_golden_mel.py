"""Write tests/golden/frontend_mel.pt: the reference's prompt-mel recipe (inference/infer_tool.py:170-181) run literally with
torchaudio transforms, in fp32 (as the reference runs it) and fp64 (Resample(..., dtype=torch.float64),
MelSpectrogram(...).double()), on the reference's own dataset/1/1.wav and dataset/2/2.wav (44.1 kHz) and on seeded synthetic
signals at 16 000, 22 050, 24 000 and 48 000 Hz.  Every input is stored as int16 samples (x = pcm / 32768, as torchaudio reads
16-bit PCM).

The file stays small: oracle/mel_oracle.py reproduces torchaudio's runs (asserted here on every full output: fp64 to 1e-12, fp32
bit for bit), so the tests rebuild the full outputs from the oracle, and the fixture keeps what pins it - per case the lengths,
the recipe's own fp32-vs-fp64 errors e_ref (from the full outputs), and torchaudio's values at two frames of the mel and at a
strided sample of the resampled signal (pin_frames / pin_samples, in fp64 and fp32); torchaudio's phase tables and filterbank are
stored as the nonzero span of each row (sparse_rows / dense_rows, bit-exact).

    python oracle/make_golden_mel.py        (reference tree from $NS2VC_REFERENCE, as the other generators; needs torchaudio)
"""
from __future__ import annotations

import math
import os
import sys
import wave

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import mel_oracle  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "frontend_mel.pt")
RATE_PAIRS = [(16000, 24000), (22050, 24000), (48000, 24000), (44100, 24000), (44100, 16000)]
SYNTH_RATES = [16000, 22050, 24000, 48000]


def read_wav_int16(path: str):
    with wave.open(path, "rb") as w:
        assert w.getsampwidth() == 2 and w.getnchannels() == 1, path
        sr = w.getframerate()
        pcm = torch.frombuffer(bytearray(w.readframes(w.getnframes())), dtype=torch.int16).clone()
    return pcm, sr


def chirp(sr: int, seconds: float, seed: int) -> torch.Tensor:
    """A 60 Hz -> 0.45 sr log chirp with light noise, and an exact-silence stretch over its middle fifth."""
    g = torch.Generator().manual_seed(seed)
    n = int(sr * seconds)
    t = torch.arange(n, dtype=torch.float64) / sr
    f0, f1 = 60.0, 0.45 * sr
    k = math.log(f1 / f0) / seconds
    x = 0.5 * torch.sin(2 * math.pi * f0 * (torch.exp(k * t) - 1) / k) + 0.01 * torch.randn(n, generator=g, dtype=torch.float64)
    x[2 * n // 5: 3 * n // 5] = 0.0
    return x.float()


def pin_frames(F: int) -> torch.Tensor:
    """Mel frames whose torchaudio values the fixture keeps: the middle one and the last (where the reflect padding acts)."""
    return torch.tensor(sorted({F // 2, F - 1}))


def pin_samples(n24: int) -> torch.Tensor:
    """Resampled samples whose torchaudio values the fixture keeps (a stride over the signal and its last three)."""
    return torch.unique(torch.cat([torch.arange(0, n24, max(1, n24 // 61)), torch.arange(max(0, n24 - 3), n24)]))


def to_pcm(x: torch.Tensor) -> torch.Tensor:
    return torch.round(x * 32768.0).clamp(-32768, 32767).to(torch.int16)


def sparse_rows(m: torch.Tensor) -> dict:
    """A 2-D fp32 table as the span [first, last] of nonzero entries of each row; the zeros are `fill` (torchaudio's clamped sinc
    taps are all -0.0, the filterbank's zeros +0.0) except the flat indices `other_zeros`, which hold the other signed zero.
    dense_rows() rebuilds the table bit for bit."""
    lo, cnt, vals = [], [], []
    for row in m:
        nz = torch.nonzero(row).flatten()
        a, b = (int(nz[0]), int(nz[-1]) + 1) if len(nz) else (0, 0)
        lo.append(a)
        cnt.append(b - a)
        vals.append(row[a:b])
    zeros = m[m == 0]
    fill = -0.0 if 2 * int(torch.signbit(zeros).sum()) > len(zeros) else 0.0      # the more frequent signed zero
    flat = m.contiguous().view(-1)
    other = torch.nonzero((flat == 0) & (flat.view(torch.int32) != torch.tensor([fill]).view(torch.int32))).flatten()
    sp = dict(shape=tuple(m.shape), lo=torch.tensor(lo, dtype=torch.int32), count=torch.tensor(cnt, dtype=torch.int32),
              values=torch.cat(vals).clone(), fill=fill, other_zeros=other.to(torch.int32))
    assert torch.equal(dense_rows(sp).view(torch.int32), m.contiguous().view(torch.int32))
    return sp


def dense_rows(sp: dict) -> torch.Tensor:
    out = torch.full(sp["shape"], sp["fill"], dtype=torch.float32)
    off = 0
    for r, (a, n) in enumerate(zip(sp["lo"].tolist(), sp["count"].tolist())):
        out[r, a:a + n] = sp["values"][off:off + n]
        off += n
    idx = sp["other_zeros"].long()
    out.view(-1)[idx] = -out.view(-1)[idx]
    return out


def input_length_for(sr: int, n24: int) -> int:
    """Smallest input length at sr whose resampled length is n24, or 0 when no input length gives it (16 kHz: ceil(1.5 n))."""
    n = max(1, int(n24 * sr / 24000) - 4)
    while mel_oracle.out_length(sr, 24000, n) < n24:
        n += 1
    return n if mel_oracle.out_length(sr, 24000, n) == n24 else 0


def edge_lengths(sr: int):
    """24 kHz lengths 513 (the shortest the reflect padding takes), 768 (a multiple of the hop) and the first reachable
    k * 256 + 255, k >= 4 (one sample short of the next frame) -> input lengths at sr."""
    out = [("513", input_length_for(sr, 513)), ("768", input_length_for(sr, 768))]
    k = 4
    while not input_length_for(sr, k * 256 + 255):
        k += 1
    out.append((str(k * 256 + 255), input_length_for(sr, k * 256 + 255)))
    assert all(n for _, n in out), (sr, out)
    return out


def recipe(torchaudio, wav: torch.Tensor, sr: int, dtype: torch.dtype):
    """inference/infer_tool.py:170-181 with the transforms in dtype."""
    x = wav.to(dtype)[None]
    if dtype == torch.float64:
        wav24 = torchaudio.transforms.Resample(sr, 24000, dtype=torch.float64)(x)
        spec = torchaudio.transforms.MelSpectrogram(sample_rate=24000, n_fft=1024, hop_length=256, n_mels=100, center=True,
                                                    power=1).double()(wav24)
    else:
        wav24 = torchaudio.transforms.Resample(sr, 24000)(x)
        spec = torchaudio.transforms.MelSpectrogram(sample_rate=24000, n_fft=1024, hop_length=256, n_mels=100, center=True,
                                                    power=1)(wav24)
    return wav24[0], torch.log(torch.clip(spec, min=1e-7))[0]


def main(ref_root: str) -> None:
    import torchaudio
    torch.manual_seed(0)
    cases = {}

    def add(name, pcm, sr):
        wav = pcm.float() / 32768.0
        r32, m32 = recipe(torchaudio, wav, sr, torch.float32)
        r64, m64 = recipe(torchaudio, wav, sr, torch.float64)
        o64 = mel_oracle.log_mel(wav, sr, torch.float64)
        o_r64 = mel_oracle.resample(wav, sr, 24000, torch.float64)
        assert o64.shape == m64.shape and o_r64.shape == r64.shape, name
        e_res, e_mel = (o_r64 - r64).abs().max().item(), (o64 - m64).abs().max().item()
        assert e_res < 1e-12 and e_mel < 1e-12, (name, e_res, e_mel)
        assert torch.equal(mel_oracle.resample(wav, sr, 24000, torch.float32), r32) and torch.equal(mel_oracle.log_mel(wav, sr, torch.float32), m32), name
        F, n24 = m64.shape[-1], r64.shape[-1]
        fr, sm = pin_frames(F), pin_samples(n24)
        c = dict(sr=sr, n=wav.shape[-1], pcm_int16=pcm, len24=n24, frames=F,
                 e_ref_resample=(r32.double() - r64).abs().max().item(), e_ref=(m32.double() - m64).abs().max().item(),
                 pin_mel_f64=m64[:, fr].clone(), pin_mel_f32=m32[:, fr].clone(), pin_wav24_f64=r64[sm].clone(), pin_wav24_f32=r32[sm].clone())
        cases[name] = c
        print(f"{name:>16}: sr {sr} n {c['n']} -> {c['len24']} samples, {c['frames']} frames; e_ref_resample {c['e_ref_resample']:.2e} "
              f"e_ref {c['e_ref']:.2e}; oracle-vs-torchaudio fp64 {e_res:.1e} / {e_mel:.1e}, fp32 bit-identical")

    for i in (1, 2):
        pcm, sr = read_wav_int16(os.path.join(ref_root, "dataset", str(i), f"{i}.wav"))
        add(f"{i}.wav", pcm, sr)
    for j, sr in enumerate(SYNTH_RATES):
        add(f"chirp_{sr}", to_pcm(chirp(sr, 0.15, seed=100 + j)), sr)
        for tag, n in edge_lengths(sr):
            add(f"edge{tag}_{sr}", to_pcm(chirp(sr, n / sr + 1e-9, seed=200 + j)[:n]), sr)
    tables = {}
    for o, n in RATE_PAIRS:
        r = torchaudio.transforms.Resample(o, n)
        tables[f"{o}_{n}"] = dict(kernel=sparse_rows(r.kernel.reshape(r.kernel.shape[0], -1)), width=r.width)
    fb = torchaudio.functional.melscale_fbanks(513, 0.0, 12000.0, 100, 24000, norm=None, mel_scale="htk")
    torch.save(dict(cases=cases, tables=tables, fbanks_t=sparse_rows(fb.t()), torchaudio_version=torchaudio.__version__), OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main(os.environ.get("NS2VC_REFERENCE", "/root/reference"))
