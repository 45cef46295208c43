"""Write tests/golden/preprocess.pt: the reference's ``process_one`` (preprocess.py:26-60) run on the CPU for eight short
waveforms at 16, 22.05, 24, 44.1 and 48 kHz (two stereo, one at the shortest length the GPU path accepts), with torchaudio's
transforms as the reference calls them and ``oracle/content_oracle.py`` in fp32 standing in for fairseq's HuBERT at a small
seeded ContentVec configuration (``synth.make_contentvec_state_dict``; 256 output channels, as the condition encoders take).

Per item it stores the input as int16 PCM (x = pcm / 32768, as torchaudio reads 16-bit files), the reference's fp32 outputs
``wav16k``, ``wav24k``, ``soft`` [1, 256, U] and ``spec`` [1, 100, N24 // 256 + 1], ``frames`` = N24 // 256, and the recipe's
own fp32 errors against the same recipe in fp64 (torchaudio ``Resample(dtype=float64)`` / ``MelSpectrogram().double()``, the
content oracle in fp64): ``e_ref_16k`` / ``e_ref_24k`` (max |.|) and ``e_ref_mel``, the bounds' units in the tests.  Before writing
it asserts that ``oracle/mel_oracle.py`` reproduces torchaudio's fp64 outputs (1e-12), so the tests can rebuild the fp64 truths.

It also stores the reference's own ``utils.resize_f0`` (imported from the reference tree, librosa stubbed) on stub f0 arrays
with unvoiced runs, and the output names of a few paths.  The names restate ``process_one``'s three replacements here, because
they are inline in ``process_one``, which needs torchaudio's file I/O and a HuBERT.

    NS2VC_REFERENCE=<reference tree> python oracle/make_golden_preprocess.py        (needs torchaudio)
"""
from __future__ import annotations

import math
import os
import sys
from unittest.mock import MagicMock

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, REPO)
from ns2vc_b200.synth import CONTENTVEC_SMALL, make_contentvec_state_dict, state_dict_checksum  # noqa: E402
from oracle import content_oracle, mel_oracle  # noqa: E402

OUT = os.path.join(REPO, "tests", "golden", "preprocess.pt")
CV_CFG = dict(CONTENTVEC_SMALL, final_dim=256)
CV_SEED, CV_REGIME = 5, "trained_like"
# (rate, channels, samples): 1100 samples at 44.1 kHz are the fewest that give ContentVec's 400 samples at 16 kHz
ITEMS = [(16000, 1, 3000), (22050, 2, 4000), (24000, 1, 4800), (44100, 1, 9000), (48000, 2, 7200), (44100, 1, 1100),
         (22050, 1, 5513), (48000, 1, 5760)]
F0_CASES = [(50, 37), (20, 64), (33, 33), (7, 1), (128, 95)]
PATHS = [("dataset/spk1/a.wav", "dataset"), ("dataset/spk1/b.flac", "dataset"), ("corpus/x.mp3/c.mp3", "corpus"),
         ("data/v1.wav/d.wav", "data"), ("/abs/data/spk/e.flac", "/abs/data")]


def signal(sr: int, channels: int, n: int, seed: int) -> torch.Tensor:
    """int16 PCM [channels, n]: a log chirp per channel (different start pitch), light noise, a DC offset, a silent stretch."""
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(n, dtype=torch.float64) / sr
    out = []
    for c in range(channels):
        f0, f1 = 90.0 + 70.0 * c + 10.0 * seed, 0.4 * sr
        dur = max(n / sr, 1e-3)
        k = math.log(f1 / f0) / dur
        x = 0.4 * torch.sin(2 * math.pi * f0 * (torch.exp(k * t) - 1) / k) + 0.02 * torch.randn(n, generator=g, dtype=torch.float64)
        x += 0.03 * (c + 1)
        x[n // 2: n // 2 + n // 8] = 0.0
        out.append(torch.round(x * 32767).clamp(-32768, 32767).to(torch.int16))
    return torch.stack(out)


def output_names(filename: str, in_dir: str):
    wav = filename.replace(in_dir, in_dir + "_processed").replace('.mp3', '.wav').replace('.flac', '.wav')
    return dict(wav=wav, soft=wav + ".soft.pt", f0=wav + ".f0.npy", spec=wav.replace(".wav", ".spec.pt"))


def stub_f0(n: int, seed: int) -> np.ndarray:
    """A pitch track with unvoiced (0) runs at the start, in the middle and at the end, rounded to 0.1 Hz as DIO's output is."""
    rng = np.random.default_rng(seed)
    f0 = np.round(120 + 40 * np.sin(np.arange(n) / 5.0) + rng.normal(0, 3, n), 1)
    f0[: max(1, n // 10)] = 0
    f0[n // 2: n // 2 + n // 6] = 0
    if n > 4:
        f0[-2:] = 0
    return f0


def main(ref: str) -> None:
    import torchaudio.transforms as T
    sys.path.insert(0, ref)
    sys.modules.setdefault("librosa", MagicMock())
    import utils as ref_utils

    sd = make_contentvec_state_dict(CV_SEED, CV_REGIME, **CV_CFG)
    heads = CV_CFG["num_heads"]
    items = []
    for k, (sr, C, n) in enumerate(ITEMS):
        pcm = signal(sr, C, n, k)
        wav = pcm.float() / 32768.0
        if wav.shape[0] > 1:                                                   # process_one, step by step
            wav = wav.mean(dim=0, keepdim=True)
        wav16k = T.Resample(sr, 16000)(wav)
        wav24k = T.Resample(sr, 24000)(wav)
        spec_tf = T.MelSpectrogram(sample_rate=24000, n_fft=1024, hop_length=256, n_mels=100, center=True, power=1)
        spec = torch.log(torch.clip(spec_tf(wav24k), min=1e-7))
        with torch.no_grad():
            soft = content_oracle.extract(sd, wav16k, heads, dtype=torch.float32).transpose(1, 2)
            w64 = wav.double()
            w16_64 = T.Resample(sr, 16000, dtype=torch.float64)(w64)
            w24_64 = T.Resample(sr, 24000, dtype=torch.float64)(w64)
            spec64 = torch.log(torch.clip(spec_tf.double()(w24_64), min=1e-7))
            soft64 = content_oracle.extract(sd, w16_64, heads).transpose(1, 2)
        assert (mel_oracle.resample(wav[0], sr, 16000) - w16_64[0]).abs().max().item() <= 1e-12, k
        assert (mel_oracle.resample(wav[0], sr, 24000) - w24_64[0]).abs().max().item() <= 1e-12, k
        assert (mel_oracle.log_mel(wav[0], sr) - spec64[0]).abs().max().item() <= 1e-12, k
        frames = wav24k.shape[-1] // 256
        assert spec.shape == (1, 100, frames + 1) and soft.shape == (1, 256, content_oracle.num_frames(wav16k.shape[-1])), k
        items.append(dict(sr=sr, pcm_int16=pcm, wav16k=wav16k, wav24k=wav24k, soft=soft.float().contiguous(), spec=spec,
                          frames=frames, e_ref_16k=(wav16k.double() - w16_64).abs().max().item(),
                          e_ref_24k=(wav24k.double() - w24_64).abs().max().item(),
                          e_ref_mel=(spec.double() - spec64).abs().max().item(),
                          e_ref_soft=(soft.double() - soft64).abs().max().item()))
        print(f"item {k}: {sr} Hz x{C}, {n} samples -> N16 {wav16k.shape[-1]}, N24 {wav24k.shape[-1]}, U {soft.shape[-1]}, "
              f"frames {frames}")
    f0 = []
    for s, (n, target) in enumerate(F0_CASES):
        x = stub_f0(n, s)
        f0.append(dict(f0=x, target_len=target, resized=np.asarray(ref_utils.resize_f0(x, target))))
    names = [dict(filename=f, in_dir=d, **output_names(f, d)) for f, d in PATHS]
    torch.save(dict(cv_cfg=CV_CFG, cv_seed=CV_SEED, cv_regime=CV_REGIME, cv_checksum=state_dict_checksum(sd), items=items,
                    resize_f0=f0, names=names), OUT)
    print(f"wrote {OUT}")


if __name__ == "__main__":
    main(os.environ.get("NS2VC_REFERENCE", "/root/reference"))
