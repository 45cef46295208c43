"""Write tests/golden/slicer.pt: the reference's silence slicer (inference/slicer.py, imported unmodified) run on synthetic
16-bit signals.  librosa is not needed: a stub ``librosa`` module supplies only what slicer.py calls, ``feature.rms`` (the
numpy restatement in oracle/slicer_oracle.py) and ``to_mono``.  ``chunks2audio`` reads its file through ``torchaudio.load``,
which is pointed at the case's samples.

Per case the fixture keeps the samples (int16, zlib-compressed; x = pcm / 32768 as a 16-bit WAV reads), the rate, the
threshold and min_length, hop and win, the rms frames, ``Slicer.slice``'s chunk dict and ``chunks2audio``'s list as
(is_silence, start, stop) spans of the samples.  The cases cover 16, 22.05, 44.1, 48 and 11.025 kHz, leading and trailing
silence, gaps shorter than min_interval, silences up to max_sil_kept, between it and twice it and longer, digital zeros (rms
ties for argmin), a file of no more than min_length samples and a file shorter than win.

    NS2VC_REFERENCE=<reference tree> python oracle/make_golden_slicer.py
"""
from __future__ import annotations

import importlib.util
import os
import sys
import types
import zlib

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import slicer_oracle  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "slicer.pt")


def _voice(rng, sr, dur, period, amp):
    """A voiced stand-in that compresses: one random period of ``period`` samples, repeated."""
    cycle = amp * rng.standard_normal(period)
    return np.tile(cycle, int(dur * sr) // period + 1)[:int(dur * sr)]


def _dense(rng, sr, dur, amp):
    return amp * rng.standard_normal(int(dur * sr))


def _noise(rng, sr, dur, db):
    return 10 ** (db / 20) * rng.standard_normal(int(dur * sr))


def _zeros(rng, sr, dur):
    return np.zeros(int(dur * sr))


def cases():
    rng = np.random.default_rng(2026)
    V, D, N, Z = _voice, _dense, _noise, _zeros
    spec = [
        # name, sr, threshold dB, min_length ms, segments
        ("16k_gaps_trailing", 16000, -40, 500,
         [(Z, 0.7), (V, 1.3, 89, 0.3), (N, 0.2, -62), (V, 1.1, 73, 0.25), (N, 1.5, -66), (V, 0.9, 101, 0.2), (Z, 0.8)]),
        ("22k_long_leading", 22050, -30, 500, [(N, 5.2, -66), (V, 1.5, 97, 0.3), (Z, 0.6), (V, 1.0, 61, 0.2)]),
        ("44k_short_gaps", 44100, -40, 500, [(V, 0.9, 211, 0.3), (N, 0.45, -70), (V, 0.8, 149, 0.25), (Z, 0.35)]),
        ("48k_zeros_ties", 48000, -40, 500, [(Z, 0.25), (V, 1.0, 307, 0.2), (Z, 0.5), (V, 0.7, 113, 0.3), (N, 0.1, -65)]),
        ("11k_cli_long_silences", 11025, -40, 5000,
         [(V, 5.5, 83, 0.2), (N, 7.0, -66), (V, 5.2, 59, 0.15), (Z, 11.0), (V, 5.1, 71, 0.2), (N, 0.2, -70)]),
        ("11k_min_len_300", 11025, -30, 300, [(V, 0.5, 67, 0.3), (Z, 0.45), (V, 0.4, 53, 0.3), (N, 0.29, -62)]),
        ("16k_at_most_min_length", 16000, -40, 5000, [(D, 0.015, 0.3)]),
        ("44k_shorter_than_win", 44100, -40, 5000, [(D, 0.068, 0.3)]),
    ]
    out = []
    for name, sr, db, min_len, segs in spec:
        x = np.concatenate([s[0](rng, sr, *s[1:]) for s in segs])
        pcm = np.clip(np.round(x * 32768), -32768, 32767).astype(np.int16)
        out.append(dict(name=name, sr=sr, db=db, min_len=min_len, pcm=pcm))
    return out


def samples(case) -> np.ndarray:
    """The fixture's float32 samples of one case."""
    return np.frombuffer(zlib.decompress(case["pcm_zlib"]), dtype=np.int16).astype(np.float32) / np.float32(32768)


def load_reference_slicer(ref: str):
    librosa = types.ModuleType("librosa")
    librosa.feature = types.SimpleNamespace(rms=lambda y, frame_length, hop_length: slicer_oracle.rms(y, frame_length, hop_length))
    librosa.to_mono = lambda y: np.mean(y, axis=0)
    sys.modules["librosa"] = librosa
    spec = importlib.util.spec_from_file_location("reference_slicer", os.path.join(ref, "inference", "slicer.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    ref = os.environ.get("NS2VC_REFERENCE")
    if not ref:
        raise SystemExit("set NS2VC_REFERENCE to the reference tree")
    mod = load_reference_slicer(ref)
    fixture = []
    for c in cases():
        y = c["pcm"].astype(np.float32) / np.float32(32768)
        p = slicer_oracle.slicer_params(c["sr"], c["db"], c["min_len"])
        sl = mod.Slicer(sr=c["sr"], threshold=c["db"], min_length=c["min_len"])
        assert (sl.hop_size, sl.win_size) == (p["hop"], p["win"])
        chunks = sl.slice(y)
        audio = torch.from_numpy(y.copy())
        mod.torchaudio = types.SimpleNamespace(load=lambda path, a=audio, sr=c["sr"]: (a.unsqueeze(0), sr))
        pieces, sr = mod.chunks2audio("<samples>", chunks)
        spans = []
        for tag, arr in pieces:      # views of one array (chunks2audio's channel mean, a copy of the samples)
            root = arr
            while root.base is not None and isinstance(root.base, np.ndarray):
                root = root.base
            start = (arr.__array_interface__["data"][0] - root.__array_interface__["data"][0]) // 4
            assert np.array_equal(arr, y[start:start + arr.shape[0]])
            spans.append((bool(tag), int(start), int(start + arr.shape[0])))
        r = slicer_oracle.rms(y, p["win"], p["hop"])[0]
        fixture.append(dict(name=c["name"], sr=c["sr"], db=c["db"], min_len=c["min_len"], n=int(y.shape[0]), hop=p["hop"], win=p["win"],
                            pcm_zlib=zlib.compress(c["pcm"].tobytes(), 9), rms=torch.from_numpy(r.copy()), chunks=chunks, chunks2audio=spans))
        print(f"{c['name']:24s} sr={c['sr']} n={y.shape[0]} frames={r.shape[0]} chunks={len(chunks)} "
              f"{[(v['slice'], v['split_time']) for v in chunks.values()]}")
    torch.save(fixture, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main()
