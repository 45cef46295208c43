"""Throughput of the content encoder (``content.ContentVec.extract``, ContentVec's configuration with synthetic ``trained_like``
weights).

    python scripts/content_bench.py [--iters 20] [--warmup 3] [--out results/content_bench.json]

(a) ``extract`` at B=1 for 3 s and 10 s of 16 kHz audio, and at B=8 for 10 s: ms per call, audio-seconds per second, launches
    per call and algorithmic TFLOP/s (``gflop`` below: the work from shapes, the 3xBF16 split not counted).
(b) the 16-slice list of scripts/ragged_bench.py (lengths uniform in [150, 1000] frames of 256 samples at 24 kHz, seed 0, here
    converted to 16 kHz samples): one ``extract`` per slice at B = 1 against ``api.content_utterances(max_batch=8)``.
(c) transformers' eager fp32 ``HubertModel`` at the same configuration on the same GPU, when transformers is importable: a
    stand-in for fairseq's eager HubertModel, NOT fairseq.  Its TF32 flags are recorded.

Timing: CUDA events around the timed calls after ``--warmup`` untimed passes, the mean of ``--iters`` calls.  Prints the card's
name and power limit with the numbers.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ns2vc_b200 import api  # noqa: E402
from ns2vc_b200.content import CONTENTVEC, CONV_LAYERS, ContentVec  # noqa: E402
from ns2vc_b200.synth import make_contentvec_state_dict  # noqa: E402
from scripts.ragged_bench import card  # noqa: E402

SR = 16000


def gflop(n: int, c=CONTENTVEC) -> dict:
    """Algorithmic GFLOP (2 per multiply-add) of one utterance of n samples, by part"""
    C0, D, FF, K, G = c["conv_dim"], c["embed_dim"], c["ffn_dim"], c["pos_conv_kernel"], c["pos_conv_groups"]
    conv, t = 0, n
    for l, (k, s) in enumerate(CONV_LAYERS):
        t = (t - k) // s + 1
        conv += 2 * t * C0 * (1 if l == 0 else C0) * k
    T = t
    return {"conv_feature_encoder": conv / 1e9,
            "layers_without_attention": 2 * c["num_layers"] * T * (4 * D * D + 2 * D * FF) / 1e9,
            "attention": 2 * c["num_layers"] * 2 * T * T * D / 1e9,
            "positional_conv": 2 * T * D * (D // G) * K / 1e9,
            "projections": 2 * T * (C0 * D + D * c["final_dim"]) / 1e9}


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b) / 1e3 / iters


def transformers_hubert():
    try:
        import transformers
    except ImportError:
        return None
    c = CONTENTVEC
    hc = transformers.HubertConfig(
        hidden_size=c["embed_dim"], num_hidden_layers=c["num_layers"], num_attention_heads=c["num_heads"], intermediate_size=c["ffn_dim"],
        conv_dim=(c["conv_dim"],) * 7, conv_stride=tuple(s for _, s in CONV_LAYERS), conv_kernel=tuple(k for k, _ in CONV_LAYERS),
        num_conv_pos_embeddings=c["pos_conv_kernel"], num_conv_pos_embedding_groups=c["pos_conv_groups"], feat_extract_norm="group",
        conv_bias=False, do_stable_layer_norm=False, hidden_act="gelu", apply_spec_augment=False)
    try:
        m = transformers.HubertModel(hc, attn_implementation="eager")
    except TypeError:
        m = transformers.HubertModel(hc)
    proj = torch.nn.Linear(c["embed_dim"], c["final_dim"])
    return m.cuda().eval(), proj.cuda().eval()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("content_bench needs a CUDA device")
    sd = make_contentvec_state_dict(0, "trained_like")
    m = ContentVec.from_state_dict(sd).cuda().eval()
    res = {"card": card(), "gflop_per_10s": {k: round(v, 2) for k, v in gflop(10 * SR).items()}, "extract": {}, "slices": {},
           "transformers_fp32_eager_stand_in": "not measured"}
    res["gflop_per_10s"]["total"] = round(sum(gflop(10 * SR).values()), 1)
    print("card", res["card"], "GFLOP per 10 s", res["gflop_per_10s"], flush=True)
    torch.set_grad_enabled(False)
    g = torch.Generator().manual_seed(1)
    for B, sec_audio in ((1, 3), (1, 10), (8, 10)):
        n = sec_audio * SR
        wav = (0.1 * torch.randn((B, n), generator=g)).cuda()
        _, sec = timed(lambda: m.extract(wav), args.iters, args.warmup)
        row = {"ms": round(sec * 1e3, 3), "audio_seconds_per_second": round(B * sec_audio / sec, 1),
               "tflops": round(B * sum(gflop(n).values()) / sec / 1e3, 1), "launches": m.launch_count()}
        res["extract"][f"B={B},{sec_audio}s"] = row
        print("extract", B, sec_audio, row, flush=True)

    gs = torch.Generator().manual_seed(0)
    frames = torch.randint(150, 1001, (16,), generator=gs).tolist()
    lengths = [f * 256 * SR // 24000 for f in frames]
    wavs = [(0.1 * torch.randn(n, generator=gs)).cuda() for n in lengths]
    audio_s = sum(lengths) / SR
    modes = [("B=1", lambda: [m.extract(w[None])[0][0] for w in wavs]),
             ("content_utterances(max_batch=8)", lambda: api.content_utterances(m, wavs, max_batch=8))]
    ref = None
    for name, fn in modes:
        out, sec = timed(fn, max(1, args.iters // 4), args.warmup)
        row = {"ms": round(sec * 1e3, 3), "audio_seconds_per_second": round(audio_s / sec, 1)}
        if ref is None:
            ref = out
        else:
            row["speedup_vs_B1"] = round(res["slices"]["B=1"]["ms"] / row["ms"], 2)
            row["bit_identical_to_B1"] = sum(int(torch.equal(a.t(), r)) for a, r in zip(out, ref))
        res["slices"][name] = row
        print("slices", name, row, flush=True)

    th = transformers_hubert()
    if th is not None:
        hub, proj = th
        flags = {"matmul.allow_tf32": torch.backends.cuda.matmul.allow_tf32, "cudnn.allow_tf32": torch.backends.cudnn.allow_tf32}
        st = {"what": "transformers HubertModel, eager fp32, same configuration (a stand-in for fairseq, NOT fairseq)", "tf32_flags": flags}
        wav10 = (0.1 * torch.randn((1, 10 * SR), generator=g)).cuda()
        _, sec = timed(lambda: proj(hub(wav10).last_hidden_state), max(1, args.iters // 4), 1)
        st["B=1,10s"] = {"ms": round(sec * 1e3, 3), "audio_seconds_per_second": round(10 / sec, 1)}
        _, sec = timed(lambda: [proj(hub(w[None]).last_hidden_state) for w in wavs], max(1, args.iters // 4), 1)
        st["slices B=1"] = {"ms": round(sec * 1e3, 3), "audio_seconds_per_second": round(audio_s / sec, 1)}
        res["transformers_fp32_eager_stand_in"] = st
        print("stand-in", st, flush=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
