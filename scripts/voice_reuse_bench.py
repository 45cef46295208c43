"""What encoding each target voice once saves: the condition encoders split into a voice half (``Pre_model.encode_voices``) and
a content half (``Pre_model.infer_content``), against the fused ragged encoders run on every row.

    python scripts/voice_reuse_bench.py [--steps 30] [--reps 5] [--out results/voice_reuse_bench.json]

Full-size models with synthetic weights (ContentVec, the shipped condition encoders, the 66 M-parameter denoiser, the
vocos-mel-24khz vocoder shapes), UniPC.  Three measurements, each with the card's name, power limit and maximum SM clock:

- encoder stage: 8 items of 500 frames with one voice of 300 frames, ``Pre_model.infer(per_utterance=True)`` on the batch
  against ``encode_voices`` once plus ``infer_content``; CUDA events, median of ``--reps`` after a warm-up;
- ``convert_files``: 2 files of ~20 s against V = 1, 2 and 4 voices; wall time (host clock around a synchronised call),
  the rows ContentVec extracted and the rows the prompt encoder ran;
- ``StreamConverter``: time per tick (CUDA events, median over ``--reps`` ticks after two warm-up ticks) with 1 and 8
  streams and prompts of ~3 s and ~10 s.

The ``fused`` rows run the same calls with ``convert.encode_front`` replaced by the fused encoders on every row, as the
conversion ran before voices were reused: every row through the resampling, ContentVec and all three encoders.  Needs a
CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from convert_bench import PRE_CFG, card  # noqa: E402
from ns2vc_b200 import api, convert, frontend, stream  # noqa: E402
from ns2vc_b200.arch import ns2vc_denoiser_config  # noqa: E402
from ns2vc_b200.content import ContentVec  # noqa: E402
from ns2vc_b200.pre_model import Pre_model, Voice  # noqa: E402
from ns2vc_b200.synth import make_contentvec_state_dict, make_pre_state_dict, make_state_dict, make_vocos_state_dict  # noqa: E402
from ns2vc_b200.unet import UNet1DConditionModel  # noqa: E402
from ns2vc_b200.vocoder import Vocos  # noqa: E402

SR = 44100
MEL_OF = {}          # id(Voice) -> the mel it was encoded from, for the fused rows


def recording(encode):
    def run(pre_model, mels, max_batch=8):
        voices = encode(pre_model, mels, max_batch)
        MEL_OF.update({id(v): m for v, m in zip(voices, mels)})
        return voices
    return run


def fused_front(content_model, pre_model, wavs, sr, prompts, plans, dev, cache=None):
    """``convert.encode_front`` with the fused ragged encoders on every row, as before voices were reused (a ``Voice`` prompt
    is replaced by its mel)."""
    B = len(wavs)
    n = [int(w.shape[0]) for w in wavs]
    prompts = [MEL_OF[id(p)] if isinstance(p, Voice) else p for p in prompts]
    tl, sl = [p["T"] for p in plans], [int(p.shape[1]) for p in prompts]
    wav = torch.zeros((B, max(n)), dtype=torch.float32, device=dev)
    for j, w in enumerate(wavs):
        wav[j, :n[j]] = w.to(dev, torch.float32)
    w24, _ = frontend.resample(wav, sr, convert.TARGET_SR, torch.tensor(n))
    w16, _ = frontend.resample(w24, convert.TARGET_SR, convert.CONTENT_SR, torch.tensor([p["n24"] for p in plans]))
    units_all, _ = content_model.extract(w16, torch.tensor([p["n16"] for p in plans]))
    units = [units_all[j, :p["units"]].t() for j, p in enumerate(plans)]
    cs = [frontend.repeat_expand_2d(u, t) for u, t in zip(units, tl)]
    c = torch.zeros((B, units_all.shape[2], max(tl)), dtype=torch.float32, device=dev)
    refer = torch.zeros((B, 100, max(sl)), dtype=torch.float32, device=dev)
    for j in range(B):
        c[j, :, :tl[j]] = cs[j]
        refer[j, :, :sl[j]] = prompts[j].to(dev)
    content, prompt = pre_model.infer((c, refer, None, None, None, torch.tensor(tl), torch.tensor(sl), None), per_utterance=True)
    return dict(units=units, c=cs, tl=tl, content=content, prompt=prompt)


class Rows:
    """Counts the rows of every call of ``obj.name`` (the first dim of its first argument, or of that argument's first tensor)."""

    def __init__(self, obj, name):
        self.n, fn = 0, getattr(obj, name)

        def call(x, *a, **k):
            self.n += int((x[0] if isinstance(x, tuple) else x).shape[0])
            return fn(x, *a, **k)
        setattr(obj, name, call)


def signal(n, g):
    t = torch.arange(n) / SR
    f0 = 100 + 200 * torch.rand(1, generator=g)
    return (0.3 * torch.sin(2 * torch.pi * f0 * t) * (1 + 0.5 * torch.sin(2 * torch.pi * 3 * t)) + 0.02 * torch.randn(n, generator=g)).float()


def events(fn, reps):
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("voice_reuse_bench needs a CUDA device")
    dev = torch.device("cuda")
    res = dict(card=card(), steps=args.steps)
    print(res["card"], flush=True)
    cfg = ns2vc_denoiser_config()
    unet = UNet1DConditionModel(in_channels=cfg.in_channels, out_channels=cfg.out_channels, block_out_channels=cfg.block_out_channels,
                                layers_per_block=list(cfg.layers_per_block), norm_num_groups=cfg.norm_num_groups,
                                cross_attention_dim=cfg.cross_attention_dim, attention_head_dim=cfg.num_heads,
                                addition_embed_type=cfg.addition_embed_type, addition_embed_type_num_heads=cfg.addition_embed_type_num_heads,
                                resnet_time_scale_shift=cfg.resnet_time_scale_shift)
    unet.load_state_dict(make_state_dict(cfg, 0))
    unet = unet.to(dev).eval()
    cv = ContentVec.from_state_dict(make_contentvec_state_dict(0, "trained_like")).to(dev)
    pre = Pre_model(PRE_CFG)
    pre.load_state_dict(make_pre_state_dict(PRE_CFG, 0))
    pre = pre.to(dev).eval()
    voc = Vocos.from_state_dict(make_vocos_state_dict(0, "trained_like")).to(dev)
    models = (cv, pre, unet, voc)
    convert.encode_voices = recording(convert.encode_voices)
    stream.encode_voices = recording(stream.encode_voices)
    g = torch.Generator().manual_seed(0)

    def mel(seconds):
        return frontend.log_mel_spectrogram((0.2 * torch.randn(int(seconds * 24000), generator=g)).float().to(dev), 24000)[0]

    # ---- encoder stage: 8 items, one voice
    B, T, S = 8, 500, 300
    c = torch.randn((B, 256, T), generator=g).to(dev)
    refer1 = (torch.randn((1, 100, S), generator=g) - 4).to(dev)
    lengths, rl1 = torch.tensor([T - 37 * j for j in range(B)]), torch.tensor([S])
    fused = lambda: pre.infer((c, refer1.expand(B, -1, -1), None, None, None, lengths, rl1.expand(B), None), per_utterance=True)

    def split():
        v = pre.encode_voices(refer1, rl1)[0]
        return pre.infer_content(c, lengths, [v] * B)
    fused(), split()
    same = torch.equal(fused()[0], split())
    v1 = pre.encode_voices(refer1, rl1)[0]
    res["encoders"] = dict(B=B, T=T, S=S, fused_ms=events(fused, args.reps), split_ms=events(split, args.reps),
                           content_only_ms=events(lambda: pre.infer_content(c, lengths, [v1] * B), args.reps), content_equal=same)
    print("encoders", res["encoders"], flush=True)

    # ---- convert_files: 2 files of ~20 s against V = 1, 2, 4 voices
    files = [(signal(int(20.3 * SR), g).numpy(), SR), (signal(int(19.6 * SR), g).numpy(), SR)]
    voices = [((0.2 * torch.randn(int(d * 24000), generator=g)).float(), 24000) for d in (3.0, 4.5, 2.5, 6.0)]
    ext, enc, fus = Rows(cv, "extract"), Rows(pre, "encode_voices"), Rows(pre, "infer")
    own_front = convert.encode_front
    res["convert_files"] = []
    for V in (1, 2, 4):
        for mode in ("split", "fused"):
            convert.encode_front = own_front if mode == "split" else fused_front
            run = lambda: convert.convert_files(*models, files, voices[:V], clip_seconds=0, steps=args.steps, max_batch=8)
            torch.manual_seed(1)
            run()                                           # warm-up: builds every shape of this run
            ext.n = enc.n = fus.n = 0
            torch.manual_seed(1)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = run()
            torch.cuda.synchronize()
            sec = time.perf_counter() - t0
            r = dict(V=V, mode=mode, seconds=sec, contentvec_rows=ext.n, voice_rows=enc.n, fused_encoder_rows=fus.n,
                     audio_s=sum(len(o) for f in out for o in f) / convert.TARGET_SR)
            if mode == "split":
                ref = out
            else:
                r["equal_to_split"] = all(np.array_equal(a, b) for fa, fb in zip(out, ref) for a, b in zip(fa, fb))
            res["convert_files"].append(r)
            print("convert_files", r, flush=True)
    convert.encode_front = own_front

    # ---- StreamConverter: time per tick
    res["stream"] = []
    mels = {3: mel(3.0), 10: mel(10.0)}
    for nstreams in (1, 8):
        for ps in (3, 10):
            for mode in ("split", "fused"):
                convert.encode_front = own_front if mode == "split" else fused_front
                sess = stream.StreamConverter(*models, [mels[ps]] * nstreams, 16000, steps=args.steps)
                blocks = [0.1 * torch.randn((nstreams, sess.plan["block_in"]), generator=g).to(dev) for _ in range(args.reps + 2)]
                it = iter(blocks)
                sess.push(next(it))
                sess.push(next(it))
                ms = events(lambda: sess.push(next(it)), args.reps)
                r = dict(streams=nstreams, prompt_s=ps, mode=mode, tick_ms=ms, block_ms=1000 * sess.plan["Nb"] / convert.TARGET_SR)
                res["stream"].append(r)
                print("stream", r, flush=True)
    convert.encode_front = own_front
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
