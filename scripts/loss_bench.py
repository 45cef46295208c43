"""Cost of the training objective under no_grad (``ns2vc_b200.loss``) per evaluated timestep, at the reference's training crop:
full-size synthetic models, B = 8, T = 400, S = 200.

    python scripts/loss_bench.py [--ks 1,4,16,64] [--shape 8x400x200] [--out results/loss_bench.json]

For each K, three ways to evaluate K timesteps of one batch, alternated within one timed loop:
  profile   one ``loss_profile`` call: encoders, prepare_cond, q_sample and the reduction once, K denoiser forwards
  calls     K ``diffusion_loss`` calls with a [B] ``t``: everything redone per timestep
  port      K passes of ``NaturalSpeech2.forward``'s body written out with torch ops around ``Pre_model.infer`` and the drop-in
            UNet's generic forward (what a port of the reference's loop does): encoders and conditioning redone per timestep
and, for the profile, where the time goes: encoders / prepare_cond / K forwards / q_sample + reduction.  The three are asserted
to agree on the losses (rtol 1e-3).  Timing: CUDA events after warm-up.  Prints the card's name, power limit and clocks with the
numbers.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ns2vc_b200 import coefs  # noqa: E402
from ns2vc_b200.api import sequence_mask  # noqa: E402
from ns2vc_b200.arch import ns2vc_denoiser_config  # noqa: E402
from ns2vc_b200.fused import get_session  # noqa: E402
from ns2vc_b200.loss import diffusion_loss, loss_profile, mse_rows, q_sample  # noqa: E402
from ns2vc_b200.pre_model import Pre_model  # noqa: E402
from ns2vc_b200.synth import make_pre_inputs, make_pre_state_dict, make_state_dict  # noqa: E402
from ns2vc_b200.unet import UNet1DConditionModel  # noqa: E402

PRE_CFG = {"phoneme_encoder": dict(in_channels=256, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2),
           "prompt_encoder": dict(in_channels=100, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2)}


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable: {e}"


def timed_ms(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


@torch.no_grad()
def port_loss(pre, unet, data, t, noise, buf):
    """NaturalSpeech2.forward's body (model.py:706-734) for one [B] t, with torch ops."""
    c, refer, _, spec, _, lengths, refer_lengths, _ = data
    B, _, T = spec.shape
    x_mask = sequence_mask(lengths, T).unsqueeze(1).to(spec.dtype)
    x_start = spec * x_mask
    content, prompt = pre.infer(data)
    noise = noise * x_mask
    ext = lambda a: a.gather(-1, t).reshape(B, 1, 1)
    x = ext(buf["sqrt_alphas_cumprod"]) * x_start + ext(buf["sqrt_one_minus_alphas_cumprod"]) * noise
    assert torch.isnan(x).any() == False  # noqa: E712   (Diffusion_Encoder.forward's host check, model.py:404)
    p = prompt.permute(1, 0, 2)
    xin = torch.cat([x, content.permute(1, 2, 0)], dim=1)
    out = unet(xin, t, p, encoder_attention_mask=sequence_mask(refer_lengths, p.size(1)).to(torch.bool)).sample
    sq = ((out - x_start) ** 2).reshape(B, -1)
    return (sq * ext(buf["loss_weight"])).mean()


@torch.no_grad()
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,4,16,64")
    ap.add_argument("--shape", default="8x400x200")
    ap.add_argument("--budget-ms", type=float, default=1500.0, help="timed window per variant (sets the repeat count)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("loss_bench needs a CUDA device")
    B, T, S = (int(v) for v in args.shape.split("x"))
    dev = torch.device("cuda", 0)
    unet = UNet1DConditionModel(in_channels=356, out_channels=100, block_out_channels=(128, 256, 384, 512), norm_num_groups=8,
                                cross_attention_dim=256, attention_head_dim=8, addition_embed_type="text", resnet_time_scale_shift="scale_shift")
    unet.load_state_dict(make_state_dict(ns2vc_denoiser_config(), seed=0))
    pre = Pre_model(PRE_CFG)
    pre.load_state_dict(make_pre_state_dict(PRE_CFG, seed=0))
    unet, pre = unet.to(dev).eval(), pre.to(dev).eval()
    pin = make_pre_inputs(B, T, S, ragged=True, seed=1)
    spec = torch.randn((B, 100, T), generator=torch.Generator().manual_seed(2))
    data = (pin["c"].to(dev), pin["refer"].to(dev), None, spec.to(dev), None, pin["lengths"].to(dev), pin["refer_lengths"].to(dev), None)
    noise = torch.randn((B, 100, T), generator=torch.Generator().manual_seed(3)).to(dev)
    buf = {k: v.to(dev) for k, v in coefs.loss_buffers(1000).items()}
    res = {"card": card(), "shape": dict(B=B, T=T, S=S), "rows": []}
    print(res["card"])
    for K in (int(v) for v in args.ks.split(",")):
        grid = [int(v) for v in torch.linspace(0, 999, K).round().tolist()] if K > 1 else [500]
        tk = torch.tensor(grid, dtype=torch.int64, device=dev)[:, None].expand(K, B).contiguous()
        profile = lambda: loss_profile(pre, unet, data, t_grid=grid, noise=noise).loss
        calls = lambda: torch.stack([diffusion_loss(pre, unet, data, t=tk[k], noise=noise).loss for k in range(K)])
        port = lambda: torch.stack([port_loss(pre, unet, data, tk[k], noise, buf) for k in range(K)])
        # the profile's parts
        len_r = data[6]

        def encoders():
            return pre.infer(data)
        content, prompt = encoders()
        sess = get_session(unet, content.permute(1, 2, 0), prompt.permute(1, 0, 2), sequence_mask(len_r, S))
        x_start, x = q_sample(data[3], noise, data[5], tk)
        out = torch.empty_like(x)
        loss_kernels = lambda: mse_rows(out, q_sample(data[3], noise, data[5], tk)[0], tk)
        forwards = lambda: sess.eval_x_start(x, tk, out)         # = prepare_cond + time_table + K forwards
        want = profile()
        for name, fn in (("calls", calls), ("port", port)):
            got = fn()
            rel = ((got - want).abs() / want.abs()).max().item()
            assert rel <= 1e-3, f"K={K}: {name} and profile disagree (rel {rel:.2e})"
        for fn in (profile, calls, port, encoders, sess.prepare, forwards, loss_kernels):
            fn()                                                 # warm-up of every shape the timed loops use
        one = timed_ms(profile, 1)
        reps = max(2, min(50, int(args.budget_ms / max(one, 1e-3))))
        t_prof, t_calls, t_port = [], [], []
        for _ in range(3):                                       # alternate the three so drift hits them alike
            t_prof.append(timed_ms(profile, reps))
            t_calls.append(timed_ms(calls, max(1, reps // 2)))
            t_port.append(timed_ms(port, max(1, reps // 2)))
        med = lambda v: sorted(v)[len(v) // 2]
        t_enc, t_prep = timed_ms(encoders, 20), timed_ms(sess.prepare, 20)
        t_fwd, t_loss = timed_ms(forwards, max(2, reps)), timed_ms(loss_kernels, 50)
        row = dict(K=K, reps=reps, profile_ms=med(t_prof), calls_ms=med(t_calls), port_ms=med(t_port),
                   profile_ms_runs=t_prof, calls_ms_runs=t_calls, port_ms_runs=t_port,
                   profile_ms_per_t=med(t_prof) / K, calls_ms_per_t=med(t_calls) / K, port_ms_per_t=med(t_port) / K,
                   encoders_ms=t_enc, prepare_ms=t_prep, forwards_ms=t_fwd - t_prep, forward_ms_each=(t_fwd - t_prep) / K,
                   loss_kernels_ms=t_loss)
        res["rows"].append(row)
        print(json.dumps({k: (round(v, 3) if isinstance(v, float) else v) for k, v in row.items() if not k.endswith("_runs")}))
    res["card_after"] = card()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
