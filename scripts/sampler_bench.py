"""Denoiser-steps/s (B x UNet forwards per second, bench.py's unit) of the fused DDIM-100 and DDPM-1000 loops
(``DenoiserSession.sample_ddim`` / ``sample_ddpm``) against the reference's own loop (``ddim_sample`` / ``p_sample_loop``, model.py:535-601) written out with the drop-in UNet's generic forward: the
Diffusion_Encoder closure, ``extract`` gathers and scalar math as torch ops, ``randn_like`` and the per-call NaN assert.

    python scripts/sampler_bench.py [--shapes 1x256x128,8x1024x256] [--generic-ddpm-steps 100] [--out results/sampler_bench.json]

Shapes are BxTxS (batch, frames, prompt frames); the 66 M-parameter denoiser with synthetic weights.  Timing: CUDA events after
warm-up (the fused loops are timed once their chunk graphs are captured).  The generic DDPM loop is timed over its first
``--generic-ddpm-steps`` steps (its per-step cost does not depend on t).  Each pair of runs from one seed is asserted to agree
(rtol 1e-3 / atol 1e-4).  Prints the card's name and power limit with the numbers.  Needs a CUDA device.
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
from ns2vc_b200.arch import ns2vc_denoiser_config  # noqa: E402
from ns2vc_b200.fused import DenoiserSession  # noqa: E402
from ns2vc_b200.synth import make_inputs, make_state_dict  # noqa: E402
from ns2vc_b200.unet import UNet1DConditionModel  # noqa: E402


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable: {e}"


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b) / 1e3


def agree(a, b, what):
    err = (a - b).abs()
    worst = (err / (1e-4 + 1e-3 * b.abs())).max().item()
    assert worst <= 1.0, f"{what}: fused and generic disagree (max_abs {err.max().item():.3e}, worst err/tol {worst:.2f})"
    return round(worst, 3)


def generic_loops(unet, inp):
    """The reference's ddim_sample / p_sample_loop bodies around the drop-in UNet's generic forward."""
    dev = "cuda"
    content, prompt, plen = inp["content"].to(dev), inp["prompt"].to(dev), inp["refer_lengths"].to(dev)
    buf = {k: v.to(dev) for k, v in coefs.diffusion_buffers(1000).items()}

    def extract(a, t, x_shape):
        return a.gather(-1, t).reshape(t.shape[0], *((1,) * (len(x_shape) - 1)))

    def model_predictions(x, t):
        assert torch.isnan(x).any() == False                 # noqa: E712  (model.py:404)
        p = prompt.permute(1, 0, 2)
        xin = torch.cat([x, content.permute(1, 2, 0)], dim=1)
        mask = (torch.arange(p.size(1), device=dev).unsqueeze(0) < plen.unsqueeze(1)).to(torch.bool)
        x_start = unet(xin, t, p, encoder_attention_mask=mask).sample
        t = t.type(torch.int64)
        pred_noise = (extract(buf["sqrt_recip_alphas_cumprod"], t, x.shape) * x - x_start) / extract(buf["sqrt_recipm1_alphas_cumprod"], t, x.shape)
        return pred_noise, x_start

    def ddim(img, S, eta=0.0):
        for time, time_next in coefs.ddim_time_pairs(1000, S):
            pred_noise, x_start = model_predictions(img, torch.full((img.shape[0],), time, device=dev, dtype=torch.long))
            if time_next < 0:
                img = x_start
                continue
            alpha, alpha_next = buf["alphas_cumprod"][time], buf["alphas_cumprod"][time_next]
            sigma = eta * ((1 - alpha / alpha_next) * (1 - alpha_next) / (1 - alpha)).sqrt()
            c = (1 - alpha_next - sigma ** 2).sqrt()
            img = x_start * alpha_next.sqrt() + c * pred_noise + sigma * torch.randn_like(img)
        return img

    def ddpm(img, timesteps):
        for t in timesteps:
            bt = torch.full((img.shape[0],), t, device=dev, dtype=torch.long)
            _pn, x_start = model_predictions(img, bt)
            mean = extract(buf["posterior_mean_coef1"], bt, img.shape) * x_start + extract(buf["posterior_mean_coef2"], bt, img.shape) * img
            noise = torch.randn_like(img) if t > 0 else 0.
            img = mean + (0.5 * extract(buf["posterior_log_variance_clipped"], bt, img.shape)).exp() * noise
        return img
    return ddim, ddpm


@torch.no_grad()
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1x256x128,8x1024x256")
    ap.add_argument("--generic-ddpm-steps", type=int, default=100)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "sampler_bench needs a CUDA device"
    info = card()
    print(f"card: {info}")
    cfg = ns2vc_denoiser_config()
    unet = UNet1DConditionModel(in_channels=356, out_channels=100, block_out_channels=(128, 256, 384, 512), norm_num_groups=8,
                                cross_attention_dim=256, attention_head_dim=8, addition_embed_type="text", resnet_time_scale_shift="scale_shift")
    unet.load_state_dict(make_state_dict(cfg, seed=0))
    unet = unet.cuda().eval()
    rows = []
    for shape in args.shapes.split(","):
        B, T, S = (int(v) for v in shape.split("x"))
        inp = make_inputs(B, T, S, ragged=True, seed=B + T)
        content = inp["content"].permute(1, 2, 0).contiguous().cuda()
        prompt = inp["prompt"].permute(1, 0, 2).contiguous().cuda()
        mask = (torch.arange(S).unsqueeze(0) < inp["refer_lengths"].unsqueeze(1)).cuda()
        sess = DenoiserSession(unet, content, prompt, mask)
        ddim_g, ddpm_g = generic_loops(unet, inp)
        x = inp["x"].cuda()
        row = dict(B=B, T=T, S=S, unit="denoiser-steps/s")
        # DDIM, 100 steps (sample()'s default sampling_timesteps), eta 0
        for _ in range(DenoiserSession.CAPTURE_AFTER):
            sess.sample_ddim(x, 100)
        torch.cuda.manual_seed(1)
        fused, t_f = timed(lambda: sess.sample_ddim(x, 100))
        ddim_g(x, 6)                                          # warm-up
        torch.cuda.manual_seed(1)
        generic, t_g = timed(lambda: ddim_g(x, 100))
        row["ddim100"] = dict(fused=round(B * 100 / t_f, 1), generic=round(B * 100 / t_g, 1), speedup=round(t_g / t_f, 2),
                              worst_err_over_tol=agree(fused, generic, "ddim100"))
        # DDPM, all 1000 steps; the generic loop over its first steps (and the fused loop over the same steps for the check)
        for _ in range(DenoiserSession.CAPTURE_AFTER):
            sess.sample_ddpm(x)
        torch.cuda.manual_seed(2)
        _out, t_f = timed(lambda: sess.sample_ddpm(x))
        n = args.generic_ddpm_steps
        ts = list(range(999, 999 - n, -1))
        torch.cuda.manual_seed(3)
        part_f = sess.sample_ddpm(x, ts)
        torch.cuda.manual_seed(3)
        part_g, t_g = timed(lambda: ddpm_g(x, ts))
        row["ddpm1000"] = dict(fused=round(B * 1000 / t_f, 1), generic=round(B * n / t_g, 1),
                               speedup=round((t_g / n) / (t_f / 1000), 2), generic_steps_timed=n,
                               worst_err_over_tol=agree(part_f, part_g, f"ddpm first {n} steps"))
        rows.append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
