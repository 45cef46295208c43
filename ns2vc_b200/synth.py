"""Deterministic synthetic weights and inputs (no checkpoints or datasets exist offline).

The generator is keyed by parameter NAME (not by module construction order), so the same
``state_dict`` is reproduced on any box with the same torch build — fixtures under
``tests/golden`` therefore only store outputs plus a checksum of the weights.

Distributions follow PyTorch's default initialisers used by the reference modules
(``nn.Conv1d`` / ``nn.Linear``: U(-1/sqrt(fan_in), 1/sqrt(fan_in)); norms: weight 1, bias 0;
``AttentionPooling.positional_embedding``: N(0,1)/sqrt(dim), reference ``embeddings.py:505``).
Norm affine parameters are additionally perturbed so that parity tests exercise gamma/beta.
"""
from __future__ import annotations

import hashlib
import math
from typing import Dict

import torch

from .arch import UNetConfig, param_shapes


def _seed_for(name: str, seed: int) -> int:
    h = hashlib.sha256(f"{seed}:{name}".encode()).digest()
    return int.from_bytes(h[:7], "little")


def make_state_dict(cfg: UNetConfig, seed: int = 0, perturb_norms: bool = True) -> Dict[str, torch.Tensor]:
    sd: Dict[str, torch.Tensor] = {}
    shapes = param_shapes(cfg)
    for name, shape in shapes.items():
        g = torch.Generator().manual_seed(_seed_for(name, seed))
        leaf = name.rsplit(".", 1)[-1]
        owner = name.rsplit(".", 1)[0]
        is_norm = (len(shape) == 1 and owner.split(".")[-1].startswith(("norm", "conv_norm_out")))
        if name.endswith("positional_embedding"):
            t = torch.randn(shape, generator=g) / math.sqrt(shape[-1])
        elif is_norm:
            if leaf == "weight":
                t = torch.ones(shape)
                if perturb_norms:
                    t = t + 0.1 * torch.randn(shape, generator=g)
            else:
                t = torch.zeros(shape)
                if perturb_norms:
                    t = 0.1 * torch.randn(shape, generator=g)
        else:
            wshape = shapes[owner + ".weight"]
            fan_in = 1
            for d in wshape[1:]:
                fan_in *= d
            bound = 1.0 / math.sqrt(fan_in)
            t = (torch.rand(shape, generator=g) * 2 - 1) * bound
        sd[name] = t.to(torch.float32).contiguous()
    return sd


def make_pre_state_dict(cfg: dict, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Synthetic `Pre_model` weights keyed by parameter name: norms 1 + 0.1 N(0,1) / 0.1 N(0,1), everything else
    U(-b, b) with b = fan_in^-1/2 (ConvTBC weights [k, c_in, c_out]: fan_in = k c_in)."""
    from .pre_model import pre_param_shapes
    sd: Dict[str, torch.Tensor] = {}
    for name, shape in pre_param_shapes(cfg).items():
        g = torch.Generator().manual_seed(_seed_for(name, seed))
        owner, leaf = name.rsplit(".", 1)
        if len(shape) == 1 and "norm" in owner.rsplit(".", 1)[-1]:
            t = (1.0 if leaf == "weight" else 0.0) + 0.1 * torch.randn(shape, generator=g)
        else:
            fan_in = 1
            for d in (shape[1:] if len(shape) > 1 else shape):
                fan_in *= d
            if name.endswith("conv.weight") and len(shape) == 3 and "spk_proj" not in name:
                fan_in = shape[0] * shape[1]
            t = (torch.rand(shape, generator=g) * 2 - 1) / math.sqrt(max(fan_in, 1))
        sd[name] = t.to(torch.float32).contiguous()
    return sd


VOCOS_REGIMES = ("init", "trained_like", "clip", "large_phase", "ln_offset")


def make_vocos_state_dict(seed: int = 0, regime: str = "init", input_channels: int = 100, dim: int = 512, intermediate_dim: int = 1536,
                          num_layers: int = 8, n_fft: int = 1024) -> Dict[str, torch.Tensor]:
    """Synthetic ``Vocos`` weights keyed by parameter name.  Regimes:

    init          the package's own init (trunc-normal std 0.02 conv / linear weights, zero biases, layer scale 1 / num_layers,
                  LayerNorms 1 / 0, periodic Hann window)
    trained_like  biases 0.05 N(0,1), LayerNorms 1 + 0.1 N / 0.1 N, layer scale U(0.05, 1); head log-magnitude bias -3 + 0.5 N,
                  phase bias U(-20, 20) rad
    clip          trained_like with log-magnitude biases of +6 on a quarter of the bins (exp > 100: clipped) and +200 on a
                  twentieth (exp overflows fp32 to +inf before the clip)
    large_phase   trained_like with the phase rows of head.out (weights and bias) x 100: sin / cos range reduction
    ln_offset     trained_like with embed bias + 30: the backbone LayerNorm's row statistics at |mean| >> std
    """
    from .vocoder import vocos_init, vocos_param_shapes
    if regime not in VOCOS_REGIMES:
        raise ValueError(f"unknown regime {regime!r} ({' | '.join(VOCOS_REGIMES)})")
    nb = n_fft // 2 + 1
    sd: Dict[str, torch.Tensor] = {}
    for name, shape in vocos_param_shapes(input_channels, dim, intermediate_dim, num_layers, n_fft).items():
        g = torch.Generator().manual_seed(_seed_for(name, seed))
        t = vocos_init(name, shape, num_layers, generator=g)
        leaf = name.rsplit(".", 1)[-1]
        if regime != "init" and not name.endswith("istft.window"):
            if leaf == "gamma":
                t = 0.05 + 0.95 * torch.rand(shape, generator=g)
            elif ".norm." in name or "final_layer_norm" in name:
                t = t + 0.1 * torch.randn(shape, generator=g)
            elif name == "head.out.bias":
                t = torch.cat([-3.0 + 0.5 * torch.randn((nb,), generator=g), 40.0 * torch.rand((nb,), generator=g) - 20.0])
                if regime == "clip":
                    u = torch.rand((nb,), generator=g)
                    t[:nb][u < 0.25] = 6.0
                    t[:nb][u < 0.05] = 200.0
            elif leaf == "bias":
                t = 0.05 * torch.randn(shape, generator=g)
            if regime == "large_phase" and name.startswith("head.out."):
                t[nb:] *= 100.0
            if regime == "ln_offset" and name == "backbone.embed.bias":
                t = t + 30.0
        sd[name] = t.to(torch.float32).contiguous()
    return sd


def make_pre_inputs(B: int, T: int, S: int, content_ch: int = 256, ragged: bool = False, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Synthetic `Pre_model.infer` inputs: c ~ N(0,1) [B, 256, T] (ContentVec features), refer ~ N(0,1) [B, 100, S] (mel prompt)."""
    g = torch.Generator().manual_seed(seed + 11)
    c = torch.randn((B, content_ch, T), generator=g)
    refer = torch.randn((B, 100, S), generator=g)
    if ragged:
        lengths = torch.tensor([max(1, T - 37 * (i % 8)) for i in range(B)], dtype=torch.int64)
        refer_lengths = torch.tensor([max(1, S - 17 * (i % 8)) for i in range(B)], dtype=torch.int64)
    else:
        lengths = torch.full((B,), T, dtype=torch.int64)
        refer_lengths = torch.full((B,), S, dtype=torch.int64)
    return dict(c=c, refer=refer, lengths=lengths, refer_lengths=refer_lengths)


def make_utterance_loss_inputs(T: int, S: int, seed: int) -> Dict[str, torch.Tensor]:
    """One utterance of the per-utterance objective: c [256, T] and refer [100, S] (``make_pre_inputs`` at B = 1), the target
    mel spec [100, T] ~ N(0,1) (seed+1) and the noise [100, T] ~ N(0,1) (seed+2)."""
    pin = make_pre_inputs(1, T, S, seed=seed)
    spec = torch.randn((1, 100, T), generator=torch.Generator().manual_seed(seed + 1))
    noise = torch.randn((1, 100, T), generator=torch.Generator().manual_seed(seed + 2))
    return dict(c=pin["c"][0], refer=pin["refer"][0], spec=spec[0], noise=noise[0])


def state_dict_checksum(sd: Dict[str, torch.Tensor]) -> str:
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(sd[k].detach().cpu().contiguous().numpy().tobytes())
    return h.hexdigest()[:16]


def make_inputs(B: int, T: int, S: int, latent_ch: int = 100, content_ch: int = 256,
                ragged: bool = False, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Synthetic denoiser inputs per SURVEY.md §8(d): content ~ N(0,1) [T,B,256] (seed+1),
    prompt ~ N(0,1) [S,B,256] (seed+2), x_T ~ N(0,1) [B,100,T] (seed+3); ragged prompt lengths
    S - 17*i (i = sample index mod 8), floored at 1, for parity runs."""
    def gen(k):
        return torch.Generator().manual_seed(seed + k)
    content = torch.randn((T, B, content_ch), generator=gen(1))
    prompt = torch.randn((S, B, content_ch), generator=gen(2))
    x = torch.randn((B, latent_ch, T), generator=gen(3))
    lengths = torch.full((B,), T, dtype=torch.int64)
    if ragged:
        refer_lengths = torch.tensor([max(1, S - 17 * (i % 8)) for i in range(B)], dtype=torch.int64)
    else:
        refer_lengths = torch.full((B,), S, dtype=torch.int64)
    return dict(content=content, prompt=prompt, x=x, lengths=lengths, refer_lengths=refer_lengths)


def linear_betas(timesteps: int = 1000) -> torch.Tensor:
    """fp32 copy of the reference's linear beta schedule (``model.py:426-433, 473``):
    float64 linspace cast to float32 by ``register_buffer``."""
    scale = 1000 / timesteps
    return torch.linspace(scale * 0.0001, scale * 0.02, timesteps, dtype=torch.float64).to(torch.float32)


CONTENTVEC_REGIMES = ("init", "trained_like", "sharp", "large_v", "ln_offset")
CONTENTVEC_SMALL = dict(conv_dim=128, embed_dim=128, ffn_dim=256, num_layers=2, num_heads=2, pos_conv_kernel=16, pos_conv_groups=4,
                        final_dim=32)


def make_contentvec_state_dict(seed: int = 0, regime: str = "init", **cfg) -> Dict[str, torch.Tensor]:
    """Synthetic fairseq ``HubertModel`` weights (ContentVec's configuration unless ``cfg`` overrides it), fairseq-named, in one
    of five regimes:

    * ``init``: fairseq's initialisation (Kaiming-normal convs, N(0, 0.02) linears, zero biases, unit LayerNorms, the positional
      conv N(0, sqrt(4 / (K D))) with g = ||v||);
    * ``trained_like``: perturbed norms and biases, and a ``final_proj`` whose output has unit scale (the dataset's ``.soft.pt``
      units have mean -0.02 and std 1.0);
    * ``sharp``: q and k scaled to an attention-score std of about 4;
    * ``large_v``: v_proj x 256 and out_proj x 1/256;
    * ``ln_offset``: ``trained_like`` with a +100 offset on four residual channels (post_extract_proj, out_proj and fc2 biases),
      so that every post-LN sees rows whose mean is far from their spread."""
    from .content import CONTENTVEC, contentvec_param_shapes
    if regime not in CONTENTVEC_REGIMES:
        raise ValueError(f"unknown regime {regime!r}")
    c = {**CONTENTVEC, **cfg}
    D, K = c["embed_dim"], c["pos_conv_kernel"]
    g = torch.Generator().manual_seed(1000 + seed)
    sd: Dict[str, torch.Tensor] = {}
    trained = regime != "init"
    for k, shape in contentvec_param_shapes(**c).items():
        leaf = k.rsplit(".", 1)[-1]
        if k.startswith("feature_extractor.conv_layers.") and k.endswith(".0.weight"):
            t = torch.randn(shape, generator=g) * math.sqrt(2.0 / (shape[1] * shape[2]))
        elif k == "encoder.pos_conv.0.weight_v":
            t = torch.randn(shape, generator=g) * math.sqrt(4.0 / (K * D))
        elif k == "encoder.pos_conv.0.weight_g":
            continue                                           # after weight_v: g = ||v|| per tap (weight_norm's initial value)
        elif "norm" in k or k.startswith("feature_extractor.conv_layers.0.2."):
            if leaf == "weight":
                t = 1.0 + (0.1 * torch.randn(shape, generator=g) if trained else torch.zeros(shape))
            else:
                t = 0.1 * torch.randn(shape, generator=g) if trained else torch.zeros(shape)
        elif leaf == "bias":
            t = 0.02 * torch.randn(shape, generator=g) if trained else torch.zeros(shape)
        else:
            t = 0.02 * torch.randn(shape, generator=g)
        sd[k] = t
    v = sd["encoder.pos_conv.0.weight_v"]
    sd["encoder.pos_conv.0.weight_g"] = v.pow(2).sum(dim=(0, 1), keepdim=True).sqrt() * (1.5 if trained else 1.0)
    sd = {k: sd[k] for k in contentvec_param_shapes(**c)}     # registry order
    if trained:
        sd["final_proj.weight"] = torch.randn(sd["final_proj.weight"].shape, generator=g) / math.sqrt(D)
        sd["final_proj.bias"] = torch.full_like(sd["final_proj.bias"], -0.02)
    for i in range(c["num_layers"]):
        p = f"encoder.layers.{i}.self_attn."
        if regime == "sharp":
            s = 2.0 / math.sqrt(D) / 0.02
            sd[p + "q_proj.weight"] = sd[p + "q_proj.weight"] * s
            sd[p + "k_proj.weight"] = sd[p + "k_proj.weight"] * s
        if regime == "large_v":
            sd[p + "v_proj.weight"] = sd[p + "v_proj.weight"] * 256.0
            sd[p + "v_proj.bias"] = sd[p + "v_proj.bias"] * 256.0
            sd[p + "out_proj.weight"] = sd[p + "out_proj.weight"] / 256.0
    if regime == "ln_offset":
        ch = torch.tensor([3, 17, 40, D - 1])
        for k in ["post_extract_proj.bias"] + [f"encoder.layers.{i}.{m}.bias" for i in range(c["num_layers"])
                                               for m in ("self_attn.out_proj", "fc2")]:
            t = sd[k].clone()
            t[ch] += 100.0
            sd[k] = t
    return {k: t.to(torch.float32).contiguous() for k, t in sd.items()}
