"""Functional ATen restatement of the content units ``utils.get_hubert_content`` computes with ContentVec (a fairseq
``HubertModel``: extractor_mode "default", layer_norm_first False, no conv biases): ``extract_features(source, padding_mask = all
False, output_layer = L)`` then ``final_proj``, on fairseq's parameter names, in fp32 or fp64.

Each row of a batch is computed alone on its own samples (``lengths``), which is what the reference does: it runs one slice at
a time.  The per-stage functions let the tests feed a stage the GPU's own input for it.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn.functional as F

CONV_LAYERS = [(10, 5)] + [(3, 2)] * 4 + [(2, 2)] * 2     # fairseq's default conv_feature_layers (kernel, stride)
EPS = 1e-5


def num_frames(n: int) -> int:
    """Frames of n samples: T = floor((T - k) / s) + 1 through the seven convs (0 if the input is too short)."""
    for k, s in CONV_LAYERS:
        n = 0 if n < k else (n - k) // s + 1
    return n


def _c(sd, k, dtype):
    return sd[k].to(dtype)


def fold_weight_norm(g: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """torch.nn.utils.weight_norm(dim=2): W = g v / ||v||, the norm over (out, in) for each tap."""
    return g * v / v.pow(2).sum(dim=(0, 1), keepdim=True).sqrt()


def pos_conv_weight(sd: Dict[str, torch.Tensor], dtype=torch.float64) -> torch.Tensor:
    p = "encoder.pos_conv.0."
    if p + "weight_g" in sd:
        g, v = sd[p + "weight_g"], sd[p + "weight_v"]
    else:
        g, v = sd[p + "parametrizations.weight.original0"], sd[p + "parametrizations.weight.original1"]
    return fold_weight_norm(g.to(dtype), v.to(dtype))


def conv_layer(sd, l: int, x: torch.Tensor) -> torch.Tensor:
    """Conv l of the feature encoder on token-major [T, C] input (l = 0: the waveform [N]) -> [T_l, C0] (GroupNorm + GELU for l = 0)."""
    k, s = CONV_LAYERS[l]
    w = _c(sd, f"feature_extractor.conv_layers.{l}.0.weight", x.dtype)
    inp = x[None, None, :] if l == 0 else x.t()[None]
    y = F.conv1d(inp, w, stride=s)
    if l == 0:
        y = F.group_norm(y, w.shape[0], _c(sd, "feature_extractor.conv_layers.0.2.weight", x.dtype),
                         _c(sd, "feature_extractor.conv_layers.0.2.bias", x.dtype), EPS)
    return F.gelu(y)[0].t()


def layer_norm(sd, name: str, x: torch.Tensor) -> torch.Tensor:
    return F.layer_norm(x, x.shape[-1:], _c(sd, name + ".weight", x.dtype), _c(sd, name + ".bias", x.dtype), EPS)


def linear(sd, name: str, x: torch.Tensor) -> torch.Tensor:
    return F.linear(x, _c(sd, name + ".weight", x.dtype), _c(sd, name + ".bias", x.dtype))


def pos_conv(sd, x: torch.Tensor) -> torch.Tensor:
    """x + GELU(SamePad(pos_conv(x))) on [T, D]"""
    w = pos_conv_weight(sd, x.dtype)
    K, groups = w.shape[-1], x.shape[-1] // w.shape[1]
    y = F.conv1d(x.t()[None], w, _c(sd, "encoder.pos_conv.0.bias", x.dtype), padding=K // 2, groups=groups)
    if K % 2 == 0:
        y = y[:, :, :-1]
    return x + F.gelu(y)[0].t()


def attention_block(sd, i: int, x: torch.Tensor, heads: int) -> torch.Tensor:
    """self_attn_layer_norm(x + out_proj(attn(x))) of layer i on [T, D]"""
    p = f"encoder.layers.{i}."
    T, D = x.shape
    dh = D // heads
    q = linear(sd, p + "self_attn.q_proj", x) * dh ** -0.5
    k = linear(sd, p + "self_attn.k_proj", x)
    v = linear(sd, p + "self_attn.v_proj", x)
    q, k, v = (t.reshape(T, heads, dh).transpose(0, 1) for t in (q, k, v))
    a = torch.softmax(q @ k.transpose(1, 2), dim=-1) @ v
    a = a.transpose(0, 1).reshape(T, D)
    return layer_norm(sd, p + "self_attn_layer_norm", x + linear(sd, p + "self_attn.out_proj", a))


def ffn_block(sd, i: int, x: torch.Tensor) -> torch.Tensor:
    p = f"encoder.layers.{i}."
    return layer_norm(sd, p + "final_layer_norm", x + linear(sd, p + "fc2", F.gelu(linear(sd, p + "fc1", x))))


def stages(sd, wav: torch.Tensor, heads: int, dtype=torch.float64) -> Dict[str, torch.Tensor]:
    """Every stage of one utterance wav [N] (N >= 400) under the tap names of the engine: [T, C] each."""
    x = wav.to(dtype)
    out: Dict[str, torch.Tensor] = {}
    for l in range(len(CONV_LAYERS)):
        x = conv_layer(sd, l, x)
        out[f"feature_extractor.conv_layers.{l}"] = x
    x = out["layer_norm"] = layer_norm(sd, "layer_norm", x)
    x = out["post_extract_proj"] = linear(sd, "post_extract_proj", x)
    x = out["encoder.pos_conv"] = pos_conv(sd, x)
    x = out["encoder.layer_norm"] = layer_norm(sd, "encoder.layer_norm", x)
    i = 0
    while f"encoder.layers.{i}.fc1.weight" in sd:
        x = out[f"encoder.layers.{i}.self_attn_layer_norm"] = attention_block(sd, i, x, heads)
        x = out[f"encoder.layers.{i}"] = ffn_block(sd, i, x)
        i += 1
    out["final_proj"] = linear(sd, "final_proj", x)
    return out


def stage_fn(sd, name: str, heads: int):
    """The function of one stage (tap name) of its input (the previous stage's output; the waveform for conv 0)."""
    if name.startswith("feature_extractor.conv_layers."):
        l = int(name.rsplit(".", 1)[1])
        return lambda x: conv_layer(sd, l, x)
    if name == "layer_norm" or name == "encoder.layer_norm":
        return lambda x: layer_norm(sd, name, x)
    if name in ("post_extract_proj", "final_proj"):
        return lambda x: linear(sd, name, x)
    if name == "encoder.pos_conv":
        return lambda x: pos_conv(sd, x)
    if name.endswith(".self_attn_layer_norm"):
        i = int(name.split(".")[2])
        return lambda x: attention_block(sd, i, x, heads)
    i = int(name.split(".")[2])
    return lambda x: ffn_block(sd, i, x)


def stage_names(num_layers: int) -> List[str]:
    names = [f"feature_extractor.conv_layers.{l}" for l in range(len(CONV_LAYERS))]
    names += ["layer_norm", "post_extract_proj", "encoder.pos_conv", "encoder.layer_norm"]
    for i in range(num_layers):
        names += [f"encoder.layers.{i}.self_attn_layer_norm", f"encoder.layers.{i}"]
    return names + ["final_proj"]


def extract(sd, wav: torch.Tensor, heads: int, lengths: Optional[Sequence[int]] = None, dtype=torch.float64) -> torch.Tensor:
    """units [B, T, final_dim] of wav [B, N]: row b computed alone on wav[b, :lengths[b]], zero past its own frames"""
    B, N = wav.shape
    lengths = [N] * B if lengths is None else [int(n) for n in lengths]
    T = num_frames(N)
    out = None
    for b in range(B):
        u = stages(sd, wav[b, :lengths[b]], heads, dtype)["final_proj"]
        if out is None:
            out = torch.zeros((B, T, u.shape[1]), dtype=dtype, device=wav.device)
        out[b, :u.shape[0]] = u
    return out
