"""TEST INFRASTRUCTURE ONLY — CPU fp32 restatement of the reference's condition encoders (`Pre_model`), the step
immediately BEFORE the denoiser hot path (SURVEY.md §8(f) rank 1).  Nothing in the product imports this file.

Functional style over a reference `state_dict` (same parameter names), same ATen ops in the same order:
  * Pre_model.infer                     model.py:360-377
  * PhoneEncoder / PromptEncoder        model.py:98-190
  * ConvLayer (LayerNorm + ConvTBC k=1) model.py:77-96, 63-75
  * TransformerEncoderLayer -> EncSALayer(c, 8 heads, conv-FFN k=9 'SAME')   model.py:50-59, operations.py:953-964, 784-821
  * MultiheadAttention (torch F.multi_head_attention_forward path, packed in_proj, no biases)   operations.py:304-441
  * TransformerFFNLayer (k shifted Linears, * k^-0.5, ReLU, Linear)          operations.py:644-690
  * ref_enc = TextTimeEmbedding(100, 100, 1)                                  model.py:340, unet1d/embeddings.py:421-434
Pinned against the unmodified reference by oracle/make_golden_pre.py (tests/golden/pre_model_*.pt).
"""
from __future__ import annotations

import math
from typing import Dict, Tuple

import torch
import torch.nn.functional as F

from .unet_oracle import sequence_mask, text_time_embedding

Tensor = torch.Tensor
SD = Dict[str, Tensor]
N_HEADS = 8          # operations.py:961  EncSALayer(c, 8, ...)
FFN_KERNEL = 9       # operations.py:963


def conv_layer(sd: SD, p: str, x_tbc: Tensor, pad_mask_bt: Tensor) -> Tensor:
    """ConvLayer.forward (model.py:86-96): zero the padded frames, LayerNorm over channels, ConvTBC with k=1."""
    x = x_tbc.masked_fill(pad_mask_bt.t().unsqueeze(-1), 0)
    x = F.layer_norm(x, (x.shape[-1],), sd[p + ".layer_norm.weight"], sd[p + ".layer_norm.bias"], 1e-5)
    w = sd[p + ".conv.weight"]                               # [k, c_in, c_out]
    return torch.conv_tbc(x.contiguous(), w, sd[p + ".conv.bias"], w.shape[0] // 2)


def self_attention(sd: SD, p: str, x_tbc: Tensor, pad_mask_bt: Tensor) -> Tensor:
    """MultiheadAttention self-attention as F.multi_head_attention_forward evaluates it with need_weights=True
    (operations.py:412-421): packed in_proj, q scaled by head_dim^-0.5, -inf on padded keys, softmax, out_proj."""
    T, B, C = x_tbc.shape
    dh = C // N_HEADS
    q, k, v = F.linear(x_tbc, sd[p + ".in_proj_weight"]).chunk(3, dim=-1)
    q = q.contiguous().view(T, B * N_HEADS, dh).transpose(0, 1)
    k = k.contiguous().view(T, B * N_HEADS, dh).transpose(0, 1)
    v = v.contiguous().view(T, B * N_HEADS, dh).transpose(0, 1)
    bias = torch.zeros((B, 1, 1, T), dtype=x_tbc.dtype).masked_fill(pad_mask_bt.view(B, 1, 1, T), float("-inf"))
    bias = bias.expand(-1, N_HEADS, -1, -1).reshape(B * N_HEADS, 1, T)
    w = torch.baddbmm(bias, q * math.sqrt(1.0 / dh), k.transpose(-2, -1))
    w = torch.softmax(w, dim=-1)
    o = torch.bmm(w, v).transpose(0, 1).contiguous().view(T * B, C)
    return F.linear(o, sd[p + ".out_proj.weight"]).view(T, B, C)


def conv_ffn(sd: SD, p: str, x_tbc: Tensor) -> Tensor:
    """TransformerFFNLayer with kernel_size 9, 'SAME' padding (operations.py:664-690)."""
    k = FFN_KERNEL
    first = -((k - 1) // 2)
    last = first + k - 1
    padded = F.pad(x_tbc, (0, 0, 0, 0, -first, last))
    T = x_tbc.shape[0]
    res = None
    for i in range(k):
        shifted = padded[i:T + i] if i else x_tbc            # NB: tap 0 reads the UNPADDED input (reference quirk, :681)
        y = F.linear(shifted, sd[f"{p}.ffn_1.{i}.weight"], sd.get(f"{p}.ffn_1.{i}.bias"))
        res = y if res is None else res + y
    x = res * k ** -0.5
    x = F.relu(x)
    return F.linear(x, sd[p + ".ffn_2.weight"], sd[p + ".ffn_2.bias"])


def enc_sa_layer(sd: SD, p: str, x_tbc: Tensor, pad_mask_bt: Tensor) -> Tensor:
    """EncSALayer.forward (operations.py:798-821), eval mode (dropout off)."""
    keep = (1 - pad_mask_bt.to(x_tbc.dtype)).transpose(0, 1)[..., None]
    r = x_tbc
    x = F.layer_norm(x_tbc, (x_tbc.shape[-1],), sd[p + ".layer_norm1.weight"], sd[p + ".layer_norm1.bias"], 1e-5)
    x = self_attention(sd, p + ".self_attn", x, pad_mask_bt)
    x = (r + x) * keep
    r = x
    y = F.layer_norm(x, (x.shape[-1],), sd[p + ".layer_norm2.weight"], sd[p + ".layer_norm2.bias"], 1e-5)
    y = conv_ffn(sd, p + ".ffn", y)
    return (r + y) * keep


def _encoder(sd: SD, p: str, x_tbc: Tensor, lengths: Tensor, n_layers: int, tap=None) -> Tensor:
    pad = ~sequence_mask(lengths, x_tbc.shape[0]).to(torch.bool)           # [B, T], True = padding
    keep = (1 - pad.to(x_tbc.dtype)).transpose(0, 1)[..., None]
    x = conv_layer(sd, p + ".pre", x_tbc, pad) * keep
    if tap is not None:
        tap[p + ".pre"] = x.clone()
    for i in range(n_layers):
        x = enc_sa_layer(sd, f"{p}.layers.{i}.op", x, pad)
        if tap is not None:
            tap[f"{p}.layers.{i}"] = x.clone()
    x = conv_layer(sd, p + ".out_proj", x, pad)
    x = F.layer_norm(x, (x.shape[-1],), sd[p + ".layer_norm.weight"], sd[p + ".layer_norm.bias"], 1e-5)
    return x * keep


def phone_encoder(sd: SD, p: str, c_bct: Tensor, lengths: Tensor, g_bc1: Tensor, n_layers: int, tap=None) -> Tensor:
    """PhoneEncoder.forward (model.py:128-148): content + spk_proj(g), then the encoder stack.  Returns [T, B, C_out]."""
    x = c_bct + F.conv1d(g_bc1, sd[p + ".spk_proj.weight"], sd[p + ".spk_proj.bias"])
    return _encoder(sd, p, x.permute(2, 0, 1), lengths, n_layers, tap)


def prompt_encoder(sd: SD, p: str, refer_bct: Tensor, lengths: Tensor, n_layers: int, tap=None) -> Tensor:
    """PromptEncoder.forward (model.py:173-190).  Returns [S, B, C_out]."""
    return _encoder(sd, p, refer_bct.permute(2, 0, 1), lengths, n_layers, tap)


def pre_model_infer(sd: SD, c_padded: Tensor, refer_padded: Tensor, lengths: Tensor, refer_lengths: Tensor,
                    n_layers_phone: int = 6, n_layers_prompt: int = 6, tap=None) -> Tuple[Tensor, Tensor]:
    """Pre_model.infer (model.py:360-377): returns (content [T,B,C], audio_prompt [S,B,C]) — exactly the two tensors
    Diffusion_Encoder.forward receives (model.py:403-415)."""
    g = text_time_embedding(sd, "ref_enc", refer_padded.transpose(1, 2), 1).unsqueeze(-1)      # [B, 100, 1]
    if tap is not None:
        tap["ref_enc"] = g.clone()
    audio_prompt = prompt_encoder(sd, "prompt_encoder", refer_padded, refer_lengths, n_layers_prompt, tap)
    content = phone_encoder(sd, "phoneme_encoder", c_padded, lengths, g, n_layers_phone, tap)
    return content, audio_prompt


def synth_state_dict(shapes: Dict[str, Tuple[int, ...]], seed: int = 0) -> SD:
    """Deterministic weights keyed by parameter name (so fixtures store shapes + outputs, not weights):
    LayerNorm-like vectors ~ 1 + 0.1 N(0,1) / 0.1 N(0,1), everything else U(-b, b) with b = fan_in^-0.5."""
    import hashlib
    sd: SD = {}
    for name, shape in shapes.items():
        h = int.from_bytes(hashlib.sha256(f"{seed}:{name}".encode()).digest()[:4], "little")
        g = torch.Generator().manual_seed(h)
        leaf = name.rsplit(".", 1)[-1]
        owner = name.rsplit(".", 1)[0].rsplit(".", 1)[-1]
        if len(shape) == 1 and ("norm" in owner):
            t = (1.0 if leaf == "weight" else 0.0) + 0.1 * torch.randn(shape, generator=g)
        else:
            fan_in = 1
            for d in (shape[1:] if len(shape) > 1 else shape):
                fan_in *= d
            if leaf == "weight" and len(shape) == 3 and name.endswith("conv.weight"):    # ConvTBC: [k, c_in, c_out]
                fan_in = shape[0] * shape[1]
            t = (torch.rand(shape, generator=g) * 2 - 1) / math.sqrt(max(fan_in, 1))
        sd[name] = t.to(torch.float32).contiguous()
    return sd
