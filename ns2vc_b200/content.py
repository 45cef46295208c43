"""``ContentVec`` — drop-in for the content encoder the reference runs before the condition encoders:
``utils.get_hubert_content(hmodel, wav_16k)`` with ContentVec (``checkpoint_best_legacy_500.pt``), a fairseq ``HubertModel``
(HuBERT-base: conv feature encoder of extractor_mode "default", post-LN transformer, no conv biases), i.e.
``extract_features(source, padding_mask = all False, output_layer = 12)`` then ``final_proj``.

Same parameter names and shapes as ``HubertModel.state_dict()`` without the training-only ``mask_emb`` / ``label_embs_concat``.
``extract`` takes a padded batch of 16 kHz waveforms and per-row ``lengths``: row b then equals that utterance run alone (a
padded fairseq batch does not: the first conv's GroupNorm and the positional conv read the padding).  The math runs in the
sm_90a engine behind the C-ABI (``include/ns2vc_b200.h``, ``csrc/content.cu``); this module owns the parameters and marshals
pointers.  No CPU path; inference only.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch
import torch.nn as nn

from . import _lib
from .unet import _insert

CONV_LAYERS = [(10, 5)] + [(3, 2)] * 4 + [(2, 2)] * 2     # fairseq's default conv_feature_layers (kernel, stride)
MIN_SAMPLES = 400                                          # the shortest input that gives one frame
CONTENTVEC = dict(conv_dim=512, embed_dim=768, ffn_dim=3072, num_layers=12, num_heads=12, pos_conv_kernel=128, pos_conv_groups=16,
                  final_dim=256)
TRAINING_ONLY = ("mask_emb", "label_embs_concat")


def num_frames(n: int) -> int:
    """Frames of n samples at 16 kHz (one per 320 samples): T = floor((T - k) / s) + 1 through the seven convs; 0 below 400."""
    n = int(n)
    for k, s in CONV_LAYERS:
        n = 0 if n < k else (n - k) // s + 1
    return n


def contentvec_param_shapes(conv_dim: int = 512, embed_dim: int = 768, ffn_dim: int = 3072, num_layers: int = 12, num_heads: int = 12,
                            pos_conv_kernel: int = 128, pos_conv_groups: int = 16, final_dim: int = 256) -> Dict[str, Tuple[int, ...]]:
    """``HubertModel.state_dict()`` keys -> shapes without mask_emb / label_embs_concat, in its order (a module's own parameters
    before its children's; children in registration order: feature_extractor, post_extract_proj, encoder, layer_norm,
    final_proj; fairseq's MultiheadAttention registers k, v, q, out)."""
    s: Dict[str, Tuple[int, ...]] = {}
    for l, (k, _) in enumerate(CONV_LAYERS):
        s[f"feature_extractor.conv_layers.{l}.0.weight"] = (conv_dim, 1 if l == 0 else conv_dim, k)
        if l == 0:
            s["feature_extractor.conv_layers.0.2.weight"] = (conv_dim,); s["feature_extractor.conv_layers.0.2.bias"] = (conv_dim,)
    s["post_extract_proj.weight"] = (embed_dim, conv_dim); s["post_extract_proj.bias"] = (embed_dim,)
    s["encoder.pos_conv.0.bias"] = (embed_dim,)
    s["encoder.pos_conv.0.weight_g"] = (1, 1, pos_conv_kernel)
    s["encoder.pos_conv.0.weight_v"] = (embed_dim, embed_dim // pos_conv_groups, pos_conv_kernel)
    for i in range(num_layers):
        p = f"encoder.layers.{i}."
        for m in ("k_proj", "v_proj", "q_proj", "out_proj"):
            s[p + f"self_attn.{m}.weight"] = (embed_dim, embed_dim); s[p + f"self_attn.{m}.bias"] = (embed_dim,)
        s[p + "self_attn_layer_norm.weight"] = (embed_dim,); s[p + "self_attn_layer_norm.bias"] = (embed_dim,)
        s[p + "fc1.weight"] = (ffn_dim, embed_dim); s[p + "fc1.bias"] = (ffn_dim,)
        s[p + "fc2.weight"] = (embed_dim, ffn_dim); s[p + "fc2.bias"] = (embed_dim,)
        s[p + "final_layer_norm.weight"] = (embed_dim,); s[p + "final_layer_norm.bias"] = (embed_dim,)
    s["encoder.layer_norm.weight"] = (embed_dim,); s["encoder.layer_norm.bias"] = (embed_dim,)
    s["layer_norm.weight"] = (conv_dim,); s["layer_norm.bias"] = (conv_dim,)
    s["final_proj.weight"] = (final_dim, embed_dim); s["final_proj.bias"] = (final_dim,)
    return s


def _norm_keys(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """The parametrizations form of the positional conv's weight norm under the legacy names (both fold to the same weight)"""
    p = "encoder.pos_conv.0."
    ren = {p + "parametrizations.weight.original0": p + "weight_g", p + "parametrizations.weight.original1": p + "weight_v"}
    return {ren.get(k, k): v for k, v in sd.items()}


class ContentVec(_lib.EngineModule):
    _prefix, _cfg_struct, _requirement = "ns2vc_cv_", _lib.CvCfg, "this content encoder needs fp32 parameters on {device}"

    def __init__(self, conv_dim: int = 512, embed_dim: int = 768, ffn_dim: int = 3072, num_layers: int = 12, num_heads: int = 12,
                 pos_conv_kernel: int = 128, pos_conv_groups: int = 16, final_dim: int = 256) -> None:
        super().__init__()
        self.cfg = dict(conv_dim=conv_dim, embed_dim=embed_dim, ffn_dim=ffn_dim, num_layers=num_layers, num_heads=num_heads,
                        pos_conv_kernel=pos_conv_kernel, pos_conv_groups=pos_conv_groups, final_dim=final_dim)
        for key, shape in contentvec_param_shapes(**self.cfg).items():
            init = torch.ones(shape) if key.endswith(("norm.weight", "conv_layers.0.2.weight", "weight_g")) else torch.zeros(shape)
            _insert(self, key, nn.Parameter(init))

    # ------------------------------------------------------------------ loading
    @classmethod
    def from_state_dict(cls, sd: Dict[str, torch.Tensor], num_heads: int = 12) -> "ContentVec":
        """A ``ContentVec`` with the weights of ``sd`` (``torch.load(ckpt)["model"]`` of a fairseq HubertModel; mask_emb /
        label_embs_concat are accepted and not loaded).  The configuration is read off the shapes (the head count is not in
        them).  A missing, unexpected or mis-shaped key raises ValueError naming it, and so do the "layer_norm" extractor mode
        and conv biases."""
        sd = _norm_keys({k: v for k, v in sd.items() if k not in TRAINING_ONLY})
        for k in sd:
            if k.startswith("feature_extractor.conv_layers.") and ".2.1." in k:
                raise ValueError(f"{k}: the 'layer_norm' extractor mode is not supported (ContentVec uses 'default')")
            if k.startswith("feature_extractor.conv_layers.") and k.endswith(".0.bias"):
                raise ValueError(f"{k}: conv biases (conv_bias=True) are not supported")

        def need(k):
            if k not in sd:
                raise ValueError(f"missing key {k} in the HubertModel state_dict")
            return sd[k]
        conv_dim = need("feature_extractor.conv_layers.0.0.weight").shape[0]
        embed_dim = need("post_extract_proj.weight").shape[0]
        v = need("encoder.pos_conv.0.weight_v")
        num_layers = 0
        while f"encoder.layers.{num_layers}.fc1.weight" in sd:
            num_layers += 1
        ffn_dim = need("encoder.layers.0.fc1.weight").shape[0] if num_layers else 4 * embed_dim
        final_dim = need("final_proj.weight").shape[0]
        groups = embed_dim // v.shape[1] if v.dim() == 3 and v.shape[1] else 1
        m = cls(int(conv_dim), int(embed_dim), int(ffn_dim), num_layers, int(num_heads), int(v.shape[-1]), int(groups), int(final_dim))
        return m._load_checked(sd, "HubertModel")

    @classmethod
    def from_fairseq(cls, obj) -> "ContentVec":
        """The drop-in for a fairseq ``HubertModel`` object (``svc.hubert_model``): its weights, on the device of its parameters.
        Only the post-LN encoder (``layer_norm_first = False``) exists here."""
        enc = obj.encoder
        if getattr(enc, "layer_norm_first", False):
            raise ValueError("encoder.layer_norm_first = True: only the post-LN encoder (ContentVec, HuBERT-base) is supported")
        heads = getattr(enc.layers[0].self_attn, "num_heads", 12) if hasattr(enc, "layers") and len(enc.layers) else 12
        sd = obj.state_dict()
        m = cls.from_state_dict(sd, num_heads=int(heads))
        dev = sd["final_proj.weight"].device
        return m.to(dev)

    @staticmethod
    def num_frames(n: int) -> int:
        return num_frames(n)

    def _lengths(self, lengths, B: int, N: int, dev: torch.device) -> Optional[torch.Tensor]:
        if lengths is None:
            return None
        t = torch.as_tensor(lengths)
        if not torch.cuda.is_current_stream_capturing():       # (under capture the engine clamps into [400, N] instead)
            lv = t.tolist()
            if t.dim() != 1 or len(lv) != B:
                raise ValueError(f"lengths must have {B} entries, got shape {tuple(t.shape)}")
            for b, n in enumerate(lv):
                if not MIN_SAMPLES <= int(n) <= N:
                    raise ValueError(f"lengths[{b}] = {n}: each row needs {MIN_SAMPLES} .. {N} samples (under {MIN_SAMPLES} gives no frame)")
        return t.to(dev, torch.int64).contiguous()

    # ------------------------------------------------------------------ API
    def extract(self, wav: torch.Tensor, lengths=None) -> Tuple[torch.Tensor, torch.Tensor]:
        """16 kHz waveforms wav [B, N] (CUDA) -> (units [B, T, final_dim] fp32 with T = num_frames(N), frames [B] int64).  With
        ``lengths`` [B] (each in [400, N]) row b equals the utterance wav[b, :lengths[b]] run alone: its frames >= frames[b] are 0
        and its samples >= lengths[b] are never read."""
        if not wav.is_cuda:
            raise RuntimeError("ns2vc_b200.content.ContentVec has no CPU path: move the module and inputs to an H100 ('cuda')")
        if torch.is_grad_enabled() and (wav.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise RuntimeError("this content encoder runs inference only: call extract under torch.no_grad()")
        if wav.dim() != 2:
            raise ValueError(f"wav must be [B, N], got {tuple(wav.shape)}")
        B, N = wav.shape
        if N < MIN_SAMPLES:
            raise ValueError(f"wav has {N} samples: at least {MIN_SAMPLES} are needed for one frame")
        dev = wav.device
        x = wav.to(torch.float32).contiguous()
        lens = self._lengths(lengths, B, N, dev)
        h = self.engine(dev)
        ws = self.workspace(B, N, dev)
        units = torch.empty((B, num_frames(N), self.cfg["final_dim"]), dtype=torch.float32, device=dev)
        frames = torch.empty((B,), dtype=torch.int64, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().ns2vc_cv_extract(h, x.data_ptr(), N, None if lens is None else lens.data_ptr(), units.data_ptr(),
                                                   frames.data_ptr(), B, N, ws.data_ptr(), stream))
        return units, frames

    def forward(self, wav: torch.Tensor, lengths=None):
        return self.extract(wav, lengths)

    # diagnostics for the parity tests -------------------------------------------------------
    @torch.no_grad()
    def taps(self, wav: torch.Tensor, lengths=None) -> Dict[str, torch.Tensor]:
        """Activations of one ``extract`` (token-major [B, T_stage, C]) under the oracle's stage names, plus ``"units"``."""
        B, _ = wav.shape
        self.extract(wav, lengths)                               # builds the program for this shape
        (units, frames), bufs = self._collect_taps(wav.device, B, lambda: self.extract(wav, lengths))
        bufs["units"], bufs["frames"] = units, frames
        return bufs


def get_hubert_content(model: ContentVec, wav_16k_tensor: torch.Tensor) -> torch.Tensor:
    """Drop-in for the reference's ``utils.get_hubert_content(hmodel, wav_16k_tensor)``: a 2-D input is averaged over its last
    dimension; returns the units [1, final_dim, T] on the input's device."""
    feats = wav_16k_tensor
    if feats.dim() == 2:
        feats = feats.mean(-1)
    assert feats.dim() == 1, feats.dim()
    dev = next(model.parameters()).device
    with torch.no_grad():
        units, _ = model.extract(feats.reshape(1, -1).to(dev, torch.float32))
    return units.transpose(1, 2).to(wav_16k_tensor.device)
