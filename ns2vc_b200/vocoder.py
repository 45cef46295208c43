"""``Vocos`` — drop-in for the vocoder the reference calls after sampling (``model.py:689-691``: ``vocos.to(audio.device);
audio = vocos.decode(audio)``), the ``charactr/vocos-mel-24khz`` configuration of the ``vocos`` package: ``VocosBackbone``
(``vocos/models.py``: Conv1d embed, LayerNorm, eight ``ConvNeXtBlock`` of ``vocos/modules.py``, final LayerNorm) and
``ISTFTHead`` (``vocos/heads.py``, the "same"-padded ISTFT of ``vocos/spectral_ops.py``).

Same parameter names and shapes as ``Vocos.state_dict()`` without the ``feature_extractor.*`` entries (the prompt mel is
``frontend.log_mel_spectrogram``), same ``decode(features_input)``.  ``decode`` also takes per-row ``lengths``: row b of a
padded batch is then decoded as if it were alone.  The math runs in the sm_90a engine behind the C-ABI
(``include/ns2vc_b200.h``, ``csrc/vocoder.cu``); this module owns the parameters and marshals pointers.  No CPU path;
inference only.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch
import torch.nn as nn

from . import _lib
from .fused import check_lengths
from .unet import _insert

KERNEL = 7           # embed and depthwise convs (vocos/models.py, vocos/modules.py)


def vocos_param_shapes(input_channels: int = 100, dim: int = 512, intermediate_dim: int = 1536, num_layers: int = 8,
                       n_fft: int = 1024) -> Dict[str, Tuple[int, ...]]:
    """``Vocos.state_dict()`` keys -> shapes after ``feature_extractor.*``, in its order (a module's own parameters before its
    children's: ``gamma`` leads each block)."""
    s: Dict[str, Tuple[int, ...]] = {}
    s["backbone.embed.weight"] = (dim, input_channels, KERNEL); s["backbone.embed.bias"] = (dim,)
    s["backbone.norm.weight"] = (dim,); s["backbone.norm.bias"] = (dim,)
    for i in range(num_layers):
        b = f"backbone.convnext.{i}"
        s[b + ".gamma"] = (dim,)
        s[b + ".dwconv.weight"] = (dim, 1, KERNEL); s[b + ".dwconv.bias"] = (dim,)
        s[b + ".norm.weight"] = (dim,); s[b + ".norm.bias"] = (dim,)
        s[b + ".pwconv1.weight"] = (intermediate_dim, dim); s[b + ".pwconv1.bias"] = (intermediate_dim,)
        s[b + ".pwconv2.weight"] = (dim, intermediate_dim); s[b + ".pwconv2.bias"] = (dim,)
    s["backbone.final_layer_norm.weight"] = (dim,); s["backbone.final_layer_norm.bias"] = (dim,)
    s["head.out.weight"] = (n_fft + 2, dim); s["head.out.bias"] = (n_fft + 2,)
    s["head.istft.window"] = (n_fft,)
    return s


def vocos_init(key: str, shape: Tuple[int, ...], num_layers: int, generator: Optional[torch.Generator] = None) -> torch.Tensor:
    """The package's initial value of one entry: trunc-normal std 0.02 conv / linear weights, zero biases (VocosBackbone
    ._init_weights), layer scale 1 / num_layers, LayerNorms 1 / 0, and the periodic Hann window of the ISTFT."""
    leaf = key.rsplit(".", 1)[-1]
    if key.endswith("istft.window"):
        return torch.hann_window(shape[0])
    if leaf == "gamma":
        return torch.full(shape, 1.0 / num_layers)
    if ".norm." in key or "final_layer_norm" in key:
        return torch.ones(shape) if leaf == "weight" else torch.zeros(shape)
    if leaf == "bias":
        return torch.zeros(shape)
    return torch.nn.init.trunc_normal_(torch.empty(shape), std=0.02, generator=generator)


class Vocos(_lib.EngineModule):
    _prefix, _cfg_struct, _requirement = "ns2vc_voc_", _lib.VocCfg, "this vocoder needs fp32 parameters on {device}"

    def __init__(self, input_channels: int = 100, dim: int = 512, intermediate_dim: int = 1536, num_layers: int = 8,
                 n_fft: int = 1024, hop_length: int = 256) -> None:
        super().__init__()
        if n_fft != 4 * hop_length:
            raise ValueError(f"n_fft {n_fft} must be 4 * hop_length ({hop_length})")
        self.cfg = dict(input_channels=input_channels, dim=dim, intermediate_dim=intermediate_dim, num_layers=num_layers,
                        n_fft=n_fft, hop_length=hop_length)
        for key, shape in vocos_param_shapes(input_channels, dim, intermediate_dim, num_layers, n_fft).items():
            # the window is a buffer in the package; here it is a frozen parameter, so that a change re-packs the engine
            _insert(self, key, nn.Parameter(vocos_init(key, shape, num_layers), requires_grad=not key.endswith("istft.window")))

    @property
    def hop_length(self) -> int:
        return self.cfg["hop_length"]

    # ------------------------------------------------------------------ loading
    @classmethod
    def from_state_dict(cls, sd: Dict[str, torch.Tensor], hop_length: int = 256) -> "Vocos":
        """A ``Vocos`` with the weights of ``sd`` (a ``Vocos.state_dict()``; ``feature_extractor.*`` entries are skipped).  The
        configuration is read off the shapes; a missing, unexpected or mis-shaped key raises ValueError naming it, and so does
        an AdaLayerNorm (the encodec variant)."""
        sd = {k: v for k, v in sd.items() if not k.startswith("feature_extractor.")}
        for k in sd:
            if k.endswith((".scale.weight", ".shift.weight")) and ".norm." in k:
                raise ValueError(f"{k}: AdaLayerNorm (the encodec variant of Vocos) is not supported")

        def need(k):
            if k not in sd:
                raise ValueError(f"missing key {k} in the Vocos state_dict")
            return sd[k]
        dim, input_channels = need("backbone.embed.weight").shape[:2]
        num_layers = 0
        while f"backbone.convnext.{num_layers}.dwconv.weight" in sd:
            num_layers += 1
        intermediate_dim = need("backbone.convnext.0.pwconv1.weight").shape[0] if num_layers else 3 * dim
        n_fft = need("head.out.weight").shape[0] - 2
        if n_fft != 4 * hop_length:
            raise ValueError(f"head.out.weight gives n_fft {n_fft}; with hop_length {hop_length} only n_fft = 4 * hop_length is supported")
        m = cls(int(input_channels), int(dim), int(intermediate_dim), num_layers, int(n_fft), int(hop_length))
        return m._load_checked(sd, "Vocos")

    @classmethod
    def from_vocos(cls, obj) -> "Vocos":
        """The drop-in for a ``vocos.Vocos`` object (``Vocos.from_pretrained("charactr/vocos-mel-24khz")``): its weights, its hop
        length, on the device of its parameters.  Only the "same" ISTFT padding exists here."""
        istft = obj.head.istft
        padding = getattr(istft, "padding", "same")
        if padding != "same":
            raise ValueError(f"head.istft.padding = {padding!r}: only the 'same' padding is supported")
        sd = obj.state_dict()
        m = cls.from_state_dict(sd, hop_length=int(istft.hop_length))
        dev = sd["head.out.weight"].device
        return m.to(dev)

    def _lengths(self, lengths, B: int, T: int, dev: torch.device) -> Optional[torch.Tensor]:
        if lengths is None:
            return None
        if not torch.cuda.is_current_stream_capturing():       # (under capture the engine clamps into [1, T] instead)
            check_lengths(lengths, B, T, "lengths")
        return torch.as_tensor(lengths).to(dev, torch.int64).contiguous()

    # ------------------------------------------------------------------ reference API
    def decode(self, features_input: torch.Tensor, lengths=None) -> torch.Tensor:
        """``Vocos.decode``: mel features [B, input_channels, T] (CUDA) -> audio [B, T * hop_length] fp32.  With ``lengths`` [B]
        (each in [1, T]) row b equals ``decode(features_input[b:b+1, :, :lengths[b]])`` and its samples >= lengths[b] * hop_length
        are 0; features past a length are never read."""
        if not features_input.is_cuda:
            raise RuntimeError("ns2vc_b200.vocoder.Vocos has no CPU path: move the module and inputs to an H100 ('cuda')")
        if torch.is_grad_enabled() and (features_input.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise RuntimeError("this vocoder runs inference only: call decode under torch.no_grad()")
        ci = self.cfg["input_channels"]
        if features_input.dim() != 3 or features_input.shape[1] != ci:
            raise ValueError(f"features_input must be [B, {ci}, T], got {tuple(features_input.shape)}")
        B, _, T = features_input.shape
        dev = features_input.device
        mel = features_input.to(torch.float32).contiguous()
        lens = self._lengths(lengths, B, T, dev)
        h = self.engine(dev)
        ws = self.workspace(B, T, dev)
        audio = torch.empty((B, T * self.hop_length), dtype=torch.float32, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().ns2vc_voc_decode(h, mel.data_ptr(), ci * T, None if lens is None else lens.data_ptr(), audio.data_ptr(),
                                                   B, T, ws.data_ptr(), stream))
        return audio

    def forward(self, audio_input, **kwargs):
        raise NotImplementedError("Vocos.forward runs the feature extractor, which this module does not replace: compute the mel with "
                                  "ns2vc_b200.frontend.log_mel_spectrogram and call decode()")

    # diagnostics for the parity tests -------------------------------------------------------
    @torch.no_grad()
    def istft(self, head_out: torch.Tensor, lengths=None) -> torch.Tensor:
        """The head's ISTFT stage alone: head_out [B, T, n_fft + 2] (log-magnitudes, then phases) -> audio [B, T * hop_length]."""
        B, T, N = head_out.shape
        if N != self.cfg["n_fft"] + 2 or not head_out.is_cuda:
            raise ValueError(f"head_out must be a CUDA [B, T, {self.cfg['n_fft'] + 2}] tensor, got {tuple(head_out.shape)}")
        dev = head_out.device
        x = head_out.to(torch.float32).contiguous()
        lens = self._lengths(lengths, B, T, dev)
        audio = torch.empty((B, T * self.hop_length), dtype=torch.float32, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().ns2vc_voc_istft(self.engine(dev), x.data_ptr(), None if lens is None else lens.data_ptr(),
                                                  audio.data_ptr(), B, T, stream))
        return audio

    @torch.no_grad()
    def taps(self, features_input: torch.Tensor, lengths=None) -> Dict[str, torch.Tensor]:
        """Activations of one ``decode`` (token-major [B, T, C]: after backbone.norm, each convnext block, final_layer_norm and
        head.out) plus its result under ``"audio"``."""
        B = features_input.shape[0]
        self.decode(features_input, lengths)                     # builds the program for this shape
        audio, bufs = self._collect_taps(features_input.device, B, lambda: self.decode(features_input, lengths))
        bufs["audio"] = audio
        bufs["head.out"] = bufs["head.out"][:, :, :self.cfg["n_fft"] + 2]
        return bufs
