"""``Pre_model`` — drop-in for the reference's condition encoders (``model.py:328-377``): ``ref_enc``
(``TextTimeEmbedding(100, 100, 1)``), ``PromptEncoder`` and ``PhoneEncoder`` (``model.py:98-190``, six
``EncSALayer`` each, ``operations.py:784-821``).  It is the step immediately BEFORE the denoiser
(SURVEY.md §8(f) rank 1): ``NaturalSpeech2.sample`` calls ``self.pre_model.infer(data)`` and hands the two
results to the sampler (``model.py:631-633, 666-668``).

Same constructor argument (the ``cfg`` dict with ``phoneme_encoder`` / ``prompt_encoder`` keyword sets), same
``state_dict`` key names and shapes (34 923 404 parameters for the shipped configuration, ``demo.ipynb:447``), same
``infer(data)`` / ``forward(data)`` signatures and return layouts (``[T, B, C]`` / ``[S, B, C]``).  The math runs in the
sm_90a engine behind the C-ABI (``include/ns2vc_b200.h``, ``csrc/pre_engine.cu``); this module owns the parameters and
marshals pointers.  No CPU path; inference only (the reference's training forward applies dropout and needs autograd).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Sequence, Tuple

import torch
import torch.nn as nn

from . import _lib
from .unet import _insert

N_HEADS = 8          # operations.py:961  EncSALayer(c, 8, ...)
FFN_KERNEL = 9       # operations.py:963
REF_DIM = 100        # model.py:340      TextTimeEmbedding(100, 100, 1)


def _enc_args(d: dict, default_hidden: int) -> Tuple[int, int, int, int]:
    """(in_channels, hidden_channels, out_channels, n_layers) with the reference's defaults (model.py:99-105, 151-157)."""
    return (int(d.get("in_channels", 128)), int(d.get("hidden_channels", default_hidden)), int(d.get("out_channels", 512)),
            int(d.get("n_layers", 6)))


def pre_param_shapes(cfg: dict) -> Dict[str, Tuple[int, ...]]:
    """Reference ``Pre_model(cfg).state_dict()`` key -> shape (compared with the C registry and the reference in tests)."""
    shapes: Dict[str, Tuple[int, ...]] = {}

    def encoder(p: str, cin: int, H: int, cout: int, L: int, spk: bool):
        F = 4 * H
        for i in range(L):
            b = f"{p}.layers.{i}.op"
            shapes[b + ".layer_norm1.weight"] = (H,); shapes[b + ".layer_norm1.bias"] = (H,)
            shapes[b + ".self_attn.in_proj_weight"] = (3 * H, H)
            shapes[b + ".self_attn.out_proj.weight"] = (H, H)
            shapes[b + ".layer_norm2.weight"] = (H,); shapes[b + ".layer_norm2.bias"] = (H,)
            for j in range(FFN_KERNEL):
                shapes[f"{b}.ffn.ffn_1.{j}.weight"] = (F, H)
                if j == 0:
                    shapes[f"{b}.ffn.ffn_1.{j}.bias"] = (F,)
            shapes[b + ".ffn.ffn_2.weight"] = (H, F); shapes[b + ".ffn.ffn_2.bias"] = (H,)

        def last_ln():
            shapes[p + ".layer_norm.weight"] = (cout,); shapes[p + ".layer_norm.bias"] = (cout,)

        if not spk:                     # registration order of the reference modules (model.py:118-123 vs 166-170)
            last_ln()
        shapes[p + ".pre.layer_norm.weight"] = (cin,); shapes[p + ".pre.layer_norm.bias"] = (cin,)
        shapes[p + ".pre.conv.weight"] = (1, cin, H); shapes[p + ".pre.conv.bias"] = (H,)
        shapes[p + ".out_proj.layer_norm.weight"] = (H,); shapes[p + ".out_proj.layer_norm.bias"] = (H,)
        shapes[p + ".out_proj.conv.weight"] = (1, H, cout); shapes[p + ".out_proj.conv.bias"] = (cout,)
        if spk:
            last_ln()
            shapes[p + ".spk_proj.weight"] = (H, REF_DIM, 1); shapes[p + ".spk_proj.bias"] = (H,)

    encoder("phoneme_encoder", *_enc_args(cfg["phoneme_encoder"], 512), True)
    encoder("prompt_encoder", *_enc_args(cfg["prompt_encoder"], 256), False)
    R = REF_DIM
    shapes["ref_enc.norm1.weight"] = (R,); shapes["ref_enc.norm1.bias"] = (R,)
    shapes["ref_enc.pool.positional_embedding"] = (1, R)
    for n in ("k_proj", "q_proj", "v_proj"):
        shapes[f"ref_enc.pool.{n}.weight"] = (R, R); shapes[f"ref_enc.pool.{n}.bias"] = (R,)
    shapes["ref_enc.proj.weight"] = (R, R); shapes["ref_enc.proj.bias"] = (R,)
    shapes["ref_enc.norm2.weight"] = (R,); shapes["ref_enc.norm2.bias"] = (R,)
    return shapes


@dataclass(eq=False)
class Voice:
    """A target voice encoded once by ``Pre_model.encode_voices``: everything the condition encoders derive from its prompt mel.
    ``spk`` [phone_hidden] is ``phoneme_encoder.spk_proj(ref_enc(mel))``, the one vector by which the voice enters the content
    encoder; ``prompt`` [S_v, prompt_out] is the prompt encoder's output.  Both live on the device of the ``Pre_model`` that
    encoded them, and only that module (on that device) may use them."""
    spk: torch.Tensor
    prompt: torch.Tensor
    pre_model: "Pre_model"

    @property
    def S_v(self) -> int:
        return int(self.prompt.shape[0])

    @property
    def device(self) -> torch.device:
        return self.prompt.device


class Pre_model(_lib.EngineModule):
    _prefix, _cfg_struct, _requirement = "ns2vc_pre_", _lib.PreCfg, "these condition encoders need fp32 parameters on {device}"

    def __init__(self, cfg: dict) -> None:
        super().__init__()
        self.cfg = cfg
        for name in ("phoneme_encoder", "prompt_encoder"):
            if not cfg[name].get("last_ln", True):
                raise NotImplementedError(f"{name}: last_ln=False is not supported by these condition encoders")
        shapes = pre_param_shapes(cfg)
        for key, shape in shapes.items():
            owner, leaf = key.rsplit(".", 1)
            tail = owner.rsplit(".", 1)[-1]
            if "norm" in tail and len(shape) == 1:
                t = torch.ones(shape) if leaf == "weight" else torch.zeros(shape)
            elif key.endswith("positional_embedding"):
                t = torch.randn(shape) / math.sqrt(shape[-1])
            elif key.endswith("conv.weight") and len(shape) == 3 and "spk_proj" not in key:     # ConvTBC [k, c_in, c_out]: model.py:80-84
                t = torch.randn(shape) * math.sqrt(4 * 0.8 / (shape[0] * shape[1]))
            elif leaf == "bias":
                t = torch.zeros(shape)
            else:
                fan_in = 1
                for d in shape[1:]:
                    fan_in *= d
                t = torch.empty(shape).uniform_(-1.0 / math.sqrt(fan_in), 1.0 / math.sqrt(fan_in))
            _insert(self, key, nn.Parameter(t))

    # ------------------------------------------------------------------ engine management
    def _c_cfg(self) -> "_lib.PreCfg":
        pi, ph, po, pl = _enc_args(self.cfg["phoneme_encoder"], 512)
        ri, rh, ro, rl = _enc_args(self.cfg["prompt_encoder"], 256)
        c = self._cfg_struct()
        c.phone_in, c.phone_hidden, c.phone_out, c.phone_layers = pi, ph, po, pl
        c.prompt_in, c.prompt_hidden, c.prompt_out, c.prompt_layers = ri, rh, ro, rl
        c.ref_dim, c.ref_heads, c.n_heads, c.ffn_kernel = REF_DIM, 1, N_HEADS, FFN_KERNEL
        return c

    # ------------------------------------------------------------------ reference API
    @torch.no_grad()
    def infer(self, data, auto_predict_f0=None, per_utterance: bool = False):
        """``Pre_model.infer`` (model.py:360-377): data = (c_padded [B, C, T], refer_padded [B, 100, S], f0, spec, wav, lengths [B],
        refer_lengths [B], uv) -> (content [T, B, C_out], audio_prompt [S, B, C_out]); frames past a length are exactly zero.

        The default runs the padded batch as the reference does: ``ref_enc`` pools over all S prompt frames and the conv-FFN of
        a short row reads the batch's padding.  ``per_utterance=True`` runs a ragged batch instead: row b equals ``infer`` of
        ``c_padded[b:b+1, :, :lengths[b]]``, ``refer_padded[b:b+1, :, :refer_lengths[b]]`` alone, and input values past the
        lengths (which must lie in [1, T] / [1, S]) are never read."""
        c_padded, refer_padded, _f0, _spec, _wav, lengths, refer_lengths, _uv = data
        if not c_padded.is_cuda:
            raise RuntimeError("ns2vc_b200.Pre_model has no CPU path: move the module and inputs to an H100 ('cuda')")
        dev = c_padded.device
        pi, _ph, po, _pl = _enc_args(self.cfg["phoneme_encoder"], 512)
        ri, _rh, ro, _rl = _enc_args(self.cfg["prompt_encoder"], 256)
        if c_padded.dim() != 3 or c_padded.shape[1] != pi:
            raise ValueError(f"c_padded must be [B, {pi}, T], got {tuple(c_padded.shape)}")
        B, _, T = c_padded.shape
        if refer_padded.dim() == 3 and refer_padded.shape[0] == 1 and B > 1:
            # one prompt for the whole batch: the reference's encoders broadcast it (`sample()` even cuts a 2-row prompt down to its
            # first row, model.py:610-611); row-wise that is the same prompt repeated
            refer_padded = refer_padded.expand(B, -1, -1)
        if refer_padded.dim() != 3 or refer_padded.shape[0] != B or refer_padded.shape[1] != ri:
            raise ValueError(f"refer_padded must be [B, {ri}, S], got {tuple(refer_padded.shape)}")
        S = refer_padded.shape[2]
        c = c_padded.to(torch.float32).contiguous()
        refer = refer_padded.to(dev, torch.float32).contiguous()
        len_c = lengths.to(dev, torch.int64).contiguous()
        len_r = refer_lengths.to(dev, torch.int64).contiguous()
        if len_c.shape != (B,) or len_r.shape != (B,):
            raise ValueError("lengths / refer_lengths must be [B]")
        if per_utterance:
            from .fused import check_lengths
            check_lengths(lengths, B, T, "lengths")
            check_lengths(refer_lengths, B, S, "refer_lengths")
        L = _lib.lib()
        h = self.engine(dev)
        ws = self.workspace(B, T, S, dev)
        content = torch.empty((B, T, po), dtype=torch.float32, device=dev)
        prompt = torch.empty((B, S, ro), dtype=torch.float32, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        run = L.ns2vc_pre_infer_ragged if per_utterance else L.ns2vc_pre_infer
        with torch.cuda.device(dev):
            _lib.check(run(h, c.data_ptr(), refer.data_ptr(), len_c.data_ptr(), len_r.data_ptr(), content.data_ptr(),
                                         prompt.data_ptr(), B, T, S, ws.data_ptr(), stream))
        # the reference's layouts are the [T, B, C] / [S, B, C] views of the same values (model.py:147, 189)
        return content.transpose(0, 1).to(c_padded.dtype), prompt.transpose(0, 1).to(c_padded.dtype)

    def voice_widths(self) -> Tuple[int, int]:
        """(phone_hidden, prompt_out): the widths of a ``Voice``'s ``spk`` and ``prompt`` rows."""
        return _enc_args(self.cfg["phoneme_encoder"], 512)[1], _enc_args(self.cfg["prompt_encoder"], 256)[2]

    def check_voice(self, v, device: torch.device, what: str = "voice") -> Voice:
        """``v`` if it is a ``Voice`` this module encoded on ``device``; ValueError otherwise."""
        ph, ro = self.voice_widths()
        if not isinstance(v, Voice):
            raise ValueError(f"{what}: expected a Voice, got {type(v).__name__}")
        if v.pre_model is not self:
            raise ValueError(f"{what}: this Voice was encoded by another Pre_model")
        if v.spk.device != device or v.prompt.device != device:
            raise ValueError(f"{what}: this Voice lives on {v.device}, the call runs on {device}")
        if tuple(v.spk.shape) != (ph,) or v.prompt.dim() != 2 or v.prompt.shape[1] != ro or v.S_v < 1:
            raise ValueError(f"{what}: expected spk [{ph}] and prompt [S_v >= 1, {ro}], got {tuple(v.spk.shape)} and {tuple(v.prompt.shape)}")
        return v

    @torch.no_grad()
    def encode_voices(self, refer: torch.Tensor, refer_lengths: torch.Tensor) -> List[Voice]:
        """The voice half of ``infer(per_utterance=True)``: refer [B, 100, S] (mel prompts, zero-padded), refer_lengths [B] in
        [1, S] -> one ``Voice`` per row, whose ``prompt`` is row b of ``infer``'s prompt output cut to S_b frames and whose
        ``spk`` is the speaker vector its content rows add; both equal those of the fused call byte for byte."""
        if not refer.is_cuda:
            raise RuntimeError("ns2vc_b200.Pre_model has no CPU path: move the module and inputs to an H100 ('cuda')")
        dev = refer.device
        _pi, ph, _po, _pl = _enc_args(self.cfg["phoneme_encoder"], 512)
        ri, _rh, ro, _rl = _enc_args(self.cfg["prompt_encoder"], 256)
        if refer.dim() != 3 or refer.shape[1] != ri:
            raise ValueError(f"refer must be [B, {ri}, S], got {tuple(refer.shape)}")
        B, _, S = refer.shape
        from .fused import check_lengths
        sl = check_lengths(refer_lengths, B, S, "refer_lengths")
        ref = refer.to(torch.float32).contiguous()
        len_r = refer_lengths.to(dev, torch.int64).contiguous()
        h = self.engine(dev)
        ws = self.workspace(B, 1, S, dev)
        spk = torch.empty((B, ph), dtype=torch.float32, device=dev)
        prompt = torch.empty((B, S, ro), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().ns2vc_pre_encode_voices_ragged(h, ref.data_ptr(), len_r.data_ptr(), spk.data_ptr(), prompt.data_ptr(),
                                                                 B, S, ws.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
        return [Voice(spk[b], prompt[b, :int(sl[b])], self) for b in range(B)]

    @torch.no_grad()
    def infer_content(self, c: torch.Tensor, lengths: torch.Tensor, voices: Sequence[Voice]) -> torch.Tensor:
        """The content half of ``infer(per_utterance=True)``: c [B, C, T] (stretched ContentVec units), lengths [B] in [1, T] and
        row b's ``Voice`` -> content [T, B, C_out], row b equal byte for byte to ``infer``'s content row for that voice's prompt
        mel; frames past T_b are exactly 0."""
        dev = c.device
        voices = [self.check_voice(v, dev, f"voice {b}") for b, v in enumerate(voices)]
        if not c.is_cuda:
            raise RuntimeError("ns2vc_b200.Pre_model has no CPU path: move the module and inputs to an H100 ('cuda')")
        pi, _ph, po, _pl = _enc_args(self.cfg["phoneme_encoder"], 512)
        if c.dim() != 3 or c.shape[1] != pi:
            raise ValueError(f"c must be [B, {pi}, T], got {tuple(c.shape)}")
        B, _, T = c.shape
        if len(voices) != B:
            raise ValueError(f"{len(voices)} voices for {B} rows")
        from .fused import check_lengths
        check_lengths(lengths, B, T, "lengths")
        cc = c.to(torch.float32).contiguous()
        len_c = lengths.to(dev, torch.int64).contiguous()
        spk = torch.stack([v.spk for v in voices]).contiguous()
        h = self.engine(dev)
        ws = self.workspace(B, T, 1, dev)
        content = torch.empty((B, T, po), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().ns2vc_pre_infer_content_ragged(h, cc.data_ptr(), len_c.data_ptr(), spk.data_ptr(), content.data_ptr(),
                                                                 B, T, ws.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
        return content.transpose(0, 1)

    def forward(self, data, g=None):
        """``Pre_model.forward`` (model.py:341-359) in eval mode: (content, audio_prompt, lf0, lf0_pred) with lf0 = lf0_pred = 0."""
        if self.training and torch.is_grad_enabled():
            raise NotImplementedError("these condition encoders run inference only (the reference's training forward applies "
                                      "dropout and needs autograd): call .eval() under torch.no_grad()")
        content, prompt = self.infer(data)
        return content, prompt, 0, 0

    # diagnostics for the parity tests -------------------------------------------------------
    def taps(self, data, per_utterance: bool = False) -> Dict[str, torch.Tensor]:
        """Per-layer activations of one ``infer`` (token-major [B, rows, C]; the speaker vector as [B, 1, 100])."""
        c_padded = data[0]
        self.infer(data, per_utterance=per_utterance)          # builds the program for this shape
        _, bufs = self._collect_taps(c_padded.device, c_padded.shape[0], lambda: self.infer(data, per_utterance=per_utterance))
        return bufs
