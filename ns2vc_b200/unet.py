"""``UNet1DConditionModel`` — drop-in for the reference's ``unet1d/unet_1d_condition.py`` class.

Same constructor keywords (``unet_1d_condition.py:151-203``), same ``state_dict`` key names and
shapes (SURVEY.md Appendix B), same ``forward`` signature and ``UNet1DConditionOutput(.sample)``
return (``:743-757, 1034-1037``).  The math runs in the sm_90a engine behind the C-ABI
(``include/ns2vc_b200.h``); this module only owns the parameters and marshals pointers.

There is NO CPU fallback: a forward on CPU tensors, or without the built extension, raises.
Autograd through the fused kernels is not implemented yet (SURVEY.md §8f rank 2); a forward
that would need gradients raises instead of silently detaching.
"""
from __future__ import annotations

import math
import threading
from collections import OrderedDict
from dataclasses import dataclass, fields
from typing import Any, Dict, Optional, Tuple, Union

import torch
import torch.nn as nn

from . import _lib
from .arch import UNetConfig, build_plan, param_shapes


class BaseOutput(OrderedDict):
    """Minimal stand-in for the reference's ``outputs.BaseOutput``: attribute + key + index access."""

    def __getitem__(self, k):
        if isinstance(k, str):
            return super().__getitem__(k)
        return tuple(self.values())[k]

    def to_tuple(self):
        return tuple(self.values())


class UNet1DConditionOutput(BaseOutput):
    def __init__(self, sample: torch.Tensor = None):
        super().__init__()
        self["sample"] = sample

    @property
    def sample(self) -> torch.Tensor:
        return self["sample"]


class _Node(nn.Module):
    """Parameter container; children are created on demand from dotted state_dict keys."""


def _insert(root: nn.Module, key: str, p: nn.Parameter) -> None:
    parts = key.split(".")
    mod = root
    i = 0
    while i < len(parts) - 1:
        name = parts[i]
        nxt = parts[i + 1]
        if nxt.isdigit() and i + 1 < len(parts) - 1:
            lst = getattr(mod, name, None)
            if lst is None:
                lst = nn.ModuleList()
                setattr(mod, name, lst)
            idx = int(nxt)
            while len(lst) <= idx:
                lst.append(_Node())
            mod = lst[idx]
            i += 2
        else:
            child = getattr(mod, name, None)
            if child is None:
                child = _Node()
                setattr(mod, name, child)
            mod = child
            i += 1
    mod.register_parameter(parts[-1], p)


_trace = threading.local()


class trace_calls:
    """Context manager used by the fused samplers to observe which denoiser calls a model closure
    makes (see ``fused.py``)."""

    def __enter__(self):
        self.prev = getattr(_trace, "records", None)
        _trace.records = []
        return _trace.records

    def __exit__(self, *exc):
        _trace.records = self.prev
        return False


@dataclass
class CallRecord:
    unet: "UNet1DConditionModel"
    sample: torch.Tensor
    timesteps: torch.Tensor
    ehs: torch.Tensor
    mask: Optional[torch.Tensor]
    output: torch.Tensor


class UNet1DConditionModel(_lib.EngineModule):
    _prefix, _cfg_struct = "ns2vc_unet_", _lib.UNetCfg
    _requirement = "this denoiser needs fp32 parameters on {device} (module.to('cuda'))"

    def __init__(
        self,
        sample_size: Optional[int] = None,
        in_channels: int = 4,
        out_channels: int = 4,
        center_input_sample: bool = False,
        flip_sin_to_cos: bool = True,
        freq_shift: int = 0,
        down_block_types: Tuple[str, ...] = ("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"),
        mid_block_type: Optional[str] = "UNetMidBlock2DCrossAttn",
        up_block_types: Tuple[str, ...] = ("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D"),
        only_cross_attention: Union[bool, Tuple[bool, ...]] = False,
        block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280),
        layers_per_block: Union[int, Tuple[int, ...]] = 2,
        downsample_padding: int = 1,
        mid_block_scale_factor: float = 1,
        act_fn: str = "silu",
        norm_num_groups: Optional[int] = 32,
        norm_eps: float = 1e-5,
        cross_attention_dim: Union[int, Tuple[int, ...]] = 1280,
        transformer_layers_per_block: Union[int, Tuple[int, ...]] = 1,
        encoder_hid_dim: Optional[int] = None,
        encoder_hid_dim_type: Optional[str] = None,
        attention_head_dim: Union[int, Tuple[int, ...]] = 8,
        num_attention_heads: Optional[Union[int, Tuple[int, ...]]] = None,
        dual_cross_attention: bool = False,
        use_linear_projection: bool = False,
        class_embed_type: Optional[str] = None,
        addition_embed_type: Optional[str] = None,
        addition_time_embed_dim: Optional[int] = None,
        num_class_embeds: Optional[int] = None,
        upcast_attention: bool = False,
        resnet_time_scale_shift: str = "default",
        resnet_skip_time_act: bool = False,
        resnet_out_scale_factor: float = 1.0,
        time_embedding_type: str = "positional",
        time_embedding_dim: Optional[int] = None,
        time_embedding_act_fn: Optional[str] = None,
        timestep_post_act: Optional[str] = None,
        time_cond_proj_dim: Optional[int] = None,
        conv_in_kernel: int = 3,
        conv_out_kernel: int = 3,
        projection_class_embeddings_input_dim: Optional[int] = None,
        class_embeddings_concat: bool = False,
        mid_block_only_cross_attention: Optional[bool] = None,
        cross_attention_norm: Optional[str] = None,
        addition_embed_type_num_heads: int = 64,
        latent_channels: Optional[int] = None,
    ):
        super().__init__()
        self.sample_size = sample_size
        if num_attention_heads is not None:
            raise ValueError(
                "At the moment it is not possible to define the number of attention heads via `num_attention_heads` "
                "because of a naming issue (reference unet_1d_condition.py:208-211).")
        num_attention_heads = attention_head_dim

        def _only(name, val, allowed):
            if val not in allowed:
                raise ValueError(f"`{name}`={val!r} is not supported by this denoiser (supported: {allowed})")

        n = len(block_out_channels)
        _only("center_input_sample", center_input_sample, (False,))
        _only("only_cross_attention", only_cross_attention if isinstance(only_cross_attention, bool) else any(only_cross_attention), (False,))
        _only("downsample_padding", downsample_padding, (1,))
        _only("mid_block_scale_factor", mid_block_scale_factor, (1, 1.0))
        _only("act_fn", act_fn, ("silu", "swish"))
        _only("transformer_layers_per_block", transformer_layers_per_block if isinstance(transformer_layers_per_block, int) else max(transformer_layers_per_block), (1,))
        _only("encoder_hid_dim", encoder_hid_dim, (None,))
        _only("encoder_hid_dim_type", encoder_hid_dim_type, (None,))
        _only("dual_cross_attention", dual_cross_attention, (False,))
        _only("use_linear_projection", use_linear_projection, (False,))
        _only("class_embed_type", class_embed_type, (None,))
        _only("num_class_embeds", num_class_embeds, (None,))
        _only("upcast_attention", upcast_attention, (False,))
        _only("resnet_skip_time_act", resnet_skip_time_act, (False,))
        _only("resnet_out_scale_factor", resnet_out_scale_factor, (1, 1.0))
        _only("time_embedding_type", time_embedding_type, ("positional",))
        _only("time_embedding_dim", time_embedding_dim, (None,))
        _only("time_embedding_act_fn", time_embedding_act_fn, (None,))
        _only("timestep_post_act", timestep_post_act, (None,))
        _only("time_cond_proj_dim", time_cond_proj_dim, (None,))
        _only("conv_in_kernel", conv_in_kernel, (3,))
        _only("conv_out_kernel", conv_out_kernel, (3,))
        _only("class_embeddings_concat", class_embeddings_concat, (False,))
        _only("cross_attention_norm", cross_attention_norm, (None,))
        if norm_num_groups is None:
            raise ValueError("`norm_num_groups`=None is not supported by this denoiser")
        if not isinstance(num_attention_heads, int):
            if len(set(num_attention_heads)) != 1:
                raise ValueError("per-block `attention_head_dim` tuples must be uniform")
            num_attention_heads = num_attention_heads[0]
        if not isinstance(cross_attention_dim, int):
            if len(set(cross_attention_dim)) != 1:
                raise ValueError("per-block `cross_attention_dim` tuples must be uniform")
            cross_attention_dim = cross_attention_dim[0]

        self.cfg = UNetConfig(
            in_channels=in_channels, out_channels=out_channels, block_out_channels=tuple(block_out_channels),
            down_block_types=tuple(down_block_types), mid_block_type=mid_block_type, up_block_types=tuple(up_block_types),
            layers_per_block=layers_per_block, norm_num_groups=norm_num_groups, norm_eps=norm_eps,
            cross_attention_dim=cross_attention_dim, num_heads=num_attention_heads,
            addition_embed_type=addition_embed_type, addition_embed_type_num_heads=addition_embed_type_num_heads,
            resnet_time_scale_shift=resnet_time_scale_shift, flip_sin_to_cos=flip_sin_to_cos, freq_shift=freq_shift)
        for i, t in enumerate(self.cfg.down_block_types):
            if (t == "DownBlock2D") != (self.cfg.up_block_types[n - 1 - i] == "UpBlock2D"):
                raise ValueError("down/up block types must mirror each other (reference default layout)")
        # conv_in channel split: Diffusion_Encoder builds in_channels = latent + hidden and
        # cross_attention_dim = hidden (reference model.py:391-397); the hidden (content) share is
        # step-invariant and its conv_in contribution is hoisted by the fused samplers.
        if latent_channels is None:
            latent_channels = in_channels - cross_attention_dim if in_channels > cross_attention_dim else in_channels
        self.latent_channels = int(latent_channels)

        # `.config` mirrors the reference's registered config dict (:561-607)
        self.config = dict(
            sample_size=sample_size, in_channels=in_channels, out_channels=out_channels, center_input_sample=center_input_sample,
            flip_sin_to_cos=flip_sin_to_cos, freq_shift=freq_shift, down_block_types=tuple(down_block_types),
            mid_block_type=mid_block_type, up_block_types=tuple(up_block_types), only_cross_attention=[False] * n,
            block_out_channels=tuple(block_out_channels), layers_per_block=list(self.cfg.layers_per_block),
            downsample_padding=downsample_padding, mid_block_scale_factor=mid_block_scale_factor, act_fn=act_fn,
            norm_num_groups=norm_num_groups, norm_eps=norm_eps, cross_attention_dim=(cross_attention_dim,) * n,
            transformer_layers_per_block=[1] * n, encoder_hid_dim=None, encoder_hid_dim_type=None,
            attention_head_dim=(attention_head_dim,) * n if isinstance(attention_head_dim, int) else tuple(attention_head_dim),
            num_attention_heads=(num_attention_heads,) * n, dual_cross_attention=False, use_linear_projection=False,
            class_embed_type=None, addition_embed_type=addition_embed_type, addition_time_embed_dim=addition_time_embed_dim,
            num_class_embeds=None, upcast_attention=False, resnet_time_scale_shift=resnet_time_scale_shift,
            resnet_skip_time_act=False, resnet_out_scale_factor=resnet_out_scale_factor, time_embedding_type="positional",
            time_embedding_dim=None, time_embedding_act_fn=None, timestep_post_act=None, time_cond_proj_dim=None,
            conv_in_kernel=3, conv_out_kernel=3, projection_class_embeddings_input_dim=projection_class_embeddings_input_dim,
            class_embeddings_concat=False, mid_block_only_cross_attention=False, cross_attention_norm=None,
            addition_embed_type_num_heads=addition_embed_type_num_heads)

        # parameters, registered under the reference's key names with PyTorch-default initialisers
        shapes = param_shapes(self.cfg)
        for key, shape in shapes.items():
            owner, leaf = key.rsplit(".", 1)
            if key.endswith("positional_embedding"):
                t = torch.randn(shape) / math.sqrt(shape[-1])
            elif len(shape) == 1 and owner.split(".")[-1].startswith(("norm", "conv_norm_out")):
                t = torch.ones(shape) if leaf == "weight" else torch.zeros(shape)
            else:
                wshape = shapes[owner + ".weight"]
                fan_in = 1
                for d in wshape[1:]:
                    fan_in *= d
                bound = 1.0 / math.sqrt(fan_in)
                t = torch.empty(shape).uniform_(-bound, bound)
            _insert(self, key, nn.Parameter(t))

    # ------------------------------------------------------------------ engine management
    def _c_cfg(self) -> _lib.UNetCfg:
        cfg = self.cfg
        c = self._cfg_struct()
        c.in_channels, c.latent_channels, c.out_channels = cfg.in_channels, self.latent_channels, cfg.out_channels
        c.n_levels = len(cfg.block_out_channels)
        n = c.n_levels
        for i in range(n):
            c.block_out_channels[i] = cfg.block_out_channels[i]
            c.layers_per_block[i] = cfg.layers_per_block[i]
            c.down_has_attn[i] = int(cfg.down_block_types[i] == "CrossAttnDownBlock2D")
            c.up_has_attn[i] = int(cfg.up_block_types[i] == "CrossAttnUpBlock2D")
        c.num_heads, c.cross_attention_dim = cfg.num_heads, cfg.cross_attention_dim
        c.norm_num_groups, c.norm_eps = cfg.norm_num_groups, cfg.norm_eps
        c.time_scale_shift = int(cfg.resnet_time_scale_shift == "scale_shift")
        c.add_embed_text = int(cfg.addition_embed_type == "text")
        c.add_embed_heads = cfg.addition_embed_type_num_heads
        c.flip_sin_to_cos, c.freq_shift = int(cfg.flip_sin_to_cos), float(cfg.freq_shift)
        return c

    def plan_string(self) -> str:
        return "".join(f"{o.kind}|{o.prefix}|{o.cin}|{o.cout}|{o.level}\n" for o in build_plan(self.cfg))

    # ------------------------------------------------------------------ forward
    def forward(
        self,
        sample: torch.FloatTensor,
        timestep: Union[torch.Tensor, float, int],
        encoder_hidden_states: torch.Tensor,
        class_labels: Optional[torch.Tensor] = None,
        timestep_cond: Optional[torch.Tensor] = None,
        attention_mask: Optional[torch.Tensor] = None,
        cross_attention_kwargs: Optional[Dict[str, Any]] = None,
        added_cond_kwargs: Optional[Dict[str, torch.Tensor]] = None,
        down_block_additional_residuals: Optional[Tuple[torch.Tensor]] = None,
        mid_block_additional_residual: Optional[torch.Tensor] = None,
        encoder_attention_mask: Optional[torch.Tensor] = None,
        return_dict: bool = True,
    ) -> Union[UNet1DConditionOutput, Tuple]:
        for name, v in (("class_labels", class_labels), ("timestep_cond", timestep_cond), ("attention_mask", attention_mask),
                        ("cross_attention_kwargs", cross_attention_kwargs), ("added_cond_kwargs", added_cond_kwargs),
                        ("down_block_additional_residuals", down_block_additional_residuals),
                        ("mid_block_additional_residual", mid_block_additional_residual)):
            if v is not None and not (isinstance(v, dict) and not v):
                raise NotImplementedError(f"`{name}` is not supported by this denoiser")
        if not sample.is_cuda:
            raise RuntimeError("ns2vc_b200.UNet1DConditionModel has no CPU path: move the module and inputs to an H100 ('cuda')")
        if torch.is_grad_enabled() and (sample.requires_grad or encoder_hidden_states.requires_grad
                                        or any(p.requires_grad for p in self.parameters())):
            raise NotImplementedError(
                "backward through the fused sm_90a denoiser is not implemented yet; call under torch.no_grad() "
                "(inference) — training is tracked as SURVEY.md §8(f) rank 2")
        dev = sample.device
        if sample.dim() != 3 or sample.shape[1] != self.cfg.in_channels:
            raise ValueError(f"sample must be [B, {self.cfg.in_channels}, T], got {tuple(sample.shape)}")
        B, _, T = sample.shape
        if encoder_hidden_states.dim() != 3 or encoder_hidden_states.shape[0] != B or encoder_hidden_states.shape[2] != self.cfg.cross_attention_dim:
            raise ValueError(f"encoder_hidden_states must be [B, S, {self.cfg.cross_attention_dim}], got {tuple(encoder_hidden_states.shape)}")
        S = encoder_hidden_states.shape[1]

        # timestep normalisation, reference :825-839 (python number / 0-d / [B]; int or float)
        timesteps = timestep
        if not torch.is_tensor(timesteps):
            timesteps = torch.tensor([timesteps], dtype=torch.float64 if isinstance(timestep, float) else torch.int64, device=dev)
        elif timesteps.dim() == 0:
            timesteps = timesteps[None].to(dev)
        t32 = timesteps.to(dev).expand(B).to(torch.float32).contiguous()

        x = sample.to(torch.float32)
        if not x.is_contiguous():
            x = x.contiguous()
        ehs = encoder_hidden_states.to(torch.float32).contiguous()
        mask_u8 = None
        if encoder_attention_mask is not None:
            if encoder_attention_mask.shape != (B, S):
                raise ValueError(f"encoder_attention_mask must be [B, S]={B, S}, got {tuple(encoder_attention_mask.shape)}")
            # the reference converts with .to(sample.dtype): any non-zero float counts as its value;
            # NS2VC only ever passes bool masks (model.py:411)
            mask_u8 = encoder_attention_mask.to(torch.bool).to(torch.uint8).contiguous()

        L = _lib.lib()
        h = self.engine(dev)
        ws = self.workspace(B, T, S, dev)
        out = torch.empty((B, self.cfg.out_channels, T), dtype=torch.float32, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        Cl, Cin = self.latent_channels, self.cfg.in_channels
        content_ptr = x.data_ptr() + 4 * Cl * T if Cin > Cl else None
        with torch.cuda.device(dev):
            self.__dict__["_cond_owner"] = None
            _lib.check(L.ns2vc_unet_prepare_cond(h, content_ptr, Cin * T, ehs.data_ptr(),
                                                 mask_u8.data_ptr() if mask_u8 is not None else None, B, T, S, ws.data_ptr(), stream))
            _lib.check(L.ns2vc_unet_forward(h, x.data_ptr(), Cin * T, t32.data_ptr(), out.data_ptr(), B, T, S, ws.data_ptr(), stream))
        out = out.to(sample.dtype)
        recs = getattr(_trace, "records", None)
        if recs is not None:
            recs.append(CallRecord(self, sample, t32, encoder_hidden_states, encoder_attention_mask, out))
        if not return_dict:
            return (out,)
        return UNet1DConditionOutput(sample=out)
