"""Static description of the denoiser UNet1D: config normalisation, block plan and the
state_dict contract (key names + shapes).

This is the single place where the block structure of the reference's
``UNet1DConditionModel`` (reference ``unet1d/unet_1d_condition.py:151-560``, block factories
``unet1d/unet_1d_blocks.py:31,226``) is restated.  The Python module (``unet.py``), the CPU
oracle (``oracle/unet_oracle.py``) and the weight packer of the CUDA engine all derive their
layer lists from :func:`build_plan`, so they cannot drift apart.

Only the block types the reference's denoiser instantiates (``model.py:391-400``) are supported;
anything else is rejected loudly (SURVEY.md §8b).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

SUPPORTED_DOWN = ("CrossAttnDownBlock2D", "DownBlock2D")
SUPPORTED_UP = ("UpBlock2D", "CrossAttnUpBlock2D")
SUPPORTED_MID = ("UNetMidBlock2DCrossAttn",)


def _tup(v, n):
    if isinstance(v, (list, tuple)):
        if len(v) != n:
            raise ValueError(f"expected {n} entries, got {v!r}")
        return tuple(v)
    return (v,) * n


@dataclass
class UNetConfig:
    """Normalised constructor arguments (same names/defaults as the reference ctor,
    ``unet_1d_condition.py:151-203``)."""

    in_channels: int = 4
    out_channels: int = 4
    block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    down_block_types: Tuple[str, ...] = (
        "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D")
    mid_block_type: Optional[str] = "UNetMidBlock2DCrossAttn"
    up_block_types: Tuple[str, ...] = (
        "UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D")
    layers_per_block: Tuple[int, ...] = (2, 2, 2, 2)
    norm_num_groups: int = 32
    norm_eps: float = 1e-5
    cross_attention_dim: int = 1280
    num_heads: int = 8                      # reference: attention_head_dim reinterpreted (:219)
    addition_embed_type: Optional[str] = None
    addition_embed_type_num_heads: int = 64
    resnet_time_scale_shift: str = "default"
    flip_sin_to_cos: bool = True
    freq_shift: int = 0
    time_embed_dim: int = 0                 # filled in: 4 * block_out_channels[0]

    def __post_init__(self):
        n = len(self.block_out_channels)
        self.block_out_channels = tuple(int(c) for c in self.block_out_channels)
        self.down_block_types = tuple(self.down_block_types)
        self.up_block_types = tuple(self.up_block_types)
        self.layers_per_block = _tup(self.layers_per_block, n)
        if len(self.down_block_types) != len(self.up_block_types):
            raise ValueError("Must provide the same number of `down_block_types` as `up_block_types`.")
        if len(self.block_out_channels) != len(self.down_block_types):
            raise ValueError("Must provide the same number of `block_out_channels` as `down_block_types`.")
        for t in self.down_block_types:
            if t not in SUPPORTED_DOWN:
                raise ValueError(f"{t} is not supported by this denoiser (supported: {SUPPORTED_DOWN})")
        for t in self.up_block_types:
            if t not in SUPPORTED_UP:
                raise ValueError(f"{t} is not supported by this denoiser (supported: {SUPPORTED_UP})")
        if self.mid_block_type not in SUPPORTED_MID:
            raise ValueError(f"unknown mid_block_type : {self.mid_block_type}")
        if self.resnet_time_scale_shift not in ("default", "scale_shift"):
            raise ValueError(f"unknown time_embedding_norm : {self.resnet_time_scale_shift} ")
        if self.addition_embed_type not in (None, "text"):
            raise ValueError(f"addition_embed_type: {self.addition_embed_type} must be None or 'text'.")
        g = self.norm_num_groups
        for c in self.block_out_channels:
            if c % g or c % self.num_heads:
                raise ValueError(f"block width {c} must be divisible by groups {g} and heads {self.num_heads}")
        if not self.time_embed_dim:
            self.time_embed_dim = 4 * self.block_out_channels[0]


# ---------------------------------------------------------------------------------------------
# Block plan: a flat op list the oracle interprets and the CUDA engine mirrors (engine.cu builds
# the same list from the same config; tests compare the two).
# ---------------------------------------------------------------------------------------------
@dataclass
class Op:
    kind: str                      # 'resnet' | 'xformer' | 'down' | 'up' | 'push' | 'pop_cat'
    prefix: str = ""               # state_dict prefix, e.g. 'down_blocks.0.resnets.1'
    cin: int = 0
    cout: int = 0
    level: int = 0                 # resolution level of the OUTPUT of this op


def build_plan(cfg: UNetConfig) -> List[Op]:
    """Sequence of ops between conv_in and conv_norm_out (reference forward
    ``unet_1d_condition.py:943-1026`` + block forwards ``unet_1d_blocks.py:949-1016, 1071-1097,
    602-623, 2070-2131, 2182-2207``).  'push' records a skip tensor, 'pop_cat' concatenates the
    most recent skip after the running tensor along channels."""
    ops: List[Op] = [Op("push", level=0, cout=cfg.block_out_channels[0])]
    boc = cfg.block_out_channels
    n = len(boc)
    skip_ch: List[int] = [boc[0]]
    ch = boc[0]
    level = 0
    for i, btype in enumerate(cfg.down_block_types):
        cout = boc[i]
        for j in range(cfg.layers_per_block[i]):
            ops.append(Op("resnet", f"down_blocks.{i}.resnets.{j}", ch, cout, level))
            ch = cout
            if btype == "CrossAttnDownBlock2D":
                ops.append(Op("xformer", f"down_blocks.{i}.attentions.{j}", ch, ch, level))
            ops.append(Op("push", level=level, cout=ch))
            skip_ch.append(ch)
        if i != n - 1:
            level += 1
            ops.append(Op("down", f"down_blocks.{i}.downsamplers.0", ch, ch, level))
            ops.append(Op("push", level=level, cout=ch))
            skip_ch.append(ch)
    # mid
    ops.append(Op("resnet", "mid_block.resnets.0", ch, ch, level))
    ops.append(Op("xformer", "mid_block.attentions.0", ch, ch, level))
    ops.append(Op("resnet", "mid_block.resnets.1", ch, ch, level))
    # up
    rboc = list(reversed(boc))
    rlayers = list(reversed(cfg.layers_per_block))
    for i, btype in enumerate(cfg.up_block_types):
        cout = rboc[i]
        for j in range(rlayers[i] + 1):
            sk = skip_ch.pop()
            ops.append(Op("pop_cat", cin=ch, cout=ch + sk, level=level))
            ops.append(Op("resnet", f"up_blocks.{i}.resnets.{j}", ch + sk, cout, level))
            ch = cout
            if btype == "CrossAttnUpBlock2D":
                ops.append(Op("xformer", f"up_blocks.{i}.attentions.{j}", ch, ch, level))
        if i != n - 1:
            level -= 1
            ops.append(Op("up", f"up_blocks.{i}.upsamplers.0", ch, ch, level))
    assert not skip_ch and level == 0
    return ops


def level_lengths(T: int, n_levels: int) -> List[int]:
    """Sequence length per resolution level: conv k3 s2 p1 => floor((T-1)/2)+1
    (reference ``resnet.py:200``; SURVEY Appendix C)."""
    out = [T]
    for _ in range(n_levels - 1):
        out.append((out[-1] - 1) // 2 + 1)
    return out


def param_shapes(cfg: UNetConfig) -> "Dict[str, Tuple[int, ...]]":
    """state_dict contract: every key of the reference module with its shape, in the reference's
    registration order (SURVEY Appendix B; verified against the reference in
    oracle/make_golden.py)."""
    P: Dict[str, Tuple[int, ...]] = {}
    boc = cfg.block_out_channels
    c0 = boc[0]
    ted = cfg.time_embed_dim
    xd = cfg.cross_attention_dim

    def conv(p, co, ci, k):
        P[p + ".weight"] = (co, ci, k)
        P[p + ".bias"] = (co,)

    def lin(p, co, ci, bias=True):
        P[p + ".weight"] = (co, ci)
        if bias:
            P[p + ".bias"] = (co,)

    def norm(p, c):
        P[p + ".weight"] = (c,)
        P[p + ".bias"] = (c,)

    def resnet(p, ci, co):
        norm(p + ".norm1", ci)
        conv(p + ".conv1", co, ci, 3)
        lin(p + ".time_emb_proj", 2 * co if cfg.resnet_time_scale_shift == "scale_shift" else co, ted)
        norm(p + ".norm2", co)
        conv(p + ".conv2", co, co, 3)
        if ci != co:
            conv(p + ".conv_shortcut", co, ci, 1)

    def xformer(p, c):
        norm(p + ".norm", c)
        conv(p + ".proj_in", c, c, 1)
        b = p + ".transformer_blocks.0"
        norm(b + ".norm1", c)
        for w in ("to_q", "to_k", "to_v"):
            lin(f"{b}.attn1.{w}", c, c, bias=False)
        lin(b + ".attn1.to_out.0", c, c)
        norm(b + ".norm2", c)
        lin(b + ".attn2.to_q", c, c, bias=False)
        lin(b + ".attn2.to_k", c, xd, bias=False)
        lin(b + ".attn2.to_v", c, xd, bias=False)
        lin(b + ".attn2.to_out.0", c, c)
        norm(b + ".norm3", c)
        lin(b + ".ff.net.0.proj", 8 * c, c)
        lin(b + ".ff.net.2", c, 4 * c)
        conv(p + ".proj_out", c, c, 1)

    conv("conv_in", c0, cfg.in_channels, 3)
    lin("time_embedding.linear_1", ted, c0)
    lin("time_embedding.linear_2", ted, ted)
    if cfg.addition_embed_type == "text":
        norm("add_embedding.norm1", xd)
        P["add_embedding.pool.positional_embedding"] = (1, xd)
        for w in ("k_proj", "q_proj", "v_proj"):
            lin(f"add_embedding.pool.{w}", xd, xd)
        lin("add_embedding.proj", ted, xd)
        norm("add_embedding.norm2", ted)

    # The reference registers attentions before resnets inside each block, then resamplers;
    # down blocks, then up blocks, then mid block (module registration order).
    plan = build_plan(cfg)
    by_block: Dict[str, List[Op]] = {}
    for op in plan:
        if op.prefix:
            blk = ".".join(op.prefix.split(".")[:2]) if not op.prefix.startswith("mid_block") else "mid_block"
            by_block.setdefault(blk, []).append(op)
    order = [f"down_blocks.{i}" for i in range(len(boc))] + \
            [f"up_blocks.{i}" for i in range(len(boc))] + ["mid_block"]
    for blk in order:
        ops = by_block.get(blk, [])
        for op in ops:
            if op.kind == "xformer":
                xformer(op.prefix, op.cout)
        for op in ops:
            if op.kind == "resnet":
                resnet(op.prefix, op.cin, op.cout)
        for op in ops:
            if op.kind in ("down", "up"):
                conv(op.prefix + ".conv", op.cout, op.cin, 3)
    norm("conv_norm_out", c0)
    conv("conv_out", cfg.out_channels, c0, 3)
    return P


def ns2vc_denoiser_config(in_channels=100, hidden_channels=256, out_channels=100, n_heads=8) -> UNetConfig:
    """The fixed hyper-parameters of the reference's ``Diffusion_Encoder`` (``model.py:391-400``)."""
    return UNetConfig(
        in_channels=in_channels + hidden_channels, out_channels=out_channels,
        block_out_channels=(128, 256, 384, 512), norm_num_groups=8,
        cross_attention_dim=hidden_channels, num_heads=n_heads,
        addition_embed_type="text", resnet_time_scale_shift="scale_shift")
