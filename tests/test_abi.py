"""C-ABI library: loads, exports every symbol include/ns2vc_b200.h declares, host-only helpers are
bit-exact, the C++ layer plan equals the Python plan, and the Python drop-in exposes the reference's
state_dict contract.  No GPU compute here."""
import ctypes as C
import os
import re

import pytest
import torch

from conftest import REPO, tiny_config
from ns2vc_b200 import _lib
from ns2vc_b200.arch import build_plan, level_lengths, ns2vc_denoiser_config, param_shapes
from ns2vc_b200.unet import UNet1DConditionModel


def header_symbols():
    src = open(os.path.join(REPO, "include", "ns2vc_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(ns2vc_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    L = _lib.lib()
    syms = header_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(L, s), f"{s} declared in include/ns2vc_b200.h but not exported"
    assert set(syms) == set(_lib.SIGNATURES), set(syms) ^ set(_lib.SIGNATURES)
    assert b"sm_90a" in L.ns2vc_build_info()


def test_nearest_index_bit_exact(gold):
    L = _lib.lib()
    for (tin, tout), ref in gold("nearest_index.pt").items():
        buf = (C.c_int * tout)()
        assert L.ns2vc_nearest_index(tin, tout, buf) == 0
        assert list(buf) == ref.tolist(), (tin, tout)


def test_down_length_matches_conv_rule():
    L = _lib.lib()
    for t in (1, 2, 8, 17, 131, 1000, 1023, 1024):
        conv = torch.nn.functional.conv1d(torch.zeros(1, 1, t), torch.zeros(1, 1, 3), stride=2, padding=1).shape[-1]
        assert L.ns2vc_down_length(t) == conv
    assert level_lengths(131, 4) == [131, 66, 33, 17]
    assert level_lengths(1000, 4) == [1000, 500, 250, 125]


def _create(unet):
    L = _lib.lib()
    h = C.c_void_p()
    cfg = unet._c_cfg()
    _lib.check(L.ns2vc_unet_create(C.byref(cfg), C.byref(h)))
    return L, h


@pytest.mark.parametrize("which", ["tiny", "full", "lpb1"])
def test_engine_plan_and_weight_registry_match_python(which):
    if which == "tiny":
        c = tiny_config()
        kw = dict(in_channels=36, out_channels=20, block_out_channels=(32, 64, 64, 96), norm_num_groups=8, cross_attention_dim=16,
                  attention_head_dim=8, addition_embed_type="text", addition_embed_type_num_heads=4, resnet_time_scale_shift="scale_shift")
    else:
        c = ns2vc_denoiser_config()
        kw = dict(in_channels=356, out_channels=100, block_out_channels=(128, 256, 384, 512), norm_num_groups=8, cross_attention_dim=256,
                  attention_head_dim=8, addition_embed_type="text", resnet_time_scale_shift="scale_shift")
        if which == "lpb1":
            kw["layers_per_block"] = 1      # BASELINE config 1
    unet = UNet1DConditionModel(**kw)
    L, h = _create(unet)
    try:
        assert L.ns2vc_unet_plan_string(h).decode() == unet.plan_string()
        shapes = param_shapes(unet.cfg)
        assert L.ns2vc_unet_num_weights(h) == len(shapes)
        got = {}
        for i in range(len(shapes)):
            name, shp, nd = C.c_char_p(), (C.c_int64 * 4)(), C.c_int()
            _lib.check(L.ns2vc_unet_weight_info(h, i, C.byref(name), shp, C.byref(nd)))
            got[name.value.decode()] = tuple(shp[k] for k in range(nd.value))
        assert got == shapes
        assert list(unet.state_dict().keys()) == list(shapes.keys())
        assert all(tuple(v.shape) == shapes[k] for k, v in unet.state_dict().items())
    finally:
        L.ns2vc_unet_destroy(h)
    if which == "full":
        assert unet.latent_channels == 100
        assert sum(p.numel() for p in unet.parameters()) == 66076900
        assert unet.config["addition_embed_type"] == "text" and unet.config["center_input_sample"] is False


def test_errors_are_reported_not_swallowed():
    L = _lib.lib()
    unet = UNet1DConditionModel(in_channels=36, out_channels=20, block_out_channels=(32, 64, 64, 96), norm_num_groups=8,
                                cross_attention_dim=16, attention_head_dim=8)
    L, h = _create(unet)
    try:
        n = C.c_size_t()
        rc = L.ns2vc_unet_workspace_bytes(h, 1, 16, 4, C.byref(n))     # before finalize
        assert rc != 0 and b"finalize" in L.ns2vc_last_error()
        shape = (C.c_int64 * 1)(3)
        rc = L.ns2vc_unet_load_weight(h, b"not.a.key", 1, shape, 1, None)
        assert rc != 0 and b"Unexpected key" in L.ns2vc_last_error()
    finally:
        L.ns2vc_unet_destroy(h)
    with pytest.raises(_lib.Ns2vcError):
        _lib.check(-1)


def test_unsupported_configs_rejected_loudly():
    with pytest.raises(ValueError):
        UNet1DConditionModel(down_block_types=("AttnDownBlock2D",) * 4)
    with pytest.raises(ValueError):
        UNet1DConditionModel(dual_cross_attention=True)
    with pytest.raises(ValueError):
        UNet1DConditionModel(num_attention_heads=8)
    with pytest.raises(ValueError):
        UNet1DConditionModel(block_out_channels=(32, 64), down_block_types=("DownBlock2D",) * 4)


def test_no_cpu_fallback():
    unet = UNet1DConditionModel(in_channels=36, out_channels=20, block_out_channels=(32, 64, 64, 96), norm_num_groups=8,
                                cross_attention_dim=16, attention_head_dim=8)
    with torch.no_grad(), pytest.raises(RuntimeError, match="no CPU path"):
        unet(torch.zeros(1, 36, 16), 3, torch.zeros(1, 4, 16))


def test_product_never_imports_oracle():
    pkg = os.path.join(REPO, "ns2vc_b200")
    for root, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh")):
                txt = open(os.path.join(root, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt, f
