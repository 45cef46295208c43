import os
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

GOLD = os.path.join(REPO, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: run with -m gpu)")


@pytest.fixture(scope="session")
def gold():
    import torch

    def load(name):
        return torch.load(os.path.join(GOLD, name), map_location="cpu", weights_only=False)
    return load


def tiny_config():
    from ns2vc_b200.arch import UNetConfig
    return UNetConfig(in_channels=36, out_channels=20, block_out_channels=(32, 64, 64, 96), norm_num_groups=8,
                      cross_attention_dim=16, num_heads=8, addition_embed_type="text", addition_embed_type_num_heads=4,
                      resnet_time_scale_shift="scale_shift")


def tiny_inputs():
    import torch
    from ns2vc_b200.synth import make_inputs
    inp = make_inputs(2, 37, 11, latent_ch=20, content_ch=16, ragged=True, seed=10)
    inp["refer_lengths"] = torch.tensor([11, 7])
    return inp
