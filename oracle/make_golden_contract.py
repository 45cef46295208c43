"""``python oracle/make_golden_contract.py``: from the UNMODIFIED reference tree, write tests/golden/contract.pt (shipped config,
``Pre_model`` / ``diff_model.unet.`` state_dict keys, shapes and parameter counts) and repeat_expand.pt (``utils.repeat_expand_2d``
on the seeded inputs of tests/test_frontend.py)."""
from __future__ import annotations

import json
import os
import sys
from unittest.mock import MagicMock

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("NS2VC_REFERENCE", "/root/reference")
sys.path.insert(0, REPO)
sys.path.insert(0, REF)
GOLD = os.path.join(REPO, "tests", "golden")

for _name in ("matplotlib", "matplotlib.pyplot", "vocos", "accelerate", "librosa", "soundfile", "tensorboardX"):
    sys.modules.setdefault(_name, MagicMock())


def main() -> None:
    import model as ref_model
    import utils as ref_utils
    import importlib.util
    spec = importlib.util.spec_from_file_location("test_frontend", os.path.join(REPO, "tests", "test_frontend.py"))
    tf = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tf)
    CASES, reference_input = tf.CASES, tf.reference_input

    cfg = json.load(open(os.path.join(REF, "config.json")))
    pre = ref_model.Pre_model(cfg)
    ns2 = ref_model.NaturalSpeech2(cfg)
    unet = ns2.diff_model.unet
    contract = {
        "config": cfg,
        "pre_model_state": [[k, list(v.shape)] for k, v in pre.state_dict().items()],
        "pre_model_params": sum(p.numel() for p in pre.parameters()),
        "unet_keys": [k[len("diff_model.unet."):] for k in ns2.state_dict() if k.startswith("diff_model.unet.")],
        "unet_params": sum(p.numel() for p in unet.parameters()),
        "unet_latent_channels": cfg["diffusion_encoder"]["in_channels"],
    }
    torch.save(contract, os.path.join(GOLD, "contract.pt"))
    outs = {f"{src}_{tgt}": ref_utils.repeat_expand_2d(reference_input(src, tgt), tgt) for src, tgt in CASES}
    torch.save(outs, os.path.join(GOLD, "repeat_expand.pt"))
    print("wrote contract.pt, repeat_expand.pt")


if __name__ == "__main__":
    main()
