"""Our ``Pre_model`` and denoiser UNet, built from the reference's shipped config, have the state_dict keys (order, shapes) and
parameter counts of the reference's modules (tests/golden/contract.pt, from oracle/make_golden_contract.py)."""
import pytest
import torch

from ns2vc_b200.arch import ns2vc_denoiser_config, param_shapes


def test_our_modules_have_the_reference_checkpoint_contract(gold):
    ref = gold("contract.pt")
    cfg = ref["config"]
    from ns2vc_b200.pre_model import Pre_model
    pre = Pre_model(cfg)
    ours = [[k, list(v.shape)] for k, v in pre.state_dict().items()]
    assert ours == ref["pre_model_state"]                   # same keys, order and shapes as the reference's Pre_model
    assert sum(p.numel() for p in pre.parameters()) == ref["pre_model_params"] == 34923404
    pre.load_state_dict({k: torch.zeros(s) for k, s in ref["pre_model_state"]}, strict=True)

    from ns2vc_b200.unet import UNet1DConditionModel
    de = cfg["diffusion_encoder"]
    unet = UNet1DConditionModel(in_channels=de["in_channels"] + de["hidden_channels"], out_channels=de["out_channels"],
                                block_out_channels=(128, 256, 384, 512), norm_num_groups=8,
                                cross_attention_dim=de["hidden_channels"], attention_head_dim=de["n_heads"],
                                addition_embed_type="text", resnet_time_scale_shift="scale_shift")
    assert sum(p.numel() for p in unet.parameters()) == ref["unet_params"] == 66076900
    assert unet.latent_channels == ref["unet_latent_channels"]
    # a checkpoint written by the reference has exactly these keys under diff_model.unet.
    assert list(unet.state_dict().keys()) == ref["unet_keys"]
    assert list(param_shapes(ns2vc_denoiser_config()).keys()) == ref["unet_keys"]


def test_install_aliases_the_reference_module_paths(monkeypatch):
    """install() points the reference's import paths at our modules, install_pre_model() replaces model.Pre_model (stub
    packages stand in for the reference tree)."""
    import sys
    import types

    import ns2vc_b200
    from ns2vc_b200 import dpm_solver, uni_pc, unet
    from ns2vc_b200.pre_model import Pre_model
    for name in ("unet1d", "unet1d.unet_1d_condition", "sampler", "sampler.dpm_solver", "sampler.uni_pc", "model"):
        monkeypatch.delitem(sys.modules, name, raising=False)
    ns2vc_b200.install()
    import unet1d.unet_1d_condition as ref_unet
    from sampler.dpm_solver import DPM_Solver, NoiseScheduleVP, model_wrapper
    from sampler.uni_pc import UniPC
    assert ref_unet is unet and (DPM_Solver, NoiseScheduleVP, model_wrapper) == (dpm_solver.DPM_Solver, dpm_solver.NoiseScheduleVP, dpm_solver.model_wrapper)
    assert UniPC is uni_pc.UniPC
    with pytest.raises(RuntimeError):
        ns2vc_b200.install_pre_model()                      # model.py not imported yet
    for name in ("model", "other"):
        mod = types.ModuleType(name)
        mod.Pre_model = object
        if name == "model":
            monkeypatch.setitem(sys.modules, "model", mod)
            ns2vc_b200.install_pre_model()
        else:
            ns2vc_b200.install_pre_model(mod)
        assert mod.Pre_model is Pre_model
