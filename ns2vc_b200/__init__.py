"""ns2vc_b200 — H100-native (sm_90a) implementation of the NS2VC diffusion-denoiser hot path.

Drop-in surface (same names as the reference):
    ns2vc_b200.unet.UNet1DConditionModel          <- unet1d/unet_1d_condition.py
    ns2vc_b200.dpm_solver.{NoiseScheduleVP, model_wrapper, DPM_Solver}   <- sampler/dpm_solver.py
    ns2vc_b200.uni_pc.{NoiseScheduleVP, model_wrapper, UniPC}            <- sampler/uni_pc.py
    ns2vc_b200.pre_model.Pre_model                <- model.py:328-377 (condition encoders; ``install_pre_model(model)``)
    ns2vc_b200.frontend.repeat_expand_2d          <- utils.py:482-496 (feature stretch in front of the encoders)
    ns2vc_b200.diffusion.{p_sample_loop, ddim_sample} <- model.py:544-603 (DDPM / DDIM; ``install_diffusion(model)``)
    ns2vc_b200.loss.diffusion_loss                <- model.py:706-734 (``NaturalSpeech2.forward``'s objective, no gradients)
``ns2vc_b200.install()`` aliases those module paths so the reference's model.py / infer.py import
them unchanged (see INTEGRATION.md).
"""
from __future__ import annotations

import sys
import types

__version__ = "0.1.0"


def install() -> None:
    """Make ``unet1d.unet_1d_condition``, ``sampler.dpm_solver`` and ``sampler.uni_pc`` resolve to
    the CUDA implementations (call before ``import model`` in the reference tree).  The reference's
    own ``unet1d`` / ``sampler`` packages stay importable for their other submodules
    (``model.py:6`` imports ``unet1d.embeddings``); only the three hot-path modules are aliased."""
    import importlib
    import importlib.util

    from . import dpm_solver, uni_pc, unet

    def parent(name):
        m = sys.modules.get(name)
        if m is None:
            try:
                spec = importlib.util.find_spec(name)
            except (ImportError, ValueError):
                spec = None
            if spec is not None:
                m = importlib.import_module(name)
            else:                                   # no reference tree on sys.path: stub package
                m = types.ModuleType(name)
                m.__path__ = []
                sys.modules[name] = m
        return m

    for pkg, sub, mod in (("unet1d", "unet_1d_condition", unet), ("sampler", "dpm_solver", dpm_solver),
                          ("sampler", "uni_pc", uni_pc)):
        p = parent(pkg)
        sys.modules[f"{pkg}.{sub}"] = mod
        setattr(p, sub, mod)


def install_pre_model(model_module=None) -> None:
    """Make the reference's ``model.Pre_model`` (defined inside ``model.py`` itself, :328) the CUDA implementation: call after
    ``import model`` and before ``NaturalSpeech2(cfg)`` is constructed (``model.py:451`` looks the class up by its global name)."""
    from .pre_model import Pre_model
    if model_module is None:
        model_module = sys.modules.get("model")
    if model_module is None or not hasattr(model_module, "Pre_model"):
        raise RuntimeError("install_pre_model: import the reference's model.py first (or pass the module)")
    model_module.Pre_model = Pre_model


def install_diffusion(model_module=None) -> None:
    """Make the reference's ``NaturalSpeech2.p_sample_loop`` / ``.ddim_sample`` (``sample_method='ddpm'`` / ``'ddim'``, model.py:544-603)
    take the fused DDPM / DDIM loops when the denoiser is our UNet (``ns2vc_b200.diffusion``), and add
    ``NaturalSpeech2.validation_loss``: ``forward``'s objective under ``no_grad`` on the device path.  Call after ``import model``."""
    from . import diffusion
    if model_module is None:
        model_module = sys.modules.get("model")
    if model_module is None or not hasattr(model_module, "NaturalSpeech2"):
        raise RuntimeError("install_diffusion: import the reference's model.py first (or pass the module)")
    model_module.NaturalSpeech2.p_sample_loop = diffusion.p_sample_loop
    model_module.NaturalSpeech2.ddim_sample = diffusion.ddim_sample
    # the training objective under no_grad (model.py:706-734); `forward` itself stays the reference's
    model_module.NaturalSpeech2.validation_loss = diffusion.validation_loss
