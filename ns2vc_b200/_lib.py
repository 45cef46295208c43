"""ctypes binding of ``libns2vc_b200.so`` (C-ABI declared in ``include/ns2vc_b200.h``).

There is no CPU fallback: if the library is missing every CUDA entry point raises.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_C", os.environ.get("NS2VC_LIB_NAME", "libns2vc_b200.so"))   # (NS2VC_LIB_NAME: A/B builds during development)

MAX_LEVELS = 8


class UNetCfg(C.Structure):
    _fields_ = [
        ("in_channels", C.c_int), ("latent_channels", C.c_int), ("out_channels", C.c_int), ("n_levels", C.c_int),
        ("block_out_channels", C.c_int * MAX_LEVELS), ("layers_per_block", C.c_int * MAX_LEVELS),
        ("down_has_attn", C.c_int * MAX_LEVELS), ("up_has_attn", C.c_int * MAX_LEVELS),
        ("num_heads", C.c_int), ("cross_attention_dim", C.c_int), ("norm_num_groups", C.c_int), ("norm_eps", C.c_float),
        ("time_scale_shift", C.c_int), ("add_embed_text", C.c_int), ("add_embed_heads", C.c_int),
        ("flip_sin_to_cos", C.c_int), ("freq_shift", C.c_float),
    ]


class PreCfg(C.Structure):
    _fields_ = [("phone_in", C.c_int), ("phone_hidden", C.c_int), ("phone_out", C.c_int), ("phone_layers", C.c_int),
                ("prompt_in", C.c_int), ("prompt_hidden", C.c_int), ("prompt_out", C.c_int), ("prompt_layers", C.c_int),
                ("ref_dim", C.c_int), ("ref_heads", C.c_int), ("n_heads", C.c_int), ("ffn_kernel", C.c_int)]


class VocCfg(C.Structure):
    _fields_ = [("input_channels", C.c_int), ("dim", C.c_int), ("intermediate_dim", C.c_int), ("num_layers", C.c_int),
                ("n_fft", C.c_int), ("hop_length", C.c_int)]


class CvCfg(C.Structure):
    _fields_ = [("conv_dim", C.c_int), ("embed_dim", C.c_int), ("ffn_dim", C.c_int), ("num_layers", C.c_int), ("num_heads", C.c_int),
                ("pos_conv_kernel", C.c_int), ("pos_conv_groups", C.c_int), ("final_dim", C.c_int)]


class DpmCoef(C.Structure):
    _fields_ = [("alpha_s", C.c_float), ("sigma_s", C.c_float), ("c_x", C.c_float), ("c_m", C.c_float),
                ("c_d", C.c_float), ("inv_r0", C.c_float), ("order", C.c_int)]


class UniPcCoef(C.Structure):
    _fields_ = [("alpha_t", C.c_float), ("sigma_t", C.c_float), ("c_x", C.c_float), ("c_m", C.c_float),
                ("ab", C.c_float), ("rk", C.c_float), ("rho0", C.c_float), ("rho1", C.c_float), ("corr_order", C.c_int),
                ("n_c_x", C.c_float), ("n_c_m", C.c_float), ("nab", C.c_float), ("nrk", C.c_float), ("pred_order", C.c_int)]


class DdpmCoef(C.Structure):
    _fields_ = [("c_x0", C.c_float), ("c_x", C.c_float), ("c_noise", C.c_float), ("add_noise", C.c_int)]


class DdimCoef(C.Structure):
    _fields_ = [("sqrt_recip", C.c_float), ("sqrt_recipm1", C.c_float), ("sqrt_alpha_next", C.c_float), ("c", C.c_float),
                ("sigma", C.c_float), ("last", C.c_int)]


# symbol -> (restype, argtypes); also the export list checked by tests/test_abi.py
_P = C.c_void_p
SIGNATURES = {
    "ns2vc_last_error": (C.c_char_p, []),
    "ns2vc_build_info": (C.c_char_p, []),
    "ns2vc_unet_create": (C.c_int, [C.POINTER(UNetCfg), C.POINTER(_P)]),
    "ns2vc_unet_destroy": (None, [_P]),
    "ns2vc_unet_num_weights": (C.c_int, [_P]),
    "ns2vc_unet_weight_info": (C.c_int, [_P, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int64), C.POINTER(C.c_int)]),
    "ns2vc_unet_load_weight": (C.c_int, [_P, C.c_char_p, _P, C.POINTER(C.c_int64), C.c_int, _P]),
    "ns2vc_unet_finalize": (C.c_int, [_P, _P]),
    "ns2vc_unet_workspace_bytes": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "ns2vc_unet_prepare_cond": (C.c_int, [_P, _P, C.c_longlong, _P, _P, C.c_int, C.c_int, C.c_int, _P, _P]),
    "ns2vc_unet_prepare_cond_ragged": (C.c_int, [_P, _P, C.c_longlong, _P, _P, _P, C.c_int, C.c_int, C.c_int, _P, _P]),
    "ns2vc_unet_forward": (C.c_int, [_P, _P, C.c_longlong, _P, _P, C.c_int, C.c_int, C.c_int, _P, _P]),
    "ns2vc_unet_film_width": (C.c_int, [_P]),
    "ns2vc_unet_time_table_floats": (C.c_size_t, [_P, C.c_int]),
    "ns2vc_unet_time_table": (C.c_int, [_P, _P, C.c_int, _P, C.c_int, C.c_int, C.c_int, _P, _P]),
    "ns2vc_unet_forward_film": (C.c_int, [_P, _P, C.c_longlong, _P, _P, C.c_int, C.c_int, C.c_int, _P, _P]),
    "ns2vc_dpm_step": (C.c_int, [_P, _P, _P, C.POINTER(DpmCoef), _P, _P, C.c_size_t, _P, _P]),
    "ns2vc_unipc_step": (C.c_int, [_P, _P, _P, _P, _P, C.POINTER(UniPcCoef), _P, _P, _P, C.c_size_t, _P, _P]),
    "ns2vc_ddpm_step": (C.c_int, [_P, _P, _P, _P, _P, C.c_size_t, _P, _P]),     # (the coefficient struct is a device pointer)
    "ns2vc_ddim_step": (C.c_int, [_P, _P, _P, _P, _P, C.c_size_t, _P, _P]),
    "ns2vc_mask_bias": (C.c_int, [_P, C.c_int, _P, _P]),
    "ns2vc_nearest_index": (C.c_int, [C.c_int, C.c_int, C.POINTER(C.c_int)]),
    "ns2vc_down_length": (C.c_int, [C.c_int]),
    "ns2vc_unet_num_taps": (C.c_int, [_P]),
    "ns2vc_unet_tap_info": (C.c_int, [_P, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "ns2vc_unet_set_tap": (C.c_int, [_P, C.c_int, _P]),
    "ns2vc_unet_plan_string": (C.c_char_p, [_P]),
    "ns2vc_unet_launch_count": (C.c_int, [_P]),
    "ns2vc_unet_set_profiling": (C.c_int, [_P, C.c_int]),
    "ns2vc_unet_set_trace": (C.c_int, [_P, _P, C.c_int]),
    "ns2vc_unet_set_attn_trace": (C.c_int, [_P, _P, C.c_int]),
    "ns2vc_unet_set_span_trace": (C.c_int, [_P, _P, C.c_int]),
    "ns2vc_unet_launch_kind": (C.c_int, [_P, C.c_int]),
    "ns2vc_profile_num_kinds": (C.c_int, []),
    "ns2vc_profile_kind_name": (C.c_char_p, [C.c_int]),
    "ns2vc_unet_profile_read": (C.c_int, [_P, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_longlong)]),
    "ns2vc_unet_profile_dump": (C.c_int, [_P, C.c_char_p]),
    "ns2vc_unet_profile_reset": (C.c_int, [_P]),
    # condition encoders (Pre_model)
    "ns2vc_pre_create": (C.c_int, [C.POINTER(PreCfg), C.POINTER(_P)]),
    "ns2vc_pre_destroy": (None, [_P]),
    "ns2vc_pre_num_weights": (C.c_int, [_P]),
    "ns2vc_pre_weight_info": (C.c_int, [_P, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int64), C.POINTER(C.c_int)]),
    "ns2vc_pre_load_weight": (C.c_int, [_P, C.c_char_p, _P, C.POINTER(C.c_int64), C.c_int, _P]),
    "ns2vc_pre_finalize": (C.c_int, [_P, _P]),
    "ns2vc_pre_workspace_bytes": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "ns2vc_pre_infer": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int, _P, _P]),
    "ns2vc_pre_infer_ragged": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int, _P, _P]),
    "ns2vc_pre_num_taps": (C.c_int, [_P]),
    "ns2vc_pre_tap_info": (C.c_int, [_P, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "ns2vc_pre_set_tap": (C.c_int, [_P, C.c_int, _P]),
    "ns2vc_pre_launch_count": (C.c_int, [_P]),
    # vocoder (Vocos.decode)
    "ns2vc_voc_create": (C.c_int, [C.POINTER(VocCfg), C.POINTER(_P)]),
    "ns2vc_voc_destroy": (None, [_P]),
    "ns2vc_voc_num_weights": (C.c_int, [_P]),
    "ns2vc_voc_weight_info": (C.c_int, [_P, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int64), C.POINTER(C.c_int)]),
    "ns2vc_voc_load_weight": (C.c_int, [_P, C.c_char_p, _P, C.POINTER(C.c_int64), C.c_int, _P]),
    "ns2vc_voc_finalize": (C.c_int, [_P, _P]),
    "ns2vc_voc_workspace_bytes": (C.c_int, [_P, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "ns2vc_voc_decode": (C.c_int, [_P, _P, C.c_longlong, _P, _P, C.c_int, C.c_int, _P, _P]),
    "ns2vc_voc_istft": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, _P]),
    "ns2vc_voc_num_taps": (C.c_int, [_P]),
    "ns2vc_voc_tap_info": (C.c_int, [_P, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "ns2vc_voc_set_tap": (C.c_int, [_P, C.c_int, _P]),
    "ns2vc_voc_launch_count": (C.c_int, [_P]),
    # content encoder (ContentVec / HubertModel units)
    "ns2vc_cv_create": (C.c_int, [C.POINTER(CvCfg), C.POINTER(_P)]),
    "ns2vc_cv_destroy": (None, [_P]),
    "ns2vc_cv_num_weights": (C.c_int, [_P]),
    "ns2vc_cv_weight_info": (C.c_int, [_P, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int64), C.POINTER(C.c_int)]),
    "ns2vc_cv_load_weight": (C.c_int, [_P, C.c_char_p, _P, C.POINTER(C.c_int64), C.c_int, _P]),
    "ns2vc_cv_finalize": (C.c_int, [_P, _P]),
    "ns2vc_cv_workspace_bytes": (C.c_int, [_P, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "ns2vc_cv_num_frames": (C.c_int, [C.c_longlong]),
    "ns2vc_cv_extract": (C.c_int, [_P, _P, C.c_longlong, _P, _P, _P, C.c_int, C.c_int, _P, _P]),
    "ns2vc_cv_num_taps": (C.c_int, [_P]),
    "ns2vc_cv_tap_info": (C.c_int, [_P, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "ns2vc_cv_set_tap": (C.c_int, [_P, C.c_int, _P]),
    "ns2vc_cv_launch_count": (C.c_int, [_P]),
    # prompt-mel front end (resampler + log-mel spectrogram)
    "ns2vc_resample_out_length": (C.c_longlong, [C.c_int, C.c_int, C.c_longlong]),
    "ns2vc_resample_table": (C.c_int, [C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), _P]),
    "ns2vc_mel_filterbank": (C.c_int, [_P]),
    "ns2vc_resampler_create": (C.c_int, [C.c_int, C.c_int, C.POINTER(_P)]),
    "ns2vc_resampler_destroy": (None, [_P]),
    "ns2vc_resample": (C.c_int, [_P, _P, C.c_longlong, C.c_longlong, _P, _P, C.c_longlong, C.c_longlong, C.c_int, _P]),
    "ns2vc_mel_create": (C.c_int, [_P, _P, C.POINTER(_P)]),
    "ns2vc_mel_destroy": (None, [_P]),
    "ns2vc_log_mel": (C.c_int, [_P, _P, C.c_longlong, C.c_longlong, _P, _P, C.c_int, C.c_int, _P]),
    # live conversion (SOLA join of one tick)
    "ns2vc_stream_sola": (C.c_int, [_P, C.c_longlong, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, _P]),
    # silence slicer (framewise RMS)
    "ns2vc_slice_rms_frames": (C.c_longlong, [C.c_longlong, C.c_int, C.c_int]),
    "ns2vc_slice_rms": (C.c_int, [_P, C.c_longlong, _P, _P, _P, C.c_int, C.c_int, _P]),
}

_lib: Optional[C.CDLL] = None


class Ns2vcError(RuntimeError):
    pass


def lib() -> C.CDLL:
    """Load the shared library (once).  Raises loudly when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise Ns2vcError(
                f"{LIB_PATH} not found: the ns2vc_b200 CUDA extension is not built "
                "(run ./build.sh or __graft_entry__.build()); there is no CPU fallback.")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(rc: int) -> None:
    if rc != 0:
        msg = lib().ns2vc_last_error()
        raise Ns2vcError((msg or b"unknown error").decode("utf-8", "replace") + f" (code {rc})")


def engine_handle(mod, prefix: str, device, requirement: str) -> int:
    """The engine handle of ``mod`` (a module with ``_c_cfg()`` and ``_release()``) on ``device``, with its current parameter
    values loaded and packed.  ``prefix`` selects the C-ABI (``"ns2vc_unet_"`` / ``"ns2vc_pre_"`` / ``"ns2vc_voc_"`` / ``"ns2vc_cv_"``).  The handle is created on
    the device if needed; every state_dict entry is loaded and the weights are finalized again whenever a parameter changed
    (optimizer step, load_state_dict, .to()).  ``requirement`` ends the error raised for a parameter that is not fp32 on
    ``device``; ``{device}`` in it is filled in."""
    # (storage, version) pairs over a cached list of the Parameter objects: the module tree is fixed after construction,
    # `.to()` / `load_state_dict` / optimizers change storage or bump versions of the SAME objects (the recursive
    # `self.parameters()` walk on every forward of the generic path was ~1 ms of host time per call)
    plist = mod.__dict__.get("_plist")
    if plist is None:
        plist = mod.__dict__["_plist"] = list(mod.parameters())
    sig = tuple((p.data_ptr(), p._version) for p in plist)
    if mod._handle is not None and mod._wsig == sig and mod._handle_device == device:
        return mod._handle
    plist = mod.__dict__["_plist"] = list(mod.parameters())     # something changed: re-walk the tree before re-packing
    sig = tuple((p.data_ptr(), p._version) for p in plist)
    L = lib()
    stream = torch.cuda.current_stream(device).cuda_stream
    with torch.cuda.device(device):
        if mod._handle is None or mod._handle_device != device:
            mod._release()
            h = C.c_void_p()
            ccfg = mod._c_cfg()
            check(getattr(L, prefix + "create")(C.byref(ccfg), C.byref(h)))
            mod._handle = h.value
            mod._handle_device = device
        load = getattr(L, prefix + "load_weight")
        for key, p in mod.state_dict().items():
            if p.device != device or p.dtype != torch.float32:
                raise RuntimeError(f"parameter {key} is {p.dtype} on {p.device}; " + requirement.format(device=device))
            t = p.detach().contiguous()
            shape = (C.c_int64 * t.dim())(*t.shape)
            check(load(mod._handle, key.encode(), t.data_ptr(), shape, t.dim(), stream))
        check(getattr(L, prefix + "finalize")(mod._handle, stream))
    mod._wsig = sig
    return mod._handle


def release_engine(mod, prefix: str) -> bool:
    """Destroy the engine handle of ``mod``; False if it had none.  Plain ``__dict__`` writes: ``nn.Module.__setattr__`` may
    already be torn down at interpreter shutdown."""
    if mod.__dict__.get("_handle") is None:
        return False
    try:
        getattr(lib(), prefix + "destroy")(mod._handle)
    except Exception:
        pass
    mod.__dict__["_handle"] = None
    return True
