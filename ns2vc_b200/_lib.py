"""ctypes binding of ``libns2vc_b200.so`` (C-ABI declared in ``include/ns2vc_b200.h``), and the base class of the modules
that run in its engines.

There is no CPU fallback: if the library is missing every CUDA entry point raises.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Any, Callable, Dict, Optional, Tuple

import torch
import torch.nn as nn

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


# the row step's methods (NS2VC_ROW_* of the header)
ROW_DPM, ROW_UNIPC, ROW_DDPM, ROW_DDIM = 0, 1, 2, 3


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
    "ns2vc_unet_prepare_cond_rows": (C.c_int, [_P, _P, C.c_longlong, _P, _P, _P, C.POINTER(C.c_int), C.c_int, C.c_int, C.c_int,
                                               C.c_int, _P, _P]),
    "ns2vc_unet_forward": (C.c_int, [_P, _P, C.c_longlong, _P, _P, C.c_int, C.c_int, C.c_int, _P, _P]),
    "ns2vc_unet_film_width": (C.c_int, [_P]),
    "ns2vc_unet_time_table_floats": (C.c_size_t, [_P, C.c_int]),
    "ns2vc_unet_time_table": (C.c_int, [_P, _P, C.c_int, _P, C.c_int, C.c_int, C.c_int, _P, _P]),
    "ns2vc_unet_time_table_rows": (C.c_int, [_P, _P, C.c_int, C.POINTER(C.c_int), C.c_int, _P, C.c_int, C.c_int, C.c_int, _P, _P]),
    "ns2vc_unet_forward_film": (C.c_int, [_P, _P, C.c_longlong, _P, _P, C.c_int, C.c_int, C.c_int, _P, _P]),
    "ns2vc_dpm_step": (C.c_int, [_P, _P, _P, C.POINTER(DpmCoef), _P, _P, C.c_size_t, _P, _P]),
    "ns2vc_unipc_step": (C.c_int, [_P, _P, _P, _P, _P, C.POINTER(UniPcCoef), _P, _P, _P, C.c_size_t, _P, _P]),
    "ns2vc_dpm_step_rows": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, C.c_size_t, C.c_int, _P, _P]),   # (device coefficient arrays)
    "ns2vc_unipc_step_rows": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_size_t, C.c_int, _P, _P]),
    "ns2vc_sampler_step_rows": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_size_t, C.c_int, _P, _P]),
    "ns2vc_ddpm_step": (C.c_int, [_P, _P, _P, _P, _P, C.c_size_t, _P, _P]),     # (the coefficient struct is a device pointer)
    "ns2vc_ddim_step": (C.c_int, [_P, _P, _P, _P, _P, C.c_size_t, _P, _P]),
    "ns2vc_sampler_step_rows_seeded": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_int, _P, _P, _P, _P, _P, _P, C.c_size_t,
                                                 C.c_int, _P, _P]),
    "ns2vc_noise_normal_rows": (C.c_int, [_P, C.c_uint32, C.c_int, C.c_int, _P, _P, C.c_int, _P]),
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
    "ns2vc_pre_encode_voices_ragged": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_int, _P, _P]),
    "ns2vc_pre_infer_content_ragged": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_int, _P, _P]),
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
    "ns2vc_resample_check": (C.c_int, [C.c_int, C.c_int]),
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
    # training objective (q_sample and the SNR-weighted per-row MSE)
    "ns2vc_q_sample": (C.c_int, [_P, _P, C.c_int, _P, _P, _P, _P, C.c_int, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, _P]),
    "ns2vc_mse_workspace_bytes": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "ns2vc_mse_rows": (C.c_int, [_P, _P, C.c_int, _P, _P, C.c_int, C.c_float, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P]),
    "ns2vc_mse_ragged_workspace_bytes": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "ns2vc_mse_rows_ragged": (C.c_int, [_P, _P, C.c_int, _P, _P, _P, C.c_int, C.c_float, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int,
                                        _P, _P]),
    # kernel checks (tests only; the argument structs are mirrored in tests/test_kernels_fp64.py, tests/test_norm_kernels_fp64.py and
    # tests/test_audio_kernels_fp64.py)
    "ns2vc_check_pack_b": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P,
                                     C.c_int, C.c_int, _P]),
    "ns2vc_check_gemm": (C.c_int, [_P, C.c_char_p, C.c_int, _P]),
    "ns2vc_check_attention": (C.c_int, [_P, C.c_char_p, C.c_int, _P]),
    "ns2vc_check_prep": (C.c_int, [_P, C.c_char_p, C.c_int, _P]),
    "ns2vc_check_ln": (C.c_int, [_P, C.c_char_p, C.c_int, _P]),
    "ns2vc_check_voc_norm": (C.c_int, [_P, C.c_char_p, C.c_int, _P]),
    "ns2vc_check_small_linear": (C.c_int, [_P, C.c_char_p, C.c_int, _P]),
    "ns2vc_check_pool": (C.c_int, [_P, C.c_char_p, C.c_int, _P]),
    "ns2vc_check_nct_split": (C.c_int, [_P, C.c_char_p, C.c_int, _P]),
    "ns2vc_check_cv_conv0": (C.c_int, [_P, C.c_char_p, C.c_int, _P]),
    "ns2vc_check_cv_pos_conv": (C.c_int, [_P, C.c_char_p, C.c_int, _P]),
    "ns2vc_check_down_conv": (C.c_int, [_P, C.c_char_p, C.c_int, _P]),
    "ns2vc_check_cv_conv": (C.c_int, [_P, C.c_char_p, C.c_int, _P]),
    "ns2vc_check_istft": (C.c_int, [_P, C.c_char_p, C.c_int, _P]),
    # the packed-weight record (tests/test_packed_weights_fp64.py)
    "ns2vc_check_packed_count": (C.c_int, [C.c_int, _P]),
    "ns2vc_check_packed": (C.c_int, [C.c_int, _P, C.c_int, C.c_char_p, C.c_int, _P, _P, _P, _P, _P, _P, _P]),
    "ns2vc_check_fold_vector": (C.c_int, [C.c_int, _P, C.c_int, C.c_int, C.c_char_p, C.c_int, _P, _P, _P]),
    # the run loops' launch observer (tests/test_program_launches_fp64.py)
    "ns2vc_check_set_launch_hook": (C.c_int, [C.c_int, _P, _P, _P]),
    # the sampler noise's generator (tests/test_seeded_noise.py)
    "ns2vc_check_philox": (C.c_int, [_P, _P, C.c_int, _P, _P, _P]),
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


class EngineModule(nn.Module):
    """A module whose parameters run in one of the engines behind the C-ABI.  A subclass sets ``_prefix`` (which C-ABI:
    ``"ns2vc_unet_"`` / ``"ns2vc_pre_"`` / ``"ns2vc_voc_"`` / ``"ns2vc_cv_"``), ``_cfg_struct`` (its create argument, filled
    from the ``self.cfg`` dict unless the subclass overrides ``_c_cfg``) and ``_requirement`` (the end of the error raised for a
    parameter that is not fp32 on the device; ``{device}`` in it is filled in)."""
    _prefix: str
    _cfg_struct: type
    _requirement: str

    def __init__(self) -> None:
        super().__init__()
        self._handle: Optional[int] = None
        self._handle_device = None
        self._wsig = None
        self._ws: Optional[torch.Tensor] = None
        self._ws_need: Dict[Tuple[int, ...], int] = {}

    def _c_cfg(self):
        c = self._cfg_struct()
        for k, v in self.cfg.items():
            setattr(c, k, int(v))
        return c

    def _fn(self, name: str):
        return getattr(lib(), self._prefix + name)

    def engine(self, device: torch.device) -> int:
        """Opaque engine handle on ``device`` with the current parameter values loaded and packed.  The handle is created on
        the device if needed; every state_dict entry is loaded and the weights are finalized again whenever a parameter
        changed (optimizer step, load_state_dict, .to())."""
        # (storage, version) pairs over a cached list of the Parameter objects: the module tree is fixed after construction,
        # `.to()` / `load_state_dict` / optimizers change storage or bump versions of the SAME objects (the recursive
        # `self.parameters()` walk on every forward of the generic path was ~1 ms of host time per call)
        plist = self.__dict__.get("_plist")
        if plist is None:
            plist = self.__dict__["_plist"] = list(self.parameters())
        sig = tuple((p.data_ptr(), p._version) for p in plist)
        if self._handle is not None and self._wsig == sig and self._handle_device == device:
            return self._handle
        plist = self.__dict__["_plist"] = list(self.parameters())     # something changed: re-walk the tree before re-packing
        sig = tuple((p.data_ptr(), p._version) for p in plist)
        stream = torch.cuda.current_stream(device).cuda_stream
        with torch.cuda.device(device):
            if self._handle is None or self._handle_device != device:
                self._release()
                h = C.c_void_p()
                ccfg = self._c_cfg()
                check(self._fn("create")(C.byref(ccfg), C.byref(h)))
                self._handle = h.value
                self._handle_device = device
            load = self._fn("load_weight")
            for key, p in self.state_dict().items():
                if p.device != device or p.dtype != torch.float32:
                    raise RuntimeError(f"parameter {key} is {p.dtype} on {p.device}; " + self._requirement.format(device=device))
                t = p.detach().contiguous()
                shape = (C.c_int64 * t.dim())(*t.shape)
                check(load(self._handle, key.encode(), t.data_ptr(), shape, t.dim(), stream))
            check(self._fn("finalize")(self._handle, stream))
        self._wsig = sig
        self._ws_need = {}                  # (re)packed: the workspace sizes are asked again
        return self._handle

    def _release(self):
        """Destroy the engine handle and drop the workspace.  Plain ``__dict__`` writes: ``nn.Module.__setattr__`` may already
        be torn down at interpreter shutdown."""
        if self.__dict__.get("_handle") is None:
            return
        try:
            self._fn("destroy")(self._handle)
        except Exception:
            pass
        self.__dict__["_handle"] = None
        self.__dict__["_ws"] = None

    def __del__(self):
        try:
            self._release()
        except Exception:
            pass

    def workspace(self, *dims_and_device) -> torch.Tensor:
        """``workspace(*dims, device)``: the scratch buffer of a call of shape ``dims`` (the dims of the engine's
        ``_workspace_bytes``).  ONE grow-only buffer per module, shared by every shape (the CLI feeds a different T per slice: a
        fresh multi-hundred-MB allocation per shape was most of a cold call).  Calls are stream-ordered and never concurrent,
        and every program rebuilds or re-prepares what it keeps there after a shape switch, so shapes can alias the same
        memory.  Growing it invalidates the captured loops that baked the old pointer (the module's sessions are dropped)."""
        *dims, device = dims_and_device
        key = tuple(dims)
        need = self._ws_need.get(key)
        if need is None:
            n = C.c_size_t()
            check(self._fn("workspace_bytes")(self.engine(device), *dims, C.byref(n)))
            need = int(n.value)
            if len(self._ws_need) > 256:
                self._ws_need.clear()
            self._ws_need[key] = need
        ws = self._ws
        if ws is None or ws.device != device or ws.numel() < need:
            self.__dict__.get("_sessions", {}).clear()
            self._ws = ws = None            # (the old buffer is freed before the new one is allocated)
            self._ws = ws = torch.empty(int(need * 1.25) if need < (8 << 30) else need, dtype=torch.uint8, device=device)
        return ws

    def launch_count(self) -> int:
        """Launches of the engine's last run (tap copies not counted); 0 before the first."""
        return int(self._fn("launch_count")(self._handle)) if self._handle is not None else 0

    def _collect_taps(self, device: torch.device, B: int, run: Callable[[], Any],
                      rows: Callable[[int], int] = lambda r: r) -> Tuple[Any, Dict[str, torch.Tensor]]:
        """Sets every tap of the engine's current program to a fresh zeroed [B, rows(r), C] buffer (r, C: the tap's info; r is a
        row count, or the denoiser's level), calls ``run()`` (which must run that program without building another),
        synchronises and clears the taps whatever happens.  Returns (run's result, {tap name: buffer}) in the engine's
        token-major layout."""
        h = self.engine(device)
        num, info, set_tap = self._fn("num_taps"), self._fn("tap_info"), self._fn("set_tap")
        n = num(h)
        bufs = {}
        try:
            for i in range(n):
                name, r, ch = C.c_char_p(), C.c_int(), C.c_int()
                check(info(h, i, C.byref(name), C.byref(r), C.byref(ch)))
                t = torch.zeros((B, rows(r.value), ch.value), dtype=torch.float32, device=device)
                check(set_tap(h, i, t.data_ptr()))
                bufs[name.value.decode()] = t
            with torch.no_grad():
                res = run()
            torch.cuda.synchronize(device)
        finally:
            for i in range(n):
                set_tap(h, i, None)
        return res, bufs

    def _load_checked(self, sd: Dict[str, torch.Tensor], what: str) -> "EngineModule":
        """Loads ``sd`` (as fp32) after checking it holds exactly this module's keys and shapes; ValueError names the first
        missing, unexpected or mis-shaped key (``what``: the reference model the state_dict comes from)."""
        want = self.state_dict()
        for k in want:
            if k not in sd:
                raise ValueError(f"missing key {k} in the {what} state_dict")
        for k, v in sd.items():
            if k not in want:
                raise ValueError(f"unexpected key {k} in the {what} state_dict")
            if tuple(v.shape) != tuple(want[k].shape):
                raise ValueError(f"size mismatch for {k}: expected {tuple(want[k].shape)}, got {tuple(v.shape)}")
        self.load_state_dict({k: v.detach().to(torch.float32) for k, v in sd.items()})
        return self
