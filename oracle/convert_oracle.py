"""TEST INFRASTRUCTURE ONLY - the reference's waveform-to-waveform conversion restated for ONE slice alone, and the CLI's
slicing loop restated literally.  Nothing in the product imports this file.

``convert_one`` is ``Svc.infer`` (inference/infer_tool.py:141-206) -> ``NaturalSpeech2.sample`` (model.py:605-696) at B = 1,
stage by stage over the other oracles:
  * wav = resample(x, sr, 24000)                         infer_tool.py:143 (librosa.load(sr=24000); here torchaudio's filter)
                                                         mel_oracle.resample
  * T = len(wav) // 256                                  the f0 length: utils.py:159-160 (compute_f0_parselmouth)
  * wav16k = resample(wav, 24000, 16000)                 infer_tool.py:162
  * c = repeat_expand_2d(hubert(wav16k), T)              infer_tool.py:164-165; content_oracle.extract, utils.py:482-496
  * content, prompt = Pre_model.infer(...)               model.py:631-633; pre_model_oracle.pre_model_infer
  * mel = UniPC-bh2 / DPM-Solver++(2M) from x_T          model.py:620-686; sampler_oracle.unipc_bh / dpmpp_2m over
                                                         unet_oracle.denoiser_forward
  * audio = vocos.decode(mel)                            model.py:689-691; vocos_oracle.decode
``cli_loop`` is infer.py:99-141 for one (file, prompt) pair with Python lists, ``pad_array`` and ``split_list_by_n`` as written
there (inference/infer_tool.py:100-113), the per-slice conversion injected.
"""
from __future__ import annotations

from typing import Callable, Dict

import numpy as np
import torch

from . import content_oracle, mel_oracle, pre_model_oracle, sampler_oracle, unet_oracle, vocos_oracle

TARGET_SR, HOP = 24000, 256


def lengths(n: int, sr: int) -> Dict[str, int]:
    """Host lengths of one slice of n samples at sr: 24 kHz samples, frames T, 16 kHz samples, ContentVec frames."""
    n24 = mel_oracle.out_length(sr, TARGET_SR, n)
    n16 = mel_oracle.out_length(TARGET_SR, 16000, n24)
    return dict(n24=n24, T=n24 // HOP, n16=n16, units=content_oracle.num_frames(n16))


def repeat_expand_2d(content: torch.Tensor, target_len: int) -> torch.Tensor:
    """utils.py:482-496, as written there."""
    src_len = content.shape[-1]
    target = torch.zeros([content.shape[0], target_len], dtype=content.dtype).to(content.device)
    temp = torch.arange(src_len + 1) * target_len / src_len
    current_pos = 0
    for i in range(target_len):
        if i < temp[current_pos + 1]:
            target[:, i] = content[:, current_pos]
        else:
            current_pos += 1
            target[:, i] = content[:, current_pos]
    return target


def convert_one(models: dict, wav: torch.Tensor, sr: int, prompt_mel: torch.Tensor, x_T: torch.Tensor, method: str, steps: int,
                dtype=torch.float64) -> Dict[str, torch.Tensor]:
    """One slice alone.  models: cv_sd / cv_heads, pre_sd / pre_layers (phone, prompt), unet_sd / unet_cfg, voc_sd.  Returns every
    stage: units [D, F], content [T, C], prompt [S, C], latent [100, T], audio [T * 256]."""
    wav24 = mel_oracle.resample(wav, sr, TARGET_SR, dtype)
    T = wav24.shape[0] // HOP
    wav16 = mel_oracle.resample(wav24, TARGET_SR, 16000, dtype)
    units = content_oracle.extract(models["cv_sd"], wav16[None], models["cv_heads"], dtype=dtype)[0].t()
    c = repeat_expand_2d(units, T)
    pre_sd = {k: v.to(dtype) for k, v in models["pre_sd"].items()}
    S = prompt_mel.shape[1]
    content, prompt = pre_model_oracle.pre_model_infer(pre_sd, c[None], prompt_mel[None].to(dtype), torch.tensor([T]), torch.tensor([S]),
                                                       *models["pre_layers"])
    unet_sd = {k: v.to(dtype) for k, v in models["unet_sd"].items()}
    fn = lambda x, t: unet_oracle.denoiser_forward(unet_sd, models["unet_cfg"], x, content, prompt, torch.tensor([S]), t.to(dtype))
    sch = sampler_oracle.OracleSchedule(models["betas"])
    x = x_T.reshape(1, 100, T).to(dtype)
    if method == "unipc":
        lat = sampler_oracle.unipc_bh(fn, sch, x, steps, variant="bh2")
    else:
        lat = sampler_oracle.dpmpp_2m(fn, sch, x, steps)
    audio = vocos_oracle.decode(models["voc_sd"], lat, HOP, dtype=dtype)[0]
    return dict(units=units, content=content[:, 0], prompt=prompt[:, 0], latent=lat[0], audio=audio)


# ------------------------------------------------------------------------------------------------ infer.py:99-141, literally
def pad_array(arr, target_length):
    current_length = arr.shape[0]
    if current_length >= target_length:
        return arr
    else:
        pad_width = target_length - current_length
        pad_left = pad_width // 2
        pad_right = pad_width - pad_left
        padded_arr = np.pad(arr, (pad_left, pad_right), 'constant', constant_values=(0, 0))
        return padded_arr


def split_list_by_n(list_collection, n, pre=0):
    for i in range(0, len(list_collection), n):
        yield list_collection[i - pre if i - pre >= 0 else i: i + n]


def cli_loop(audio_data, audio_sr: int, convert: Callable[[np.ndarray], np.ndarray], pad_seconds=0.5, clip=0, lg=0, lgr=0.75,
             target_sample: int = TARGET_SR) -> np.ndarray:
    """``convert(dat)`` gets each padded voice sub-slice (float64 at audio_sr) and returns its float32 24 kHz audio
    (``out_audio.cpu().numpy()``).  Returns the array ``soundfile.write`` receives."""
    per_size = int(clip * audio_sr)
    lg_size = int(lg * audio_sr)
    lg_size_r = int(lg_size * lgr)
    lg_size_c_l = (lg_size - lg_size_r) // 2
    lg_size_c_r = lg_size - lg_size_r - lg_size_c_l
    lg = np.linspace(0, 1, lg_size_r) if lg_size != 0 else 0
    audio = []
    for (slice_tag, data) in audio_data:
        length = int(np.ceil(len(data) / audio_sr * target_sample))
        if slice_tag:
            _audio = np.zeros(length)
            audio.extend(list(pad_array(_audio, length)))
            continue
        if per_size != 0:
            datas = split_list_by_n(data, per_size, lg_size)
        else:
            datas = [data]
        for k, dat in enumerate(datas):
            per_length = int(np.ceil(len(dat) / audio_sr * target_sample)) if clip != 0 else length
            pad_len = int(audio_sr * pad_seconds)
            dat = np.concatenate([np.zeros([pad_len]), dat, np.zeros([pad_len])])
            _audio = convert(dat)
            pad_len = int(target_sample * pad_seconds)
            _audio = _audio[pad_len:-pad_len]
            _audio = pad_array(_audio, per_length)
            if lg_size != 0 and k != 0:
                lg1 = audio[-(lg_size_r + lg_size_c_r):-lg_size_c_r] if lgr != 1 else audio[-lg_size:]
                lg2 = _audio[lg_size_c_l:lg_size_c_l + lg_size_r] if lgr != 1 else _audio[0:lg_size]
                lg_pre = lg1 * (1 - lg) + lg2 * lg
                audio = audio[0:-(lg_size_r + lg_size_c_r)] if lgr != 1 else audio[0:-lg_size]
                audio.extend(lg_pre)
                _audio = _audio[lg_size_c_l + lg_size_r:] if lgr != 1 else _audio[lg_size:]
            audio.extend(list(_audio))
    return np.asarray(audio, dtype=np.float64) if audio else np.zeros(0)
