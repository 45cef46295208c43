"""The launch count of each engine's program, pinned at one small shape without lengths and one with: a change to how a program
is built or run that adds, drops or merges a launch shows here.  Tap copies are not counted, nor is the denoiser's MASKBIAS when
prepare_cond has no mask.  The values were recorded from the engines as they stood when the launch records became typed."""
import pytest
import torch

pytestmark = pytest.mark.gpu

EXPECTED = {
    "denoiser": {"padded": {"prepare_cond": 12, "forward": 216, "forward_film": 213},
                 "ragged": {"prepare_cond": 11, "forward": 216, "forward_film": 213}},
    "pre": {"padded": 46, "ragged": 46},
    "vocoder": {"padded": 13, "ragged": 13},
    "content": {"padded": 34, "ragged": 34},
}

PRE_CFG = {"phoneme_encoder": dict(in_channels=32, hidden_channels=32, out_channels=32, n_layers=2),
           "prompt_encoder": dict(in_channels=100, hidden_channels=32, out_channels=32, n_layers=2)}


def denoiser_counts(dev):
    from ns2vc_b200 import _lib
    from ns2vc_b200.arch import UNetConfig
    from ns2vc_b200.fused import DenoiserSession
    from ns2vc_b200.synth import make_inputs, make_state_dict
    from ns2vc_b200.unet import UNet1DConditionModel
    kw = dict(in_channels=36, out_channels=20, block_out_channels=(32, 64, 64, 96), norm_num_groups=8, cross_attention_dim=16,
              addition_embed_type="text", addition_embed_type_num_heads=4, resnet_time_scale_shift="scale_shift")
    m = UNet1DConditionModel(attention_head_dim=8, **kw)
    m.load_state_dict(make_state_dict(UNetConfig(num_heads=8, **kw), 0))
    m = m.to(dev).eval()
    L, h = _lib.lib(), m.engine(dev)
    B, T, S = 2, 37, 11
    inp = make_inputs(B, T, S, latent_ch=20, content_ch=16, seed=10)
    content, prompt = inp["content"].permute(1, 2, 0).contiguous().to(dev), inp["prompt"].permute(1, 0, 2).contiguous().to(dev)
    x, t = inp["x"].to(dev), torch.tensor([500.5, 37.25], device=dev)
    out = torch.empty((B, 20, T), device=dev)
    counts = {}
    for name, sess in (("padded", DenoiserSession(m, content, prompt, torch.ones((B, S), dtype=torch.bool, device=dev))),
                       ("ragged", DenoiserSession(m, content, prompt, None, content_lengths=[37, 20], prompt_lengths=[11, 4]))):
        c = {}
        sess.prepare()
        c["prepare_cond"] = L.ns2vc_unet_launch_count(h)
        sess.forward(x, t, out)
        c["forward"] = L.ns2vc_unet_launch_count(h)
        table = torch.empty(L.ns2vc_unet_time_table_floats(h, B), device=dev)
        sess.time_table(t, table)
        sess.forward(x, t, out, film_rows=table)
        c["forward_film"] = L.ns2vc_unet_launch_count(h)
        counts[name] = c
    torch.cuda.synchronize(dev)
    return counts


def pre_counts(dev):
    from ns2vc_b200.pre_model import Pre_model
    from ns2vc_b200.synth import make_pre_inputs, make_pre_state_dict
    m = Pre_model(PRE_CFG)
    m.load_state_dict(make_pre_state_dict(PRE_CFG, 0), strict=True)
    m = m.to(dev).eval()
    counts = {}
    for name, ragged in (("padded", False), ("ragged", True)):
        d = make_pre_inputs(3, 29, 17, content_ch=32, ragged=True, seed=2)
        m.infer((d["c"].to(dev), d["refer"].to(dev), None, None, None, d["lengths"], d["refer_lengths"], None), per_utterance=ragged)
        counts[name] = m.launch_count()
    return counts


def vocoder_counts(dev):
    from ns2vc_b200.synth import make_vocos_state_dict
    from ns2vc_b200.vocoder import Vocos
    m = Vocos.from_state_dict(make_vocos_state_dict(0, "init", input_channels=100, dim=128, intermediate_dim=384, num_layers=2)).to(dev).eval()
    mel = torch.randn((3, 100, 40), generator=torch.Generator().manual_seed(3)).to(dev)
    counts = {}
    for name, lengths in (("padded", None), ("ragged", torch.tensor([40, 23, 1]))):
        m.decode(mel, lengths)
        counts[name] = m.launch_count()
    return counts


def content_counts(dev):
    from ns2vc_b200.content import ContentVec
    from ns2vc_b200.synth import CONTENTVEC_SMALL, make_contentvec_state_dict
    m = ContentVec.from_state_dict(make_contentvec_state_dict(0, "init", **CONTENTVEC_SMALL), num_heads=CONTENTVEC_SMALL["num_heads"])
    m = m.to(dev).eval()
    wav = torch.randn((3, 4000), generator=torch.Generator().manual_seed(4)).to(dev)
    counts = {}
    for name, lengths in (("padded", None), ("ragged", torch.tensor([4000, 2500, 400]))):
        m.extract(wav, lengths)
        counts[name] = m.launch_count()
    return counts


def launch_counts():
    dev = torch.device("cuda", torch.cuda.current_device())
    with torch.no_grad():
        return {"denoiser": denoiser_counts(dev), "pre": pre_counts(dev), "vocoder": vocoder_counts(dev), "content": content_counts(dev)}


def test_launch_counts_are_pinned():
    assert launch_counts() == EXPECTED
