"""Small full-architecture run for compute-sanitizer: one ``utterance_losses`` call over five utterances whose lengths are off the
kernels' tile edges (two ragged batches: the encoders' and denoiser's ragged programs, q_sample and the ragged reduction)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from ns2vc_b200.arch import ns2vc_denoiser_config  # noqa: E402
from ns2vc_b200.loss import utterance_losses  # noqa: E402
from ns2vc_b200.pre_model import Pre_model  # noqa: E402
from ns2vc_b200.synth import make_pre_state_dict, make_state_dict  # noqa: E402
from ns2vc_b200.unet import UNet1DConditionModel  # noqa: E402

PRE_CFG = {"phoneme_encoder": dict(in_channels=256, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2),
           "prompt_encoder": dict(in_channels=100, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2)}
unet = UNet1DConditionModel(in_channels=356, out_channels=100, block_out_channels=(128, 256, 384, 512), norm_num_groups=8,
                            cross_attention_dim=256, attention_head_dim=8, addition_embed_type="text", resnet_time_scale_shift="scale_shift")
unet.load_state_dict(make_state_dict(ns2vc_denoiser_config(), 0))
pre = Pre_model(PRE_CFG)
pre.load_state_dict(make_pre_state_dict(PRE_CFG, 0))
unet, pre = unet.cuda().eval(), pre.cuda().eval()
g = torch.Generator().manual_seed(5)
items = [(torch.randn(256, T, generator=g), torch.randn(100, T, generator=g), torch.randn(100, S, generator=g))
         for T, S in ((37, 18), (65, 7), (130, 55), (201, 23), (97, 40))]
torch.manual_seed(0)
r = utterance_losses(pre, unet, items, max_batch=3)
torch.cuda.synchronize()
print("ok", r.t.tolist(), [f"{v:.4e}" for v in r.loss.tolist()])
