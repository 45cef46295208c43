"""Write tests/golden/content_tiny.pt: transformers' eager ``HubertModel`` (a port of fairseq's HubertModel) at a tiny
ContentVec-shaped configuration, its seeded initial weights renamed to fairseq's ``HubertModel`` names, two inputs (0.6 s and
0.4 s at 16 kHz, each run alone), transformers' ``last_hidden_state`` of each, and ``final_proj`` of it (transformers has no
final_proj: its weights are seeded here).  It asserts that ``oracle/content_oracle.py`` reproduces transformers in fp32 (within
1e-5 relative) before writing, so the fixture pins the oracle with no transformers at test time.

What this pins: the oracle's arithmetic (conv stack, GroupNorm, SamePad, weight norm, post-LN layers) against an independent
production implementation.  What it does not: fairseq itself or the ContentVec checkpoint (both absent), and the fairseq key
names, which only the strict loader checks.

    python oracle/make_golden_content.py        (needs transformers; reads nothing outside this repository)
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import content_oracle  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "content_tiny.pt")
CFG = dict(conv_dim=32, embed_dim=32, ffn_dim=64, num_layers=2, num_heads=2, pos_conv_kernel=16, pos_conv_groups=4, final_dim=16)
LENGTHS = [9600, 6400]
SEED = 20


def to_fairseq(name: str):
    """transformers HubertModel key -> fairseq HubertModel key (None: not a fairseq inference weight)"""
    n = name
    if n == "masked_spec_embed":
        return None
    if n.startswith("feature_extractor.conv_layers."):
        return n.replace(".conv.weight", ".0.weight").replace(".layer_norm.", ".2.")
    if n.startswith("feature_projection.layer_norm."):
        return n.replace("feature_projection.", "")
    if n.startswith("feature_projection.projection."):
        return n.replace("feature_projection.projection", "post_extract_proj")
    if n.startswith("encoder.pos_conv_embed.conv."):
        leaf = n[len("encoder.pos_conv_embed.conv."):]
        leaf = {"parametrizations.weight.original0": "weight_g", "parametrizations.weight.original1": "weight_v"}.get(leaf, leaf)
        return "encoder.pos_conv.0." + leaf
    if n.startswith("encoder.layers."):
        return (n.replace(".attention.", ".self_attn.").replace(".layer_norm.", ".self_attn_layer_norm.")
                .replace(".feed_forward.intermediate_dense.", ".fc1.").replace(".feed_forward.output_dense.", ".fc2."))
    return n                                                   # encoder.layer_norm.*


def main() -> None:
    import transformers
    c = CFG
    hc = transformers.HubertConfig(
        hidden_size=c["embed_dim"], num_hidden_layers=c["num_layers"], num_attention_heads=c["num_heads"], intermediate_size=c["ffn_dim"],
        conv_dim=(c["conv_dim"],) * 7, conv_stride=(5, 2, 2, 2, 2, 2, 2), conv_kernel=(10, 3, 3, 3, 3, 2, 2),
        num_conv_pos_embeddings=c["pos_conv_kernel"], num_conv_pos_embedding_groups=c["pos_conv_groups"], feat_extract_norm="group",
        conv_bias=False, do_stable_layer_norm=False, hidden_act="gelu", feat_extract_activation="gelu", feat_proj_layer_norm=True,
        layer_norm_eps=1e-5, hidden_dropout=0.0, attention_dropout=0.0, activation_dropout=0.0, feat_proj_dropout=0.0, layerdrop=0.0,
        apply_spec_augment=False)
    torch.manual_seed(SEED)
    model = transformers.HubertModel(hc).eval()
    g = torch.Generator().manual_seed(SEED + 1)
    sd = {}
    for k, v in model.state_dict().items():
        fk = to_fairseq(k)
        if fk is not None:
            # LayerNorm / GroupNorm affine and biases start at 1 / 0 in transformers: perturb them so that the fixture exercises them
            t = v.detach().clone().float()
            if fk.endswith(".bias") or fk.endswith("norm.weight") or fk.endswith(".2.weight"):
                t = t + 0.1 * torch.randn(t.shape, generator=g)
            sd[fk] = t
    model.load_state_dict({k: sd[to_fairseq(k)] for k in model.state_dict() if to_fairseq(k) is not None}, strict=False)
    sd["final_proj.weight"] = torch.randn((c["final_dim"], c["embed_dim"]), generator=g) / c["embed_dim"] ** 0.5
    sd["final_proj.bias"] = 0.02 * torch.randn(c["final_dim"], generator=g)
    N = max(LENGTHS)
    wav = torch.zeros((len(LENGTHS), N))
    t = torch.arange(N) / 16000.0
    wav[0] = 0.1 * torch.randn(N, generator=g) + 0.2 * torch.sin(2 * torch.pi * 220.0 * t)
    wav[1, :LENGTHS[1]] = 0.1 * torch.randn(LENGTHS[1], generator=g) + 0.05
    T = content_oracle.num_frames(N)
    hidden = torch.zeros((len(LENGTHS), T, c["embed_dim"]))
    with torch.no_grad():
        for b, n in enumerate(LENGTHS):
            hs = model(wav[b:b + 1, :n]).last_hidden_state[0]
            hidden[b, :hs.shape[0]] = hs
        units = torch.nn.functional.linear(hidden, sd["final_proj.weight"], sd["final_proj.bias"])
        for b, n in enumerate(LENGTHS):
            units[b, content_oracle.num_frames(n):] = 0
    got = content_oracle.extract(sd, wav, c["num_heads"], LENGTHS, dtype=torch.float32)
    rel = ((got - units).abs().max() / units.abs().max()).item()
    assert rel <= 1e-5, rel
    torch.save(dict(cfg=c, state_dict=sd, wav=wav, lengths=torch.tensor(LENGTHS), last_hidden_state=hidden, units=units,
                    transformers_version=transformers.__version__), OUT)
    print(f"wrote {OUT}: oracle vs transformers {rel:.2e} relative")


if __name__ == "__main__":
    main()
