"""Block-isolated accuracy of the denoiser and of the condition encoders against fp64.

The denoiser does not compute in fp32: its GEMMs are 3xBF16, its attention scores are 3xBF16, its softmax weights are fp16
once there are >= 256 keys (V is then an fp16 hi/lo pair), its LayerNorms are folded into the consumer GEMM as
rstd (x W' - mu g), and its GroupNorm statistics are one-pass sums.  The parity tests elsewhere compare whole forwards with
the fp32 CPU oracle on the synthetic init, where attention is nearly uniform and activations are centred.  Here:

* every op of ``arch.build_plan`` (and conv_in and the output head) is re-run by the oracle on the GPU's OWN input for that
  op, taken from the engine's taps, once in fp64 (the truth) and once in fp32 (the yardstick's own error), so each block is
  judged on its own error and an error in one block is not averaged into the rest of the network;
* the weights are the synthetic init and four named transformations of it ("regimes") that each push one precision trick
  off the synthetic init's easy ground:

    sharp      to_q, to_k of every attention x g, g set so that the fp64 pre-softmax score std is ~4: 3xBF16 Q K^T, fp16 P
    large_v    to_v x 256 and to_out.0.weight x 1/256 (block outputs unchanged): the fp16 hi/lo V operand
    gn_offset  +30 rms on conv_in's and every resnet conv2's bias: GroupNorm statistics from one-pass sums
    ln_offset  proj_in.bias + 100: the folded LayerNorm's cancellation at |row mean| >> row std

* the shapes put ragged key lengths on the 64-key tile edges (1, 63-65, 255-257), mix the v1 and the TMA-fed attention
  kernel in one program (S = 800), and fill the staged-bias capacity exactly (S = 1024).

Contract per block (ref = fp64 output, e32 = max |fp32 - fp64| of the same block on the same input):
  elementwise  |gpu - ref| <= max(1e-3 |ref| + 1e-4 rms(ref), 2 e32)
  normwise     ||gpu - ref||_2 / ||inc||_2 <= 1e-4, inc = ref - residual input for resnet and transformer blocks (the
               block's own contribution: an attention error is not diluted by the stream it is added to), ref otherwise
"""
import math
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from ns2vc_b200.arch import build_plan, ns2vc_denoiser_config
from ns2vc_b200.synth import make_inputs, make_state_dict
from oracle import pre_model_oracle as po
from oracle import unet_oracle

pytestmark = pytest.mark.gpu
RTOL, ATOL_RMS, NORM_TOL = 1e-3, 1e-4, 1e-4
TARGET_SCORE_STD = 4.0
P_MODE = "split" if os.environ.get("NS2VC_ATTN_P", "").startswith("s") else "fp16"

# id: (B, T, S, refer_lengths)
SHAPES = {
    "A": (4, 1024, 256, (256, 255, 65, 1)),   # fp16 P: self-attention at levels 0-2; split P at level 3 and in cross-attention
    "B": (2, 520, 200, (200, 64)),            # split-P cross-attention; 520 / 260 / 130 / 65 rows are not multiples of 64
    "C": (1, 256, 800, (800,)),               # level 0 (dh 16, > 768 biased keys) on the v1 kernel, levels 1-3 on v2
    "D": (2, 136, 1024, (1024, 1000)),        # dh >= 32 at exactly the 1024-key staged-bias capacity
}
REGIMES = ("synthetic", "sharp", "large_v", "gn_offset", "ln_offset")
CASES = [("A", r) for r in REGIMES] + [(s, r) for s in "BCD" for r in ("synthetic", "sharp")]

_cache = {}


# ------------------------------------------------------------------ measurement helpers
def contract(got, ref, e32, inc):
    """(worst elementwise err / tol, normwise ||got - ref|| / ||inc||) of the rule in the module docstring."""
    got, ref = got.double(), ref.double()
    err = (got - ref).abs()
    rms = ref.pow(2).mean().sqrt()
    tol = torch.clamp(RTOL * ref.abs() + ATOL_RMS * rms, min=2 * e32)
    return (err / tol).max().item(), ((got - ref).norm() / inc.double().norm().clamp_min(1e-300)).item()


class ScoreStd:
    """Records the std of the pre-softmax scores q k^T / sqrt(dh) over the unmasked keys of every attention the oracle runs
    (the denoiser's Attention or the encoders' MultiheadAttention), keyed by the layer prefix."""

    def __init__(self, module, name, scores):
        self.module, self.name, self.scores, self.std = module, name, scores, {}

    def __enter__(self):
        orig = self.orig = getattr(self.module, self.name)

        def wrapped(sd, p, *a, **kw):
            s, keep = self.scores(sd, p, *a, **kw)
            s = s.masked_select(keep.expand_as(s))
            self.std[p] = s.std().item()
            return orig(sd, p, *a, **kw)
        setattr(self.module, self.name, wrapped)
        return self

    def __exit__(self, *exc):
        setattr(self.module, self.name, self.orig)


def _unet_scores(sd, p, hs, ehs, mask_bias, heads):
    B = hs.shape[0]
    q = F.linear(hs, sd[p + ".to_q.weight"])
    k = F.linear(hs if ehs is None else ehs, sd[p + ".to_k.weight"])
    dh = q.shape[-1] // heads
    s = torch.einsum("bqhd,bkhd->bhqk", q.view(B, -1, heads, dh), k.view(B, -1, heads, dh)) / math.sqrt(dh)
    keep = torch.ones((B, 1, 1, k.shape[1]), dtype=torch.bool) if mask_bias is None else (mask_bias == 0)[:, None]
    return s, keep


def _pre_scores(sd, p, x_tbc, pad_mask_bt):
    T, B, C = x_tbc.shape
    dh = C // po.N_HEADS
    q, k, _ = F.linear(x_tbc, sd[p + ".in_proj_weight"]).chunk(3, dim=-1)
    s = torch.einsum("qbhd,kbhd->bhqk", q.reshape(T, B, po.N_HEADS, dh), k.reshape(T, B, po.N_HEADS, dh)) / math.sqrt(dh)
    return s, ~pad_mask_bt[:, None, None, :]


# ------------------------------------------------------------------ denoiser: oracle side
CFG = ns2vc_denoiser_config()


def case_inputs(shape):
    B, T, S, lens = SHAPES[shape]
    inp = make_inputs(B, T, S, seed=300 + ord(shape))
    inp["refer_lengths"] = torch.tensor(lens, dtype=torch.int64)
    x = torch.cat([inp["x"], inp["content"].permute(1, 2, 0)], 1)
    ehs = inp["prompt"].permute(1, 0, 2).contiguous()
    mask = unet_oracle.sequence_mask(inp["refer_lengths"], S)
    t = torch.linspace(17.5, 941.25, B)
    return x, t, ehs, mask


def oracle_forward(sd, shape, dtype):
    """Full oracle forward of a case in `dtype`; returns (out, {tap name: activation})."""
    x, t, ehs, mask = case_inputs(shape)
    taps = {}
    sdd = {k: v.to(dtype) for k, v in sd.items()}
    with torch.no_grad():
        out = unet_oracle.unet_forward(sdd, CFG, x.to(dtype), t, ehs.to(dtype), mask, tap=lambda n, v: taps.__setitem__(n, v))
    return out, taps


def synthetic_reference(shape):
    """fp64 oracle run of the synthetic init (cached): its taps and its per-layer score std."""
    key = ("synthetic64", shape)
    if key not in _cache:
        with ScoreStd(unet_oracle, "attention", _unet_scores) as rec:
            out, taps = oracle_forward(make_state_dict(CFG, 0), shape, torch.float64)
        _cache[key] = (out, taps, rec.std)
    return _cache[key]


def sharp_gain():
    """Gain on to_q and to_k (scores scale by g^2) that takes the synthetic init's mean score std (shape A, fp64) to ~4."""
    std = synthetic_reference("A")[2]
    s0 = sum(std.values()) / len(std)
    return math.sqrt(TARGET_SCORE_STD / s0), s0


def regime_state_dict(regime):
    sd = make_state_dict(CFG, 0)
    if regime == "sharp":
        g, _ = sharp_gain()
        for k in sd:
            if re.search(r"\.attn[12]\.to_[qk]\.weight$", k):
                sd[k] = sd[k] * g
    elif regime == "large_v":
        for k in sd:
            if re.search(r"\.attn[12]\.to_v\.weight$", k):
                sd[k] = sd[k] * 256.0
            elif re.search(r"\.attn[12]\.to_out\.0\.weight$", k):
                sd[k] = sd[k] / 256.0
    elif regime == "gn_offset":
        # the same offset on every channel of a group: the group mean becomes large against the group std
        taps = synthetic_reference("A")[1]
        rms = lambda n: taps[n].pow(2).mean().sqrt().item()
        sd["conv_in.bias"] = sd["conv_in.bias"] + 30 * rms("conv_in")
        for op in build_plan(CFG):
            if op.kind == "resnet":
                sd[op.prefix + ".conv2.bias"] = sd[op.prefix + ".conv2.bias"] + 30 * rms(op.prefix)
    elif regime == "ln_offset":
        for k in sd:
            if k.endswith("proj_in.bias"):
                sd[k] = sd[k] + 100.0
    else:
        assert regime == "synthetic", regime
    return sd


def block_table(sd, shape, gpu_out, gpu_taps, emb64):
    """Every block re-run in fp64 and fp32 on the GPU's own input for it.  Returns [(block, elem ratio, normwise, e32)]."""
    x, t, ehs, mask = case_inputs(shape)
    sd64 = {k: v.double() for k, v in sd.items()}
    mb64 = ((1 - mask.double()) * -10000.0).unsqueeze(1)
    mb32 = ((1 - mask.float()) * -10000.0).unsqueeze(1)
    emb32 = emb64.float()
    rows = []

    def judge(name, fn64, fn32, h_in, got, residual, gn_input=False):
        with torch.no_grad():
            ref = fn64(h_in.double())
            r32 = fn32(h_in.float())
        e32 = (r32.double() - ref).abs().max().item()
        inc = ref - h_in.double() if residual else ref
        elem, norm = contract(got, ref, e32, inc)
        n32 = ((r32.double() - ref).norm() / inc.norm()).item()
        rows.append((name, elem, norm, e32, n32, norm_allowance(h_in) if gn_input else NORM_TOL))

    judge("conv_in", lambda h: F.conv1d(h, sd64["conv_in.weight"], sd64["conv_in.bias"], padding=1),
          lambda h: F.conv1d(h, sd["conv_in.weight"], sd["conv_in.bias"], padding=1), x, gpu_taps["conv_in"], False)
    h = gpu_taps["conv_in"].double()
    skips = []
    for op in build_plan(CFG):
        if op.kind in ("push", "pop_cat"):
            h = unet_oracle.block_forward(sd64, CFG, op, h, skips, emb64, ehs.double(), mb64)
            continue
        got = gpu_taps[op.prefix]
        residual = op.kind in ("resnet", "xformer") and op.cin == op.cout
        judge(op.prefix,
              lambda v, op=op: unet_oracle.block_forward(sd64, CFG, op, v, list(skips), emb64, ehs.double(), mb64),
              lambda v, op=op: unet_oracle.block_forward(sd, CFG, op, v, [s.float() for s in skips], emb32, ehs, mb32),
              h, got, residual, gn_input=op.kind in ("resnet", "xformer"))
        h = got.double()
    judge("head", lambda v: unet_oracle.head_forward(sd64, CFG, v), lambda v: unet_oracle.head_forward(sd, CFG, v), h, gpu_out, False,
          gn_input=True)
    return rows


def norm_allowance(h_in):
    """Normwise bound of a block that starts with a GroupNorm of its input.  The engine normalises the input inside the consumer
    GEMM from the input's bf16 hi/lo pair, which keeps 16 significant bits: |x - (hi + lo)| <= 2^-17 |x|.  After the GroupNorm
    that error is <= 2^-17 |x| / sigma_g, i.e. 2^-17 r relative to the normalised values' unit scale, with r = max over
    (sample, group) of rms(x) / std(x).  On centred activations r ~ 1 and the contract's 1e-4 holds with room to spare; a
    group mean far from 0 (the 'gn_offset' regime: r up to ~100) makes this term the larger one."""
    B, C, T = h_in.shape
    g = h_in.double().reshape(B, CFG.norm_num_groups, -1)
    r = (g.pow(2).mean(-1).sqrt() / g.std(-1, unbiased=False)).max().item()
    return max(NORM_TOL, 2.0 ** -17 * r)


# ------------------------------------------------------------------ denoiser: GPU side
@pytest.fixture(scope="module")
def unet():
    from ns2vc_b200.unet import UNet1DConditionModel
    m = UNet1DConditionModel(in_channels=CFG.in_channels, out_channels=CFG.out_channels, block_out_channels=CFG.block_out_channels,
                             layers_per_block=list(CFG.layers_per_block), norm_num_groups=CFG.norm_num_groups,
                             cross_attention_dim=CFG.cross_attention_dim, attention_head_dim=CFG.num_heads,
                             addition_embed_type=CFG.addition_embed_type, resnet_time_scale_shift=CFG.resnet_time_scale_shift)
    m.load_state_dict(make_state_dict(CFG, 0), strict=True)
    return m.to("cuda").eval()


def gpu_forward(m, sd, shape):
    from ns2vc_b200.debug import forward_with_taps
    m.load_state_dict(sd, strict=True)
    x, t, ehs, mask = case_inputs(shape)
    out, taps = forward_with_taps(m, x.cuda(), t.cuda(), ehs.cuda(), mask.cuda())
    return out.cpu(), {k: v.cpu() for k, v in taps.items()}


def run_case(m, shape, regime):
    """One case: GPU forward with taps, fp64/fp32 oracle end to end and per block.  Cached per (shape, regime)."""
    key = ("case", shape, regime)
    if key in _cache:
        return _cache[key]
    sd = regime_state_dict(regime)
    gpu_out, gpu_taps = gpu_forward(m, sd, shape)
    score = None
    if regime == "sharp" and shape == "A":
        with ScoreStd(unet_oracle, "attention", _unet_scores) as rec:
            ref, taps64 = oracle_forward(sd, shape, torch.float64)
        score = rec.std
    else:
        ref, taps64 = oracle_forward(sd, shape, torch.float64)
    ref32, _ = oracle_forward(sd, shape, torch.float32)
    e2e = contract(gpu_out, ref, (ref32.double() - ref).abs().max().item(), ref)
    rows = block_table(sd, shape, gpu_out, gpu_taps, taps64["emb"])
    res = dict(rows=rows, e2e=e2e, score=score, e32=(ref32.double() - ref).abs().max().item())
    _cache[key] = res
    return res


def worst(rows):
    """The rows with the worst elementwise ratio and the worst normwise error relative to its bound."""
    we = max(rows, key=lambda r: r[1])
    wn = max(rows, key=lambda r: r[2] / r[5])
    return we, wn


@pytest.mark.parametrize("shape,regime", CASES, ids=[f"{s}_{r}" for s, r in CASES])
def test_denoiser_blocks_vs_fp64(unet, shape, regime):
    B, T, S, lens = SHAPES[shape]
    res = run_case(unet, shape, regime)
    tag = f"{shape}_{regime}"
    print(f"\n== {tag}  B={B} T={T} S={S} refer_lengths={list(lens)}  softmax weights P: {P_MODE} (fp16: self-attention over >= 256 keys)")
    if regime == "sharp":
        g, s0 = sharp_gain()
        print(f"   sharp gain g={g:.3f} (synthetic mean score std {s0:.3f})")
        if res["score"]:
            sv = sorted(res["score"].values())
            print(f"   fp64 score std under 'sharp': min {sv[0]:.2f} mean {sum(sv) / len(sv):.2f} max {sv[-1]:.2f} over {len(sv)} attentions")
    print(f"   {'block':44s} {'elem err/tol':>12s} {'norm err':>10s} {'norm bound':>10s} {'fp32 max':>10s} {'fp32 norm':>10s}")
    for name, elem, norm, e32, n32, nb in res["rows"]:
        print(f"   {name:44s} {elem:12.3f} {norm:10.2e} {nb:10.2e} {e32:10.2e} {n32:10.2e}")
    we, wn = worst(res["rows"])
    print(f"   end to end: elem err/tol {res['e2e'][0]:.3f}, ||err||/||ref|| {res['e2e'][1]:.2e}, fp32 max {res['e32']:.2e}")
    print(f"WORST {tag} P={P_MODE} elem {we[1]:.4f} ({we[0]}) norm {wn[2]:.3e} ({wn[0]}, bound {wn[5]:.2e})")
    bad = [f"{n}: elem err/tol {e:.3f}, norm {nm:.2e} (bound {nb:.2e})" for n, e, nm, _, _, nb in res["rows"] if e > 1.0 or nm > nb]
    assert not bad, f"{tag}: blocks outside the contract (elem err/tol <= 1, norm <= bound):\n" + "\n".join(bad)
    assert res["e2e"][0] <= 1.0, f"{tag}: end-to-end output elem err/tol {res['e2e'][0]:.3f}"


def test_fp16_softmax_weights_against_the_split_path(unet):
    """Shape A under 'sharp' again with NS2VC_ATTN_P=split (bf16 hi/lo softmax weights everywhere) in a child process: it must
    pass too, and both paths' worst block errors are printed side by side - the price of fp16 P where it matters."""
    here = run_case(unet, "A", "sharp")
    child_env = dict(os.environ, NS2VC_ATTN_P="split")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "-s", "-m", "gpu", "-p", "no:cacheprovider",
                        "-k", "test_denoiser_blocks_vs_fp64 and A_sharp"], env=child_env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and " passed" in r.stdout, f"split P:\n{r.stdout[-3000:]}\n{r.stderr[-500:]}"
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("WORST A_sharp P=split")]
    assert line, r.stdout[-3000:]
    we, wn = worst(here["rows"])
    e2e = [ln for ln in r.stdout.splitlines() if ln.startswith("   end to end")]
    print(f"\nA_sharp worst blocks, P={P_MODE}: elem {we[1]:.4f} ({we[0]}) norm {wn[2]:.3e} ({wn[0]}); "
          f"end to end elem err/tol {here['e2e'][0]:.3f}")
    print(line[0] + ("; split P" + e2e[0].strip()[len("end to end"):] if e2e else ""))
    per_block = [ln for ln in r.stdout.splitlines() if ln.startswith("   ") and "attentions" in ln]
    print("split-P transformer blocks (block, elem err/tol, norm err, norm bound, fp32 max, fp32 norm):\n" + "\n".join(per_block))


# ------------------------------------------------------------------ condition encoders (Pre_model.infer)
PRE_FULL = {"phoneme_encoder": dict(in_channels=256, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2),
            "prompt_encoder": dict(in_channels=100, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2)}
PRE_B, PRE_T, PRE_S = 6, 129, 257
PRE_LENGTHS = (129, 128, 65, 64, 63, 1)
PRE_REFER_LENGTHS = (257, 256, 129, 64, 2, 1)


def pre_inputs():
    g = torch.Generator().manual_seed(41)
    c = torch.randn((PRE_B, 256, PRE_T), generator=g)
    refer = torch.randn((PRE_B, 100, PRE_S), generator=g)
    return c, refer, torch.tensor(PRE_LENGTHS), torch.tensor(PRE_REFER_LENGTHS)


def _bf16_pair(t):
    hi = t.to(torch.bfloat16).to(t.dtype)
    return hi, (t - hi).to(torch.bfloat16).to(t.dtype)


def _self_attention_3xbf16_scores(sd, p, x_tbc, pad_mask_bt):
    """po.self_attention in exact arithmetic except for the scores, which are formed as the encoders' attention kernels form
    them: q and k as bf16 hi/lo pairs, s = qh kh^T + ql kh^T + qh kl^T (the ql kl^T term dropped), scaled afterwards."""
    T, B, C = x_tbc.shape
    H = po.N_HEADS
    dh = C // H
    q, k, v = F.linear(x_tbc, sd[p + ".in_proj_weight"]).chunk(3, dim=-1)
    heads = lambda t: t.contiguous().view(T, B * H, dh).transpose(0, 1)
    (qh, ql), (kh, kl), v = _bf16_pair(heads(q)), _bf16_pair(heads(k)), heads(v)
    s = (qh @ kh.transpose(1, 2) + ql @ kh.transpose(1, 2) + qh @ kl.transpose(1, 2)) * math.sqrt(1.0 / dh)
    bias = torch.zeros((B, 1, 1, T), dtype=x_tbc.dtype).masked_fill(pad_mask_bt.view(B, 1, 1, T), float("-inf"))
    s = s + bias.expand(-1, H, -1, -1).reshape(B * H, 1, T)
    o = torch.bmm(torch.softmax(s, dim=-1), v).transpose(0, 1).contiguous().view(T * B, C)
    return F.linear(o, sd[p + ".out_proj.weight"]).view(T, B, C)


def pre_oracle(sd, dtype, tap=None):
    c, refer, lengths, refer_lengths = pre_inputs()
    with torch.no_grad():
        return po.pre_model_infer({k: v.to(dtype) for k, v in sd.items()}, c.to(dtype), refer.to(dtype), lengths, refer_lengths, 6, 6, tap=tap)


@pytest.mark.parametrize("regime", ["synthetic", "sharp"])
def test_condition_encoders_vs_fp64(regime):
    from ns2vc_b200.pre_model import Pre_model
    m = Pre_model(PRE_FULL)
    sd = po.synth_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}, seed=1)
    if regime == "sharp":
        with ScoreStd(po, "self_attention", _pre_scores) as rec:
            pre_oracle(sd, torch.float64)
        s0 = sum(rec.std.values()) / len(rec.std)
        g = math.sqrt(TARGET_SCORE_STD / s0)
        for k in sd:
            if k.endswith("self_attn.in_proj_weight"):
                C = sd[k].shape[1]
                sd[k] = torch.cat([sd[k][:2 * C] * g, sd[k][2 * C:]])
        with ScoreStd(po, "self_attention", _pre_scores) as rec:
            pre_oracle(sd, torch.float64)
        sv = sorted(rec.std.values())
        print(f"\nsharp gain g={g:.3f} (synthetic mean score std {s0:.3f}); fp64 score std now {sv[0]:.2f}-{sv[-1]:.2f}")
    m.load_state_dict(sd, strict=True)
    m = m.to("cuda").eval()
    c, refer, lengths, refer_lengths = pre_inputs()
    data = (c.cuda(), refer.cuda(), None, None, None, lengths.cuda(), refer_lengths.cuda(), None)
    content, prompt = (v.cpu() for v in m.infer(data))
    taps = m.taps(data)
    taps64 = {}
    ref_c, ref_p = pre_oracle(sd, torch.float64, tap=taps64)
    r32_c, r32_p = pre_oracle(sd, torch.float32)
    # The precision term fp32 does not have: Q K^T on bf16 hi/lo pairs (16 significant bits per operand), whose absolute score
    # error grows with the scores themselves.  Its size here is the fp64 oracle's own output change when only the scores are
    # formed that way; like e32 it enters the elementwise rule as 2x its max.
    orig = po.self_attention
    po.self_attention = _self_attention_3xbf16_scores
    try:
        qk_c, qk_p = pre_oracle(sd, torch.float64)
    finally:
        po.self_attention = orig
    print(f"\n== encoders {regime}: B={PRE_B} T={PRE_T} lengths={list(PRE_LENGTHS)} S={PRE_S} refer_lengths={list(PRE_REFER_LENGTHS)}")
    for k, ref in taps64.items():                    # diagnostics only: these inputs are the oracle's, not the GPU's
        ref = ref.squeeze(-1).unsqueeze(1) if k == "ref_enc" else ref.transpose(0, 1)
        got = taps[k].cpu().double()
        print(f"   tap {k:32s} max|err| {(got - ref).abs().max().item():.2e}  ||err||/||ref|| {((got - ref).norm() / ref.norm()).item():.2e}")
    bad = []
    for name, got, ref, r32, rqk in (("content", content, ref_c, r32_c, qk_c), ("prompt", prompt, ref_p, r32_p, qk_p)):
        e32 = (r32.double() - ref).abs().max().item()
        eqk = (rqk - ref).abs().max().item()
        elem, norm = contract(got, ref, max(e32, eqk), ref)
        print(f"   {name:8s} elem err/tol {elem:.3f}  ||err||/||ref|| {norm:.2e}  fp32 max {e32:.2e}  3xBF16-score max {eqk:.2e}")
        if elem > 1.0:
            bad.append(f"{name}: elem err/tol {elem:.3f}")
    assert not bad, f"encoders {regime}: " + "; ".join(bad)
    for b in range(PRE_B):
        assert (content[PRE_LENGTHS[b]:, b] == 0).all(), f"content row {b}: padded frames are not exactly 0"
        assert (prompt[PRE_REFER_LENGTHS[b]:, b] == 0).all(), f"prompt row {b}: padded frames are not exactly 0"
