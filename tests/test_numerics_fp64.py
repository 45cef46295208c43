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
  kernel in one program (S = 800), and fill the staged-bias capacity exactly (S = 1024);
* ragged programs (per-utterance lengths T_b, S_b) are judged row by row against the oracle of each utterance ALONE, on the
  row's own GPU input [:T_b,l] of every block, under the same regimes; each row is also run through our own B = 1 padded
  program, every tap must be exactly 0 past the row's length, and a forward on a workspace full of NaN bytes must be
  bit-identical to one on a zeroed workspace.

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
import time

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


def oracle_run(sd, x, t, ehs, mask, dtype):
    """Full oracle forward in `dtype` (mask: bool [B, S] or None); returns (out, {tap name: activation})."""
    taps = {}
    sdd = {k: v.to(dtype) for k, v in sd.items()}
    with torch.no_grad():
        out = unet_oracle.unet_forward(sdd, CFG, x.to(dtype), t, ehs.to(dtype), mask, tap=lambda n, v: taps.__setitem__(n, v))
    return out, taps


def oracle_forward(sd, shape, dtype):
    """Full oracle forward of a padded case in `dtype`; returns (out, {tap name: activation})."""
    return oracle_run(sd, *case_inputs(shape), dtype)


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


def mask_bias(mask):
    """The reference's cross-attention bias [B, 1, S] of a bool keep mask (0 / -10000, exact in fp32 and fp64)."""
    return ((1 - mask.double()) * -10000.0).unsqueeze(1)


def block_table(sd, x, ehs, mb, emb64, gpu_out, gpu_taps):
    """Every block re-run in fp64 and fp32 on the GPU's own input for it.  x: conv_in's input [B, Cin, T]; ehs: the prompt
    [B, S, C]; mb: the cross-attention bias [B, 1, S] or None; emb64: the fp64 oracle's time embedding of the same run; gpu_out,
    gpu_taps: the GPU's output and taps of exactly these B rows and T frames.
    Returns [(block, elem err/tol, normwise, e32, fp32 normwise, normwise bound)]."""
    sd64 = {k: v.double() for k, v in sd.items()}
    mb64 = None if mb is None else mb.double()
    mb32 = None if mb is None else mb.float()
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
    ehs64, ehs32 = ehs.double(), ehs.float()
    for op in build_plan(CFG):
        if op.kind in ("push", "pop_cat"):
            h = unet_oracle.block_forward(sd64, CFG, op, h, skips, emb64, ehs64, mb64)
            continue
        got = gpu_taps[op.prefix]
        residual = op.kind in ("resnet", "xformer") and op.cin == op.cout
        judge(op.prefix,
              lambda v, op=op: unet_oracle.block_forward(sd64, CFG, op, v, list(skips), emb64, ehs64, mb64),
              lambda v, op=op: unet_oracle.block_forward(sd, CFG, op, v, [s.float() for s in skips], emb32, ehs32, mb32),
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
    x, _, ehs, mask = case_inputs(shape)
    rows = block_table(sd, x, ehs, mask_bias(mask), taps64["emb"], gpu_out, gpu_taps)
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


# ------------------------------------------------------------------ denoiser: ragged programs, each row against fp64 alone
# The ragged contract: row b equals utterance b run alone.  So the reference of row b is the oracle of that utterance alone
# (x[b, :, :T_b], content[:T_b], prompt[:S_b], no mask), and each block is judged on the GPU's own rows [:T_b,l] of its input,
# T_b,l = ceil(T_b / 2^l).  id: (B, T, S, rows (T_b, S_b))
RAGGED = {
    # per-entry key counts on the 64-key tile edges (1/64/65/128/129/255/257); short rows that the padded level length puts on
    # fp16 softmax weights (255 and 150 keys at level 0, 75 at level 1, 38 at level 2); a single prompt key; a single frame at
    # every level (GroupNorm over one row)
    "R1": (7, 1024, 256, ((1024, 256), (255, 40), (150, 1), (257, 65), (513, 64), (65, 255), (1, 256))),
    # level 0 (dh 16, > 768 biased prompt keys) on the fp32 kernel with the 0 / -inf self-attention key bias; levels 1-3 per-entry
    "R2": (3, 256, 800, ((256, 800), (100, 1), (33, 769))),
    # S > 1024: every transformer on the fp32 kernel
    "R3": (2, 300, 1100, ((300, 1100), (97, 300))),
}
RAGGED_CASES = [("R1", r) for r in REGIMES] + [(c, r) for c in ("R2", "R3") for r in ("synthetic", "sharp")]
NLEV = len(CFG.block_out_channels)


def ragged_inputs(case):
    """(x [B, 100, T], content [B, 256, T], prompt [B, S, 256], t [B]) of a ragged case, values everywhere."""
    B, T, S, _ = RAGGED[case]
    inp = make_inputs(B, T, S, seed=500 + int(case[1:]))
    return inp["x"], inp["content"].permute(1, 2, 0).contiguous(), inp["prompt"].permute(1, 0, 2).contiguous(), torch.linspace(17.5, 941.25, B)


def ragged_session(m, case):
    """A DenoiserSession of the case's ragged program (inputs on the GPU)."""
    from ns2vc_b200.fused import DenoiserSession
    _, _, _, rows = RAGGED[case]
    _, content, prompt, _ = ragged_inputs(case)
    return DenoiserSession(m, content.cuda(), prompt.cuda(), None, content_lengths=[r[0] for r in rows],
                           prompt_lengths=[r[1] for r in rows])


def gpu_alone(m, xin, t, ehs):
    """Our own B = 1 padded forward of one utterance (xin [1, Cin, T_b], ehs [1, S_b, C], no mask)."""
    from ns2vc_b200.fused import DenoiserSession
    Cl = m.latent_channels
    sess = DenoiserSession(m, xin[:, Cl:].contiguous().cuda(), ehs.contiguous().cuda(), None)
    out = torch.empty((1, CFG.out_channels, xin.shape[2]), device="cuda")
    sess.forward(xin[:, :Cl].contiguous().cuda(), t.cuda(), out)
    return out.cpu()


def run_ragged_case(m, case, regime):
    """One ragged forward with taps; per row: every tap and the output exactly 0 past the row's length, every block against
    fp64 on the row's own GPU input, the row end to end and our own B = 1 run of it against the fp64 oracle of the utterance
    alone.  Cached per (case, regime)."""
    key = ("ragged", case, regime)
    if key in _cache:
        return _cache[key]
    from ns2vc_b200.arch import level_lengths
    from ns2vc_b200.debug import session_forward_with_taps
    B, T, S, rows = RAGGED[case]
    sd = regime_state_dict(regime)
    m.load_state_dict(sd, strict=True)
    x, content, prompt, t = ragged_inputs(case)
    gpu_out, gpu_taps = session_forward_with_taps(ragged_session(m, case), x.cuda(), t.cuda())
    gpu_out, gpu_taps = gpu_out.cpu(), {k: v.cpu() for k, v in gpu_taps.items()}
    Tl = level_lengths(T, NLEV)
    per_row, oracle_s = [], 0.0
    for b, (Tb, Sb) in enumerate(rows):
        tb = level_lengths(Tb, NLEV)
        mine, stale = {}, []
        for name, v in gpu_taps.items():
            lvl = Tl.index(v.shape[2])
            mine[name] = v[b:b + 1, :, :tb[lvl]]
            if v[b, :, tb[lvl]:].any():
                stale.append(name)
        if gpu_out[b, :, Tb:].any():
            stale.append("output")
        xin, tb_t, ehs = torch.cat([x[b:b + 1, :, :Tb], content[b:b + 1, :, :Tb]], 1), t[b:b + 1], prompt[b:b + 1, :Sb]
        got = gpu_out[b:b + 1, :, :Tb]
        alone = gpu_alone(m, xin, tb_t, ehs)
        t0 = time.perf_counter()
        ref, taps64 = oracle_run(sd, xin, tb_t, ehs, None, torch.float64)
        ref32, _ = oracle_run(sd, xin, tb_t, ehs, None, torch.float32)
        e32 = (ref32.double() - ref).abs().max().item()
        blocks = block_table(sd, xin, ehs, None, taps64["emb"], got, mine)
        oracle_s += time.perf_counter() - t0
        per_row.append(dict(Tb=Tb, Sb=Sb, rows=blocks, e2e=contract(got, ref, e32, ref), alone=contract(alone, ref, e32, ref),
                            stale=stale, e32=e32))
    res = dict(rows=per_row, oracle_s=oracle_s)
    _cache[key] = res
    return res


@pytest.mark.parametrize("case,regime", RAGGED_CASES, ids=[f"{c}_{r}" for c, r in RAGGED_CASES])
def test_ragged_rows_blocks_vs_fp64(unet, case, regime):
    B, T, S, rows = RAGGED[case]
    res = run_ragged_case(unet, case, regime)
    tag = f"{case}_{regime}"
    print(f"\n== {tag}  ragged B={B} T={T} S={S} rows (T_b, S_b)={list(rows)}  softmax weights P: {P_MODE}  "
          f"(CPU oracle {res['oracle_s']:.0f} s)")
    print("   per block and row: elem err/tol | norm err / norm bound")
    print(f"   {'block':44s}" + "".join(f" {f'{Tb},{Sb}':>13s}" for Tb, Sb in rows))
    for i, name in enumerate(r[0] for r in res["rows"][0]["rows"]):
        cells = [rr["rows"][i] for rr in res["rows"]]
        print(f"   {name:44s}" + "".join(f" {c[1]:6.3f}|{c[2] / c[5]:6.3f}" for c in cells))
    print(f"   {'end to end, ragged row':44s}" + "".join(f" {rr['e2e'][0]:13.3f}" for rr in res["rows"]))
    print(f"   {'end to end, our own B=1 padded run':44s}" + "".join(f" {rr['alone'][0]:13.3f}" for rr in res["rows"]))
    bad = []
    for rr in res["rows"]:
        at = f"{tag} row (T_b={rr['Tb']}, S_b={rr['Sb']})"
        bad += [f"{at} {n}: elem err/tol {e:.3f}, norm {nm:.2e} (bound {nb:.2e})" for n, e, nm, _, _, nb in rr["rows"] if e > 1.0 or nm > nb]
        if rr["stale"]:
            bad.append(f"{at}: not exactly 0 past the row's length in {', '.join(rr['stale'])}")
        if rr["e2e"][0] > 1.0:
            bad.append(f"{at} end to end: elem err/tol {rr['e2e'][0]:.3f}")
    we = max(((rr["Tb"], rr["Sb"]) + r for rr in res["rows"] for r in rr["rows"]), key=lambda r: r[3])
    print(f"WORST {tag} P={P_MODE} elem {we[3]:.4f} ({we[2]}, row {we[0]},{we[1]}) end to end ragged "
          f"{max(rr['e2e'][0] for rr in res['rows']):.4f} / B=1 {max(rr['alone'][0] for rr in res['rows']):.4f}")
    assert not bad, f"{tag}: rows outside the contract (elem err/tol <= 1, norm <= bound, exact zeros past the length):\n" + "\n".join(bad)


# The padded program's fp16 softmax weights (self-attention over >= 256 keys) under 'sharp': the B = 1 runs of R1's 257- and
# 513-frame rows end at 1.004 and 1.075 of the tolerance (bf16 hi/lo weights everywhere, NS2VC_ATTN_P=split: 0.69 / 0.68).
# Split weights everywhere cost 1.2 % of the cfg2 throughput (1808 -> 1787 denoiser-steps/s on an H100 80GB HBM3 at 700 W), so
# the padded rule is kept for now and this case is an expected failure of the fp16 path: it fails the suite (strict) once it
# passes.
_B1_KNOWN = pytest.mark.xfail(P_MODE == "fp16", strict=True,
                              reason="fp16 softmax weights of the padded program exceed the end-to-end tolerance under 'sharp'")
B1_CASES = [pytest.param(c, r, id=f"{c}_{r}", marks=_B1_KNOWN if (c, r) == ("R1", "sharp") else ()) for c, r in RAGGED_CASES]


@pytest.mark.parametrize("case,regime", B1_CASES)
def test_padded_b1_rows_vs_fp64(unet, case, regime):
    """Each ragged row's utterance through our own B = 1 padded program, against the same fp64 reference end to end: the
    padded program at small, odd B = 1 shapes under the regimes."""
    res = run_ragged_case(unet, case, regime)
    bad = [f"{case}_{regime} row (T_b={rr['Tb']}, S_b={rr['Sb']}) our own B=1 padded run end to end: elem err/tol {rr['alone'][0]:.3f}"
           for rr in res["rows"] if rr["alone"][0] > 1.0]
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("program", ["ragged", "padded"])
def test_poisoned_workspace_changes_nothing(unet, program):
    """Every value a forward reads from the shared workspace was written by this prepare + forward: with the workspace filled
    with 0xFF bytes (NaN as fp32, bf16 and fp64) before the prepare, the output and every tap are bit-identical to the same run
    on a zeroed workspace.  Covers split columns between C and the row pitch, rows past a view's T, and the padded rows."""
    from ns2vc_b200.debug import run_with_taps
    from ns2vc_b200.fused import DenoiserSession
    B, T, S, _ = RAGGED["R1"]
    unet.load_state_dict(regime_state_dict("synthetic"), strict=True)
    x, content, prompt, t = (v.cuda() for v in ragged_inputs("R1"))
    sess = ragged_session(unet, "R1") if program == "ragged" else DenoiserSession(unet, content, prompt, None)
    out = torch.empty((B, CFG.out_channels, T), device="cuda")
    sess.forward(x, t, out)                                    # builds the program
    ws = unet.workspace(B, T, S, sess.dev)
    assert ws.data_ptr() == sess.ws.data_ptr()

    def run(byte):
        def go():
            ws.fill_(byte)
            sess.prepare()
            sess.forward(x, t, out)
            return out.clone()
        o, taps = run_with_taps(unet, sess.dev, B, T, go)
        return dict(taps, output=o)

    clean, dirty = run(0), run(0xFF)
    bits = lambda v: v.contiguous().view(torch.int32)
    bad = [f"{k}: {(~torch.isfinite(dirty[k])).sum().item()} non-finite, {(bits(dirty[k]) != bits(v)).sum().item()} of {v.numel()} differ"
           for k, v in clean.items() if not torch.equal(bits(dirty[k]), bits(v))]
    assert torch.isfinite(clean["output"]).all()
    assert not bad, f"{program} program on a 0xFF-filled workspace:\n" + "\n".join(bad)


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
