"""Load time: every engine's packed weights and load-time folds against fp64 folds of the reference state_dict
(oracle/pack_oracle.py).

CPU tier: the oracle's folds equal the reference math they replace, in fp64 on random inputs (the conv-FFN's k shifted
Linears, proj_out o ff.net.2, the positional conv's weight norm, fairseq's q scaling, Vocos' layer scale, the LayerNorm folded
into the condition encoders' out_proj with its conv bias), and the fold bounds are not vacuous: an fp32-accumulated fold breaks
them by 16x or more somewhere in the `fold_stress` regime.

GPU tier: each engine is packed (its C-ABI create / load / finalize) under its synthetic weights and under `fold_stress`, and
its packed-weight record is read back (ns2vc_check_packed / ns2vc_check_fold_vector).  Three things are asserted:

* coverage: the record names exactly the oracle's operands, in packing order, each once, with the oracle's shapes;
* exact images: the whole hi / lo image of every operand equals split(f32) bit for bit, padding included (columns past
  n_logical, channels past a segment's ncin: +0), where f32 is the packer's arithmetic emulated bit for bit (a copy, the TBC
  transpose, gamma W, the conv-FFN taps' two roundings, the layer scale, the q scaling and the weight norm in its kernel's
  order), or the engine's own fp32 Wp W2 for the merged feed-forward; segments never overlap (pack_oracle.assemble);
* bounded folds: every double-accumulated fold (ln_fold_vec, matmul_nn, matvec_bias) and the fp64 weight norm and q scaling
  lie within one fp32 rounding plus the fp64 sums, 2^-24 |exact| + (n + 2) 2^-53 sum |a_i b_i|; the conv-FFN taps within their
  two fp32 roundings.  Each family's worst ratio is printed.
"""
from __future__ import annotations

import ctypes as C
import math
import time
from collections import defaultdict

import pytest
import torch

from ns2vc_b200 import _lib
from oracle import pack_oracle as po

F64, F32 = torch.float64, torch.float32
ULP = 2.0 ** -24


# ------------------------------------------------------------------------------------------------------------------ CPU tier
def _rand(*shape, seed=0, scale=1.0):
    return scale * torch.randn(shape, generator=torch.Generator().manual_seed(seed), dtype=F64)


@pytest.mark.parametrize("k", [3, 5, 7, 9])
def test_ffn_fold_equals_shifted_linears(k):
    """TransformerFFNLayer's first stage (operations.py:678-684: zero pad by (k-1)/2, Linear i over padded[i:T+i] for i >= 1,
    Linear 0 over the unpadded x, sum, times k^-0.5) equals the oracle's (k-1)-tap conv (tap j at row offset j + 1 - (k-1)/2)."""
    T, B, H, F = 11, 2, 6, 10
    x = _rand(T, B, H, seed=k)
    ws = [_rand(F, H, seed=100 + j).float().double() for j in range(k)]
    b0 = _rand(F, seed=99)
    p = (k - 1) // 2
    padded = torch.cat([torch.zeros(p, B, H, dtype=F64), x, torch.zeros(p, B, H, dtype=F64)])
    ref = sum((padded[i:T + i] if i else x) @ ws[i].t() for i in range(k)) + b0
    ref = ref * k ** -0.5
    segs = po.ffn_taps([w.float() for w in ws])
    got = torch.zeros(T, B, F, dtype=F64)
    for j, s in enumerate(segs):
        off = j + 1 - p
        src = torch.zeros(T, B, H, dtype=F64)
        lo, hi = max(0, -off), min(T, T - off)
        src[lo:hi] = x[lo + off:hi + off]
        got += src @ s.exact.t()
    got += b0 * k ** -0.5
    assert (got - ref).abs().max().item() <= 1e-12 * ref.abs().max().item()
    # the folded bias and the fp32 emulation's two roundings
    s32 = po.ffn_scale(k)
    assert abs(s32 - k ** -0.5) <= ULP * k ** -0.5
    for s in segs:
        assert ((s.f32.double() - s.exact).abs() <= s.bound).all()


def test_ff2p_merge_equals_proj_out_of_ff2():
    """[Wp W2 | Wp] with bias Wp b2 + bp over K = [GEGLU output g | residual h] equals proj_out(ff.net.2(g) + h)."""
    from ns2vc_b200.arch import UNetConfig
    from ns2vc_b200.synth import make_state_dict
    cfg = UNetConfig(in_channels=36, out_channels=20, block_out_channels=(32, 64), norm_num_groups=8, cross_attention_dim=16,
                     num_heads=8, down_block_types=("CrossAttnDownBlock2D", "DownBlock2D"),
                     up_block_types=("UpBlock2D", "CrossAttnUpBlock2D"), layers_per_block=(1, 1))
    sd = make_state_dict(cfg, 3)
    ops = {o.name: o for o in po.denoiser(sd, cfg)}
    name = next(n for n in ops if n.endswith(".ff2p"))
    o = ops[name]
    p = name[:-len(".ff2p")]
    C = o.n_logical
    M = po.assemble(o, "exact")[:C]
    g, h = _rand(7, 4 * C, seed=1), _rand(7, C, seed=2)
    A = torch.zeros(7, 64 * o.nkb, dtype=F64)
    A[:, :4 * C] = g
    A[:, 64 * po.nkb_of(4 * C):64 * po.nkb_of(4 * C) + C] = h
    got = A @ M.t() + o.vecs["bias_ff2p"].exact
    b = p + ".transformer_blocks.0"
    ff2 = g @ sd[b + ".ff.net.2.weight"].double().t() + sd[b + ".ff.net.2.bias"].double()
    ref = (ff2 + h) @ sd[p + ".proj_out.weight"][:, :, 0].double().t() + sd[p + ".proj_out.bias"].double()
    assert (got - ref).abs().max().item() <= 1e-12 * ref.abs().max().item()


def test_weight_norm_equals_torch():
    """The oracle's fp64 weight norm equals torch._weight_norm(v, g, dim=2), its kernel emulation lies within the fold bound,
    and an all-zero column gives NaN in both (torch divides by the zero norm too)."""
    v = _rand(24, 6, 5, seed=4).float()
    g = (_rand(1, 1, 5, seed=5).abs() + 0.1).float()
    v[:, :, 0] *= 1e-20
    v[:, :, 2] = 0
    g[..., 1] = 0
    ref = torch._weight_norm(v.double(), g.double(), 2)
    w64 = po.weight_norm_f64(v, g)
    assert torch.equal(torch.isnan(ref), torch.isnan(w64)) and torch.isnan(ref[:, :, 2]).all()
    fin = ~torch.isnan(ref)
    assert ((w64 - ref).abs()[fin] <= 1e-14 * ref.abs()[fin]).all()
    emu = po.weight_norm_emulate(v, g).double()
    assert torch.equal(torch.isnan(emu), torch.isnan(ref))
    assert ((emu - w64).abs()[fin] <= po.fold_bound(w64, w64.abs(), 24 * 6)[fin]).all()


def test_qscale_stack_equals_fairseq_q_scaling():
    """The content encoder's [q_proj * scaling | k_proj | v_proj] stack and bias equal fairseq MHA's q_proj(x) * scaling,
    k_proj(x), v_proj(x)."""
    from ns2vc_b200.synth import CONTENTVEC_SMALL, make_contentvec_state_dict
    cfg = dict(CONTENTVEC_SMALL)
    sd = make_contentvec_state_dict(0, "trained_like", **cfg)
    o = next(x for x in po.content(sd, cfg) if x.name == "encoder.layers.1.qkv")
    D = cfg["embed_dim"]
    Wst = po.assemble(o, "exact")[:3 * D, :D]
    x = _rand(5, D, seed=6)
    got = x @ Wst.t() + o.vecs["bias"].exact
    a = "encoder.layers.1.self_attn."
    lin = lambda m: x @ sd[a + m + ".weight"].double().t() + sd[a + m + ".bias"].double()
    scaling = (D // cfg["num_heads"]) ** -0.5
    ref = torch.cat([lin("q_proj") * scaling, lin("k_proj"), lin("v_proj")], 1)
    assert (got - ref).abs().max().item() <= 1e-13 * ref.abs().max().item()


def test_layer_scale_equals_gamma_times_pwconv2():
    from ns2vc_b200.synth import make_vocos_state_dict
    cfg = dict(input_channels=100, dim=128, intermediate_dim=384, num_layers=2, n_fft=1024)
    sd = po.fold_stress(make_vocos_state_dict(0, "trained_like", dim=128, intermediate_dim=384, num_layers=2), 1)
    o = next(x for x in po.vocoder(sd, cfg) if x.name == "backbone.convnext.1.pw2")
    x = _rand(5, 384, seed=7)
    got = x @ po.assemble(o, "exact")[:128, :384].t() + o.vecs["bias"].exact
    p = "backbone.convnext.1."
    ref = sd[p + "gamma"].double() * (x @ sd[p + "pwconv2.weight"].double().t() + sd[p + "pwconv2.bias"].double())
    assert (got - ref).abs().max().item() <= 1e-12 * ref.abs().max().item()
    gam = sd[p + "gamma"]
    assert (gam == 0).any() and (gam < 0).any() and (gam == torch.tensor(1e-6)).any()


def test_out_proj_ln_fold_with_conv_bias():
    """LN(x; gamma, beta) W + b (the condition encoders' out_proj: LayerNorm then a k=1 ConvTBC with bias) equals
    rstd (x (gamma W)^T - mean g) + bf with the oracle's packed gamma W and its g / bf (the conv bias folded into bf)."""
    H, cout = 40, 24
    sd = {"w": _rand(1, H, cout, seed=8).float(), "g": (1 + 0.1 * _rand(H, seed=9)).float(), "b": _rand(H, seed=10).float(),
          "cb": _rand(cout, seed=11).float()}
    wt = sd["w"][0].t()
    seg = po._scaled(wt, sd["g"], 0)
    v = po.ln_fold(wt, sd["g"], sd["b"], sd["cb"], "g_out", "bf_out")
    x = _rand(9, H, seed=12, scale=3.0) + 5.0
    mean, var = x.mean(1, keepdim=True), x.var(1, unbiased=False, keepdim=True)
    rstd = 1 / (var + 1e-5).sqrt()
    ref = ((x - mean) * rstd * sd["g"].double() + sd["b"].double()) @ wt.double().t() + sd["cb"].double()
    got = rstd * (x @ seg.exact.t() - mean * v["g_out"].exact) + v["bf_out"].exact
    assert (got - ref).abs().max().item() <= 1e-12 * ref.abs().max().item()


def _stress_denoiser_small():
    from ns2vc_b200.arch import UNetConfig
    from ns2vc_b200.synth import make_state_dict
    cfg = UNetConfig(in_channels=36, out_channels=20, block_out_channels=(32, 64, 64, 96), norm_num_groups=8, cross_attention_dim=16,
                     num_heads=8, addition_embed_type="text", addition_embed_type_num_heads=4, resnet_time_scale_shift="scale_shift")
    return cfg, po.fold_stress(make_state_dict(cfg, 0), 2)


def test_fold_bounds_are_not_vacuous():
    """In fold_stress, each double-accumulated fold computed with fp32 accumulation leaves its bound by >= 16x somewhere."""
    cfg, sd = _stress_denoiser_small()
    worst = defaultdict(float)
    for o in po.denoiser(sd, cfg):
        b = o.name[:-len(".qkv")] + ".transformer_blocks.0" if o.name.endswith(".qkv") else None
        if b:
            W = torch.cat([sd[f"{b}.attn1.to_{t}.weight"] for t in "qkv"])
            for vn, vec in (("g_qkv", sd[b + ".norm1.weight"]), ("bf_qkv", sd[b + ".norm1.bias"])):
                acc = torch.zeros(W.shape[0], dtype=F32)
                for c in range(W.shape[1]):                                    # fp32 accumulation in the kernel's own order
                    acc = acc + W[:, c] * vec[c]
                v = o.vecs[vn]
                worst["ln_fold_vec"] = max(worst["ln_fold_vec"], ((acc.double() - v.exact).abs() / po.fold_bound(v.exact, v.absum, v.nterms)).max().item())
        if o.name.endswith(".ff2p"):
            p = o.name[:-len(".ff2p")]
            b = p + ".transformer_blocks.0"
            Wp, W2 = sd[p + ".proj_out.weight"][:, :, 0], sd[b + ".ff.net.2.weight"]
            v = o.vecs["Wm"]
            acc = torch.zeros(Wp.shape[0], W2.shape[1], dtype=F32)
            for c in range(Wp.shape[1]):
                acc = acc + Wp[:, c:c + 1] * W2[c:c + 1]
            worst["matmul_nn"] = max(worst["matmul_nn"], ((acc.double().reshape(-1) - v.exact).abs() / po.fold_bound(v.exact, v.absum, v.nterms)).max().item())
            v = o.vecs["bias_ff2p"]
            acc = sd[p + ".proj_out.bias"].clone()
            for c in range(Wp.shape[1]):
                acc = acc + Wp[:, c] * sd[b + ".ff.net.2.bias"][c]
            worst["matvec_bias"] = max(worst["matvec_bias"], ((acc.double() - v.exact).abs() / po.fold_bound(v.exact, v.absum, v.nterms)).max().item())
    from ns2vc_b200.synth import CONTENTVEC_SMALL, make_contentvec_state_dict
    csd = po.fold_stress(make_contentvec_state_dict(0, "trained_like", **CONTENTVEC_SMALL), 3)
    v, g = csd["encoder.pos_conv.0.weight_v"], csd["encoder.pos_conv.0.weight_g"]
    w64 = po.weight_norm_f64(v, g)
    w32 = (g * v / v.pow(2).sum(dim=(0, 1), keepdim=True).sqrt()).double()
    fin = torch.isfinite(w64)
    r = (w32 - w64).abs() / po.fold_bound(w64, w64.abs(), v.shape[0] * v.shape[1])
    worst["weight_norm"] = r[fin].nan_to_num(nan=math.inf).max().item()
    print("fp32-accumulated folds / bound:", {k: f"{x:.3g}" for k, x in worst.items()})
    for fam in ("ln_fold_vec", "matmul_nn", "matvec_bias", "weight_norm"):
        assert worst[fam] >= 16, (fam, worst[fam])


def test_oracle_segments_never_overlap_and_stay_inside():
    cfg, sd = _stress_denoiser_small()
    for o in po.denoiser(sd, cfg):
        if o.Npad:
            po.assemble(o, "exact")
    bad = po.Operand("x", 64, 128, 2, [po._copy(torch.ones(64, 64), 0, 0), po._copy(torch.ones(64, 10), 60, 0)])
    with pytest.raises(ValueError, match="overlap"):
        po.assemble(bad, "exact")


# ------------------------------------------------------------------------------------------------------------------ GPU tier
KINDS = {"ns2vc_unet_": 0, "ns2vc_pre_": 1, "ns2vc_cv_": 2, "ns2vc_voc_": 3}


class Packed:
    """An engine handle created, loaded with `sd` and finalized through the C-ABI (no module), destroyed on exit."""

    def __init__(self, prefix, ccfg, sd, dev):
        self.prefix, self.kind, self.L = prefix, KINDS[prefix], _lib.lib()
        h = C.c_void_p()
        _lib.check(getattr(self.L, prefix + "create")(C.byref(ccfg), C.byref(h)))
        self.h = h.value
        self.stream = torch.cuda.current_stream().cuda_stream
        self.keep = []
        for key, t in sd.items():
            t = t.to(dev, F32).contiguous()
            self.keep.append(t)
            shape = (C.c_int64 * t.dim())(*t.shape)
            _lib.check(getattr(self.L, prefix + "load_weight")(self.h, key.encode(), t.data_ptr(), shape, t.dim(), self.stream))

    def finalize(self):
        _lib.check(getattr(self.L, self.prefix + "finalize")(self.h, self.stream))

    def __enter__(self):
        return self

    def __exit__(self, *a):
        torch.cuda.synchronize()
        getattr(self.L, self.prefix + "destroy")(self.h)

    def read(self):
        """[(name, Npad, nkb, n_logical, hi, lo, {vector name: fp32 tensor})] of the record"""
        L, dev = self.L, torch.device("cuda")
        n = L.ns2vc_check_packed_count(self.kind, self.h)
        if n < 0:
            _lib.check(-1)
        out = []
        for i in range(n):
            name = C.create_string_buffer(256)
            Np, nkb, nl, nv = C.c_int(), C.c_int(), C.c_int(), C.c_int()
            _lib.check(L.ns2vc_check_packed(self.kind, self.h, i, name, 256, C.byref(Np), C.byref(nkb), C.byref(nl), C.byref(nv), None, None, None))
            hi = torch.empty(nkb.value * Np.value * 64, dtype=torch.bfloat16, device=dev)
            lo = torch.empty_like(hi)
            _lib.check(L.ns2vc_check_packed(self.kind, self.h, i, None, 0, None, None, None, None, hi.data_ptr(), lo.data_ptr(), self.stream))
            vecs = {}
            for j in range(nv.value):
                vn, ln = C.create_string_buffer(64), C.c_longlong()
                _lib.check(L.ns2vc_check_fold_vector(self.kind, self.h, i, j, vn, 64, C.byref(ln), None, None))
                t = torch.empty(ln.value, dtype=F32, device=dev)
                _lib.check(L.ns2vc_check_fold_vector(self.kind, self.h, i, j, None, 0, None, t.data_ptr(), self.stream))
                vecs[vn.value.decode()] = t
            out.append((name.value.decode(), Np.value, nkb.value, nl.value, hi, lo, vecs))
        torch.cuda.synchronize()
        return out


def _bits_equal(got: torch.Tensor, want: torch.Tensor) -> torch.Tensor:
    """elementwise: same bits, or both NaN"""
    nan = torch.isnan(want.float())
    return (got.view(torch.int16) == want.view(torch.int16)) | (nan & torch.isnan(got.float()))


def check_record(rec, ops, worst, tag):
    """coverage, exact images and bounded folds of one packed engine against the oracle's operands"""
    names = [r[0] for r in rec]
    assert len(set(names)) == len(names), f"{tag}: an operand recorded twice"
    assert names == [o.name for o in ops], f"{tag}: recorded {set(names) ^ set(o.name for o in ops)} differ from the plan's sites"
    for (name, Np, nkb, nl, hi, lo, vecs), o in zip(rec, ops):
        assert (Np, nkb, nl if Np else 0) == (o.Npad, o.nkb, o.n_logical if o.Npad else 0), f"{tag} {name}: shape {(Np, nkb, nl)}"
        assert sorted(vecs) == sorted(o.vecs), f"{tag} {name}: vectors {sorted(vecs)}"
        for vn, v in o.vecs.items():
            got = vecs[vn]
            assert got.numel() == v.exact.numel(), f"{tag} {name}.{vn}: length {got.numel()}"
            if v.f32 is not None:
                ok = (got.view(torch.int32) == v.f32.view(torch.int32)) | (torch.isnan(got) & torch.isnan(v.f32))
                assert ok.all(), f"{tag} {name}.{vn}: {int((~ok).sum())} values differ from the fp32 fold bit for bit"
            if v.absum is not None:
                r = ((got.double() - v.exact).abs() / po.fold_bound(v.exact, v.absum, v.nterms)).max().item()
                worst[v.family] = max(worst[v.family], r)
                assert r <= 1.0, f"{tag} {name}.{vn}: {r:.3g} x the fold bound"
        if not o.Npad:
            continue
        f32 = po.assemble(o, "f32", vecs)
        want_hi, want_lo = f32.to(torch.bfloat16), (f32 - f32.to(torch.bfloat16).float()).to(torch.bfloat16)
        got_hi, got_lo = po.unswizzle(hi, Np, nkb), po.unswizzle(lo, Np, nkb)
        ok = _bits_equal(got_hi, want_hi) & _bits_equal(got_lo, want_lo)
        if not ok.all():
            n, k = [int(x) for x in (~ok).nonzero()[0]]
            raise AssertionError(f"{tag} {name}: {int((~ok).sum())} of {ok.numel()} image elements differ, first at column {n}, "
                                 f"channel {k}: got {got_hi[n, k].item()} + {got_lo[n, k].item()}, want {f32[n, k].item()}")
        # the emulated fp32 operand against the fp64 fold
        fam = {s.family for s in o.segs if s.bound is not None and s.f32 is not None}
        if fam:
            ex, bd = po.assemble(o, "exact"), po.assemble(o, "bound")
            fin = torch.isfinite(ex)
            r = ((f32.double() - ex).abs() / bd.clamp_min(1e-300))[fin].max().item()
            for fm in fam:
                worst[fm] = max(worst[fm], r)
            assert r <= 1.0, f"{tag} {name}: the fp32 fold is {r:.3g} x its bound from fp64"


# configurations ------------------------------------------------------------------------------------------------------------
def _denoiser_cases():
    from ns2vc_b200.arch import UNetConfig, ns2vc_denoiser_config
    tiny = dict(in_channels=36, out_channels=20, block_out_channels=(32, 64, 64, 96), norm_num_groups=8, cross_attention_dim=16,
                num_heads=8)
    return {"tiny": UNetConfig(**tiny, addition_embed_type="text", addition_embed_type_num_heads=4, resnet_time_scale_shift="scale_shift"),
            "tiny_plain": UNetConfig(**tiny),
            "full": ns2vc_denoiser_config()}


def _unet_ccfg(cfg):
    from ns2vc_b200.unet import UNet1DConditionModel
    m = UNet1DConditionModel.__new__(UNet1DConditionModel)
    m.__dict__.update(cfg=cfg, latent_channels=cfg.in_channels - cfg.cross_attention_dim if cfg.in_channels > cfg.cross_attention_dim
                      else cfg.in_channels)
    return UNet1DConditionModel._c_cfg(m)


PRE_FULL = {"phoneme_encoder": dict(in_channels=256, hidden_channels=256, out_channels=256, n_layers=6),
            "prompt_encoder": dict(in_channels=100, hidden_channels=256, out_channels=256, n_layers=6)}
PRE_NARROW = {"phoneme_encoder": dict(in_channels=96, hidden_channels=96, out_channels=40, n_layers=2),      # widths not multiples of 64
              "prompt_encoder": dict(in_channels=100, hidden_channels=160, out_channels=36, n_layers=2)}
PRE_CASES = {"full": (PRE_FULL, 9), "k3": (PRE_FULL, 3), "k5_narrow": (PRE_NARROW, 5)}

CV_FULL = dict(conv_dim=512, embed_dim=768, ffn_dim=3072, num_layers=12, num_heads=12, pos_conv_kernel=128, pos_conv_groups=16, final_dim=256)
VOC_SMALL = dict(input_channels=100, dim=128, intermediate_dim=384, num_layers=2, n_fft=1024, hop_length=256)
VOC_FULL = dict(input_channels=100, dim=512, intermediate_dim=1536, num_layers=8, n_fft=1024, hop_length=256)

WORST = defaultdict(float)


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.time()
    yield
    if WORST:
        print(f"\nload-time folds, worst |got - fp64| / bound per family ({time.time() - t0:.1f} s):")
        for k in sorted(WORST):
            print(f"  {k:12s} {WORST[k]:.3g}")


def _run(prefix, ccfg, sd, ops_fn, tag):
    dev = torch.device("cuda")
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    with Packed(prefix, ccfg, sd_dev, dev) as e:
        e.finalize()
        rec = e.read()
    check_record(rec, ops_fn(sd_dev), WORST, tag)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["synthetic", "fold_stress"])
@pytest.mark.parametrize("config", ["tiny", "tiny_plain", "full"])
def test_denoiser_packed(config, regime):
    from ns2vc_b200.synth import make_state_dict
    cfg = _denoiser_cases()[config]
    sd = make_state_dict(cfg, 0)
    if regime == "fold_stress":
        sd = po.fold_stress(sd, 11)
    _run("ns2vc_unet_", _unet_ccfg(cfg), sd, lambda s: po.denoiser(s, cfg), f"denoiser {config} {regime}")


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["synthetic", "fold_stress"])
@pytest.mark.parametrize("config", list(PRE_CASES))
def test_encoders_packed(config, regime):
    from ns2vc_b200.pre_model import REF_DIM, Pre_model, _enc_args
    from ns2vc_b200.synth import make_pre_state_dict
    pcfg, k = PRE_CASES[config]
    sd = {key: t for key, t in make_pre_state_dict(pcfg, 0).items() if not any(f".ffn_1.{j}." in key for j in range(k, 9))}
    if regime == "fold_stress":
        sd = po.fold_stress(sd, 12, ffn_kernel=k)
    m = Pre_model.__new__(Pre_model)
    m.__dict__.update(cfg=pcfg)
    ccfg = Pre_model._c_cfg(m)
    ccfg.ffn_kernel = k
    phone, prompt = _enc_args(pcfg["phoneme_encoder"], 512), _enc_args(pcfg["prompt_encoder"], 256)
    _run("ns2vc_pre_", ccfg, sd, lambda s: po.encoders(s, phone, prompt, k, REF_DIM), f"encoders {config} {regime}")


def _cv_ccfg(cfg):
    c = _lib.CvCfg()
    for key, v in cfg.items():
        setattr(c, key, int(v))
    return c


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["init", "trained_like", "sharp", "large_v", "ln_offset", "fold_stress"])
@pytest.mark.parametrize("config", ["small", "full"])
def test_content_packed(config, regime):
    from ns2vc_b200.synth import CONTENTVEC_SMALL, make_contentvec_state_dict
    if config == "full" and regime not in ("trained_like", "fold_stress"):
        pytest.skip("the full configuration runs the synthetic and fold_stress weights")
    cfg = dict(CONTENTVEC_SMALL) if config == "small" else dict(CV_FULL)
    sd = make_contentvec_state_dict(0, "trained_like" if regime == "fold_stress" else regime, **cfg)
    if regime == "fold_stress":
        sd = po.fold_stress(sd, 13)
    _run("ns2vc_cv_", _cv_ccfg(cfg), sd, lambda s: po.content(s, cfg), f"content {config} {regime}")


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["init", "trained_like", "clip", "large_phase", "ln_offset", "fold_stress"])
@pytest.mark.parametrize("config", ["small", "full"])
def test_vocoder_packed(config, regime):
    from ns2vc_b200.synth import make_vocos_state_dict
    if config == "full" and regime not in ("trained_like", "fold_stress"):
        pytest.skip("the full configuration runs the synthetic and fold_stress weights")
    cfg = dict(VOC_SMALL if config == "small" else VOC_FULL)
    sd = make_vocos_state_dict(0, "trained_like" if regime == "fold_stress" else regime, dim=cfg["dim"],
                               intermediate_dim=cfg["intermediate_dim"], num_layers=cfg["num_layers"])
    if regime == "fold_stress":
        sd = po.fold_stress(sd, 14)
    c = _lib.VocCfg()
    for key in ("input_channels", "dim", "intermediate_dim", "num_layers", "n_fft", "hop_length"):
        setattr(c, key, cfg[key])
    _run("ns2vc_voc_", c, sd, lambda s: po.vocoder(s, cfg), f"vocoder {config} {regime}")


@pytest.mark.gpu
def test_record_argument_errors():
    from ns2vc_b200.synth import make_vocos_state_dict
    L, dev = _lib.lib(), torch.device("cuda")
    cfg = dict(VOC_SMALL)
    sd = make_vocos_state_dict(0, "trained_like", dim=cfg["dim"], intermediate_dim=cfg["intermediate_dim"], num_layers=cfg["num_layers"])
    c = _lib.VocCfg()
    for key in ("input_channels", "dim", "intermediate_dim", "num_layers", "n_fft", "hop_length"):
        setattr(c, key, cfg[key])

    def err(rc):
        assert rc < 0
        return L.ns2vc_last_error().decode()

    with Packed("ns2vc_voc_", c, {k: v.to(dev) for k, v in sd.items()}, dev) as e:
        assert "not packed" in err(L.ns2vc_check_packed_count(3, e.h))           # loaded, not finalized
        e.finalize()
        n = L.ns2vc_check_packed_count(3, e.h)
        assert n == 2 + 2 * cfg["num_layers"]
        assert "engine kind 7" in err(L.ns2vc_check_packed_count(7, e.h))
        assert "null handle" in err(L.ns2vc_check_packed_count(3, None))
        assert "out of range" in err(L.ns2vc_check_packed(3, e.h, n, None, 0, None, None, None, None, None, None, None))
        assert "out of range" in err(L.ns2vc_check_packed(3, e.h, -1, None, 0, None, None, None, None, None, None, None))
        buf = C.create_string_buffer(8)
        assert "name buffer" in err(L.ns2vc_check_packed(3, e.h, 0, buf, 8, None, None, None, None, None, None, None))   # backbone.embed
        assert L.ns2vc_check_packed(3, e.h, 0, C.create_string_buffer(15), 15, None, None, None, None, None, None, None) == 0
        assert "out of range" in err(L.ns2vc_check_fold_vector(3, e.h, 0, 0, None, 0, None, None, None))                 # embed: none
        assert "name buffer" in err(L.ns2vc_check_fold_vector(3, e.h, 2, 0, C.create_string_buffer(4), 4, None, None, None))
        # re-loading a weight unpacks the handle until the next finalize
        t = sd["head.out.weight"].to(dev)
        shape = (C.c_int64 * 2)(*t.shape)
        _lib.check(L.ns2vc_voc_load_weight(e.h, b"head.out.weight", t.data_ptr(), shape, 2, e.stream))
        assert "not packed" in err(L.ns2vc_check_packed_count(3, e.h))
