"""fp64 oracle of the engines' load-time packing: every operand the launch programs read, as a list of segments in the packer's
column and k-block order, and every load-time vector beside it, computed from the reference ``state_dict`` alone.

A packed operand is a bf16 hi / lo pair of images [nkb k-blocks][Npad columns][64 channels], each 128-byte row XOR-swizzled
(``unswizzle``).  Its logical content is the dense [Npad, 64 nkb] matrix ``assemble`` builds from the segments: segment s puts
its [rows, ncin] block at columns n0.. and channels 64 kb0.., zeros everywhere else.  Each segment carries

* ``exact``: the fp64 value of the fold (the reference's own arithmetic, in real numbers);
* ``f32``:   the fp32 value the packer feeds to the split, emulated bit for bit where the packer's arithmetic is a fixed sequence of
             fp32 or fp64 roundings (copies, the TBC transpose, gamma W, the conv-FFN taps, the layer scale, the q scaling, the weight
             norm in its kernel's order), or None where the engine keeps the fp32 operand itself as a load-time vector
             (``from_vec``: the denoiser's Wp W2).

Each vector carries ``exact`` and either ``f32`` (bit-exact families) or ``absum`` / ``n`` (double-accumulated folds, checked with
``fold_bound``).  Every function takes tensors on any device and computes there.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch

F64, F32 = torch.float64, torch.float32


def pad128(n: int) -> int:
    return (n + 127) // 128 * 128


def nkb_of(c: int) -> int:
    return (c + 63) // 64


@dataclass
class Seg:
    exact: torch.Tensor                   # fp64 [rows, ncin]
    f32: Optional[torch.Tensor]           # fp32 [rows, ncin], or None: the vector `from_vec` of the operand, reshaped
    n0: int
    kb0: int
    family: str
    bound: Optional[torch.Tensor] = None  # fp64 [rows, ncin]: allowed |f32 - exact| (None: f32 is the rounding of exact)
    from_vec: Optional[str] = None


@dataclass
class Vec:
    exact: torch.Tensor                   # fp64 [n]
    family: str
    f32: Optional[torch.Tensor] = None    # bit-exact families
    absum: Optional[torch.Tensor] = None  # double-accumulated folds: sum_i |a_i b_i|
    nterms: int = 0


@dataclass
class Operand:
    name: str
    n_logical: int = 0
    Npad: int = 0                         # 0: vectors only
    nkb: int = 0
    segs: List[Seg] = field(default_factory=list)
    vecs: Dict[str, Vec] = field(default_factory=dict)


def fold_bound(exact: torch.Tensor, absum: torch.Tensor, nterms: int) -> torch.Tensor:
    """One fp32 rounding of the result plus the fp64 sum's own error: 2^-24 |exact| + (n + 2) 2^-53 sum |a_i b_i|."""
    return 2.0 ** -24 * exact.abs() + (nterms + 2) * 2.0 ** -53 * absum


def unswizzle(img: torch.Tensor, Npad: int, nkb: int) -> torch.Tensor:
    """A packed image (flat, nkb * Npad * 64) -> [Npad, 64 nkb]: element (kb, n, kk) lives at
    (kb Npad + n) 64 + ((kk >> 3) ^ (n & 7)) 8 + (kk & 7)."""
    dev = img.device
    kb, n, kk = torch.meshgrid(torch.arange(nkb, device=dev), torch.arange(Npad, device=dev), torch.arange(64, device=dev), indexing="ij")
    idx = ((kb * Npad + n) * 64 + ((((kk >> 3) ^ (n & 7)) << 3) + (kk & 7))).reshape(-1)
    return img[idx].reshape(nkb, Npad, 64).permute(1, 0, 2).reshape(Npad, nkb * 64)


def assemble(op: Operand, which: str, vecs: Optional[Dict[str, torch.Tensor]] = None) -> torch.Tensor:
    """The dense [Npad, 64 nkb] matrix of `which` ('exact' | 'f32' | 'bound'); a segment without an f32 value takes the recorded
    vector `vecs[seg.from_vec]`.  Raises on segments that overlap or leave the image."""
    dev = op.segs[0].exact.device
    dt = F32 if which == "f32" else F64
    out = torch.zeros(op.Npad, op.nkb * 64, dtype=dt, device=dev)
    used = torch.zeros(op.Npad, op.nkb * 64, dtype=torch.int32, device=dev)
    for s in op.segs:
        rows, ncin = s.exact.shape
        k0 = 64 * s.kb0
        if s.n0 < 0 or s.n0 + rows > op.Npad or s.kb0 < 0 or k0 + 64 * nkb_of(ncin) > 64 * op.nkb:
            raise ValueError(f"{op.name}: segment at column {s.n0}, k-block {s.kb0} leaves the [{op.Npad}, {op.nkb}] image")
        # a segment owns its whole k-blocks: channels past ncin are its zeros
        used[s.n0:s.n0 + rows, k0:k0 + 64 * nkb_of(ncin)] += 1
        if which == "exact":
            v = s.exact
        elif which == "bound":
            v = s.bound if s.bound is not None else 2.0 ** -24 * s.exact.abs()
        else:
            v = s.f32 if s.f32 is not None else vecs[s.from_vec].reshape(rows, ncin)
        out[s.n0:s.n0 + rows, k0:k0 + ncin] = v.to(dt)
    if int(used.max()) > 1:
        raise ValueError(f"{op.name}: segments overlap")
    return out


def _copy(w: torch.Tensor, n0: int, kb0: int, family: str = "copy") -> Seg:
    return Seg(w.to(F64), w.to(F32), n0, kb0, family)


def _scaled(w: torch.Tensor, gamma: torch.Tensor, n0: int, family: str = "ln_gamma") -> Seg:
    """gamma W (per input channel): one fp32 product, as pack_b's cscale"""
    return Seg(w.to(F64) * gamma.to(F64), w.to(F32) * gamma.to(F32), n0, 0, family)


def _taps(w: torch.Tensor, nkb_tap: int, family: str = "copy") -> List[Seg]:
    """conv weight [rows, cin, k]: tap j at k-block j nkb_tap"""
    return [_copy(w[:, :, j], 0, j * nkb_tap, family) for j in range(w.shape[2])]


def ln_fold(W: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, bias: Optional[torch.Tensor], gname: str,
            bname: str) -> Dict[str, Vec]:
    """g[n] = sum_c gamma_c W[n, c], bf[n] = sum_c beta_c W[n, c] (+ bias[n]) of a linear that consumes LayerNorm(gamma, beta)"""
    W64 = W.to(F64)
    g = W64 @ gamma.to(F64)
    bf = W64 @ beta.to(F64)
    sb = W64.abs() @ beta.to(F64).abs()
    if bias is not None:
        bf = bf + bias.to(F64)
        sb = sb + bias.to(F64).abs()
    C = W.shape[1]
    return {gname: Vec(g, "ln_fold_vec", absum=W64.abs() @ gamma.to(F64).abs(), nterms=C),
            bname: Vec(bf, "ln_fold_vec", absum=sb, nterms=C + (bias is not None))}


def geglu_interleave(w: torch.Tensor, half: int) -> torch.Tensor:
    """rows of a GEGLU projection [2 half, ...] in packed order: 128-row blocks [64 value | 64 gate]"""
    blocks = [torch.cat([w[64 * j:64 * j + 64], w[half + 64 * j:half + 64 * j + 64]]) for j in range(half // 64)]
    return torch.cat(blocks)


# ------------------------------------------------------------------------------------------------------------------ denoiser
def denoiser(sd: Dict[str, torch.Tensor], cfg) -> List[Operand]:
    """pack_all (csrc/engine.cu) of UNet1DConditionModel's state_dict; `cfg` an arch.UNetConfig."""
    from ns2vc_b200.arch import build_plan
    c0, ci, co = cfg.block_out_channels[0], cfg.in_channels, cfg.out_channels
    xd = cfg.cross_attention_dim
    Cl = ci - xd if ci > xd else ci
    Cc = ci - Cl
    ops: List[Operand] = []
    w = sd["conv_in.weight"]
    ops.append(Operand("conv_in.latent", c0, pad128(c0), 3 * nkb_of(Cl), _taps(w[:, :Cl], nkb_of(Cl))))
    if Cc > 0:
        ops.append(Operand("conv_in.content", c0, pad128(c0), 3 * nkb_of(Cc), _taps(w[:, Cl:], nkb_of(Cc))))
    xformers, resnets = [], []
    for o in build_plan(cfg):
        p = o.prefix
        if o.kind == "resnet":
            ni, no = nkb_of(o.cin), nkb_of(o.cout)
            resnets.append(p)
            ops.append(Operand(p + ".conv1", o.cout, pad128(o.cout), 3 * ni, _taps(sd[p + ".conv1.weight"], ni)))
            segs = _taps(sd[p + ".conv2.weight"], no)
            b2 = sd[p + ".conv2.bias"]
            if o.cin != o.cout:
                segs.append(_copy(sd[p + ".conv_shortcut.weight"][:, :, 0], 0, 3 * no))
                bs = sd[p + ".conv_shortcut.bias"]
                bias2 = Vec(b2.to(F64) + bs.to(F64), "add_vec", f32=b2.to(F32) + bs.to(F32))
            else:
                bias2 = Vec(b2.to(F64), "add_vec", f32=b2.to(F32))
            ops.append(Operand(p + ".conv2", o.cout, pad128(o.cout), 3 * no + (ni if o.cin != o.cout else 0), segs, {"bias2": bias2}))
        elif o.kind == "xformer":
            C, nk = o.cout, nkb_of(o.cout)
            b = p + ".transformer_blocks.0"
            xformers.append((b, C))
            ops.append(Operand(p + ".proj_in", C, pad128(C), nk, [_copy(sd[p + ".proj_in.weight"][:, :, 0], 0, 0)]))
            g1, g2, g3 = (sd[f"{b}.norm{i}.weight"] for i in (1, 2, 3))
            be1, be2, be3 = (sd[f"{b}.norm{i}.bias"] for i in (1, 2, 3))
            qkv = [sd[f"{b}.attn1.to_{t}.weight"] for t in "qkv"]
            v1 = ln_fold(torch.cat(qkv), g1, be1, None, "g_qkv", "bf_qkv")
            ops.append(Operand(p + ".qkv", 3 * C, pad128(3 * C), nk, [_scaled(qkv[i], g1, i * C) for i in range(3)], v1))
            ops.append(Operand(p + ".out1", C, pad128(C), nk, [_copy(sd[b + ".attn1.to_out.0.weight"], 0, 0)]))
            q2 = sd[b + ".attn2.to_q.weight"]
            ops.append(Operand(p + ".q2", C, pad128(C), nk, [_scaled(q2, g2, 0)], ln_fold(q2, g2, be2, None, "g_q2", "bf_q2")))
            ops.append(Operand(p + ".out2", C, pad128(C), nk, [_copy(sd[b + ".attn2.to_out.0.weight"], 0, 0)]))
            w1, bb1 = sd[b + ".ff.net.0.proj.weight"], sd[b + ".ff.net.0.proj.bias"]
            ops.append(Operand(p + ".ff1", 4 * C, pad128(8 * C), nk, [_scaled(geglu_interleave(w1, 4 * C), g3, 0, "ln_gamma")],
                               ln_fold(w1, g3, be3, bb1, "g_ff1", "bf_ff1")))
            # proj_out o ff.net.2: K = [Wp W2 over the 4C GEGLU channels | Wp over the C residual channels]
            Wp, W2 = sd[p + ".proj_out.weight"][:, :, 0].to(F64), sd[b + ".ff.net.2.weight"].to(F64)
            b2, bp = sd[b + ".ff.net.2.bias"].to(F64), sd[p + ".proj_out.bias"].to(F64)
            Wm, Wm_abs = Wp @ W2, Wp.abs() @ W2.abs()
            segs = [Seg(Wm, None, 0, 0, "matmul_nn", bound=fold_bound(Wm, Wm_abs, C), from_vec="Wm"),
                    _copy(sd[p + ".proj_out.weight"][:, :, 0], 0, nkb_of(4 * C))]
            vecs = {"Wm": Vec(Wm.reshape(-1), "matmul_nn", absum=Wm_abs.reshape(-1), nterms=C),
                    "bias_ff2p": Vec(Wp @ b2 + bp, "matvec_bias", absum=Wp.abs() @ b2.abs() + bp.abs(), nterms=C + 1)}
            ops.append(Operand(p + ".ff2p", C, pad128(C), nkb_of(4 * C) + nk, segs, vecs))
        elif o.kind in ("down", "up"):
            ops.append(Operand(p + ".conv", o.cout, pad128(o.cout), 3 * nkb_of(o.cout), _taps(sd[p + ".conv.weight"], nkb_of(o.cout))))
    ops.append(Operand("conv_out", co, pad128(co), 3 * nkb_of(c0), _taps(sd["conv_out.weight"], nkb_of(c0))))
    if xformers:
        k_total = sum(C for _, C in xformers)
        segs, off = [], 0
        for b, C in xformers:
            segs.append(_copy(sd[b + ".attn2.to_k.weight"], off, 0))
            segs.append(_copy(sd[b + ".attn2.to_v.weight"], k_total + off, 0))
            off += C
        ops.append(Operand("kv_all", 2 * k_total, pad128(2 * k_total), nkb_of(xd), segs))
    fw = torch.cat([sd[p + ".time_emb_proj.weight"].reshape(-1) for p in resnets])
    fb = torch.cat([sd[p + ".time_emb_proj.bias"] for p in resnets])
    ops.append(Operand("time_emb_proj", vecs={"film_W": Vec(fw.to(F64), "concat", f32=fw.to(F32)),
                                              "film_b": Vec(fb.to(F64), "concat", f32=fb.to(F32))}))
    if cfg.addition_embed_type == "text":
        ops.append(_pool_kv(sd, "add_embedding.pool"))
    return ops


def _pool_kv(sd, pool: str) -> Operand:
    W = torch.cat([sd[pool + ".k_proj.weight"].reshape(-1), sd[pool + ".v_proj.weight"].reshape(-1)])
    b = torch.cat([sd[pool + ".k_proj.bias"], sd[pool + ".v_proj.bias"]])
    return Operand(pool + ".kv", vecs={"W": Vec(W.to(F64), "concat", f32=W.to(F32)), "b": Vec(b.to(F64), "concat", f32=b.to(F32))})


# ------------------------------------------------------------------------------------------------------------------ condition encoders
def ffn_scale(k: int) -> float:
    """the conv-FFN's fp32 scale: k^-0.5 in fp64, rounded once"""
    return float(torch.tensor(float(k) ** -0.5, dtype=F64).to(F32))


def ffn_centre(k: int) -> int:
    """the packed tap that also carries the reference's tap 0 (which reads the unshifted input: row offset 0)"""
    return (k - 1) // 2 - 1


def ffn_taps(ws: List[torch.Tensor]) -> List[Seg]:
    """TransformerFFNLayer's k Linears [F, H] -> the (k - 1)-tap conv: tap j (row offset j + 1 - (k - 1) / 2) = s W_{j+1}, the
    centre tap s (W_{j+1} + W_0); fp32: the sum, then the product with the fp32 scale (two roundings)."""
    k = len(ws)
    s32, s64 = ffn_scale(k), float(k) ** -0.5
    H = ws[0].shape[1]
    segs = []
    for j in range(k - 1):
        a = ws[j + 1]
        if j == ffn_centre(k):
            e = (a.to(F64) + ws[0].to(F64)) * s64
            f = (a.to(F32) + ws[0].to(F32)) * s32
            bound = 2.0 ** -24 * (a.to(F64).abs() + ws[0].to(F64).abs()) * s64 * 2 + 2.0 ** -24 * e.abs()
        else:
            e, f = a.to(F64) * s64, a.to(F32) * s32
            bound = 2 * 2.0 ** -24 * e.abs()
        segs.append(Seg(e, f, 0, j * nkb_of(H), "ffn_taps", bound=bound))
    return segs


def encoders(sd: Dict[str, torch.Tensor], phone: tuple, prompt: tuple, ffn_kernel: int, ref_dim: int) -> List[Operand]:
    """pack (csrc/pre_engine.cu) of Pre_model's state_dict; phone / prompt: (in, hidden, out, layers) of each encoder."""
    ops: List[Operand] = []
    k = ffn_kernel
    for p, (cin, H, cout, L) in (("phoneme_encoder", phone), ("prompt_encoder", prompt)):
        nh, F = nkb_of(H), 4 * H
        ops.append(Operand(p + ".pre", H, pad128(H), nkb_of(cin), [_copy(sd[p + ".pre.conv.weight"][0].t(), 0, 0, "tbc")]))
        for i in range(L):
            b = f"{p}.layers.{i}.op"
            site = f"{p}.layers.{i}"
            win = sd[b + ".self_attn.in_proj_weight"]
            g1, b1 = sd[b + ".layer_norm1.weight"], sd[b + ".layer_norm1.bias"]
            ops.append(Operand(site + ".qkv", 3 * H, pad128(3 * H), nh, [_scaled(win, g1, 0)], ln_fold(win, g1, b1, None, "g_qkv", "bf_qkv")))
            ops.append(Operand(site + ".out", H, pad128(H), nh, [_copy(sd[b + ".self_attn.out_proj.weight"], 0, 0)]))
            ws = [sd[f"{b}.ffn.ffn_1.{j}.weight"] for j in range(k)]
            b0 = sd[b + ".ffn.ffn_1.0.bias"]
            bvec = Vec(b0.to(F64) * float(k) ** -0.5, "ffn_taps", f32=b0.to(F32) * ffn_scale(k))
            ops.append(Operand(site + ".ffn1", F, pad128(F), (k - 1) * nh, ffn_taps(ws), {"b_ffn1": bvec}))
            ops.append(Operand(site + ".ffn2", H, pad128(H), nkb_of(F), [_copy(sd[b + ".ffn.ffn_2.weight"], 0, 0)]))
        wt = sd[p + ".out_proj.conv.weight"][0].t()              # ConvTBC [1, H, cout] -> [cout, H]
        go, bo, cb = sd[p + ".out_proj.layer_norm.weight"], sd[p + ".out_proj.layer_norm.bias"], sd[p + ".out_proj.conv.bias"]
        ops.append(Operand(p + ".out_proj", cout, pad128(cout), nh, [_scaled(wt, go, 0)], ln_fold(wt, go, bo, cb, "g_out", "bf_out")))
    ops.append(_pool_kv(sd, "ref_enc.pool"))
    return ops


# ------------------------------------------------------------------------------------------------------------------ content encoder
def cv_conv_k(l: int) -> int:
    return 10 if l == 0 else 3 if l < 5 else 2


def weight_norm_f64(v: torch.Tensor, g: torch.Tensor) -> torch.Tensor:
    """torch._weight_norm(v, g, dim=2) in fp64: w[o, i, j] = g[j] v[o, i, j] / ||v[:, :, j]||"""
    v64 = v.to(F64)
    return g.to(F64).reshape(1, 1, -1) * v64 / v64.pow(2).sum(dim=(0, 1), keepdim=True).sqrt()


def weight_norm_emulate(v: torch.Tensor, g: torch.Tensor) -> torch.Tensor:
    """cv_weight_norm_kernel bit for bit: per tap, thread t of 256 sums the squares of rows t, t + 256, ... in fp64 (each square
    exact), thread 0 adds the 256 partials in thread order, f = g / sqrt(sum) in fp64, w = fp32(f v)."""
    D, gw, K = v.shape
    rows = D * gw
    v64 = v.to(F64).reshape(rows, K)
    nchunk = (rows + 255) // 256
    vp = torch.zeros(nchunk * 256, K, dtype=F64, device=v.device)
    vp[:rows] = v64
    vp = vp.reshape(nchunk, 256, K)
    part = torch.zeros(256, K, dtype=F64, device=v.device)
    for i in range(nchunk):
        part = part + vp[i] * vp[i]
    t = torch.zeros(K, dtype=F64, device=v.device)
    for i in range(256):
        t = t + part[i]
    f = g.reshape(-1).to(F64) / t.sqrt()
    return (f.reshape(1, K) * v64).to(F32).reshape(D, gw, K)


def qscale_of(D: int, heads: int) -> float:
    return 1.0 / math.sqrt(D // heads)


def content(sd: Dict[str, torch.Tensor], cfg: dict) -> List[Operand]:
    """pack_with (csrc/content.cu) of ContentVec's (HubertModel's) state_dict; `cfg` the ContentVec constructor arguments."""
    C0, D, K, G = cfg["conv_dim"], cfg["embed_dim"], cfg["pos_conv_kernel"], cfg["pos_conv_groups"]
    gw = D // G
    ops: List[Operand] = []
    for l in range(1, 7):
        key = f"feature_extractor.conv_layers.{l}"
        ops.append(Operand(key, C0, pad128(C0), cv_conv_k(l) * nkb_of(C0), _taps(sd[key + ".0.weight"], nkb_of(C0))))
    ops.append(Operand("post_extract_proj", D, pad128(D), nkb_of(C0), [_copy(sd["post_extract_proj.weight"], 0, 0)]))
    v, g = sd["encoder.pos_conv.0.weight_v"], sd["encoder.pos_conv.0.weight_g"]
    w64, w32 = weight_norm_f64(v, g), weight_norm_emulate(v, g)
    bound = fold_bound(w64, w64.abs(), D * gw)
    for gi in range(G):
        r = slice(gi * gw, (gi + 1) * gw)
        segs = [Seg(w64[r, :, j], w32[r, :, j], 0, j, "weight_norm", bound=bound[r, :, j]) for j in range(K)]
        ops.append(Operand(f"encoder.pos_conv.{gi}", gw, pad128(gw), K, segs))
    qs = qscale_of(D, cfg["num_heads"])
    for i in range(cfg["num_layers"]):
        p = f"encoder.layers.{i}"
        a = p + ".self_attn."
        qw, qb = sd[a + "q_proj.weight"], sd[a + "q_proj.bias"]
        # q's rows times qscale (an fp64 product rounded once), then k and v as loaded
        e_q, f_q = qw.to(F64) / math.sqrt(D // cfg["num_heads"]), (qw.to(F64) * qs).to(F32)
        segs = [Seg(e_q, f_q, 0, 0, "qscale", bound=fold_bound(e_q, e_q.abs(), 1)),
                _copy(sd[a + "k_proj.weight"], D, 0), _copy(sd[a + "v_proj.weight"], 2 * D, 0)]
        e_b = torch.cat([qb.to(F64) / math.sqrt(D // cfg["num_heads"]), sd[a + "k_proj.bias"].to(F64), sd[a + "v_proj.bias"].to(F64)])
        f_b = torch.cat([(qb.to(F64) * qs).to(F32), sd[a + "k_proj.bias"].to(F32), sd[a + "v_proj.bias"].to(F32)])
        ops.append(Operand(p + ".qkv", 3 * D, pad128(3 * D), nkb_of(D), segs, {"bias": Vec(e_b, "qscale", f32=f_b)}))
        ops.append(Operand(p + ".out_proj", D, pad128(D), nkb_of(D), [_copy(sd[a + "out_proj.weight"], 0, 0)]))
        ops.append(Operand(p + ".fc1", cfg["ffn_dim"], pad128(cfg["ffn_dim"]), nkb_of(D), [_copy(sd[p + ".fc1.weight"], 0, 0)]))
        ops.append(Operand(p + ".fc2", D, pad128(D), nkb_of(cfg["ffn_dim"]), [_copy(sd[p + ".fc2.weight"], 0, 0)]))
    fd = cfg["final_dim"]
    ops.append(Operand("final_proj", fd, pad128(fd), nkb_of(D), [_copy(sd["final_proj.weight"], 0, 0)]))
    return ops


# ------------------------------------------------------------------------------------------------------------------ vocoder
def vocoder(sd: Dict[str, torch.Tensor], cfg: dict) -> List[Operand]:
    """pack (csrc/vocoder.cu) of Vocos' state_dict; `cfg` the Vocos constructor arguments."""
    D, Fi, cin, nf = cfg["dim"], cfg["intermediate_dim"], cfg["input_channels"], cfg["n_fft"]
    ops = [Operand("backbone.embed", D, pad128(D), 7 * nkb_of(cin), _taps(sd["backbone.embed.weight"], nkb_of(cin)))]
    for i in range(cfg["num_layers"]):
        p = f"backbone.convnext.{i}"
        ops.append(Operand(p + ".pw1", Fi, pad128(Fi), nkb_of(D), [_copy(sd[p + ".pwconv1.weight"], 0, 0)]))
        gam, W2, b2 = sd[p + ".gamma"], sd[p + ".pwconv2.weight"], sd[p + ".pwconv2.bias"]
        seg = Seg(gam.to(F64)[:, None] * W2.to(F64), gam.to(F32)[:, None] * W2.to(F32), 0, 0, "layer_scale")
        bias = Vec(gam.to(F64) * b2.to(F64), "layer_scale", f32=gam.to(F32) * b2.to(F32))
        ops.append(Operand(p + ".pw2", D, pad128(D), nkb_of(Fi), [seg], {"bias": bias}))
    ops.append(Operand("head.out", nf + 2, pad128(nf + 2), nkb_of(D), [_copy(sd["head.out.weight"], 0, 0)]))
    return ops


# ------------------------------------------------------------------------------------------------------------------ fold_stress
def _cancel_pairs(shape, axis: int, g: torch.Generator, scale: float = 1e4) -> torch.Tensor:
    """scale N(0, 1) with odd entries along `axis` = -(1 + 2^-10 N(0, 1)) x the even one before: sums over `axis` (against
    pairwise-equal factors) cancel about 10 bits"""
    t = scale * torch.randn(shape, generator=g, dtype=F64)
    t = t.movedim(axis, 0)
    m = t.shape[0] // 2 * 2
    t[1:m:2] = -t[0:m:2] * (1 + 2.0 ** -10 * torch.randn(t[1:m:2].shape, generator=g, dtype=F64))
    return t.movedim(0, axis).to(F32).contiguous()


def _equal_pairs(t: torch.Tensor, axis: int = 0) -> torch.Tensor:
    t = t.movedim(axis, 0).clone()
    m = t.shape[0] // 2 * 2
    t[1:m:2] = t[0:m:2]
    return t.movedim(0, axis).contiguous()


def stress_gamma(n: int, g: torch.Generator) -> torch.Tensor:
    """a LayerNorm / layer-scale gamma with exact zeros, negatives and 1e-6 entries (Vocos' layer-scale init), pairwise equal"""
    t = (0.5 + 1.5 * torch.rand(n, generator=g)) * torch.where(torch.rand(n, generator=g) < 0.3, -1.0, 1.0)
    t[0::7] = 0.0
    t[2::7] = 1e-6
    t[4::11] = -1e-6
    return _equal_pairs(t.to(F32))


def fold_stress(sd: Dict[str, torch.Tensor], seed: int = 0, ffn_kernel: int = 9) -> Dict[str, torch.Tensor]:
    """The `fold_stress` regime of any engine's state_dict: the weights each load-time fold reads, replaced so that the folds
    cancel 8+ bits (W gamma, Wp W2, Wp b2, the conv-FFN centre-tap sum, conv2 + shortcut biases), with gammas holding exact
    zeros, negatives and 1e-6, weight-norm columns of 1e-20 (whose squares underflow in fp32), g = 0 in one tap and an all-zero
    v column (0 / 0: NaN, as torch._weight_norm gives)."""
    g = torch.Generator().manual_seed(seed)
    out = dict(sd)
    for key, t in sd.items():
        shp = tuple(t.shape)
        if any(key.endswith(f"norm{i}.weight") for i in (1, 2, 3)) and ".transformer_blocks." in key or \
                key.endswith(("layer_norm1.weight", "out_proj.layer_norm.weight")) or key.endswith(".gamma"):
            out[key] = stress_gamma(shp[0], g)
        elif any(key.endswith(f"norm{i}.bias") for i in (1, 2, 3)) and ".transformer_blocks." in key or \
                key.endswith(("layer_norm1.bias", "out_proj.layer_norm.bias")):
            out[key] = _equal_pairs(torch.randn(shp, generator=g))
        elif key.endswith((".attn1.to_q.weight", ".attn1.to_k.weight", ".attn1.to_v.weight", ".attn2.to_q.weight",
                           ".ff.net.0.proj.weight", "self_attn.in_proj_weight")):
            out[key] = _cancel_pairs(shp, 1, g)
        elif key.endswith("out_proj.conv.weight"):                   # ConvTBC [1, H, cout]: H is the folded axis
            out[key] = _cancel_pairs(shp, 1, g)
        elif key.endswith(".proj_out.weight"):
            out[key] = _equal_pairs(1e4 * torch.randn(shp, generator=g), 1)
        elif key.endswith((".ff.net.2.weight", ".ff.net.2.bias")):
            out[key] = _cancel_pairs(shp, 0, g)
        elif key.endswith(".conv_shortcut.bias"):
            b2 = out[key.replace("conv_shortcut", "conv2")] = 1e4 * torch.randn(shp, generator=g)
            out[key] = (-b2.to(F64) * (1 + 2.0 ** -10 * torch.randn(shp, generator=g, dtype=F64))).to(F32)
        elif key.endswith(("q_proj.weight", "q_proj.bias", "pwconv2.weight", "pwconv2.bias")) and "pool" not in key:
            out[key] = 1e4 * torch.randn(shp, generator=g)
        elif key.endswith("pos_conv.0.weight_v"):
            v = torch.randn(shp, generator=g)
            v[:, :, 0] *= 1e-20
            v[:, :, 2] = 0.0
            out[key] = v
        elif key.endswith("pos_conv.0.weight_g"):
            w = torch.rand(shp, generator=g) + 0.5
            w[..., 1] = 0.0
            out[key] = w
    for key in sd:
        if key.endswith(".ffn.ffn_1.0.weight"):                     # tap 0 nearly cancels the centre tap it is summed into
            b = key[:-len("0.weight")]
            for j in range(1, ffn_kernel):
                out[f"{b}{j}.weight"] = 1e4 * torch.randn(tuple(sd[key].shape), generator=g)
            c = out[f"{b}{ffn_centre(ffn_kernel) + 1}.weight"].to(F64)
            out[key] = (-c * (1 + 2.0 ** -10 * torch.randn(c.shape, generator=g, dtype=F64))).to(F32)
    return {k: v.to(F32).contiguous() for k, v in out.items()}
