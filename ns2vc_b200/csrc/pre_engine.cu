// Condition-encoder engine: `Pre_model.infer` of the reference (model.py:359-377) as one launch program per (B, T, S) over the
// denoiser's own kernels - the wgmma 3xBF16 GEMM (gemm_tc.cu, ENC instantiation for the ReLU / padding-mask epilogues), the
// flash attention kernels (key-padding bias), the LayerNorm split - plus the handful of small kernels in pre_kernels.cu.
//
//   g            = ref_enc(refer^T)                      TextTimeEmbedding(100, 100, 1)      model.py:340, 362; embeddings.py:421-434
//   audio_prompt = PromptEncoder(refer, refer_lengths)   model.py:173-190
//   content      = PhoneEncoder(c + spk_proj(g), lengths) model.py:125-145
//
// Encoder (token-major [B, T, C] throughout; the reference's [T, B, C] is the transposed view of the same values):
//   x0 = (input) * keep                      -> LayerNorm -> k=1 ConvTBC + bias, * keep                  ConvLayer, model.py:88-96, 134-135
//   per layer (EncSALayer, operations.py:798-821):
//     q|k|v = LN1(x) in_proj^T        LayerNorm FOLDED into the GEMM (gamma in the weights, mean / rstd in the epilogue, row sums
//                                      accumulated by the producer's epilogue): no LayerNorm kernel
//     a     = softmax(q k^T dh^-0.5 + key padding bias) v                                                operations.py:412-421
//     x     = (x + a out_proj^T) * keep                                                                  :812-813
//     y     = LN2(x)                   explicit (ln_split): the conv-FFN reads NEIGHBOUR rows, whose statistics differ per tap;
//                                      padded frames of x are zero, so y = beta there - exactly what the reference's FFN sees
//     f     = relu(k^-0.5 sum_i y[t + off_i] W_i^T + b)   ONE implicit GEMM over 8 row-shifted views (tap 0 of the reference reads
//                                      the unshifted input, like the centre tap: both weights are summed at load time)      :678-684
//     x     = (x + f ffn_2^T + b2) * keep                                                                :689-691, 819-820
//   out = LN(LN_o(x) conv_o + b_o) * keep   (LN_o folded into the k=1 conv; final LayerNorm + mask: ln_mask)  model.py:141-144
#include "common.cuh"
#include "../../include/ns2vc_b200.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

using namespace ns2vc;

namespace {

struct WSlot {
  std::string name;
  std::vector<int64_t> shape;
  float* d = nullptr;
  bool loaded = false;
  size_t numel() const { size_t n = 1; for (auto s : shape) n *= (size_t)s; return n; }
};
struct PackedB {
  __nv_bfloat16* hi = nullptr;
  __nv_bfloat16* lo = nullptr;
  float* f32 = nullptr;
  int Npad = 0, nkb = 0, n_logical = 0;
};
inline int pad_to(int v, int m) { return (v + m - 1) / m * m; }
inline int nkb_of(int c) { return (c + 63) / 64; }

struct Arena {
  uint8_t* base = nullptr;
  size_t off = 0;
  template <class T> T* get(size_t n) {
    off = (off + 255) & ~(size_t)255;
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += n * sizeof(T);
    return p;
  }
};

struct LayerSite {
  PackedB qkv, out, ffn1, ffn2;
  float* g_qkv = nullptr; float* bf_qkv = nullptr;     // folded layer_norm1
  float* b_ffn1 = nullptr;                             // k^-0.5 * ffn_1.0.bias
};
struct EncSite {
  std::string p;
  int cin = 0, H = 0, cout = 0, L = 0;
  bool spk = false;
  PackedB pre, outp;
  float* g_out = nullptr; float* bf_out = nullptr;     // folded out_proj.layer_norm (+ conv bias)
  std::vector<LayerSite> layers;
};

struct PLaunch {
  enum Kind { MEMSET, SEQMASK, ENC_INPUT, LN_SPLIT, GEMM, ATTN, LN_MASK, NCT2TOK, LN_APPLY, POOL_CLS, LINEAR, POOL_ATT, TAP } kind;
  GemmOp gemm; AttnOp attn; LinOp lin; SplitBuf split;
  const float* a = nullptr; const float* b = nullptr; const float* c = nullptr; const float* d = nullptr; float* o = nullptr; float* o2 = nullptr;
  int i0 = 0, i1 = 0, i2 = 0, i3 = 0; float f0 = 0;
  void* mem = nullptr; size_t mem_bytes = 0;
  int patch = 0;             // SEQMASK: 1 lengths, 2 refer_lengths; ENC_INPUT: 1 c, 2 refer; NCT2TOK: 2 refer; LN_MASK: 1 content, 2 prompt
  int tap_index = -1;
};

}  // namespace

struct ns2vc_pre {
  ns2vc_pre_cfg cfg;
  std::vector<WSlot> weights;
  std::unordered_map<std::string, int> windex;
  bool finalized = false, simt = false;
  EncSite phone, prompt;
  float* ref_kvW = nullptr; float* ref_kvb = nullptr;   // ref_enc.pool k_proj | v_proj as one [2R, R] operator
  std::vector<void*> owned;
  // cached program
  int pB = 0, pT = 0, pS = 0; void* pws = nullptr;
  std::vector<PLaunch> prog;
  std::vector<std::string> tap_names; std::vector<int> tap_rows, tap_ch; std::vector<float*> tap_dst;
  int last_launches = 0;
  const float* W(const std::string& n) const {
    auto it = windex.find(n);
    return it == windex.end() ? nullptr : weights[it->second].d;
  }
};

namespace {

void add_w(ns2vc_pre* h, const std::string& n, std::vector<int64_t> shape) {
  h->windex[n] = (int)h->weights.size();
  WSlot s; s.name = n; s.shape = std::move(shape);
  h->weights.push_back(std::move(s));
}
void add_norm(ns2vc_pre* h, const std::string& p, int c) { add_w(h, p + ".weight", {c}); add_w(h, p + ".bias", {c}); }
void add_lin(ns2vc_pre* h, const std::string& p, int co, int ci, bool bias = true) { add_w(h, p + ".weight", {co, ci}); if (bias) add_w(h, p + ".bias", {co}); }

// reference parameter names / shapes (model.py:98-127, 156-172; operations.py:784-797, 304-340, 644-663)
void register_encoder(ns2vc_pre* h, const std::string& p, int cin, int H, int cout, int L, bool spk) {
  const int k = h->cfg.ffn_kernel, F = 4 * H;
  for (int i = 0; i < L; ++i) {
    const std::string b = p + ".layers." + std::to_string(i) + ".op";
    add_norm(h, b + ".layer_norm1", H);
    add_w(h, b + ".self_attn.in_proj_weight", {3 * H, H});
    add_w(h, b + ".self_attn.out_proj.weight", {H, H});
    add_norm(h, b + ".layer_norm2", H);
    for (int j = 0; j < k; ++j) add_lin(h, b + ".ffn.ffn_1." + std::to_string(j), F, H, j == 0);
    add_lin(h, b + ".ffn.ffn_2", H, F);
  }
  add_norm(h, p + ".layer_norm", cout);
  add_norm(h, p + ".pre.layer_norm", cin);
  add_w(h, p + ".pre.conv.weight", {1, cin, H}); add_w(h, p + ".pre.conv.bias", {H});
  add_norm(h, p + ".out_proj.layer_norm", H);
  add_w(h, p + ".out_proj.conv.weight", {1, H, cout}); add_w(h, p + ".out_proj.conv.bias", {cout});
  if (spk) { add_w(h, p + ".spk_proj.weight", {H, h->cfg.ref_dim, 1}); add_w(h, p + ".spk_proj.bias", {H}); }
}

void register_weights(ns2vc_pre* h) {
  const ns2vc_pre_cfg& c = h->cfg;
  register_encoder(h, "phoneme_encoder", c.phone_in, c.phone_hidden, c.phone_out, c.phone_layers, true);
  register_encoder(h, "prompt_encoder", c.prompt_in, c.prompt_hidden, c.prompt_out, c.prompt_layers, false);
  const int R = c.ref_dim;
  add_norm(h, "ref_enc.norm1", R);
  add_w(h, "ref_enc.pool.positional_embedding", {1, R});
  add_lin(h, "ref_enc.pool.k_proj", R, R); add_lin(h, "ref_enc.pool.q_proj", R, R); add_lin(h, "ref_enc.pool.v_proj", R, R);
  add_lin(h, "ref_enc.proj", R, R);
  add_norm(h, "ref_enc.norm2", R);
}

template <class T>
int dev_alloc(ns2vc_pre* h, T** p, size_t n, bool zero) {
  void* q = nullptr;
  NS_CHECK_CUDA(cudaMalloc(&q, std::max<size_t>(n, 1) * sizeof(T)));
  if (zero) NS_CHECK_CUDA(cudaMemset(q, 0, std::max<size_t>(n, 1) * sizeof(T)));
  h->owned.push_back(q);
  *p = reinterpret_cast<T*>(q);
  return 0;
}
int alloc_packed(ns2vc_pre* h, PackedB& pb, int n_logical, int nkb) {
  pb.n_logical = n_logical; pb.Npad = pad_to(n_logical, 128); pb.nkb = nkb;
  const size_t elems = (size_t)nkb * pb.Npad * 64;
  if (dev_alloc(h, &pb.hi, elems, true) || dev_alloc(h, &pb.lo, elems, true)) return -2;
  if (h->simt && dev_alloc(h, &pb.f32, elems, true)) return -2;
  return 0;
}
// w: [n_rows, cin, ktaps] fp32 (device); tap `tap` -> k-blocks kb0.. of the packed operand
int pack(PackedB& pb, const float* w, int n_rows, int cin, int ktaps, int tap, int kb0, cudaStream_t st, const float* cscale = nullptr) {
  PackSeg ps;
  ps.w = w; ps.n_rows = n_rows; ps.cin_total = cin; ps.ktaps = ktaps; ps.tap = tap; ps.cin0 = 0; ps.ncin = cin; ps.n_dst0 = 0; ps.kb0 = kb0;
  ps.nkb = nkb_of(cin); ps.geglu_half = 0; ps.cscale = cscale;
  return launch_pack_b(ps, pb.hi, pb.lo, pb.f32, pb.Npad, st);
}

int pack_encoder(ns2vc_pre* h, EncSite& e, const std::string& p, int cin, int H, int cout, int L, bool spk, cudaStream_t st) {
  const int k = h->cfg.ffn_kernel, F = 4 * H, nh = nkb_of(H);
  e.p = p; e.cin = cin; e.H = H; e.cout = cout; e.L = L; e.spk = spk;
  e.layers.clear();
  int rc;
  auto need = [&](const std::string& n) -> const float* { const float* w = h->W(n); if (!w) set_error("pack: weight %s missing", n.c_str()); return w; };
  // pre: ConvTBC k=1 [1, cin, H] -> [H, cin, 1]
  {
    const float* w = need(p + ".pre.conv.weight"); if (!w) return -1;
    float* wt = nullptr; if (dev_alloc(h, &wt, (size_t)cin * H, false)) return -2;
    if ((rc = launch_tbc_weight(w, 1, cin, H, wt, st))) return rc;
    if ((rc = alloc_packed(h, e.pre, H, nkb_of(cin)))) return rc;
    if ((rc = pack(e.pre, wt, H, cin, 1, 0, 0, st))) return rc;
  }
  for (int i = 0; i < L; ++i) {
    const std::string b = p + ".layers." + std::to_string(i) + ".op";
    LayerSite ls;
    const float* win = need(b + ".self_attn.in_proj_weight"); const float* g1 = need(b + ".layer_norm1.weight"); const float* b1 = need(b + ".layer_norm1.bias");
    if (!win || !g1 || !b1) return -1;
    if ((rc = alloc_packed(h, ls.qkv, 3 * H, nh))) return rc;
    if ((rc = pack(ls.qkv, win, 3 * H, H, 1, 0, 0, st, g1))) return rc;
    if (dev_alloc(h, &ls.g_qkv, (size_t)3 * H, false) || dev_alloc(h, &ls.bf_qkv, (size_t)3 * H, false)) return -2;
    if ((rc = launch_ln_fold_vec(win, g1, b1, nullptr, ls.g_qkv, ls.bf_qkv, 3 * H, H, st))) return rc;
    const float* wo = need(b + ".self_attn.out_proj.weight"); if (!wo) return -1;
    if ((rc = alloc_packed(h, ls.out, H, nh))) return rc;
    if ((rc = pack(ls.out, wo, H, H, 1, 0, 0, st))) return rc;
    // conv-FFN: k Linears -> one (k-1)-tap conv weight, scaled by k^-0.5 (see pre_kernels.cu)
    const float* wt[16];
    for (int j = 0; j < k; ++j) { wt[j] = need(b + ".ffn.ffn_1." + std::to_string(j) + ".weight"); if (!wt[j]) return -1; }
    const float* b0 = need(b + ".ffn.ffn_1.0.bias"); if (!b0) return -1;
    const float scale = (float)std::pow((double)k, -0.5);
    float* wm = nullptr; if (dev_alloc(h, &wm, (size_t)F * H * (k - 1), false)) return -2;
    if ((rc = launch_ffn_taps(wt, k, F, H, (k - 1) / 2 - 1, scale, wm, st))) return rc;
    if (dev_alloc(h, &ls.b_ffn1, (size_t)F, false)) return -2;
    if ((rc = launch_scale_vec(b0, scale, ls.b_ffn1, F, st))) return rc;
    if ((rc = alloc_packed(h, ls.ffn1, F, (k - 1) * nh))) return rc;
    for (int j = 0; j < k - 1; ++j)
      if ((rc = pack(ls.ffn1, wm, F, H, k - 1, j, j * nh, st))) return rc;
    const float* w2 = need(b + ".ffn.ffn_2.weight"); if (!w2) return -1;
    if ((rc = alloc_packed(h, ls.ffn2, H, nkb_of(F)))) return rc;
    if ((rc = pack(ls.ffn2, w2, H, F, 1, 0, 0, st))) return rc;
    e.layers.push_back(ls);
  }
  // out_proj: LayerNorm folded into the k=1 ConvTBC
  {
    const float* w = need(p + ".out_proj.conv.weight"); const float* go = need(p + ".out_proj.layer_norm.weight"); const float* bo = need(p + ".out_proj.layer_norm.bias");
    const float* cb = need(p + ".out_proj.conv.bias");
    if (!w || !go || !bo || !cb) return -1;
    float* wt = nullptr; if (dev_alloc(h, &wt, (size_t)H * cout, false)) return -2;
    if ((rc = launch_tbc_weight(w, 1, H, cout, wt, st))) return rc;
    if ((rc = alloc_packed(h, e.outp, cout, nh))) return rc;
    if ((rc = pack(e.outp, wt, cout, H, 1, 0, 0, st, go))) return rc;
    if (dev_alloc(h, &e.g_out, (size_t)cout, false) || dev_alloc(h, &e.bf_out, (size_t)cout, false)) return -2;
    if ((rc = launch_ln_fold_vec(wt, go, bo, cb, e.g_out, e.bf_out, cout, H, st))) return rc;
  }
  return 0;
}

struct PBuilder {
  ns2vc_pre* h;
  Arena ar;
  int B;
  bool dry;
  std::vector<PLaunch>* out;
  int err = 0;

  SplitBuf split(int Tn, int C) {
    SplitBuf s{}; s.T = Tn; s.C = C; s.ld = pad_to(C, 8);
    s.hi = ar.get<__nv_bfloat16>((size_t)B * Tn * s.ld);
    s.lo = ar.get<__nv_bfloat16>((size_t)B * Tn * s.ld);
    return s;
  }
  GemmOp gemm_base(const PackedB& w, int T_out) {
    GemmOp g; memset(&g, 0, sizeof(g));
    g.B = B; g.T_out = T_out;
    g.w_hi = w.hi; g.w_lo = w.lo; g.w_f32 = w.f32; g.N = w.Npad; g.n_valid = w.n_logical;
    g.f16_col0 = 0x7fffffff; g.ksplit = 1;
    return g;
  }
  void seg(GemmOp& g, int src, int nch, int tap) {
    GSeg& s = g.seg[g.nseg++];
    s.src = src; s.c0 = 0; s.nkb = nkb_of(nch); s.tap = tap;
    g.nkb_total += s.nkb;
  }
  GemmOp lin(const PackedB& w, const SplitBuf& in, int T_out) {
    GemmOp g = gemm_base(w, T_out);
    g.src[0] = in; g.nsrc = 1;
    seg(g, 0, in.C, 0);
    return g;
  }
  void emit_gemm(GemmOp& g, const PackedB& w) {
    PLaunch l; l.kind = PLaunch::GEMM;
    if (!dry) {
      if (g.nkb_total != w.nkb) { set_error("internal: K mismatch %d vs %d", g.nkb_total, w.nkb); err = -1; }
      plan_gemm(g);
      if (!h->simt) { const int rc = encode_tmaps(g); if (rc) err = rc; }
    }
    l.gemm = g;
    out->push_back(l);
  }
  void emit_tap(const std::string& name, const float* src, int rows, int C) {
    if (dry) return;
    PLaunch l; l.kind = PLaunch::TAP; l.a = src; l.i0 = B * rows * C; l.tap_index = (int)h->tap_names.size();
    out->push_back(l);
    h->tap_names.push_back(name); h->tap_rows.push_back(rows); h->tap_ch.push_back(C);
  }
};

// One encoder over Tn frames.  in_patch: 1 = c / lengths / content output, 2 = refer / refer_lengths / prompt output.
void build_encoder(PBuilder& bld, const EncSite& e, int Tn, int in_patch, const float* spk, double*& stat_cur) {
  ns2vc_pre* h = bld.h;
  Arena& ar = bld.ar;
  const int B = bld.B, H = e.H, F = 4 * H, k = h->cfg.ffn_kernel, heads = h->cfg.n_heads, dh = H / heads;
  const size_t M = (size_t)B * Tn;
  const int ldin = pad_to(e.cin, 8);
  float* keep = ar.get<float>(M);
  float* kbias = ar.get<float>(M);
  float* X0 = ar.get<float>(M * ldin);
  float* XA = ar.get<float>(M * H);
  float* XB = ar.get<float>(M * H);
  float* QKV = ar.get<float>(M * 3 * H);
  float* OUTP = ar.get<float>(M * e.cout);
  const SplitBuf s_in = bld.split(Tn, e.cin), s_ln = bld.split(Tn, H), s_qkv = bld.split(Tn, 3 * H), s_att = bld.split(Tn, H),
                 s_y = bld.split(Tn, H), s_ff = bld.split(Tn, F);
  auto new_rowstats = [&]() { double* p = stat_cur; if (stat_cur) stat_cur += 2 * M; return p; };
  auto emits_ln_input = [&](GemmOp& g, double* rs) { g.flags |= EPI_OUT_SPLIT | EPI_ROWSTATS; g.out_hi = s_ln.hi; g.out_lo = s_ln.lo; g.out_split_ld = s_ln.ld; g.row_stats = rs; };
  auto consumes_ln = [&](GemmOp& g, const double* rs, const float* gv, const float* bf) {
    g.flags |= EPI_LNFOLD | EPI_BIAS; g.ln_stats = rs; g.ln_g = gv; g.bias = bf; g.ln_C = H; g.ln_eps = 1e-5f; };
  auto masked = [&](GemmOp& g) { g.flags |= EPI_ROWMASK; g.rowmask = keep; };

  { PLaunch l; l.kind = PLaunch::SEQMASK; l.patch = in_patch; l.i0 = Tn; l.o = keep; l.o2 = kbias; bld.out->push_back(l); }
  { PLaunch l; l.kind = PLaunch::ENC_INPUT; l.patch = in_patch; l.b = spk; l.c = keep; l.i0 = e.cin; l.i1 = Tn; l.o = X0; l.i2 = ldin; bld.out->push_back(l); }
  { PLaunch l; l.kind = PLaunch::LN_SPLIT; l.a = X0; l.i0 = ldin; l.i1 = (int)M; l.i2 = e.cin; l.f0 = 1e-5f;
    l.b = h->W(e.p + ".pre.layer_norm.weight"); l.c = h->W(e.p + ".pre.layer_norm.bias"); l.split = s_in; bld.out->push_back(l); }
  double* rs = new_rowstats();
  { GemmOp g = bld.lin(e.pre, s_in, Tn);
    g.flags = EPI_BIAS | EPI_OUT_F32; g.bias = h->W(e.p + ".pre.conv.bias"); g.out = XA; g.out_ld = H;
    masked(g); emits_ln_input(g, rs);
    bld.emit_gemm(g, e.pre); }
  bld.emit_tap(e.p + ".pre", XA, Tn, H);
  const bool av2 = !h->simt && attention_v2_supported(dh, Tn, true);
  for (int i = 0; i < e.L; ++i) {
    const LayerSite& ls = e.layers[i];
    const std::string b = e.p + ".layers." + std::to_string(i) + ".op";
    { GemmOp g = bld.lin(ls.qkv, s_ln, Tn);
      if (av2) { g.flags = EPI_OUT_SPLIT; g.out_hi = s_qkv.hi; g.out_lo = s_qkv.lo; g.out_split_ld = s_qkv.ld; }   // (V stays a bf16 split: p_split below)
      else { g.flags = EPI_OUT_F32; g.out = QKV; g.out_ld = 3 * H; }
      consumes_ln(g, rs, ls.g_qkv, ls.bf_qkv);
      bld.emit_gemm(g, ls.qkv); }
    { PLaunch l; l.kind = PLaunch::ATTN; AttnOp& a = l.attn; memset(&a, 0, sizeof(a));
      a.q = QKV; a.q_ld = 3 * H; a.k = QKV + H; a.k_ld = 3 * H; a.v = QKV + 2 * H; a.v_ld = 3 * H; a.bias = kbias;
      a.out_hi = s_att.hi; a.out_lo = s_att.lo; a.out_split_ld = s_att.ld;
      a.B = B; a.H = heads; a.Tq = Tn; a.Tk = Tn; a.dh = dh; a.scale = 1.0f / sqrtf((float)dh);
      // bf16 hi/lo softmax weights: with a few dozen keys the 2^-12 rounding of fp16 weights (the denoiser's default over 256-2048
      // keys) does not average out - measured on the shipped configuration at S = 32: worst err/tol 1.16 with fp16 weights, 0.24 split
      if (av2) { a.v2 = 1; a.p_split = 1; a.qs = s_qkv; a.ks = s_qkv; a.vs = s_qkv; a.q_c0 = 0; a.k_c0 = H; a.v_c0 = 2 * H;
                 if (!bld.dry) { const int rc = encode_attn_tmaps(a); if (rc) bld.err = rc; } }
      bld.out->push_back(l); }
    { GemmOp g = bld.lin(ls.out, s_att, Tn);
      g.flags = EPI_RESIDUAL | EPI_OUT_F32; g.res = XA; g.res_ld = H; g.out = XB; g.out_ld = H;
      masked(g);
      bld.emit_gemm(g, ls.out); }
    { PLaunch l; l.kind = PLaunch::LN_SPLIT; l.a = XB; l.i0 = H; l.i1 = (int)M; l.i2 = H; l.f0 = 1e-5f;
      l.b = h->W(b + ".layer_norm2.weight"); l.c = h->W(b + ".layer_norm2.bias"); l.split = s_y; bld.out->push_back(l); }
    { GemmOp g = bld.gemm_base(ls.ffn1, Tn);
      g.src[0] = s_y; g.nsrc = 1;
      for (int j = 0; j < k - 1; ++j) bld.seg(g, 0, H, j + 1 - (k - 1) / 2);     // row offsets -3 .. +4 for k = 9
      g.flags = EPI_BIAS | EPI_RELU | EPI_OUT_SPLIT; g.bias = ls.b_ffn1;
      g.out_hi = s_ff.hi; g.out_lo = s_ff.lo; g.out_split_ld = s_ff.ld;
      bld.emit_gemm(g, ls.ffn1); }
    rs = new_rowstats();
    { GemmOp g = bld.lin(ls.ffn2, s_ff, Tn);
      g.flags = EPI_BIAS | EPI_RESIDUAL | EPI_OUT_F32; g.bias = h->W(b + ".ffn.ffn_2.bias"); g.res = XB; g.res_ld = H; g.out = XA; g.out_ld = H;
      masked(g); emits_ln_input(g, rs);
      bld.emit_gemm(g, ls.ffn2); }
    bld.emit_tap(e.p + ".layers." + std::to_string(i), XA, Tn, H);
  }
  { GemmOp g = bld.lin(e.outp, s_ln, Tn);
    g.flags = EPI_OUT_F32; g.out = OUTP; g.out_ld = e.cout;
    consumes_ln(g, rs, e.g_out, e.bf_out);
    bld.emit_gemm(g, e.outp); }
  { PLaunch l; l.kind = PLaunch::LN_MASK; l.patch = in_patch; l.a = OUTP; l.i0 = e.cout; l.i1 = (int)M; l.i2 = e.cout; l.f0 = 1e-5f;
    l.b = h->W(e.p + ".layer_norm.weight"); l.c = h->W(e.p + ".layer_norm.bias"); l.d = keep; bld.out->push_back(l); }
}

int build_program(ns2vc_pre* h, int B, int T, int S, void* ws, size_t* bytes_out) {
  const ns2vc_pre_cfg& c = h->cfg;
  const bool dry = ws == nullptr;
  NS_REQUIRE(B >= 1 && T >= 1 && S >= 1, "bad shape B=%d T=%d S=%d", B, T, S);
  std::vector<PLaunch> prog;
  if (!dry) { h->tap_names.clear(); h->tap_rows.clear(); h->tap_ch.clear(); }
  PBuilder bld{h, Arena{(uint8_t*)ws, 0}, B, dry, &prog};
  Arena& ar = bld.ar;
  // LayerNorm row sums (double [rows][2] per folded LayerNorm), zeroed by the program's only memset
  const size_t stat_doubles = (size_t)2 * B * ((size_t)T * (c.phone_layers + 1) + (size_t)S * (c.prompt_layers + 1));
  double* stat_arena = ar.get<double>(stat_doubles);
  double* stat_cur = stat_arena;
  { PLaunch l; l.kind = PLaunch::MEMSET; l.mem = stat_arena; l.mem_bytes = stat_doubles * sizeof(double); prog.push_back(l); }
  // ---- ref_enc: TextTimeEmbedding over ALL S prompt frames (the reference does not mask them: model.py:362)
  const int R = c.ref_dim;
  float* rt = ar.get<float>((size_t)B * S * R);
  float* rn = ar.get<float>((size_t)B * S * R);
  float* rtok = ar.get<float>((size_t)B * (S + 1) * R);
  float* rq = ar.get<float>((size_t)B * R);
  float* rkv = ar.get<float>((size_t)B * (S + 1) * 2 * R);
  float* rpool = ar.get<float>((size_t)B * R);
  float* rproj = ar.get<float>((size_t)B * R);
  float* g = ar.get<float>((size_t)B * R);
  float* spk = ar.get<float>((size_t)B * c.phone_hidden);
  { PLaunch l; l.kind = PLaunch::NCT2TOK; l.patch = 2; l.i0 = R; l.i1 = S; l.o = rt; prog.push_back(l); }
  { PLaunch l; l.kind = PLaunch::LN_APPLY; l.a = rt; l.i0 = R; l.i1 = B * S; l.i2 = R; l.f0 = 1e-5f; l.b = h->W("ref_enc.norm1.weight"); l.c = h->W("ref_enc.norm1.bias"); l.o = rn; l.i3 = R; prog.push_back(l); }
  { PLaunch l; l.kind = PLaunch::POOL_CLS; l.a = rn; l.b = h->W("ref_enc.pool.positional_embedding"); l.i0 = S; l.i1 = R; l.o = rtok; prog.push_back(l); }
  { PLaunch l; l.kind = PLaunch::LINEAR; LinOp& o = l.lin; memset(&o, 0, sizeof(o));
    o.x = rtok; o.x_ld = (S + 1) * R; o.M = B; o.K = R; o.W = h->W("ref_enc.pool.q_proj.weight"); o.bias = h->W("ref_enc.pool.q_proj.bias"); o.N = R; o.out = rq; o.out_ld = R; prog.push_back(l); }
  { PLaunch l; l.kind = PLaunch::LINEAR; LinOp& o = l.lin; memset(&o, 0, sizeof(o));
    o.x = rtok; o.x_ld = R; o.M = B * (S + 1); o.K = R; o.W = h->ref_kvW; o.bias = h->ref_kvb; o.N = 2 * R; o.out = rkv; o.out_ld = 2 * R; prog.push_back(l); }
  { PLaunch l; l.kind = PLaunch::POOL_ATT; l.a = rq; l.b = rkv; l.i0 = S + 1; l.i1 = R; l.i2 = c.ref_heads; l.o = rpool; prog.push_back(l); }
  { PLaunch l; l.kind = PLaunch::LINEAR; LinOp& o = l.lin; memset(&o, 0, sizeof(o));
    o.x = rpool; o.x_ld = R; o.M = B; o.K = R; o.W = h->W("ref_enc.proj.weight"); o.bias = h->W("ref_enc.proj.bias"); o.N = R; o.out = rproj; o.out_ld = R; prog.push_back(l); }
  { PLaunch l; l.kind = PLaunch::LN_APPLY; l.a = rproj; l.i0 = R; l.i1 = B; l.i2 = R; l.f0 = 1e-5f; l.b = h->W("ref_enc.norm2.weight"); l.c = h->W("ref_enc.norm2.bias"); l.o = g; l.i3 = R; prog.push_back(l); }
  bld.emit_tap("ref_enc", g, 1, R);
  // spk_proj: Conv1d(100, hidden, 1) on g [B, 100, 1] (model.py:123, 127)
  { PLaunch l; l.kind = PLaunch::LINEAR; LinOp& o = l.lin; memset(&o, 0, sizeof(o));
    o.x = g; o.x_ld = R; o.M = B; o.K = R; o.W = h->W("phoneme_encoder.spk_proj.weight"); o.bias = h->W("phoneme_encoder.spk_proj.bias"); o.N = c.phone_hidden; o.out = spk; o.out_ld = c.phone_hidden; prog.push_back(l); }
  build_encoder(bld, h->prompt, S, 2, nullptr, stat_cur);
  build_encoder(bld, h->phone, T, 1, spk, stat_cur);
  if (bld.err) return bld.err;
  if (bytes_out) *bytes_out = ar.off + 256;
  if (!dry) {
    h->prog = std::move(prog);
    h->tap_dst.assign(h->tap_names.size(), nullptr);
    h->pB = B; h->pT = T; h->pS = S; h->pws = ws;
  }
  return 0;
}

int run_program(ns2vc_pre* h, const float* c, const float* refer, const long long* lengths, const long long* refer_lengths, float* content,
                float* prompt, cudaStream_t st) {
  int rc = 0, count = 0;
  const int B = h->pB;
  for (PLaunch& l : h->prog) {
    switch (l.kind) {
      case PLaunch::MEMSET: {
        cudaError_t e = cudaMemsetAsync(l.mem, 0, l.mem_bytes, st);
        if (e != cudaSuccess) { set_error("memset failed: %s", cudaGetErrorString(e)); rc = -2; }
        break;
      }
      case PLaunch::SEQMASK: rc = launch_seq_mask(l.patch == 1 ? lengths : refer_lengths, B, l.i0, l.o, l.o2, st); break;
      case PLaunch::ENC_INPUT: {
        const float* src = l.patch == 1 ? c : refer;
        rc = launch_enc_input(src, (long long)l.i0 * l.i1, l.b, l.c, B, l.i0, l.i1, l.o, l.i2, st);
        break;
      }
      case PLaunch::LN_SPLIT: rc = launch_ln_split(l.a, l.i0, l.i1, l.i2, l.f0, l.b, l.c, l.split, st); break;
      case PLaunch::GEMM: rc = h->simt ? launch_gemm_simt(l.gemm, st) : launch_gemm_tc(l.gemm, st); break;
      case PLaunch::ATTN: rc = (l.attn.v2 && !h->simt) ? launch_attention_v2(l.attn, st) : launch_attention(l.attn, st, h->simt); break;
      case PLaunch::LN_MASK: rc = launch_ln_mask(l.a, l.i0, l.i1, l.i2, l.f0, l.b, l.c, l.d, l.patch == 1 ? content : prompt, l.i2, st); break;
      case PLaunch::NCT2TOK: rc = launch_nct_to_tokens(refer, (long long)l.i0 * l.i1, B, l.i0, l.i1, l.o, l.i0, l.i0, st); break;
      case PLaunch::LN_APPLY: rc = launch_ln_apply(l.a, l.i0, l.i1, l.i2, l.f0, l.b, l.c, l.o, l.i3, st); break;
      case PLaunch::POOL_CLS: rc = launch_pool_class_token(l.a, l.b, B, l.i0, l.i1, l.o, st); break;
      case PLaunch::LINEAR: rc = launch_small_linear(l.lin, st); break;
      case PLaunch::POOL_ATT: rc = launch_pool_attend_wide(l.a, l.b, B, l.i0, l.i1, l.i2, l.o, st); break;
      case PLaunch::TAP:
        --count;
        if (l.tap_index >= 0 && l.tap_index < (int)h->tap_dst.size() && h->tap_dst[l.tap_index]) {
          cudaError_t e = cudaMemcpyAsync(h->tap_dst[l.tap_index], l.a, (size_t)l.i0 * sizeof(float), cudaMemcpyDeviceToDevice, st);
          if (e != cudaSuccess) { set_error("tap copy failed: %s", cudaGetErrorString(e)); rc = -2; }
        }
        break;
    }
    if (rc) return rc;
    ++count;
  }
  h->last_launches = count;
  return 0;
}

}  // namespace

extern "C" {

int ns2vc_pre_create(const ns2vc_pre_cfg* cfg, ns2vc_pre** out) {
  NS_REQUIRE(cfg && out, "null argument");
  NS_REQUIRE(cfg->n_heads >= 1 && cfg->ref_heads >= 1 && cfg->ref_dim >= 1 && cfg->ref_dim % cfg->ref_heads == 0, "bad head configuration");
  NS_REQUIRE(cfg->ffn_kernel >= 3 && cfg->ffn_kernel <= 9 && (cfg->ffn_kernel & 1), "ffn_kernel %d unsupported (odd, 3..9: the taps run as up to %d GEMM segments)", cfg->ffn_kernel, kMaxSeg);
  NS_REQUIRE(cfg->phone_in == cfg->phone_hidden, "PhoneEncoder adds spk_proj(g) [hidden] to the content [in]: in_channels %d != hidden_channels %d (model.py:130)", cfg->phone_in, cfg->phone_hidden);
  NS_REQUIRE(cfg->prompt_in == cfg->ref_dim, "ref_enc and the prompt encoder read the same mel prompt: prompt_in %d != ref_dim %d", cfg->prompt_in, cfg->ref_dim);
  const int Hs[2] = {cfg->phone_hidden, cfg->prompt_hidden};
  for (int H : Hs) {
    NS_REQUIRE(H >= 8 && H % cfg->n_heads == 0 && H % 8 == 0 && H <= 1024, "hidden width %d must be a multiple of 8 and of the %d heads, <= 1024", H, cfg->n_heads);
    NS_REQUIRE(H / cfg->n_heads <= 64 && (H / cfg->n_heads) % 4 == 0, "head width %d unsupported", H / cfg->n_heads);
  }
  NS_REQUIRE(cfg->phone_layers >= 0 && cfg->prompt_layers >= 0 && cfg->phone_out >= 1 && cfg->prompt_out >= 1 && cfg->phone_in >= 1 && cfg->prompt_in >= 1 &&
             cfg->phone_in <= 1024 && cfg->prompt_in <= 1024, "bad encoder configuration");
  ns2vc_pre* h = new ns2vc_pre();
  h->cfg = *cfg;
  const char* be = getenv("NS2VC_GEMM_BACKEND");
  h->simt = be && strcmp(be, "simt") == 0;
  register_weights(h);
  *out = h;
  return 0;
}

void ns2vc_pre_destroy(ns2vc_pre* h) {
  if (!h) return;
  for (auto& w : h->weights) if (w.d) cudaFree(w.d);
  for (void* p : h->owned) cudaFree(p);
  delete h;
}

int ns2vc_pre_num_weights(const ns2vc_pre* h) { return h ? (int)h->weights.size() : -1; }

int ns2vc_pre_weight_info(const ns2vc_pre* h, int i, const char** name, int64_t shape[4], int* ndim) {
  NS_REQUIRE(h && i >= 0 && i < (int)h->weights.size(), "weight index %d out of range", i);
  const WSlot& w = h->weights[i];
  if (name) *name = w.name.c_str();
  if (ndim) *ndim = (int)w.shape.size();
  if (shape) for (size_t k = 0; k < w.shape.size() && k < 4; ++k) shape[k] = w.shape[k];
  return 0;
}

int ns2vc_pre_load_weight(ns2vc_pre* h, const char* key, const float* dptr, const int64_t* shape, int ndim, ns2vc_stream stream) {
  NS_REQUIRE(h && key && dptr, "null argument");
  auto it = h->windex.find(key);
  NS_REQUIRE(it != h->windex.end(), "Unexpected key in state_dict: %s", key);
  WSlot& w = h->weights[it->second];
  NS_REQUIRE(ndim == (int)w.shape.size(), "size mismatch for %s: expected %d dims, got %d", key, (int)w.shape.size(), ndim);
  for (int k = 0; k < ndim; ++k) NS_REQUIRE(shape[k] == w.shape[k], "size mismatch for %s at dim %d: expected %lld, got %lld", key, k, (long long)w.shape[k], (long long)shape[k]);
  if (!w.d) NS_CHECK_CUDA(cudaMalloc(&w.d, w.numel() * sizeof(float)));
  NS_CHECK_CUDA(cudaMemcpyAsync(w.d, dptr, w.numel() * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  w.loaded = true;
  h->finalized = false;
  return 0;
}

int ns2vc_pre_finalize(ns2vc_pre* h, ns2vc_stream stream) {
  NS_REQUIRE(h, "null handle");
  for (auto& w : h->weights) NS_REQUIRE(w.loaded, "Missing key in state_dict: %s", w.name.c_str());
  for (void* p : h->owned) cudaFree(p);
  h->owned.clear();
  h->prog.clear(); h->pB = h->pT = h->pS = 0; h->pws = nullptr;
  const ns2vc_pre_cfg& c = h->cfg;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = pack_encoder(h, h->phone, "phoneme_encoder", c.phone_in, c.phone_hidden, c.phone_out, c.phone_layers, true, st);
  if (rc) return rc;
  rc = pack_encoder(h, h->prompt, "prompt_encoder", c.prompt_in, c.prompt_hidden, c.prompt_out, c.prompt_layers, false, st);
  if (rc) return rc;
  {
    const int R = c.ref_dim;
    if (dev_alloc(h, &h->ref_kvW, (size_t)2 * R * R, false) || dev_alloc(h, &h->ref_kvb, (size_t)2 * R, false)) return -2;
    NS_CHECK_CUDA(cudaMemcpyAsync(h->ref_kvW, h->W("ref_enc.pool.k_proj.weight"), (size_t)R * R * 4, cudaMemcpyDeviceToDevice, st));
    NS_CHECK_CUDA(cudaMemcpyAsync(h->ref_kvW + (size_t)R * R, h->W("ref_enc.pool.v_proj.weight"), (size_t)R * R * 4, cudaMemcpyDeviceToDevice, st));
    NS_CHECK_CUDA(cudaMemcpyAsync(h->ref_kvb, h->W("ref_enc.pool.k_proj.bias"), (size_t)R * 4, cudaMemcpyDeviceToDevice, st));
    NS_CHECK_CUDA(cudaMemcpyAsync(h->ref_kvb + R, h->W("ref_enc.pool.v_proj.bias"), (size_t)R * 4, cudaMemcpyDeviceToDevice, st));
  }
  NS_CHECK_CUDA(cudaGetLastError());
  h->finalized = true;
  return 0;
}

int ns2vc_pre_workspace_bytes(const ns2vc_pre* h, int B, int T, int S, size_t* bytes) {
  NS_REQUIRE(h && bytes, "null argument");
  NS_REQUIRE(h->finalized, "ns2vc_pre_finalize() has not been called");
  return build_program(const_cast<ns2vc_pre*>(h), B, T, S, nullptr, bytes);
}

int ns2vc_pre_infer(ns2vc_pre* h, const float* c, const float* refer, const int64_t* lengths, const int64_t* refer_lengths, float* content,
                    float* prompt, int B, int T, int S, void* ws, ns2vc_stream stream) {
  NS_REQUIRE(h && c && refer && lengths && refer_lengths && content && prompt, "null argument");
  NS_REQUIRE(h->finalized, "ns2vc_pre_finalize() has not been called");
  NS_REQUIRE(ws != nullptr, "workspace is NULL");
  if (!(h->pB == B && h->pT == T && h->pS == S && h->pws == ws)) {
    const int rc = build_program(h, B, T, S, ws, nullptr);
    if (rc) return rc;
  }
  return run_program(h, c, refer, reinterpret_cast<const long long*>(lengths), reinterpret_cast<const long long*>(refer_lengths), content, prompt,
                     (cudaStream_t)stream);
}

int ns2vc_pre_num_taps(const ns2vc_pre* h) { return h ? (int)h->tap_names.size() : -1; }
int ns2vc_pre_tap_info(const ns2vc_pre* h, int i, const char** name, int* rows, int* channels) {
  NS_REQUIRE(h && i >= 0 && i < (int)h->tap_names.size(), "tap index %d out of range", i);
  if (name) *name = h->tap_names[i].c_str();
  if (rows) *rows = h->tap_rows[i];
  if (channels) *channels = h->tap_ch[i];
  return 0;
}
int ns2vc_pre_set_tap(ns2vc_pre* h, int i, float* dst) {
  NS_REQUIRE(h && i >= 0 && i < (int)h->tap_dst.size(), "tap index %d out of range", i);
  h->tap_dst[i] = dst;
  return 0;
}
int ns2vc_pre_launch_count(const ns2vc_pre* h) { return h ? h->last_launches : -1; }

}  // extern "C"
