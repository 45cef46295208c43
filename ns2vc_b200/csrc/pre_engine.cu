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
#include "engine_host.cuh"
#include "../../include/ns2vc_b200.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

using namespace ns2vc;

namespace {

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

}  // namespace

struct ns2vc_pre : SingleProgramEngine {
  ns2vc_pre_cfg cfg;
  bool simt = false;
  EncSite phone, prompt;
  PoolKV ref_kv;                                       // ref_enc.pool k_proj | v_proj as one [2R, R] operator
};

namespace ns2vc {
const EngineBase* engine_base(const ns2vc_pre* h) { return h; }
}  // namespace ns2vc

namespace {

// reference parameter names / shapes (model.py:98-127, 156-172; operations.py:784-797, 304-340, 644-663)
void register_encoder(ns2vc_pre* h, const std::string& p, int cin, int H, int cout, int L, bool spk) {
  WeightRegistry& w = h->weights;
  const int k = h->cfg.ffn_kernel, F = 4 * H;
  for (int i = 0; i < L; ++i) {
    const std::string b = p + ".layers." + std::to_string(i) + ".op";
    w.add_norm(b + ".layer_norm1", H);
    w.add(b + ".self_attn.in_proj_weight", {3 * H, H});
    w.add(b + ".self_attn.out_proj.weight", {H, H});
    w.add_norm(b + ".layer_norm2", H);
    for (int j = 0; j < k; ++j) w.add_lin(b + ".ffn.ffn_1." + std::to_string(j), F, H, j == 0);
    w.add_lin(b + ".ffn.ffn_2", H, F);
  }
  w.add_norm(p + ".layer_norm", cout);
  w.add_norm(p + ".pre.layer_norm", cin);
  w.add(p + ".pre.conv.weight", {1, cin, H}); w.add(p + ".pre.conv.bias", {H});
  w.add_norm(p + ".out_proj.layer_norm", H);
  w.add(p + ".out_proj.conv.weight", {1, H, cout}); w.add(p + ".out_proj.conv.bias", {cout});
  if (spk) w.add_conv(p + ".spk_proj", H, h->cfg.ref_dim, 1);
}

void register_weights(ns2vc_pre* h) {
  const ns2vc_pre_cfg& c = h->cfg;
  register_encoder(h, "phoneme_encoder", c.phone_in, c.phone_hidden, c.phone_out, c.phone_layers, true);
  register_encoder(h, "prompt_encoder", c.prompt_in, c.prompt_hidden, c.prompt_out, c.prompt_layers, false);
  WeightRegistry& w = h->weights;
  const int R = c.ref_dim;
  w.add_norm("ref_enc.norm1", R);
  w.add("ref_enc.pool.positional_embedding", {1, R});
  w.add_lin("ref_enc.pool.k_proj", R, R); w.add_lin("ref_enc.pool.q_proj", R, R); w.add_lin("ref_enc.pool.v_proj", R, R);
  w.add_lin("ref_enc.proj", R, R);
  w.add_norm("ref_enc.norm2", R);
}

int pack_encoder(ns2vc_pre* h, EncSite& e, const std::string& p, int cin, int H, int cout, int L, bool spk, cudaStream_t st) {
  const int k = h->cfg.ffn_kernel, F = 4 * H, nh = nkb_of(H);
  e.p = p; e.cin = cin; e.H = H; e.cout = cout; e.L = L; e.spk = spk;
  e.layers.clear();
  DeviceMem& mem = h->mem;
  int rc;
  auto need = [&](const std::string& n) -> const float* { const float* w = h->weights.W(n); if (!w) set_error("pack: weight %s missing", n.c_str()); return w; };
  // pre: ConvTBC k=1 [1, cin, H] -> [H, cin, 1]
  {
    const float* w = need(p + ".pre.conv.weight"); if (!w) return -1;
    float* wt = mem.alloc<float>((size_t)cin * H); if (!wt) return -2;
    if ((rc = launch_tbc_weight(w, 1, cin, H, wt, st))) return rc;
    if ((rc = mem.alloc_packed(e.pre, H, H, nkb_of(cin), h->simt))) return rc;
    if ((rc = pack_seg(e.pre, wt, H, cin, 1, 0, 0, cin, 0, 0, 0, st))) return rc;
    h->packed.add(p + ".pre", e.pre);
  }
  for (int i = 0; i < L; ++i) {
    const std::string b = p + ".layers." + std::to_string(i) + ".op";
    LayerSite ls;
    const float* win = need(b + ".self_attn.in_proj_weight"); const float* g1 = need(b + ".layer_norm1.weight"); const float* b1 = need(b + ".layer_norm1.bias");
    if (!win || !g1 || !b1) return -1;
    if ((rc = mem.alloc_packed(ls.qkv, 3 * H, 3 * H, nh, h->simt))) return rc;
    if ((rc = pack_seg(ls.qkv, win, 3 * H, H, 1, 0, 0, H, 0, 0, 0, st, g1))) return rc;
    if (!(ls.g_qkv = mem.alloc<float>((size_t)3 * H)) || !(ls.bf_qkv = mem.alloc<float>((size_t)3 * H))) return -2;
    if ((rc = launch_ln_fold_vec(win, g1, b1, nullptr, ls.g_qkv, ls.bf_qkv, 3 * H, H, st))) return rc;
    const float* wo = need(b + ".self_attn.out_proj.weight"); if (!wo) return -1;
    if ((rc = mem.alloc_packed(ls.out, H, H, nh, h->simt))) return rc;
    if ((rc = pack_seg(ls.out, wo, H, H, 1, 0, 0, H, 0, 0, 0, st))) return rc;
    // conv-FFN: k Linears -> one (k-1)-tap conv weight, scaled by k^-0.5 (see pre_kernels.cu)
    const float* wt[16];
    for (int j = 0; j < k; ++j) { wt[j] = need(b + ".ffn.ffn_1." + std::to_string(j) + ".weight"); if (!wt[j]) return -1; }
    const float* b0 = need(b + ".ffn.ffn_1.0.bias"); if (!b0) return -1;
    const float scale = (float)std::pow((double)k, -0.5);
    float* wm = mem.alloc<float>((size_t)F * H * (k - 1)); if (!wm) return -2;
    if ((rc = launch_ffn_taps(wt, k, F, H, (k - 1) / 2 - 1, scale, wm, st))) return rc;
    if (!(ls.b_ffn1 = mem.alloc<float>((size_t)F))) return -2;
    if ((rc = launch_scale_vec(b0, scale, ls.b_ffn1, F, st))) return rc;
    if ((rc = mem.alloc_packed(ls.ffn1, F, F, (k - 1) * nh, h->simt))) return rc;
    for (int j = 0; j < k - 1; ++j)
      if ((rc = pack_seg(ls.ffn1, wm, F, H, k - 1, j, 0, H, 0, j * nh, 0, st))) return rc;
    const float* w2 = need(b + ".ffn.ffn_2.weight"); if (!w2) return -1;
    if ((rc = mem.alloc_packed(ls.ffn2, H, H, nkb_of(F), h->simt))) return rc;
    if ((rc = pack_seg(ls.ffn2, w2, H, F, 1, 0, 0, F, 0, 0, 0, st))) return rc;
    const std::string site = p + ".layers." + std::to_string(i);
    h->packed.add(site + ".qkv", ls.qkv, {{"g_qkv", ls.g_qkv, 3 * H}, {"bf_qkv", ls.bf_qkv, 3 * H}});
    h->packed.add(site + ".out", ls.out);
    h->packed.add(site + ".ffn1", ls.ffn1, {{"b_ffn1", ls.b_ffn1, F}});
    h->packed.add(site + ".ffn2", ls.ffn2);
    e.layers.push_back(ls);
  }
  // out_proj: LayerNorm folded into the k=1 ConvTBC
  {
    const float* w = need(p + ".out_proj.conv.weight"); const float* go = need(p + ".out_proj.layer_norm.weight"); const float* bo = need(p + ".out_proj.layer_norm.bias");
    const float* cb = need(p + ".out_proj.conv.bias");
    if (!w || !go || !bo || !cb) return -1;
    float* wt = mem.alloc<float>((size_t)H * cout); if (!wt) return -2;
    if ((rc = launch_tbc_weight(w, 1, H, cout, wt, st))) return rc;
    if ((rc = mem.alloc_packed(e.outp, cout, cout, nh, h->simt))) return rc;
    if ((rc = pack_seg(e.outp, wt, cout, H, 1, 0, 0, H, 0, 0, 0, st, go))) return rc;
    if (!(e.g_out = mem.alloc<float>((size_t)cout)) || !(e.bf_out = mem.alloc<float>((size_t)cout))) return -2;
    if ((rc = launch_ln_fold_vec(wt, go, bo, cb, e.g_out, e.bf_out, cout, H, st))) return rc;
    h->packed.add(p + ".out_proj", e.outp, {{"g_out", e.g_out, cout}, {"bf_out", e.bf_out, cout}});
  }
  return 0;
}

int pack(ns2vc_pre* h, cudaStream_t st) {
  const ns2vc_pre_cfg& c = h->cfg;
  int rc;
  if ((rc = pack_encoder(h, h->phone, "phoneme_encoder", c.phone_in, c.phone_hidden, c.phone_out, c.phone_layers, true, st))) return rc;
  if ((rc = pack_encoder(h, h->prompt, "prompt_encoder", c.prompt_in, c.prompt_hidden, c.prompt_out, c.prompt_layers, false, st))) return rc;
  if ((rc = concat_pool_kv(h->mem, h->weights, "ref_enc.pool", c.ref_dim, h->ref_kv, st))) return rc;
  h->packed.add("ref_enc.pool.kv", PackedB{}, {{"W", h->ref_kv.W, 2LL * c.ref_dim * c.ref_dim}, {"b", h->ref_kv.b, 2LL * c.ref_dim}});
  return 0;
}

// The call arguments of one encoder: its lengths, its [B, C, T] input, its [B, T, C_out] output and (SPK or NONE) the speaker
// rows added to its input when the call supplies them.
struct EncIo { Launch::Input lengths, in, out, spk = Launch::NONE; };

// One encoder over Tn frames.  `ragged`: LN2's split is 0 on rows past the entry's length, so the conv-FFN reads zeros there as
// an unpadded run reads its zero padding.  `ilens`: where SEQMASK also writes the lengths as int [B], clamped to [1, Tn], or nullptr.
void build_encoder(ns2vc_pre* h, ProgramBuilder& bld, TapSet& taps, const EncSite& e, int Tn, EncIo io, const float* spk, double*& stat_cur,
                   bool ragged, int* ilens) {
  Arena& ar = bld.ar;
  const WeightRegistry& w = h->weights;
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
  auto masked = [&](GemmOp& g) { g.flags |= EPI_ROWMASK; g.rowmask = keep; };

  bld.emit(Launch::SEQMASK, SeqMaskOp{nullptr, B, Tn, keep, kbias, ilens}, io.lengths);
  bld.emit(Launch::ENC_INPUT, TokensOp{nullptr, 0, B, e.cin, Tn, X0, ldin, spk, keep}, io.in).input2 = io.spk;
  bld.emit_ln_split(X0, ldin, (int)M, e.cin, w.W(e.p + ".pre.layer_norm.weight"), w.W(e.p + ".pre.layer_norm.bias"), s_in);
  double* rs = new_rowstats();
  { GemmOp g = bld.lin(e.pre, s_in, Tn);
    g.flags = EPI_BIAS | EPI_OUT_F32; g.bias = w.W(e.p + ".pre.conv.bias"); g.out = XA; g.out_ld = H;
    masked(g); bld.emits_ln_input(g, s_ln, rs);
    bld.emit_gemm(g, e.pre); }
  bld.emit_tap(taps, e.p + ".pre", XA, Tn, H, Tn);
  const bool av2 = !h->simt && attention_v2_supported(dh, Tn, true);
  for (int i = 0; i < e.L; ++i) {
    const LayerSite& ls = e.layers[i];
    const std::string b = e.p + ".layers." + std::to_string(i) + ".op";
    { GemmOp g = bld.lin(ls.qkv, s_ln, Tn);
      if (av2) { g.flags = EPI_OUT_SPLIT; g.out_hi = s_qkv.hi; g.out_lo = s_qkv.lo; g.out_split_ld = s_qkv.ld; }   // (V stays a bf16 split: p_split below)
      else { g.flags = EPI_OUT_F32; g.out = QKV; g.out_ld = 3 * H; }
      bld.consumes_ln(g, rs, ls.g_qkv, ls.bf_qkv, H);
      bld.emit_gemm(g, ls.qkv); }
    { AttnOp a; memset(&a, 0, sizeof(a));
      a.q = QKV; a.q_ld = 3 * H; a.k = QKV + H; a.k_ld = 3 * H; a.v = QKV + 2 * H; a.v_ld = 3 * H; a.bias = kbias;
      a.out_hi = s_att.hi; a.out_lo = s_att.lo; a.out_split_ld = s_att.ld;
      a.B = B; a.H = heads; a.Tq = Tn; a.Tk = Tn; a.dh = dh; a.scale = 1.0f / sqrtf((float)dh);
      // bf16 hi/lo softmax weights: with a few dozen keys the 2^-12 rounding of fp16 weights (the denoiser's default over 256-2048
      // keys) does not average out - measured on the shipped configuration at S = 32: worst err/tol 1.16 with fp16 weights, 0.24 split
      if (av2) { a.v2 = 1; a.p_split = 1; a.qs = s_qkv; a.ks = s_qkv; a.vs = s_qkv; a.q_c0 = 0; a.k_c0 = H; a.v_c0 = 2 * H; }
      bld.emit_attention(a); }
    { GemmOp g = bld.lin(ls.out, s_att, Tn);
      g.flags = EPI_RESIDUAL | EPI_OUT_F32; g.res = XA; g.res_ld = H; g.out = XB; g.out_ld = H;
      masked(g);
      bld.emit_gemm(g, ls.out); }
    bld.emit_ln_split(XB, H, (int)M, H, w.W(b + ".layer_norm2.weight"), w.W(b + ".layer_norm2.bias"), s_y, ragged ? keep : nullptr);
    { GemmOp g = bld.gemm_base(ls.ffn1, Tn);
      const int src = bld.add_src(g, s_y);
      for (int j = 0; j < k - 1; ++j) bld.seg(g, src, 0, H, j + 1 - (k - 1) / 2);     // row offsets -3 .. +4 for k = 9
      g.flags = EPI_BIAS | EPI_RELU | EPI_OUT_SPLIT; g.bias = ls.b_ffn1;
      g.out_hi = s_ff.hi; g.out_lo = s_ff.lo; g.out_split_ld = s_ff.ld;
      bld.emit_gemm(g, ls.ffn1); }
    rs = new_rowstats();
    { GemmOp g = bld.lin(ls.ffn2, s_ff, Tn);
      g.flags = EPI_BIAS | EPI_RESIDUAL | EPI_OUT_F32; g.bias = w.W(b + ".ffn.ffn_2.bias"); g.res = XB; g.res_ld = H; g.out = XA; g.out_ld = H;
      masked(g); bld.emits_ln_input(g, s_ln, rs);
      bld.emit_gemm(g, ls.ffn2); }
    bld.emit_tap(taps, e.p + ".layers." + std::to_string(i), XA, Tn, H, Tn);
  }
  { GemmOp g = bld.lin(e.outp, s_ln, Tn);
    g.flags = EPI_OUT_F32; g.out = OUTP; g.out_ld = e.cout;
    bld.consumes_ln(g, rs, e.g_out, e.bf_out, H);
    bld.emit_gemm(g, e.outp); }
  bld.emit(Launch::LN_MASK, LnOp{OUTP, e.cout, (int)M, e.cout, 1e-5f, w.W(e.p + ".layer_norm.weight"), w.W(e.p + ".layer_norm.bias"), keep,
                                 nullptr, e.cout, SplitBuf{}}, io.out);
}

// `ragged`: row b is the utterance c[b, :, :T_b], refer[b, :, :S_b] encoded alone (ns2vc_pre_infer_ragged).  Besides the masked
// LN2 splits, ref_enc pools over each entry's 1 + S_b tokens; the prompt encoder runs first so that its SEQMASK launch writes the
// int prompt lengths ref_enc reads.  Same launches as the padded program.
// The two halves of the ragged program, each the same launches as its part of it:
//   T = 0: the voice program (ns2vc_pre_encode_voices_ragged): prompt encoder, ref_enc and spk_proj, which writes the call's SPK;
//   S = 0: the content program (ns2vc_pre_infer_content_ragged): the phone encoder, whose input adds the call's SPK rows.
// Each half zeroes its own LayerNorm statistics, so their launch counts add up to the ragged program's plus one memset.
int finish_program(ns2vc_pre* h, const ProgramBuilder& bld, std::vector<Launch> prog, TapSet taps, size_t* bytes_out) {
  if (bld.err) return bld.err;
  if (bytes_out) *bytes_out = bld.ar.off + 256;
  if (!bld.dry) {
    h->cp.prog = std::move(prog);
    h->cp.taps = std::move(taps);
  }
  return 0;
}

int build_program(ns2vc_pre* h, int B, int T, int S, bool ragged, void* ws, size_t* bytes_out) {
  const ns2vc_pre_cfg& c = h->cfg;
  const bool dry = ws == nullptr;
  NS_REQUIRE(B >= 1 && T >= 0 && S >= 0 && T + S >= 1 && (ragged || (T >= 1 && S >= 1)), "bad shape B=%d T=%d S=%d", B, T, S);
  std::vector<Launch> prog;
  TapSet taps;
  ProgramBuilder bld{Arena{(uint8_t*)ws, 0}, B, dry, h->simt, &prog};
  Arena& ar = bld.ar;
  // LayerNorm row sums (double [rows][2] per folded LayerNorm), zeroed by the program's only memset
  const size_t stat_doubles = (size_t)2 * B * ((size_t)T * (c.phone_layers + 1) + (size_t)S * (c.prompt_layers + 1));
  double* stat_arena = ar.get<double>(stat_doubles);
  double* stat_cur = stat_arena;
  bld.emit_memset(stat_arena, stat_doubles * sizeof(double));
  if (S == 0) {
    build_encoder(h, bld, taps, h->phone, T, {Launch::LENGTHS, Launch::C, Launch::CONTENT_OUT, Launch::SPK}, nullptr, stat_cur, true, nullptr);
    return finish_program(h, bld, std::move(prog), std::move(taps), bytes_out);
  }
  int* plens = ragged ? ar.get<int>(B) : nullptr;
  if (ragged) build_encoder(h, bld, taps, h->prompt, S, {Launch::REFER_LENGTHS, Launch::REFER, Launch::PROMPT_OUT}, nullptr, stat_cur, true, plens);
  // ---- ref_enc: TextTimeEmbedding over ALL S prompt frames (the reference does not mask them: model.py:362), or S_b when ragged
  const int R = c.ref_dim;
  float* rt = ar.get<float>((size_t)B * S * R);
  TextTimeEmbedding tte;
  tte.reserve(ar, B, S, R, R);
  float* g = ar.get<float>((size_t)B * R);
  float* spk = ar.get<float>((size_t)B * c.phone_hidden);
  bld.emit(Launch::NCT2TOK, TokensOp{nullptr, 0, B, R, S, rt, R, nullptr, nullptr}, Launch::REFER);
  tte.emit(bld, h->weights, "ref_enc", rt, Launch::NONE, S, R, R, c.ref_heads, Launch::POOL_ATT_WIDE, h->ref_kv, g, plens);
  bld.emit_tap(taps, "ref_enc", g, 1, R, 1);
  // spk_proj: Conv1d(100, hidden, 1) on g [B, 100, 1] (model.py:123, 127)
  bld.emit_linear(linear_op(g, R, B, R, h->weights.W("phoneme_encoder.spk_proj.weight"), h->weights.W("phoneme_encoder.spk_proj.bias"),
                            c.phone_hidden, spk, c.phone_hidden), T == 0 ? Launch::SPK : Launch::NONE);
  if (!ragged) build_encoder(h, bld, taps, h->prompt, S, {Launch::REFER_LENGTHS, Launch::REFER, Launch::PROMPT_OUT}, nullptr, stat_cur, false, nullptr);
  if (T > 0) build_encoder(h, bld, taps, h->phone, T, {Launch::LENGTHS, Launch::C, Launch::CONTENT_OUT}, spk, stat_cur, ragged, nullptr);
  return finish_program(h, bld, std::move(prog), std::move(taps), bytes_out);
}

int run_program(ns2vc_pre* h, const float* c, const float* refer, const long long* lengths, const long long* refer_lengths, float* content,
                float* prompt, float* spk, cudaStream_t st) {
  const int T = h->cp.dims[1], S = h->cp.dims[2];
  CallArgs in{};
  in[Launch::C] = {c, (long long)h->cfg.phone_in * T};
  in[Launch::REFER] = {refer, (long long)h->cfg.prompt_in * S};
  in[Launch::LENGTHS] = {lengths}; in[Launch::REFER_LENGTHS] = {refer_lengths};
  in[Launch::CONTENT_OUT] = {content}; in[Launch::PROMPT_OUT] = {prompt}; in[Launch::SPK] = {spk};
  return run_cached(h, h->simt, in, st, no_launcher);
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

void ns2vc_pre_destroy(ns2vc_pre* h) { destroy_engine(h); }
int ns2vc_pre_num_weights(const ns2vc_pre* h) { return num_weights(h); }
int ns2vc_pre_weight_info(const ns2vc_pre* h, int i, const char** name, int64_t shape[4], int* ndim) { return weight_info(h, i, name, shape, ndim); }
int ns2vc_pre_load_weight(ns2vc_pre* h, const char* key, const float* dptr, const int64_t* shape, int ndim, ns2vc_stream stream) {
  return load_weight(h, key, dptr, shape, ndim, (cudaStream_t)stream);
}
int ns2vc_pre_finalize(ns2vc_pre* h, ns2vc_stream stream) { return finalize_engine(h, [&] { return pack(h, (cudaStream_t)stream); }); }

int ns2vc_pre_workspace_bytes(const ns2vc_pre* h, int B, int T, int S, size_t* bytes) {
  NS_REQUIRE(h && bytes, "null argument");
  NS_REQUIRE(h->finalized, "ns2vc_pre_finalize() has not been called");
  // one workspace serves every program of a shape: the padded and ragged ones, the voice program of (B, S) and the content
  // program of (B, T)
  size_t need[4] = {0, 0, 0, 0};
  ns2vc_pre* hm = const_cast<ns2vc_pre*>(h);
  int rc = build_program(hm, B, T, S, false, nullptr, &need[0]);
  if (!rc) rc = build_program(hm, B, T, S, true, nullptr, &need[1]);
  if (!rc) rc = build_program(hm, B, 0, S, true, nullptr, &need[2]);
  if (!rc) rc = build_program(hm, B, T, 0, true, nullptr, &need[3]);
  if (!rc) *bytes = *std::max_element(need, need + 4);
  return rc;
}

}  // extern "C"

namespace {
// T = 0 / S = 0: the voice / content program (build_program), cached under that shape like the others
int infer(ns2vc_pre* h, const float* c, const float* refer, const int64_t* lengths, const int64_t* refer_lengths, float* content, float* prompt,
          float* spk, int B, int T, int S, void* ws, bool ragged, cudaStream_t st) {
  const int rc = ensure_program(h, "ns2vc_pre", B, T, S, ragged, ws, [&] { return build_program(h, B, T, S, ragged, ws, nullptr); });
  if (rc) return rc;
  return run_program(h, c, refer, reinterpret_cast<const long long*>(lengths), reinterpret_cast<const long long*>(refer_lengths), content,
                     prompt, spk, st);
}
}  // namespace

extern "C" {

int ns2vc_pre_infer(ns2vc_pre* h, const float* c, const float* refer, const int64_t* lengths, const int64_t* refer_lengths, float* content,
                    float* prompt, int B, int T, int S, void* ws, ns2vc_stream stream) {
  NS_REQUIRE(h && c && refer && lengths && refer_lengths && content && prompt, "null argument");
  NS_REQUIRE(T >= 1 && S >= 1, "bad shape B=%d T=%d S=%d", B, T, S);
  return infer(h, c, refer, lengths, refer_lengths, content, prompt, nullptr, B, T, S, ws, false, (cudaStream_t)stream);
}

int ns2vc_pre_infer_ragged(ns2vc_pre* h, const float* c, const float* refer, const int64_t* lengths, const int64_t* refer_lengths, float* content,
                           float* prompt, int B, int T, int S, void* ws, ns2vc_stream stream) {
  NS_REQUIRE(h && c && refer && lengths && refer_lengths && content && prompt, "null argument");
  NS_REQUIRE(T >= 1 && S >= 1, "bad shape B=%d T=%d S=%d", B, T, S);
  return infer(h, c, refer, lengths, refer_lengths, content, prompt, nullptr, B, T, S, ws, true, (cudaStream_t)stream);
}

int ns2vc_pre_encode_voices_ragged(ns2vc_pre* h, const float* refer, const int64_t* refer_lengths, float* spk, float* prompt, int B, int S,
                                   void* ws, ns2vc_stream stream) {
  NS_REQUIRE(h && refer && refer_lengths && spk && prompt, "null argument");
  NS_REQUIRE(S >= 1, "bad shape B=%d S=%d", B, S);
  return infer(h, nullptr, refer, nullptr, refer_lengths, nullptr, prompt, spk, B, 0, S, ws, true, (cudaStream_t)stream);
}

int ns2vc_pre_infer_content_ragged(ns2vc_pre* h, const float* c, const int64_t* lengths, const float* spk, float* content, int B, int T,
                                   void* ws, ns2vc_stream stream) {
  NS_REQUIRE(h && c && lengths && spk && content, "null argument");
  NS_REQUIRE(T >= 1, "bad shape B=%d T=%d", B, T);
  return infer(h, c, nullptr, lengths, nullptr, content, nullptr, const_cast<float*>(spk), B, T, 0, ws, true, (cudaStream_t)stream);
}

int ns2vc_pre_num_taps(const ns2vc_pre* h) { return num_taps(h); }
int ns2vc_pre_tap_info(const ns2vc_pre* h, int i, const char** name, int* rows, int* channels) { return tap_info(h, i, name, rows, channels); }
int ns2vc_pre_set_tap(ns2vc_pre* h, int i, float* dst) { return set_tap(h, i, dst); }
int ns2vc_pre_launch_count(const ns2vc_pre* h) { return launch_count(h); }

}  // extern "C"
