// Host-side machinery shared by the engines (engine.cu: the denoiser, pre_engine.cu: the condition encoders, vocoder.cu: the
// vocoder, content.cu: the content encoder): the weight registry, owned device memory and weight packing, the launch record,
// the program-builder base, the runner of the launch kinds the engines share, the taps, the TextTimeEmbedding of the first
// two, and the handle lifecycle (load, finalize, destroy; the cached program and counted run of the single-program engines).
#pragma once
#include "common.cuh"

#include <algorithm>
#include <array>
#include <cstring>
#include <string>
#include <unordered_map>
#include <variant>
#include <vector>

namespace ns2vc {

struct PackedB {
  __nv_bfloat16* hi = nullptr;
  __nv_bfloat16* lo = nullptr;
  float* f32 = nullptr;
  int Npad = 0, nkb = 0, n_logical = 0;
};

inline int pad_to(int v, int m) { return (v + m - 1) / m * m; }
inline int nkb_of(int c) { return (c + 63) / 64; }

// Bump allocator over the caller's workspace (or a dry run when base == nullptr).  A row view (rows > 1) replays the
// allocations of a build at B = rows from a build at B = 1: each request of n elements reserves n * rows, as the B = rows
// build did, and returns the start of row `row` of that [rows, n] buffer.
struct Arena {
  uint8_t* base = nullptr;
  size_t off = 0;
  size_t rows = 1, row = 0;
  template <class T> T* get(size_t n) {
    off = (off + 255) & ~(size_t)255;
    T* p = base ? reinterpret_cast<T*>(base + off) + row * n : nullptr;
    off += n * rows * sizeof(T);
    return p;
  }
};

// The reference state_dict: keys and shapes in registration order (the order the C-ABI lists them), each with an owned fp32 copy.
struct WeightRegistry {
  struct Slot {
    std::string name;
    std::vector<int64_t> shape;
    float* d = nullptr;
    bool loaded = false;
    size_t numel() const { size_t n = 1; for (auto s : shape) n *= (size_t)s; return n; }
  };
  std::vector<Slot> slots;
  std::unordered_map<std::string, int> index;

  void add(const std::string& n, std::vector<int64_t> shape) {
    index[n] = (int)slots.size();
    Slot s; s.name = n; s.shape = std::move(shape);
    slots.push_back(std::move(s));
  }
  void add_conv(const std::string& p, int co, int ci, int k) { add(p + ".weight", {co, ci, k}); add(p + ".bias", {co}); }
  void add_lin(const std::string& p, int co, int ci, bool bias = true) { add(p + ".weight", {co, ci}); if (bias) add(p + ".bias", {co}); }
  void add_norm(const std::string& p, int c) { add(p + ".weight", {c}); add(p + ".bias", {c}); }

  const float* W(const std::string& n) const {
    auto it = index.find(n);
    return it == index.end() ? nullptr : slots[it->second].d;
  }
  int size() const { return (int)slots.size(); }

  int load(const char* key, const float* dptr, const int64_t* shape, int ndim, cudaStream_t st) {
    auto it = index.find(key);
    NS_REQUIRE(it != index.end(), "Unexpected key in state_dict: %s", key);
    Slot& w = slots[it->second];
    NS_REQUIRE(ndim == (int)w.shape.size(), "size mismatch for %s: expected %d dims, got %d", key, (int)w.shape.size(), ndim);
    for (int k = 0; k < ndim; ++k) NS_REQUIRE(shape[k] == w.shape[k], "size mismatch for %s at dim %d: expected %lld, got %lld", key, k, (long long)w.shape[k], (long long)shape[k]);
    if (!w.d) NS_CHECK_CUDA(cudaMalloc(&w.d, w.numel() * sizeof(float)));
    NS_CHECK_CUDA(cudaMemcpyAsync(w.d, dptr, w.numel() * sizeof(float), cudaMemcpyDeviceToDevice, st));
    w.loaded = true;
    return 0;
  }
  int info(int i, const char** name, int64_t shape[4], int* ndim) const {
    NS_REQUIRE(i >= 0 && i < size(), "weight index %d out of range", i);
    const Slot& w = slots[i];
    if (name) *name = w.name.c_str();
    if (ndim) *ndim = (int)w.shape.size();
    if (shape) for (size_t k = 0; k < w.shape.size() && k < 4; ++k) shape[k] = w.shape[k];
    return 0;
  }
  int require_all_loaded() const {
    for (auto& w : slots) NS_REQUIRE(w.loaded, "Missing key in state_dict: %s", w.name.c_str());
    return 0;
  }
  void release() {
    for (auto& w : slots) if (w.d) { cudaFree(w.d); w.d = nullptr; }
  }
};

// Device memory owned by the packed model (freed together when the weights are re-packed or the handle is destroyed).
struct DeviceMem {
  std::vector<void*> ptrs;
  // nullptr on failure (the error is set)
  template <class T> T* alloc(size_t n, bool zero = false) {
    void* q = nullptr;
    cudaError_t e = cudaMalloc(&q, std::max<size_t>(n, 1) * sizeof(T));
    if (e == cudaSuccess && zero) {
      e = cudaMemset(q, 0, std::max<size_t>(n, 1) * sizeof(T));
      if (e != cudaSuccess) cudaFree(q);
    }
    if (e != cudaSuccess) { set_error("device allocation of %zu bytes failed: %s", n * sizeof(T), cudaGetErrorString(e)); return nullptr; }
    ptrs.push_back(q);
    return reinterpret_cast<T*>(q);
  }
  // n_logical output columns of which the first n_packed (padded to 128) are stored, nkb 64-channel k-blocks
  int alloc_packed(PackedB& pb, int n_logical, int n_packed, int nkb, bool with_f32) {
    pb.n_logical = n_logical;
    pb.Npad = pad_to(n_packed, 128);
    pb.nkb = nkb;
    const size_t elems = (size_t)nkb * pb.Npad * 64;
    if (!(pb.hi = alloc<__nv_bfloat16>(elems, true)) || !(pb.lo = alloc<__nv_bfloat16>(elems, true))) return -2;
    if (with_f32 && !(pb.f32 = alloc<float>(elems, true))) return -2;
    return 0;
  }
  void release() {
    for (void* p : ptrs) cudaFree(p);
    ptrs.clear();
  }
};

// Pack `w` ([n_rows, cin_total, ktaps] fp32, device) channels [cin0, cin0+ncin) of tap `tap` at k-block kb0, columns n_dst0..
inline int pack_seg(PackedB& pb, const float* w, int n_rows, int cin_total, int ktaps, int tap, int cin0, int ncin, int n_dst0,
                    int kb0, int geglu_half, cudaStream_t st, const float* cscale = nullptr) {
  PackSeg ps;
  ps.cscale = cscale;
  ps.w = w; ps.n_rows = n_rows; ps.cin_total = cin_total; ps.ktaps = ktaps; ps.tap = tap; ps.cin0 = cin0; ps.ncin = ncin;
  ps.n_dst0 = n_dst0; ps.kb0 = kb0; ps.nkb = nkb_of(ncin); ps.geglu_half = geglu_half;
  return launch_pack_b(ps, pb.hi, pb.lo, pb.f32, pb.Npad, st);
}

// AttentionPooling's k_proj | v_proj as one [2R, R] operator (and its [2R] bias): one small linear over every token
struct PoolKV { float* W = nullptr; float* b = nullptr; };
inline int concat_pool_kv(DeviceMem& mem, const WeightRegistry& w, const std::string& pool, int R, PoolKV& kv, cudaStream_t st) {
  if (!(kv.W = mem.alloc<float>((size_t)2 * R * R)) || !(kv.b = mem.alloc<float>((size_t)2 * R))) return -2;
  NS_CHECK_CUDA(cudaMemcpyAsync(kv.W, w.W(pool + ".k_proj.weight"), (size_t)R * R * 4, cudaMemcpyDeviceToDevice, st));
  NS_CHECK_CUDA(cudaMemcpyAsync(kv.W + (size_t)R * R, w.W(pool + ".v_proj.weight"), (size_t)R * R * 4, cudaMemcpyDeviceToDevice, st));
  NS_CHECK_CUDA(cudaMemcpyAsync(kv.b, w.W(pool + ".k_proj.bias"), (size_t)R * 4, cudaMemcpyDeviceToDevice, st));
  NS_CHECK_CUDA(cudaMemcpyAsync(kv.b + R, w.W(pool + ".v_proj.bias"), (size_t)R * 4, cudaMemcpyDeviceToDevice, st));
  return 0;
}

// The arguments of the launch kinds that run without a launcher of common.cuh: two copies, and the kernels private to
// vocoder.cu and content.cu (whose hooks pass them the call arguments they read)
struct MemsetOp { void* p; size_t bytes; };
struct CopyOp { const float* src; size_t bytes; float* dst; };   // TAP: dst is the tap's buffer (TapSet); COPY: the call's output
struct VocLensOp { int B, T; int* lens; float* keep; };          // lengths -> lens [B] and keep [B, T]
struct IstftOp { const float* h; int ld, B, T; };                // head output [B, T, ld] -> audio
struct CvLensOp { int B, N; };                                   // lengths -> the content encoder's length tables
struct CvGnStatsOp { int B, N, C0; const float* w0; float eps; float2* stats; };
struct CvConv0Op { int B, N, rows; const float* w0; const float2* stats; const float* gamma; const float* beta; SplitBuf out; };
struct CvPosWinOp { const float* x; int B, T, D, G, gw, K; const long long* frames; SplitBuf win; };
struct CvAddOp { float* p; const float* x; long long n4; };     // p += x over n4 float4
struct SplitTapOp { SplitBuf s; int B, rows, T, C; };            // tap of a split [B, rows, s.ld]: its first T rows, C channels

// One launch of a per-shape program: its kind and that kind's arguments.
struct Launch {
  // The denoiser's kinds keep their numbers: ns2vc_unet_launch_kind() and ns2vc_profile_kind_name() expose them.  The
  // condition encoders' own kinds follow TAP, then the vocoder's, then the content encoder's.
  enum Kind { GEMM, ATTN, LN_SPLIT, LN_APPLY, LINEAR, NCT2SPLIT, POOL_CLS, POOL_ATT, MASKBIAS, PREP, MEMSET, TAP,
              SEQMASK, ENC_INPUT, LN_MASK, NCT2TOK, POOL_ATT_WIDE,
              VOC_LENS, VOC_NORM, VOC_ISTFT,
              COPY, CV_LENS, CV_GN_STATS, CV_CONV0, CV_POS_WIN, CV_ADD, CV_SPLIT_TAP } kind = GEMM;
  // The call argument a launch reads or writes instead of a program buffer (bind_input puts it into the payload)
  enum Input { NONE,
               X, T, OUT, CONTENT, PROMPT, MASK,                               // ns2vc_unet_prepare_cond / _forward
               C, REFER, LENGTHS, REFER_LENGTHS, CONTENT_OUT, PROMPT_OUT,      // ns2vc_pre_infer
               SPK,                                                           // ns2vc_pre_encode_voices_ragged / _infer_content_ragged
               MEL,                                                           // ns2vc_voc_decode (+ LENGTHS)
               NUM_INPUTS                                                     // (ns2vc_cv_extract: OUT)
  } input = NONE;
  Input input2 = NONE;       // a second call argument (the condition encoders' content program: ENC_INPUT's speaker rows, SPK)
  std::variant<std::monostate, GemmOp, AttnOp, LnOp, LinOp, NctSplitOp, TokensOp, PoolClsOp, PoolAttOp, MaskBiasOp, PrepOp, SeqMaskOp,
               VocNormOp, MemsetOp, CopyOp, VocLensOp, IstftOp, CvLensOp, CvGnStatsOp, CvConv0Op, CvPosWinOp, CvAddOp, SplitTapOp> op;
  int tap_index = -1;
  int reads_film = 0;        // denoiser: reads the FiLM rows (pointers are rebased when the caller supplies precomputed rows)
  int time_path = 0;         // denoiser: timestep path (sinusoid -> MLP -> FiLM rows): skipped when the caller supplies precomputed FiLM rows
  template <class Op> Op& get() { return std::get<Op>(op); }
  template <class Op> const Op& get() const { return std::get<Op>(op); }
};

// A call argument: its pointer and (the [B, C, T] inputs) its batch stride in elements.  Each C entry point fills the table of
// the arguments its programs read.
struct CallArg { const void* p = nullptr; long long bstride = 0; };
using CallArgs = std::array<CallArg, Launch::NUM_INPUTS>;

// Puts the call argument `a` (the one named `which`) into the field of l's payload that reads it.
inline int bind_input(Launch& l, Launch::Input which, const CallArg& a) {
  float* p = (float*)a.p;
  if (which == Launch::SPK) {     // the speaker rows [B, phone_hidden]: written by spk_proj, or added to the content encoder's input
    if (l.kind == Launch::LINEAR) { l.get<LinOp>().out = p; return 0; }
    if (l.kind == Launch::ENC_INPUT) { l.get<TokensOp>().rowbias = p; return 0; }
    set_error("internal: launch kind %d reads no speaker rows", (int)l.kind); return -1;
  }
  switch (l.kind) {
    case Launch::GEMM: l.get<GemmOp>().out = p; return 0;
    case Launch::ATTN: return 0;   // MASK: the denoiser drops the key-padding bias when its prepare_cond had no mask
    case Launch::LN_APPLY: l.get<LnOp>().x = p; return 0;
    case Launch::LN_MASK: l.get<LnOp>().y = p; return 0;
    case Launch::LINEAR: l.get<LinOp>().x = p; return 0;
    case Launch::PREP: l.get<PrepOp>().src1 = p; return 0;
    case Launch::NCT2SPLIT: { NctSplitOp& o = l.get<NctSplitOp>(); o.x = p; o.bstride = a.bstride; return 0; }
    case Launch::ENC_INPUT: case Launch::NCT2TOK: { TokensOp& o = l.get<TokensOp>(); o.x = p; o.bstride = a.bstride; return 0; }
    case Launch::MASKBIAS: l.get<MaskBiasOp>().mask = (const uint8_t*)a.p; return 0;
    case Launch::SEQMASK: l.get<SeqMaskOp>().len = (const long long*)a.p; return 0;
    case Launch::VOC_NORM: l.get<VocNormOp>().len = (const long long*)a.p; return 0;
    case Launch::COPY: l.get<CopyOp>().dst = p; return 0;
    default: set_error("internal: launch kind %d reads no call argument", (int)l.kind); return -1;
  }
}

// Named activations a program can copy out after the launch that produced them (diagnostics: per-layer parity tests).
struct TapSet {
  std::vector<std::string> names;
  std::vector<int> rows, ch;   // rows: the level (denoiser) or the row count per batch entry (condition encoders)
  std::vector<float*> dst;
  int add(const std::string& name, int r, int c) {
    names.push_back(name); rows.push_back(r); ch.push_back(c); dst.push_back(nullptr);
    return (int)names.size() - 1;
  }
  int size() const { return (int)names.size(); }
  int info(int i, const char** name, int* r, int* c) const {
    NS_REQUIRE(i >= 0 && i < size(), "tap index %d out of range", i);
    if (name) *name = names[i].c_str();
    if (r) *r = rows[i];
    if (c) *c = ch[i];
    return 0;
  }
  int set(int i, float* p) {
    NS_REQUIRE(i >= 0 && i < size(), "tap index %d out of range", i);
    dst[i] = p;
    return 0;
  }
  int copy(const Launch& l, cudaStream_t st) const {
    if (l.tap_index >= 0 && l.tap_index < size() && dst[l.tap_index]) {
      const CopyOp& c = l.get<CopyOp>();
      cudaError_t e = cudaMemcpyAsync(dst[l.tap_index], c.src, c.bytes, cudaMemcpyDeviceToDevice, st);
      if (e != cudaSuccess) { set_error("tap copy failed: %s", cudaGetErrorString(e)); return -2; }
    }
    return 0;
  }
};

// Builds a launch program over a workspace arena (a dry run sizes the workspace: no device work, no tensor maps).
struct ProgramBuilder {
  Arena ar;
  int B;
  bool dry;
  bool simt;
  std::vector<Launch>* out;
  int err = 0;

  SplitBuf split(int Tn, int C) {
    SplitBuf s{}; s.T = Tn; s.C = C; s.ld = pad_to(C, 8);
    s.hi = ar.get<__nv_bfloat16>((size_t)B * Tn * s.ld);
    s.lo = ar.get<__nv_bfloat16>((size_t)B * Tn * s.ld);
    return s;
  }
  // view of a (larger) scratch split as [B, Tn, C]
  static SplitBuf view(const SplitBuf& base, int Tn, int C) {
    SplitBuf s = base; s.T = Tn; s.C = C; s.ld = pad_to(C, 8); return s;
  }
  GemmOp gemm_base(const PackedB& w, int T_out) {
    GemmOp g; memset(&g, 0, sizeof(g));
    g.B = B; g.T_out = T_out;
    g.w_hi = w.hi; g.w_lo = w.lo; g.w_f32 = w.f32; g.N = w.Npad; g.n_valid = w.n_logical;
    g.f16_col0 = 0x7fffffff;
    g.ksplit = 1;
    return g;
  }
  int add_src(GemmOp& g, const SplitBuf& s) { g.src[g.nsrc] = s; return g.nsrc++; }
  void seg(GemmOp& g, int src, int c0, int nch, int tap) {
    GSeg& s = g.seg[g.nseg++];
    s.src = src; s.c0 = c0; s.nkb = nkb_of(nch); s.tap = tap;
    g.nkb_total += s.nkb;
  }
  // ---- panel mode (GemmOp::xmode): raw split sources normalised inside the GEMM
  void xseg(GemmOp& g, int src, int c0, int nch, int ntap, int kb0, int kb_stride, int xf, int aff_c0) {
    XSeg& x = g.xs[g.nxs++];
    x.src = src; x.c0 = c0; x.ncb = nkb_of(nch); x.ntap = ntap; x.xf = xf; x.aff_c0 = aff_c0;
    for (int j = 0; j < 3; ++j) x.kb_tap[j] = kb0 + j * kb_stride;
    g.nkb_total += x.ncb * ntap;
    g.xmode = 1;
  }
  // a linear layer: one unshifted segment over all channels of `in`
  GemmOp lin(const PackedB& w, const SplitBuf& in, int T_out) {
    GemmOp g = gemm_base(w, T_out);
    seg(g, add_src(g, in), 0, in.C, 0);
    return g;
  }
  // ---- LayerNorm (eps 1e-5) folded into its consumer GEMM (EPI_LNFOLD):
  //   LN(x) W^T = rstd * (x (gamma*W)^T - mean * g) + (beta W^T + bias),   g[n] = sum_c gamma_c W[n,c]
  // The producer of x also writes its raw split `s` and the per-row sums `rs`; the consumer runs on `s` with gamma packed into
  // its weights and applies mean / rstd over the C channels with the load-time vectors `gv` = g and `bf` = beta W^T + bias.
  static void emits_ln_input(GemmOp& g, const SplitBuf& s, double* rs) {
    g.flags |= EPI_OUT_SPLIT | EPI_ROWSTATS; g.out_hi = s.hi; g.out_lo = s.lo; g.out_split_ld = s.ld; g.row_stats = rs;
  }
  static void consumes_ln(GemmOp& g, const double* rs, const float* gv, const float* bf, int C) {
    g.flags |= EPI_LNFOLD | EPI_BIAS; g.ln_stats = rs; g.ln_g = gv; g.bias = bf; g.ln_C = C; g.ln_eps = 1e-5f;
  }
  template <class Op> Launch& emit(Launch::Kind kind, const Op& op, Launch::Input in = Launch::NONE) {
    Launch l; l.kind = kind; l.input = in; l.op = op;
    out->push_back(l);
    return out->back();
  }
  Launch& emit_gemm(GemmOp& g, const PackedB& w, Launch::Input in = Launch::NONE) {
    if (!dry) {
      if (g.nkb_total != w.nkb) { set_error("internal: K mismatch %d vs %d", g.nkb_total, w.nkb); err = -1; }
      plan_gemm(g);
      if (!simt) { const int rc = encode_tmaps(g); if (rc) err = rc; }
    }
    return emit(Launch::GEMM, g, in);
  }
  void emit_attention(const AttnOp& a, Launch::Input in = Launch::NONE) {
    AttnOp& op = emit(Launch::ATTN, a, in).get<AttnOp>();
    if (a.v2 && !dry) { const int rc = encode_attn_tmaps(op); if (rc) err = rc; }
  }
  // LayerNorm (eps 1e-5) of M rows of C channels at pitch ld; `keep`: rows whose factor is 0 are stored as zeros, or nullptr
  void emit_ln_split(const float* x, int ld, int M, int C, const float* gamma, const float* beta, const SplitBuf& o, const float* keep = nullptr) {
    LnOp op{x, ld, M, C, 1e-5f, gamma, beta, keep, nullptr, 0, o};
    emit(Launch::LN_SPLIT, op);
  }
  void emit_ln_apply(const float* x, Launch::Input in, int M, int C, const float* gamma, const float* beta, float* y) {
    LnOp op{x, C, M, C, 1e-5f, gamma, beta, nullptr, y, C, SplitBuf{}};
    emit(Launch::LN_APPLY, op, in);
  }
  void emit_linear(const LinOp& o, Launch::Input in = Launch::NONE, int time_path = 0) {
    emit(Launch::LINEAR, o, in).time_path = time_path;
  }
  void emit_memset(void* p, size_t bytes) { emit(Launch::MEMSET, MemsetOp{p, bytes}); }
  // copy-out point of a named activation ([B, rows, C] fp32): only in real programs, whose taps can be read
  void emit_tap(TapSet& taps, const std::string& name, const float* src, int tap_rows, int C, int rows) {
    if (dry) return;
    emit(Launch::TAP, CopyOp{src, (size_t)B * rows * C * sizeof(float), nullptr}).tap_index = taps.add(name, tap_rows, C);
  }
};

// The GroupNorm part of a prep descriptor over Tn rows of B entries: statistics of up to two concatenated producers (st1 / st2:
// [B, C] sums | [B, C] sums of squares, as the producers' EPI_STATS epilogues lay them out; st2 nullptr without a concat), the
// norm's weights, the FiLM rows (nullptr: none; the panel-mode GEMM passes its own as GemmOp::pre_film) and the group count.
// The engines and the kernel checks fill every GroupNorm descriptor through this.
inline void set_group_norm(PrepOp& p, int B, const double* st1, int C1, const double* st2, int C2, int Tn, int G, float eps,
                           const float* gamma, const float* beta, const float* film, int film_ld) {
  p.gn.sum1 = st1; p.gn.sq1 = st1 ? st1 + (size_t)B * C1 : nullptr;
  p.gn.sum2 = st2; p.gn.sq2 = st2 ? st2 + (size_t)B * C2 : nullptr;
  p.gn.gamma = gamma; p.gn.beta = beta; p.gn.film = film; p.gn.film_ld = film_ld; p.gn.G = G; p.gn.eps = eps;
  p.gn.inv_n = 1.0 / ((double)Tn * ((C1 + C2) / G));
}

// The denoiser's Downsample1D (engine.cu), shared by its emit_down and the kernel checks: conv k3 s2 p1 of a [B, Tin, C] input
// as one GEMM over its even rows E[t] = x[2t] and odd rows O[t] = x[2t+1] (bias included; the caller adds the outputs):
//   out[t] = W0 O[t-1] + W1 E[t] + W2 O[t],   t < ceil(Tin / 2)
// With `views` and Tin >= 2, E and O are views of the raw split `raw` [B, Tin, raw.ld] as row pairs (no copy, nprep = 0);
// otherwise the two prep launches prep[0..1] decimate the fp32 input x [B, Tin, C] into e_buf / o_buf first.  The weights are
// [C, C, 3] packed by pack_resample_conv (which packs Upsample1D's conv too).
struct DownConv { GemmOp g; PrepOp prep[2]; int nprep; };
int pack_resample_conv(PackedB& pb, const float* w, int C, cudaStream_t st);
DownConv down_conv(ProgramBuilder& bld, const PackedB& w, const float* bias, const float* x, const SplitBuf& raw, int Tin, int C,
                   bool views, const SplitBuf& e_buf, const SplitBuf& o_buf);

// The content encoder's launchers (content.cu), shared by its run_program and the kernel checks.  conv 0's two launches read the
// call's waveform (batch stride bstride) and lengths; convs 1-6 are one GEMM each (cv_conv_gemm over the weights pack_cv_conv
// packs); the positional conv is the windows, one GEMM per group (cv_pos_group_gemm over the weights pack_cv_pos_group packs),
// then the residual add.
int launch_cv_gn_stats(const CvGnStatsOp& o, const float* wav, long long bstride, const long long* lengths, cudaStream_t st);
int launch_cv_conv0(const CvConv0Op& o, const float* wav, long long bstride, const long long* lengths, cudaStream_t st);
int launch_cv_pos_windows(const CvPosWinOp& o, cudaStream_t st);
int launch_cv_add(const CvAddOp& o, cudaStream_t st);
int cv_conv_taps(int l);
int pack_cv_conv(PackedB& pb, const float* w, int C0, int l, cudaStream_t st);
GemmOp cv_conv_gemm(ProgramBuilder& bld, const PackedB& w, const SplitBuf& in, int rows_in, int rows_out, int l, const float* keep,
                    const SplitBuf& out_split, float* out);
int pack_cv_pos_group(PackedB& pb, const float* wg, int gw, int K, cudaStream_t st);
GemmOp cv_pos_group_gemm(ProgramBuilder& bld, const PackedB& w, const SplitBuf& win, int G, int g, int gw, int T, int K, const float* bias,
                         const float* keep, float* out, int out_ld);

// The vocoder's ISTFT (vocoder.cu): its tables, and the launch of one head output [B, T, ld] -> audio [B, T hop] with them
struct IstftTables {
  const float* window;      // [n_fft] head.istft.window as loaded
  const float2* tw_half;    // [M / 2] exp(+2 pi i j / M), M = n_fft / 2: the inverse complex FFT
  const float2* tw_full;    // [M / 2 + 1] exp(+2 pi i k / n_fft): the split step of the real inverse
};
void istft_twiddles(int n_fft, std::vector<float2>& tw_half, std::vector<float2>& tw_full);
int istft_log2m(int n_fft);
size_t istft_smem_bytes(int n_fft);
int launch_istft(const IstftTables& tb, const float* h, int ld, const long long* len, float* audio, int B, int T, int n_fft, int hop, int log2m,
                 size_t smem, cudaStream_t st);

inline LinOp linear_op(const float* x, int x_ld, int M, int K, const float* W, const float* bias, int N, float* y, int y_ld) {
  LinOp o; memset(&o, 0, sizeof(o));
  o.x = x; o.x_ld = x_ld; o.M = M; o.K = K; o.W = W; o.bias = bias; o.N = N; o.out = y; o.out_ld = y_ld;
  return o;
}

// TextTimeEmbedding (reference embeddings.py:421-434) over a token-major [B, S, R] input `x` (or the call argument `x_in`):
//   LayerNorm -> AttentionPooling (class token; q of the class token, k|v of every token as one [2R, R] operator) -> Linear
//   to E channels -> LayerNorm into `y` [B, E].
// The scratch buffers are placed by reserve() so that each engine keeps its own workspace layout.
struct TextTimeEmbedding {
  float* norm = nullptr; float* tok = nullptr; float* q = nullptr; float* kv = nullptr; float* pool = nullptr; float* proj = nullptr;
  void reserve(Arena& ar, int B, int S, int R, int E) {
    norm = ar.get<float>((size_t)B * S * R);
    tok = ar.get<float>((size_t)B * (S + 1) * R);
    q = ar.get<float>((size_t)B * R);
    kv = ar.get<float>((size_t)B * (S + 1) * 2 * R);
    pool = ar.get<float>((size_t)B * R);
    proj = ar.get<float>((size_t)B * E);
  }
  // `attend`: POOL_ATT (denoiser) or POOL_ATT_WIDE (condition encoders) - their sums run in different orders.
  // `lens`: per-entry prompt lengths [B] (the denoiser's ragged programs pool over each entry's own frames), or nullptr.
  void emit(ProgramBuilder& bld, const WeightRegistry& w, const std::string& p, const float* x, Launch::Input x_in, int S, int R,
            int E, int heads, Launch::Kind attend, const PoolKV& pkv, float* y, const int* lens = nullptr) const {
    const int B = bld.B;
    bld.emit_ln_apply(x, x_in, B * S, R, w.W(p + ".norm1.weight"), w.W(p + ".norm1.bias"), norm);
    bld.emit(Launch::POOL_CLS, PoolClsOp{norm, w.W(p + ".pool.positional_embedding"), B, S, R, tok, lens});
    bld.emit_linear(linear_op(tok, (S + 1) * R, B, R, w.W(p + ".pool.q_proj.weight"), w.W(p + ".pool.q_proj.bias"), R, q, R));
    bld.emit_linear(linear_op(tok, R, B * (S + 1), R, pkv.W, pkv.b, 2 * R, kv, 2 * R));
    bld.emit(attend, PoolAttOp{q, kv, B, S + 1, R, heads, pool, lens});
    bld.emit_linear(linear_op(pool, R, B, R, w.W(p + ".proj.weight"), w.W(p + ".proj.bias"), E, proj, E));
    bld.emit_ln_apply(proj, Launch::NONE, B, E, w.W(p + ".norm2.weight"), w.W(p + ".norm2.bias"), y);
  }
};

// Launches every kind whose launcher common.cuh declares, with the arguments of the record (bound, patched or as built);
// returns kEngineKind for the kinds an engine launches itself.
constexpr int kEngineKind = 1;
struct Runner {
  bool simt;
  const TapSet* taps;
  cudaStream_t st;

  int run(const Launch& l) const {
    switch (l.kind) {
      case Launch::GEMM: { const GemmOp& g = l.get<GemmOp>(); return simt ? launch_gemm_simt(g, st) : launch_gemm_tc(g, st); }
      case Launch::ATTN: { const AttnOp& a = l.get<AttnOp>(); return (a.v2 && !simt) ? launch_attention_v2(a, st) : launch_attention(a, st, simt); }
      case Launch::LN_SPLIT: return launch_ln_split(l.get<LnOp>(), st);
      case Launch::LN_APPLY: return launch_ln_apply(l.get<LnOp>(), st);
      case Launch::LN_MASK: return launch_ln_mask(l.get<LnOp>(), st);
      case Launch::LINEAR: return launch_small_linear(l.get<LinOp>(), st);
      case Launch::NCT2SPLIT: return launch_nct_to_split(l.get<NctSplitOp>(), st);
      case Launch::NCT2TOK: return launch_nct_to_tokens(l.get<TokensOp>(), st);
      case Launch::ENC_INPUT: return launch_enc_input(l.get<TokensOp>(), st);
      case Launch::POOL_CLS: return launch_pool_class_token(l.get<PoolClsOp>(), st);
      case Launch::POOL_ATT: return launch_pool_attend(l.get<PoolAttOp>(), st);
      case Launch::POOL_ATT_WIDE: return launch_pool_attend_wide(l.get<PoolAttOp>(), st);
      case Launch::MASKBIAS: return launch_mask_bias(l.get<MaskBiasOp>(), st);
      case Launch::PREP: return launch_prep_split(l.get<PrepOp>(), st);
      case Launch::SEQMASK: return launch_seq_mask(l.get<SeqMaskOp>(), st);
      case Launch::VOC_NORM: return launch_voc_norm(l.get<VocNormOp>(), st);
      case Launch::MEMSET: {
        const MemsetOp& m = l.get<MemsetOp>();
        const cudaError_t e = cudaMemsetAsync(m.p, 0, m.bytes, st);
        if (e != cudaSuccess) { set_error("memset failed: %s", cudaGetErrorString(e)); return -2; }
        return 0;
      }
      case Launch::COPY: {
        const CopyOp& c = l.get<CopyOp>();
        NS_CHECK_CUDA(cudaMemcpyAsync(c.dst, c.src, c.bytes, cudaMemcpyDeviceToDevice, st));
        return 0;
      }
      case Launch::TAP: return taps->copy(l, st);
      default: return kEngineKind;
    }
  }
};

inline int no_launcher(const Launch& l) {
  set_error("internal: launch kind %d has no launcher", (int)l.kind);
  return -1;
}

// The record to launch for `l`: `l` itself, or (when it reads a call argument) `tmp` holding a copy with the argument bound
inline const Launch* bound(const Launch& l, const CallArgs& in, Launch& tmp, int& rc) {
  rc = 0;
  if (l.input == Launch::NONE && l.input2 == Launch::NONE) return &l;
  tmp = l;
  if (l.input != Launch::NONE) rc = bind_input(tmp, l.input, in[l.input]);
  if (!rc && l.input2 != Launch::NONE) rc = bind_input(tmp, l.input2, in[l.input2]);
  return &tmp;
}

// The operands a packer built, in packing order: each under its site name, with the load-time vectors (folded LayerNorm
// vectors, merged biases and operators, concatenations) the launch programs read beside it.  Host bookkeeping only: the
// pointers are the engine's own device memory and stay valid until the next finalize.  The kernel checks read it back
// (ns2vc_check_packed), so that the tests can compare every packed image and fold with an fp64 fold of the state_dict.
struct PackedRecord {
  struct Vec { std::string name; const float* p; long long n; };
  struct Entry { std::string name; PackedB pb; std::vector<Vec> vecs; };   // pb.Npad == 0: vectors only
  std::vector<Entry> entries;
  void add(const std::string& name, const PackedB& pb, std::vector<Vec> vecs = {}) { entries.push_back(Entry{name, pb, std::move(vecs)}); }
};

// A test-only observer of the run loops (ns2vc_check_set_launch_hook): while `fn` is set, every launch of a run is preceded
// (phase 0) and followed (phase 1) by observe_launch(), which synchronises the stream and hands the record as launched (index:
// its position in the program) to the caller's function.  Unset, the loops do what they do without it.
struct LaunchHook { void* fn = nullptr; void* user = nullptr; };
int observe_launch(const LaunchHook& hook, int index, int phase, const Launch& l, cudaStream_t st);   // kernel_check.cu

// What every engine handle holds: the reference state_dict, the device memory of its packed weights and their record, whether
// the loaded weights are packed, the number of launches of its last run, and the launch observer.  Each handle also has a
// drop_programs() that forgets the launch programs built over the packed weights.
struct EngineBase {
  WeightRegistry weights;
  DeviceMem mem;
  PackedRecord packed;
  bool finalized = false;
  int last_launches = 0;
  LaunchHook hook;
};

// The C-ABI's <engine>_num_weights / _weight_info / _load_weight / _launch_count
inline int num_weights(const EngineBase* h) { return h ? h->weights.size() : -1; }
inline int weight_info(const EngineBase* h, int i, const char** name, int64_t shape[4], int* ndim) {
  NS_REQUIRE(h, "weight index %d out of range", i);
  return h->weights.info(i, name, shape, ndim);
}
inline int load_weight(EngineBase* h, const char* key, const float* dptr, const int64_t* shape, int ndim, cudaStream_t st) {
  NS_REQUIRE(h && key && dptr, "null argument");
  const int rc = h->weights.load(key, dptr, shape, ndim, st);
  if (rc) return rc;
  h->finalized = false;          // packed from the old values until the next finalize
  return 0;
}
inline int launch_count(const EngineBase* h) { return h ? h->last_launches : -1; }

// <engine>_finalize: (re)packs every loaded weight with the engine's `pack()`, after freeing the previous packing and the
// programs that point into it.
template <class Engine, class Pack> int finalize_engine(Engine* h, Pack pack) {
  NS_REQUIRE(h, "null handle");
  int rc = h->weights.require_all_loaded();
  if (rc) return rc;
  h->mem.release();
  h->packed.entries.clear();
  h->drop_programs();
  if ((rc = pack())) return rc;
  NS_CHECK_CUDA(cudaGetLastError());
  h->finalized = true;
  return 0;
}

// <engine>_destroy
template <class Engine> void destroy_engine(Engine* h) {
  if (!h) return;
  h->weights.release();
  h->mem.release();
  h->drop_programs();
  delete h;
}

// The launch program of the condition encoders, the vocoder and the content encoder: one per handle, for the last shape
// (B, and up to two more dims: T, S or N), ragged flag and workspace it ran with.
struct CachedProgram {
  int dims[3] = {0, 0, 0};
  bool ragged = false;
  void* ws = nullptr;
  std::vector<Launch> prog;
  TapSet taps;
};

struct SingleProgramEngine : EngineBase {
  CachedProgram cp;
  void drop_programs() { cp = CachedProgram(); }
};

// The C-ABI's <engine>_num_taps / _tap_info / _set_tap: the taps of the cached program
inline int num_taps(const SingleProgramEngine* h) { return h ? h->cp.taps.size() : -1; }
inline int tap_info(const SingleProgramEngine* h, int i, const char** name, int* rows, int* channels) {
  NS_REQUIRE(h, "tap index %d out of range", i);
  return h->cp.taps.info(i, name, rows, channels);
}
inline int set_tap(SingleProgramEngine* h, int i, float* dst) {
  NS_REQUIRE(h, "tap index %d out of range", i);
  return h->cp.taps.set(i, dst);
}

// Makes h->cp the program of (B, d1, d2, ragged, ws), calling `build()` (which fills cp.prog and cp.taps) unless it already is.
// `engine`: the C-ABI prefix named in the error of an unfinalized handle.
template <class Build> int ensure_program(SingleProgramEngine* h, const char* engine, int B, int d1, int d2, bool ragged, void* ws,
                                          Build build) {
  NS_REQUIRE(h->finalized, "%s_finalize() has not been called", engine);
  NS_REQUIRE(ws != nullptr, "workspace is NULL");
  CachedProgram& cp = h->cp;
  if (cp.dims[0] == B && cp.dims[1] == d1 && cp.dims[2] == d2 && cp.ragged == ragged && cp.ws == ws) return 0;
  const int rc = build();
  if (rc) return rc;
  cp.dims[0] = B; cp.dims[1] = d1; cp.dims[2] = d2; cp.ragged = ragged; cp.ws = ws;
  return 0;
}

// Runs h->cp over the call arguments `in` and records its launch count in h->last_launches.  `own(l)` launches the kinds
// Runner leaves to the engine.  Tap copies (the launches with a tap index) are not counted: they are diagnostics, not part of
// the computation.
template <class Own> int run_cached(SingleProgramEngine* h, bool simt, const CallArgs& in, cudaStream_t st, Own own) {
  const Runner run{simt, &h->cp.taps, st};
  Launch tmp;
  int count = 0, index = 0;
  for (const Launch& rec : h->cp.prog) {
    int rc;
    const Launch* l = bound(rec, in, tmp, rc);
    if (!rc && h->hook.fn) rc = observe_launch(h->hook, index, 0, *l, st);
    if (!rc) rc = run.run(*l);
    if (rc == kEngineKind) rc = own(*l);
    if (!rc && h->hook.fn) rc = observe_launch(h->hook, index, 1, *l, st);
    ++index;
    if (rc) return rc;
    if (rec.tap_index < 0) ++count;
  }
  h->last_launches = count;
  return 0;
}

}  // namespace ns2vc

struct ns2vc_unet; struct ns2vc_pre; struct ns2vc_cv; struct ns2vc_voc;

namespace ns2vc {
// The EngineBase of each handle type, defined beside the type (kernel_check.cu sees the handles as opaque)
const EngineBase* engine_base(const ns2vc_unet* h);
const EngineBase* engine_base(const ns2vc_pre* h);
const EngineBase* engine_base(const ns2vc_cv* h);
const EngineBase* engine_base(const ns2vc_voc* h);
}  // namespace ns2vc
