// Test-only entry points into the product launchers: one weight packing, one wgmma GEMM, one flash attention, one activation
// prep, one LayerNorm, one small linear, the AttentionPooling pieces, one [B, C, T] -> split conversion, the content encoder's
// first conv, strided convs 1-6 and positional conv, the denoiser's Downsample1D conv, and the vocoder's ISTFT, each described
// by a flat C struct (include/ns2vc_b200.h, "kernel checks") and run through exactly the host code the engines use (pack_seg,
// the ProgramBuilder helpers, set_group_norm, linear_op, down_conv / pack_resample_conv, cv_conv_gemm / pack_cv_conv,
// plan_gemm / encode_tmaps / launch_gemm_tc, encode_attn_tmaps / the attention dispatch, the launchers of common.cuh and
// engine_host.cuh).  tests/test_kernels_fp64.py, tests/test_norm_kernels_fp64.py, tests/test_audio_kernels_fp64.py and
// tests/test_strided_conv_fp64.py drive them at the shapes and edges the models never reach.  The launches the models make are
// checked through the launch observer (ns2vc_check_set_launch_hook, observe_launch): the run loops hand each GEMM and attention
// record, as bound to the call, to tests/test_program_launches_fp64.py in the same flat structs, before and after it runs (the
// programs that module steps through are listed in its docstring and in DESIGN.md).  Nothing here is a kernel: every launch
// is the product's own.  The packed-weight record (ns2vc_check_packed, ns2vc_check_fold_vector) gives back what each engine's
// packer built, for tests/test_packed_weights_fp64.py.  The one kernel here, philox_check_kernel, runs the sampler
// noise's device functions (philox.cuh) on a list of counters and keys for tests/test_seeded_noise.py.
#include "engine_host.cuh"
#include "philox.cuh"
#include "../../include/ns2vc_b200.h"

#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

namespace ns2vc {
namespace {

SplitBuf to_split(const ns2vc_check_split& s) {
  SplitBuf b{};
  b.hi = (__nv_bfloat16*)s.hi; b.lo = (__nv_bfloat16*)s.lo; b.T = s.T; b.C = s.C; b.ld = s.ld; b.bpitch = s.bpitch;
  return b;
}

// The EngineBase of the handle of engine `kind` (0 denoiser, 1 condition encoders, 2 content encoder, 3 vocoder); nullptr (the
// error, prefixed by `fn`, is set) for another kind or a null handle
const EngineBase* base_of(int kind, const void* handle, const char* fn) {
  const EngineBase* e = nullptr;
  switch (kind) {
    case 0: e = engine_base((const ns2vc_unet*)handle); break;
    case 1: e = engine_base((const ns2vc_pre*)handle); break;
    case 2: e = engine_base((const ns2vc_cv*)handle); break;
    case 3: e = engine_base((const ns2vc_voc*)handle); break;
    default: set_error("%s: engine kind %d (0 denoiser, 1 condition encoders, 2 content encoder, 3 vocoder)", fn, kind); return nullptr;
  }
  if (!handle) { set_error("%s: null handle", fn); return nullptr; }
  return e;
}

// The packed record of the handle of engine `kind`; nullptr (the error is set) as for base_of, or for weights that are not packed
const PackedRecord* packed_record(int kind, const void* handle) {
  const EngineBase* e = base_of(kind, handle, "check_packed");
  if (!e) return nullptr;
  if (!e->finalized) { set_error("check_packed: the weights are not packed (finalize has not run since the last load)"); return nullptr; }
  return &e->packed;
}

// copies `name` into the caller's buffer (may be null)
int copy_name(const std::string& name, char* out, int out_len) {
  if (!out) return 0;
  NS_REQUIRE(out_len > (int)name.size(), "check_packed: name buffer of %d bytes for %s (%d + 1 needed)", out_len, name.c_str(), (int)name.size());
  memcpy(out, name.c_str(), name.size() + 1);
  return 0;
}

// the kernel and template arguments a launch selected, for the caller's `desc` (may be null)
template <class... A> void report(char* desc, int desc_len, const char* fmt, A... args) {
  if (desc && desc_len > 0) snprintf(desc, (size_t)desc_len, fmt, args...);
}

// the template arguments launch_gemm_tc selects for a planned operator
void report_gemm(const GemmOp& g, char* desc, int desc_len) {
  const int f = g.flags;
  const bool voc = (f & EPI_GELU) != 0, enc = !voc && (f & (EPI_RELU | EPI_ROWMASK));
  report(desc, desc_len, "gemm_tc<%d,LNF=%d,XF=%d,ENC=%d,RAG=%d,VOC=%d>", g.bn, (f & EPI_LNFOLD) ? 1 : 0, g.xmode ? 1 : 0, enc ? 1 : 0,
         g.row_len ? 1 : 0, voc ? 1 : 0);
}

// the kernel the attention dispatch launches for an operator (v2: after encode_attn_tmaps)
void report_attn(const AttnOp& op, char* desc, int desc_len) {
  if (op.v2) {
    const bool pf16 = attention_v2_p_fp16() && !op.p_split;
    report(desc, desc_len, "attn_v2<%d,PB=%d,BIAS=%d,PF16=%d,RAGK=%d>", op.dh, op.pb, op.bias ? 1 : 0, pf16 ? 1 : 0, op.key_len ? 1 : 0);
  } else {
    const int dhp = op.dh <= 16 ? 16 : op.dh <= 32 ? 32 : op.dh <= 48 ? 48 : 64;
    report(desc, desc_len, "attn_tc<%d>", dhp);
  }
}

ns2vc_check_split from_split(const SplitBuf& s) { return ns2vc_check_split{s.hi, s.lo, s.T, s.C, s.ld, s.bpitch}; }

// The flat description of a program's GEMM: its segments as ns2vc_check_gemm takes them, and (panel mode) the affine of its
// device-side descriptor, read back (the stream is synchronised)
int flat_gemm(const GemmOp& g, ns2vc_check_gemm_args& a) {
  memset(&a, 0, sizeof(a));
  a.B = g.B; a.T_out = g.T_out;
  a.nsrc = g.nsrc;
  for (int i = 0; i < g.nsrc; ++i) a.src[i] = from_split(g.src[i]);
  a.nseg = g.nseg;
  for (int i = 0; i < g.nseg; ++i) {
    const GSeg& s = g.seg[i];
    a.seg[i][0] = s.src; a.seg[i][1] = s.c0; a.seg[i][2] = 64 * s.nkb; a.seg[i][3] = s.tap;
  }
  a.nxs = g.xmode ? g.nxs : 0;
  for (int i = 0; i < a.nxs; ++i) {
    const XSeg& x = g.xs[i];
    const int v[8] = {x.src, x.c0, 64 * x.ncb, x.ntap, x.kb_tap[0], x.ntap > 1 ? x.kb_tap[1] - x.kb_tap[0] : 0, x.xf, x.aff_c0};
    memcpy(a.xseg[i], v, sizeof(v));
  }
  a.w_hi = g.w_hi; a.w_lo = g.w_lo; a.N = g.N; a.n_valid = g.n_valid; a.nkb_w = g.nkb_total;
  a.flags = g.flags;
  a.bias = g.bias; a.rowbias = g.rowbias; a.rowbias_ld = g.rowbias_ld; a.res = g.res; a.res_ld = g.res_ld;
  a.out = g.out; a.out_ld = g.out_ld; a.out_hi = g.out_hi; a.out_lo = g.out_lo; a.out_split_ld = g.out_split_ld;
  a.f16_col0 = g.f16_col0 == 0x7fffffff ? -1 : g.f16_col0;
  a.ln_stats = g.ln_stats; a.ln_g = g.ln_g; a.ln_C = g.ln_C; a.ln_eps = g.ln_eps;
  a.row_stats = g.row_stats; a.stat_sum = g.stat_sum; a.stat_sq = g.stat_sq;
  a.rowmask = g.rowmask; a.row_len = g.row_len; a.len_shift = g.len_shift;
  a.ksplit = g.ksplit; a.bn = g.bn; a.tma_out = g.tma_out;
  if (!g.xmode || !g.pre) return 0;
  PrepOp p;
  NS_CHECK_CUDA(cudaMemcpy(&p, g.pre, sizeof(p), cudaMemcpyDeviceToHost));
  a.pre_mode = p.mode;
  if (p.scale) {
    a.pre_scale = p.scale; a.pre_shift = p.shift; a.pre_C = p.C1 + p.C2;
    return 0;
  }
  // the flat record carries what set_group_norm derives from its arguments: check that this descriptor is one it built
  const int Cg = p.C1 + p.C2;
  NS_REQUIRE(p.gn.G >= 1 && Cg % p.gn.G == 0 && p.gn.sq1 == p.gn.sum1 + (size_t)g.B * p.C1 &&
             (p.C2 ? p.gn.sq2 == p.gn.sum2 + (size_t)g.B * p.C2 : !p.gn.sum2) &&
             std::fabs(p.gn.inv_n * (double)g.T_out * (Cg / p.gn.G) - 1.0) < 1e-12,
             "launch hook: a panel GroupNorm descriptor the flat record cannot express");
  a.gn_stats1 = p.gn.sum1; a.gn_stats2 = p.gn.sum2; a.gn_C1 = p.C1; a.gn_C2 = p.C2; a.gn_G = p.gn.G; a.gn_eps = p.gn.eps;
  a.gn_gamma = p.gn.gamma; a.gn_beta = p.gn.beta; a.gn_film = g.pre_film; a.gn_film_ld = p.gn.film_ld;
  return 0;
}

void flat_attn(const AttnOp& op, ns2vc_check_attn_args& a) {
  memset(&a, 0, sizeof(a));
  a.B = op.B; a.H = op.H; a.Tq = op.Tq; a.Tk = op.Tk; a.dh = op.dh; a.scale = op.scale; a.v2 = op.v2;
  a.q = op.q; a.q_ld = op.q_ld; a.k = op.k; a.k_ld = op.k_ld; a.v = op.v; a.v_ld = op.v_ld;
  a.qs = from_split(op.qs); a.ks = from_split(op.ks); a.vs = from_split(op.vs);
  a.q_c0 = op.q_c0; a.k_c0 = op.k_c0; a.v_c0 = op.v_c0;
  a.p_split = op.p_split; a.key_len = op.key_len; a.key_shift = op.key_shift; a.bias = op.bias;
  a.out = op.out; a.out_ld = op.out_ld; a.out_hi = op.out_hi; a.out_lo = op.out_lo; a.out_split_ld = op.out_split_ld;
  a.pb = op.pb;
}

}  // namespace

int observe_launch(const LaunchHook& hook, int index, int phase, const Launch& l, cudaStream_t st) {
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  NS_CHECK_CUDA(cudaStreamIsCapturing(st, &cs));
  NS_REQUIRE(cs == cudaStreamCaptureStatusNone, "launch hook: the stream is capturing (the observer synchronises it: remove it to capture)");
  NS_CHECK_CUDA(cudaStreamSynchronize(st));
  ns2vc_check_gemm_args ga;
  ns2vc_check_attn_args aa;
  const ns2vc_check_gemm_args* gp = nullptr;
  const ns2vc_check_attn_args* ap = nullptr;
  char desc[96] = "";
  if (l.kind == Launch::GEMM) {
    const GemmOp& g = l.get<GemmOp>();
    const int rc = flat_gemm(g, ga);
    if (rc) return rc;
    report_gemm(g, desc, sizeof(desc));
    gp = &ga;
  } else if (l.kind == Launch::ATTN) {
    const AttnOp& a = l.get<AttnOp>();
    flat_attn(a, aa);
    report_attn(a, desc, sizeof(desc));
    ap = &aa;
  }
  const int r = ((ns2vc_check_launch_fn)hook.fn)(hook.user, index, phase, (int)l.kind, gp, ap, desc);
  NS_REQUIRE(r == 0, "launch hook: the observer returned %d at launch %d (phase %d)", r, index, phase);
  NS_CHECK_CUDA(cudaStreamSynchronize(st));
  return 0;
}

}  // namespace ns2vc

using namespace ns2vc;

namespace ns2vc {
// Entry j: raw[j] = Philox4x32-10(counters[j], keys[j]); normals[j] = (z0, z1) of the pair (x, y), then of (z, w).
__global__ void philox_check_kernel(const uint32_t* counters, const uint32_t* keys, int n, uint32_t* raw, float* normals) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint32_t* c = counters + 4 * (size_t)j;
  const PhiloxOut o = philox4x32_10(c[0], c[1], c[2], c[3], keys[2 * (size_t)j], keys[2 * (size_t)j + 1]);
  uint32_t* r = raw + 4 * (size_t)j;
  r[0] = o.x; r[1] = o.y; r[2] = o.z; r[3] = o.w;
  float* z = normals + 4 * (size_t)j;
  z[0] = box_muller(o.x, o.y, false); z[1] = box_muller(o.x, o.y, true);
  z[2] = box_muller(o.z, o.w, false); z[3] = box_muller(o.z, o.w, true);
}
}  // namespace ns2vc

extern "C" {

int ns2vc_check_pack_b(const float* w, int n_rows, int cin_total, int ktaps, int tap, int cin0, int ncin, int n_dst0, int kb0,
                       int geglu_half, const float* cscale, void* w_hi, void* w_lo, int Npad, int nkb_total, ns2vc_stream stream) {
  NS_REQUIRE(w && w_hi && w_lo, "check_pack_b: null argument");
  NS_REQUIRE(n_rows >= 1 && ktaps >= 1 && tap >= 0 && tap < ktaps && cin0 >= 0 && ncin >= 1 && cin0 + ncin <= cin_total,
             "check_pack_b: bad weight slice n_rows=%d cin=%d+%d of %d tap=%d of %d", n_rows, cin0, ncin, cin_total, tap, ktaps);
  NS_REQUIRE(Npad % 128 == 0 && n_dst0 >= 0 && n_dst0 + n_rows <= Npad, "check_pack_b: columns %d+%d do not fit Npad=%d", n_dst0, n_rows, Npad);
  NS_REQUIRE(kb0 >= 0 && kb0 + nkb_of(ncin) <= nkb_total, "check_pack_b: k-blocks %d+%d do not fit %d", kb0, nkb_of(ncin), nkb_total);
  NS_REQUIRE(geglu_half == 0 || 2 * geglu_half == n_rows, "check_pack_b: a GEGLU weight has 2 * geglu_half rows");
  PackedB pb;
  pb.hi = (__nv_bfloat16*)w_hi; pb.lo = (__nv_bfloat16*)w_lo; pb.Npad = Npad; pb.nkb = nkb_total;
  return pack_seg(pb, w, n_rows, cin_total, ktaps, tap, cin0, ncin, n_dst0, kb0, geglu_half, (cudaStream_t)stream, cscale);
}

int ns2vc_check_gemm(const ns2vc_check_gemm_args* a, char* desc, int desc_len, ns2vc_stream stream) {
  NS_REQUIRE(a, "check_gemm: null argument");
  NS_REQUIRE(a->B >= 1 && a->T_out >= 1, "check_gemm: bad sizes B=%d T_out=%d", a->B, a->T_out);
  NS_REQUIRE(a->nsrc >= 1 && a->nsrc <= kMaxSrc && a->nseg >= 0 && a->nseg <= kMaxSeg && a->nxs >= 0 && a->nxs <= kMaxXSeg,
             "check_gemm: %d sources (1..%d), %d segments (0..%d), %d panel segments (0..%d)", a->nsrc, kMaxSrc, a->nseg, kMaxSeg,
             a->nxs, kMaxXSeg);
  NS_REQUIRE((a->nseg > 0) != (a->nxs > 0), "check_gemm: either plain segments or panel segments");
  NS_REQUIRE(a->w_hi && a->w_lo, "check_gemm: null weights");
  const int f = a->flags;
  NS_REQUIRE(!(f & (EPI_OUT_F32 | EPI_OUT_NCT)) || a->out, "check_gemm: fp32 output without a buffer");
  NS_REQUIRE(!(f & EPI_OUT_SPLIT) || (a->out_hi && a->out_lo), "check_gemm: split output without buffers");
  NS_REQUIRE(!(f & (EPI_BIAS | EPI_GEGLU)) || a->bias, "check_gemm: bias flag without a bias");
  NS_REQUIRE(!(f & EPI_RESIDUAL) || a->res, "check_gemm: residual flag without a residual");
  NS_REQUIRE(!(f & EPI_ROWBIAS) || a->rowbias, "check_gemm: row-bias flag without a row bias");
  NS_REQUIRE(!(f & EPI_LNFOLD) || (a->ln_stats && a->ln_g && a->ln_C > 0), "check_gemm: folded LayerNorm without statistics");
  NS_REQUIRE(!(f & EPI_ROWSTATS) || a->row_stats, "check_gemm: row statistics without a buffer");
  NS_REQUIRE(!(f & EPI_STATS) || (a->stat_sum && a->stat_sq), "check_gemm: column statistics without buffers");

  PackedB w;
  w.hi = (__nv_bfloat16*)a->w_hi; w.lo = (__nv_bfloat16*)a->w_lo; w.Npad = a->N; w.nkb = a->nkb_w; w.n_logical = a->n_valid;
  ProgramBuilder bld{Arena{}, a->B, false, false, nullptr};
  GemmOp g = bld.gemm_base(w, a->T_out);
  for (int i = 0; i < a->nsrc; ++i) bld.add_src(g, to_split(a->src[i]));
  for (int i = 0; i < a->nseg; ++i) {
    const int* s = a->seg[i];
    NS_REQUIRE(s[0] >= 0 && s[0] < a->nsrc && s[1] >= 0 && s[2] >= 1, "check_gemm: bad segment %d", i);
    bld.seg(g, s[0], s[1], s[2], s[3]);
  }
  for (int i = 0; i < a->nxs; ++i) {
    const int* x = a->xseg[i];
    NS_REQUIRE(x[0] >= 0 && x[0] < a->nsrc && x[1] >= 0 && x[1] % 64 == 0 && x[2] >= 1 && (x[3] == 1 || x[3] == 3),
               "check_gemm: bad panel segment %d", i);
    NS_REQUIRE(!x[6] || (x[7] >= 0 && x[7] + nkb_of(x[2]) * 64 <= kXfMaxC), "check_gemm: panel segment %d outside the affine table", i);
    bld.xseg(g, x[0], x[1], x[2], x[3], x[4], x[5], x[6], x[7]);
  }
  NS_REQUIRE(g.nkb_total == a->nkb_w, "check_gemm: the segments cover %d k-blocks, the weights %d", g.nkb_total, a->nkb_w);
  if (g.xmode) for (int i = 0; i < g.nxs; ++i) for (int j = 0; j < g.xs[i].ntap; ++j)
    NS_REQUIRE(g.xs[i].kb_tap[j] >= 0 && g.xs[i].kb_tap[j] + g.xs[i].ncb <= a->nkb_w, "check_gemm: panel segment %d tap %d outside the weights", i, j);
  g.flags = f;
  g.bias = a->bias; g.rowbias = a->rowbias; g.rowbias_ld = a->rowbias_ld; g.res = a->res; g.res_ld = a->res_ld;
  g.out = a->out; g.out_ld = a->out_ld;
  g.out_hi = (__nv_bfloat16*)a->out_hi; g.out_lo = (__nv_bfloat16*)a->out_lo; g.out_split_ld = a->out_split_ld;
  if (a->f16_col0 >= 0) g.f16_col0 = a->f16_col0;
  g.ln_stats = a->ln_stats; g.ln_g = a->ln_g; g.ln_C = a->ln_C; g.ln_eps = a->ln_eps;
  g.row_stats = a->row_stats; g.stat_sum = a->stat_sum; g.stat_sq = a->stat_sq;
  g.rowmask = a->rowmask; g.row_len = a->row_len; g.len_shift = a->len_shift;
  g.ksplit = a->ksplit;

  cudaStream_t st = (cudaStream_t)stream;
  PrepOp* pre_dev = nullptr;
  if (g.xmode && (a->pre_scale || a->gn_stats1)) {
    NS_REQUIRE(a->pre_mode == PREP_AFFINE || a->pre_mode == PREP_AFFINE_SILU, "check_gemm: panel affine mode %d", a->pre_mode);
    PrepOp p; memset(&p, 0, sizeof(p));
    p.B = a->B; p.T_src = a->T_out; p.T_dst = a->T_out; p.mode = a->pre_mode;
    if (a->pre_scale) {
      NS_REQUIRE(a->pre_shift && a->pre_C >= 1 && a->pre_C <= kXfMaxC, "check_gemm: panel affine needs scale, shift and 1..%d channels", kXfMaxC);
      p.C1 = a->pre_C;
      p.scale = a->pre_scale; p.shift = a->pre_shift;
    } else {
      // the GroupNorm descriptor as the denoiser's normed_input builds it in panel mode; the FiLM rows travel in GemmOp::pre_film
      const int Cg = a->gn_C1 + a->gn_C2;
      NS_REQUIRE(a->gn_C1 >= 1 && a->gn_C2 >= 0 && (a->gn_C2 == 0) == (a->gn_stats2 == nullptr) && Cg <= kXfMaxC,
                 "check_gemm: GroupNorm sources %d + %d channels (up to %d)", a->gn_C1, a->gn_C2, kXfMaxC);
      NS_REQUIRE(a->gn_G >= 1 && a->gn_G <= 64 && Cg % a->gn_G == 0 && a->gn_gamma && a->gn_beta,
                 "check_gemm: GroupNorm of %d channels in %d groups", Cg, a->gn_G);
      NS_REQUIRE(!a->gn_film || a->gn_film_ld >= 2 * Cg, "check_gemm: FiLM rows of %d < %d", a->gn_film_ld, 2 * Cg);
      p.C1 = a->gn_C1; p.C2 = a->gn_C2;
      set_group_norm(p, a->B, a->gn_stats1, a->gn_C1, a->gn_stats2, a->gn_C2, a->T_out, a->gn_G, a->gn_eps, a->gn_gamma, a->gn_beta,
                     nullptr, a->gn_film_ld);
      g.pre_film = a->gn_film;
    }
    p.row_len = a->row_len; p.len_shift = a->len_shift;
    NS_CHECK_CUDA(cudaMallocAsync((void**)&pre_dev, sizeof(PrepOp), st));
    NS_CHECK_CUDA(cudaMemcpyAsync(pre_dev, &p, sizeof(PrepOp), cudaMemcpyHostToDevice, st));
    g.pre = pre_dev;
  }
  plan_gemm(g);
  int rc = encode_tmaps(g);
  if (!rc) rc = launch_gemm_tc(g, st);
  if (pre_dev) NS_CHECK_CUDA(cudaFreeAsync(pre_dev, st));
  if (rc) return rc;
  report_gemm(g, desc, desc_len);
  return 0;
}

int ns2vc_check_attention(const ns2vc_check_attn_args* a, char* desc, int desc_len, ns2vc_stream stream) {
  NS_REQUIRE(a, "check_attention: null argument");
  NS_REQUIRE(a->B >= 1 && a->H >= 1 && a->dh >= 1, "check_attention: bad sizes B=%d H=%d dh=%d", a->B, a->H, a->dh);
  NS_REQUIRE(a->out || (a->out_hi && a->out_lo), "check_attention: no output");
  AttnOp op; memset(&op, 0, sizeof(op));
  op.B = a->B; op.H = a->H; op.Tq = a->Tq; op.Tk = a->Tk; op.dh = a->dh; op.scale = a->scale;
  op.bias = a->bias;
  op.out = a->out; op.out_ld = a->out_ld;
  op.out_hi = (__nv_bfloat16*)a->out_hi; op.out_lo = (__nv_bfloat16*)a->out_lo; op.out_split_ld = a->out_split_ld;
  cudaStream_t st = (cudaStream_t)stream;
  if (a->v2) {
    NS_REQUIRE(a->qs.hi && a->qs.lo && a->ks.hi && a->ks.lo && a->vs.hi && a->vs.lo, "check_attention: v2 needs split q / k / v");
    op.v2 = 1;
    op.qs = to_split(a->qs); op.ks = to_split(a->ks); op.vs = to_split(a->vs);
    op.q_c0 = a->q_c0; op.k_c0 = a->k_c0; op.v_c0 = a->v_c0;
    op.key_len = a->key_len; op.key_shift = a->key_shift; op.p_split = a->p_split;
    int rc = encode_attn_tmaps(op);
    if (!rc) rc = launch_attention_v2(op, st);
    if (rc) return rc;
    report_attn(op, desc, desc_len);
    return 0;
  }
  NS_REQUIRE(a->q && a->k && a->v, "check_attention: v1 needs fp32 q / k / v");
  NS_REQUIRE(!a->key_len, "check_attention: per-entry key counts are a v2 feature");
  op.q = a->q; op.q_ld = a->q_ld; op.k = a->k; op.k_ld = a->k_ld; op.v = a->v; op.v_ld = a->v_ld;
  const int rc = launch_attention(op, st, false);
  if (rc) return rc;
  report_attn(op, desc, desc_len);
  return 0;
}

int ns2vc_check_prep(const ns2vc_check_prep_args* a, char* desc, int desc_len, ns2vc_stream stream) {
  NS_REQUIRE(a, "check_prep: null argument");
  NS_REQUIRE(a->B >= 1 && a->T_src >= 1 && a->T_dst >= 1 && a->C1 >= 1 && a->C2 >= 0 && a->src1 && (a->C2 == 0 || a->src2),
             "check_prep: bad sizes B=%d T=%d->%d C=%d+%d", a->B, a->T_src, a->T_dst, a->C1, a->C2);
  NS_REQUIRE(a->out.hi && a->out.lo, "check_prep: no output");
  NS_REQUIRE(a->mode >= PREP_RAW && a->mode <= PREP_AFFINE_SILU, "check_prep: mode %d", a->mode);
  PrepOp p; memset(&p, 0, sizeof(p));
  p.src1 = a->src1; p.ld1 = a->ld1; p.C1 = a->C1; p.src2 = a->src2; p.ld2 = a->ld2; p.C2 = a->C2;
  p.B = a->B; p.T_src = a->T_src; p.T_dst = a->T_dst;
  p.row_mul = a->row_mul; p.row_add = a->row_add; p.rowmap = a->rowmap; p.mode = a->mode;
  p.out = to_split(a->out);
  if (a->raw.hi) p.raw = to_split(a->raw);
  p.row_len = a->row_len; p.len_shift = a->len_shift;
  if (a->mode != PREP_RAW) {
    if (a->scale) {
      NS_REQUIRE(a->shift, "check_prep: scale without shift");
      p.scale = a->scale; p.shift = a->shift;
    } else {
      NS_REQUIRE(a->stats1 && (a->C2 == 0 || a->stats2) && a->gamma && a->beta && a->G >= 1, "check_prep: GroupNorm without its sums or weights");
      set_group_norm(p, a->B, a->stats1, a->C1, a->C2 ? a->stats2 : nullptr, a->C2, a->T_src, a->G, a->eps, a->gamma, a->beta, a->film,
                     a->film_ld);
    }
  }
  const int rc = launch_prep_split(p, (cudaStream_t)stream);
  if (rc) return rc;
  report(desc, desc_len, "prep_split<RAG=%d>", p.row_len ? 1 : 0);
  return 0;
}

int ns2vc_check_ln(const ns2vc_check_ln_args* a, char* desc, int desc_len, ns2vc_stream stream) {
  NS_REQUIRE(a && a->x && a->gamma && a->beta, "check_ln: null argument");
  NS_REQUIRE(a->M >= 1 && a->C >= 1 && a->ld >= a->C, "check_ln: bad sizes M=%d C=%d ld=%d", a->M, a->C, a->ld);
  LnOp op{a->x, a->ld, a->M, a->C, a->eps, a->gamma, a->beta, a->keep, a->y, a->y_ld, to_split(a->split)};
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  switch (a->kind) {
    case 0:
      NS_REQUIRE(op.split.hi && op.split.lo, "check_ln: ln_split without a split output");
      if ((rc = launch_ln_split(op, st))) return rc;
      report(desc, desc_len, "ln_split<KEEP=%d>", op.keep ? 1 : 0);
      return 0;
    case 1:
      NS_REQUIRE(op.y, "check_ln: ln_apply without an output");
      if ((rc = launch_ln_apply(op, st))) return rc;
      report(desc, desc_len, "%s", "ln_apply");
      return 0;
    case 2:
      NS_REQUIRE(op.y && op.keep, "check_ln: ln_mask without an output or keep factors");
      if ((rc = launch_ln_mask(op, st))) return rc;
      report(desc, desc_len, "%s", "ln_mask");
      return 0;
  }
  set_error("check_ln: kind %d", a->kind);
  return -1;
}

int ns2vc_check_voc_norm(const ns2vc_check_voc_norm_args* a, char* desc, int desc_len, ns2vc_stream stream) {
  NS_REQUIRE(a && a->x && a->gamma && a->beta, "check_voc_norm: null argument");
  NS_REQUIRE(a->B >= 1 && a->T >= 1 && a->C >= 128 && a->C <= 1024 && a->C % 128 == 0, "check_voc_norm: bad sizes B=%d T=%d C=%d", a->B,
             a->T, a->C);
  NS_REQUIRE(a->out || (a->split.hi && a->split.lo), "check_voc_norm: no output");
  VocNormOp op{a->x, a->B, a->T, a->C, a->dw, a->gamma, a->beta, a->eps, (const long long*)a->len, a->out, to_split(a->split)};
  const int rc = launch_voc_norm(op, (cudaStream_t)stream);
  if (rc) return rc;
  report(desc, desc_len, "voc_norm<DW=%d>", a->dw ? 1 : 0);
  return 0;
}

int ns2vc_check_small_linear(const ns2vc_check_linear_args* a, char* desc, int desc_len, ns2vc_stream stream) {
  NS_REQUIRE(a && a->x && a->W && a->out, "check_small_linear: null argument");
  NS_REQUIRE(a->M >= 1 && a->K >= 1 && a->N >= 1 && a->in_mode >= LIN_RAW && a->in_mode <= LIN_SINUSOID,
             "check_small_linear: bad sizes M=%d K=%d N=%d mode %d", a->M, a->K, a->N, a->in_mode);
  LinOp op = linear_op(a->x, a->x_ld, a->M, a->K, a->W, a->bias, a->N, a->out, a->out_ld);
  op.add = a->add; op.add_ld = a->add_ld; op.add_rows = a->add_rows;
  op.in_mode = a->in_mode; op.flip_sin_to_cos = a->flip_sin_to_cos; op.freq_shift = a->freq_shift; op.out_silu = a->out_silu;
  const int rc = launch_small_linear(op, (cudaStream_t)stream);
  if (rc) return rc;
  report(desc, desc_len, "%s", "small_linear");
  return 0;
}

int ns2vc_check_pool(const ns2vc_check_pool_args* a, char* desc, int desc_len, ns2vc_stream stream) {
  NS_REQUIRE(a && (a->tokens || a->out), "check_pool: nothing to launch");
  NS_REQUIRE(a->B >= 1 && a->S >= 1 && a->C >= 1, "check_pool: bad sizes B=%d S=%d C=%d", a->B, a->S, a->C);
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if (a->tokens) {
    NS_REQUIRE(a->x && a->pos, "check_pool: class token without input");
    if ((rc = launch_pool_class_token(PoolClsOp{a->x, a->pos, a->B, a->S, a->C, a->tokens, a->lens}, st))) return rc;
  }
  if (a->out) {
    NS_REQUIRE(a->q && a->kv && a->heads >= 1, "check_pool: attention without q / kv");
    const PoolAttOp op{a->q, a->kv, a->B, a->S + 1, a->C, a->heads, a->out, a->lens};
    if ((rc = a->wide ? launch_pool_attend_wide(op, st) : launch_pool_attend(op, st))) return rc;
  }
  report(desc, desc_len, "%s%s%s<RAG=%d>", a->tokens ? "pool_class_token" : "", a->tokens && a->out ? "+" : "",
         a->out ? (a->wide ? "pool_attend_wide" : "pool_attend") : "", a->lens ? 1 : 0);
  return 0;
}

int ns2vc_check_nct_split(const ns2vc_check_nct_split_args* a, char* desc, int desc_len, ns2vc_stream stream) {
  NS_REQUIRE(a && a->x && a->out.hi && a->out.lo, "check_nct_split: null argument");
  NS_REQUIRE(a->B >= 1 && a->C >= 1 && a->T >= 1 && a->out.ld >= a->C && a->out.ld % 8 == 0, "check_nct_split: bad sizes B=%d C=%d T=%d ld=%d",
             a->B, a->C, a->T, a->out.ld);
  const int rc = launch_nct_to_split(NctSplitOp{a->x, a->bstride, a->B, a->C, a->T, to_split(a->out), a->row_len, nullptr, 0}, (cudaStream_t)stream);
  if (rc) return rc;
  report(desc, desc_len, "nct_to_split<RAG=%d>", a->row_len ? 1 : 0);
  return 0;
}

int ns2vc_check_cv_conv0(const ns2vc_check_cv_conv0_args* a, char* desc, int desc_len, ns2vc_stream stream) {
  NS_REQUIRE(a && a->wav && a->w0 && a->gamma && a->beta && a->stats && a->out.hi && a->out.lo, "check_cv_conv0: null argument");
  NS_REQUIRE(a->B >= 1 && a->B <= 65535 && a->N >= 400 && a->bstride >= a->N && a->rows >= 1, "check_cv_conv0: bad sizes B=%d N=%d bstride=%lld rows=%d",
             a->B, a->N, a->bstride, a->rows);
  NS_REQUIRE(a->C0 >= 128 && a->C0 <= 1024 && a->C0 % 128 == 0 && a->out.C == a->C0 && a->out.ld >= a->C0 && a->out.ld % 8 == 0,
             "check_cv_conv0: C0=%d (a multiple of 128 up to 1024), out C=%d ld=%d", a->C0, a->out.C, a->out.ld);
  cudaStream_t st = (cudaStream_t)stream;
  const long long* len = (const long long*)a->lengths;
  float2* stats = (float2*)a->stats;
  int rc = launch_cv_gn_stats(CvGnStatsOp{a->B, a->N, a->C0, a->w0, a->eps, stats}, a->wav, a->bstride, len, st);
  if (rc) return rc;
  rc = launch_cv_conv0(CvConv0Op{a->B, a->N, a->rows, a->w0, stats, a->gamma, a->beta, to_split(a->out)}, a->wav, a->bstride, len, st);
  if (rc) return rc;
  report(desc, desc_len, "cv_gn_stats+cv_conv0<%d>", a->C0 / 2);
  return 0;
}

int ns2vc_check_cv_pos_conv(const ns2vc_check_cv_pos_conv_args* a, char* desc, int desc_len, ns2vc_stream stream) {
  NS_REQUIRE(a && a->x && a->frames && a->win_hi && a->win_lo, "check_cv_pos_conv: null argument");
  NS_REQUIRE(a->B >= 1 && a->B <= 65535 && a->T >= 1 && a->G >= 1 && a->D % a->G == 0 && a->D % 4 == 0, "check_cv_pos_conv: bad sizes B=%d T=%d D=%d G=%d",
             a->B, a->T, a->D, a->G);
  const int gw = a->D / a->G;
  NS_REQUIRE(gw <= 64 && gw % 4 == 0 && a->K >= 16 && a->K <= 16 * kMaxSeg && a->K % 16 == 0, "check_cv_pos_conv: group width %d, K=%d", gw, a->K);
  cudaStream_t st = (cudaStream_t)stream;
  const SplitBuf win{(__nv_bfloat16*)a->win_hi, (__nv_bfloat16*)a->win_lo, a->T + a->K, 1024, 1024, 0};
  int rc = launch_cv_pos_windows(CvPosWinOp{a->x, a->B, a->T, a->D, a->G, gw, a->K, (const long long*)a->frames, win}, st);
  if (rc) return rc;
  if (a->windows_only) {
    report(desc, desc_len, "%s", "cv_pos_windows");
    return 0;
  }
  NS_REQUIRE(a->w && a->bias && a->keep && a->out, "check_cv_pos_conv: the GEMMs need weights, bias, keep and out");
  ProgramBuilder bld{Arena{}, a->B, false, false, nullptr};
  PackedB pb;
  pb.Npad = pad_to(gw, 128); pb.nkb = a->K; pb.n_logical = gw;
  const size_t elems = (size_t)pb.nkb * pb.Npad * 64;
  NS_CHECK_CUDA(cudaMallocAsync((void**)&pb.hi, elems * sizeof(__nv_bfloat16), st));
  NS_CHECK_CUDA(cudaMallocAsync((void**)&pb.lo, elems * sizeof(__nv_bfloat16), st));
  int bn = 0;
  for (int g = 0; g < a->G && !rc; ++g) {
    if (cudaMemsetAsync(pb.hi, 0, elems * sizeof(__nv_bfloat16), st) != cudaSuccess || cudaMemsetAsync(pb.lo, 0, elems * sizeof(__nv_bfloat16), st) != cudaSuccess) {
      set_error("check_cv_pos_conv: memset failed");
      rc = -2;
      break;
    }
    if ((rc = pack_cv_pos_group(pb, a->w + (size_t)g * gw * gw * a->K, gw, a->K, st))) break;
    GemmOp op = cv_pos_group_gemm(bld, pb, win, a->G, g, gw, a->T, a->K, a->bias, a->keep, a->out, a->D);
    plan_gemm(op);
    bn = op.bn;
    if (!(rc = encode_tmaps(op))) rc = launch_gemm_tc(op, st);
  }
  NS_CHECK_CUDA(cudaFreeAsync(pb.hi, st));
  NS_CHECK_CUDA(cudaFreeAsync(pb.lo, st));
  if (rc) return rc;
  if ((rc = launch_cv_add(CvAddOp{a->out, a->x, (long long)a->B * a->T * a->D / 4}, st))) return rc;
  report(desc, desc_len, "cv_pos_windows+%dxgemm_tc<%d,LNF=0,XF=0,ENC=0,RAG=0,VOC=1>+cv_add", a->G, bn);
  return 0;
}

int ns2vc_check_down_conv(const ns2vc_check_down_conv_args* a, char* desc, int desc_len, ns2vc_stream stream) {
  NS_REQUIRE(a && a->x && a->in_hi && a->in_lo && a->w && a->bias, "check_down_conv: null argument");
  NS_REQUIRE(a->B >= 1 && a->B <= 65535 && a->Tin >= 1 && a->C >= 1, "check_down_conv: bad sizes B=%d Tin=%d C=%d", a->B, a->Tin, a->C);
  NS_REQUIRE(a->ld >= a->C && a->ld % 8 == 0, "check_down_conv: input ld=%d (a multiple of 8, at least C=%d)", a->ld, a->C);
  NS_REQUIRE(a->out || (a->out_hi && a->out_lo), "check_down_conv: no output");
  NS_REQUIRE(!a->row_len || a->len_shift >= 1, "check_down_conv: ragged output level %d (at least 1)", a->len_shift);
  cudaStream_t st = (cudaStream_t)stream;
  const int C = a->C, Cp = pad_to(C, 8), TL = (a->Tin - 1) / 2 + 1, To = std::max(a->Tin / 2, 1);
  PackedB pb;
  pb.Npad = pad_to(C, 128); pb.nkb = 3 * nkb_of(C); pb.n_logical = C;
  const size_t welems = (size_t)pb.nkb * pb.Npad * 64;
  NS_CHECK_CUDA(cudaMallocAsync((void**)&pb.hi, welems * sizeof(__nv_bfloat16), st));
  NS_CHECK_CUDA(cudaMallocAsync((void**)&pb.lo, welems * sizeof(__nv_bfloat16), st));
  // the prep path's dense even / odd splits (allocated either way: the views do not touch them)
  SplitBuf e{}, o{};
  e.T = TL; o.T = To; e.C = o.C = C; e.ld = o.ld = Cp;
  NS_CHECK_CUDA(cudaMallocAsync((void**)&e.hi, (size_t)a->B * TL * Cp * sizeof(__nv_bfloat16), st));
  NS_CHECK_CUDA(cudaMallocAsync((void**)&e.lo, (size_t)a->B * TL * Cp * sizeof(__nv_bfloat16), st));
  NS_CHECK_CUDA(cudaMallocAsync((void**)&o.hi, (size_t)a->B * To * Cp * sizeof(__nv_bfloat16), st));
  NS_CHECK_CUDA(cudaMallocAsync((void**)&o.lo, (size_t)a->B * To * Cp * sizeof(__nv_bfloat16), st));
  int rc = 0;
  if (cudaMemsetAsync(pb.hi, 0, welems * sizeof(__nv_bfloat16), st) != cudaSuccess || cudaMemsetAsync(pb.lo, 0, welems * sizeof(__nv_bfloat16), st) != cudaSuccess) {
    set_error("check_down_conv: memset failed");
    rc = -2;
  }
  if (!rc) rc = pack_resample_conv(pb, a->w, C, st);
  ProgramBuilder bld{Arena{}, a->B, false, false, nullptr};
  const SplitBuf raw{(__nv_bfloat16*)a->in_hi, (__nv_bfloat16*)a->in_lo, a->Tin, C, a->ld, 0};
  DownConv d = down_conv(bld, pb, a->bias, a->x, raw, a->Tin, C, !a->force_prep, e, o);
  for (int i = 0; i < d.nprep && !rc; ++i) rc = launch_prep_split(d.prep[i], st);
  GemmOp& g = d.g;
  if (a->out) { g.flags |= EPI_OUT_F32; g.out = a->out; g.out_ld = C; }
  if (a->out_hi) { g.flags |= EPI_OUT_SPLIT; g.out_hi = (__nv_bfloat16*)a->out_hi; g.out_lo = (__nv_bfloat16*)a->out_lo; g.out_split_ld = Cp; }
  g.row_len = a->row_len; g.len_shift = a->len_shift;
  if (!rc) {
    plan_gemm(g);
    if (!(rc = encode_tmaps(g))) rc = launch_gemm_tc(g, st);
  }
  for (void* p : {(void*)pb.hi, (void*)pb.lo, (void*)e.hi, (void*)e.lo, (void*)o.hi, (void*)o.lo}) NS_CHECK_CUDA(cudaFreeAsync(p, st));
  if (rc) return rc;
  report(desc, desc_len, "%sgemm_tc<%d,LNF=0,XF=0,ENC=0,RAG=%d,VOC=0>", d.nprep ? "2xprep_split<RAG=0>+" : "", g.bn, g.row_len ? 1 : 0);
  return 0;
}

int ns2vc_check_cv_conv(const ns2vc_check_cv_conv_args* a, char* desc, int desc_len, ns2vc_stream stream) {
  NS_REQUIRE(a && a->in_hi && a->in_lo && a->w && a->keep, "check_cv_conv: null argument");
  NS_REQUIRE(a->l >= 1 && a->l <= 6, "check_cv_conv: conv index %d (1 .. 6)", a->l);
  NS_REQUIRE(a->C0 >= 128 && a->C0 <= 1024 && a->C0 % 128 == 0, "check_cv_conv: C0=%d (a multiple of 128 up to 1024)", a->C0);
  NS_REQUIRE(a->B >= 1 && a->B <= 65535 && a->rows_in >= 2 && a->rows_out >= 1, "check_cv_conv: bad sizes B=%d rows_in=%d rows_out=%d", a->B,
             a->rows_in, a->rows_out);
  NS_REQUIRE(a->rows_in % 2 == 0, "check_cv_conv: rows_in=%d is odd (a row pair would straddle two entries)", a->rows_in);
  NS_REQUIRE((a->out != nullptr) != (a->out_hi != nullptr) && (a->out_hi != nullptr) == (a->out_lo != nullptr),
             "check_cv_conv: exactly one output, fp32 or split");
  cudaStream_t st = (cudaStream_t)stream;
  const int C0 = a->C0;
  PackedB pb;
  pb.Npad = C0; pb.nkb = cv_conv_taps(a->l) * nkb_of(C0); pb.n_logical = C0;
  const size_t welems = (size_t)pb.nkb * pb.Npad * 64;
  NS_CHECK_CUDA(cudaMallocAsync((void**)&pb.hi, welems * sizeof(__nv_bfloat16), st));
  NS_CHECK_CUDA(cudaMallocAsync((void**)&pb.lo, welems * sizeof(__nv_bfloat16), st));
  int rc = pack_cv_conv(pb, a->w, C0, a->l, st);
  ProgramBuilder bld{Arena{}, a->B, false, false, nullptr};
  const SplitBuf in{(__nv_bfloat16*)a->in_hi, (__nv_bfloat16*)a->in_lo, a->rows_in, C0, C0, 0};
  const SplitBuf out{(__nv_bfloat16*)a->out_hi, (__nv_bfloat16*)a->out_lo, a->rows_out, C0, C0, 0};
  GemmOp g = cv_conv_gemm(bld, pb, in, a->rows_in, a->rows_out, a->l, a->keep, out, a->out);
  if (!rc) {
    plan_gemm(g);
    if (!(rc = encode_tmaps(g))) rc = launch_gemm_tc(g, st);
  }
  NS_CHECK_CUDA(cudaFreeAsync(pb.hi, st));
  NS_CHECK_CUDA(cudaFreeAsync(pb.lo, st));
  if (rc) return rc;
  report(desc, desc_len, "gemm_tc<%d,LNF=0,XF=0,ENC=0,RAG=0,VOC=1>", g.bn);
  return 0;
}

int ns2vc_check_istft(const ns2vc_check_istft_args* a, char* desc, int desc_len, ns2vc_stream stream) {
  NS_REQUIRE(a && a->h && a->window && a->audio, "check_istft: null argument");
  const int n_fft = a->n_fft, hop = n_fft / 4;
  NS_REQUIRE(n_fft >= 64 && n_fft <= 2048 && (n_fft & (n_fft - 1)) == 0, "check_istft: n_fft %d (a power of two, 64 .. 2048)", n_fft);
  NS_REQUIRE(a->B >= 1 && a->B <= 65535 && a->T >= 1 && (long long)a->T * hop <= INT32_MAX && a->ld >= n_fft + 2, "check_istft: bad sizes B=%d T=%d ld=%d",
             a->B, a->T, a->ld);
  cudaStream_t st = (cudaStream_t)stream;
  std::vector<float2> th, tf;
  istft_twiddles(n_fft, th, tf);
  float2 *d_th = nullptr, *d_tf = nullptr;
  NS_CHECK_CUDA(cudaMallocAsync((void**)&d_th, th.size() * sizeof(float2), st));
  NS_CHECK_CUDA(cudaMallocAsync((void**)&d_tf, tf.size() * sizeof(float2), st));
  NS_CHECK_CUDA(cudaMemcpyAsync(d_th, th.data(), th.size() * sizeof(float2), cudaMemcpyHostToDevice, st));
  NS_CHECK_CUDA(cudaMemcpyAsync(d_tf, tf.data(), tf.size() * sizeof(float2), cudaMemcpyHostToDevice, st));
  const int log2m = istft_log2m(n_fft);
  const size_t smem = istft_smem_bytes(n_fft);
  const int rc = launch_istft(IstftTables{a->window, d_th, d_tf}, a->h, a->ld, (const long long*)a->len, a->audio, a->B, a->T, n_fft, hop, log2m,
                              smem, st);
  NS_CHECK_CUDA(cudaFreeAsync(d_th, st));
  NS_CHECK_CUDA(cudaFreeAsync(d_tf, st));
  if (rc) return rc;
  report(desc, desc_len, "voc_istft<log2m=%d,smem=%zu>", log2m, smem);
  return 0;
}

int ns2vc_check_packed_count(int kind, const void* handle) {
  const PackedRecord* r = packed_record(kind, handle);
  return r ? (int)r->entries.size() : -1;
}

int ns2vc_check_packed(int kind, const void* handle, int i, char* name, int name_len, int* Npad, int* nkb, int* n_logical, int* nvec,
                       void* hi_out, void* lo_out, ns2vc_stream stream) {
  const PackedRecord* r = packed_record(kind, handle);
  if (!r) return -1;
  NS_REQUIRE(i >= 0 && i < (int)r->entries.size(), "check_packed: operand %d out of range (%d recorded)", i, (int)r->entries.size());
  const PackedRecord::Entry& e = r->entries[i];
  int rc = copy_name(e.name, name, name_len);
  if (rc) return rc;
  if (Npad) *Npad = e.pb.Npad;
  if (nkb) *nkb = e.pb.nkb;
  if (n_logical) *n_logical = e.pb.n_logical;
  if (nvec) *nvec = (int)e.vecs.size();
  const size_t bytes = (size_t)e.pb.nkb * e.pb.Npad * 64 * sizeof(__nv_bfloat16);
  cudaStream_t st = (cudaStream_t)stream;
  if (hi_out && bytes) NS_CHECK_CUDA(cudaMemcpyAsync(hi_out, e.pb.hi, bytes, cudaMemcpyDeviceToDevice, st));
  if (lo_out && bytes) NS_CHECK_CUDA(cudaMemcpyAsync(lo_out, e.pb.lo, bytes, cudaMemcpyDeviceToDevice, st));
  return 0;
}

int ns2vc_check_fold_vector(int kind, const void* handle, int i, int j, char* name, int name_len, long long* n, float* out,
                            ns2vc_stream stream) {
  const PackedRecord* r = packed_record(kind, handle);
  if (!r) return -1;
  NS_REQUIRE(i >= 0 && i < (int)r->entries.size(), "check_fold_vector: operand %d out of range (%d recorded)", i, (int)r->entries.size());
  const PackedRecord::Entry& e = r->entries[i];
  NS_REQUIRE(j >= 0 && j < (int)e.vecs.size(), "check_fold_vector: vector %d of %s out of range (%d recorded)", j, e.name.c_str(), (int)e.vecs.size());
  const PackedRecord::Vec& v = e.vecs[j];
  int rc = copy_name(v.name, name, name_len);
  if (rc) return rc;
  if (n) *n = v.n;
  if (out && v.n) NS_CHECK_CUDA(cudaMemcpyAsync(out, v.p, (size_t)v.n * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}

int ns2vc_check_set_launch_hook(int kind, void* handle, ns2vc_check_launch_fn fn, void* user) {
  EngineBase* e = const_cast<EngineBase*>(base_of(kind, handle, "check_set_launch_hook"));
  if (!e) return -1;
  e->hook.fn = (void*)fn;
  e->hook.user = fn ? user : nullptr;
  return 0;
}

int ns2vc_check_philox(const uint32_t* counters, const uint32_t* keys, int n, uint32_t* raw, float* normals, ns2vc_stream stream) {
  NS_REQUIRE(counters && keys && raw && normals && n >= 1, "check_philox: null argument or n = %d", n);
  philox_check_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(counters, keys, n, raw, normals);
  NS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
