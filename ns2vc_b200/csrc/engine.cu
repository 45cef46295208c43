// Denoiser engine: layer plan, weight registry + packing, per-shape launch program, C-ABI.
//
// The plan restates the block structure of the reference UNet1DConditionModel
// (unet1d/unet_1d_condition.py:421-559, forward :943-1032) — see ns2vc_b200/arch.py for the
// Python twin that the oracle uses; tests compare the two plan strings.
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

struct PlanOp {
  enum Kind { PUSH, POP_CAT, RESNET, XFORMER, DOWN, UP } kind;
  std::string prefix;
  int cin = 0, cout = 0, level = 0;
  int c1 = 0, c2 = 0;       // RESNET: channels of the running tensor and of the concatenated skip
  int site = -1;            // RESNET / XFORMER / DOWN / UP: index of its ResnetSite / XformerSite / ConvSite (set by pack_all)
  bool skip = false;        // its output is pushed as a skip (the next op is a PUSH)
};

struct ResnetSite {
  std::string p;
  int c1, c2, cin, cout;
  bool shortcut;
  PackedB conv1, conv2;      // conv2 also carries the 1x1 shortcut K-blocks
  float* bias2 = nullptr;    // conv2.bias (+ conv_shortcut.bias)
  int film_off = 0;
};
struct XformerSite {
  std::string p;
  int c;
  PackedB proj_in, qkv, out1, q2, out2, ff1;
  // ff.net.2 and proj_out have no non-linearity between them (reference attention.py:203 -> transformer_1d.py:289-295):
  //   proj_out(ff2(g) + b2 + h) + bp = g (Wp W2)^T + h Wp^T + (Wp b2 + bp)
  // so both run as ONE GEMM over K = [GEGLU output (4C) | residual stream h (C)] with the product matrix packed at load time.
  PackedB ff2p; float* bias_ff2p = nullptr;
  int kv_off = 0;            // column offset of this block's K in the cross K/V cache (all K first ...)
  int v_off = 0;             // ... then all V: column offset of this block's V
  // LayerNorm folded into the consumer GEMM (norm1 -> qkv, norm2 -> q2, norm3 -> ff1): the packed weights carry gamma,
  // g[n] = sum_c gamma_c W[n,c] and bf[n] = sum_c beta_c W[n,c] (+ bias[n]) feed the epilogue (EPI_LNFOLD)
  float* g_qkv = nullptr; float* bf_qkv = nullptr;
  float* g_q2 = nullptr; float* bf_q2 = nullptr;
  float* g_ff1 = nullptr; float* bf_ff1 = nullptr;
};
struct ConvSite { std::string p; int c; PackedB w; };

// The launch programs of one (B, T, S, ragged, workspace) key.
struct Program {
  int B = 0, T = 0, S = 0; void* ws = nullptr;
  bool ragged = false;       // per-utterance content / prompt lengths (ns2vc_unet_prepare_cond_ragged)
  RaggedTables rt{};         // ragged: the length and key-bias tables (static buffer) its prepare_cond fills
  bool has_mask = false;
  bool cond_ready = false;   // the conditioning program has run for this key since it last became active
  std::vector<Launch> prog_cond, prog_fwd;
  // ragged: entry b's conditioning alone (ns2vc_unet_prepare_cond_rows), built when b is first asked for; empty until then
  std::vector<std::vector<Launch>> prog_cond_row;
  size_t cond_end = 0;                                    // workspace offset where the conditioning's buffers end
  float* film_base = nullptr;                             // FiLM rows [B, film_total] (workspace)
  float* aug = nullptr;                                   // add_embedding output [B, ted] (workspace)
  TapSet taps;
};

}  // namespace

struct ns2vc_unet : EngineBase {
  ns2vc_unet_cfg cfg;
  int ted = 0;                                   // time_embed_dim
  std::vector<PlanOp> plan;
  bool simt = false;
  std::string plan_str;

  std::vector<ResnetSite> resnets;
  std::vector<XformerSite> xformers;
  std::vector<ConvSite> resamplers;
  PackedB convin_lat, convin_content, conv_out, kv_all;
  int kv_total = 0, k_total = 0, film_total = 0;
  float* film_W = nullptr; float* film_b = nullptr;       // concatenated time_emb_proj
  PoolKV pool_kv;                                         // concatenated k_proj | v_proj

  // Cached programs, least recently active first; the active one (if any) is progs[active].  Other keys stay cached for the
  // sub-batch lanes of a multi-stream sampler and for callers that alternate shapes.
  static constexpr size_t kMaxInactive = 16;
  std::vector<Program> progs;
  int active = -1;
  // Per-program STATIC device data (GroupNorm descriptors, nearest-upsample index tables) lives outside the caller's workspace:
  // several shapes may share one workspace, and captured graphs keep reading these tables, so they are only released when the
  // weights are re-packed or the handle is destroyed (~20 KB per shape ever seen)
  std::vector<void*> static_bufs;
  void drop_programs() {
    progs.clear();
    active = -1;
    for (void* p : static_bufs) cudaFree(p);
    static_bufs.clear();
  }
  bool profiling = false;
  const float* film_ext = nullptr;   // caller-supplied FiLM rows for one forward (replace the active program's film_base)
  unsigned long long* trace = nullptr; int trace_cap = 0;
  unsigned long long* attn_trace = nullptr; int attn_trace_cap = 0;
  unsigned long long* span = nullptr; int span_cap = 0;   // [launch][2] grid spans
  struct ProfRec { int kind; cudaEvent_t a, b; int M, N, K, nseg, ctas; };
  std::vector<ProfRec> prof;
};

namespace ns2vc {

const EngineBase* engine_base(const ns2vc_unet* h) { return h; }

// A resampler's (Downsample1D's, Upsample1D's) conv weights [C, C, 3]: tap j at k-block j nkb(C)
int pack_resample_conv(PackedB& pb, const float* w, int C, cudaStream_t st) {
  for (int j = 0; j < 3; ++j) {
    const int rc = pack_seg(pb, w, C, C, 3, j, 0, C, 0, j * nkb_of(C), 0, st);
    if (rc) return rc;
  }
  return 0;
}

DownConv down_conv(ProgramBuilder& bld, const PackedB& w, const float* bias, const float* x, const SplitBuf& raw, int Tin, int C,
                   bool views, const SplitBuf& e_buf, const SplitBuf& o_buf) {
  const int TL = (Tin - 1) / 2 + 1, To = Tin / 2;          // even rows, odd rows
  DownConv d;
  memset(&d, 0, sizeof(d));
  SplitBuf ev = e_buf, od = o_buf;
  if (views && To >= 1) {
    // the raw split seen as row PAIRS [B, ceil(Tin/2), 2*ld]: even rows are the first half of a pair, odd rows the second
    // (one row fewer when Tin is odd: rows past it are the TMA unit's zero fill).  The entries stay Tin rows apart.
    ev = raw; ev.T = TL; ev.ld = 2 * raw.ld; ev.bpitch = (long long)Tin * raw.ld;
    od = ev; od.hi += raw.ld; od.lo += raw.ld; od.T = To;
  } else {
    // E[t] = x[2t], O[t] = x[2t+1] decimated into dense splits (Tin = 1: O is one row of zeros past the input)
    for (int j = 0; j < 2; ++j) {
      PrepOp& p = d.prep[j];
      p.src1 = x; p.ld1 = C; p.C1 = C; p.B = bld.B; p.T_src = Tin; p.T_dst = j ? std::max(To, 1) : TL;
      p.row_mul = 2; p.row_add = j; p.mode = PREP_RAW; p.out = j ? od : ev;
    }
    d.nprep = 2;
  }
  d.g = bld.gemm_base(w, TL);
  const int ie = bld.add_src(d.g, ev), io = bld.add_src(d.g, od);
  bld.seg(d.g, io, 0, C, -1); bld.seg(d.g, ie, 0, C, 0); bld.seg(d.g, io, 0, C, 0);
  d.g.flags = EPI_BIAS; d.g.bias = bias;
  return d;
}

}  // namespace ns2vc

namespace {

int level_len(int T, int level) {
  for (int i = 0; i < level; ++i) T = (T - 1) / 2 + 1;
  return T;
}

void build_plan(ns2vc_unet* h) {
  const ns2vc_unet_cfg& c = h->cfg;
  const int n = c.n_levels;
  std::vector<int> skip;
  auto push = [&](int ch, int level) {
    if (!h->plan.empty()) h->plan.back().skip = true;   // (the first push keeps conv_in's output, which precedes the plan)
    PlanOp o; o.kind = PlanOp::PUSH; o.cout = ch; o.level = level; h->plan.push_back(o); skip.push_back(ch);
  };
  int ch = c.block_out_channels[0], level = 0;
  push(ch, 0);
  for (int i = 0; i < n; ++i) {
    const int cout = c.block_out_channels[i];
    for (int j = 0; j < c.layers_per_block[i]; ++j) {
      PlanOp r; r.kind = PlanOp::RESNET; r.prefix = "down_blocks." + std::to_string(i) + ".resnets." + std::to_string(j);
      r.cin = ch; r.cout = cout; r.level = level; r.c1 = ch; r.c2 = 0; h->plan.push_back(r);
      ch = cout;
      if (c.down_has_attn[i]) {
        PlanOp x; x.kind = PlanOp::XFORMER; x.prefix = "down_blocks." + std::to_string(i) + ".attentions." + std::to_string(j);
        x.cin = x.cout = ch; x.level = level; h->plan.push_back(x);
      }
      push(ch, level);
    }
    if (i != n - 1) {
      ++level;
      PlanOp d; d.kind = PlanOp::DOWN; d.prefix = "down_blocks." + std::to_string(i) + ".downsamplers.0"; d.cin = d.cout = ch; d.level = level;
      h->plan.push_back(d);
      push(ch, level);
    }
  }
  auto res = [&](const std::string& p, int c1, int c2, int cout) {
    PlanOp r; r.kind = PlanOp::RESNET; r.prefix = p; r.cin = c1 + c2; r.cout = cout; r.level = level; r.c1 = c1; r.c2 = c2; h->plan.push_back(r);
  };
  auto xf = [&](const std::string& p, int cc) {
    PlanOp x; x.kind = PlanOp::XFORMER; x.prefix = p; x.cin = x.cout = cc; x.level = level; h->plan.push_back(x);
  };
  res("mid_block.resnets.0", ch, 0, ch);
  xf("mid_block.attentions.0", ch);
  res("mid_block.resnets.1", ch, 0, ch);
  for (int i = 0; i < n; ++i) {
    const int cout = c.block_out_channels[n - 1 - i];
    const int layers = c.layers_per_block[n - 1 - i] + 1;
    for (int j = 0; j < layers; ++j) {
      const int sk = skip.back(); skip.pop_back();
      PlanOp pc; pc.kind = PlanOp::POP_CAT; pc.cin = ch; pc.cout = ch + sk; pc.level = level; h->plan.push_back(pc);
      res("up_blocks." + std::to_string(i) + ".resnets." + std::to_string(j), ch, sk, cout);
      ch = cout;
      if (c.up_has_attn[i]) xf("up_blocks." + std::to_string(i) + ".attentions." + std::to_string(j), ch);
    }
    if (i != n - 1) {
      --level;
      PlanOp u; u.kind = PlanOp::UP; u.prefix = "up_blocks." + std::to_string(i) + ".upsamplers.0"; u.cin = u.cout = ch; u.level = level;
      h->plan.push_back(u);
    }
  }
  // plan string (compared with ns2vc_b200.arch.build_plan in tests)
  static const char* kn[] = {"push", "pop_cat", "resnet", "xformer", "down", "up"};
  for (auto& o : h->plan) {
    char buf[256];
    snprintf(buf, sizeof(buf), "%s|%s|%d|%d|%d\n", kn[o.kind], o.prefix.c_str(), o.cin, o.cout, o.level);
    h->plan_str += buf;
  }
}

void register_weights(ns2vc_unet* h) {
  const ns2vc_unet_cfg& c = h->cfg;
  WeightRegistry& w = h->weights;
  const int c0 = c.block_out_channels[0], ted = h->ted, xd = c.cross_attention_dim;
  w.add_conv("conv_in", c0, c.in_channels, 3);
  w.add_lin("time_embedding.linear_1", ted, c0);
  w.add_lin("time_embedding.linear_2", ted, ted);
  if (c.add_embed_text) {
    w.add_norm("add_embedding.norm1", xd);
    w.add("add_embedding.pool.positional_embedding", {1, xd});
    w.add_lin("add_embedding.pool.k_proj", xd, xd);
    w.add_lin("add_embedding.pool.q_proj", xd, xd);
    w.add_lin("add_embedding.pool.v_proj", xd, xd);
    w.add_lin("add_embedding.proj", ted, xd);
    w.add_norm("add_embedding.norm2", ted);
  }
  for (auto& o : h->plan) {
    if (o.kind == PlanOp::RESNET) {
      const std::string& p = o.prefix;
      w.add_norm(p + ".norm1", o.cin);
      w.add_conv(p + ".conv1", o.cout, o.cin, 3);
      w.add_lin(p + ".time_emb_proj", c.time_scale_shift ? 2 * o.cout : o.cout, ted);
      w.add_norm(p + ".norm2", o.cout);
      w.add_conv(p + ".conv2", o.cout, o.cout, 3);
      if (o.cin != o.cout) w.add_conv(p + ".conv_shortcut", o.cout, o.cin, 1);
    } else if (o.kind == PlanOp::XFORMER) {
      const std::string& p = o.prefix; const int cc = o.cout;
      w.add_norm(p + ".norm", cc);
      w.add_conv(p + ".proj_in", cc, cc, 1);
      const std::string b = p + ".transformer_blocks.0";
      w.add_norm(b + ".norm1", cc);
      w.add_lin(b + ".attn1.to_q", cc, cc, false); w.add_lin(b + ".attn1.to_k", cc, cc, false); w.add_lin(b + ".attn1.to_v", cc, cc, false);
      w.add_lin(b + ".attn1.to_out.0", cc, cc);
      w.add_norm(b + ".norm2", cc);
      w.add_lin(b + ".attn2.to_q", cc, cc, false); w.add_lin(b + ".attn2.to_k", cc, xd, false); w.add_lin(b + ".attn2.to_v", cc, xd, false);
      w.add_lin(b + ".attn2.to_out.0", cc, cc);
      w.add_norm(b + ".norm3", cc);
      w.add_lin(b + ".ff.net.0.proj", 8 * cc, cc);
      w.add_lin(b + ".ff.net.2", cc, 4 * cc);
      w.add_conv(p + ".proj_out", cc, cc, 1);
    } else if (o.kind == PlanOp::DOWN || o.kind == PlanOp::UP) {
      w.add_conv(o.prefix + ".conv", o.cout, o.cin, 3);
    }
  }
  w.add_norm("conv_norm_out", c0);
  w.add_conv("conv_out", c.out_channels, c0, 3);
}

// g / bf of a [N, C] linear that consumes LayerNorm(gamma, beta) (rows n_dst0.. of the output vectors)
int ln_fold_vectors(ns2vc_unet* h, const std::string& wname, const std::string& bname, const std::string& norm, int N, int C,
                    float* g, float* bf, int n_dst0, cudaStream_t st) {
  const float* W = h->weights.W(wname); const float* ga = h->weights.W(norm + ".weight"); const float* be = h->weights.W(norm + ".bias");
  NS_REQUIRE(W && ga && be, "ln fold: %s / %s missing", wname.c_str(), norm.c_str());
  const float* bias = bname.empty() ? nullptr : h->weights.W(bname);
  return launch_ln_fold_vec(W, ga, be, bias, g + n_dst0, bf + n_dst0, N, C, st);
}

// pack_seg() of the registered weight `wname`
int pack_named(ns2vc_unet* h, PackedB& pb, const std::string& wname, int n_rows, int cin_total, int ktaps, int tap, int cin0,
               int ncin, int n_dst0, int kb0, int geglu_half, cudaStream_t st, const float* cscale = nullptr) {
  const float* w = h->weights.W(wname);
  NS_REQUIRE(w != nullptr, "pack: weight %s missing", wname.c_str());
  return pack_seg(pb, w, n_rows, cin_total, ktaps, tap, cin0, ncin, n_dst0, kb0, geglu_half, st, cscale);
}

// Wm[n, k] = sum_c Wp[n, c] W2[c, k]  (load time; double accumulation): the product matrix of ff.net.2 followed by proj_out
__global__ void matmul_nn_kernel(const float* __restrict__ Wp, const float* __restrict__ W2, float* __restrict__ Wm, int N, int Cmid, int K) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x, n = blockIdx.y;
  if (k >= K || n >= N) return;
  double acc = 0;
  for (int c = 0; c < Cmid; ++c) acc += (double)Wp[(long long)n * Cmid + c] * (double)W2[(long long)c * K + k];
  Wm[(long long)n * K + k] = (float)acc;
}
// bm[n] = sum_c Wp[n, c] b2[c] + bp[n]
__global__ void matvec_bias_kernel(const float* __restrict__ Wp, const float* __restrict__ b2, const float* __restrict__ bp, float* __restrict__ bm, int N, int Cmid) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  double acc = bp[n];
  for (int c = 0; c < Cmid; ++c) acc += (double)Wp[(long long)n * Cmid + c] * (double)b2[c];
  bm[n] = (float)acc;
}

__global__ void add_vec_kernel(const float* a, const float* b, float* o, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) o[i] = a[i] + (b ? b[i] : 0.f);
}

int pack_all(ns2vc_unet* h, cudaStream_t st) {
  const ns2vc_unet_cfg& c = h->cfg;
  const int c0 = c.block_out_channels[0];
  const int Cl = c.latent_channels, Cc = c.in_channels - c.latent_channels;
  int rc;
  // conv_in: latent part and (hoisted) content part
  {
    const int nl = nkb_of(Cl);
    if ((rc = h->mem.alloc_packed(h->convin_lat, c0, c0, 3 * nl, h->simt))) return rc;
    for (int j = 0; j < 3; ++j)
      if ((rc = pack_named(h, h->convin_lat, "conv_in.weight", c0, c.in_channels, 3, j, 0, Cl, 0, j * nl, 0, st))) return rc;
    h->packed.add("conv_in.latent", h->convin_lat);
    if (Cc > 0) {
      const int nc = nkb_of(Cc);
      if ((rc = h->mem.alloc_packed(h->convin_content, c0, c0, 3 * nc, h->simt))) return rc;
      for (int j = 0; j < 3; ++j)
        if ((rc = pack_named(h, h->convin_content, "conv_in.weight", c0, c.in_channels, 3, j, Cl, Cc, 0, j * nc, 0, st))) return rc;
      h->packed.add("conv_in.content", h->convin_content);
    }
  }
  // resnets / transformers / resamplers in plan order
  h->resnets.clear(); h->xformers.clear(); h->resamplers.clear();
  int film_off = 0, kv_off = 0;
  for (auto& o : h->plan) {
    if (o.kind == PlanOp::RESNET) {
      ResnetSite s; s.p = o.prefix; s.c1 = o.c1; s.c2 = o.c2; s.cin = o.cin; s.cout = o.cout; s.shortcut = o.cin != o.cout;
      const int ni = nkb_of(s.cin), no = nkb_of(s.cout);
      if ((rc = h->mem.alloc_packed(s.conv1, s.cout, s.cout, 3 * ni, h->simt))) return rc;
      for (int j = 0; j < 3; ++j)
        if ((rc = pack_named(h, s.conv1, s.p + ".conv1.weight", s.cout, s.cin, 3, j, 0, s.cin, 0, j * ni, 0, st))) return rc;
      const int nsc = s.shortcut ? ni : 0;
      if ((rc = h->mem.alloc_packed(s.conv2, s.cout, s.cout, 3 * no + nsc, h->simt))) return rc;
      for (int j = 0; j < 3; ++j)
        if ((rc = pack_named(h, s.conv2, s.p + ".conv2.weight", s.cout, s.cout, 3, j, 0, s.cout, 0, j * no, 0, st))) return rc;
      if (s.shortcut)
        if ((rc = pack_named(h, s.conv2, s.p + ".conv_shortcut.weight", s.cout, s.cin, 1, 0, 0, s.cin, 0, 3 * no, 0, st))) return rc;
      if (!(s.bias2 = h->mem.alloc<float>(s.cout))) return -2;
      add_vec_kernel<<<ceil_div(s.cout, 256), 256, 0, st>>>(h->weights.W(s.p + ".conv2.bias"), s.shortcut ? h->weights.W(s.p + ".conv_shortcut.bias") : nullptr, s.bias2, s.cout);
      h->packed.add(s.p + ".conv1", s.conv1);
      h->packed.add(s.p + ".conv2", s.conv2, {{"bias2", s.bias2, s.cout}});
      s.film_off = film_off;
      film_off += c.time_scale_shift ? 2 * s.cout : s.cout;
      o.site = (int)h->resnets.size();
      h->resnets.push_back(s);
    } else if (o.kind == PlanOp::XFORMER) {
      XformerSite x; x.p = o.prefix; x.c = o.cout;
      const int C = x.c, nk = nkb_of(C);
      const std::string b = x.p + ".transformer_blocks.0";
      if ((rc = h->mem.alloc_packed(x.proj_in, C, C, nk, h->simt))) return rc;
      if ((rc = pack_named(h, x.proj_in, x.p + ".proj_in.weight", C, C, 1, 0, 0, C, 0, 0, 0, st))) return rc;
      if ((rc = h->mem.alloc_packed(x.qkv, 3 * C, 3 * C, nk, h->simt))) return rc;
      const char* qkvn[3] = {".attn1.to_q.weight", ".attn1.to_k.weight", ".attn1.to_v.weight"};
      for (int i = 0; i < 3; ++i)
        if ((rc = pack_named(h, x.qkv, b + qkvn[i], C, C, 1, 0, 0, C, i * C, 0, 0, st, h->weights.W(b + ".norm1.weight")))) return rc;
      if (!(x.g_qkv = h->mem.alloc<float>((size_t)3 * C)) || !(x.bf_qkv = h->mem.alloc<float>((size_t)3 * C))) return -2;
      if (!(x.g_q2 = h->mem.alloc<float>((size_t)C)) || !(x.bf_q2 = h->mem.alloc<float>((size_t)C))) return -2;
      if (!(x.g_ff1 = h->mem.alloc<float>((size_t)8 * C)) || !(x.bf_ff1 = h->mem.alloc<float>((size_t)8 * C))) return -2;
      for (int i = 0; i < 3; ++i)
        if ((rc = ln_fold_vectors(h, b + qkvn[i], "", b + ".norm1", C, C, x.g_qkv, x.bf_qkv, i * C, st))) return rc;
      if ((rc = ln_fold_vectors(h, b + ".attn2.to_q.weight", "", b + ".norm2", C, C, x.g_q2, x.bf_q2, 0, st))) return rc;
      if ((rc = ln_fold_vectors(h, b + ".ff.net.0.proj.weight", b + ".ff.net.0.proj.bias", b + ".norm3", 8 * C, C, x.g_ff1, x.bf_ff1, 0, st))) return rc;
      if ((rc = h->mem.alloc_packed(x.out1, C, C, nk, h->simt))) return rc;
      if ((rc = pack_named(h, x.out1, b + ".attn1.to_out.0.weight", C, C, 1, 0, 0, C, 0, 0, 0, st))) return rc;
      if ((rc = h->mem.alloc_packed(x.q2, C, C, nk, h->simt))) return rc;
      if ((rc = pack_named(h, x.q2, b + ".attn2.to_q.weight", C, C, 1, 0, 0, C, 0, 0, 0, st, h->weights.W(b + ".norm2.weight")))) return rc;
      if ((rc = h->mem.alloc_packed(x.out2, C, C, nk, h->simt))) return rc;
      if ((rc = pack_named(h, x.out2, b + ".attn2.to_out.0.weight", C, C, 1, 0, 0, C, 0, 0, 0, st))) return rc;
      NS_REQUIRE((4 * C) % 64 == 0, "transformer width %d: 4C must be a multiple of 64", C);
      if ((rc = h->mem.alloc_packed(x.ff1, 4 * C, 8 * C, nk, h->simt))) return rc;
      if ((rc = pack_named(h, x.ff1, b + ".ff.net.0.proj.weight", 8 * C, C, 1, 0, 0, C, 0, 0, 4 * C, st, h->weights.W(b + ".norm3.weight")))) return rc;
      {
        // proj_out o ff.net.2 as one operator: K blocks [Wp W2 over the 4C GEGLU channels | Wp over the C residual channels]
        const float* Wp = h->weights.W(x.p + ".proj_out.weight"); const float* W2 = h->weights.W(b + ".ff.net.2.weight");
        NS_REQUIRE(Wp && W2, "pack: %s feed-forward / proj_out weights missing", x.p.c_str());
        float* Wm = nullptr;
        if (!(Wm = h->mem.alloc<float>((size_t)C * 4 * C)) || !(x.bias_ff2p = h->mem.alloc<float>((size_t)C))) return -2;
        matmul_nn_kernel<<<dim3(ceil_div(4 * C, 128), C), 128, 0, st>>>(Wp, W2, Wm, C, C, 4 * C);
        matvec_bias_kernel<<<ceil_div(C, 128), 128, 0, st>>>(Wp, h->weights.W(b + ".ff.net.2.bias"), h->weights.W(x.p + ".proj_out.bias"), x.bias_ff2p, C, C);
        if ((rc = h->mem.alloc_packed(x.ff2p, C, C, nkb_of(4 * C) + nk, h->simt))) return rc;
        if ((rc = pack_seg(x.ff2p, Wm, C, 4 * C, 1, 0, 0, 4 * C, 0, 0, 0, st))) return rc;
        if ((rc = pack_named(h, x.ff2p, x.p + ".proj_out.weight", C, C, 1, 0, 0, C, 0, nkb_of(4 * C), 0, st))) return rc;
        h->packed.add(x.p + ".proj_in", x.proj_in);
        h->packed.add(x.p + ".qkv", x.qkv, {{"g_qkv", x.g_qkv, 3 * C}, {"bf_qkv", x.bf_qkv, 3 * C}});
        h->packed.add(x.p + ".out1", x.out1);
        h->packed.add(x.p + ".q2", x.q2, {{"g_q2", x.g_q2, C}, {"bf_q2", x.bf_q2, C}});
        h->packed.add(x.p + ".out2", x.out2);
        h->packed.add(x.p + ".ff1", x.ff1, {{"g_ff1", x.g_ff1, 8 * C}, {"bf_ff1", x.bf_ff1, 8 * C}});
        h->packed.add(x.p + ".ff2p", x.ff2p, {{"Wm", Wm, (long long)C * 4 * C}, {"bias_ff2p", x.bias_ff2p, C}});
      }
      x.kv_off = kv_off;
      kv_off += C;
      o.site = (int)h->xformers.size();
      h->xformers.push_back(x);
    } else if (o.kind == PlanOp::DOWN || o.kind == PlanOp::UP) {
      ConvSite s; s.p = o.prefix; s.c = o.cout;
      const float* w = h->weights.W(s.p + ".conv.weight");
      NS_REQUIRE(w != nullptr, "pack: weight %s missing", (s.p + ".conv.weight").c_str());
      if ((rc = h->mem.alloc_packed(s.w, s.c, s.c, 3 * nkb_of(s.c), h->simt))) return rc;
      if ((rc = pack_resample_conv(s.w, w, s.c, st))) return rc;
      h->packed.add(s.p + ".conv", s.w);
      o.site = (int)h->resamplers.size();
      h->resamplers.push_back(s);
    }
  }
  h->film_total = film_off;
  h->k_total = kv_off;                                   // cache columns: [K of every block | V of every block]
  for (auto& x : h->xformers) x.v_off = h->k_total + x.kv_off;
  h->kv_total = 2 * kv_off;
  // conv_out
  {
    const int nk = nkb_of(c0);
    if ((rc = h->mem.alloc_packed(h->conv_out, c.out_channels, c.out_channels, 3 * nk, h->simt))) return rc;
    for (int j = 0; j < 3; ++j)
      if ((rc = pack_named(h, h->conv_out, "conv_out.weight", c.out_channels, c0, 3, j, 0, c0, 0, j * nk, 0, st))) return rc;
    h->packed.add("conv_out", h->conv_out);
  }
  // all cross-attention K|V projections as one GEMM over the prompt
  if (h->kv_total > 0) {
    const int xd = c.cross_attention_dim;
    if ((rc = h->mem.alloc_packed(h->kv_all, h->kv_total, h->kv_total, nkb_of(xd), h->simt))) return rc;
    for (auto& x : h->xformers) {
      const std::string b = x.p + ".transformer_blocks.0";
      if ((rc = pack_named(h, h->kv_all, b + ".attn2.to_k.weight", x.c, xd, 1, 0, 0, xd, x.kv_off, 0, 0, st))) return rc;
      if ((rc = pack_named(h, h->kv_all, b + ".attn2.to_v.weight", x.c, xd, 1, 0, 0, xd, x.v_off, 0, 0, st))) return rc;
    }
    h->packed.add("kv_all", h->kv_all);
  }
  // concatenated FiLM projection [film_total, ted]
  if (!(h->film_W = h->mem.alloc<float>((size_t)h->film_total * h->ted))) return -2;
  if (!(h->film_b = h->mem.alloc<float>((size_t)h->film_total))) return -2;
  for (auto& s : h->resnets) {
    const int rows = c.time_scale_shift ? 2 * s.cout : s.cout;
    NS_CHECK_CUDA(cudaMemcpyAsync(h->film_W + (size_t)s.film_off * h->ted, h->weights.W(s.p + ".time_emb_proj.weight"), (size_t)rows * h->ted * 4, cudaMemcpyDeviceToDevice, st));
    NS_CHECK_CUDA(cudaMemcpyAsync(h->film_b + s.film_off, h->weights.W(s.p + ".time_emb_proj.bias"), (size_t)rows * 4, cudaMemcpyDeviceToDevice, st));
  }
  h->packed.add("time_emb_proj", PackedB{}, {{"film_W", h->film_W, (long long)h->film_total * h->ted}, {"film_b", h->film_b, h->film_total}});
  if (c.add_embed_text) {
    const int xd = c.cross_attention_dim;
    if ((rc = concat_pool_kv(h->mem, h->weights, "add_embedding.pool", xd, h->pool_kv, st))) return rc;
    h->packed.add("add_embedding.pool.kv", PackedB{}, {{"W", h->pool_kv.W, 2LL * xd * xd}, {"b", h->pool_kv.b, 2LL * xd}});
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------
// Program construction
// ---------------------------------------------------------------------------------------------
// ATen nearest_idx (UpSample.h), as ns2vc_nearest_index() below; IEEE fp32 division / product / floor: bit-identical on host and device
__global__ void nearest_index_kernel(int t_in, int t_out, int* idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= t_out) return;
  idx[i] = nearest_src_index(i, t_in, t_out);
}

// The timestep path over M rows of timesteps `t` as small linears into temb1, emb [M, ted] and film [M, film_total]; returns their
// number (the FiLM projection only when some resnet has one).  Reference embeddings.py:24-64, 157-218 (sinusoid -> linear_1 ->
// SiLU -> linear_2), unet_1d_condition.py:869-883 (+ aug_emb: row m adds row m % B of `aug`), resnet.py:619-629 (time_emb_proj
// of SiLU(emb) for every resnet at once).
int time_path_ops(const ns2vc_unet* h, const float* t, int M, int B, const float* aug, float* temb1, float* emb, float* film, LinOp ops[3]) {
  const ns2vc_unet_cfg& c = h->cfg;
  const int ted = h->ted;
  ops[0] = linear_op(t, 1, M, c.block_out_channels[0], h->weights.W("time_embedding.linear_1.weight"), h->weights.W("time_embedding.linear_1.bias"),
                     ted, temb1, ted);
  ops[0].in_mode = LIN_SINUSOID; ops[0].flip_sin_to_cos = c.flip_sin_to_cos; ops[0].freq_shift = c.freq_shift; ops[0].out_silu = 1;
  ops[1] = linear_op(temb1, ted, M, ted, h->weights.W("time_embedding.linear_2.weight"), h->weights.W("time_embedding.linear_2.bias"), ted, emb, ted);
  if (c.add_embed_text) { ops[1].add = aug; ops[1].add_ld = ted; ops[1].add_rows = B; }
  if (h->film_total <= 0) return 2;
  ops[2] = linear_op(emb, ted, M, ted, h->film_W, h->film_b, h->film_total, film, h->film_total);
  ops[2].in_mode = LIN_SILU;
  return 3;
}

// An activation that leaves a block: fp32 token-major tensor, its raw bf16 hi/lo split (the A operand of the panel-mode
// GEMMs that consume it; written by the same epilogue) and the per-(b, channel) sums for the consumer's GroupNorm.
struct Act { float* p = nullptr; SplitBuf sp{}; int c = 0; double* st = nullptr; };

// The forward's scratch, shared by every block: each block views these at its own level's rows and width (Builder::reserve_forward).
struct Scratch {
  float* rot[3]; SplitBuf rot_sp[3];   // outputs of the blocks whose output no skip keeps, in rotation, and their raw splits
  float *H1, *T0, *T1, *QKV;
  SplitBuf SP_A, SP_R, SP_H, SP_X, SP_ATT, SP_FF, SP_QKV, SP_LN;
};

// Builds the conditioning and forward programs of one (B, T, S, ragged, workspace) key into `pg`: emit_cond, then
// reserve_forward, emit_entry, one emitter per plan op in plan order and emit_head.  Each step takes its buffers from the
// workspace arena and the static buffer as it goes, so this order fixes every offset.
struct Builder : ProgramBuilder {
  ns2vc_unet* h;
  Program& pg;
  const int T, S;
  const bool ragged;
  std::vector<int> Tl;                                     // rows per entry at each level
  const bool xf_on;                                        // panel mode is possible (wgmma backend)
  const int* rag_lens = nullptr;                           // ragged programs: content lengths [B] (device), else nullptr
  const int* rag_plens = nullptr;                          // ragged programs: prompt lengths [B] (device), else nullptr
  Arena sar;                                               // the program's static buffer (see ns2vc_unet::static_bufs)
  // conditioning outputs the forward reads
  float* P = nullptr;                                      // conv_in(content) + bias
  float* kvc = nullptr;                                    // cross-attention K | V of every transformer
  SplitBuf kvs{};                                          // the same cache as bf16 hi/lo (attention v2 reads it by TMA)
  float* maskbias = nullptr;
  float* aug = nullptr;                                    // add_embedding output [B, ted]
  // per-step buffers of the forward
  SplitBuf s_xin{};
  float* temb1 = nullptr; float* emb = nullptr; float* film = nullptr;
  // per-(b, channel) sum | sum-of-squares of every fp32 activation that feeds a GroupNorm, accumulated by the producing GEMM
  // epilogues; one contiguous arena, zeroed by one memset at the top of the forward
  double* stat_arena = nullptr;
  size_t stat_doubles = 0, stat_used = 0;
  Scratch sc{};
  // the walk: the running activation, the skip stack and the skip popped for the next resnet's concat
  Act cur, cat2;
  std::vector<Act> skips;
  int rot_i = 0;

  Builder(ns2vc_unet* h_, Program& pg_, void* ws, int B_, int T_, int S_, bool ragged_)
      : ProgramBuilder{Arena{(uint8_t*)ws, 0}, B_, ws == nullptr, h_->simt, &pg_.prog_cond}, h(h_), pg(pg_), T(T_), S(S_),
        ragged(ragged_), Tl(h_->cfg.n_levels), xf_on(!h_->simt) {
    for (int l = 0; l < (int)Tl.size(); ++l) Tl[l] = level_len(T, l);
  }

  void conv3(GemmOp& g, const SplitBuf& s) {           // k=3, stride 1, pad 1 over one split source
    const int i = add_src(g, s);
    for (int j = 0; j < 3; ++j) seg(g, i, 0, s.C, j - 1);
  }
  void emit_gemm(GemmOp& g, const PackedB& w, Launch::Input in = Launch::NONE) {
    if (g.xmode) {
      // few-tile, deep-K launches (the two coarsest levels at B = 8: 64 tiles of 24-64 k-blocks each): two CTAs per tile, each
      // half of the channel blocks; worth it when both halves still have a few panels and all pairs are resident at once
      const int tiles = B * ceil_div(g.T_out, 128) * (w.Npad / 64);
      int panels = 0;
      for (int i = 0; i < g.nxs; ++i) panels += g.xs[i].ncb;
      if (2 * tiles <= gemm_sm_count() && panels >= 8) g.ksplit = 2;
    }
    Launch& l = ProgramBuilder::emit_gemm(g, w, in);
    if (g.pre_film || (g.flags & EPI_ROWBIAS)) l.reads_film = 1;
  }
  // GroupNorm descriptors of the panel-mode GEMMs: one array in the static buffer, copied to the device in ONE copy when the
  // program is complete
  std::vector<PrepOp> aff_host; PrepOp* aff_dev = nullptr; int aff_cap = 0;
  void reserve_affine(int n) { aff_cap = n; aff_dev = sar.get<PrepOp>((size_t)n); aff_host.reserve(n); }
  int upload_affine(cudaStream_t st) {
    if (dry || aff_host.empty()) return 0;
    // pageable source: the runtime stages it before returning, so the vector may die with the builder
    return cudaMemcpyAsync(aff_dev, aff_host.data(), aff_host.size() * sizeof(PrepOp), cudaMemcpyHostToDevice, st) == cudaSuccess ? 0 : -2;
  }
  void emit_prep(const float* s1, int C1, const float* s2, int C2, int T_src, int T_dst, int mode, const float* scale,
                 const float* shift, const SplitBuf& o, const SplitBuf* raw = nullptr, int row_mul = 1, int row_add = 0,
                 const int* rowmap = nullptr, Launch::Input in = Launch::NONE) {
    PrepOp p; memset(&p, 0, sizeof(p));
    p.src1 = s1; p.ld1 = C1; p.C1 = C1; p.src2 = s2; p.ld2 = C2; p.C2 = C2; p.B = B; p.T_src = T_src; p.T_dst = T_dst;
    p.row_mul = row_mul; p.row_add = row_add; p.rowmap = rowmap; p.mode = mode; p.scale = scale; p.shift = shift; p.out = o;
    if (raw) p.raw = *raw;
    emit(Launch::PREP, p, in);
  }

  // ragged programs: rows past each entry's length (every level derives its own: ceil(T_b / 2^l)) are zeros
  void rag(GemmOp& g, int level) const { g.row_len = rag_lens; g.len_shift = level; }
  void rag_prep(const int* len, int level) { PrepOp& p = out->back().get<PrepOp>(); p.row_len = len; p.len_shift = level; }
  double* new_stats(int C) { return new_rowstats((size_t)B * C); }   // per-(b, channel) sums | sums of squares
  double* new_rowstats(size_t nrows) { double* p = stat_arena ? stat_arena + stat_used : nullptr; stat_used += 2 * nrows; return p; }
  void with_stats(GemmOp& g, double* st_, int C) const { g.flags |= EPI_STATS; g.stat_sum = st_; g.stat_sq = st_ ? st_ + (size_t)B * C : nullptr; }
  SplitBuf scratch_split(size_t elems) { SplitBuf s{}; s.hi = ar.get<__nv_bfloat16>(elems); s.lo = ar.get<__nv_bfloat16>(elems); return s; }

  // fp16 softmax weights (one P x [V_hi | V_lo] MMA per k-step) only where enough keys average their 2^-12 rounding out: over a few
  // dozen keys (short prompts, the coarsest levels of short utterances) the weights are a bf16 hi/lo split - those launches are
  // cheap anyway.  Measured on the reference's 40-step pipeline fixture (S = 40): worst err/tol 1.35 with fp16 weights everywhere.
  // Only self-attention uses fp16 weights.  Cross-attention keeps the split whatever its key count: a key count cannot see how
  // sharp the prompt attention is, and with fp16 weights in both attentions, scores of std ~4 (tests/test_numerics_fp64.py,
  // regime 'sharp' at B=4, T=1024, S=256) put the output at 1.51x the elementwise tolerance against fp64 on an H100.
  // Ragged programs never use them: entry b of a self-attention attends over its own T_b,l keys, known only on the device, and
  // one built program serves every length vector, so the padded T_l says nothing about how many keys average the rounding.
  static constexpr int kFp16MinKeys = 256;
  bool p16(int keys) const { return !ragged && attention_v2_p_fp16() && keys >= kFp16MinKeys; }

  // Can the GroupNorm in front of a GEMM over (cur [+ skip]) channels run inside the GEMM?  (64-channel blocks may not
  // straddle the concat seam; the affine table holds kXfMaxC channels)
  bool xf_ok(int c1, int c2) const { return xf_on && (c2 == 0 || c1 % 64 == 0) && c1 + c2 <= kXfMaxC && h->cfg.norm_num_groups <= 64; }

  // The GroupNorm(+FiLM)(+SiLU) of one or two concatenated producers (statistics from their epilogues) as the A operand of `g`,
  // a conv of `taps` taps (3: k3 p1, or 1).  Panel mode (`panel`, which xf_ok allows): the GEMM reads the producers' raw splits
  // and normalises them with the descriptor, parked in the static buffer; the FiLM rows travel in GemmOp::pre_film.  Otherwise
  // the descriptor is a prep launch into `o` (with `raw`: also the input's raw split, for a prep-mode shortcut) and the GEMM
  // reads `o` in plain segments.
  void normed_input(GemmOp& g, bool panel, const Act& a1, const Act& a2, const std::string& norm, float eps, int mode,
                    const float* film, int film_ld, int taps, int level, const SplitBuf& o, const SplitBuf* raw = nullptr) {
    const int Tn = Tl[level], C = a1.c + a2.c;
    PrepOp p; memset(&p, 0, sizeof(p));
    p.C1 = a1.c; p.C2 = a2.c; p.B = B; p.T_src = Tn; p.T_dst = Tn; p.mode = mode; p.row_len = rag_lens; p.len_shift = level;
    set_group_norm(p, B, a1.st, a1.c, a2.st, a2.c, Tn, h->cfg.norm_num_groups, eps, h->weights.W(norm + ".weight"),
                   h->weights.W(norm + ".bias"), panel ? nullptr : film, film_ld);
    if (panel) {
      const int kb_stride = taps == 1 ? 0 : nkb_of(C);       // k-blocks per tap
      const int i1 = add_src(g, a1.sp);
      xseg(g, i1, 0, a1.c, taps, 0, kb_stride, 1, 0);
      if (a2.c) { const int i2 = add_src(g, a2.sp); xseg(g, i2, 0, a2.c, taps, nkb_of(a1.c), kb_stride, 1, a1.c); }
      g.pre_film = film;
      if ((int)aff_host.size() >= aff_cap) { err = -1; set_error("internal: affine descriptor table full"); return; }
      aff_host.push_back(p);
      g.pre = aff_dev ? aff_dev + (aff_host.size() - 1) : reinterpret_cast<const PrepOp*>(uintptr_t(16));   // (dry run: any non-null value)
    } else {
      p.src1 = a1.p; p.ld1 = a1.c; p.src2 = a2.p; p.ld2 = a2.c; p.row_mul = 1; p.out = o;
      if (raw) p.raw = *raw;
      emit(Launch::PREP, p).reads_film = film != nullptr;
      const int i = add_src(g, o);
      for (int j = 0; j < taps; ++j) seg(g, i, 0, C, j - taps / 2);
    }
  }

  // The GEMM `g` that ends a block at `level` writes the block's output of C channels: fp32, (panel mode) its raw split and its
  // statistics, into a buffer of its own when a skip keeps it, else into the next of the three rotating ones; ragged rows past
  // each entry's length are zeros.  The output becomes the running activation, tapped as `name`.
  void emit_block_out(GemmOp& g, const PackedB& w, int level, int C, bool is_skip, const std::string& name) {
    const int TL = Tl[level];
    Act a; a.c = C;
    if (is_skip) { a.p = ar.get<float>((size_t)B * TL * C); if (xf_on) a.sp = view(scratch_split((size_t)B * TL * pad_to(C, 8)), TL, C); }
    else { a.p = sc.rot[rot_i]; if (xf_on) a.sp = view(sc.rot_sp[rot_i], TL, C); rot_i = (rot_i + 1) % 3; }
    a.st = new_stats(C);
    g.flags |= EPI_OUT_F32; g.out = a.p; g.out_ld = C;
    if (xf_on) { g.flags |= EPI_OUT_SPLIT; g.out_hi = a.sp.hi; g.out_lo = a.sp.lo; g.out_split_ld = a.sp.ld; }
    with_stats(g, a.st, C);
    rag(g, level);
    emit_gemm(g, w);
    cur = a;
    emit_tap(pg.taps, name, a.p, level, C, TL);
  }

  // ================= conditioning program =================
  // conv_in of the content, the cross-attention K | V of every transformer over the prompt, the mask bias and the pooled prompt
  // embedding; its outputs stay in the workspace for every forward
  void emit_cond() {
    const ns2vc_unet_cfg& c = h->cfg;
    const int c0 = c.block_out_channels[0], Cc = c.in_channels - c.latent_channels, xd = c.cross_attention_dim, ted = h->ted;
    const int* plens = rag_plens;
    P = (Cc > 0) ? ar.get<float>((size_t)B * T * c0) : nullptr;
    kvc = ar.get<float>((size_t)B * S * std::max(h->kv_total, 1));
    kvs.T = S; kvs.C = std::max(h->kv_total, 8); kvs.ld = pad_to(kvs.C, 8);
    kvs.hi = ar.get<__nv_bfloat16>((size_t)B * S * kvs.ld);
    kvs.lo = ar.get<__nv_bfloat16>((size_t)B * S * kvs.ld);
    maskbias = ar.get<float>((size_t)B * S);
    aug = ar.get<float>((size_t)B * ted);
    // conditioning scratch
    const SplitBuf s_content = (Cc > 0) ? split(T, Cc) : SplitBuf{};
    const SplitBuf s_prompt = split(S, xd);
    TextTimeEmbedding tte;
    tte.reserve(ar, B, S, xd, ted);

    if (Cc > 0) {
      emit(Launch::NCT2SPLIT, NctSplitOp{nullptr, 0, B, Cc, T, s_content, rag_lens, nullptr, 0}, Launch::CONTENT);
      GemmOp g = gemm_base(h->convin_content, T);
      conv3(g, s_content);
      g.flags = EPI_BIAS | EPI_OUT_F32; g.bias = h->weights.W("conv_in.bias"); g.out = P; g.out_ld = c0;
      emit_gemm(g, h->convin_content);
    }
    emit(Launch::MASKBIAS, MaskBiasOp{nullptr, B * S, maskbias}, Launch::MASK);
    if (h->kv_total > 0) {
      emit_prep(nullptr, xd, nullptr, 0, S, S, PREP_RAW, nullptr, nullptr, s_prompt, nullptr, 1, 0, nullptr, Launch::PROMPT);
      rag_prep(plens, 0);                                    // (ragged: prompt frames past S_b are zeros, so is their K / V)
      GemmOp g = lin(h->kv_all, s_prompt, S);
      g.flags = EPI_OUT_F32 | EPI_OUT_SPLIT; g.out = kvc; g.out_ld = h->kv_total;
      g.out_hi = kvs.hi; g.out_lo = kvs.lo; g.out_split_ld = kvs.ld;   // (V stays a bf16 split: cross-attention weights are split)
      emit_gemm(g, h->kv_all);
    }
    if (c.add_embed_text)   // TextTimeEmbedding of the prompt (embeddings.py:421-434)
      tte.emit(*this, h->weights, "add_embedding", nullptr, Launch::PROMPT, S, xd, ted, c.add_embed_heads, Launch::POOL_ATT, h->pool_kv, aug, plens);
  }

  // ================= forward program =================
  // per-step buffers, the statistics arena and the scratch the blocks share
  void reserve_forward() {
    const ns2vc_unet_cfg& c = h->cfg;
    const int c0 = c.block_out_channels[0];
    s_xin = split(T, c.latent_channels);
    temb1 = ar.get<float>((size_t)B * h->ted);
    emb = ar.get<float>((size_t)B * h->ted);
    film = ar.get<float>((size_t)B * std::max(h->film_total, 1));
    stat_doubles = (size_t)2 * B * c0;
    for (auto& o : h->plan) {
      if (o.kind == PlanOp::RESNET) stat_doubles += (size_t)4 * B * o.cout;
      else if (o.kind == PlanOp::XFORMER || o.kind == PlanOp::DOWN || o.kind == PlanOp::UP) stat_doubles += (size_t)2 * B * o.cout;
      if (o.kind == PlanOp::XFORMER) stat_doubles += (size_t)3 * 2 * B * Tl[o.level];   // three LayerNorm row-statistics buffers
    }
    stat_arena = ar.get<double>(stat_doubles);
    // activation buffers
    size_t max_act = (size_t)B * T * c0, max_cat = 0, max_ff = 1, max_qkv = 1;
    for (auto& o : h->plan) {
      const size_t rows = (size_t)B * Tl[o.level];
      if (o.kind == PlanOp::RESNET) { max_act = std::max(max_act, rows * o.cout); max_cat = std::max(max_cat, rows * o.cin); }
      if (o.kind == PlanOp::DOWN || o.kind == PlanOp::UP) { max_act = std::max(max_act, rows * o.cout); max_cat = std::max(max_cat, rows * o.cout); }
      if (o.kind == PlanOp::XFORMER) { max_act = std::max(max_act, rows * o.cout); max_ff = std::max(max_ff, rows * 4 * o.cout); max_qkv = std::max(max_qkv, rows * 3 * o.cout); }
    }
    max_cat = std::max(max_cat, max_act);
    for (int i = 0; i < 3; ++i) sc.rot[i] = ar.get<float>(max_act);
    sc.H1 = ar.get<float>(max_act);
    sc.T0 = ar.get<float>(max_act);
    sc.T1 = ar.get<float>(max_act);
    sc.QKV = ar.get<float>(max_qkv);
    sc.SP_A = scratch_split(max_cat);      // conv1 / resample input
    sc.SP_R = scratch_split(max_cat);      // raw shortcut operand / odd rows of a stride-2 conv
    sc.SP_H = scratch_split(max_act);      // conv2 input, out-head input
    sc.SP_X = scratch_split(max_act);      // GN-normalised transformer input (when the GroupNorm is a prep launch)
    sc.SP_ATT = scratch_split(max_act);    // attention output
    sc.SP_FF = scratch_split(max_ff);      // GEGLU output
    sc.SP_QKV = scratch_split(max_qkv);    // q | k | v of the self-attention (q of the cross-attention)
    sc.SP_LN = scratch_split(max_act);     // raw (un-normalised) split of the transformer's residual stream (folded LayerNorms)
    for (int i = 0; i < 3; ++i) sc.rot_sp[i] = xf_on ? scratch_split(max_act) : SplitBuf{};   // (panel mode only)
  }

  // entry: the statistics memset, x -> split tokens, the time path and conv_in (whose output is the first skip)
  void emit_entry() {
    const ns2vc_unet_cfg& c = h->cfg;
    const int c0 = c.block_out_channels[0], Cc = c.in_channels - c.latent_channels;
    emit_memset(stat_arena, stat_doubles * sizeof(double));
    emit(Launch::NCT2SPLIT, NctSplitOp{nullptr, 0, B, c.latent_channels, T, s_xin, rag_lens, nullptr, 0}, Launch::X);
    LinOp tp[3];
    const int n = time_path_ops(h, nullptr, B, B, aug, temb1, emb, film, tp);
    for (int i = 0; i < n; ++i) emit_linear(tp[i], i == 0 ? Launch::T : Launch::NONE, 1);

    GemmOp g = gemm_base(h->convin_lat, T);
    conv3(g, s_xin);
    if (Cc > 0) { g.flags |= EPI_RESIDUAL; g.res = P; g.res_ld = c0; }
    else { g.flags |= EPI_BIAS; g.bias = h->weights.W("conv_in.bias"); }
    emit_block_out(g, h->convin_lat, 0, c0, true, "conv_in");
  }

  // ResnetBlock1D (reference resnet.py:597-612): norm1 + SiLU -> conv1 (+ FiLM bias) -> norm2 (+ FiLM scale / shift) + SiLU ->
  // conv2, plus the block input or its 1x1 conv_shortcut.  The input is the running tensor, concatenated in the up path with
  // the popped skip.  Panel mode normalises both inputs inside the convs, with no fp32 h; the 1x1 shortcut reads the raw splits
  // of the block input(s) as extra 1-tap segments.  Otherwise two prep launches, the first also writing the input's raw split
  // for the shortcut.  The whole block takes one mode: conv2's shortcut reads the input as conv1's mode leaves it.
  void emit_resnet(const PlanOp& o) {
    const ns2vc_unet_cfg& c = h->cfg;
    const ResnetSite& s = h->resnets[o.site];
    const int TL = Tl[o.level];
    const bool panel = xf_ok(s.c1, s.c2) && xf_ok(s.cout, 0);
    const SplitBuf a_h = view(sc.SP_H, TL, s.cout), a_raw = view(sc.SP_R, TL, s.cin);
    const Act h1{sc.H1, a_h, s.cout, new_stats(s.cout)};   // conv1's output: its raw split (panel mode) or fp32
    {
      GemmOp g = gemm_base(s.conv1, TL);
      normed_input(g, panel, cur, cat2, s.p + ".norm1", c.norm_eps, PREP_AFFINE_SILU, nullptr, 0, 3, o.level, view(sc.SP_A, TL, s.cin),
                   s.shortcut ? &a_raw : nullptr);
      g.flags = EPI_BIAS; g.bias = h->weights.W(s.p + ".conv1.bias");
      if (!c.time_scale_shift) { g.flags |= EPI_ROWBIAS; g.rowbias = film + s.film_off; g.rowbias_ld = h->film_total; }
      if (panel) { g.flags |= EPI_OUT_SPLIT; g.out_hi = a_h.hi; g.out_lo = a_h.lo; g.out_split_ld = a_h.ld; }
      else { g.flags |= EPI_OUT_F32; g.out = h1.p; g.out_ld = s.cout; }
      with_stats(g, h1.st, s.cout);
      rag(g, o.level);
      emit_gemm(g, s.conv1);
    }
    {
      GemmOp g = gemm_base(s.conv2, TL);
      // panel mode: the raw 1x1 shortcut panels go first: their MMAs run while the transform warps still derive the GroupNorm affine
      if (s.shortcut && panel) {
        const int no = nkb_of(s.cout), n1 = nkb_of(s.c1);
        const int a0 = add_src(g, cur.sp);
        xseg(g, a0, 0, s.c1, 1, 3 * no, 0, 0, 0);
        if (s.c2) { const int a1 = add_src(g, cat2.sp); xseg(g, a1, 0, s.c2, 1, 3 * no + n1, 0, 0, 0); }
      }
      normed_input(g, panel, h1, Act{}, s.p + ".norm2", c.norm_eps, PREP_AFFINE_SILU, c.time_scale_shift ? film + s.film_off : nullptr,
                   h->film_total, 3, o.level, a_h);
      if (s.shortcut && !panel) { const int i = add_src(g, a_raw); seg(g, i, 0, s.cin, 0); }
      g.flags |= EPI_BIAS; g.bias = s.bias2;
      if (!s.shortcut) { g.flags |= EPI_RESIDUAL; g.res = cur.p; g.res_ld = s.c1; }
      emit_block_out(g, s.conv2, o.level, s.cout, o.skip, s.p);
    }
    cat2 = Act{};
  }

  // Transformer1DModel with one BasicTransformerBlock (reference transformer_1d.py, attention.py)
  void emit_xformer(const PlanOp& o) {
    const XformerSite& x = h->xformers[o.site];
    const int TL = Tl[o.level], C = x.c, H = h->cfg.num_heads, dh = C / H;
    const size_t rows = (size_t)B * TL;
    const std::string b = x.p + ".transformer_blocks.0";
    const SplitBuf satt = view(sc.SP_ATT, TL, C), sff = view(sc.SP_FF, TL, 4 * C);
    // Folded LayerNorms (reference attention.py:83,102,118 nn.LayerNorm): proj_in, out1 and out2 each emit the raw split of
    // the residual stream into `sln` and its per-row sums; qkv, q2 and ff1 read `sln` - no LayerNorm kernel, no extra pass.
    const SplitBuf sln = view(sc.SP_LN, TL, C);
    double* rs1 = new_rowstats(rows); double* rs2 = new_rowstats(rows); double* rs3 = new_rowstats(rows);
    { GemmOp g = gemm_base(x.proj_in, TL);              // GroupNorm (eps 1e-6) of the block input, then proj_in
      normed_input(g, xf_ok(C, 0), cur, Act{}, x.p + ".norm", 1e-6f, PREP_AFFINE, nullptr, 0, 1, o.level, view(sc.SP_X, TL, C));
      g.flags = EPI_BIAS | EPI_OUT_F32; g.bias = h->weights.W(x.p + ".proj_in.bias"); g.out = sc.T0; g.out_ld = C;
      emits_ln_input(g, sln, rs1);
      rag(g, o.level);
      emit_gemm(g, x.proj_in); }
    const bool av2 = !h->simt && attention_v2_supported(dh, TL, false) && attention_v2_supported(dh, S, true);
    const SplitBuf sqkv = view(sc.SP_QKV, TL, 3 * C), sq2 = view(sc.SP_QKV, TL, C);
    { GemmOp g = lin(x.qkv, sln, TL);
      if (av2) { g.flags = EPI_OUT_SPLIT; g.out_hi = sqkv.hi; g.out_lo = sqkv.lo; g.out_split_ld = sqkv.ld;
                 if (p16(TL)) g.f16_col0 = 2 * C; }
      else { g.flags = EPI_OUT_F32; g.out = sc.QKV; g.out_ld = 3 * C; }
      consumes_ln(g, rs1, x.g_qkv, x.bf_qkv, C);
      emit_gemm(g, x.qkv); }
    { AttnOp a; memset(&a, 0, sizeof(a));
      a.q = sc.QKV; a.q_ld = 3 * C; a.k = sc.QKV + C; a.k_ld = 3 * C; a.v = sc.QKV + 2 * C; a.v_ld = 3 * C;
      a.out_hi = satt.hi; a.out_lo = satt.lo; a.out_split_ld = satt.ld;
      a.B = B; a.H = H; a.Tq = TL; a.Tk = TL; a.dh = dh; a.scale = 1.0f / sqrtf((float)dh);
      // ragged: v2 attends over each entry's own keys (per-entry key count); the fp32 kernel takes a 0 / -inf key bias
      if (ragged && av2) { a.key_len = rag_lens; a.key_shift = o.level; }
      else if (ragged) a.bias = pg.rt.key_bias[o.level];
      if (av2) { a.v2 = 1; a.p_split = p16(TL) ? 0 : 1; a.qs = sqkv; a.ks = sqkv; a.vs = sqkv; a.q_c0 = 0; a.k_c0 = C; a.v_c0 = 2 * C; }
      emit_attention(a); }
    { GemmOp g = lin(x.out1, satt, TL); g.flags = EPI_BIAS | EPI_RESIDUAL | EPI_OUT_F32; g.bias = h->weights.W(b + ".attn1.to_out.0.bias"); g.res = sc.T0; g.res_ld = C; g.out = sc.T1; g.out_ld = C;
      emits_ln_input(g, sln, rs2);
      emit_gemm(g, x.out1); }
    { GemmOp g = lin(x.q2, sln, TL);
      if (av2) { g.flags = EPI_OUT_SPLIT; g.out_hi = sq2.hi; g.out_lo = sq2.lo; g.out_split_ld = sq2.ld; }
      else { g.flags = EPI_OUT_F32; g.out = sc.QKV; g.out_ld = C; }
      consumes_ln(g, rs2, x.g_q2, x.bf_q2, C);
      emit_gemm(g, x.q2); }
    { AttnOp a; memset(&a, 0, sizeof(a));
      a.q = sc.QKV; a.q_ld = C; a.k = kvc + x.kv_off; a.k_ld = h->kv_total; a.v = kvc + x.v_off; a.v_ld = h->kv_total; a.bias = maskbias;
      a.out_hi = satt.hi; a.out_lo = satt.lo; a.out_split_ld = satt.ld;
      a.B = B; a.H = H; a.Tq = TL; a.Tk = S; a.dh = dh; a.scale = 1.0f / sqrtf((float)dh);
      if (av2) { a.v2 = 1; a.p_split = 1; a.qs = sq2; a.ks = kvs; a.vs = kvs; a.q_c0 = 0; a.k_c0 = x.kv_off; a.v_c0 = x.v_off; }
      if (ragged) { a.bias = pg.rt.prompt_bias; emit_attention(a); }   // the prompt-length bias of the ragged tables
      else emit_attention(a, Launch::MASK); }     // the key-padding bias comes from the call's mask (dropped without one)
    { GemmOp g = lin(x.out2, satt, TL); g.flags = EPI_BIAS | EPI_RESIDUAL | EPI_OUT_F32; g.bias = h->weights.W(b + ".attn2.to_out.0.bias"); g.res = sc.T1; g.res_ld = C; g.out = sc.T0; g.out_ld = C;
      emits_ln_input(g, sln, rs3);
      emit_gemm(g, x.out2); }
    { GemmOp g = lin(x.ff1, sln, TL); g.flags = EPI_GEGLU | EPI_OUT_SPLIT;
      g.out_hi = sff.hi; g.out_lo = sff.lo; g.out_split_ld = sff.ld;
      consumes_ln(g, rs3, x.g_ff1, x.bf_ff1, C); g.flags &= ~EPI_BIAS;   // GEGLU reads its (folded) biases through g.bias itself
      emit_gemm(g, x.ff1); }
    { // ff.net.2 + proj_out as one GEMM over K = [GEGLU output | residual stream]:  out = g (Wp W2)^T + h Wp^T + (Wp b2 + bp) + x_in
      GemmOp g = gemm_base(x.ff2p, TL);
      const int i0 = add_src(g, sff); seg(g, i0, 0, 4 * C, 0);
      const int i1 = add_src(g, sln); seg(g, i1, 0, C, 0);          // raw split of the residual stream, written by out2's epilogue
      g.flags = EPI_BIAS | EPI_RESIDUAL; g.bias = x.bias_ff2p; g.res = cur.p; g.res_ld = C;
      emit_block_out(g, x.ff2p, o.level, C, o.skip, x.p); }
  }

  // Downsample1D: conv k3 s2 p1 (down_conv): in panel mode over row-pair views of the block input's raw split, else (and at
  // Tin = 1) over its even and odd rows decimated by two prep launches.
  void emit_down(const PlanOp& o) {
    const ConvSite& s = h->resamplers[o.site];
    const int TL = Tl[o.level], Tin = Tl[o.level - 1];
    DownConv d = down_conv(*this, s.w, h->weights.W(s.p + ".conv.bias"), cur.p, cur.sp, Tin, s.c, xf_on, view(sc.SP_A, TL, s.c),
                           view(sc.SP_R, std::max(Tin / 2, 1), s.c));
    for (int i = 0; i < d.nprep; ++i) emit(Launch::PREP, d.prep[i]);
    emit_block_out(d.g, s.w, o.level, s.c, o.skip, s.p);
  }

  // Upsample1D: nearest-neighbour 2x (to the finer level's length), then conv k3 p1
  int emit_up(const PlanOp& o, cudaStream_t st) {
    const ConvSite& s = h->resamplers[o.site];
    const int TL = Tl[o.level], Tin = Tl[o.level + 1];
    // nearest-neighbour source rows of F.interpolate(size=TL) (reference resnet.py:160): a table in the static buffer, filled on
    // the device with the same fp32 rule as ns2vc_nearest_index() (stream-ordered: no allocation, no host sync)
    int* map_d = sar.get<int>((size_t)TL);
    if (!dry) {
      nearest_index_kernel<<<ceil_div(TL, 256), 256, 0, st>>>(Tin, TL, map_d);
      NS_CHECK_CUDA(cudaGetLastError());
    }
    const SplitBuf up = view(sc.SP_A, TL, s.c);
    emit_prep(cur.p, s.c, nullptr, 0, Tin, TL, PREP_RAW, nullptr, nullptr, up, nullptr, 1, 0, map_d);
    // ragged: each entry's rows come from its OWN (T_b,l+1 -> T_b,l) nearest rule (the padded table can differ from it in
    // fp32), and rows past the entry's length at this level are zeros
    rag_prep(rag_lens, o.level);
    GemmOp g = gemm_base(s.w, TL);
    conv3(g, up);
    g.flags = EPI_BIAS; g.bias = h->weights.W(s.p + ".conv.bias");
    emit_block_out(g, s.w, o.level, s.c, o.skip, s.p);
    return 0;
  }

  // output head: GN -> SiLU -> conv_out, stored channel-major [B, out_channels, T]
  void emit_head() {
    const ns2vc_unet_cfg& c = h->cfg;
    const int c0 = c.block_out_channels[0];
    GemmOp g = gemm_base(h->conv_out, T);
    normed_input(g, xf_ok(c0, 0), cur, Act{}, "conv_norm_out", c.norm_eps, PREP_AFFINE_SILU, nullptr, 0, 3, 0, view(sc.SP_H, T, c0));
    g.flags = EPI_BIAS | EPI_OUT_NCT; g.bias = h->weights.W("conv_out.bias"); g.out = nullptr;
    rag(g, 0);                                             // (ragged: output frames past T_b are exact zeros)
    emit_gemm(g, h->conv_out, Launch::OUT);
  }
};

// Builds the programs of (B, T, S, ragged, ws) into *prog, or (ws == nullptr) sizes their workspace into *bytes_out.
// A ragged program takes no more workspace than the padded one: its tables live in the program's static buffer.
int build_programs(ns2vc_unet* h, int B, int T, int S, void* ws, size_t* bytes_out, Program* prog, cudaStream_t st = nullptr,
                   bool ragged = false) {
  const int nlev = h->cfg.n_levels;
  const bool dry = (ws == nullptr);
  Program pg;
  Builder bld(h, pg, ws, B, T, S, ragged);
  const std::vector<int>& Tl = bld.Tl;
  NS_REQUIRE(Tl[nlev - 1] >= 1 && T >= 1 && B >= 1 && S >= 1, "bad shape B=%d T=%d S=%d", B, T, S);
  NS_REQUIRE(!ragged || (!h->simt && nlev <= kRagMaxLevels), "ragged programs need the wgmma backend and at most %d levels", kRagMaxLevels);
  std::vector<bool> xf_level(nlev, false);                 // levels with a transformer (their self-attention needs a key bias)
  for (auto& o : h->plan) if (o.kind == PlanOp::XFORMER) xf_level[o.level] = true;

  if (!dry) {
    // building a program allocates its static tables and copies them to the device: illegal under stream capture (header contract:
    // run a new shape once eagerly first)
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(st, &cs) == cudaSuccess && cs != cudaStreamCaptureStatusNone) {
      set_error("the first call for a new (B=%d, T=%d, S=%d, workspace) builds its launch program and must not run under stream capture", B, T, S);
      return -1;
    }
  }
  {
    const int n_aff = 2 * (int)h->resnets.size() + (int)h->xformers.size() + 2;
    size_t sbytes = 1024 + (size_t)n_aff * sizeof(PrepOp);
    for (auto& o : h->plan) if (o.kind == PlanOp::UP) sbytes += 256 + (size_t)Tl[o.level] * sizeof(int);
    if (ragged) {
      sbytes += 512 + (size_t)2 * B * sizeof(int) + (size_t)B * S * sizeof(float);
      for (int l = 0; l < nlev; ++l) if (xf_level[l]) sbytes += 256 + (size_t)B * Tl[l] * sizeof(float);
    }
    if (!dry) {
      void* sb = nullptr;
      NS_CHECK_CUDA(cudaMalloc(&sb, sbytes));
      h->static_bufs.push_back(sb);
      bld.sar = Arena{(uint8_t*)sb, 0};
    }
    bld.reserve_affine(n_aff);
    if (ragged) {
      pg.ragged = true;
      RaggedTables& rt = pg.rt;
      rt.B = B; rt.T = T; rt.S = S; rt.nlev = nlev;
      rt.lens = bld.sar.get<int>((size_t)2 * B);           // content lengths [B] | prompt lengths [B]
      rt.prompt_bias = bld.sar.get<float>((size_t)B * S);
      for (int l = 0; l < nlev; ++l) { rt.Tl[l] = Tl[l]; rt.key_bias[l] = xf_level[l] ? bld.sar.get<float>((size_t)B * Tl[l]) : nullptr; }
      bld.rag_lens = rt.lens;
      bld.rag_plens = rt.lens + B;
    }
  }

  bld.emit_cond();
  pg.cond_end = bld.ar.off;
  bld.out = &pg.prog_fwd;
  bld.reserve_forward();
  bld.emit_entry();
  for (const PlanOp& o : h->plan) {
    switch (o.kind) {
      case PlanOp::PUSH: bld.skips.push_back(bld.cur); break;
      case PlanOp::POP_CAT: bld.cat2 = bld.skips.back(); bld.skips.pop_back(); break;
      case PlanOp::RESNET: bld.emit_resnet(o); break;
      case PlanOp::XFORMER: bld.emit_xformer(o); break;
      case PlanOp::DOWN: bld.emit_down(o); break;
      case PlanOp::UP: { const int rc = bld.emit_up(o, st); if (rc) return rc; break; }
    }
  }
  bld.emit_head();

  if (!bld.err && bld.upload_affine(st)) { set_error("affine descriptor upload failed"); return -2; }
  if (bld.err) return bld.err;
  if (bytes_out) *bytes_out = bld.ar.off + 256;
  if (!dry) {
    pg.B = B; pg.T = T; pg.S = S; pg.ws = ws;
    pg.film_base = bld.film; pg.aug = bld.aug;
    *prog = std::move(pg);
  }
  return 0;
}

// Entry b's conditioning program of the ragged program `pg`: emit_cond at B = 1 over row b of every buffer the full program
// placed there (an Arena row view of the same workspace), reading entry b's lengths.  Each of its launches is row-local:
// the GEMMs' tiles, the split and prep rows, the LayerNorm rows, the small linears' rows and the pooling CTAs each cover one
// entry, and no ragged launch reads another entry's length.  So it writes the bytes the full program writes for row b, and
// nothing of any other row.
int build_cond_row(ns2vc_unet* h, Program& pg, int b) {
  Builder rb(h, pg, pg.ws, 1, pg.T, pg.S, true);
  rb.ar.rows = (size_t)pg.B; rb.ar.row = (size_t)b;
  std::vector<Launch> prog;
  rb.out = &prog;
  rb.rag_lens = pg.rt.lens + b;
  rb.rag_plens = pg.rt.lens + pg.B + b;
  rb.emit_cond();
  if (rb.err) return rb.err;
  // every buffer emit_cond takes must be [B, ...]: then the row view ends where the full build's conditioning ended
  NS_REQUIRE(rb.ar.off == pg.cond_end, "internal: entry %d's conditioning ends at workspace offset %zu, the full program's at %zu",
             b, rb.ar.off, pg.cond_end);
  pg.prog_cond_row[b] = std::move(prog);
  return 0;
}

// Checks a caller's list of n distinct entries of a batch of B.
int check_rows(const int* rows, int n, int B, const char* fn) {
  NS_REQUIRE(n >= 0 && n <= B && (rows || n == 0), "%s: %d rows of a batch of %d", fn, n, B);
  std::vector<char> seen((size_t)B, 0);
  for (int i = 0; i < n; ++i) {
    NS_REQUIRE(rows[i] >= 0 && rows[i] < B, "%s: row %d out of range [0, %d)", fn, rows[i], B);
    NS_REQUIRE(!seen[rows[i]], "%s: row %d listed twice", fn, rows[i]);
    seen[rows[i]] = 1;
  }
  return 0;
}

// Runs `prog` over the call arguments `in`.  Before Runner launches a record, the denoiser's own patches go into a copy of it:
// the FiLM rows of ns2vc_unet_forward_film, the cross-attention without a mask, and the span / trace / profiling diagnostics.
int run_program(ns2vc_unet* h, const Program& pg, const std::vector<Launch>& prog, const CallArgs& in, cudaStream_t st) {
  int rc = 0, count = 0, gemm_idx = 0, attn_idx = 0;
  // Precomputed FiLM rows (ns2vc_unet_time_table): the timestep path of this forward is skipped and every reader is rebased.
  const float* film_ext = h->film_ext;
  auto rebase = [&](const float* p) { return (film_ext && p) ? film_ext + (p - pg.film_base) : p; };
  const Runner run{h->simt, &pg.taps, st};
  Launch tmp;
  for (const Launch& rec : prog) {
    if (film_ext && rec.time_path) continue;
    cudaEvent_t ev_a = nullptr, ev_b = nullptr;
    const bool prof = h->profiling && rec.kind != Launch::TAP;
    if (prof) {
      cudaEventCreate(&ev_a); cudaEventCreate(&ev_b);
      cudaEventRecord(ev_a, st);
    }
    unsigned long long* span = (h->span && count < h->span_cap) ? h->span + 2 * count : nullptr;
    const Launch* l = bound(rec, in, tmp, rc);
    auto patched = [&]() { if (l != &tmp) { tmp = rec; l = &tmp; } return &tmp; };
    bool skip = false;
    switch (rec.kind) {
      case Launch::GEMM:
        if (film_ext && rec.reads_film) {
          GemmOp& g = patched()->get<GemmOp>();
          g.rowbias = rebase(g.rowbias);
          g.pre_film = rebase(g.pre_film);
        }
        if (span) patched()->get<GemmOp>().span = span;
        if (h->trace && gemm_idx < h->trace_cap) patched()->get<GemmOp>().trace = h->trace + 32 * gemm_idx;
        ++gemm_idx;
        break;
      case Launch::ATTN:
        if (rec.input == Launch::MASK && !pg.has_mask) patched()->get<AttnOp>().bias = nullptr;
        if (span) patched()->get<AttnOp>().span = span;
        if (h->attn_trace && attn_idx < h->attn_trace_cap) patched()->get<AttnOp>().trace = h->attn_trace + 2048 * attn_idx;
        ++attn_idx;
        break;
      case Launch::PREP:
        if (film_ext && rec.reads_film) { PrepOp& p = patched()->get<PrepOp>(); p.gn.film = rebase(p.gn.film); }
        if (span) patched()->get<PrepOp>().span = span;
        break;
      case Launch::NCT2SPLIT:   // the forward's first launch: it warms the step's FiLM rows into L2
        if (film_ext && rec.input == Launch::X) { NctSplitOp& o = patched()->get<NctSplitOp>(); o.warm = film_ext; o.warm_bytes = (long long)pg.B * h->film_total * 4; }
        break;
      case Launch::MASKBIAS: skip = !in[Launch::MASK].p; break;   // no mask: the cross-attention runs without the bias
      default: break;
    }
    const int index = (int)(&rec - prog.data());
    if (!rc && !skip && h->hook.fn) rc = observe_launch(h->hook, index, 0, *l, st);
    if (!rc && !skip) {
      rc = run.run(*l);
      if (rc == kEngineKind) rc = no_launcher(rec);
    }
    if (!rc && !skip && h->hook.fn) rc = observe_launch(h->hook, index, 1, *l, st);
    if (prof) {
      cudaEventRecord(ev_b, st);
      ns2vc_unet::ProfRec pr{(int)rec.kind, ev_a, ev_b, 0, 0, 0, 0, 0};
      if (rec.kind == Launch::GEMM) { const GemmOp& g = rec.get<GemmOp>(); pr.M = g.B * g.T_out; pr.N = g.n_valid; pr.K = g.nkb_total * 64; pr.nseg = g.nseg; }
      if (rec.kind == Launch::PREP) { const PrepOp& p = rec.get<PrepOp>(); pr.M = p.B * p.T_dst; pr.N = p.C1 + p.C2; }
      if (rec.kind == Launch::ATTN) { const AttnOp& a = rec.get<AttnOp>(); pr.M = a.Tq; pr.N = a.Tk; pr.K = a.dh; }
      h->prof.push_back(pr);
    }
    if (rc) return rc;
    if (rec.tap_index < 0 && !skip) ++count;
  }
  h->last_launches = count;
  return 0;
}

// Make the program for (B,T,S,ragged,ws) the active one, building it if it is not cached.
int ensure_program(ns2vc_unet* h, int B, int T, int S, void* ws, cudaStream_t st, bool ragged = false) {
  NS_REQUIRE(h->finalized, "ns2vc_unet_finalize() has not been called");
  NS_REQUIRE(ws != nullptr, "workspace is NULL");
  auto is = [&](const Program& p) { return p.B == B && p.T == T && p.S == S && p.ws == ws && p.ragged == ragged; };
  if (h->active >= 0) {
    if (is(h->progs[h->active])) return 0;
    // programs of different shapes may share one workspace (the caller's grow-only scratch buffer): the conditioning an inactive
    // program prepared is gone once another program has run there, so it must be prepared again when it comes back
    h->progs[h->active].cond_ready = false;
    h->active = -1;
  }
  auto it = std::find_if(h->progs.begin(), h->progs.end(), is);
  if (it != h->progs.end()) {
    std::rotate(it, it + 1, h->progs.end());             // most recently active last
  } else {
    Program p;
    const int rc = build_programs(h, B, T, S, ws, nullptr, &p, st, ragged);
    if (rc) return rc;
    // bounded: drop the least recently active program (it owns no device memory: everything lives in its workspace)
    if (h->progs.size() > ns2vc_unet::kMaxInactive) h->progs.erase(h->progs.begin());
    h->progs.push_back(std::move(p));
  }
  h->active = (int)h->progs.size() - 1;
  return 0;
}

// forward / forward_film / time_table run the variant the last prepare_cond of this (B,T,S,ws) chose: ragged or padded.  When
// another key has run since, neither variant is prepared any more; the call then takes the variant that is cached (the ragged
// one only if it is the sole one), so that it fails on the missing prepare_cond without building a program for nothing.
int ensure_program_for_call(ns2vc_unet* h, int B, int T, int S, void* ws, cudaStream_t st) {
  auto key = [&](const Program& p) { return p.B == B && p.T == T && p.S == S && p.ws == ws; };
  bool ragged = false;
  if (h->active >= 0 && key(h->progs[h->active])) {
    ragged = h->progs[h->active].ragged;
  } else {
    bool have_padded = false, have_ragged = false;
    for (const Program& p : h->progs) if (key(p)) (p.ragged ? have_ragged : have_padded) = true;
    ragged = have_ragged && !have_padded;
  }
  return ensure_program(h, B, T, S, ws, st, ragged);
}

}  // namespace

// =============================================================================================
// C-ABI
// =============================================================================================
extern "C" {

const char* ns2vc_last_error(void) { return ns2vc::get_error(); }

const char* ns2vc_build_info(void) { return "ns2vc_b200 sm_90a wgmma/3xBF16 engine, built " __DATE__ " " __TIME__; }

int ns2vc_down_length(int t) { return (t - 1) / 2 + 1; }

int ns2vc_nearest_index(int t_in, int t_out, int* idx) {
  // ATen nearest_idx (UpSample.h): identity if sizes match, >>1 for exact 2x, else
  // min(int(floorf(dst * (float)in/out)), in-1) with the scale held in fp32.
  if (t_in <= 0 || t_out <= 0 || !idx) { ns2vc::set_error("nearest_index: bad sizes %d -> %d", t_in, t_out); return -1; }
  const float scale = (float)t_in / (float)t_out;
  for (int i = 0; i < t_out; ++i) {
    int s;
    if (t_out == t_in) s = i;
    else if (t_out == 2 * t_in) s = i >> 1;
    else s = std::min((int)floorf((float)i * scale), t_in - 1);
    idx[i] = s;
  }
  return 0;
}

int ns2vc_unet_create(const ns2vc_unet_cfg* cfg, ns2vc_unet** out) {
  NS_REQUIRE(cfg && out, "null argument");
  NS_REQUIRE(cfg->n_levels >= 1 && cfg->n_levels <= NS2VC_MAX_LEVELS, "n_levels %d out of range", cfg->n_levels);
  NS_REQUIRE(cfg->latent_channels >= 1 && cfg->latent_channels <= cfg->in_channels, "latent_channels %d invalid", cfg->latent_channels);
  for (int i = 0; i < cfg->n_levels; ++i) {
    const int c = cfg->block_out_channels[i];
    NS_REQUIRE(c % cfg->norm_num_groups == 0 && c % cfg->num_heads == 0 && c % 16 == 0,
               "block width %d must be divisible by groups %d, heads %d and 16", c, cfg->norm_num_groups, cfg->num_heads);
    NS_REQUIRE(cfg->layers_per_block[i] >= 1, "layers_per_block must be >= 1");
  }
  NS_REQUIRE(cfg->cross_attention_dim % 8 == 0, "cross_attention_dim must be a multiple of 8");
  if (cfg->add_embed_text)
    NS_REQUIRE(cfg->cross_attention_dim % cfg->add_embed_heads == 0 && cfg->cross_attention_dim / cfg->add_embed_heads <= 16,
               "addition_embed heads %d unsupported for dim %d", cfg->add_embed_heads, cfg->cross_attention_dim);
  ns2vc_unet* h = new ns2vc_unet();
  h->cfg = *cfg;
  h->ted = 4 * cfg->block_out_channels[0];
  const char* be = getenv("NS2VC_GEMM_BACKEND");
  h->simt = be && strcmp(be, "simt") == 0;
  build_plan(h);
  register_weights(h);
  *out = h;
  return 0;
}

void ns2vc_unet_destroy(ns2vc_unet* h) { destroy_engine(h); }
int ns2vc_unet_num_weights(const ns2vc_unet* h) { return num_weights(h); }
int ns2vc_unet_weight_info(const ns2vc_unet* h, int i, const char** name, int64_t shape[4], int* ndim) { return weight_info(h, i, name, shape, ndim); }
int ns2vc_unet_load_weight(ns2vc_unet* h, const char* key, const float* dptr, const int64_t* shape, int ndim, ns2vc_stream stream) {
  return load_weight(h, key, dptr, shape, ndim, (cudaStream_t)stream);
}
int ns2vc_unet_finalize(ns2vc_unet* h, ns2vc_stream stream) { return finalize_engine(h, [&] { return pack_all(h, (cudaStream_t)stream); }); }

int ns2vc_unet_workspace_bytes(const ns2vc_unet* h, int B, int T, int S, size_t* bytes) {
  NS_REQUIRE(h && bytes, "null argument");
  NS_REQUIRE(h->finalized, "ns2vc_unet_finalize() has not been called");
  return build_programs(const_cast<ns2vc_unet*>(h), B, T, S, nullptr, bytes, nullptr);
}

int ns2vc_unet_prepare_cond(ns2vc_unet* h, const float* content, long long content_bstride, const float* prompt, const uint8_t* mask,
                            int B, int T, int S, void* ws, ns2vc_stream stream) {
  NS_REQUIRE(h && prompt, "null argument");
  int rc = ensure_program(h, B, T, S, ws, (cudaStream_t)stream);
  if (rc) return rc;
  const int Cc = h->cfg.in_channels - h->cfg.latent_channels;
  NS_REQUIRE(Cc == 0 || content != nullptr, "content is NULL but the model has %d content channels", Cc);
  Program& pg = h->progs[h->active];
  pg.has_mask = mask != nullptr;
  CallArgs in{};
  in[Launch::CONTENT] = {content, content_bstride}; in[Launch::PROMPT] = {prompt}; in[Launch::MASK] = {mask};
  rc = run_program(h, pg, pg.prog_cond, in, (cudaStream_t)stream);
  if (rc) return rc;
  pg.cond_ready = true;
  return 0;
}

int ns2vc_unet_prepare_cond_ragged(ns2vc_unet* h, const float* content, long long content_bstride, const float* prompt,
                                   const int64_t* content_lengths, const int64_t* prompt_lengths, int B, int T, int S, void* ws,
                                   ns2vc_stream stream) {
  NS_REQUIRE(h && prompt && content_lengths && prompt_lengths, "null argument");
  int rc = ensure_program(h, B, T, S, ws, (cudaStream_t)stream, true);
  if (rc) return rc;
  const int Cc = h->cfg.in_channels - h->cfg.latent_channels;
  NS_REQUIRE(Cc == 0 || content != nullptr, "content is NULL but the model has %d content channels", Cc);
  Program& pg = h->progs[h->active];
  pg.has_mask = false;                                     // (the cross-attention reads the ragged program's prompt-length bias)
  rc = launch_ragged_tables(reinterpret_cast<const long long*>(content_lengths), reinterpret_cast<const long long*>(prompt_lengths), pg.rt,
                            (cudaStream_t)stream);
  if (rc) return rc;
  CallArgs in{};
  in[Launch::CONTENT] = {content, content_bstride}; in[Launch::PROMPT] = {prompt};
  rc = run_program(h, pg, pg.prog_cond, in, (cudaStream_t)stream);
  if (rc) return rc;
  pg.cond_ready = true;
  return 0;
}

int ns2vc_unet_prepare_cond_rows(ns2vc_unet* h, const float* content, long long content_bstride, const float* prompt,
                                 const int64_t* content_lengths, const int64_t* prompt_lengths, const int* rows, int n_rows, int B,
                                 int T, int S, void* ws, ns2vc_stream stream) {
  NS_REQUIRE(h && prompt && content_lengths && prompt_lengths, "null argument");
  int rc = check_rows(rows, n_rows, B, "ns2vc_unet_prepare_cond_rows");
  if (rc) return rc;
  rc = ensure_program(h, B, T, S, ws, (cudaStream_t)stream, true);
  if (rc) return rc;
  const int Cc = h->cfg.in_channels - h->cfg.latent_channels;
  NS_REQUIRE(Cc == 0 || content != nullptr, "content is NULL but the model has %d content channels", Cc);
  Program& pg = h->progs[h->active];
  NS_REQUIRE(pg.cond_ready, "ns2vc_unet_prepare_cond_ragged() must have prepared the same (B,T,S,workspace) before ns2vc_unet_prepare_cond_rows()");
  const cudaStream_t st = (cudaStream_t)stream;
  const long long* clen = reinterpret_cast<const long long*>(content_lengths);
  const long long* plen = reinterpret_cast<const long long*>(prompt_lengths);
  if (n_rows == B) {                                       // every entry: the full program writes exactly these rows
    if ((rc = launch_ragged_tables(clen, plen, pg.rt, st))) return rc;
    CallArgs in{};
    in[Launch::CONTENT] = {content, content_bstride}; in[Launch::PROMPT] = {prompt};
    return run_program(h, pg, pg.prog_cond, in, st);
  }
  if (pg.prog_cond_row.empty()) pg.prog_cond_row.resize(B);
  const size_t prompt_row = (size_t)S * h->cfg.cross_attention_dim;
  int launches = 0;
  for (int i = 0; i < n_rows; ++i) {
    const int b = rows[i];
    if (pg.prog_cond_row[b].empty() && (rc = build_cond_row(h, pg, b))) return rc;
    if ((rc = launch_ragged_tables(clen, plen, pg.rt, st, b, 1))) return rc;
    CallArgs in{};
    in[Launch::CONTENT] = {content ? content + (size_t)b * content_bstride : nullptr, content_bstride};
    in[Launch::PROMPT] = {prompt + (size_t)b * prompt_row};
    if ((rc = run_program(h, pg, pg.prog_cond_row[b], in, st))) return rc;
    launches += 1 + h->last_launches;
  }
  h->last_launches = launches;
  return 0;
}

int ns2vc_unet_forward(ns2vc_unet* h, const float* x, long long x_bstride, const float* t, float* out, int B, int T, int S, void* ws,
                       ns2vc_stream stream) {
  NS_REQUIRE(h && x && t && out, "null argument");
  int rc0 = ensure_program_for_call(h, B, T, S, ws, (cudaStream_t)stream);
  if (rc0) return rc0;
  const Program& pg = h->progs[h->active];
  NS_REQUIRE(pg.cond_ready, "ns2vc_unet_prepare_cond%s() must be called with the same (B,T,S,workspace) before forward", pg.ragged ? "_ragged" : "");
  CallArgs in{};
  in[Launch::X] = {x, x_bstride}; in[Launch::T] = {t}; in[Launch::OUT] = {out};
  return run_program(h, pg, pg.prog_fwd, in, (cudaStream_t)stream);
}

int ns2vc_unet_film_width(const ns2vc_unet* h) { return h ? h->film_total : -1; }

size_t ns2vc_unet_time_table_floats(const ns2vc_unet* h, int n_rows) {
  if (!h || n_rows <= 0) return 0;
  return (size_t)n_rows * ((size_t)std::max(h->film_total, 1) + 2 * (size_t)h->ted);
}

int ns2vc_unet_time_table(ns2vc_unet* h, const float* t_rows, int n_rows, float* table, int B, int T, int S, void* ws, ns2vc_stream stream) {
  NS_REQUIRE(h && t_rows && table, "null argument");
  NS_REQUIRE(n_rows > 0 && n_rows % B == 0, "time table: %d rows is not a multiple of the batch %d", n_rows, B);
  int rc = ensure_program_for_call(h, B, T, S, ws, (cudaStream_t)stream);
  if (rc) return rc;
  const Program& pg = h->progs[h->active];
  NS_REQUIRE(pg.cond_ready || !h->cfg.add_embed_text, "ns2vc_unet_prepare_cond() must precede ns2vc_unet_time_table() (the pooled prompt embedding is added to every row)");
  float* film = table;
  float* temb1 = table + (size_t)n_rows * std::max(h->film_total, 1);
  float* emb = temb1 + (size_t)n_rows * h->ted;
  LinOp tp[3];
  const int n = time_path_ops(h, t_rows, n_rows, B, pg.aug, temb1, emb, film, tp);
  for (int i = 0; i < n; ++i)
    if ((rc = launch_small_linear(tp[i], (cudaStream_t)stream))) return rc;
  return 0;
}

int ns2vc_unet_time_table_rows(ns2vc_unet* h, const float* t_rows, int n_steps, const int* rows, int n_rows, float* table, int B, int T,
                               int S, void* ws, ns2vc_stream stream) {
  NS_REQUIRE(h && t_rows && table, "null argument");
  NS_REQUIRE(n_steps > 0, "time table rows: %d steps", n_steps);
  int rc = check_rows(rows, n_rows, B, "ns2vc_unet_time_table_rows");
  if (rc) return rc;
  rc = ensure_program_for_call(h, B, T, S, ws, (cudaStream_t)stream);
  if (rc) return rc;
  const Program& pg = h->progs[h->active];
  NS_REQUIRE(pg.cond_ready || !h->cfg.add_embed_text, "ns2vc_unet_prepare_cond() must precede ns2vc_unet_time_table_rows() (the pooled prompt embedding is added to every row)");
  // ns2vc_unet_time_table's layout for n_steps x B rows; entry b's rows k * B + b are one strided M = n_steps pass per linear
  // (the small linear computes each row on its own, so a row is the same at any M and pitch)
  const int M = n_steps * B, ted = h->ted, fw = h->film_total;
  float* film = table;
  float* temb1 = table + (size_t)M * std::max(fw, 1);
  float* emb = temb1 + (size_t)M * ted;
  if (n_rows == B) {                                       // every entry: the whole table, three launches
    LinOp tp[3];
    const int n = time_path_ops(h, t_rows, M, B, pg.aug, temb1, emb, film, tp);
    for (int j = 0; j < n; ++j)
      if ((rc = launch_small_linear(tp[j], (cudaStream_t)stream))) return rc;
    return 0;
  }
  for (int i = 0; i < n_rows; ++i) {
    const int b = rows[i];
    LinOp tp[3];
    const int n = time_path_ops(h, t_rows + b, n_steps, 1, pg.aug ? pg.aug + (size_t)b * ted : nullptr, temb1 + (size_t)b * ted,
                                emb + (size_t)b * ted, film + (size_t)b * std::max(fw, 1), tp);
    tp[0].x_ld = B; tp[0].out_ld = B * ted;
    tp[1].x_ld = B * ted; tp[1].out_ld = B * ted;
    if (n > 2) { tp[2].x_ld = B * ted; tp[2].out_ld = B * fw; }
    for (int j = 0; j < n; ++j)
      if ((rc = launch_small_linear(tp[j], (cudaStream_t)stream))) return rc;
  }
  return 0;
}

int ns2vc_unet_forward_film(ns2vc_unet* h, const float* x, long long x_bstride, const float* film_rows, float* out, int B, int T, int S,
                            void* ws, ns2vc_stream stream) {
  NS_REQUIRE(h && x && film_rows && out, "null argument");
  int rc0 = ensure_program_for_call(h, B, T, S, ws, (cudaStream_t)stream);
  if (rc0) return rc0;
  const Program& pg = h->progs[h->active];
  NS_REQUIRE(pg.cond_ready, "ns2vc_unet_prepare_cond%s() must be called with the same (B,T,S,workspace) before forward", pg.ragged ? "_ragged" : "");
  NS_REQUIRE(h->film_total > 0, "the model has no FiLM rows");
  h->film_ext = film_rows;
  CallArgs in{};
  in[Launch::X] = {x, x_bstride}; in[Launch::OUT] = {out};
  const int rc = run_program(h, pg, pg.prog_fwd, in, (cudaStream_t)stream);
  h->film_ext = nullptr;
  return rc;
}

int ns2vc_mask_bias(const uint8_t* mask, int n, float* bias, ns2vc_stream stream) {
  NS_REQUIRE(mask && bias && n >= 0, "bad argument");
  return launch_mask_bias(MaskBiasOp{mask, n, bias}, (cudaStream_t)stream);
}

int ns2vc_unet_num_taps(const ns2vc_unet* h) { return h ? (h->active >= 0 ? h->progs[h->active].taps.size() : 0) : -1; }
int ns2vc_unet_tap_info(const ns2vc_unet* h, int i, const char** name, int* level, int* channels) {
  NS_REQUIRE(h && h->active >= 0, "tap index %d out of range", i);
  return h->progs[h->active].taps.info(i, name, level, channels);
}
int ns2vc_unet_set_tap(ns2vc_unet* h, int i, float* dst) {
  NS_REQUIRE(h && h->active >= 0, "tap index %d out of range", i);
  return h->progs[h->active].taps.set(i, dst);
}
int ns2vc_unet_set_attn_trace(ns2vc_unet* h, unsigned long long* dbuf, int n_launches) {
  if (!h) return -1;
  h->attn_trace = dbuf; h->attn_trace_cap = n_launches;
  return 0;
}
int ns2vc_unet_set_trace(ns2vc_unet* h, unsigned long long* dbuf, int n_gemms) {
  NS_REQUIRE(h, "null handle");
  h->trace = dbuf; h->trace_cap = n_gemms;
  return 0;
}
int ns2vc_unet_set_span_trace(ns2vc_unet* h, unsigned long long* dbuf, int n_launches) {
  NS_REQUIRE(h, "null handle");
  h->span = dbuf; h->span_cap = n_launches;
  return 0;
}
int ns2vc_unet_launch_kind(const ns2vc_unet* h, int i) {
  if (!h || i < 0 || h->active < 0) return -1;
  int c = 0;
  for (auto& l : h->progs[h->active].prog_fwd) {
    if (l.kind == Launch::TAP) continue;
    if (c == i) return (int)l.kind;
    ++c;
  }
  return -1;
}
int ns2vc_unet_set_profiling(ns2vc_unet* h, int on) {
  NS_REQUIRE(h, "null handle");
  h->profiling = on != 0;
  return 0;
}
// the denoiser's profiled kinds: every Launch::Kind before TAP (taps are copies, not kernels)
static const char* const kKindNames[] = {"gemm_tc", "attention", "ln_split", "ln_apply", "small_linear", "nct_to_split",   // = Launch::Kind order
                                         "pool_class_token", "pool_attend", "mask_bias", "prep_split", "memset"};
static_assert(sizeof(kKindNames) / sizeof(kKindNames[0]) == Launch::TAP, "one profile name per Launch::Kind before TAP");
int ns2vc_profile_num_kinds(void) { return Launch::TAP; }
const char* ns2vc_profile_kind_name(int k) { return (k >= 0 && k < Launch::TAP) ? kKindNames[k] : ""; }
int ns2vc_unet_profile_read(ns2vc_unet* h, int kind, double* ms_total, long long* launches) {
  NS_REQUIRE(h && ms_total && launches, "null argument");
  double ms = 0; long long n = 0;
  for (auto& r : h->prof) {
    if (r.kind != kind) continue;
    NS_CHECK_CUDA(cudaEventSynchronize(r.b));
    float e = 0;
    NS_CHECK_CUDA(cudaEventElapsedTime(&e, r.a, r.b));
    ms += e; ++n;
  }
  *ms_total = ms; *launches = n;
  return 0;
}
int ns2vc_unet_profile_dump(ns2vc_unet* h, const char* path) {
  NS_REQUIRE(h && path, "null argument");
  FILE* f = fopen(path, "w");
  NS_REQUIRE(f, "cannot open %s", path);
  fprintf(f, "idx,kind,us,M,N,K,nseg\n");
  int i = 0;
  for (auto& r : h->prof) {
    cudaEventSynchronize(r.b);
    float e = 0; cudaEventElapsedTime(&e, r.a, r.b);
    fprintf(f, "%d,%s,%.2f,%d,%d,%d,%d\n", i++, ns2vc_profile_kind_name(r.kind), e * 1e3f, r.M, r.N, r.K, r.nseg);
  }
  fclose(f);
  return 0;
}
int ns2vc_unet_profile_reset(ns2vc_unet* h) {
  NS_REQUIRE(h, "null handle");
  for (auto& r : h->prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  h->prof.clear();
  return 0;
}
const char* ns2vc_unet_plan_string(const ns2vc_unet* h) { return h ? h->plan_str.c_str() : ""; }
int ns2vc_unet_launch_count(const ns2vc_unet* h) { return launch_count(h); }

}  // extern "C"
