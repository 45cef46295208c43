// Content encoder: the units `utils.get_hubert_content` computes with ContentVec (a fairseq HubertModel, HuBERT-base: conv
// feature encoder of extractor_mode "default", post-LN transformer), `extract_features(output_layer = 12)` then `final_proj`,
// as one launch program per (B, N, workspace) over the wgmma 3xBF16 GEMM (gemm_tc.cu) plus the small kernels below.
//
// Token-major [B, T, C] throughout.  Ragged batches: row b is computed as if alone on its first N_b = lengths[b] samples (the
// reference's padding_mask is all False: nothing of a padded batch would be masked before the transformer, and the first conv's
// GroupNorm normalises over the whole time axis).  Every level's rows at or past the row's own frame count are exact zeros, so
// the strided convs and the positional conv read the zero padding of the utterance alone.
//
//   conv 0   (C0, k 10, s 5) -> GroupNorm(C0, C0) -> GELU   cv_gn_stats_kernel (fp64 sums over the row's own frames) +
//                                                            cv_conv0_kernel (recomputes the conv, writes layer 1's split)
//   conv 1-4 (C0, k 3, s 2) -> GELU                          GEMM, VOC instantiation, over row-pair views [B, T/2, 2 C0] of the
//   conv 5-6 (C0, k 2, s 2) -> GELU                          previous level (segments: pair | next pair's first half); row mask
//   layer_norm (C0) -> post_extract_proj (C0 -> D)           voc_norm_kernel + GEMM (ENC: row mask)
//   x + GELU(pos_conv(x))                                    per group: windows of 16 frames x 64 channels (cv_pos_windows_kernel),
//                                                            one GEMM of K / 16 row-shifted segments (VOC: GELU, row mask), then
//                                                            cv_add_kernel; weight norm folded at load in fp64
//   encoder.layer_norm, then per layer (post-LN):
//     x = self_attn_layer_norm(x + out_proj(attn(q, k, v)))  QKV GEMM (q's scaling folded at load), attention v2 with the row's
//                                                            own key count, GEMM (bias + residual), voc_norm_kernel
//     x = final_layer_norm(x + fc2(gelu(fc1(x))))           GEMM (VOC: GELU), GEMM (bias + residual), voc_norm_kernel
//   final_proj (D -> F)                                      GEMM (ENC: row mask)
#include "common.cuh"
#include "engine_host.cuh"
#include "gemm_common.cuh"
#include "launch.cuh"
#include "../../include/ns2vc_b200.h"

#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

namespace ns2vc {
namespace {

constexpr int kLevels = 7;                                   // the feature encoder's convs (fairseq's default conv_feature_layers)
constexpr int kMinSamples = 400;                             // the shortest input that gives one frame
constexpr int kWinTaps = 16;                                 // positional-conv taps per window row (16 x 64 channels = 1024)
constexpr int kStatCh = 8, kStatLanes = 32;                  // cv_gn_stats_kernel: channels x time lanes per CTA
constexpr int kConv0Frames = 16;                             // cv_conv0_kernel: frames per CTA

#define NS_CV_LAUNCH_CHECK()                                                                   \
  do {                                                                                         \
    cudaError_t _e = cudaGetLastError();                                                       \
    if (_e != cudaSuccess) {                                                                   \
      set_error("%s:%d launch failed: %s", __FILE__, __LINE__, cudaGetErrorString(_e));        \
      return -2;                                                                               \
    }                                                                                          \
  } while (0)

// kernel and stride of conv l: (10, 5), then (3, 2) four times, then (2, 2) twice
__host__ __device__ constexpr int conv_k(int l) { return l == 0 ? 10 : l < 5 ? 3 : 2; }
__host__ __device__ constexpr int conv_s(int l) { return l == 0 ? 5 : 2; }
__host__ __device__ __forceinline__ int conv_frames(int n, int l) { return n < conv_k(l) ? 0 : (n - conv_k(l)) / conv_s(l) + 1; }

// Row b's sample count: lengths[b] clamped into [kMinSamples, N], or N without lengths.
__device__ __forceinline__ int cv_samples(const long long* len, int b, int N) {
  return len ? (int)min(max(__ldg(len + b), (long long)kMinSamples), (long long)N) : N;
}

struct LenTables {
  int* frames;                 // [kLevels][B]: row b's frame count at each level
  long long* frames64;         // [B] frames of the last level (voc_norm_kernel's lengths)
  float* keep[kLevels];        // keep[l][b * rows[l] + t] = t < frames[l][b] (levels 1 ..; the row masks of the GEMM epilogues)
  int rows[kLevels];           // rows per entry of each level's buffer
};

__global__ void cv_lengths_kernel(const long long* __restrict__ len, int B, int N, LenTables lt, long long* __restrict__ frames_out) {
  pdl_trigger();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * lt.rows[1]) return;
  const int b = (int)(i / lt.rows[1]), t = (int)(i - (long long)b * lt.rows[1]);
  int n = cv_samples(len, b, N);
  for (int l = 0; l < kLevels; ++l) {
    n = conv_frames(n, l);
    if (l > 0 && t < lt.rows[l]) lt.keep[l][(long long)b * lt.rows[l] + t] = t < n ? 1.f : 0.f;
    if (t == 0) lt.frames[l * B + b] = n;
  }
  if (t == 0) {
    lt.frames64[b] = n;
    if (frames_out) frames_out[b] = n;
  }
}

// y[t, c] = sum_j w[c][j] x[5 t + j]: the first conv of one frame and channel (fp32, taps in order)
__device__ __forceinline__ float conv0_at(const float* w, const float* x) {
  float y = 0.f;
#pragma unroll
  for (int j = 0; j < 10; ++j) y = fmaf(w[j], x[j], y);
  return y;
}

// GroupNorm(C0, C0) statistics of the first conv's output over the row's own T0_b frames: per (row, channel) mean and 1 / std
// (biased variance, eps).  Time lane q of a CTA sums the frames t = q mod kStatLanes in fp64; the lanes are then added in lane
// order.  Neither depends on the rest of the batch.
__global__ void __launch_bounds__(kStatCh * kStatLanes) cv_gn_stats_kernel(const float* __restrict__ wav, long long bstride,
                                                                           const long long* __restrict__ len, int N,
                                                                           const float* __restrict__ w0, float eps, int C0,
                                                                           float2* __restrict__ stats) {
  __shared__ double red[2][kStatLanes][kStatCh];
  pdl_trigger();
  const int b = blockIdx.y, ci = threadIdx.x % kStatCh, q = threadIdx.x / kStatCh, c = blockIdx.x * kStatCh + ci;
  float w[10];
#pragma unroll
  for (int j = 0; j < 10; ++j) w[j] = __ldg(w0 + c * 10 + j);
  pdl_wait();
  const int T0 = conv_frames(cv_samples(len, b, N), 0);
  const float* xb = wav + (size_t)b * bstride;
  double s = 0.0, s2 = 0.0;
  for (int t = q; t < T0; t += kStatLanes) {
    float x[10];
#pragma unroll
    for (int j = 0; j < 10; ++j) x[j] = __ldg(xb + 5 * t + j);
    const double y = (double)conv0_at(w, x);
    s += y;
    s2 = fma(y, y, s2);
  }
  red[0][q][ci] = s;
  red[1][q][ci] = s2;
  __syncthreads();
  if (q == 0) {
    double a = 0.0, a2 = 0.0;
    for (int k = 0; k < kStatLanes; ++k) { a += red[0][k][ci]; a2 += red[1][k][ci]; }
    const double mean = a / T0;
    const double var = fmax(a2 / T0 - mean * mean, 0.0);
    stats[(size_t)b * C0 + c] = make_float2((float)mean, (float)(1.0 / sqrt(var + (double)eps)));
  }
}

// The first conv again, normalised (GroupNorm affine), erf-GELU, stored as layer 1's bf16 hi/lo split [B, rows, C0].  One CTA of
// C0 / 2 threads (two channels each) per kConv0Frames frames; frames at or past T0_b are stored as 0 and their samples are not
// read.
__global__ void __launch_bounds__(512) cv_conv0_kernel(const float* __restrict__ wav, long long bstride, const long long* __restrict__ len,
                                                       int N, int rows, const float* __restrict__ w0, const float2* __restrict__ stats,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta, SplitBuf out) {
  __shared__ float xs[5 * (kConv0Frames - 1) + 10];
  pdl_trigger();
  const int b = blockIdx.y, t0 = blockIdx.x * kConv0Frames, c = 2 * threadIdx.x, C0 = 2 * blockDim.x;
  float w[2][10];
#pragma unroll
  for (int k = 0; k < 2; ++k)
#pragma unroll
    for (int j = 0; j < 10; ++j) w[k][j] = __ldg(w0 + (c + k) * 10 + j);
  const float g[2] = {__ldg(gamma + c), __ldg(gamma + c + 1)}, be[2] = {__ldg(beta + c), __ldg(beta + c + 1)};
  pdl_wait();
  const int nb = cv_samples(len, b, N), T0 = conv_frames(nb, 0);
  const float2 st[2] = {__ldg(stats + (size_t)b * C0 + c), __ldg(stats + (size_t)b * C0 + c + 1)};
  const float* xb = wav + (size_t)b * bstride;
  for (int i = threadIdx.x; i < 5 * (kConv0Frames - 1) + 10; i += blockDim.x) {
    const long long s = 5LL * t0 + i;
    xs[i] = s < nb ? __ldg(xb + s) : 0.f;
  }
  __syncthreads();
  for (int i = 0; i < kConv0Frames; ++i) {
    const int t = t0 + i;
    if (t >= rows) break;
    float v[2] = {0.f, 0.f};
    if (t < T0) {
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const float y = (conv0_at(w[k], xs + 5 * i) - st[k].x) * st[k].y * g[k] + be[k];
        v[k] = 0.5f * y * (1.0f + erff(y * 0.70710678118654752440f));
      }
    }
    uint32_t hi, lo;
    split2(v[0], v[1], hi, lo);
    const size_t o = ((size_t)b * rows + t) * out.ld + c;
    *reinterpret_cast<uint32_t*>(out.hi + o) = hi;
    *reinterpret_cast<uint32_t*>(out.lo + o) = lo;
  }
}

// Window rows of the positional conv's group g: win[b, g, r, p * 64 + i] = x[b, r - K / 2 + p, g * gw + i] for p < kWinTaps,
// i < gw (0 outside the row's own frames and for i >= gw), as a bf16 hi/lo split of T + K rows.  Tap j = kWinTaps a + p of
// output frame t is then row t + kWinTaps a of the window: K / kWinTaps row-shifted segments of 1024 channels.
__global__ void __launch_bounds__(128) cv_pos_windows_kernel(const float* __restrict__ x, int T, int D, int G, int gw, int K,
                                                             const long long* __restrict__ frames, __nv_bfloat16* __restrict__ hi,
                                                             __nv_bfloat16* __restrict__ lo) {
  pdl_trigger();
  pdl_wait();
  const int r = blockIdx.x, g = blockIdx.y, b = blockIdx.z;
  const int L = (int)min(max(__ldg(frames + b), 1LL), (long long)T);
  const int e0 = threadIdx.x * 8, p = e0 >> 6, i0 = e0 & 63;
  const int src = r - K / 2 + p;
  float v[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int i = i0 + k;
    v[k] = (src >= 0 && src < L && i < gw) ? __ldg(x + ((size_t)b * T + src) * D + g * gw + i) : 0.f;
  }
  uint4 h, l;
  split8(v, h, l);
  const size_t o = (((size_t)b * G + g) * (T + K) + r) * (kWinTaps * 64) + e0;
  *reinterpret_cast<uint4*>(hi + o) = h;
  *reinterpret_cast<uint4*>(lo + o) = l;
}

// p += x (the positional conv's residual, [n / 4] float4)
__global__ void cv_add_kernel(float4* __restrict__ p, const float4* __restrict__ x, long long n4) {
  pdl_trigger();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 a = p[i];
  const float4 c = __ldg(x + i);
  a.x += c.x; a.y += c.y; a.z += c.z; a.w += c.w;
  p[i] = a;
}

// Tap of a split activation: dst[b, t, c] = hi + lo for t < T of a [B, rows, ld] split
__global__ void cv_split_tap_kernel(SplitBuf s, int rows, int T, int C, float* __restrict__ dst, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = (int)(i % C);
  const long long bt = i / C;
  const int t = (int)(bt % T), b = (int)(bt / T);
  const size_t o = ((size_t)b * rows + t) * s.ld + c;
  dst[i] = __bfloat162float(s.hi[o]) + __bfloat162float(s.lo[o]);
}

// Weight norm of the positional conv (dim = 2): W[o, i, j] = g[j] v[o, i, j] / ||v[:, :, j]||, the norm and the product in fp64.
// One CTA per tap j; the partial sums of squares are added in thread order.
__global__ void __launch_bounds__(256) cv_weight_norm_kernel(const float* __restrict__ g, const float* __restrict__ v, int rows, int K,
                                                             float* __restrict__ w) {
  __shared__ double part[256];
  const int j = blockIdx.x;
  double s = 0.0;
  for (int r = threadIdx.x; r < rows; r += 256) { const double a = v[(size_t)r * K + j]; s = fma(a, a, s); }
  part[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int k = 0; k < 256; ++k) t += part[k];
    part[0] = (double)g[j] / sqrt(t);
  }
  __syncthreads();
  const double f = part[0];
  for (int r = threadIdx.x; r < rows; r += 256) w[(size_t)r * K + j] = (float)(f * (double)v[(size_t)r * K + j]);
}

// q_proj | k_proj | v_proj as one [3D, D] operator and its [3D] bias, q's rows (weight and bias) times `qscale` (fp64, rounded once)
__global__ void cv_qkv_kernel(const float* __restrict__ qw, const float* __restrict__ kw, const float* __restrict__ vw, const float* __restrict__ qb,
                              const float* __restrict__ kb, const float* __restrict__ vb, int D, double qscale, float* __restrict__ w,
                              float* __restrict__ bias) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long DD = (long long)D * D;
  if (i < 3 * DD) {
    const int part = (int)(i / DD);
    const long long k = i - part * DD;
    w[i] = part == 0 ? (float)(qscale * (double)qw[k]) : part == 1 ? kw[k] : vw[k];
  }
  if (i < 3LL * D) {
    const int part = (int)(i / D), k = (int)(i - (long long)part * D);
    bias[i] = part == 0 ? (float)(qscale * (double)qb[k]) : part == 1 ? kb[k] : vb[k];
  }
}

int launch_check(cudaError_t e, const char* what) {
  if (e != cudaSuccess) { set_error("%s launch failed: %s", what, cudaGetErrorString(e)); return -2; }
  return 0;
}

}  // namespace

// The launchers of the kernels above (engine_host.cuh): run_program and the kernel checks launch them through these
int launch_cv_gn_stats(const CvGnStatsOp& o, const float* wav, long long bstride, const long long* lengths, cudaStream_t st) {
  return launch_check(launch_k(cv_gn_stats_kernel, dim3(o.C0 / kStatCh, o.B), dim3(kStatCh * kStatLanes), 0, st, wav, bstride, lengths, o.N,
                               o.w0, o.eps, o.C0, o.stats), "cv_gn_stats");
}

int launch_cv_conv0(const CvConv0Op& o, const float* wav, long long bstride, const long long* lengths, cudaStream_t st) {
  return launch_check(launch_k(cv_conv0_kernel, dim3(ceil_div(o.rows, kConv0Frames), o.B), dim3(o.out.C / 2), 0, st, wav, bstride, lengths, o.N,
                               o.rows, o.w0, o.stats, o.gamma, o.beta, o.out), "cv_conv0");
}

int launch_cv_pos_windows(const CvPosWinOp& o, cudaStream_t st) {
  return launch_check(launch_k(cv_pos_windows_kernel, dim3(o.win.T, o.G, o.B), dim3(kWinTaps * 64 / 8), 0, st, o.x, o.T, o.D, o.G, o.gw, o.K,
                               o.frames, o.win.hi, o.win.lo), "cv_pos_windows");
}

int launch_cv_add(const CvAddOp& o, cudaStream_t st) {
  return launch_check(launch_k(cv_add_kernel, dim3((unsigned)((o.n4 + 255) / 256)), dim3(256), 0, st, reinterpret_cast<float4*>(o.p),
                               reinterpret_cast<const float4*>(o.x), o.n4), "cv_add");
}

int cv_conv_taps(int l) { return conv_k(l); }

// Conv l's weights (w: [C0, C0, k]) into pb (Npad C0, k nkb(C0) k-blocks): tap j at k-block j nkb(C0), so that taps 0, 1 are
// one row pair's channels in order
int pack_cv_conv(PackedB& pb, const float* w, int C0, int l, cudaStream_t st) {
  for (int j = 0; j < conv_k(l); ++j) {
    const int rc = pack_seg(pb, w, C0, C0, conv_k(l), j, 0, C0, 0, j * nkb_of(C0), 0, st);
    if (rc) return rc;
  }
  return 0;
}

// Conv l (1 .. 6: k 3 or 2, stride 2, no bias) + GELU over level l - 1's split `in` [B, rows_in, C0] (ld C0; rows_in even, so
// that no pair straddles two entries) seen as row pairs [B, rows_in / 2, 2 C0]: output row t reads pair t (taps 0, 1) and, for
// k = 3, the next pair's first row (tap 2).  Rows whose factor in keep [B, rows_out] is 0 are stored as zeros; the output is
// the split `out_split` [B, rows_out, C0] (hi non-null) or fp32 `out` [B, rows_out, C0].
GemmOp cv_conv_gemm(ProgramBuilder& bld, const PackedB& w, const SplitBuf& in, int rows_in, int rows_out, int l, const float* keep,
                    const SplitBuf& out_split, float* out) {
  const SplitBuf pairs = ProgramBuilder::view(in, rows_in / 2, 2 * in.C);
  const int C0 = in.C;
  GemmOp g = bld.gemm_base(w, rows_out);
  const int src = bld.add_src(g, pairs);
  bld.seg(g, src, 0, 2 * C0, 0);                             // taps 0, 1: the pair itself
  if (conv_k(l) == 3) bld.seg(g, src, 0, C0, 1);             // tap 2: the next pair's first row
  g.flags = EPI_GELU | EPI_ROWMASK; g.rowmask = keep;
  if (out_split.hi) { g.flags |= EPI_OUT_SPLIT; g.out_hi = out_split.hi; g.out_lo = out_split.lo; g.out_split_ld = out_split.ld; }
  else { g.flags |= EPI_OUT_F32; g.out = out; g.out_ld = C0; }
  return g;
}

// Group g's weights of the folded positional conv (wg: [gw, gw, K]) into pb (Npad 128, K k-blocks): k-block j = tap j
int pack_cv_pos_group(PackedB& pb, const float* wg, int gw, int K, cudaStream_t st) {
  for (int j = 0; j < K; ++j) {
    const int rc = pack_seg(pb, wg, gw, gw, K, j, 0, gw, 0, j, 0, st);
    if (rc) return rc;
  }
  return 0;
}

// The positional conv's GEMM of group g over the windows `win` (CvPosWinOp::win: G groups of T + K rows): K / kWinTaps segments
// of 1024 channels at row shifts kWinTaps a, bias + GELU, the row mask `keep` [B, T], fp32 out at column g gw of out [B, T, out_ld]
GemmOp cv_pos_group_gemm(ProgramBuilder& bld, const PackedB& w, const SplitBuf& win, int G, int g, int gw, int T, int K, const float* bias,
                         const float* keep, float* out, int out_ld) {
  const size_t gsz = (size_t)win.T * kWinTaps * 64;
  const SplitBuf s{win.hi + g * gsz, win.lo + g * gsz, win.T, kWinTaps * 64, kWinTaps * 64,
                   (long long)G * win.T * kWinTaps * 64};
  GemmOp op = bld.gemm_base(w, T);
  const int src = bld.add_src(op, s);
  for (int a = 0; a < K / kWinTaps; ++a) bld.seg(op, src, 0, kWinTaps * 64, kWinTaps * a);
  op.flags = EPI_BIAS | EPI_GELU | EPI_OUT_F32 | EPI_ROWMASK; op.bias = bias + g * gw; op.out = out + g * gw; op.out_ld = out_ld;
  op.rowmask = keep;
  return op;
}

}  // namespace ns2vc

using namespace ns2vc;

struct ns2vc_cv : SingleProgramEngine {
  ns2vc_cv_cfg cfg;
  PackedB conv[kLevels];                                    // conv[1 ..]: the strided convs
  PackedB proj, fin;
  std::vector<PackedB> pos;                                 // per positional-conv group
  std::vector<PackedB> qkv, out, fc1, fc2;
  std::vector<float*> qkv_b;
  LenTables lt{};                                           // the cached program's length tables (in its workspace)
};

namespace ns2vc {
const EngineBase* engine_base(const ns2vc_cv* h) { return h; }
}  // namespace ns2vc

namespace {

std::string layer(int i) { return "encoder.layers." + std::to_string(i); }
std::string conv_key(int l) { return "feature_extractor.conv_layers." + std::to_string(l); }

// HubertModel.state_dict() order without the training-only mask_emb / label_embs_concat (a module's own parameters precede its
// children's; children in registration order: feature_extractor, post_extract_proj, encoder, layer_norm, final_proj)
void register_weights(ns2vc_cv* h) {
  const ns2vc_cv_cfg& c = h->cfg;
  WeightRegistry& w = h->weights;
  for (int l = 0; l < kLevels; ++l) {
    w.add(conv_key(l) + ".0.weight", {c.conv_dim, l == 0 ? 1 : c.conv_dim, conv_k(l)});
    if (l == 0) w.add_norm(conv_key(0) + ".2", c.conv_dim);
  }
  w.add_lin("post_extract_proj", c.embed_dim, c.conv_dim);
  w.add("encoder.pos_conv.0.bias", {c.embed_dim});
  w.add("encoder.pos_conv.0.weight_g", {1, 1, c.pos_conv_kernel});
  w.add("encoder.pos_conv.0.weight_v", {c.embed_dim, c.embed_dim / c.pos_conv_groups, c.pos_conv_kernel});
  for (int i = 0; i < c.num_layers; ++i) {
    const std::string p = layer(i);
    for (const char* m : {".self_attn.k_proj", ".self_attn.v_proj", ".self_attn.q_proj", ".self_attn.out_proj"}) w.add_lin(p + m, c.embed_dim, c.embed_dim);
    w.add_norm(p + ".self_attn_layer_norm", c.embed_dim);
    w.add_lin(p + ".fc1", c.ffn_dim, c.embed_dim);
    w.add_lin(p + ".fc2", c.embed_dim, c.ffn_dim);
    w.add_norm(p + ".final_layer_norm", c.embed_dim);
  }
  w.add_norm("encoder.layer_norm", c.embed_dim);
  w.add_norm("layer_norm", c.conv_dim);
  w.add_lin("final_proj", c.final_dim, c.embed_dim);
}

int pack_lin(DeviceMem& mem, PackedB& pb, const float* W, int n, int k, cudaStream_t st) {
  int rc;
  if ((rc = mem.alloc_packed(pb, n, n, nkb_of(k), false))) return rc;
  return pack_seg(pb, W, n, k, 1, 0, 0, k, 0, 0, 0, st);
}

// `scratch`: at least max(D gw K, 3 D^2) floats, used in stream order (the folded positional weight, then one layer's QKV at a time)
int pack_with(ns2vc_cv* h, cudaStream_t st, float* scratch) {
  const ns2vc_cv_cfg& c = h->cfg;
  const WeightRegistry& w = h->weights;
  DeviceMem& mem = h->mem;
  const int C0 = c.conv_dim, D = c.embed_dim, K = c.pos_conv_kernel, G = c.pos_conv_groups, gw = D / G;
  int rc;
  for (int l = 1; l < kLevels; ++l) {
    PackedB& pb = h->conv[l];
    if ((rc = mem.alloc_packed(pb, C0, C0, conv_k(l) * nkb_of(C0), false))) return rc;
    if ((rc = pack_cv_conv(pb, w.W(conv_key(l) + ".0.weight"), C0, l, st))) return rc;
    h->packed.add(conv_key(l), pb);
  }
  if ((rc = pack_lin(mem, h->proj, w.W("post_extract_proj.weight"), D, C0, st))) return rc;
  h->packed.add("post_extract_proj", h->proj);
  {
    float* wpos = scratch;
    cv_weight_norm_kernel<<<K, 256, 0, st>>>(w.W("encoder.pos_conv.0.weight_g"), w.W("encoder.pos_conv.0.weight_v"), D * gw, K, wpos);
    NS_CV_LAUNCH_CHECK();
    h->pos.assign(G, PackedB());
    for (int g = 0; g < G; ++g) {
      if ((rc = mem.alloc_packed(h->pos[g], gw, gw, K, false))) return rc;   // gw <= 64 channels, zero beyond
      if ((rc = pack_cv_pos_group(h->pos[g], wpos + (size_t)g * gw * gw * K, gw, K, st))) return rc;
      h->packed.add("encoder.pos_conv." + std::to_string(g), h->pos[g]);
    }
  }
  const int L = c.num_layers;
  h->qkv.assign(L, PackedB()); h->out.assign(L, PackedB()); h->fc1.assign(L, PackedB()); h->fc2.assign(L, PackedB());
  h->qkv_b.assign(L, nullptr);
  float* wqkv = scratch;
  const double qscale = 1.0 / std::sqrt((double)(D / c.num_heads));
  for (int i = 0; i < L; ++i) {
    const std::string p = layer(i) + ".self_attn.";
    if (!(h->qkv_b[i] = mem.alloc<float>((size_t)3 * D))) return -2;
    cv_qkv_kernel<<<ceil_div(3 * D * D, 256), 256, 0, st>>>(w.W(p + "q_proj.weight"), w.W(p + "k_proj.weight"), w.W(p + "v_proj.weight"),
                                                           w.W(p + "q_proj.bias"), w.W(p + "k_proj.bias"), w.W(p + "v_proj.bias"), D, qscale,
                                                           wqkv, h->qkv_b[i]);
    NS_CV_LAUNCH_CHECK();
    if ((rc = pack_lin(mem, h->qkv[i], wqkv, 3 * D, D, st))) return rc;
    if ((rc = pack_lin(mem, h->out[i], w.W(p + "out_proj.weight"), D, D, st))) return rc;
    if ((rc = pack_lin(mem, h->fc1[i], w.W(layer(i) + ".fc1.weight"), c.ffn_dim, D, st))) return rc;
    if ((rc = pack_lin(mem, h->fc2[i], w.W(layer(i) + ".fc2.weight"), D, c.ffn_dim, st))) return rc;
    h->packed.add(layer(i) + ".qkv", h->qkv[i], {{"bias", h->qkv_b[i], 3 * D}});
    h->packed.add(layer(i) + ".out_proj", h->out[i]);
    h->packed.add(layer(i) + ".fc1", h->fc1[i]);
    h->packed.add(layer(i) + ".fc2", h->fc2[i]);
  }
  if ((rc = pack_lin(mem, h->fin, w.W("final_proj.weight"), c.final_dim, D, st))) return rc;
  h->packed.add("final_proj", h->fin);
  return 0;
}

// Packs every operator; the load-time scratch is freed again in stream order, whatever the outcome
int pack(ns2vc_cv* h, cudaStream_t st) {
  const ns2vc_cv_cfg& c = h->cfg;
  const int D = c.embed_dim;
  const size_t n = std::max((size_t)D * (D / c.pos_conv_groups) * c.pos_conv_kernel, (size_t)3 * D * D);
  float* scratch = nullptr;
  NS_CHECK_CUDA(cudaMallocAsync(&scratch, n * sizeof(float), st));
  const int rc = pack_with(h, st, scratch);
  const cudaError_t e = cudaFreeAsync(scratch, st);
  if (rc) return rc;
  NS_CHECK_CUDA(e);
  return 0;
}

int build_program(ns2vc_cv* h, int B, int N, void* ws, size_t* bytes_out) {
  const ns2vc_cv_cfg& c = h->cfg;
  const bool dry = ws == nullptr;
  NS_REQUIRE(B >= 1 && B <= 65535 && N >= kMinSamples && N <= (1 << 28), "bad shape B=%d N=%d (N must be at least %d samples)", B, N, kMinSamples);
  const int C0 = c.conv_dim, D = c.embed_dim, FF = c.ffn_dim, G = c.pos_conv_groups, gw = D / G, K = c.pos_conv_kernel;
  int Tl[kLevels], rows[kLevels];
  for (int l = 0, n = N; l < kLevels; ++l) {
    Tl[l] = n = conv_frames(n, l);
    rows[l] = l + 1 < kLevels ? Tl[l] + (Tl[l] & 1) : Tl[l];    // even, so that the next conv's row-pair view stays inside the entry
  }
  const int T = Tl[kLevels - 1];
  std::vector<Launch> prog;
  TapSet taps;
  ProgramBuilder bld{Arena{(uint8_t*)ws, 0}, B, dry, false, &prog};
  Arena& ar = bld.ar;
  const WeightRegistry& w = h->weights;
  const size_t M = (size_t)B * T;
  LenTables lt{};
  lt.frames = ar.get<int>((size_t)kLevels * B);
  lt.frames64 = ar.get<long long>(B);
  for (int l = 0; l < kLevels; ++l) {
    lt.rows[l] = rows[l];
    lt.keep[l] = l ? ar.get<float>((size_t)B * rows[l]) : nullptr;
  }
  const int* frames_last = lt.frames + (kLevels - 1) * B;
  float2* gn = ar.get<float2>((size_t)B * C0);
  // levels 0, 2, 4 share one split, levels 1, 3, 5 another
  const SplitBuf lv_even = bld.split(rows[0], C0), lv_odd = bld.split(rows[1], C0);
  float* H6 = ar.get<float>(M * C0);                         // conv 6 output
  float* Fn = ar.get<float>(M * C0);                         // the feature LayerNorm's (voc_norm_kernel's x and out must not alias)
  const SplitBuf s_feat = bld.split(T, C0), s_x = bld.split(T, D), s_qkv = bld.split(T, 3 * D), s_att = bld.split(T, D), s_ff = bld.split(T, FF);
  float* Fp = ar.get<float>(M * D);                          // post_extract_proj output (the positional conv's input and residual)
  float* P = ar.get<float>(M * D);                           // positional conv, then x + it
  float* X = ar.get<float>(M * D);                           // residual stream (normalised)
  float* Y = ar.get<float>(M * D);
  float* U = ar.get<float>(M * c.final_dim);
  const int Tw = T + K;                                     // window rows: frames -K/2 .. T + K/2 - 1
  const size_t win_elems = (size_t)B * G * Tw * kWinTaps * 64;
  __nv_bfloat16* win_hi = ar.get<__nv_bfloat16>(win_elems);
  __nv_bfloat16* win_lo = ar.get<__nv_bfloat16>(win_elems);

  auto tap_f32 = [&](const std::string& name, const float* src, int C) { bld.emit_tap(taps, name, src, T, C, T); };
  auto tap_split_of = [&](const std::string& name, const SplitBuf& s, int rws, int Tn) {
    if (dry) return;
    bld.emit(Launch::CV_SPLIT_TAP, SplitTapOp{s, B, rws, Tn, C0}).tap_index = taps.add(name, Tn, C0);
  };
  auto norm = [&](const float* in, const std::string& ln, int C, float* out, const SplitBuf& split) {
    bld.emit(Launch::VOC_NORM, VocNormOp{in, B, T, C, nullptr, w.W(ln + ".weight"), w.W(ln + ".bias"), 1e-5f, lt.frames64, out, split});
  };
  auto rowmask = [&](GemmOp& g, int l) { g.flags |= EPI_ROWMASK; g.rowmask = lt.keep[l]; };

  const float* w0 = w.W(conv_key(0) + ".0.weight");
  bld.emit(Launch::CV_LENS, CvLensOp{B, N});
  bld.emit(Launch::CV_GN_STATS, CvGnStatsOp{B, N, C0, w0, 1e-5f, gn});
  bld.emit(Launch::CV_CONV0, CvConv0Op{B, N, rows[0], w0, gn, w.W(conv_key(0) + ".2.weight"), w.W(conv_key(0) + ".2.bias"), lv_even});
  tap_split_of(conv_key(0), lv_even, rows[0], Tl[0]);
  for (int l = 1; l < kLevels; ++l) {
    const SplitBuf in = (l & 1) ? lv_even : lv_odd;          // level l - 1
    const SplitBuf out = ProgramBuilder::view((l & 1) ? lv_odd : lv_even, rows[l], C0);
    GemmOp g = cv_conv_gemm(bld, h->conv[l], in, rows[l - 1], rows[l], l, lt.keep[l], l + 1 < kLevels ? out : SplitBuf{}, H6);
    bld.emit_gemm(g, h->conv[l]);
    if (l + 1 < kLevels) tap_split_of(conv_key(l), out, rows[l], Tl[l]);
    else tap_f32(conv_key(l), H6, C0);
  }
  norm(H6, "layer_norm", C0, Fn, s_feat);
  tap_f32("layer_norm", Fn, C0);
  { GemmOp g = bld.lin(h->proj, s_feat, T);
    g.flags = EPI_BIAS | EPI_OUT_F32; g.bias = w.W("post_extract_proj.bias"); g.out = Fp; g.out_ld = D;
    rowmask(g, kLevels - 1);
    bld.emit_gemm(g, h->proj); }
  tap_f32("post_extract_proj", Fp, D);
  const SplitBuf win{win_hi, win_lo, Tw, kWinTaps * 64, kWinTaps * 64, 0};
  bld.emit(Launch::CV_POS_WIN, CvPosWinOp{Fp, B, T, D, G, gw, K, lt.frames64, win});
  for (int g_ = 0; g_ < G; ++g_) {
    GemmOp g = cv_pos_group_gemm(bld, h->pos[g_], win, G, g_, gw, T, K, w.W("encoder.pos_conv.0.bias"), lt.keep[kLevels - 1], P, D);
    bld.emit_gemm(g, h->pos[g_]);
  }
  bld.emit(Launch::CV_ADD, CvAddOp{P, Fp, (long long)(M * D / 4)});
  tap_f32("encoder.pos_conv", P, D);
  norm(P, "encoder.layer_norm", D, X, s_x);
  tap_f32("encoder.layer_norm", X, D);
  const int dh = D / c.num_heads;
  for (int i = 0; i < c.num_layers; ++i) {
    const std::string p = layer(i);
    { GemmOp g = bld.lin(h->qkv[i], s_x, T);
      g.flags = EPI_BIAS | EPI_OUT_SPLIT; g.bias = h->qkv_b[i]; g.out_hi = s_qkv.hi; g.out_lo = s_qkv.lo; g.out_split_ld = s_qkv.ld;
      bld.emit_gemm(g, h->qkv[i]); }
    { AttnOp a; memset(&a, 0, sizeof(a));
      a.out_hi = s_att.hi; a.out_lo = s_att.lo; a.out_split_ld = s_att.ld;
      a.B = B; a.H = c.num_heads; a.Tq = T; a.Tk = T; a.dh = dh; a.scale = 1.0f;   // (q's scaling is folded into q_proj)
      a.v2 = 1; a.p_split = 1; a.qs = s_qkv; a.ks = s_qkv; a.vs = s_qkv; a.q_c0 = 0; a.k_c0 = D; a.v_c0 = 2 * D;
      a.key_len = frames_last; a.key_shift = 0;             // each row attends over its own frames; padded key tiles are skipped
      bld.emit_attention(a); }
    { GemmOp g = bld.lin(h->out[i], s_att, T);
      g.flags = EPI_BIAS | EPI_RESIDUAL | EPI_OUT_F32; g.bias = w.W(p + ".self_attn.out_proj.bias"); g.res = X; g.res_ld = D; g.out = Y; g.out_ld = D;
      bld.emit_gemm(g, h->out[i]); }
    norm(Y, p + ".self_attn_layer_norm", D, X, s_x);
    tap_f32(p + ".self_attn_layer_norm", X, D);
    { GemmOp g = bld.lin(h->fc1[i], s_x, T);
      g.flags = EPI_BIAS | EPI_GELU | EPI_OUT_SPLIT; g.bias = w.W(p + ".fc1.bias"); g.out_hi = s_ff.hi; g.out_lo = s_ff.lo; g.out_split_ld = s_ff.ld;
      bld.emit_gemm(g, h->fc1[i]); }
    { GemmOp g = bld.lin(h->fc2[i], s_ff, T);
      g.flags = EPI_BIAS | EPI_RESIDUAL | EPI_OUT_F32; g.bias = w.W(p + ".fc2.bias"); g.res = X; g.res_ld = D; g.out = Y; g.out_ld = D;
      bld.emit_gemm(g, h->fc2[i]); }
    norm(Y, p + ".final_layer_norm", D, X, s_x);
    tap_f32(p, X, D);
  }
  { GemmOp g = bld.lin(h->fin, s_x, T);
    g.flags = EPI_BIAS | EPI_OUT_F32; g.bias = w.W("final_proj.bias"); g.out = U; g.out_ld = c.final_dim;
    rowmask(g, kLevels - 1);
    bld.emit_gemm(g, h->fin); }
  tap_f32("final_proj", U, c.final_dim);
  bld.emit(Launch::COPY, CopyOp{U, M * c.final_dim * sizeof(float), nullptr}, Launch::OUT);
  if (bld.err) return bld.err;
  if (bytes_out) *bytes_out = ar.off + 256;
  if (!dry) {
    h->cp.prog = std::move(prog);
    h->cp.taps = std::move(taps);
    h->lt = lt;
  }
  return 0;
}

}  // namespace

namespace {

int run_program(ns2vc_cv* h, const float* wav, long long bstride, const long long* lengths, float* units, long long* frames_out, cudaStream_t st) {
  CallArgs in{};
  in[Launch::OUT] = {units};
  return run_cached(h, false, in, st, [&](const Launch& l) {
    switch (l.kind) {
      case Launch::CV_LENS: {
        const CvLensOp& o = l.get<CvLensOp>();
        const LenTables& lt = h->lt;
        return launch_check(launch_k(cv_lengths_kernel, dim3(ceil_div(o.B * lt.rows[1], 256)), dim3(256), 0, st, lengths, o.B, o.N, lt, frames_out), "cv_lengths");
      }
      case Launch::CV_GN_STATS: return launch_cv_gn_stats(l.get<CvGnStatsOp>(), wav, bstride, lengths, st);
      case Launch::CV_CONV0: return launch_cv_conv0(l.get<CvConv0Op>(), wav, bstride, lengths, st);
      case Launch::CV_POS_WIN: return launch_cv_pos_windows(l.get<CvPosWinOp>(), st);
      case Launch::CV_ADD: return launch_cv_add(l.get<CvAddOp>(), st);
      case Launch::CV_SPLIT_TAP: {
        float* dst = h->cp.taps.dst[l.tap_index];
        if (dst) {
          const SplitTapOp& o = l.get<SplitTapOp>();
          const long long n = (long long)o.B * o.T * o.C;
          cv_split_tap_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(o.s, o.rows, o.T, o.C, dst, n);
          NS_CV_LAUNCH_CHECK();
        }
        return 0;
      }
      default: return no_launcher(l);
    }
  });
}

}  // namespace

extern "C" {

int ns2vc_cv_create(const ns2vc_cv_cfg* cfg, ns2vc_cv** out) {
  NS_REQUIRE(cfg && out, "null argument");
  const ns2vc_cv_cfg& c = *cfg;
  NS_REQUIRE(c.conv_dim >= 128 && c.conv_dim <= 1024 && c.conv_dim % 128 == 0, "conv_dim %d unsupported (a multiple of 128 up to 1024)", c.conv_dim);
  NS_REQUIRE(c.embed_dim >= 128 && c.embed_dim <= 1024 && c.embed_dim % 128 == 0, "embed_dim %d unsupported (a multiple of 128 up to 1024)", c.embed_dim);
  NS_REQUIRE(c.num_heads >= 1 && c.embed_dim % c.num_heads == 0, "embed_dim %d is not a multiple of num_heads %d", c.embed_dim, c.num_heads);
  const int dh = c.embed_dim / c.num_heads;
  NS_REQUIRE(dh == 16 || dh == 32 || dh == 48 || dh == 64, "head dim %d unsupported (16, 32, 48 or 64)", dh);
  NS_REQUIRE(c.ffn_dim >= 64 && c.ffn_dim % 64 == 0, "ffn_dim %d unsupported (a multiple of 64)", c.ffn_dim);
  NS_REQUIRE(c.num_layers >= 0 && c.num_layers <= 64, "num_layers %d unsupported", c.num_layers);
  NS_REQUIRE(c.final_dim >= 4 && c.final_dim % 4 == 0, "final_dim %d unsupported (a multiple of 4)", c.final_dim);
  NS_REQUIRE(c.pos_conv_groups >= 1 && c.embed_dim % c.pos_conv_groups == 0, "embed_dim %d is not a multiple of pos_conv_groups %d", c.embed_dim,
             c.pos_conv_groups);
  const int gw = c.embed_dim / c.pos_conv_groups;
  NS_REQUIRE(gw <= 64 && gw % 4 == 0, "positional-conv group width %d unsupported (a multiple of 4 up to 64: one 64-channel TMA box per tap, "
             "16-byte aligned group columns)", gw);
  NS_REQUIRE(c.pos_conv_kernel >= kWinTaps && c.pos_conv_kernel <= kWinTaps * kMaxSeg && c.pos_conv_kernel % kWinTaps == 0,
             "pos_conv_kernel %d unsupported (a multiple of %d up to %d)", c.pos_conv_kernel, kWinTaps, kWinTaps * kMaxSeg);
  ns2vc_cv* h = new ns2vc_cv();
  h->cfg = c;
  register_weights(h);
  *out = h;
  return 0;
}

void ns2vc_cv_destroy(ns2vc_cv* h) { destroy_engine(h); }
int ns2vc_cv_num_weights(const ns2vc_cv* h) { return num_weights(h); }
int ns2vc_cv_weight_info(const ns2vc_cv* h, int i, const char** name, int64_t shape[4], int* ndim) { return weight_info(h, i, name, shape, ndim); }
int ns2vc_cv_load_weight(ns2vc_cv* h, const char* key, const float* dptr, const int64_t* shape, int ndim, ns2vc_stream stream) {
  return load_weight(h, key, dptr, shape, ndim, (cudaStream_t)stream);
}
int ns2vc_cv_finalize(ns2vc_cv* h, ns2vc_stream stream) { return finalize_engine(h, [&] { return pack(h, (cudaStream_t)stream); }); }

int ns2vc_cv_workspace_bytes(const ns2vc_cv* h, int B, int N, size_t* bytes) {
  NS_REQUIRE(h && bytes, "null argument");
  NS_REQUIRE(h->finalized, "ns2vc_cv_finalize() has not been called");
  return build_program(const_cast<ns2vc_cv*>(h), B, N, nullptr, bytes);
}

int ns2vc_cv_num_frames(long long n) {
  if (n < kMinSamples || n > (1 << 28)) return 0;
  int t = (int)n;
  for (int l = 0; l < kLevels; ++l) t = conv_frames(t, l);
  return t;
}

int ns2vc_cv_extract(ns2vc_cv* h, const float* wav, long long wav_bstride, const int64_t* lengths, float* units, int64_t* frames, int B, int N,
                     void* ws, ns2vc_stream stream) {
  NS_REQUIRE(h && wav && units, "null argument");
  NS_REQUIRE(wav_bstride >= N, "waveform batch stride %lld shorter than a row of %d samples", wav_bstride, N);
  const int rc = ensure_program(h, "ns2vc_cv", B, N, 0, false, ws, [&] { return build_program(h, B, N, ws, nullptr); });
  if (rc) return rc;
  return run_program(h, wav, wav_bstride, reinterpret_cast<const long long*>(lengths), units, reinterpret_cast<long long*>(frames),
                     (cudaStream_t)stream);
}

int ns2vc_cv_num_taps(const ns2vc_cv* h) { return num_taps(h); }
int ns2vc_cv_tap_info(const ns2vc_cv* h, int i, const char** name, int* rows, int* channels) { return tap_info(h, i, name, rows, channels); }
int ns2vc_cv_set_tap(ns2vc_cv* h, int i, float* dst) { return set_tap(h, i, dst); }
int ns2vc_cv_launch_count(const ns2vc_cv* h) { return launch_count(h); }

}  // extern "C"
