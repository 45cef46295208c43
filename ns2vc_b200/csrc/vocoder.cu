// Vocoder engine: `Vocos.decode` (vocos/pretrained.py) of the mel configuration the reference loads at model.py:689-691
// (charactr/vocos-mel-24khz: VocosBackbone(100, 512, 1536, 8), ISTFTHead(512, 1024, 256, padding="same")), as one launch
// program per (B, T, workspace) over the wgmma 3xBF16 GEMM (gemm_tc.cu) plus the three small kernels below.
//
// Token-major [B, T, C] throughout (the reference's [B, C, T] is the transposed view of the same values).  Ragged batches:
// row b is decoded as if alone on its first T_b = lengths[b] frames; the residual stream is exactly 0 at frames >= T_b, so every
// k = 7 convolution reads the zero padding of the utterance alone.
//
//   x  = embed(mel)                        Conv1d(in, dim, 7, pad 3)      ONE implicit GEMM over 7 row-shifted views of the
//                                                                         mel split (frames >= T_b zeroed by nct_to_split)
//   x  = backbone.norm(x) * keep           LayerNorm eps 1e-6             voc_norm_kernel<false>     (vocos/models.py)
//   per ConvNeXtBlock (vocos/modules.py):
//     y = norm(dwconv(x))                  depthwise k = 7 + LayerNorm    voc_norm_kernel<true>: the row is local to the CTA
//     y = gelu_erf(y W1^T + b1)                                           GEMM, VOC instantiation (EPI_GELU)
//     x = (x + y (gamma W2)^T + gamma b2) * keep                          GEMM, ENC instantiation (residual + row mask);
//                                                                         layer scale folded into pwconv2 at load (fp64)
//   x  = final_layer_norm(x)                                              voc_norm_kernel<false>
//   h  = head.out(x)                       Linear(dim, n_fft + 2)         GEMM
//   audio = ISTFT_same(clip(exp(h[:513]), 100) * e^(i h[513:]))           voc_istft_kernel          (vocos/heads.py,
//                                                                         vocos/spectral_ops.py)
#include "common.cuh"
#include "engine_host.cuh"
#include "gemm_common.cuh"
#include "launch.cuh"
#include "../../include/ns2vc_b200.h"

#include <cmath>
#include <string>
#include <vector>

namespace ns2vc {
namespace {

constexpr int kTaps = 7;                  // ConvNeXt's depthwise conv and the embed conv (vocos/models.py, modules.py)
constexpr int kNormRows = 16;             // rows per voc_norm_kernel CTA
constexpr int kIstftFrames = 16;          // frames per voc_istft_kernel CTA (one warp each, two rounds of 8 warps)
constexpr int kIstftThreads = 256;
constexpr int kFramesPerSample = 4;       // n_fft = 4 hop_length: every output sample overlaps 4 frames

#define NS_VOC_LAUNCH_CHECK()                                                                  \
  do {                                                                                         \
    cudaError_t _e = cudaGetLastError();                                                       \
    if (_e != cudaSuccess) {                                                                   \
      set_error("%s:%d launch failed: %s", __FILE__, __LINE__, cudaGetErrorString(_e));        \
      return -2;                                                                               \
    }                                                                                          \
  } while (0)

// Row b's frame count: lengths[b] clamped into [1, T], or T without lengths.
__device__ __forceinline__ int voc_len(const long long* len, int b, int T) {
  return len ? (int)min(max(__ldg(len + b), 1LL), (long long)T) : T;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// lens[b] (the frame count, for nct_to_split) and keep[b, t] = t < lens[b] (the row mask of the pwconv2 epilogue)
__global__ void voc_lengths_kernel(const long long* __restrict__ len, int B, int T, int* __restrict__ lens, float* __restrict__ keep) {
  pdl_trigger();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * T) return;
  const int b = (int)(i / T), t = (int)(i - (long long)b * T);
  const int L = voc_len(len, b, T);
  keep[i] = t < L ? 1.f : 0.f;
  if (t == 0) lens[b] = L;
}

// LayerNorm (eps) over the C channels of each row, optionally after the 7-tap depthwise conv of ConvNeXtBlock (DW).  One CTA of
// C / 4 threads per kNormRows rows of one batch entry, four channels per thread.  Input rows at or past the entry's length read
// as zero (taps included); output rows at or past it are stored as 0.  Statistics in two passes (mean, then the mean square
// deviation), so a row offset large against the row's spread does not cancel.  Outputs: fp32 [B, T, C] and / or the bf16
// hi/lo split of the next GEMM.  dw: [C][8] = the 7 taps and the bias of each channel.
template <bool DW>
__global__ void __launch_bounds__(256) voc_norm_kernel(const float* __restrict__ x, int T, int C, const float4* __restrict__ dw,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                                       const long long* __restrict__ len, float* __restrict__ out, SplitBuf split) {
  __shared__ float red[kNormRows][8];
  pdl_trigger();
  const int b = blockIdx.y, t0 = blockIdx.x * kNormRows;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nwarps = blockDim.x >> 5;
  const int c = tid * 4;
  float w[4][8];
  if constexpr (DW) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float4 lo = __ldg(dw + 2 * (c + k)), hi = __ldg(dw + 2 * (c + k) + 1);
      w[k][0] = lo.x; w[k][1] = lo.y; w[k][2] = lo.z; w[k][3] = lo.w; w[k][4] = hi.x; w[k][5] = hi.y; w[k][6] = hi.z; w[k][7] = hi.w;
    }
  }
  const float4 g4 = __ldg(reinterpret_cast<const float4*>(gamma + c)), b4 = __ldg(reinterpret_cast<const float4*>(beta + c));
  pdl_wait();
  const int L = voc_len(len, b, T);
  const float* xb = x + (size_t)b * T * C + c;
  auto row = [&](int t) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t >= 0 && t < L) v = __ldg(reinterpret_cast<const float4*>(xb + (size_t)t * C));
    return v;
  };
  float y[kNormRows][4];
  if constexpr (DW) {
#pragma unroll
    for (int i = 0; i < kNormRows; ++i)
#pragma unroll
      for (int k = 0; k < 4; ++k) y[i][k] = w[k][7];
    // input row t0 - 3 + r feeds output row i = r - j through tap j: each output sums its taps in order 0 .. 6
#pragma unroll
    for (int r = 0; r < kNormRows + kTaps - 1; ++r) {
      const float4 v4 = row(t0 - kTaps / 2 + r);
      const float v[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
      for (int j = 0; j < kTaps; ++j) {
        const int i = r - j;
        if (i >= 0 && i < kNormRows) {
#pragma unroll
          for (int k = 0; k < 4; ++k) y[i][k] = fmaf(w[k][j], v[k], y[i][k]);
        }
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < kNormRows; ++i) {
      const float4 v4 = row(t0 + i);
      y[i][0] = v4.x; y[i][1] = v4.y; y[i][2] = v4.z; y[i][3] = v4.w;
    }
  }
  const float inv_c = 1.0f / (float)C;
  float mean[kNormRows], rstd[kNormRows];
#pragma unroll
  for (int i = 0; i < kNormRows; ++i) {
    const float s = warp_sum((y[i][0] + y[i][1]) + (y[i][2] + y[i][3]));
    if (lane == 0) red[i][warp] = s;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < kNormRows; ++i) {
    float s = 0.f;
    for (int q = 0; q < nwarps; ++q) s += red[i][q];
    mean[i] = s * inv_c;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < kNormRows; ++i) {
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) { const float d = y[i][k] - mean[i]; q = fmaf(d, d, q); }
    q = warp_sum(q);
    if (lane == 0) red[i][warp] = q;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < kNormRows; ++i) {
    float q = 0.f;
    for (int p = 0; p < nwarps; ++p) q += red[i][p];
    rstd[i] = 1.0f / sqrtf(q * inv_c + eps);
  }
  const float g[4] = {g4.x, g4.y, g4.z, g4.w}, be[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
  for (int i = 0; i < kNormRows; ++i) {
    const int t = t0 + i;
    if (t >= T) break;
    float o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) o[k] = t < L ? (y[i][k] - mean[i]) * rstd[i] * g[k] + be[k] : 0.f;
    const size_t m = (size_t)b * T + t;
    if (out) *reinterpret_cast<float4*>(out + m * C + c) = make_float4(o[0], o[1], o[2], o[3]);
    if (split.hi) {
      uint2 h, l;
      split2(o[0], o[1], h.x, l.x);
      split2(o[2], o[3], h.y, l.y);
      *reinterpret_cast<uint2*>(split.hi + m * split.ld + c) = h;
      *reinterpret_cast<uint2*>(split.lo + m * split.ld + c) = l;
    }
  }
}

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

// Bin k of S = clip(exp(mag), max=100) * (cos p + i sin p) from the head's row (log-magnitudes [nb], then phases [nb]).  The
// clip keeps NaN (as torch.clip does).  The imaginary parts of bins 0 and M do not enter a real inverse FFT.
__device__ __forceinline__ float2 spectrum_bin(const float* hrow, int nb, int k) {
  const float e = expf(__ldg(hrow + k));
  const float mag = e > 100.f ? 100.f : e;
  float s, c;
  sincosf(__ldg(hrow + nb + k), &s, &c);
  return make_float2(mag * c, (k == 0 || k == nb - 1) ? 0.f : mag * s);
}

// ISTFT with padding "same" (vocos/spectral_ops.py ISTFT): frames = irfft(S, n_fft) * window, overlap-added at hop_length,
// divided by the overlap-added window^2 and trimmed by pad = (n_fft - hop) / 2 on both ends; T frames give T * hop samples.
// Row b uses its frames < T_b only, its envelope counts those frames only, and its samples >= T_b * hop are 0.
// One CTA per (row, G = kIstftFrames - 3 output hops): its warps compute the G + 3 frames those hops overlap (one warp per frame,
// a 1024-point real inverse FFT as a 512-point complex radix-2 FFT after the inverse split step), keep them windowed in shared
// memory, then every thread overlap-adds its samples over their 4 frames in frame order (no atomics).
__global__ void __launch_bounds__(kIstftThreads) voc_istft_kernel(const float* __restrict__ h, int ld, int T, const long long* __restrict__ len,
                                                                  float* __restrict__ audio, int n_fft, int hop, int log2m, IstftTables tb) {
  extern __shared__ float s_fr[];                            // [kIstftFrames][n_fft]: windowed frames f0, f0 + 1, ...
  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.y;
  const int M = n_fft >> 1, nb = M + 1;
  constexpr int G = kIstftFrames - (kFramesPerSample - 1);
  const int k0 = 1 + blockIdx.x * G;                         // first hop block [k hop, (k + 1) hop) of the padded signal here
  const int f0 = k0 - (kFramesPerSample - 1);
  const int L = voc_len(len, b, T);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float inv_n = 1.0f / (float)n_fft;
  for (int q = warp; q < kIstftFrames; q += kIstftThreads / 32) {
    const int f = f0 + q;
    if (f < 0 || f >= L) continue;
    float2* z = reinterpret_cast<float2*>(s_fr + (size_t)q * n_fft);
    const float* hrow = h + ((size_t)b * T + f) * ld;
    // Z[k] = E[k] + i O[k], E[k] = X[k] + conj X[M-k], O[k] = (X[k] - conj X[M-k]) w^k (w = e^(2 pi i / n_fft)): the complex
    // sequence whose M-point inverse FFT is x[2m] + i x[2m+1] (times n_fft).  Z[M-k] uses w^(M-k) = -conj(w^k).  Stored
    // bit-reversed for the decimation-in-time stages.
    for (int k = lane; k <= M / 2; k += 32) {
      const float2 xk = spectrum_bin(hrow, nb, k), xn = spectrum_bin(hrow, nb, M - k);
      const float2 w = __ldg(tb.tw_full + k);
      {
        const float2 o = cmul(make_float2(xk.x - xn.x, xk.y + xn.y), w);
        z[__brev(k) >> (32 - log2m)] = make_float2((xk.x + xn.x) - o.y, (xk.y - xn.y) + o.x);
      }
      if (k != 0 && 2 * k != M) {
        const float2 o = cmul(make_float2(xn.x - xk.x, xn.y + xk.y), make_float2(-w.x, w.y));
        z[__brev(M - k) >> (32 - log2m)] = make_float2((xn.x + xk.x) - o.y, (xn.y - xk.y) + o.x);
      }
    }
    __syncwarp();
    for (int half = 1, tws = M >> 1; half < M; half <<= 1, tws >>= 1) {
      for (int u = lane; u < (M >> 1); u += 32) {
        const int pos = u & (half - 1);
        const int i0 = 2 * (u - pos) + pos, i1 = i0 + half;
        const float2 a = z[i0];
        const float2 c = cmul(z[i1], __ldg(tb.tw_half + pos * tws));
        z[i0] = make_float2(a.x + c.x, a.y + c.y);
        z[i1] = make_float2(a.x - c.x, a.y - c.y);
      }
      __syncwarp();
    }
    float* fr = s_fr + (size_t)q * n_fft;                    // z[m] = (x[2m], x[2m+1]): the frame in sample order
    for (int n = lane; n < n_fft; n += 32) fr[n] = (fr[n] * inv_n) * __ldg(tb.window + n);
    __syncwarp();
  }
  __syncthreads();
  const int pad = (n_fft - hop) >> 1;
  float* ab = audio + (size_t)b * T * hop;
  for (int i = threadIdx.x; i < G * hop; i += kIstftThreads) {
    const long long p = (long long)k0 * hop + i;             // sample of the padded signal
    const long long n = p - pad;                             // sample of the output
    if (n >= (long long)T * hop) break;
    if (n < 0) continue;
    float v = 0.f;
    if (n < (long long)L * hop) {
      const int kb = k0 + i / hop;
      const int fa = max(kb - (kFramesPerSample - 1), 0), fz = min(kb, L - 1);
      float y = 0.f, env = 0.f;
      for (int f = fa; f <= fz; ++f) {
        const int off = (int)(p - (long long)f * hop);
        const float wv = __ldg(tb.window + off);
        y += s_fr[(size_t)(f - f0) * n_fft + off];
        env += wv * wv;
      }
      v = y / env;
    }
    ab[n] = v;
  }
}

// Layer scale folded into pwconv2 (load time): w' = gamma[n] W[n, :], b' = gamma[n] b[n], products in fp64 rounded once
__global__ void voc_layer_scale_kernel(const float* __restrict__ W, const float* __restrict__ bias, const float* __restrict__ gamma, int N, int K,
                                       float* __restrict__ wo, float* __restrict__ bo) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)N * K) return;
  const int n = (int)(i / K);
  wo[i] = (float)((double)gamma[n] * (double)W[i]);
  if (i % K == 0) bo[n] = (float)((double)gamma[n] * (double)bias[n]);
}

}  // namespace

// (also the content encoder's LayerNorms: content.cu)
int launch_voc_norm(const VocNormOp& op, cudaStream_t st) {
  const dim3 grid(ceil_div(op.T, kNormRows), op.B), block(op.C / 4);
  cudaError_t e = op.dw ? launch_k(voc_norm_kernel<true>, grid, block, 0, st, op.x, op.T, op.C, reinterpret_cast<const float4*>(op.dw), op.gamma,
                                   op.beta, op.eps, op.len, op.out, op.split)
                        : launch_k(voc_norm_kernel<false>, grid, block, 0, st, op.x, op.T, op.C, (const float4*)nullptr, op.gamma, op.beta,
                                   op.eps, op.len, op.out, op.split);
  if (e != cudaSuccess) { set_error("voc_norm launch failed: %s", cudaGetErrorString(e)); return -2; }
  return 0;
}

// twiddles: fp64 formulas rounded to fp32 (the kernels evaluate no sin / cos besides the phases')
void istft_twiddles(int n_fft, std::vector<float2>& th, std::vector<float2>& tf) {
  const int M = n_fft / 2;
  const double pi = 3.141592653589793;
  th.resize(M / 2);
  tf.resize(M / 2 + 1);
  for (int j = 0; j < M / 2; ++j) th[j] = make_float2((float)std::cos(2.0 * pi * j / M), (float)std::sin(2.0 * pi * j / M));
  for (int k = 0; k <= M / 2; ++k) tf[k] = make_float2((float)std::cos(2.0 * pi * k / n_fft), (float)std::sin(2.0 * pi * k / n_fft));
}

int istft_log2m(int n_fft) {                                 // M = n_fft / 2 = 2^log2m
  int log2m = 0;
  while ((2 << log2m) < n_fft) ++log2m;
  return log2m;
}

size_t istft_smem_bytes(int n_fft) { return (size_t)kIstftFrames * n_fft * sizeof(float); }

int launch_istft(const IstftTables& tb, const float* head_out, int ld, const long long* len, float* audio, int B, int T, int n_fft, int hop,
                 int log2m, size_t smem, cudaStream_t st) {
  static size_t smem_set = 0;
  if (smem > 48 * 1024 && smem > smem_set) {
    const cudaError_t e = cudaFuncSetAttribute(voc_istft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("voc_istft: cannot set %zu B dynamic smem: %s", smem, cudaGetErrorString(e)); return -2; }
    smem_set = smem;
  }
  constexpr int G = kIstftFrames - (kFramesPerSample - 1);
  const cudaError_t e = launch_k(voc_istft_kernel, dim3(ceil_div(T + 1, G), B), dim3(kIstftThreads), smem, st, head_out, ld, T, len, audio, n_fft,
                                 hop, log2m, tb);
  if (e != cudaSuccess) { set_error("voc_istft launch failed: %s", cudaGetErrorString(e)); return -2; }
  return 0;
}

}  // namespace ns2vc

using namespace ns2vc;

struct ns2vc_voc : SingleProgramEngine {
  ns2vc_voc_cfg cfg;
  PackedB embed, head;
  std::vector<PackedB> pw1, pw2;
  std::vector<float*> b2;                                   // gamma * pwconv2.bias per block
  std::vector<float*> dw;                                   // [dim][8]: dwconv taps and bias per block
  float2* tw_half = nullptr; float2* tw_full = nullptr;
  int log2m = 0;
  size_t istft_smem = 0;
};

namespace ns2vc {
const EngineBase* engine_base(const ns2vc_voc* h) { return h; }
}  // namespace ns2vc

namespace {

std::string blk(int i) { return "backbone.convnext." + std::to_string(i); }

// Vocos.state_dict() order (feature_extractor.* is not part of decode): a module's own parameters precede its children's
void register_weights(ns2vc_voc* h) {
  const ns2vc_voc_cfg& c = h->cfg;
  WeightRegistry& w = h->weights;
  w.add_conv("backbone.embed", c.dim, c.input_channels, kTaps);
  w.add_norm("backbone.norm", c.dim);
  for (int i = 0; i < c.num_layers; ++i) {
    w.add(blk(i) + ".gamma", {c.dim});
    w.add_conv(blk(i) + ".dwconv", c.dim, 1, kTaps);
    w.add_norm(blk(i) + ".norm", c.dim);
    w.add_lin(blk(i) + ".pwconv1", c.intermediate_dim, c.dim);
    w.add_lin(blk(i) + ".pwconv2", c.dim, c.intermediate_dim);
  }
  w.add_norm("backbone.final_layer_norm", c.dim);
  w.add_lin("head.out", c.n_fft + 2, c.dim);
  w.add("head.istft.window", {c.n_fft});
}

int pack(ns2vc_voc* h, cudaStream_t st) {
  const ns2vc_voc_cfg& c = h->cfg;
  const WeightRegistry& w = h->weights;
  DeviceMem& mem = h->mem;
  const int D = c.dim, F = c.intermediate_dim, cin = c.input_channels;
  int rc;
  if ((rc = mem.alloc_packed(h->embed, D, D, kTaps * nkb_of(cin), false))) return rc;
  for (int j = 0; j < kTaps; ++j)
    if ((rc = pack_seg(h->embed, w.W("backbone.embed.weight"), D, cin, kTaps, j, 0, cin, 0, j * nkb_of(cin), 0, st))) return rc;
  h->packed.add("backbone.embed", h->embed);
  h->pw1.assign(c.num_layers, PackedB()); h->pw2.assign(c.num_layers, PackedB());
  h->b2.assign(c.num_layers, nullptr); h->dw.assign(c.num_layers, nullptr);
  float* scaled = c.num_layers ? mem.alloc<float>((size_t)D * F) : nullptr;   // scratch: gamma * W2 of one block at a time (stream order)
  if (c.num_layers && !scaled) return -2;
  for (int i = 0; i < c.num_layers; ++i) {
    const std::string p = blk(i);
    if ((rc = mem.alloc_packed(h->pw1[i], F, F, nkb_of(D), false))) return rc;
    if ((rc = pack_seg(h->pw1[i], w.W(p + ".pwconv1.weight"), F, D, 1, 0, 0, D, 0, 0, 0, st))) return rc;
    if (!(h->b2[i] = mem.alloc<float>(D))) return -2;
    voc_layer_scale_kernel<<<ceil_div(D * F, 256), 256, 0, st>>>(w.W(p + ".pwconv2.weight"), w.W(p + ".pwconv2.bias"), w.W(p + ".gamma"), D, F,
                                                                  scaled, h->b2[i]);
    NS_VOC_LAUNCH_CHECK();
    if ((rc = mem.alloc_packed(h->pw2[i], D, D, nkb_of(F), false))) return rc;
    if ((rc = pack_seg(h->pw2[i], scaled, D, F, 1, 0, 0, F, 0, 0, 0, st))) return rc;
    h->packed.add(p + ".pw1", h->pw1[i]);
    h->packed.add(p + ".pw2", h->pw2[i], {{"bias", h->b2[i], D}});
    float* d = h->dw[i] = mem.alloc<float>((size_t)D * 8);
    if (!d) return -2;
    NS_CHECK_CUDA(cudaMemcpy2DAsync(d, 8 * sizeof(float), w.W(p + ".dwconv.weight"), kTaps * sizeof(float), kTaps * sizeof(float), D,
                                    cudaMemcpyDeviceToDevice, st));
    NS_CHECK_CUDA(cudaMemcpy2DAsync(d + kTaps, 8 * sizeof(float), w.W(p + ".dwconv.bias"), sizeof(float), sizeof(float), D,
                                    cudaMemcpyDeviceToDevice, st));
  }
  if ((rc = mem.alloc_packed(h->head, c.n_fft + 2, c.n_fft + 2, nkb_of(D), false))) return rc;
  if ((rc = pack_seg(h->head, w.W("head.out.weight"), c.n_fft + 2, D, 1, 0, 0, D, 0, 0, 0, st))) return rc;
  h->packed.add("head.out", h->head);
  std::vector<float2> th, tf;
  istft_twiddles(c.n_fft, th, tf);
  if (!(h->tw_half = mem.alloc<float2>(th.size())) || !(h->tw_full = mem.alloc<float2>(tf.size()))) return -2;
  NS_CHECK_CUDA(cudaMemcpy(h->tw_half, th.data(), th.size() * sizeof(float2), cudaMemcpyHostToDevice));
  NS_CHECK_CUDA(cudaMemcpy(h->tw_full, tf.data(), tf.size() * sizeof(float2), cudaMemcpyHostToDevice));
  return 0;
}

int launch_istft(const ns2vc_voc* h, const float* head_out, int ld, const long long* len, float* audio, int B, int T, cudaStream_t st) {
  const IstftTables tb{h->weights.W("head.istft.window"), h->tw_half, h->tw_full};
  return launch_istft(tb, head_out, ld, len, audio, B, T, h->cfg.n_fft, h->cfg.hop_length, h->log2m, h->istft_smem, st);
}

int head_ld(const ns2vc_voc_cfg& c) { return pad_to(c.n_fft + 2, 4); }   // a TMA-storable row pitch for the head's output

int build_program(ns2vc_voc* h, int B, int T, void* ws, size_t* bytes_out) {
  const ns2vc_voc_cfg& c = h->cfg;
  const bool dry = ws == nullptr;
  NS_REQUIRE(B >= 1 && B <= 65535 && T >= 1 && (long long)T * c.hop_length <= INT32_MAX, "bad shape B=%d T=%d", B, T);
  std::vector<Launch> prog;
  TapSet taps;
  ProgramBuilder bld{Arena{(uint8_t*)ws, 0}, B, dry, false, &prog};
  Arena& ar = bld.ar;
  const WeightRegistry& w = h->weights;
  const int D = c.dim, ldh = head_ld(c);
  const size_t M = (size_t)B * T;
  int* lens = ar.get<int>(B);
  float* keep = ar.get<float>(M);
  const SplitBuf s_mel = bld.split(T, c.input_channels), s_x = bld.split(T, D), s_ff = bld.split(T, c.intermediate_dim);
  const SplitBuf none{};
  float* E = ar.get<float>(M * D);                          // embed output, later final_layer_norm's (for its tap)
  float* x = ar.get<float>(M * D);                          // residual stream (ping-pong)
  float* y = ar.get<float>(M * D);
  float* H = ar.get<float>(M * ldh);
  auto norm = [&](const float* in, const float* dwp, const std::string& ln, float* out, const SplitBuf& split) {
    bld.emit(Launch::VOC_NORM, VocNormOp{in, B, T, D, dwp, w.W(ln + ".weight"), w.W(ln + ".bias"), 1e-6f, nullptr, out, split}, Launch::LENGTHS);
  };
  bld.emit(Launch::VOC_LENS, VocLensOp{B, T, lens, keep});
  bld.emit(Launch::NCT2SPLIT, NctSplitOp{nullptr, 0, B, c.input_channels, T, s_mel, lens, nullptr, 0}, Launch::MEL);
  { GemmOp g = bld.gemm_base(h->embed, T);
    const int src = bld.add_src(g, s_mel);
    for (int j = 0; j < kTaps; ++j) bld.seg(g, src, 0, c.input_channels, j - kTaps / 2);
    g.flags = EPI_BIAS | EPI_OUT_F32; g.bias = w.W("backbone.embed.bias"); g.out = E; g.out_ld = D;
    bld.emit_gemm(g, h->embed); }
  norm(E, nullptr, "backbone.norm", x, none);
  bld.emit_tap(taps, "backbone.norm", x, T, D, T);
  for (int i = 0; i < c.num_layers; ++i) {
    const std::string p = blk(i);
    norm(x, h->dw[i], p + ".norm", nullptr, s_x);
    { GemmOp g = bld.lin(h->pw1[i], s_x, T);
      g.flags = EPI_BIAS | EPI_GELU | EPI_OUT_SPLIT; g.bias = w.W(p + ".pwconv1.bias");
      g.out_hi = s_ff.hi; g.out_lo = s_ff.lo; g.out_split_ld = s_ff.ld;
      bld.emit_gemm(g, h->pw1[i]); }
    { GemmOp g = bld.lin(h->pw2[i], s_ff, T);
      g.flags = EPI_BIAS | EPI_RESIDUAL | EPI_ROWMASK | EPI_OUT_F32; g.bias = h->b2[i]; g.res = x; g.res_ld = D; g.out = y; g.out_ld = D;
      g.rowmask = keep;
      bld.emit_gemm(g, h->pw2[i]); }
    bld.emit_tap(taps, p, y, T, D, T);
    std::swap(x, y);
  }
  norm(x, nullptr, "backbone.final_layer_norm", E, s_x);
  bld.emit_tap(taps, "backbone.final_layer_norm", E, T, D, T);
  { GemmOp g = bld.lin(h->head, s_x, T);
    g.flags = EPI_BIAS | EPI_OUT_F32; g.bias = w.W("head.out.bias"); g.out = H; g.out_ld = ldh;
    bld.emit_gemm(g, h->head); }
  bld.emit_tap(taps, "head.out", H, T, ldh, T);
  bld.emit(Launch::VOC_ISTFT, IstftOp{H, ldh, B, T});
  if (bld.err) return bld.err;
  if (bytes_out) *bytes_out = ar.off + 256;
  if (!dry) {
    h->cp.prog = std::move(prog);
    h->cp.taps = std::move(taps);
  }
  return 0;
}

int run_program(ns2vc_voc* h, const float* mel, long long mel_bstride, const long long* lengths, float* audio, cudaStream_t st) {
  CallArgs in{};
  in[Launch::MEL] = {mel, mel_bstride}; in[Launch::LENGTHS] = {lengths};
  return run_cached(h, false, in, st, [&](const Launch& l) {
    switch (l.kind) {
      case Launch::VOC_LENS: {
        const VocLensOp& o = l.get<VocLensOp>();
        voc_lengths_kernel<<<ceil_div(o.B * o.T, 256), 256, 0, st>>>(lengths, o.B, o.T, o.lens, o.keep);
        NS_VOC_LAUNCH_CHECK();
        return 0;
      }
      case Launch::VOC_ISTFT: { const IstftOp& o = l.get<IstftOp>(); return launch_istft(h, o.h, o.ld, lengths, audio, o.B, o.T, st); }
      default: return no_launcher(l);
    }
  });
}

}  // namespace

extern "C" {

int ns2vc_voc_create(const ns2vc_voc_cfg* cfg, ns2vc_voc** out) {
  NS_REQUIRE(cfg && out, "null argument");
  NS_REQUIRE(cfg->input_channels >= 1 && cfg->input_channels <= 1024, "input_channels %d unsupported (1 .. 1024)", cfg->input_channels);
  NS_REQUIRE(cfg->dim >= 128 && cfg->dim <= 1024 && cfg->dim % 128 == 0, "dim %d unsupported (a multiple of 128 up to 1024)", cfg->dim);
  NS_REQUIRE(cfg->intermediate_dim >= 64 && cfg->intermediate_dim % 64 == 0, "intermediate_dim %d unsupported (a multiple of 64)", cfg->intermediate_dim);
  NS_REQUIRE(cfg->num_layers >= 0 && cfg->num_layers <= 256, "num_layers %d unsupported", cfg->num_layers);
  NS_REQUIRE(cfg->hop_length >= 1 && cfg->n_fft == 4 * cfg->hop_length, "n_fft %d must be 4 * hop_length (%d): every sample overlaps 4 frames",
             cfg->n_fft, cfg->hop_length);
  NS_REQUIRE(cfg->n_fft >= 64 && cfg->n_fft <= 2048 && (cfg->n_fft & (cfg->n_fft - 1)) == 0, "n_fft %d unsupported (a power of two, 64 .. 2048)", cfg->n_fft);
  ns2vc_voc* h = new ns2vc_voc();
  h->cfg = *cfg;
  h->log2m = istft_log2m(cfg->n_fft);
  h->istft_smem = istft_smem_bytes(cfg->n_fft);
  register_weights(h);
  *out = h;
  return 0;
}

void ns2vc_voc_destroy(ns2vc_voc* h) { destroy_engine(h); }
int ns2vc_voc_num_weights(const ns2vc_voc* h) { return num_weights(h); }
int ns2vc_voc_weight_info(const ns2vc_voc* h, int i, const char** name, int64_t shape[4], int* ndim) { return weight_info(h, i, name, shape, ndim); }
int ns2vc_voc_load_weight(ns2vc_voc* h, const char* key, const float* dptr, const int64_t* shape, int ndim, ns2vc_stream stream) {
  return load_weight(h, key, dptr, shape, ndim, (cudaStream_t)stream);
}
int ns2vc_voc_finalize(ns2vc_voc* h, ns2vc_stream stream) { return finalize_engine(h, [&] { return pack(h, (cudaStream_t)stream); }); }

int ns2vc_voc_workspace_bytes(const ns2vc_voc* h, int B, int T, size_t* bytes) {
  NS_REQUIRE(h && bytes, "null argument");
  NS_REQUIRE(h->finalized, "ns2vc_voc_finalize() has not been called");
  return build_program(const_cast<ns2vc_voc*>(h), B, T, nullptr, bytes);
}

int ns2vc_voc_decode(ns2vc_voc* h, const float* mel, long long mel_bstride, const int64_t* lengths, float* audio, int B, int T, void* ws,
                     ns2vc_stream stream) {
  NS_REQUIRE(h && mel && audio, "null argument");
  NS_REQUIRE(mel_bstride >= (long long)h->cfg.input_channels * T, "mel batch stride %lld shorter than a [%d, %d] row", mel_bstride,
             h->cfg.input_channels, T);
  const int rc = ensure_program(h, "ns2vc_voc", B, T, 0, false, ws, [&] { return build_program(h, B, T, ws, nullptr); });
  if (rc) return rc;
  return run_program(h, mel, mel_bstride, reinterpret_cast<const long long*>(lengths), audio, (cudaStream_t)stream);
}

int ns2vc_voc_istft(ns2vc_voc* h, const float* head_out, const int64_t* lengths, float* audio, int B, int T, ns2vc_stream stream) {
  NS_REQUIRE(h && head_out && audio, "null argument");
  NS_REQUIRE(h->finalized, "ns2vc_voc_finalize() has not been called");
  NS_REQUIRE(B >= 1 && B <= 65535 && T >= 1 && (long long)T * h->cfg.hop_length <= INT32_MAX, "bad shape B=%d T=%d", B, T);
  return launch_istft(h, head_out, h->cfg.n_fft + 2, reinterpret_cast<const long long*>(lengths), audio, B, T, (cudaStream_t)stream);
}

int ns2vc_voc_num_taps(const ns2vc_voc* h) { return num_taps(h); }
int ns2vc_voc_tap_info(const ns2vc_voc* h, int i, const char** name, int* rows, int* channels) { return tap_info(h, i, name, rows, channels); }
int ns2vc_voc_set_tap(ns2vc_voc* h, int i, float* dst) { return set_tap(h, i, dst); }
int ns2vc_voc_launch_count(const ns2vc_voc* h) { return launch_count(h); }

}  // extern "C"
