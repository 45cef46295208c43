// Prompt-mel front end (reference inference/infer_tool.py:170-181, preprocess.py:27-31, 49-59): torchaudio's
// Resample(orig, new) (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99) and
// MelSpectrogram(24000, n_fft=1024, hop=256, n_mels=100, center=True, power=1) followed by log(clip(., 1e-7)),
// per utterance of a ragged batch.  Latency-sized fp32 SIMT work: no tensor cores, no vendor FFT.
//
//   resample_kernel  polyphase FIR: output j = sum_i table[j mod new][i] * x[(j div new) * orig - width + i], the input
//                    outside [0, len_b) reading as zero (torchaudio's pad + conv1d(stride=orig)); each CTA stages its
//                    contiguous input window in shared memory.
//   log_mel_kernel   one CTA per (utterance, 8 frames), one warp per frame: reflect-padded staging at the utterance's own
//                    length, periodic Hann window, 1024-point real FFT as a 512-point complex radix-2 FFT plus the split
//                    step, magnitudes, sparse HTK mel projection, log(max(., 1e-7)), [B, 100, S] stores through shared memory.
//
// Every table (phase table, window, twiddles, filterbank) is built on the host once per handle; the kernels evaluate no
// sin / cos.  Each output element depends only on its own row and a fixed summation order, so a row of a ragged batch is
// bit-identical to the same row computed alone.
#include "common.cuh"
#include "../../include/ns2vc_b200.h"

#include <algorithm>
#include <cmath>
#include <numeric>
#include <vector>

namespace ns2vc {
namespace {

constexpr int kNfft = NS2VC_MEL_N_FFT;
constexpr int kHop = NS2VC_MEL_HOP;
constexpr int kMels = NS2VC_MEL_N_MELS;
constexpr int kBins = kNfft / 2 + 1;                       // 513 one-sided bins
constexpr int kHalf = kNfft / 2;                           // 512: complex FFT length, and the reflect pad of center=True
constexpr int kFrames = 8;                                 // frames per CTA (one warp each)
constexpr int kMelThreads = 32 * kFrames;
constexpr int kStage = kFrames * kHop + kNfft - kHop;      // staged samples per CTA
constexpr int kMelPitch = kFrames + 1;
constexpr int kResThreads = 256;                           // outputs per resample CTA (one per thread)
constexpr int kResMaxWindow = 48 * 1024 / 4;               // staged input floats per resample CTA

// ---------------------------------------------------------------------------------------------------------------------
// Host tables
// ---------------------------------------------------------------------------------------------------------------------
struct Ratio { int orig, nw, width, taps; double base; };

Ratio resample_ratio(int orig_freq, int new_freq) {
  const int g = std::gcd(orig_freq, new_freq);
  Ratio r;
  r.orig = orig_freq / g;
  r.nw = new_freq / g;
  r.base = (double)std::min(r.orig, r.nw) * 0.99;           // base_freq *= rolloff
  r.width = (int)std::ceil(6.0 * r.orig / r.base);           // ceil(lowpass_filter_width * orig / base_freq), 6 * orig exact
  r.taps = 2 * r.width + r.orig;
  return r;
}

// torchaudio _get_sinc_resample_kernel (dtype=None): idx in fp64, the phase offsets -p/new as fp32 (an int64 arange true-
// divided in the default dtype), everything after in fp64, the result rounded to fp32.  [nw][taps], phase-major.
std::vector<float> sinc_table(const Ratio& r) {
  std::vector<float> k((size_t)r.nw * r.taps);
  const double pi = 3.141592653589793;
  for (int p = 0; p < r.nw; ++p) {
    const double ph = (double)((float)(-p) / (float)r.nw);
    for (int i = 0; i < r.taps; ++i) {
      double t = (ph + (double)(i - r.width) / r.orig) * r.base;
      t = std::min(std::max(t, -6.0), 6.0);
      const double c = std::cos(t * pi / 6.0 / 2.0);
      const double win = c * c;
      t *= pi;
      const double s = t == 0.0 ? 1.0 : std::sin(t) / t;
      k[(size_t)p * r.taps + i] = (float)(s * (win * (r.base / r.orig)));
    }
  }
  return k;
}

// torchaudio melscale_fbanks(513, 0, 12000, 100, 24000, norm=None, mel_scale="htk") in its own fp32 operation order:
// torch.linspace (start + step * i below the halfway point, end - step * (steps - 1 - i) above it, each one fused multiply-
// add), _mel_to_hz, and the triangular filterbank of _create_triangular_filterbank.  [513][100], bin-major like the
// reference's matrix.  torch's vectorised powf may differ from the C library's in the last bit, so the matrix agrees with
// torchaudio's to a few fp32 ulps rather than bit for bit.
std::vector<float> mel_filterbank() {
  auto linspace = [](float a, float b, int n) {
    std::vector<float> v(n);
    const float step = (b - a) / (float)(n - 1);
    for (int i = 0; i < n; ++i) v[i] = i < n / 2 ? fmaf(step, (float)i, a) : fmaf(-step, (float)(n - 1 - i), b);
    return v;
  };
  const std::vector<float> freqs = linspace(0.f, (float)(NS2VC_MEL_SAMPLE_RATE / 2), kBins);
  const double m_max = 2595.0 * std::log10(1.0 + (NS2VC_MEL_F_MAX / 700.0));
  std::vector<float> f_pts = linspace(0.f, (float)m_max, kMels + 2);
  for (float& m : f_pts) m = 700.0f * (powf(10.0f, m / 2595.0f) - 1.0f);
  std::vector<float> fb((size_t)kBins * kMels);
  for (int k = 0; k < kBins; ++k)
    for (int m = 0; m < kMels; ++m) {
      const float down = (-1.0f * (f_pts[m] - freqs[k])) / (f_pts[m + 1] - f_pts[m]);
      const float up = (f_pts[m + 2] - freqs[k]) / (f_pts[m + 2] - f_pts[m + 1]);
      fb[(size_t)k * kMels + m] = std::max(0.0f, std::min(down, up));
    }
  return fb;
}

long long out_length(const Ratio& r, long long n) {
  // torchaudio: ceil(torch.as_tensor(new * n / orig)).long() - an fp64 quotient rounded to fp32 before the ceiling
  return (long long)std::ceil((float)((double)(r.nw * n) / (double)r.orig));
}

// input floats a resample CTA stages for its kResThreads outputs; a ratio whose window passes kResMaxWindow is refused
long long resample_window(const Ratio& r) {
  return (long long)((kResThreads - 1) / r.nw + 1) * r.orig + r.taps;
}

// ---------------------------------------------------------------------------------------------------------------------
// Kernels
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kResThreads)
resample_kernel(const float* __restrict__ x, long long x_bstride, long long n, const long long* __restrict__ lengths,
                float* __restrict__ y, long long y_bstride, long long n_out, const float* __restrict__ table,
                const int2* __restrict__ range, int orig, int nw, int width, int taps) {
  extern __shared__ float s_x[];
  const int b = blockIdx.y;
  const long long j0 = (long long)blockIdx.x * kResThreads;
  const long long L = lengths ? min(max(lengths[b], 0LL), n) : n;
  const long long L_out = (long long)ceilf(__double2float_rn(__ddiv_rn((double)(nw * L), (double)orig)));
  const long long k0 = j0 / nw;
  const long long in0 = k0 * orig - width;                  // input index of tap 0 of output block k0
  const long long j_last = min(j0 + kResThreads, n_out) - 1;
  const int span = (int)((j_last / nw - k0) * orig + taps);
  const float* xb = x + b * x_bstride;
  for (int i = threadIdx.x; i < span; i += kResThreads) {
    const long long s = in0 + i;
    s_x[i] = (s >= 0 && s < L) ? __ldg(xb + s) : 0.f;
  }
  __syncthreads();
  const long long j = j0 + threadIdx.x;
  if (j >= n_out) return;
  float acc = 0.f;
  if (j < L_out) {
    const long long k = j / nw;
    const int p = (int)(j - k * nw);
    const float* w = table + (size_t)p * taps;
    const float* xs = s_x + (k - k0) * orig;
    // [first, last] nonzero tap of this phase, fixed order, accumulated in fp64 and rounded once: resampling to a lower rate
    // leaves the top mel bands holding little but the resampler's rounding noise, so the log-mel there sees every fp32 rounding
    const int2 r = range[p];
    double a = (double)__ldg(w + r.x) * (double)xs[r.x];
    for (int i = r.x + 1; i <= r.y; ++i) a = fma((double)__ldg(w + i), (double)xs[i], a);
    acc = (float)a;
  }
  y[b * y_bstride + j] = acc;
}

struct MelTables {
  const float* window;    // [1024] periodic Hann
  const float2* tw512;    // [256] exp(-2 pi i k / 512)
  const float2* tw1024;   // [257] exp(-2 pi i k / 1024)
  const int2* band;       // [100] (first bin, nonzero bins)
  const int* band_off;    // [100] offset of band m's weights
  const float* weights;   // packed nonzero filterbank weights, band-major
};

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

__global__ void __launch_bounds__(kMelThreads)
log_mel_kernel(const float* __restrict__ x, long long x_bstride, long long n, const long long* __restrict__ lengths,
               float* __restrict__ mel, int S, MelTables t) {
  __shared__ float s_x[kStage];
  __shared__ float2 s_fft[kFrames][kHalf];
  __shared__ float s_mel[kMels * kMelPitch];
  const int b = blockIdx.y;
  const int s0 = blockIdx.x * kFrames;
  // out-of-contract lengths are clamped into the row, so no index below can leave it
  const long long L = lengths ? min(max(lengths[b], 1LL), n) : n;
  const int n_frames = (int)min(1 + L / kHop, (long long)S);
  const int nf = max(0, min(kFrames, n_frames - s0));       // frames this CTA computes; the rest of its tile is zero
  const float* xb = x + b * x_bstride;
  const long long p0 = (long long)s0 * kHop - kHalf;        // sample under padded position s0 * hop
  for (int i = threadIdx.x; i < nf * kHop + kNfft - kHop && nf > 0; i += kMelThreads) {
    long long s = p0 + i;
    s = s < 0 ? -s : s;                                     // reflect about sample 0 ...
    s = s >= L ? 2 * (L - 1) - s : s;                       // ... and about sample L-1
    s = min(max(s, 0LL), L - 1);
    s_x[i] = __ldg(xb + s);
  }
  __syncthreads();
  const int f = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (f < nf) {
    float2* z = s_fft[f];
    const float* fr = s_x + f * kHop;
    for (int q = lane; q < kHalf; q += 32)                  // z[q] = w x[2q] + i w x[2q+1], stored bit-reversed
      z[__brev(q) >> 23] = make_float2(fr[2 * q] * __ldg(t.window + 2 * q), fr[2 * q + 1] * __ldg(t.window + 2 * q + 1));
    __syncwarp();
    for (int half = 1, tws = kHalf / 2; half < kHalf; half <<= 1, tws >>= 1) {
      for (int u = lane; u < kHalf / 2; u += 32) {
        const int pos = u & (half - 1);
        const int i0 = 2 * (u - pos) + pos, i1 = i0 + half;
        const float2 a = z[i0];
        const float2 c = cmul(z[i1], __ldg(t.tw512 + pos * tws));
        z[i0] = make_float2(a.x + c.x, a.y + c.y);
        z[i1] = make_float2(a.x - c.x, a.y - c.y);
      }
      __syncwarp();
    }
    // split step: X[k] = Xe + W^k Xo, X[512-k] = conj(Xe - W^k Xo), Xe = (Z[k] + conj Z[512-k]) / 2, Xo = (Z[k] - conj Z[512-k]) / 2i
    constexpr int kPairs = (kHalf / 2 + 32) / 32;           // k = 0 .. 256
    float mk[kPairs], mn[kPairs];
#pragma unroll
    for (int i = 0; i < kPairs; ++i) {
      const int k = lane + 32 * i;
      if (k <= kHalf / 2) {
        const float2 zk = z[k], zn = z[(kHalf - k) & (kHalf - 1)];
        const float2 xe = make_float2(0.5f * (zk.x + zn.x), 0.5f * (zk.y - zn.y));
        const float2 xo = make_float2(0.5f * (zk.y + zn.y), -0.5f * (zk.x - zn.x));
        const float2 wx = cmul(__ldg(t.tw1024 + k), xo);
        const float ar = xe.x + wx.x, ai = xe.y + wx.y, br = xe.x - wx.x, bi = xe.y - wx.y;
        mk[i] = sqrtf(ar * ar + ai * ai);
        mn[i] = sqrtf(br * br + bi * bi);
      }
    }
    __syncwarp();
    float* mag = reinterpret_cast<float*>(z);               // [513] magnitudes over the consumed spectrum
#pragma unroll
    for (int i = 0; i < kPairs; ++i) {
      const int k = lane + 32 * i;
      if (k <= kHalf / 2) {
        mag[k] = mk[i];
        mag[kHalf - k] = mn[i];                             // k = 256 writes the same value twice
      }
    }
    __syncwarp();
    for (int m = lane; m < kMels; m += 32) {
      const int2 band = __ldg(t.band + m);
      const float* w = t.weights + __ldg(t.band_off + m);
      float acc = 0.f;
      for (int i = 0; i < band.y; ++i) acc = fmaf(__ldg(w + i), mag[band.x + i], acc);
      // torch.clip(., min=1e-7) keeps NaN (fmaxf would return 1e-7 for it): a NaN sample reaches the prompt mel as NaN
      s_mel[m * kMelPitch + f] = logf(acc < 1e-7f ? 1e-7f : acc);
    }
  }
  __syncthreads();
  float* mb = mel + (size_t)b * kMels * S;
  for (int i = threadIdx.x; i < kMels * kFrames; i += kMelThreads) {
    const int m = i / kFrames, ff = i % kFrames, s = s0 + ff;
    if (s < S) mb[(size_t)m * S + s] = ff < nf ? s_mel[m * kMelPitch + ff] : 0.f;
  }
}

}  // namespace
}  // namespace ns2vc

struct ns2vc_resampler {
  ns2vc::Ratio r;
  bool identity;
  int window;             // staged input floats per CTA
  float* table = nullptr; // device [nw][taps]
  int2* range = nullptr;  // device [nw]
};

struct ns2vc_mel {
  void* mem = nullptr;
  ns2vc::MelTables t;
};

using namespace ns2vc;

extern "C" {

long long ns2vc_resample_out_length(int orig_freq, int new_freq, long long n) {
  if (orig_freq <= 0 || new_freq <= 0 || n < 0) { set_error("resample_out_length: bad arguments %d -> %d, n=%lld", orig_freq, new_freq, n); return -1; }
  if (orig_freq == new_freq) return n;
  return out_length(resample_ratio(orig_freq, new_freq), n);
}

int ns2vc_resample_table(int orig_freq, int new_freq, int* phases, int* taps, int* width, float* table) {
  NS_REQUIRE(orig_freq > 0 && new_freq > 0 && orig_freq != new_freq, "resample_table: bad rates %d -> %d", orig_freq, new_freq);
  const Ratio r = resample_ratio(orig_freq, new_freq);
  if (phases) *phases = r.nw;
  if (taps) *taps = r.taps;
  if (width) *width = r.width;
  if (table) {
    const std::vector<float> k = sinc_table(r);
    std::copy(k.begin(), k.end(), table);
  }
  return 0;
}

int ns2vc_mel_filterbank(float* fb) {
  NS_REQUIRE(fb, "mel_filterbank: null argument");
  const std::vector<float> v = mel_filterbank();
  std::copy(v.begin(), v.end(), fb);
  return 0;
}

int ns2vc_resample_check(int orig_freq, int new_freq) {
  NS_REQUIRE(orig_freq > 0 && new_freq > 0, "resample_check: bad rates %d -> %d", orig_freq, new_freq);
  if (orig_freq == new_freq) return 0;
  const Ratio r = resample_ratio(orig_freq, new_freq);
  NS_REQUIRE(resample_window(r) <= kResMaxWindow, "resample_check: %d -> %d Hz reduces to %d:%d, whose %lld-sample input window per %d "
             "outputs exceeds %d", orig_freq, new_freq, r.orig, r.nw, resample_window(r), kResThreads, kResMaxWindow);
  return 0;
}

int ns2vc_resampler_create(int orig_freq, int new_freq, ns2vc_resampler** out) {
  NS_REQUIRE(out, "resampler_create: null argument");
  NS_REQUIRE(orig_freq > 0 && new_freq > 0, "resampler_create: bad rates %d -> %d", orig_freq, new_freq);
  auto* h = new ns2vc_resampler();
  h->identity = orig_freq == new_freq;
  std::vector<float> table;
  std::vector<int2> range;
  if (h->identity) {                                        // torchaudio returns the input: one phase, one unit tap
    h->r = Ratio{1, 1, 0, 1, 1.0};
    table = {1.0f};
    range = {make_int2(0, 0)};
  } else {
    h->r = resample_ratio(orig_freq, new_freq);
    table = sinc_table(h->r);
    for (int p = 0; p < h->r.nw; ++p) {                     // the taps past the zero crossings clamp to exactly 0 in fp32
      const float* w = table.data() + (size_t)p * h->r.taps;
      int lo = 0, hi = h->r.taps - 1;
      while (lo < hi && w[lo] == 0.f) ++lo;
      while (hi > lo && w[hi] == 0.f) --hi;
      range.push_back(make_int2(lo, hi));
    }
  }
  const Ratio r = h->r;                                     // a copy: the refusal below reads it after deleting h
  h->window = (int)std::min<long long>(resample_window(r), INT32_MAX);
  if (h->window > kResMaxWindow) {
    delete h;
    set_error("resampler_create: %d -> %d Hz reduces to %d:%d, whose %d-sample input window per %d outputs exceeds %d",
              orig_freq, new_freq, r.orig, r.nw, (int)resample_window(r), kResThreads, kResMaxWindow);
    return -1;
  }
  cudaError_t e = cudaMalloc(&h->table, table.size() * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&h->range, range.size() * sizeof(int2));
  if (e == cudaSuccess) e = cudaMemcpy(h->table, table.data(), table.size() * sizeof(float), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(h->range, range.data(), range.size() * sizeof(int2), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    cudaFree(h->table);
    cudaFree(h->range);
    delete h;
    set_error("resampler_create: %s", cudaGetErrorString(e));
    return -2;
  }
  *out = h;
  return 0;
}

void ns2vc_resampler_destroy(ns2vc_resampler* h) {
  if (!h) return;
  cudaFree(h->table);
  cudaFree(h->range);
  delete h;
}

int ns2vc_resample(const ns2vc_resampler* h, const float* x, long long x_bstride, long long n, const int64_t* lengths, float* y,
                   long long y_bstride, long long n_out, int B, ns2vc_stream stream) {
  NS_REQUIRE(h && x && y, "resample: null argument");
  NS_REQUIRE(B >= 1 && B <= 65535 && n >= 0 && n_out >= 0, "resample: bad sizes B=%d n=%lld n_out=%lld", B, n, n_out);
  NS_REQUIRE(x_bstride >= n && y_bstride >= n_out, "resample: batch strides %lld / %lld shorter than the rows", x_bstride, y_bstride);
  const long long n_need = h->identity ? n : out_length(h->r, n);
  NS_REQUIRE(n_out <= n_need, "resample: %lld output samples requested, %lld input samples give %lld", n_out, n, n_need);
  if (n_out == 0) return 0;
  const long long blocks = (n_out + kResThreads - 1) / kResThreads;
  NS_REQUIRE(blocks <= INT32_MAX, "resample: %lld output samples per row is too many", n_out);
  const Ratio& r = h->r;
  resample_kernel<<<dim3((unsigned)blocks, B), kResThreads, h->window * sizeof(float), (cudaStream_t)stream>>>(
      x, x_bstride, n, reinterpret_cast<const long long*>(lengths), y, y_bstride, n_out, h->table, h->range, r.orig, r.nw,
      r.width, r.taps);
  NS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int ns2vc_mel_create(const float* window_in, const float* fb_in, ns2vc_mel** out) {
  NS_REQUIRE(out, "mel_create: null argument");
  // twiddles: fp64 formulas rounded to fp32.  Window and filterbank: the caller's fp32 tables, else the periodic Hann window
  // in fp64 rounded to fp32 and mel_filterbank()
  std::vector<float> window(kNfft);
  std::vector<float2> tw512(kHalf / 2), tw1024(kHalf / 2 + 1);
  const double pi = 3.141592653589793;
  for (int i = 0; i < kNfft; ++i) window[i] = window_in ? window_in[i] : (float)(0.5 - 0.5 * std::cos(2.0 * pi * i / kNfft));
  for (int k = 0; k < kHalf / 2; ++k) tw512[k] = make_float2((float)std::cos(2.0 * pi * k / kHalf), (float)-std::sin(2.0 * pi * k / kHalf));
  for (int k = 0; k <= kHalf / 2; ++k) tw1024[k] = make_float2((float)std::cos(2.0 * pi * k / kNfft), (float)-std::sin(2.0 * pi * k / kNfft));
  const std::vector<float> fb = fb_in ? std::vector<float>(fb_in, fb_in + (size_t)kBins * kMels) : mel_filterbank();
  std::vector<int2> band(kMels);
  std::vector<int> band_off(kMels);
  std::vector<float> weights;
  for (int m = 0; m < kMels; ++m) {
    int lo = 0, hi = kBins - 1;
    while (lo < kBins && fb[(size_t)lo * kMels + m] == 0.f) ++lo;
    while (hi >= lo && fb[(size_t)hi * kMels + m] == 0.f) --hi;
    band[m] = make_int2(std::min(lo, kBins - 1), std::max(hi - lo + 1, 0));
    band_off[m] = (int)weights.size();
    for (int k = lo; k <= hi; ++k) weights.push_back(fb[(size_t)k * kMels + m]);
  }
  // one allocation, 16-byte aligned pieces
  auto pad = [](size_t b) { return (b + 15) & ~size_t(15); };
  const size_t o_win = 0, o_tw512 = o_win + pad(window.size() * 4), o_tw1024 = o_tw512 + pad(tw512.size() * 8),
               o_band = o_tw1024 + pad(tw1024.size() * 8), o_off = o_band + pad(band.size() * 8), o_w = o_off + pad(band_off.size() * 4),
               total = o_w + pad(weights.size() * 4);
  std::vector<char> host(total, 0);
  memcpy(host.data() + o_win, window.data(), window.size() * 4);
  memcpy(host.data() + o_tw512, tw512.data(), tw512.size() * 8);
  memcpy(host.data() + o_tw1024, tw1024.data(), tw1024.size() * 8);
  memcpy(host.data() + o_band, band.data(), band.size() * 8);
  memcpy(host.data() + o_off, band_off.data(), band_off.size() * 4);
  memcpy(host.data() + o_w, weights.data(), weights.size() * 4);
  auto* h = new ns2vc_mel();
  cudaError_t e = cudaMalloc(&h->mem, total);
  if (e == cudaSuccess) e = cudaMemcpy(h->mem, host.data(), total, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    cudaFree(h->mem);
    delete h;
    set_error("mel_create: %s", cudaGetErrorString(e));
    return -2;
  }
  char* d = static_cast<char*>(h->mem);
  h->t = MelTables{reinterpret_cast<const float*>(d + o_win), reinterpret_cast<const float2*>(d + o_tw512),
                   reinterpret_cast<const float2*>(d + o_tw1024), reinterpret_cast<const int2*>(d + o_band),
                   reinterpret_cast<const int*>(d + o_off), reinterpret_cast<const float*>(d + o_w)};
  *out = h;
  return 0;
}

void ns2vc_mel_destroy(ns2vc_mel* h) {
  if (!h) return;
  cudaFree(h->mem);
  delete h;
}

int ns2vc_log_mel(const ns2vc_mel* h, const float* x, long long x_bstride, long long n, const int64_t* lengths, float* mel, int S,
                  int B, ns2vc_stream stream) {
  NS_REQUIRE(h && x && mel, "log_mel: null argument");
  NS_REQUIRE(B >= 1 && B <= 65535 && S >= 1 && n > kHalf, "log_mel: bad sizes B=%d S=%d n=%lld (rows need more than %d samples)", B, S, n, kHalf);
  NS_REQUIRE(x_bstride >= n, "log_mel: batch stride %lld shorter than the row (%lld)", x_bstride, n);
  NS_REQUIRE(S <= 1 + n / kHop, "log_mel: %d frames requested, %lld samples give %lld", S, n, 1 + n / kHop);
  log_mel_kernel<<<dim3((S + kFrames - 1) / kFrames, B), kMelThreads, 0, (cudaStream_t)stream>>>(
      x, x_bstride, n, reinterpret_cast<const long long*>(lengths), mel, S, h->t);
  NS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
