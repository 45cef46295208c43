// Framewise RMS of the silence slicer: librosa 0.10's feature.rms(y, frame_length=win, hop_length=hop) (center=True,
// pad_mode="constant") for a ragged batch of files, bit for bit.  librosa pads win/2 zeros at both ends, frames the padded
// signal with util.frame and takes np.mean(np.square(frame), axis=-2) in float32, then np.sqrt.  The squared frame view is
// F-contiguous, so numpy sums each frame with its pairwise float32 sum (PW_BLOCKSIZE 128, 8 interleaved accumulators per
// leaf) and divides by win in float32; this kernel restates that association exactly.  One thread per frame.  The squares
// and sums are __fmul_rn / __fadd_rn so that nvcc cannot contract them into FMAs, and the square root is IEEE.
#include "common.cuh"
#include "../../include/ns2vc_b200.h"

namespace ns2vc {
namespace {

constexpr int kRmsThreads = 128;
constexpr int kPwBlock = 128;   // numpy's PW_BLOCKSIZE
constexpr int kPwDepth = 8;     // levels of halving above the leaves that the kernel unrolls

// the square of padded sample j of a row of n samples (the centre padding and the tail are zeros; nothing past n is read)
__device__ __forceinline__ float sq(const float* __restrict__ x, long long n, long long j) {
  if (j < 0 || j >= n) return 0.0f;
  const float v = __ldg(x + j);
  return __fmul_rn(v, v);
}

// numpy's pairwise_sum for m <= 128 elements starting at padded sample j0
__device__ __noinline__ float pw_leaf(const float* __restrict__ x, long long n, long long j0, int m) {
  if (m < 8) {
    float r = 0.0f;
    for (int i = 0; i < m; ++i) r = __fadd_rn(r, sq(x, n, j0 + i));
    return r;
  }
  float r0 = sq(x, n, j0), r1 = sq(x, n, j0 + 1), r2 = sq(x, n, j0 + 2), r3 = sq(x, n, j0 + 3);
  float r4 = sq(x, n, j0 + 4), r5 = sq(x, n, j0 + 5), r6 = sq(x, n, j0 + 6), r7 = sq(x, n, j0 + 7);
  int i = 8;
  for (; i < m - (m % 8); i += 8) {
    r0 = __fadd_rn(r0, sq(x, n, j0 + i));
    r1 = __fadd_rn(r1, sq(x, n, j0 + i + 1));
    r2 = __fadd_rn(r2, sq(x, n, j0 + i + 2));
    r3 = __fadd_rn(r3, sq(x, n, j0 + i + 3));
    r4 = __fadd_rn(r4, sq(x, n, j0 + i + 4));
    r5 = __fadd_rn(r5, sq(x, n, j0 + i + 5));
    r6 = __fadd_rn(r6, sq(x, n, j0 + i + 6));
    r7 = __fadd_rn(r7, sq(x, n, j0 + i + 7));
  }
  float res = __fadd_rn(__fadd_rn(__fadd_rn(r0, r1), __fadd_rn(r2, r3)), __fadd_rn(__fadd_rn(r4, r5), __fadd_rn(r6, r7)));
  for (; i < m; ++i) res = __fadd_rn(res, sq(x, n, j0 + i));
  return res;
}

// above 128 elements numpy splits at n2 = n/2 - (n/2 mod 8) and adds the two halves' sums
template <int D>
__device__ __forceinline__ float pw(const float* __restrict__ x, long long n, long long j0, int m) {
  if (m <= kPwBlock) return pw_leaf(x, n, j0, m);
  int m2 = m / 2;
  m2 -= m2 % 8;
  return __fadd_rn(pw<D - 1>(x, n, j0, m2), pw<D - 1>(x, n, j0 + m2, m - m2));
}

template <>
__device__ __forceinline__ float pw<0>(const float* __restrict__ x, long long n, long long j0, int m) {
  return pw_leaf(x, n, j0, m);
}

__global__ void __launch_bounds__(kRmsThreads) slice_rms_kernel(const float* __restrict__ wav, long long bstride,
                                                                const int64_t* __restrict__ lengths,
                                                                const int* __restrict__ hop_win, float* __restrict__ rms,
                                                                int F) {
  const int b = blockIdx.y;
  const int f = blockIdx.x * kRmsThreads + threadIdx.x;
  if (f >= F) return;
  const int hop = hop_win[2 * b], win = hop_win[2 * b + 1];
  const long long n = lengths[b];
  float out = 0.0f;
  // frames past the row's count are 0; a (hop, win) the host would have rejected computes nothing (and reads nothing)
  if (hop >= 1 && win >= 1 && n >= 0 && n + 2 * (win / 2) >= win && f < 1 + (n + 2 * (win / 2) - win) / hop) {
    const float s = pw<kPwDepth>(wav + (long long)b * bstride, n, (long long)f * hop - win / 2, win);
    out = __fsqrt_rn(__fdiv_rn(s, (float)win));
  }
  rms[(long long)b * F + f] = out;
}

// levels of halving numpy's pairwise sum takes above its 128-element leaves for m elements
int pw_depth(long long m) {
  if (m <= kPwBlock) return 0;
  long long m2 = m / 2;
  m2 -= m2 % 8;
  const int a = pw_depth(m2), c = pw_depth(m - m2);
  return 1 + (a > c ? a : c);
}

}  // namespace
}  // namespace ns2vc

using namespace ns2vc;

extern "C" {

long long ns2vc_slice_rms_frames(long long n, int hop, int win) {
  if (n < 0 || hop < 1 || win < 1 || n + 2 * (win / 2) < win || pw_depth(win) > kPwDepth) {
    set_error("slice_rms_frames: bad arguments n=%lld hop=%d win=%d (needs hop, win >= 1, a padded length n + 2 (win/2) >= win "
              "and a win whose pairwise sum splits at most %d times, about %d samples)", n, hop, win, kPwDepth,
              kPwBlock << kPwDepth);
    return -1;
  }
  return 1 + (n + 2 * (win / 2) - win) / hop;
}

int ns2vc_slice_rms(const float* wav, long long wav_bstride, const int64_t* lengths, const int* hop_win, float* rms, int F, int B,
                    ns2vc_stream stream) {
  NS_REQUIRE(wav && lengths && hop_win && rms, "slice_rms: null argument");
  NS_REQUIRE(B >= 1 && B <= 65535 && F >= 1 && wav_bstride >= 0, "slice_rms: bad sizes B=%d F=%d bstride=%lld", B, F, wav_bstride);
  dim3 grid((F + kRmsThreads - 1) / kRmsThreads, B);
  slice_rms_kernel<<<grid, kRmsThreads, 0, (cudaStream_t)stream>>>(wav, wav_bstride, lengths, hop_win, rms, F);
  NS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
