// SOLA (synchronized overlap-add) for live conversion: joins the output of one sliding-window tick to the tail kept from the
// last tick.  One CTA per slot.  For every offset k in [0, Ns] it correlates seg[k : k + Nc] with the tail, normalised by the
// segment's energy, picks the best offset, cross-fades the tail into the segment there, emits Nb samples and keeps the next
// tail.  Both sums of every k run in fp64 in one fixed order (one thread per k, ascending i), so the chosen offset does not
// depend on the launch.
#include "common.cuh"
#include "../../include/ns2vc_b200.h"

#include <cfloat>
#include <climits>

namespace ns2vc {
namespace {

constexpr int kSolaThreads = 256;
constexpr int kSolaMaxSmem = 47 * 1024;   // dynamic shared memory, leaving the static reduction slots under the 48 KB default

struct Best {
  double r;
  int k;
};

// a beats b: higher ratio, or the same ratio at a lower offset
__device__ __forceinline__ bool beats(const Best& a, const Best& b) { return a.r > b.r || (a.r == b.r && a.k < b.k); }

__global__ void __launch_bounds__(kSolaThreads) sola_kernel(const float* __restrict__ seg, long long seg_bstride,
                                                            float* __restrict__ tail, const float* __restrict__ fade_in,
                                                            float* __restrict__ out, int* __restrict__ offset, int Nb, int Nc,
                                                            int Ns) {
  extern __shared__ float sm[];
  float* s_seg = sm;                  // seg[0 : Nc + Ns]
  float* s_tail = sm + Nc + Ns;       // tail[0 : Nc]
  __shared__ Best s_best[kSolaThreads / 32];
  __shared__ int s_k;
  const int b = blockIdx.x;
  const float* row = seg + (long long)b * seg_bstride;
  float* trow = tail + (long long)b * Nc;
  for (int i = threadIdx.x; i < Nc + Ns; i += blockDim.x) s_seg[i] = row[i];
  for (int i = threadIdx.x; i < Nc; i += blockDim.x) s_tail[i] = trow[i];
  __syncthreads();

  Best best{-DBL_MAX, INT_MAX};
  for (int k = threadIdx.x; k <= Ns; k += blockDim.x) {
    double num = 0.0, den = 0.0;
    for (int i = 0; i < Nc; ++i) {
      const double s = s_seg[k + i];
      num = fma(s, (double)s_tail[i], num);
      den = fma(s, s, den);
    }
    const Best c{num / sqrt(den + 1e-8), k};
    if (beats(c, best)) best = c;
  }
  for (int o = 16; o > 0; o >>= 1) {
    Best other{__shfl_down_sync(0xffffffffu, best.r, o), __shfl_down_sync(0xffffffffu, best.k, o)};
    if (beats(other, best)) best = other;
  }
  if ((threadIdx.x & 31) == 0) s_best[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    Best w = s_best[0];
    for (int j = 1; j < kSolaThreads / 32; ++j)
      if (beats(s_best[j], w)) w = s_best[j];
    // every ratio NaN (a NaN in seg or tail) compares false everywhere: fall back to k = 0 rather than an out-of-range offset
    const int k = (w.k >= 0 && w.k <= Ns) ? w.k : 0;
    s_k = k;
    offset[b] = k;
  }
  __syncthreads();

  const int k = s_k;
  float* orow = out + (long long)b * Nb;
  for (int i = threadIdx.x; i < Nb; i += blockDim.x) {
    const float s = row[k + i];
    orow[i] = i < Nc ? s * fade_in[i] + s_tail[i] * (1.0f - fade_in[i]) : s;
  }
  // the tail is read from shared memory only, so overwriting it in global memory races with nothing above
  for (int i = threadIdx.x; i < Nc; i += blockDim.x) trow[i] = row[k + Nb + i];
}

}  // namespace
}  // namespace ns2vc

using namespace ns2vc;

extern "C" {

int ns2vc_stream_sola(const float* seg, long long seg_bstride, float* tail, const float* fade_in, float* out, int* offset, int B,
                      int Nb, int Nc, int Ns, ns2vc_stream stream) {
  NS_REQUIRE(seg && tail && fade_in && out && offset, "stream_sola: null argument");
  NS_REQUIRE(B >= 1 && B <= 65535 && Nc >= 1 && Ns >= 0 && Nb >= Nc, "stream_sola: bad sizes B=%d Nb=%d Nc=%d Ns=%d", B, Nb, Nc, Ns);
  NS_REQUIRE(seg_bstride >= (long long)Nb + Nc + Ns, "stream_sola: batch stride %lld is shorter than Nb + Nc + Ns = %d", seg_bstride,
             Nb + Nc + Ns);
  const size_t smem = (size_t)(2 * Nc + Ns) * sizeof(float);
  NS_REQUIRE(smem <= (size_t)kSolaMaxSmem, "stream_sola: 2 Nc + Ns = %d samples do not fit %d B of shared memory", 2 * Nc + Ns,
             kSolaMaxSmem);
  sola_kernel<<<B, kSolaThreads, smem, (cudaStream_t)stream>>>(seg, seg_bstride, tail, fade_in, out, offset, Nb, Nc, Ns);
  NS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
