// The training objective of NaturalSpeech2.forward (reference model.py:698-734) around the denoiser, evaluated under no_grad at K
// timesteps per batch: q_sample in front of the K denoiser forwards, and the SNR-weighted per-row MSE behind them.
//
// q_sample_kernel restates the reference's five element-wise torch ops (spec * mask, randn * mask, a[t] * x_start,
// s[t] * noise, their sum) with explicitly rounded multiplies and adds, so no FMA is contracted and the result equals the
// torch expression on the same device bit for bit.  The mask is a 0/1 FACTOR as in the reference: a non-finite input value
// past a row's length turns into NaN there exactly as it does in the reference.  Inputs must be finite.
//
// The MSE is deterministic: every row is cut into chunks of kMseChunk elements, one CTA per chunk, fp64 accumulation in a fixed
// order inside the CTA, the partial sums written to a workspace and added by mse_finish_kernel in index order.  No atomics: the
// result depends on neither the launch nor the scheduling.
//
// The ragged MSE (per-utterance objective) applies the same scheme to each row's own C * T_b elements and reads nothing past a
// row's length, so a row's value does not depend on the batch it sits in.
#include "common.cuh"
#include "../../include/ns2vc_b200.h"

#include <cmath>

namespace ns2vc {
namespace {

constexpr int kQThreads = 256;
constexpr int kMseThreads = 256;
constexpr int kMseChunk = 8192;      // elements of one row per CTA: the partition depends on the row length only
constexpr int kFinishThreads = 128;

__global__ void __launch_bounds__(kQThreads) q_sample_kernel(const float* __restrict__ spec, const float* __restrict__ noise,
                                                             long long noise_kstride, const int64_t* __restrict__ lengths,
                                                             const int64_t* __restrict__ t,
                                                             const float* __restrict__ sqrt_ac,
                                                             const float* __restrict__ sqrt_1mac, int timesteps,
                                                             float* __restrict__ x_start, float* __restrict__ noise_m,
                                                             float* __restrict__ x, int B, int T, int n) {
  const int i = blockIdx.x * kQThreads + threadIdx.x;    // element of the row's [C, T]
  if (i >= n) return;
  const int b = blockIdx.y, k = blockIdx.z;
  const long long tb = t[(long long)k * B + b];
  // a timestep outside the schedule reads no table entry and gives NaN
  const bool ok = tb >= 0 && tb < timesteps;
  const float a = ok ? sqrt_ac[tb] : nanf("");
  const float s = ok ? sqrt_1mac[tb] : nanf("");
  const float m = (i % T) < lengths[b] ? 1.0f : 0.0f;
  const long long row = (long long)b * n + i;
  const float xs = __fmul_rn(spec[row], m);
  const float nm = __fmul_rn(noise[(long long)k * noise_kstride + row], m);
  if (k == 0) x_start[row] = xs;
  if (noise_m != nullptr && (k == 0 || noise_kstride != 0)) noise_m[(long long)k * noise_kstride + row] = nm;
  x[((long long)k * B + b) * n + i] = __fadd_rn(__fmul_rn(a, xs), __fmul_rn(s, nm));
}

// partial[r * P + p] = sum over chunk p of row r of (out - target)^2, r = k * B + b
__global__ void __launch_bounds__(kMseThreads) mse_rows_kernel(const float* __restrict__ out, const float* __restrict__ target,
                                                               long long target_kstride, double* __restrict__ partial, int B,
                                                               int n) {
  __shared__ double s_warp[kMseThreads / 32];
  const int p = blockIdx.x, r = blockIdx.y;
  const int k = r / B, b = r - k * B;
  const float* o = out + (long long)r * n;
  const float* g = target + (long long)k * target_kstride + (long long)b * n;
  const int lo = p * kMseChunk;
  const int hi = min(n, lo + kMseChunk);
  double acc = 0.0;
  for (int i = lo + threadIdx.x; i < hi; i += kMseThreads) {
    const double d = (double)o[i] - (double)g[i];
    acc = fma(d, d, acc);
  }
  for (int w = 16; w > 0; w >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, w);
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double sum = s_warp[0];
    for (int j = 1; j < kMseThreads / 32; ++j) sum += s_warp[j];
    partial[(long long)r * gridDim.x + p] = sum;
  }
}

// One CTA per k: the rows' means, their weights, and the batch's loss.  The reference multiplies the [B, C*T] squared errors by
// the [B, 1, 1] weights (model.py:723-726: its `reduce` flattens without averaging), which broadcasts to [B, B, C*T]; the mean
// of that is mean_b(weight) * mean_b(row MSE), and that product is the number `forward` returns.
__global__ void __launch_bounds__(kFinishThreads) mse_finish_kernel(const double* __restrict__ partial, double* __restrict__ rows,
                                                                    const int64_t* __restrict__ t,
                                                                    const float* __restrict__ loss_weight, int timesteps,
                                                                    float min_snr_gamma, float* __restrict__ loss_row,
                                                                    float* __restrict__ loss_weighted, float* __restrict__ loss,
                                                                    int B, int P, int n) {
  const int k = blockIdx.x;
  for (int b = threadIdx.x; b < B; b += kFinishThreads) {
    const long long r = (long long)k * B + b;
    double sum = 0.0;
    for (int p = 0; p < P; ++p) sum += partial[r * P + p];
    const double mean = sum / (double)n;
    const long long tb = t[r];
    float w = (tb >= 0 && tb < timesteps) ? loss_weight[tb] : nanf("");
    if (min_snr_gamma > 0.0f) w = fminf(w, min_snr_gamma);
    rows[2 * r] = mean;
    rows[2 * r + 1] = (double)w;
    loss_row[r] = (float)mean;
    loss_weighted[r] = (float)(mean * (double)w);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double sum_m = 0.0, sum_w = 0.0;
    for (int b = 0; b < B; ++b) {
      sum_m += rows[2 * ((long long)k * B + b)];
      sum_w += rows[2 * ((long long)k * B + b) + 1];
    }
    loss[k] = (float)((sum_w / (double)B) * (sum_m / (double)B));
  }
}

// The ragged reduction: row r = k * B + b holds C * T_b valid elements, frame f < T_b of channel c at c * T + f of the padded
// [C, T] row.  Element j of the row's own [C, T_b] order is cut into chunks of kMseChunk exactly as mse_rows_kernel cuts a row of
// n = C * T_b, and every thread walks its chunk with the same stride, so the additions and their order depend on (C, T_b) only:
// an utterance's value has the same bits whatever T, B or row it gets.  CTAs past the row's last chunk return at once.  A
// length outside [1, T] gives NaN (mse_ragged_finish_kernel); nothing past a row's length is read.
__global__ void __launch_bounds__(kMseThreads) mse_rows_ragged_kernel(const float* __restrict__ out,
                                                                      const float* __restrict__ target, long long target_kstride,
                                                                      const int64_t* __restrict__ lengths,
                                                                      double* __restrict__ partial, int B, int T, int n) {
  __shared__ double s_warp[kMseThreads / 32];
  const int p = blockIdx.x, r = blockIdx.y;
  const int k = r / B, b = r - k * B;
  const long long len = lengths[b];
  if (len < 1 || len > T) return;
  const int Tb = (int)len;
  const int nb = (n / T) * Tb;                             // C * T_b
  const int lo = p * kMseChunk;
  if (lo >= nb) return;
  const int hi = min(nb, lo + kMseChunk);
  const float* o = out + (long long)r * n;
  const float* g = target + (long long)k * target_kstride + (long long)b * n;
  double acc = 0.0;
  for (int j = lo + threadIdx.x; j < hi; j += kMseThreads) {
    const int c = j / Tb;
    const int i = c * T + (j - c * Tb);
    const double d = (double)o[i] - (double)g[i];
    acc = fma(d, d, acc);
  }
  for (int w = 16; w > 0; w >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, w);
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double sum = s_warp[0];
    for (int j = 1; j < kMseThreads / 32; ++j) sum += s_warp[j];
    partial[(long long)r * gridDim.x + p] = sum;
  }
}

// One thread per row: the row's own chunks added in index order, / (C * T_b), the weight of its t.
__global__ void __launch_bounds__(kFinishThreads) mse_ragged_finish_kernel(const double* __restrict__ partial,
                                                                           const int64_t* __restrict__ lengths,
                                                                           const int64_t* __restrict__ t,
                                                                           const float* __restrict__ loss_weight, int timesteps,
                                                                           float min_snr_gamma, float* __restrict__ loss_row,
                                                                           float* __restrict__ loss_weighted, int rows, int B, int T,
                                                                           int C, int P) {
  const int r = blockIdx.x * kFinishThreads + threadIdx.x;
  if (r >= rows) return;
  const long long len = lengths[r % B];
  double mean = nan("");
  if (len >= 1 && len <= T) {
    const int nb = C * (int)len;
    const int pb = (nb + kMseChunk - 1) / kMseChunk;
    double sum = 0.0;
    for (int p = 0; p < pb; ++p) sum += partial[(long long)r * P + p];
    mean = sum / (double)nb;
  }
  const long long tb = t[r];
  float w = (tb >= 0 && tb < timesteps) ? loss_weight[tb] : nanf("");
  if (min_snr_gamma > 0.0f) w = fminf(w, min_snr_gamma);
  loss_row[r] = (float)mean;
  loss_weighted[r] = (float)(mean * (double)w);
}

inline int mse_chunks(long long n) { return (int)((n + kMseChunk - 1) / kMseChunk); }

}  // namespace
}  // namespace ns2vc

using namespace ns2vc;

extern "C" {

int ns2vc_q_sample(const float* spec, const float* noise, int noise_per_k, const int64_t* lengths, const int64_t* t,
                   const float* sqrt_alphas_cumprod, const float* sqrt_one_minus_alphas_cumprod, int timesteps, float* x_start,
                   float* noise_masked, float* x, int K, int B, int C, int T, ns2vc_stream stream) {
  NS_REQUIRE(spec && noise && lengths && t && sqrt_alphas_cumprod && sqrt_one_minus_alphas_cumprod && x_start && x,
             "q_sample: null argument");
  NS_REQUIRE(K >= 1 && K <= 65535 && B >= 1 && B <= 65535 && C >= 1 && T >= 1 && timesteps >= 1,
             "q_sample: bad sizes K=%d B=%d C=%d T=%d timesteps=%d", K, B, C, T, timesteps);
  const long long n = (long long)C * T;
  NS_REQUIRE(n <= 0x7fffffffLL - kQThreads, "q_sample: C * T = %lld is too long for one row", n);
  const dim3 grid((unsigned)((n + kQThreads - 1) / kQThreads), (unsigned)B, (unsigned)K);
  q_sample_kernel<<<grid, kQThreads, 0, (cudaStream_t)stream>>>(spec, noise, noise_per_k ? (long long)B * n : 0LL, lengths, t,
                                                               sqrt_alphas_cumprod, sqrt_one_minus_alphas_cumprod, timesteps,
                                                               x_start, noise_masked, x, B, T, (int)n);
  NS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int ns2vc_mse_workspace_bytes(int K, int B, int C, int T, size_t* bytes) {
  NS_REQUIRE(bytes != nullptr, "mse_workspace_bytes: null argument");
  NS_REQUIRE(K >= 1 && B >= 1 && C >= 1 && T >= 1, "mse_workspace_bytes: bad sizes K=%d B=%d C=%d T=%d", K, B, C, T);
  const long long rows = (long long)K * B;
  *bytes = (size_t)rows * (size_t)(mse_chunks((long long)C * T) + 2) * sizeof(double);
  return 0;
}

int ns2vc_mse_rows(const float* out, const float* target, int target_per_k, const int64_t* t, const float* loss_weight, int timesteps,
                   float min_snr_gamma, float* loss_row, float* loss_weighted, float* loss, int K, int B, int C, int T, void* ws,
                   ns2vc_stream stream) {
  NS_REQUIRE(out && target && t && loss_weight && loss_row && loss_weighted && loss && ws, "mse_rows: null argument");
  NS_REQUIRE(K >= 1 && B >= 1 && (long long)K * B <= 65535 && C >= 1 && T >= 1 && timesteps >= 1,
             "mse_rows: bad sizes K=%d B=%d (K * B <= 65535) C=%d T=%d timesteps=%d", K, B, C, T, timesteps);
  const long long n = (long long)C * T;
  NS_REQUIRE(n <= 0x7fffffffLL, "mse_rows: C * T = %lld is too long for one row", n);
  NS_REQUIRE(((uintptr_t)ws & 7) == 0, "mse_rows: the workspace must be 8-byte aligned");
  const int P = mse_chunks(n);
  double* partial = (double*)ws;
  double* rows = partial + (long long)K * B * P;
  mse_rows_kernel<<<dim3((unsigned)P, (unsigned)(K * B)), kMseThreads, 0, (cudaStream_t)stream>>>(
      out, target, target_per_k ? (long long)B * n : 0LL, partial, B, (int)n);
  NS_CHECK_CUDA(cudaGetLastError());
  mse_finish_kernel<<<K, kFinishThreads, 0, (cudaStream_t)stream>>>(partial, rows, t, loss_weight, timesteps, min_snr_gamma,
                                                                   loss_row, loss_weighted, loss, B, P, (int)n);
  NS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int ns2vc_mse_ragged_workspace_bytes(int K, int B, int C, int T, size_t* bytes) {
  NS_REQUIRE(bytes != nullptr, "mse_ragged_workspace_bytes: null argument");
  NS_REQUIRE(K >= 1 && B >= 1 && C >= 1 && T >= 1, "mse_ragged_workspace_bytes: bad sizes K=%d B=%d C=%d T=%d", K, B, C, T);
  *bytes = (size_t)K * B * (size_t)mse_chunks((long long)C * T) * sizeof(double);
  return 0;
}

int ns2vc_mse_rows_ragged(const float* out, const float* target, int target_per_k, const int64_t* lengths, const int64_t* t,
                          const float* loss_weight, int timesteps, float min_snr_gamma, float* loss_row, float* loss_weighted, int K,
                          int B, int C, int T, void* ws, ns2vc_stream stream) {
  NS_REQUIRE(out && target && lengths && t && loss_weight && loss_row && loss_weighted && ws, "mse_rows_ragged: null argument");
  NS_REQUIRE(K >= 1 && B >= 1 && (long long)K * B <= 65535 && C >= 1 && T >= 1 && timesteps >= 1,
             "mse_rows_ragged: bad sizes K=%d B=%d (K * B <= 65535) C=%d T=%d timesteps=%d", K, B, C, T, timesteps);
  const long long n = (long long)C * T;
  NS_REQUIRE(n <= 0x7fffffffLL - kMseChunk, "mse_rows_ragged: C * T = %lld is too long for one row", n);
  NS_REQUIRE(((uintptr_t)ws & 7) == 0, "mse_rows_ragged: the workspace must be 8-byte aligned");
  const int P = mse_chunks(n);
  const int rows = K * B;
  mse_rows_ragged_kernel<<<dim3((unsigned)P, (unsigned)rows), kMseThreads, 0, (cudaStream_t)stream>>>(
      out, target, target_per_k ? (long long)B * n : 0LL, lengths, (double*)ws, B, T, (int)n);
  NS_CHECK_CUDA(cudaGetLastError());
  mse_ragged_finish_kernel<<<(rows + kFinishThreads - 1) / kFinishThreads, kFinishThreads, 0, (cudaStream_t)stream>>>(
      (const double*)ws, lengths, t, loss_weight, timesteps, min_snr_gamma, loss_row, loss_weighted, rows, B, T, C, P);
  NS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
