// Small kernels of the condition encoders (`Pre_model`, reference model.py:98-190, 328-377): sequence masks, the
// [B, C, T] -> token-major entry with the speaker bias and the padding mask, the masked final LayerNorm, the
// single-head AttentionPooling of `ref_enc`, and the load-time weight reshapes (ConvTBC layout, conv-FFN taps).
// Once per utterance, HBM/L2-bound, none worth tensor cores; the contractions run on gemm_tc.cu / attention*.cu.
#include "common.cuh"
#include "launch.cuh"
#include <math.h>

namespace ns2vc {

#define NS_PRE_LAUNCH_CHECK()                                                                  \
  do {                                                                                         \
    cudaError_t _e = cudaGetLastError();                                                       \
    if (_e != cudaSuccess) {                                                                   \
      set_error("%s:%d launch failed: %s", __FILE__, __LINE__, cudaGetErrorString(_e));        \
      return -2;                                                                               \
    }                                                                                          \
  } while (0)

namespace {
__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float wmax(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
}  // namespace

// sequence_mask (reference modules/commons.py:149-153): keep[b, t] = t < len[b]; the attention's key-padding bias uses the
// denoiser's finite form (1 - keep) * -10000 instead of -inf (operations.py:412-421): exp(-10000 - max) is exactly 0 in fp32
// as long as one key is valid (lengths >= 1), so the softmax weights are identical.  `ilen` (ragged programs, or nullptr): the
// lengths as int [B], clamped to [1, T], for the kernels that take per-entry key counts.
__global__ void seq_mask_kernel(const long long* __restrict__ len, int B, int T, float* __restrict__ keep, float* __restrict__ kbias,
                                int* __restrict__ ilen) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * T) return;
  const int b = i / T, t = i - b * T;
  const float k = ((long long)t < len[b]) ? 1.f : 0.f;
  keep[i] = k;
  kbias[i] = (1.0f - k) * -10000.0f;
  if (ilen && t == 0) ilen[b] = (int)max(1LL, min((long long)T, len[b]));
}
int launch_seq_mask(const SeqMaskOp& op, cudaStream_t st) {
  seq_mask_kernel<<<ceil_div(op.B * op.T, 256), 256, 0, st>>>(op.len, op.B, op.T, op.keep, op.kbias, op.ilen);
  NS_PRE_LAUNCH_CHECK();
  return 0;
}

// Encoder entry (PhoneEncoder.forward model.py:127-128 + ConvLayer.forward :92-93): [B, C, T] (+ spk[b, c]) -> token-major fp32
// [B, T, ld] with padded frames and channels >= C zeroed.  32x32 shared-memory transpose, coalesced on both sides.
__global__ void enc_input_kernel(const float* __restrict__ x, long long bstride, const float* __restrict__ rowbias, const float* __restrict__ keep,
                                 int C, int T, float* __restrict__ out, int ld) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const float* xb = x + (long long)b * bstride;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, t = t0 + threadIdx.x;
    float v = 0.f;
    if (c < C && t < T) v = xb[(long long)c * T + t] + (rowbias ? rowbias[(long long)b * C + c] : 0.f);
    tile[i][threadIdx.x] = v;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int t = t0 + i, c = c0 + threadIdx.x;
    if (t < T && c < ld) {
      const float k = keep[(long long)b * T + t];
      out[((long long)b * T + t) * ld + c] = (k != 0.f && c < C) ? tile[threadIdx.x][i] : 0.f;   // masked_fill(pad, 0): exact zeros
    }
  }
}
int launch_enc_input(const TokensOp& op, cudaStream_t st) {
  dim3 grid(ceil_div(op.T, 32), ceil_div(op.ld, 32), op.B), block(32, 8);
  enc_input_kernel<<<grid, block, 0, st>>>(op.x, op.bstride, op.rowbias, op.keep, op.C, op.T, op.out, op.ld);
  NS_PRE_LAUNCH_CHECK();
  return 0;
}

// Encoder exit (model.py:142-144): y = LayerNorm(x) * keep; one warp per row, two-pass statistics.
__global__ void __launch_bounds__(256) ln_mask_kernel(const float* __restrict__ x, int ld, int M, int C, float eps, const float* __restrict__ gamma,
                                                      const float* __restrict__ beta, const float* __restrict__ keep, float* __restrict__ y, int y_ld) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const float* xr = x + (long long)row * ld;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += xr[c];
  const float mean = wsum(s) / (float)C;
  float q = 0.f;
  for (int c = lane; c < C; c += 32) { const float d = xr[c] - mean; q += d * d; }
  const float rstd = 1.0f / sqrtf(wsum(q) / (float)C + eps);
  const float k = keep[row];
  float* yr = y + (long long)row * y_ld;
  for (int c = lane; c < C; c += 32) yr[c] = ((xr[c] - mean) * rstd * gamma[c] + beta[c]) * k;
}
int launch_ln_mask(const LnOp& op, cudaStream_t st) {
  ln_mask_kernel<<<ceil_div(op.M, 8), 256, 0, st>>>(op.x, op.ld, op.M, op.C, op.eps, op.gamma, op.beta, op.keep, op.y, op.y_ld);
  NS_PRE_LAUNCH_CHECK();
  return 0;
}

// AttentionPooling attend step for any head width (reference unet1d/embeddings.py:521-546; `ref_enc` has ONE head of 100
// channels): one block per (b, head); scores of the S1 keys in shared memory, softmax, then one thread per output channel.
// RAG: over the class token and the entry's first lens[b] frames only (kv rows keep the stride S1).
template <bool RAG>
__global__ void __launch_bounds__(256) pool_attend_wide_kernel(const float* __restrict__ q, const float* __restrict__ kv, int S1, int C, int heads,
                                                               float* __restrict__ out, const int* __restrict__ lens) {
  extern __shared__ float sc_[];                            // [S1] scores -> weights
  __shared__ float red[8];
  __shared__ float bcast;
  const int b = blockIdx.x / heads, h = blockIdx.x % heads;
  const int K1 = RAG ? lens[b] + 1 : S1;
  const int dph = C / heads;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float s4 = 1.0f / sqrtf(sqrtf((float)dph));
  const float* qh = q + (long long)b * C + h * dph;
  float mx = -INFINITY;
  for (int j = tid; j < K1; j += 256) {
    const float* kr = kv + ((long long)b * S1 + j) * 2 * C + h * dph;
    float s = 0.f;
    for (int d = 0; d < dph; ++d) s += (qh[d] * s4) * (kr[d] * s4);
    sc_[j] = s;
    mx = fmaxf(mx, s);
  }
  mx = wmax(mx);
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  if (tid == 0) { float m = red[0]; for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w]); bcast = m; }
  __syncthreads();
  mx = bcast;
  float den = 0.f;
  for (int j = tid; j < K1; j += 256) { const float p = expf(sc_[j] - mx); sc_[j] = p; den += p; }
  den = wsum(den);
  __syncthreads();
  if (lane == 0) red[warp] = den;
  __syncthreads();
  if (tid == 0) { float a = 0.f; for (int w = 0; w < 8; ++w) a += red[w]; bcast = a; }
  __syncthreads();
  den = bcast;
  for (int d = tid; d < dph; d += 256) {
    float a = 0.f;
    for (int j = 0; j < K1; ++j) a += sc_[j] * kv[((long long)b * S1 + j) * 2 * C + C + h * dph + d];
    out[(long long)b * C + h * dph + d] = a / den;
  }
}
int launch_pool_attend_wide(const PoolAttOp& op, cudaStream_t st) {
  if (op.heads < 1 || op.C % op.heads) { set_error("pool_attend: dim/heads %d/%d unsupported", op.C, op.heads); return -1; }
  const size_t smem = (size_t)op.S1 * sizeof(float);
  if (smem > 48 * 1024) { set_error("pool_attend: %d keys do not fit the score buffer", op.S1); return -1; }
  if (op.lens) pool_attend_wide_kernel<true><<<op.B * op.heads, 256, smem, st>>>(op.q, op.kv, op.S1, op.C, op.heads, op.out, op.lens);
  else pool_attend_wide_kernel<false><<<op.B * op.heads, 256, smem, st>>>(op.q, op.kv, op.S1, op.C, op.heads, op.out, op.lens);
  NS_PRE_LAUNCH_CHECK();
  return 0;
}

// ---- load-time reshapes
// ConvTBC weight [k, c_in, c_out] (reference model.py:63-75) -> the conv1d layout [c_out, c_in, k] the weight packer reads
__global__ void tbc_weight_kernel(const float* __restrict__ w, int k, int cin, int cout, float* __restrict__ o) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)k * cin * cout) return;
  const int n = (int)(i % cout), c = (int)((i / cout) % cin), j = (int)(i / ((long long)cout * cin));
  o[((long long)n * cin + c) * k + j] = w[i];
}
int launch_tbc_weight(const float* w, int k, int cin, int cout, float* o, cudaStream_t st) {
  tbc_weight_kernel<<<ceil_div(k * cin * cout, 256), 256, 0, st>>>(w, k, cin, cout, o);
  NS_PRE_LAUNCH_CHECK();
  return 0;
}

// TransformerFFNLayer first stage (reference operations.py:664-692): k Linear layers over k row shifts of the input, summed,
// times k^-0.5.  With `padded` = the input zero-padded by (k-1)/2 frames on both sides, tap i >= 1 reads padded[t + i], i.e. input
// row t + i - (k-1)/2; tap 0 reads the UNPADDED input (the reference's `shifted = padded[i:T+i] if i else x`), i.e. row t - the
// same rows as the centre tap.  Packed here as ONE (k-1)-tap conv weight [F, H, k-1] for the row offsets 1-(k-1)/2 .. (k-1)/2:
// tap j = scale * W_{j+1}, and the centre tap (j = `centre`) also carries scale * W_0.  (ReLU(s z) = s ReLU(z), s > 0.)
struct FfnTaps { const float* w[16]; };
__global__ void ffn_taps_kernel(FfnTaps taps, int k, int F, int H, int centre, float scale, float* __restrict__ o) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)F * H) return;
  for (int j = 0; j < k - 1; ++j) {
    float v = taps.w[j + 1][i];
    if (j == centre) v += taps.w[0][i];
    o[i * (k - 1) + j] = v * scale;
  }
}
__global__ void scale_vec_kernel(const float* __restrict__ a, float s, float* __restrict__ o, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) o[i] = a[i] * s;
}
int launch_ffn_taps(const float* const* w, int k, int F, int H, int centre, float scale, float* o, cudaStream_t st) {
  if (k < 2 || k > 16) { set_error("ffn taps: kernel size %d unsupported", k); return -1; }
  FfnTaps t{};
  for (int i = 0; i < k; ++i) t.w[i] = w[i];
  ffn_taps_kernel<<<ceil_div(F * H, 256), 256, 0, st>>>(t, k, F, H, centre, scale, o);
  NS_PRE_LAUNCH_CHECK();
  return 0;
}
// g[n] = sum_c gamma_c W[n, c],  bf[n] = sum_c beta_c W[n, c] (+ bias[n]): the vectors of a LayerNorm folded into its consumer
// GEMM (EPI_LNFOLD; load time, double accumulation).  Used by both engines.
__global__ void ln_fold_vec_kernel(const float* __restrict__ W, const float* __restrict__ gamma, const float* __restrict__ beta,
                                   const float* __restrict__ bias, float* __restrict__ g, float* __restrict__ bf, int N, int C) {
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (n >= N) return;
  double sg = 0, sb = 0;
  for (int c = lane; c < C; c += 32) { const double w = W[(long long)n * C + c]; sg += w * gamma[c]; sb += w * beta[c]; }
  for (int o = 16; o > 0; o >>= 1) { sg += __shfl_xor_sync(0xffffffffu, sg, o); sb += __shfl_xor_sync(0xffffffffu, sb, o); }
  if (lane == 0) { g[n] = (float)sg; bf[n] = (float)(sb + (bias ? (double)bias[n] : 0.0)); }
}
int launch_ln_fold_vec(const float* W, const float* gamma, const float* beta, const float* bias, float* g, float* bf, int N, int C, cudaStream_t st) {
  ln_fold_vec_kernel<<<ceil_div(N, 8), 256, 0, st>>>(W, gamma, beta, bias, g, bf, N, C);
  NS_PRE_LAUNCH_CHECK();
  return 0;
}
int launch_scale_vec(const float* a, float s, float* o, int n, cudaStream_t st) {
  scale_vec_kernel<<<ceil_div(n, 256), 256, 0, st>>>(a, s, o, n);
  NS_PRE_LAUNCH_CHECK();
  return 0;
}

}  // namespace ns2vc
