// Small HBM/L2-bound kernels of the denoiser step: layout conversion, GroupNorm/LayerNorm
// statistics, the timestep/FiLM GEMV and AttentionPooling pieces.
// All are coalesced/vectorised; none is worth tensor cores.
#include "gemm_common.cuh"
#include "prep_common.cuh"
#include "launch.cuh"
#include <cstdarg>
#include <cstdio>
#include <math.h>

namespace ns2vc {

static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* get_error() { return g_err; }

#define NS_LAUNCH_CHECK()                                                                      \
  do {                                                                                         \
    cudaError_t _e = cudaGetLastError();                                                       \
    if (_e != cudaSuccess) {                                                                   \
      set_error("%s:%d launch failed: %s", __FILE__, __LINE__, cudaGetErrorString(_e));        \
      return -2;                                                                               \
    }                                                                                          \
  } while (0)

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---------------------------------------------------------------------------------------------
// Layout conversion.  32x32 smem tile transpose, coalesced on both sides.
// ---------------------------------------------------------------------------------------------
__global__ void nct_to_tokens_kernel(const float* __restrict__ x, long long bstride, int C, int T,
                                     float* __restrict__ out, int ldo, int Cpad) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const float* xb = x + (long long)b * bstride;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int c = c0 + i, t = t0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && t < T) ? xb[(long long)c * T + t] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int t = t0 + i, c = c0 + threadIdx.x;
    if (t < T && c < Cpad) out[((long long)b * T + t) * ldo + c] = tile[threadIdx.x][i];
  }
}
int launch_nct_to_tokens(const TokensOp& op, cudaStream_t st) {
  dim3 grid(ceil_div(op.T, 32), ceil_div(op.ld, 32), op.B), block(32, 8);
  nct_to_tokens_kernel<<<grid, block, 0, st>>>(op.x, op.bstride, op.C, op.T, op.out, op.ld, op.ld);
  NS_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------------
// LayerNorm row statistics (one warp per row; two-pass in registers, C <= 2048).
// ---------------------------------------------------------------------------------------------
template <bool APPLY>
__global__ void __launch_bounds__(256) ln_kernel(const float* __restrict__ x, int ld, int M, int C, float eps,
                                                 float* __restrict__ stats, const float* __restrict__ gamma,
                                                 const float* __restrict__ beta, float* __restrict__ y, int y_ld) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const float* xr = x + (long long)row * ld;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += xr[c];
  const float mean = warp_sum(s) / (float)C;
  float q = 0.f;
  for (int c = lane; c < C; c += 32) { float d = xr[c] - mean; q += d * d; }
  const float var = warp_sum(q) / (float)C;
  const float rstd = 1.0f / sqrtf(var + eps);
  if (APPLY) {
    float* yr = y + (long long)row * y_ld;
    for (int c = lane; c < C; c += 32) yr[c] = (xr[c] - mean) * rstd * gamma[c] + beta[c];
  } else if (lane == 0) {
    stats[2 * row] = mean;
    stats[2 * row + 1] = rstd;
  }
}
int launch_ln_apply(const LnOp& op, cudaStream_t st) {
  ln_kernel<true><<<ceil_div(op.M, 8), 256, 0, st>>>(op.x, op.ld, op.M, op.C, op.eps, nullptr, op.gamma, op.beta, op.y, op.y_ld);
  NS_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------------
// Activation prep: concat(src1, src2) -> [per-(b,c) affine (+SiLU)] -> bf16 hi/lo split, optionally a
// second untransformed split (the resnet's 1x1 shortcut operand).  One thread = 8 channels of one
// row (two 16-byte loads, 16-byte hi + lo stores); rows may be remapped (stride-2 decimation for
// the downsample convs, nearest-upsample index table).
// ---------------------------------------------------------------------------------------------
// RAG: ragged programs (op.row_len): rows past the entry's length are zeros, the GroupNorm counts only the valid rows
template <bool RAG>
__global__ void __launch_bounds__(256) prep_split_kernel(PrepOp op) {
  span_begin(op.span);
  pdl_trigger();
  extern __shared__ float aff[];                         // [2][C] scale | shift of this block's batch entry
  const int C = op.C1 + op.C2;
  float pg[kPrepSlots], pb[kPrepSlots];
  prep_fetch_norm_weights(op, C, pg, pb, threadIdx.x, blockDim.x);   // weights: before griddepcontrol.wait
  pdl_wait();
  const int b = blockIdx.y;
  const int chunks = op.out.ld >> 3;                     // 8-channel chunks per output row (incl. zero padding)
  const int total = op.T_dst * chunks;
  const int stride = gridDim.x * blockDim.x;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  // the first chunk's loads are in flight while the block derives the GroupNorm affine
  PrepChunk k0;
  const bool have = i < total;
  if (have) prep_load_at<RAG>(op, b, C, i / chunks, i % chunks, k0);
  float fs[kPrepSlots], fb[kPrepSlots];
  prep_fetch_film(op, op.gn.film, b, C, fs, fb, threadIdx.x, blockDim.x);
  prep_affine<RAG>(op, b, C, C, aff, pg, pb, fs, fb, threadIdx.x, blockDim.x, BlockSync());
  if (have) prep_finish(op, b, C, aff, k0);
  for (i += stride; i < total; i += stride) {
    PrepChunk k;
    prep_load_at<RAG>(op, b, C, i / chunks, i % chunks, k);
    prep_finish(op, b, C, aff, k);
  }
  span_end(op.span);
}
int launch_prep_split(const PrepOp& op, cudaStream_t st) {
  if ((op.out.ld & 7) || (op.raw.hi && op.raw.ld != op.out.ld)) { set_error("prep_split: bad pitch"); return -1; }
  const int C = op.C1 + op.C2;
  if (op.mode != PREP_RAW && !op.scale && (C % op.gn.G)) { set_error("prep_split: %d channels not divisible by %d groups", C, op.gn.G); return -1; }
  const int total = op.T_dst * (op.out.ld >> 3);
  int bx = (total + 255) / 256;
  const int cap = (132 * 8 + op.B - 1) / op.B;           // ~8 blocks per SM over the whole grid
  if (bx > cap) bx = cap;
  if (bx < 1) bx = 1;
  const size_t smem = (op.mode != PREP_RAW) ? (size_t)prep_affine_floats(C) * sizeof(float) : 0;
  if (smem > 48 * 1024 || (op.mode != PREP_RAW && !op.scale && (C > kPrepSlots * 256 || op.gn.G > 64))) { set_error("prep_split: C=%d too large", C); return -1; }
  cudaError_t e = op.row_len ? launch_k(prep_split_kernel<true>, dim3(bx, op.B), dim3(256), smem, st, op)
                             : launch_k(prep_split_kernel<false>, dim3(bx, op.B), dim3(256), smem, st, op);
  if (e != cudaSuccess) { set_error("prep_split launch failed: %s", cudaGetErrorString(e)); return -2; }
  return 0;
}

// LayerNorm + split: one warp per row, two-pass statistics in registers (C <= 1024).
// KEEP: rows with keep[row] == 0 store hi = lo = 0 (the condition encoders' ragged programs: a k > 1 conv over the split then
// reads zeros past an entry's length, as an unpadded run reads its zero padding).
template <bool KEEP>
__global__ void __launch_bounds__(256) ln_split_kernel(const float* __restrict__ x, int ld, int M, int C, float eps,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                                       SplitBuf out, unsigned long long* span, const float* __restrict__ keep) {
  span_begin(span);
  pdl_trigger();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  constexpr int kMaxChunks = 4;                            // 8-channel chunks per lane: C <= 32*8*4
  // gamma / beta are weights: fetch them while the producer of x is still running (before griddepcontrol.wait)
  float gm[kMaxChunks][8], bt[kMaxChunks][8];
#pragma unroll
  for (int k = 0; k < kMaxChunks; ++k) {
    const int c0 = (lane + 32 * k) * 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) { gm[k][j] = 0.f; bt[k][j] = 0.f; }
    if (c0 + 8 <= C && ((reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(beta)) & 15) == 0) {
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c0)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + c0) + 1);
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + c0)), b1 = __ldg(reinterpret_cast<const float4*>(beta + c0) + 1);
      gm[k][0] = g0.x; gm[k][1] = g0.y; gm[k][2] = g0.z; gm[k][3] = g0.w; gm[k][4] = g1.x; gm[k][5] = g1.y; gm[k][6] = g1.z; gm[k][7] = g1.w;
      bt[k][0] = b0.x; bt[k][1] = b0.y; bt[k][2] = b0.z; bt[k][3] = b0.w; bt[k][4] = b1.x; bt[k][5] = b1.y; bt[k][6] = b1.z; bt[k][7] = b1.w;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) if (c0 + j < C) { gm[k][j] = __ldg(gamma + c0 + j); bt[k][j] = __ldg(beta + c0 + j); }
    }
  }
  pdl_wait();
  if (row >= M) { span_end(span); return; }
  const float* xr = x + (long long)row * ld;
  float v[kMaxChunks][8];
  const int chunks = (C + 7) >> 3;
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < kMaxChunks; ++k) {
    const int ck = lane + 32 * k;
#pragma unroll
    for (int j = 0; j < 8; ++j) v[k][j] = 0.f;
    if (ck < chunks) {
      const int c0 = ck * 8;
      if (c0 + 8 <= C && ((ld & 3) == 0)) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(xr + c0)), b4 = __ldg(reinterpret_cast<const float4*>(xr + c0) + 1);
        v[k][0] = a.x; v[k][1] = a.y; v[k][2] = a.z; v[k][3] = a.w; v[k][4] = b4.x; v[k][5] = b4.y; v[k][6] = b4.z; v[k][7] = b4.w;
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) if (c0 + j < C) v[k][j] = xr[c0 + j];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[k][j];
    }
  }
  const float mean = warp_sum(s) / (float)C;
  float q = 0.f;
#pragma unroll
  for (int k = 0; k < kMaxChunks; ++k) {
    const int ck = lane + 32 * k;
    if (ck < chunks) {
#pragma unroll
      for (int j = 0; j < 8; ++j) if (ck * 8 + j < C) { const float d = v[k][j] - mean; q += d * d; }
    }
  }
  const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)C + eps);
  const bool live = !KEEP || keep[row] != 0.f;
  const int ochunks = out.ld >> 3;
#pragma unroll
  for (int k = 0; k < kMaxChunks; ++k) {
    const int ck = lane + 32 * k;
    if (ck < ochunks) {
      const int c0 = ck * 8;
      float y[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = c0 + j;
        y[j] = (c < C && live) ? (v[k][j] - mean) * rstd * gm[k][j] + bt[k][j] : 0.f;
      }
      uint4 hi, lo;
      split8(y, hi, lo);
      *reinterpret_cast<uint4*>(out.hi + (long long)row * out.ld + c0) = hi;
      *reinterpret_cast<uint4*>(out.lo + (long long)row * out.ld + c0) = lo;
    }
  }
  span_end(span);
}
int launch_ln_split(const LnOp& op, cudaStream_t st) {
  const SplitBuf& out = op.split;
  if (op.C > 1024 || (out.ld & 7) || out.ld > 1024) { set_error("ln_split: C=%d / pitch %d unsupported", op.C, out.ld); return -1; }
  unsigned long long* span = nullptr;
  const dim3 grid(ceil_div(op.M, 8)), block(256);
  if (op.keep) launch_k(ln_split_kernel<true>, grid, block, 0, st, op.x, op.ld, op.M, op.C, op.eps, op.gamma, op.beta, out, span, op.keep);
  else launch_k(ln_split_kernel<false>, grid, block, 0, st, op.x, op.ld, op.M, op.C, op.eps, op.gamma, op.beta, out, span, op.keep);
  NS_LAUNCH_CHECK();
  return 0;
}

// [B, C, T] fp32 -> split token-major [B, T, out.ld]; 32x32 smem transpose, zero-fills c >= C (RAG: and t >= row_len[b]).
template <bool RAG>
__global__ void nct_to_split_kernel(const float* __restrict__ x, long long bstride, int C, int T, SplitBuf out,
                                    const char* warm, long long warm_bytes, const int* __restrict__ row_len) {
  pdl_trigger();
  // first kernel of a forward: pull this step's FiLM rows (a slice of the run's timestep table, cold in L2) towards L2 so that
  // the 22 conv2 launches that read them later do not each wait for HBM
  if (warm) {
    const long long line = ((long long)(blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) * (blockDim.x * blockDim.y) + threadIdx.y * blockDim.x + threadIdx.x;
    if (line * 128 < warm_bytes) asm volatile("prefetch.global.L2 [%0];" ::"l"(warm + line * 128));
  }
  pdl_wait();
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const float* xb = x + (long long)b * bstride;
  int Tv = T;
  if constexpr (RAG) Tv = min(T, __ldg(row_len + b));
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int c = c0 + i, t = t0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && t < Tv) ? xb[(long long)c * T + t] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int t = t0 + i, c = c0 + threadIdx.x;
    if (t < T && c < out.ld) {
      const float v = tile[threadIdx.x][i];
      const __nv_bfloat16 h = __float2bfloat16_rn(v);
      const long long off = ((long long)b * T + t) * out.ld + c;
      out.hi[off] = h;
      out.lo[off] = __float2bfloat16_rn(v - __bfloat162float(h));
    }
  }
}
int launch_nct_to_split(const NctSplitOp& op, cudaStream_t st) {
  dim3 grid(ceil_div(op.T, 32), ceil_div(op.out.ld, 32), op.B), block(32, 8);
  const char* warm = (const char*)op.warm;
  if (op.row_len) launch_k(nct_to_split_kernel<true>, grid, block, 0, st, op.x, op.bstride, op.C, op.T, op.out, warm, op.warm_bytes, op.row_len);
  else launch_k(nct_to_split_kernel<false>, grid, block, 0, st, op.x, op.bstride, op.C, op.T, op.out, warm, op.warm_bytes, op.row_len);
  NS_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------------
// Small-M linear (timestep MLP, batched FiLM projections, AttentionPooling projections).
// One warp per output column n; the input rows (<= 8 at a time) live in shared memory.
// HBM-bound on W (read once per launch when M <= 8).
// ---------------------------------------------------------------------------------------------
constexpr int kLinRows = 8;
__global__ void __launch_bounds__(256) small_linear_kernel(LinOp op) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ float xs[];   // [kLinRows][K]
  const int m0 = blockIdx.y * kLinRows;
  const int rows = min(kLinRows, op.M - m0);
  const int K = op.K;
  const bool vec_in = op.in_mode != LIN_SINUSOID && op.x_ld == K && (K & 3) == 0 && (reinterpret_cast<uintptr_t>(op.x) & 15) == 0;
  if (vec_in) {
    // contiguous input rows: all 16-byte loads of this thread are in flight before the first use
    const float4* xin = reinterpret_cast<const float4*>(op.x + (long long)m0 * K);
    const int n4 = rows * K / 4;
    for (int i0 = threadIdx.x; i0 < n4; i0 += 4 * blockDim.x) {
      float4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) { const int i = i0 + u * blockDim.x; v[u] = (i < n4) ? __ldg(xin + i) : make_float4(0.f, 0.f, 0.f, 0.f); }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + u * blockDim.x;
        if (i < n4) {
          if (op.in_mode == LIN_SILU) {
            v[u].x = v[u].x / (1.0f + expf(-v[u].x)); v[u].y = v[u].y / (1.0f + expf(-v[u].y));
            v[u].z = v[u].z / (1.0f + expf(-v[u].z)); v[u].w = v[u].w / (1.0f + expf(-v[u].w));
          }
          reinterpret_cast<float4*>(xs)[i] = v[u];
        }
      }
    }
  }
  for (int i = threadIdx.x; !vec_in && i < rows * K; i += blockDim.x) {
    int r = i / K, k = i % K;
    float v;
    if (op.in_mode == LIN_SINUSOID) {
      // reference embeddings.py:41-59: emb = t * exp(-ln(1e4) * i / (half - shift)); [sin | cos], flipped
      const int half = K / 2;
      const float t = op.x[(long long)(m0 + r) * op.x_ld];
      if (k >= 2 * half) {
        v = 0.f;
      } else {
        bool first = k < half;
        int i2 = first ? k : k - half;
        float ex = (-9.210340371976184f * (float)i2) / ((float)half - op.freq_shift);
        float arg = t * expf(ex);
        bool use_cos = op.flip_sin_to_cos ? first : !first;
        v = use_cos ? cosf(arg) : sinf(arg);
      }
    } else {
      v = op.x[(long long)(m0 + r) * op.x_ld + k];
      if (op.in_mode == LIN_SILU) v = v / (1.0f + expf(-v));
    }
    xs[r * K + k] = v;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= op.N) return;
  const float* wr = op.W + (long long)n * K;
  float acc[kLinRows];
#pragma unroll
  for (int r = 0; r < kLinRows; ++r) acc[r] = 0.f;
  if ((K & 127) == 0 && (reinterpret_cast<uintptr_t>(wr) & 15) == 0) {
    // the weight row is the only HBM traffic: issue up to four 16-byte loads per lane before the first FMA so a warp
    // pays one memory latency per 512 weights instead of one per 32
    for (int k0 = 0; k0 < K; k0 += 512) {
      float4 w[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int k = k0 + u * 128 + lane * 4;
        w[u] = (k < K) ? __ldg(reinterpret_cast<const float4*>(wr + k)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int k = k0 + u * 128 + lane * 4;
        if (k < K) {
#pragma unroll
          for (int r = 0; r < kLinRows; ++r) {
            const float4 xv = *reinterpret_cast<const float4*>(xs + r * K + k);
            acc[r] = fmaf(xv.x, w[u].x, acc[r]); acc[r] = fmaf(xv.y, w[u].y, acc[r]);
            acc[r] = fmaf(xv.z, w[u].z, acc[r]); acc[r] = fmaf(xv.w, w[u].w, acc[r]);
          }
        }
      }
    }
  } else {
    for (int k = lane; k < K; k += 32) {
      const float w = __ldg(wr + k);
#pragma unroll
      for (int r = 0; r < kLinRows; ++r) acc[r] = fmaf(xs[r * K + k], w, acc[r]);
    }
  }
#pragma unroll
  for (int r = 0; r < kLinRows; ++r) acc[r] = warp_sum(acc[r]);
  if (lane == 0) {
    const float bv = op.bias ? op.bias[n] : 0.f;
    for (int r = 0; r < rows; ++r) {
      float v = acc[r] + bv;
      if (op.add) v += op.add[(long long)(op.add_rows > 0 ? (m0 + r) % op.add_rows : (m0 + r)) * op.add_ld + n];
      if (op.out_silu) v = v / (1.0f + expf(-v));
      op.out[(long long)(m0 + r) * op.out_ld + n] = v;
    }
  }
}
int launch_small_linear(const LinOp& op, cudaStream_t st) {
  size_t smem = (size_t)kLinRows * op.K * sizeof(float);
  if (smem > 48 * 1024) { set_error("small_linear: K=%d too large", op.K); return -1; }
  dim3 grid(ceil_div(op.N, 8), ceil_div(op.M, kLinRows));
  launch_k(small_linear_kernel, grid, dim3(256), smem, st, op);
  NS_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------------
// AttentionPooling pieces (reference embeddings.py:499-546); once per utterance.
// ---------------------------------------------------------------------------------------------
// RAG: the class token is the mean over the entry's first lens[b] frames (the utterance's own prompt)
template <bool RAG>
__global__ void pool_class_token_kernel(const float* __restrict__ xn, const float* __restrict__ pos, int S, int C,
                                        float* __restrict__ tokens, const int* __restrict__ lens) {
  const int b = blockIdx.x;
  const int Sb = RAG ? lens[b] : S;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f;
    for (int t = 0; t < Sb; ++t) s += xn[((long long)b * S + t) * C + c];
    tokens[((long long)b * (S + 1)) * C + c] = s / (float)Sb + pos[c];
    for (int t = 0; t < S; ++t) tokens[((long long)b * (S + 1) + 1 + t) * C + c] = xn[((long long)b * S + t) * C + c];
  }
}
int launch_pool_class_token(const PoolClsOp& op, cudaStream_t st) {
  if (op.lens) pool_class_token_kernel<true><<<op.B, 256, 0, st>>>(op.x, op.pos, op.S, op.C, op.tokens, op.lens);
  else pool_class_token_kernel<false><<<op.B, 256, 0, st>>>(op.x, op.pos, op.S, op.C, op.tokens, op.lens);
  NS_LAUNCH_CHECK();
  return 0;
}

// one warp per (b, head): softmax over S1 keys of (q*s).(k*s), s = dph^-1/4; out = sum_j w_j v_j
// RAG: over the class token and the entry's first lens[b] frames only
template <bool RAG>
__global__ void pool_attend_kernel(const float* __restrict__ q, const float* __restrict__ kv, int S1, int C, int heads,
                                   float* __restrict__ out, const int* __restrict__ lens) {
  const int b = blockIdx.x / heads, h = blockIdx.x % heads;
  const int K1 = RAG ? lens[b] + 1 : S1;                 // keys attended (kv rows keep the stride S1)
  const int dph = C / heads;
  const int lane = threadIdx.x;
  const float sc = 1.0f / sqrtf(sqrtf((float)dph));
  const float* qh = q + (long long)b * C + h * dph;
  float mx = -INFINITY;
  for (int j = lane; j < K1; j += 32) {
    const float* kr = kv + ((long long)b * S1 + j) * 2 * C + h * dph;
    float s = 0.f;
    for (int d = 0; d < dph; ++d) s += (qh[d] * sc) * (kr[d] * sc);
    mx = fmaxf(mx, s);
  }
  mx = warp_max(mx);
  float den = 0.f;
  float acc[16];
  for (int d = 0; d < 16; ++d) acc[d] = 0.f;
  for (int j = lane; j < K1; j += 32) {
    const float* kr = kv + ((long long)b * S1 + j) * 2 * C + h * dph;
    float s = 0.f;
    for (int d = 0; d < dph; ++d) s += (qh[d] * sc) * (kr[d] * sc);
    float p = expf(s - mx);
    den += p;
    const float* vr = kr + C;
    for (int d = 0; d < dph && d < 16; ++d) acc[d] += p * vr[d];
  }
  den = warp_sum(den);
  for (int d = 0; d < dph && d < 16; ++d) {
    float a = warp_sum(acc[d]);
    if (lane == 0) out[(long long)b * C + h * dph + d] = a / den;
  }
}
int launch_pool_attend(const PoolAttOp& op, cudaStream_t st) {
  if (op.C % op.heads || op.C / op.heads > 16) { set_error("pool_attend: dim/head %d/%d unsupported", op.C, op.heads); return -1; }
  if (op.lens) pool_attend_kernel<true><<<op.B * op.heads, 32, 0, st>>>(op.q, op.kv, op.S1, op.C, op.heads, op.out, op.lens);
  else pool_attend_kernel<false><<<op.B * op.heads, 32, 0, st>>>(op.q, op.kv, op.S1, op.C, op.heads, op.out, op.lens);
  NS_LAUNCH_CHECK();
  return 0;
}

// bool mask -> additive bias, bit-exact with (1 - m) * -10000 (reference unet_1d_condition.py:817)
__global__ void mask_bias_kernel(const uint8_t* __restrict__ mask, int n, float* __restrict__ bias) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) bias[i] = (1.0f - (mask[i] ? 1.0f : 0.0f)) * -10000.0f;
}
int launch_mask_bias(const MaskBiasOp& op, cudaStream_t st) {
  mask_bias_kernel<<<ceil_div(op.n, 256), 256, 0, st>>>(op.mask, op.n, op.bias);
  NS_LAUNCH_CHECK();
  return 0;
}

// Ragged programs: one block per batch entry turns its content / prompt lengths into the program's tables.  The key biases are
// -inf (not the reference mask's -10000): the attention kernels already stage -inf for keys past Tk, so a masked key contributes
// exactly 0 to the online softmax, and the staged bias row of a short utterance equals that of the utterance run alone.
// Block i fills entry b0 + i, so one entry's tables can be rewritten without touching the others'.
__global__ void ragged_tables_kernel(const long long* __restrict__ clen, const long long* __restrict__ plen, RaggedTables r, int b0) {
  const int b = b0 + blockIdx.x;
  const int T = (int)min(max(clen[b], 1LL), (long long)r.T), S = (int)min(max(plen[b], 1LL), (long long)r.S);
  if (threadIdx.x == 0) { r.lens[b] = T; r.lens[r.B + b] = S; }
  for (int s = threadIdx.x; s < r.S; s += blockDim.x) r.prompt_bias[(long long)b * r.S + s] = s < S ? 0.f : -INFINITY;
  for (int l = 0; l < r.nlev; ++l) {
    if (!r.key_bias[l]) continue;
    const int Tl = r.Tl[l], tb = ((T - 1) >> l) + 1;
    for (int t = threadIdx.x; t < Tl; t += blockDim.x) r.key_bias[l][(long long)b * Tl + t] = t < tb ? 0.f : -INFINITY;
  }
}
int launch_ragged_tables(const long long* content_lengths, const long long* prompt_lengths, const RaggedTables& r, cudaStream_t st,
                         int b0, int n) {
  if (r.nlev > kRagMaxLevels) { set_error("ragged tables: %d levels", r.nlev); return -1; }
  if (n <= 0) n = r.B;
  if (b0 < 0 || b0 + n > r.B) { set_error("ragged tables: entries [%d, %d) of %d", b0, b0 + n, r.B); return -1; }
  ragged_tables_kernel<<<n, 256, 0, st>>>(content_lengths, prompt_lengths, r, b0);
  NS_LAUNCH_CHECK();
  return 0;
}

}  // namespace ns2vc
