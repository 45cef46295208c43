// Scaled-dot-product attention (reference attention_processor.py:1025-1036 -> F.scaled_dot_product_attention):
//   out = softmax(q k^T * dh^-0.5 + bias) v,   8 heads, dh = C/8, no positional term.
// v1: fp32 flash-style kernel on the FMA pipes — one query row per thread, K/V tiles staged in
// shared memory (all threads read the same K/V element: broadcast, conflict-free), online softmax
// over 16-key chunks with exp2f and the scale*log2(e) folded into q.
// Self-attention: k/v come from the fused QKV buffer; cross-attention: from the per-utterance
// K/V cache with the additive mask bias (0 / -10000, NOT -inf: reference unet_1d_condition.py:817).
#include "flash_mma.cuh"
#include "tc_common.cuh"
#include "launch.cuh"
#include <math.h>

namespace ns2vc {

constexpr int kAttnThreads = 128;   // query rows per CTA
constexpr int kAttnKeys = 64;       // keys per shared-memory tile
constexpr int kChunk = 16;

template <int DH>
__global__ void __launch_bounds__(kAttnThreads) attn_kernel(AttnOp op) {
  __shared__ float Ks[kAttnKeys][DH];
  __shared__ float Vs[kAttnKeys][DH];
  __shared__ float Bs[kAttnKeys];
  const int b = blockIdx.z, h = blockIdx.y;
  const int tq = blockIdx.x * kAttnThreads + threadIdx.x;
  const bool qv = tq < op.Tq;
  const float qs = op.scale * 1.4426950408889634f;       // fold log2(e): softmax via exp2
  float q[DH], o[DH];
#pragma unroll
  for (int d = 0; d < DH; ++d) { q[d] = 0.f; o[d] = 0.f; }
  if (qv) {
    const float* qp = op.q + ((long long)b * op.Tq + tq) * op.q_ld + h * DH;
#pragma unroll
    for (int d = 0; d < DH; ++d) q[d] = qp[d] * qs;
  }
  float mrun = -INFINITY, lrun = 0.f;
  for (int k0 = 0; k0 < op.Tk; k0 += kAttnKeys) {
    const int nk = min(kAttnKeys, op.Tk - k0);
    __syncthreads();
    for (int i = threadIdx.x; i < kAttnKeys * DH; i += kAttnThreads) {
      const int j = i / DH, d = i % DH;
      float kv = 0.f, vv = 0.f;
      if (j < nk) {
        const long long row = (long long)b * op.Tk + k0 + j;
        kv = op.k[row * op.k_ld + h * DH + d];
        vv = op.v[row * op.v_ld + h * DH + d];
      }
      Ks[j][d] = kv;
      Vs[j][d] = vv;
    }
    for (int j = threadIdx.x; j < kAttnKeys; j += kAttnThreads)
      Bs[j] = (j < nk) ? (op.bias ? op.bias[(long long)b * op.Tk + k0 + j] * 1.4426950408889634f : 0.f) : -INFINITY;
    __syncthreads();
#pragma unroll 1
    for (int c0 = 0; c0 < kAttnKeys; c0 += kChunk) {
      if (c0 >= nk) break;
      float s[kChunk];
      float cmax = -INFINITY;
#pragma unroll
      for (int j = 0; j < kChunk; ++j) {
        float a = Bs[c0 + j];
#pragma unroll
        for (int d = 0; d < DH; ++d) a = fmaf(q[d], Ks[c0 + j][d], a);
        s[j] = a;
        cmax = fmaxf(cmax, a);
      }
      const float mnew = fmaxf(mrun, cmax);
      const float corr = exp2f(mrun - mnew);           // mrun = -inf on the first chunk -> 0
      lrun *= corr;
#pragma unroll
      for (int d = 0; d < DH; ++d) o[d] *= corr;
#pragma unroll
      for (int j = 0; j < kChunk; ++j) {
        const float p = exp2f(s[j] - mnew);            // padded keys: s = -inf -> 0
        lrun += p;
#pragma unroll
        for (int d = 0; d < DH; ++d) o[d] = fmaf(p, Vs[c0 + j][d], o[d]);
      }
      mrun = mnew;
    }
  }
  if (qv) {
    const float inv = 1.0f / lrun;
    if (op.out) {
      float* po = op.out + ((long long)b * op.Tq + tq) * op.out_ld + h * DH;
#pragma unroll
      for (int d = 0; d < DH; ++d) po[d] = o[d] * inv;
    }
    if (op.out_hi) {
      __nv_bfloat16* ph = op.out_hi + ((long long)b * op.Tq + tq) * op.out_split_ld + h * DH;
      __nv_bfloat16* pl = op.out_lo + ((long long)b * op.Tq + tq) * op.out_split_ld + h * DH;
#pragma unroll
      for (int d = 0; d < DH; ++d) {
        const float v = o[d] * inv;
        const __nv_bfloat16 hi = __float2bfloat16_rn(v);
        ph[d] = hi;
        pl[d] = __float2bfloat16_rn(v - __bfloat162float(hi));
      }
    }
  }
}

template <int DH>
static int launch_dh(const AttnOp& op, cudaStream_t st) {
  dim3 grid(ceil_div(op.Tq, kAttnThreads), op.H, op.B);
  attn_kernel<DH><<<grid, kAttnThreads, 0, st>>>(op);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_error("attention launch failed: %s", cudaGetErrorString(e)); return -2; }
  return 0;
}

static int launch_attention_simt(const AttnOp& op, cudaStream_t st) {
  switch (op.dh) {
    case 4: return launch_dh<4>(op, st);
    case 8: return launch_dh<8>(op, st);
    case 12: return launch_dh<12>(op, st);
    case 16: return launch_dh<16>(op, st);
    case 24: return launch_dh<24>(op, st);
    case 32: return launch_dh<32>(op, st);
    case 48: return launch_dh<48>(op, st);
    case 64: return launch_dh<64>(op, st);
    default: set_error("attention: head dim %d not supported (4,8,12,16,24,32,48,64)", op.dh); return -1;
  }
}


// =============================================================================================
// Tensor-core flash attention for fp32 q / k / v (head dims the v2 kernel does not take, and long biased key rows).
//   CTA = 128 queries of one (batch, head), 8 warps of 16 query rows; key tiles of 64.  Q/K/V are read as fp32 rows
//   (fused QKV buffer or the cross-attention K/V cache), split on the fly into bf16 hi/lo and written as SWIZZLE_128B row
//   images [rows][64 channels]; S = Q K^T and O += P V then run on the tensor cores (flash_mma.cuh), exp2 with the softmax
//   scale and log2(e) folded into Q.  The next tile's global loads are in flight while the current one is computed.
// =============================================================================================
constexpr int AQ = 128, AKT = 64;
constexpr int kAttnTcThreads = 256;
constexpr int kOffQ = 0;                 // Q hi [128][64] bf16, lo follows
constexpr int kOffK = 32768;             // K hi [64][64], lo follows
constexpr int kOffV = kOffK + 16384;     // V hi [64 keys][64], lo follows
constexpr int kOffBias = kOffV + 16384;  // 64 floats
constexpr int kAttnSmem = kOffBias + 256 + 1024 /*alignment slack*/;

__device__ __forceinline__ void load8(const float* p, bool row_ok, int d0, int dh, bool vec, float* v) {
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = 0.f;
  if (!row_ok || d0 >= dh) return;
  if (vec) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(p + d0)), b = __ldg(reinterpret_cast<const float4*>(p + d0) + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) if (d0 + j < dh) v[j] = __ldg(p + d0 + j);
  }
}

template <int DHP>
__global__ void __launch_bounds__(kAttnTcThreads, 1) attn_tc_kernel(const AttnOp op) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (base - raw);
  float* bias_s = reinterpret_cast<float*>(smem + kOffBias);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * AQ;
  const int dh = op.dh;
  constexpr int CK = DHP / 8;                              // 8-wide chunks per row
  const float qscale = op.scale * 1.4426950408889634f;
  const bool vq = ((op.q_ld | (h * dh) | dh) & 3) == 0 && (dh & 7) == 0;
  const bool vk = ((op.k_ld | (h * dh)) & 3) == 0 && (dh & 7) == 0;
  const bool vv = ((op.v_ld | (h * dh)) & 3) == 0 && (dh & 7) == 0;

  span_begin(op.span);
  pdl_trigger();
  pdl_wait();

  // ---- Q tile -> smem (scaled, split)
  for (int i = tid; i < AQ * CK; i += kAttnTcThreads) {
    const int row = i / CK, ck = i % CK;
    const int q = q0 + row;
    float v[8];
    load8(op.q + ((long long)b * op.Tq + q) * op.q_ld + h * dh, q < op.Tq, ck * 8, dh, vq, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] *= qscale;
    uint4 hi, lo;
    split8(v, hi, lo);
    const int off = row * 128 + ((ck ^ (row & 7)) << 4);
    *reinterpret_cast<uint4*>(smem + kOffQ + off) = hi;
    *reinterpret_cast<uint4*>(smem + kOffQ + 16384 + off) = lo;
  }

  constexpr int KCH = (AKT * CK + kAttnTcThreads - 1) / kAttnTcThreads;   // K/V chunks per thread
  float kreg[KCH][8], vreg[KCH][8];
  auto load_kv = [&](int k0) {
#pragma unroll
    for (int u = 0; u < KCH; ++u) {
      const int i = tid + u * kAttnTcThreads;
      const int key = i / CK, ck = i % CK;
      const bool ok = (i < AKT * CK) && (k0 + key < op.Tk);
      const long long rowi = (long long)b * op.Tk + k0 + key;
      load8(op.k + rowi * op.k_ld + h * dh, ok, ck * 8, dh, vk, kreg[u]);
      load8(op.v + rowi * op.v_ld + h * dh, ok, ck * 8, dh, vv, vreg[u]);
    }
  };
  auto store_kv = [&](int k0) {
#pragma unroll
    for (int u = 0; u < KCH; ++u) {
      const int i = tid + u * kAttnTcThreads;
      if (i < AKT * CK) {
        const int key = i / CK, ck = i % CK;
        const int off = key * 128 + ((ck ^ (key & 7)) << 4);
        uint4 hi, lo;
        split8(kreg[u], hi, lo);
        *reinterpret_cast<uint4*>(smem + kOffK + off) = hi;
        *reinterpret_cast<uint4*>(smem + kOffK + 8192 + off) = lo;
        split8(vreg[u], hi, lo);
        *reinterpret_cast<uint4*>(smem + kOffV + off) = hi;
        *reinterpret_cast<uint4*>(smem + kOffV + 8192 + off) = lo;
      }
    }
    if (tid < AKT) {
      const int key = k0 + tid;
      bias_s[tid] = (key < op.Tk) ? (op.bias ? __ldg(op.bias + (long long)b * op.Tk + key) * 1.4426950408889634f : 0.f) : -INFINITY;
    }
  };

  const uint32_t sQ = base + kOffQ, sK = base + kOffK, sV = base + kOffV;
  FlashWarp<DHP, 128, false> fw;
  const int ntiles = (op.Tk + AKT - 1) / AKT;
  load_kv(0);
  for (int j = 0; j < ntiles; ++j) {
    store_kv(j * AKT);
    __syncthreads();                                       // Q (first tile), K, V and the bias row are in shared memory
    if (j == 0) fw.load_q(sQ, sQ + 16384, 16 * warp, lane);
    if (j + 1 < ntiles) load_kv((j + 1) * AKT);            // global loads overlap the MMAs + softmax
    fw.tile(sK, sK + 8192, sV, sV + 8192, bias_s, 1.0f, AKT, lane);
    __syncthreads();                                       // every warp is done with K / V before the next store
  }
  fw.store(op, b, h, q0 + 16 * warp, lane);
  span_end(op.span);
}

template <int DHP>
static int launch_attn_tc(const AttnOp& op, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(attn_tc_kernel<DHP>, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnSmem);
    if (e != cudaSuccess) { set_error("attention: cannot set %d B dynamic smem: %s", kAttnSmem, cudaGetErrorString(e)); return -2; }
    attr_set = true;
  }
  dim3 grid(ceil_div(op.Tq, AQ), op.H, op.B);
  cudaError_t e = launch_k(attn_tc_kernel<DHP>, grid, dim3(kAttnTcThreads), (size_t)kAttnSmem, st, op);
  if (e != cudaSuccess) { set_error("attention launch failed: %s", cudaGetErrorString(e)); return -2; }
  return 0;
}

int launch_attention(const AttnOp& op, cudaStream_t st, bool simt) {
  if (op.Tk <= 0 || op.Tq <= 0) { set_error("attention: empty sequence"); return -1; }
  if (simt) return launch_attention_simt(op, st);
  if (op.dh <= 16) return launch_attn_tc<16>(op, st);
  if (op.dh <= 32) return launch_attn_tc<32>(op, st);
  if (op.dh <= 48) return launch_attn_tc<48>(op, st);
  if (op.dh <= 64) return launch_attn_tc<64>(op, st);
  set_error("attention: head dim %d > 64 not supported", op.dh);
  return -1;
}

}  // namespace ns2vc
