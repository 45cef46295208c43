// Warp-level flash-attention core on the sm_90 tensor cores (mma.sync m16n8k16, fp32 accumulators in registers).
// One warp owns 16 query rows.  Per tile of 64 keys: S = Q K^T as three bf16 MMAs over the hi/lo splits (fp32-level
// products, see gemm_tc.cu), online softmax in registers, then O += P V with P straight from the score registers (the C
// fragment of two adjacent n8 tiles is the A fragment of one k16 step) and V read with ldmatrix.trans.  P is fp16 (the
// weights ARE the rounded values: numerator and row sum agree) or a bf16 hi/lo split.
// Q / K / V tiles are rows of PB bytes (32 / 64 / 128) in shared memory, in the TMA's SWIZZLE_<PB>B pattern.
#pragma once
#include "gemm_common.cuh"
#include <math.h>

namespace ns2vc {

// Shared-memory address of byte `a` of a SWIZZLE_<PB>B tile: 16-byte chunk bits [4, 4 + log2(PB/16)) XOR address bits [7, ...)
template <int PB>
__device__ __forceinline__ uint32_t swz(uint32_t a) { return a ^ (((a >> 7) & (uint32_t)(PB / 16 - 1)) << 4); }

__device__ __forceinline__ float ex2f(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

__device__ __forceinline__ void ldsm_x4(uint32_t a, uint32_t* r) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t a, uint32_t* r) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
#define NS2VC_MMA(name, ty)                                                                                                      \
  __device__ __forceinline__ void name(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {                               \
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32." ty "." ty ".f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};" \
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1)); }
NS2VC_MMA(mma_bf16, "bf16")
NS2VC_MMA(mma_f16, "f16")
#undef NS2VC_MMA

// Fragment ownership (g = lane / 4, t = lane % 4): score s[n][e] is row g + 8 (e / 2), key 8 n + 2 t + e % 2; output o[n][e] is
// row g + 8 (e / 2), head channel 8 n + 2 t + e % 2.
template <int DHP, int PB, bool PF16>
struct FlashWarp {
  static constexpr int KS = DHP / 16;   // k16 steps of Q K^T
  static constexpr int NO = DHP / 8;    // n8 tiles of O
  uint32_t qh[KS][4], ql[KS][4];
  float o[NO][4];
  float m[2], l[2];

  // Q fragments of rows [r0, r0 + 16) of the hi / lo tiles
  __device__ __forceinline__ void load_q(uint32_t sqh, uint32_t sql, int r0, int lane) {
    const uint32_t off = (uint32_t)((r0 + (lane & 7) + 8 * ((lane >> 3) & 1)) * PB + 16 * (lane >> 4));
#pragma unroll
    for (int k = 0; k < KS; ++k) { ldsm_x4(swz<PB>(sqh + off + 32 * k), qh[k]); ldsm_x4(swz<PB>(sql + off + 32 * k), ql[k]); }
#pragma unroll
    for (int n = 0; n < NO; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
    m[0] = m[1] = -INFINITY;
    l[0] = l[1] = 0.f;
  }

  // One tile of 64 keys: K / V hi and lo tiles [64 keys][PB bytes].  score = raw * qs + bias[key] (bias: log2(e)-scaled, -inf
  // past the last key) or, without bias, raw * qs for keys < nvalid and -inf beyond.
  __device__ __forceinline__ void tile(uint32_t skh, uint32_t skl, uint32_t svh, uint32_t svl, const float* bias, float qs, int nvalid, int lane) {
    float s[8][4];
#pragma unroll
    for (int n = 0; n < 8; ++n) s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
    const uint32_t koff = (uint32_t)(((lane & 7) + 8 * (lane >> 4)) * PB + 16 * ((lane >> 3) & 1));
#pragma unroll
    for (int k = 0; k < KS; ++k) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {                      // keys [16 np, 16 np + 16): n8 tiles 2 np, 2 np + 1
        uint32_t kh[4], kl[4];
        const uint32_t a = (uint32_t)(16 * np * PB) + koff + 32 * k;
        ldsm_x4(swz<PB>(skh + a), kh);
        ldsm_x4(swz<PB>(skl + a), kl);
        mma_bf16(s[2 * np], qh[k], kh[0], kh[1]);
        mma_bf16(s[2 * np], ql[k], kh[0], kh[1]);
        mma_bf16(s[2 * np], qh[k], kl[0], kl[1]);
        mma_bf16(s[2 * np + 1], qh[k], kh[2], kh[3]);
        mma_bf16(s[2 * np + 1], ql[k], kh[2], kh[3]);
        mma_bf16(s[2 * np + 1], qh[k], kl[2], kl[3]);
      }
    }
    const int t = lane & 3;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int n = 0; n < 8; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = 8 * n + 2 * t + (e & 1);
        float v = s[n][e] * qs;
        if (bias) v += bias[key];
        else if (key >= nvalid) v = -INFINITY;
        s[n][e] = v;
        mx[e >> 1] = fmaxf(mx[e >> 1], v);
      }
    float corr[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 1));
      mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 2));
      const float mn = fmaxf(m[i], mx[i]);
      corr[i] = ex2f(m[i] - mn);
      m[i] = mn;
      l[i] *= corr[i];
    }
#pragma unroll
    for (int n = 0; n < NO; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) o[n][e] *= corr[e >> 1];
    const uint32_t voff = (uint32_t)(((lane & 7) + 8 * ((lane >> 3) & 1)) * PB + 16 * (lane >> 4));
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {                        // keys [16 kk, 16 kk + 16)
      uint32_t ph[4], pl[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {                         // a0..a3 = (n 2kk, rows g), (2kk, g+8), (2kk+1, g), (2kk+1, g+8)
        float* sv = s[2 * kk + (u >> 1)] + 2 * (u & 1);
        const float p0 = ex2f(sv[0] - m[u & 1]), p1 = ex2f(sv[1] - m[u & 1]);
        if (PF16) {
          ph[u] = pack_f16x2(p0, p1);
          l[u & 1] += f16lo_to_f32(ph[u]) + f16hi_to_f32(ph[u]);
        } else {
          split2(p0, p1, ph[u], pl[u]);
          l[u & 1] += p0 + p1;
        }
      }
#pragma unroll
      for (int dp = 0; dp < NO / 2; ++dp) {                 // head channels [16 dp, 16 dp + 16): n8 tiles 2 dp, 2 dp + 1
        uint32_t vh[4], vl[4];
        const uint32_t a = (uint32_t)(16 * kk * PB) + voff + 32 * dp;
        ldsm_x4_t(swz<PB>(svh + a), vh);
        ldsm_x4_t(swz<PB>(svl + a), vl);
        if (PF16) {
          mma_f16(o[2 * dp], ph, vh[0], vh[1]);
          mma_f16(o[2 * dp], ph, vl[0], vl[1]);
          mma_f16(o[2 * dp + 1], ph, vh[2], vh[3]);
          mma_f16(o[2 * dp + 1], ph, vl[2], vl[3]);
        } else {
          mma_bf16(o[2 * dp], ph, vh[0], vh[1]);
          mma_bf16(o[2 * dp], pl, vh[0], vh[1]);
          mma_bf16(o[2 * dp], ph, vl[0], vl[1]);
          mma_bf16(o[2 * dp + 1], ph, vh[2], vh[3]);
          mma_bf16(o[2 * dp + 1], pl, vh[2], vh[3]);
          mma_bf16(o[2 * dp + 1], ph, vl[2], vl[3]);
        }
      }
    }
  }

  // Normalise and store rows [r0, r0 + 16) (query index q0 + row) of head h: fp32 and / or bf16 hi/lo split output, a channel
  // pair per store where the addresses allow it.
  __device__ __forceinline__ void store(const AttnOp& op, int b, int h, int q0, int lane) {
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      l[i] += __shfl_xor_sync(0xffffffffu, l[i], 1);
      l[i] += __shfl_xor_sync(0xffffffffu, l[i], 2);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int q = q0 + g + 8 * i;
      if (q >= op.Tq) continue;
      const float inv = 1.0f / l[i];
      const long long orow = (long long)b * op.Tq + q;
#pragma unroll
      for (int n = 0; n < NO; ++n) {
        const int d = 8 * n + 2 * t;                        // this thread's channel pair d, d + 1
        if (d >= op.dh) continue;
        const float v0 = o[n][2 * i] * inv, v1 = o[n][2 * i + 1] * inv;
        const long long of = orow * op.out_ld + h * op.dh + d, os = orow * op.out_split_ld + h * op.dh + d;
        if (op.out && d + 1 < op.dh && ((of | (long long)(reinterpret_cast<uintptr_t>(op.out) >> 2)) & 1) == 0) {
          *reinterpret_cast<float2*>(op.out + of) = make_float2(v0, v1);
        } else if (op.out) {
          op.out[of] = v0;
          if (d + 1 < op.dh) op.out[of + 1] = v1;
        }
        if (op.out_hi && d + 1 < op.dh &&
            ((os | (long long)(reinterpret_cast<uintptr_t>(op.out_hi) >> 1) | (long long)(reinterpret_cast<uintptr_t>(op.out_lo) >> 1)) & 1) == 0) {
          uint32_t hi, lo;
          split2(v0, v1, hi, lo);
          *reinterpret_cast<uint32_t*>(op.out_hi + os) = hi;
          *reinterpret_cast<uint32_t*>(op.out_lo + os) = lo;
        } else if (op.out_hi) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            if (d + e >= op.dh) break;
            const float v = e ? v1 : v0;
            const __nv_bfloat16 hi = __float2bfloat16_rn(v);
            op.out_hi[os + e] = hi;
            op.out_lo[os + e] = __float2bfloat16_rn(v - __bfloat162float(hi));
          }
        }
      }
    }
  }
};

}  // namespace ns2vc
