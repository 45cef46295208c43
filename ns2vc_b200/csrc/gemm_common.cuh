// Device helpers shared by the wgmma GEMM, the SIMT debug GEMM and the prep kernels.
#pragma once
#include "common.cuh"

namespace ns2vc {

// x * sigmoid(x) = x * rcp(1 + 2^(-x log2 e)): MUFU.EX2 + MUFU.RCP (1-2 ulp each) and three FP32 ops.  For very negative v the
// exponential overflows to +inf (or the reciprocal flushes to 0): the product is -0, which is the limit.  (__fdividef adds a
// range test and two scaling multiplies per element; the panel-mode transform is instruction-issue bound.)
__device__ __forceinline__ float silu_f(float v) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(v * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return v * r;
}

// erf-GELU, as F.gelu default (reference attention.py:295)
// erf via Abramowitz & Stegun 7.1.26 (|error| <= 1.5e-7, far inside the fp32 parity budget); the libm
// erff costs ~3x the instructions and the GEGLU epilogue is issue-latency bound.
__device__ __forceinline__ float gelu_erf_f(float v) {
  const float x = fabsf(v) * 0.70710678118654752440f;
  const float t = __fdividef(1.0f, fmaf(0.3275911f, x, 1.0f));
  float p = fmaf(t, 1.061405429f, -1.453152027f);
  p = fmaf(t, p, 1.421413741f);
  p = fmaf(t, p, -0.284496736f);
  p = fmaf(t, p, 0.254829592f);
  const float erf_abs = 1.0f - p * t * __expf(-x * x);
  return 0.5f * v * (1.0f + copysignf(erf_abs, v));
}

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}

// fp32 pairs packed in one 64-bit value.  sm_90 has no packed fp32x2 arithmetic: each helper is two scalar operations, which
// the compiler sees through (the packing is a register-pair move).
__device__ __forceinline__ unsigned long long pk2(float a, float b) { unsigned long long r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ void upk2(unsigned long long v, float& a, float& b) { asm("mov.b64 {%0, %1}, %2;" : "=f"(a), "=f"(b) : "l"(v)); }
__device__ __forceinline__ unsigned long long ffma2(unsigned long long a, unsigned long long b, unsigned long long c) {
  float a0, a1, b0, b1, c0, c1; upk2(a, a0, a1); upk2(b, b0, b1); upk2(c, c0, c1); return pk2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1)); }
__device__ __forceinline__ unsigned long long fadd2(unsigned long long a, unsigned long long b) {
  float a0, a1, b0, b1; upk2(a, a0, a1); upk2(b, b0, b1); return pk2(__fadd_rn(a0, b0), __fadd_rn(a1, b1)); }
__device__ __forceinline__ unsigned long long fsub2(unsigned long long a, unsigned long long b) {
  float a0, a1, b0, b1; upk2(a, a0, a1); upk2(b, b0, b1); return pk2(__fsub_rn(a0, b0), __fsub_rn(a1, b1)); }
__device__ __forceinline__ unsigned long long fmul2(unsigned long long a, unsigned long long b) {
  float a0, a1, b0, b1; upk2(a, a0, a1); upk2(b, b0, b1); return pk2(__fmul_rn(a0, b0), __fmul_rn(a1, b1)); }

// (a, b) -> packed bf16 hi = rn(a), rn(b) and lo = rn(a - hi_a), rn(b - hi_b): x = hi + lo to ~2^-17 relative.
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  hi = pack_bf16x2(a, b);
  const float ha = __uint_as_float(hi << 16), hb = __uint_as_float(hi & 0xffff0000u);
  float la, lb;
  upk2(fsub2(pk2(a, b), pk2(ha, hb)), la, lb);
  lo = pack_bf16x2(la, lb);
}

// erf-GELU of two values at once (same A&S 7.1.26 polynomial as gelu_erf_f)
__device__ __forceinline__ unsigned long long gelu_erf2(unsigned long long v2) {
  float a, b;
  upk2(v2, a, b);
  const unsigned long long x2 = pk2(fabsf(a) * 0.70710678118654752440f, fabsf(b) * 0.70710678118654752440f);
  float da, db;
  upk2(ffma2(pk2(0.3275911f, 0.3275911f), x2, pk2(1.0f, 1.0f)), da, db);
  float ta, tb;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(ta) : "f"(da));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(tb) : "f"(db));
  const unsigned long long t2 = pk2(ta, tb);
  unsigned long long p2 = ffma2(t2, pk2(1.061405429f, 1.061405429f), pk2(-1.453152027f, -1.453152027f));
  p2 = ffma2(t2, p2, pk2(1.421413741f, 1.421413741f));
  p2 = ffma2(t2, p2, pk2(-0.284496736f, -0.284496736f));
  p2 = ffma2(t2, p2, pk2(0.254829592f, 0.254829592f));
  float ea, eb;
  upk2(fmul2(fmul2(x2, x2), pk2(-1.4426950408889634f, -1.4426950408889634f)), ea, eb);
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(ea) : "f"(ea));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(eb) : "f"(eb));
  float ra, rb;
  upk2(fsub2(pk2(1.0f, 1.0f), fmul2(fmul2(p2, t2), pk2(ea, eb))), ra, rb);     // erf(|x|)
  const unsigned long long one_plus = fadd2(pk2(1.0f, 1.0f), pk2(copysignf(ra, a), copysignf(rb, b)));
  return fmul2(fmul2(v2, pk2(0.5f, 0.5f)), one_plus);
}

// silu of a packed pair
__device__ __forceinline__ unsigned long long silu2(unsigned long long y2) {
  float z0, z1, e0, e1, r0, r1, d0, d1;
  upk2(fmul2(y2, pk2(-1.4426950408889634f, -1.4426950408889634f)), z0, z1);
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e0) : "f"(z0));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e1) : "f"(z1));
  upk2(fadd2(pk2(e0, e1), pk2(1.0f, 1.0f)), d0, d1);
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r0) : "f"(d0));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r1) : "f"(d1));
  return fmul2(y2, pk2(r0, r1));
}

// fp16 flavour of split2 / split8 (operands of the attention's fp16 P x V product)
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) { uint32_t r; asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo)); return r; }
__device__ __forceinline__ float f16lo_to_f32(uint32_t h2) { float f; asm("{.reg .f16 l, h; mov.b32 {l, h}, %1; cvt.f32.f16 %0, l;}" : "=f"(f) : "r"(h2)); return f; }
__device__ __forceinline__ float f16hi_to_f32(uint32_t h2) { float f; asm("{.reg .f16 l, h; mov.b32 {l, h}, %1; cvt.f32.f16 %0, h;}" : "=f"(f) : "r"(h2)); return f; }
__device__ __forceinline__ void split2_f16(float a, float b, uint32_t& hi, uint32_t& lo) {
  hi = pack_f16x2(a, b);
  float la, lb;
  upk2(fsub2(pk2(a, b), pk2(f16lo_to_f32(hi), f16hi_to_f32(hi))), la, lb);
  lo = pack_f16x2(la, lb);
}
__device__ __forceinline__ void split8_f16(const float* v, uint4& hi, uint4& lo) {
  split2_f16(v[0], v[1], hi.x, lo.x); split2_f16(v[2], v[3], hi.y, lo.y);
  split2_f16(v[4], v[5], hi.z, lo.z); split2_f16(v[6], v[7], hi.w, lo.w);
}

// 8 fp32 values -> 16 bytes of bf16 hi and 16 bytes of bf16 lo
__device__ __forceinline__ void split8(const float* v, uint4& hi, uint4& lo) {
  split2(v[0], v[1], hi.x, lo.x); split2(v[2], v[3], hi.y, lo.y);
  split2(v[4], v[5], hi.z, lo.z); split2(v[6], v[7], hi.w, lo.w);
}

// One A element of a segment, as the TMA path sees it (zero outside the source).
__device__ __forceinline__ float a_fetch_split(const GemmOp& op, const GSeg& s, int b, int t, int c) {
  const SplitBuf& src = op.src[s.src];
  const int r = t + s.tap, ch = s.c0 + c;
  if (r < 0 || r >= src.T || ch >= src.C) return 0.f;
  const long long off = (src.bpitch ? (long long)b * src.bpitch + (long long)r * src.ld : ((long long)b * src.T + r) * src.ld) + ch;
  return __bfloat162float(src.hi[off]) + __bfloat162float(src.lo[off]);
}

// LayerNorm statistics of row m from the producer's accumulated row sums (biased variance, reference nn.LayerNorm)
__device__ __forceinline__ void ln_row_stats(const GemmOp& op, long long m, float& mu, float& rstd) {
  const double s = op.ln_stats[m * 2], q = op.ln_stats[m * 2 + 1];
  const double mean = s / (double)op.ln_C;
  double var = q / (double)op.ln_C - mean * mean;
  if (var < 0) var = 0;
  mu = (float)mean;
  rstd = rsqrtf((float)var + op.ln_eps);
}

// Epilogue for one accumulator value at (m = b*T_out + t, logical column n).  For GEGLU the caller
// passes the value accumulator in `acc` and the gate accumulator in `acc_gate`.
template <bool LNF = true, bool VOC = false>
__device__ __forceinline__ float epi_value(const GemmOp& op, int b, long long m, int n, float acc, float acc_gate) {
  if (LNF && (op.flags & EPI_LNFOLD)) {
    float mu, rstd;
    ln_row_stats(op, m, mu, rstd);
    acc = rstd * (acc - mu * __ldg(op.ln_g + n));
    if (op.flags & EPI_GEGLU) acc_gate = rstd * (acc_gate - mu * __ldg(op.ln_g + op.n_valid + n));
  }
  float v = acc;
  if (op.flags & EPI_GEGLU) {
    const int half = op.n_valid;   // = 4C
    v = (acc + __ldg(op.bias + n)) * gelu_erf_f(acc_gate + __ldg(op.bias + half + n));
  } else if (op.flags & EPI_BIAS) {
    v += __ldg(op.bias + n);
  }
  if (op.flags & EPI_ROWBIAS) v += __ldg(op.rowbias + (long long)b * op.rowbias_ld + n);
  if (op.flags & EPI_RESIDUAL) v += __ldg(op.res + m * op.res_ld + n);
  if (VOC && (op.flags & EPI_GELU)) v = gelu_erf_f(v);
  if (op.flags & EPI_RELU) v = fmaxf(v, 0.f);
  if (op.flags & EPI_ROWMASK) v *= __ldg(op.rowmask + m);
  return v;
}

}  // namespace ns2vc
