// Activation prep shared by the stand-alone prep kernel (kernels_misc.cu) and the GEMM's fused prologue (gemm_tc.cu):
//   concat(src1, src2) -> [per-(b,c) affine (+SiLU)] -> bf16 hi/lo split (+ an untransformed second split)
// One work item = 8 channels of one output row (two 16-byte loads, 16-byte hi + lo stores); rows may be remapped
// (stride-2 decimation for the downsample convs, nearest-upsample index table).
#pragma once
#include "gemm_common.cuh"

namespace ns2vc {

struct PrepChunk { float v[8]; int t, c0; bool rowok; };
constexpr int kPrepSlots = 4;                              // per-thread channel slots of the affine: C <= kPrepSlots * blockDim.x

// Valid rows of batch entry b in a ragged program: ceil(len / 2^shift), the stride-2 conv length rule applied `shift` times
__device__ __forceinline__ int ragged_rows(const int* len, int b, int shift) { return ((__ldg(len + b) - 1) >> shift) + 1; }

// Fetch 8 channels [ck*8, ck*8+8) of output row t (zero outside the sources; RAG: also past the entry's length).
template <bool RAG = false>
__device__ __forceinline__ void prep_load_at(const PrepOp& op, int b, int C, int t, int ck, PrepChunk& k) {
  k.t = t;
  k.c0 = ck * 8;
  int ts;
  if constexpr (RAG) {
    // nearest upsample (rowmap set): this entry's own rule from its length one level down (len_shift + 1) to its length here
    ts = op.rowmap ? nearest_src_index(t, ragged_rows(op.row_len, b, op.len_shift + 1), ragged_rows(op.row_len, b, op.len_shift))
                   : t * op.row_mul + op.row_add;
  } else {
    ts = op.rowmap ? __ldg(op.rowmap + t) : t * op.row_mul + op.row_add;
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) k.v[j] = 0.f;
  k.rowok = ts >= 0 && ts < op.T_src;
  if constexpr (RAG) k.rowok = k.rowok && t < ragged_rows(op.row_len, b, op.len_shift);
  if (k.rowok && k.c0 < C) {
    const int c0 = k.c0;
    const bool in1 = c0 < op.C1;
    const float* p = in1 ? op.src1 + ((long long)b * op.T_src + ts) * op.ld1 + c0
                         : op.src2 + ((long long)b * op.T_src + ts) * op.ld2 + (c0 - op.C1);
    const int lim = in1 ? op.C1 - c0 : C - c0;             // channels left in this source
    const int ldx = in1 ? op.ld1 : op.ld2;
    if (lim >= 8 && ((ldx | (in1 ? c0 : c0 - op.C1)) & 3) == 0) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(p)), c4 = __ldg(reinterpret_cast<const float4*>(p) + 1);
      k.v[0] = a.x; k.v[1] = a.y; k.v[2] = a.z; k.v[3] = a.w; k.v[4] = c4.x; k.v[5] = c4.y; k.v[6] = c4.z; k.v[7] = c4.w;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = c0 + j;
        if (c < C) k.v[j] = (c < op.C1) ? op.src1[((long long)b * op.T_src + ts) * op.ld1 + c]
                                        : op.src2[((long long)b * op.T_src + ts) * op.ld2 + (c - op.C1)];
      }
    }
  }
}

// Transform + split + store one work item.  aff: [C] scale | [C] shift of batch entry b (shared memory).
__device__ __forceinline__ void prep_finish(const PrepOp& op, int b, int C, const float* aff, PrepChunk& k) {
  const long long orow = (long long)b * op.T_dst + k.t;
  if (op.raw.hi) {
    uint4 hi, lo;
    split8(k.v, hi, lo);
    *reinterpret_cast<uint4*>(op.raw.hi + orow * op.raw.ld + k.c0) = hi;
    *reinterpret_cast<uint4*>(op.raw.lo + orow * op.raw.ld + k.c0) = lo;
  }
  if (op.mode != PREP_RAW && k.rowok) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = k.c0 + j;
      if (c < C) {
        float y = fmaf(k.v[j], aff[c], aff[C + c]);
        if (op.mode == PREP_AFFINE_SILU) y = silu_f(y);
        k.v[j] = y;
      }
    }
  }
  uint4 hi, lo;
  split8(k.v, hi, lo);
  *reinterpret_cast<uint4*>(op.out.hi + orow * op.out.ld + k.c0) = hi;
  *reinterpret_cast<uint4*>(op.out.lo + orow * op.out.ld + k.c0) = lo;
}

// The affine is derived by a group of `nthr` threads (the whole block of the prep kernel, or the 8 transform warps of the
// GEMM) identified by tid in [0, nthr); `sync` is that group's barrier.
struct BlockSync { __device__ __forceinline__ void operator()() const { __syncthreads(); } };

// GroupNorm gamma / beta are weights: they can be fetched before the producer of the activations has finished.
__device__ __forceinline__ void prep_fetch_norm_weights(const PrepOp& op, int C, float* pg, float* pb, int tid, int nthr) {
#pragma unroll
  for (int k = 0; k < kPrepSlots; ++k) {
    const int c = tid + k * nthr;
    const bool ok = op.mode != PREP_RAW && !op.scale && c < C;
    pg[k] = ok ? __ldg(op.gn.gamma + c) : 0.f;
    pb[k] = ok ? __ldg(op.gn.beta + c) : 0.f;
  }
}

// FiLM rows are produced by the timestep path (an earlier kernel): fetched right after the dependency wait, in flight together
// with the statistics and the first activation loads instead of behind the group reduction.
__device__ __forceinline__ void prep_fetch_film(const PrepOp& op, const float* film, int b, int C, float* fs, float* fb, int tid, int nthr) {
#pragma unroll
  for (int k = 0; k < kPrepSlots; ++k) {
    const int c = tid + k * nthr;
    const bool ok = film && op.mode != PREP_RAW && !op.scale && c < C;
    fs[k] = ok ? 1.f + film[(long long)b * op.gn.film_ld + c] : 1.f;
    fb[k] = ok ? film[(long long)b * op.gn.film_ld + C + c] : 0.f;
  }
}

// Per-(b, channel) scale / shift of batch entry b into aff[0..C) | aff[Cs..Cs+C) (Cs = stride of the shift row; uses
// aff[2*Cs .. 2*Cs + 2G) as scratch).  GroupNorm finalise from the per-channel sums the producer epilogues accumulated
// (reference nn.GroupNorm: biased variance over T x C/G elements; resnet.py:536,557, transformer_1d.py:134), then
// (1 + scale) / shift of the FiLM row (resnet.py:627-629).  Called by every thread of the group; ends with sync().
// RAG: the statistics cover the entry's valid rows only (the producers stored zeros past them): n = rows_b x C/G.
template <bool RAG = false, class Sync>
__device__ __forceinline__ void prep_affine(const PrepOp& op, int b, int C, int Cs, float* aff, const float* pg, const float* pb,
                                            const float* fs, const float* fb, int tid, int nthr, Sync sync) {
  if (op.mode == PREP_RAW) return;
  if (op.scale) {
    for (int c = tid; c < C; c += nthr) { aff[c] = op.scale[(long long)b * C + c]; aff[Cs + c] = op.shift[(long long)b * C + c]; }
  } else {
    const GnStats& g = op.gn;
    const int cpg = C / g.G;
    float* gmean = aff + 2 * Cs;                         // [G] mean | [G] rstd
    for (int grp = tid >> 5; grp < g.G; grp += nthr >> 5) {
      double s = 0, q = 0;
      for (int ii = tid & 31; ii < cpg; ii += 32) {
        const int c = grp * cpg + ii;
        s += (c < op.C1) ? g.sum1[(long long)b * op.C1 + c] : g.sum2[(long long)b * op.C2 + (c - op.C1)];
        q += (c < op.C1) ? g.sq1[(long long)b * op.C1 + c] : g.sq2[(long long)b * op.C2 + (c - op.C1)];
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); q += __shfl_xor_sync(0xffffffffu, q, o); }
      if ((tid & 31) == 0) {
        double inv;
        if constexpr (RAG) inv = 1.0 / ((double)ragged_rows(op.row_len, b, op.len_shift) * cpg);
        else inv = g.inv_n != 0.0 ? g.inv_n : 1.0 / ((double)op.T_src * cpg);   // (a double division is ~0.1 us on the launch's critical path)
        const double mean = s * inv;
        double var = q * inv - mean * mean;
        if (var < 0) var = 0;
        gmean[grp] = (float)mean;
        gmean[g.G + grp] = rsqrtf((float)var + g.eps);
      }
    }
    sync();
#pragma unroll
    for (int k = 0; k < kPrepSlots; ++k) {
      const int c = tid + k * nthr;
      if (c >= C) break;
      const int grp = c / cpg;
      float ga = pg[k] * gmean[g.G + grp];
      float be = pb[k] - gmean[grp] * ga;
      ga = ga * fs[k];                                       // FiLM: x * (1 + scale) + shift (identity when there is none)
      be = be * fs[k] + fb[k];
      aff[c] = ga;
      aff[Cs + c] = be;
    }
  }
  sync();
}

// Shared-memory floats prep_affine() needs for C channels
__host__ __device__ constexpr int prep_affine_floats(int C) { return 2 * C + 2 * 64; }

}  // namespace ns2vc
