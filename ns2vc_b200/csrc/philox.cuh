// Counter-based sampler noise: Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011; the generator
// curand's Philox4_32_10 and torch's CUDA generator are built on) and a Box-Muller transform of its outputs.
//
// Layout, fixed for every kernel that draws sampler noise:
//   key     = the utterance's 64-bit seed (lo, hi)
//   counter = (t >> 2, c, step, 0): one call yields frames t & ~3 .. t | 3 of channel c
//   step    = the row's own step index k within its schedule; kXtStep (0xFFFFFFFF) is reserved for the utterance's x_T
//   frames  t & 3 = 0, 1: z0, z1 of the output pair (x, y); t & 3 = 2, 3: z0, z1 of the pair (z, w)
// So the value at (seed, step, c, t) depends on nothing else: not on T, the row's length, the batch size, the row's slot or the
// launch geometry.  Box-Muller of a pair (a, b):
//   u = fp32((a >> 8) + 0.5) * 2^-24 in (0, 1],  v = (b >> 8) * 2^-24 in [0, 1)
//   r = sqrt(-2 log u),  z0 = r cospi(2v),  z1 = r sinpi(2v)
// v is exact; the sum in u needs 25 bits from 2^23 up and is rounded once to nearest even (u = 1 gives r = 0, never inf or NaN).
// The transform is one __noinline__ function, so every kernel of this translation unit that draws runs the same instructions and
// gets the same bits (the build has no fast-math; logf / sincospif are the precise library functions).
#pragma once
#include <cstdint>

namespace ns2vc {

constexpr uint32_t kXtStep = 0xFFFFFFFFu;

struct PhiloxOut {
  uint32_t x, y, z, w;
};

__host__ __device__ __forceinline__ PhiloxOut philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                                            uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r > 0) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    const uint64_t p0 = (uint64_t)0xD2511F53u * c0;
    const uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
    const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
    const uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
    c1 = (uint32_t)p1;
    c3 = (uint32_t)p0;
    c0 = n0;
    c2 = n2;
  }
  return {c0, c1, c2, c3};
}

// z0 (sin_part false) or z1 (true) of the Box-Muller pair (a, b).
static __device__ __noinline__ float box_muller(uint32_t a, uint32_t b, bool sin_part) {
  const float u = __fmul_rn(__fadd_rn((float)(a >> 8), 0.5f), 5.9604644775390625e-8f);   // 2^-24
  const float v = __fmul_rn((float)(b >> 8), 5.9604644775390625e-8f);
  const float r = __fsqrt_rn(__fmul_rn(-2.0f, logf(u)));
  const float v2 = __fmul_rn(2.0f, v);
  return __fmul_rn(r, sin_part ? sinpif(v2) : cospif(v2));
}

// The normal at (seed, step, c, t) of the layout above.
__device__ __forceinline__ float seeded_normal(uint64_t seed, uint32_t step, uint32_t c, uint32_t t) {
  const PhiloxOut o = philox4x32_10(t >> 2, c, step, 0u, (uint32_t)seed, (uint32_t)(seed >> 32));
  const bool second = (t & 2u) != 0;
  return box_muller(second ? o.z : o.x, second ? o.w : o.y, (t & 1u) != 0);
}

}  // namespace ns2vc
