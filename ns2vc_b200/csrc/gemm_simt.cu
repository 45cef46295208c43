// (1) Weight packing into the wgmma B-operand layout (+ optional fp32 copy for the debug GEMM).
// (2) SIMT fp32 GEMM over the same GemmOp descriptor.  DEBUG/TEST backend only: it is selected
//     with NS2VC_GEMM_BACKEND=simt and exists so the wgmma kernel can be differentially
//     tested on the device; the product path is gemm_tc.cu.
#include "gemm_common.cuh"

namespace ns2vc {

// ---------------------------------------------------------------------------------------------
// Packed B layout: for k-block kb (64 K-values) and packed column n:
//     row (kb*Npad + n) is 128 bytes = 64 bf16 along K, whose 16-byte chunks are XOR-swizzled
//     with (n & 7)  — exactly the shared-memory image of a K-major SWIZZLE_128B wgmma operand,
//     so one contiguous cp.async.bulk of BN*128 bytes loads a [BN x 64] tile.
// w_hi = bf16(w), w_lo = bf16(w - float(w_hi))   (3xBF16 split: hi*hi + hi*lo + lo*hi).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) pack_b_kernel(PackSeg ps, __nv_bfloat16* __restrict__ w_hi,
                                                     __nv_bfloat16* __restrict__ w_lo, float* __restrict__ w_f32,
                                                     int Npad) {
  const long long total = (long long)ps.n_rows * ps.nkb * 64;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int kk = (int)(i % 64);
    const int kbl = (int)((i / 64) % ps.nkb);
    const int nl = (int)(i / (64LL * ps.nkb));          // row within this segment's n range (packed order)
    int n_src = nl;
    if (ps.geglu_half > 0) {
      // packed: 128-column blocks [64 value | 64 gate]; value rows [0,half), gate rows [half, 2*half)
      const int blk = nl / 128, r = nl % 128;
      n_src = (r < 64) ? (blk * 64 + r) : (ps.geglu_half + blk * 64 + (r - 64));
    }
    const int c = kbl * 64 + kk;                          // channel within the segment
    float w = 0.f;
    if (c < ps.ncin) {
      w = ps.w[((long long)n_src * ps.cin_total + ps.cin0 + c) * ps.ktaps + ps.tap];
      if (ps.cscale) w *= ps.cscale[ps.cin0 + c];
    }
    const int n = ps.n_dst0 + nl;
    const int kb = ps.kb0 + kbl;
    const long long row = (long long)kb * Npad + n;
    const int chunk = (kk >> 3) ^ (n & 7);
    const long long off = row * 64 + chunk * 8 + (kk & 7);
    const __nv_bfloat16 hi = __float2bfloat16_rn(w);
    const __nv_bfloat16 lo = __float2bfloat16_rn(w - __bfloat162float(hi));
    w_hi[off] = hi;
    w_lo[off] = lo;
    if (w_f32) w_f32[((long long)kb * 64 + kk) * Npad + n] = w;
  }
}

int launch_pack_b(const PackSeg& ps, __nv_bfloat16* w_hi, __nv_bfloat16* w_lo, float* w_f32, int Npad,
                  cudaStream_t st) {
  const long long total = (long long)ps.n_rows * ps.nkb * 64;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  if (blocks < 1) blocks = 1;
  pack_b_kernel<<<blocks, 256, 0, st>>>(ps, w_hi, w_lo, w_f32, Npad);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_error("pack_b launch failed: %s", cudaGetErrorString(e)); return -2; }
  return 0;
}

// ---------------------------------------------------------------------------------------------
// SIMT debug GEMM: 64x64 tile, BK=16, 256 threads x (4x4) accumulators (x2 for GEGLU).  Reads the
// same split activations the TMA path reads (A = hi + lo) and the fp32 copy of the weights, so a
// disagreement with gemm_tc isolates the TMA / wgmma machinery.
// ---------------------------------------------------------------------------------------------
template <bool GEGLU>
__global__ void __launch_bounds__(256) gemm_simt_kernel(const __grid_constant__ GemmOp op) {
  __shared__ float As[16][64 + 4];
  __shared__ float Bs[GEGLU ? 2 : 1][16][64 + 4];
  const int tid = threadIdx.x;
  const int tiles_per_batch = (op.T_out + 63) / 64;
  const int b = blockIdx.x / tiles_per_batch;
  const int t0 = (blockIdx.x % tiles_per_batch) * 64;
  const int jn = blockIdx.y;                       // output column tile (64 logical columns)
  const int pcol0 = GEGLU ? jn * 128 : jn * 64;    // first packed column
  const int ty = tid / 16, tx = tid % 16;
  float acc[4][4], accg[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) { acc[i][j] = 0.f; accg[i][j] = 0.f; }

  const int ar = tid / 4, ak = (tid % 4) * 4;      // A-load assignment: row ar, 4 channels of each 16-wide slab
  const int at = t0 + ar;
  const int bk = tid / 16, bn = (tid % 16) * 4;    // B-load assignment

  int kb_glob = 0;
  for (int si = 0; si < op.nseg; ++si) {
    const GSeg& s = op.seg[si];
    const int kmax = s.nkb * 64;
    for (int k0 = 0; k0 < kmax; k0 += 16) {
#pragma unroll
      for (int j = 0; j < 4; ++j) As[ak + j][ar] = (at < op.T_out) ? a_fetch_split(op, s, b, at, k0 + ak + j) : 0.f;
      const long long krow = ((long long)kb_glob * 64 + k0 + bk) * op.N;
      const float4 bv = *reinterpret_cast<const float4*>(op.w_f32 + krow + pcol0 + bn);
      Bs[0][bk][bn] = bv.x; Bs[0][bk][bn + 1] = bv.y; Bs[0][bk][bn + 2] = bv.z; Bs[0][bk][bn + 3] = bv.w;
      if (GEGLU) {
        const float4 gv = *reinterpret_cast<const float4*>(op.w_f32 + krow + pcol0 + 64 + bn);
        Bs[GEGLU ? 1 : 0][bk][bn] = gv.x; Bs[GEGLU ? 1 : 0][bk][bn + 1] = gv.y; Bs[GEGLU ? 1 : 0][bk][bn + 2] = gv.z; Bs[GEGLU ? 1 : 0][bk][bn + 3] = gv.w;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < 16; ++kk) {
        float a[4], bb[4], gg[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
        for (int j = 0; j < 4; ++j) { bb[j] = Bs[0][kk][tx * 4 + j]; gg[j] = GEGLU ? Bs[GEGLU ? 1 : 0][kk][tx * 4 + j] : 0.f; }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
            if (GEGLU) accg[i][j] = fmaf(a[i], gg[j], accg[i][j]);
          }
      }
      __syncthreads();
    }
    kb_glob += s.nkb;
  }

#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int t = t0 + ty * 4 + i;
    if (t >= op.T_out) continue;
    const long long m = (long long)b * op.T_out + t;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = jn * 64 + tx * 4 + j;       // logical output column
      if (n >= op.n_valid) continue;
      const float v = epi_value(op, b, m, n, acc[i][j], accg[i][j]);
      if (op.flags & EPI_OUT_NCT) op.out[((long long)b * op.n_valid + n) * op.T_out + t] = v;
      if (op.flags & EPI_OUT_F32) op.out[m * op.out_ld + n] = v;
      if (op.flags & EPI_STATS) {
        atomicAdd(op.stat_sum + (long long)b * op.n_valid + n, (double)v);
        atomicAdd(op.stat_sq + (long long)b * op.n_valid + n, (double)v * (double)v);
      }
      if (op.flags & EPI_ROWSTATS) {
        atomicAdd(op.row_stats + m * 2, (double)v);
        atomicAdd(op.row_stats + m * 2 + 1, (double)v * (double)v);
      }
      if (op.flags & EPI_OUT_SPLIT) {
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        op.out_hi[m * op.out_split_ld + n] = h;
        op.out_lo[m * op.out_split_ld + n] = __float2bfloat16_rn(v - __bfloat162float(h));
      }
    }
  }
}

int launch_gemm_simt(const GemmOp& op, cudaStream_t st) {
  if (!op.w_f32) { set_error("SIMT debug GEMM requested but fp32 weights were not packed (set NS2VC_GEMM_BACKEND=simt before creating the engine)"); return -1; }
  const bool geglu = (op.flags & EPI_GEGLU) != 0;
  const int ncols = geglu ? op.N / 2 : op.N;
  dim3 grid(op.B * ceil_div(op.T_out, 64), ncols / 64);
  if (geglu) gemm_simt_kernel<true><<<grid, 256, 0, st>>>(op);
  else gemm_simt_kernel<false><<<grid, 256, 0, st>>>(op);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_error("gemm_simt launch failed: %s", cudaGetErrorString(e)); return -2; }
  return 0;
}

}  // namespace ns2vc
