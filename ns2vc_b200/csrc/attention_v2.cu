// Flash attention, v2 (product path): TMA-fed and warp-specialised, sm_90a.
//   out = softmax(q k^T * dh^-0.5 + bias) v      (reference attention_processor.py:1025-1036)
//
// CTA = 128 queries of one (batch, head); key tiles of 64; 288 threads:
//   warp 0      one elected thread is the TMA producer: Q once, then a ring of {K_hi, K_lo, V_hi, V_lo} tiles, plain 3-D
//               boxes of the hi/lo "split" tensors the projection GEMMs wrote (no conversion, no transpose).
//   warps 1-8   16 query rows each (flash_mma.cuh); a warp hands a ring stage back as soon as it is done with it.
// Shared-memory rows of the Q/K/V tiles are `PB` bytes wide (32/64/128 = the TMA box width and swizzle mode), so a dh=16
// head moves 32 B per key instead of a padded 128 B row.
#include "flash_mma.cuh"
#include "tc_common.cuh"
#include "launch.cuh"
#include <math.h>
#include <cstdlib>

namespace ns2vc {

namespace {

constexpr int kQ = 128, kKeys = 64;
constexpr int kThreadsV2 = 288;                          // warp 0: TMA producer (one elected thread); warps 1-8: 16 query rows each

template <int DHP, int PB, bool PF16, bool BIAS> struct ACfg {
  static constexpr int NST = (PB == 128) ? 2 : 3;
  static constexpr int kQBytes = kQ * PB;            // Q hi (lo follows)
  static constexpr int kTBytes = kKeys * PB;         // one K or V tile (hi or lo)
  static constexpr int kStageBytes = 4 * kTBytes;    // K_hi | K_lo | V_hi | V_lo
  static constexpr int kOffQ = 0;
  static constexpr int kOffKV = 2 * kQBytes;
  static constexpr int kOffBar = kOffKV + NST * kStageBytes;
  static constexpr int kOffBias = kOffBar + 256;     // additive bias * log2(e) (or -inf past Tk) for up to kBiasKeys keys
  static constexpr int kBiasKeys = (PB == 32) ? 768 : 1024;
  static constexpr int kSmem = kOffBias + (BIAS ? 4 * kBiasKeys : 0) + 1024 /*alignment slack*/;
  // The scores, output and Q fragments of a warp's 16 rows live in registers.  128-byte rows (d_h 48 / 64) need ~150-170 per
  // thread: one CTA per SM without spills measured faster than two with spills (H100, 741 vs 837 us of attention per forward).
  static constexpr int kMinCtas = (PB == 128) ? 1 : (kSmem <= 113 * 1024) ? 2 : 1;
};

// RAGK: per-entry key counts (op.key_len, the denoiser's ragged self-attention): entry b runs exactly the key tiles, and the tail
// mask, of a run over its own keys alone
template <int DHP, int PB, bool BIAS, bool PF16, bool RAGK = false>
__global__ void __launch_bounds__(kThreadsV2, ACfg<DHP, PB, PF16, BIAS>::kMinCtas) attn_v2_kernel(const __grid_constant__ AttnOp op) {
  using C = ACfg<DHP, PB, PF16, BIAS>;
  constexpr int NST = C::NST;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (base - raw);
  const uint32_t bar0 = base + C::kOffBar;
  const uint32_t q_full = bar0;
  auto kv_full = [&](int s) { return bar0 + 8u + 8u * s; };
  auto kv_empty = [&](int s) { return bar0 + 8u + 8u * (NST + s); };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * kQ;
  const int dh = op.dh;
  const int ntiles = (op.Tk + kKeys - 1) / kKeys;

  span_begin(op.span);
  // diagnostics: [start, end, SM id] of every CTA at trace[256 + 3 * linear CTA id] (globaltimer ns)
  const int cta_lin = (blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
  if (op.trace && tid == 0 && cta_lin < 597) {
    unsigned smid; asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    op.trace[256 + 3 * cta_lin] = gtime_ns();
    op.trace[256 + 3 * cta_lin + 2] = smid;
  }
  if (tid == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < NST; ++s) { mbar_init(kv_full(s), 1); mbar_init(kv_empty(s), 8); }
    mbar_fence_init();
  }
  if (warp == 0 && lane == 0) {
#pragma unroll
    for (int i = 0; i < 6; ++i) prefetch_tmap(&op.tm[i]);
  }
  pdl_trigger();
  __syncthreads();
  const uint32_t sQ = base + C::kOffQ, sKV = base + C::kOffKV;

  if (warp == 0) {
    if (elect_one()) {
      auto load_kv = [&](int j) {
        const int stage = j % NST;
        const uint32_t dst = sKV + stage * C::kStageBytes;
        mbar_arrive_expect_tx(kv_full(stage), (uint32_t)C::kStageBytes);
        tma_load_3d(dst, &op.tm[2], op.k_c0 + h * dh, j * kKeys, b, kv_full(stage));
        tma_load_3d(dst + C::kTBytes, &op.tm[3], op.k_c0 + h * dh, j * kKeys, b, kv_full(stage));
        tma_load_3d(dst + 2 * C::kTBytes, &op.tm[4], op.v_c0 + h * dh, j * kKeys, b, kv_full(stage));
        tma_load_3d(dst + 3 * C::kTBytes, &op.tm[5], op.v_c0 + h * dh, j * kKeys, b, kv_full(stage));
      };
      pdl_wait();                                           // q / k / v are the previous kernels' outputs
      int nt = ntiles;
      if constexpr (RAGK) nt = min(ntiles, (((__ldg(op.key_len + b) - 1) >> op.key_shift) + kKeys) / kKeys);
      mbar_arrive_expect_tx(q_full, 2u * C::kQBytes);
      tma_load_3d(sQ, &op.tm[0], op.q_c0 + h * dh, q0, b, q_full);
      tma_load_3d(sQ + C::kQBytes, &op.tm[1], op.q_c0 + h * dh, q0, b, q_full);
      for (int j = 0; j < nt; ++j) {
        if (j >= NST) mbar_wait(kv_empty(j % NST), (uint32_t)(((j / NST) & 1) ^ 1));   // every warp is done with tile j - NST
        load_kv(j);
      }
    }
  } else {
    // ===================== attention warps =====================
    float* bias_s = reinterpret_cast<float*>(smem + C::kOffBias);
    const float qscale = op.scale * 1.4426950408889634f;
    pdl_wait();                                             // the mask bias and the output buffers belong to earlier kernels
    int tk = op.Tk, nt = ntiles;
    if constexpr (RAGK) { tk = min(tk, ((__ldg(op.key_len + b) - 1) >> op.key_shift) + 1); nt = (tk + kKeys - 1) / kKeys; }
    if (BIAS) {                                             // additive mask bias * log2(e); -inf past Tk
      const float* bias = op.bias + (long long)b * op.Tk;
      for (int i = tid - 32; i < ntiles * kKeys; i += 256)
        bias_s[i] = (i < op.Tk) ? __ldg(bias + i) * 1.4426950408889634f : -INFINITY;
      asm volatile("bar.sync 1, 256;" ::: "memory");
    }
    FlashWarp<DHP, PB, PF16> fw;
    const int r0 = 16 * (warp - 1);
    mbar_wait(q_full, 0);
    fw.load_q(sQ, sQ + C::kQBytes, r0, lane);
    for (int j = 0; j < nt; ++j) {
      const int stage = j % NST;
      mbar_wait_quiet(kv_full(stage), (uint32_t)((j / NST) & 1));
      const uint32_t kst = sKV + stage * C::kStageBytes;
      fw.tile(kst, kst + C::kTBytes, kst + 2 * C::kTBytes, kst + 3 * C::kTBytes, BIAS ? bias_s + j * kKeys : nullptr, qscale,
              (RAGK ? tk : op.Tk) - j * kKeys, lane);
      __syncwarp();
      if (lane == 0) mbar_arrive(kv_empty(stage));
    }
    fw.store(op, b, h, q0 + r0, lane);
  }
  __syncthreads();
  span_end(op.span);
  if (op.trace && tid == 0 && cta_lin < 597) op.trace[256 + 3 * cta_lin + 1] = gtime_ns();
}

template <int DHP, int PB, bool BIAS, bool PF16, bool RAGK = false>
int launch_v2b(const AttnOp& op, cudaStream_t st) {
  using C = ACfg<DHP, PB, PF16, BIAS>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(attn_v2_kernel<DHP, PB, BIAS, PF16, RAGK>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmem);
    if (e != cudaSuccess) { set_error("attention v2: cannot set %d B dynamic smem: %s", C::kSmem, cudaGetErrorString(e)); return -2; }
    // ask for the largest shared-memory carve-out: the CTA count per SM is what the smem budget above was sized for
    cudaFuncSetAttribute(attn_v2_kernel<DHP, PB, BIAS, PF16, RAGK>, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared);
    if (getenv("NS2VC_DEBUG")) {
      int nb = 0;
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, attn_v2_kernel<DHP, PB, BIAS, PF16, RAGK>, kThreadsV2, (size_t)C::kSmem);
      fprintf(stderr, "ns2vc: attn_v2<%d,%d,bias=%d,f16=%d> smem %d B, planned %d CTAs/SM, occupancy API says %d\n", DHP, PB, (int)BIAS, (int)PF16, C::kSmem, C::kMinCtas, nb);
    }
    attr_set = true;
  }
  dim3 grid(ceil_div(op.Tq, kQ), op.H, op.B);
  cudaError_t e = launch_k(attn_v2_kernel<DHP, PB, BIAS, PF16, RAGK>, grid, dim3(kThreadsV2), (size_t)C::kSmem, st, op);
  if (e != cudaSuccess) { set_error("attention v2 launch failed: %s", cudaGetErrorString(e)); return -2; }
  return 0;
}
// Softmax weights: fp16 (one P*[V_hi|V_lo] MMA per k-step; the weights are DEFINED as the rounded values, so the result
// is an exact weighted mean with weights perturbed by <= 2^-12 relative) or bf16 hi/lo split (NS2VC_ATTN_P=split).
bool p_fp16() { return attention_v2_p_fp16(); }
template <int DHP, int PB>
int launch_v2(const AttnOp& op, cudaStream_t st) {
  if (op.key_len) {
    if (op.bias) { set_error("attention v2: per-entry key counts take no additive bias"); return -1; }
    return (p_fp16() && !op.p_split) ? launch_v2b<DHP, PB, false, true, true>(op, st) : launch_v2b<DHP, PB, false, false, true>(op, st);
  }
  if (op.bias) {
    if (ceil_div(op.Tk, kKeys) * kKeys > ACfg<DHP, PB, true, true>::kBiasKeys) { set_error("attention v2: %d biased keys exceed the staged-bias capacity", op.Tk); return -1; }
    return (p_fp16() && !op.p_split) ? launch_v2b<DHP, PB, true, true>(op, st) : launch_v2b<DHP, PB, true, false>(op, st);
  }
  return (p_fp16() && !op.p_split) ? launch_v2b<DHP, PB, false, true>(op, st) : launch_v2b<DHP, PB, false, false>(op, st);
}

int natural_pb(int dh) { return dh == 16 ? 32 : dh == 32 ? 64 : 128; }

}  // namespace

bool attention_v2_p_fp16() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("NS2VC_ATTN_P"); v = (e && e[0] == 's') ? 0 : 1; }
  return v == 1;
}

bool attention_v2_supported(int dh, int Tk, bool biased) {
  if (!(dh == 16 || dh == 32 || dh == 48 || dh == 64)) return false;
  return !biased || ceil_div(Tk, kKeys) * kKeys <= (dh == 16 ? 768 : 1024);   // the additive bias of a row of keys is staged in shared memory
}

int encode_attn_tmaps(AttnOp& op) {
  op.pb = natural_pb(op.dh);                                // (padded 128-byte rows for every head dim were measured slower in r01)
  const int bc = op.pb / 2;                                 // box width in channels
  int rc = 0;
  if ((rc = encode_tmap_rows(&op.tm[0], op.qs.hi, op.qs.C, op.qs.T, op.B, op.qs.ld, bc, kQ, op.pb))) return rc;
  if ((rc = encode_tmap_rows(&op.tm[1], op.qs.lo, op.qs.C, op.qs.T, op.B, op.qs.ld, bc, kQ, op.pb))) return rc;
  if ((rc = encode_tmap_rows(&op.tm[2], op.ks.hi, op.ks.C, op.ks.T, op.B, op.ks.ld, bc, kKeys, op.pb))) return rc;
  if ((rc = encode_tmap_rows(&op.tm[3], op.ks.lo, op.ks.C, op.ks.T, op.B, op.ks.ld, bc, kKeys, op.pb))) return rc;
  if ((rc = encode_tmap_rows(&op.tm[4], op.vs.hi, op.vs.C, op.vs.T, op.B, op.vs.ld, bc, kKeys, op.pb))) return rc;
  if ((rc = encode_tmap_rows(&op.tm[5], op.vs.lo, op.vs.C, op.vs.T, op.B, op.vs.ld, bc, kKeys, op.pb))) return rc;
  return 0;
}

int launch_attention_v2(const AttnOp& op, cudaStream_t st) {
  if (op.Tk <= 0 || op.Tq <= 0) { set_error("attention: empty sequence"); return -1; }
  if (op.qs.T != op.Tq || op.ks.T != op.Tk || op.vs.T != op.Tk) { set_error("attention v2: split buffer / sequence length mismatch"); return -1; }
  const int dh = op.dh;
  if (op.pb == 128) {
    if (dh == 48) return launch_v2<48, 128>(op, st);
    if (dh == 64) return launch_v2<64, 128>(op, st);
  } else if (op.pb == 64 && dh == 32) {
    return launch_v2<32, 64>(op, st);
  } else if (op.pb == 32 && dh == 16) {
    return launch_v2<16, 32>(op, st);
  }
  set_error("attention v2: unsupported head dim %d / box %d", dh, op.pb);
  return -1;
}

}  // namespace ns2vc
