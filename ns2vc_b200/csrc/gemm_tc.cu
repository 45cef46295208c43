// wgmma implicit-GEMM kernel for every contraction of the denoiser step (k=3 convs, 1x1 convs,
// linears), sm_90a.
//
//   D[128 x BN] (fp32, registers) += A_hi*B_hi + A_lo*B_hi + A_hi*B_lo          (3xBF16 split)
//
// fp32-level parity with the reference (rtol 1e-3 / atol 1e-4) cannot be met by single-pass
// bf16/tf32 MMAs (SURVEY.md Appendix D), so both operands are split x = hi + lo (bf16 each) and
// three bf16 wgmmas accumulate into the same fp32 tile (the lo*lo term, ~2^-16 relative, is dropped).
//
// A operand: the pre-normalised "split" activations [B, T, C] (bf16 hi / lo), fetched by TMA
// (cp.async.bulk.tensor.3d, SWIZZLE_128B) as {64 channels x 128 rows} boxes of ONE batch entry.
// A conv tap is the same box shifted by one row; rows before 0 / past T and channels past C are
// zero-filled by the TMA unit, which is the conv's zero padding and the ragged-edge handling at
// once.  Channel concats are just two tensor maps.
// B operand: weights pre-packed as the swizzled smem image, one cp.async.bulk per hi/lo tile.
//
// One output tile per CTA, 384 threads:
//   warp 0      TMA producer (one elected lane): 3-4 stage mbarrier ring
//   warps 1-3   idle (they keep warps 4-11 aligned to warpgroups)
//   warps 4-11  two warpgroups (tile rows [0, 64) / [64, 128)): wgmma into registers, parked in shared memory as a fp32 tile;
//               the epilogue reads it one row per thread -> bias / GEGLU / residual -> TMA bulk stores (fp32, 16-bit hi/lo)
#include "gemm_common.cuh"
#include "prep_common.cuh"
#include "tc_common.cuh"
#include "launch.cuh"
#include <cuda.h>
#include <cuda_fp16.h>
#include <cstdlib>

namespace ns2vc {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int kEpiWarps = 8;                            // two per SMSP: the epilogue is issue-latency bound
constexpr int kThreads = (4 + kEpiWarps) * 32;
constexpr int kATileBytes = BM * BK * 2;                // 16 KB: one bf16 [128 x 64] A tile (hi or lo)

constexpr int kMaxStages = 4;
// Per-warp staging area of the epilogue: 8 KB per warp =
//   [0, 4096)    fp32 chunk  [32 rows][32 cols]  as a SWIZZLE_128B box image
//   [4096, 6144) 16-bit hi   [32 rows][32 cols]  as a SWIZZLE_64B box image,  [6144, 8192) 16-bit lo
constexpr int kStagePerWarp = 8192;
constexpr int kStageOff = 8192;                         // the staging area starts with two GroupNorm partial-sum buffers (tile parity), <= 4 KB each
constexpr int kStagingBytes = kStageOff + kEpiWarps * kStagePerWarp;   // 68 KB

// Panel mode (GemmOp::xmode): per 64-channel block the hi and lo panels of 136 rows (130 used: t0-1 .. t0+128) go through a
// three-stage ring (TMA -> normalise -> MMA), the weight tiles (hi | lo) of up to three taps through a two-stage ring of
// their own; the affine table sits behind them.
constexpr int kPanelRows = BM + 2;
constexpr int kPanelBytes = 136 * 128;                   // 17 KB: 1024-byte aligned so that hi and lo panels share the swizzle phase
constexpr int kXAStageBytes = 2 * kPanelBytes;           // hi | lo panel of one 64-channel block
constexpr int kXBStageBytes = 3 * 2 * (64 * BK * 2);     // weight tiles (hi | lo) of up to three taps
constexpr int kXAStages = 3;                             // TMA -> normalise -> MMA: three panels in flight
constexpr int kXBStages = 2;
constexpr int kXOffB = kXAStages * kXAStageBytes;        // 104 448
constexpr int kXOffAff = kXOffB + kXBStages * kXBStageBytes;   // [Cs] scale | [Cs] shift | [2 G] group statistics (floats), Cs = kXfMaxC
constexpr int kXAffBytes = (2 * kXfMaxC + 2 * 64) * 4;

template <int BN_> struct TileCfg {
  static constexpr int BN = BN_;
  static constexpr int kBTileBytes = BN_ * BK * 2;      // one bf16 [BN x 64] B tile (hi or lo)
  static constexpr int kStageBytes = 2 * kATileBytes + 2 * kBTileBytes;
  // once the main loop is done the epilogue uses the idle stage buffers: staging area, then the parked accumulator tile
  static constexpr int kStagesSingle = (BN_ == 128) ? 3 : 4;
  static constexpr int kOffAcc = kStagingBytes;
  static constexpr int kPipeBytes = (kStagesSingle * kStageBytes > kXOffAff + kXAffBytes) ? kStagesSingle * kStageBytes : kXOffAff + kXAffBytes;
  static constexpr int kOffBar = kPipeBytes;
  static constexpr int kOffDesc = kOffBar + 1024;
  static constexpr int kOffLnG = kOffDesc + 3072;         // [8 warps][4][32] floats: folded-LayerNorm g and bias vectors of the warp's chunk
  static constexpr int kSmemBytes = kOffLnG + 4096 + 1024 /*alignment slack*/;
};
static_assert(TileCfg<64>::kSmemBytes <= 227 * 1024 && TileCfg<128>::kSmemBytes <= 227 * 1024, "shared memory budget");
static_assert(kXOffAff + kXAffBytes <= TileCfg<64>::kPipeBytes && kPrepSlots * kEpiWarps * 32 >= kXfMaxC, "panel mode: stages + affine table inside the pipeline area");
// panel mode: the accumulator is parked in the weight ring, behind the area a split-K partner writes its partial tile into
constexpr int kXOffAcc = kXOffB + 8 * 256 * 16;
static_assert(kXOffAcc + BM * 64 * 4 <= kXOffAff, "panel mode: parked accumulator inside the weight ring");
static_assert(TileCfg<64>::kOffAcc + BM * 64 * 4 <= TileCfg<64>::kStagesSingle * TileCfg<64>::kStageBytes &&
              TileCfg<128>::kOffAcc + BM * 128 * 4 <= TileCfg<128>::kStagesSingle * TileCfg<128>::kStageBytes, "parked accumulator inside the stage buffers");


__device__ __forceinline__ float* stage_f32_ptr(uint8_t* st, int row, int c4) {      // 16-byte group c4 (0..7) of row
  return reinterpret_cast<float*>(st + row * 128 + ((c4 ^ (row & 7)) << 4));
}

// ---- Cold paths, OUT OF LINE.  Partial chunks (n_valid not a multiple of 32), unaligned leading dimensions and the channel-major
// output of the head are rare; inlined into the epilogue (32-fold unrolled element code) they were half of the kernel's
// instructions and raised its register pressure: 2.90 -> 2.74 ms per forward with them compiled out.  The thread parks its 32
// values in its row of the warp's fp32 staging chunk and these element loops work on that row.

// Element-wise epilogue (bias / GEGLU / row bias / residual / folded LayerNorm) of this thread's parked row; gate values of a
// GEGLU chunk are parked as plain [32 rows][32] floats behind the fp32 chunk (the 16-bit staging area).
template <bool LNF, bool VOC = false>
__device__ __noinline__ void epi_cold(const GemmOp& op, int b, long long m, int nbase, uint8_t* st, int lane, bool with_gate) {
#pragma unroll 1
  for (int j = 0; j < 32; ++j) {
    float* pv = stage_f32_ptr(st, lane, j >> 2) + (j & 3);
    const float g = with_gate ? reinterpret_cast<const float*>(st + 4096)[lane * 32 + j] : 0.f;
    *pv = (nbase + j < op.n_valid) ? epi_value<LNF, VOC>(op, b, m, nbase + j, *pv, g) : 0.f;
  }
}
// Element-wise stores of this thread's parked row in the layout(s) `flags` asks for (channel-major, fp32 or split rows).
__device__ __noinline__ void store_cold(const GemmOp& op, int flags, int b, int t, long long m, int nbase, uint8_t* st, int lane) {
  const bool f16 = nbase >= op.f16_col0;
#pragma unroll 1
  for (int j = 0; j < 32; ++j) {
    const int n = nbase + j;
    if (n >= op.n_valid) break;
    const float v = stage_f32_ptr(st, lane, j >> 2)[j & 3];
    if (flags & EPI_OUT_NCT) { op.out[((long long)b * op.n_valid + n) * op.T_out + t] = v; continue; }
    if (flags & EPI_OUT_F32) op.out[m * op.out_ld + n] = v;
    if (flags & EPI_OUT_SPLIT) {
      const long long o = m * op.out_split_ld + n;
      if (f16) {
        const __half h = __float2half_rn(v);
        reinterpret_cast<__half*>(op.out_hi)[o] = h;
        reinterpret_cast<__half*>(op.out_lo)[o] = __float2half_rn(v - __half2float(h));
      } else {
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        op.out_hi[o] = h;
        op.out_lo[o] = __float2bfloat16_rn(v - __bfloat162float(h));
      }
    }
  }
}
__device__ __forceinline__ void park_row(uint8_t* st, int lane, const float* val) {
#pragma unroll
  for (int j = 0; j < 8; ++j) *reinterpret_cast<float4*>(stage_f32_ptr(st, lane, j)) = make_float4(val[4 * j], val[4 * j + 1], val[4 * j + 2], val[4 * j + 3]);
}
__device__ __forceinline__ void fetch_row(uint8_t* st, int lane, float* val) {
#pragma unroll
  for (int j = 0; j < 8; ++j) { const float4 v = *reinterpret_cast<const float4*>(stage_f32_ptr(st, lane, j)); val[4 * j] = v.x; val[4 * j + 1] = v.y; val[4 * j + 2] = v.z; val[4 * j + 3] = v.w; }
}

// Store one 32-column chunk of this warp's 32 rows.  val: this thread's row (already zero for rows past T_out).
__device__ __forceinline__ void emit_chunk(const GemmOp& op, const TMap* tmo, uint8_t* st, int lane, bool leader, bool stage_f32, int b, int t,
                                           int t_warp0, long long m, bool mv, int nbase, const float* val, bool with_split = true,
                                           unsigned long long* stamp = nullptr) {
  if (stage_f32) {
#pragma unroll
    for (int j = 0; j < 8; ++j) *reinterpret_cast<float4*>(stage_f32_ptr(st, lane, j)) = make_float4(val[4 * j], val[4 * j + 1], val[4 * j + 2], val[4 * j + 3]);
  }
  const int tma = with_split ? op.tma_out : (op.tma_out & ~2);
  if (tma & 2) {
    const bool f16 = nbase >= op.f16_col0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint4 hi, lo;
      if (f16) split8_f16(val + 8 * j, hi, lo); else split8(val + 8 * j, hi, lo);
      const int off = lane * 64 + ((j ^ ((lane >> 1) & 3)) << 4);
      *reinterpret_cast<uint4*>(st + 4096 + off) = hi;
      *reinterpret_cast<uint4*>(st + 6144 + off) = lo;
    }
  }
  if (stamp) { long long t; asm volatile("mov.u64 %0, %%clock64;" : "=l"(t)); stamp[12] = t; }     // staging written
  if (tma & 3) {
    fence_proxy_async();
    __syncwarp();
    if (stamp) { long long t; asm volatile("mov.u64 %0, %%clock64;" : "=l"(t)); stamp[13] = t; }   // fence + syncwarp done
    // the warp's elected thread (elect.sync once per warp: `leader`) issues the fp32 / hi / lo stores back to back as ONE bulk
    // group; behind lane tests every UTMASTG sat in a serialisation loop (~0.4 us per store)
    if (leader) {
      const uint32_t sa = smem_u32(st);
      if (tma & 1) tma_store_3d(&tmo[0], sa, nbase, t_warp0, b);
      if (tma & 2) { tma_store_3d(&tmo[1], sa + 4096u, nbase, t_warp0, b); tma_store_3d(&tmo[2], sa + 6144u, nbase, t_warp0, b); }
      bulk_commit();
    }
  }
  // whatever does not go through TMA (channel-major output, unaligned leading dimensions)
  const int direct = ((op.flags & EPI_OUT_NCT) ? EPI_OUT_NCT : 0) | (((op.flags & EPI_OUT_F32) && !(op.tma_out & 1)) ? EPI_OUT_F32 : 0) |
                     (((op.flags & EPI_OUT_SPLIT) && with_split && !(op.tma_out & 2)) ? EPI_OUT_SPLIT : 0);
  if (direct) {                                             // (warp-uniform; cold)
    if (!stage_f32) park_row(st, lane, val);
    if (mv) store_cold(op, direct, b, t, m, nbase, st, lane);
  }
}

__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
// panel-mode stamps of the first transform thread of CTA 0: slots 16.. of the 32-slot trace record
#define XTRACE(i) do { if (op_param.trace && blockIdx.x == 0 && tid == 128) op_param.trace[16 + (i)] = gtime(); } while (0)
#define TRACE(i) do { if (op.trace && blockIdx.x == 0 && blockIdx.y == 0) op.trace[i] = gtime(); } while (0)
// epilogue sub-steps of warp 4 / lane 0 of CTA (0,0), SM clock: slots 8..15 of the 16-slot trace record
__device__ __forceinline__ long long gclk() { long long t; asm volatile("mov.u64 %0, %%clock64;" : "=l"(t)); return t; }
#define ETRACE(i) do { if (op.trace && blockIdx.x == 0 && blockIdx.y == 0 && warp == 4 && lane == 0) op.trace[8 + (i)] = gclk(); } while (0)

// only the fields in front of the tensor maps are copied to shared memory (the maps are used by address)
constexpr int kGemmOpHotBytes = (int)offsetof(GemmOp, tmap);
static_assert(kGemmOpHotBytes % 16 == 0 && kGemmOpHotBytes <= 2688 && sizeof(PrepOp) <= 320, "GemmOp's hot part must fit the shared-memory descriptor copy");

// LNF: instantiation for the consumers of a folded LayerNorm (EPI_LNFOLD); the other GEMMs run the LNF = false code, which
// keeps the epilogue free of the extra live values (the epilogue is register-bound).
// XF: instantiation with the panel-mode paths (GroupNorm of the A operand applied in shared memory; BN = 64, one tile per CTA)
// ENC: instantiation for the condition encoders (pre_engine.cu): ReLU and the per-row keep mask in the epilogue (EPI_RELU /
// EPI_ROWMASK); the denoiser's instantiations do not carry that code
// RAG: instantiation for the denoiser's ragged programs (GemmOp::row_len): rows past each utterance's length at this level are
// stored as exact zeros, and in panel mode they read as the conv's zero padding and drop out of the GroupNorm statistics
// VOC: instantiation for the vocoder (vocoder.cu): the erf-GELU epilogue of ConvNeXt's pwconv1 (EPI_GELU)
// and of the content encoder (content.cu), whose row mask (EPI_ROWMASK) stores the rows a zero keep factor marks as exact zeros
template <int BN_, bool LNF, bool XF, bool ENC = false, bool RAG = false, bool VOC = false>
__global__ void __launch_bounds__(kThreads, 1) gemm_tc_kernel(const __grid_constant__ GemmOp op_param) {
  using Cfg = TileCfg<BN_>;
  constexpr int BN = Cfg::BN;
  constexpr int kStageBytes = Cfg::kStageBytes;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;             // SWIZZLE_128B atoms need 1024 B alignment
  uint8_t* smem = smem_raw + (base - raw);
  const uint32_t bar_base = base + Cfg::kOffBar;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (kMaxStages + s); };
  // panel mode: A ring = full_bar / empty_bar (0..2); weight ring of its own
  auto b_full = [&](int s) { return bar_base + 8u * (19 + s); };
  auto b_empty = [&](int s) { return bar_base + 8u * (21 + s); };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // The 1.7 KB operator descriptor lives in the kernel-parameter constant bank, which is cold at every
  // launch: reading its fields one by one costs a chain of constant-cache misses on the critical path
  // (producer start-up, epilogue).  Copy it to shared memory once, with all loads in flight together,
  // before the first __syncthreads (i.e. inside the PDL window); everything below reads the copy.
  // TMA still gets the tensor maps by their parameter-space address.
  {
    const uint4* src = reinterpret_cast<const uint4*>(&op_param);
    uint4* dst = reinterpret_cast<uint4*>(smem + Cfg::kOffDesc);
    for (int i = tid; i < kGemmOpHotBytes / 16; i += kThreads) dst[i] = src[i];
    // GroupNorm parameters of a panel-mode launch (device memory, static): parked behind the operator copy
    if (XF && op_param.xmode && op_param.pre) {
      const uint4* ps = reinterpret_cast<const uint4*>(op_param.pre);
      uint4* pd = reinterpret_cast<uint4*>(smem + Cfg::kOffDesc + 2688);
      for (int i = tid; i < (int)(sizeof(PrepOp) / 16); i += kThreads) pd[i] = __ldg(ps + i);
    }
  }
  const GemmOp& op = *reinterpret_cast<const GemmOp*>(smem + Cfg::kOffDesc);
  const TMap* tmaps = op_param.tmap;
  // One tile per CTA (tile = m_tile * n_tiles + n_tile; launch_bn's grid is the tile count): the epilogue stages its output
  // and parks the accumulator in the stage buffers, which only a CTA without a next tile may do.
  const int tiles_per_batch = (op_param.T_out + BM - 1) / BM;
  const int n_tiles = op_param.N / BN;
  // split-K (panel mode only): the `ks` CTAs of a cluster share one tile; kr = this CTA's share of the channel blocks
  const int ks = (XF && op_param.xmode && op_param.ksplit > 1) ? op_param.ksplit : 1;
  const int kr = (int)blockIdx.x % ks, bid = (int)blockIdx.x / ks;
  const int nst = Cfg::kStagesSingle;
  uint8_t* stage_area = smem;
  float* acc_tile = reinterpret_cast<float*>(smem + (XF ? kXOffAcc : Cfg::kOffAcc));
  const int wg = (warp - 4) >> 2;                           // consumer warpgroup: tile rows [64 wg, 64 wg + 64)
  float acc_d[BN / 2];                                      // this thread's part of the warpgroup's m64 x BN accumulator
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc_d[i] = 0.f;
  // one 16-wide k-step of the 3xBF16 product: A rows [64 wg, 64 wg + 64) at a_hi / a_lo, B rows [0, BN) at b_hi / b_lo
  auto mma3 = [&](uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo) {
    wgmma_bf16<BN>(acc_d, wg_desc(a_hi), wg_desc(b_hi));
    wgmma_bf16<BN>(acc_d, wg_desc(a_lo), wg_desc(b_hi));
    wgmma_bf16<BN>(acc_d, wg_desc(a_hi), wg_desc(b_lo));
  };
  const int nkb = op_param.nkb_total;
  const bool tr0 = blockIdx.x == 0;
  auto xr_ready = [&]() { return bar_base + 8u * 23; };     // split-K: the first CTA's rings are idle, the partner may write
  auto xr_full = [&]() { return bar_base + 8u * 24; };      // split-K: the partner's partial tile has landed (8 warps)
  if (tid == 0 && op_param.trace && tr0) op_param.trace[0] = gtime();
  span_begin(op_param.span);

  if (warp == 1 && lane == 0) {
    for (int s = 0; s < kMaxStages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), kEpiWarps); }
    if (XF) { mbar_init(xr_ready(), 1); mbar_init(xr_full(), kEpiWarps); for (int a = 0; a < kXBStages; ++a) { mbar_init(b_full(a), 1); mbar_init(b_empty(a), kEpiWarps); } }
    mbar_fence_init();
  }
  if (warp == 0 && lane == 0) {
    for (int i = 0; i < 2 * op_param.nsrc; ++i) prefetch_tmap(&tmaps[i]);
    // the store maps too: the first bulk store through a cold descriptor costs a ~0.5 us fetch on the epilogue's critical path
    const TMap* pm = op_param.tmap_out;
    if (op_param.tma_out & 1) prefetch_tmap(&pm[0]);
    if (op_param.tma_out & 2) { prefetch_tmap(&pm[1]); prefetch_tmap(&pm[2]); }
  }
  pdl_trigger();
  __syncthreads();                                          // descriptor copy + armed barriers
  if (tid == 0 && tr0) TRACE(1);
  if constexpr (XF) if (ks > 1) cluster_sync_all();          // split-K: the partner's mbarriers exist before anyone arrives on them remotely

  // ============================================================================================================
  // Panel mode: one tile per CTA (grid == tile count).  warp 0: panels + weight tiles by TMA; warps 4-11: normalise
  // each panel in place, issue the wgmmas over three row-shifted views of the panel per tap, then (below) the ordinary
  // epilogue.
  // ============================================================================================================
  constexpr bool xpanel = XF;                               // the XF instantiation IS the panel mode (launch_gemm_tc): no plain main loop in it
  if constexpr (XF) {
    const int tile = bid, mtile = tile / n_tiles;
    const int xb = mtile / tiles_per_batch, xt0 = (mtile % tiles_per_batch) * BM, xn0 = (tile % n_tiles) * BN;
    int ncblk = 0;
    for (int si = 0; si < op.nxs; ++si) ncblk += op.xs[si].ncb;
    const int p_lo = ncblk * kr / ks, p_hi = ncblk * (kr + 1) / ks;   // this CTA's channel blocks (global panel indices)
    if (warp == 0) {
      if (elect_one()) {
        // weights of the first two channel blocks before the dependency wait, activations after it
        auto issue_w = [&](const XSeg& xs, int cb, int sb) {
          const uint32_t b0 = base + kXOffB + sb * kXBStageBytes;
          mbar_arrive_expect_tx(b_full(sb), (uint32_t)xs.ntap * 2u * Cfg::kBTileBytes);
          for (int j = 0; j < xs.ntap; ++j) {
            const size_t eoff = ((size_t)(xs.kb_tap[j] + cb) * op.N + xn0) * 64;
            bulk_g2s(b0 + j * 2 * Cfg::kBTileBytes, op.w_hi + eoff, Cfg::kBTileBytes, b_full(sb));
            bulk_g2s(b0 + j * 2 * Cfg::kBTileBytes + Cfg::kBTileBytes, op.w_lo + eoff, Cfg::kBTileBytes, b_full(sb));
          }
        };
        { int it = 0, gp = 0;
          for (int si = 0; si < op.nxs && it < kXBStages; ++si)
            for (int cb = 0; cb < op.xs[si].ncb && it < kXBStages; ++cb, ++gp) {
              if (gp < p_lo || gp >= p_hi) continue;
              issue_w(op.xs[si], cb, it); ++it;
            } }
        pdl_wait();
        if (tr0) TRACE(2);
        int it = 0, gp = 0;
        for (int si = 0; si < op.nxs; ++si) {
          const XSeg& xs = op.xs[si];
          for (int cb = 0; cb < xs.ncb; ++cb, ++gp) {
            if (gp < p_lo || gp >= p_hi) continue;
            const int sa = it % kXAStages, sb = it % kXBStages;
            if (it >= kXAStages) mbar_wait(empty_bar(sa), (uint32_t)(((it / kXAStages) & 1) ^ 1));
            const uint32_t a_hi = base + sa * kXAStageBytes;
            const uint32_t rows = xs.ntap == 3 ? (uint32_t)kPanelRows : (uint32_t)BM;
            const int c = xs.c0 + cb * 64, trow = xt0 + (xs.ntap == 3 ? -1 : 0);
            mbar_arrive_expect_tx(full_bar(sa), 2u * rows * 128u);
            tma_load_3d(a_hi, &tmaps[2 * xs.src], c, trow, xb, full_bar(sa));
            tma_load_3d(a_hi + kPanelBytes, &tmaps[2 * xs.src + 1], c, trow, xb, full_bar(sa));
            if (it >= kXBStages) { mbar_wait(b_empty(sb), (uint32_t)(((it / kXBStages) & 1) ^ 1)); issue_w(xs, cb, sb); }
            ++it;
          }
        }
      }
    } else if (warp >= 4) {
      // ---- transform + MMA warps (the epilogue warps; 256 threads) ----
      const int xt = tid - 128;
      float* aff = reinterpret_cast<float*>(smem + kXOffAff);
      const PrepOp& pr = *reinterpret_cast<const PrepOp*>(smem + Cfg::kOffDesc + 2688);
      const bool have_aff = op.pre != nullptr;
      const int C = have_aff ? pr.C1 + pr.C2 : 0;
      auto sync256 = [] { asm volatile("bar.sync 1, 256;" ::: "memory"); };
      float pg[kPrepSlots], pbv[kPrepSlots], fs[kPrepSlots], fbv[kPrepSlots];
      if (have_aff) prep_fetch_norm_weights(pr, C, pg, pbv, xt, 256);
      pdl_wait();
      XTRACE(0);
      if (have_aff) prep_fetch_film(pr, op.pre_film, xb, C, fs, fbv, xt, 256);
      bool aff_done = !have_aff;                              // derived when the first normalised segment comes up: raw (shortcut)
                                                              // panels queued before it are released to the MMA warp at once
      const bool silu = have_aff && pr.mode == PREP_AFFINE_SILU;
      int it = 0, gp = 0;
      for (int si = 0; si < op.nxs; ++si) {
        const XSeg& xs = op.xs[si];
        const int rows = xs.ntap == 3 ? kPanelRows : BM, tfirst = xt0 + (xs.ntap == 3 ? -1 : 0);
        int Tsrc = op.src[xs.src].T;
        if constexpr (RAG) Tsrc = min(Tsrc, ragged_rows(op.row_len, xb, op.len_shift));   // (panel sources sit at the output's level)
        if (xs.xf && !aff_done && gp < p_hi && gp + xs.ncb > p_lo) {   // (only if some of this segment's panels are this CTA's)
          for (int c = C + xt; c < ((C + 63) & ~63); c += 256) { aff[c] = 0.f; aff[kXfMaxC + c] = 0.f; }   // padding channels of the last block
          prep_affine<RAG>(pr, xb, C, kXfMaxC, aff, pg, pbv, fs, fbv, xt, 256, sync256);
          aff_done = true;
          XTRACE(1);
        }
        for (int cb = 0; cb < xs.ncb; ++cb, ++gp) {
          if (gp < p_lo || gp >= p_hi) continue;
          const int sa = it % kXAStages;
          // this thread's 16-byte chunk column q = xt % 8 is the same for every row it touches: its 8 scale / shift values
          // are fetched once per panel, before the panel itself has landed
          const int q = xt & 7;
          float scv[8], shv[8];
          if (xs.xf) {
            const float* sc = aff + xs.aff_c0 + cb * 64 + q * 8;
            const float4 s0 = *reinterpret_cast<const float4*>(sc), s1 = *reinterpret_cast<const float4*>(sc + 4);
            const float4 b0 = *reinterpret_cast<const float4*>(sc + kXfMaxC), b1 = *reinterpret_cast<const float4*>(sc + kXfMaxC + 4);
            scv[0] = s0.x; scv[1] = s0.y; scv[2] = s0.z; scv[3] = s0.w; scv[4] = s1.x; scv[5] = s1.y; scv[6] = s1.z; scv[7] = s1.w;
            shv[0] = b0.x; shv[1] = b0.y; shv[2] = b0.z; shv[3] = b0.w; shv[4] = b1.x; shv[5] = b1.y; shv[6] = b1.z; shv[7] = b1.w;
          }
          mbar_wait(full_bar(sa), (uint32_t)((it / kXAStages) & 1));
          if (it == 0) XTRACE(2);
          if (xs.xf) {
            uint8_t* p_hi = smem + sa * kXAStageBytes;
            uint8_t* p_lo = p_hi + kPanelBytes;
            auto xform = [&](int r, uint4& h4, uint4& l4) {     // one 16-byte chunk (8 channels) of row r, in place (branch-free)
              const int t = tfirst + r;
              const float keep = (t >= 0 && t < Tsrc) ? 1.f : 0.f;   // rows outside the sequence: the conv's zero padding (of the NORMALISED activation)
              const uint32_t hw[4] = {h4.x, h4.y, h4.z, h4.w}, lw[4] = {l4.x, l4.y, l4.z, l4.w};
              float v[8];
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                float x0, x1;
                upk2(fadd2(pk2(__uint_as_float(hw[j] << 16), __uint_as_float(hw[j] & 0xffff0000u)),
                           pk2(__uint_as_float(lw[j] << 16), __uint_as_float(lw[j] & 0xffff0000u))), x0, x1);
                unsigned long long y2 = ffma2(pk2(x0, x1), pk2(scv[2 * j], scv[2 * j + 1]), pk2(shv[2 * j], shv[2 * j + 1]));
                if (silu) y2 = silu2(y2);
                upk2(fmul2(y2, pk2(keep, keep)), v[2 * j], v[2 * j + 1]);
              }
              split8(v, h4, l4);
            };
            // this thread: chunk column q of rows r, r + 32, r + 64, r + 96 (always inside the panel) - four independent
            // chains in flight - and of row r + 128 for the two halo rows of a k=3 panel
            const int rb = xt >> 3;
            uint4 h4[4], l4[4];
            int off[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              const int r = rb + 32 * u;
              off[u] = r * 128 + ((q ^ (r & 7)) << 4);
              h4[u] = *reinterpret_cast<const uint4*>(p_hi + off[u]);
              l4[u] = *reinterpret_cast<const uint4*>(p_lo + off[u]);
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) xform(rb + 32 * u, h4[u], l4[u]);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              *reinterpret_cast<uint4*>(p_hi + off[u]) = h4[u];
              *reinterpret_cast<uint4*>(p_lo + off[u]) = l4[u];
            }
            if (rb + 128 < rows) {
              const int r = rb + 128, o = r * 128 + ((q ^ (r & 7)) << 4);
              uint4 hh = *reinterpret_cast<const uint4*>(p_hi + o), ll = *reinterpret_cast<const uint4*>(p_lo + o);
              xform(r, hh, ll);
              *reinterpret_cast<uint4*>(p_hi + o) = hh; *reinterpret_cast<uint4*>(p_lo + o) = ll;
            }
            fence_proxy_async();
          }
          asm volatile("bar.sync 1, 256;" ::: "memory");      // the whole panel is normalised
          if (it == 0) XTRACE(3);
          const int sb = it % kXBStages;
          mbar_wait(b_full(sb), (uint32_t)((it / kXBStages) & 1));
          const uint32_t a_hi = base + sa * kXAStageBytes + wg * 64 * 128, a_lo = a_hi + kPanelBytes, b0 = base + kXOffB + sb * kXBStageBytes;
          wgmma_fence();
          for (int j = 0; j < xs.ntap; ++j) {              // tap j = panel rows [j, j + 128): start address + 128 B per row
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) {
              const uint32_t bh = b0 + j * 2 * Cfg::kBTileBytes + k * 32;
              mma3(a_hi + j * 128 + k * 32, a_lo + j * 128 + k * 32, bh, bh + Cfg::kBTileBytes);
            }
          }
          wgmma_commit();
          wgmma_wait<1>();                                   // the previous panel's wgmmas have retired: release its buffers
          if (it > 0 && lane == 0) { mbar_arrive(empty_bar((it - 1) % kXAStages)); mbar_arrive(b_empty((it - 1) % kXBStages)); }
          ++it;
        }
      }
      wgmma_wait<0>();
      XTRACE(4);
    }
  }

  // The weights do not depend on the previous kernel: the first tile's first stages are in flight before
  // griddepcontrol.wait; the activations (written by the previous kernel) only after it.
  const int npf = nkb < nst ? nkb : nst;
  if constexpr (!xpanel) if (warp == 0 && elect_one()) {
    const int n0 = (bid % n_tiles) * BN;
    for (int kb = 0; kb < npf; ++kb) {
      const uint32_t b_hi = base + kb * kStageBytes + 2 * kATileBytes;
      mbar_arrive_expect_tx(full_bar(kb), 2u * kATileBytes + 2u * Cfg::kBTileBytes);
      const size_t eoff = ((size_t)kb * op.N + n0) * 64;
      bulk_g2s(b_hi, op.w_hi + eoff, Cfg::kBTileBytes, full_bar(kb));
      bulk_g2s(b_hi + Cfg::kBTileBytes, op.w_lo + eoff, Cfg::kBTileBytes, full_bar(kb));
    }
  }
  __syncwarp();

  if (warp == 0) {
    // ===================== TMA producer =====================
    if constexpr (!xpanel) if (elect_one()) {
      const int npre = npf;
      pdl_wait();
      if (tr0) TRACE(2);
      {
        const int mt = bid / n_tiles, n0 = (bid % n_tiles) * BN;
        const int b = mt / tiles_per_batch, t0 = (mt % tiles_per_batch) * BM;
        int si = 0, kbl = 0;
        for (int kb = 0; kb < nkb; ++kb) {
          const int stage = kb % nst;
          const GSeg& s = op.seg[si];
          const uint32_t a_hi = base + stage * kStageBytes;
          const uint32_t a_lo = a_hi + kATileBytes;
          const uint32_t b_hi = a_lo + kATileBytes;
          if (kb >= npre) {
            if (kb >= nst) mbar_wait(empty_bar(stage), (uint32_t)(((kb / nst) & 1) ^ 1));
            mbar_arrive_expect_tx(full_bar(stage), 2u * kATileBytes + 2u * Cfg::kBTileBytes);
            const size_t eoff = ((size_t)kb * op.N + n0) * 64;
            bulk_g2s(b_hi, op.w_hi + eoff, Cfg::kBTileBytes, full_bar(stage));
            bulk_g2s(b_hi + Cfg::kBTileBytes, op.w_lo + eoff, Cfg::kBTileBytes, full_bar(stage));
          }
          const int c = s.c0 + kbl * 64;
          tma_load_3d(a_hi, &tmaps[2 * s.src], c, t0 + s.tap, b, full_bar(stage));
          tma_load_3d(a_lo, &tmaps[2 * s.src + 1], c, t0 + s.tap, b, full_bar(stage));
          if (++kbl == s.nkb) { kbl = 0; ++si; }
        }
      }
    }
  } else if (warp >= 4) {
    // ===================== main loop + epilogue (warps 4..11) =====================
    pdl_wait();                                             // residual reads / output writes follow the previous kernel
    __syncwarp();
    const bool leader = elect_one();                        // this warp's bulk-store thread (issues, commits and waits for its groups)
    const int q = warp & 3;                                 // row quarter of the tile this warp's epilogue handles
    const int r = q * 32 + lane;
    const int cc0 = (warp - 4) >> 2;
    uint8_t* st = stage_area + kStageOff + (warp - 4) * kStagePerWarp;   // this warp's staging area
    const TMap* tmo = op_param.tmap_out;
    bool staged_once = false;
    {
      constexpr int it = 0;                                 // the CTA's only tile (tile-parity indexing below)
      const int mt = bid / n_tiles, nt = bid % n_tiles, n0 = nt * BN;
      const int b = mt / tiles_per_batch, t0 = (mt % tiles_per_batch) * BM;
      const int t = t0 + r;
      const bool mv = t < op.T_out;
      const long long m = (long long)b * op.T_out + t;
      bool rv = mv;                                         // row inside its utterance (RAG: stored as zeros otherwise)
      if constexpr (RAG) rv = mv && t < ragged_rows(op.row_len, b, op.len_shift);
      if constexpr (VOC) if (op.flags & EPI_ROWMASK) rv = mv && __ldg(op.rowmask + m) != 0.f;   // (content.cu: exact zeros past a row's frames)
      if constexpr (!xpanel) {
        for (int kb = 0; kb < nkb; ++kb) {
          const int stage = kb % nst;
          mbar_wait(full_bar(stage), (uint32_t)((kb / nst) & 1));
          if (kb == 0 && tr0 && warp == 4 && lane == 0) TRACE(3);
          const uint32_t a_hi = base + stage * kStageBytes + wg * 64 * 128;
          const uint32_t a_lo = a_hi + kATileBytes;
          const uint32_t b_hi = base + stage * kStageBytes + 2 * kATileBytes;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / 16; ++k) mma3(a_hi + k * 32, a_lo + k * 32, b_hi + k * 32, b_hi + Cfg::kBTileBytes + k * 32);
          wgmma_commit();
          wgmma_wait<1>();                                   // the previous k-block's wgmmas have retired: release its stage
          if (kb > 0 && lane == 0) mbar_arrive(empty_bar((kb - 1) % nst));
        }
        wgmma_wait<0>();
        if (lane == 0) mbar_arrive(empty_bar((nkb - 1) % nst));
        if (it == 0 && tr0 && warp == 4 && lane == 0) TRACE(4);
      }
      // once every wgmma of BOTH warpgroups has retired the stage buffers are idle: park the accumulator there
      asm volatile("bar.sync 1, 256;" ::: "memory");
      acc_park<BN>(acc_tile, acc_d, wg, tid & 127);
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc_d[i] = 0.f;
      asm volatile("bar.sync 1, 256;" ::: "memory");
      const int t_warp0 = t0 + q * 32;                      // first row of this warp's 32-row slab
      // bias and residual values of this thread's first 32-column chunk
      float pre[32];                                        // bias + residual of chunk cc0 (plain path); GEGLU: value bias
      float preg[32];                                       // GEGLU: gate bias
      bool pre_ok = false;
      // folded LayerNorm: this row's mean / rstd (sums accumulated by the producer's epilogue) and the g vectors of the
      // warp's first chunk (shared by all rows: parked in shared memory, one column per lane)
      float ln_mu = 0.f, ln_rstd = 1.f;
      float* sg = reinterpret_cast<float*>(smem + Cfg::kOffLnG) + (warp - 4) * 128;   // g (value | gate) | folded bias (value | gate)
      if constexpr (LNF) {
        // LNF instantiation: every per-column vector lives in shared memory (no register copies: the epilogue is register-bound)
        if (mv) ln_row_stats(op, m, ln_mu, ln_rstd);
        __syncwarp();
        if constexpr (BN == 128) {                          // (BN = 128 <=> GEGLU: plan_gemm, checked at launch)
          const int nb = nt * 64 + cc0 * 32 + lane;
          const bool ok = nb < op.n_valid;
          sg[lane] = ok ? __ldg(op.ln_g + nb) : 0.f;
          sg[32 + lane] = ok ? __ldg(op.ln_g + op.n_valid + nb) : 0.f;
          sg[64 + lane] = ok ? __ldg(op.bias + nb) : 0.f;
          sg[96 + lane] = ok ? __ldg(op.bias + op.n_valid + nb) : 0.f;
          pre_ok = BN == 128 && nt * 64 + cc0 * 32 + 32 <= op.n_valid;
        } else {
          const int nb = n0 + cc0 * 32 + lane;
          const bool ok = nb < op.n_valid;
          sg[lane] = ok ? __ldg(op.ln_g + nb) : 0.f;
          sg[64 + lane] = (ok && (op.flags & EPI_BIAS)) ? __ldg(op.bias + nb) : 0.f;
          pre_ok = mv && n0 + cc0 * 32 + 32 <= op.n_valid && !(op.flags & (EPI_ROWBIAS | EPI_RESIDUAL));
        }
        __syncwarp();
      }
      if constexpr (!LNF) {
      if constexpr (BN == 128) {
        const int nb = nt * 64 + cc0 * 32;
        if (BN == 128 && nb + 32 <= op.n_valid) {
          pre_ok = true;
          const float4* bv = reinterpret_cast<const float4*>(op.bias + nb);
          const float4* bg = reinterpret_cast<const float4*>(op.bias + op.n_valid + nb);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float4 x = __ldg(bv + j), y = __ldg(bg + j);
            pre[4 * j] = x.x; pre[4 * j + 1] = x.y; pre[4 * j + 2] = x.z; pre[4 * j + 3] = x.w;
            preg[4 * j] = y.x; preg[4 * j + 1] = y.y; preg[4 * j + 2] = y.z; preg[4 * j + 3] = y.w;
          }
        }
      } else {
        const int nb = n0 + cc0 * 32;
        if (mv && nb + 32 <= op.n_valid && !(op.flags & EPI_ROWBIAS) && (!(op.flags & EPI_RESIDUAL) || (op.res_ld & 3) == 0)) {
          pre_ok = true;
#pragma unroll
          for (int j = 0; j < 32; ++j) pre[j] = 0.f;
          if (op.flags & EPI_BIAS) {
            const float4* pb = reinterpret_cast<const float4*>(op.bias + nb);
#pragma unroll
            for (int j = 0; j < 8; ++j) { const float4 v = __ldg(pb + j); pre[4 * j] = v.x; pre[4 * j + 1] = v.y; pre[4 * j + 2] = v.z; pre[4 * j + 3] = v.w; }
          }
          if (op.flags & EPI_RESIDUAL) {
            const float4* pr = reinterpret_cast<const float4*>(op.res + m * op.res_ld + nb);
#pragma unroll
            for (int j = 0; j < 8; ++j) { const float4 v = __ldg(pr + j); pre[4 * j] += v.x; pre[4 * j + 1] += v.y; pre[4 * j + 2] += v.z; pre[4 * j + 3] += v.w; }
          }
        }
      }
      }   // !LNF
      float enc_keep = 1.f;
      if constexpr (ENC) if ((op.flags & EPI_ROWMASK) && mv) enc_keep = __ldg(op.rowmask + m);
      if (it == 0 && tr0 && warp == 4 && lane == 0) TRACE(5);
      if (it == 0 && tr0) ETRACE(0);
      auto wait_staging = [&]() {                           // the TMA unit must have read the previous chunk out of the staging area
        if (staged_once && op.tma_out) {
          if (leader) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
          __syncwarp();
        }
      };
      if constexpr (BN == 128) {
        {
          const int hh = cc0;                               // the two warps of a lane quarter take one half each
          float val[32], gate[32];
          acc_row32<BN>(acc_tile, r, hh * 32, val);
          acc_row32<BN>(acc_tile, r, 64 + hh * 32, gate);
          const int nbase = nt * 64 + hh * 32;              // logical output column
          if (nbase < op.n_valid) {                         // (uniform across the warp)
            if (!rv) {
#pragma unroll
              for (int j = 0; j < 32; ++j) val[j] = 0.f;
            } else if (pre_ok) {                            // biases were fetched before the accumulator wait
              if constexpr (LNF) {
#pragma unroll
                for (int j = 0; j < 32; j += 2) {
                  const float v0 = fmaf(ln_rstd, val[j] - ln_mu * sg[j], sg[64 + j]), v1 = fmaf(ln_rstd, val[j + 1] - ln_mu * sg[j + 1], sg[65 + j]);
                  const float g0 = fmaf(ln_rstd, gate[j] - ln_mu * sg[32 + j], sg[96 + j]), g1 = fmaf(ln_rstd, gate[j + 1] - ln_mu * sg[33 + j], sg[97 + j]);
                  upk2(fmul2(pk2(v0, v1), gelu_erf2(pk2(g0, g1))), val[j], val[j + 1]);
                }
              } else {
#pragma unroll
                for (int j = 0; j < 32; j += 2)
                  upk2(fmul2(fadd2(pk2(val[j], val[j + 1]), pk2(pre[j], pre[j + 1])), gelu_erf2(fadd2(pk2(gate[j], gate[j + 1]), pk2(preg[j], preg[j + 1])))),
                       val[j], val[j + 1]);
              }
            } else {                                        // cold: partial chunk - out of line, through the staging row
              wait_staging();
              park_row(st, lane, val);
#pragma unroll
              for (int j = 0; j < 8; ++j) reinterpret_cast<float4*>(st + 4096)[lane * 8 + j] = make_float4(gate[4 * j], gate[4 * j + 1], gate[4 * j + 2], gate[4 * j + 3]);
              epi_cold<LNF>(op, b, m, nbase, st, lane, true);
              fetch_row(st, lane, val);
            }
            wait_staging();
            emit_chunk(op, tmo, st, lane, leader, false, b, t, t_warp0, m, mv, nbase, val);
            staged_once = true;
          }
        }
      } else {
        float* sm_part = reinterpret_cast<float*>(stage_area) + (it & 1) * (4 * BN * 2);   // [4 quarters][BN][2] GroupNorm partial sums (per tile parity)
        const bool stage_f32 = (op.tma_out & 1) || (op.flags & EPI_STATS);
#pragma unroll 1
        for (int cc = cc0; cc < BN / 32; cc += 2) {         // the two warps of a lane quarter alternate chunks
          float acc[32];
          acc_row32<BN>(acc_tile, r, cc * 32, acc);
          if (it == 0 && tr0) ETRACE(1);
          if constexpr (XF) if (ks > 1) {
            // split-K: the partner CTA's fp32 partial of this thread's 32 values travels through THIS tile owner's shared
            // memory (its weight ring is idle once its own accumulator is complete): [8 x float4][256 threads]
            const int te = tid - 128;
            if (kr != 0) {
              mbar_wait_cluster(xr_ready(), 0);              // the owner has finished its main loop
              const uint32_t rbase = mapa_u32(base + kXOffB, 0);
#pragma unroll
              for (int j = 0; j < 8; ++j) st_remote_f32x4(rbase + (uint32_t)((j * 256 + te) * 16), acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]);
              asm volatile("fence.acq_rel.cluster;" ::: "memory");
              __syncwarp();
              if (lane == 0) mbar_arrive_remote(mapa_u32(xr_full(), 0));
              continue;                                      // no epilogue of its own: the owner stores the tile
            }
            if (warp == 4 && lane == 0) mbar_arrive_remote(mapa_u32(xr_ready(), 1));   // (our wgmmas have retired: the rings are idle)
            mbar_wait_cluster(xr_full(), 0);
            const float4* xr = reinterpret_cast<const float4*>(smem + kXOffB);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float4 v = xr[j * 256 + te];
              acc[4 * j] += v.x; acc[4 * j + 1] += v.y; acc[4 * j + 2] += v.z; acc[4 * j + 3] += v.w;
            }
          }
          const int nbase = n0 + cc * 32;
          const bool cvalid = nbase < op.n_valid;           // (uniform across the warp)
          if (cvalid) {
            const bool fullc = nbase + 32 <= op.n_valid;
            bool enc_hot = ENC && mv;                       // (the out-of-line path applies ReLU / mask itself: epi_value)
            bool voc_hot = VOC;                             // (likewise the GELU)
            if (!rv) {
#pragma unroll
              for (int j = 0; j < 32; ++j) acc[j] = 0.f;
            } else if (cc == cc0 && pre_ok) {
              if constexpr (LNF) {
#pragma unroll
                for (int j = 0; j < 32; ++j) acc[j] = fmaf(ln_rstd, acc[j] - ln_mu * sg[j], sg[64 + j]);
              } else {
#pragma unroll
                for (int j = 0; j < 32; ++j) acc[j] += pre[j];
              }
            } else if (!LNF && fullc && !(op.flags & EPI_ROWBIAS) && (!(op.flags & EPI_RESIDUAL) || (op.res_ld & 3) == 0)) {
              if (op.flags & EPI_BIAS) {
                const float4* pb = reinterpret_cast<const float4*>(op.bias + nbase);
#pragma unroll
                for (int j = 0; j < 8; ++j) { const float4 v = __ldg(pb + j); acc[4 * j] += v.x; acc[4 * j + 1] += v.y; acc[4 * j + 2] += v.z; acc[4 * j + 3] += v.w; }
              }
              if (op.flags & EPI_RESIDUAL) {
                const float4* pr = reinterpret_cast<const float4*>(op.res + m * op.res_ld + nbase);
#pragma unroll
                for (int j = 0; j < 8; ++j) { const float4 v = __ldg(pr + j); acc[4 * j] += v.x; acc[4 * j + 1] += v.y; acc[4 * j + 2] += v.z; acc[4 * j + 3] += v.w; }
              }
            } else {                                        // cold: partial chunk / row bias / unaligned residual - out of line
              wait_staging();
              park_row(st, lane, acc);
              epi_cold<LNF, VOC>(op, b, m, nbase, st, lane, false);
              fetch_row(st, lane, acc);
              enc_hot = false;
              voc_hot = false;
            }
            if constexpr (VOC) if (voc_hot && (op.flags & EPI_GELU)) {
#pragma unroll
              for (int j = 0; j < 32; j += 2) upk2(gelu_erf2(pk2(acc[j], acc[j + 1])), acc[j], acc[j + 1]);
            }
            if constexpr (ENC) if (enc_hot) {
              if (op.flags & EPI_RELU) {
#pragma unroll
                for (int j = 0; j < 32; ++j) acc[j] = fmaxf(acc[j], 0.f);
              }
              if (op.flags & EPI_ROWMASK) {
#pragma unroll
                for (int j = 0; j < 32; ++j) acc[j] *= enc_keep;
              }
            }
            if (it == 0 && tr0) ETRACE(2);
            if ((op.flags & EPI_ROWSTATS) && mv) {          // LayerNorm statistics of this row for the consumer GEMM
              float rs = 0.f, rq = 0.f;
#pragma unroll
              for (int j = 0; j < 32; ++j) { rs += acc[j]; rq = fmaf(acc[j], acc[j], rq); }   // columns >= n_valid are zero
              atomicAdd(op.row_stats + m * 2, (double)rs);
              atomicAdd(op.row_stats + m * 2 + 1, (double)rq);
            }
            wait_staging();
            emit_chunk(op, tmo, st, lane, leader, stage_f32, b, t, t_warp0, m, mv, nbase, acc, true,
                       (it == 0 && tr0 && warp == 4 && lane == 0) ? op.trace : nullptr);
            staged_once = true;
            if (it == 0 && tr0) ETRACE(3);
            if (op.flags & EPI_STATS) {
              // per-(b, column) sum / sum-of-squares over this tile's rows for the consumer's GroupNorm: read the staged
              // chunk column-wise (one column per lane; a row's 32 columns are one permuted 128-byte line: conflict-free);
              // the four lane quarters' partials are combined below so each column costs one atomic per CTA.
              __syncwarp();
              float cs = 0.f, cq = 0.f;
#pragma unroll
              for (int rr = 0; rr < 32; ++rr) { const float v = stage_f32_ptr(st, rr, lane >> 2)[lane & 3]; cs += v; cq += v * v; }
              sm_part[(q * BN + cc * 32 + lane) * 2] = cs;
              sm_part[(q * BN + cc * 32 + lane) * 2 + 1] = cq;
              if (it == 0 && tr0) ETRACE(4);
            }
          } else if (op.flags & EPI_STATS) {
            sm_part[(q * BN + cc * 32 + lane) * 2] = 0.f;
            sm_part[(q * BN + cc * 32 + lane) * 2 + 1] = 0.f;
          }
        }
        if ((op.flags & EPI_STATS) && kr == 0) {            // (a split-K partner has no output of its own)
          asm volatile("bar.sync 1, 256;" ::: "memory");    // the 8 epilogue warps
          if (it == 0 && tr0) ETRACE(5);
          const int col = tid - 128;                        // 0..127
          if (col < BN && n0 + col < op.n_valid) {
            double cs = 0, cq = 0;
#pragma unroll
            for (int w = 0; w < 4; ++w) { cs += (double)sm_part[(w * BN + col) * 2]; cq += (double)sm_part[(w * BN + col) * 2 + 1]; }
            atomicAdd(op.stat_sum + (long long)b * op.n_valid + n0 + col, cs);
            atomicAdd(op.stat_sq + (long long)b * op.n_valid + n0 + col, cq);
          }
        }
      }
    }
    // Shared memory must outlive the TMA unit's reads of the staged chunks; the writes themselves are made visible to the
    // dependent grid by grid completion (griddepcontrol.wait on the other side), as in CUTLASS' tma_store_wait.
    if (op.tma_out && leader) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
  }

  if (warp == 4 && lane == 0 && tr0) TRACE(6);
  if (tr0) ETRACE(6);
  __syncthreads();
  if (tr0) ETRACE(7);
  if (tid == 0 && tr0) TRACE(7);
  span_end(op.span);
}

// ---------------------------------------------------------------------------------------------
// Host: TMA descriptor encoding (driver entry point fetched through the runtime; no -lcuda)
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int encode_tmap_any(TMap* out, const void* base, int elem_bytes, int C, int T, int B, int ld, int box_c, int box_rows, int swizzle_bytes,
                    long long bpitch) {
  static_assert(sizeof(CUtensorMap) == sizeof(TMap), "CUtensorMap size");
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point not available"); return -2; }
  if (((long long)ld * elem_bytes) % 16 || (reinterpret_cast<uintptr_t>(base) & 15)) { set_error("buffer not TMA-aligned (ld=%d)", ld); return -1; }
  const CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                               : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE;
  const cuuint64_t gdim[3] = {(cuuint64_t)C, (cuuint64_t)T, (cuuint64_t)B};
  const cuuint64_t gstr[2] = {(cuuint64_t)ld * elem_bytes, (cuuint64_t)(bpitch ? bpitch : (long long)T * ld) * elem_bytes};
  const cuuint32_t box[3] = {(cuuint32_t)box_c, (cuuint32_t)box_rows, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(reinterpret_cast<CUtensorMap*>(out), elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3,
                  const_cast<void*>(base), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d) C=%d T=%d B=%d ld=%d box=%dx%d sw=%d", (int)r, C, T, B, ld, box_c, box_rows, swizzle_bytes); return -2; }
  return 0;
}
int encode_tmap_rows(TMap* out, const __nv_bfloat16* base, int C, int T, int B, int ld, int box_c, int box_rows, int swizzle_bytes) {
  return encode_tmap_any(out, base, 2, C, T, B, ld, box_c, box_rows, swizzle_bytes);
}

static int encode_one(TMap* out, const __nv_bfloat16* base, const SplitBuf& s, int B, int box_rows) {
  return encode_tmap_any(out, base, 2, s.C, s.T, B, s.ld, 64, box_rows, 128, s.bpitch);
}

int encode_tmaps(GemmOp& op) {
  // Outputs: the epilogue stages each warp's 32 x 32 chunk in shared memory and hands it to the TMA unit
  // (one thread per row storing straight to global memory would cost 32 LSU wavefronts per 128-bit store instruction).
  op.tma_out = 0;
  if (!(op.flags & EPI_OUT_NCT)) {
    // (the GEGLU epilogue does not stage its fp32 chunk for a bulk store: its fp32 output takes the element-wise path)
    if ((op.flags & EPI_OUT_F32) && !(op.flags & EPI_GEGLU) && op.out && (op.out_ld & 3) == 0 && (reinterpret_cast<uintptr_t>(op.out) & 15) == 0) {
      int rc = encode_tmap_any(&op.tmap_out[0], op.out, 4, op.n_valid, op.T_out, op.B, op.out_ld, 32, 32, 128);
      if (rc) return rc;
      op.tma_out |= 1;
    }
    // (per-thread 16-byte stores of the split instead of two TMA stores were measured in r02: 3.46 vs 3.16 ms per forward)
    if ((op.flags & EPI_OUT_SPLIT) && (op.out_split_ld & 7) == 0 && (reinterpret_cast<uintptr_t>(op.out_hi) & 15) == 0 &&
        (reinterpret_cast<uintptr_t>(op.out_lo) & 15) == 0) {
      int rc = encode_tmap_any(&op.tmap_out[1], op.out_hi, 2, op.n_valid, op.T_out, op.B, op.out_split_ld, 32, 32, 64);
      if (rc) return rc;
      rc = encode_tmap_any(&op.tmap_out[2], op.out_lo, 2, op.n_valid, op.T_out, op.B, op.out_split_ld, 32, 32, 64);
      if (rc) return rc;
      op.tma_out |= 2;
    }
  }
  for (int i = 0; i < op.nsrc; ++i) {
    int box_rows = BM;
    if (op.xmode)                                           // panel mode: a k=3 source is fetched as one 130-row panel per channel block
      for (int k = 0; k < op.nxs; ++k) if (op.xs[k].src == i && op.xs[k].ntap == 3) box_rows = kPanelRows;
    int rc = encode_one(&op.tmap[2 * i], op.src[i].hi, op.src[i], op.B, box_rows);
    if (rc) return rc;
    rc = encode_one(&op.tmap[2 * i + 1], op.src[i].lo, op.src[i], op.B, box_rows);
    if (rc) return rc;
  }
  return 0;
}

static int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

template <int BN_, bool LNF, bool XF, bool ENC = false, bool RAG = false, bool VOC = false>
static int launch_bn(const GemmOp& op, cudaStream_t st) {
  using Cfg = TileCfg<BN_>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_tc_kernel<BN_, LNF, XF, ENC, RAG, VOC>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) { set_error("gemm_tc: cannot set %d B dynamic smem: %s", Cfg::kSmemBytes, cudaGetErrorString(e)); return -2; }
    attr_set = true;
  }
  const int tiles = op.B * ceil_div(op.T_out, BM) * (op.N / BN_);
  int grid = tiles;                                         // one tile per CTA (the epilogue reuses the stage buffers)
  dim3 cluster(1, 1, 1);
  if (XF && op.xmode && op.ksplit > 1) { grid = tiles * op.ksplit; cluster.x = (unsigned)op.ksplit; }   // split-K: the CTAs of a cluster share a tile
  cudaError_t e = launch_kc(gemm_tc_kernel<BN_, LNF, XF, ENC, RAG, VOC>, dim3(grid), dim3(kThreads), (size_t)Cfg::kSmemBytes, st, cluster, op);
  if (e != cudaSuccess) { set_error("gemm_tc launch failed: %s", cudaGetErrorString(e)); return -2; }
  return 0;
}

int gemm_sm_count() { return sm_count(); }

void plan_gemm(GemmOp& op) {
  // N tile: 64 wide (more, smaller tiles balance better over the SMs); the GEGLU epilogue pairs
  // value|gate inside a 128-column block and needs BN = 128.
  op.bn = (op.flags & EPI_GEGLU) ? 128 : 64;
}

int launch_gemm_tc(const GemmOp& op, cudaStream_t st) {
  if (op.N % 128) { set_error("gemm_tc: packed N=%d is not a multiple of 128", op.N); return -1; }
  const bool lnf = (op.flags & EPI_LNFOLD) != 0;
  const bool rag = op.row_len != nullptr;
  if (rag && (lnf || op.bn != 64 || (op.flags & (EPI_GEGLU | EPI_RELU | EPI_ROWMASK)))) {
    set_error("gemm_tc: ragged row masks need a plain 64-wide tile without a folded LayerNorm");
    return -1;
  }
  if (op.flags & EPI_GELU) {
    if (lnf || rag || op.xmode || op.bn != 64 || (op.flags & (EPI_GEGLU | EPI_RELU))) {
      set_error("gemm_tc: the GELU epilogue needs a plain 64-wide tile without a folded LayerNorm or ReLU");
      return -1;
    }
    if ((op.flags & EPI_ROWMASK) && !op.rowmask) { set_error("gemm_tc: EPI_ROWMASK without a mask"); return -1; }
    if (op.nkb_total <= 0) { set_error("gemm_tc: empty K"); return -1; }
    return launch_bn<64, false, false, false, false, true>(op, st);
  }
  if (op.flags & (EPI_RELU | EPI_ROWMASK)) {
    if (lnf || op.xmode || op.bn != 64 || (op.flags & EPI_GEGLU)) { set_error("gemm_tc: ReLU / row-mask epilogues need a plain 64-wide tile"); return -1; }
    if ((op.flags & EPI_ROWMASK) && !op.rowmask) { set_error("gemm_tc: EPI_ROWMASK without a mask"); return -1; }
    if (op.nkb_total <= 0) { set_error("gemm_tc: empty K"); return -1; }
    return launch_bn<64, false, false, true>(op, st);
  }
  if (op.xmode) {
    if (lnf || op.bn != 64 || op.nxs < 1 || op.nxs > kMaxXSeg) { set_error("gemm_tc: panel mode needs a plain 64-wide tile and 1..%d segments", kMaxXSeg); return -1; }
    if (op.pre == nullptr) { set_error("gemm_tc: panel mode without GroupNorm parameters"); return -1; }
    if (op.ksplit != 1 && op.ksplit != 2) { set_error("gemm_tc: ksplit must be 1 or 2"); return -1; }
    return rag ? launch_bn<64, false, true, false, true>(op, st) : launch_bn<64, false, true>(op, st);
  }
  if (op.nkb_total <= 0) { set_error("gemm_tc: empty K"); return -1; }
  if ((op.bn == 128) != ((op.flags & EPI_GEGLU) != 0)) { set_error("gemm_tc: the 128-wide tile is the GEGLU instantiation (plan_gemm)"); return -1; }
  if (op.bn == 128) return lnf ? launch_bn<128, true, false>(op, st) : launch_bn<128, false, false>(op, st);
  if (op.bn != 64) { set_error("gemm_tc: plan_gemm() was not called"); return -1; }
  if (rag) return launch_bn<64, false, false, false, true>(op, st);
  return lnf ? launch_bn<64, true, false>(op, st) : launch_bn<64, false, false>(op, st);
}

}  // namespace ns2vc
