// Thin inline-PTX wrappers for the sm_90a primitives used by the tensor-core kernels:
// mbarrier, TMA (bulk + tensor), clusters, wgmma and its shared-memory descriptors.
#pragma once
#include "common.cuh"
#include <cstdio>

namespace ns2vc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug becomes a trap (CUDA error) instead of a hung GPU.  The message (a printf call site per wait:
// code size and registers in every role loop) is compiled in with -DNS2VC_WAIT_MESSAGES only.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 24)) {
#ifdef NS2VC_WAIT_MESSAGES
      printf("ns2vc: mbarrier timeout (block %d,%d,%d thread %d bar %u parity %u)\n", blockIdx.x, blockIdx.y, blockIdx.z,
             threadIdx.x, bar, parity);
#endif
      __trap();
    }
  }
}
// Same bound, no message: no printf call (and its register / stack cost) inside register-starved loops.
__device__ __forceinline__ void mbar_wait_quiet(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) { if (++spins > (1u << 24)) __trap(); }
}
// One lane of a CONVERGED warp: ptxas knows that the region guarded by elect.sync runs on a single thread and issues the
// uniform-datapath instructions (UTMALDG, UBLKCP...) directly; behind a `lane == 0` test it wraps every one of them
// in an ELECT / BRA.U.ANY serialisation loop.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// 3-D tiled TMA load at (c, t, b); out-of-range coordinates are zero-filled
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const TMap* tmap, int c, int t, int b, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c), "r"(t), "r"(b)
      : "memory");
}

// 3-D tiled TMA store of a shared-memory box to (c, t, b); parts of the box outside the tensor are not written
__device__ __forceinline__ void tma_store_3d(const TMap* tmap, uint32_t src, int c, int t, int b) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(src), "r"(c), "r"(t), "r"(b)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ---- distributed shared memory (thread-block cluster): remote address, remote arrive, remote store, cluster-scope wait
__device__ __forceinline__ uint32_t mapa_u32(uint32_t local_saddr, uint32_t cta_rank) {
  uint32_t r; asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_saddr), "r"(cta_rank)); return r;
}
__device__ __forceinline__ void mbar_arrive_remote(uint32_t remote_bar) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote_bar) : "memory");
}
__device__ __forceinline__ void st_remote_f32x4(uint32_t raddr, float a, float b, float c, float d) {
  asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(raddr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ void mbar_wait_cluster(uint32_t bar, uint32_t parity) {   // acquire at cluster scope: a peer CTA's writes / arrive
  uint32_t spins = 0, ok = 0;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    if (!ok && ++spins > (1u << 24)) {
#ifdef NS2VC_WAIT_MESSAGES
      printf("ns2vc: cluster mbarrier timeout (block %d thread %d)\n", blockIdx.x, threadIdx.x);
#endif
      __trap();
    }
  } while (!ok);
}
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }

__device__ __forceinline__ void prefetch_tmap(const TMap* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}

// K-major SWIZZLE_128B wgmma descriptor: [0,14) start>>4 | [16,30) LBO>>4 = 1 (unused) | [32,46) SBO>>4 = 1024>>4 | [62,64) 1 =
// SWIZZLE_128B.  The swizzle follows the address bits: a start advanced by 32 B (k-step) or by 128-byte rows stays consistent.
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// d[64 x N] (fp32, registers of the warpgroup) += A[64 x 16] * B[N x 16]^T, both bf16 K-major in shared memory.
// Thread t of the warpgroup holds d[i] = D[16 (t/32) + (t%32)/4 + 8 ((i/2)%2)][8 (i/4) + 2 (t%4) + i%2].
template <int N>
__device__ __forceinline__ void wgmma_bf16(float* d, uint64_t adesc, uint64_t bdesc);
#define NS2VC_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define NS2VC_D32(i) NS2VC_D8(i), NS2VC_D8(i + 8), NS2VC_D8(i + 16), NS2VC_D8(i + 24)
template <>
__device__ __forceinline__ void wgmma_bf16<64>(float* d, uint64_t adesc, uint64_t bdesc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
               "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
               "%32, %33, p, 1, 1, 0, 0;\n\t}" : NS2VC_D32(0) : "l"(adesc), "l"(bdesc), "r"(1));
}
template <>
__device__ __forceinline__ void wgmma_bf16<128>(float* d, uint64_t adesc, uint64_t bdesc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
               "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
               "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
               "%64, %65, p, 1, 1, 0, 0;\n\t}" : NS2VC_D32(0), NS2VC_D32(32) : "l"(adesc), "l"(bdesc), "r"(1));
}
#undef NS2VC_D32
#undef NS2VC_D8

// Park a warpgroup's m64 x N accumulator in a [128][N] fp32 shared-memory tile (rows 64 g .. 64 g + 63), 16-byte chunk c of
// row r stored at chunk c ^ (r & 7): the epilogue then reads one row per thread, 32 consecutive columns, conflict-free.
template <int N>
__device__ __forceinline__ void acc_park(float* tile, const float* d, int g, int t) {
  const int w = t >> 5, l = t & 31;
#pragma unroll
  for (int i = 0; i < N / 2; i += 2) {
    const int r = 64 * g + 16 * w + (l >> 2) + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + 2 * (l & 3);
    *reinterpret_cast<float2*>(tile + r * N + ((((c >> 2) ^ (r & 7))) << 2) + (c & 3)) = make_float2(d[i], d[i + 1]);
  }
}
// v[i] = row r, column c0 + i of the parked tile, i < 32 (c0 a multiple of 32)
template <int N>
__device__ __forceinline__ void acc_row32(const float* tile, int r, int c0, float* v) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 x = *reinterpret_cast<const float4*>(tile + r * N + ((((c0 >> 2) + j) ^ (r & 7)) << 2));
    v[4 * j] = x.x; v[4 * j + 1] = x.y; v[4 * j + 2] = x.z; v[4 * j + 3] = x.w;
  }
}
}  // namespace ns2vc
