// The sampler steps: one element-wise kernel per step of DPM-Solver++(2M), UniPC-bh2, DDPM and DDIM after the denoiser returned
// x0, their launches and their C entry points.  Every arithmetic op uses the round-to-nearest intrinsics so that the compiler
// cannot contract a*b+c into an FMA: the reference evaluates each product and sum as a separate fp32 tensor op
// (dpm_solver.py:291-292, 437-439, 569-576, 813-831; uni_pc.py:533-536, 561-567; model.py:535-542, 586-601), and the result
// here is bit-identical to that sequence.  Each method's element update is written once: the batch kernels run it over n
// elements with one coefficient struct, the row kernels over the rows of a batch that are at different steps.
#include "common.cuh"
#include "launch.cuh"
#include "philox.cuh"
#include "../../include/ns2vc_b200.h"

#include <cooperative_groups.h>

namespace ns2vc {

__device__ __forceinline__ float x0_round_trip(float x, float o, float alpha, float sigma) {
  // noise = (x - alpha*out)/sigma  (model_wrapper, x_start)  ;  x0 = (x - sigma*noise)/alpha
  float noise = __fdiv_rn(__fsub_rn(x, __fmul_rn(alpha, o)), sigma);
  return __fdiv_rn(__fsub_rn(x, __fmul_rn(sigma, noise)), alpha);
}

// Each update does element i and ORs into `bad` whether its input x is NaN: the reference asserts on that before every denoiser
// call (model.py:404), the kernels raise a flag instead.  (The test is accumulated here, next to the load, rather than returned:
// a returned bool compiles to a byte-wide accumulator and different SASS.)
__device__ __forceinline__ void dpm_update(bool& bad, const float* x, const float* o, const float* mp, const ns2vc_dpm_coef& c,
                                           float* mc, float* xn, size_t i) {
  const float xv = x[i];
  bad |= (xv != xv);
  const float m0 = x0_round_trip(xv, o[i], c.alpha_s, c.sigma_s);
  mc[i] = m0;
  if (c.order != 0) {                                      // order 0 writes no x_next
    float r = __fsub_rn(__fmul_rn(c.c_x, xv), __fmul_rn(c.c_m, m0));
    if (c.order == 2) {
      float d1 = __fmul_rn(c.inv_r0, __fsub_rn(m0, mp[i]));
      r = __fsub_rn(r, __fmul_rn(c.c_d, d1));
    }
    xn[i] = r;
  }
}

// kAlwaysXt: x_t is written at corr_order 0 too (x_t = x_eval), as the row kernel needs; the batch kernel leaves it alone there
// (x_t may then be NULL).
template <bool kAlwaysXt>
__device__ __forceinline__ void unipc_update(bool& bad, const float* xp, const float* xe, const float* o, const float* m0p,
                                             const float* m1p, const ns2vc_unipc_coef& c, float* mt_out, float* xt_out,
                                             float* xpred_out, size_t i) {
  const float xev = xe[i];
  bad |= (xev != xev);
  const float mt = x0_round_trip(xev, o[i], c.alpha_t, c.sigma_t);
  mt_out[i] = mt;
  float xt = xev;
  float m0 = 0.f;
  if (c.corr_order > 0) {
    m0 = m0p[i];
    const float xbar = __fsub_rn(__fmul_rn(c.c_x, xp[i]), __fmul_rn(c.c_m, m0));
    const float d1t = __fsub_rn(mt, m0);
    float inner;
    if (c.corr_order == 2) {
      const float d1 = __fdiv_rn(__fsub_rn(m1p[i], m0), c.rk);
      inner = __fadd_rn(__fmul_rn(c.rho0, d1), __fmul_rn(c.rho1, d1t));
    } else {
      inner = __fmul_rn(c.rho1, d1t);     // 0 + 0.5*D1_t
    }
    xt = __fsub_rn(xbar, __fmul_rn(c.ab, inner));
  }
  if (kAlwaysXt || c.corr_order > 0) xt_out[i] = xt;
  if (c.pred_order > 0) {
    const float nbar = __fsub_rn(__fmul_rn(c.n_c_x, xt), __fmul_rn(c.n_c_m, mt));
    float xpred = nbar;
    if (c.pred_order == 2) {
      const float d1n = __fdiv_rn(__fsub_rn(m0, mt), c.nrk);
      xpred = __fsub_rn(nbar, __fmul_rn(c.nab, __fmul_rn(0.5f, d1n)));
    }
    xpred_out[i] = xpred;
  }
}

// x_next may be x itself: each element is read before it is written.  `noise` is element i's noise value, a load or an
// in-register draw; it is produced (and used) only where the step adds noise (add_noise / !last), which the caller tests.
__device__ __forceinline__ void ddpm_update(bool& bad, const float* x, const float* x0, float noise, const ns2vc_ddpm_coef& c,
                                            float* x_next, size_t i) {
  const float xv = x[i];
  bad |= (xv != xv);
  // q_posterior mean (:509-512), then mean + exp(0.5 * logvar) * noise; at t == 0 the reference adds exp(.) * 0. (:540-541)
  const float mean = __fadd_rn(__fmul_rn(c.c_x0, x0[i]), __fmul_rn(c.c_x, xv));
  x_next[i] = __fadd_rn(mean, c.add_noise ? __fmul_rn(c.c_noise, noise) : 0.0f);
}

__device__ __forceinline__ void ddim_update(bool& bad, const float* x, const float* x0, float noise, const ns2vc_ddim_coef& c,
                                            float* x_next, size_t i) {
  const float xv = x[i];
  bad |= (xv != xv);
  const float x0v = x0[i];
  if (c.last) {                                            // the pair (t, -1): img = x_start (:589-592)
    x_next[i] = x0v;
  } else {
    // predict_noise_from_start (:498-503), then x0 * sqrt(a_next) + c * pred_noise + sigma * noise (:599-601); the sigma term is
    // kept at eta = 0: it decides the sign of zero results
    const float pn = __fdiv_rn(__fsub_rn(__fmul_rn(c.sqrt_recip, xv), x0v), c.sqrt_recipm1);
    const float r = __fadd_rn(__fmul_rn(x0v, c.sqrt_alpha_next), __fmul_rn(c.c, pn));
    x_next[i] = __fadd_rn(r, __fmul_rn(c.sigma, noise));
  }
}

// The batch kernels: update(bad, i) over a grid-stride loop of n elements, one flag for a NaN anywhere.
template <class Update>
__device__ __forceinline__ void batch_step(size_t n, int* nan_flag, const Update& update) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  bool bad = false;
  for (; i < n; i += stride) update(bad, i);
  if (bad && nan_flag) atomicOr(nan_flag, 1);
}

// Every kernel waits for its predecessor (programmatic dependent launch) before it reads global memory.
__global__ void __launch_bounds__(256) dpm_step_kernel(const float* __restrict__ x, const float* __restrict__ o,
                                                       const float* __restrict__ mp, ns2vc_dpm_coef c, float* __restrict__ mc,
                                                       float* __restrict__ xn, size_t n, int* nan_flag) {
  pdl_trigger();
  pdl_wait();
  batch_step(n, nan_flag, [&](bool& bad, size_t i) { dpm_update(bad, x, o, mp, c, mc, xn, i); });
}

__global__ void __launch_bounds__(256) unipc_step_kernel(const float* __restrict__ xp, const float* __restrict__ xe,
                                                         const float* __restrict__ o, const float* __restrict__ m0p,
                                                         const float* __restrict__ m1p, ns2vc_unipc_coef c,
                                                         float* __restrict__ mt_out, float* __restrict__ xt_out,
                                                         float* __restrict__ xpred_out, size_t n, int* nan_flag) {
  pdl_trigger();
  pdl_wait();
  batch_step(n, nan_flag,
             [&](bool& bad, size_t i) { unipc_update<false>(bad, xp, xe, o, m0p, m1p, c, mt_out, xt_out, xpred_out, i); });
}

// The row kernel: row b of a [B, row_n] batch takes step k[b] of its own run, so the rows of one batch can be at different steps
// (requests that joined at different ticks) and of different methods.  Row b's method is method[b] (uniform_method for every row
// when method is NULL) and its struct is dpm, unipc, ddpm or ddim[base[b] + k[b]] (base NULL: 0), so one device table per
// struct type holds every schedule in use.  Both methods share one buffer layout (see ns2vc_sampler_step_rows in the header);
// a DPM row never reads m1 or x_prev and never writes x_t.  A DDPM or DDIM row reads x_in and o (its x0) only, writes x_new only
// (which may be x_in itself: each element is read before it is written) and draws its noise in-register at (seeds[b], k[b], c,
// t) with row element i = c * T + t.  Each row is one cluster of kRowCtas CTAs (grid kRowCtas x B); an
// empty row (k[b] < 0) zeroes m_new and x_t (when given) and x_new and raises nothing.  Every CTA reads k[b] before the cluster
// barrier and CTA 0 advances it after, so a captured tick replays with no host write in between.  The NaN flag is per row.
constexpr int kRowCtas = 8;

__global__ void __launch_bounds__(256) sampler_step_rows_kernel(const float* x_in, const float* __restrict__ o,
                                                                const float* __restrict__ m0, const float* __restrict__ m1,
                                                                const float* __restrict__ x_prev,
                                                                const ns2vc_dpm_coef* __restrict__ dpm,
                                                                const ns2vc_unipc_coef* __restrict__ unipc,
                                                                const ns2vc_ddpm_coef* __restrict__ ddpm,
                                                                const ns2vc_ddim_coef* __restrict__ ddim,
                                                                const int64_t* __restrict__ seeds, unsigned T,
                                                                const int* __restrict__ method, int uniform_method,
                                                                const int* __restrict__ base, int* k, float* __restrict__ m_new,
                                                                float* __restrict__ x_t, float* x_new, size_t row_n,
                                                                int* nan_flags) {
  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.y;
  const int kb = k[b];
  const size_t off = (size_t)b * row_n;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  if (kb < 0) {
    for (; i < row_n; i += stride) {
      if (m_new) m_new[off + i] = 0.f;
      if (x_t) x_t[off + i] = 0.f;
      x_new[off + i] = 0.f;
    }
  } else {
    const int entry = (base ? base[b] : 0) + kb;
    const int m = method ? method[b] : uniform_method;
    bool bad = false;
    if (m == NS2VC_ROW_DPM) {
      const ns2vc_dpm_coef c = dpm[entry];
      for (; i < row_n; i += stride) dpm_update(bad, x_in, o, m0, c, m_new, x_new, off + i);
    } else if (m == NS2VC_ROW_UNIPC) {
      const ns2vc_unipc_coef c = unipc[entry];
      for (; i < row_n; i += stride) unipc_update<true>(bad, x_prev, x_in, o, m0, m1, c, m_new, x_t, x_new, off + i);
    } else if (m == NS2VC_ROW_DDPM) {
      const ns2vc_ddpm_coef c = ddpm[entry];
      const uint64_t seed = (uint64_t)seeds[b];
      for (; i < row_n; i += stride)
        ddpm_update(bad, x_in, o, c.add_noise ? seeded_normal(seed, kb, (unsigned)i / T, (unsigned)i % T) : 0.f, c, x_new, off + i);
    } else {
      const ns2vc_ddim_coef c = ddim[entry];
      const uint64_t seed = (uint64_t)seeds[b];
      for (; i < row_n; i += stride)
        ddim_update(bad, x_in, o, c.last ? 0.f : seeded_normal(seed, kb, (unsigned)i / T, (unsigned)i % T), c, x_new, off + i);
    }
    if (bad && nan_flags) atomicOr(nan_flags + b, 1);
  }
  cooperative_groups::this_cluster().sync();               // every CTA of the row has read k[b]
  if (kb >= 0 && blockIdx.x == 0 && threadIdx.x == 0) k[b] = kb + 1;
}

// DDPM and DDIM read their struct from device memory, so a captured chunk of steps serves any window of a run: the host refills
// the coefficient window before each replay.
__global__ void __launch_bounds__(256) ddpm_step_kernel(const float* x, const float* __restrict__ x0, const float* __restrict__ noise,
                                                        const ns2vc_ddpm_coef* __restrict__ cp, float* x_next, size_t n, int* nan_flag) {
  pdl_trigger();
  pdl_wait();
  const ns2vc_ddpm_coef c = *cp;
  batch_step(n, nan_flag, [&](bool& bad, size_t i) { ddpm_update(bad, x, x0, c.add_noise ? noise[i] : 0.f, c, x_next, i); });
}

__global__ void __launch_bounds__(256) ddim_step_kernel(const float* x, const float* __restrict__ x0, const float* __restrict__ noise,
                                                        const ns2vc_ddim_coef* __restrict__ cp, float* x_next, size_t n, int* nan_flag) {
  pdl_trigger();
  pdl_wait();
  const ns2vc_ddim_coef c = *cp;
  batch_step(n, nan_flag, [&](bool& bad, size_t i) { ddim_update(bad, x, x0, c.last ? 0.f : noise[i], c, x_next, i); });
}

// out[b, c, t] = the normal at (seeds[b], step, c, t) for t < T_b (lengths[b], or T), 0 past it.  Grid (x: elements, y: rows).
__global__ void __launch_bounds__(256) noise_normal_rows_kernel(const int64_t* __restrict__ seeds, uint32_t step, int C, int T,
                                                                const int64_t* __restrict__ lengths, float* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.y;
  const uint64_t seed = (uint64_t)seeds[b];
  const int64_t Tb = lengths ? lengths[b] : T;
  const size_t row_n = (size_t)C * T;
  float* row = out + (size_t)b * row_n;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < row_n; i += (size_t)gridDim.x * blockDim.x) {
    const unsigned c = (unsigned)i / (unsigned)T, t = (unsigned)i % (unsigned)T;
    row[i] = (int64_t)t < Tb ? seeded_normal(seed, step, c, t) : 0.f;
  }
}

namespace {

// A batch kernel over n elements: one per thread, at most 8 CTAs of 256 threads per SM of the H100's 132, grid-stride beyond.
template <typename... KArgs, typename... Args>
int launch_batch(void (*kernel)(KArgs...), size_t n, int* nan_flag, ns2vc_stream stream, Args... args) {
  int blocks = (int)((n + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  launch_k(kernel, dim3(blocks), dim3(256), 0, (cudaStream_t)stream, args..., n, nan_flag);
  NS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// The row kernel over B rows.  dpm_step_rows and unipc_step_rows are this launch with one method for every row and one schedule.
// Every row entry is this launch: the tables, seeds and T an entry does not take are NULL / 0.
int launch_rows(int B, ns2vc_stream stream, const float* x_in, const float* unet_out, const float* m0, const float* m1,
                const float* x_prev, const ns2vc_dpm_coef* dpm, const ns2vc_unipc_coef* unipc, const ns2vc_ddpm_coef* ddpm,
                const ns2vc_ddim_coef* ddim, const int64_t* seeds, int T, const int* method, int uniform_method, const int* base, int* k,
                float* m_new, float* x_t, float* x_new, size_t row_n, int* nan_flags) {
  launch_kc(sampler_step_rows_kernel, dim3(kRowCtas, B), dim3(256), 0, (cudaStream_t)stream, dim3(kRowCtas, 1, 1), x_in, unet_out, m0,
            m1, x_prev, dpm, unipc, ddpm, ddim, seeds, (unsigned)T, method, uniform_method, base, k, m_new, x_t, x_new, row_n, nan_flags);
  NS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace
}  // namespace ns2vc

using namespace ns2vc;

extern "C" {

int ns2vc_dpm_step(const float* x, const float* unet_out, const float* m_prev, const ns2vc_dpm_coef* c, float* m_cur, float* x_next,
                   size_t n, int* nan_flag, ns2vc_stream stream) {
  NS_REQUIRE(x && unet_out && c && m_cur, "null argument");
  NS_REQUIRE(c->order == 0 || x_next, "x_next is NULL");
  NS_REQUIRE(c->order < 2 || m_prev, "m_prev is NULL for a second-order step");
  return launch_batch(dpm_step_kernel, n, nan_flag, stream, x, unet_out, m_prev, *c, m_cur, x_next);
}

int ns2vc_unipc_step(const float* x_prev, const float* x_eval, const float* unet_out, const float* m0, const float* m1,
                     const ns2vc_unipc_coef* c, float* m_t, float* x_t, float* x_pred, size_t n, int* nan_flag, ns2vc_stream stream) {
  NS_REQUIRE(x_eval && unet_out && c && m_t, "null argument");
  NS_REQUIRE(c->corr_order == 0 || (x_prev && m0 && x_t), "corrector inputs missing");
  NS_REQUIRE(c->corr_order < 2 || m1, "m1 is NULL for an order-2 corrector");
  NS_REQUIRE(c->pred_order == 0 || x_pred, "x_pred is NULL");
  NS_REQUIRE(c->pred_order < 2 || c->corr_order > 0, "order-2 predictor needs the previous model output");
  return launch_batch(unipc_step_kernel, n, nan_flag, stream, x_prev, x_eval, unet_out, m0, m1, *c, m_t, x_t, x_pred);
}

int ns2vc_dpm_step_rows(const float* x, const float* unet_out, const float* m_prev, const ns2vc_dpm_coef* coefs, int* k, float* m_cur,
                        float* x_next, size_t row_n, int B, int* nan_flags, ns2vc_stream stream) {
  NS_REQUIRE(x && unet_out && m_prev && coefs && k && m_cur && x_next, "null argument");
  NS_REQUIRE(B >= 1 && B <= 65535 && row_n >= 1, "bad row batch %d x %zu", B, row_n);
  return launch_rows(B, stream, x, unet_out, m_prev, nullptr, nullptr, coefs, nullptr, nullptr, nullptr, nullptr, 0, nullptr,
                     NS2VC_ROW_DPM, nullptr, k, m_cur, nullptr, x_next, row_n, nan_flags);
}

int ns2vc_unipc_step_rows(const float* x_prev, const float* x_eval, const float* unet_out, const float* m0, const float* m1,
                          const ns2vc_unipc_coef* coefs, int* k, float* m_t, float* x_t, float* x_pred, size_t row_n, int B,
                          int* nan_flags, ns2vc_stream stream) {
  NS_REQUIRE(x_prev && x_eval && unet_out && m0 && m1 && coefs && k && m_t && x_t && x_pred, "null argument");
  NS_REQUIRE(B >= 1 && B <= 65535 && row_n >= 1, "bad row batch %d x %zu", B, row_n);
  return launch_rows(B, stream, x_eval, unet_out, m0, m1, x_prev, nullptr, coefs, nullptr, nullptr, nullptr, 0, nullptr,
                     NS2VC_ROW_UNIPC, nullptr, k, m_t, x_t, x_pred, row_n, nan_flags);
}

int ns2vc_sampler_step_rows(const float* x_in, const float* unet_out, const float* m0, const float* m1, const float* x_prev,
                            const ns2vc_dpm_coef* dpm_coefs, const ns2vc_unipc_coef* unipc_coefs, const int* method, const int* base,
                            int* k, float* m_new, float* x_t, float* x_new, size_t row_n, int B, int* nan_flags, ns2vc_stream stream) {
  NS_REQUIRE(x_in && unet_out && m0 && m1 && x_prev && method && base && k && m_new && x_t && x_new, "null argument");
  NS_REQUIRE(dpm_coefs || unipc_coefs, "no coefficient table");
  NS_REQUIRE(B >= 1 && B <= 65535 && row_n >= 1, "bad row batch %d x %zu", B, row_n);
  return launch_rows(B, stream, x_in, unet_out, m0, m1, x_prev, dpm_coefs, unipc_coefs, nullptr, nullptr, nullptr, 0, method, -1, base,
                     k, m_new, x_t, x_new, row_n, nan_flags);
}

int ns2vc_sampler_step_rows_seeded(const float* x_in, const float* unet_out, const float* m0, const float* m1, const float* x_prev,
                                   const ns2vc_dpm_coef* dpm_coefs, const ns2vc_unipc_coef* unipc_coefs, const ns2vc_ddpm_coef* ddpm_coefs,
                                   const ns2vc_ddim_coef* ddim_coefs, const int64_t* seeds, int T, const int* method, const int* base,
                                   int* k, float* m_new, float* x_t, float* x_new, size_t row_n, int B, int* nan_flags,
                                   ns2vc_stream stream) {
  NS_REQUIRE(x_in && unet_out && method && base && k && x_new, "null argument");
  NS_REQUIRE(dpm_coefs || unipc_coefs || ddpm_coefs || ddim_coefs, "no coefficient table");
  NS_REQUIRE(!(dpm_coefs || unipc_coefs) || (m0 && m1 && x_prev && m_new && x_t), "DPM-Solver++ / UniPC buffers missing");
  NS_REQUIRE(!(ddpm_coefs || ddim_coefs) || seeds, "seeds is NULL with a DDPM / DDIM table");
  NS_REQUIRE(B >= 1 && B <= 65535 && row_n >= 1, "bad row batch %d x %zu", B, row_n);
  NS_REQUIRE(T >= 1 && row_n % (size_t)T == 0 && row_n <= 0xFFFFFFFFu, "row_n %zu is not C * T with T = %d", row_n, T);
  return launch_rows(B, stream, x_in, unet_out, m0, m1, x_prev, dpm_coefs, unipc_coefs, ddpm_coefs, ddim_coefs, seeds, T, method, -1,
                     base, k, m_new, x_t, x_new, row_n, nan_flags);
}

int ns2vc_noise_normal_rows(const int64_t* seeds, uint32_t step, int C, int T, const int64_t* lengths, float* out, int B,
                            ns2vc_stream stream) {
  NS_REQUIRE(seeds && out, "null argument");
  NS_REQUIRE(B >= 1 && B <= 65535 && C >= 1 && T >= 1 && (size_t)C * T <= 0xFFFFFFFFu, "bad noise shape [%d, %d, %d]", B, C, T);
  int blocks = (int)(((size_t)C * T + 255) / 256);
  if (blocks > 64) blocks = 64;
  launch_k(noise_normal_rows_kernel, dim3(blocks, B), dim3(256), 0, (cudaStream_t)stream, seeds, step, C, T, lengths, out);
  NS_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int ns2vc_ddpm_step(const float* x, const float* x0, const float* noise, const ns2vc_ddpm_coef* c, float* x_next, size_t n,
                    int* nan_flag, ns2vc_stream stream) {
  NS_REQUIRE(x && x0 && c && x_next, "null argument");
  return launch_batch(ddpm_step_kernel, n, nan_flag, stream, x, x0, noise, c, x_next);
}

int ns2vc_ddim_step(const float* x, const float* x0, const float* noise, const ns2vc_ddim_coef* c, float* x_next, size_t n,
                    int* nan_flag, ns2vc_stream stream) {
  NS_REQUIRE(x && x0 && c && x_next, "null argument");
  return launch_batch(ddim_step_kernel, n, nan_flag, stream, x, x0, noise, c, x_next);
}

}  // extern "C"
