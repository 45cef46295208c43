/* ns2vc_b200 — C-ABI of the H100-native NS2VC denoiser hot path.
 *
 * The reference (adelacvg/NS2VC) is pure Python/PyTorch and defines no FFI; its boundary for this
 * path is the Python object graph (SURVEY.md §8b).  This header is the C boundary the Python
 * drop-in modules (ns2vc_b200/unet.py, fused.py) bind with ctypes; each entry point names the
 * reference interface it stands in for.  Plain C types, raw device pointers + cudaStream_t,
 * int return (0 = ok, <0 = error; ns2vc_last_error() returns the message).  No exceptions or C++
 * types cross the ABI; the caller owns every buffer, the handle owns only its packed weights and, per
 * (B, T, S, workspace) it has seen, a launch program with ~20 KB of static device tables.
 * All calls are stream-ordered.  The FIRST prepare_cond / forward / time_table for a new (B, T, S, workspace)
 * builds that program (host work, one cudaMalloc, one host-to-device copy): it must not run under stream
 * capture - run a shape once eagerly, after which its calls allocate nothing, never synchronise and are
 * capturable in a CUDA graph.  One workspace may serve several shapes one after another (prepare_cond again
 * after a switch).  One handle per device, one run at a time; not thread-safe per handle.
 */
#ifndef NS2VC_B200_H
#define NS2VC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ns2vc_unet ns2vc_unet;
typedef void* ns2vc_stream;   /* cudaStream_t */

#define NS2VC_MAX_LEVELS 8

/* Constructor arguments of UNet1DConditionModel (reference unet1d/unet_1d_condition.py:151-203,
 * as called from model.py:391-400). */
typedef struct ns2vc_unet_cfg {
  int in_channels;            /* conv_in input channels = latent + content (356)                 */
  int latent_channels;        /* leading channels that change every step (100); the rest is the  */
                              /* step-invariant content embedding whose conv_in share is hoisted  */
  int out_channels;           /* 100                                                              */
  int n_levels;
  int block_out_channels[NS2VC_MAX_LEVELS];
  int layers_per_block[NS2VC_MAX_LEVELS];
  int down_has_attn[NS2VC_MAX_LEVELS];   /* CrossAttnDownBlock2D (1) / DownBlock2D (0)           */
  int up_has_attn[NS2VC_MAX_LEVELS];     /* CrossAttnUpBlock2D (1) / UpBlock2D (0)               */
  int num_heads;              /* reference: attention_head_dim reinterpreted as head count (:219) */
  int cross_attention_dim;
  int norm_num_groups;
  float norm_eps;
  int time_scale_shift;       /* resnet_time_scale_shift == 'scale_shift'                         */
  int add_embed_text;         /* addition_embed_type == 'text'                                    */
  int add_embed_heads;        /* addition_embed_type_num_heads (64)                               */
  int flip_sin_to_cos;
  float freq_shift;
} ns2vc_unet_cfg;

const char* ns2vc_last_error(void);

/* Build the layer plan for cfg (reference ctor, unet_1d_condition.py:421-559). */
int ns2vc_unet_create(const ns2vc_unet_cfg* cfg, ns2vc_unet** out);
void ns2vc_unet_destroy(ns2vc_unet* h);

/* state_dict contract (reference key names and shapes, SURVEY.md Appendix B). */
int ns2vc_unet_num_weights(const ns2vc_unet* h);
int ns2vc_unet_weight_info(const ns2vc_unet* h, int i, const char** name, int64_t shape[4], int* ndim);
/* Copy one parameter (device fp32, contiguous) into the handle: load_state_dict per key. */
int ns2vc_unet_load_weight(ns2vc_unet* h, const char* key, const float* dptr, const int64_t* shape, int ndim,
                           ns2vc_stream stream);
/* Pack every contraction weight into the wgmma operand layout (bf16 hi/lo, swizzled tiles);
 * fails if any key is missing (strict load, reference inference/infer_tool.py:27). */
int ns2vc_unet_finalize(ns2vc_unet* h, ns2vc_stream stream);

int ns2vc_unet_workspace_bytes(const ns2vc_unet* h, int B, int T, int S, size_t* bytes);

/* Step-invariant conditioning (the part of Diffusion_Encoder.forward / UNet forward that does not
 * depend on x or t: model.py:406-411, unet_1d_condition.py:816-818, 869-870, cross-attention K/V
 * attention_processor.py:1017-1020).
 *   content : [B, in_channels-latent_channels, T] fp32, batch stride content_bstride floats (may be NULL if 0 ch)
 *   prompt  : [B, S, cross_attention_dim] fp32 contiguous (encoder_hidden_states)
 *   mask    : [B, S] uint8 (1 = attend), or NULL (no encoder_attention_mask)                    */
int ns2vc_unet_prepare_cond(ns2vc_unet* h, const float* content, long long content_bstride, const float* prompt,
                            const uint8_t* mask, int B, int T, int S, void* ws, ns2vc_stream stream);

/* The same for a ragged batch: utterance b has content_lengths[b] <= T frames and prompt_lengths[b] <= S prompt frames
 * (int64 [B] device arrays; values are clamped to [1, T] / [1, S]).  It selects the RAGGED program of (B, T, S, workspace),
 * whose tables these lengths fill: the ns2vc_unet_forward / _forward_film / _time_table calls that follow run it, and
 * row b of their output equals utterance b run alone on x[b, :, :T_b], content[b, :, :T_b], prompt[b, :S_b] (no mask).
 * Output frames >= T_b are exact zeros; input values past the lengths are never read.  Lengths may change between calls
 * without a rebuild (one program and one captured graph serve every length vector).  The padded program of the same key
 * is untouched: ns2vc_unet_prepare_cond selects it again. */
int ns2vc_unet_prepare_cond_ragged(ns2vc_unet* h, const float* content, long long content_bstride, const float* prompt,
                                   const int64_t* content_lengths, const int64_t* prompt_lengths, int B, int T, int S, void* ws,
                                   ns2vc_stream stream);

/* ns2vc_unet_prepare_cond_ragged for the n_rows entries listed in rows (host array of distinct indices in [0, B)) only:
 * their length and key-bias tables, content conditioning, pooled prompt embedding and cross-attention K/V are recomputed
 * from the same arguments (content_lengths / prompt_lengths are the full int64 [B] device arrays) and written exactly as
 * the full call writes them; no byte of any other entry changes.  The ragged program of (B, T, S, workspace) must already
 * have been prepared by ns2vc_unet_prepare_cond_ragged (and no other key run on the handle since).  Each listed entry is
 * its own launches at B = 1 (listing every entry runs the full program once).  Stream-ordered, no host sync. */
int ns2vc_unet_prepare_cond_rows(ns2vc_unet* h, const float* content, long long content_bstride, const float* prompt,
                                 const int64_t* content_lengths, const int64_t* prompt_lengths, const int* rows, int n_rows,
                                 int B, int T, int S, void* ws, ns2vc_stream stream);

/* UNet1DConditionModel.forward (unet_1d_condition.py:743-1037) given prepared conditioning.
 *   x [B, latent_channels, T] fp32 (batch stride x_bstride floats), t [B] fp32 -> out [B, out_channels, T] */
int ns2vc_unet_forward(ns2vc_unet* h, const float* x, long long x_bstride, const float* t, float* out, int B, int T,
                       int S, void* ws, ns2vc_stream stream);

/* The timestep path of many forwards at once (the sampler knows every evaluation time when the run starts):
 * Timesteps -> TimestepEmbedding (+ the pooled prompt embedding) -> time_emb_proj of all resnets
 * (reference embeddings.py:24-64, 157-218; unet_1d_condition.py:825-883; resnet.py:619-629).
 *   t_rows [n_rows] fp32 device, n_rows = steps x B in step-major order (row r belongs to batch entry r % B)
 *   table  device buffer of ns2vc_unet_time_table_floats(h, n_rows) floats; its first n_rows x film_width floats are the
 *          FiLM rows, the rest is scratch.  Needs ns2vc_unet_prepare_cond() on the same (B,T,S,workspace) first.        */
int ns2vc_unet_film_width(const ns2vc_unet* h);
size_t ns2vc_unet_time_table_floats(const ns2vc_unet* h, int n_rows);
int ns2vc_unet_time_table(ns2vc_unet* h, const float* t_rows, int n_rows, float* table, int B, int T, int S, void* ws,
                          ns2vc_stream stream);
/* The FiLM rows k * B + b of such a table for the entries b listed in rows (host array of n_rows distinct indices in [0, B))
 * and every step k < n_steps, bit-identical to what ns2vc_unet_time_table(t_rows, n_steps * B, ...) writes there; every
 * other FiLM row is left as it was.  t_rows and table are laid out as for that call.  Each listed entry is three launches
 * of n_steps rows (listing every entry computes the whole table in three launches). */
int ns2vc_unet_time_table_rows(ns2vc_unet* h, const float* t_rows, int n_steps, const int* rows, int n_rows, float* table, int B,
                               int T, int S, void* ws, ns2vc_stream stream);
/* ns2vc_unet_forward with the timestep path taken from B rows of such a table (film_rows = table + step * B * film_width). */
int ns2vc_unet_forward_film(ns2vc_unet* h, const float* x, long long x_bstride, const float* film_rows, float* out, int B,
                            int T, int S, void* ws, ns2vc_stream stream);

/* Per-step sampler math fused into one element-wise kernel (bit-exact fp32 op order).
 * DPM-Solver++(2M): model_wrapper x_start->noise (sampler/dpm_solver.py:291-292), data_prediction_fn
 * (:437-439), dpm_solver_first_update (:569-576), multistep_dpm_solver_second_update (:813-831). */
typedef struct ns2vc_dpm_coef {
  float alpha_s, sigma_s;     /* at the time the UNet was evaluated (x0 round trip)                */
  float c_x;                  /* sigma_t / sigma_s                                                 */
  float c_m;                  /* alpha_t * expm1(-h)                                               */
  float c_d;                  /* 0.5 * c_m                                                         */
  float inv_r0;               /* 1 / r0 (order 2 only)                                             */
  int order;                  /* 0: x0 round trip only; 1 / 2: + first / second order update       */
} ns2vc_dpm_coef;
/* x_next = (c_x*x - c_m*m_cur) - c_d*(inv_r0*(m_cur - m_prev)), the last term at order 2 only */
/* nan_flag (device int, may be NULL): set to 1 when x holds a NaN - the reference asserts on that every denoiser call
 * (model.py:404); the fused loop checks the flag once after the run instead of syncing every step. */
int ns2vc_dpm_step(const float* x, const float* unet_out, const float* m_prev, const ns2vc_dpm_coef* c, float* m_cur,
                   float* x_next, size_t n, int* nan_flag, ns2vc_stream stream);

/* UniPC-bh2 (sampler/uni_pc.py:471-588): corrector at t and predictor to the next time. */
typedef struct ns2vc_unipc_coef {
  float alpha_t, sigma_t;     /* x0 round trip at t                                                */
  /* corrector at t from (x_prev, m0, m1): x_t = xbar - ab*(rho0*D1 + rho1*(m_t - m0))                */
  float c_x, c_m;             /* xbar = c_x*x_prev - c_m*m0                                        */
  float ab;                   /* alpha_t * B_h                                                     */
  float rk;                   /* D1 = (m1 - m0) / rk (order-2 corrector)                           */
  float rho0, rho1;
  int corr_order;             /* 0: no corrector (the first step: history only), 1, 2              */
  /* predictor to the next time from (x_t, m_t, m0): x_pred = nbar - nab*(0.5*D1n), D1n = (m0 - m_t)/nrk */
  float n_c_x, n_c_m;         /* nbar = n_c_x*x_t - n_c_m*m_t                                      */
  float nab, nrk;
  int pred_order;             /* 0: none, 1: nbar only, 2: with D1n                                */
} ns2vc_unipc_coef;
int ns2vc_unipc_step(const float* x_prev, const float* x_eval, const float* unet_out, const float* m0, const float* m1,
                     const ns2vc_unipc_coef* c, float* m_t, float* x_t, float* x_pred, size_t n, int* nan_flag,
                     ns2vc_stream stream);

/* The two steps above for rows at different steps: row b of a [B, row_n] batch (row_n = Cl * T elements per row) takes step
 * k[b] of a run whose coefficient structs are the DEVICE array coefs (one per step; k[b] must be below their count).
 *   k [B] int32 device: each row's step, or -1 for an empty row.  An occupied row's results are bit-identical to the scalar entry
 *     run on that row with struct coefs[k[b]]; an empty row writes 0 to every output and raises no flag.  Each occupied k[b] is
 *     advanced by one, so a captured step replays with no host write in between.
 *   nan_flags [B] int32 device (may be NULL): entry b is set to 1 when row b's x (x_eval) holds a NaN.
 * Every buffer pointer is required (any row may need any operand).  UniPC: a row at its first step (corr_order == 0) writes
 * x_t = x_eval, so the rotation m1 <- m0 <- m_t, x_prev <- x_t, x_eval <- x_pred is the same for every row. */
int ns2vc_dpm_step_rows(const float* x, const float* unet_out, const float* m_prev, const ns2vc_dpm_coef* coefs, int* k, float* m_cur,
                        float* x_next, size_t row_n, int B, int* nan_flags, ns2vc_stream stream);
int ns2vc_unipc_step_rows(const float* x_prev, const float* x_eval, const float* unet_out, const float* m0, const float* m1,
                          const ns2vc_unipc_coef* coefs, int* k, float* m_t, float* x_t, float* x_pred, size_t row_n, int B,
                          int* nan_flags, ns2vc_stream stream);

/* One row step for rows of either method: row b of a [B, row_n] batch takes step k[b] of its own schedule.
 *   method [B] int32 device: NS2VC_ROW_DPM (DPM-Solver++) or NS2VC_ROW_UNIPC (UniPC-bh2); read only for occupied rows.
 *   base [B] int32 device: where row b's schedule starts in its method's table, so row b's struct is
 *     dpm_coefs[base[b] + k[b]] or unipc_coefs[base[b] + k[b]].  Each table holds the structs of every schedule of that method
 *     in use, back to back; a table no occupied row selects may be NULL.
 *   k [B] int32 device: each row's step within its schedule, or -1 for an empty row; each occupied k[b] is advanced by one.
 *   nan_flags [B] int32 device (may be NULL): entry b is set to 1 when row b's x_in holds a NaN.
 * Both methods use one buffer layout, so the rotation after the step is the same four copies for every row:
 *   plane     DPM-Solver++   UniPC
 *   x_in      x              x_eval      (the denoiser input)
 *   m0        m_prev         m0
 *   m1        -              m1
 *   x_prev    -              x_prev
 *   m_new     m_cur          m_t         (written)
 *   x_t       -              x_t         (written; x_eval at a row's first step)
 *   x_new     x_next         x_pred      (written)
 * and the rotation is m1 <- m0, m0 <- m_new, x_prev <- x_t, x_in <- x_new.  A DPM row never reads m1 or x_prev and never writes
 * x_t.  An occupied row's results are bit-identical to ns2vc_dpm_step / ns2vc_unipc_step run on that row with its struct; an
 * empty row writes 0 to m_new, x_t and x_new and raises no flag.  Every pointer except nan_flags and one of the tables is
 * required.  ns2vc_dpm_step_rows and ns2vc_unipc_step_rows are this step with one method and one schedule (base 0). */
#define NS2VC_ROW_DPM 0
#define NS2VC_ROW_UNIPC 1
int ns2vc_sampler_step_rows(const float* x_in, const float* unet_out, const float* m0, const float* m1, const float* x_prev,
                            const ns2vc_dpm_coef* dpm_coefs, const ns2vc_unipc_coef* unipc_coefs, const int* method, const int* base,
                            int* k, float* m_new, float* x_t, float* x_new, size_t row_n, int B, int* nan_flags, ns2vc_stream stream);

/* DDPM p_sample (model.py:535-542) and DDIM (model.py:586-601) steps after the denoiser returned x0 = x_start.
 * UNLIKE the two entries above, `c` is a DEVICE pointer to one coefficient struct, read by the kernel: a captured chunk of
 * steps then serves every chunk of a long run (the host refills a device window of structs before each replay).
 * x, x0, noise, x_next: n fp32 device values; x_next may equal x (in place).  noise is not read when the step adds none
 * (add_noise == 0 / last != 0) and may then be NULL.  nan_flag as for ns2vc_dpm_step (NaN in the step's input x). */
typedef struct ns2vc_ddpm_coef {
  float c_x0;                 /* posterior_mean_coef1[t]                                                      */
  float c_x;                  /* posterior_mean_coef2[t]                                                      */
  float c_noise;              /* exp(0.5 * posterior_log_variance_clipped[t])                                 */
  int add_noise;              /* t > 0; otherwise x_next = mean + 0.0f (the reference adds exp(.) * 0.)      */
} ns2vc_ddpm_coef;
/* x_next = (c_x0*x0 + c_x*x) + c_noise*noise */
int ns2vc_ddpm_step(const float* x, const float* x0, const float* noise, const ns2vc_ddpm_coef* c, float* x_next, size_t n,
                    int* nan_flag, ns2vc_stream stream);

typedef struct ns2vc_ddim_coef {
  float sqrt_recip;           /* sqrt_recip_alphas_cumprod[t]                                                 */
  float sqrt_recipm1;         /* sqrt_recipm1_alphas_cumprod[t]                                               */
  float sqrt_alpha_next;      /* alphas_cumprod[t_next].sqrt()                                                */
  float c;                    /* (1 - alpha_next - sigma**2).sqrt()                                           */
  float sigma;                /* eta * ((1 - alpha/alpha_next) * (1 - alpha_next) / (1 - alpha)).sqrt()       */
  int last;                   /* t_next < 0: x_next = x0                                                      */
} ns2vc_ddim_coef;
/* pn = (sqrt_recip*x - x0) / sqrt_recipm1 ; x_next = (x0*sqrt_alpha_next + c*pn) + sigma*noise (also at eta = 0) */
int ns2vc_ddim_step(const float* x, const float* x0, const float* noise, const ns2vc_ddim_coef* c, float* x_next, size_t n,
                    int* nan_flag, ns2vc_stream stream);

/* Seeded sampler noise (csrc/philox.cuh): the normal at (seed, step, c, t) is a pure function of those four values, Philox4x32-10
 * keyed by the 64-bit seed with counter (t >> 2, c, step, 0) and a Box-Muller transform of its outputs, so an utterance's noise does
 * not depend on its batch, slot, padding or launch.  Step NS2VC_XT_STEP is reserved for the utterance's x_T.
 *   ns2vc_noise_normal_rows: out [B, C, T] fp32 device, out[b, c, t] = the normal at (seeds[b], step, c, t) for t < T_b and 0 past
 *   it; seeds [B] int64 device (>= 0), lengths [B] int64 device (T_b in [1, T]) or NULL (every T_b = T). */
#define NS2VC_XT_STEP 0xFFFFFFFFu
int ns2vc_noise_normal_rows(const int64_t* seeds, uint32_t step, int C, int T, const int64_t* lengths, float* out, int B,
                            ns2vc_stream stream);

/* ns2vc_sampler_step_rows with seeded DDPM and DDIM rows as well: method[b] may also be
 *   NS2VC_ROW_DDPM: struct ddpm_coefs[base[b] + k[b]];  NS2VC_ROW_DDIM: struct ddim_coefs[base[b] + k[b]].
 * Such a row reads x_in (x) and unet_out (x0) only and writes x_new only (x_new may equal x_in); it never reads m0, m1 or x_prev
 * and never writes m_new or x_t, so the four-copy rotation above stays the same for every row.  Its step noise is drawn
 * in-register at (seeds[b], k[b], c, t), where row element i = c * T + t (row_n = C * T), bit-identical to
 * ns2vc_noise_normal_rows(seeds, k[b], ...); its x_next is bit-identical to ns2vc_ddpm_step / ns2vc_ddim_step fed with that
 * tensor.  seeds [B] int64 device is required when a DDPM or DDIM table is given; m0, m1, x_prev, m_new and x_t when a DPM-Solver++
 * or UniPC table is.  A table no occupied row selects may be NULL.  DPM-Solver++ and UniPC rows, empty rows, k and the NaN flags are
 * as for ns2vc_sampler_step_rows (an empty row leaves a NULL m_new or x_t alone). */
#define NS2VC_ROW_DDPM 2
#define NS2VC_ROW_DDIM 3
int ns2vc_sampler_step_rows_seeded(const float* x_in, const float* unet_out, const float* m0, const float* m1, const float* x_prev,
                                   const ns2vc_dpm_coef* dpm_coefs, const ns2vc_unipc_coef* unipc_coefs, const ns2vc_ddpm_coef* ddpm_coefs,
                                   const ns2vc_ddim_coef* ddim_coefs, const int64_t* seeds, int T, const int* method, const int* base,
                                   int* k, float* m_new, float* x_t, float* x_new, size_t row_n, int B, int* nan_flags,
                                   ns2vc_stream stream);

/* Bit-exact index helpers (host, no GPU): nearest-neighbour source index of F.interpolate(size=)
 * (reference resnet.py:160) and the stride-2 conv length rule (resnet.py:200). */
int ns2vc_nearest_index(int t_in, int t_out, int* idx /* [t_out] */);
int ns2vc_down_length(int t);

/* encoder_attention_mask -> additive attention bias, (1 - m) * -10000 (reference unet_1d_condition.py:816-818): the kernel
 * prepare_cond runs, exposed for the bit-exact test.  mask [n] uint8 device, bias [n] fp32 device. */
int ns2vc_mask_bias(const uint8_t* mask, int n, float* bias, ns2vc_stream stream);

/* Diagnostics used by the parity tests. */
int ns2vc_unet_num_taps(const ns2vc_unet* h);
int ns2vc_unet_tap_info(const ns2vc_unet* h, int i, const char** name, int* level, int* channels);
int ns2vc_unet_set_tap(ns2vc_unet* h, int i, float* dst /* device [B, T_level, C] token-major, or NULL */);
const char* ns2vc_unet_plan_string(const ns2vc_unet* h);
int ns2vc_unet_launch_count(const ns2vc_unet* h);  /* kernels launched by the last forward */
const char* ns2vc_build_info(void);

/* Per-kernel-kind device timing (CUDA events around every launch on the caller's stream); used by
 * bench.py for the roofline line.  Off by default; never enable inside a timed region. */
int ns2vc_unet_set_profiling(ns2vc_unet* h, int on);
/* In-kernel stamps of CTA (0,0) of every GEMM launch of the next forwards, 32 slots per launch: [0,8) %globaltimer
 * (entry, prologue, PDL wait, first stage full, MMAs issued, accumulator ready, epilogue done, exit), [8,16) SM-clock
 * stamps of the epilogue sub-steps, [16,22) %globaltimer stamps of the fused prep (dependency wait done, loads issued,
 * affine ready, rows stored, all preps done, published to the cluster).  NULL disables. */
int ns2vc_unet_set_trace(ns2vc_unet* h, unsigned long long* device_buf, int n_gemms);
/* Diagnostics: attention launch i of the next forward writes per-key-tile SM-clock stamps of its CTA (0,0,0)
 * to device_buf[2048*i ...] ([16 tiles][16 slots], then [start ns, end ns, SM id] of up to 597 CTAs; see attention_v2.cu).
 * NULL disables. */
int ns2vc_unet_set_attn_trace(ns2vc_unet* h, unsigned long long* device_buf, int n_launches);
/* [min entry, max exit] %globaltimer of every launch of the next forwards (buffer pre-set to {~0, 0} pairs). */
int ns2vc_unet_set_span_trace(ns2vc_unet* h, unsigned long long* device_buf, int n_launches);
int ns2vc_unet_launch_kind(const ns2vc_unet* h, int launch_index);   /* index into ns2vc_profile_kind_name */
int ns2vc_profile_num_kinds(void);
const char* ns2vc_profile_kind_name(int kind);
int ns2vc_unet_profile_read(ns2vc_unet* h, int kind, double* ms_total, long long* launches);
int ns2vc_unet_profile_dump(ns2vc_unet* h, const char* csv_path);   /* one row per launch */
int ns2vc_unet_profile_reset(ns2vc_unet* h);

/* ------------------------------------------------------------------------------------------------------------------
 * Condition encoders: `Pre_model.infer` (reference model.py:359-377) - the step immediately BEFORE the denoiser
 * (SURVEY.md 8(f) rank 1): ref_enc (TextTimeEmbedding, unet1d/embeddings.py:421-434), PromptEncoder and PhoneEncoder
 * (model.py:98-190: ConvLayer -> n x EncSALayer (operations.py:784-821: LayerNorm, 8-head self-attention with key padding,
 * LayerNorm, k=9 conv-FFN) -> ConvLayer -> LayerNorm), all frames past an utterance's length exactly zero.
 * Same conventions as the denoiser handle above: raw device pointers, caller-owned workspace, stream-ordered, int errors.
 * The first call for a new (B, T, S, workspace) builds the launch program on the host (no device allocation). */
typedef struct ns2vc_pre ns2vc_pre;
typedef struct ns2vc_pre_cfg {       /* reference config.json "phoneme_encoder" / "prompt_encoder" (model.py:332-340)        */
  int phone_in, phone_hidden, phone_out, phone_layers;       /* PhoneEncoder(in_channels, hidden_channels, out_channels, n_layers) */
  int prompt_in, prompt_hidden, prompt_out, prompt_layers;   /* PromptEncoder(...)                                          */
  int ref_dim;                       /* TextTimeEmbedding(100, 100, 1): width of the mel prompt (= prompt_in)                 */
  int ref_heads;                     /* 1                                                                                     */
  int n_heads;                       /* EncSALayer(c, 8, ...) (operations.py:961)                                             */
  int ffn_kernel;                    /* 9 (operations.py:963)                                                                 */
} ns2vc_pre_cfg;
int ns2vc_pre_create(const ns2vc_pre_cfg* cfg, ns2vc_pre** out);
void ns2vc_pre_destroy(ns2vc_pre* h);
int ns2vc_pre_num_weights(const ns2vc_pre* h);                                  /* state_dict contract: reference key names / shapes */
int ns2vc_pre_weight_info(const ns2vc_pre* h, int i, const char** name, int64_t shape[4], int* ndim);
int ns2vc_pre_load_weight(ns2vc_pre* h, const char* key, const float* dptr, const int64_t* shape, int ndim, ns2vc_stream stream);
int ns2vc_pre_finalize(ns2vc_pre* h, ns2vc_stream stream);                      /* strict: fails on a missing key                   */
/* One size serves every program of the handle at (B, T, S): ns2vc_pre_infer, _infer_ragged, _encode_voices_ragged of (B, S) and
 * _infer_content_ragged of (B, T). */
int ns2vc_pre_workspace_bytes(const ns2vc_pre* h, int B, int T, int S, size_t* bytes);
/* Pre_model.infer:
 *   c [B, phone_in, T] fp32, refer [B, prompt_in, S] fp32 (contiguous), lengths / refer_lengths [B] int64 (device, each >= 1)
 *   -> content [B, T, phone_out], prompt [B, S, prompt_out] fp32 token-major (the reference returns the [T, B, C] / [S, B, C]
 *      views of the same values: model.py:145, 189).                                                                        */
int ns2vc_pre_infer(ns2vc_pre* h, const float* c, const float* refer, const int64_t* lengths, const int64_t* refer_lengths,
                    float* content, float* prompt, int B, int T, int S, void* ws, ns2vc_stream stream);
/* Ragged batch, same arguments: row b equals ns2vc_pre_infer of c[b, :, :T_b], refer[b, :, :S_b] alone (B = 1, T = T_b, S = S_b),
 * T_b = lengths[b] in [1, T], S_b = refer_lengths[b] in [1, S]; frames past T_b / S_b are exactly 0 and input values there are
 * never read.  A second program per (B, T, S, workspace); the workspace size above serves both. */
int ns2vc_pre_infer_ragged(ns2vc_pre* h, const float* c, const float* refer, const int64_t* lengths, const int64_t* refer_lengths,
                           float* content, float* prompt, int B, int T, int S, void* ws, ns2vc_stream stream);
/* The ragged program in two halves, so that a target voice is encoded once and reused with any content:
 * the voice half reads refer [B, prompt_in, S] and refer_lengths [B] (S_b in [1, S]) and writes
 *   spk [B, phone_hidden]           phoneme_encoder.spk_proj(ref_enc(refer)), the one vector by which the voice enters the content,
 *   prompt [B, S, prompt_out]        the prompt encoder's output, exactly 0 past S_b;
 * the content half reads c [B, phone_in, T], lengths [B] (T_b in [1, T]) and row b's speaker vector spk[b] and writes
 *   content [B, T, phone_out]        exactly 0 past T_b.
 * Row b of each equals, byte for byte, the same row of ns2vc_pre_infer_ragged on that prompt and content: both halves are its
 * launches, split after spk_proj.  Each is one more program per shape and workspace (size: ns2vc_pre_workspace_bytes above), and
 * each zeroes its own LayerNorm statistics, so their launch counts add up to ns2vc_pre_infer_ragged's plus one. */
int ns2vc_pre_encode_voices_ragged(ns2vc_pre* h, const float* refer, const int64_t* refer_lengths, float* spk, float* prompt, int B, int S,
                                   void* ws, ns2vc_stream stream);
int ns2vc_pre_infer_content_ragged(ns2vc_pre* h, const float* c, const int64_t* lengths, const float* spk, float* content, int B, int T,
                                   void* ws, ns2vc_stream stream);
/* Diagnostics for the parity tests: per-layer activations (token-major [B, rows, channels]; rows = 1 for the speaker vector). */
int ns2vc_pre_num_taps(const ns2vc_pre* h);
int ns2vc_pre_tap_info(const ns2vc_pre* h, int i, const char** name, int* rows, int* channels);
int ns2vc_pre_set_tap(ns2vc_pre* h, int i, float* dst);
int ns2vc_pre_launch_count(const ns2vc_pre* h);   /* kernels launched by the last call of any of the four programs */

/* ------------------------------------------------------------------------------------------------------------------
 * Prompt-mel front end: the recipe of reference inference/infer_tool.py:170-181 (and preprocess.py:27-31, 49-59) per
 * utterance of a ragged batch - torchaudio Resample(orig, new) (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99),
 * then MelSpectrogram at the fixed parameters below, then log(max(., 1e-7)).
 * Same conventions as above: raw device pointers, device int64 lengths, caller-owned outputs, int errors, stream-ordered.
 * create builds and uploads the handle's tables on the current device; the calls allocate nothing and never synchronise.
 * A handle is read-only after create: it may serve several streams at once. */
#define NS2VC_MEL_SAMPLE_RATE 24000   /* Hz                                                                  */
#define NS2VC_MEL_N_FFT 1024          /* periodic Hann window of n_fft, center=True with reflect padding of  */
#define NS2VC_MEL_HOP 256             /* n_fft / 2 at each utterance's own ends, one-sided magnitude          */
#define NS2VC_MEL_N_MELS 100          /* HTK mel scale, 0 .. NS2VC_MEL_F_MAX Hz, norm=None                    */
#define NS2VC_MEL_F_MAX 12000.0
#define NS2VC_MEL_LOG_CLIP 1e-7f
typedef struct ns2vc_resampler ns2vc_resampler;
typedef struct ns2vc_mel ns2vc_mel;
/* Host-only, no GPU: torchaudio's output length of Resample(orig, new) for n input samples, ceil(fp32(new * n / orig))
 * with the ratio reduced by its gcd and the quotient taken in fp64 (NOT the exact integer ceiling); n when orig == new;
 * -1 on bad arguments. */
long long ns2vc_resample_out_length(int orig_freq, int new_freq, long long n);
/* Host-only: the resampler's fp32 phase table [phases][taps] (phases = new / gcd, taps = 2 * width + orig / gcd) as torchaudio
 * builds it in fp64 and rounds it; table may be NULL to query the sizes.  orig == new has no table (error). */
int ns2vc_resample_table(int orig_freq, int new_freq, int* phases, int* taps, int* width, float* table);
/* Host-only: the dense fp32 mel filterbank [513][100] (torchaudio melscale_fbanks at the parameters above). */
int ns2vc_mel_filterbank(float* fb);
/* Host-only, no GPU: 0 when ns2vc_resampler_create accepts the rate pair, else -1 with the reason (a bad rate, or a ratio whose
 * input window per CTA exceeds 48 KB of shared memory), so a caller can reject an input before any device work. */
int ns2vc_resample_check(int orig_freq, int new_freq);
int ns2vc_resampler_create(int orig_freq, int new_freq, ns2vc_resampler** out);   /* orig == new: a copy */
void ns2vc_resampler_destroy(ns2vc_resampler* h);
/* x [B, n] fp32 (batch stride x_bstride floats), lengths [B] int64 device (each <= n; NULL: every row n)
 *   -> y [B, n_out] (batch stride y_bstride), n_out <= ns2vc_resample_out_length(orig, new, n).  Row b is
 *   Resample(orig, new)(x[b, :lengths[b]]); samples at or past its output length are exactly 0. */
int ns2vc_resample(const ns2vc_resampler* h, const float* x, long long x_bstride, long long n, const int64_t* lengths, float* y,
                   long long y_bstride, long long n_out, int B, ns2vc_stream stream);
/* window [1024] and fb [513][100]: host fp32 tables, or NULL for the library's own (the periodic Hann window in fp64 rounded to
 * fp32; ns2vc_mel_filterbank()).  The reference's recipe uses torch's fp32 tables, whose vectorised cosf / powf round some
 * entries 1 ulp apart from the C library's; a quiet mel band notices that more than the kernel's own rounding, so a caller
 * matching the reference passes torch.hann_window(1024) and torch's melscale_fbanks (ns2vc_b200.frontend does). */
int ns2vc_mel_create(const float* window, const float* fb, ns2vc_mel** out);
void ns2vc_mel_destroy(ns2vc_mel* h);
/* x [B, n] fp32 at 24 kHz (batch stride x_bstride floats), lengths [B] int64 device (each in (512, n]; NULL: every row n)
 *   -> mel [B, 100, S] fp32 contiguous, S <= 1 + n / 256: log(max(MelSpectrogram(x[b, :len]), 1e-7)); frames at or past
 *   1 + lengths[b] / 256 are exactly 0. */
int ns2vc_log_mel(const ns2vc_mel* h, const float* x, long long x_bstride, long long n, const int64_t* lengths, float* mel, int S,
                  int B, ns2vc_stream stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Vocoder: `Vocos.decode` (vocos/pretrained.py) of the mel configuration the reference loads (charactr/vocos-mel-24khz,
 * model.py:689-691): VocosBackbone (vocos/models.py: Conv1d embed k=7, LayerNorm, ConvNeXtBlocks of vocos/modules.py, final
 * LayerNorm; no AdaLayerNorm) and ISTFTHead (vocos/heads.py: Linear to n_fft + 2, exp / clip 100 / phase, the "same"-padded
 * ISTFT of vocos/spectral_ops.py).  A ragged batch decodes row b as if it were decoded alone on its first lengths[b] frames.
 * Same conventions as the encoders: raw device pointers, caller-owned workspace, stream-ordered, int errors; the first call for
 * a new (B, T, workspace) builds the launch program on the host, later calls allocate nothing and may be captured. */
typedef struct ns2vc_voc ns2vc_voc;
typedef struct ns2vc_voc_cfg {       /* VocosBackbone(input_channels, dim, intermediate_dim, num_layers) + ISTFTHead(dim, n_fft,  */
  int input_channels, dim, intermediate_dim, num_layers, n_fft, hop_length;   /* hop_length, padding="same")                     */
} ns2vc_voc_cfg;
/* Only the "same" padding and no AdaLayerNorm exist here; the configuration must have n_fft = 4 hop_length (a power of two,
 * 64 .. 2048), dim a multiple of 128 up to 1024 and intermediate_dim a multiple of 64. */
int ns2vc_voc_create(const ns2vc_voc_cfg* cfg, ns2vc_voc** out);
void ns2vc_voc_destroy(ns2vc_voc* h);
int ns2vc_voc_num_weights(const ns2vc_voc* h);                                  /* backbone.* / head.* keys of Vocos.state_dict() */
int ns2vc_voc_weight_info(const ns2vc_voc* h, int i, const char** name, int64_t shape[4], int* ndim);
int ns2vc_voc_load_weight(ns2vc_voc* h, const char* key, const float* dptr, const int64_t* shape, int ndim, ns2vc_stream stream);
int ns2vc_voc_finalize(ns2vc_voc* h, ns2vc_stream stream);                      /* strict: fails on a missing key                   */
int ns2vc_voc_workspace_bytes(const ns2vc_voc* h, int B, int T, size_t* bytes);
/* Vocos.decode: mel [B, input_channels, T] fp32 (row-contiguous, batch stride mel_bstride floats), lengths [B] int64 device or
 * NULL (every row T; values are clamped into [1, T]) -> audio [B, T * hop_length] fp32.  Row b equals the row decoded alone on
 * mel[b, :, :lengths[b]]; its samples >= lengths[b] * hop_length are exactly 0 and mel frames past lengths[b] are never read. */
int ns2vc_voc_decode(ns2vc_voc* h, const float* mel, long long mel_bstride, const int64_t* lengths, float* audio, int B, int T,
                     void* ws, ns2vc_stream stream);
/* The head's ISTFT stage alone: head_out [B, T, n_fft + 2] fp32 token-major (log-magnitudes, then phases) -> audio as above. */
int ns2vc_voc_istft(ns2vc_voc* h, const float* head_out, const int64_t* lengths, float* audio, int B, int T, ns2vc_stream stream);
/* Diagnostics for the parity tests: activations after backbone.norm, each convnext block, final_layer_norm ([B, T, dim]) and
 * head.out ([B, T, channels] with channels = n_fft + 2 rounded up to a multiple of 4: columns past n_fft + 2 are padding). */
int ns2vc_voc_num_taps(const ns2vc_voc* h);
int ns2vc_voc_tap_info(const ns2vc_voc* h, int i, const char** name, int* rows, int* channels);
int ns2vc_voc_set_tap(ns2vc_voc* h, int i, float* dst);
int ns2vc_voc_launch_count(const ns2vc_voc* h);   /* kernels launched by the last decode */

/* ------------------------------------------------------------------------------------------------------------------
 * Content encoder: the units of `utils.get_hubert_content` (ContentVec, a fairseq HubertModel of extractor_mode "default",
 * layer_norm_first False, no conv biases): `extract_features(source, padding_mask = all False, output_layer = num_layers)` then
 * `final_proj`.  The feature encoder's convs are fairseq's default [(C, 10, 5)] + [(C, 3, 2)] * 4 + [(C, 2, 2)] * 2.  A ragged
 * batch computes row b as if it were run alone on its first lengths[b] samples.  Same conventions as the vocoder. */
typedef struct ns2vc_cv ns2vc_cv;
typedef struct ns2vc_cv_cfg {        /* ContentVec legacy: 512, 768, 3072, 12, 12, 128, 16, 256 */
  int conv_dim, embed_dim, ffn_dim, num_layers, num_heads, pos_conv_kernel, pos_conv_groups, final_dim;
} ns2vc_cv_cfg;
/* Rejected: conv_dim or embed_dim not a multiple of 128 up to 1024, a head dim other than 16 / 32 / 48 / 64, ffn_dim not a
 * multiple of 64, final_dim not a multiple of 4, positional-conv groups wider than 64 channels or not a multiple of 4, and
 * pos_conv_kernel not a multiple of 16 up to 128. */
int ns2vc_cv_create(const ns2vc_cv_cfg* cfg, ns2vc_cv** out);
void ns2vc_cv_destroy(ns2vc_cv* h);
int ns2vc_cv_num_weights(const ns2vc_cv* h);     /* HubertModel.state_dict() keys without mask_emb / label_embs_concat, in its order */
int ns2vc_cv_weight_info(const ns2vc_cv* h, int i, const char** name, int64_t shape[4], int* ndim);
int ns2vc_cv_load_weight(ns2vc_cv* h, const char* key, const float* dptr, const int64_t* shape, int ndim, ns2vc_stream stream);
int ns2vc_cv_finalize(ns2vc_cv* h, ns2vc_stream stream);   /* strict: fails on a missing key; folds the weight norm and q's scaling */
int ns2vc_cv_workspace_bytes(const ns2vc_cv* h, int B, int N, size_t* bytes);
/* Frames of n samples (0 below 400): T = floor((T - k) / s) + 1 through the seven convs. */
int ns2vc_cv_num_frames(long long n);
/* wav [B, N] fp32 at 16 kHz (batch stride wav_bstride floats), lengths [B] int64 device or NULL (every row N; values are clamped
 * into [400, N]) -> units [B, T, final_dim] fp32 with T = ns2vc_cv_num_frames(N), frames [B] int64 device (or NULL): each row's
 * frame count.  Row b equals the row run alone on wav[b, :lengths[b]]; its frames >= frames[b] are exactly 0 and samples past
 * lengths[b] are never read. */
int ns2vc_cv_extract(ns2vc_cv* h, const float* wav, long long wav_bstride, const int64_t* lengths, float* units, int64_t* frames, int B, int N,
                     void* ws, ns2vc_stream stream);
/* Diagnostics for the parity tests: activations ([B, rows, C] fp32) after each conv of the feature encoder, layer_norm,
 * post_extract_proj, the positional conv's residual sum, encoder.layer_norm, each layer's self_attn_layer_norm and output, and
 * final_proj. */
int ns2vc_cv_num_taps(const ns2vc_cv* h);
int ns2vc_cv_tap_info(const ns2vc_cv* h, int i, const char** name, int* rows, int* channels);
int ns2vc_cv_set_tap(ns2vc_cv* h, int i, float* dst);
int ns2vc_cv_launch_count(const ns2vc_cv* h);   /* kernels launched by the last extract */

/* ------------------------------------------------------------------------------------------------------------------
 * Live conversion: the SOLA (synchronized overlap-add) join of one sliding-window tick, per slot b of B (one CTA each).
 *   seg     [B, Nb + Nc + Ns] fp32 (batch stride seg_bstride floats): the end of the tick's converted window
 *   tail    [B, Nc] fp32 contiguous, in place: the samples kept from the last tick; on return seg[b, k + Nb : k + Nb + Nc]
 *   fade_in [Nc] fp32: the cross-fade's rising half (the caller's table; ns2vc_b200.stream builds sin^2(pi/2 i/(Nc-1)))
 *   out     [B, Nb] fp32 contiguous, offset [B] int32: the emitted block and the chosen k
 * k maximises sum_i seg[k+i] tail[i] / sqrt(sum_i seg[k+i]^2 + 1e-8) over k in [0, Ns] (i < Nc), both sums in fp64 in a fixed
 * order, the lowest k on ties (an all-zero tail gives 0).  out[i] = seg[k+i], cross-faded with tail[i] for i < Nc.
 * Needs Nb >= Nc and (2 Nc + Ns) * 4 bytes <= 47 KB.  Stream-ordered, allocates nothing, capturable. */
int ns2vc_stream_sola(const float* seg, long long seg_bstride, float* tail, const float* fade_in, float* out, int* offset, int B,
                      int Nb, int Nc, int Ns, ns2vc_stream stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Silence slicer: framewise RMS, librosa 0.10 feature.rms(y, frame_length=win, hop_length=hop) with center=True and
 * pad_mode="constant", bit for bit (numpy's pairwise float32 sum of each squared frame, divided by win in float32, IEEE sqrt).
 * Host-only: the frame count 1 + (n + 2 (win/2) - win) / hop of a row of n samples, or -1 for bad arguments (hop or win < 1,
 * a padded length n + 2 (win/2) shorter than win, or a win too long for the kernel's unrolled pairwise sum, about 32768). */
long long ns2vc_slice_rms_frames(long long n, int hop, int win);
/* wav [B, *] fp32 (batch stride wav_bstride floats), lengths [B] int64 device, hop_win [B, 2] int32 device (row b's hop and
 * win, each accepted by ns2vc_slice_rms_frames) -> rms [B, F] fp32 contiguous: frame f of row b, 0 for f at or past that
 * row's frame count.  Samples past lengths[b] are never read.  Stream-ordered, allocates nothing, capturable. */
int ns2vc_slice_rms(const float* wav, long long wav_bstride, const int64_t* lengths, const int* hop_win, float* rms, int F, int B,
                    ns2vc_stream stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Training objective of NaturalSpeech2.forward (model.py:698-734) under no_grad, at K timesteps per batch of B rows.
 * q_sample: x_start = spec * mask, noise_m = noise * mask, x[k] = sqrt_ac[t[k,b]] * x_start + sqrt_1mac[t[k,b]] * noise_m with
 * mask[b, :, f] = (f < lengths[b]) as a 0/1 factor, every product and the sum rounded separately: bit-identical to the
 * reference's torch expression on the device.  Inputs must be finite (a non-finite value past a length gives NaN there, as
 * in the reference).
 *   spec [B, C, T] fp32, lengths [B] int64, t [K, B] int64 (a value outside [0, timesteps) gives NaN), all device
 *   noise [K, B, C, T] (noise_per_k != 0) or one [B, C, T] shared by every k (noise_per_k == 0)
 *   sqrt_alphas_cumprod, sqrt_one_minus_alphas_cumprod [timesteps] fp32 device
 *   x_start [B, C, T], x [K, B, C, T]; noise_masked: NULL, or the shape of noise
 * Stream-ordered, allocates nothing, capturable. */
int ns2vc_q_sample(const float* spec, const float* noise, int noise_per_k, const int64_t* lengths, const int64_t* t,
                   const float* sqrt_alphas_cumprod, const float* sqrt_one_minus_alphas_cumprod, int timesteps, float* x_start,
                   float* noise_masked, float* x, int K, int B, int C, int T, ns2vc_stream stream);
/* Host-only: bytes of the scratch buffer ns2vc_mse_rows needs (its contents on entry do not matter). */
int ns2vc_mse_workspace_bytes(int K, int B, int C, int T, size_t* bytes);
/* loss_row[k, b] = mean over C * T of (out[k, b] - target[b])^2 (padded frames included, as F.mse_loss over the padded row),
 * loss_weighted[k, b] = loss_row * w with w = loss_weight[t[k, b]], clamped to min_snr_gamma when that is > 0,
 * loss[k] = mean_b(w) * mean_b(loss_row[k, b]): the number forward() returns, whose [B, C*T] x [B, 1, 1] product broadcasts over
 * a second batch axis (model.py:723-726); it equals mean_b(loss_weighted) when every row has the same t.  out [K, B, C, T]; target [K, B, C, T] (target_per_k != 0) or [B, C, T];
 * K * B <= 65535.  Sums run in fp64 over a partition and in an order that depend on C * T only, without atomics, so two
 * launches give the same bits; every fp32 output is rounded once from fp64.  ws: 8-byte aligned device scratch.
 * Stream-ordered, allocates nothing, capturable. */
int ns2vc_mse_rows(const float* out, const float* target, int target_per_k, const int64_t* t, const float* loss_weight, int timesteps,
                   float min_snr_gamma, float* loss_row, float* loss_weighted, float* loss, int K, int B, int C, int T, void* ws,
                   ns2vc_stream stream);
/* Host-only: bytes of the scratch buffer ns2vc_mse_rows_ragged needs (its contents on entry do not matter). */
int ns2vc_mse_ragged_workspace_bytes(int K, int B, int C, int T, size_t* bytes);
/* The per-utterance reduction of a ragged batch: loss_row[k, b] = mean over the C * T_b elements of frames f < T_b = lengths[b]
 * of (out[k, b] - target[b])^2, loss_weighted[k, b] = loss_row * w with w as for ns2vc_mse_rows.  out, target as for
 * ns2vc_mse_rows; lengths [B] int64 device (a length outside [1, T] gives NaN in its rows).  Nothing past a row's length is read,
 * so non-finite padding has no effect.  The partition of a row and the order of every addition depend on (C, T_b) only: a row's
 * result has the same bits whatever T, B or position it has (and equals ns2vc_mse_rows on the unpadded row).  No atomics;
 * every fp32 output is rounded once from fp64.  K * B <= 65535.  ws: 8-byte aligned device scratch.
 * Stream-ordered, allocates nothing, capturable. */
int ns2vc_mse_rows_ragged(const float* out, const float* target, int target_per_k, const int64_t* lengths, const int64_t* t,
                          const float* loss_weight, int timesteps, float min_snr_gamma, float* loss_row, float* loss_weighted, int K,
                          int B, int C, int T, void* ws, ns2vc_stream stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Kernel checks (tests only): one weight packing, one wgmma GEMM, one flash attention or one other launch (or short run of
 * launches) through the engines' own host code and launchers, described by flat structs.  Every pointer is device memory; invalid combinations come back as the
 * launchers' error codes.  `desc` (desc_len bytes, may be NULL) receives the kernel and template arguments launched.
 * Stream-ordered (the GEMM allocates and frees its panel-affine descriptor on the stream). */
typedef struct ns2vc_check_split {   /* a bf16 hi/lo split activation [B, T, ld] (16-bit elements), C valid channels */
  const void* hi; const void* lo;
  int T, C, ld;
  long long bpitch;                  /* elements between batch entries; 0: T * ld */
} ns2vc_check_split;
typedef struct ns2vc_check_gemm_args {
  int B, T_out;
  int nsrc; ns2vc_check_split src[4];
  int nseg; int seg[8][4];           /* plain segments: source, first channel, channels, row offset (tap) */
  int nxs; int xseg[4][8];           /* panel segments: source, c0, channels, taps (1 | 3), k-block of tap 0, k-block stride of the
                                        taps, normalise (0 | 1), first channel of the affine table */
  const void* w_hi; const void* w_lo; /* packed weights (ns2vc_check_pack_b), N columns x nkb_w k-blocks */
  int N, n_valid, nkb_w;
  int flags;                         /* EPI_* bits of the GEMM epilogue (csrc/common.cuh) */
  const float* bias; const float* rowbias; int rowbias_ld;
  const float* res; int res_ld;
  float* out; int out_ld;
  void* out_hi; void* out_lo; int out_split_ld;
  int f16_col0;                      /* split columns >= f16_col0 stored as fp16 hi/lo; < 0: none */
  const double* ln_stats; const float* ln_g; int ln_C; float ln_eps;
  double* row_stats; double* stat_sum; double* stat_sq;
  const float* rowmask;
  const int* row_len; int len_shift;
  const float* pre_scale; const float* pre_shift; /* panel mode: the affine [B, pre_C] applied to the normalised segments */
  int pre_mode;                      /* 1: x * scale + shift, 2: then SiLU */
  int pre_C;
  int ksplit;                        /* panel mode: 1 or 2 CTAs per tile */
  /* panel mode without pre_scale: the GroupNorm (mode pre_mode) of gn_C1 + gn_C2 channels in gn_G groups over T_out rows (row_len:
     each entry's own rows) from per-(entry, channel) sums gn_stats1 [2][B][gn_C1] | gn_stats2 [2][B][gn_C2] (sums, then sums of
     squares, as EPI_STATS writes them; NULL: no second source), with FiLM rows gn_film [B, gn_film_ld] (scale | shift) or NULL -
     the descriptor the denoiser builds */
  const double* gn_stats1; const double* gn_stats2; int gn_C1, gn_C2, gn_G; float gn_eps;
  const float* gn_gamma; const float* gn_beta; const float* gn_film; int gn_film_ld;
  int bn, tma_out;                   /* the launch hook's report of the N tile and TMA stores a program chose (ignored by
                                        ns2vc_check_gemm, which plans its own) */
} ns2vc_check_gemm_args;
typedef struct ns2vc_check_attn_args {
  int B, H, Tq, Tk, dh;
  float scale;
  int v2;                            /* 1: the TMA-fed kernel over split q / k / v; 0: the fp32-input tensor-core kernel */
  const float* q; int q_ld; const float* k; int k_ld; const float* v; int v_ld;
  ns2vc_check_split qs, ks, vs;      /* v2; head h of x at channels [x_c0 + h dh, x_c0 + (h + 1) dh) */
  int q_c0, k_c0, v_c0;
  int p_split;
  const int* key_len; int key_shift;
  const float* bias;                 /* additive [B, Tk] or NULL */
  float* out; int out_ld;
  void* out_hi; void* out_lo; int out_split_ld;
  int pb;                            /* the launch hook's report of the v2 box width (ignored by ns2vc_check_attention) */
} ns2vc_check_attn_args;
int ns2vc_check_pack_b(const float* w, int n_rows, int cin_total, int ktaps, int tap, int cin0, int ncin, int n_dst0, int kb0,
                       int geglu_half, const float* cscale, void* w_hi, void* w_lo, int Npad, int nkb_total, ns2vc_stream stream);
int ns2vc_check_gemm(const ns2vc_check_gemm_args* args, char* desc, int desc_len, ns2vc_stream stream);
int ns2vc_check_attention(const ns2vc_check_attn_args* args, char* desc, int desc_len, ns2vc_stream stream);

/* One activation prep (prep_split_kernel): concat(src1, src2) rows remapped -> [affine (+ SiLU)] -> split `out` (+ the untransformed
 * split `raw`).  The affine is either given (scale / shift) or the GroupNorm (+ FiLM) of the sums, as the denoiser builds it. */
typedef struct ns2vc_check_prep_args {
  const float* src1; int ld1, C1;
  const float* src2; int ld2, C2;    /* NULL / 0: no concat */
  int B, T_src, T_dst;
  int row_mul, row_add;              /* source row of output row t: rowmap ? rowmap[t] : t * row_mul + row_add */
  const int* rowmap;                 /* [T_dst] or NULL; with row_len: the nearest-upsample rule of each entry's own lengths */
  int mode;                          /* 0: raw, 1: affine, 2: affine then SiLU */
  const float* scale; const float* shift; /* [B, C1 + C2], or NULL: GroupNorm from stats1 / stats2 */
  const double* stats1; const double* stats2; /* [2][B][C1] / [2][B][C2]: sums, then sums of squares, over T_src rows */
  const float* gamma; const float* beta; int G; float eps;
  const float* film; int film_ld;    /* [B, film_ld]: scale at [b, c], shift at [b, C1 + C2 + c]; or NULL */
  ns2vc_check_split out, raw;        /* raw.hi NULL: no raw output */
  const int* row_len; int len_shift; /* ragged: level-0 lengths [B] or NULL */
} ns2vc_check_prep_args;
int ns2vc_check_prep(const ns2vc_check_prep_args* args, char* desc, int desc_len, ns2vc_stream stream);

/* One LayerNorm launch of M rows of C channels (pitch ld): kind 0 ln_split (into `split`; keep: rows whose factor is 0 are stored
 * as zeros, or NULL), 1 ln_apply (into y), 2 ln_mask (into y, times keep). */
typedef struct ns2vc_check_ln_args {
  int kind;
  const float* x; int ld, M, C; float eps;
  const float* gamma; const float* beta;
  const float* keep;
  float* y; int y_ld;
  ns2vc_check_split split;
} ns2vc_check_ln_args;
int ns2vc_check_ln(const ns2vc_check_ln_args* args, char* desc, int desc_len, ns2vc_stream stream);

/* One voc_norm_kernel launch: LayerNorm of token-major [B, T, C] rows, after the 7-tap depthwise conv dw ([C][8]: taps, bias) or
 * not (NULL), rows at or past len[b] (int64, or NULL) zero; into out and / or split. */
typedef struct ns2vc_check_voc_norm_args {
  const float* x; int B, T, C;
  const float* dw; const float* gamma; const float* beta; float eps;
  const int64_t* len;
  float* out; ns2vc_check_split split;
} ns2vc_check_voc_norm_args;
int ns2vc_check_voc_norm(const ns2vc_check_voc_norm_args* args, char* desc, int desc_len, ns2vc_stream stream);

/* One small linear: out[m, n] = f(x[m, :]) . W[n, :] + bias[n] (+ add[m % add_rows (add_rows > 0) or m, n]) (then SiLU);
 * in_mode 0: x, 1: SiLU(x), 2: the K-wide sinusoid of t = x[m * x_ld]. */
typedef struct ns2vc_check_linear_args {
  const float* x; int x_ld, M, K;
  const float* W; const float* bias; int N;
  const float* add; int add_ld, add_rows;
  float* out; int out_ld;
  int in_mode, flip_sin_to_cos; float freq_shift; int out_silu;
} ns2vc_check_linear_args;
int ns2vc_check_small_linear(const ns2vc_check_linear_args* args, char* desc, int desc_len, ns2vc_stream stream);

/* AttentionPooling pieces: with `tokens`, the class token (mean of x's first lens[b] or S rows + pos) and the copied rows; with
 * `out`, the attention of q [B, C] over kv [B, S + 1, 2C] (k | v) in `heads` heads (wide: the any-width kernel). */
typedef struct ns2vc_check_pool_args {
  const float* x; const float* pos; int B, S, C;
  float* tokens;
  const float* q; const float* kv; int heads, wide;
  float* out;
  const int* lens;
} ns2vc_check_pool_args;
int ns2vc_check_pool(const ns2vc_check_pool_args* args, char* desc, int desc_len, ns2vc_stream stream);

/* [B, C, T] fp32 (batch stride bstride) -> split token-major [B, T, out.ld]; frames past row_len[b] (or NULL) are zeros. */
typedef struct ns2vc_check_nct_split_args {
  const float* x; long long bstride; int B, C, T;
  ns2vc_check_split out;
  const int* row_len;
} ns2vc_check_nct_split_args;
int ns2vc_check_nct_split(const ns2vc_check_nct_split_args* args, char* desc, int desc_len, ns2vc_stream stream);

/* The content encoder's first conv: the GroupNorm statistics launch (stats [B, C0] of (mean, 1 / std) float pairs over each row's
 * own frames), then the conv 0 launch into the split `out` [B, rows, out.ld] (out.C = C0); wav [B, bstride], lengths int64 [B]
 * (clamped into [400, N]) or NULL. */
typedef struct ns2vc_check_cv_conv0_args {
  const float* wav; long long bstride; const int64_t* lengths; int B, N, C0;
  const float* w0; const float* gamma; const float* beta; float eps;   /* w0 [C0, 1, 10]; the GroupNorm's weights [C0] */
  float* stats;
  ns2vc_check_split out; int rows;
} ns2vc_check_cv_conv0_args;
int ns2vc_check_cv_conv0(const ns2vc_check_cv_conv0_args* args, char* desc, int desc_len, ns2vc_stream stream);

/* The content encoder's positional conv out = x + GELU(SamePad(conv(x))) over x [B, T, D] with frames[b] (int64) valid rows:
 * the window launch into win_hi / win_lo ([B, G, T + K, 1024] bf16 each), then (windows_only = 0) one GEMM per group over the
 * folded weight w [D, D / G, K] packed as the engine packs it, with bias [D] and the row mask keep [B, T], then the residual add. */
typedef struct ns2vc_check_cv_pos_conv_args {
  const float* x; int B, T, D, G, K;
  const int64_t* frames;
  const float* w; const float* bias; const float* keep;
  void* win_hi; void* win_lo;
  float* out;
  int windows_only;
} ns2vc_check_cv_pos_conv_args;
int ns2vc_check_cv_pos_conv(const ns2vc_check_cv_pos_conv_args* args, char* desc, int desc_len, ns2vc_stream stream);

/* The denoiser's Downsample1D (conv k3 s2 p1 + bias) of x [B, Tin, C] as the engine launches it: one GEMM over row-pair views of
 * the raw split (in_hi / in_lo [B, Tin, ld], ld a multiple of 8 >= C), or (force_prep, or Tin = 1) two prep launches decimating
 * the fp32 x into dense even / odd splits first.  w [C, C, 3] is packed as the engine packs it.  Outputs [B, ceil(Tin / 2), C]:
 * fp32 `out` and / or the split out_hi / out_lo (row pitch pad_to(C, 8)); ragged: level-0 lengths row_len [B] (int32) and the
 * output level len_shift >= 1 (rows past each entry's own length are zeros), or NULL. */
typedef struct ns2vc_check_down_conv_args {
  int B, Tin, C;
  const float* x;
  const void* in_hi; const void* in_lo; int ld;
  const float* w; const float* bias;
  const int* row_len; int len_shift;
  float* out;
  void* out_hi; void* out_lo;
  int force_prep;
} ns2vc_check_down_conv_args;
int ns2vc_check_down_conv(const ns2vc_check_down_conv_args* args, char* desc, int desc_len, ns2vc_stream stream);

/* The content encoder's conv l (1 .. 6: k 3, or 2 for l >= 5; stride 2, no bias) + GELU as the engine launches it: one GEMM over
 * the row-pair view of the previous level's split in_hi / in_lo [B, rows_in, C0] (rows_in even), the row mask keep [B, rows_out],
 * into the split out_hi / out_lo or the fp32 out ([B, rows_out, C0], exactly one of them).  w [C0, C0, k] is packed as the
 * engine packs it; C0 a multiple of 128 up to 1024. */
typedef struct ns2vc_check_cv_conv_args {
  int B, rows_in, rows_out, C0, l;
  const void* in_hi; const void* in_lo;
  const float* w; const float* keep;
  float* out;
  void* out_hi; void* out_lo;
} ns2vc_check_cv_conv_args;
int ns2vc_check_cv_conv(const ns2vc_check_cv_conv_args* args, char* desc, int desc_len, ns2vc_stream stream);

/* The vocoder's ISTFT of a head output h [B, T, ld] (log-magnitudes, then phases; ld >= n_fft + 2) with window [n_fft] and
 * hop n_fft / 4 into audio [B, T * hop]; len int64 [B] (clamped into [1, T]) or NULL.  The twiddles are the engine's. */
typedef struct ns2vc_check_istft_args {
  const float* h; int ld; const int64_t* len; int B, T, n_fft;
  const float* window;
  float* audio;
} ns2vc_check_istft_args;
int ns2vc_check_istft(const ns2vc_check_istft_args* args, char* desc, int desc_len, ns2vc_stream stream);

/* The packed-weight record: the operands engine `kind` (0 denoiser ns2vc_unet, 1 condition encoders ns2vc_pre, 2 content encoder
 * ns2vc_cv, 3 vocoder ns2vc_voc) built at its last finalize, in packing order, each with its site name and the load-time vectors
 * (folded LayerNorm vectors, merged biases and operators, concatenations) read beside it.  Errors: another kind, a null handle,
 * weights not packed since the last load, an index out of range, a name buffer shorter than the name and its NUL.
 * _count returns the number of operands (-1 on error).  _packed: name (or NULL), the packed image's Npad columns (0: an entry of
 * vectors only), nkb k-blocks and n_logical columns, nvec vectors; hi_out / lo_out (device, nkb * Npad * 64 bf16 each, or NULL)
 * receive the swizzled hi / lo images.  _fold_vector: vector j of operand i, its name (or NULL), length n and (out: device
 * fp32 [n], or NULL) values.  Stream-ordered copies. */
int ns2vc_check_packed_count(int kind, const void* handle);
int ns2vc_check_packed(int kind, const void* handle, int i, char* name, int name_len, int* Npad, int* nkb, int* n_logical, int* nvec,
                       void* hi_out, void* lo_out, ns2vc_stream stream);
int ns2vc_check_fold_vector(int kind, const void* handle, int i, int j, char* name, int name_len, long long* n, float* out,
                            ns2vc_stream stream);

/* The launch observer of engine `kind` (numbered as for ns2vc_check_packed): while set, every run of the handle's programs
 * calls fn(user, index, phase, launch_kind, gemm, attn, desc) before (phase 0) and after (phase 1) each launch, with the stream
 * synchronised, index the launch's position in its program and launch_kind its kind (ns2vc_unet_launch_kind numbering).  For a
 * GEMM, `gemm` describes the launch as bound to the call's arguments (plain or panel segments; a panel GroupNorm as gn_*), for
 * an attention `attn`; the other is NULL, and both are NULL for the other kinds.  desc: the kernel and template arguments, as
 * ns2vc_check_gemm / ns2vc_check_attention report them ("" for the other kinds).  A nonzero return from fn ends the run with an
 * error.  fn NULL removes the observer.  A run on a capturing stream fails while an observer is set.  Errors: another kind, a
 * null handle. */
typedef int (*ns2vc_check_launch_fn)(void* user, int index, int phase, int launch_kind, const ns2vc_check_gemm_args* gemm,
                                     const ns2vc_check_attn_args* attn, const char* desc);
int ns2vc_check_set_launch_hook(int kind, void* handle, ns2vc_check_launch_fn fn, void* user);

/* The sampler noise's generator (ns2vc_noise_normal_rows): for each of n entries, raw [n, 4] = Philox4x32-10 of counters [n, 4]
 * under keys [n, 2] (key lo, hi), and normals [n, 4] = the Box-Muller pair (z0, z1) of outputs (x, y), then of (z, w). */
int ns2vc_check_philox(const uint32_t* counters, const uint32_t* keys, int n, uint32_t* raw, float* normals, ns2vc_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* NS2VC_B200_H */
