// Shared declarations for the ns2vc_b200 denoiser engine (sm_90a only).
//
// Internal activation layout: TOKEN-MAJOR fp32 [B, T_l, C] ("rows" = B*T_l tokens, channels
// contiguous).  The reference keeps [B, C, T] and permutes around every transformer block
// (reference unet1d/transformer_1d.py:264, 289); here the convs are implicit GEMMs over
// token rows (tap j of a k=3 conv is the same matrix shifted by j-1 rows), so no permute exists.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stddef.h>

namespace ns2vc {

// ---------------------------------------------------------------------------------------------
// Error handling: C-ABI returns negative codes; the message is kept per thread.
// ---------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
const char* get_error();

#define NS_CHECK_CUDA(expr)                                                                    \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      ns2vc::set_error("%s:%d CUDA error %s: %s", __FILE__, __LINE__, cudaGetErrorName(_e),    \
                       cudaGetErrorString(_e));                                                \
      return -2;                                                                               \
    }                                                                                          \
  } while (0)

#define NS_REQUIRE(cond, ...)                                                                  \
  do {                                                                                         \
    if (!(cond)) {                                                                             \
      ns2vc::set_error(__VA_ARGS__);                                                           \
      return -1;                                                                               \
    }                                                                                          \
  } while (0)

// ---------------------------------------------------------------------------------------------
// "Split" activations: every GEMM A operand is stored as two bf16 tensors hi = bf16(x),
// lo = bf16(x - hi), token-major [B, T, ld].  They are written ONCE by the op that produces or
// normalises the activation (prep kernels below, or a GEMM/attention epilogue) and then read by
// TMA straight into the swizzled shared-memory image wgmma wants — for every conv tap and
// every N tile — instead of re-running GroupNorm/SiLU in the GEMM's load path.
// ---------------------------------------------------------------------------------------------
struct SplitBuf {
  __nv_bfloat16* hi;
  __nv_bfloat16* lo;
  int T;              // rows per batch entry
  int C;              // valid channels
  int ld;             // row pitch in elements (multiple of 8)
  long long bpitch;   // elements between batch entries; 0 = T * ld (dense).  Views over row PAIRS of a tensor with an odd
                      // number of rows (the stride-2 conv's even / odd rows) need their own value
};

struct alignas(128) TMap { unsigned long long v[16]; };   // CUtensorMap storage (driver-encoded)

// ---------------------------------------------------------------------------------------------
// Activation prep: (concat of up to two fp32 sources) -> [GroupNorm affine (+FiLM) (+SiLU)] -> split
// ---------------------------------------------------------------------------------------------
enum PrepMode : int { PREP_RAW = 0, PREP_AFFINE = 1, PREP_AFFINE_SILU = 2 };
// GroupNorm source statistics: per-(b, channel) sums accumulated by the producing GEMM epilogues.
struct GnStats {
  const double* sum1; const double* sq1;   // [B, C1]
  const double* sum2; const double* sq2;   // [B, C2]
  const float* gamma; const float* beta;   // [C1+C2]
  const float* film; int film_ld;          // nullptr or [B, film_ld]: scale at film[b,c], shift at film[b,C+c]
  int G; float eps;
  double inv_n;                            // 1 / (T * C/G): elements per group, reciprocal taken on the host (0: derive it on the device)
};
struct alignas(16) PrepOp {      // (16-byte multiples: arrays of descriptors are copied with 128-bit loads)
  const float* src1; int ld1; int C1;
  const float* src2; int ld2; int C2;     // nullptr / 0 when there is no concat
  int B, T_src, T_dst;
  int row_mul, row_add;                   // src row = rowmap ? rowmap[t] : t*row_mul + row_add
  const int* rowmap;                      // nearest-upsample index table [T_dst] or nullptr
  int mode;
  const float* scale; const float* shift; // [B, C1+C2] precomputed affine, or nullptr: derive it from `gn`
  GnStats gn;
  SplitBuf out;                           // transformed
  SplitBuf raw;                           // optional second output without the transform (hi == nullptr: none)
  unsigned long long* span;               // diagnostics
  // ragged programs: per-utterance lengths [B] at level 0 (nullptr: every row of T_dst is valid).  Output rows
  // t >= ((row_len[b] - 1) >> len_shift) + 1 are written as zeros and the GroupNorm statistics count only the valid rows; a
  // nearest upsample (rowmap set) derives each entry's source rows from its own lengths at levels len_shift + 1 and len_shift.
  const int* row_len; int len_shift;
};

// GEMM / implicit-conv operator (shared by the wgmma kernel and the SIMT debug kernel):
//
//   out[b, t, n] = epilogue( sum_seg sum_{c < 64*nkb} A_seg[b, t + tap, c0 + c] * W[kofs_seg + c, n] )
//
// A_seg rows outside [0, src.T) and channels >= src.C read as zero (TMA out-of-bounds fill), which
// is exactly a conv's zero padding of the already-normalised activations (reference resnet.py:597-612).
// Strided (downsample) and nearest-upsample convs get their row mapping from the prep kernel, so
// every segment here is a unit-stride window.
constexpr int kMaxSrc = 4;
constexpr int kMaxSeg = 8;

struct GSeg {
  int src;            // index into GemmOp::src
  int c0;             // first channel
  int nkb;            // 64-wide k-blocks
  int tap;            // row offset
};

enum EpiFlags : int {
  EPI_BIAS = 1,       // + bias[n]
  EPI_RESIDUAL = 2,   // + res[m*res_ld + n]
  EPI_GEGLU = 4,      // packed N pairs 64 value | 64 gate columns: out = (v+bv) * gelu_erf(g+bg)
  EPI_OUT_NCT = 8,    // store fp32 out[b, n, t] (channel-major, n < n_valid)
  EPI_ROWBIAS = 16,   // + rowbias[b*rowbias_ld + n]   (per-sample bias, time_embedding 'default')
  EPI_OUT_F32 = 32,   // store fp32 token-major out[m*out_ld + n]
  EPI_OUT_SPLIT = 64, // store bf16 hi/lo token-major (feeds the next GEMM's TMA)
  EPI_STATS = 128,    // accumulate per-(b, column) sum / sum-of-squares of the fp32 output (GroupNorm of the consumer)
  EPI_LNFOLD = 256,   // the A operand is the RAW input of a LayerNorm whose gamma is folded into the weights:
                      //   acc <- rstd_row * (acc - mean_row * ln_g[n]);  bias then carries beta.W + bias   (see engine.cu)
  EPI_ROWSTATS = 512, // accumulate per-row sum / sum-of-squares of the fp32 output (LayerNorm statistics for the consumer)
  // condition encoders (pre_engine.cu; the ENC instantiation of the wgmma kernel):
  EPI_RELU = 1024,    // max(v, 0) after bias / residual              (conv-FFN, reference operations.py:689)
  EPI_ROWMASK = 2048, // v *= rowmask[m] after everything else         (x * (1 - padding_mask), reference operations.py:813, 820)
                      //   (VOC instantiation: rows whose rowmask is 0 are stored as exact zeros)
  // vocoder (vocoder.cu) and content encoder (content.cu; the VOC instantiation of the wgmma kernel):
  EPI_GELU = 4096,    // gelu_erf(v) after bias / residual             (ConvNeXtBlock pwconv1 -> act, vocos/modules.py)
};

// One panel segment of a panel-mode GEMM: `ncb` 64-channel blocks of one raw split source
constexpr int kMaxXSeg = 4;
struct XSeg {
  int src;            // index into GemmOp::src
  int c0;             // first channel within the source (multiple of 64)
  int ncb;            // 64-channel blocks
  int ntap;           // 3: k=3 conv (panel rows t0-1 .. t0+128), 1: 1x1 operand (rows t0 .. t0+127)
  int kb_tap[3];      // packed-weight k-block of tap j for channel block 0 (block cb: + cb)
  int xf;             // 1: normalise the panel in shared memory, 0: raw operand (1x1 shortcut)
  int aff_c0;         // channel of the affine table that corresponds to c0
};

struct GemmOp {
  SplitBuf src[kMaxSrc];
  int nsrc;
  GSeg seg[kMaxSeg];
  int nseg;
  int nkb_total;
  int B, T_out;
  // B operand
  const __nv_bfloat16* w_hi;   // packed [kb][Npad][64] (128B-swizzled rows)
  const __nv_bfloat16* w_lo;
  const float* w_f32;          // debug SIMT backend: [K_pad][Npad] fp32 (nullptr unless enabled)
  int N;                       // packed output columns (multiple of 128)
  // epilogue
  int flags;
  const float* bias;           // [N] (GEGLU: [2*N_out] in the reference's value|gate order)
  const float* rowbias;
  int rowbias_ld;
  const float* res;
  int res_ld;
  float* out;
  int out_ld;
  __nv_bfloat16* out_hi;       // EPI_OUT_SPLIT
  __nv_bfloat16* out_lo;
  int out_split_ld;
  int n_valid;                 // logical output columns written (<= N, or N/2 for GEGLU)
  const double* ln_stats;      // EPI_LNFOLD: [B*T_out][2] row sum / sum of squares of the LayerNorm input (over ln_C channels)
  const float* ln_g;           // EPI_LNFOLD: [n logical] sum_c gamma_c W[n, c]  (GEGLU: value rows then gate rows, like bias)
  int ln_C; float ln_eps;
  double* row_stats;           // EPI_ROWSTATS: [B*T_out][2], pre-zeroed
  int f16_col0;                // split output columns >= f16_col0 (a multiple of 32) are written as FP16 hi/lo instead of bf16
  double* stat_sum;            // EPI_STATS: [B, n_valid] each, pre-zeroed
  double* stat_sq;
  unsigned long long* trace;   // diagnostics: 8 globaltimer stamps of CTA (0,0), or nullptr
  unsigned long long* span;    // diagnostics: [min entry, max exit] of the grid, or nullptr
  int tma_out;                 // bit 0: fp32 output goes through tmap_out[0]; bit 1: split output through tmap_out[1..2]
  int bn;                      // N tile (64 / 128), chosen by plan_gemm()
  // Panel mode (xmode = 1): the GroupNorm(+FiLM)(+SiLU) of the A operand is applied INSIDE this kernel (reference
  // resnet.py:597-612, transformer_1d.py:256-262).  The A sources are the RAW bf16 hi/lo splits the producers' epilogues wrote.
  // Per 64-channel block the TMA unit drops ONE panel of 130 rows (t0-1 .. t0+128; 128 rows for a 1x1 operand) of each split
  // into shared memory; the eight epilogue warps (idle during the main loop: one tile per CTA) normalise the panel in place
  // (x = hi + lo, y = silu(x * scale[b,c] + shift[b,c]), re-split; rows outside [0, T) stay zero = the conv's zero padding);
  // the three taps of a k=3 conv are three row-shifted views of the same panel (descriptor start address + 128 B per row:
  // the 128B swizzle is a function of the shared-memory address bits), so a conv reads and normalises each activation once.
  int xmode;
  int ksplit;                  // 1, or 2: the channel blocks are divided between the two CTAs of a cluster (few-tile, deep-K launches);
                               // the second CTA ships its fp32 partial tile into the first one's shared memory, which runs the epilogue
  int nxs;
  XSeg xs[kMaxXSeg];
  const PrepOp* pre;           // GroupNorm parameters of the normalised segments (device memory; only the affine part is used)
  const float* pre_film;       // FiLM rows read by that affine (nullptr: none) - kept here because they change per forward
  const float* rowmask;        // EPI_ROWMASK: [B*T_out] keep factor (1 = frame inside the utterance, 0 = padding)
  // Ragged programs (the RAG instantiation): per-utterance lengths [B] at level 0, or nullptr.  Rows t >= ((row_len[b] - 1) >>
  // len_shift) + 1 of the output are stored as exact zeros, and panel-mode rows past that length read as the conv's zero padding.
  const int* row_len;
  int len_shift;
  // ---- tensor maps last: the TMA unit reads them by address (kernel-parameter space); the kernel copies only the fields
  // ---- before them into shared memory (kGemmOpHotBytes)
  TMap tmap[2 * kMaxSrc];      // [2*i] = hi, [2*i+1] = lo of src[i]; box = {64 ch, 128 rows, 1} (130 rows for a panel-mode k=3 source)
  TMap tmap_out[3];            // TMA store maps: fp32 out (box 32 cols x 32 rows, SWIZZLE_128B), out_hi, out_lo (SWIZZLE_64B)
};
// Choose the N tile for op (fills op.bn); must precede encode_tmaps().
void plan_gemm(GemmOp& op);
constexpr int kXfMaxC = 1024;         // channels a panel-mode GEMM may normalise (affine slots per thread x the 256 transform threads)
int gemm_sm_count();

// Launchers (each returns 0 or a negative error code; all stream-ordered, no host sync).
int launch_gemm_tc(const GemmOp& op, cudaStream_t st);
int launch_gemm_simt(const GemmOp& op, cudaStream_t st);
// Encode the TMA descriptors of op.src[] into op.tmap[] (host; needs a CUDA context).
int encode_tmaps(GemmOp& op);

// Weight packing (device side, load time).  Source W is the reference parameter layout
// [n_rows, cin_total, ktaps] fp32 (ktaps = 1 for nn.Linear / 1x1 conv).
struct PackSeg {
  const float* w;     // device pointer
  int n_rows;         // rows of w used (output channels from this tensor)
  int cin_total;
  int ktaps;
  int tap;            // which tap (0..ktaps-1)
  int cin0, ncin;     // channel range of w's input axis covered by this segment
  int n_dst0;         // first packed column
  int kb0;            // first k-block in the packed K order
  int nkb;
  int geglu_half;     // 0: plain. >0: interleave value/gate (value rows [0,half), gate rows [half,2*half))
  const float* cscale; // optional per-input-channel multiplier [cin_total] (LayerNorm gamma folded into the weights), or nullptr
};
int launch_pack_b(const PackSeg& ps, __nv_bfloat16* w_hi, __nv_bfloat16* w_lo, float* w_f32, int Npad,
                  cudaStream_t st);
// g[n] = sum_c gamma_c W[n, c], bf[n] = sum_c beta_c W[n, c] (+ bias[n]) of a [N, C] linear that consumes LayerNorm(gamma, beta)
// (EPI_LNFOLD; load time, pre_kernels.cu)
int launch_ln_fold_vec(const float* W, const float* gamma, const float* beta, const float* bias, float* g, float* bf, int N, int C, cudaStream_t st);

int launch_prep_split(const PrepOp& op, cudaStream_t st);

// LayerNorm (eps) of M rows of C channels (row pitch ld), one warp per row
struct LnOp {
  const float* x; int ld, M, C; float eps;
  const float* gamma; const float* beta;
  const float* keep;           // [M] row keep factors or nullptr: ln_split stores zeros where keep == 0, ln_mask multiplies by keep
  float* y; int y_ld;          // ln_apply / ln_mask: fp32 output
  SplitBuf split;              // ln_split: bf16 hi/lo output
};
// LayerNorm + split in one pass: split = ((x-mean)*rstd*gamma + beta) as bf16 hi/lo
int launch_ln_split(const LnOp& op, cudaStream_t st);

// ---------------------------------------------------------------------------------------------
// Attention
// ---------------------------------------------------------------------------------------------
struct AttnOp {
  const float* q; int q_ld;       // [B, Tq, q_ld], head h at column h*dh
  const float* k; int k_ld;       // [B, Tk, k_ld]
  const float* v; int v_ld;
  const float* bias;              // additive [B, Tk] or nullptr      (reference: 0 / -10000)
  float* out; int out_ld;         // [B, Tq, out_ld] fp32 (may be nullptr when out_hi is set)
  __nv_bfloat16* out_hi;          // optional split output (feeds the out-projection GEMM)
  __nv_bfloat16* out_lo;
  int out_split_ld;
  int B, H, Tq, Tk, dh;
  float scale;                    // dh^-0.5
  unsigned long long* span;       // diagnostics
  unsigned long long* trace;      // diagnostics (v2): per-tile clock64 stamps of CTA (0,0,0): [16 tiles][16 slots]
  // v2 (TMA-fed, attention_v2.cu): q / k / v as split activations written by the projection GEMMs' epilogues.
  // Head h of tensor x lives at columns [x_c0 + h*dh, x_c0 + (h+1)*dh) of its split buffer.
  SplitBuf qs, ks, vs;
  int q_c0, k_c0, v_c0;
  int v2;                         // 1: launch the v2 kernel (needs dh % 16 == 0 and encode_attn_tmaps())
  int pb;                         // byte width of the Q/K/V TMA boxes = shared-memory row pitch (32 / 64 / 128)
  const int* key_len;             // v2, the denoiser's ragged programs: per-entry lengths [B] at level 0 (nullptr: Tk keys).  Entry b attends
  int key_shift;                  // over its first ((key_len[b] - 1) >> key_shift) + 1 keys only; later key tiles are not even loaded
  int p_split;                    // 1: softmax weights as a bf16 hi/lo split whatever NS2VC_ATTN_P says (V must then be a bf16 split too).  The
                                  // condition encoders attend over a few dozen keys: the 2^-12 rounding of fp16 weights does not average out there
  TMap tm[6];                     // q hi, q lo (box pb x 128 rows), k hi, k lo, v hi, v lo (box pb x 64 rows)
};
int launch_attention(const AttnOp& op, cudaStream_t st, bool simt_debug);
int launch_attention_v2(const AttnOp& op, cudaStream_t st);
// Can the v2 kernel run this shape?  (head dim 16/32/48/64; a biased key row must fit the staged-bias buffer)
bool attention_v2_supported(int dh, int Tk, bool biased);
// v2 softmax weights as fp16 (then V must be an fp16 hi/lo split) or as a bf16 hi/lo split (NS2VC_ATTN_P=split)
bool attention_v2_p_fp16();
// Host: pick the box width and encode op.tm[] (needs a CUDA context).
int encode_attn_tmaps(AttnOp& op);
// Generic 3-D tiled bf16 tensor map over a token-major [B, T, ld] buffer with C valid channels.
int encode_tmap_rows(TMap* out, const __nv_bfloat16* base, int C, int T, int B, int ld, int box_c, int box_rows, int swizzle_bytes);
// Same for fp32 data (elem_bytes = 4) / bf16 (elem_bytes = 2)
int encode_tmap_any(TMap* out, const void* base, int elem_bytes, int C, int T, int B, int ld, int box_c, int box_rows, int swizzle_bytes,
                    long long bpitch = 0);

// ---------------------------------------------------------------------------------------------
// Norm statistics and small kernels (kernels_misc.cu)
// ---------------------------------------------------------------------------------------------
// y = (x-mean)*rstd*gamma + beta
int launch_ln_apply(const LnOp& op, cudaStream_t st);

// [B, C, T] fp32 (batch stride bstride) -> token-major fp32 [B, T, ld], channels >= C zero-filled up to ld
struct TokensOp {
  const float* x; long long bstride; int B, C, T;
  float* out; int ld;
  const float* rowbias;        // enc_input: + rowbias[b, c], or nullptr
  const float* keep;           // enc_input: [B, T] rows with keep == 0 are stored as zeros
};
int launch_nct_to_tokens(const TokensOp& op, cudaStream_t st);
// [B, C, T] fp32 -> split token-major [B, T, out.ld] (channels >= C zero-filled up to out.ld)
struct NctSplitOp {
  const float* x; long long bstride; int B, C, T;
  SplitBuf out;
  const int* row_len;          // per-entry valid frames [B] (ragged programs): frames past them are written as zeros; or nullptr
  const void* warm; long long warm_bytes;   // optional region prefetched into L2 by the same launch (the step's FiLM rows)
};
int launch_nct_to_split(const NctSplitOp& op, cudaStream_t st);

enum LinIn : int { LIN_RAW = 0, LIN_SILU = 1, LIN_SINUSOID = 2 };
// Small-M linear: out[m, n] = f(x[m, :]) . W[n, :] + bias[n] (+ add[m, n]);  W row-major [N, K].
// LIN_SINUSOID: x is t[m] and the input row is the K-wide sinusoidal embedding
// (reference embeddings.py:24-64, flip_sin_to_cos / freq_shift as given).
struct LinOp {
  const float* x; int x_ld; int M; int K;
  const float* W; const float* bias; int N;
  const float* add; int add_ld;
  int add_rows;                // > 0: row m reads add row (m % add_rows)  (the timestep table: rows = steps x batch entries)
  float* out; int out_ld;
  int in_mode; int flip_sin_to_cos; float freq_shift;
  int out_silu;
};
int launch_small_linear(const LinOp& op, cudaStream_t st);

// AttentionPooling pieces (reference embeddings.py:499-546)
// lens: per-entry prompt lengths [B] (ragged programs: pool over the first lens[b] frames only), or nullptr (all S)
struct PoolClsOp {
  const float* x; const float* pos; int B, S, C;   // x: [B, S, C] LayerNorm'd, pos: [C]
  float* tokens;                                   // [B, S+1, C]: row 0 = class token, rows 1.. = x
  const int* lens;
};
int launch_pool_class_token(const PoolClsOp& op, cudaStream_t st);
// POOL_ATT (launch_pool_attend: head width <= 16) and POOL_ATT_WIDE (launch_pool_attend_wide: any head width)
struct PoolAttOp {
  const float* q; const float* kv; int B, S1, C, heads;   // q: [B, C], kv: [B, S1, 2C] k | v
  float* out;                                             // [B, C]
  const int* lens;
};
int launch_pool_attend(const PoolAttOp& op, cudaStream_t st);
struct MaskBiasOp { const uint8_t* mask; int n; float* bias; };
int launch_mask_bias(const MaskBiasOp& op, cudaStream_t st);

// Ragged programs: per-utterance lengths -> the device tables the program reads (written by ns2vc_unet_prepare_cond_ragged).
constexpr int kRagMaxLevels = 8;
struct RaggedTables {
  int B, T, S, nlev;
  int* lens;                          // [2B]: content lengths | prompt lengths, clamped to [1, T] / [1, S]
  float* prompt_bias;                 // [B, S]: 0 / -inf key bias of the cross-attention
  float* key_bias[kRagMaxLevels];     // [B, Tl] 0 / -inf key bias of the self-attention at level l (nullptr: no transformer there)
  int Tl[kRagMaxLevels];
};
// Entries [b0, b0 + n) (n = 0: all B); the lengths are read at the same entries.
int launch_ragged_tables(const long long* content_lengths, const long long* prompt_lengths, const RaggedTables& r, cudaStream_t st,
                         int b0 = 0, int n = 0);

// ---------------------------------------------------------------------------------------------
// Condition encoders (pre_kernels.cu; program in pre_engine.cu)
// ---------------------------------------------------------------------------------------------
struct SeqMaskOp {
  const long long* len; int B, T;
  float* keep; float* kbias;   // [B, T]
  int* ilen;                   // the lengths as int [B], clamped to [1, T], or nullptr
};
int launch_seq_mask(const SeqMaskOp& op, cudaStream_t st);
int launch_enc_input(const TokensOp& op, cudaStream_t st);
// y = LayerNorm(x) * keep
int launch_ln_mask(const LnOp& op, cudaStream_t st);
int launch_pool_attend_wide(const PoolAttOp& op, cudaStream_t st);
int launch_tbc_weight(const float* w, int k, int cin, int cout, float* o, cudaStream_t st);
int launch_ffn_taps(const float* const* w, int k, int F, int H, int centre, float scale, float* o, cudaStream_t st);
int launch_scale_vec(const float* a, float s, float* o, int n, cudaStream_t st);

// LayerNorm (eps) of token-major [B, T, C] rows (vocoder.cu's voc_norm_kernel; C a multiple of 128 up to 1024), optionally after
// a 7-tap depthwise conv (dw: [C][8] taps and bias).  Rows at or past len[b] (int64 [B], clamped into [1, T]; nullptr: T) read
// and store 0.  Outputs: fp32 `out` and / or the bf16 hi/lo `split`.
struct VocNormOp {
  const float* x; int B, T, C;
  const float* dw; const float* gamma; const float* beta; float eps;
  const long long* len;
  float* out; SplitBuf split;
};
int launch_voc_norm(const VocNormOp& op, cudaStream_t st);

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// Source row of output row i of F.interpolate(size=t_out, mode='nearest') from t_in rows: ATen nearest_idx (UpSample.h), with
// IEEE fp32 division / product / floor as ns2vc_nearest_index() on the host.  In fp32 this is NOT always i >> 1 when t_out is
// 2 t_in - 1 (e.g. t_in = 2095, t_out = 4189, i = 4187 -> 2094): a table depends on both lengths.
__device__ __forceinline__ int nearest_src_index(int i, int t_in, int t_out) {
  if (t_out == t_in) return i;
  if (t_out == 2 * t_in) return i >> 1;
  const float scale = __fdiv_rn((float)t_in, (float)t_out);
  return min((int)floorf(__fmul_rn((float)i, scale)), t_in - 1);
}

}  // namespace ns2vc
