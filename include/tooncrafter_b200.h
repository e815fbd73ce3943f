/* tooncrafter_b200 — C ABI of the H100-native DDIM/UNet/VAE-decoder hot path.
 *
 * The reference (Doubiiu/ToonCrafter) has no FFI: its "plugin" seam is Python-object instantiation
 * (utils/utils.py:27-34) and every kernel is a torch library call.  This header is therefore the
 * boundary: the entry points our Python mirror of lvdm.* calls instead of
 * torch.nn.functional.  Each entry cites the reference call site(s) it replaces.
 *
 * Conventions
 *   - plain C, raw device pointers, caller owns all memory (no allocation, no sync inside);
 *   - every function enqueues on `stream` (a cudaStream_t passed as void*), is CUDA-graph-capturable;
 *   - returns 0 on success, negative on error; tc_last_error() gives a thread-local message;
 *   - activations are fp16 ("half") channels-last: a video tensor is [B][T][H][W][C]; "frames" N = B*T;
 *   - single host thread per process (same as the reference: gradio_app.py:81 max_threads=1).
 */
#ifndef TOONCRAFTER_B200_H
#define TOONCRAFTER_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TC_OK 0
#define TC_ERR_INVALID (-1)
#define TC_ERR_CUDA (-2)
#define TC_ERR_UNSUPPORTED (-3)

#define TC_MAX_TAPS 9
#define TC_GN_MAX_PARTIALS 296 /* GroupNorm statistics blocks per stat group (workspace sizing) */
#define TC_DDIM_PARTIALS 64     /* DDIM-step reduction blocks per sample (workspace sizing) */

/* epilogue flags of tc_conv_gemm */
#define TC_EPI_GEGLU 1 /* weight rows packed per N-tile as [a-half | gate-half]; out = a * gelu_erf(gate) */

const char* tc_last_error(void);
int tc_version(void);
/* number of kernels launched by this library since load (bench.py's gpu_launches claim) */
unsigned long long tc_launch_count(void);
/* SM count of the current device (grid sizing of the persistent kernels) */
int tc_sm_count(void);

/* ------------------------------------------------------------------------------------------------
 * Implicit-GEMM convolution / linear layer on the Hopper tensor cores (wgmma, TMA-fed, register accumulators).
 *
 *   out[m, j] = epilogue( sum_{tap, c} A[n + dn[tap], y + dy[tap], x + dx[tap], c] * Wt[j, tap*C + c] )
 *
 * with m = (n*oH + y)*oW + x over the output pixel grid [oN][oH][oW]; A reads outside [a_N][a_H][a_W]
 * are zero (TMA out-of-bounds fill == the conv's zero padding).
 * epilogue: a = ln_stats ? rstd_m*(acc - mean_m*ln_u[j]) : acc;  v = a + bias[j] + bias2[m / bias2_rows_per][j];
 *           v = v*acc_scale + res[m][j];  (GEGLU optional; optional per-row {sum, sumsq} of the outputs)
 *
 * Replaces (reference call sites): nn.Conv2d 3x3 / 1x1 (openaimodel3d.py:68,96,154,179,187,386,545;
 * autoencoder_dualref.py:52-69,914-935), nn.Conv3d (3,1,1) (openaimodel3d.py:255-266; autoencoder_dualref.py
 * :601-648), nn.Linear (attention.py:53-57,269,290,336,362,418,438), nn.Conv1d k=1 (attention.py:332-334,360).
 * C must be a multiple of 64 (callers zero-pad 4/8/3-channel inputs).
 * Refused with TC_ERR_INVALID (nothing is launched): a, b, out, res or bias2 not 16-byte aligned; A strides, ldb, ldc,
 * ldr or bias2_ld not multiples of 8 elements; n_cols > b_rows; ldc < the output width; ldr < n_cols with a residual;
 * GEGLU with res, bias2, acc_scale != 1 or n_cols % block_n != 0.
 */
typedef struct {
  /* A operand: [a_N][a_H][a_W][C] halfs, C contiguous, strides in elements */
  const void* a;
  int a_N, a_H, a_W, a_C;
  long long a_sN, a_sH, a_sW;
  /* B operand (weights): [b_rows][taps*C] halfs, row stride ldb (elements) */
  const void* b;
  int b_rows;
  long long ldb;
  /* filter taps: per-tap coordinate offsets into A */
  int taps;
  int tap_dx[TC_MAX_TAPS], tap_dy[TC_MAX_TAPS], tap_dn[TC_MAX_TAPS];
  /* output pixel grid and output matrix [oN*oH*oW][n_out] halfs, row stride ldc (elements) */
  int oN, oH, oW;
  void* out;
  long long ldc;
  int n_cols; /* GEMM N (rows of Wt used); output width is n_cols, or n_cols/2 with TC_EPI_GEGLU */
  /* epilogue */
  const float* bias;   /* [n_cols] or NULL */
  const void* bias2;   /* halfs [groups][bias2_ld] or NULL (per-sample timestep-embedding add) */
  long long bias2_ld;
  int bias2_rows_per;  /* output rows per bias2 group */
  const void* res;     /* halfs [M][ldr] or NULL */
  long long ldr;
  float acc_scale;     /* 1.0f for plain layers */
  int flags;
  int block_n;         /* 0 = auto */
  /* folded LayerNorm of the A operand (attention.py:225-227,243-245): with Wt pre-multiplied by gamma,
   * LN(x) @ W^T = rstd_m * (acc - mean_m * ln_u[j]) (+ bias' = beta @ W^T + b).  ln_stats = {mean, rstd} per output
   * row from tc_row_stats, ln_u[j] = sum_k Wt[j][k].  Both NULL for plain layers. */
  const float* ln_stats; /* [M][2], or with ln_nslots > 0: [M][ln_nslots][2] partial {sum, sum of squares} */
  const float* ln_u;     /* [n_cols] */
  /* ln_nslots > 0: ln_stats holds the partial row sums a producer GEMM wrote through row_stats (below); the epilogue
   * finishes them itself: mean = S1/C, rstd = rsqrt(S2/C - mean^2 + ln_eps) with C = a_C (taps must be 1). */
  int ln_nslots;
  float ln_eps;
  /* producer side: per output row, {sum, sum of squares} of the fp16-rounded outputs this launch writes, one slot per
   * N tile: slot = j / block_n, [M][row_stats_slots][2] floats, where row_stats_slots must equal
   * ceil(n_cols/block_n) (so block_n must be given).  Feeds the LayerNorm fold of the consumer without a
   * separate statistics pass over the activation.  NULL = off. */
  float* row_stats;
  int row_stats_slots;
  /* optional scratch for split-K (long K loops on few output tiles): caller-owned, any contents, at least
   * TC_GEMM_WS_TICKET_BYTES of it zeroed ONCE before the first launch that uses it (the library leaves it zeroed).  NULL or too
   * small: no split-K.  One workspace per stream (launches on one stream are ordered). */
  void* workspace;
  long long workspace_bytes;
} TcConvGemm;
#define TC_GEMM_WS_TICKET_BYTES (64 * 1024) /* head of the workspace: per-tile tickets (4 bytes each) */

int tc_conv_gemm(const TcConvGemm* desc, void* stream);
/* profiling aid: bits 8..11 of mode cap the k-slices of later tc_conv_gemm launches (0 = heuristic); other bits are ignored */
int tc_debug_set_gemm_mode(int mode);
/* tests: {block_n, cta pair (always 0), k-slices, pipeline stages} of the process' most recent tc_conv_gemm launch */
int tc_debug_last_gemm_config(int* out4);
/* kept for ABI compatibility: the GEMM kernel records no timeline, so this returns TC_ERR_INVALID */
int tc_debug_read_gemm_trace(unsigned long long* host_dst, int count);
/* kept for ABI compatibility: the attention kernel records no timeline, so this returns TC_ERR_INVALID */
int tc_debug_read_attn_trace(unsigned long long* host_dst, int count);

/* ------------------------------------------------------------------------------------------------
 * GroupNorm (+ optional SiLU), fp32 statistics, channels-last fp16 in/out.
 * x: [groups_of_frames * frames_per_stat][HW][C]; statistics are taken over (frames_per_stat, HW, C/G):
 *   frames_per_stat = 1  -> per-frame GN of a 4-D (N,C,H,W) tensor   (basics.py:76-87; attention.py:265)
 *   frames_per_stat = T  -> 5-D GN over all frames of a clip          (openaimodel3d.py:256-265; attention.py:331;
 *                                                                       autoencoder_dualref.py:601,626)
 * Output may be written into a channel slice of a wider tensor (ldy >= C); input likewise (ldx).
 * `ws` needs 2*n_stat*G*TC_GN_MAX_PARTIALS floats (n_stat = frames/frames_per_stat).
 * Refused (TC_ERR_INVALID, nothing launched): x or y not 16-byte aligned, ldx or ldy not a multiple of 8 or below C.
 */
int tc_groupnorm(const void* x, long long ldx, void* y, long long ldy, const float* gamma, const float* beta,
                 int frames, int frames_per_stat, int hw, int C, int G, float eps, int silu, float* ws,
                 void* stream);

/* per-row {mean, rstd} of [rows][C] halfs (the statistics half of nn.LayerNorm, attention.py:225-227); the
 * normalisation itself is folded into the consuming tc_conv_gemm (ln_stats / ln_u).
 * Refused: x not 16-byte or stats not 8-byte aligned, ldx not a multiple of 8 or below C. */
int tc_row_stats(const void* x, long long ldx, int rows, int C, float eps, float* stats, void* stream);

/* LayerNorm over the last dim of [rows][C] halfs (attention.py:225-227), fp32 math, fp16 out.
 * Refused: x or y not 16-byte aligned, ldx or ldy not a multiple of 8 or below C. */
int tc_layernorm(const void* x, long long ldx, void* y, long long ldy, const float* gamma, const float* beta,
                 int rows, int C, float eps, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Fused attention, head dim 64 (or 80), on mma.sync tensor-core MMAs (QK^T and PV), online softmax in fp32.
 * q:  [q_batches][Lq][heads*D] (row stride ldq), kv segment s: k/v [kv_batches_s][Lk_s][heads*D], D = head dim.
 * Query batch b attends to kv batch b / kv_div[s].  With two segments the two softmax-attention
 * results are summed (text + image cross attention, attention.py:128-142,153-207); with one it is plain
 * attention (attention.py:103-120,175; autoencoder_dualref.py:270-341).
 * head_dim 80 (the OpenCLIP ViT-H/14 vision tower: 16 heads of 80) and causal = 1 (key j masked for query i when
 * j > i: the OpenCLIP text tower's attn_mask) take one segment.  Both fields 0 = head dim 64, no mask.
 */
typedef struct {
  const void* q; long long ldq; int q_batches; int Lq; int heads;
  int n_seg;
  const void* k[2]; const void* v[2]; long long ldk[2]; long long ldv[2]; int Lk[2]; int kv_div[2];
  void* out; long long ldo;
  float scale;
  int head_dim; /* 0 or 64, or 80 */
  int causal;   /* 0 or 1 */
} TcAttention;
int tc_attention(const TcAttention* desc, void* stream);

/* Temporal self-attention over the frame axis (attention.py:365-412 'only_self_att', einsum path :103-120):
 * tokens x[b][t][p][heads*64]; for each (b, p, head) softmax(q k^T * scale) v over t in [0,T), T <= 64.
 * Refused: q, k, v or out not 16-byte aligned, ld or ldo not a multiple of 8 or below heads*64. */
int tc_temporal_attention(const void* q, const void* k, const void* v, long long ld, void* out, long long ldo,
                          int B, int T, int P, int heads, float scale, void* stream);

/* Fused single-head attention with a wide head (D = 64..512, D % 64 == 0, D % 128 == 0 above 256): the VAE mid-block
 * AttnBlock (autoencoder_dualref.py:172-206: q/k/v 1x1 convs -> softmax(q k^T / sqrt(C)) v over the H*W tokens of a frame,
 * C = 512 at full width; also the encoder's mid block).  q/k/v: [batches][L][D] halfs with row strides ldq/ldk/ldv (they
 * may be channel slices of one fused qkv tensor), out: [batches][Lq][D] with row stride ldo.  Scores stay on chip. */
int tc_attention_wide(const void* q, const void* k, const void* v, long long ldq, long long ldk, long long ldv,
                      void* out, long long ldo, int batches, int Lq, int Lk, int D, float scale, void* stream);

/* row softmax of fp16 scores [rows][cols] scaled by `scale`, in place (unfused form of the VAE mid-block attention, d = 512:
 * autoencoder_dualref.py:172-200).  Any sign of `scale`: the maximum is taken over the scaled scores.  Refused: lds < cols. */
int tc_softmax_rows(void* s, long long lds, int rows, int cols, float scale, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Data-movement / elementwise helpers (reference: rearrange/cat/interpolate sites)
 */
/* NCTHW fp32 (B,Cin,T,H,W) -> channels-last fp16 [B][T][H][W][Cpad], zero-padded channels, written at channel
 * offset `coff` of a Cpad-wide tensor (used twice to realise cat([x, c_concat], dim=1), ddpm3d.py:1260-1262);
 * values are multiplied by `scale` (1/scale_factor of decode_core, ddpm3d.py:655). */
int tc_ncthw_to_cl(const float* x, void* y, int B, int C, int T, int H, int W, int Cpad, int coff, float scale,
                   void* stream);
/* channels-last fp16 [B][T][H][W][ld] (first C channels) -> NCTHW fp16 or fp32 (openaimodel3d.py:602) */
int tc_cl_to_ncthw(const void* x, long long ldx, void* y, int out_fp32, int B, int C, int T, int H, int W,
                   void* stream);
/* nearest 2x upsample of [N][H][W][C] (openaimodel3d.py:101-103) */
int tc_upsample2x(const void* x, void* y, int N, int H, int W, int C, void* stream);
/* stride-2 phase split: x [N][H][W][C] -> y [4][N][H/2][W/2][C], phase = (row parity)*2 + col parity
 * (so a stride-2 3x3 conv becomes 9 stride-1 taps; openaimodel3d.py:66-69) */
int tc_phase_split2(const void* x, void* y, int N, int H, int W, int C, void* stream);
/* strided 2-D copy of halfs: dst[r][0:cols] = src[r][0:cols] (torch.cat on channels, openaimodel3d.py:596) */
int tc_copy2d(const void* src, long long lds, void* dst, long long ldd, long long rows, int cols, void* stream);
/* y[r][c] += x[r][c] (Combiner add into first / last frame, autoencoder_dualref.py:357-368) */
int tc_add2d(const void* x, long long ldx, void* y, long long ldy, long long rows, int cols, void* stream);
/* y[r][c] = GELU(x[r][c]), exact erf form (nn.GELU of the Resampler feed-forward, lvdm/modules/encoders/resampler.py:27-34);
 * y may alias x */
int tc_gelu2d(const void* x, long long ldx, void* y, long long ldy, long long rows, int cols, void* stream);

/* One interpolated segment into the joined uint8 video (scripts/evaluation/inference.py:148-153, 262-270):
 * x16: the decoder's fp16 [T][3][H][W] output of the 16-frame pass; x14: NULL or the [T-2][3][H][W] output of the
 * 14-frame pass of the same clip, whose frames T/2-2 and T/2-1 replace frames T/2-1 and T/2 (the middle-frame splice).
 * Frames f_begin <= f < f_end are written to out[f - f_begin][H][W][3] (uint8, NTHWC; `out` points at the first of
 * them) as u = (uint8)(((clamp(x, -1, 1) + 1) / 2) * 255), fp32 ops in that order, truncation toward zero.
 * Any H, W; the vectorised path needs H*W % 8 == 0, 16-byte aligned inputs and an 8-byte aligned `out`. */
int tc_video_u8(const void* x16, const void* x14, int T, int H, int W, int f_begin, int f_end, void* out, void* stream);

/* sinusoidal embedding (utils_diffusion.py:8-28) + Linear -> SiLU -> Linear MLP (openaimodel3d.py:370-382,550-577):
 * out[b][:] (+)= W2 * silu(W1 * sincos(t[b]) + b1) + b2, fp32 output.  dim = model_channels. */
int tc_time_embed(const float* t, int B, int dim, const void* w1, const float* b1, const void* w2, const float* b2,
                  int hidden, float* out, int accumulate, float* ws, void* stream);
/* y[b][j] = sum_k act(x[b][k]) * W[j][k] + bias[j]; x fp32 [B][K], W half [J][K], y half [B][ldy]
 * (ResBlock.emb_layers for all blocks at once: openaimodel3d.py:168-174,219) */
int tc_small_linear(const float* x, int B, int K, const void* w, const float* bias, int J, void* y, long long ldy,
                    int silu_in, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Fused DDIM update (ddim.py:221-277 + utils_diffusion.py:147-158 + ddpm3d.py:240-252), v-parameterisation.
 *   v   = e_uc + s*(e_c - e_uc)            (fp16 arithmetic like the reference under autocast)
 *   v   = phi * v * std(e_c)/std(v) + (1-phi) * v        per sample, if phi > 0
 *   eps = sqrt_ac*v + sqrt_1mac*x ; x0 = sqrt_ac*x - sqrt_1mac*v ; x0 *= rescale
 *   x_prev = sqrt_aprev*x0 + dir_coef*eps + sigma*noise
 * e_c/e_uc: fp16 NCTHW [B][n], x/noise/x_prev/pred_x0: fp32 [B][n].  coef = {s, phi, sqrt_ac, sqrt_1mac,
 * rescale, sqrt_aprev, dir_coef, sigma} (device pointer: 8 floats, so a captured graph can be replayed
 * with new coefficients).  ws: 4*B*TC_DDIM_PARTIALS doubles scratch.
 */
int tc_ddim_step(const void* e_c, const void* e_uc, const float* x, const float* noise, float* x_prev,
                 float* pred_x0, const float* coef, int B, long long n, double* ws, void* stream);

/* Three-way guidance of the multi-condition sampler (lvdm/models/samplers/ddim_multiplecond.py:214-234):
 *   v = e_uc + cfg_img*(e_img - e_uc) + s*(e_c - e_img)   (fp16 arithmetic, one rounding per torch op, left to right)
 * followed by the same guidance rescale against std(e_c) and the same v -> (eps, x0) -> x_prev update as tc_ddim_step.
 * coef holds 9 floats: the 8 of tc_ddim_step and cfg_img. */
int tc_ddim_step3(const void* e_c, const void* e_uc, const void* e_img, const float* x, const float* noise,
                  float* x_prev, float* pred_x0, const float* coef, int B, long long n, double* ws, void* stream);

/* DPM-Solver++(2M) step: tc_ddim_step / tc_ddim_step3 (e_img NULL / not NULL) plus the second-order correction
 *   x_prev += c * (pred_x0 - prev_pred_x0)     (fp32, each op rounded on its own)
 * prev_pred_x0: the previous step's pred_x0, fp32 [B][n], a buffer other than pred_x0 (the caller swaps the two each
 * step).  c = coef[8] (tc_dpm_step) or coef[9] (tc_dpm_step3, after cfg_img).  c == 0 is a first-order step: the
 * result is the DDIM step's bit for bit and prev_pred_x0 is not read. */
int tc_dpm_step(const void* e_c, const void* e_uc, const float* x, const float* noise, const float* prev_pred_x0,
                float* x_prev, float* pred_x0, const float* coef, int B, long long n, double* ws, void* stream);
int tc_dpm_step3(const void* e_c, const void* e_uc, const void* e_img, const float* x, const float* noise,
                 const float* prev_pred_x0, float* x_prev, float* pred_x0, const float* coef, int B, long long n,
                 double* ws, void* stream);

/* Forward diffusion of a clean latent, in place on x (fp32 [B][n]); row b takes a = coef[2b], c = coef[2b+1]:
 *   q = clean ? x0 : a*x0 + c*noise        (q_sample / stochastic_encode: ddpm3d.py:306-309, ddim.py:309-318)
 *   x = mask ? q*m + (1 - m)*x : q         (the masked step blend of ddim.py:172-180)
 * x0, noise, mask: fp32 [B][n] (noise and coef may be NULL with clean; mask NULL: x = q).  Each multiply and add is
 * rounded on its own in that order (no contraction), so x equals torch's fp32 arithmetic bit for bit.  x may not
 * alias x0, noise or mask.  coef is a device pointer (2B floats), so a captured graph can be replayed with new ones. */
int tc_q_sample(float* x, const float* x0, const float* noise, const float* mask, const float* coef, int clean, int B,
                long long n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TOONCRAFTER_B200_H */
