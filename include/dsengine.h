/* dsengine.h — C ABI of libdsengine.so, the sm_90a kernel library behind diffsensei_b200.
 *
 * The reference (jianzongwu/DiffSensei) has no FFI: every kernel on its UNet sampling path is a
 * PyTorch library call.  Each entry point below therefore names the reference call site whose
 * arithmetic it replaces (paths relative to the reference repo root); the Python adapters in
 * diffsensei_b200/ bind them with ctypes (see INTEGRATION.md).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless a comment says "host";
 *   - activations are bf16, channels-last: images are NHWC [B][H][W][C], token tensors [B][N][C]
 *     (the same memory — a transformer block needs no transpose);
 *   - norm/bias parameters are fp32; GEMM/conv weights are bf16, K-major ([out][in]);
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it, nothing synchronises;
 *   - no entry point allocates device memory: scratch is passed in by the caller;
 *   - return value 0 = ok, otherwise a DS_ERR_* code; ds_last_error() gives the message
 *     (thread-local).  There is no CPU fallback: on a box without an sm_90 device every compute
 *     entry point returns DS_ERR_CUDA.
 */
#ifndef DSENGINE_H_
#define DSENGINE_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DS_OK 0
#define DS_ERR_INVALID 1 /* bad argument / unsupported shape */
#define DS_ERR_CUDA 2    /* CUDA runtime / driver error      */

/* library version (major*10000 + minor*100 + patch) and last error message of the calling thread */
int ds_version(void);
const char* ds_last_error(void);
/* number of kernels this library has launched in the calling process (for bench.py's gpu_launches) */
uint64_t ds_launch_count(void);
/* cudaMemsetAsync(ptr, 0, bytes) on `stream`: a memset node (not a fill kernel) for the statistics pools the step clears */
int ds_zero_async(void* ptr, int64_t bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * GroupNorm (+ optional SiLU), NHWC bf16.                     [HBM-bound]
 * Replaces diffusers ResnetBlock2D.norm1/norm2 + nonlinearity (GroupNorm(32, eps=1e-5) -> SiLU),
 * Transformer2DModel.norm (eps=1e-6, no SiLU) and conv_norm_out+conv_act reached from
 * src/models/unet.py:251-261,281-290,316-338 — and the torch.cat([hidden, skip], 1) in front of every up-block
 * ResnetBlock2D (:316-332), which is never materialised.
 *
 * Statistics are per (sample, CHANNEL): fp64 [B][C][2] {sum, sum of squares} of the bf16 tensor.  They normally
 * come from the epilogue of the ds_gemm_bf16 / ds_conv3x3_nhwc call that produced the tensor (`chan_stats`), so the
 * GroupNorm itself is ONE pass: read x, write y (the algorithmic 4 B/element).  Per-channel sums compose: the
 * statistics of a channel concatenation are the two tensors' statistics side by side.
 *   ds_channel_stats   : statistics of a tensor that has no such producer; ACCUMULATES into `stats` (caller zeroes).
 *   ds_groupnorm_apply : y[B][HW][C1+C2] = act(GroupNorm([x1 | x2])) from stats1 [B][C1][2] / stats2 [B][C2][2];
 *                        x2 / stats2 NULL and C2 = 0 for a single source.  The channel sums are folded into the
 *                        `groups` group statistics in shared memory in a fixed order; normalisation, affine and SiLU
 *                        in fp32, one rounding to bf16.  y must not alias x1 / x2 when C2 > 0.
 *   ds_groupnorm_silu  : stand-alone form = zero scratch + ds_channel_stats + ds_groupnorm_apply (two passes over x).
 *                        `stats`: scratch of ds_groupnorm_scratch_floats(B, C) floats, 16-byte aligned.
 * All pointers 16-byte aligned; C, C1, C2 multiples of 8; (C1 + C2) % groups == 0; groups <= 64.
 * --------------------------------------------------------------------------------------------- */
int ds_channel_stats(const void* x, double* stats, int B, int HW, int C, void* stream);
int ds_groupnorm_apply(const void* x1, const double* stats1, int C1, const void* x2, const double* stats2, int C2,
                       void* y, const float* gamma, const float* beta, int B, int HW, int groups, float eps,
                       int apply_silu, void* stream);
int64_t ds_groupnorm_scratch_floats(int B, int C);
int ds_groupnorm_silu(const void* x, void* y, const float* gamma, const float* beta, float* stats, int B, int HW,
                      int C, int groups, float eps, int apply_silu, void* stream);

/* LayerNorm over the last dim, bf16 in/out, fp32 affine.     [HBM-bound]
 * Replaces BasicTransformerBlock.norm1/2/3 (eps 1e-5) and Resampler LayerNorms
 * (src/models/resampler.py:14,40-41,104). rows x C, C % 8 == 0, C <= 5120. */
int ds_layernorm(const void* x, void* y, const float* gamma, const float* beta, int rows, int C, float eps,
                 void* stream);

/* Dialog-bbox embedding add, in place on the NHWC conv_in output.   [HBM-bound]
 * Replaces UNetMangaModel.encode_dialog_bbox (src/models/unet.py:88-114):
 *   sample[b, y, x, :] += emb[:]  iff (x, y) lies in the union of the half-open pixel boxes
 *   [int(x1*W), int(x2*W)) x [int(y1*H), int(y2*H)), clamped to the image.
 * `dialog_bbox` is [B][num_dialogs][4] fp32 holding values ALREADY rounded to the unet dtype
 * (the reference multiplies in the unet dtype before int(): src/models/unet.py:102-105); set
 * `round_bf16` = 1 to reproduce the bf16 product rounding (int(bf16(0.9)*152) = 137), 0 for fp32. */
int ds_dialog_embed_add(void* sample, const float* emb, const float* dialog_bbox, int B, int H, int W, int C,
                        int num_dialogs, int round_bf16, void* stream);

/* Stand-alone IP attention mask (parity aid only — the fused cross-attention kernel computes the
 * same predicate in registers and never materialises it).
 * Replaces MaskedIPAttnProcessor2_0.prepare_attention_mask_ip (src/models/attention_processor.py:115-169).
 *   bbox : [B][num_ips][4] fp32;  mask out: [B][N][num_dummy + num_ips*tokens_per_ip] fp32 in {0,-10000}
 *   (identical across heads, so the head dim is not materialised). (H', W') are re-derived from
 *   (N, aspect_ratio) exactly as the reference does (:131-139). */
int ds_ip_mask(const float* bbox, float* mask, int B, int N, double aspect_ratio, int num_ips, int tokens_per_ip,
               int num_dummy, void* stream);

/* ---------------------------------------------------------------------------------------------
 * bf16 GEMM on wgmma tensor cores, TMA-fed, fp32 accumulation in registers.   [tensor-bound]
 *   out[M][Nout] = epilogue( A[M][K] * W[N][K]^T )
 * Replaces every nn.Linear on the path: attn.to_q/to_k/to_v/to_out (src/models/attention_processor.py:
 * 56,63-64,84,207,225-226,245-246,261), diffusers FeedForward/GEGLU, Transformer2D proj_in/proj_out,
 * ResnetBlock2D.time_emb_proj, TimestepEmbedding, Resampler linears (src/models/resampler.py:15-17,43-45,
 * 100-103), and 1x1 shortcut convs.
 * Epilogue, applied in fp32 before one rounding to bf16:
 *   v = acc + bias[n] + rowbias[row / rows_per_batch][n]
 *   DS_EPI_GEGLU: W/bias rows are packed in blocks of 128 "value" rows followed by their 128 "gate"
 *                 rows (see diffsensei_b200.weights.pack_geglu); out[:, j] = v_val * gelu_erf(v_gate),
 *                 Nout = N/2.  gelu_erf(x) = x * Phi(x) is evaluated as x * sigmoid(2k(x + a x^3 + b x^5)) with
 *                 (k, a, b) fitted to Phi: |abs err| <= 2.6e-5 for all x (the bf16 output rounding is >= 10x larger).
 *   DS_EPI_GELU / DS_EPI_SILU / DS_EPI_QUICKGELU : v = act(v)
 *   then v += residual[row][n] (bf16) and v *= out_scale (if != 0).
 * LayerNorm fusion (diffusers BasicTransformerBlock.norm1/2/3 -> the linears on either side of them):
 *   consumer: with ln_stats != NULL, A holds the UN-normalised rows and the caller passes pre-folded weights
 *             W' = W * gamma (per input feature), bias' = bias + W beta, ln_colsum[n] = sum_k W'[n][k]; then
 *             acc is replaced by rstd[row] * (acc - mean[row] * ln_colsum[n]) before anything else, where
 *             mean = sum/K, rstd = rsqrt(sumsq/K - mean^2 + ln_eps) from ln_stats[row] = {sum, sumsq}.
 *             Algebraically identical to LayerNorm(A) W^T + bias.
 *   producer: with row_stats_out != NULL the call zeroes it (unless row_stats_zeroed), then accumulates {sum, sum
 *             of squares} of every output row (fp32 values, before the bf16 rounding; per-tile fp32 partials are
 *             combined with fp64 atomics, which is exact, so the statistics do not depend on the arrival order) —
 *             bf16 outputs with 16-byte rows only.  zero_rows != NULL: the call also resets that [M][2] buffer (the first n-tile of
 *             every m-tile does it), which lets a chain of GEMMs rotate three statistics buffers without any
 *             memset node: the consumer of buffer k clears buffer k+2.
 * Split-K tail: the kernel is persistent (one CTA per SM, static round-robin over 128 x BN output tiles);
 *   when the tile count is not a multiple of the resident CTAs, the tiles of the partial last round are cut along
 *   K into slices that run on different CTAs, reduced in fp32 through `splitk_ws` (vector red.global.add) and
 *   finished by whichever slice arrives last.  The caller provides a 16-byte aligned workspace that is ALL ZERO on
 *   entry (ds_gemm_splitk_ws_bytes() bytes cover every shape; the kernel leaves it all zero again) and must not be
 *   shared by GEMMs running concurrently on different streams.  NULL simply disables the feature.
 * Mixed-width schedule (default on, DS_GEMM_TAIL=0 disables): when the last round of the persistent schedule would
 *   fill less than ~45 % of the CTAs, the m-rows that fall into it run as 128-column units (twice as many, half
 *   as long) appended to the 256-column units of the same launch, instead of paying a whole round for a handful of
 *   tiles.  Results are bit-identical to the plain schedule (same K order per output element).
 * Constraints: K % 8 == 0, lda % 8 == 0 (16-byte TMA strides). M, N, K tails are handled by TMA
 * zero-fill and masked stores.
 * --------------------------------------------------------------------------------------------- */
#define DS_EPI_NONE 0
#define DS_EPI_GEGLU 1
#define DS_EPI_GELU 2
#define DS_EPI_SILU 3
#define DS_EPI_QUICKGELU 4 /* v * sigmoid(1.702 v): CLIP-L text encoder MLP (hidden_act "quick_gelu") */

typedef struct {
  const void* a;        /* bf16 [M][lda]                                  */
  const void* w;        /* bf16 [N][ldw]  (row = output feature, K-major) */
  void* out;            /* bf16 [M][ldo]  (or fp32 when out_fp32 != 0)    */
  const float* bias;    /* [N] or NULL                                    */
  const float* rowbias; /* [ceil(M/rows_per_batch)][N] or NULL            */
  const void* residual; /* bf16 [M][ldres] or NULL                        */
  int32_t M, N, K;
  int32_t lda, ldw, ldo, ldres;
  int32_t rows_per_batch; /* only read when rowbias != NULL                */
  int32_t rowbias_ld;     /* row stride of rowbias in floats; 0 means N     */
  int32_t epilogue;       /* DS_EPI_*                                      */
  int32_t out_fp32;       /* 1: `out` is fp32                              */
  float out_scale;        /* 0 or 1: no scaling                            */
  const double* ln_stats; /* [M][2] fp64 (sum, sumsq) of A's rows, or NULL  */
  const float* ln_colsum; /* [N] fp32; required with ln_stats               */
  float ln_eps;
  double* row_stats_out;  /* [M][2] fp64 or NULL (see "producer" above)     */
  double* zero_rows;      /* [M][2] fp64 or NULL: rows reset to 0 by this call */
  int32_t row_stats_zeroed; /* 1: row_stats_out is already 0, skip the memset  */
  void* splitk_ws;        /* split-K workspace (see below) or NULL             */
  int64_t splitk_ws_bytes;
  /* second A operand (optional): the GEMM reads [a | a2] along K without the concatenation ever being written —
   * the 1x1 shortcut of an up-block ResnetBlock2D on torch.cat([hidden, skip], 1) (src/models/unet.py:316-332).
   * a2: bf16 [M][lda2], its K2 = K - K1 columns follow a's K1 columns; K1 % 64 == 0.  NULL: off (K1 ignored). */
  const void* a2;
  int32_t K1, lda2;
  /* producer-side GroupNorm statistics (optional): fp64 [M/stats_rows_per_sample][N][2] (sum, sum of squares) per
   * (sample, output channel) of the bf16-rounded outputs, ACCUMULATED with atomics (the caller zeroes it) — read by
   * ds_groupnorm_apply, so the GroupNorm that follows needs no statistics pass over the tensor.  Needs the bf16
   * TMA epilogue (16-byte rows), no GEGLU, stats_rows_per_sample % 128 == 0.  NULL: off. */
  double* chan_stats;
  int32_t stats_rows_per_sample;
  /* 1: `w` is constant data (model weights: never written by a kernel that can still be in flight) — the kernel may
   * then request its first weight tiles before it waits for the preceding kernel (programmatic dependent launch).
   * 0: `w` may have been produced by a preceding kernel (an activation used as the B operand): fetched after the wait. */
  int32_t w_is_constant;
} ds_gemm_args;

int ds_gemm_bf16(const ds_gemm_args* args, void* stream);
/* bytes of split-K workspace that suffice for any ds_gemm_bf16 / ds_conv3x3_nhwc call on the current device */
int64_t ds_gemm_splitk_ws_bytes(void);

/* A CHAIN of n (<= ds_gemm_chain_max()) dependent GEMMs as ONE persistent launch: args[q+1].a must be args[q].out
 * (the BasicTransformerBlock sequences attn.to_out -> attn2.to_q and attn2.to_out -> ff.net.0 -> ff.net.2 -> next
 * attn1.to_qkv of diffusers' BasicTransformerBlock.forward, each a torch.nn.Linear call in the reference; the
 * LayerNorms between them are folded as in ds_gemm_bf16).  Results are bit-identical to n ds_gemm_bf16 calls: same
 * tiles, same K order; only the schedule differs — the CTAs walk the problems back to back and a tile of problem
 * q+1 on row block m starts as soon as all column tiles of problem q for those 128 rows are written (a counter per
 * (problem, row block) in `dep`), so launch / prologue / drain are paid once and the partial last round of one
 * problem is filled with the first tiles of the next.  Every problem: same M > 128, bf16 output with 16-byte
 * addressable rows, no chan_stats, no split-K; residual / ln_stats / row_stats_out / zero_rows may refer to buffers
 * written by EARLIER problems of the chain for the same rows.
 * dep: dep_len >= ds_gemm_chain_max() * ceil(M / 128) + 1 ints, ALL ZERO on entry; the kernel leaves them all
 *      zero again (no memset between launches or graph replays); not to be shared by chains running concurrently. */
int ds_gemm_chain(const ds_gemm_args* args, int n, int* dep, int dep_len, void* stream);
int ds_gemm_chain_max(void);

/* ---------------------------------------------------------------------------------------------
 * 3x3 convolution, padding 1, stride 1 or 2, NHWC bf16, as an implicit GEMM on wgmma:
 * the A operand is gathered by 4-D TMA tiles (one 8x16-pixel patch x 64 channels per filter tap;
 * the halo / zero padding is TMA out-of-bounds fill), never materialised.       [tensor-bound]
 * Replaces nn.Conv2d 3x3 in diffusers ResnetBlock2D.conv1/conv2, Downsample2D.conv (stride 2),
 * Upsample2D.conv and conv_out, reached from src/models/unet.py:251-261,281-290,316-338.
 *   x   : [B][H][W][Cin]          w: [Cout][3][3][Cin] bf16 (tap-major K; see weights.pack_conv3x3)
 *   out : [B][Ho][Wo][Cout],  Ho = (H-1)/stride+1 (same for Wo)
 *   rowbias : [B][Cout] fp32 or NULL — the ResnetBlock2D time-embedding projection, broadcast over pixels
 *   residual: bf16 [B][Ho][Wo][Cout] or NULL — the block's skip / shortcut branch
 * Constraints: Cin % 64 == 0 (conv_in with Cin=4 has its own entry point below).
 * --------------------------------------------------------------------------------------------- */
typedef struct {
  const void* x;
  const void* w;
  void* out;
  const float* bias;
  const float* rowbias;
  const void* residual;
  int32_t B, H, W, Cin, Cout;
  int32_t stride;
  int32_t rowbias_ld; /* row stride of rowbias in floats; 0 means Cout */
  int32_t out_fp32;
  float out_scale;
  void* splitk_ws;    /* as in ds_gemm_args */
  int64_t splitk_ws_bytes;
  double* chan_stats; /* fp64 [B][Cout][2] producer-side GroupNorm statistics, as in ds_gemm_args; NULL: off */
  /* 1: out = conv3x3(nearest_x2(x)) — diffusers Upsample2D (F.interpolate(scale_factor=2, mode="nearest") + conv,
   * reached from src/models/unet.py:335-338) — WITHOUT materialising the upsampled tensor: four 2x2 convolutions of x,
   * one per output-pixel parity, whose taps are the pre-summed 3x3 taps that read the same input pixel (16 instead of
   * 36 MACs per input pixel).  x: [B][H][W][Cin], out: [B][2H][2W][Cout] bf16, w: [4][Cout][2][2][Cin] bf16 from
   * weights.pack_conv3x3_up2 (phase = 2*row_parity + col_parity).  stride 1, no residual / rowbias. */
  int32_t upsample2;
  /* 1: padding (left 0, right 1, top 0, bottom 1) instead of 1 on every side, stride 2 only — diffusers Downsample2D
   * of the AutoencoderKL encoder (F.pad(x, (0, 1, 0, 1)) + Conv2d(stride=2, padding=0)): out [B][H/2][W/2][Cout],
   * output pixel i reads input pixels 2i .. 2i+2.  0: the convolution described above. */
  int32_t pad_bottom_right;
} ds_conv3x3_args;

int ds_conv3x3_nhwc(const ds_conv3x3_args* args, void* stream);

/* conv_in: 3x3, Cin = 4 (latent channels), direct CUDA-core kernel (K = 36 is not GEMM-shaped; the op is
 * bound by writing the [B][H][W][Cout] output).  x: NHWC bf16 [B][H][W][4]; w: fp32 [Cout][3][3][4].
 * Replaces UNet2DConditionModel.conv_in (src/models/unet.py:206).                       [HBM-bound] */
int ds_conv_in_3x3(const void* x, const float* w, const float* bias, void* out, int B, int H, int W, int Cout,
                   void* stream);
/* The same conv on the tensor cores: ds_im2col_latent writes A[B*H*W][64] bf16 (column tap*4 + c, taps row-major over
 * the 3x3 window, zero padding outside the image, columns 36..63 zero) and ds_gemm_bf16 with the weights packed as
 * [Cout][64] (weights.pack_conv_in) does the rest — bias, GroupNorm statistics of the output (chan_stats) and the
 * coalesced TMA store in its epilogue.  x: NHWC bf16 [B][H][W][4].                        [HBM-bound] */
int ds_im2col_latent(const void* x, void* a, int B, int H, int W, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Fused self-attention, head_dim 64, no mask: softmax(Q K^T / 8) V.              [tensor-bound]
 * Replaces F.scaled_dot_product_attention in AttnProcessor2_0.__call__
 * (src/models/attention_processor.py:69-81).
 *   qkv : bf16 [B][N][3*C] — the fused to_q|to_k|to_v projection output (C = heads*64); head h reads
 *         columns h*64.. of each third, via TMA boxes, so no head transpose is ever materialised
 *   out : bf16 [B][N][C]
 * --------------------------------------------------------------------------------------------- */
int ds_attention_self(const void* qkv, void* out, int B, int N, int heads, void* stream);
/* Perturbed-attention guidance (diffusers' PAGCFGIdentitySelfAttnProcessor2_0): ds_attention_self on batch rows
 * [0, first_perturbed_row), bit for bit, and the identity attention map on rows [first_perturbed_row, B): out = the V
 * columns [2C, 3C) of qkv, copied exactly.  One launch; the CTAs of perturbed rows copy instead of attending.
 * 0 <= first_perturbed_row <= B (B: no perturbed row). */
int ds_attention_self_pag(const void* qkv, void* out, int B, int N, int heads, int first_perturbed_row,
                          void* stream);

/* Fused text + masked-IP cross-attention, head_dim 64:                              [HBM-bound]
 *   out = softmax(Q Kt^T/8) Vt + scale * softmax(Q Kip^T/8 + M(bbox)) Vip
 * Replaces both SDPA calls, prepare_attention_mask_ip and the blend in
 * MaskedIPAttnProcessor2_0.__call__ (src/models/attention_processor.py:231-258).
 *   q    : bf16 [B][N][C]
 *   kv_t : bf16 [B][n_text][2*C]  (to_k | to_v of the text tokens; timestep-invariant)
 *   kv_ip: bf16 [B][n_ip][2*C]    (to_k_ip | to_v_ip of the image tokens, n_ip = num_dummy + num_ips*tokens_per_ip)
 *   bbox : fp32 [B][num_ips][4];  the additive mask is evaluated in registers with the reference's
 *          closed-interval linspace membership and derived (H', W') (:131-163); masked keys get -10000.
 * n_text, n_ip: any positive lengths; both key sets stay resident in shared memory when they take <= 4 64-key tiles
 * together, and stream otherwise.  num_ips <= 16. */
typedef struct {
  const void* q;
  const void* kv_text;
  const void* kv_ip;
  const float* bbox;
  void* out;
  int32_t B, N, heads;
  int32_t n_text, n_ip;
  int32_t num_ips, tokens_per_ip, num_dummy;
  double aspect_ratio; /* latent H / W as a Python float (double): pipeline_diffsensei.py:272 */
  float ip_scale;
} ds_cross_ip_args;

int ds_attention_cross_ip(const ds_cross_ip_args* args, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Layout / glue kernels (all HBM-bound, vectorised)
 * --------------------------------------------------------------------------------------------- */
/* NCHW (fp32 or bf16) <-> NHWC bf16 at the diffusers-facing boundary of UNetMangaModel.forward */
int ds_nchw_to_nhwc(const void* src, int src_is_fp32, void* dst_bf16, int B, int C, int H, int W, void* stream);
int ds_nhwc_to_nchw(const void* src_bf16, void* dst, int dst_is_fp32, int B, int C, int H, int W, void* stream);
/* nearest-neighbour resize to (Ho, Wo) (Upsample2D's F.interpolate; src index = floor(dst * in/out)) */
int ds_upsample_nearest(const void* x, void* y, int B, int H, int W, int C, int Ho, int Wo, void* stream);
/* channel concat of two NHWC tensors: y[..., :C1] = a, y[..., C1:] = b  (torch.cat([hidden, skip], 1)) */
int ds_concat_channels(const void* a, const void* b, void* y, int pixels, int C1, int C2, void* stream);
/* elementwise y = silu(x), n bf16 elements */
int ds_silu(const void* x, void* y, int64_t n, void* stream);
/* Timesteps(num_channels, flip_sin_to_cos=True, downscale_freq_shift=0): out[r][:] = [cos | sin](t[r]*w) bf16 */
int ds_timestep_embedding(const float* t, void* out, int rows, int dim, void* stream);

/* ---------------------------------------------------------------------------------------------
 * CFG blend + DDIM (eta = 0, epsilon-prediction) update, fused.                    [HBM-bound]
 * Replaces src/pipelines/pipeline_diffsensei.py:315,332-337 (chunk, u + g*(t-u), scheduler.step,
 * and the torch.cat([latents]*2) for the next step):
 *   eps   = e_uncond + guidance * (e_text - e_uncond)
 *   x0    = (x - sqrt(1-a_t) * eps) / sqrt(a_t)
 *   x_new = sqrt(a_prev) * x0 + sqrt(1-a_prev) * eps
 *   noise_pred : bf16 NHWC [2*bs][H][W][4] (uncond half first)
 *   latents    : fp32 [bs][H][W][4] updated in place (fp32 master copy)
 *   model_in   : bf16 NHWC [2*bs][H][W][4] — x_new duplicated for both CFG halves (next step's UNet input)
 *   coef       : device pointer to 2 floats {alpha_prod_t, alpha_prod_t_prev} for this step
 * --------------------------------------------------------------------------------------------- */
int ds_cfg_ddim_step(const void* noise_pred, float* latents, void* model_in, const float* coef, float guidance,
                     int bs, int HW, int C, void* stream);

/* ---------------------------------------------------------------------------------------------
 * CFG blend + Euler (EulerDiscreteScheduler, s_churn = 0, epsilon-prediction) update + the next
 * step's scale_model_input, fused.                                                 [HBM-bound]
 * Replaces src/pipelines/pipeline_diffsensei.py:315-317,332-337 (chunk, u + g*(t-u), scheduler.step,
 * the torch.cat([latents]*2) and scheduler.scale_model_input for the next step), fp32, each operation
 * rounded separately in this order:
 *   eps     = e_uncond + guidance * (e_text - e_uncond)
 *   x0      = x - sigma * eps
 *   d       = (x - x0) / sigma
 *   x_new   = x + d * (sigma_next - sigma)
 *   noise_pred : bf16 NHWC [2*bs][H][W][4] (uncond half first)
 *   latents    : fp32 [bs][H][W][4] updated in place (fp32 master copy)
 *   model_in   : bf16 NHWC [2*bs][H][W][4] — x_new / sqrt(sigma_next^2 + 1) for both CFG halves
 *   coef       : device pointer to 3 floats {sigma, sigma_next, sqrt(sigma_next^2 + 1)} for this step
 * --------------------------------------------------------------------------------------------- */
int ds_cfg_euler_step(const void* noise_pred, float* latents, void* model_in, const float* coef, float guidance,
                      int bs, int HW, int C, void* stream);

/* ---------------------------------------------------------------------------------------------
 * The two updates above followed by the inpaint blend of diffusers' StableDiffusionXLInpaintPipeline with a
 * 4-channel UNet, fused.                                                           [HBM-bound]
 *   init  = c0 * z + c1 * n        (add_noise of the image latents at the next timestep; {1, 0} on the last step;
 *                                   each product and the sum rounded on its own)
 *   x_new = mask ? x_new : init    ((1 - m) * init + m * x_new with a binary m)
 * and the next UNet input is computed from the blended x_new.  A pixel with mask != 0 is the plain kernel's result
 * bit for bit.
 *   coef          : DDIM {alpha_prod_t, alpha_prod_t_prev, c0, c1}; Euler {sigma, sigma_next,
 *                   sqrt(sigma_next^2 + 1), c0, c1} (device pointer)
 *   image_latents : fp32 NHWC [bs][H][W][4] (z, scaling_factor * posterior sample), 16-byte aligned
 *   noise         : fp32 NHWC [bs][H][W][4] (n, the noise the start latents were drawn with), 16-byte aligned
 *   mask          : uint8 [bs][H][W], 1 = regenerate, 0 = keep the image
 * --------------------------------------------------------------------------------------------- */
int ds_cfg_ddim_inpaint_step(const void* noise_pred, float* latents, void* model_in, const float* coef, float guidance,
                             const float* image_latents, const float* noise, const uint8_t* mask, int bs, int HW,
                             int C, void* stream);
int ds_cfg_euler_inpaint_step(const void* noise_pred, float* latents, void* model_in, const float* coef,
                              float guidance, const float* image_latents, const float* noise, const uint8_t* mask,
                              int bs, int HW, int C, void* stream);

/* ---------------------------------------------------------------------------------------------
 * CFG + perturbed-attention guidance (diffusers' PAGMixin, do_classifier_free_guidance) fused with the four updates
 * above.                                                                           [HBM-bound]
 *   noise_pred : bf16 NHWC [3*bs][H][W][4], chunks [uncond ; text ; perturbed]
 *   eps        = (e_uncond + guidance * (e_text - e_uncond)) + s * (e_text - e_perturbed)
 * then the DDIM / Euler update (and the inpaint blend) of the matching CFG kernel, every operation rounded on its
 * own in diffusers' eager order (the DDIM update too); model_in : bf16 NHWC [3*bs][H][W][4], the next UNet input
 * in all three chunks.  s is the LAST entry of the step's coefficient row, read on the device:
 *   DDIM {a_t, a_prev, s}                 Euler {sigma, sigma_next, sqrt(sigma_next^2 + 1), s}
 *   DDIM inpaint {a_t, a_prev, c0, c1, s} Euler inpaint {sigma, sigma_next, sqrt(sigma_next^2 + 1), c0, c1, s}
 * --------------------------------------------------------------------------------------------- */
int ds_cfg_pag_ddim_step(const void* noise_pred, float* latents, void* model_in, const float* coef, float guidance,
                         int bs, int HW, int C, void* stream);
int ds_cfg_pag_euler_step(const void* noise_pred, float* latents, void* model_in, const float* coef, float guidance,
                          int bs, int HW, int C, void* stream);
int ds_cfg_pag_ddim_inpaint_step(const void* noise_pred, float* latents, void* model_in, const float* coef,
                                 float guidance, const float* image_latents, const float* noise, const uint8_t* mask,
                                 int bs, int HW, int C, void* stream);
int ds_cfg_pag_euler_inpaint_step(const void* noise_pred, float* latents, void* model_in, const float* coef,
                                  float guidance, const float* image_latents, const float* noise, const uint8_t* mask,
                                  int bs, int HW, int C, void* stream);

/* Perceiver attention of the character Resampler: 16 latent queries x (n_kv) keys per (character, head),
 * q and k each pre-scaled by dim_head^-0.25, fp32 softmax (src/models/resampler.py:64-74).
 *   q: bf16 [Bc][nq][C], kv: bf16 [Bc][n_kv][2*C] (k | v), out: bf16 [Bc][nq][C]; C = heads*64 */
int ds_resampler_attn(const void* q, const void* kv, void* out, int Bc, int nq, int n_kv, int heads, void* stream);

/* ---------------------------------------------------------------------------------------------
 * AutoencoderKL decoder helpers (SURVEY.md §8f rank 1: the step right after the denoise loop,
 * src/pipelines/pipeline_diffsensei.py:339-367).  The decoder's convs / GroupNorms / linears / upsampling run on
 * the entry points above; these cover what is specific to it.                               [HBM-bound]
 *   ds_latent_pointwise : out[b][p][0..4) = W (latents[b][:][p] * inv_scale) + bias — `latents / scaling_factor`
 *                         followed by AutoencoderKL.post_quant_conv (1x1, 4 -> 4).  latents fp32 NCHW [B][4][HW],
 *                         w fp32 [4][4] (out, in), bias fp32 [4] or NULL, out bf16 NHWC [B][HW][4].
 *   ds_softmax_rows     : P[r][:] = softmax(scale * S[r][:]), S fp32 [rows][lds], P bf16 [rows][ldp], n <= 32768
 *                         columns — between the QK^T and PV GEMMs of the decoder's single 512-wide attention head.
 *   ds_image_postprocess: out = clamp(x / 2 + 0.5, 0, 1), x bf16 NHWC [B][HW][C] -> out fp32 NCHW [B][C][HW]
 *                         (VaeImageProcessor.postprocess with do_denormalize, output_type "pt").
 * --------------------------------------------------------------------------------------------- */
int ds_latent_pointwise(const float* latents, const float* w, const float* bias, void* out, float inv_scale, int B,
                        int HW, void* stream);
int ds_softmax_rows(const float* S, void* P, int rows, int n, int64_t lds, int64_t ldp, float scale, void* stream);
int ds_image_postprocess(const void* x, float* out, int B, int HW, int C, void* stream);
/* The AutoencoderKL encoder's posterior, from its conv_out output x fp32 NHWC [B][HW][8] (diffusers
 * AutoencoderKL.encode -> DiagonalGaussianDistribution, then StableDiffusionXLImg2ImgPipeline.prepare_latents):
 *   moments = quant_conv(x) (w fp32 [8][8] (out, in), bias fp32 [8]);  mean = moments[:4],
 *   logvar = clamp(moments[4:], -30, 20);  z = mean + exp(0.5 logvar) * eps  (eps NULL: z = mean, i.e. mode());
 *   z = scale * z;  out[b * repeat + r] = c0 * z + c1 * noise[b * repeat + r] for r < repeat, with {c0, c1} = coef, a
 *   DEVICE pointer: {sqrt(alpha_bar_t), sqrt(1 - alpha_bar_t)} for DDIM's add_noise, {1, sigma} for Euler's (noise NULL:
 *   out = z repeated).  fp32 throughout, each operation rounded on its own.
 *   mean / logvar / eps: fp32 NCHW [B][4][HW], each optional output may be NULL;  noise / out: fp32 NCHW
 *   [B * repeat][4][HW].  x 16-byte aligned. */
int ds_vae_posterior(const float* x, const float* w, const float* bias, const float* eps, float scale,
                     const float* noise, const float* coef, int repeat, float* mean, float* logvar, float* out, int B,
                     int HW, void* stream);

/* The decoder's mid-block attention (diffusers Attention(heads=1, dim_head=D)) in ONE launch for the whole batch:
 *   out[b] = softmax(q[b] k[b]^T / sqrt(D)) v[b]                                                     [compute-bound]
 *   q / k / v : bf16 [B][N][ld] — rows of D elements with one shared row stride ld (elements, >= D, a multiple of 8),
 *               images N * ld apart, so column slices of one fused q|k|v projection may be passed as they are
 *   out       : bf16 [B][N][D], dense
 *   D = 128 or 512 (the last block_out_channels of TINY_VAE / SDXL's VAE); any other D returns DS_ERR_INVALID.
 *   Any N >= 1 and B <= 65535; pointers 16-byte aligned.  fp32 scores, running max / sum and accumulation, P rounded
 *   to bf16 before the PV product.  No scratch memory: a flash (online-softmax) pass over 32-key tiles.
 * Replaces the decoder's QK^T GEMM -> ds_softmax_rows -> PV GEMM, which materialised the [N][N] scores. */
int ds_attention_single_head(const void* q, const void* k, const void* v, void* out, int B, int N, int D, int64_t ld,
                             void* stream);

/* ---------------------------------------------------------------------------------------------
 * Conditioning-encoder helpers (SURVEY.md §8f ranks 2-3: CLIP ViT-H / Magi ViT-MAE image encoders,
 * src/pipelines/pipeline_diffsensei.py:125-128, and the two SDXL CLIP text encoders of encode_prompt, :232-245).
 * Their linears run on ds_gemm_bf16 and their LayerNorms on ds_layernorm.                    [latency-bound]
 *   ds_attention_small : out = softmax(scale * Q K^T [+ causal mask]) V for short sequences (Nk <= 320) and any
 *                        head_dim that is a multiple of 8 up to 256 (80 for ViT-H, 160 for the MLLM input resampler: outside the flash
 *                        kernel's 64).
 *                        q/k/v/out: bf16 [B][N][ld*] with head h at columns [h*head_dim, (h+1)*head_dim); the row
 *                        strides ld* are in elements, so q/k/v may point into one fused [B][N][3C] projection.
 *                        causal != 0: key j visible from query i iff j <= i (CLIP text), needs Nq == Nk.
 *   ds_embed_tokens    : out[b][t][:] = tok_emb[ids[b][t]][:] + pos_emb[t][:], bf16, ids int32 [B][L] (clamped to
 *                        the vocabulary) — CLIPTextEmbeddings.
 * --------------------------------------------------------------------------------------------- */
int ds_attention_small(const void* q, const void* k, const void* v, void* out, int B, int Nq, int Nk, int heads,
                       int head_dim, int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo, float scale, int causal,
                       void* stream);
int ds_embed_tokens(const int* ids, const void* tok_emb, const void* pos_emb, void* out, int B, int L, int C, int vocab,
                    void* stream);

/* Image processors of prepare_ip_image_embeds (src/pipelines/pipeline_diffsensei.py:70-71,125-126: transformers'
 * CLIPImageProcessor / ViTImageProcessor, shipped defaults, PIL backend), bit-exact:
 *   DS_IMG_CLIP : shortest edge -> 224 (long edge int(224 * long / short)), Pillow bicubic, centre crop 224 x 224,
 *                 (x / 255 - OPENAI_CLIP_MEAN) / OPENAI_CLIP_STD
 *   DS_IMG_VIT  : 224 x 224, Pillow bilinear, (x / 255 - 0.5) / 0.5
 * The resize is Pillow's 8-bit fixed-point resampler (22-bit coefficients, horizontal pass into a uint8
 * intermediate, then vertical; a pass whose size does not change is skipped); see image_kernels.cu.
 *   src     : uint8 RGB HWC images packed in one buffer; image i starts at byte offsets[i]
 *   offsets : HOST int64 [n];  sizes: HOST int32 [n][2] {height, width}, each side in [1, 65535]
 *   out     : fp32 NCHW [n][3][224][224]
 *   scratch : ds_image_preprocess_scratch_bytes(sizes, n, mode) bytes, 16-byte aligned (coefficient tables and the
 *             uint8 intermediate; no fixed tap limit).  The query is pure host arithmetic; it returns -1 for
 *             arguments the entry point rejects.
 * Three launches per 16 images. */
#define DS_IMG_CLIP 0
#define DS_IMG_VIT 1
int64_t ds_image_preprocess_scratch_bytes(const int* sizes, int n, int mode);
int ds_image_preprocess(const uint8_t* src, const int64_t* offsets, const int* sizes, int n, int mode, float* out,
                        void* scratch, int64_t scratch_bytes, void* stream);

/* Image preprocessing of the AutoencoderKL encoder (diffusers VaeImageProcessor.preprocess, default config:
 * do_resize with Pillow LANCZOS, do_normalize), bit-exact with Pillow + numpy / torch fp32:
 *   ds_vae_image_preprocess : one uint8 RGB HWC image [H][W][3] -> Image.resize((out_w, out_h), LANCZOS) (skipped when
 *                             the size does not change), then x = float32(u8) / 255, 2x - 1.  Writes `out` fp32 NCHW
 *                             [3][out_h][out_w] and / or `out_nhwc4` bf16 NHWC [out_h][out_w][4] with a zero 4th
 *                             channel (the input of the encoder's conv_in); either may be NULL.  Same 8-bit fixed-point
 *                             resampler as ds_image_preprocess; the Lanczos tap tables are built on the host (with the
 *                             host libm's sin, as Pillow does) and copied into the scratch, so the call is not
 *                             graph-capturable.  scratch: ds_vae_image_preprocess_scratch_bytes(...) bytes, 16-byte
 *                             aligned (-1: sizes the entry point rejects; sides in [1, 65535]).
 *   ds_vae_image_pack       : a float NCHW [B][3][HW] image that is already at its size -> (normalize ? 2x - 1 : x) as
 *                             fp32 NCHW `out` (may alias x) and / or bf16 NHWC `out_nhwc4` [B][HW][4], 4th channel 0. */
int64_t ds_vae_image_preprocess_scratch_bytes(int H, int W, int out_h, int out_w);
int ds_vae_image_preprocess(const uint8_t* src, int H, int W, int out_h, int out_w, float* out, void* out_nhwc4,
                            void* scratch, int64_t scratch_bytes, void* stream);
int ds_vae_image_pack(const float* x, float* out, void* out_nhwc4, int B, int HW, int normalize, void* stream);

/* Inpaint mask preprocessing (diffusers VaeImageProcessor(do_normalize=False, do_binarize=True,
 * do_convert_grayscale=True).preprocess, then prepare_mask_latents' F.interpolate(nearest) to H/8 x W/8):
 *   ds_vae_mask_preprocess : one uint8 HWC image with C = 1 ("L") or C = 3 ("RGB") channels -> Image.resize((out_w,
 *                            out_h), LANCZOS) in its own mode (same resampler and host-built tap tables as
 *                            ds_vae_image_preprocess) -> for RGB, Pillow's convert("L") of the resized pixels,
 *                            (19595 R + 38470 G + 7471 B + 0x8000) >> 16 -> binarize float32(L) / 255 at 0.5, i.e.
 *                            L >= 128.  Writes `out` fp32 [out_h][out_w] in {0, 1} and / or `out_latent` uint8
 *                            [out_h/8][out_w/8] = the mask at (8i, 8j); either may be NULL (out_latent needs sizes that
 *                            are multiples of 8).  Not graph-capturable (host tables).  scratch:
 *                            ds_vae_mask_preprocess_scratch_bytes(...) bytes, 16-byte aligned (-1: rejected sizes).
 *   ds_vae_mask_pack       : a float mask already at its size [H][W] -> (x >= 0.5) as `out` fp32 and / or
 *                            `out_latent` uint8 [H/8][W/8]. */
int64_t ds_vae_mask_preprocess_scratch_bytes(int H, int W, int C, int out_h, int out_w);
int ds_vae_mask_preprocess(const uint8_t* src, int H, int W, int C, int out_h, int out_w, float* out,
                           uint8_t* out_latent, void* scratch, int64_t scratch_bytes, void* stream);
int ds_vae_mask_pack(const float* x, int H, int W, float* out, uint8_t* out_latent, void* stream);

/* ---------------------------------------------------------------------------------------------
 * LLaMA decoder of the MLLM agent (SURVEY.md §8f-4: ContinuousLVLM.generate, src/models/mllm/seed_x.py:90-171, over
 * LlamaForCausalLM of src/models/mllm/modeling_llama_xformer.py).  Every kernel that depends on the sequence position
 * reads it from a DEVICE int32 (`pos`), so one captured graph serves every decode step.
 *   ds_gemv_bf16       : y[M][N] = x[M][K] W[N][K]^T (+ residual[M][N]), bf16 in, fp32 accumulation, bf16 or fp32
 *                        (out_fp32) out, 1 <= M <= 8, K % 8 == 0, M*K*2 bytes <= 227 KB.  W is streamed once with
 *                        16-byte non-allocating loads; x is staged in shared memory.  y may alias residual.
 *                        The decode linears (fused q|k|v, o_proj, fused gate|up, down_proj, lm_head).  [HBM-bound]
 *   ds_rmsnorm         : LlamaRMSNorm: y = x * rsqrt(mean(x^2) + eps) * gamma, fp32 statistics, one rounding to
 *                        bf16; x / y bf16 [rows][C], gamma fp32 [C]; C % 8 == 0, C <= 8192.
 *   ds_rope_kv_append  : qkv bf16 [M][3][H][D] (the fused projection); row m has position *pos + m.  Rotates q and k
 *                        (rotate-half, inv_freq = theta^(-2i/D) in fp32), writes q_out bf16 [M][H][D] and appends the
 *                        rotated k and v to kv_layer bf16 [2][H][L_max][D] (one layer of a [layer][2][H][L_max][D]
 *                        cache).  Rows at positions >= L_max are skipped.  D = 64 or 128.
 *   ds_attention_kv    : out[m] = softmax(q[m] K^T / sqrt(D)) V over cache keys 0 .. *pos + m (bottom-right causal),
 *                        q / out bf16 [M][H][D].  Keys are cut into ceil(L_max / chunk) splits of `chunk` keys that
 *                        run on separate CTAs (splits past the current length exit at once) and a combine pass merges
 *                        them; ws: fp32 workspace of >= M * H * splits * (D + 2) * 4 bytes.  D = 64 or 128.
 *   ds_silu_mul        : out[m][i] = silu(g[m][i]) * u[m][i] from gate_up bf16 [M][2I] = [g | u]; I % 8 == 0.
 *   ds_agent_next_token: one greedy step at batch 1.  state: int32 {pos, generated, done, last token}.  When done is
 *                        set the call changes nothing.  Otherwise: hidden[pos] = hidden_src (bf16 [C], skipped when
 *                        NULL); the image-token rule of AutoImageTokenGenerationProcessor (src/models/mllm/
 *                        generation.py:18-30) on logits fp32 [V], IN PLACE: if `last` is in img_ids[0 .. n_img-2],
 *                        the next entry's score becomes max + 10, else the scores of img_ids[1 ..] become 0.0; then
 *                        tok = argmax (first index on ties); out_ids[generated] = tok; next_x = embed[tok] (bf16
 *                        [V][C]); pos += 1; generated += 1; last = tok; done = (tok == eos || generated >= max_new).
 * B sequences decoded together, one row each (B <= 8 in the engine, the GEMV's limit).  Row b has its own position
 * pos[b * pos_stride] (device int32; the engine passes its [B][4] state with pos_stride 4) and its own cache slice
 * kv + b * seq_stride elements, laid out [2][H][L_cap][D].  Each row computes what the batch-1 kernel computes for
 * that sequence alone, bit for bit (same split boundaries when `chunk` is the batch-1 decode's).
 *   ds_rope_kv_append_rows  : ds_rope_kv_append of row b of qkv bf16 [B][3][H][D] at position pos[b]: q_out[b],
 *                             k / v appended at row pos[b] of its slice.  Rows at positions >= L_cap are skipped.
 *   ds_attention_kv_rows    : out[b] = softmax(q[b] K_b^T / sqrt(D)) V_b over keys 0 .. pos[b] of slice b; q / out
 *                             bf16 [B][H][D].  ceil(L_cap / chunk) splits per (row, head) and a combine pass; ws:
 *                             fp32 workspace of >= B * H * splits * (D + 2) * 4 bytes.  D = 64 or 128.
 *   ds_agent_next_token_rows: ds_agent_next_token for every row b on its own: logits fp32 [B][V], state int32 [B][4],
 *                             out_ids int32 [B][max_new], next_x bf16 [B][C], hidden bf16 rows of row b at hidden +
 *                             b * hidden_stride elements (hidden_stride % 8 == 0), hidden_src bf16 [B][C] or NULL.
 *                             img_ids, eos and max_new are shared.  A row whose done is set changes nothing.
 * --------------------------------------------------------------------------------------------- */
int ds_gemv_bf16(const void* x, const void* w, const void* residual, void* y, int M, int N, int K, int out_fp32,
                 void* stream);
int ds_rmsnorm(const void* x, const float* gamma, void* y, int rows, int C, float eps, void* stream);
int ds_rope_kv_append(const void* qkv, void* q_out, void* kv_layer, const int* pos, int M, int H, int D, int L_max,
                      float theta, void* stream);
int ds_attention_kv(const void* q, const void* kv_layer, void* out, float* ws, int64_t ws_bytes, const int* pos, int M,
                    int H, int D, int L_max, int chunk, void* stream);
int ds_silu_mul(const void* gate_up, void* out, int M, int I, void* stream);
int ds_agent_next_token(float* logits, int V, const int* img_ids, int n_img, int* state, int* out_ids, int max_new,
                        int eos, const void* embed, void* next_x, const void* hidden_src, void* hidden, int C,
                        void* stream);
int ds_rope_kv_append_rows(const void* qkv, void* q_out, void* kv, int64_t seq_stride, const int* pos, int pos_stride,
                           int B, int H, int D, int L_cap, float theta, void* stream);
int ds_attention_kv_rows(const void* q, const void* kv, int64_t seq_stride, void* out, float* ws, int64_t ws_bytes,
                         const int* pos, int pos_stride, int B, int H, int D, int L_cap, int chunk, void* stream);
int ds_agent_next_token_rows(float* logits, int V, const int* img_ids, int n_img, int* state, int* out_ids, int max_new,
                             int eos, const void* embed, void* next_x, const void* hidden_src, void* hidden,
                             int64_t hidden_stride, int C, int B, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DSENGINE_H_ */
