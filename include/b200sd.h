/* b200sd.h — C ABI of libb200sd.so, the sm_90a (H100) compute library behind the local-GPU worker.
 *
 * Boundary being replaced (reference = papuSpartan/stable-diffusion-webui-distributed @ 8fd65ebd):
 *   scripts/spartan/worker.py:288-504  Worker.request()  — the reference posts the job to a remote sdwui
 *   (`session.post(full_url("txt2img"|"img2img"))`, worker.py:432-435) whose process_images() runs
 *   UNet x steps + VAE decode.  The reference contains none of that arithmetic (SURVEY.md §0.2); these
 *   entry points are what a local executor binds instead of the HTTP call: every function below is one
 *   op of the per-step model evaluation and sampler update / final decode (SURVEY.md §8 a-ext x1..x11), taking
 *   raw device pointers and an explicit stream.  The sampler updates take an eps-prediction model (SD1.x, SDXL);
 *   the `_v` twins take a v-prediction model (SD 2.x 768-v and v-prediction finetunes): they convert the
 *   CFG-combined v to eps = sqrt(1-a) x_in + sqrt(a) v in fp32, next to the fp32 latents, before the same update.
 *
 * Conventions
 *   - caller owns all device memory; the library never allocates, never synchronises, never throws
 *   - activations are NHWC ("pixels x channels") fp16 (dtype 0) or bf16 (dtype 1); `ld*` / `pitch` are row
 *     pitches in ELEMENTS, so channel slices of wider buffers (skip-concat buffers) are addressed in place
 *   - weights are pre-packed [N][K] (K contiguous); conv weights [Cout][ky][kx][Cin]
 *   - all pointers 16-byte aligned, pitches multiples of 8 elements
 *   - `stream` is a cudaStream_t passed as void* (torch.cuda.current_stream().cuda_stream)
 *   - return value: 0 ok, <0 error (B200SD_ERR_*); the call launched nothing if it failed
 */
#ifndef B200SD_H_
#define B200SD_H_

#ifdef __cplusplus
extern "C" {
#endif

#define B200SD_OK 0
#define B200SD_ERR_INVALID (-1)
#define B200SD_ERR_CUDA (-2)
#define B200SD_ERR_TMAP (-3)
#define B200SD_ERR_UNSUPPORTED (-4)

#define B200SD_F16 0
#define B200SD_BF16 1

/* epilogue flags for b200sd_linear / b200sd_conv2d */
#define B200SD_EPI_GEGLU 1 /* tile columns [0,bn/2) = value, [bn/2,bn) = gate: out = v * gelu_erf(g) */
#define B200SD_EPI_SILU 2  /* out = silu(acc + bias (+ residual)) */
#define B200SD_EPI_LRELU 4 /* b200sd_conv2d_scaled only: v = leaky_relu(acc + bias, 0.2) */

/* The residual may be the output itself (residual == D and ldr == ldd: D += epi(...) in place, e.g. a ControlNet zero
 * conv adding into a channel slice of a skip-concat buffer): each output tile reads its residual tile before it
 * stores that tile, and no two tiles overlap.  Any other overlap of residual and D is undefined. */
typedef struct b200sd_epilogue {
  const float* bias;      /* [groups][N] fp32 or NULL */
  int bias_group_rows;    /* output rows sharing one bias row (H*W for a per-image bias); <=0: one row */
  const void* residual;   /* [M][N_out] same dtype as the output, or NULL (may equal D, see above) */
  long long ldr;          /* residual row pitch (elements) */
  int flags;              /* B200SD_EPI_* */
} b200sd_epilogue;

/* library / build identification: returns a static string "b200sd <version> sm_90a" */
const char* b200sd_version(void);

/* ---- tensor-core ops (wgmma + TMA) -------------------------------------------------------------- */

/* D[M,N_out] = epi(A[M,K] . Wt[N,K]^T).  Linear layers and 1x1 convs (upstream ldm CrossAttention.to_q/k/v/
 * to_out, FeedForward.net, SpatialTransformer.proj_in/out, ResBlock.skip_connection).
 * K % 64 == 0, N % block_n == 0, block_n in {32,64,...,256}.  max_ctas <= 0: one CTA per SM. */
int b200sd_linear(const void* A, long long lda, const void* Wt, void* D, long long ldd, int M, int N, int K,
                  int block_n, const b200sd_epilogue* epi, int dtype, int max_ctas, void* stream);

/* NHWC convolution as implicit GEMM: X[NB,Hin,Win,C] (channel pitch `pitch_c`), Wt[Cout][k*k*C],
 * ksize in {1,3}, stride in {1,2}, zero padding `pad` before / `pad_end` after each spatial dim.
 * D rows are output pixels in (n, y, x) order.  (upstream ResBlock.in_layers/out_layers conv, Upsample.conv,
 * Downsample.op, AutoencoderKL Decoder/Encoder convs.)  C % 64 == 0. */
int b200sd_conv2d(const void* X, long long pitch_c, int NB, int Hin, int Win, int C, const void* Wt, int ksize,
                  int stride, int pad, int pad_end, void* D, long long ldd, int Cout, int block_n,
                  const b200sd_epilogue* epi, int dtype, int max_ctas, void* stream);
/* b200sd_conv2d with the epilogue of ESRGAN's RRDBNet (basicsr ResidualDenseBlock / RRDB): v = acc + bias, then
 * v = leaky_relu(v, 0.2) if epi->flags has B200SD_EPI_LRELU, then D = residual + res_scale * v if epi->residual is set
 * (else D = v).  epi->flags may hold B200SD_EPI_LRELU only; block_n in {32, 64}; dtype B200SD_F16 only (the upscaler runs
 * in fp16 for every model family; bf16 returns B200SD_ERR_INVALID).  The residual may equal D as for b200sd_conv2d.
 * C % 64 == 0. */
int b200sd_conv2d_scaled(const void* X, long long pitch_c, int NB, int Hin, int Win, int C, const void* Wt, int ksize,
                         int stride, int pad, int pad_end, void* D, long long ldd, int Cout, int block_n,
                         const b200sd_epilogue* epi, float res_scale, int dtype, int max_ctas, void* stream);

/* O[b,s,h*d] = softmax(Q K^T * scale) V per (batch, head); Q/K/V rows are tokens, head h occupies columns
 * [h*d_pad, h*d_pad+d) (zero padded to d_pad, a multiple of 64).  (upstream CrossAttention.forward)
 * v_ones_col != 0 (needs d < d_pad): V[:, h*d_pad + d] == 1 for every head — the P.V tensor-core product then also
 * yields the softmax denominators (column d of the accumulator), so no CUDA-core row sums are computed. */
int b200sd_attention(const void* Q, long long ldq, const void* K, long long ldk, const void* V, long long ldv,
                     void* O, long long ldo, int B, int heads, int Sq, int Skv, int d, int d_pad, float scale,
                     int v_ones_col, int dtype, void* stream);
/* b200sd_attention with a key count per batch row: row b attends to keys [0, kv_len[b]) of K/V buffers that are Skv
 * rows long.  kv_len is a DEVICE array of B ints, read by the kernel (one captured graph serves any lengths); each
 * length is clamped to [1, Skv].  Row b is bitwise equal to b200sd_attention on the first kv_len[b] key rows, provided
 * the buffer rows from kv_len[b] up to the next multiple of the key tile (128 when d <= 64, else 64) or Skv hold
 * finite values.  (sdwui evaluates a cond
 * and an uncond context of different lengths in separate UNet calls; this evaluates them in one batch.) */
int b200sd_attention_varlen(const void* Q, long long ldq, const void* K, long long ldk, const void* V, long long ldv,
                            void* O, long long ldo, int B, int heads, int Sq, int Skv, const int* kv_len, int d,
                            int d_pad, float scale, int v_ones_col, int dtype, void* stream);

/* ---- HBM-bound ops ------------------------------------------------------------------------------- */

/* GroupNorm statistics: stats[n][g] = (sum, sumsq) over the group's channels and all HW pixels, bit-reproducible
 * run to run (per-CTA partial sums combined in a fixed order; no floating-point atomics).
 * `stats` holds b200sd_groupnorm_stats_floats() floats: the [NB][G][2] results first, then the kernel's scratch.
 * The buffer must be zero-filled once when it is allocated (the scratch contains arrival counters that the kernel
 * leaves at zero); it may be shared by successive calls on one stream. (upstream GroupNorm32 / Normalize) */
long long b200sd_groupnorm_stats_floats(int NB, int HW, int C, int G);
int b200sd_groupnorm_stats(const void* X, long long pitch, int NB, int HW, int C, int G, float* stats, int dtype,
                           void* stream);
/* Y = (X - mean) * rstd * gamma + beta, optional SiLU; mean/rstd from `stats`. */
int b200sd_groupnorm_apply(const void* X, long long pitch_x, void* Y, long long pitch_y, int NB, int HW, int C, int G,
                           const float* stats, const float* gamma, const float* beta, float eps, int silu, int dtype,
                           void* stream);
/* GroupNorm in one call: b200sd_groupnorm_stats, then b200sd_groupnorm_apply on the same stream.  How the pixels of an
 * image are split between CTAs depends on HW and C only, never on NB, so an image's bits do not depend on the batch it
 * travels in.  `stats` as for b200sd_groupnorm_stats. */
int b200sd_groupnorm(const void* X, long long pitch_x, void* Y, long long pitch_y, int NB, int HW, int C, int G,
                     float* stats, const float* gamma, const float* beta, float eps, int silu, int dtype, void* stream);
/* LayerNorm over the last dim of [rows, C]. (upstream BasicTransformerBlock.norm1/2/3) */
int b200sd_layernorm(const void* X, long long ldx, void* Y, long long ldy, int rows, int C, const float* gamma,
                     const float* beta, float eps, int dtype, void* stream);
/* nearest-neighbour 2x upsample, NHWC. (upstream Upsample before its conv) */
int b200sd_upsample2x(const void* X, long long pitch_x, void* Y, long long pitch_y, int NB, int H, int W, int C,
                      int dtype, void* stream);
/* circular padding, NHWC: X[NB,H,W,C] (pixel pitch pitch_x) -> Y[NB,H+2p,W+2p,C] (pixel pitch pitch_y), the interior X and
 * the halo copied from the opposite edges, as torch.nn.functional.pad(mode="circular").  A pure copy: the output is
 * bitwise defined.  0 <= p <= H and p <= W (H = 1 or W = 1 with p = 1 wraps onto itself); C % 8 == 0.  A circular 3x3
 * conv (sdwui's tiling: padding_mode 'circular' on every Conv2d) is this copy with p = 1, then b200sd_conv2d with
 * pad = pad_end = 0 on Y. */
int b200sd_pad_circular(const void* X, long long pitch_x, void* Y, long long pitch_y, int NB, int H, int W, int C, int p,
                        int dtype, void* stream);
/* row softmax of an fp16/bf16 matrix in place, fp32 math (VAE mid-block attention, d=512 single head).  Any cols >= 1
 * (the VAE calls it with cols = latent pixels: 16384 at 1024^2, 36864 at 1536^2). */
int b200sd_softmax_rows(void* S, long long lds, int rows, int cols, float scale, int dtype, void* stream);
/* Y[rows, C] = silu(X) elementwise (emb_layers SiLU). */
int b200sd_silu(const void* X, void* Y, long long n, int dtype, void* stream);

/* ---- sampler / conditioning / output ------------------------------------------------------------- */

/* sinusoidal timestep embedding (cos first, then sin), out [T][dim] fp16/bf16. (ldm timestep_embedding) */
int b200sd_timestep_embedding(const float* t, int T, int dim, void* out, long long ldo, int dtype, void* stream);
/* table[step][c] (fp32) = conv_bias[c] + emb[step][c]; folds the per-step time embedding into conv biases. */
int b200sd_fold_bias(const void* emb, long long lde, const float* bias, float* table, int T, int C, int dtype,
                     void* stream);
/* cur[0..n) = table[*step_counter][0..n) : selects this sampler step's rows on the device (graph replay safe). */
int b200sd_select_step(const float* table, long long row_len, const int* step_counter, float* cur, void* stream);
/* prompt editing: ctx[row][0..cap) = bank[e][0..entry_len[e]) followed by zeros, and kv_len[row] = entry_len[e], where
 * e = sched[*step_counter][row].  bank [n_entries][cap][ctx_dim] and ctx [rows][cap][ctx_dim] are fp16 or bf16 (a
 * 16-byte copy: the type does not enter), 16-byte aligned, ctx_dim % 8 == 0; sched [*][rows] int32 (the caller keeps
 * its entries in [0, n_entries); out-of-range ones are clamped); entry lengths are clamped to [1, cap].  Reads the
 * step counter on the device like b200sd_select_step (graph replay safe). */
int b200sd_select_context(const void* bank, const int* entry_len, int n_entries, const int* sched,
                          const int* step_counter, void* ctx, int* kv_len, int rows, int cap, int ctx_dim,
                          void* stream);
/* latents fp32 NHWC [B,HW,4] -> UNet input [2B,HW,pitch] (cond half and uncond half identical, channels >= 4
 * untouched: they are zero from allocation) */
int b200sd_pack_unet_input(const float* x, void* xin, long long pitch, int B, int HW, float in_scale, int dtype,
                           void* stream);
/* classifier-free guidance + one DDIM (eta = 0) update, then re-pack the next UNet input and advance
 * *step_counter.  eps [2B,HW,pitch_e] (cond first, uncond second), coef[step] = {sqrt(a_t), sqrt(1-a_t),
 * sqrt(a_prev), sqrt(1-a_prev)}.  (sdwui CFGDenoiser + sd_samplers_timesteps_impl.ddim) */
int b200sd_cfg_ddim_step(const void* eps, long long pitch_e, float* x, void* xin, long long pitch_x, int B, int HW,
                         float cfg_scale, const float* coef, int* step_counter, int dtype, void* stream);
/* Euler-ancestral step on sigma-space latents (k-diffusion sample_euler_ancestral); noise may be NULL when
 * sigma_up == 0.  coef[step] = {sigma, sigma_next_down, sigma_up, in_scale_next}. */
int b200sd_cfg_euler_a_step(const void* eps, long long pitch_e, float* x, const float* noise, void* xin,
                            long long pitch_x, int B, int HW, float cfg_scale, const float* coef, int* step_counter,
                            int dtype, void* stream);
/* DPM-Solver++(2M) step on sigma-space latents (k-diffusion sample_dpmpp_2m; sdwui "DPM++ 2M" / "DPM++ 2M Karras"):
 * old_denoised [B,HW,4] fp32 carries the previous step's x0 prediction (ignored when c2 == 0).
 * coef[step] = {sigma, sigma_next/sigma, c1, c2, in_scale_next, 0, 0, 0} — 8 floats per row. */
int b200sd_cfg_dpmpp_2m_step(const void* eps, long long pitch_e, float* x, float* old_denoised, void* xin,
                             long long pitch_x, int B, int HW, float cfg_scale, const float* coef, int* step_counter,
                             int dtype, void* stream);
/* v-prediction twins of the three fused steps: same arguments; `eps` holds the UNet's v output.  The CFG-combined v is
 * converted with the kernel's own pre-update fp32 x (the point the UNet evaluated), then the eps step runs unchanged.
 *   _ddim_step_v:     same 4-float rows; eps = sqrt(1-a_t) x + sqrt(a_t) v  (sdwui CompVisTimestepsVDenoiser)
 *   _euler_a_step_v:  8-float rows {sigma, sigma_down, sigma_up, in_scale_next, kx, kv, 0, 0}
 *   _dpmpp_2m_step_v: the 8-float rows with kx, kv in columns 5 and 6
 * with kx = sigma/(sigma^2+1), kv = 1/sqrt(sigma^2+1): eps = kx x + kv v is to_d of k-diffusion's CompVisVDenoiser
 * (sigma_data 1) on sigma-space x. */
int b200sd_cfg_ddim_step_v(const void* eps, long long pitch_e, float* x, void* xin, long long pitch_x, int B, int HW,
                           float cfg_scale, const float* coef, int* step_counter, int dtype, void* stream);
int b200sd_cfg_euler_a_step_v(const void* eps, long long pitch_e, float* x, const float* noise, void* xin,
                              long long pitch_x, int B, int HW, float cfg_scale, const float* coef, int* step_counter,
                              int dtype, void* stream);
int b200sd_cfg_dpmpp_2m_step_v(const void* eps, long long pitch_e, float* x, float* old_denoised, void* xin,
                               long long pitch_x, int B, int HW, float cfg_scale, const float* coef, int* step_counter,
                               int dtype, void* stream);
/* ---- generic sampler building blocks: every sampler of the reference's ETA table (scripts/spartan/worker.py:75-94)
 * beyond the four fused ones above is, per model evaluation, one b200sd_cfg_eps plus a few b200sd_latent_lincomb on
 * fp32 NHWC latents [B,HW,4], with coefficient rows selected on the device by *step_counter (graph replay safe). */
/* e = eps_uncond + cfg_scale * (eps_cond - eps_uncond), fp32 [B,HW,4].  (sdwui CFGDenoiser; equals k-diffusion
 * to_d(x, sigma, denoised) for the eps-prediction CompVisDenoiser.  For a v-prediction model this is the CFG-combined v,
 * and one b200sd_latent_lincomb e = kx x + kv e converts it to eps.) */
int b200sd_cfg_eps(const void* eps, long long pitch_e, float* e, int B, int HW, float cfg_scale, int dtype, void* stream);
/* dst = sum_{k<n_src} c[k] * srcs[k], c = coef + (*step_counter) * ld + col0.  srcs / idx_strides are HOST arrays of
 * n_src (<= 8) device pointers / element strides: a source with idx_strides[k] != 0 is a stack of tensors and tensor
 * (int)coef[(*step_counter) * ld + idx_col] of it is read (per-step noise draws).  xin != NULL: dst * c[n_src] is also
 * packed as the next UNet input [2B,HW,pitch_x].  dst may alias a source. */
int b200sd_latent_lincomb(float* dst, const float* const* srcs, const long long* idx_strides, int n_src,
                          const float* coef, int ld, int col0, int idx_col, const int* step_counter, void* xin,
                          long long pitch_x, int B, int HW, int dtype, void* stream);
/* *step_counter += 1 on the device. */
int b200sd_bump_step(int* step_counter, void* stream);
/* decoded image [B,HW,pitch] (first 3 channels RGB in [-1,1]) -> uint8 [B,HW,3]:
 * trunc(255 * clamp((v+1)/2, 0, 1))  (sdwui process_images_inner) */
int b200sd_quantize_u8(const void* img, long long pitch, unsigned char* out, int B, int HW, int dtype, void* stream);

/* img2img input: uint8 [B,HW,3] RGB -> [B,HW,pitch] with channel c < 3 = 2*x/255 - 1 (channels >= 3 untouched: zero
 * from allocation).  (sdwui StableDiffusionProcessingImg2Img.init) */
int b200sd_image_to_nhwc(const unsigned char* img, void* out, long long pitch, int B, int HW, int dtype, void* stream);
/* ControlNet hint: uint8 [B,HW,3] RGB -> [B,HW,pitch] with channel c < 3 = x/255 and channels 3..pitch-1 = 0 (ldm
 * ControlNet input_hint_block input, sd-webui-controlnet's HWC3(image) / 255).  Not 2x/255 - 1: the hint block's zero
 * padding at the image borders must stand for black. */
int b200sd_hint_to_nhwc(const unsigned char* img, void* out, long long pitch, int B, int HW, int dtype, void* stream);
/* inpainting-model conditioning image: uint8 [B,HW,3] RGB and mask uint8 [HW] (NULL: all ones) -> [B,HW,pitch] with
 * channel c < 3 = (2*x/255 - 1) * (1 - weight * [mask >= 128]) (channels >= 3 untouched).  sdwui
 * inpainting_image_conditioning: torch.lerp(s, s * (1 - M), inpainting_mask_weight), M = round(mask / 255).  Where the mask
 * is 0 the output is bitwise b200sd_image_to_nhwc's. */
int b200sd_masked_image_to_nhwc(const unsigned char* img, const unsigned char* mask, float weight, void* out,
                                long long pitch, int B, int HW, int dtype, void* stream);
/* inpainting-model UNet input: z fp32 [B,h*w,4] (VAE latents of the conditioning image) and the pixel mask uint8
 * [f*h, f*w] (NULL: all ones) -> channel 4 = [mask[f*i, f*j] >= 128] (nearest F.interpolate to the latent size) and
 * channels 5..8 = z of rows b and B+b of xin [2B,h*w,pitch] ([cond | uncond]).  No other channel is touched.
 * pitch >= 9 and pitch % 4 == 0, z 16-byte and xin 8-byte aligned. */
int b200sd_pack_image_cond(const float* z, const unsigned char* mask, void* xin, long long pitch, int B, int h, int w,
                           int f, int dtype, void* stream);
/* VAE encoder moments [B,HW,pitch] (first 4 channels = posterior mean) -> scaled latents fp32 [B,HW,4] = mean * scale
 * (AutoencoderKL.encode(...).mean * scale_factor) */
int b200sd_unpack_latent(const void* moments, long long pitch, float* x, int B, int HW, float scale, int dtype,
                         void* stream);
/* hires fix, "Latent" upscaler: fp32 NHWC latents [B,H*W,4] -> [B,Ho*Wo,4], bilinear, half-pixel centres, no antialias
 * (torch.nn.functional.interpolate(mode="bilinear") in sdwui StableDiffusionProcessingTxt2Img.sample_hr_pass) */
int b200sd_resize_latent_bilinear(const float* x, float* y, int B, int H, int W, int Ho, int Wo, void* stream);
/* hires fix, the other "Latent (...)" upscalers: fp32 NHWC latents [B,H*W,4] -> [B,Ho*Wo,4] by separable DEVICE tables:
 * y[b,oy,ox] = sum_j wy[oy*ky+j] * (sum_i wx[ox*kx+i] * x[b, iy[oy*ky+j], ix[ox*kx+i]]), sums in tap order.  The host
 * builds the tables of F.interpolate's nearest, nearest-exact, bicubic (A = -0.75, clamped taps) and antialiased
 * bilinear / bicubic modes; unused taps carry weight 0 and a valid index. */
int b200sd_resize_latent_table(const float* x, float* y, int B, int H, int W, int Ho, int Wo, const int* ix,
                               const float* wx, int kx, const int* iy, const float* wy, int ky, void* stream);

/* ---- hires fix pixel upscalers (sdwui images.resize_image / upscaler_utils.upscale_with_model) ---------------------- */
/* one pass of Pillow's ImagingResample on RGB uint8 [B,Hin,Win,3] -> [B,Hout,Wout,3] along x (vertical = 0: Hout == Hin)
 * or y (vertical = 1: Wout == Win).  bounds [out][2] = {first input, count} and kk [out][ksize] are Pillow's fixed-point
 * coefficients (22 fraction bits), DEVICE arrays; out = clip8((1 << 21 + sum in * kk) >> 22).  Pillow resizes
 * horizontally first and skips a pass whose size does not change; a NEAREST resize is the same two passes with one
 * tap of weight 1 << 22 at Pillow's nearest source index. */
int b200sd_resample_u8(const unsigned char* in, unsigned char* out, int B, int Hin, int Win, int Hout, int Wout,
                       int vertical, const int* bounds, const int* kk, int ksize, void* stream);
/* sdwui images.combine_grid: upscaled tiles uint8 [B*rows*cols, th, tw, 3] (row-major per image) -> [B,H,W,3].  Tile (r,c)
 * sits at (xs[c], ys[r]) (DEVICE arrays, may be negative); within a row each tile not at x == 0 blends its first
 * `overlap` columns over the row through mask[column] with Pillow's paste-with-mask integer arithmetic, then the rows
 * are stacked the same way through mask[row]; bitwise equal to the sequence of PIL pastes. */
int b200sd_combine_tiles_u8(const unsigned char* tiles, unsigned char* out, int B, int H, int W, int th, int tw,
                            int rows, int cols, const int* ys, const int* xs, const unsigned char* mask, int overlap,
                            void* stream);
/* ESRGAN output [B,HW,pitch] (channels 0..2 nominally in [0,1]) -> uint8 [B,HW,3] = round_half_even(255 * clamp(v, 0, 1))
 * (sdwui torch_bgr_to_pil_image; not the truncating b200sd_quantize_u8 of VAE images).  dtype B200SD_F16 only. */
int b200sd_quantize_unit_u8(const void* img, long long pitch, unsigned char* out, int B, int HW, int dtype, void* stream);
/* Y[r, c] += alpha * X[r, c] for c < C, fp32 math (basicsr RRDB: x + 0.2 * rdb3(...)).  dtype B200SD_F16 only. */
int b200sd_scaled_add(const void* X, long long pitch_x, void* Y, long long pitch_y, long long rows, int C, float alpha,
                      int dtype, void* stream);

/* inpainting: x[b,p,:] = x[b,p,:] * latmask[p] + init[b,p,:] * (1 - latmask[p]) on fp32 NHWC latents [B,HW,4]; latmask [HW]
 * is the request's latent-resolution mask (1 = repaint).  (sdwui CFGDenoiser.apply_blend, before every model call of the
 * timestep samplers, and once more after sampling) */
int b200sd_blend_latent(float* x, const float* init, const float* latmask, int B, int HW, void* stream);

/* ---- token merging (tomesd bipartite soft matching on the 2x2 grid, as sdwui's token_merging_ratio applies it to the
 * self-attention of the UNet's full-resolution transformer blocks).  fp16 only: bf16 is B200SD_ERR_UNSUPPORTED.
 * Tokens of a batch row are the H*W latent pixels t = y*W + x (H, W even); the top-left token of every 2x2 block is a
 * dst token (index j = (y/2)*(W/2) + x/2), the other Ns = 3/4 N are src tokens, numbered in ascending token order.
 * A merged sequence of Nm = N - r slots: slots [0, Ns - r) are the unmerged src tokens in ascending token order, slot
 * Ns - r + j is dst token j with the src tokens merged into it. */
/* bytes of the caller-owned workspace b200sd_tome_match takes (-1: unsupported shape; C must be 64 or 320) */
long long b200sd_tome_match_workspace_bytes(int B, int H, int W, int C);
/* matching of X [B,H*W,C] (row pitch `pitch`), per batch row: metric = X / ||X|| rounded to fp16; for every src token
 * a, node_max / node_idx = max / argmax over dst b of metric_a . metric_b (fp32 accumulation, ties to the lowest dst
 * index; a fused wgmma kernel, no score matrix is stored); the r src tokens with the largest (node_max desc, src index
 * asc) keys are merged into their node_idx dst (1 <= r <= Ns).  Outputs int32: slot [B][N] (the slot of every token),
 * members [B][N] (tokens ordered by slot, ascending within a slot), seg [B][Nm+1] (slot s holds members[seg[s] ..
 * seg[s+1])). */
int b200sd_tome_match(const void* X, long long pitch, int B, int H, int W, int C, int r, int* slot, int* members,
                      int* seg, void* workspace, long long workspace_bytes, int dtype, void* stream);
/* Y[b,s,:] = mean of X[b,t,:] over the members t of slot s: fp32 sum in ascending token order, divided by the count and
 * rounded once (tomesd merge: scatter_reduce "mean", include_self).  X [B,N,C], Y [B,Nm,C]; C % 8 == 0. */
int b200sd_tome_merge(const void* X, long long pitch_x, const int* members, const int* seg, void* Y, long long pitch_y,
                      int B, int N, int Nm, int C, int dtype, void* stream);
/* out[b,t,:] = round(R[b,t,:] + Y[b, slot[b,t], :]) (tomesd unmerge, then the block's residual add).  R, out [B,N,C],
 * Y [B,Nm,C]. */
int b200sd_tome_unmerge_add(const void* R, long long pitch_r, const void* Y, long long pitch_y, const int* slot,
                            void* out, long long pitch_o, int B, int N, int Nm, int C, int dtype, void* stream);

/* ---- LoRA networks merged into packed weights (sdwui networks.py network_apply_weights, `<lora:name:te:unet>`) ---- */
/* One target: W[rows, cols] (row pitch ldw elements, fp16 / bf16) is rewritten from its pristine copy P (same layout and
 * pitch) as W[i,k] = round_rn(P[i,k] + s), s = sum_{j < R} U[i,j] * D[j,k] accumulated in fp32 by fmaf in ascending j
 * from 0 (bitwise the same on every device and run, whatever the tiling); where s == 0 (R == 0: a restore; a zero row of
 * U) W = P bitwise.  U [rows, R] and D [R, cols] are fp32, row-major and dense.  W must not overlap P, U or D. */
typedef struct b200sd_lora_target {
  void* W;
  const void* P;
  const float* U;
  const float* D;
  long long ldw;
  int rows, cols, R;
  int reserved; /* 0 */
} b200sd_lora_target;
/* every target of the DEVICE-resident table targets[n_targets] in one persistent launch (register-tiled fp32 FMA; the
 * rank loops in chunks of 32).  Targets must not overlap each other's W. */
int b200sd_lora_merge(const b200sd_lora_target* targets, int n_targets, int dtype, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200SD_H_ */
