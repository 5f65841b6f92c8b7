/* libmarigold_b200 — C ABI of the H100-native (sm_90a) Marigold denoising hot path.
 *
 * The reference (prs-eth/Marigold) has no FFI: its hot path is the Python object protocol
 *   vae.encoder / vae.quant_conv            marigold/marigold_depth_pipeline.py:491-492
 *   scheduler.set_timesteps / .timesteps    marigold/marigold_depth_pipeline.py:423-424
 *   unet(x, t, encoder_hidden_states)       marigold/marigold_depth_pipeline.py:461-463
 *   scheduler.step(...).prev_sample         marigold/marigold_depth_pipeline.py:466-468
 *   vae.post_quant_conv / vae.decoder       marigold/marigold_depth_pipeline.py:512-513
 *   ensemble_depth / ensemble_normals       marigold/util/ensemble.py:39,199
 * Each entry point below names the call(s) it replaces. INTEGRATION.md shows the ctypes stub.
 *
 * Conventions
 *   - Every pointer named *_dev is a CUDA device pointer owned by the caller; image-like tensors
 *     are contiguous NCHW fp32 (the reference's layout). NHWC/bf16 is an internal detail.
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it and the call returns
 *     without synchronising unless stated otherwise.
 *   - Every function returns 0 (MGB_OK) or a negative mgb_status; mgb_last_error() has the text.
 *   - A handle is not thread-safe: one handle per process per GPU.
 *   - There is no CPU fallback anywhere behind this ABI.
 */
#ifndef MARIGOLD_B200_H_
#define MARIGOLD_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  MGB_OK = 0,
  MGB_ERR_INVALID = -1,      /* bad argument (shape, null pointer, unknown key ...) */
  MGB_ERR_CUDA = -2,         /* a CUDA runtime/driver call failed */
  MGB_ERR_STATE = -3,        /* call order violated (e.g. denoise before finalize_weights) */
  MGB_ERR_NOMEM = -4,
  MGB_ERR_UNSUPPORTED = -5   /* valid request this build does not implement */
} mgb_status;

typedef enum { MGB_F32 = 0, MGB_BF16 = 1, MGB_F16 = 2 } mgb_dtype;
typedef enum { MGB_DECODE_DEPTH = 0, MGB_DECODE_NORMALS = 1, MGB_DECODE_RAW3 = 2, MGB_DECODE_UNIT3 = 3 } mgb_decode_mode;

typedef struct mgb_handle mgb_handle;

/* Architecture description (diffusers config.json fields; SURVEY.md App. A).
 * Channel counts must be multiples of 64; attention head_dim is 64 (SD-2: "attention_head_dim"
 * there is a head COUNT, C/64). */
typedef struct {
  int32_t unet_in_channels;        /* 8 = rgb latent (4) | target latent (4); IID with n targets: 4 (n + 1) */
  int32_t unet_out_channels;       /* 4; IID: 4 n (n <= 4)                                          */
  int32_t unet_block_channels[4];  /* 320, 640, 1280, 1280                                          */
  int32_t unet_layers_per_block;   /* 2                                                             */
  int32_t unet_cross_dim;          /* 1024                                                          */
  int32_t vae_block_channels[4];   /* 128, 256, 512, 512                                            */
  int32_t vae_layers_per_block;    /* 2                                                             */
  int32_t vae_latent_channels;     /* 4                                                             */
  int32_t norm_groups;             /* 32                                                            */
  float latent_scale;              /* 0.18215 (marigold_depth_pipeline.py:118)                      */
} mgb_config;

/* ---- lifecycle ------------------------------------------------------------------------------ */
int mgb_create(const mgb_config* cfg, mgb_handle** out);
void mgb_destroy(mgb_handle* h);
const char* mgb_last_error(void);
/* library build info: "libmarigold_b200 sm_90a: wgmma ..." */
const char* mgb_build_info(void);

/* ---- weights (replaces DiffusionPipeline.from_pretrained state-dict loading) ---------------- */
/* `key` is the diffusers state-dict name prefixed by the sub-model: "unet.conv_in.weight",
 * "vae.decoder.mid_block.attentions.0.to_q.bias", ... `data` is a HOST pointer, contiguous,
 * in the PyTorch layout ([out,in,kh,kw] conv, [out,in] linear). */
int mgb_load_tensor(mgb_handle* h, const char* key, const void* data, const int64_t* shape, int32_t ndim,
                    int32_t dtype);
/* Repack to kernel layouts (bf16, tap-major conv weights, fused QKV, GEGLU-interleaved FF) and
 * verify that every tensor the architecture needs was loaded. */
int mgb_finalize_weights(mgb_handle* h);

/* ---- conditioning --------------------------------------------------------------------------- */
/* Empty-prompt embedding [n_tokens, cross_dim] fp32 HOST (marigold_depth_pipeline.py:381-394,
 * 438-442; n_tokens == 2). Cross-attention K/V of every block are folded here, once.
 * A call rejected for its arguments changes nothing; a call that fails after that leaves no embedding set, so
 * denoising returns MGB_ERR_STATE until a later call succeeds. */
int mgb_set_text_embedding(mgb_handle* h, const float* embed_host, int32_t n_tokens);

/* scheduler.set_timesteps + the per-step coefficients of scheduler.step, computed by the host in
 * float64 (marigold_b200/schedulers.py) so scheduler-config handling stays in Python:
 *     x_prev = kx[i] * x + kv[i] * model_output + kz[i] * noise_i
 * (DDIM eta=0: kz = 0; LCM: kz != 0 on every step but the last). All arrays have n entries.
 * A call that fails for any reason leaves the previous schedule in place and usable. */
int mgb_set_schedule(mgb_handle* h, int32_t n, const int32_t* timesteps, const float* kx, const float* kv,
                     const float* kz);

/* ---- the hot path --------------------------------------------------------------------------- */
/* encode_rgb: vae.encoder + quant_conv, mean half, * latent_scale  (…pipeline.py:479-496).
 * rgb_dev [B,3,H,W] in [-1,1]; latent_dev [B,4,H/8,W/8] (floor). Any H, W >= 8: like the reference, sizes that are not
 * multiples of 8 lose the remainder rows / columns in the VAE's stride-2 convs.
 * Supported maximum (this call and mgb_decode): B * H * W <= 2^26 pixels (one 8192 x 8192 image); larger batches return
 * MGB_ERR_UNSUPPORTED before anything is allocated or launched. */
int mgb_encode(mgb_handle* h, const float* rgb_dev, int32_t B, int32_t H, int32_t W, float* latent_dev,
               void* stream);
/* One denoising iteration i: cat -> unet -> scheduler.step (…pipeline.py:456-468).
 * target_dev [B,Ct,h,w] (Ct = unet_out_channels: 4, or 4 n for an n-target IID model, marigold_iid_pipeline.py:538-551)
 * is updated in place; noise_dev (or NULL) is this step's z; if model_out_dev != NULL it also receives the raw UNet
 * output [B,Ct,h,w]. Any h, w >= 1 (odd sizes follow diffusers' `upsample_size` path). */
int mgb_unet_step(mgb_handle* h, const float* rgb_latent_dev, float* target_dev, const float* noise_dev,
                  float* model_out_dev, int32_t step_index, int32_t B, int32_t lh, int32_t lw, void* stream);
/* The whole loop (…pipeline.py:455-468): steps 0..n-1 of the current schedule.
 * step_noise_dev: [n-1, B, Ct, h, w] or NULL (required when any kz != 0). */
int mgb_denoise(mgb_handle* h, const float* rgb_latent_dev, float* target_dev, const float* step_noise_dev,
                int32_t B, int32_t lh, int32_t lw, void* stream);
/* Steps [first_step, first_step + num_steps) of the current schedule only (bench.py times K steps of a
 * longer schedule with it). step_noise_dev is indexed by absolute step: [n-1, B, 4, h, w]. */
int mgb_denoise_range(mgb_handle* h, const float* rgb_latent_dev, float* target_dev, const float* step_noise_dev,
                      int32_t first_step, int32_t num_steps, int32_t B, int32_t lh, int32_t lw, void* stream);
/* decode_depth / decode_normals + the clip / shift / normalise that follow
 * (…depth_pipeline.py:498-516,473-475; …normals_pipeline.py:463-479,438-440).
 * out_dev: DEPTH [B,1,H,W] in [0,1]; NORMALS [B,3,H,W] unit vectors; RAW3 [B,3,H,W]; UNIT3 [B,3,H,W] = (clip(x,-1,1)+1)/2
 * (one IID target, marigold_iid_pipeline.py:562-565,578-585: the caller loops over the targets' 4-channel slices).
 * B * 8 lh * 8 lw output pixels within the supported maximum of mgb_encode. */
int mgb_decode(mgb_handle* h, const float* latent_dev, int32_t B, int32_t lh, int32_t lw, int32_t mode,
               float* out_dev, void* stream);

/* ---- one image on several GPUs: the attentions' query rows split over the ranks --------------- */
/* Exchange of one attention's output: buf_dev holds world chunks of chunk_bytes; on entry chunk `rank` holds this rank's
 * rows. On return (in stream order) every chunk must hold its rank's rows: an in-place all-gather. Runs on `stream`, the
 * call's stream. Returns 0, or a non-zero status that fails the call. */
typedef int32_t (*mgb_exchange_fn)(void* ctx, void* buf_dev, size_t chunk_bytes, int32_t rank, int32_t world,
                                   void* stream);
/* Row-split mode of this handle. With fn installed, every attention of mgb_encode, mgb_unet_step, mgb_denoise(_range) and
 * mgb_decode computes only this rank's share of its query rows, then calls fn once with the attention's output (16 calls
 * per UNet step, one per encode, one per decode): of T rows, chunk = ceil(ceil(T / 128) / world) * 128 rows per rank,
 * rank r's rows [r chunk, (r + 1) chunk) within [0, T) (a rank may have none; it still calls fn). Every other layer runs
 * whole on every rank, so when every rank runs the same call with the same inputs, every rank's outputs are
 * bit-identical to the same call without the split. fn is called even at world 1. While installed, the calls take
 * B = 1 only (MGB_ERR_INVALID before any launch otherwise), and denoising runs each step eagerly: no CUDA graph is
 * captured or replayed. fn = NULL clears the mode; the handle then runs, sizes and lays out its work exactly as one that
 * never had it. MGB_ERR_INVALID for world < 1 or rank outside [0, world). */
int mgb_set_row_split(mgb_handle* h, int32_t rank, int32_t world, mgb_exchange_fn fn, void* ctx);

/* ---- ensembling (marigold/util/ensemble.py) ------------------------------------------------- */
/* cost_fn of ensemble_depth (ensemble.py:138-152) at one point, in ONE host sync:
 * depth_dev [E,HW] fp32; param_host = [s_0..s_{E-1}, t_0..t_{E-1}] (or only s when !shift);
 * returns sum_{i<j} RMSE(a_i - a_j) + reg * (|min(med)| + |1 - max(med)|). Synchronises. */
int mgb_ens_depth_cost(mgb_handle* h, const float* depth_dev, const double* param_host, int32_t E, int64_t HW,
                       int32_t scale_invariant, int32_t shift_invariant, int32_t reduction_median,
                       double regularizer, double* cost_out, void* stream);
/* That objective and the points of one forward-difference gradient in ONE host sync (scipy approx_derivative as BFGS
 * calls it, ensemble.py:165-171): base_host [n] is the current point, pert_host [n] the same vector with EVERY
 * coordinate moved to its perturbed value x_i + h_i; costs_out_host [1 + n]: [0] = cost(base), [1 + i] = cost(base with
 * coordinate i perturbed), each bit-identical to mgb_ens_depth_cost of that vector. n = 2E (or E when !shift); any E
 * from 1 (no pairs: the regulariser alone) to mgb_ens_max_members(). */
int mgb_ens_depth_cost_fd(mgb_handle* h, const float* depth_dev, const double* base_host, const double* pert_host,
                          int32_t E, int64_t HW, int32_t scale_invariant, int32_t shift_invariant,
                          int32_t reduction_median, double regularizer, double* costs_out_host, void* stream);
/* Largest ensemble size the ensembling entry points accept (sizes <= 16 run register-resident kernels). */
int mgb_ens_max_members(void);
/* init_param statistics (ensemble.py:91-105): per-member min and max. Synchronises. */
int mgb_ens_minmax(mgb_handle* h, const float* depth_dev, int32_t E, int64_t HW, float* min_host, float* max_host,
                   void* stream);
/* align + ensemble + min-max renormalise (ensemble.py:178-196). pred_dev [HW]; uncert_dev [HW] or NULL.
 * member_idx_dev (int32 [HW] or NULL) receives the index of the member picked by the (lower) median. */
int mgb_ens_depth_reduce(mgb_handle* h, const float* depth_dev, const double* param_host, int32_t E, int64_t HW,
                         int32_t scale_invariant, int32_t shift_invariant, int32_t reduction_median,
                         float* pred_dev, float* uncert_dev, int32_t* member_idx_dev, void* stream);
/* ensemble_normals (ensemble.py:199-249): normals_dev [E,3,HW]; out_dev [3,HW]; uncert_dev [HW] or NULL;
 * member_idx_dev int32 [HW] or NULL = argmax index. reduction_closest: 1 = "closest", 0 = "mean". */
int mgb_ens_normals(mgb_handle* h, const float* normals_dev, int32_t E, int64_t HW, int32_t reduction_closest,
                    float* out_dev, float* uncert_dev, int32_t* member_idx_dev, void* stream);

/* ensemble_iid (ensemble.py:252-270): targets_dev [E, N] (N = 3 n H W) -> pred_dev [N] = lower median (or mean) over the
 * members; uncert_dev [N] or NULL = median absolute deviation (or unbiased std). No alignment, no renormalisation. */
int mgb_ens_iid(mgb_handle* h, const float* targets_dev, int32_t E, int64_t N, int32_t reduction_median, float* pred_dev,
                float* uncert_dev, void* stream);

/* ---- pre / post-processing bookends and the evaluation step ------------------------------------ */
/* torchvision resize(antialias=True) as resize_max_res calls it (marigold/util/image_util.py:90-120) and for the final
 * prediction (marigold_depth_pipeline.py:306-312). src_dev [NC,H,W] uint8 (src_is_u8) or fp32 -> dst_dev fp32 [NC,h,w].
 * mode 0 bilinear, 1 bicubic (both antialiased), 2 nearest-exact. arith selects whose arithmetic the antialiased modes
 * reproduce bit for bit (tap windows, weights and accumulation): 0 torch's CPU kernel (the reference resizes the image
 * on the host), 1 torch's CUDA kernel (the reference resizes the prediction on the device).
 * post 0: none; 1: clamp to [0,255] and round half to even (a uint8 image stays uint8-valued); 2: that, then x / 255 * 2 - 1 with a true division
 * (marigold_depth_pipeline.py:252 on the host); 3: x / 255 * 2 - 1 alone (a float image). tmp_dev: NC*H*w floats. */
int mgb_resize_ex(const void* src_dev, int32_t src_is_u8, int32_t NC, int32_t H, int32_t W, float* dst_dev, int32_t h,
                  int32_t w, int32_t mode, int32_t arith, int32_t post, float* tmp_dev, void* stream);
/* colorize_depth_maps + chw2hwc + uint8 (image_util.py:38-76, marigold_depth_pipeline.py:326-331): depth_dev fp32 [HW] ->
 * out_hwc_dev uint8 [HW,3]; lut_dev uint8 [256,3] = the colour map's 256-entry table * 255, truncated. */
int mgb_colorize(const float* depth_dev, int64_t HW, float dmin, float dmax, const uint8_t* lut_dev, uint8_t* out_hwc_dev,
                 void* stream);
/* Least-squares scale / shift alignment to the ground truth over the valid pixels (src/util/alignment.py:35-82), the
 * clips of script/depth/eval.py:201-207 and the masked depth metrics of src/util/metric.py:64-191 in two passes and ONE
 * synchronisation. mask_dev uint8 [HW] or NULL; aligned_out_dev fp32 [HW] or NULL; ws_dev: mgb_eval_ws_bytes() bytes.
 * out_host[13] = {scale, shift, n_valid, abs_rel, sq_rel, rmse, rmse_log, log10, delta1, delta2, delta3, i_rmse, silog}.
 * NaN metrics when n_valid == 0; scale = shift = 0 when the fit has no pixel (np.linalg.lstsq of no rows). */
size_t mgb_eval_ws_bytes(void);
int mgb_eval_depth(const float* pred_dev, const float* gt_dev, const uint8_t* mask_dev, int64_t HW, int32_t least_squares,
                   float dmin, float dmax, float* aligned_out_dev, void* ws_dev, double* out_host, void* stream);
/* mgb_eval_depth with every alignment of script/depth/eval.py:171-207 (same workspace, same out_host[13]). alignment: 0 none,
 * 1 least_square, 2 least_square_disparity (:179-199: fit pred to 1 / gt over valid & gt > 0 & pred > 0, clip the aligned
 * disparity to >= 1e-3 and take its reciprocal before the dataset clip). The metrics always use mask_dev. fit_rows_dev /
 * fit_cols_dev: int32 [fit_h] / [fit_w] source row / column of each pixel of the downsampled maps the fit uses
 * (align_depth_least_square's max_resolution, src/util/alignment.py:48-59), or both NULL to fit at full resolution. */
int mgb_eval_depth_ex(const float* pred_dev, const float* gt_dev, const uint8_t* mask_dev, int32_t H, int32_t W,
                      int32_t alignment, const int32_t* fit_rows_dev, const int32_t* fit_cols_dev, int32_t fit_h, int32_t fit_w,
                      float dmin, float dmax, float* aligned_out_dev, void* ws_dev, double* out_host, void* stream);
/* Surface-normals evaluation of one sample (script/normals/eval.py:145-157): the angular error of compute_cosine_error(
 * masked=True) (src/util/metric.py:194-219) and the metrics of metric.py:222-257, in four launches and ONE synchronisation.
 * pred_dev, gt_dev fp32 [3,H,W]; a pixel is valid where ||gt|| > 0 and mask_dev (uint8 [H,W], or NULL) is non-zero.
 * error_out_dev: fp32 [H,W] angular error in degrees, NaN where not valid, or NULL. ws_dev: mgb_eval_normals_ws_bytes(H*W).
 * out_host[9] = {n_valid, mean, median (np.median of the errors, exact), rmse, sub5, sub7.5, sub11.25, sub22.5, sub30}
 * (percentages, unrounded); NaN metrics when n_valid == 0. Deterministic: equal inputs give equal bits. */
size_t mgb_eval_normals_ws_bytes(int64_t HW);
int mgb_eval_normals(const float* pred_dev, const float* gt_dev, const uint8_t* mask_dev, int32_t H, int32_t W,
                     float* error_out_dev, void* ws_dev, double* out_host, void* stream);
/* Intrinsic-image evaluation of one (sample, target) pair: compute_iid_metric (src/util/metric.py:263-338) as
 * script/iid/eval.py:182-213 calls it, for PSNR and SSIM (torchmetrics, data_range 1), in ONE synchronisation (the
 * reference does a torch.linalg.lstsq, a torch.quantile read back with float(), one .item() per metric and a 121-tap
 * grouped conv2d over five stacked maps). pred_dev, gt_dev fp32 [3,H,W]; mask_dev uint8 [3,H,W] (per channel) or NULL.
 *   transform (applied to both maps first): 0 none, 1 x ** 2.2 (srgb2linear), 2 x ** (1/2.2) (linear2srgb)
 *   up_to_scale (shading, residual; metric.py:266-270): s = lstsq of the masked elements of all three channels
 *     (sum pg / sum p^2, 0 when sum p^2 == 0), pred = s * pred; q = torch.quantile(brightness, 0.9) of
 *     0.3 g0 + 0.59 g1 + 0.11 g2 over the pixels valid in mask channel 0 (float32 rank fl(0.9 (n-1)), exact order
 *     statistics, torch's lerp; NaN if any brightness is NaN); k = 0 if q < 1e-4 else fl(fl(1 / q) * 0.8) (torch's
 *     0.8 / q); gt = clamp(k gt, 0, 1), pred = clamp(k pred, 0, 1)
 *   PSNR = 10 log10(1 / (SSE / n)) over the masked elements (all 3HW without a mask); +inf when SSE = 0, NaN when n = 0
 *   SSIM: invalid elements set to 0, Gaussian sigma 1.5 (11 taps), c1 = 0.01^2, c2 = 0.03^2, variances clamped at 0,
 *     the mean over the 3 (H-10)(W-10) windows inside the image (torchmetrics pads by reflection and crops 5 per side)
 * ws_dev: mgb_eval_iid_ws_bytes(H, W). out_host[6] = {n_valid (masked elements), psnr, ssim, s, q, k}; s = k = 1,
 * q = NaN when !up_to_scale. MGB_ERR_INVALID for H or W < 11, and for up_to_scale with no pixel valid in mask channel 0
 * (torch.quantile of an empty tensor raises). Deterministic: equal inputs give equal bits. */
size_t mgb_eval_iid_ws_bytes(int32_t H, int32_t W);
int mgb_eval_iid(const float* pred_dev, const float* gt_dev, const uint8_t* mask_dev, int32_t H, int32_t W,
                 int32_t up_to_scale, int32_t transform, void* ws_dev, double* out_host, void* stream);
/* LPIPS weights: torchmetrics' LearnedPerceptualImagePatchSimilarity(net_type="alex"). conv_w[l], conv_b[l]: host fp32
 * torchvision alexnet().features.{0,3,6,8,10} weight [Cout, Cin, k, k] and bias [Cout]; conv_w_shape[l]: that weight's
 * shape; lin_w[l]: host fp32 lin{l}.model.1.weight [1, Cout, 1, 1] of lin_channels[l] elements. The handle owns bf16
 * copies of the convolutions (conv1 repacked for the factor-4 space-to-depth operand) and fp32 lin weights.
 * MGB_ERR_INVALID for any shape but AlexNet's (64x3x11x11, 192x64x5x5, 384x192x3x3, 256x384x3x3, 256x256x3x3). */
typedef struct mgb_lpips mgb_lpips;
int mgb_lpips_create(const float* const conv_w[5], const int32_t conv_w_shape[5][4], const float* const conv_b[5],
                     const float* const lin_w[5], const int32_t lin_channels[5], mgb_lpips** out);
/* LPIPS weights of any of torchmetrics' three backbones (net_type "alex", "vgg", "squeeze"). conv_w[i], conv_b[i]: host
 * fp32 weight [Cout, Cin, k, k] and bias [Cout] of the net's i-th convolution in torchvision's order, conv_w_shape[4 i ..
 * 4 i + 3] that weight's shape; lin_w[l]: host fp32 lin{l}.model.1.weight of lin_channels[l] elements.
 *   MGB_LPIPS_ALEX     5 convs:  alexnet().features.{0,3,6,8,10}; 5 lin layers of 64, 192, 384, 256, 256 channels
 *   MGB_LPIPS_VGG      13 convs: vgg16().features.{0,2,5,7,10,12,14,17,19,21,24,26,28}; 5 lin layers of 64, 128, 256, 512,
 *                      512 channels (relu1_2, relu2_2, relu3_3, relu4_3, relu5_3)
 *   MGB_LPIPS_SQUEEZE  25 convs: squeezenet1_1().features.0, then features.{3,4,6,7,9,10,11,12}.{squeeze, expand1x1,
 *                      expand3x3}; 7 lin layers of 64, 128, 256, 384, 384, 512, 512 channels
 * MGB_ERR_INVALID for an unknown net_type and for any count or shape but the net's. mgb_lpips_create is this call with
 * MGB_LPIPS_ALEX. */
typedef enum { MGB_LPIPS_ALEX = 0, MGB_LPIPS_VGG = 1, MGB_LPIPS_SQUEEZE = 2 } mgb_lpips_net_type;
int mgb_lpips_create_net(int32_t net_type, int32_t n_conv, const float* const* conv_w, const int32_t* conv_w_shape,
                         const float* const* conv_b, int32_t n_lin, const float* const* lin_w, const int32_t* lin_channels,
                         mgb_lpips** out);
void mgb_lpips_destroy(mgb_lpips* h);
/* The smallest H (and W) for which every tapped layer of the net is non-empty: 31 (AlexNet), 16 (VGG16), 17 (SqueezeNet
 * 1.1); 0 for an unknown net_type. */
int32_t mgb_lpips_min_size(int32_t net_type);
/* Workspace of mgb_eval_iid_lpips with the AlexNet weights (it includes mgb_eval_iid's); 0 when H or W < 31. */
size_t mgb_lpips_ws_bytes(int32_t H, int32_t W);
/* Workspace of mgb_eval_iid_lpips with the weights h; 0 when H or W is below the net's minimum size. */
size_t mgb_lpips_ws_bytes_h(const mgb_lpips* h, int32_t H, int32_t W);
/* mgb_eval_iid, then LPIPS of the same maps (compute_iid_metric with "lpips", src/util/metric.py:263-288), in ONE
 * synchronisation. The maps the metric sees are SSIM's (mapped, invalid elements 0); they must lie in [0, 1]
 * (normalize=True), else MGB_ERR_INVALID with torchmetrics' message (a NaN fails). Then 2 x - 1, the scaling layer,
 * the net's conv + ReLU layers and pools (bf16 operands, fp32 accumulation and features), per tapped layer the
 * unit-normalised (x / sqrt(1e-8 + sum x^2)) squared difference weighted by lin and averaged over the pixels, and the
 * float32 sum of the means in layer order. out_host[7] = mgb_eval_iid's six values, then lpips. H, W >= the net's
 * minimum size (mgb_lpips_min_size; 31 for AlexNet, whose second pool needs a 3 x 3 input). ws_dev:
 * mgb_lpips_ws_bytes_h. Deterministic: equal inputs give equal bits; for the targets that are not up to scale, swapping
 * pred and gt gives the same lpips. */
int mgb_eval_iid_lpips(const float* pred_dev, const float* gt_dev, const uint8_t* mask_dev, int32_t H, int32_t W,
                       int32_t up_to_scale, int32_t transform, const mgb_lpips* lpips, void* ws_dev, double* out_host,
                       void* stream);

/* ---- capacity ------------------------------------------------------------------------------- */
/* Bytes of the activation arena the handle holds for images of H x W with B members per batch; 0 beyond the supported
 * maximum of mgb_encode / mgb_decode. */
size_t mgb_workspace_bytes(mgb_handle* h, int32_t B, int32_t H, int32_t W);
/* Bytes of device workspace the handle holds now (activation arena, split-K and barrier scratch); a call that needs more
 * frees it before allocating the larger size. */
size_t mgb_workspace_held_bytes(mgb_handle* h);
/* Number of kernel launches enqueued by this library since creation (for bench.py gpu_launches). Memsets and copies
   are not counted; a replay of a captured CUDA graph counts the kernels the graph holds. */
int64_t mgb_launch_count(void);

/* ---- operator-level entry points (layer parity tests; tests/test_ops_gpu.py) ---------------- */
/* D[M,N] = A[M,K] W[N,K]^T with the fused epilogue. A, W bf16 row-major (device). */
int mgb_op_linear(const void* a_bf16_dev, const void* w_bf16_dev, const float* bias_dev, const float* residual_dev,
                  float* out_f32_dev, void* out_bf16_dev, int32_t M, int32_t N, int32_t K, int32_t flags,
                  int32_t block_n, int32_t splits, int32_t stages, float* splitk_ws_dev, void* stream);
/* 3x3 / 1x1 / 5x5 convolution on NHWC bf16. kind: 0 = 3x3 stride 1 pad 1, 1 = 1x1, 2 = 3x3 stride 2 pad 1
 * (x is the 4-plane space-to-depth tensor), 3 = 3x3 stride 2 with pad (0,1,0,1) (VAE; same planes),
 * 4 = 3x3 stride 1 without padding (LPIPS conv1 over factor-4 space-to-depth blocks): only through mgb_op_conv2d_ex,
 *   with the source extent Hsrc >= Hout + 2, Wsrc >= Wout + 2 (anything smaller, and every call of mgb_op_conv2d,
 *   returns MGB_ERR_INVALID before launching),
 * 5 = 5x5 stride 1 pad 2 (25 taps). Epilogue flag 256 (EPI_RELU): out = max(acc + bias, 0).
 * Hout, Wout: OUTPUT size. w_dev: bf16 [Cout, taps*Cin] tap-major. */
int mgb_op_conv2d(const void* x_bf16_dev, const void* w_bf16_dev, const float* bias_dev, const float* residual_dev,
                  float* out_f32_dev, void* out_bf16_dev, int32_t NB, int32_t Hout, int32_t Wout, int32_t Cin,
                  int32_t Cout, int32_t kind, int32_t flags, int32_t block_n, int32_t splits, int32_t stages,
                  float* splitk_ws_dev, void* stream);
/* The same two operators with every input the network's GEMMs use (test entry points: each reaches a path of the
 * network that the plain calls above cannot):
 *   a2_bf16_dev [M, K2] (or NULL): K concatenation A = [a | a2], w [N, K + K2]  (ff.net.2 + proj_out as one GEMM)
 *   x2_bf16_dev NHWC [NB, Hout, Wout, Cin2] (or NULL, kinds 0 / 1): a 1x1 convolution appended along K, w
 *     [Cout, taps*Cin + Cin2]                                                    (ResnetBlock conv2 + 1x1 shortcut)
 *   ldo: row stride of residual / outputs (0: N, or N / 2 with GEGLU); the conv always uses Cout
 *   Hsrc, Wsrc: extent of the tensor the taps address (one parity plane for kinds 2 / 3: ceil(Hin / 2) x ceil(Win / 2));
 *     0 = the output size
 *   scale (EPI_SCALE), sched_x / sched_z / sched_k_dev {kx, kv, kz} / aux_out (EPI_SCHED): see the epilogue flags.
 * block_n <= 0 picks the tile; a special epilogue (EPI_SCHED / DEPTH / NORMALS / NCHW) always takes block_n 16, and
 * an explicit block_n != 16 or N > 16 with one of them returns MGB_ERR_INVALID before anything is launched. */
int mgb_op_linear_ex(const void* a_bf16_dev, const void* a2_bf16_dev, const void* w_bf16_dev, const float* bias_dev,
                     const float* residual_dev, float* out_f32_dev, void* out_bf16_dev, int32_t M, int32_t N, int32_t K,
                     int32_t K2, int32_t ldo, int32_t flags, float scale, const float* sched_x_dev,
                     const float* sched_z_dev, const float* sched_k_dev, float* aux_out_dev, int32_t block_n,
                     int32_t splits, int32_t stages, float* splitk_ws_dev, void* stream);
int mgb_op_conv2d_ex(const void* x_bf16_dev, const void* x2_bf16_dev, const void* w_bf16_dev, const float* bias_dev,
                     const float* residual_dev, float* out_f32_dev, void* out_bf16_dev, int32_t NB, int32_t Hout,
                     int32_t Wout, int32_t Cin, int32_t Cin2, int32_t Cout, int32_t kind, int32_t Hsrc, int32_t Wsrc,
                     int32_t flags, float scale, const float* sched_x_dev, const float* sched_z_dev,
                     const float* sched_k_dev, float* aux_out_dev, int32_t block_n, int32_t splits, int32_t stages,
                     float* splitk_ws_dev, void* stream);
/* Flash self-attention, head size 64 (replaces F.scaled_dot_product_attention under diffusers' Attention, reached
 * from marigold_depth_pipeline.py:461-463). qkv: [NB*T, 3C] (Q | K | V column blocks), out: [NB*T, C]. Long
 * sequences are split over KV ranges and merged by a second kernel; the operator-level entry point keeps the
 * split workspace in a process-wide buffer that it grows on demand (a synchronising cudaMalloc on first use or
 * growth) and is therefore not re-entrant across threads. The network path carves the workspace out of its arena. */
int mgb_op_flash_attn64(const void* qkv_bf16_dev, void* out_bf16_dev, int32_t NB, int32_t T, int32_t C, float scale,
                        void* stream);
/* The same on the 128-row query blocks [q_block_begin, q_block_end) of every (image, head) only: the rows of out_bf16_dev
 * outside them are not written. The KV split and its workspace are chosen for the whole (NB, T, C) problem, so each row
 * written is bit-identical to mgb_op_flash_attn64's. An empty range launches nothing; a range outside
 * [0, ceil(T / 128)] returns MGB_ERR_INVALID. */
int mgb_op_flash_attn64_ex(const void* qkv_bf16_dev, void* out_bf16_dev, int32_t NB, int32_t T, int32_t C, float scale,
                           int32_t q_block_begin, int32_t q_block_end, void* stream);
/* GroupNorm (+SiLU) -> bf16, one launch with a grid-wide barrier, run-to-run deterministic (replaces torch.nn.GroupNorm
 * + F.silu under diffusers' ResnetBlock2D / Transformer2DModel, reached from marigold_depth_pipeline.py:461-463).
 * ws_dev: mgb_op_groupnorm_ws_bytes(NB, HW, C, G) bytes of scratch (0 = unsupported shape). */
size_t mgb_op_groupnorm_ws_bytes(int32_t NB, int32_t HW, int32_t C, int32_t G);
int mgb_op_groupnorm(const float* x_dev, void* y_bf16_dev, const float* gamma_dev, const float* beta_dev,
                     float* ws_dev, int32_t NB, int32_t HW, int32_t C, int32_t G, float eps, int32_t silu,
                     void* stream);
/* GroupNorm over the channel concat [xa | xb] (xb NULL with Cb = 0: one source), groups may straddle the boundary;
 * raw_copy_bf16_dev (or NULL): bf16 copy of the un-normalised concat. ws_dev: mgb_op_groupnorm_ws_bytes(NB, HW, Ca + Cb, G). */
int mgb_op_groupnorm_ex(const float* xa_dev, int32_t Ca, const float* xb_dev, int32_t Cb, void* y_bf16_dev,
                        void* raw_copy_bf16_dev, const float* gamma_dev, const float* beta_dev, float* ws_dev, int32_t NB,
                        int32_t HW, int32_t G, float eps, int32_t silu, void* stream);
int mgb_op_layernorm(const float* x_dev, void* y_bf16_dev, const float* gamma_dev, const float* beta_dev, int32_t M,
                     int32_t C, float eps, void* stream);
/* attn2 of diffusers' BasicTransformerBlock against the FIXED two-token context CLIP(""), collapsed (marigold_depth_pipeline.py
 * :381-394,438-442,461-463), with the LayerNorm before it (norm2) and after it (norm3):
 *   z = LN2(x);  y = x + c1 + sum_h sigmoid(scale * z . G_h) U_h;  a = LN3(y)        (y, a stored as bf16)
 * GU_bf16_dev: [2][H][C] (G rows, then U rows) and c1_dev [C] are what mgb_set_text_embedding folds from to_q / to_k / to_v /
 * to_out and the text embedding. One launch; one warp per token, or four for C = 1280 with few tokens. */
int mgb_op_xattn2(const float* x_dev, void* y_bf16_dev, void* a_bf16_dev, const float* ln2_g_dev, const float* ln2_b_dev,
                  const float* ln3_g_dev, const float* ln3_b_dev, const void* GU_bf16_dev, const float* c1_dev, int32_t M,
                  int32_t C, int32_t H, float scale, float eps, void* stream);
int mgb_op_space_to_depth(const float* x_dev, void* y_bf16_dev, int32_t NB, int32_t H, int32_t W, int32_t C,
                          void* stream);
int mgb_op_upsample2x(const float* x_dev, void* y_bf16_dev, int32_t NB, int32_t H, int32_t W, int32_t C,
                      void* stream);
/* nearest upsampling to Ho x Wo, Ho in {2H - 1, 2H}, Wo in {2W - 1, 2W} (the UNet's crop to an odd skip size) */
int mgb_op_upsample2x_ex(const float* x_dev, void* y_bf16_dev, int32_t NB, int32_t H, int32_t W, int32_t C, int32_t Ho,
                         int32_t Wo, void* stream);
/* VAE attention helpers. Row softmax: fp32 s[M, ld] (first n columns valid) -> bf16 p[M, ld], columns [n, ld) zero.
 * Transpose: bf16 x[M, N] -> bf16 y[N, ld], columns [M, ld) zero. */
int mgb_op_softmax_rows(const float* s_dev, void* p_bf16_dev, int32_t M, int32_t n, int32_t ld, void* stream);
int mgb_op_transpose_bf16(const void* x_bf16_dev, void* y_bf16_dev, int32_t M, int32_t N, int32_t ld, void* stream);
/* The decoder's input: z = post_quant_conv(latent * inv_scale), a 1x1 conv 4 -> 4 in fp32, written as bf16 NHWC with
 * 64 channels (4..63 zero). latent_dev fp32 NCHW [NB, 4, HW]; w_dev fp32 [4, 4]; b_dev fp32 [4]; out [NB * HW, 64]. */
int mgb_op_pack_decoder_latent(const float* latent_dev, const float* w_dev, const float* b_dev, float inv_scale,
                               void* out_bf16_dev, int32_t NB, int32_t HW, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MARIGOLD_B200_H_ */
