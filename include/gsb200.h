/* gsb200.h -- C ABI of libgsb200.so, the H100-native (sm_90a) replacement for the native code
 * under InstantSplat's training hot path.  Plain pointers and sizes only; no torch types.
 * All pointers are DEVICE pointers unless the name ends in _host.  All tensors fp32, contiguous.
 * Every entry point enqueues work on `stream` and returns 0 on success or a negative error code
 * (GSB_ERR_*); none of them throws.  Buffers are caller-owned (the Python layer uses torch
 * allocations), sized with the gsb_*_bytes() helpers.
 *
 * What each entry point replaces in the reference (files of the InstantSplat tree):
 *
 *   gsb_preprocess + gsb_render   ->  diff_gaussian_rasterization._C.rasterize_gaussians, called by
 *                                     GaussianRasterizer.forward at gaussian_renderer/__init__.py:126-135
 *                                     (settings built at :60-76).  With `pose` set they also absorb
 *                                     the pose pre-transform (:81-89), the activations
 *                                     (scene/gaussian_model.py:101-121) and the feature cat (:113-117).
 *   gsb_backward                  ->  _C.rasterize_gaussians_backward (autograd of the call above,
 *                                     triggered by train.py:177) plus the ATen backward of
 *                                     utils/pose_utils.py:57-104 (quad2rotation / quadmultiply) that
 *                                     yields gaussians.P.grad.
 *   gsb_mark_visible              ->  _C.mark_visible (GaussianRasterizer.markVisible).
 *   gsb_preprocess_ex / _backward_ex, gsb_mip_filter3d
 *                                 ->  Mip-Splatting (Yu et al., CVPR 2024), listed as a TODO in the reference's
 *                                     README.md:31-34: the 2D Mip filter (GaussianRasterizationSettings.kernel_size)
 *                                     and the 3D smoothing filter (GaussianModel.compute_3D_filter,
 *                                     get_scaling_with_3D_filter / get_opacity_with_3D_filter).  DESIGN.md 4.7.
 *   gsb_ssim_forward/backward     ->  fused_ssim.fused_ssim, train.py:39-43,172-173
 *                                     (fallback utils/loss_utils.py:55-85).
 *   gsb_loss_forward/backward     ->  train.py:171-176: l1_loss (utils/loss_utils.py:39-40) + SSIM +
 *                                     the (1-l)*L1 + l*(1-ssim) combine, fused.
 *   gsb_adam_step                 ->  scene/per_point_adam.py:34-98 (PerPointAdam.step) for up to
 *                                     GSB_ADAM_MAX_TENSORS tensors in one launch.
 *                                     GsbAdamTensor.grad_scale folds in the x 1/G after the NCCL sum of
 *                                     per-Gaussian gradients (SURVEY.md section 8e).
 */
#ifndef GSB200_H_
#define GSB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define GSB_API __attribute__((visibility("default")))
#else
#define GSB_API
#endif

typedef void* gsb_stream_t; /* cudaStream_t */

#define GSB_OK 0
#define GSB_ERR_INVALID (-1)  /* bad argument (shape / NULL / alignment) */
#define GSB_ERR_CUDA (-2)     /* a CUDA call failed; see gsb_last_error() */
#define GSB_ERR_CAPACITY (-3) /* caller-provided buffer too small */

#define GSB_ADAM_MAX_TENSORS 8

/* Rasterizer settings: GaussianRasterizationSettings of the reference
 * (gaussian_renderer/__init__.py:60-76).  viewmatrix/projmatrix are stored transposed
 * (row-vector convention, scene/cameras.py:54-56): p_view = [p,1] @ viewmatrix. */
typedef struct GsbCamera {
  int32_t width, height;
  float tanfovx, tanfovy;
  float scale_modifier;
  int32_t sh_degree;       /* active degree D (0..3) */
  int32_t sh_coeffs;       /* M: coefficients stored per Gaussian (1, 4, 9 or 16) */
  int32_t exact_cull;      /* 1: lossless alpha<1/255 tile culling (default); 0: reference rect only */
  const float* bg;         /* [3] */
  const float* viewmatrix; /* [16] */
  const float* projmatrix; /* [16] */
  const float* campos;     /* [3] */
} GsbCamera;

/* Gaussian inputs.  Exactly one of (sh_dc[,sh_rest]) / colors_precomp and one of
 * (scales+rotations) / cov3D_precomp must be given. */
typedef struct GsbGaussians {
  int32_t P;
  int32_t sh_packed;           /* 1: sh_dc points at a packed [P,M,3] tensor (B2 boundary);
                                  0: sh_dc [P,3] and sh_rest [P,M-1,3] (the model's own tensors) */
  int32_t raw_params;          /* 1: scales are log-scales and opacities logits (activations fused) */
  int32_t reserved;
  const float* means3D;        /* [P,3] */
  const float* scales;         /* [P,3] */
  const float* rotations;      /* [P,4] raw quaternions, real first, never normalised */
  const float* opacities;      /* [P] */
  const float* sh_dc;
  const float* sh_rest;
  const float* colors_precomp; /* [P,3] or NULL */
  const float* cov3D_precomp;  /* [P,6] or NULL */
  const float* pose;           /* [7] = qw,qx,qy,qz,tx,ty,tz or NULL: fused InstantSplat pre-transform */
} GsbGaussians;

/* Gradients w.r.t. the tensors of GsbGaussians (dense, every row written).  NULL = not wanted. */
typedef struct GsbGrads {
  float* dL_dmeans3D;   /* [P,3] */
  float* dL_dmeans2D;   /* [P,3]  d/d(ndc x,y), z = 0 */
  float* dL_dscales;    /* [P,3] */
  float* dL_drotations; /* [P,4] */
  float* dL_dopacities; /* [P] */
  float* dL_dsh_dc;     /* layout mirrors sh_dc / sh_rest */
  float* dL_dsh_rest;
  float* dL_dcolors;    /* [P,3] (colors_precomp) */
  float* dL_dcov3D;     /* [P,6] (cov3D_precomp) */
  float* dL_dpose;      /* [7] (pose) */
} GsbGrads;

GSB_API size_t gsb_geom_bytes(int32_t P);
GSB_API size_t gsb_binning_bytes(int64_t R, int32_t width, int32_t height);
GSB_API size_t gsb_image_bytes(int32_t width, int32_t height);

/* Forward, phase 1: per-Gaussian projection (+ fused pose / activations / SH->RGB), lossless tile culling,
 * instance counts per Gaussian and per tile, tile-segment offsets.  Writes radii [P] (int32).  The number of
 * (Gaussian, tile) instances R stays on the device; if status_host != NULL (pinned host memory, 8 words) the
 * status words {R, 0, longest tile list, 0, long lists, very long lists, forward serial number, -} are copied there asynchronously (valid once the stream reaches
 * this point) -- a caller that wants an exactly-sized binning buffer waits for it, nobody else has to. */
GSB_API int gsb_preprocess(const GsbCamera* cam, const GsbGaussians* g, void* geom, size_t geom_bytes,
                   int32_t* radii, uint32_t* status_host, gsb_stream_t stream);

/* Forward, phase 2: binning (scatter into per-tile segments, per-tile depth sort in shared memory, slab
 * gather) and the per-tile blend.  R is the instance CAPACITY the binning buffer was sized for
 * (gsb_binning_bytes(R, w, h) <= binning_bytes); it need not be the exact count.  If the true count exceeds
 * it the tile lists are truncated (memory-safe, image approximate) and status word 1 (overflow) is set.
 * status_host (optional, pinned, 8 words): {R true, overflow, longest list, tiles sorted by the slow global
 * path, #lists > 2048, #lists > 8192, forward serial number, -}, copied asynchronously after the blend has been enqueued.  out_color [3,H,W]. */
GSB_API int gsb_render(const GsbCamera* cam, int32_t P, void* geom, void* binning, size_t binning_bytes,
               int64_t R, void* image, float* out_color, uint32_t* status_host, gsb_stream_t stream);

/* Device address of the 8 status words inside `geom` ([0] R, [1] overflow, [2] longest list, [3] slow-path
 * tiles): lets device code (e.g. gsb_adam_step's skip flag) react to an overflow without a host round trip. */
GSB_API uint32_t* gsb_status_device(void* geom, int32_t P);

/* Backward of gsb_preprocess + gsb_render (same R as given to gsb_render).  dL_dout [3,H,W]. */
GSB_API int gsb_backward(const GsbCamera* cam, const GsbGaussians* g, void* geom, void* binning, int64_t R,
                 void* image, const float* dL_dout, const GsbGrads* grads, gsb_stream_t stream);

/* Mip-Splatting filters (DESIGN.md section 4.7).  A NULL GsbFilter is the reference path.
 * flags & GSB_FILTER_MIP2D: the 2D Mip filter, kernel_size * I replaces the 0.3 px^2 dilation of the screen-space
 *   covariance and the opacity is multiplied by sqrt(max(2.5e-5, det(cov2D) / det(cov2D + kernel_size I))).
 *   (kernel_size 0.3 is the upstream rasterizer's later `antialiasing` mode.)
 * filter3D ([P], or NULL): the 3D smoothing filter, raw_params only: scale s -> sqrt(s^2 + f^2) before
 *   scale_modifier, opacity * prod_k s_k / sqrt(s_k^2 + f^2).  f is a constant: it receives no gradient.
 * The record opacity every later stage reads (cull threshold, tile keep mask, 1/255 cutoff, blend) is the filtered one. */
#define GSB_FILTER_MIP2D 1
typedef struct GsbFilter {
  float kernel_size;
  int32_t flags;
  const float* filter3D;
} GsbFilter;

/* gsb_preprocess / gsb_backward with filters; those two are these with filt = NULL.  Like cam and g, the same filter
 * must be passed to a forward and its backward.  With GSB_FILTER_MIP2D a pose-only backward takes the full 9-value
 * blend backward (the filtered opacity depends on the pose). */
GSB_API int gsb_preprocess_ex(const GsbCamera* cam, const GsbGaussians* g, const GsbFilter* filt, void* geom,
                              size_t geom_bytes, int32_t* radii, uint32_t* status_host, gsb_stream_t stream);
GSB_API int gsb_backward_ex(const GsbCamera* cam, const GsbGaussians* g, const GsbFilter* filt, void* geom,
                            void* binning, int64_t R, void* image, const float* dL_dout, const GsbGrads* grads,
                            gsb_stream_t stream);

/* Densification statistics of the reference loop (train.py:197-199 with gaussian_model.py:476-478), accumulated by
 * the per-Gaussian backward from the same dL/dmeans2D it writes to GsbGrads.dL_dmeans2D.  All arrays are [P]:
 * radii is the forward's output (gsb_preprocess), the other three are read and updated in place.  For every Gaussian
 * with radii > 0 (the reference's visibility_filter):
 *   grad_accum += |dL/dmeans2D[:2]|,  denom += 1,  max_radii2D = max(max_radii2D, radii).
 * Nothing is updated when the forward's binning capacity was exceeded (status word 1), so that a repeated
 * iteration counts once.  One thread per Gaussian, no atomics: the result is bit-reproducible. */
typedef struct GsbDensifyStats {
  const int32_t* radii;
  float* grad_accum;
  float* denom;
  float* max_radii2D;
} GsbDensifyStats;

/* gsb_backward_ex that also accumulates the densification statistics; gsb_backward_ex is this with stats = NULL. */
GSB_API int gsb_backward_stats(const GsbCamera* cam, const GsbGaussians* g, const GsbFilter* filt,
                               const GsbDensifyStats* stats, void* geom, void* binning, int64_t R, void* image,
                               const float* dL_dout, const GsbGrads* grads, gsb_stream_t stream);

/* Size of the 3D smoothing filter (Mip-Splatting's GaussianModel.compute_3D_filter) from the training views' pose
 * table: poses7 [n_views, 7] (the rows gsb_preprocess takes as GsbGaussians.pose, p = R x + t), xyz [P, 3] world
 * points, one shared intrinsics (width, height, tanfovx, tanfovy).  A view counts for a point when p_z > 0.2 and
 * its projection lies in the frame widened by 15 % on every side; d = the smallest p_z over the views that count
 * (points no view counts for take the largest d found); out [P] = d / fx * sqrt(0.2).  Deterministic (min / max
 * reductions only). */
GSB_API int gsb_mip_filter3d(int32_t P, const float* xyz, int32_t n_views, const float* poses7, int32_t width,
                             int32_t height, float tanfovx, float tanfovy, float* out, gsb_stream_t stream);

GSB_API int gsb_mark_visible(int32_t P, const float* means3D, const float* viewmatrix,
                     const float* projmatrix, uint8_t* present, gsb_stream_t stream);

/* SSIM (11x11, sigma 1.5, zero 'same' padding, C1=1e-4, C2=9e-4), images [B,C,H,W].
 * forward: sums2[1] += sum of the SSIM map (double[2]; caller zeroes it and divides by B*C*H*W);
 * if maps != NULL ([3,B,C,H,W]) the three partial-derivative maps are stored for backward. */
GSB_API int gsb_ssim_forward(int32_t BC, int32_t H, int32_t W, const float* img1, const float* img2,
                     double* sums2, float* maps, gsb_stream_t stream);
/* dL_dimg1 = scale_host * d(sum ssim)/d(img1) * (*dL_dmean_scale if not NULL) */
GSB_API int gsb_ssim_backward(int32_t BC, int32_t H, int32_t W, const float* img1, const float* img2,
                      const float* maps, float scale_host, const float* dL_dmean_scale,
                      float* dL_dimg1, gsb_stream_t stream);

/* Fused training loss of train.py:171-176 on one image [C,H,W]:
 * sums[0] += sum|img-gt|, sums[1] += sum ssim_map (double[2], caller zeroes it). */
GSB_API int gsb_loss_forward(int32_t C, int32_t H, int32_t W, const float* img, const float* gt,
                     double* sums, float* maps, gsb_stream_t stream);
/* dL_dimg = (1-lambda)/N * sign(img-gt) - lambda/N * d(sum ssim)/d(img), N = C*H*W */
GSB_API int gsb_loss_backward(int32_t C, int32_t H, int32_t W, const float* img, const float* gt,
                      const float* maps, float lambda_dssim, float* dL_dimg, gsb_stream_t stream);

/* ---- pose-only tracking mode (render.py:99-170: Gaussians frozen, Adam on the 7 pose parameters of one view) ----
 * Masked L1 (utils/loss_utils.py:17-23 with the mask of render.py:137-138), forward and backward in one pass:
 * mask = (img > threshold) per element; sums[0] += sum |img-gt|*mask, sums[1] += sum mask (double[2], caller zeroes);
 * dL_dimg = sign(img-gt)*mask -- NOT yet divided by sum(mask): gsb_track_step applies that factor to dL/dpose. */
GSB_API int gsb_l1_mask_fwd_bwd(int32_t C, int32_t H, int32_t W, const float* img, const float* gt, float threshold,
                                double* sums, float* dL_dimg, gsb_stream_t stream);
/* One optimiser step of render.py:118-151 entirely on the device (all pointers are device pointers):
 * loss = sums2[0]/sums2[1]; g = dpose7_raw/sums2[1] + weight_decay*pose; torch.optim.Adam update with step count
 * `step` (1-based) and learning rates lr_q (pose[0..3]) / lr_T (pose[4..6]) -- the caller evaluates the cosine
 * schedule on the host; then, if loss < best8[0]: best8 = {loss, pose AFTER the step} (render.py:146-151).
 * loss_out (optional) receives the loss.  gsb_backward with only GsbGrads.dL_dpose set produces dpose7_raw through a
 * blend backward specialised for this mode (8 accumulated values per Gaussian instead of 9). */
GSB_API int gsb_track_step(float* pose7, const float* dpose7_raw, const double* sums2, float* exp_avg7,
                           float* exp_avg_sq7, float* best8, float* loss_out, int32_t step, float lr_q, float lr_T,
                           float beta1, float beta2, float eps, float weight_decay, gsb_stream_t stream);

/* ---- batched tracking: render.py:99-170 for V test views at once (the loop over test cameras at :99, each view's
 * 500-iteration pose optimisation at :113-161).  The views share one cloud (frozen), one GsbCamera (intrinsics,
 * background) and one GsbFilter; each has its own pose, row v of a [V, 7] table.  Every kernel of the single-view
 * path runs once for the whole batch with a view index: record id v*P + i, global tile v*T + t (T = tiles of one
 * frame), one fixed-point unit M per view.  Each view's result is bit-identical to the single-view call on it, and
 * V = 1 is the single-view path (the single-view entry points are that case of the same kernels).
 * Status words are one set per batch: [0] is the total R of all views, [1] (overflow) is set if any tile list was
 * truncated (memory-safe, as in gsb_render).
 *
 * Sizes: geom grows by ~145 bytes per (view, Gaussian), the image buffer and out_color by V frames, binning by
 * 8 bytes per tile and view; at V = 1 each is at least the single-view size.
 *
 * Batched training (several views per optimizer step, JointTrainer.step_batch): gsb_backward_batch writes the
 * per-Gaussian gradients of all V views SUMMED in view order -- for every element ((g_0 + g_1) + g_2) + ... in fp32,
 * bit-identical to V single-view backward calls whose outputs are added in that order -- plus dL/dpose per view.  It
 * stages each Gaussian slice once and loops over the views inside one launch; no per-view gradient copy is written.
 * gsb_loss_forward_batch / gsb_loss_backward_batch are the training loss on V images, each view's sums and dL/dimg
 * exactly those of gsb_loss_forward / gsb_loss_backward on it.  gsb_backward_batch_stats also accumulates the
 * densification statistics of the batch's first views; batched tracking (gsb_backward_pose_batch) takes none. */
GSB_API size_t gsb_geom_bytes_batch(int32_t P, int32_t V, int32_t width, int32_t height);
GSB_API size_t gsb_binning_bytes_batch(int64_t R, int32_t width, int32_t height, int32_t V);
GSB_API size_t gsb_image_bytes_batch(int32_t width, int32_t height, int32_t V);
/* Device address of the status words inside a batch's geom buffer (gsb_status_device for V views). */
GSB_API uint32_t* gsb_status_device_batch(void* geom, int32_t P, int32_t V);
/* gsb_preprocess_ex for V poses: g must hold raw parameters; g->pose is ignored and poses7 [V, 7] used instead.
 * radii [V, P] (int32). */
GSB_API int gsb_preprocess_batch(const GsbCamera* cam, const GsbGaussians* g, const GsbFilter* filt, int32_t V,
                                 const float* poses7, void* geom, size_t geom_bytes, int32_t* radii,
                                 uint32_t* status_host, gsb_stream_t stream);
/* gsb_render for the batch; R is the instance capacity of the binning buffer for all views.  out_color [V, 3, H, W]. */
GSB_API int gsb_render_batch(const GsbCamera* cam, int32_t P, int32_t V, void* geom, void* binning,
                             size_t binning_bytes, int64_t R, void* image, float* out_color, uint32_t* status_host,
                             gsb_stream_t stream);
/* Pose-only backward of the batch (gsb_backward_ex with only dL_dpose set, per view): dL_dout [V, 3, H, W] ->
 * dpose7 [V, 7].  No per-Gaussian gradient is written. */
GSB_API int gsb_backward_pose_batch(const GsbCamera* cam, const GsbGaussians* g, const GsbFilter* filt, int32_t V,
                                    const float* poses7, void* geom, void* binning, int64_t R, void* image,
                                    const float* dL_dout, float* dpose7, gsb_stream_t stream);
/* gsb_backward_ex for the batch with every per-Gaussian gradient of `grads` summed over the V views (see above);
 * dL_dout [V, 3, H, W], dpose7 [V, 7] (grads->dL_dpose is ignored).  Needs SH colours and scale / rotation (no
 * dL_dcolors / dL_dcov3D); the 2D and 3D Mip filters of filt apply to every view.  V = 1 gives gsb_backward_ex's bits. */
GSB_API int gsb_backward_batch(const GsbCamera* cam, const GsbGaussians* g, const GsbFilter* filt, int32_t V,
                               const float* poses7, void* geom, void* binning, int64_t R, void* image,
                               const float* dL_dout, const GsbGrads* grads, float* dpose7, gsb_stream_t stream);
/* gsb_backward_batch that also accumulates the densification statistics (train.py:197-199) of views 0 .. n_stats-1,
 * in view order: for each such view v and every Gaussian with radii[v*P + i] > 0, grad_accum += |dL/dmeans2D[:2]| of
 * view v's own loss (not of the sum), denom += 1, max_radii2D = max(max_radii2D, radii[v*P + i]).  stats->radii is
 * the batch's [V, P] radii (gsb_preprocess_batch); the other three are [P].  The result is bit-identical to n_stats
 * gsb_backward_stats calls made in view order; nothing is counted when the batch's binning capacity was exceeded
 * (status word 1).  n_stats must be in 0..V and stats non-NULL when n_stats > 0 (else GSB_ERR_INVALID);
 * gsb_backward_batch is this with stats = NULL and n_stats = 0. */
GSB_API int gsb_backward_batch_stats(const GsbCamera* cam, const GsbGaussians* g, const GsbFilter* filt, int32_t V,
                                     int32_t n_stats, const GsbDensifyStats* stats, const float* poses7, void* geom,
                                     void* binning, int64_t R, void* image, const float* dL_dout,
                                     const GsbGrads* grads, float* dpose7, gsb_stream_t stream);
/* Per-view backgrounds (JointTrainer's random background): gsb_render_batch and gsb_backward_batch_stats with view v
 * blended over bg[3 v .. 3 v + 2] of a device [V, 3] fp32 table instead of cam->bg (which is then not read by the
 * blend).  Each view's image and gradients are bit-identical to those of the shared-background call with cam->bg
 * holding that view's row.  The backward must get the table its forward used.  Only blend version 2 (the default)
 * takes a table; with gsb_set_option("blend_version", 1) both return GSB_ERR_INVALID. */
GSB_API int gsb_render_batch_bg(const GsbCamera* cam, int32_t P, int32_t V, const float* bg, void* geom, void* binning,
                                size_t binning_bytes, int64_t R, void* image, float* out_color, uint32_t* status_host,
                                gsb_stream_t stream);
GSB_API int gsb_backward_batch_stats_bg(const GsbCamera* cam, const GsbGaussians* g, const GsbFilter* filt, int32_t V,
                                        const float* bg, int32_t n_stats, const GsbDensifyStats* stats,
                                        const float* poses7, void* geom, void* binning, int64_t R, void* image,
                                        const float* dL_dout, const GsbGrads* grads, float* dpose7,
                                        gsb_stream_t stream);
/* gsb_loss_forward / gsb_loss_backward on V images img [V, C, H, W]: view v's target is the [C, H, W] block
 * gt + gt_row[v] * C*H*W (gt_row: device int32 [V], so that one captured launch serves any choice of targets).
 * sums [V, 2] (double, caller zeroes), maps [3, V, C, H, W]; dL_dimg [V, C, H, W], each view scaled by 1/N with
 * N = C*H*W as in gsb_loss_backward (a mean over views is the caller's factor). */
GSB_API int gsb_loss_forward_batch(int32_t V, int32_t C, int32_t H, int32_t W, const float* img, const float* gt,
                                   const int32_t* gt_row, double* sums, float* maps, gsb_stream_t stream);
GSB_API int gsb_loss_backward_batch(int32_t V, int32_t C, int32_t H, int32_t W, const float* img, const float* gt,
                                    const int32_t* gt_row, const float* maps, float lambda_dssim, float* dL_dimg,
                                    gsb_stream_t stream);
/* gsb_l1_mask_fwd_bwd on V images [V, C, H, W] at once; sums [V, 2] (double, caller zeroes). */
GSB_API int gsb_l1_mask_fwd_bwd_batch(int32_t V, int32_t C, int32_t H, int32_t W, const float* img, const float* gt,
                                      float threshold, double* sums, float* dL_dimg, gsb_stream_t stream);
/* gsb_track_step for V views: pose7, dpose7_raw, exp_avg7, exp_avg_sq7 [V, 7], sums2 [V, 2], best8 [V, 8]; view v's
 * loss goes to loss_out[v * loss_stride] when loss_out is not NULL. */
GSB_API int gsb_track_step_batch(int32_t V, float* pose7, const float* dpose7_raw, const double* sums2, float* exp_avg7,
                                 float* exp_avg_sq7, float* best8, float* loss_out, int64_t loss_stride, int32_t step,
                                 float lr_q, float lr_T, float beta1, float beta2, float eps, float weight_decay,
                                 gsb_stream_t stream);

/* ---- evaluation metrics (train.py:256-290 training_report, metrics.py:55-84) ----
 * img [V, C, H, W]; view v is compared with block gt_row[v] of gt (gt + gt_row[v] * C*H*W, gt_row: device int32 [V]).
 * mode: GSB_METRIC_CLAMP (both clamped to [0,1], train.py training_report) or GSB_METRIC_PNG8 (both through
 * save_image's 8-bit quantisation uint8(clamp(x*255 + 0.5, 0, 255)) and to_tensor's /255, render.py -> metrics.py).
 * out [V, 2 + C] doubles: sum|a-b|, sum of the SSIM map (the training loss's SSIM), per-channel sum (a-b)^2.
 * Every CTA writes its partial sums to scratch (at least gsb_image_metrics_scratch_bytes(V, C, H, W) bytes) and a
 * second kernel adds each view's partials in a fixed order: no atomics, and view v's result is bit-identical across
 * runs, whatever V is and whichever views share the batch.  V * C must not exceed 65535; an unknown mode or a short
 * scratch is GSB_ERR_INVALID. */
#define GSB_METRIC_CLAMP 1
#define GSB_METRIC_PNG8 2
GSB_API size_t gsb_image_metrics_scratch_bytes(int32_t V, int32_t C, int32_t H, int32_t W);
GSB_API int gsb_image_metrics_batch(int32_t V, int32_t C, int32_t H, int32_t W, const float* img, const float* gt,
                                    const int32_t* gt_row, int32_t mode, double* out, void* scratch,
                                    size_t scratch_bytes, gsb_stream_t stream);

/* ---- 8-bit frames (render.py:91-93, torchvision.utils.save_image of one [3, H, W] image) ----
 * img [V, 3, H, W] fp32 -> out [V, H, W, 3] uint8: uint8(clamp(x*255 + 0.5, 0, 255)) per value, each operation rounded
 * as torch rounds it, truncating (the level GSB_METRIC_PNG8 compares), with the channels interleaved per pixel as PIL
 * takes an RGB image.  One memory-bound pass, 12 bytes read and 3 written per pixel.  V must not exceed 65535 and
 * H * W must fit in int32. */
GSB_API int gsb_frames_u8_batch(int32_t V, int32_t H, int32_t W, const float* img, uint8_t* out, gsb_stream_t stream);

/* ---- PNG encoding of 8-bit RGB frames (save_image's files, re-compressed; DESIGN.md 4.19) ----
 * rgb [V, H, W, 3] uint8 (gsb_frames_u8_batch's layout) -> out [V, gsb_png_bound(H, W)] uint8: frame v's zlib stream
 * (the concatenated IDAT data of its PNG) at out + v * gsb_png_bound(H, W), its length in sizes[v] (device int64).
 * The scanlines are filtered as Pillow filters them (of None, Sub, Up and Paeth, the least sum of |int8|, the first on
 * a tie), so the stream inflates to Pillow's filtered bytes; the deflate itself differs from zlib's, so the files are
 * not byte-identical to Pillow's.  A frame's bytes depend on its pixels only: not on V, its place in the batch, the
 * stream or the timing.
 * gsb_png_bound: the largest stream a frame needs (every 32 KiB segment stored, plus the zlib framing); 0 for a bad
 * size.  gsb_png_scratch_bytes: the scratch one call needs.  H, W >= 1, H (3W + 1) below 2^31 - 4096, V <= 65535;
 * scratch 16-byte and sizes 8-byte aligned; else GSB_ERR_INVALID. */
GSB_API size_t gsb_png_bound(int32_t H, int32_t W);
GSB_API size_t gsb_png_scratch_bytes(int32_t V, int32_t H, int32_t W);
GSB_API int gsb_png_encode_batch(int32_t V, int32_t H, int32_t W, const uint8_t* rgb, void* scratch,
                                 size_t scratch_bytes, uint8_t* out, int64_t* sizes, gsb_stream_t stream);

/* ---- Pillow's bicubic resize of 8-bit RGB images (PILtoTorch's pil_image.resize; DESIGN.md 4.21) ----
 * in [V, H, W, 3] uint8 -> out [V, Ho, Wo, 3] uint8, byte for byte what Image.resize((Wo, Ho)) gives each view: a
 * horizontal pass when Wo != W, then a vertical pass when Ho != H, each output channel
 * clamp((2^21 + sum_k src[first + k] * coef[k]) >> 22, 0, 255) in int32 over Pillow's integer tables.  Per axis the
 * tables are device int32: bounds [out, 2] (first source index, tap count) and coefs [out, ksize] (Pillow's weights
 * times 2^22, rounded half away from zero), built on the host (resample.py coefficients); an axis that keeps its size
 * takes no tables (NULL).  Both axes unchanged is a copy.  scratch: the horizontal pass's V * H * Wo * 3 bytes, needed
 * only when both axes change.  A view's bytes depend on its own pixels only.  V, H and Ho in 1..65535, W and Wo >= 1
 * with 3 W and 3 Wo at most 65535 * 256, ksize >= 1 for an axis that changes; else GSB_ERR_INVALID. */
GSB_API int gsb_resample_u8_batch(int32_t V, int32_t H, int32_t W, int32_t Ho, int32_t Wo, const uint8_t* in,
                                  uint8_t* out, const int32_t* x_bounds, const int32_t* x_coefs, int32_t x_ksize,
                                  const int32_t* y_bounds, const int32_t* y_coefs, int32_t y_ksize, void* scratch,
                                  size_t scratch_bytes, gsb_stream_t stream);

/* ---- point_cloud.ply vertex records (GaussianModel.save_ply / load_ply, scene/gaussian_model.py:261-278, 285-;
 * DESIGN.md 4.23) ----
 * A record is R <= GSB_PLY_MAX_FLOATS 32-bit words, filled column by column by up to GSB_PLY_MAX_SEGMENTS segments in
 * record order.  Segment s is a [P, width] array of 32-bit words (row p at data + p * width); its row, read as
 * [width / inner, inner], is stored transposed: element (r, k) at record column col_s + k * (width / inner) + r, col_s
 * the sum of the earlier segments' widths.  inner == width keeps the row as it is; f_rest [P, M-1, 3] takes inner 3
 * (construct_list_of_attributes' channel-major f_rest_*, transpose(1, 2).flatten(1)).  Words are copied, never
 * converted (NaN payloads, -0 and denormals survive), and offsets are 64-bit.  The record buffer is device memory or
 * pinned host memory the device can reach, 4-byte aligned (any 16-byte phase); segment data 4-byte aligned.  Width
 * and inner >= 1 with inner dividing width, R <= GSB_PLY_MAX_FLOATS, P >= 0 (0: nothing launched); else
 * GSB_ERR_INVALID. */
#define GSB_PLY_MAX_SEGMENTS 8
#define GSB_PLY_MAX_FLOATS 64
typedef struct GsbPlySegment {
  void* data;     /* pack: read, NULL for zeros (the normals); unpack: written, NULL to skip the columns */
  int32_t width;  /* words per record */
  int32_t inner;  /* the row's minor extent, made major in the record */
} GsbPlySegment;
/* Replaces save_ply's np.concatenate of the attributes and the structured array PlyData writes: P records, P * R * 4
 * bytes, into out. */
GSB_API int gsb_ply_pack(int64_t P, int32_t n_segments, const GsbPlySegment* segments, void* out,
                         gsb_stream_t stream);
/* Replaces load_ply's per-property np.asarray columns: P records from in into the segments' arrays. */
GSB_API int gsb_ply_unpack(int64_t P, const void* in, int32_t n_segments, const GsbPlySegment* segments,
                           gsb_stream_t stream);

/* ---- Baseline JPEG decoding (PIL.Image.open(path) on libjpeg-turbo; DESIGN.md 4.24) ----
 * One call decodes n files of any sizes, each a single interleaved Huffman scan of 8-bit YCbCr with chroma 1x1 and
 * luma sampling 1x1, 2x1, 1x2 or 2x2, into out[out_offset .. + height * width * 3) as RGB bytes: jdhuff.c's decode,
 * the DC prediction in int32 per component reset at each restart, jidctint.c's islow IDCT, jdsample.c's fancy
 * upsampling and jdcolor.c's fixed-point conversion, so the bytes are Pillow's.  The host parses the marker segments
 * (quantisation and derived Huffman tables, DRI); data holds each file's entropy-coded segment exactly as stored
 * (stuffed bytes and RSTn included), file after file: files[i].data_offset is the sum of the earlier data_bytes.
 * Without restart markers the scan is split into subseq_bits-bit subsequences decoded in parallel and synchronised
 * (Weissenberger & Schmidt, ICPP 2018); the call blocks until the decode is done, the synchronisation's rounds
 * reading a counter each.  status[i] (device int32) is 0 for a file decoded exactly, else GSB_JPEG_* bits naming the
 * stream libjpeg would warn about or handle in ways not reproduced here; such a file's pixels are undefined and the
 * caller decodes it another way.  n <= 65535; subseq_bits a multiple of 8 in 32..2^20; width, height in 1..65535;
 * each entropy segment below 2^28 bytes; scratch 256-byte aligned, at least gsb_jpeg_scratch_bytes; else
 * GSB_ERR_INVALID. */
#define GSB_JPEG_LOOKAHEAD 9
typedef struct GsbJpegHuff {
  uint16_t look[1 << GSB_JPEG_LOOKAHEAD]; /* codes of <= 9 bits, indexed by the next 9 bits: (length << 8) | symbol,
                                             0 for a longer code */
  int32_t maxcode[18];   /* jpeg_make_d_derived_tbl's: the largest code of each length, -1 when there is none */
  int32_t valoffset[18]; /* huffval index = code + valoffset[length] */
  uint8_t huffval[256];
} GsbJpegHuff;
typedef struct GsbJpegFile {
  int32_t width, height;
  int32_t h, v;             /* luma sampling factors, 1 or 2; both chroma components 1x1 */
  int32_t restart_interval; /* MCUs per restart interval, 0 for none */
  int32_t reserved;
  int64_t data_offset;      /* the entropy-coded segment in data */
  int64_t data_bytes;
  int64_t out_offset;       /* the [height, width, 3] image in out */
  uint16_t quant[3][64];    /* per component (Y, Cb, Cr), natural order */
  GsbJpegHuff dc[3], ac[3]; /* per component */
} GsbJpegFile;
#define GSB_JPEG_BAD_CODE 1       /* a code with no table entry */
#define GSB_JPEG_PAST_END 2       /* bits needed past the end of an entropy segment or restart interval */
#define GSB_JPEG_RUN_PAST_63 4    /* a run past coefficient 63 */
#define GSB_JPEG_RESTART 8        /* RSTn missing, extra or out of sequence */
#define GSB_JPEG_MCUS_LEFT 16     /* a segment or interval ended with MCUs left to decode */
#define GSB_JPEG_TRAILING 32      /* a whole byte or more left after an interval's last MCU */
#define GSB_JPEG_COEF_RANGE 64    /* a dequantised coefficient outside int16, or a DC sum outside int32 */
#define GSB_JPEG_UNSYNCED 128     /* the subsequences did not synchronise */
GSB_API size_t gsb_jpeg_scratch_bytes(int32_t n, const GsbJpegFile* files, int32_t subseq_bits);
GSB_API int gsb_jpeg_decode_batch(int32_t n, const GsbJpegFile* files, const uint8_t* data, int32_t subseq_bits,
                                  void* scratch, size_t scratch_bytes, uint8_t* out, int32_t* status,
                                  gsb_stream_t stream);

/* ---- LPIPS, VGG16 v0.1(metrics.py:69 lpips(render, gt, net_type='vgg'); lpipsPyTorch/modules/lpips.py,
 * networks.py BaseNet / VGG16, utils.py normalize_activation).  DESIGN.md 4.15.  fp32 FFMA, NHWC activations, every
 * sum in one fixed order: an image's values are bit-identical from run to run and whatever else is in the batch.
 *
 * gsb_lpips_prepare       ->  BaseNet.z_score: x, y [V, 3, H, W] -> out [2V, H, W, 3], images 0..V-1 from x and
 *                             V..2V-1 from y, (v - mean) / std in fp32.
 * gsb_lpips_conv3x3_relu  ->  one Conv2d(Cin, Cout, 3, padding=1) + ReLU of vgg16().features: in [N, H, W, Cin] ->
 *                             out [N, H, W, Cout].  w_packed [Cin, 3, 3, Cout] (weight.permute(1, 2, 3, 0)), bias
 *                             [Cout].  Cin is 3 or a multiple of 8, Cout a multiple of 64; w_packed, out (and in when
 *                             Cin > 3) 16-byte aligned.
 * gsb_lpips_maxpool2      ->  MaxPool2d(2, 2), floor mode: in [N, H, W, C] -> out [N, H / 2, W / 2, C]; C a multiple
 *                             of 4, both 16-byte aligned.
 * gsb_lpips_head          ->  normalize_activation of both feature maps, (fx - fy)^2, the lin layer's 1x1 conv and
 *                             the sum over H x W: feats [2V, H, W, C] (x's V images, then y's), lin_w [C]; writes
 *                             out[v * 5 + layer] (fp64), the sum over pixels (the mean is out / (H W)).  partials: at
 *                             least V * GSB_LPIPS_HEAD_PARTS doubles; C a multiple of 32.
 * gsb_lpips_scratch_bytes ->  what one call of a V-pair batch at H x W needs: two activation buffers of
 *                             2V * H * W * 64 floats each (the largest activation, relu1_x) followed by the head's
 *                             V * GSB_LPIPS_HEAD_PARTS doubles. */
#define GSB_LPIPS_HEAD_PARTS 128
GSB_API size_t gsb_lpips_scratch_bytes(int32_t V, int32_t H, int32_t W);
GSB_API int gsb_lpips_prepare(int32_t V, int32_t H, int32_t W, const float* x, const float* y, float* out,
                              gsb_stream_t stream);
GSB_API int gsb_lpips_conv3x3_relu(int32_t N, int32_t H, int32_t W, int32_t Cin, int32_t Cout, const float* in,
                                   const float* w_packed, const float* bias, float* out, gsb_stream_t stream);
GSB_API int gsb_lpips_maxpool2(int32_t N, int32_t H, int32_t W, int32_t C, const float* in, float* out,
                               gsb_stream_t stream);
GSB_API int gsb_lpips_head(int32_t V, int32_t H, int32_t W, int32_t C, const float* feats, const float* lin_w,
                           int32_t layer, double* out, double* partials, gsb_stream_t stream);

/* Per-point Adam (scene/per_point_adam.py:34-98), n tensors in one launch. */
typedef struct GsbAdamTensor {
  float* param;
  const float* grad;
  float* exp_avg;
  float* exp_avg_sq;
  const float* per_point_lr; /* [rows] or NULL */
  int64_t numel;
  int32_t row_len;           /* numel / rows (elements sharing one per_point_lr entry) */
  float grad_scale;          /* gradient is multiplied by this first (1/G after an NCCL sum) */
  double step_size;          /* lr * sqrt(1-b2^t) / (1-b1^t), computed on the host in double */
  double beta1, beta2, eps, weight_decay;
} GsbAdamTensor;
/* flags: [n] uint32 scratch (device); gate g.norm()>0 per tensor is evaluated on the device (see gsb_adam_gate). */
GSB_API int gsb_adam_step(int32_t n, const GsbAdamTensor* tensors_host, uint32_t* flags, gsb_stream_t stream);
/* Same, but the whole update is skipped on the device when *skip_if_nonzero != 0 (device pointer, may be NULL):
 * pass gsb_status_device(geom, P) + 1 so that a binning overflow leaves the parameters untouched and the
 * caller can redo the iteration with a larger buffer once it notices -- no host sync on the normal path. */
GSB_API int gsb_adam_step_gated(int32_t n, const GsbAdamTensor* tensors_host, uint32_t* flags,
                                const uint32_t* skip_if_nonzero, gsb_stream_t stream);

/* flags[k] = GSB_ADAM_FLAG_NONZERO if tensor k's scaled gradient has a non-zero element, | GSB_ADAM_FLAG_NAN if it has
 * a NaN; the gate half of gsb_adam_step, exposed so the multi-GPU path can all-reduce the flags before the fused
 * exchange kernel.  The moments are updated when 1 <= flag < GSB_ADAM_FLAG_NAN: the reference's gate grad.norm() > 0
 * is false for a NaN anywhere in the tensor.  Flags summed over at most 8 ranks keep that meaning. */
#define GSB_ADAM_FLAG_NONZERO 1u
#define GSB_ADAM_FLAG_NAN 256u
GSB_API int gsb_adam_gate(int32_t n, const GsbAdamTensor* tensors_host, uint32_t* flags, gsb_stream_t stream);

/* ---- multi-GPU: fused reduce-scatter -> per-point Adam -> all-gather over NVLink peer memory ----------
 * (new functionality, SURVEY.md section 8e; the NCCL all-reduce + gsb_adam_step pair is the baseline it
 * replaces).  Peer-visible buffers are cudaMalloc'ed here and shared between the per-GPU processes with
 * CUDA IPC handles (64 bytes). */
GSB_API int gsb_ipc_alloc(size_t bytes, void** dev_ptr, unsigned char* handle64);
GSB_API int gsb_ipc_open(const unsigned char* handle64, void** dev_ptr);
GSB_API int gsb_ipc_close(void* dev_ptr);
GSB_API int gsb_ipc_free(void* dev_ptr);

/* Flag barrier / small exchange over peer memory (replace the tiny NCCL collectives around the fused kernel).
 * peer_signal: host array of `world` device pointers to every rank's signal buffer (gsb_peer_signal_bytes() bytes,
 * allocated zeroed with gsb_ipc_alloc, own rank included).  epoch: the optimizer step, 1, 2, 3, ... (same on all
 * ranks); epoch 0 = use the device-resident epoch (word 61 of the local signal buffer, advanced by every
 * gsb_peer_exchange and re-used by the gsb_peer_barrier of the same step), which makes both launches replayable from a
 * CUDA graph.  Do not mix the two conventions on one signal buffer.  gsb_peer_exchange (channel 0): flags8[0..6] gate flags, overflow_word (device, may be NULL) and
 * pose_grad[n_pose] are replaced IN PLACE by their sums over the ranks (flags8[7] = number of ranks whose
 * overflow_word was set); it is also the barrier "every rank's gradients are written".  gsb_peer_barrier: pure
 * barrier on `channel` (use 1 after the fused kernel: "every rank's parameter stores have landed").  A wait that
 * exceeds ~3 s sets word 60 of the local signal buffer and returns (the GPU is never hung on a dead peer). */
GSB_API size_t gsb_peer_signal_bytes(void);
GSB_API int gsb_peer_barrier(int32_t world, int32_t rank, void* const* peer_signal, uint32_t epoch, int32_t channel,
                             gsb_stream_t stream);
GSB_API int gsb_peer_exchange(int32_t world, int32_t rank, void* const* peer_signal, uint32_t epoch, uint32_t* flags8,
                              const uint32_t* overflow_word, float* pose_grad, int32_t n_pose, gsb_stream_t stream);

/* Same again, with the per-tensor step sizes read from a DEVICE array (float[n], step_sizes_dev[k] replaces
 * tensors_host[k].step_size) when it is not NULL: the launch can then sit in a CUDA graph and be replayed while the
 * host refreshes the array (learning-rate schedule, bias correction) before every replay. */
GSB_API int gsb_adam_step_ex(int32_t n, const GsbAdamTensor* tensors_host, uint32_t* flags,
                             const uint32_t* skip_if_nonzero, const float* step_sizes_dev, gsb_stream_t stream);

typedef struct GsbShardPiece { /* (one tensor's segment) intersected with (this rank's shard) */
  int64_t begin, end;          /* flat-buffer element range, multiples of 4 */
  int64_t seg_begin;           /* where the tensor's segment starts in the flat buffer */
  const float* per_point_lr;   /* [rows] of the whole tensor, or NULL */
  int32_t row_len;
  int32_t flag_index;          /* which gate flag applies */
  double step_size, beta1, beta2, eps;
} GsbShardPiece;

/* step_sizes_dev (device, may be NULL): float[GSB_ADAM_MAX_TENSORS], entry flag_index replaces the piece's step_size
 * (CUDA-graph replay: the host refreshes the array before every replay).
 * skip_if_nonzero (device, may be NULL): when the word is non-zero the kernel returns without touching anything
 * (the sum over ranks of the forward's overflow words, so every replica takes the same decision).
 * peer_grads / peer_params: host arrays of `world` device pointers to every rank's flat gradient / parameter
 * buffer (own rank included).  exp_avg / exp_avg_sq: this rank's shard only, indexed by (element - shard_begin). */
GSB_API int gsb_fused_rs_adam_ag(int32_t world, int32_t rank, const float* const* peer_grads,
                                 float* const* peer_params, float* exp_avg_shard, float* exp_avg_sq_shard,
                                 int64_t shard_begin, int32_t n_pieces, const GsbShardPiece* pieces,
                                 const uint32_t* flags, const uint32_t* skip_if_nonzero, float grad_scale,
                                 const float* step_sizes_dev, gsb_stream_t stream);

/* simple_knn._C.distCUDA2 (scene/gaussian_model.py:20,156-160; init only, SURVEY.md section 8 row f1):
 * out[i] = mean squared distance from point i to its 3 nearest neighbours (exact).  points [P,3], out [P]. */
GSB_API size_t gsb_knn_scratch_bytes(int32_t P);
GSB_API int gsb_knn_mean_dist2(int32_t P, const float* points, float* out, void* scratch, size_t scratch_bytes,
                               gsb_stream_t stream);

/* Optional instrumentation (bench.py): per-kernel CUDA-event timing on the launching stream and a
 * count of this library's kernel launches (every launch on the path is the library's own). */
enum {
  GSB_K_PREPROCESS = 0, GSB_K_SORT_DEPTH /* unused since ABI 2 */, GSB_K_SCAN /* tile scan */,
  GSB_K_DUPLICATE /* scatter */, GSB_K_SORT_TILE /* per-tile sort + slab gather */, GSB_K_GATHER /* unused */,
  GSB_K_BLEND_FWD, GSB_K_BLEND_BWD, GSB_K_PREPROCESS_BWD, GSB_K_LOSS_FWD, GSB_K_LOSS_BWD, GSB_K_ADAM,
  GSB_K_COUNT
};
/* Pair statistics of the blend kernels on the buffers of the last forward (and backward if dL_dout != NULL):
 * stats (device, 8 x uint64) = {fwd warp iterations (64 evaluated pixel-Gaussian pairs each), fwd contributing
 * pairs, bwd warp iterations, bwd contributing pairs, bwd warp iterations that reached the reduction, 0, 0, 0}. */
GSB_API int gsb_blend_stats(const GsbCamera* cam, int32_t P, void* geom, void* binning, int64_t R, void* image,
                            float* out_color, const float* dL_dout, unsigned long long* stats, gsb_stream_t stream);
GSB_API void gsb_profile_enable(int on);
GSB_API int gsb_profile_collect(double* ms_sum, int64_t* count, int n_ids);
GSB_API uint64_t gsb_launch_count(void);
/* Tuning switches: "blend_version" = 1 (one pixel per lane, 8 warps per tile; the in-library cross-check) | 2 (two
 * pixels per lane; default); "stage_bulk" = 1 (slab chunks staged with cp.async.bulk/TMA +
 * mbarrier, double buffered; default) | 0; "blend_bwd_batch" = 1 (the v2 blend backward reduces its per-Gaussian
 * moments in per-warp batches; default) | 0 (one warp butterfly per list entry: the bit-for-bit reference). */
GSB_API int gsb_set_option(const char* name, int value);

GSB_API const char* gsb_last_error(void);
GSB_API int gsb_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* GSB200_H_ */
