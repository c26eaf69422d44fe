/*
 * brush_b200.h -- C ABI of libbrush_b200.so: the sm_90a CUDA hot path of the
 * differentiable Gaussian-splat rasterizer, behind the operator boundary of
 * ArthurBrussee/brush.  Plain pointers and sizes only; no torch / burn types.
 *
 * Every entry point replaces one Rust-side operator of the reference (cited
 * per function, paths relative to the reference checkout).  INTEGRATION.md
 * shows the `extern "C"` block + `impl SplatOps / SplatBwdOps / LossOps`
 * shim a Brush maintainer would add on the Rust side.
 *
 * Conventions (modelled on apps/brush-c/src/lib.rs:14-163, the reference's
 * only C ABI):
 *   - every call returns int32_t status (BG_OK == 0); nothing panics/aborts;
 *     null or inconsistent arguments give BG_ERR_NULL / BG_ERR_INVALID;
 *   - all array pointers are DEVICE pointers on the context's device unless
 *     the parameter comment says "host"; arrays are dense, row major, f32 or
 *     u32, 16-byte aligned;
 *   - every call takes the cudaStream_t (as void*) to enqueue on and returns
 *     without synchronising: there is no device->host readback inside the
 *     forward (the reference blocks on one, render.rs:146-168).  Counters are
 *     mirrored into pinned host memory and are valid after the caller
 *     synchronises the stream;
 *   - the context owns the scratch arena (sort buffers, intersection lists,
 *     saved forward state).  One context serves one logical task at a time
 *     (the reference's threading contract, brush-async/src/lib.rs:1-17);
 *     distinct contexts are independent and may be used from different
 *     threads / streams concurrently.
 */
#ifndef BRUSH_B200_H
#define BRUSH_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BG_ABI_VERSION 7u

/* f32 lanes per projected splat: a 64-byte row, four aligned 128-bit loads.  Lanes 0..8 are the reference
 * layout (kernels/helpers.rs:49-53: xy_x, xy_y, conic_x, conic_y, conic_z, color_a, color_r, color_g, color_b).
 * Lanes 9..12 are derived values cached for the blend kernels: 9 = log2(e)/2 * conic_z, 10 = log2(e)/2 * conic_x,
 * 11 = log2(e) * conic_y (so that alpha = opacity * 2^-(l10 dx^2 + l9 dy^2 + l11 dx dy) costs three FMA-class
 * operations and one MUFU per pixel), 12 = ln(255 * opacity) (the block-cull threshold); 13..15 pad (the blend
 * kernels' shared-memory copy of a row carries the splat's depth in lane 13 when depth is rendered). */
#define BG_PROJECTED_STRIDE 16u
/* f32 lanes per row of v_combined (bwd/burn_glue.rs:36-43). */
#define BG_VCOMBINED_STRIDE 10u

typedef enum {
    BG_OK = 0,
    BG_ERR_NULL = 1,        /* a required pointer was null */
    BG_ERR_INVALID = 2,     /* inconsistent sizes / unsupported K / zero image size */
    BG_ERR_CUDA = 3,        /* a CUDA runtime call failed; see bg_last_error_string */
    BG_ERR_CAPACITY = 4,    /* request exceeds what the context was created for */
    BG_ERR_UNSUPPORTED = 5  /* camera model / feature not built */
} BgStatus;

/* gaussian_splats.rs:27-48 RasterPass */
typedef enum { BG_PASS_FORWARD = 0, BG_PASS_BACKWARD = 1, BG_PASS_BACKWARD_SMOOTH = 2 } BgPass;

/* kernels/camera_model/mod.rs:32-39 CameraModel.  The reference bakes the distortion coefficients into the
 * kernel at compile time; here they travel in BgCamera.model_params:
 *   KANNALA_BRANDT_4    (kannala_brandt_4.rs:10-16)      k1 k2 k3 k4
 *   RADIAL_TANGENTIAL_8 (radial_tangential_8.rs:12-21)   k1 k2 k3 k4 k5 k6 p1 p2
 *   THIN_PRISM_FISHEYE  (thin_prism_fisheye.rs:25-31)    k1 k2 k3 k4 p1 p2 sx1 sy1 */
typedef enum {
    BG_CAMERA_PINHOLE = 0,
    BG_CAMERA_KANNALA_BRANDT_4 = 1,
    BG_CAMERA_RADIAL_TANGENTIAL_8 = 2,
    BG_CAMERA_THIN_PRISM_FISHEYE = 3
} BgCameraModel;

/* Host struct.  Mirror of ProjectUniforms (shaders.rs:17-66, kernels/types.rs:51-80) minus the
 * sizes that are passed as arguments.  viewmat = camera.world_to_local(), top 3 rows, column
 * major: column i at viewmat[3*i .. 3*i+3], column 3 is the translation. */
typedef struct {
    float viewmat[12];
    float fx, fy, cx, cy;                              /* PinholeParams, camera.rs:64-73 */
    float cam_pos[3];                                  /* camera.position */
    float lim_pos_x, lim_pos_y, lim_neg_x, lim_neg_y;  /* JacobianClampLimits, camera.rs:200-254 */
    float half_max_render_fov;                         /* render.rs:70-71 */
    uint32_t camera_model;                             /* BgCameraModel */
    float model_params[8];                             /* distortion coefficients of camera_model, zero padded */
} BgCamera;

/* Saved forward state handed to the backward calls: mirror of the non-image fields of
 * RenderOutput (render_aux.rs:16-28) + GaussianBackwardState (bwd/burn_glue.rs:95-112).
 * Pointers refer to the context arena and stay valid until the next bg_render_forward on
 * the same context. */
typedef struct {
    const float *projected;                 /* [num_visible, BG_PROJECTED_STRIDE] depth-sorted */
    const uint32_t *compact_gid_from_isect; /* [num_intersections] tile-major, depth order inside a tile */
    const uint32_t *global_from_compact_gid;/* [num_visible] */
    const uint32_t *compact_from_global_gid;/* [n] inverse map; 0xFFFFFFFF for culled Gaussians */
    const uint32_t *tile_offsets;           /* [tiles_y, tiles_x, 2] (start,end); end trimmed when pass != FORWARD */
    const float *depths;                    /* [num_visible] sorted camera-space z (diagnostic) */
    const uint32_t *tile_id_from_isect;     /* [num_intersections] sorted tile ids (diagnostic) */
    const uint32_t *counters_dev;           /* device [4]: num_visible, num_intersections, overflow flag, reserved */
    const volatile uint32_t *counters_host; /* host (pinned) mirror of counters_dev; valid after stream sync */
    uint32_t n, k, w, h, tiles_x, tiles_y;
    int32_t mip, pass;
} BgRenderState;

typedef struct BgContext BgContext;

/* Version / capability probe.  Returns BG_ABI_VERSION. */
uint32_t bg_abi_version(void);
/* Thread-local description of the last BG_ERR_CUDA / BG_ERR_INVALID on this thread. */
const char *bg_last_error_string(void);

/* Creates the scratch arena on `device`.  max_intersections bounds num_intersections
 * (the reference sizes these buffers after a blocking readback, render.rs:146-168,211-213);
 * 0 picks max(16*max_splats, 1<<22).  Exceeding it at run time sets counters[2] != 0 and the
 * extra intersections are dropped (never written out of bounds). */
int32_t bg_ctx_create(int32_t device, uint32_t max_splats, uint32_t max_w, uint32_t max_h,
                      uint64_t max_intersections, BgContext **out_ctx);
int32_t bg_ctx_destroy(BgContext *ctx);
/* Bytes of device memory held by the arena (for sizing against 180 GB HBM3e). */
uint64_t bg_ctx_arena_bytes(const BgContext *ctx);

/* Replaces <MainBackendBase as SplatOps>::render, brush-render/src/render.rs:37-315
 * (trait: brush-render/src/lib.rs:54-77).
 *   transforms [n,10] means(3)+quat wxyz(4)+log_scales(3); sh [n,k,3], k in {1,4,9,16,25};
 *   raw_opac [n]; bg: host float[3].
 *   out_img: [h,w,4] f32 when pass != FORWARD, [h,w] u32 rgba8 when pass == FORWARD.
 *   visible [n] f32 (written only when pass != FORWARD, may be null otherwise); max_radius [n].
 * Panics of the reference (render.rs:50-64, dim_check.rs) become BG_ERR_INVALID. */
int32_t bg_render_forward(BgContext *ctx, void *stream, const BgCamera *cam, uint32_t w, uint32_t h,
                          uint32_t n, uint32_t k, const float *transforms, const float *sh,
                          const float *raw_opac, int32_t mip, const float *bg, int32_t pass,
                          void *out_img, float *visible, float *max_radius, BgRenderState *state_out);

/* Replaces SplatBwdOps::rasterize_bwd, bwd/render_bwd.rs:22-99 (kernel:
 * bwd/kernels/rasterize_backwards.rs:100-391).  v_combined: [rows, 10] with rows >= num_visible
 * (n rows always suffice); the first min(rows, n) rows are zeroed here, as float_zeros does.
 * Preconditions (the state is valid until the next bg_render_forward on the same context; the backward replays
 * what that forward recorded in the arena), each BG_ERR_INVALID with v_combined untouched when violated:
 *   smooth_cutoff != 0 exactly when state->pass == BG_PASS_BACKWARD_SMOOTH (the reference passes
 *   state.pass.smooth_cutoff(), bwd/burn_glue.rs:152); `state` comes from this context's last forward. */
int32_t bg_rasterize_backward(BgContext *ctx, void *stream, const BgRenderState *state, const float *out_img,
                              const float *v_output, const float *bg, int32_t smooth_cutoff,
                              float *v_combined, uint32_t v_combined_rows);

/* ---- Differentiable depth (DESIGN.md §4.6; no reference operator).
 * bg_render_forward_depth is bg_render_forward for the f32 passes (BG_PASS_BACKWARD, BG_PASS_BACKWARD_SMOOTH;
 * BG_PASS_FORWARD is BG_ERR_INVALID) that also writes the accumulated depth
 *     out_depth[y,x] = D = sum_i vis_i z_i          (device [h,w] f32)
 * with vis_i = alpha_i T_i the weight the colour uses (same cutoffs, the stopping splat not blended) and z_i the
 * splat mean's camera-space z (the depth-sort key, state->depths).  There is no background term; the expected depth
 * is D / out_img[y,x,3], formed by the caller.  out_img, visible, max_radius, the state and the tile ranges are
 * bit-identical to bg_render_forward's.
 * bg_rasterize_backward_depth is bg_rasterize_backward with the upstream gradient v_depth [h,w] of D: depth enters
 * v_alpha like a fourth colour channel with colour z_i, so v_combined also carries the depth terms (its refine weight
 * is formed from the total screen-space gradient), and v_z (device [v_combined_rows]) receives
 * v_z[cgid] = sum over pixels of vis v_depth, indexed by compact id like v_combined; its first min(rows, n) entries
 * are zeroed here.  Besides the preconditions of bg_rasterize_backward, the state must come from this context's last
 * forward AND that forward must have been bg_render_forward_depth (out_depth is its output): otherwise BG_ERR_INVALID
 * with v_combined and v_z untouched.  The state stays valid until the next forward on the context, of either kind.
 * bg_project_backward_depth is bg_project_backward followed by v_transforms[gid, 0:3] += v_z[cgid] * R[2,:]
 * (R = the view rotation, R[2,:] = viewmat[2], viewmat[5], viewmat[8]); Gaussians with v_z == 0 keep
 * bg_project_backward's output bits. */
int32_t bg_render_forward_depth(BgContext *ctx, void *stream, const BgCamera *cam, uint32_t w, uint32_t h,
                                uint32_t n, uint32_t k, const float *transforms, const float *sh,
                                const float *raw_opac, int32_t mip, const float *bg, int32_t pass,
                                float *out_img /*[h,w,4]*/, float *out_depth /*[h,w]*/, float *visible,
                                float *max_radius, BgRenderState *state_out);
int32_t bg_rasterize_backward_depth(BgContext *ctx, void *stream, const BgRenderState *state, const float *out_img,
                                    const float *out_depth, const float *v_output, const float *v_depth /*[h,w]*/,
                                    const float *bg, int32_t smooth_cutoff, float *v_combined,
                                    uint32_t v_combined_rows, float *v_z /*[v_combined_rows]*/);
int32_t bg_project_backward_depth(BgContext *ctx, void *stream, const BgCamera *cam, const BgRenderState *state,
                                  const float *transforms, const float *sh, const float *raw_opac,
                                  const float *v_combined, const float *v_z, float *v_transforms, float *v_sh,
                                  float *v_raw_opac, float *v_refine);

/* Measurement aid (not a reference operator): counters of the blend loop for the state of this context's last
 * BG_PASS_BACKWARD forward.  out4 (host): [0] warp-splat iterations of the backward walk (64 pixel-splat pairs each),
 * [1] pixel-splat pairs that blended, [2] pairs that stopped a pixel, [3] tile-list entries (num_intersections).
 * v_combined_scratch: device [n,10] scratch that receives the gradients of the counting run.  Synchronises `stream`. */
int32_t bg_debug_blend_stats(BgContext *ctx, void *stream, const BgRenderState *state, const float *out_img,
                             const float *v_output, const float *bg, float *v_combined_scratch,
                             unsigned long long *out4);

/* Replaces SplatBwdOps::project_bwd, bwd/render_bwd.rs:102-171 (kernel:
 * bwd/kernels/project_backwards.rs:99-254).  Dense outputs; every row is written (zeros for
 * Gaussians that received no gradient), so no separate zero-fill is needed. */
int32_t bg_project_backward(BgContext *ctx, void *stream, const BgCamera *cam, const BgRenderState *state,
                            const float *transforms, const float *sh, const float *raw_opac,
                            const float *v_combined, float *v_transforms, float *v_sh, float *v_raw_opac,
                            float *v_refine);

/* Counter-based N(0,1) draws (Philox4x32-10 + Box-Muller): out[i], i < count, is a pure function of (seed, offset, i);
 * the reference draws the mean noise with burn's Tensor::random(Normal) from an unseeded generator (train.rs:395-399). */
int32_t bg_normal_noise(BgContext *ctx, void *stream, uint64_t seed, uint64_t offset, uint64_t count, float *out);

/* SplatTrainer::step (brush-train/src/train.rs:176-429) as one call: render forward -> L1 + SSIM loss value and
 * gradient -> rasterize / project backward -> AdamScaled on transforms, SH, opacity -> refine statistics -> mean noise.
 * Every launch goes to `stream`; nothing is read back (the step can be captured in a CUDA graph).  Parameters, Adam
 * moments and the refine record are updated in place.  Scratch comes from `workspace` (device, 256-byte aligned,
 * bg_train_step_workspace_bytes(n, k, w, h) bytes).  Learning rates are the step's values: the caller evaluates the
 * schedule lr_mean(n) = lr_mean * decay^(n-1) * median_scale (train.rs:328-333).  `step` is the 1-based Adam step.
 * noise_scale = lr_mean * mean_noise_weight (0 disables the noise); the draw is bg_normal_noise(seed, step). */
typedef struct {
    BgCamera cam;
    uint32_t w, h, n, k;
    int32_t mip;
    float background[3];
    float *transforms, *sh, *raw_opac;              /* [n,10] [n,k,3] [n], updated in place */
    float *m_t, *v_t, *m_sh, *v_sh, *m_o, *v_o;     /* Adam moments; v_sh is [n] (row-reduced, adam_scaled.rs:152-165) */
    float *refine_norm, *vis_weight, *max_screen;   /* RefineRecord (stats.rs:15-50), [n] each */
    const uint32_t *gt_packed;                      /* device [h,w] rgba8 (scene.rs:97-136) */
    float l1_weight, ssim_weight;                   /* train.rs:228-232: 1 - w, -w */
    int32_t has_composite_bg;
    float composite_bg[3];
    int32_t mask;                                   /* AlphaMode::Masked */
    int32_t channels;                               /* 3, or 4 when the alpha channel is matched (train.rs:236-249) */
    float alpha_weight;                             /* match_alpha_weight */
    float lr_mean, lr_rotation, lr_scale, lr_coeffs_dc, lr_coeffs_sh_scale, lr_opac;
    float noise_scale, median_scale;
    uint64_t seed;
    int32_t step;
    void *workspace;
    uint64_t workspace_bytes;
    float *loss_out;                                /* device scalar */
    BgRenderState state_out;                        /* the step's render state (counters etc.) */
} BgTrainStepArgs;
uint64_t bg_train_step_workspace_bytes(uint32_t n, uint32_t k, uint32_t w, uint32_t h);
int32_t bg_train_step(BgContext *ctx, void *stream, BgTrainStepArgs *args);

/* Depth supervision (DESIGN.md section 4.7; not a reference operator).  target: device [h,w] metric camera-space z of the
 * view; a pixel is valid when its target is finite and > 0 (0 = no measurement).  With a = out_img[...,3], ed = D / a
 * and a pixel active when it is valid and a >= 1/255, the term is
 *   L_d = (weight / valid_count) * sum over active pixels of |ed - t|.
 * valid_count is the number of valid pixels, counted by the host when the map was loaded (never read back here). */
typedef struct {
    const float *target;      /* device [h,w] f32; may be null when weight == 0 or valid_count == 0 */
    float weight;             /* w_d >= 0, finite */
    uint32_t valid_count;     /* |valid pixels| */
    float *depth_loss_out;    /* device scalar: L_d (0 when the term is skipped) */
} BgDepthSupervision;

/* One pass of the depth term over a depth render (bg_render_forward_depth): with chain = weight / valid_count and
 * s = sign(ed - t) (sign(0) = 0), writes v_depth = chain * s / a on active pixels and 0 elsewhere, ADDS -v_depth * ed to
 * v_output[...,3] on active pixels only (that slot may already hold the image loss's alpha gradient), and writes per-block
 * partial sums of |ed - t| (device float[bg_depth_loss_num_partials(h, w)]; L_d = chain * their sum).  IEEE division, no
 * float atomics.  out_img and v_output: [h,w,4], 16-byte aligned.  chain must be finite and >= 0. */
uint32_t bg_depth_loss_num_partials(uint32_t h, uint32_t w);
int32_t bg_depth_loss_fused(BgContext *ctx, void *stream, const float *out_img /*[h,w,4]*/, const float *depth /*[h,w]*/,
                            const float *target /*[h,w]*/, uint32_t h, uint32_t w, float chain /* w_d/|valid| */,
                            float *v_output /*[h,w,4], channel 3 +=*/, float *v_depth /*[h,w]*/, float *partials);

/* bg_train_step with the depth term: bg_render_forward_depth -> image loss -> bg_depth_loss_fused ->
 * bg_rasterize_backward_depth -> bg_project_backward_depth -> the same update pass.  *args->loss_out = image loss + L_d;
 * *depth->depth_loss_out = L_d.  Nothing is read back (capturable in a CUDA graph).  workspace:
 * bg_train_step_depth_workspace_bytes(n, k, w, h) bytes (else BG_ERR_CAPACITY).  weight == 0 or valid_count == 0 runs
 * bg_train_step itself (bit-identical results) and writes 0 to depth_loss_out.  A negative or non-finite weight is
 * BG_ERR_INVALID; a null args, depth or depth_loss_out (or a null target when the term runs) is BG_ERR_NULL. */
uint64_t bg_train_step_depth_workspace_bytes(uint32_t n, uint32_t k, uint32_t w, uint32_t h);
int32_t bg_train_step_depth(BgContext *ctx, void *stream, BgTrainStepArgs *args, const BgDepthSupervision *depth);

/* The parameter update of one step as ONE pass over the Gaussians (update.cu): AdamScaled::step on the three parameter
 * tensors (brush-train/src/adam_scaled.rs:75-165, train.rs:328-381), RefineRecord::gather_stats (stats.rs:40-50) and the
 * mean noise (train.rs:389-416; the draw is bg_normal_noise(seed, (step-1)*ceil(3n/4) ..)).  Gradients are the dense
 * outputs of bg_project_backward; v_refine / visible / max_radius are the step's statistics.  bg_train_step and
 * bg_train_step_views end with this pass; it is exported for hosts that drive the operators themselves. */
typedef struct {
    uint32_t n, k;
    float *transforms, *sh, *raw_opac;              /* [n,10] [n,k,3] [n], updated in place */
    float *m_t, *v_t, *m_sh, *v_sh, *m_o, *v_o;     /* Adam moments; v_sh is [n] */
    float *refine_norm, *vis_weight, *max_screen;   /* RefineRecord, [n] each */
    const float *v_transforms, *v_sh_grad, *v_raw_opac;   /* gradients [n,10] [n,k,3] [n] */
    const float *v_refine, *visible, *max_radius;   /* [n] each */
    float lr_mean, lr_rotation, lr_scale, lr_coeffs_dc, lr_coeffs_sh_scale, lr_opac;
    float noise_scale, median_scale;
    uint64_t seed;
    int32_t step;                                   /* 1-based Adam step; step == 1 initialises the moments */
} BgTrainUpdateArgs;
int32_t bg_train_update(BgContext *ctx, void *stream, const BgTrainUpdateArgs *args);

/* SplatTrainer::refine (brush-train/src/train.rs:431-893) on the device: prune (opacity < 1/255, scale or position
 * beyond max_allowed, non-finite) -> replace the pruned splats by splitting survivors sampled by opacity x visibility
 * -> force-split splats larger than split_at_screen_size on screen -> sample growth_select_fraction of the splats whose
 * refine weight exceeds growth_grad_threshold -> split (refine_splats, :665-821: child opacity 1-(1-o)^(1/sqrt2),
 * per-axis shrink, +-offset along the rotated scale, zero Adam moments on both halves) -> opacity decay.
 * Weighted sampling without replacement (multinomial.rs:1-26) is Efraimidis-Spirakis on the device: keys
 * log(u_i)/w_i from the counter-based stream (seed, refine_index), the context's radix sort, the k best taken.
 * Sources are [n,...]; destinations have `capacity` rows (capacity >= min(2n, max(n, max_splats)) always suffices).
 * The call synchronises `stream` once, at its end, to return the counts; BG_ERR_CAPACITY if capacity was too small.
 * The refine record (refine_norm, vis_weight, max_screen) restarts at zero after a refine (train.rs:442-445): the
 * caller allocates it for stats_out->total_splats. */
typedef struct {
    uint32_t num_added, num_split_oversized, num_split_high_grad, num_pruned, num_pruned_non_finite, total_splats;
} BgRefineStats;
typedef struct {
    uint32_t n, k, capacity;
    const float *transforms, *sh, *raw_opac;                /* [n,10] [n,k,3] [n] */
    const float *m_t, *v_t, *m_sh, *v_sh, *m_o, *v_o;       /* Adam moments (v_sh: [n]) */
    const float *refine_norm, *vis_weight, *max_screen;     /* RefineRecord since the last refine */
    float *transforms_out, *sh_out, *raw_opac_out;          /* [capacity,...] */
    float *m_t_out, *v_t_out, *m_sh_out, *v_sh_out, *m_o_out, *v_o_out;
    float bounds_center[3];                                 /* self.bounds.center */
    float max_allowed;                                      /* self.bounds.extent.max_element() * 100 */
    float split_at_screen_size, growth_grad_threshold, growth_select_fraction;
    uint32_t max_splats;
    int32_t growth_enabled;                                 /* iter < growth_stop_iter */
    float opac_decay_minus;                                 /* opac_decay * (1 - clamp(iter / total_iters, 0, 1)) */
    uint64_t seed;
    uint32_t refine_index;                                  /* selects the random stream (the iteration number) */
    void *workspace;
    uint64_t workspace_bytes;                               /* >= bg_refine_workspace_bytes(n) */
} BgRefineArgs;
uint64_t bg_refine_workspace_bytes(uint32_t n);
int32_t bg_refine(BgContext *ctx, void *stream, const BgRefineArgs *args, BgRefineStats *stats_out /* host */);

/* bounds_from_pos (brush-train/src/splat_init.rs:130-160): per axis the ((1-p)/2, (1+p)/2) order statistics of the
 * finite means, through three radix sorts.  out6 (host): (lo, hi) for x, y, z; NaN when no finite value exists.
 * workspace: bg_refine_workspace_bytes(n).  Synchronises `stream`. */
int32_t bg_bounds_percentile(BgContext *ctx, void *stream, uint32_t n, const float *transforms, float percentile,
                             void *workspace, uint64_t workspace_bytes, float *out6);

/* Mip-Splatting 3D smoothing filter (scale floor).
 * bg_compute_min_scale  <- compute_min_scale (brush-train/src/train.rs:102-125):
 *     f[i] = sqrt(factor) * min_v(|mean_i - cam_v| / max(focal_v, 1e-6)); view_cams: DEVICE [views,4] =
 *     (x, y, z, focal_px), 16-byte aligned.  views == 0 or factor <= 0 is BG_ERR_INVALID (the reference
 *     returns None: the caller simply has no floor).
 * bg_fold_min_scale_forward <- fold_min_scale (brush-render/src/gaussian_splats.rs:86-111): scales become
 *     sqrt(s^2+f^2), opacity is multiplied by sqrt(det(s^2)/det(s^2+f^2)) and clamped to [1e-6, 1-1e-6];
 *     outputs may alias the inputs (Splats::bake_min_scale, :245-252).
 * bg_fold_min_scale_backward: what burn's autodiff derives for that fold.  IN PLACE: on entry
 *     v_transforms[:,7:10] / v_raw_opac hold the gradients w.r.t. the FOLDED values (as written by
 *     bg_project_backward on a render of the folded parameters), on exit w.r.t. the learned ones.
 *     transforms / raw_opac are the learned (un-folded) parameters; f is a constant. */
int32_t bg_compute_min_scale(BgContext *ctx, void *stream, uint32_t n, const float *transforms,
                             const float *view_cams, uint32_t views, float factor, float *f_out);
int32_t bg_fold_min_scale_forward(BgContext *ctx, void *stream, uint32_t n, const float *transforms,
                                  const float *raw_opac, const float *f, float *transforms_out,
                                  float *raw_opac_out);
int32_t bg_fold_min_scale_backward(BgContext *ctx, void *stream, uint32_t n, const float *transforms,
                                   const float *raw_opac, const float *f, float *v_transforms,
                                   float *v_raw_opac);

/* ---- LOD baking (brush-train/src/lod.rs).
 * bg_pup_accumulate <- the per-view step of compute_pup_scores (lod.rs:78-142): with J = (v_transforms[i, 0:3],
 *     v_transforms[i, 7:10]) (the gradient w.r.t. means and log-scales of one view), H_i += J J^T in f32, product and sum
 *     rounded separately.  fisher: [21, n] entry-major upper triangle (rows 00,01,..,05,11,..,15,22,..,55); first != 0
 *     writes 0 + J J^T (the reference's zero-initialised accumulator), so no zero-fill is needed.  The per-view chain
 *     before it (render with a zero background and the hard cutoff -> L1 gradient of the mean over [h,w,3] ->
 *     bg_rasterize_backward -> bg_project_backward_factored -> bg_fold_min_scale_backward when a floor exists) stays
 *     with the host, as in the reference.
 * bg_pup_log_det <- log_det_6x6 (lod.rs:44-69): scores[i] = 2 * sum ln(l_jj) of the f32 Cholesky factor of H_i, in the
 *     reference's loop order with IEEE sqrt / division and the deterministic log; -inf as soon as a pivot is <= 0; a NaN
 *     entry gives NaN. */
int32_t bg_pup_accumulate(BgContext *ctx, void *stream, uint32_t n, const float *v_transforms, int32_t first,
                          float *fisher);
int32_t bg_pup_log_det(BgContext *ctx, void *stream, uint32_t n, const float *fisher, float *scores);

/* decimate_to_count (lod.rs:13-40) without a readback: keeps the `target` highest scores, rows in DESCENDING score order,
 * index order among equal scores (the reference's stable sort_by); -inf ranks below every finite score and NaN scores
 * go last, in index order.  Gathers transforms, SH, opacity and, when min_scale is not NULL, the scale floor (so the
 * kept splats render exactly as before).  target >= n (or 0): nothing is written -- the reference returns its input
 * unchanged, and the caller keeps the source arrays.  Arrays 16-byte aligned; destinations hold `target` rows and must
 * not overlap the sources.  kept_ids_out (optional, [target]): the source index of each kept row.  The sort runs on
 * the context's radix sort: n <= the context's sort capacity, else BG_ERR_CAPACITY. */
typedef struct {
    uint32_t n, k, target;
    const float *scores;                                    /* [n] */
    const float *transforms, *sh, *raw_opac;                /* [n,10] [n,k,3] [n] */
    const float *min_scale;                                 /* [n] or NULL */
    float *transforms_out, *sh_out, *raw_opac_out;          /* [target,10] [target,k,3] [target] */
    float *min_scale_out;                                   /* [target]; required when min_scale != NULL */
    uint32_t *kept_ids_out;                                 /* [target] or NULL */
    void *workspace;                                        /* device, 256-byte aligned */
    uint64_t workspace_bytes;                               /* >= bg_decimate_workspace_bytes(n) */
} BgDecimateArgs;
uint64_t bg_decimate_workspace_bytes(uint32_t n);
int32_t bg_decimate_to_count(BgContext *ctx, void *stream, const BgDecimateArgs *args);

/* ---- View-sharded data parallelism behind the boundary (SURVEY.md section 8e; the reference is single-device).
 * A communicator is one NCCL rank bound to the context's device.  Rank 0 calls bg_dp_unique_id and ships the 128 bytes
 * to the other ranks by any side channel (the Python mirror uses torch.distributed's store; a Rust host would use
 * its own rendezvous); every rank then calls bg_dp_comm_create (collective).  NCCL is bound at run time
 * (libnccl.so.2); without it these calls return BG_ERR_UNSUPPORTED and everything else works. */
typedef struct BgDpComm BgDpComm;
#define BG_DP_UNIQUE_ID_BYTES 128
int32_t bg_dp_unique_id(uint8_t *out_id /* host [128] */);
int32_t bg_dp_comm_create(BgContext *ctx, const uint8_t *id /* host [128] */, int32_t rank, int32_t world,
                          BgDpComm **out_comm);
int32_t bg_dp_comm_destroy(BgDpComm *comm);

/* Exchange buffers for n Gaussians and `local_views` views per rank, interleaved per Gaussian (so that a slice of the
 * Gaussian range is one contiguous piece of each):
 *   small  [n][12]               v_transforms (10) | v_raw_opac | visible, summed over the rank's views  (all-reduce SUM)
 *   stat   [n][2]                v_refine | max_radius, MAX over the rank's views                       (all-reduce MAX)
 *   record [n][3 local_views]    v_color of each local view                                             (all-gather)
 *   recv   world * record floats the gathered records, per slice [world][len][3 local_views]
 * bg_dp_pack_view folds one view's operator outputs (bg_project_backward_factored, the forward's visible / max_radius)
 * into `small` / `stat` / `record`: the first view of a step assigns, the others accumulate. */
uint64_t bg_dp_small_floats(uint32_t n);
uint64_t bg_dp_stat_floats(uint32_t n);
uint64_t bg_dp_record_floats(uint32_t n, uint32_t local_views);
int32_t bg_dp_pack_view(BgContext *ctx, void *stream, uint32_t n, uint32_t local_views, uint32_t view, int32_t first,
                        const float *v_transforms, const float *v_raw_opac, const float *v_color, const float *v_refine,
                        const float *visible, const float *max_radius, float *small, float *stat, float *record);

/* The gradient exchange of one step on its own: all-gather of the records, all-reduce of `small` (SUM) and `stat` (MAX)
 * in place, all on the communicator's stream behind everything already enqueued on `stream`; `stream` waits for the
 * result.  chunks (1..16) slices the Gaussian range (one group of collectives per slice). */
int32_t bg_dp_exchange(BgContext *ctx, BgDpComm *comm, void *stream, uint32_t n, uint32_t local_views,
                       float *small, float *stat, const float *record, float *recv, uint32_t chunks);

/* One optimizer step over views_total = world * local_views views (BASELINE config [4]): the loss is the mean of the
 * per-view losses (train.rs:254-260 per view), i.e. the step equals accumulating the views' gradients on one GPU.
 * Per rank: for each local view render -> L1+SSIM loss -> rasterize / project backward (SH gradient kept in its
 * rank-one form).  The exchange runs on the communicator's stream in two parts: the all-gather of the colour records
 * starts right behind the last view's rasterize backward and travels UNDER its projection backward; the all-reduces of
 * `small` / `stat` follow.  The SH part of the update pass (bg_train_update's kernel in its factored form: it needs the
 * records only) runs UNDER the all-reduces, the rest of the update behind them.  comm == NULL runs the same step on one device.  Every rank must pass the same
 * n, local_views, learning rates, seed and step; cams / gt_packed are this rank's views, global view index =
 * rank * local_views + i.  min_scale (optional, [n]): the Mip-Splatting scale floor folded in for the renders and
 * chained out of the gradients (gaussian_splats.rs:86-111).  loss_out: mean loss of this rank's views. */
typedef struct {
    uint32_t w, h, n, k;
    int32_t mip;
    float background[3];
    uint32_t local_views;
    const BgCamera *cams;                           /* host [local_views] */
    const uint32_t *const *gt_packed;               /* host [local_views] device pointers, each [h,w] rgba8 */
    float *transforms, *sh, *raw_opac;
    float *m_t, *v_t, *m_sh, *v_sh, *m_o, *v_o;
    float *refine_norm, *vis_weight, *max_screen;
    const float *min_scale;                         /* device [n] or NULL */
    float l1_weight, ssim_weight;
    int32_t has_composite_bg;
    float composite_bg[3];
    int32_t mask, channels;
    float alpha_weight;
    float lr_mean, lr_rotation, lr_scale, lr_coeffs_dc, lr_coeffs_sh_scale, lr_opac;
    float noise_scale, median_scale;
    uint64_t seed;
    int32_t step;
    uint32_t chunks;                                /* reserved, pass 0 (<= 16) */
    void *workspace;
    uint64_t workspace_bytes;
    float *loss_out;
    BgRenderState state_out;                        /* render state of the last local view */
} BgTrainViewsArgs;
uint64_t bg_train_step_views_workspace_bytes(uint32_t n, uint32_t k, uint32_t w, uint32_t h, uint32_t local_views,
                                             uint32_t world);
int32_t bg_train_step_views(BgContext *ctx, BgDpComm *comm, void *stream, BgTrainViewsArgs *args);

/* Building blocks of the exchange for hosts that drive the operators themselves.  The SH part of the
 * gradient of ONE view is rank one per Gaussian: v_sh[g,k,:] = Y_k(dir(mean_g, camera)) * v_color[g,:]
 * (kernels/sh.rs:265-355).  bg_project_backward_factored is bg_project_backward without the dense v_sh:
 * it writes v_color [n,3] instead (zeros where no gradient).  Ranks all-reduce v_transforms / v_raw_opac,
 * all-gather their v_color rows (12 B instead of 12K B per Gaussian), and bg_sh_grad_from_views rebuilds
 *   v_sh[g,k,:] = out_scale * sum_v Y_k(dir(mean_g, cam_positions[v])) * v_color_all[v,g,:]
 * in view order (bit-identical on every rank).  cam_positions: host float[views*3]; views <= 16.
 * view_stride: floats between the colour blocks of consecutive views (0 = n*3, dense); larger when each view's
 * all-gathered record also carries other per-Gaussian values (refine weight, radius) behind its colours. */
int32_t bg_project_backward_factored(BgContext *ctx, void *stream, const BgCamera *cam, const BgRenderState *state,
                                     const float *transforms, const float *sh, const float *raw_opac,
                                     const float *v_combined, float *v_transforms, float *v_color,
                                     float *v_raw_opac, float *v_refine);
int32_t bg_sh_grad_from_views(BgContext *ctx, void *stream, uint32_t n, uint32_t k, const float *transforms,
                              const float *cam_positions, uint32_t views, const float *v_color_all,
                              uint64_t view_stride, float out_scale, float *v_sh);

/* Replaces brush_sort::radix_argsort, brush-sort/src/lib.rs:16-125: stable ascending sort of
 * (key,value) pairs on the low `bits` bits.  n_dev (device, may be null) overrides n with a
 * device-resident count <= n. */
int32_t bg_radix_argsort_u32(BgContext *ctx, void *stream, const uint32_t *keys, const uint32_t *vals,
                             uint32_t n, const uint32_t *n_dev, uint32_t bits, uint32_t *keys_out,
                             uint32_t *vals_out);

/* Replaces brush_prefix_sum::prefix_sum, brush-prefix-sum/src/lib.rs:11-89 (inclusive). */
int32_t bg_inclusive_scan_u32(BgContext *ctx, void *stream, const uint32_t *in, uint32_t n, uint32_t *out);

/* Replaces LossOps::image_loss_forward / image_loss_backward, brush-loss/src/lib.rs:718-733
 * (kernels lib.rs:180-359, 370-661).  pred and dl_dpred are addressed as
 * p[c*stride_c + y*stride_y + x*stride_x] so both the reference's CHW-permuted tensor (stride_c=h*w,
 * stride_y=w, stride_x=1) and the rasterizer's [h,w,4] image (stride_c=1, stride_y=4w, stride_x=4)
 * are accepted without a permute; loss_map and dl_dmap are dense [channels,h,w].
 * channels in {3,4}; channel 3 is the alpha-match path.  bg: host float[3] or null (no compositing). */
int32_t bg_image_loss_forward(BgContext *ctx, void *stream, const float *pred, const uint32_t *gt_packed,
                              uint32_t channels, uint32_t h, uint32_t w, int64_t stride_c, int64_t stride_y,
                              int64_t stride_x, float l1_weight, float ssim_weight, const float *bg,
                              int32_t mask, float *loss_map);
int32_t bg_image_loss_backward(BgContext *ctx, void *stream, const float *pred, const uint32_t *gt_packed,
                               const float *dl_dmap, uint32_t channels, uint32_t h, uint32_t w,
                               int64_t stride_c, int64_t stride_y, int64_t stride_x, float l1_weight,
                               float ssim_weight, const float *bg, int32_t mask, float *dl_dpred);

/* Train-path fusion of the two calls above for a mean-reduced loss (brush-train/src/train.rs:254-260:
 * loss = mean(map) [+ match_alpha_weight * mean(alpha map)], so dL/dmap is one constant per channel):
 * writes dL/dpred and per-block partial sums of the loss map in ONE pass.  chain_per_channel: host
 * float[channels] (= dL/dmap per channel).  loss_partials: device float[bg_image_loss_num_partials()];
 * sum of partials of channel blocks = sum of that channel's map.  Partials are laid out channel-major:
 * partials[ch * (n/channels) .. (ch+1) * (n/channels)). */
uint32_t bg_image_loss_num_partials(uint32_t channels, uint32_t h, uint32_t w);
int32_t bg_image_loss_fused(BgContext *ctx, void *stream, const float *pred, const uint32_t *gt_packed,
                            uint32_t channels, uint32_t h, uint32_t w, int64_t stride_c, int64_t stride_y,
                            int64_t stride_x, float l1_weight, float ssim_weight, const float *bg, int32_t mask,
                            const float *chain_per_channel, float *dl_dpred, float *loss_partials);

/* Replaces AdamScaled::step for one parameter tensor, brush-train/src/adam_scaled.rs:75-165.
 * p,g,m: [rows,cols]; v: [rows,cols], or [rows] when reduce_v (second moment = row mean of g^2).
 * lr_scale_per_col: device [cols] or null.  t: 1-based step count (t == 1 initialises the moments). */
int32_t bg_adam_step(BgContext *ctx, void *stream, float *p, const float *g, float *m, float *v,
                     uint64_t rows, uint32_t cols, const float *lr_scale_per_col, float lr, float beta1,
                     float beta2, float eps, int32_t t, int32_t reduce_v);

/* Replaces RefineRecord::gather_stats (brush-train/src/stats.rs:40-50) and the mean-noise update
 * (brush-train/src/train.rs:389-416) in one pass over the Gaussians.  noise: device [n,3] standard
 * normal draws (null skips the noise update). */
int32_t bg_refine_stats_noise(BgContext *ctx, void *stream, uint32_t n, const float *v_refine,
                              const float *visible, const float *max_radius, float *refine_weight_norm,
                              float *vis_weight, float *max_screen_size, float *transforms,
                              const float *raw_opac, const float *noise, float noise_scale,
                              float median_scale);

#ifdef __cplusplus
}
#endif
#endif /* BRUSH_B200_H */
