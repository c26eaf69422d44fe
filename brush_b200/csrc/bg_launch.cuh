// bg_launch.cuh -- every host-callable function that a kernel file defines and api.cu calls, declared once, with the
// parameter names of its definition.  Included by api.cu and by each defining .cu, grouped by defining file.
// (dp.cu, update.cu and refine.cu keep theirs beside the types they share with api.cu: bg_dp.cuh, bg_update.cuh,
// bg_refine.cuh.)
//
// Pointers are device pointers unless a comment says host.  `s` is the stream every launch goes to; `grid` is the CTA
// count of a persistent kernel, chosen by the caller from the SM count.  `ctl` is the control block of bg_common.cuh.
// A look-back chain takes its state words `lb`, the per-context device epoch word `epoch_base` and the index
// `epoch_off` of the launch inside the API call.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/brush_b200.h"

namespace bg {

// ---- project.cu
// K1: culls and projects all n Gaussians in index order.  Writes, per visible splat in index order, depth_keys / gids
// (the unsorted depth-sort input), and by global id counts [n] (tiles hit), max_radius [n], row_by_gid [n,16] (the
// finished projected row + tile hit bits) and cgid_from_gid [n] = 0xFFFFFFFF; counts the depth-key digits into ctl.
cudaError_t launch_project_cull(cudaStream_t s, int grid, bool mip, int deg, const float *transforms, const float *sh,
                                const float *raw_opac, uint32_t n, const BgCamera &u, uint32_t w, uint32_t h,
                                uint32_t tx, uint32_t ty, uint32_t *depth_keys, uint32_t *gids, uint32_t *counts,
                                float *max_radius, uint32_t *cgid_from_gid, float *row_by_gid, uint32_t *ctl,
                                unsigned long long *lb, const uint32_t *epoch_base, uint32_t epoch_off);
// out[i] = inclusive sum of in[gather_idx[i]] (in[i] when gather_idx is null) over i < min(n_host, *n_dev).  total_out
// gets the last sum clamped to capacity, overflow_flag is set when it was clamped; n_dev, total_out and overflow_flag
// may be null.
cudaError_t launch_gather_scan(cudaStream_t s, int grid, const uint32_t *in, const uint32_t *gather_idx,
                               uint32_t n_host, const uint32_t *n_dev, uint32_t *out, uint32_t *total_out,
                               uint32_t capacity, uint32_t *overflow_flag, uint32_t *ticket,
                               unsigned long long *lb, const uint32_t *epoch_base, uint32_t epoch_off);
// K2+K3: in depth order (gid_sorted, cum from launch_gather_scan) gathers row_by_gid into projected [visible,16] and
// emits the unsorted (tile_keys, isect_vals) pairs, at most cap; sets cgid_from_gid of the visible splats to their
// depth-sorted compact id.  With tile_bits <= 16 it also counts the tile-key digits into ctl.
cudaError_t launch_project_visible_emit(cudaStream_t s, int grid, const float *row_by_gid, const uint32_t *gid_sorted,
                                        const uint32_t *cum, uint32_t tx, uint32_t ty, float *projected,
                                        uint32_t *tile_keys, uint32_t *isect_vals, uint32_t cap,
                                        uint32_t *cgid_from_gid, uint32_t *ctl, uint32_t tile_bits);
// K4: tile_offsets [num_tiles,2] = [first, one past last) of each tile in the sorted tile_ids (zeroed by the caller)
cudaError_t launch_tile_offsets(cudaStream_t s, int grid, const uint32_t *tile_ids, const uint32_t *ctl,
                                uint32_t num_tiles, uint32_t *tile_offsets);

// ---- sort.cu
// hist [passes,256] += digit counts of the low `bits` bits of the first min(n_host, *n_dev) keys (n_dev may be null)
cudaError_t launch_radix_hist(cudaStream_t s, int grid, const uint32_t *keys, uint32_t n_host, const uint32_t *n_dev,
                              uint32_t bits, uint32_t passes, uint32_t *hist);
// One stable pass on the `width`-bit digit at `shift`.  hist [256]: this digit's counts; ticket: one zeroed word;
// lb [tiles,256] and lb_group: the two levels of the look-back (sort_max_tiles sizes them).
cudaError_t launch_onesweep_pass(cudaStream_t s, int grid, const uint32_t *keys_in, const uint32_t *vals_in,
                                 uint32_t *keys_out, uint32_t *vals_out, uint32_t n_host, const uint32_t *n_dev,
                                 uint32_t shift, uint32_t width, const uint32_t *hist, uint32_t *ticket,
                                 unsigned long long *lb, unsigned long long *lb_group, const uint32_t *epoch_base,
                                 uint32_t epoch_off);
// the most tiles a pass over n keys walks
uint64_t sort_max_tiles(uint64_t n);
// once per API call, ahead of its look-back chains
cudaError_t launch_bump_epoch(cudaStream_t s, uint32_t *epoch_base);

// ---- blend_fwd.cu
// K5.  out_img: packed RGBA8 [h,w] u32 without bwd_info, float4 [h,w] with it.  bwd_info also writes visible [n] and the
// hand-off to the backward (live_masks, warp_batches: blend_common.cuh) and trims tile_offsets to the entries used.
// bg: host [3].  depths [visible] and out_depth [h,w]: both set (depth forward, bwd_info only) or out_depth null.
cudaError_t launch_blend_fwd(cudaStream_t s, bool bwd_info, bool smooth, uint32_t num_tiles, const float *projected,
                             const uint32_t *cgid_from_isect, uint32_t *tile_offsets, const uint32_t *gid_from_cgid, void *out_img,
                             float *visible, uint32_t *live_masks, uint32_t *warp_batches, uint32_t tiles_x, uint32_t w,
                             uint32_t h, const float *bg, const float *depths, float *out_depth);

// ---- blend_bwd.cu
// Replays the forward's hand-off; adds into v_combined [visible,10] (zeroed by the caller).  stats [4]: null, or the
// counting variant of bg_debug_blend_stats.  bg: host [3].  depths, out_depth, v_depth [h,w] and v_z [visible] (added
// into): all set for the adjoint of a depth forward, or all null.
cudaError_t launch_blend_bwd(cudaStream_t s, bool smooth, uint32_t num_tiles, const float *projected, const uint32_t *cgid_from_isect,
                             const uint32_t *tile_offsets, const float *out_img, const float *v_output, const uint32_t *live_masks,
                             const uint32_t *warp_batches, float *v_combined, unsigned long long *stats, uint32_t tiles_x,
                             uint32_t w, uint32_t h, const float *bg, const float *depths, const float *out_depth,
                             const float *v_depth, float *v_z);

// ---- project_bwd.cu
// v_combined [visible,10] by compact id -> v_transforms [n,10], v_raw_opac [n], v_refine [n] by global id, and either
// v_sh [n,K,3] (dense) or v_color_out [n,3] (factored, for launch_sh_grad_from_views); the other of the two is null.
cudaError_t launch_project_bwd(cudaStream_t s, bool mip, int deg, const float *transforms, const float *sh,
                               const float *raw_opac, const uint32_t *cgid_from_gid, const float *v_combined,
                               uint32_t n, const BgCamera &u, float *v_transforms, float *v_sh, float *v_raw_opac,
                               float *v_refine, float *v_color_out);
// v_transforms[gid, 0:3] += v_z[compact id] * (row 2 of the view rotation)
cudaError_t launch_depth_to_means(cudaStream_t s, const uint32_t *cgid_from_gid, const float *v_z, uint32_t n,
                                  const BgCamera &u, float *v_transforms);
// v_sh [n,K,3] = out_scale * the sum over views of the SH adjoint of v_color_all[view] ([n,3], view_stride floats
// apart).  cam_pos_host: host [views,3].
cudaError_t launch_sh_grad_from_views(cudaStream_t s, int deg, const float *transforms, const float *v_color_all,
                                      uint32_t n, const float *cam_pos_host, uint32_t views, float out_scale,
                                      float *v_sh, size_t view_stride);

// ---- loss.cu
// pred [h,w,*] with element strides (sc, sy, sx); gt: packed RGBA8 [h,w]; bg: null or the host [3] composite
// background; c = 3 or 4 channels.
cudaError_t launch_image_loss_fwd(cudaStream_t s, const float *pred, const uint32_t *gt, uint32_t c, uint32_t h,
                                  uint32_t w, int64_t sc, int64_t sy, int64_t sx, float l1_w, float ssim_w,
                                  const float *bg, bool mask, float *loss_map);
cudaError_t launch_image_loss_bwd(cudaStream_t s, const float *pred, const uint32_t *gt, const float *dl_dmap,
                                  uint32_t c, uint32_t h, uint32_t w, int64_t sc, int64_t sy, int64_t sx, float l1_w,
                                  float ssim_w, const float *bg, bool mask, float *dl_dpred);
// value and gradient in one pass.  chain_per_channel: host [c], dL/d(the channel's sum); loss_partials
// [c, image_loss_fused_num_partials / c], channel major, for launch_loss_reduce
cudaError_t launch_image_loss_fused(cudaStream_t s, const float *pred, const uint32_t *gt, uint32_t c, uint32_t h,
                                    uint32_t w, int64_t sc, int64_t sy, int64_t sx, float l1_w, float ssim_w,
                                    const float *bg, bool mask, const float *chain_per_channel, float *dl_dpred,
                                    float *loss_partials);
uint32_t image_loss_fused_num_partials(uint32_t c, uint32_t h, uint32_t w);

// ---- optim.cu
// One AdamScaled step of p [rows,cols].  lr_scale: null or device [cols]; bc1, bc2 = 1 - beta^t.
cudaError_t launch_adam(cudaStream_t s, float *p, const float *g, float *m, float *v, uint64_t rows, uint32_t cols,
                        const float *lr_scale, float lr, float beta1, float beta2, float eps, float bc1, float bc2,
                        bool first, bool reduce_v);
// Folds one step's v_refine / visible / max_radius into the running statistics; with noise ([n,3], may be null) also
// perturbs the means in transforms.
cudaError_t launch_refine_stats_noise(cudaStream_t s, uint32_t n, const float *v_refine, const float *visible,
                                      const float *max_radius, float *refine_norm, float *vis_weight,
                                      float *max_screen, float *transforms, const float *raw_opac, const float *noise,
                                      float noise_scale, float median_scale);
// f_out [n]: the 3D-filter floor over the cameras cams [views,4] = (x, y, z, focal_px), 16-byte aligned
cudaError_t launch_min_scale(cudaStream_t s, uint32_t n, const float *transforms, const float *cams, uint32_t views,
                             float factor, float *f_out);
cudaError_t launch_fold_min_scale_fwd(cudaStream_t s, uint32_t n, const float *transforms, const float *raw_opac,
                                      const float *f, float *transforms_out, float *raw_opac_out);
// in place: gradients w.r.t. the folded values -> w.r.t. the learned ones
cudaError_t launch_fold_min_scale_bwd(cudaStream_t s, uint32_t n, const float *transforms, const float *raw_opac,
                                      const float *f, float *v_transforms, float *v_raw_opac);
// the same on rows vt_stride / vo_stride floats apart (the exchange rows of bg_dp.cuh)
cudaError_t launch_fold_min_scale_bwd_strided(cudaStream_t s, uint32_t n, const float *transforms, const float *raw_opac,
                                              const float *f, float *v_transforms, float *v_raw_opac, uint32_t vt_stride,
                                              uint32_t vo_stride);
// *out = mean of terms[0..count)
cudaError_t launch_loss_mean(cudaStream_t s, const float *terms, uint32_t count, float *out);
cudaError_t launch_normal_noise(cudaStream_t s, uint64_t seed, uint64_t offset, uint64_t count, float *out);
// *loss_out = sum over channels of chain[c] * (sum of the channel's per_channel partials).  chain: host [4].
cudaError_t launch_loss_reduce(cudaStream_t s, const float *partials, uint32_t channels, uint32_t per_channel,
                               const float *chain, float *loss_out);

// ---- lod.cu
// fisher [21,n]: packed upper triangle of sum J J^T, J = v_transforms[:, (0,1,2,7,8,9)]; first starts the sum from zero
cudaError_t launch_pup_accumulate(cudaStream_t s, uint32_t n, const float *v_transforms, bool first, float *fisher);
cudaError_t launch_pup_log_det(cudaStream_t s, uint32_t n, const float *fisher, float *scores);
// keys [n]: ascending key order == descending score (NaN last); vals [n] = index
cudaError_t launch_decimate_keys(cudaStream_t s, uint32_t n, const float *scores, uint32_t *keys, uint32_t *vals);
// rows ids[0..target) of each array -> the _out arrays; min_scale and min_scale_out both set or both null
cudaError_t launch_decimate_gather(cudaStream_t s, uint32_t target, uint32_t kf, const uint32_t *ids, const float *transforms,
                                   const float *sh, const float *raw_opac, const float *min_scale, float *transforms_out,
                                   float *sh_out, float *raw_opac_out, float *min_scale_out);

// ---- compress.cu
// keys [n] = 0 for a row that is kept, 1 << 30 for a dropped one (a non-finite value or a zero quaternion); bounds [7]:
// the kept count, then the ordered-u32 minima and maxima of the kept means
cudaError_t launch_compress_valid_bounds(cudaStream_t s, uint32_t n, uint32_t kf, const float *transforms, const float *sh,
                                         const float *raw_opac, uint32_t *keys, uint32_t *bounds);
// keys [n] (in: the marks above) = 30-bit Morton code of the kept means inside bounds, dropped rows stay 1 << 30;
// vals [n] = index
cudaError_t launch_compress_keys(cudaStream_t s, uint32_t n, const float *transforms, const uint32_t *bounds, uint32_t *keys,
                                 uint32_t *vals);
// Encodes the kept rows in `order` (the sorted vals), 256 per chunk; sh_out (k == 1) and order_out may be null;
// *count_out = the kept count.
cudaError_t launch_compress_chunks(cudaStream_t s, uint32_t n, uint32_t k, const float *transforms, const float *sh,
                                   const float *raw_opac, const uint32_t *bounds, const uint32_t *order, float *chunks_out,
                                   uint32_t *packed_out, uint8_t *sh_out, uint32_t *order_out, uint32_t *count_out);

// ---- mesh.cu
// img: float4 [h,w], depth [h,w]: one rendered view fused into the grid's tsdf / weight / rgb
cudaError_t launch_tsdf_integrate(cudaStream_t s, const BgTsdfGrid &g, const BgCamera &cam, uint32_t w, uint32_t h,
                                  const float *img, const float *depth, float alpha_min);
// dims: host [3]; 8x8x8-point bricks
uint32_t mesh_num_bricks(const uint32_t *dims);
// Per brick vertex / triangle counts (brick_v, brick_t) and their exclusive sums (voff, toff), all [bricks];
// header [8]: vertex total, triangle total, the dims counted.
cudaError_t launch_mesh_count(cudaStream_t s, const BgTsdfGrid &g, uint32_t *brick_v, uint32_t *brick_t, uint32_t *voff,
                              uint32_t *toff, unsigned long long *header);
// From the voff / toff of launch_mesh_count on the same grid.  vbase [points] and vmask [points] are scratch that the
// vertex pass writes and the face pass reads.
cudaError_t launch_mesh_emit(cudaStream_t s, const BgTsdfGrid &g, const uint32_t *voff, const uint32_t *toff, uint32_t *vbase,
                             uint8_t *vmask, uint32_t max_vertices, uint32_t max_triangles, float *verts, uint8_t *colors,
                             uint32_t *faces);

// ---- mesh_sparse.cu
// The grid workspace (bg_sparse_tsdf_workspace_bytes): header [8] u64 (allocated bricks, -, allocated flag, dims),
// the candidate count, the mark bitmap [ceil(bricks / 32)], per-1024-brick counts and offsets, `list` [bricks] (the
// candidates of the view being marked, then the brick of every slot) and the view's expected-depth pyramid.
constexpr uint32_t SPARSE_H_BRICKS = 0, SPARSE_H_ALLOCATED = 2, SPARSE_H_DIMS = 3;
struct SparseTsdfWs {
    unsigned long long *header;
    uint32_t *cand_count, *bitmap, *blk_cnt, *blk_off, *list;
    float2 *pyramid;
};
// The extraction workspace (bg_sparse_mesh_workspace_bytes): header [8] u64 (vertex total, triangle total, slots counted,
// dims), per-slot counts and offsets, and each pool point's vertex base and edge mask.
struct SparseMeshWs {
    unsigned long long *header;
    uint32_t *brick_v, *brick_t, *voff, *toff, *vbase;
    uint8_t *vmask;
};
uint64_t sparse_pyramid_cells(uint32_t w, uint32_t h);
// img: float4 [h,w], depth [h,w]: ORs the bricks holding a point that this view updates with f < 0 into the bitmap
cudaError_t launch_sparse_mark(cudaStream_t s, int sm_count, const BgSparseTsdfGrid &g, const BgCamera &cam, uint32_t w, uint32_t h,
                               const float *img, const float *depth, float alpha_min, const SparseTsdfWs &ws);
// Dilates the bitmap by one brick, writes g.brick_slot and the brick of every slot, header[SPARSE_H_BRICKS] = the count
cudaError_t launch_sparse_allocate(cudaStream_t s, const BgSparseTsdfGrid &g, const SparseTsdfWs &ws);
// slots: the allocated count (<= g.num_bricks)
cudaError_t launch_sparse_integrate(cudaStream_t s, const BgSparseTsdfGrid &g, uint32_t slots, const BgCamera &cam, uint32_t w,
                                    uint32_t h, const float *img, const float *depth, float alpha_min, const SparseTsdfWs &ws);
cudaError_t launch_sparse_mesh_count(cudaStream_t s, const BgSparseTsdfGrid &g, uint32_t slots, const SparseTsdfWs &ws,
                                     const SparseMeshWs &m);
cudaError_t launch_sparse_mesh_emit(cudaStream_t s, const BgSparseTsdfGrid &g, uint32_t slots, const SparseTsdfWs &ws,
                                    const SparseMeshWs &m, uint32_t max_vertices, uint32_t max_triangles, float *verts,
                                    uint8_t *colors, uint32_t *faces);

// ---- depth_loss.cu
uint32_t depth_loss_num_partials(uint32_t h, uint32_t w);
// out_img / v_output: float4 [h,w]; adds the depth term's gradient to v_output[..., 3], writes v_depth [h,w] and
// partials [depth_loss_num_partials]
cudaError_t launch_depth_loss_fused(cudaStream_t s, const float *out_img, const float *depth, const float *target, uint32_t h,
                                    uint32_t w, float chain, float *v_output, float *v_depth, float *partials);
// *depth_loss_out = chain * sum(partials); *loss_out (may be null) += the same
cudaError_t launch_depth_loss_reduce(cudaStream_t s, const float *partials, uint32_t count, float chain, float *depth_loss_out,
                                     float *loss_out);

// ---- bilagrid.cu
// grid [L,H,W,12], img / out float4 [h,w] (out may not alias img)
cudaError_t launch_bilagrid_slice(cudaStream_t s, const float *grid, const float *img, uint32_t w, uint32_t h, float *out);
// v_img = the adjoint of the slice w.r.t. img (may alias v_out); v_grid [L,H,W,12] is overwritten
cudaError_t launch_bilagrid_slice_bwd(cudaStream_t s, const float *grid, const float *img, const float *v_out, uint32_t w,
                                      uint32_t h, float *v_img, float *v_grid);
// v_grid += tv_weight * dTV/dgrid; *tv_out = tv_weight * TV(grid); *loss_out (may be null) += the same
cudaError_t launch_bilagrid_tv(cudaStream_t s, const float *grid, float *v_grid, float tv_weight, float *tv_out, float *loss_out);
// The grid update of the multi-view step (DESIGN.md section 4.11), one launch for all `slots` gradient slots: slot j is
// v_slots + j * slot_stride ([L,H,W,12], += the TV gradient) of view slot_view[j * view_stride] (device).  Each distinct view
// takes ONE update: the sum of its slots in slot order, TV then Adam (bilagrid_tv_kernel's and adam_kernel's rounding, the
// bias corrections of steps[view] + 1), steps[view] += 1.  tv_out [out_count] (and loss_terms, may be null, +=) gets the TV
// value of slots out_begin.. out_begin + out_count - 1.  grids / m / v: [num_views][L,H,W,12].
cudaError_t launch_bilagrid_update_views(cudaStream_t s, float *grids, float *m, float *v, int32_t *steps, uint32_t num_views,
                                         float lr, float tv_weight, float *v_slots, uint32_t slot_stride, const uint32_t *slot_view,
                                         uint32_t view_stride, uint32_t slots, uint32_t out_begin, uint32_t out_count,
                                         float *tv_out, float *loss_terms);

}  // namespace bg
