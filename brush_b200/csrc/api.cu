// api.cu -- the extern "C" boundary declared in include/brush_b200.h: context/arena management and
// host-side orchestration of the kernels (what <MainBackendBase as SplatOps>::render does in
// brush-render/src/render.rs:37-315, minus its blocking readback).
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdint>
#include <cstring>
#include <new>

#include "bg_common.cuh"
#include "bg_project.cuh"
#include "bg_dp.cuh"
#include "bg_update.cuh"
#include "bg_refine.cuh"

namespace bg {
// project.cu
cudaError_t launch_project_cull(cudaStream_t, int, bool, const float *, const float *, uint32_t, const BgCamera &,
                                uint32_t, uint32_t, uint32_t, uint32_t, uint32_t *, uint32_t *, uint32_t *, float *,
                                uint32_t *, unsigned long long *, uint32_t *, unsigned long long *, const uint32_t *,
                                uint32_t);
cudaError_t launch_gather_scan(cudaStream_t, int, const uint32_t *, const uint32_t *, uint32_t, const uint32_t *,
                               uint32_t *, uint32_t *, uint32_t, uint32_t *, uint32_t *, unsigned long long *,
                               const uint32_t *, uint32_t);
cudaError_t launch_project_visible_emit(cudaStream_t, int, bool, int, const float *, const float *, const float *,
                                        const uint32_t *, const uint32_t *, const BgCamera &, uint32_t, uint32_t,
                                        float *, uint32_t *, uint32_t *, uint32_t, uint32_t *, const unsigned long long *,
                                        uint32_t *, uint32_t);
cudaError_t launch_tile_offsets(cudaStream_t, int, const uint32_t *, const uint32_t *, uint32_t, uint32_t *);
// sort.cu
cudaError_t launch_radix_hist(cudaStream_t, int, const uint32_t *, uint32_t, const uint32_t *, uint32_t, uint32_t,
                              uint32_t *);
cudaError_t launch_onesweep_pass(cudaStream_t, int, const uint32_t *, const uint32_t *, uint32_t *, uint32_t *,
                                 uint32_t, const uint32_t *, uint32_t, uint32_t, const uint32_t *, uint32_t *,
                                 unsigned long long *, unsigned long long *, const uint32_t *, uint32_t);
cudaError_t launch_bump_epoch(cudaStream_t, uint32_t *);
uint64_t sort_max_tiles(uint64_t n);
// blend_fwd.cu / blend_bwd.cu
cudaError_t launch_blend_fwd(cudaStream_t, bool, bool, uint32_t, const float *, const uint32_t *, uint32_t *, const uint32_t *,
                             void *, float *, uint32_t *, uint32_t *, uint32_t, uint32_t, uint32_t, const float *, const float *,
                             float *);
cudaError_t launch_blend_bwd(cudaStream_t, bool, uint32_t, const float *, const uint32_t *, const uint32_t *, const float *,
                             const float *, const uint32_t *, const uint32_t *, float *, unsigned long long *, uint32_t,
                             uint32_t, uint32_t, const float *, const float *, const float *, const float *, float *);
// project_bwd.cu
cudaError_t launch_project_bwd(cudaStream_t, bool, int, const float *, const float *, const float *,
                               const uint32_t *, const float *, uint32_t, const BgCamera &, float *, float *, float *,
                               float *, float *);
cudaError_t launch_depth_to_means(cudaStream_t, const uint32_t *, const float *, uint32_t, const BgCamera &, float *);
cudaError_t launch_normal_noise(cudaStream_t, uint64_t, uint64_t, uint64_t, float *);
cudaError_t launch_train_fill_lr(cudaStream_t, float *, float *, uint32_t, float, float, float, float);
cudaError_t launch_loss_reduce(cudaStream_t, const float *, uint32_t, uint32_t, const float *, float *);
cudaError_t launch_min_scale(cudaStream_t, uint32_t, const float *, const float *, uint32_t, float, float *);
cudaError_t launch_fold_min_scale_fwd(cudaStream_t, uint32_t, const float *, const float *, const float *, float *, float *);
cudaError_t launch_fold_min_scale_bwd(cudaStream_t, uint32_t, const float *, const float *, const float *, float *, float *);
cudaError_t launch_fold_min_scale_bwd_strided(cudaStream_t, uint32_t, const float *, const float *, const float *, float *, float *,
                                              uint32_t, uint32_t);
cudaError_t launch_sh_grad_from_views(cudaStream_t, int, const float *, const float *, uint32_t, const float *, uint32_t,
                                      float, float *, size_t);
// loss.cu / optim.cu
cudaError_t launch_image_loss_fwd(cudaStream_t, const float *, const uint32_t *, uint32_t, uint32_t, uint32_t, int64_t,
                                  int64_t, int64_t, float, float, const float *, bool, float *);
cudaError_t launch_image_loss_bwd(cudaStream_t, const float *, const uint32_t *, const float *, uint32_t, uint32_t,
                                  uint32_t, int64_t, int64_t, int64_t, float, float, const float *, bool, float *);
cudaError_t launch_image_loss_fused(cudaStream_t, const float *, const uint32_t *, uint32_t, uint32_t, uint32_t, int64_t,
                                    int64_t, int64_t, float, float, const float *, bool, const float *, float *, float *);
uint32_t image_loss_fused_num_partials(uint32_t, uint32_t, uint32_t);
cudaError_t launch_adam(cudaStream_t, float *, const float *, float *, float *, uint64_t, uint32_t, const float *, float,
                        float, float, float, float, float, bool, bool);
cudaError_t launch_refine_stats_noise(cudaStream_t, uint32_t, const float *, const float *, const float *, float *,
                                      float *, float *, float *, const float *, const float *, float, float);
// lod.cu
cudaError_t launch_pup_accumulate(cudaStream_t, uint32_t, const float *, bool, float *);
cudaError_t launch_pup_log_det(cudaStream_t, uint32_t, const float *, float *);
cudaError_t launch_decimate_keys(cudaStream_t, uint32_t, const float *, uint32_t *, uint32_t *);
cudaError_t launch_decimate_gather(cudaStream_t, uint32_t, uint32_t, const uint32_t *, const float *, const float *,
                                   const float *, const float *, float *, float *, float *, float *);
// depth_loss.cu
uint32_t depth_loss_num_partials(uint32_t, uint32_t);
cudaError_t launch_depth_loss_fused(cudaStream_t, const float *, const float *, const float *, uint32_t, uint32_t, float, float *,
                                    float *, float *);
cudaError_t launch_depth_loss_reduce(cudaStream_t, const float *, uint32_t, float, float *, float *);
}  // namespace bg

using namespace bg;

static thread_local char g_err[512] = "";
static void set_err(const char *what, cudaError_t e) {
    snprintf(g_err, sizeof(g_err), "%s: %s", what, e == cudaSuccess ? "invalid argument" : cudaGetErrorString(e));
}

#define BG_CUDA(call)                          \
    do {                                       \
        cudaError_t e__ = (call);              \
        if (e__ != cudaSuccess) {              \
            set_err(#call, e__);               \
            return BG_ERR_CUDA;                \
        }                                      \
    } while (0)

struct BgContext {
    int device = 0;
    int sm_count = 0;
    uint32_t max_n = 0, max_w = 0, max_h = 0, max_tiles = 0;
    uint32_t max_isect = 0;
    uint32_t *epoch_dev = nullptr;          // device word: look-back epoch base, bumped on the stream per call
    uint64_t arena_bytes = 0;
    // device arena
    uint32_t *ctl = nullptr;               // CTL_WORDS u32 (forward pipeline), then CTL_WORDS (standalone ops)
    uint32_t *depth_key[2] = {nullptr, nullptr};
    uint32_t *depth_val[2] = {nullptr, nullptr};
    uint32_t *counts = nullptr, *cum = nullptr, *cgid_from_gid = nullptr;
    unsigned long long *hit_masks = nullptr;  // per-Gaussian tile hit bits from the counting pass
    float *projected = nullptr;
    uint32_t *isect_key[2] = {nullptr, nullptr};
    uint32_t *isect_val[2] = {nullptr, nullptr};
    uint32_t *tile_offsets = nullptr;
    // forward -> backward hand-off of the blend kernels (blend_common.cuh): per (tile, batch, warp) splat sets and
    // per (tile, warp) batch counts
    uint32_t *live_masks = nullptr, *warp_batches = nullptr;
    unsigned long long *blend_stats = nullptr;   // [4] development counters (bg_debug_blend_stats)
    unsigned long long *lb_scan = nullptr;  // look-back words for project/scan kernels
    unsigned long long *lb_sort = nullptr;  // look-back words for the sort passes: [tiles][256]
    uint64_t lb_scan_words = 0, lb_sort_words = 0, lb_sort_tile_words = 0;
    uint32_t *counters_host = nullptr;      // pinned [4]
    // last forward (for state pointers)
    int depth_out = 0, isect_out = 0;
    bool depth_forward = false;   // the last forward also accumulated depth (bg_render_forward_depth)
};

// Launch indices inside one API call (each look-back chain of a call gets its own epoch).
enum EpochSlots : uint32_t { EP_PROJECT = 0, EP_DEPTH_SORT = 1 /* ..4 */, EP_SCAN = 5, EP_TILE_SORT = 6 /* ..9 */ };

extern "C" uint32_t bg_abi_version(void) { return BG_ABI_VERSION; }
extern "C" const char *bg_last_error_string(void) { return g_err; }

template <typename T>
static cudaError_t arena_alloc(BgContext *c, T **p, uint64_t count) {
    uint64_t bytes = std::max<uint64_t>(count, 1) * sizeof(T);
    bytes = (bytes + 255) & ~uint64_t(255);
    cudaError_t e = cudaMalloc((void **)p, bytes);
    if (e == cudaSuccess) c->arena_bytes += bytes;
    return e;
}

extern "C" int32_t bg_ctx_destroy(BgContext *c) {
    if (!c) return BG_ERR_NULL;
    cudaSetDevice(c->device);
    void *ptrs[] = {c->ctl, c->depth_key[0], c->depth_key[1], c->depth_val[0], c->depth_val[1], c->counts, c->cum,
                    c->cgid_from_gid, c->hit_masks, c->projected, c->isect_key[0], c->isect_key[1], c->isect_val[0], c->isect_val[1],
                    c->tile_offsets, c->lb_scan, c->lb_sort, c->epoch_dev, c->live_masks, c->warp_batches, c->blend_stats};
    for (void *p : ptrs)
        if (p) cudaFree(p);
    if (c->counters_host) cudaFreeHost(c->counters_host);
    delete c;
    return BG_OK;
}

extern "C" int32_t bg_ctx_create(int32_t device, uint32_t max_splats, uint32_t max_w, uint32_t max_h,
                                 uint64_t max_intersections, BgContext **out_ctx) {
    if (!out_ctx) return BG_ERR_NULL;
    *out_ctx = nullptr;
    if (max_splats == 0 || max_w == 0 || max_h == 0) { set_err("bg_ctx_create: zero capacity", cudaSuccess); return BG_ERR_INVALID; }
    if (max_intersections == 0) max_intersections = std::max<uint64_t>(16ull * max_splats, 1ull << 22);
    if (max_intersections >= (1ull << 31)) { set_err("bg_ctx_create: max_intersections must be < 2^31", cudaSuccess); return BG_ERR_INVALID; }
    BG_CUDA(cudaSetDevice(device));
    BgContext *c = new (std::nothrow) BgContext();
    if (!c) return BG_ERR_CUDA;
    c->device = device;
    c->max_n = max_splats; c->max_w = max_w; c->max_h = max_h;
    c->max_isect = (uint32_t)max_intersections;
    c->max_tiles = ((max_w + TILE_W - 1) / TILE_W) * ((max_h + TILE_W - 1) / TILE_W);
    cudaDeviceProp prop;
    cudaError_t e = cudaGetDeviceProperties(&prop, device);
    if (e != cudaSuccess) { set_err("cudaGetDeviceProperties", e); delete c; return BG_ERR_CUDA; }
    c->sm_count = prop.multiProcessorCount;
    const uint64_t n = max_splats, I = c->max_isect;
    const uint64_t sort_tiles = sort_max_tiles(std::max<uint64_t>(n, I));
    c->lb_sort_tile_words = sort_tiles * 256;
    c->lb_sort_words = c->lb_sort_tile_words + (sort_tiles / 16 + 2) * 256;   // tile counts + group totals
    c->lb_scan_words = (n + 255) / 256 + 64;
    bool ok = true;
    ok = ok && arena_alloc(c, &c->ctl, 2 * CTL_WORDS) == cudaSuccess;
    for (int i = 0; i < 2; i++) {
        ok = ok && arena_alloc(c, &c->depth_key[i], n) == cudaSuccess;
        ok = ok && arena_alloc(c, &c->depth_val[i], n) == cudaSuccess;
        ok = ok && arena_alloc(c, &c->isect_key[i], I) == cudaSuccess;
        ok = ok && arena_alloc(c, &c->isect_val[i], I) == cudaSuccess;
    }
    ok = ok && arena_alloc(c, &c->counts, n) == cudaSuccess;
    ok = ok && arena_alloc(c, &c->cum, n) == cudaSuccess;
    ok = ok && arena_alloc(c, &c->cgid_from_gid, n) == cudaSuccess;
    ok = ok && arena_alloc(c, &c->hit_masks, n) == cudaSuccess;
    ok = ok && arena_alloc(c, &c->projected, n * BG_PROJECTED_STRIDE) == cudaSuccess;
    ok = ok && arena_alloc(c, &c->tile_offsets, (uint64_t)c->max_tiles * 2) == cudaSuccess;
    ok = ok && arena_alloc(c, &c->live_masks, (I / 32 + c->max_tiles + 2) * 4) == cudaSuccess;
    ok = ok && arena_alloc(c, &c->warp_batches, (uint64_t)c->max_tiles * 4) == cudaSuccess;
    ok = ok && arena_alloc(c, &c->blend_stats, 4) == cudaSuccess;
    ok = ok && arena_alloc(c, &c->lb_scan, c->lb_scan_words) == cudaSuccess;
    ok = ok && arena_alloc(c, &c->lb_sort, c->lb_sort_words) == cudaSuccess;
    ok = ok && arena_alloc(c, &c->epoch_dev, 1) == cudaSuccess;
    ok = ok && cudaHostAlloc((void **)&c->counters_host, 16 * sizeof(uint32_t), cudaHostAllocDefault) == cudaSuccess;
    if (ok) {
        ok = cudaMemset(c->lb_scan, 0, c->lb_scan_words * 8) == cudaSuccess &&
             cudaMemset(c->lb_sort, 0, c->lb_sort_words * 8) == cudaSuccess &&
             cudaMemset(c->ctl, 0, 2 * CTL_WORDS * 4) == cudaSuccess &&
             cudaMemset(c->epoch_dev, 0, 4) == cudaSuccess;
    }
    if (!ok) {
        set_err("bg_ctx_create: arena allocation", cudaGetLastError());
        bg_ctx_destroy(c);
        return BG_ERR_CUDA;
    }
    memset(c->counters_host, 0, 16 * sizeof(uint32_t));
    *out_ctx = c;
    return BG_OK;
}

extern "C" uint64_t bg_ctx_arena_bytes(const BgContext *c) { return c ? c->arena_bytes : 0; }

// One-sweep sort of the low `bits` bits.  bufs: ping-pong pairs; the input is (key_in,val_in); the
// result lands in (keys[out_idx], vals[out_idx]) where out_idx is returned.  `hist` must be zero.
static int32_t run_sort(BgContext *c, cudaStream_t s, const uint32_t *key_in, const uint32_t *val_in,
                        uint32_t *keys[2], uint32_t *vals[2], uint32_t n_host, const uint32_t *n_dev, uint32_t bits,
                        uint32_t *hist, uint32_t *tickets /* [1 + passes] zeroed */, int first_dst, uint32_t epoch_slot0,
                        int *out_idx, bool hist_ready = false /* the producer of the keys already counted the digits */) {
    const uint32_t passes = (bits + 7) / 8;
    *out_idx = first_dst;
    if (passes == 0 || n_host == 0) return BG_OK;
    const int grid = c->sm_count * 4;
    if (!hist_ready) BG_CUDA(launch_radix_hist(s, grid, key_in, n_host, n_dev, bits, passes, hist));
    const uint32_t *kin = key_in, *vin = val_in;
    int dst = first_dst;
    for (uint32_t p = 0; p < passes; p++) {
        const uint32_t shift = p * 8, width = std::min(8u, bits - shift);
        BG_CUDA(launch_onesweep_pass(s, c->sm_count * 3, kin, vin, keys[dst], vals[dst], n_host, n_dev, shift, width,
                                     hist + p * 256, tickets + 1 + p, c->lb_sort, c->lb_sort + c->lb_sort_tile_words, c->epoch_dev,
                                     epoch_slot0 + p));
        kin = keys[dst]; vin = vals[dst];
        *out_idx = dst;
        dst ^= 1;
    }
    return BG_OK;
}

// out_depth == nullptr: bg_render_forward; otherwise the depth forward (validated by bg_render_forward_depth)
static int32_t render_forward(BgContext *c, void *stream, const BgCamera *cam, uint32_t w, uint32_t h, uint32_t n,
                              uint32_t k, const float *transforms, const float *sh, const float *raw_opac, int32_t mip,
                              const float *bg, int32_t pass, void *out_img, float *out_depth, float *visible,
                              float *max_radius, BgRenderState *st) {
    if (!c || !cam || !bg || !out_img || !st) return BG_ERR_NULL;
    if (n > 0 && !max_radius) return BG_ERR_NULL;
    if (n > 0 && (!transforms || !sh || !raw_opac)) return BG_ERR_NULL;
    if (w == 0 || h == 0) { set_err("Can't render images with 0 size", cudaSuccess); return BG_ERR_INVALID; }
    const int deg = sh_degree_from_k(k);
    if (deg < 0) { set_err("Invalid nr. of sh bases", cudaSuccess); return BG_ERR_INVALID; }
    if (pass < 0 || pass > 2) { set_err("invalid pass", cudaSuccess); return BG_ERR_INVALID; }
    if (cam->camera_model > BG_CAMERA_THIN_PRISM_FISHEYE) return BG_ERR_UNSUPPORTED;
    const bool bwd_info = pass != BG_PASS_FORWARD;
    if (bwd_info && n > 0 && !visible) return BG_ERR_NULL;
    if ((((uintptr_t)transforms) | ((uintptr_t)sh) | ((uintptr_t)raw_opac) | ((uintptr_t)out_img)) & 15u) {
        set_err("bg_render_forward: arrays must be 16-byte aligned (bulk / 128-bit access)", cudaSuccess);
        return BG_ERR_INVALID;
    }
    const uint32_t tiles_x = (w + TILE_W - 1) / TILE_W, tiles_y = (h + TILE_W - 1) / TILE_W;
    const uint32_t num_tiles = tiles_x * tiles_y;
    if (n > c->max_n || num_tiles > c->max_tiles) { set_err("bg_render_forward: exceeds context capacity", cudaSuccess); return BG_ERR_CAPACITY; }
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    c->depth_forward = out_depth != nullptr;

    BG_CUDA(launch_bump_epoch(s, c->epoch_dev));
    BG_CUDA(cudaMemsetAsync(c->ctl, 0, CTL_WORDS * sizeof(uint32_t), s));
    BG_CUDA(cudaMemsetAsync(c->tile_offsets, 0, (size_t)num_tiles * 2 * sizeof(uint32_t), s));
    if (bwd_info && n > 0) BG_CUDA(cudaMemsetAsync(visible, 0, (size_t)n * sizeof(float), s));

    const int pgrid = c->sm_count * 5;   // project_cull: 256-thread CTAs, 48 regs
    const int vgrid = c->sm_count * 6;   // project_visible_emit: 128-thread CTAs (8 CTAs/SM would force 64 regs and spill)
    uint32_t *counters = c->ctl + CTL_COUNTERS;
    // K1: cull + compaction in index order
    BG_CUDA(launch_project_cull(s, pgrid, mip != 0, transforms, raw_opac, n, *cam, w, h, tiles_x, tiles_y,
                                c->depth_key[0], c->depth_val[0], c->counts, max_radius, c->cgid_from_gid, c->hit_masks, c->ctl,
                                c->lb_scan, c->epoch_dev, EP_PROJECT));
    // depth sort: 32-bit keys, 4 passes, (0)->(1)->(0)->(1)->(0)
    int dout = 0;
    {
        int32_t r = run_sort(c, s, c->depth_key[0], c->depth_val[0], c->depth_key, c->depth_val, n, counters + 0, 32,
                             c->ctl + CTL_HIST_DEPTH, c->ctl + CTL_TICKETS + TK_DEPTH_HIST, 1, EP_DEPTH_SORT, &dout,
                             /*hist_ready=*/true);   // counted by project_cull
        if (r != BG_OK) return r;
    }
    c->depth_out = dout;
    const uint32_t *gid_sorted = c->depth_val[dout];
    // gather counts + inclusive scan -> cum, num_intersections
    BG_CUDA(launch_gather_scan(s, c->sm_count * 2, c->counts, gid_sorted, n, counters + 0, c->cum, counters + 1,
                               c->max_isect, counters + 2, c->ctl + CTL_TICKETS + TK_SCAN, c->lb_scan, c->epoch_dev, EP_SCAN));
    // tile sort on bits = 32 - clz(num_tiles)
    uint32_t bits = 0;
    while (bits < 32 && (num_tiles >> bits) != 0) bits++;
    // K2+K3 (also counts the tile-key digits for the sort when they fit two passes)
    if (n > 0)
        BG_CUDA(launch_project_visible_emit(s, vgrid, mip != 0, deg, transforms, sh, raw_opac, gid_sorted, c->cum, *cam,
                                            tiles_x, tiles_y, c->projected, c->isect_key[0], c->isect_val[0],
                                            c->max_isect, c->cgid_from_gid, c->hit_masks, c->ctl, bits));
    int iout = 0;
    {
        const uint32_t passes = (bits + 7) / 8;
        const int first_dst = 1;
        int32_t r = run_sort(c, s, c->isect_key[0], c->isect_val[0], c->isect_key, c->isect_val, c->max_isect,
                             counters + 1, bits, c->ctl + CTL_HIST_TILE, c->ctl + CTL_TICKETS + TK_TILE_HIST, first_dst,
                             EP_TILE_SORT, &iout, /*hist_ready=*/n > 0 && bits <= 16);
        if (r != BG_OK) return r;
        (void)passes;
    }
    c->isect_out = iout;
    // K4
    BG_CUDA(launch_tile_offsets(s, c->sm_count * 16, c->isect_key[iout], c->ctl, num_tiles, c->tile_offsets));
    // K5 (BG_PASS_BACKWARD_SMOOTH: the test-only smooth alpha cutoff of the finite-difference suites)
    BG_CUDA(launch_blend_fwd(s, bwd_info, pass == BG_PASS_BACKWARD_SMOOTH, num_tiles, c->projected, c->isect_val[iout],
                             c->tile_offsets, gid_sorted, out_img, visible, c->live_masks, c->warp_batches, tiles_x, w, h, bg,
                             reinterpret_cast<const float *>(c->depth_key[dout]), out_depth));
    BG_CUDA(cudaMemcpyAsync(c->counters_host, counters, 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));

    st->projected = c->projected;
    st->compact_gid_from_isect = c->isect_val[iout];
    st->global_from_compact_gid = gid_sorted;
    st->compact_from_global_gid = c->cgid_from_gid;
    st->tile_offsets = c->tile_offsets;
    st->depths = reinterpret_cast<const float *>(c->depth_key[dout]);
    st->tile_id_from_isect = c->isect_key[iout];
    st->counters_dev = counters;
    st->counters_host = c->counters_host;
    st->n = n; st->k = k; st->w = w; st->h = h; st->tiles_x = tiles_x; st->tiles_y = tiles_y;
    st->mip = mip != 0; st->pass = pass;
    return BG_OK;
}

extern "C" int32_t bg_render_forward(BgContext *c, void *stream, const BgCamera *cam, uint32_t w, uint32_t h,
                                     uint32_t n, uint32_t k, const float *transforms, const float *sh,
                                     const float *raw_opac, int32_t mip, const float *bg, int32_t pass, void *out_img,
                                     float *visible, float *max_radius, BgRenderState *st) {
    return render_forward(c, stream, cam, w, h, n, k, transforms, sh, raw_opac, mip, bg, pass, out_img, nullptr, visible,
                          max_radius, st);
}

extern "C" int32_t bg_render_forward_depth(BgContext *c, void *stream, const BgCamera *cam, uint32_t w, uint32_t h,
                                           uint32_t n, uint32_t k, const float *transforms, const float *sh,
                                           const float *raw_opac, int32_t mip, const float *bg, int32_t pass,
                                           float *out_img, float *out_depth, float *visible, float *max_radius,
                                           BgRenderState *st) {
    if (!out_depth) return BG_ERR_NULL;
    if (pass != BG_PASS_BACKWARD && pass != BG_PASS_BACKWARD_SMOOTH) {
        set_err("bg_render_forward_depth: depth needs an f32 pass (BG_PASS_BACKWARD or BG_PASS_BACKWARD_SMOOTH)", cudaSuccess);
        return BG_ERR_INVALID;
    }
    if ((uintptr_t)out_depth % 4) { set_err("bg_render_forward_depth: out_depth must be 4-byte aligned", cudaSuccess); return BG_ERR_INVALID; }
    return render_forward(c, stream, cam, w, h, n, k, transforms, sh, raw_opac, mip, bg, pass, out_img, out_depth, visible,
                          max_radius, st);
}

// depth: out_depth / v_depth / v_z all set (bg_rasterize_backward_depth) or all null
static int32_t rasterize_backward(BgContext *c, void *stream, const BgRenderState *st, const float *out_img,
                                  const float *out_depth, const float *v_output, const float *v_depth, const float *bg,
                                  int32_t smooth, float *v_combined, uint32_t rows, float *v_z, const char *who) {
    auto invalid = [who](const char *what) {
        char m[160];
        snprintf(m, sizeof(m), "%s%s", who, what);
        set_err(m, cudaSuccess);
        return BG_ERR_INVALID;
    };
    if (st->pass == BG_PASS_FORWARD) return invalid(" requires a Backward pass state");
    const bool smooth_pass = st->pass == BG_PASS_BACKWARD_SMOOTH;
    if ((smooth != 0) != smooth_pass) return invalid(": smooth_cutoff must match the state's pass");
    if (st->tile_offsets != c->tile_offsets) return invalid(": needs the state of this context's last forward");
    if (v_z && !c->depth_forward) return invalid(": this context's last forward did not render depth");
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    const uint32_t zr = std::min(rows, std::max(st->n, 1u));
    BG_CUDA(cudaMemsetAsync(v_combined, 0, (size_t)zr * BG_VCOMBINED_STRIDE * sizeof(float), s));
    if (v_z) BG_CUDA(cudaMemsetAsync(v_z, 0, (size_t)zr * sizeof(float), s));
    // the forward of this context left its hand-off words: replay exactly the splats it used
    BG_CUDA(launch_blend_bwd(s, smooth_pass, st->tiles_x * st->tiles_y, c->projected, st->compact_gid_from_isect, st->tile_offsets,
                             out_img, v_output, c->live_masks, c->warp_batches, v_combined, nullptr, st->tiles_x, st->w, st->h, bg,
                             st->depths, out_depth, v_depth, v_z));
    return BG_OK;
}

extern "C" int32_t bg_rasterize_backward(BgContext *c, void *stream, const BgRenderState *st, const float *out_img,
                                         const float *v_output, const float *bg, int32_t smooth, float *v_combined,
                                         uint32_t rows) {
    if (!c || !st || !out_img || !v_output || !bg || !v_combined) return BG_ERR_NULL;
    return rasterize_backward(c, stream, st, out_img, nullptr, v_output, nullptr, bg, smooth, v_combined, rows, nullptr,
                              "bg_rasterize_backward");
}

extern "C" int32_t bg_rasterize_backward_depth(BgContext *c, void *stream, const BgRenderState *st, const float *out_img,
                                               const float *out_depth, const float *v_output, const float *v_depth,
                                               const float *bg, int32_t smooth, float *v_combined, uint32_t rows,
                                               float *v_z) {
    if (!c || !st || !out_img || !out_depth || !v_output || !v_depth || !bg || !v_combined || !v_z) return BG_ERR_NULL;
    if (((uintptr_t)out_depth | (uintptr_t)v_depth | (uintptr_t)v_z) % 4) {
        set_err("bg_rasterize_backward_depth: out_depth, v_depth and v_z must be 4-byte aligned", cudaSuccess);
        return BG_ERR_INVALID;
    }
    return rasterize_backward(c, stream, st, out_img, out_depth, v_output, v_depth, bg, smooth, v_combined, rows, v_z,
                              "bg_rasterize_backward_depth");
}

// Development counters of the blend loop for the last Backward-pass forward of this context:
// out[0] warp-splat iterations (64 pixel-splat pairs each), out[1] pairs that blended, out[2] pairs that stopped a
// pixel, out[3] tile-list entries (num_intersections).  Runs the backward kernel's counting variant into a scratch
// v_combined (caller-provided, [n,10]); synchronises the stream.
extern "C" int32_t bg_debug_blend_stats(BgContext *c, void *stream, const BgRenderState *st, const float *out_img,
                                        const float *v_output, const float *bg, float *v_combined_scratch,
                                        unsigned long long *out4) {
    if (!c || !st || !out_img || !v_output || !bg || !v_combined_scratch || !out4) return BG_ERR_NULL;
    if (st->pass != BG_PASS_BACKWARD || st->tile_offsets != c->tile_offsets) { set_err("bg_debug_blend_stats: needs the state of this context's last Backward pass", cudaSuccess); return BG_ERR_INVALID; }
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(cudaMemsetAsync(c->blend_stats, 0, 4 * sizeof(unsigned long long), s));
    BG_CUDA(launch_blend_bwd(s, false, st->tiles_x * st->tiles_y, c->projected, st->compact_gid_from_isect, st->tile_offsets, out_img,
                             v_output, c->live_masks, c->warp_batches, v_combined_scratch, c->blend_stats, st->tiles_x, st->w,
                             st->h, bg, nullptr, nullptr, nullptr, nullptr));
    BG_CUDA(cudaMemcpyAsync(out4, c->blend_stats, 4 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    BG_CUDA(cudaStreamSynchronize(s));
    out4[3] = st->counters_host ? st->counters_host[1] : 0;
    return BG_OK;
}

extern "C" int32_t bg_project_backward(BgContext *c, void *stream, const BgCamera *cam, const BgRenderState *st,
                                       const float *transforms, const float *sh, const float *raw_opac,
                                       const float *v_combined, float *v_transforms, float *v_sh, float *v_raw_opac,
                                       float *v_refine) {
    if (!c || !cam || !st || !v_combined || !v_transforms || !v_sh || !v_raw_opac || !v_refine) return BG_ERR_NULL;
    if (st->n > 0 && (!transforms || !sh || !raw_opac)) return BG_ERR_NULL;
    const int deg = sh_degree_from_k(st->k);
    if (deg < 0) return BG_ERR_INVALID;
    if (cam->camera_model > BG_CAMERA_THIN_PRISM_FISHEYE) return BG_ERR_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    if (((uintptr_t)sh | (uintptr_t)v_sh) % 16) {
        set_err("bg_project_backward: sh and v_sh must be 16-byte aligned (128-bit row access)", cudaSuccess);
        return BG_ERR_INVALID;
    }
    BG_CUDA(launch_project_bwd(s, st->mip != 0, deg, transforms, sh, raw_opac, st->compact_from_global_gid, v_combined,
                               st->n, *cam, v_transforms, v_sh, v_raw_opac, v_refine, nullptr));
    return BG_OK;
}

extern "C" int32_t bg_project_backward_depth(BgContext *c, void *stream, const BgCamera *cam, const BgRenderState *st,
                                             const float *transforms, const float *sh, const float *raw_opac,
                                             const float *v_combined, const float *v_z, float *v_transforms, float *v_sh,
                                             float *v_raw_opac, float *v_refine) {
    if (!v_z) return BG_ERR_NULL;
    if ((uintptr_t)v_z % 4) { set_err("bg_project_backward_depth: v_z must be 4-byte aligned", cudaSuccess); return BG_ERR_INVALID; }
    const int32_t r = bg_project_backward(c, stream, cam, st, transforms, sh, raw_opac, v_combined, v_transforms, v_sh,
                                          v_raw_opac, v_refine);
    if (r != BG_OK) return r;
    BG_CUDA(launch_depth_to_means((cudaStream_t)stream, st->compact_from_global_gid, v_z, st->n, *cam, v_transforms));
    return BG_OK;
}

extern "C" int32_t bg_project_backward_factored(BgContext *c, void *stream, const BgCamera *cam, const BgRenderState *st,
                                                const float *transforms, const float *sh, const float *raw_opac,
                                                const float *v_combined, float *v_transforms, float *v_color,
                                                float *v_raw_opac, float *v_refine) {
    if (!c || !cam || !st || !v_combined || !v_transforms || !v_color || !v_raw_opac || !v_refine) return BG_ERR_NULL;
    if (st->n > 0 && (!transforms || !sh || !raw_opac)) return BG_ERR_NULL;
    const int deg = sh_degree_from_k(st->k);
    if (deg < 0) return BG_ERR_INVALID;
    if (cam->camera_model > BG_CAMERA_THIN_PRISM_FISHEYE) return BG_ERR_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    if ((uintptr_t)sh % 16) {
        set_err("bg_project_backward_factored: sh must be 16-byte aligned (128-bit row access)", cudaSuccess);
        return BG_ERR_INVALID;
    }
    BG_CUDA(launch_project_bwd(s, st->mip != 0, deg, transforms, sh, raw_opac, st->compact_from_global_gid, v_combined,
                               st->n, *cam, v_transforms, nullptr, v_raw_opac, v_refine, v_color));
    return BG_OK;
}

extern "C" int32_t bg_sh_grad_from_views(BgContext *c, void *stream, uint32_t n, uint32_t k, const float *transforms,
                                         const float *cam_positions, uint32_t views, const float *v_color_all,
                                         uint64_t view_stride, float out_scale, float *v_sh) {
    if (!c) return BG_ERR_NULL;
    if (n == 0) return BG_OK;
    if (!transforms || !cam_positions || !v_color_all || !v_sh) return BG_ERR_NULL;
    const int deg = sh_degree_from_k(k);
    if (deg < 0 || views == 0 || views > 16) { set_err("bg_sh_grad_from_views: k must be a square <= 25, 1 <= views <= 16", cudaSuccess); return BG_ERR_INVALID; }
    BG_CUDA(cudaSetDevice(c->device));
    if (view_stride != 0 && view_stride < (uint64_t)n * 3) { set_err("bg_sh_grad_from_views: view_stride smaller than one view", cudaSuccess); return BG_ERR_INVALID; }
    BG_CUDA(launch_sh_grad_from_views((cudaStream_t)stream, deg, transforms, v_color_all, n, cam_positions, views, out_scale, v_sh,
                                      view_stride ? (size_t)view_stride : (size_t)n * 3));
    return BG_OK;
}

extern "C" int32_t bg_radix_argsort_u32(BgContext *c, void *stream, const uint32_t *keys, const uint32_t *vals,
                                        uint32_t n, const uint32_t *n_dev, uint32_t bits, uint32_t *keys_out,
                                        uint32_t *vals_out) {
    if (!c) return BG_ERR_NULL;
    if (n == 0) return BG_OK;
    if (!keys || !vals || !keys_out || !vals_out) return BG_ERR_NULL;
    if (bits > 32) { set_err("Can only sort up to 32 bits", cudaSuccess); return BG_ERR_INVALID; }
    if (n > std::max(c->max_n, c->max_isect)) { set_err("bg_radix_argsort_u32: n exceeds context capacity", cudaSuccess); return BG_ERR_CAPACITY; }
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    uint32_t *ctl2 = c->ctl + CTL_WORDS;
    BG_CUDA(launch_bump_epoch(s, c->epoch_dev));
    BG_CUDA(cudaMemsetAsync(ctl2, 0, CTL_WORDS * sizeof(uint32_t), s));
    const uint32_t passes = (bits + 7) / 8;
    if (passes == 0) {
        BG_CUDA(cudaMemcpyAsync(keys_out, keys, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
        BG_CUDA(cudaMemcpyAsync(vals_out, vals, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
        return BG_OK;
    }
    // temp = the intersection ping-pong buffer (large enough by the capacity check for n <= max_isect,
    // otherwise the depth buffers)
    uint32_t *tk = (n <= c->max_isect) ? c->isect_key[1] : c->depth_key[1];
    uint32_t *tv = (n <= c->max_isect) ? c->isect_val[1] : c->depth_val[1];
    uint32_t *kb[2] = {keys_out, tk};
    uint32_t *vb[2] = {vals_out, tv};
    const int first_dst = (passes & 1u) ? 0 : 1;  // so that the last pass writes into (keys_out, vals_out)
    int out_idx = 0;
    int32_t r = run_sort(c, s, keys, vals, kb, vb, n, n_dev, bits, ctl2 + CTL_HIST_DEPTH, ctl2 + CTL_TICKETS, first_dst,
                         EP_DEPTH_SORT, &out_idx);
    if (r != BG_OK) return r;
    if (out_idx != 0) { set_err("internal: sort parity", cudaSuccess); return BG_ERR_INVALID; }
    return BG_OK;
}

extern "C" int32_t bg_inclusive_scan_u32(BgContext *c, void *stream, const uint32_t *in, uint32_t n, uint32_t *out) {
    if (!c) return BG_ERR_NULL;
    if (n == 0) return BG_OK;
    if (!in || !out) return BG_ERR_NULL;
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    if ((uint64_t)(n + 2047) / 2048 > c->lb_scan_words) { set_err("bg_inclusive_scan_u32: n exceeds context capacity", cudaSuccess); return BG_ERR_CAPACITY; }
    uint32_t *ctl2 = c->ctl + CTL_WORDS;
    BG_CUDA(launch_bump_epoch(s, c->epoch_dev));
    BG_CUDA(cudaMemsetAsync(ctl2 + CTL_TICKETS, 0, 48 * sizeof(uint32_t), s));
    BG_CUDA(launch_gather_scan(s, c->sm_count * 2, in, nullptr, n, nullptr, out, nullptr, 0xFFFFFFFFu, nullptr,
                               ctl2 + CTL_TICKETS, c->lb_scan, c->epoch_dev, EP_SCAN));
    return BG_OK;
}

extern "C" int32_t bg_image_loss_forward(BgContext *c, void *stream, const float *pred, const uint32_t *gt,
                                         uint32_t channels, uint32_t h, uint32_t w, int64_t sc, int64_t sy, int64_t sx,
                                         float l1_w, float ssim_w, const float *bg, int32_t mask, float *loss_map) {
    if (!c || !pred || !gt || !loss_map) return BG_ERR_NULL;
    if (channels < 3 || channels > 4 || h == 0 || w == 0) { set_err("image_loss expects 3 or 4 channels and a non-empty image", cudaSuccess); return BG_ERR_INVALID; }
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_image_loss_fwd((cudaStream_t)stream, pred, gt, channels, h, w, sc, sy, sx, l1_w, ssim_w, bg, mask != 0,
                                  loss_map));
    return BG_OK;
}

extern "C" int32_t bg_image_loss_backward(BgContext *c, void *stream, const float *pred, const uint32_t *gt,
                                          const float *dl_dmap, uint32_t channels, uint32_t h, uint32_t w, int64_t sc,
                                          int64_t sy, int64_t sx, float l1_w, float ssim_w, const float *bg,
                                          int32_t mask, float *dl_dpred) {
    if (!c || !pred || !gt || !dl_dmap || !dl_dpred) return BG_ERR_NULL;
    if (channels < 3 || channels > 4 || h == 0 || w == 0) { set_err("image_loss expects 3 or 4 channels and a non-empty image", cudaSuccess); return BG_ERR_INVALID; }
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_image_loss_bwd((cudaStream_t)stream, pred, gt, dl_dmap, channels, h, w, sc, sy, sx, l1_w, ssim_w, bg,
                                  mask != 0, dl_dpred));
    return BG_OK;
}

extern "C" uint32_t bg_image_loss_num_partials(uint32_t channels, uint32_t h, uint32_t w) {
    return image_loss_fused_num_partials(channels, h, w);
}

extern "C" int32_t bg_image_loss_fused(BgContext *c, void *stream, const float *pred, const uint32_t *gt,
                                       uint32_t channels, uint32_t h, uint32_t w, int64_t sc, int64_t sy, int64_t sx,
                                       float l1_w, float ssim_w, const float *bg, int32_t mask,
                                       const float *chain_per_channel, float *dl_dpred, float *loss_partials) {
    if (!c || !pred || !gt || !chain_per_channel || !dl_dpred || !loss_partials) return BG_ERR_NULL;
    if (channels < 3 || channels > 4 || h == 0 || w == 0) { set_err("image_loss expects 3 or 4 channels and a non-empty image", cudaSuccess); return BG_ERR_INVALID; }
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_image_loss_fused((cudaStream_t)stream, pred, gt, channels, h, w, sc, sy, sx, l1_w, ssim_w, bg,
                                    mask != 0, chain_per_channel, dl_dpred, loss_partials));
    return BG_OK;
}

extern "C" uint32_t bg_depth_loss_num_partials(uint32_t h, uint32_t w) { return depth_loss_num_partials(h, w); }

extern "C" int32_t bg_depth_loss_fused(BgContext *c, void *stream, const float *out_img, const float *depth,
                                       const float *target, uint32_t h, uint32_t w, float chain, float *v_output,
                                       float *v_depth, float *partials) {
    if (!c || !out_img || !depth || !target || !v_output || !v_depth || !partials) return BG_ERR_NULL;
    if (h == 0 || w == 0) { set_err("bg_depth_loss_fused: empty image", cudaSuccess); return BG_ERR_INVALID; }
    if (!(chain >= 0.0f) || !std::isfinite(chain)) { set_err("bg_depth_loss_fused: chain must be finite and >= 0", cudaSuccess); return BG_ERR_INVALID; }
    if ((((uintptr_t)out_img) | ((uintptr_t)v_output)) & 15u) {
        set_err("bg_depth_loss_fused: out_img and v_output must be 16-byte aligned (128-bit pixel access)", cudaSuccess);
        return BG_ERR_INVALID;
    }
    if ((((uintptr_t)depth) | ((uintptr_t)target) | ((uintptr_t)v_depth) | ((uintptr_t)partials)) & 3u) {
        set_err("bg_depth_loss_fused: depth, target, v_depth and partials must be 4-byte aligned", cudaSuccess);
        return BG_ERR_INVALID;
    }
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_depth_loss_fused((cudaStream_t)stream, out_img, depth, target, h, w, chain, v_output, v_depth, partials));
    return BG_OK;
}

// compiler-rt __powisf2, what Rust's f32::powi lowers to (adam_scaled.rs:135-142)
static float powi_f32(float a, int b) {
    const bool recip = b < 0;
    float r = 1.0f;
    while (true) {
        if (b & 1) r *= a;
        b /= 2;
        if (b == 0) break;
        a *= a;
    }
    return recip ? 1.0f / r : r;
}

extern "C" int32_t bg_adam_step(BgContext *c, void *stream, float *p, const float *g, float *m, float *v,
                                uint64_t rows, uint32_t cols, const float *lr_scale, float lr, float beta1, float beta2,
                                float eps, int32_t t, int32_t reduce_v) {
    if (!c) return BG_ERR_NULL;
    if (rows == 0 || cols == 0) return BG_OK;
    if (!p || !g || !m || !v) return BG_ERR_NULL;
    if (t < 1) { set_err("bg_adam_step: t is 1-based", cudaSuccess); return BG_ERR_INVALID; }
    BG_CUDA(cudaSetDevice(c->device));
    const float bc1 = 1.0f - powi_f32(beta1, t), bc2 = 1.0f - powi_f32(beta2, t);
    BG_CUDA(launch_adam((cudaStream_t)stream, p, g, m, v, rows, cols, lr_scale, lr, beta1, beta2, eps, bc1, bc2, t == 1,
                        reduce_v != 0));
    return BG_OK;
}

extern "C" int32_t bg_refine_stats_noise(BgContext *c, void *stream, uint32_t n, const float *v_refine,
                                         const float *visible, const float *max_radius, float *refine_weight_norm,
                                         float *vis_weight, float *max_screen_size, float *transforms,
                                         const float *raw_opac, const float *noise, float noise_scale,
                                         float median_scale) {
    if (!c) return BG_ERR_NULL;
    if (n == 0) return BG_OK;
    if (!v_refine || !visible || !max_radius || !refine_weight_norm || !vis_weight || !max_screen_size) return BG_ERR_NULL;
    if (noise && (!transforms || !raw_opac)) return BG_ERR_NULL;
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_refine_stats_noise((cudaStream_t)stream, n, v_refine, visible, max_radius, refine_weight_norm,
                                      vis_weight, max_screen_size, transforms, raw_opac, noise, noise_scale,
                                      median_scale));
    return BG_OK;
}

extern "C" int32_t bg_compute_min_scale(BgContext *c, void *stream, uint32_t n, const float *transforms,
                                        const float *view_cams, uint32_t views, float factor, float *f_out) {
    if (!c) return BG_ERR_NULL;
    if (n == 0) return BG_OK;
    if (!transforms || !view_cams || !f_out) return BG_ERR_NULL;
    if (views == 0 || !(factor > 0.0f)) { set_err("bg_compute_min_scale: needs views > 0 and factor > 0 (the reference returns None)", cudaSuccess); return BG_ERR_INVALID; }
    if ((uintptr_t)view_cams % 16) { set_err("bg_compute_min_scale: view_cams must be 16-byte aligned", cudaSuccess); return BG_ERR_INVALID; }
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_min_scale((cudaStream_t)stream, n, transforms, view_cams, views, factor, f_out));
    return BG_OK;
}

extern "C" int32_t bg_fold_min_scale_forward(BgContext *c, void *stream, uint32_t n, const float *transforms,
                                             const float *raw_opac, const float *f, float *transforms_out,
                                             float *raw_opac_out) {
    if (!c) return BG_ERR_NULL;
    if (n == 0) return BG_OK;
    if (!transforms || !raw_opac || !f || !transforms_out || !raw_opac_out) return BG_ERR_NULL;
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_fold_min_scale_fwd((cudaStream_t)stream, n, transforms, raw_opac, f, transforms_out, raw_opac_out));
    return BG_OK;
}

extern "C" int32_t bg_fold_min_scale_backward(BgContext *c, void *stream, uint32_t n, const float *transforms,
                                              const float *raw_opac, const float *f, float *v_transforms,
                                              float *v_raw_opac) {
    if (!c) return BG_ERR_NULL;
    if (n == 0) return BG_OK;
    if (!transforms || !raw_opac || !f || !v_transforms || !v_raw_opac) return BG_ERR_NULL;
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_fold_min_scale_bwd((cudaStream_t)stream, n, transforms, raw_opac, f, v_transforms, v_raw_opac));
    return BG_OK;
}

extern "C" int32_t bg_normal_noise(BgContext *c, void *stream, uint64_t seed, uint64_t offset, uint64_t count, float *out) {
    if (!c) return BG_ERR_NULL;
    if (count == 0) return BG_OK;
    if (!out) return BG_ERR_NULL;
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_normal_noise((cudaStream_t)stream, seed, offset, count, out));
    return BG_OK;
}

// compiler-rt __powisf2 is defined above (powi_f32).  Fills the step-dependent constants of the update pass.
static void fill_update_consts(UpdateParams &P, float lr_mean, float lr_rotation, float lr_scale, float lr_coeffs_dc,
                               float lr_coeffs_sh_scale, float lr_opac, float noise_scale, float median_scale, uint64_t seed,
                               int32_t step, uint32_t n) {
    for (int i = 0; i < 10; i++) P.lr_t[i] = i < 3 ? lr_mean : (i < 7 ? lr_rotation : lr_scale);   // train.rs:328-350
    P.lr_sh_dc = 1.0f * lr_coeffs_dc;                                   // lr_scale_per_col * lr, as AdamScaled forms it
    P.lr_sh_rest = (1.0f / lr_coeffs_sh_scale) * lr_coeffs_dc;
    P.lr_opac = lr_opac;
    P.beta1 = 0.9f; P.beta2 = 0.999f; P.eps = 1e-15f; P.f1 = 1.0f - P.beta1; P.f2 = 1.0f - P.beta2;
    P.inv_bc1 = 1.0f / (1.0f - powi_f32(P.beta1, step)); P.inv_bc2 = 1.0f / (1.0f - powi_f32(P.beta2, step));
    P.first = step == 1;
    P.noisy = noise_scale != 0.0f;
    P.noise_scale = noise_scale; P.median_scale = median_scale;
    P.seed = seed;
    P.noise_offset = (unsigned long long)(step - 1) * (((unsigned long long)n * 3 + 3) / 4);
}

extern "C" int32_t bg_train_update(BgContext *c, void *stream, const BgTrainUpdateArgs *a) {
    if (!c || !a) return BG_ERR_NULL;
    if (a->n == 0) return BG_OK;
    if (!a->transforms || !a->sh || !a->raw_opac || !a->m_t || !a->v_t || !a->m_sh || !a->v_sh || !a->m_o || !a->v_o ||
        !a->refine_norm || !a->vis_weight || !a->max_screen || !a->v_transforms || !a->v_sh_grad || !a->v_raw_opac ||
        !a->v_refine || !a->visible || !a->max_radius)
        return BG_ERR_NULL;
    const int deg = sh_degree_from_k(a->k);
    if (deg < 0) { set_err("Invalid nr. of sh bases", cudaSuccess); return BG_ERR_INVALID; }
    if (a->step < 1) { set_err("bg_train_update: step is 1-based", cudaSuccess); return BG_ERR_INVALID; }
    BG_CUDA(cudaSetDevice(c->device));
    UpdateParams P;
    memset(&P, 0, sizeof(P));
    P.g_begin = 0; P.count = a->n;
    P.transforms = a->transforms; P.sh = a->sh; P.raw_opac = a->raw_opac;
    P.m_t = a->m_t; P.v_t = a->v_t; P.m_sh = a->m_sh; P.v_sh = a->v_sh; P.m_o = a->m_o; P.v_o = a->v_o;
    P.refine_norm = a->refine_norm; P.vis_weight = a->vis_weight; P.max_screen = a->max_screen;
    P.g_t = a->v_transforms; P.g_o = a->v_raw_opac; P.g_sh = a->v_sh_grad;
    P.grad_scale = 1.0f; P.sh_grad_scale = 1.0f;
    P.v_refine = a->v_refine; P.max_radius = a->max_radius; P.visible = a->visible;
    fill_update_consts(P, a->lr_mean, a->lr_rotation, a->lr_scale, a->lr_coeffs_dc, a->lr_coeffs_sh_scale, a->lr_opac,
                       a->noise_scale, a->median_scale, a->seed, a->step, a->n);
    BG_CUDA(launch_train_update((cudaStream_t)stream, deg, P, false));
    return BG_OK;
}

// ---- bg_train_step: SplatTrainer::step (brush-train/src/train.rs:176-429) as ONE call: every launch of the step on
// the caller's stream, nothing read back, scratch from a caller-provided workspace.
namespace {
struct TrainWs {
    float *out_img, *v_output, *partials, *v_combined, *v_t, *v_sh, *v_o, *v_r, *visible, *max_radius, *noise, *t_lr, *sh_scale;
    uint64_t bytes;
};
TrainWs carve_train_ws(void *base, uint32_t n, uint32_t k, uint32_t w, uint32_t h, uint32_t channels) {
    uint64_t off = 0;
    auto take = [&](uint64_t floats) {
        float *p = base ? reinterpret_cast<float *>(static_cast<char *>(base) + off) : nullptr;
        off += (floats * 4 + 255) / 256 * 256;
        return p;
    };
    TrainWs ws;
    const uint64_t px = (uint64_t)w * h;
    ws.out_img = take(px * 4);
    ws.v_output = take(px * 4);
    ws.partials = take(bg_image_loss_num_partials(channels, h, w));
    ws.v_combined = take((uint64_t)n * BG_VCOMBINED_STRIDE);
    ws.v_t = take((uint64_t)n * 10);
    ws.v_sh = take((uint64_t)n * k * 3);
    ws.v_o = take(n);
    ws.v_r = take(n);
    ws.visible = take(n);
    ws.max_radius = take(n);
    ws.noise = take((uint64_t)n * 3);
    ws.t_lr = take(16);
    ws.sh_scale = take((uint64_t)k * 3);
    ws.bytes = off;
    return ws;
}

// the depth step's extra scratch, behind the largest plain-step workspace
struct DepthWs {
    float *depth, *v_depth, *v_z, *partials;
    uint64_t bytes;
};
DepthWs carve_depth_ws(void *base, uint32_t n, uint32_t k, uint32_t w, uint32_t h) {
    uint64_t off = carve_train_ws(nullptr, n, k, w, h, 4).bytes;
    auto take = [&](uint64_t floats) {
        float *p = base ? reinterpret_cast<float *>(static_cast<char *>(base) + off) : nullptr;
        off += (floats * 4 + 255) / 256 * 256;
        return p;
    };
    DepthWs ws;
    const uint64_t px = (uint64_t)w * h;
    ws.depth = take(px);
    ws.v_depth = take(px);
    ws.v_z = take(std::max(n, 1u));
    ws.partials = take(depth_loss_num_partials(h, w));
    ws.bytes = off;
    return ws;
}

// argument checks shared by bg_train_step and bg_train_step_depth
int32_t check_train_args(const BgTrainStepArgs *a, const char *who) {
    if (!a->transforms || !a->sh || !a->raw_opac || !a->m_t || !a->v_t || !a->m_sh || !a->v_sh || !a->m_o || !a->v_o ||
        !a->refine_norm || !a->vis_weight || !a->max_screen || !a->gt_packed || !a->workspace || !a->loss_out)
        return BG_ERR_NULL;
    char m[160];
    auto invalid = [&](const char *what) {
        snprintf(m, sizeof(m), "%s: %s", who, what);
        set_err(m, cudaSuccess);
        return BG_ERR_INVALID;
    };
    if (a->step < 1) return invalid("step is 1-based");
    if (a->channels != 3 && a->channels != 4) return invalid("channels must be 3 or 4");
    if ((uintptr_t)a->workspace % 256) return invalid("workspace must be 256-byte aligned");
    return BG_OK;
}

// optimiser, refine statistics, mean noise (train.rs:280-416): one pass over the Gaussians
int32_t run_train_update(BgContext *c, void *stream, const BgTrainStepArgs *a, const TrainWs &ws) {
    BgTrainUpdateArgs up;
    memset(&up, 0, sizeof(up));
    up.n = a->n; up.k = a->k;
    up.transforms = a->transforms; up.sh = a->sh; up.raw_opac = a->raw_opac;
    up.m_t = a->m_t; up.v_t = a->v_t; up.m_sh = a->m_sh; up.v_sh = a->v_sh; up.m_o = a->m_o; up.v_o = a->v_o;
    up.refine_norm = a->refine_norm; up.vis_weight = a->vis_weight; up.max_screen = a->max_screen;
    up.v_transforms = ws.v_t; up.v_sh_grad = ws.v_sh; up.v_raw_opac = ws.v_o;
    up.v_refine = ws.v_r; up.visible = ws.visible; up.max_radius = ws.max_radius;
    up.lr_mean = a->lr_mean; up.lr_rotation = a->lr_rotation; up.lr_scale = a->lr_scale; up.lr_coeffs_dc = a->lr_coeffs_dc;
    up.lr_coeffs_sh_scale = a->lr_coeffs_sh_scale; up.lr_opac = a->lr_opac;
    up.noise_scale = a->noise_scale; up.median_scale = a->median_scale; up.seed = a->seed; up.step = a->step;
    return bg_train_update(c, stream, &up);
}
}  // namespace

extern "C" uint64_t bg_train_step_workspace_bytes(uint32_t n, uint32_t k, uint32_t w, uint32_t h) {
    return carve_train_ws(nullptr, n, k, w, h, 4).bytes;
}

extern "C" int32_t bg_train_step(BgContext *c, void *stream, BgTrainStepArgs *a) {
    if (!c || !a) return BG_ERR_NULL;
    if (int32_t r = check_train_args(a, "bg_train_step"); r != BG_OK) return r;
    const uint32_t n = a->n, k = a->k, w = a->w, h = a->h;
    const TrainWs ws = carve_train_ws(a->workspace, n, k, w, h, a->channels);
    if (ws.bytes > a->workspace_bytes) { set_err("bg_train_step: workspace too small (bg_train_step_workspace_bytes)", cudaSuccess); return BG_ERR_CAPACITY; }
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    int32_t r;
    // render forward (train.rs:200-216)
    r = bg_render_forward(c, stream, &a->cam, w, h, n, k, a->transforms, a->sh, a->raw_opac, a->mip, a->background, BG_PASS_BACKWARD,
                          ws.out_img, ws.visible, ws.max_radius, &a->state_out);
    if (r != BG_OK) return r;
    // loss value + gradient (train.rs:220-260): mean over [h,w,3] (+ alpha mean * weight)
    const float npx = (float)w * (float)h;
    float chain[4] = {1.0f / (3.0f * npx), 1.0f / (3.0f * npx), 1.0f / (3.0f * npx), a->channels == 4 ? a->alpha_weight / npx : 0.0f};
    BG_CUDA(cudaMemsetAsync(ws.v_output, 0, (size_t)w * h * 4 * sizeof(float), s));
    r = bg_image_loss_fused(c, stream, ws.out_img, a->gt_packed, a->channels, h, w, 1, (int64_t)w * 4, 4, a->l1_weight, a->ssim_weight,
                            a->has_composite_bg ? a->composite_bg : nullptr, a->mask, chain, ws.v_output, ws.partials);
    if (r != BG_OK) return r;
    BG_CUDA(launch_loss_reduce(s, ws.partials, a->channels, bg_image_loss_num_partials(a->channels, h, w) / a->channels, chain, a->loss_out));
    // backward (bwd/burn_glue.rs:121-182)
    r = bg_rasterize_backward(c, stream, &a->state_out, ws.out_img, ws.v_output, a->background, 0, ws.v_combined, n);
    if (r != BG_OK) return r;
    r = bg_project_backward(c, stream, &a->cam, &a->state_out, a->transforms, a->sh, a->raw_opac, ws.v_combined, ws.v_t, ws.v_sh, ws.v_o, ws.v_r);
    if (r != BG_OK) return r;
    return run_train_update(c, stream, a, ws);
}

// ---- bg_train_step_depth: bg_train_step with the depth-supervision term of DESIGN.md section 4.7
extern "C" uint64_t bg_train_step_depth_workspace_bytes(uint32_t n, uint32_t k, uint32_t w, uint32_t h) {
    return carve_depth_ws(nullptr, n, k, w, h).bytes;
}

extern "C" int32_t bg_train_step_depth(BgContext *c, void *stream, BgTrainStepArgs *a, const BgDepthSupervision *d) {
    if (!c || !a || !d || !d->depth_loss_out) return BG_ERR_NULL;
    if (!(d->weight >= 0.0f) || !std::isfinite(d->weight)) {
        set_err("bg_train_step_depth: weight must be finite and >= 0", cudaSuccess);
        return BG_ERR_INVALID;
    }
    cudaStream_t s = (cudaStream_t)stream;
    if (d->weight == 0.0f || d->valid_count == 0) {
        // no term (target may be null): the plain step, launch for launch, and a zero depth loss
        const int32_t r = bg_train_step(c, stream, a);
        if (r != BG_OK) return r;
        BG_CUDA(cudaMemsetAsync(d->depth_loss_out, 0, sizeof(float), s));
        return BG_OK;
    }
    if (!d->target) return BG_ERR_NULL;
    if (int32_t r = check_train_args(a, "bg_train_step_depth"); r != BG_OK) return r;
    const uint32_t n = a->n, k = a->k, w = a->w, h = a->h;
    const TrainWs ws = carve_train_ws(a->workspace, n, k, w, h, a->channels);
    const DepthWs dws = carve_depth_ws(a->workspace, n, k, w, h);
    if (dws.bytes > a->workspace_bytes) {
        set_err("bg_train_step_depth: workspace too small (bg_train_step_depth_workspace_bytes)", cudaSuccess);
        return BG_ERR_CAPACITY;
    }
    BG_CUDA(cudaSetDevice(c->device));
    int32_t r;
    r = bg_render_forward_depth(c, stream, &a->cam, w, h, n, k, a->transforms, a->sh, a->raw_opac, a->mip, a->background,
                                BG_PASS_BACKWARD, ws.out_img, dws.depth, ws.visible, ws.max_radius, &a->state_out);
    if (r != BG_OK) return r;
    const float npx = (float)w * (float)h;
    float chain[4] = {1.0f / (3.0f * npx), 1.0f / (3.0f * npx), 1.0f / (3.0f * npx), a->channels == 4 ? a->alpha_weight / npx : 0.0f};
    BG_CUDA(cudaMemsetAsync(ws.v_output, 0, (size_t)w * h * 4 * sizeof(float), s));
    r = bg_image_loss_fused(c, stream, ws.out_img, a->gt_packed, a->channels, h, w, 1, (int64_t)w * 4, 4, a->l1_weight, a->ssim_weight,
                            a->has_composite_bg ? a->composite_bg : nullptr, a->mask, chain, ws.v_output, ws.partials);
    if (r != BG_OK) return r;
    BG_CUDA(launch_loss_reduce(s, ws.partials, a->channels, bg_image_loss_num_partials(a->channels, h, w) / a->channels, chain, a->loss_out));
    // depth term: v_depth, v_output[...,3] += dL/da, L_d -> depth_loss_out and added to loss_out
    const float dchain = d->weight / (float)d->valid_count;
    r = bg_depth_loss_fused(c, stream, ws.out_img, dws.depth, d->target, h, w, dchain, ws.v_output, dws.v_depth, dws.partials);
    if (r != BG_OK) return r;
    BG_CUDA(launch_depth_loss_reduce(s, dws.partials, depth_loss_num_partials(h, w), dchain, d->depth_loss_out, a->loss_out));
    r = bg_rasterize_backward_depth(c, stream, &a->state_out, ws.out_img, dws.depth, ws.v_output, dws.v_depth, a->background, 0,
                                    ws.v_combined, n, dws.v_z);
    if (r != BG_OK) return r;
    r = bg_project_backward_depth(c, stream, &a->cam, &a->state_out, a->transforms, a->sh, a->raw_opac, ws.v_combined, dws.v_z,
                                  ws.v_t, ws.v_sh, ws.v_o, ws.v_r);
    if (r != BG_OK) return r;
    return run_train_update(c, stream, a, ws);
}

// ---- view-sharded data parallelism (dp.cu): communicator, exchange, the multi-view step
struct BgDpComm { DpComm *c; };

static int32_t nccl_fail(const char *what, int rc) {
    snprintf(g_err, sizeof(g_err), "%s: %s", what, rc < 0 ? "NCCL is not available (libnccl.so.2) or a CUDA call failed" : dp_nccl_error(rc));
    return rc == -1 ? BG_ERR_UNSUPPORTED : BG_ERR_CUDA;
}

extern "C" int32_t bg_dp_unique_id(uint8_t *out_id) {
    if (!out_id) return BG_ERR_NULL;
    NcclUniqueId id;
    const int rc = dp_unique_id(&id);
    if (rc != 0) return nccl_fail("bg_dp_unique_id", rc);
    memcpy(out_id, id.internal, BG_DP_UNIQUE_ID_BYTES);
    return BG_OK;
}

extern "C" int32_t bg_dp_comm_create(BgContext *c, const uint8_t *id_bytes, int32_t rank, int32_t world, BgDpComm **out) {
    if (!c || !id_bytes || !out) return BG_ERR_NULL;
    *out = nullptr;
    if (world < 1 || rank < 0 || rank >= world) { set_err("bg_dp_comm_create: rank/world", cudaSuccess); return BG_ERR_INVALID; }
    NcclUniqueId id;
    memcpy(id.internal, id_bytes, BG_DP_UNIQUE_ID_BYTES);
    int rc = 0;
    DpComm *d = dp_comm_create(c->device, id, rank, world, &rc);
    if (!d) return nccl_fail("bg_dp_comm_create", rc ? rc : -2);
    BgDpComm *h = new (std::nothrow) BgDpComm();
    if (!h) { dp_comm_destroy(d); return BG_ERR_CUDA; }
    h->c = d;
    *out = h;
    return BG_OK;
}

extern "C" int32_t bg_dp_comm_destroy(BgDpComm *h) {
    if (!h) return BG_ERR_NULL;
    dp_comm_destroy(h->c);
    delete h;
    return BG_OK;
}

extern "C" uint64_t bg_dp_small_floats(uint32_t n) { return (uint64_t)DP_SMALL_ROW * n; }
extern "C" uint64_t bg_dp_stat_floats(uint32_t n) { return (uint64_t)DP_STAT_ROW * n; }
extern "C" uint64_t bg_dp_record_floats(uint32_t n, uint32_t local) { return (uint64_t)3 * local * n; }

extern "C" int32_t bg_dp_pack_view(BgContext *c, void *stream, uint32_t n, uint32_t local, uint32_t view, int32_t first, const float *v_t,
                                   const float *v_o, const float *v_color, const float *v_refine, const float *visible,
                                   const float *max_radius, float *small, float *stat, float *record) {
    if (!c) return BG_ERR_NULL;
    if (n == 0) return BG_OK;
    if (!v_t || !v_o || !v_color || !v_refine || !visible || !max_radius || !small || !stat || !record) return BG_ERR_NULL;
    if (local == 0 || local > DP_MAX_VIEWS || view >= local) { set_err("bg_dp_pack_view: view index / views per rank", cudaSuccess); return BG_ERR_INVALID; }
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_pack_view((cudaStream_t)stream, n, local, view, first != 0, v_t, v_o, v_color, v_refine, visible, max_radius, small, stat, record));
    return BG_OK;
}

// Issues all slices of the exchange on the communicator's stream behind `s`; s waits for slice c through ev_chunk[c].
static int32_t issue_exchange(DpComm *d, cudaStream_t s, uint32_t n, uint32_t local, uint32_t chunks, float *small, float *stat,
                              const float *record, float *recv, const float *hdr, float *hdr_all) {
    BG_CUDA(cudaEventRecord(d->ev_ready, s));
    BG_CUDA(cudaStreamWaitEvent(d->stream, d->ev_ready, 0));
    if (hdr) {
        const int rc = dp_exchange_header(d, local, hdr, hdr_all);
        if (rc != 0) return nccl_fail("exchange (camera positions)", rc);
    }
    for (uint32_t ch = 0; ch < chunks; ch++) {
        const int rc = dp_exchange_chunk(d, n, local, chunks, ch, small, stat, record, recv);
        if (rc != 0) return nccl_fail("exchange", rc);
    }
    return BG_OK;
}

extern "C" int32_t bg_dp_exchange(BgContext *c, BgDpComm *h, void *stream, uint32_t n, uint32_t local, float *small, float *stat,
                                  const float *record, float *recv, uint32_t chunks) {
    if (!c || !h || !small || !stat || !record || !recv) return BG_ERR_NULL;
    if (n == 0) return BG_OK;
    if (local == 0 || local * (uint32_t)h->c->world > DP_MAX_VIEWS || chunks == 0 || chunks > DP_MAX_CHUNKS) {
        set_err("bg_dp_exchange: 1..16 views in total, 1..16 chunks", cudaSuccess);
        return BG_ERR_INVALID;
    }
    BG_CUDA(cudaSetDevice(c->device));
    cudaStream_t s = (cudaStream_t)stream;
    int32_t r = issue_exchange(h->c, s, n, local, chunks, small, stat, record, recv, nullptr, nullptr);
    if (r != BG_OK) return r;
    for (uint32_t ch = 0; ch < chunks; ch++) BG_CUDA(cudaStreamWaitEvent(s, h->c->ev_chunk[ch], 0));
    return BG_OK;
}

namespace {
struct ViewsWs {
    float *out_img, *v_output, *partials, *loss_terms, *v_combined, *small, *stat, *record, *recv, *hdr, *hdr_all;
    float *r_transforms, *r_opac, *v_t, *v_o, *v_color, *v_refine, *visible, *max_radius;
    uint64_t bytes;
};
ViewsWs carve_views_ws(void *base, uint32_t n, uint32_t k, uint32_t w, uint32_t h, uint32_t local, uint32_t world, bool fold) {
    uint64_t off = 0;
    auto take = [&](uint64_t floats) {
        float *p = base ? reinterpret_cast<float *>(static_cast<char *>(base) + off) : nullptr;
        off += (floats * 4 + 255) / 256 * 256;
        return p;
    };
    (void)k;
    ViewsWs ws;
    const uint64_t px = (uint64_t)w * h;
    const DpLayout L = dp_layout(n, local, world);
    ws.out_img = take(px * 4);
    ws.v_output = take(px * 4);
    ws.partials = take(bg_image_loss_num_partials(4, h, w));
    ws.loss_terms = take(DP_MAX_VIEWS);
    ws.v_combined = take((uint64_t)n * BG_VCOMBINED_STRIDE);
    ws.small = take(L.small_floats);
    ws.stat = take(L.stat_floats);
    ws.record = take(L.rec_floats);
    ws.recv = take(world > 1 ? L.recv_floats : 0);
    ws.hdr = take(DP_MAX_VIEWS * 4);
    ws.hdr_all = take(DP_MAX_VIEWS * 4);
    ws.r_transforms = take(fold ? (uint64_t)n * 10 : 0);
    ws.r_opac = take(fold ? n : 0);
    // one view's gradients, as the operators write them, before they are folded into the exchange rows
    ws.v_t = take((uint64_t)n * 10); ws.v_o = take(n); ws.v_color = take((uint64_t)n * 3); ws.v_refine = take(n);
    ws.visible = take(n); ws.max_radius = take(n);
    ws.bytes = off;
    return ws;
}
}  // namespace

namespace bg {
cudaError_t launch_loss_mean(cudaStream_t, const float *, uint32_t, float *);
}

// BG_DP_TRACE=1: device timeline of the multi-device step (stderr, rank 0 only; synchronises -- a debugging aid)
namespace {
struct DpTrace {
    bool on = false;
    cudaEvent_t e[12] = {};
    DpTrace() {
        const char *v = getenv("BG_DP_TRACE");
        on = v && v[0] == '1';
    }
    void mark(int i, cudaStream_t st) {
        if (!on) return;
        if (!e[i]) cudaEventCreate(&e[i]);
        cudaEventRecord(e[i], st);
    }
    void report(cudaStream_t s, cudaStream_t cs, int rank) {
        if (!on) return;
        cudaStreamSynchronize(s); cudaStreamSynchronize(cs);
        if (rank != 0) return;
        static const char *names[12] = {"step start", "blend bwd + colour pack done", "project bwd + row pack done", "records arrived (s)",
                                        "update part 1 done", "sums arrived (s)", "update part 2 done", "all-gather start (comm)",
                                        "all-gather end (comm)", "all-reduce start (comm)", "all-reduce end (comm)", ""};
        for (int i = 1; i < 11; i++) {
            float ms = 0.0f;
            if (e[i] && cudaEventElapsedTime(&ms, e[0], e[i]) == cudaSuccess) fprintf(stderr, "[bg dp trace] %-32s %8.3f ms\n", names[i], ms);
        }
    }
};
DpTrace g_dp_trace;
}  // namespace

extern "C" uint64_t bg_train_step_views_workspace_bytes(uint32_t n, uint32_t k, uint32_t w, uint32_t h, uint32_t local,
                                                        uint32_t world) {
    return carve_views_ws(nullptr, n, k, w, h, std::max(local, 1u), std::max(world, 1u), true).bytes;
}

extern "C" int32_t bg_train_step_views(BgContext *c, BgDpComm *h, void *stream, BgTrainViewsArgs *a) {
    if (!c || !a) return BG_ERR_NULL;
    if (!a->transforms || !a->sh || !a->raw_opac || !a->m_t || !a->v_t || !a->m_sh || !a->v_sh || !a->m_o || !a->v_o ||
        !a->refine_norm || !a->vis_weight || !a->max_screen || !a->cams || !a->gt_packed || !a->workspace || !a->loss_out)
        return BG_ERR_NULL;
    const uint32_t n = a->n, k = a->k, w = a->w, hh = a->h, local = a->local_views;
    const uint32_t world = h ? (uint32_t)h->c->world : 1u, rank = h ? (uint32_t)h->c->rank : 0u;
    const uint32_t views = local * world;
    if (local == 0 || views > DP_MAX_VIEWS) { set_err("bg_train_step_views: 1..16 views per step in total", cudaSuccess); return BG_ERR_INVALID; }
    if (a->step < 1) { set_err("bg_train_step_views: step is 1-based", cudaSuccess); return BG_ERR_INVALID; }
    if (a->channels != 3 && a->channels != 4) { set_err("bg_train_step_views: channels must be 3 or 4", cudaSuccess); return BG_ERR_INVALID; }
    if ((uintptr_t)a->workspace % 256) { set_err("bg_train_step_views: workspace must be 256-byte aligned", cudaSuccess); return BG_ERR_INVALID; }
    const int deg = sh_degree_from_k(k);
    if (deg < 0) { set_err("Invalid nr. of sh bases", cudaSuccess); return BG_ERR_INVALID; }
    for (uint32_t i = 0; i < local; i++)
        if (!a->gt_packed[i]) return BG_ERR_NULL;
    const bool fold = a->min_scale != nullptr;
    const ViewsWs ws = carve_views_ws(a->workspace, n, k, w, hh, local, world, fold);
    if (ws.bytes > a->workspace_bytes) { set_err("bg_train_step_views: workspace too small (bg_train_step_views_workspace_bytes)", cudaSuccess); return BG_ERR_CAPACITY; }
    if (a->chunks > DP_MAX_CHUNKS) { set_err("bg_train_step_views: at most 16 chunks", cudaSuccess); return BG_ERR_INVALID; }
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    const DpLayout L = dp_layout(n, local, world);
    int32_t r;
    // the 3D-filter floor folded into what the renderer sees (bwd/burn_glue.rs:260-270)
    const float *r_t = a->transforms, *r_o = a->raw_opac;
    if (fold) {
        r = bg_fold_min_scale_forward(c, stream, n, a->transforms, a->raw_opac, a->min_scale, ws.r_transforms, ws.r_opac);
        if (r != BG_OK) return r;
        r_t = ws.r_transforms; r_o = ws.r_opac;
    }
    const float npx = (float)w * (float)hh;
    float chain[4] = {1.0f / (3.0f * npx), 1.0f / (3.0f * npx), 1.0f / (3.0f * npx), a->channels == 4 ? a->alpha_weight / npx : 0.0f};
    BG_CUDA(cudaMemsetAsync(ws.v_output, 0, (size_t)w * hh * 4 * sizeof(float), s));
    DpHeader hdr;
    memset(&hdr, 0, sizeof(hdr));
    for (uint32_t i = 0; i < local; i++)
        for (int q = 0; q < 3; q++) hdr.pos[i][q] = a->cams[i].cam_pos[q];
    BG_CUDA(launch_write_header(s, ws.hdr, hdr, local));
    DpComm *d = world > 1 ? h->c : nullptr;
    DpTrace &tr = g_dp_trace;
    if (d) tr.mark(0, s);
    // The exchange of a step has two parts.  The colour records (all-gather) depend on the blend backward only, so they
    // leave as soon as the last local view's blend backward is done and travel UNDER its projection backward; the summed
    // small rows and the MAX statistics (all-reduces) follow once that is done.  The update pass is split the same way:
    // the SH part (70 % of its traffic) needs the records only and runs under the all-reduces, the rest follows them.
    for (uint32_t i = 0; i < local; i++) {
        const BgCamera *cam = a->cams + i;
        r = bg_render_forward(c, stream, cam, w, hh, n, k, r_t, a->sh, r_o, a->mip, a->background, BG_PASS_BACKWARD, ws.out_img, ws.visible,
                              ws.max_radius, &a->state_out);
        if (r != BG_OK) return r;
        r = bg_image_loss_fused(c, stream, ws.out_img, a->gt_packed[i], a->channels, hh, w, 1, (int64_t)w * 4, 4, a->l1_weight,
                                a->ssim_weight, a->has_composite_bg ? a->composite_bg : nullptr, a->mask, chain, ws.v_output, ws.partials);
        if (r != BG_OK) return r;
        BG_CUDA(launch_loss_reduce(s, ws.partials, a->channels, bg_image_loss_num_partials(a->channels, hh, w) / a->channels, chain,
                                   ws.loss_terms + i));
        r = bg_rasterize_backward(c, stream, &a->state_out, ws.out_img, ws.v_output, a->background, 0, ws.v_combined, n);
        if (r != BG_OK) return r;
        BG_CUDA(launch_pack_color(s, n, local, i, a->state_out.compact_from_global_gid, ws.v_combined, ws.record));
        if (d && i + 1 == local) {
            BG_CUDA(cudaEventRecord(d->ev_ready, s));
            BG_CUDA(cudaStreamWaitEvent(d->stream, d->ev_ready, 0));
            tr.mark(1, s); tr.mark(7, d->stream);
            int rc = dp_exchange_header(d, local, ws.hdr, ws.hdr_all);
            if (rc == 0) rc = dp_exchange_gather(d, n, local, ws.record, ws.recv);
            if (rc != 0) return nccl_fail("bg_train_step_views: exchange (records)", rc);
            tr.mark(8, d->stream);
        }
        r = bg_project_backward_factored(c, stream, cam, &a->state_out, r_t, a->sh, r_o, ws.v_combined, ws.v_t, ws.v_color, ws.v_o, ws.v_refine);
        if (r != BG_OK) return r;
        // fold the view into the exchange rows (sum of the small gradients, MAX statistics)
        BG_CUDA(launch_pack_view(s, n, local, i, i == 0, ws.v_t, ws.v_o, nullptr, ws.v_refine, ws.visible, ws.max_radius, ws.small, ws.stat,
                                 ws.record));
    }
    BG_CUDA(launch_loss_mean(s, ws.loss_terms, local, a->loss_out));
    UpdateParams P;
    memset(&P, 0, sizeof(P));
    P.transforms = a->transforms; P.sh = a->sh; P.raw_opac = a->raw_opac;
    P.m_t = a->m_t; P.v_t = a->v_t; P.m_sh = a->m_sh; P.v_sh = a->v_sh; P.m_o = a->m_o; P.v_o = a->v_o;
    P.refine_norm = a->refine_norm; P.vis_weight = a->vis_weight; P.max_screen = a->max_screen;
    P.small = ws.small; P.stat = ws.stat;
    P.grad_scale = 1.0f / (float)views; P.sh_grad_scale = 1.0f / (float)views;
    P.views = views; P.local = local; P.world = world;
    P.g_begin = 0; P.count = n;
    fill_update_consts(P, a->lr_mean, a->lr_rotation, a->lr_scale, a->lr_coeffs_dc, a->lr_coeffs_sh_scale, a->lr_opac, a->noise_scale,
                       a->median_scale, a->seed, a->step, n);
    auto fold_back = [&]() -> int32_t {   // chain the gradients w.r.t. the folded values back to the learned ones (linear: after the sum)
        if (fold)
            BG_CUDA(launch_fold_min_scale_bwd_strided(s, n, a->transforms, a->raw_opac, a->min_scale, ws.small, ws.small + 10, DP_SMALL_ROW,
                                                      DP_SMALL_ROW));
        return BG_OK;
    };
    if (world == 1) {
        P.records = ws.record; P.cam_all = ws.hdr;
        if ((r = fold_back()) != BG_OK) return r;
        BG_CUDA(launch_train_update(s, deg, P, true, 0));
        return BG_OK;
    }
    BG_CUDA(cudaEventRecord(d->ev_ready2, s));
    BG_CUDA(cudaStreamWaitEvent(d->stream, d->ev_ready2, 0));
    tr.mark(2, s); tr.mark(9, d->stream);
    const int rc = dp_exchange_reduce(d, n, ws.small, ws.stat);
    if (rc != 0) return nccl_fail("bg_train_step_views: exchange (sums)", rc);
    tr.mark(10, d->stream);
    P.records = ws.recv; P.cam_all = ws.hdr_all;
    BG_CUDA(cudaStreamWaitEvent(s, d->ev_chunk[0], 0));
    tr.mark(3, s);
    BG_CUDA(launch_train_update(s, deg, P, true, 1));          // SH coefficients: records only
    tr.mark(4, s);
    BG_CUDA(cudaStreamWaitEvent(s, d->ev_chunk[1], 0));
    tr.mark(5, s);
    if ((r = fold_back()) != BG_OK) return r;
    BG_CUDA(launch_train_update(s, deg, P, true, 2));          // transforms, opacity, statistics, noise
    tr.mark(6, s);
    tr.report(s, d->stream, d->rank);
    return BG_OK;
}

// ---- refine (refine.cu): every decision on the device, one readback of the counts at the end
namespace {
struct RefineWs {
    uint32_t *ctl, *keep, *keep_incl, *keys, *vals, *keys_s, *vals_s, *split, *cand, *cand_incl, *split_incl;
    float *refine_norm, *vis_weight, *max_screen, *bounds_out;
    uint64_t bytes;
};
RefineWs carve_refine_ws(void *base, uint32_t n) {
    uint64_t off = 0;
    auto take = [&](uint64_t words) {
        uint32_t *p = base ? reinterpret_cast<uint32_t *>(static_cast<char *>(base) + off) : nullptr;
        off += (words * 4 + 255) / 256 * 256;
        return p;
    };
    RefineWs w;
    w.ctl = take(64);
    w.keep = take(n); w.keep_incl = take(n); w.keys = take(n); w.vals = take(n); w.keys_s = take(n); w.vals_s = take(n);
    w.split = take(n); w.cand = take(n); w.cand_incl = take(n); w.split_incl = take(n);
    w.refine_norm = reinterpret_cast<float *>(take(n)); w.vis_weight = reinterpret_cast<float *>(take(n));
    w.max_screen = reinterpret_cast<float *>(take(n));
    w.bounds_out = reinterpret_cast<float *>(take(16));
    w.bytes = off;
    return w;
}
}  // namespace

extern "C" uint64_t bg_refine_workspace_bytes(uint32_t n) { return carve_refine_ws(nullptr, std::max(n, 1u)).bytes; }

extern "C" int32_t bg_refine(BgContext *c, void *stream, const BgRefineArgs *a, BgRefineStats *out) {
    if (!c || !a || !out) return BG_ERR_NULL;
    memset(out, 0, sizeof(*out));
    const uint32_t n0 = a->n;
    if (n0 == 0) return BG_OK;
    if (!a->transforms || !a->sh || !a->raw_opac || !a->m_t || !a->v_t || !a->m_sh || !a->v_sh || !a->m_o || !a->v_o ||
        !a->refine_norm || !a->vis_weight || !a->max_screen || !a->transforms_out || !a->sh_out || !a->raw_opac_out ||
        !a->m_t_out || !a->v_t_out || !a->m_sh_out || !a->v_sh_out || !a->m_o_out || !a->v_o_out || !a->workspace)
        return BG_ERR_NULL;
    if (sh_degree_from_k(a->k) < 0) { set_err("Invalid nr. of sh bases", cudaSuccess); return BG_ERR_INVALID; }
    if (a->capacity < n0) { set_err("bg_refine: capacity smaller than n", cudaSuccess); return BG_ERR_CAPACITY; }
    if ((uintptr_t)a->workspace % 256) { set_err("bg_refine: workspace must be 256-byte aligned", cudaSuccess); return BG_ERR_INVALID; }
    const RefineWs w = carve_refine_ws(a->workspace, n0);
    if (w.bytes > a->workspace_bytes) { set_err("bg_refine: workspace too small (bg_refine_workspace_bytes)", cudaSuccess); return BG_ERR_CAPACITY; }
    if (n0 > std::max(c->max_n, c->max_isect)) { set_err("bg_refine: n exceeds the context's sort capacity", cudaSuccess); return BG_ERR_CAPACITY; }
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    const uint32_t kf = a->k * 3;
    RefinePtrs p;
    p.transforms = a->transforms; p.sh = a->sh; p.raw_opac = a->raw_opac; p.m_t = a->m_t; p.v_t = a->v_t; p.m_sh = a->m_sh;
    p.v_sh = a->v_sh; p.m_o = a->m_o; p.v_o = a->v_o; p.refine_norm = a->refine_norm; p.vis_weight = a->vis_weight; p.max_screen = a->max_screen;
    p.transforms_out = a->transforms_out; p.sh_out = a->sh_out; p.raw_opac_out = a->raw_opac_out; p.m_t_out = a->m_t_out;
    p.v_t_out = a->v_t_out; p.m_sh_out = a->m_sh_out; p.v_sh_out = a->v_sh_out; p.m_o_out = a->m_o_out; p.v_o_out = a->v_o_out;
    p.refine_norm_tmp = w.refine_norm; p.vis_weight_tmp = w.vis_weight; p.max_screen_tmp = w.max_screen;
    int32_t r;
    BG_CUDA(cudaMemsetAsync(w.ctl, 0, 64 * sizeof(uint32_t), s));
    BG_CUDA(cudaMemsetAsync(w.split, 0, (size_t)n0 * sizeof(uint32_t), s));
    // prune mask -> flag scan -> compaction of all rows (train.rs:487-535, 848-893)
    BG_CUDA(launch_refine_classify(s, n0, kf, a->transforms, a->sh, a->raw_opac, a->bounds_center, a->max_allowed, w.keep, w.ctl));
    if ((r = bg_inclusive_scan_u32(c, stream, w.keep, n0, w.keep_incl)) != BG_OK) return r;
    BG_CUDA(launch_refine_plan_prune(s, n0, w.keep_incl, w.ctl));
    BG_CUDA(launch_refine_compact(s, n0, kf, p, w.keep, w.keep_incl, w.ctl));
    const uint64_t stream_base = (uint64_t)a->refine_index * 2;
    // replace the pruned splats: sample `pruned` survivors by opacity x visibility (train.rs:544-556)
    BG_CUDA(launch_refine_keys(s, n0, 0, p, 0.0f, a->seed, stream_base, w.keys, w.vals, w.ctl));
    if ((r = bg_radix_argsort_u32(c, stream, w.keys, w.vals, n0, w.ctl + RC_N, 32, w.keys_s, w.vals_s)) != BG_OK) return r;
    BG_CUDA(launch_refine_mark_topk(s, n0, w.vals_s, RC_PRUNED, RC_POS0, RC_SPLIT_REPLACE, w.split, w.ctl));
    // force-split what is too big on screen, in index order, within the max_splats budget (train.rs:562-586)
    BG_CUDA(launch_refine_oversize_flags(s, n0, a->split_at_screen_size, p, w.split, w.cand, w.ctl));
    if ((r = bg_inclusive_scan_u32(c, stream, w.cand, n0, w.cand_incl)) != BG_OK) return r;
    BG_CUDA(launch_refine_oversize_mark(s, n0, a->max_splats, w.cand, w.cand_incl, w.split, w.ctl));
    // growth: sample among the splats whose refine weight is above the threshold (train.rs:590-632)
    BG_CUDA(launch_refine_keys(s, n0, 1, p, a->growth_grad_threshold, a->seed, stream_base + 1, w.keys, w.vals, w.ctl));
    BG_CUDA(launch_refine_plan_growth(s, a->growth_select_fraction, a->max_splats, a->growth_enabled != 0, w.ctl));
    if ((r = bg_radix_argsort_u32(c, stream, w.keys, w.vals, n0, w.ctl + RC_N, 32, w.keys_s, w.vals_s)) != BG_OK) return r;
    BG_CUDA(launch_refine_mark_topk(s, n0, w.vals_s, RC_GROW, RC_POS1, RC_SPLIT_GROWTH, w.split, w.ctl));
    // split (refine_splats, train.rs:665-821) and opacity decay (:808-816)
    if ((r = bg_inclusive_scan_u32(c, stream, w.split, n0, w.split_incl)) != BG_OK) return r;
    BG_CUDA(launch_refine_plan_split(s, n0, w.split_incl, a->capacity, w.ctl));
    BG_CUDA(launch_refine_split(s, n0, kf, a->capacity, a->split_at_screen_size, p, w.split, w.split_incl, w.ctl));
    BG_CUDA(launch_refine_decay(s, a->capacity, a->opac_decay_minus, a->raw_opac_out, w.ctl));
    uint32_t host[RC_WORDS];
    BG_CUDA(cudaMemcpyAsync(host, w.ctl, sizeof(host), cudaMemcpyDeviceToHost, s));
    BG_CUDA(cudaStreamSynchronize(s));
    out->num_added = host[RC_REFINE_COUNT];
    out->num_split_oversized = host[RC_SPLIT_OVERSIZED];
    out->num_split_high_grad = host[RC_SPLIT_GROWTH];
    out->num_pruned = host[RC_PRUNED];
    out->num_pruned_non_finite = host[RC_NON_FINITE];
    out->total_splats = host[RC_N_NEW];
    if (host[RC_OVERFLOW]) { set_err("bg_refine: capacity of the destination arrays exceeded", cudaSuccess); return BG_ERR_CAPACITY; }
    return BG_OK;
}

extern "C" int32_t bg_bounds_percentile(BgContext *c, void *stream, uint32_t n, const float *transforms, float percentile,
                                        void *workspace, uint64_t workspace_bytes, float *out6) {
    if (!c || !out6) return BG_ERR_NULL;
    for (int i = 0; i < 6; i++) out6[i] = 0.0f;
    if (n == 0) return BG_OK;
    if (!transforms || !workspace) return BG_ERR_NULL;
    const RefineWs w = carve_refine_ws(workspace, n);
    if (w.bytes > workspace_bytes) { set_err("bg_bounds_percentile: workspace too small (bg_refine_workspace_bytes)", cudaSuccess); return BG_ERR_CAPACITY; }
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(cudaMemsetAsync(w.ctl, 0, 64 * sizeof(uint32_t), s));
    for (int axis = 0; axis < 3; axis++) {
        BG_CUDA(launch_bounds_keys(s, n, axis, transforms, w.keys, w.vals, w.ctl + axis));
        int32_t r = bg_radix_argsort_u32(c, stream, w.keys, w.vals, n, nullptr, 32, w.keys_s, w.vals_s);
        if (r != BG_OK) return r;
        BG_CUDA(launch_bounds_pick(s, w.keys_s, w.ctl + axis, percentile, w.bounds_out + 2 * axis));
    }
    BG_CUDA(cudaMemcpyAsync(out6, w.bounds_out, 6 * sizeof(float), cudaMemcpyDeviceToHost, s));
    BG_CUDA(cudaStreamSynchronize(s));
    return BG_OK;
}

// ---- LOD baking (lod.cu): PUP sensitivity scores and score-ordered decimation
extern "C" int32_t bg_pup_accumulate(BgContext *c, void *stream, uint32_t n, const float *v_transforms, int32_t first,
                                     float *fisher) {
    if (!c) return BG_ERR_NULL;
    if (n == 0) return BG_OK;
    if (!v_transforms || !fisher) return BG_ERR_NULL;
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_pup_accumulate((cudaStream_t)stream, n, v_transforms, first != 0, fisher));
    return BG_OK;
}

extern "C" int32_t bg_pup_log_det(BgContext *c, void *stream, uint32_t n, const float *fisher, float *scores) {
    if (!c) return BG_ERR_NULL;
    if (n == 0) return BG_OK;
    if (!fisher || !scores) return BG_ERR_NULL;
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_pup_log_det((cudaStream_t)stream, n, fisher, scores));
    return BG_OK;
}

namespace {
struct DecimateWs {
    uint32_t *keys, *vals, *keys_s, *vals_s;
    uint64_t bytes;
};
DecimateWs carve_decimate_ws(void *base, uint32_t n) {
    uint64_t off = 0;
    auto take = [&](uint64_t words) {
        uint32_t *p = base ? reinterpret_cast<uint32_t *>(static_cast<char *>(base) + off) : nullptr;
        off += (words * 4 + 255) / 256 * 256;
        return p;
    };
    DecimateWs w;
    w.keys = take(n); w.vals = take(n); w.keys_s = take(n); w.vals_s = take(n);
    w.bytes = off;
    return w;
}
}  // namespace

extern "C" uint64_t bg_decimate_workspace_bytes(uint32_t n) { return carve_decimate_ws(nullptr, std::max(n, 1u)).bytes; }

extern "C" int32_t bg_decimate_to_count(BgContext *c, void *stream, const BgDecimateArgs *a) {
    if (!c || !a) return BG_ERR_NULL;
    const uint32_t n = a->n, target = a->target;
    if (target == 0 || target >= n) return BG_OK;   // lod.rs:15-17: the input is returned unchanged
    if (!a->scores || !a->transforms || !a->sh || !a->raw_opac || !a->transforms_out || !a->sh_out || !a->raw_opac_out ||
        !a->workspace || (a->min_scale && !a->min_scale_out))
        return BG_ERR_NULL;
    if (sh_degree_from_k(a->k) < 0) { set_err("Invalid nr. of sh bases", cudaSuccess); return BG_ERR_INVALID; }
    const void *ptrs[] = {a->transforms, a->sh, a->raw_opac, a->min_scale, a->transforms_out, a->sh_out, a->raw_opac_out,
                          a->min_scale_out, a->workspace};
    for (const void *p : ptrs)
        if ((uintptr_t)p % 16) { set_err("bg_decimate_to_count: arrays must be 16-byte aligned", cudaSuccess); return BG_ERR_INVALID; }
    if ((uintptr_t)a->workspace % 256) { set_err("bg_decimate_to_count: workspace must be 256-byte aligned", cudaSuccess); return BG_ERR_INVALID; }
    const DecimateWs w = carve_decimate_ws(a->workspace, n);
    if (w.bytes > a->workspace_bytes) { set_err("bg_decimate_to_count: workspace too small (bg_decimate_workspace_bytes)", cudaSuccess); return BG_ERR_CAPACITY; }
    if (n > std::max(c->max_n, c->max_isect)) { set_err("bg_decimate_to_count: n exceeds the context's sort capacity", cudaSuccess); return BG_ERR_CAPACITY; }
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_decimate_keys(s, n, a->scores, w.keys, w.vals));
    int32_t r = bg_radix_argsort_u32(c, stream, w.keys, w.vals, n, nullptr, 32, w.keys_s, w.vals_s);
    if (r != BG_OK) return r;
    BG_CUDA(launch_decimate_gather(s, target, a->k * 3, w.vals_s, a->transforms, a->sh, a->raw_opac, a->min_scale,
                                   a->transforms_out, a->sh_out, a->raw_opac_out, a->min_scale_out));
    if (a->kept_ids_out) BG_CUDA(cudaMemcpyAsync(a->kept_ids_out, w.vals_s, (size_t)target * 4, cudaMemcpyDeviceToDevice, s));
    return BG_OK;
}
