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

#include "bg_adam.cuh"
#include "bg_common.cuh"
#include "bg_project.cuh"
#include "bg_dp.cuh"
#include "bg_update.cuh"
#include "bg_refine.cuh"
#include "bg_launch.cuh"

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

// ---- argument checks shared by the entry points.  Each returns BG_OK or the status, with the error text set.
// The text is "who: what", or "who what" when `what` opens with a space.
static int32_t fail(int32_t status, const char *who, const char *what) {
    char m[480];
    snprintf(m, sizeof(m), what[0] == ' ' ? "%s%s" : "%s: %s", who, what);
    set_err(m, cudaSuccess);
    return status;
}
static int32_t invalid(const char *who, const char *what) { return fail(BG_ERR_INVALID, who, what); }
static int32_t capacity(const char *who, const char *what) { return fail(BG_ERR_CAPACITY, who, what); }

// k SH coefficients per channel must be (deg + 1)^2 with deg <= 4; *deg gets the degree
static int32_t check_k(uint32_t k, int *deg = nullptr) {
    const int d = sh_degree_from_k(k);
    if (deg) *deg = d;
    if (d < 0) set_err("Invalid nr. of sh bases", cudaSuccess);
    return d < 0 ? BG_ERR_INVALID : BG_OK;
}

// A caller-provided workspace: non-null and 256-byte aligned (what Carver's blocks assume), and at least `need` bytes,
// the figure that the function named `sizer` reports.  In two parts for the entry points that check other arguments
// in between.
static int32_t check_workspace_aligned(const char *who, const void *ws) {
    if (!ws) return BG_ERR_NULL;
    if ((uintptr_t)ws % 256) return invalid(who, "workspace must be 256-byte aligned");
    return BG_OK;
}
static int32_t check_workspace_bytes(const char *who, const char *sizer, uint64_t have, uint64_t need) {
    if (need <= have) return BG_OK;
    char what[96];
    snprintf(what, sizeof(what), "workspace too small (%s)", sizer);
    return capacity(who, what);
}
static int32_t check_workspace(const char *who, const char *sizer, const void *ws, uint64_t have, uint64_t need) {
    if (int32_t r = check_workspace_aligned(who, ws); r != BG_OK) return r;
    return check_workspace_bytes(who, sizer, have, need);
}

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
    float *row_by_gid = nullptr;  // [N,16] projected rows by global id + tile hit bits (project_cull -> emit)
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

// The most keys the context's radix sort takes: its scratch is the larger of the depth and intersection ping-pong buffers.
static uint32_t sort_capacity(const BgContext *c) { return std::max(c->max_n, c->max_isect); }

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
                    c->cgid_from_gid, c->row_by_gid, c->projected, c->isect_key[0], c->isect_key[1], c->isect_val[0], c->isect_val[1],
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
    if (max_splats == 0 || max_w == 0 || max_h == 0) return invalid("bg_ctx_create", "zero capacity");
    if (max_intersections == 0) max_intersections = std::max<uint64_t>(16ull * max_splats, 1ull << 22);
    if (max_intersections >= (1ull << 31)) return invalid("bg_ctx_create", "max_intersections must be < 2^31");
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
    ok = ok && arena_alloc(c, &c->row_by_gid, n * BG_PROJECTED_STRIDE) == cudaSuccess;
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
    int deg;
    if (int32_t r = check_k(k, &deg); r != BG_OK) return r;
    if (pass < 0 || pass > 2) { set_err("invalid pass", cudaSuccess); return BG_ERR_INVALID; }
    if (cam->camera_model > BG_CAMERA_THIN_PRISM_FISHEYE) return BG_ERR_UNSUPPORTED;
    const bool bwd_info = pass != BG_PASS_FORWARD;
    if (bwd_info && n > 0 && !visible) return BG_ERR_NULL;
    if ((((uintptr_t)transforms) | ((uintptr_t)sh) | ((uintptr_t)raw_opac) | ((uintptr_t)out_img)) & 15u)
        return invalid("bg_render_forward", "arrays must be 16-byte aligned (bulk / 128-bit access)");
    const uint32_t tiles_x = (w + TILE_W - 1) / TILE_W, tiles_y = (h + TILE_W - 1) / TILE_W;
    const uint32_t num_tiles = tiles_x * tiles_y;
    if (n > c->max_n || num_tiles > c->max_tiles) return capacity("bg_render_forward", "exceeds context capacity");
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    c->depth_forward = out_depth != nullptr;

    BG_CUDA(launch_bump_epoch(s, c->epoch_dev));
    BG_CUDA(cudaMemsetAsync(c->ctl, 0, CTL_WORDS * sizeof(uint32_t), s));
    BG_CUDA(cudaMemsetAsync(c->tile_offsets, 0, (size_t)num_tiles * 2 * sizeof(uint32_t), s));
    if (bwd_info && n > 0) BG_CUDA(cudaMemsetAsync(visible, 0, (size_t)n * sizeof(float), s));

    const int pgrid = c->sm_count * 5;   // project_cull: 256-thread CTAs, 48 regs
    const int vgrid = c->sm_count * 8;   // project_visible_emit: 128-thread CTAs, __launch_bounds__(128, 8) (project.cu)
    uint32_t *counters = c->ctl + CTL_COUNTERS;
    // K1: cull + compaction in index order; finished projected rows (colour included) staged by global id
    BG_CUDA(launch_project_cull(s, pgrid, mip != 0, deg, transforms, sh, raw_opac, n, *cam, w, h, tiles_x, tiles_y,
                                c->depth_key[0], c->depth_val[0], c->counts, max_radius, c->cgid_from_gid, c->row_by_gid,
                                c->ctl, c->lb_scan, c->epoch_dev, EP_PROJECT));
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
        BG_CUDA(launch_project_visible_emit(s, vgrid, c->row_by_gid, gid_sorted, c->cum, tiles_x, tiles_y, c->projected,
                                            c->isect_key[0], c->isect_val[0], c->max_isect, c->cgid_from_gid, c->ctl,
                                            bits));
    int iout = 0;
    {
        int32_t r = run_sort(c, s, c->isect_key[0], c->isect_val[0], c->isect_key, c->isect_val, c->max_isect,
                             counters + 1, bits, c->ctl + CTL_HIST_TILE, c->ctl + CTL_TICKETS + TK_TILE_HIST, 1,
                             EP_TILE_SORT, &iout, /*hist_ready=*/n > 0 && bits <= 16);
        if (r != BG_OK) return r;
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
    if (pass != BG_PASS_BACKWARD && pass != BG_PASS_BACKWARD_SMOOTH)
        return invalid("bg_render_forward_depth", "depth needs an f32 pass (BG_PASS_BACKWARD or BG_PASS_BACKWARD_SMOOTH)");
    if ((uintptr_t)out_depth % 4) return invalid("bg_render_forward_depth", "out_depth must be 4-byte aligned");
    return render_forward(c, stream, cam, w, h, n, k, transforms, sh, raw_opac, mip, bg, pass, out_img, out_depth, visible,
                          max_radius, st);
}

// depth: out_depth / v_depth / v_z all set (bg_rasterize_backward_depth) or all null
static int32_t rasterize_backward(BgContext *c, void *stream, const BgRenderState *st, const float *out_img,
                                  const float *out_depth, const float *v_output, const float *v_depth, const float *bg,
                                  int32_t smooth, float *v_combined, uint32_t rows, float *v_z, const char *who) {
    if (st->pass == BG_PASS_FORWARD) return invalid(who, " requires a Backward pass state");
    const bool smooth_pass = st->pass == BG_PASS_BACKWARD_SMOOTH;
    if ((smooth != 0) != smooth_pass) return invalid(who, "smooth_cutoff must match the state's pass");
    if (st->tile_offsets != c->tile_offsets) return invalid(who, "needs the state of this context's last forward");
    if (v_z && !c->depth_forward) return invalid(who, "this context's last forward did not render depth");
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
    if (((uintptr_t)out_depth | (uintptr_t)v_depth | (uintptr_t)v_z) % 4)
        return invalid("bg_rasterize_backward_depth", "out_depth, v_depth and v_z must be 4-byte aligned");
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
    if (st->pass != BG_PASS_BACKWARD || st->tile_offsets != c->tile_offsets) return invalid("bg_debug_blend_stats", "needs the state of this context's last Backward pass");
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
    int deg;
    if (int32_t r = check_k(st->k, &deg); r != BG_OK) return r;
    if (cam->camera_model > BG_CAMERA_THIN_PRISM_FISHEYE) return BG_ERR_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    if (((uintptr_t)sh | (uintptr_t)v_sh) % 16)
        return invalid("bg_project_backward", "sh and v_sh must be 16-byte aligned (128-bit row access)");
    BG_CUDA(launch_project_bwd(s, st->mip != 0, deg, transforms, sh, raw_opac, st->compact_from_global_gid, v_combined,
                               st->n, *cam, v_transforms, v_sh, v_raw_opac, v_refine, nullptr));
    return BG_OK;
}

extern "C" int32_t bg_project_backward_depth(BgContext *c, void *stream, const BgCamera *cam, const BgRenderState *st,
                                             const float *transforms, const float *sh, const float *raw_opac,
                                             const float *v_combined, const float *v_z, float *v_transforms, float *v_sh,
                                             float *v_raw_opac, float *v_refine) {
    if (!v_z) return BG_ERR_NULL;
    if ((uintptr_t)v_z % 4) return invalid("bg_project_backward_depth", "v_z must be 4-byte aligned");
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
    int deg;
    if (int32_t r = check_k(st->k, &deg); r != BG_OK) return r;
    if (cam->camera_model > BG_CAMERA_THIN_PRISM_FISHEYE) return BG_ERR_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    if ((uintptr_t)sh % 16)
        return invalid("bg_project_backward_factored", "sh must be 16-byte aligned (128-bit row access)");
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
    if (deg < 0 || views == 0 || views > 16) return invalid("bg_sh_grad_from_views", "k must be a square <= 25, 1 <= views <= 16");
    BG_CUDA(cudaSetDevice(c->device));
    if (view_stride != 0 && view_stride < (uint64_t)n * 3) return invalid("bg_sh_grad_from_views", "view_stride smaller than one view");
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
    if (n > sort_capacity(c)) return capacity("bg_radix_argsort_u32", "n exceeds context capacity");
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
    if ((uint64_t)(n + 2047) / 2048 > c->lb_scan_words) return capacity("bg_inclusive_scan_u32", "n exceeds context capacity");
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
    if (h == 0 || w == 0) return invalid("bg_depth_loss_fused", "empty image");
    if (!(chain >= 0.0f) || !std::isfinite(chain)) return invalid("bg_depth_loss_fused", "chain must be finite and >= 0");
    if ((((uintptr_t)out_img) | ((uintptr_t)v_output)) & 15u)
        return invalid("bg_depth_loss_fused", "out_img and v_output must be 16-byte aligned (128-bit pixel access)");
    if ((((uintptr_t)depth) | ((uintptr_t)target) | ((uintptr_t)v_depth) | ((uintptr_t)partials)) & 3u)
        return invalid("bg_depth_loss_fused", "depth, target, v_depth and partials must be 4-byte aligned");
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_depth_loss_fused((cudaStream_t)stream, out_img, depth, target, h, w, chain, v_output, v_depth, partials));
    return BG_OK;
}

extern "C" int32_t bg_adam_step(BgContext *c, void *stream, float *p, const float *g, float *m, float *v,
                                uint64_t rows, uint32_t cols, const float *lr_scale, float lr, float beta1, float beta2,
                                float eps, int32_t t, int32_t reduce_v) {
    if (!c) return BG_ERR_NULL;
    if (rows == 0 || cols == 0) return BG_OK;
    if (!p || !g || !m || !v) return BG_ERR_NULL;
    if (t < 1) return invalid("bg_adam_step", "t is 1-based");
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
    if (views == 0 || !(factor > 0.0f)) return invalid("bg_compute_min_scale", "needs views > 0 and factor > 0 (the reference returns None)");
    if ((uintptr_t)view_cams % 16) return invalid("bg_compute_min_scale", "view_cams must be 16-byte aligned");
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

// The update pass over all n Gaussians of `a` (BgTrainUpdateArgs, BgTrainStepArgs or BgTrainViewsArgs, which name the
// trainable state and the schedule alike): the state pointers and the step-dependent constants, unit gradient scales.
// The caller sets the gradient sources.  compiler-rt __powisf2 is powi_f32 (bg_adam.cuh).
template <class A>
static UpdateParams update_params(const A *a) {
    UpdateParams P;
    memset(&P, 0, sizeof(P));
    P.g_begin = 0; P.count = a->n;
    P.transforms = a->transforms; P.sh = a->sh; P.raw_opac = a->raw_opac;
    P.m_t = a->m_t; P.v_t = a->v_t; P.m_sh = a->m_sh; P.v_sh = a->v_sh; P.m_o = a->m_o; P.v_o = a->v_o;
    P.refine_norm = a->refine_norm; P.vis_weight = a->vis_weight; P.max_screen = a->max_screen;
    P.grad_scale = 1.0f; P.sh_grad_scale = 1.0f;
    for (int i = 0; i < 10; i++) P.lr_t[i] = i < 3 ? a->lr_mean : (i < 7 ? a->lr_rotation : a->lr_scale);   // train.rs:328-350
    P.lr_sh_dc = 1.0f * a->lr_coeffs_dc;                                // lr_scale_per_col * lr, as AdamScaled forms it
    P.lr_sh_rest = (1.0f / a->lr_coeffs_sh_scale) * a->lr_coeffs_dc;
    P.lr_opac = a->lr_opac;
    P.beta1 = 0.9f; P.beta2 = 0.999f; P.eps = 1e-15f; P.f1 = 1.0f - P.beta1; P.f2 = 1.0f - P.beta2;
    P.inv_bc1 = 1.0f / (1.0f - powi_f32(P.beta1, a->step)); P.inv_bc2 = 1.0f / (1.0f - powi_f32(P.beta2, a->step));
    P.first = a->step == 1;
    P.noisy = a->noise_scale != 0.0f;
    P.noise_scale = a->noise_scale; P.median_scale = a->median_scale;
    P.seed = a->seed;
    P.noise_offset = (unsigned long long)(a->step - 1) * (((unsigned long long)a->n * 3 + 3) / 4);
    return P;
}

// The update pass reads the transforms rows and their moments as float2 and the SH spans as float4.
template <class A>
static bool update_aligned(const A *a) {
    return (uintptr_t)a->transforms % 8 == 0 && (uintptr_t)a->m_t % 8 == 0 && (uintptr_t)a->v_t % 8 == 0 &&
           (uintptr_t)a->sh % 16 == 0 && (uintptr_t)a->m_sh % 16 == 0;
}

extern "C" int32_t bg_train_update(BgContext *c, void *stream, const BgTrainUpdateArgs *a) {
    if (!c || !a) return BG_ERR_NULL;
    if (a->n == 0) return BG_OK;
    if (!a->transforms || !a->sh || !a->raw_opac || !a->m_t || !a->v_t || !a->m_sh || !a->v_sh || !a->m_o || !a->v_o ||
        !a->refine_norm || !a->vis_weight || !a->max_screen || !a->v_transforms || !a->v_sh_grad || !a->v_raw_opac ||
        !a->v_refine || !a->visible || !a->max_radius)
        return BG_ERR_NULL;
    int deg;
    if (int32_t r = check_k(a->k, &deg); r != BG_OK) return r;
    if (a->step < 1) return invalid("bg_train_update", "step is 1-based");
    if (!update_aligned(a) || (uintptr_t)a->v_transforms % 8 || (uintptr_t)a->v_sh_grad % 16)
        return invalid("bg_train_update", "transforms, m_t, v_t and v_transforms must be 8-byte aligned, sh, m_sh and v_sh_grad "
                                          "16-byte aligned (64- and 128-bit row access)");
    BG_CUDA(cudaSetDevice(c->device));
    UpdateParams P = update_params(a);
    P.g_t = a->v_transforms; P.g_o = a->v_raw_opac; P.g_sh = a->v_sh_grad;
    P.v_refine = a->v_refine; P.max_radius = a->max_radius; P.visible = a->visible;
    P.min_scale = a->min_scale;
    BG_CUDA(launch_train_update((cudaStream_t)stream, deg, P, false));
    return BG_OK;
}

// ---- bg_train_step: SplatTrainer::step (brush-train/src/train.rs:176-429) as ONE call: every launch of the step on
// the caller's stream, nothing read back, scratch from a caller-provided workspace.
namespace {
// Bump allocator over a workspace: take<T>(count) returns the next count elements and rounds the block up to 256 bytes.
// base == nullptr only sizes the workspace: off ends as its byte count.
struct Carver {
    void *base;
    uint64_t off = 0;
    template <class T = float>
    T *take(uint64_t count) {
        T *p = base ? reinterpret_cast<T *>(static_cast<char *>(base) + off) : nullptr;
        off += (count * sizeof(T) + 255) / 256 * 256;
        return p;
    }
};

// the input and the output pair of one bg_radix_argsort_u32 over n keys; the base of the workspaces that sort
struct SortWs {
    uint32_t *keys, *vals, *keys_s, *vals_s;
};
void carve_sort_ws(Carver &cv, uint32_t n, SortWs &w) {
    w.keys = cv.take<uint32_t>(n); w.vals = cv.take<uint32_t>(n); w.keys_s = cv.take<uint32_t>(n); w.vals_s = cv.take<uint32_t>(n);
}

struct TrainWs {
    float *out_img, *v_output, *partials, *v_combined, *v_t, *v_sh, *v_o, *v_r, *visible, *max_radius;
    uint64_t bytes;
};
TrainWs carve_train_ws(void *base, uint32_t n, uint32_t k, uint32_t w, uint32_t h, uint32_t channels) {
    Carver cv{base};
    TrainWs ws;
    const uint64_t px = (uint64_t)w * h;
    ws.out_img = cv.take(px * 4);
    ws.v_output = cv.take(px * 4);
    ws.partials = cv.take(bg_image_loss_num_partials(channels, h, w));
    ws.v_combined = cv.take((uint64_t)n * BG_VCOMBINED_STRIDE);
    ws.v_t = cv.take((uint64_t)n * 10);
    ws.v_sh = cv.take((uint64_t)n * k * 3);
    ws.v_o = cv.take(n);
    ws.v_r = cv.take(n);
    ws.visible = cv.take(n);
    ws.max_radius = cv.take(n);
    ws.bytes = cv.off;
    return ws;
}

// the depth term's scratch, from byte `off` on: behind the largest workspace of the same step without the term.  The
// multi-view step reuses it view after view.
struct DepthWs {
    float *depth, *v_depth, *v_z, *partials;
    uint64_t bytes;
};
DepthWs carve_depth_ws(void *base, uint64_t off, uint32_t n, uint32_t w, uint32_t h) {
    Carver cv{base, off};
    DepthWs ws;
    const uint64_t px = (uint64_t)w * h;
    ws.depth = cv.take(px);
    ws.v_depth = cv.take(px);
    ws.v_z = cv.take(std::max(n, 1u));
    ws.partials = cv.take(depth_loss_num_partials(h, w));
    ws.bytes = cv.off;
    return ws;
}

// argument checks shared by the single-view and the multi-view steps (BgTrainStepArgs / BgTrainViewsArgs)
template <class A>
int32_t check_train_args(const A *a, const char *who) {
    if (!a->transforms || !a->sh || !a->raw_opac || !a->m_t || !a->v_t || !a->m_sh || !a->v_sh || !a->m_o || !a->v_o ||
        !a->refine_norm || !a->vis_weight || !a->max_screen || !a->gt_packed || !a->workspace || !a->loss_out)
        return BG_ERR_NULL;
    if (a->step < 1) return invalid(who, "step is 1-based");
    if (a->channels != 3 && a->channels != 4) return invalid(who, "channels must be 3 or 4");
    if (int32_t r = check_workspace_aligned(who, a->workspace); r != BG_OK) return r;
    if (!update_aligned(a)) return invalid(who, "transforms, m_t and v_t must be 8-byte aligned, sh and m_sh 16-byte aligned");
    return BG_OK;
}

// Whether a view runs the depth term of DESIGN.md section 4.7.  After check_depth, a weight that is not 0 is > 0.
bool depth_term(const BgDepthSupervision &d) { return d.weight > 0.0f && d.valid_count > 0; }

int32_t check_depth(const BgDepthSupervision &d, const char *who) {
    if (!d.depth_loss_out) return BG_ERR_NULL;
    if (!(d.weight >= 0.0f) || !std::isfinite(d.weight)) return invalid(who, "weight must be finite and >= 0");
    if (depth_term(d) && !d.target) return BG_ERR_NULL;
    return BG_OK;
}

// The loss of one rendered view into *loss (train.rs:220-260): the mean over [h,w,3] (+ alpha mean * weight) of `img`
// (ws.out_img, or its bilateral-grid slice), value and gradient (into ws.v_output) from the fused kernel.  With d, also
// the depth term on the raw render: v_depth, v_output[...,3] += dL/da, L_d -> d->depth_loss_out and added to *loss.
template <class A, class W>
int32_t view_loss(BgContext *c, void *stream, const A *a, const uint32_t *gt, const W &ws, const float *img, float *loss,
                  const BgDepthSupervision *d, const DepthWs &dws) {
    cudaStream_t s = (cudaStream_t)stream;
    const uint32_t w = a->w, h = a->h;
    const float npx = (float)w * (float)h;
    float chain[4] = {1.0f / (3.0f * npx), 1.0f / (3.0f * npx), 1.0f / (3.0f * npx), a->channels == 4 ? a->alpha_weight / npx : 0.0f};
    int32_t r = bg_image_loss_fused(c, stream, img, gt, a->channels, h, w, 1, (int64_t)w * 4, 4, a->l1_weight, a->ssim_weight,
                                    a->has_composite_bg ? a->composite_bg : nullptr, a->mask, chain, ws.v_output, ws.partials);
    if (r != BG_OK) return r;
    BG_CUDA(launch_loss_reduce(s, ws.partials, a->channels, bg_image_loss_num_partials(a->channels, h, w) / a->channels, chain, loss));
    if (!d) return BG_OK;
    const float dchain = d->weight / (float)d->valid_count;
    r = bg_depth_loss_fused(c, stream, ws.out_img, dws.depth, d->target, h, w, dchain, ws.v_output, dws.v_depth, dws.partials);
    if (r != BG_OK) return r;
    BG_CUDA(launch_depth_loss_reduce(s, dws.partials, depth_loss_num_partials(h, w), dchain, d->depth_loss_out, loss));
    return BG_OK;
}

bool aligned16(const void *p) { return (uintptr_t)p % 16 == 0; }
// whether two [h,w,4] f32 images share any byte
bool overlap(const float *a, const float *b, uint32_t h, uint32_t w) {
    const uintptr_t n = (uintptr_t)h * w * 4 * sizeof(float), pa = (uintptr_t)a, pb = (uintptr_t)b;
    return pa < pb + n && pb < pa + n;
}

int32_t check_bilagrid_step(const BgBilagridStep *b, const char *who) {
    if (!b || !b->grid || !b->m || !b->v || !b->tv_loss_out) return BG_ERR_NULL;
    if (b->step < 1) return invalid(who, "bilateral grid step is 1-based");
    if (!(b->lr >= 0.0f) || !std::isfinite(b->lr) || !(b->tv_weight >= 0.0f) || !std::isfinite(b->tv_weight))
        return invalid(who, "bilateral grid lr and tv_weight must be finite and >= 0");
    if (!aligned16(b->grid) || !aligned16(b->m) || !aligned16(b->v)) return invalid(who, "grid, m and v must be 16-byte aligned");
    return BG_OK;
}

// TV into v_grid and *tv_loss_out (and *loss_out when not null), then Adam on the grid (DESIGN.md section 4.11)
cudaError_t bilagrid_update(cudaStream_t s, const BgBilagridStep *b, float *v_grid, float *loss_out) {
    cudaError_t e = launch_bilagrid_tv(s, b->grid, v_grid, b->tv_weight, b->tv_loss_out, loss_out);
    if (e != cudaSuccess) return e;
    const float beta1 = 0.9f, beta2 = 0.999f;
    return launch_adam(s, b->grid, v_grid, b->m, b->v, BG_BILAGRID_FLOATS / 4, 4, nullptr, b->lr, beta1, beta2, 1e-15f,
                       1.0f - powi_f32(beta1, b->step), 1.0f - powi_f32(beta2, b->step), b->step == 1, false);
}

// the bilateral grid's scratch of bg_train_step_bilagrid, behind the depth step's workspace
struct BilagridWs {
    float *sliced, *v_grid;
    uint64_t bytes;
};
BilagridWs carve_bilagrid_ws(void *base, uint64_t off, uint32_t w, uint32_t h) {
    Carver cv{base, off};
    BilagridWs ws;
    ws.sliced = cv.take((uint64_t)w * h * 4);
    ws.v_grid = cv.take(BG_BILAGRID_FLOATS);
    ws.bytes = cv.off;
    return ws;
}
}  // namespace

extern "C" uint64_t bg_train_step_workspace_bytes(uint32_t n, uint32_t k, uint32_t w, uint32_t h) {
    return carve_train_ws(nullptr, n, k, w, h, 4).bytes;
}

extern "C" uint64_t bg_train_step_depth_workspace_bytes(uint32_t n, uint32_t k, uint32_t w, uint32_t h) {
    return carve_depth_ws(nullptr, bg_train_step_workspace_bytes(n, k, w, h), n, w, h).bytes;
}

extern "C" uint64_t bg_train_step_bilagrid_workspace_bytes(uint32_t n, uint32_t k, uint32_t w, uint32_t h) {
    return carve_bilagrid_ws(nullptr, bg_train_step_depth_workspace_bytes(n, k, w, h), w, h).bytes;
}

// The single-view step.  d == nullptr: bg_train_step.  Otherwise the step with the depth term of DESIGN.md section 4.7
// (d validated, its term on, by bg_train_step_depth).  bl: the view's bilateral grid (DESIGN.md section 4.11, validated
// by bg_train_step_bilagrid) or null.
static int32_t train_step(BgContext *c, void *stream, BgTrainStepArgs *a, const BgDepthSupervision *d, const BgBilagridStep *bl) {
    const char *who = bl ? "bg_train_step_bilagrid" : d ? "bg_train_step_depth" : "bg_train_step";
    if (int32_t r = check_train_args(a, who); r != BG_OK) return r;
    const uint32_t n = a->n, k = a->k, w = a->w, h = a->h;
    const TrainWs ws = carve_train_ws(a->workspace, n, k, w, h, a->channels);
    // the depth term's buffers; all null without the term, which selects the plain render and blend backward
    const DepthWs dws = carve_depth_ws(d ? a->workspace : nullptr, bg_train_step_workspace_bytes(n, k, w, h), n, w, h);
    const BilagridWs bws = carve_bilagrid_ws(bl ? a->workspace : nullptr, bg_train_step_depth_workspace_bytes(n, k, w, h), w, h);
    if (int32_t r = check_workspace_bytes(who, bl ? "bg_train_step_bilagrid_workspace_bytes" : d ? "bg_train_step_depth_workspace_bytes"
                                                                                             : "bg_train_step_workspace_bytes",
                                          a->workspace_bytes, bl ? bws.bytes : d ? dws.bytes : ws.bytes); r != BG_OK) return r;
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    int32_t r;
    // render forward (train.rs:200-216)
    r = render_forward(c, stream, &a->cam, w, h, n, k, a->transforms, a->sh, a->raw_opac, a->mip, a->background, BG_PASS_BACKWARD,
                       ws.out_img, dws.depth, ws.visible, ws.max_radius, &a->state_out);
    if (r != BG_OK) return r;
    BG_CUDA(cudaMemsetAsync(ws.v_output, 0, (size_t)w * h * 4 * sizeof(float), s));
    if (bl) BG_CUDA(launch_bilagrid_slice(s, bl->grid, ws.out_img, w, h, bws.sliced));
    if ((r = view_loss(c, stream, a, a->gt_packed, ws, bl ? bws.sliced : ws.out_img, a->loss_out, d, dws)) != BG_OK) return r;
    // the gradient w.r.t. the sliced image back to the raw one, in place; the blend backward replays the RAW out_img
    if (bl) BG_CUDA(launch_bilagrid_slice_bwd(s, bl->grid, ws.out_img, ws.v_output, w, h, ws.v_output, bws.v_grid));
    // backward (bwd/burn_glue.rs:121-182); the depth gradient reaches the means through v_z
    r = rasterize_backward(c, stream, &a->state_out, ws.out_img, dws.depth, ws.v_output, dws.v_depth, a->background, 0, ws.v_combined,
                           n, dws.v_z, d ? "bg_rasterize_backward_depth" : "bg_rasterize_backward");
    if (r != BG_OK) return r;
    r = bg_project_backward(c, stream, &a->cam, &a->state_out, a->transforms, a->sh, a->raw_opac, ws.v_combined, ws.v_t, ws.v_sh,
                            ws.v_o, ws.v_r);
    if (r != BG_OK) return r;
    if (d) BG_CUDA(launch_depth_to_means(s, a->state_out.compact_from_global_gid, dws.v_z, a->state_out.n, a->cam, ws.v_t));
    // optimiser, refine statistics, mean noise (train.rs:280-416): one pass over the Gaussians, as bg_train_update
    if (n > 0) {
        UpdateParams P = update_params(a);
        P.g_t = ws.v_t; P.g_o = ws.v_o; P.g_sh = ws.v_sh;
        P.v_refine = ws.v_r; P.max_radius = ws.max_radius; P.visible = ws.visible;
        BG_CUDA(launch_train_update(s, sh_degree_from_k(k), P, false));
    }
    if (bl) BG_CUDA(bilagrid_update(s, bl, bws.v_grid, a->loss_out));
    return BG_OK;
}

extern "C" int32_t bg_train_step(BgContext *c, void *stream, BgTrainStepArgs *a) {
    if (!c || !a) return BG_ERR_NULL;
    return train_step(c, stream, a, nullptr, nullptr);
}

// ---- bg_train_step_depth: bg_train_step with the depth-supervision term of DESIGN.md section 4.7
extern "C" int32_t bg_train_step_depth(BgContext *c, void *stream, BgTrainStepArgs *a, const BgDepthSupervision *d) {
    if (!c || !a || !d) return BG_ERR_NULL;
    if (int32_t r = check_depth(*d, "bg_train_step_depth"); r != BG_OK) return r;
    if (!depth_term(*d)) {
        // no term (target may be null): the plain step, launch for launch, and a zero depth loss
        const int32_t r = train_step(c, stream, a, nullptr, nullptr);
        if (r != BG_OK) return r;
        BG_CUDA(cudaMemsetAsync(d->depth_loss_out, 0, sizeof(float), (cudaStream_t)stream));
        return BG_OK;
    }
    return train_step(c, stream, a, d, nullptr);
}

// ---- the bilateral grid of DESIGN.md section 4.11
extern "C" int32_t bg_bilagrid_slice(BgContext *c, void *stream, const float *grid, const float *img, uint32_t h, uint32_t w,
                                     float *out) {
    if (!c || !grid || !img || !out) return BG_ERR_NULL;
    if (!aligned16(grid) || !aligned16(img) || !aligned16(out))
        return invalid("bg_bilagrid_slice", "grid, img and out must be 16-byte aligned");
    if (h == 0 || w == 0) return BG_OK;
    if (overlap(img, out, h, w)) return invalid("bg_bilagrid_slice", "out must not overlap img");
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_bilagrid_slice((cudaStream_t)stream, grid, img, w, h, out));
    return BG_OK;
}

extern "C" int32_t bg_bilagrid_slice_backward(BgContext *c, void *stream, const float *grid, const float *img, const float *v_out,
                                              uint32_t h, uint32_t w, float *v_img, float *v_grid) {
    if (!c || !grid || !img || !v_out || !v_img || !v_grid) return BG_ERR_NULL;
    if (!aligned16(grid) || !aligned16(img) || !aligned16(v_out) || !aligned16(v_img) || !aligned16(v_grid))
        return invalid("bg_bilagrid_slice_backward", "grid, img, v_out, v_img and v_grid must be 16-byte aligned");
    if (overlap(img, v_img, h, w) || (v_img != v_out && overlap(v_out, v_img, h, w)))
        return invalid("bg_bilagrid_slice_backward", "v_img must not overlap img, and must be v_out itself or not overlap it");
    BG_CUDA(cudaSetDevice(c->device));
    if (h == 0 || w == 0) {
        BG_CUDA(cudaMemsetAsync(v_grid, 0, sizeof(float) * BG_BILAGRID_FLOATS, (cudaStream_t)stream));
        return BG_OK;
    }
    BG_CUDA(launch_bilagrid_slice_bwd((cudaStream_t)stream, grid, img, v_out, w, h, v_img, v_grid));
    return BG_OK;
}

extern "C" int32_t bg_bilagrid_update(BgContext *c, void *stream, const BgBilagridStep *b, float *v_grid) {
    if (!c || !v_grid) return BG_ERR_NULL;
    if (int32_t r = check_bilagrid_step(b, "bg_bilagrid_update"); r != BG_OK) return r;
    if (!aligned16(v_grid)) return invalid("bg_bilagrid_update", "v_grid must be 16-byte aligned");
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(bilagrid_update((cudaStream_t)stream, b, v_grid, nullptr));
    return BG_OK;
}

// ---- bg_train_step_bilagrid: the single-view step with the view's bilateral grid, with or without the depth term
extern "C" int32_t bg_train_step_bilagrid(BgContext *c, void *stream, BgTrainStepArgs *a, const BgDepthSupervision *d,
                                          const BgBilagridStep *bl) {
    if (!c || !a || !bl) return BG_ERR_NULL;
    if (int32_t r = check_bilagrid_step(bl, "bg_train_step_bilagrid"); r != BG_OK) return r;
    if (d) {
        if (int32_t r = check_depth(*d, "bg_train_step_bilagrid"); r != BG_OK) return r;
        if (!depth_term(*d)) {
            const int32_t r = train_step(c, stream, a, nullptr, bl);
            if (r != BG_OK) return r;
            BG_CUDA(cudaMemsetAsync(d->depth_loss_out, 0, sizeof(float), (cudaStream_t)stream));
            return BG_OK;
        }
    }
    return train_step(c, stream, a, d, bl);
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
    if (world < 1 || rank < 0 || rank >= world) return invalid("bg_dp_comm_create", "rank/world");
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
    if (local == 0 || local > DP_MAX_VIEWS || view >= local) return invalid("bg_dp_pack_view", "view index / views per rank");
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
    if (local == 0 || local * (uint32_t)h->c->world > DP_MAX_VIEWS || chunks == 0 || chunks > DP_MAX_CHUNKS)
        return invalid("bg_dp_exchange", "1..16 views in total, 1..16 chunks");
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
ViewsWs carve_views_ws(void *base, uint32_t n, uint32_t w, uint32_t h, uint32_t local, uint32_t world, bool fold) {
    Carver cv{base};
    ViewsWs ws;
    const uint64_t px = (uint64_t)w * h;
    const DpLayout L = dp_layout(n, local, world);
    ws.out_img = cv.take(px * 4);
    ws.v_output = cv.take(px * 4);
    ws.partials = cv.take(bg_image_loss_num_partials(4, h, w));
    ws.loss_terms = cv.take(DP_MAX_VIEWS);
    ws.v_combined = cv.take((uint64_t)n * BG_VCOMBINED_STRIDE);
    ws.small = cv.take(L.small_floats);
    ws.stat = cv.take(L.stat_floats);
    ws.record = cv.take(L.rec_floats);
    ws.recv = cv.take(world > 1 ? L.recv_floats : 0);
    ws.hdr = cv.take(DP_MAX_VIEWS * 4);
    ws.hdr_all = cv.take(DP_MAX_VIEWS * 4);
    ws.r_transforms = cv.take(fold ? (uint64_t)n * 10 : 0);
    ws.r_opac = cv.take(fold ? n : 0);
    // one view's gradients, as the operators write them, before they are folded into the exchange rows
    ws.v_t = cv.take((uint64_t)n * 10); ws.v_o = cv.take(n); ws.v_color = cv.take((uint64_t)n * 3); ws.v_refine = cv.take(n);
    ws.visible = cv.take(n); ws.max_radius = cv.take(n);
    ws.bytes = cv.off;
    return ws;
}

// The bilateral grids' scratch of bg_train_step_views_bilagrid, behind the views-depth workspace: the sliced image, the
// send slots (one per local view: its grid gradient, then its view index as raw bits, padded to keep the slots 16-byte
// aligned) and, with world > 1, the gathered slots of all views in global order.
constexpr uint32_t GRID_SLOT = BG_BILAGRID_FLOATS + 4;
struct ViewsGridWs {
    float *sliced, *send, *recv;
    uint64_t bytes;
};
ViewsGridWs carve_views_grid_ws(void *base, uint64_t off, uint32_t w, uint32_t h, uint32_t local, uint32_t world) {
    Carver cv{base, off};
    ViewsGridWs ws;
    ws.sliced = cv.take((uint64_t)w * h * 4);
    ws.send = cv.take((uint64_t)local * GRID_SLOT);
    ws.recv = cv.take(world > 1 ? (uint64_t)local * world * GRID_SLOT : 0);
    ws.bytes = cv.off;
    return ws;
}

// the checks of BgBilagridViews shared by the step and the operator; local_views > 0 checks the step's view indices
int32_t check_bilagrid_views(const BgBilagridViews *g, uint32_t local_views, const char *who) {
    if (!g || !g->grids || !g->m || !g->v || !g->steps || !g->tv_loss_out || (local_views && !g->view_index)) return BG_ERR_NULL;
    if (g->num_views == 0) return invalid(who, "num_views must be >= 1");
    if (!(g->lr >= 0.0f) || !std::isfinite(g->lr) || !(g->tv_weight >= 0.0f) || !std::isfinite(g->tv_weight))
        return invalid(who, "bilateral grid lr and tv_weight must be finite and >= 0");
    if (!aligned16(g->grids) || !aligned16(g->m) || !aligned16(g->v) || (uintptr_t)g->steps % 4)
        return invalid(who, "grids, m and v must be 16-byte aligned, steps 4-byte aligned");
    for (uint32_t i = 0; i < local_views; i++)
        if (g->view_index[i] >= g->num_views) return invalid(who, "view_index out of range (>= num_views)");
    return BG_OK;
}
}  // namespace

// BG_DP_TRACE=1: device timeline of the multi-device step (stderr, rank 0 only; synchronises -- a debugging aid)
namespace {
struct DpTrace {
    bool on = false;
    cudaEvent_t e[13] = {};
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
        static const char *names[13] = {"step start", "blend bwd + colour pack done", "project bwd + row pack done", "records arrived (s)",
                                        "update part 1 done", "sums arrived (s)", "update part 2 done", "all-gather start (comm)",
                                        "all-gather end (comm)", "all-reduce start (comm)", "all-reduce end (comm)",
                                        "grid gather start (comm)", "grid gather end (comm)"};
        for (int i = 1; i < 13; i++) {
            float ms = 0.0f;
            if (e[i] && cudaEventElapsedTime(&ms, e[0], e[i]) == cudaSuccess) fprintf(stderr, "[bg dp trace] %-32s %8.3f ms\n", names[i], ms);
        }
    }
};
DpTrace g_dp_trace;
}  // namespace

extern "C" uint64_t bg_train_step_views_workspace_bytes(uint32_t n, uint32_t k, uint32_t w, uint32_t h, uint32_t local,
                                                        uint32_t world) {
    (void)k;
    return carve_views_ws(nullptr, n, w, h, std::max(local, 1u), std::max(world, 1u), true).bytes;
}

extern "C" uint64_t bg_train_step_views_depth_workspace_bytes(uint32_t n, uint32_t k, uint32_t w, uint32_t h, uint32_t local,
                                                              uint32_t world) {
    return carve_depth_ws(nullptr, bg_train_step_views_workspace_bytes(n, k, w, h, local, world), n, w, h).bytes;
}

extern "C" uint64_t bg_train_step_views_bilagrid_workspace_bytes(uint32_t n, uint32_t k, uint32_t w, uint32_t h, uint32_t local,
                                                                 uint32_t world) {
    return carve_views_grid_ws(nullptr, bg_train_step_views_depth_workspace_bytes(n, k, w, h, local, world), w, h, std::max(local, 1u),
                               std::max(world, 1u)).bytes;
}

// The multi-view step.  dep == nullptr: bg_train_step_views.  Otherwise dep[local_views] (validated by
// bg_train_step_views_depth); a view whose term runs renders depth and folds its depth gradient into the exchange row, the
// other views run exactly the plain view's launches.  gr: the views' bilateral grids (validated by
// bg_train_step_views_bilagrid) or null.
static int32_t train_step_views(BgContext *c, BgDpComm *h, void *stream, BgTrainViewsArgs *a, const BgDepthSupervision *dep,
                                const BgBilagridViews *gr) {
    if (!c || !a || !a->cams) return BG_ERR_NULL;
    if (int32_t r = check_train_args(a, "bg_train_step_views"); r != BG_OK) return r;
    const uint32_t n = a->n, k = a->k, w = a->w, hh = a->h, local = a->local_views;
    const uint32_t world = h ? (uint32_t)h->c->world : 1u;
    const uint32_t views = local * world;
    if (local == 0 || views > DP_MAX_VIEWS) return invalid("bg_train_step_views", "1..16 views per step in total");
    int deg;
    if (int32_t r = check_k(k, &deg); r != BG_OK) return r;
    for (uint32_t i = 0; i < local; i++)
        if (!a->gt_packed[i]) return BG_ERR_NULL;
    const bool fold = a->min_scale != nullptr;
    const ViewsWs ws = carve_views_ws(a->workspace, n, w, hh, local, world, fold);
    if (int32_t r = check_workspace_bytes("bg_train_step_views", "bg_train_step_views_workspace_bytes", a->workspace_bytes, ws.bytes); r != BG_OK)
        return r;
    if (a->chunks > DP_MAX_CHUNKS) return invalid("bg_train_step_views", "at most 16 chunks");
    const DepthWs dws = carve_depth_ws(a->workspace, bg_train_step_views_workspace_bytes(n, k, w, hh, local, world), n, w, hh);
    if (int32_t r = check_workspace_bytes("bg_train_step_views_depth", "bg_train_step_views_depth_workspace_bytes", a->workspace_bytes,
                                          dep ? dws.bytes : 0); r != BG_OK)
        return r;
    const ViewsGridWs gws = carve_views_grid_ws(gr ? a->workspace : nullptr, bg_train_step_views_depth_workspace_bytes(n, k, w, hh, local, world),
                                                w, hh, local, world);
    if (int32_t r = check_workspace_bytes("bg_train_step_views_bilagrid", "bg_train_step_views_bilagrid_workspace_bytes",
                                          a->workspace_bytes, gr ? gws.bytes : 0); r != BG_OK)
        return r;
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    int32_t r;
    if (dep)
        for (uint32_t i = 0; i < local; i++)
            if (!depth_term(dep[i])) BG_CUDA(cudaMemsetAsync(dep[i].depth_loss_out, 0, sizeof(float), s));
    // the 3D-filter floor folded into what the renderer sees (bwd/burn_glue.rs:260-270)
    const float *r_t = a->transforms, *r_o = a->raw_opac;
    if (fold) {
        r = bg_fold_min_scale_forward(c, stream, n, a->transforms, a->raw_opac, a->min_scale, ws.r_transforms, ws.r_opac);
        if (r != BG_OK) return r;
        r_t = ws.r_transforms; r_o = ws.r_opac;
    }
    BG_CUDA(cudaMemsetAsync(ws.v_output, 0, (size_t)w * hh * 4 * sizeof(float), s));
    DpHeader hdr;
    memset(&hdr, 0, sizeof(hdr));
    for (uint32_t i = 0; i < local; i++)
        for (int q = 0; q < 3; q++) hdr.pos[i][q] = a->cams[i].cam_pos[q];
    BG_CUDA(launch_write_header(s, ws.hdr, hdr, local));
    if (gr) {
        DpGridIndex gi;
        memset(&gi, 0, sizeof(gi));
        for (uint32_t i = 0; i < local; i++) gi.view[i] = gr->view_index[i];
        BG_CUDA(launch_write_grid_index(s, gws.send + BG_BILAGRID_FLOATS, GRID_SLOT, gi, local));
    }
    DpComm *d = world > 1 ? h->c : nullptr;
    DpTrace &tr = g_dp_trace;
    if (d) tr.mark(0, s);
    // The exchange of a step has two parts.  The colour records (all-gather) depend on the blend backward only, so they
    // leave as soon as the last local view's blend backward is done and travel UNDER its projection backward; the summed
    // small rows and the MAX statistics (all-reduces) follow once that is done.  The update pass is split the same way:
    // the SH part (70 % of its traffic) needs the records only and runs under the all-reduces, the rest follows them.
    // With bilateral grids the slots of the grid gradients are gathered first, as soon as the last local view's slice
    // backward is done: they travel under its blend and projection backward.
    bool alpha_dirty = false;   // a depth view added to v_output[...,3], which the 3-channel image loss leaves as it is
    for (uint32_t i = 0; i < local; i++) {
        const BgCamera *cam = a->cams + i;
        const BgDepthSupervision *di = dep && depth_term(dep[i]) ? &dep[i] : nullptr;   // the view's depth term, if it runs
        const DepthWs vd = di ? dws : DepthWs{};   // null buffers select the plain render and blend backward
        if (alpha_dirty && a->channels == 3) BG_CUDA(cudaMemsetAsync(ws.v_output, 0, (size_t)w * hh * 4 * sizeof(float), s));
        alpha_dirty = di != nullptr;
        r = render_forward(c, stream, cam, w, hh, n, k, r_t, a->sh, r_o, a->mip, a->background, BG_PASS_BACKWARD, ws.out_img, vd.depth,
                           ws.visible, ws.max_radius, &a->state_out);
        if (r != BG_OK) return r;
        const float *grid = gr ? gr->grids + (size_t)gr->view_index[i] * BG_BILAGRID_FLOATS : nullptr;
        if (gr) BG_CUDA(launch_bilagrid_slice(s, grid, ws.out_img, w, hh, gws.sliced));
        if ((r = view_loss(c, stream, a, a->gt_packed[i], ws, gr ? gws.sliced : ws.out_img, ws.loss_terms + i, di, dws)) != BG_OK) return r;
        if (gr) {
            // back through the slice in place (the blend backward replays the RAW render); the grid gradient into slot i
            BG_CUDA(launch_bilagrid_slice_bwd(s, grid, ws.out_img, ws.v_output, w, hh, ws.v_output, gws.send + (size_t)i * GRID_SLOT));
            if (d && i + 1 == local) {
                BG_CUDA(cudaEventRecord(d->ev_ready, s));
                BG_CUDA(cudaStreamWaitEvent(d->stream, d->ev_ready, 0));
                tr.mark(11, d->stream);
                const int rc = dp_exchange_grids(d, (size_t)local * GRID_SLOT, gws.send, gws.recv);
                if (rc != 0) return nccl_fail("bg_train_step_views_bilagrid: exchange (grids)", rc);
                tr.mark(12, d->stream);
            }
        }
        r = rasterize_backward(c, stream, &a->state_out, ws.out_img, vd.depth, ws.v_output, vd.v_depth, a->background, 0, ws.v_combined, n,
                               vd.v_z, di ? "bg_rasterize_backward_depth" : "bg_rasterize_backward");
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
        // fold the view into the exchange rows (sum of the small gradients, MAX statistics); a depth view also folds in
        // its mean gradient v_z * R[2,:] on the way (the rounding of depth_to_means, no pass of its own)
        if (di)
            BG_CUDA(launch_pack_view_depth(s, n, local, i, i == 0, ws.v_t, ws.v_o, ws.v_refine, ws.visible, ws.max_radius,
                                           a->state_out.compact_from_global_gid, dws.v_z, *cam, ws.small, ws.stat, ws.record));
        else
            BG_CUDA(launch_pack_view(s, n, local, i, i == 0, ws.v_t, ws.v_o, nullptr, ws.v_refine, ws.visible, ws.max_radius, ws.small,
                                     ws.stat, ws.record));
    }
    if (gr) {
        // every rank updates the grids of all views of the step from the same slots in global order
        float *slots = d ? gws.recv : gws.send;
        if (d) BG_CUDA(cudaStreamWaitEvent(s, d->ev_chunk[2], 0));
        BG_CUDA(launch_bilagrid_update_views(s, gr->grids, gr->m, gr->v, gr->steps, gr->num_views, gr->lr, gr->tv_weight, slots,
                                             GRID_SLOT, reinterpret_cast<const uint32_t *>(slots + BG_BILAGRID_FLOATS), GRID_SLOT,
                                             views, d ? (uint32_t)d->rank * local : 0u, local, gr->tv_loss_out, ws.loss_terms));
    }
    BG_CUDA(launch_loss_mean(s, ws.loss_terms, local, a->loss_out));
    UpdateParams P = update_params(a);
    P.min_scale = a->min_scale;   // the noise gate folds the floor in, as the render did
    P.small = ws.small; P.stat = ws.stat;
    P.grad_scale = 1.0f / (float)views; P.sh_grad_scale = 1.0f / (float)views;
    P.views = views; P.local = local; P.world = world;
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

extern "C" int32_t bg_train_step_views(BgContext *c, BgDpComm *h, void *stream, BgTrainViewsArgs *a) {
    return train_step_views(c, h, stream, a, nullptr, nullptr);
}

// ---- bg_train_step_views_depth: bg_train_step_views with the depth term of DESIGN.md section 4.7 on the views that carry one.
// The depth gradient reaches v_transforms[:, 0:3] and the refine weight only, both already in the exchanged rows: the
// exchange is unchanged, and ranks with and without depth views share a step.
static int32_t check_views_depth(const BgTrainViewsArgs *a, const BgDepthSupervision *depth, const char *who) {
    for (uint32_t i = 0; i < a->local_views; i++) {
        if (int32_t r = check_depth(depth[i], who); r != BG_OK) return r;
        if (depth_term(depth[i]) && (uintptr_t)depth[i].target % 4) return invalid(who, "target must be 4-byte aligned");
    }
    return BG_OK;
}

extern "C" int32_t bg_train_step_views_depth(BgContext *c, BgDpComm *h, void *stream, BgTrainViewsArgs *a, const BgDepthSupervision *depth) {
    if (!c || !a || !depth) return BG_ERR_NULL;
    const uint32_t local = a->local_views;
    if (local == 0 || local > DP_MAX_VIEWS) return invalid("bg_train_step_views_depth", "1..16 views per step in total");
    if (int32_t r = check_views_depth(a, depth, "bg_train_step_views_depth"); r != BG_OK) return r;
    return train_step_views(c, h, stream, a, depth, nullptr);
}

// ---- bg_train_step_views_bilagrid: the multi-view step with the views' bilateral grids (DESIGN.md section 4.11), with or
// without the depth term
extern "C" int32_t bg_train_step_views_bilagrid(BgContext *c, BgDpComm *h, void *stream, BgTrainViewsArgs *a,
                                                const BgDepthSupervision *depth, const BgBilagridViews *grids) {
    const char *who = "bg_train_step_views_bilagrid";
    if (!c || !a || !grids) return BG_ERR_NULL;
    const uint32_t local = a->local_views;
    if (local == 0 || local > DP_MAX_VIEWS) return invalid(who, "1..16 views per step in total");
    if (int32_t r = check_bilagrid_views(grids, local, who); r != BG_OK) return r;
    if (depth)
        if (int32_t r = check_views_depth(a, depth, who); r != BG_OK) return r;
    return train_step_views(c, h, stream, a, depth, grids);
}

extern "C" int32_t bg_bilagrid_update_views(BgContext *c, void *stream, const BgBilagridViews *grids, uint32_t slots,
                                            const uint32_t *slot_view, float *v_grids) {
    const char *who = "bg_bilagrid_update_views";
    if (!c || !slot_view || !v_grids) return BG_ERR_NULL;
    if (int32_t r = check_bilagrid_views(grids, 0, who); r != BG_OK) return r;
    if (slots == 0 || slots > DP_MAX_VIEWS) return invalid(who, "1..16 slots");
    if (!aligned16(v_grids) || (uintptr_t)slot_view % 4) return invalid(who, "v_grids must be 16-byte aligned, slot_view 4-byte aligned");
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_bilagrid_update_views((cudaStream_t)stream, grids->grids, grids->m, grids->v, grids->steps, grids->num_views,
                                         grids->lr, grids->tv_weight, v_grids, BG_BILAGRID_FLOATS, slot_view, 1, slots, 0, slots,
                                         grids->tv_loss_out, nullptr));
    return BG_OK;
}

// ---- refine (refine.cu): every decision on the device, one readback of the counts at the end
namespace {
struct RefineWs : SortWs {
    uint32_t *ctl, *keep, *keep_incl, *split, *cand, *cand_incl, *split_incl;
    float *refine_norm, *vis_weight, *max_screen, *bounds_out;
    uint64_t bytes;
};
RefineWs carve_refine_ws(void *base, uint32_t n) {
    Carver cv{base};
    auto take = [&](uint64_t words) { return cv.take<uint32_t>(words); };
    RefineWs w;
    w.ctl = take(64);
    w.keep = take(n); w.keep_incl = take(n);
    carve_sort_ws(cv, n, w);
    w.split = take(n); w.cand = take(n); w.cand_incl = take(n); w.split_incl = take(n);
    w.refine_norm = cv.take(n); w.vis_weight = cv.take(n); w.max_screen = cv.take(n);
    w.bounds_out = cv.take(16);
    w.bytes = cv.off;
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
    int32_t r;
    if ((r = check_k(a->k)) != BG_OK) return r;
    if (a->capacity < n0) return capacity("bg_refine", "capacity smaller than n");
    const RefineWs w = carve_refine_ws(a->workspace, n0);
    if ((r = check_workspace("bg_refine", "bg_refine_workspace_bytes", a->workspace, a->workspace_bytes, w.bytes)) != BG_OK) return r;
    if (n0 > sort_capacity(c)) return capacity("bg_refine", "n exceeds the context's sort capacity");
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    const uint32_t kf = a->k * 3;
    RefinePtrs p;
    p.transforms = a->transforms; p.sh = a->sh; p.raw_opac = a->raw_opac; p.m_t = a->m_t; p.v_t = a->v_t; p.m_sh = a->m_sh;
    p.v_sh = a->v_sh; p.m_o = a->m_o; p.v_o = a->v_o; p.refine_norm = a->refine_norm; p.vis_weight = a->vis_weight; p.max_screen = a->max_screen;
    p.transforms_out = a->transforms_out; p.sh_out = a->sh_out; p.raw_opac_out = a->raw_opac_out; p.m_t_out = a->m_t_out;
    p.v_t_out = a->v_t_out; p.m_sh_out = a->m_sh_out; p.v_sh_out = a->v_sh_out; p.m_o_out = a->m_o_out; p.v_o_out = a->v_o_out;
    p.refine_norm_tmp = w.refine_norm; p.vis_weight_tmp = w.vis_weight; p.max_screen_tmp = w.max_screen;
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
    if (host[RC_OVERFLOW]) return capacity("bg_refine", "capacity of the destination arrays exceeded");
    return BG_OK;
}

extern "C" int32_t bg_bounds_percentile(BgContext *c, void *stream, uint32_t n, const float *transforms, float percentile,
                                        void *workspace, uint64_t workspace_bytes, float *out6) {
    if (!c || !out6) return BG_ERR_NULL;
    for (int i = 0; i < 6; i++) out6[i] = 0.0f;
    if (n == 0) return BG_OK;
    if (!transforms || !workspace) return BG_ERR_NULL;
    const RefineWs w = carve_refine_ws(workspace, n);
    if (int32_t r = check_workspace_bytes("bg_bounds_percentile", "bg_refine_workspace_bytes", workspace_bytes, w.bytes); r != BG_OK) return r;
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

extern "C" uint64_t bg_decimate_workspace_bytes(uint32_t n) {
    Carver cv{nullptr};
    SortWs w;
    carve_sort_ws(cv, std::max(n, 1u), w);   // the sort's buffers are all of it
    return cv.off;
}

extern "C" int32_t bg_decimate_to_count(BgContext *c, void *stream, const BgDecimateArgs *a) {
    if (!c || !a) return BG_ERR_NULL;
    const uint32_t n = a->n, target = a->target;
    if (target == 0 || target >= n) return BG_OK;   // lod.rs:15-17: the input is returned unchanged
    if (!a->scores || !a->transforms || !a->sh || !a->raw_opac || !a->transforms_out || !a->sh_out || !a->raw_opac_out ||
        !a->workspace || (a->min_scale && !a->min_scale_out))
        return BG_ERR_NULL;
    int32_t r;
    if ((r = check_k(a->k)) != BG_OK) return r;
    const void *ptrs[] = {a->transforms, a->sh, a->raw_opac, a->min_scale, a->transforms_out, a->sh_out, a->raw_opac_out,
                          a->min_scale_out, a->workspace};
    for (const void *p : ptrs)
        if ((uintptr_t)p % 16) return invalid("bg_decimate_to_count", "arrays must be 16-byte aligned");
    Carver cv{a->workspace};
    SortWs w;
    carve_sort_ws(cv, n, w);
    if ((r = check_workspace("bg_decimate_to_count", "bg_decimate_workspace_bytes", a->workspace, a->workspace_bytes, cv.off)) != BG_OK) return r;
    if (n > sort_capacity(c)) return capacity("bg_decimate_to_count", "n exceeds the context's sort capacity");
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_decimate_keys(s, n, a->scores, w.keys, w.vals));
    if ((r = bg_radix_argsort_u32(c, stream, w.keys, w.vals, n, nullptr, 32, w.keys_s, w.vals_s)) != BG_OK) return r;
    BG_CUDA(launch_decimate_gather(s, target, a->k * 3, w.vals_s, a->transforms, a->sh, a->raw_opac, a->min_scale,
                                   a->transforms_out, a->sh_out, a->raw_opac_out, a->min_scale_out));
    if (a->kept_ids_out) BG_CUDA(cudaMemcpyAsync(a->kept_ids_out, w.vals_s, (size_t)target * 4, cudaMemcpyDeviceToDevice, s));
    return BG_OK;
}

// ---- Compressed PLY encoding (compress.cu, DESIGN.md section 4.8)
namespace {
struct CompressWs : SortWs {
    uint32_t *bounds;
    uint64_t bytes;
};
CompressWs carve_compress_ws(void *base, uint32_t n) {
    Carver cv{base};
    CompressWs w;
    w.bounds = cv.take<uint32_t>(8);
    carve_sort_ws(cv, n, w);
    w.bytes = cv.off;
    return w;
}
}  // namespace

extern "C" uint64_t bg_compress_workspace_bytes(uint32_t n) { return carve_compress_ws(nullptr, std::max(n, 1u)).bytes; }

extern "C" int32_t bg_compress_splats(BgContext *c, void *stream, const BgCompressArgs *a) {
    if (!c || !a) return BG_ERR_NULL;
    const uint32_t n = a->n, k = a->k;
    if (!a->count_out) return BG_ERR_NULL;
    int32_t r;
    if ((r = check_k(k)) != BG_OK) return r;
    if ((uintptr_t)a->count_out % 4) return invalid("bg_compress_splats", "count_out must be 4-byte aligned");
    cudaStream_t s = (cudaStream_t)stream;
    if (n == 0) {
        BG_CUDA(cudaSetDevice(c->device));
        BG_CUDA(cudaMemsetAsync(a->count_out, 0, 4, s));
        return BG_OK;
    }
    if (!a->transforms || !a->sh || !a->raw_opac || !a->chunks_out || !a->packed_out || !a->workspace || (k > 1 && !a->sh_out))
        return BG_ERR_NULL;
    if (k == 1 && a->sh_out) return invalid("bg_compress_splats", "sh_out must be NULL when k == 1");
    if (((uintptr_t)a->transforms | (uintptr_t)a->packed_out) % 16 ||
        ((uintptr_t)a->sh | (uintptr_t)a->raw_opac | (uintptr_t)a->chunks_out | (uintptr_t)a->order_out) % 4)
        return invalid("bg_compress_splats", "transforms and packed_out must be 16-byte aligned, the other arrays 4-byte");
    const CompressWs w = carve_compress_ws(a->workspace, n);
    if ((r = check_workspace("bg_compress_splats", "bg_compress_workspace_bytes", a->workspace, a->workspace_bytes, w.bytes)) != BG_OK) return r;
    if (n > sort_capacity(c)) return capacity("bg_compress_splats", "n exceeds the context's sort capacity");
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_compress_valid_bounds(s, n, k * 3, a->transforms, a->sh, a->raw_opac, w.keys, w.bounds));
    BG_CUDA(launch_compress_keys(s, n, a->transforms, w.bounds, w.keys, w.vals));
    if ((r = bg_radix_argsort_u32(c, stream, w.keys, w.vals, n, nullptr, 31, w.keys_s, w.vals_s)) != BG_OK) return r;
    BG_CUDA(launch_compress_chunks(s, n, k, a->transforms, a->sh, a->raw_opac, w.bounds, w.vals_s, a->chunks_out, a->packed_out,
                                   a->sh_out, a->order_out, a->count_out));
    return BG_OK;
}

// ---- Mesh export (mesh.cu, DESIGN.md section 4.9)
namespace {
struct MeshWs {
    unsigned long long *header;   // [8]: vertex total, triangle total, dims of the counted grid
    uint32_t *brick_v, *brick_t, *voff, *toff, *vbase;
    uint8_t *vmask;
    uint64_t bytes;
};
MeshWs carve_mesh_ws(void *base, const uint32_t *dims) {
    Carver cv{base};
    MeshWs w;
    const uint64_t nb = mesh_num_bricks(dims), np = (uint64_t)dims[0] * dims[1] * dims[2];
    w.header = cv.take<unsigned long long>(8);
    w.brick_v = cv.take<uint32_t>(nb); w.brick_t = cv.take<uint32_t>(nb);
    w.voff = cv.take<uint32_t>(nb); w.toff = cv.take<uint32_t>(nb);
    w.vbase = cv.take<uint32_t>(np);
    w.vmask = cv.take<uint8_t>(np);
    w.bytes = cv.off;
    return w;
}
// Lattice checks shared by the dense and the sparse grid.
int32_t check_lattice(const float *origin, float h, float trunc, const char *who) {
    if (!(h > 0.0f) || !std::isfinite(h) || !(trunc > 0.0f) || !std::isfinite(trunc) || !std::isfinite(origin[0]) ||
        !std::isfinite(origin[1]) || !std::isfinite(origin[2]))
        return invalid(who, "grid origin must be finite, h and trunc finite and > 0");
    return BG_OK;
}
// Grid checks shared by the three calls: BG_OK, or the status with the message set.
int32_t check_grid(const BgTsdfGrid *g, const char *who) {
    if (!g->tsdf || !g->weight || !g->rgb) return BG_ERR_NULL;
    const uint64_t np = (uint64_t)g->dims[0] * g->dims[1] * g->dims[2];
    if (np == 0 || np >= (1ull << 31)) return invalid(who, "grid dims must be non-zero with dx*dy*dz < 2^31");
    if (((uintptr_t)g->tsdf | (uintptr_t)g->weight | (uintptr_t)g->rgb) % 4) return invalid(who, "grid arrays must be 4-byte aligned");
    return check_lattice(g->origin, g->h, g->trunc, who);
}
// One view's render and camera, as the integration and the marking take them.
int32_t check_view(const BgCamera *cam, uint32_t w, uint32_t h, const float *out_img, const float *out_depth, float alpha_min,
                   const char *who) {
    if (w == 0 || h == 0) return invalid(who, "empty image");
    if (!(alpha_min > 0.0f && alpha_min <= 1.0f)) return invalid(who, "alpha_min must be in (0, 1]");
    if (cam->camera_model > BG_CAMERA_THIN_PRISM_FISHEYE) return invalid(who, "unknown camera model");
    if ((uintptr_t)out_img % 16 || (uintptr_t)out_depth % 4) return invalid(who, "out_img must be 16-byte aligned, out_depth 4-byte");
    return BG_OK;
}
}  // namespace

extern "C" int32_t bg_tsdf_integrate(BgContext *c, void *stream, const BgTsdfGrid *g, const BgCamera *cam, uint32_t w, uint32_t h,
                                     const float *out_img, const float *out_depth, float alpha_min) {
    if (!c || !g || !cam || !out_img || !out_depth) return BG_ERR_NULL;
    int32_t r = check_grid(g, "bg_tsdf_integrate");
    if (r != BG_OK) return r;
    if ((r = check_view(cam, w, h, out_img, out_depth, alpha_min, "bg_tsdf_integrate")) != BG_OK) return r;
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_tsdf_integrate((cudaStream_t)stream, *g, *cam, w, h, out_img, out_depth, alpha_min));
    return BG_OK;
}

extern "C" uint64_t bg_mesh_workspace_bytes(uint32_t dx, uint32_t dy, uint32_t dz) {
    const uint32_t dims[3] = {std::max(dx, 1u), std::max(dy, 1u), std::max(dz, 1u)};
    return carve_mesh_ws(nullptr, dims).bytes;
}

extern "C" int32_t bg_mesh_count(BgContext *c, void *stream, const BgTsdfGrid *g, void *ws, uint64_t ws_bytes, uint32_t *num_vertices,
                                 uint32_t *num_triangles) {
    if (!c || !g || !num_vertices || !num_triangles) return BG_ERR_NULL;
    *num_vertices = 0;
    *num_triangles = 0;
    int32_t r = check_grid(g, "bg_mesh_count");
    if (r != BG_OK) return r;
    const MeshWs w = carve_mesh_ws(ws, g->dims);
    if ((r = check_workspace("bg_mesh_count", "bg_mesh_workspace_bytes", ws, ws_bytes, w.bytes)) != BG_OK) return r;
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_mesh_count(s, *g, w.brick_v, w.brick_t, w.voff, w.toff, w.header));
    unsigned long long host[2];
    BG_CUDA(cudaMemcpyAsync(host, w.header, sizeof(host), cudaMemcpyDeviceToHost, s));
    BG_CUDA(cudaStreamSynchronize(s));
    if (host[0] > 0xFFFFFFFFull || host[1] > 0xFFFFFFFFull) return capacity("bg_mesh_count", "more than 2^32 - 1 vertices or triangles");
    *num_vertices = (uint32_t)host[0];
    *num_triangles = (uint32_t)host[1];
    return BG_OK;
}

extern "C" int32_t bg_mesh_emit(BgContext *c, void *stream, const BgTsdfGrid *g, void *ws, uint64_t ws_bytes, uint32_t max_vertices,
                                uint32_t max_triangles, float *vertices, uint8_t *colors, uint32_t *faces) {
    if (!c || !g) return BG_ERR_NULL;
    int32_t r = check_grid(g, "bg_mesh_emit");
    if (r != BG_OK) return r;
    if ((max_vertices && (!vertices || !colors)) || (max_triangles && !faces)) return BG_ERR_NULL;
    if (((uintptr_t)vertices | (uintptr_t)faces) % 4) return invalid("bg_mesh_emit", "vertices and faces must be 4-byte aligned");
    const MeshWs w = carve_mesh_ws(ws, g->dims);
    if ((r = check_workspace("bg_mesh_emit", "bg_mesh_workspace_bytes", ws, ws_bytes, w.bytes)) != BG_OK) return r;
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    unsigned long long host[5];
    BG_CUDA(cudaMemcpyAsync(host, w.header, sizeof(host), cudaMemcpyDeviceToHost, s));
    BG_CUDA(cudaStreamSynchronize(s));
    if (host[2] != g->dims[0] || host[3] != g->dims[1] || host[4] != g->dims[2])
        return invalid("bg_mesh_emit", "the workspace holds no bg_mesh_count of a grid with these dims");
    if (host[0] > max_vertices || host[1] > max_triangles) return capacity("bg_mesh_emit", "the mesh exceeds max_vertices / max_triangles");
    if (host[0] == 0) return BG_OK;   // no vertices, so no triangles
    BG_CUDA(launch_mesh_emit(s, *g, w.voff, w.toff, w.vbase, w.vmask, max_vertices, max_triangles, vertices, colors, faces));
    return BG_OK;
}

// ---- Sparse mesh export (mesh_sparse.cu, DESIGN.md section 4.10)
namespace {
uint64_t sparse_brick_count(const uint32_t *dims) {
    return (uint64_t)((dims[0] + 7) / 8) * ((dims[1] + 7) / 8) * ((dims[2] + 7) / 8);
}
// w = h = 0: the part kept for the grid's life, without a view's pyramid
SparseTsdfWs carve_sparse_ws(void *base, const uint32_t *dims, uint32_t w, uint32_t h, uint64_t &bytes) {
    Carver cv{base};
    SparseTsdfWs s;
    const uint64_t nb = sparse_brick_count(dims), nblk = (nb + 1023) / 1024;
    s.header = cv.take<unsigned long long>(8);
    s.cand_count = cv.take<uint32_t>(1);
    s.bitmap = cv.take<uint32_t>((nb + 31) / 32);
    s.blk_cnt = cv.take<uint32_t>(nblk);
    s.blk_off = cv.take<uint32_t>(nblk);
    s.list = cv.take<uint32_t>(nb);
    s.pyramid = cv.take<float2>(w && h ? sparse_pyramid_cells(w, h) : 0);
    bytes = cv.off;
    return s;
}
SparseMeshWs carve_sparse_mesh_ws(void *base, uint32_t num_bricks, uint64_t &bytes) {
    Carver cv{base};
    SparseMeshWs m;
    const uint64_t np = (uint64_t)num_bricks * 512;
    m.header = cv.take<unsigned long long>(8);
    m.brick_v = cv.take<uint32_t>(num_bricks); m.brick_t = cv.take<uint32_t>(num_bricks);
    m.voff = cv.take<uint32_t>(num_bricks); m.toff = cv.take<uint32_t>(num_bricks);
    m.vbase = cv.take<uint32_t>(np);
    m.vmask = cv.take<uint8_t>(np);
    bytes = cv.off;
    return m;
}
// The grid and its workspace (sized for a w x h view; 0 x 0 for the calls that take no view).
int32_t check_sparse_grid(const BgSparseTsdfGrid *g, uint32_t w, uint32_t h, const char *who, SparseTsdfWs &ws) {
    if (!g->brick_slot) return BG_ERR_NULL;
    if (!g->dims[0] || !g->dims[1] || !g->dims[2] || g->dims[0] > (1u << 24) || g->dims[1] > (1u << 24) || g->dims[2] > (1u << 24) ||
        sparse_brick_count(g->dims) >= (1ull << 31))
        return invalid(who, "grid dims must be in [1, 2^24] with fewer than 2^31 bricks");
    if ((uintptr_t)g->brick_slot % 4) return invalid(who, "brick_slot must be 4-byte aligned");
    int32_t r = check_lattice(g->origin, g->h, g->trunc, who);
    if (r != BG_OK) return r;
    uint64_t need;
    ws = carve_sparse_ws(g->workspace, g->dims, w, h, need);
    return check_workspace(who, "bg_sparse_tsdf_workspace_bytes", g->workspace, g->workspace_bytes, need);
}
int32_t check_sparse_pool(const BgSparseTsdfGrid *g, const char *who) {
    if (g->num_bricks && (!g->tsdf || !g->weight || !g->rgb)) return BG_ERR_NULL;
    if (((uintptr_t)g->tsdf | (uintptr_t)g->weight | (uintptr_t)g->rgb) % 4) return invalid(who, "pool arrays must be 4-byte aligned");
    return BG_OK;
}
// Reads the grid header back: the allocated brick count, which the pool must hold.
int32_t sparse_slots(cudaStream_t s, const BgSparseTsdfGrid *g, const SparseTsdfWs &ws, const char *who, uint32_t &slots) {
    unsigned long long host[8];
    BG_CUDA(cudaMemcpyAsync(host, ws.header, sizeof(host), cudaMemcpyDeviceToHost, s));
    BG_CUDA(cudaStreamSynchronize(s));
    if (!host[SPARSE_H_ALLOCATED]) return invalid(who, "the grid is not allocated (bg_sparse_tsdf_allocate)");
    if (host[SPARSE_H_DIMS] != g->dims[0] || host[SPARSE_H_DIMS + 1] != g->dims[1] || host[SPARSE_H_DIMS + 2] != g->dims[2])
        return invalid(who, "the workspace was allocated for a grid with other dims");
    if (host[SPARSE_H_BRICKS] > g->num_bricks) return capacity(who, "num_bricks is smaller than the allocated brick count");
    slots = (uint32_t)host[SPARSE_H_BRICKS];
    return BG_OK;
}
}  // namespace

extern "C" uint64_t bg_sparse_tsdf_workspace_bytes(uint32_t dx, uint32_t dy, uint32_t dz, uint32_t max_w, uint32_t max_h) {
    const uint32_t dims[3] = {std::max(dx, 1u), std::max(dy, 1u), std::max(dz, 1u)};
    uint64_t bytes;
    carve_sparse_ws(nullptr, dims, max_w, max_h, bytes);
    return bytes;
}

extern "C" int32_t bg_sparse_tsdf_mark(BgContext *c, void *stream, const BgSparseTsdfGrid *g, const BgCamera *cam, uint32_t w,
                                       uint32_t h, const float *out_img, const float *out_depth, float alpha_min) {
    if (!c || !g || !cam || !out_img || !out_depth) return BG_ERR_NULL;
    int32_t r = check_view(cam, w, h, out_img, out_depth, alpha_min, "bg_sparse_tsdf_mark");
    if (r != BG_OK) return r;
    SparseTsdfWs ws;
    if ((r = check_sparse_grid(g, w, h, "bg_sparse_tsdf_mark", ws)) != BG_OK) return r;
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_sparse_mark((cudaStream_t)stream, c->sm_count, *g, *cam, w, h, out_img, out_depth, alpha_min, ws));
    return BG_OK;
}

extern "C" int32_t bg_sparse_tsdf_allocate(BgContext *c, void *stream, const BgSparseTsdfGrid *g, uint32_t *num_bricks) {
    if (!c || !g || !num_bricks) return BG_ERR_NULL;
    *num_bricks = 0;
    SparseTsdfWs ws;
    int32_t r = check_sparse_grid(g, 0, 0, "bg_sparse_tsdf_allocate", ws);
    if (r != BG_OK) return r;
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(launch_sparse_allocate(s, *g, ws));
    unsigned long long host;
    BG_CUDA(cudaMemcpyAsync(&host, ws.header + SPARSE_H_BRICKS, sizeof(host), cudaMemcpyDeviceToHost, s));
    BG_CUDA(cudaStreamSynchronize(s));
    *num_bricks = (uint32_t)host;   // at most the brick count, < 2^31
    return BG_OK;
}

extern "C" int32_t bg_sparse_tsdf_integrate(BgContext *c, void *stream, const BgSparseTsdfGrid *g, const BgCamera *cam, uint32_t w,
                                            uint32_t h, const float *out_img, const float *out_depth, float alpha_min) {
    if (!c || !g || !cam || !out_img || !out_depth) return BG_ERR_NULL;
    int32_t r = check_view(cam, w, h, out_img, out_depth, alpha_min, "bg_sparse_tsdf_integrate");
    if (r != BG_OK) return r;
    SparseTsdfWs ws;
    if ((r = check_sparse_grid(g, 0, 0, "bg_sparse_tsdf_integrate", ws)) != BG_OK) return r;
    if ((r = check_sparse_pool(g, "bg_sparse_tsdf_integrate")) != BG_OK) return r;
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    uint32_t slots;
    if ((r = sparse_slots(s, g, ws, "bg_sparse_tsdf_integrate", slots)) != BG_OK || slots == 0) return r;
    BG_CUDA(launch_sparse_integrate(s, *g, slots, *cam, w, h, out_img, out_depth, alpha_min, ws));
    return BG_OK;
}

extern "C" uint64_t bg_sparse_mesh_workspace_bytes(uint32_t num_bricks) {
    uint64_t bytes;
    carve_sparse_mesh_ws(nullptr, num_bricks, bytes);
    return bytes;
}

extern "C" int32_t bg_sparse_mesh_count(BgContext *c, void *stream, const BgSparseTsdfGrid *g, void *mws, uint64_t mws_bytes,
                                        uint32_t *num_vertices, uint32_t *num_triangles) {
    if (!c || !g || !num_vertices || !num_triangles) return BG_ERR_NULL;
    *num_vertices = 0;
    *num_triangles = 0;
    SparseTsdfWs ws;
    int32_t r = check_sparse_grid(g, 0, 0, "bg_sparse_mesh_count", ws);
    if (r != BG_OK) return r;
    if ((r = check_sparse_pool(g, "bg_sparse_mesh_count")) != BG_OK) return r;
    uint64_t need;
    const SparseMeshWs m = carve_sparse_mesh_ws(mws, g->num_bricks, need);
    if ((r = check_workspace("bg_sparse_mesh_count", "bg_sparse_mesh_workspace_bytes", mws, mws_bytes, need)) != BG_OK) return r;
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    uint32_t slots;
    if ((r = sparse_slots(s, g, ws, "bg_sparse_mesh_count", slots)) != BG_OK) return r;
    BG_CUDA(launch_sparse_mesh_count(s, *g, slots, ws, m));
    unsigned long long host[2];
    BG_CUDA(cudaMemcpyAsync(host, m.header, sizeof(host), cudaMemcpyDeviceToHost, s));
    BG_CUDA(cudaStreamSynchronize(s));
    if (host[0] > 0xFFFFFFFFull || host[1] > 0xFFFFFFFFull)
        return capacity("bg_sparse_mesh_count", "more than 2^32 - 1 vertices or triangles");
    *num_vertices = (uint32_t)host[0];
    *num_triangles = (uint32_t)host[1];
    return BG_OK;
}

extern "C" int32_t bg_sparse_mesh_emit(BgContext *c, void *stream, const BgSparseTsdfGrid *g, void *mws, uint64_t mws_bytes,
                                       uint32_t max_vertices, uint32_t max_triangles, float *vertices, uint8_t *colors,
                                       uint32_t *faces) {
    if (!c || !g) return BG_ERR_NULL;
    SparseTsdfWs ws;
    int32_t r = check_sparse_grid(g, 0, 0, "bg_sparse_mesh_emit", ws);
    if (r != BG_OK) return r;
    if ((r = check_sparse_pool(g, "bg_sparse_mesh_emit")) != BG_OK) return r;
    if ((max_vertices && (!vertices || !colors)) || (max_triangles && !faces)) return BG_ERR_NULL;
    if (((uintptr_t)vertices | (uintptr_t)faces) % 4) return invalid("bg_sparse_mesh_emit", "vertices and faces must be 4-byte aligned");
    uint64_t need;
    const SparseMeshWs m = carve_sparse_mesh_ws(mws, g->num_bricks, need);
    if ((r = check_workspace("bg_sparse_mesh_emit", "bg_sparse_mesh_workspace_bytes", mws, mws_bytes, need)) != BG_OK) return r;
    cudaStream_t s = (cudaStream_t)stream;
    BG_CUDA(cudaSetDevice(c->device));
    unsigned long long host[6];
    BG_CUDA(cudaMemcpyAsync(host, m.header, sizeof(host), cudaMemcpyDeviceToHost, s));
    BG_CUDA(cudaStreamSynchronize(s));
    if (host[3] != g->dims[0] || host[4] != g->dims[1] || host[5] != g->dims[2] || host[2] > g->num_bricks)
        return invalid("bg_sparse_mesh_emit", "the workspace holds no bg_sparse_mesh_count of a grid with these dims and pool");
    if (host[0] > max_vertices || host[1] > max_triangles)
        return capacity("bg_sparse_mesh_emit", "the mesh exceeds max_vertices / max_triangles");
    if (host[0] == 0) return BG_OK;   // no vertices, so no triangles
    BG_CUDA(launch_sparse_mesh_emit(s, *g, (uint32_t)host[2], ws, m, max_vertices, max_triangles, vertices, colors, faces));
    return BG_OK;
}
