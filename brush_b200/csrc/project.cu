// project.cu -- per-Gaussian forward stages (compiled with -fmad=false, see bg_math.cuh).
//
//   project_cull_kernel        <- project_forward_kernel  (kernels/project_forward.rs:20-125)
//   gather_scan_kernel         <- int_gather + prefix_sum (render.rs:185-187, brush-prefix-sum)
//   project_visible_emit_kernel<- project_visible_kernel  (kernels/project_visible.rs:22-88)
//                                 + map_gaussians_to_intersect_kernel (kernels/map_gaussians.rs:14-80)
//   tile_offsets_kernel        <- get_tile_offsets        (get_tile_offset.rs:10-58)
//
// HBM-bound in principle; in practice project_cull is issue-bound (exact tile tests) and project_visible_emit is
// gather-latency bound.  Design notes:
//   * persistent CTAs pull tiles from an atomic ticket; counts that the reference reads back to
//     the host (num_visible, num_intersections) stay on the device and downstream kernels read
//     them from the control block;
//   * compaction of visible Gaussians is a single-pass decoupled look-back in index order --
//     deterministic, unlike the reference's atomic slot (project_forward.rs:122-124);
//   * the [n,10] AoS rows of a tile are staged with one TMA bulk copy (cp.async.bulk + mbarrier),
//     double buffered; the SH rows are read in index order there too, and the depth-ordered pass gathers one
//     64-byte staged row per splat (two whole 32-byte sectors).
#include "bg_project.cuh"
#include "bg_launch.cuh"

namespace bg {

constexpr int PROJ_THREADS = 256;

struct CullResult {
    bool visible;
    float depth;
    uint32_t tiles;
    float radius;
    unsigned long long mask;  // hit bits of the bbox tiles, row major, valid when the bbox has <= 64 tiles
    // screen-space footprint, consumed by the warp-cooperative tile count
    float mx, my, c00, c01, c11, pt;
    float opac;               // compensated opacity, lane 5 of the projected row
    uint32_t min_x, min_y, bbw, ntiles;
};

// Everything of project_forward up to the tile bbox (project_forward.rs:43-117).
template <bool MIP, bool DIST>
__device__ __forceinline__ CullResult cull_one(const float *t, float raw_opac, const BgCamera &u, uint32_t img_w,
                                               uint32_t img_h, uint32_t tiles_x, uint32_t tiles_y) {
    CullResult r;
    r.visible = false; r.depth = 0.0f; r.tiles = 0; r.radius = 0.0f; r.mask = 0ull;
    r.mx = r.my = r.c00 = r.c01 = r.c11 = r.pt = r.opac = 0.0f;
    r.min_x = r.min_y = r.bbw = r.ntiles = 0;
    V3 mean_c = world_to_cam(mk3(t[0], t[1], t[2]), u);
    if (!(is_finite(mean_c) && mean_c.z <= 1.0e10f)) return r;
    if (!in_front<DIST>(mean_c, u)) return r;
    V3 scl = mk3(det_expf(t[7]), det_expf(t[8]), det_expf(t[9]));
    if (!is_finite(scl)) return r;
    Q4 qu; qu.w = t[3]; qu.x = t[4]; qu.y = t[5]; qu.z = t[6];
    float qn = dot(qu, qu);
    if (!(qn >= 1.0e-6f && is_finite(qn))) return r;
    if (!is_finite(raw_opac)) return r;
    Q4 quat = normalize(qu);
    S2 raw_cov = calc_cov2d<DIST>(scl, quat, mean_c, u);
    float comp;
    S2 cov = compensate_cov2d<MIP>(raw_cov, comp);
    float opac = det_sigmoid(raw_opac) * comp;
    if (!is_finite(cov)) return r;
    float mx, my;
    project_mean<DIST>(mean_c, u, mx, my);
    if (!(opac >= 1.0f / 255.0f)) return r;
    float pt = det_logf(opac * 255.0f);
    S2 conic = inverse(cov);
    float ex, ey;
    bbox_extent(conic, pt, ex, ey);
    if (!(ex >= 0.0f && ey >= 0.0f)) return r;
    float wf = (float)img_w, hf = (float)img_h;
    bool on_screen = mx + ex > 0.0f && mx - ex < wf && my + ey > 0.0f && my - ey < hf;
    if (!on_screen) return r;
    TileBox bb = tile_bbox(mx, my, ex, ey, tiles_x, tiles_y);
    r.visible = true;
    r.depth = mean_c.z;
    r.radius = fmaxf(ex / wf, ey / hf);
    r.mx = mx; r.my = my; r.c00 = conic.c00; r.c01 = conic.c01; r.c11 = conic.c11; r.pt = pt; r.opac = opac;
    r.min_x = bb.min_x; r.min_y = bb.min_y; r.bbw = bb.max_x - bb.min_x;
    r.ntiles = (bb.max_y - bb.min_y) * r.bbw;
    return r;
}

// count_contributing_tiles (helpers.rs:203-222) for the 32 Gaussians of a warp at once.  A per-thread
// walk costs the warp the LARGEST bbox among its lanes; here the warp's candidate tiles are flattened
// into one list and tested 32 at a time, whoever they belong to (binary search of the owner over the
// exclusive prefix of the per-lane tile counts).  Hit counts and the 64-bit hit mask are collected by the
// owner lane from the ballot of each round.
__device__ __forceinline__ void warp_count_tiles(CullResult &r) {
    const uint32_t lane = threadIdx.x & 31u;
    uint32_t incl = r.ntiles;
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= (uint32_t)o) incl += t;
    }
    const uint32_t pre = incl - r.ntiles;
    const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
    uint32_t hits_count = 0;
    unsigned long long mask = 0ull;
    for (uint32_t base = 0; base < total; base += 32) {
        const uint32_t j = base + lane;
        uint32_t own = 0;  // largest lane whose exclusive prefix is <= j
#pragma unroll
        for (int step = 16; step > 0; step >>= 1) {
            uint32_t cand = own + step;
            uint32_t pc = __shfl_sync(0xffffffffu, pre, cand & 31u);
            if (pc <= j) own = cand;
        }
        const uint32_t local = j - __shfl_sync(0xffffffffu, pre, own);
        const float mx = __shfl_sync(0xffffffffu, r.mx, own), my = __shfl_sync(0xffffffffu, r.my, own);
        S2 conic;
        conic.c00 = __shfl_sync(0xffffffffu, r.c00, own);
        conic.c01 = __shfl_sync(0xffffffffu, r.c01, own);
        conic.c11 = __shfl_sync(0xffffffffu, r.c11, own);
        const float pt = __shfl_sync(0xffffffffu, r.pt, own);
        const uint32_t min_x = __shfl_sync(0xffffffffu, r.min_x, own), min_y = __shfl_sync(0xffffffffu, r.min_y, own);
        const uint32_t bbw = __shfl_sync(0xffffffffu, r.bbw, own);
        bool hit = false;
        if (j < total) {
            const uint32_t ry = local / bbw, rx = local - ry * bbw;
            hit = tile_hit(min_x + rx, min_y + ry, mx, my, conic, pt);
        }
        // Owners collect their results from the ballot: the tiles of lane L's splat are the list positions
        // [pre, pre + ntiles), i.e. the lanes [s, e) of this round -- no atomics, nothing leaves registers.
        const uint32_t hits = __ballot_sync(0xffffffffu, hit);
        const uint32_t lo = max(pre, base), hi = min(pre + r.ntiles, base + 32u);
        if (hi > lo) {
            const uint32_t sft = lo - base, len = hi - lo;
            const uint32_t seg = (hits >> sft) & (len >= 32u ? 0xffffffffu : ((1u << len) - 1u));
            hits_count += __popc(seg);
            const uint32_t local0 = lo - pre;  // tile index (inside the bbox) of the segment's first lane
            if (local0 < 64u) mask |= (unsigned long long)seg << local0;
        }
    }
    r.tiles = hits_count;
    r.mask = mask;
}

// Colour of one splat (+0.5, non-finite -> 0, clamped), its SH row read in 128-bit pieces where the row is 16-byte
// aligned (K = 1, 9 rows are read float by float).
template <int DEG>
__device__ __forceinline__ V3 splat_color(const float *__restrict__ sh, uint32_t gid, V3 vdir) {
    constexpr int KF = (DEG + 1) * (DEG + 1) * 3;        // floats per SH row
    float coef[KF];
    if ((KF % 4) == 0) {                                 // rows of 48 B / 192 B are 16-byte aligned
        const float4 *row4 = reinterpret_cast<const float4 *>(sh + (size_t)gid * KF);
#pragma unroll
        for (int i = 0; i < KF / 4; i++) {
            float4 q = __ldg(row4 + i);
            coef[4 * i] = q.x; coef[4 * i + 1] = q.y; coef[4 * i + 2] = q.z; coef[4 * i + 3] = q.w;
        }
    } else {
        const float *row = sh + (size_t)gid * KF;
#pragma unroll
        for (int i = 0; i < KF; i++) coef[i] = __ldg(row + i);
    }
    V3 raw = sh_to_color<DEG>([&](int i) { return coef[i]; }, vdir);
    float cr = raw.x + 0.5f, cg = raw.y + 0.5f, cb = raw.z + 0.5f;
    cr = clampf(is_finite(cr) ? cr : 0.0f, -100.0f, 100.0f);
    cg = clampf(is_finite(cg) ? cg : 0.0f, -100.0f, 100.0f);
    cb = clampf(is_finite(cb) ? cb : 0.0f, -100.0f, 100.0f);
    return mk3(cr, cg, cb);
}

// K1.  One thread per Gaussian, 256 Gaussians per tile, persistent CTAs.
// Each visible splat's finished projected row (lanes 0-12, the layout of `projected`, DESIGN §3) is written here, in
// index order, to the gid-indexed staging rows `row_by_gid`, with the tile hit mask in lanes 13-14: the SH row is then a
// streamed read, and the depth-ordered emit pass gathers one 64-byte row per splat instead of the parameter rows.
// Pinhole: 5 CTAs per SM (48 registers, no spill) as before the colour moved here -- uncapped, the SH row takes the
// kernel to 52-64 registers and 4 CTAs.  Distorted models are left to the compiler (64-80 registers, no spill): capped
// at 64 their DEG >= 3 instantiations spill.
template <bool MIP, int DEG, bool DIST>
__global__ void __launch_bounds__(PROJ_THREADS, DIST ? 0 : 5)
project_cull_kernel(const float *__restrict__ transforms, const float *__restrict__ sh,
                    const float *__restrict__ raw_opac, uint32_t n,
                    BgCamera u, uint32_t img_w, uint32_t img_h, uint32_t tiles_x, uint32_t tiles_y,
                    uint32_t *__restrict__ depth_keys, uint32_t *__restrict__ gids,
                    uint32_t *__restrict__ counts_by_gid, float *__restrict__ max_radius,
                    uint32_t *__restrict__ cgid_from_gid, float *__restrict__ row_by_gid,
                    uint32_t *__restrict__ ctl,
                    unsigned long long *__restrict__ lb_state, const uint32_t *__restrict__ epoch_base, uint32_t epoch_off) {
    // look-back epoch = (per-context call counter kept ON THE DEVICE) * 32 + launch index inside the call: nothing
    // about it is baked into the launch, so the whole forward can be captured in a CUDA graph and replayed.
    const uint32_t epoch = ((*epoch_base) * 32u + epoch_off) & 0x3FFFFFFFu;
    // [n,10] AoS rows of a tile are one contiguous 10 KB block: staged with ONE TMA bulk copy
    // (cp.async.bulk -> UBLKCP) completing on an mbarrier, double buffered so the next tile's rows land
    // while this tile is processed.
    __shared__ __align__(128) float s_rows_buf[2][PROJ_THREADS * 10];
    __shared__ __align__(8) unsigned long long s_bar[2];
    __shared__ uint32_t s_scan[33];
    __shared__ uint32_t s_tile, s_tile_next, s_prefix;
    // digit histograms of the depth keys for the four one-sweep passes that follow: counted here, where the keys
    // are produced, instead of by a separate pass over them
    __shared__ uint32_t s_dhist[4 * 256];
    const uint32_t num_tiles = (n + PROJ_THREADS - 1) / PROJ_THREADS;
    if (threadIdx.x == 0) { mbar_init(&s_bar[0], 1); mbar_init(&s_bar[1], 1); }
    for (uint32_t i = threadIdx.x; i < 4 * 256; i += PROJ_THREADS) s_dhist[i] = 0;
    __syncthreads();
    auto issue = [&](uint32_t t, uint32_t b) {  // thread 0: start the bulk copy of tile t into buffer b
        const uint32_t tb = t * PROJ_THREADS;
        const uint32_t bytes = (min((uint32_t)PROJ_THREADS, n - tb) * 40u) & ~15u;
        mbar_expect_tx(&s_bar[b], bytes);
        tma_bulk_g2s(s_rows_buf[b], transforms + (size_t)tb * 10, bytes, &s_bar[b]);
    };
    if (threadIdx.x == 0) {
        uint32_t t = atomicAdd(&ctl[CTL_TICKETS + TK_PROJECT], 1u);
        s_tile = t;
        if (t < num_tiles) issue(t, 0);
    }
    __syncthreads();
    uint32_t tile = s_tile, buf = 0, phase0 = 0, phase1 = 0;
    while (tile < num_tiles) {
        if (threadIdx.x == 0) {
            uint32_t t = atomicAdd(&ctl[CTL_TICKETS + TK_PROJECT], 1u);
            s_tile_next = t;
            if (t < num_tiles) issue(t, buf ^ 1u);
        }
        const uint32_t base = tile * PROJ_THREADS;
        const uint32_t rows = min((uint32_t)PROJ_THREADS, n - base);
        float *s_rows = s_rows_buf[buf];
        if (buf == 0) { mbar_wait(&s_bar[0], phase0); phase0 ^= 1u; } else { mbar_wait(&s_bar[1], phase1); phase1 ^= 1u; }
        if (threadIdx.x == rows - 1) {  // the bulk copy moves whole 16-byte units: an odd row count leaves 8 bytes
            const uint32_t nf = rows * 10, covered = ((rows * 40u) & ~15u) >> 2;
            for (uint32_t i = covered; i < nf; i++) s_rows[i] = __ldg(transforms + (size_t)base * 10 + i);
        }
        const uint32_t gid = base + threadIdx.x;
        CullResult r;
        r.visible = false; r.depth = 0.0f; r.tiles = 0; r.radius = 0.0f; r.mask = 0ull;
        r.mx = r.my = r.c00 = r.c01 = r.c11 = r.pt = r.opac = 0.0f;
        r.min_x = r.min_y = r.bbw = r.ntiles = 0;
        float4 *row = reinterpret_cast<float4 *>(row_by_gid + (size_t)gid * BG_PROJECTED_STRIDE);
        if (threadIdx.x < rows) {
            float t[10];
#pragma unroll
            for (int j = 0; j < 10; j++) t[j] = s_rows[threadIdx.x * 10 + j];
            r = cull_one<MIP, DIST>(t, __ldg(raw_opac + gid), u, img_w, img_h, tiles_x, tiles_y);
            max_radius[gid] = r.radius;  // zero for culled splats (render_aux.rs:76-78)
            cgid_from_gid[gid] = 0xFFFFFFFFu;  // overwritten for visible splats by project_visible_emit
            // colour and row before the tile walk, so the SH coefficients are dead while it runs
            if (r.visible) {
                const V3 vdir = normalize(sub(mk3(t[0], t[1], t[2]), mk3(u.cam_pos[0], u.cam_pos[1], u.cam_pos[2])));
                const V3 col = splat_color<DEG>(sh, gid, vdir);
                const float L2E = 1.4426950408889634f;
                row[0] = make_float4(r.mx, r.my, r.c00, r.c01);
                row[1] = make_float4(r.c11, r.opac, col.x, col.y);
                row[2] = make_float4(col.z, (0.5f * L2E) * r.c11, (0.5f * L2E) * r.c00, L2E * r.c01);
            }
        }
        // The visible count is known before the (expensive) tile walk: publish the tile aggregate
        // first, count tiles, and only then look back -- by then the predecessors have published,
        // so the chained scan adds no stall.
        uint32_t total;
        uint32_t local = block_exclusive_scan(r.visible ? 1u : 0u, s_scan, &total);
        unsigned long long *st = lb_state + tile;
        if (threadIdx.x == 0) lb_store(st, epoch, tile == 0 ? LB_INCLUSIVE : LB_AGGREGATE, total);
        warp_count_tiles(r);
        if (threadIdx.x < 32) {
            uint32_t prefix = (tile == 0) ? 0u : lb_lookback_warp(lb_state, tile, epoch);
            if (threadIdx.x == 0) {
                if (tile != 0) lb_store(st, epoch, LB_INCLUSIVE, prefix + total);
                s_prefix = prefix;
                if (tile == num_tiles - 1) ctl[CTL_COUNTERS + 0] = prefix + total;  // num_visible
            }
        }
        __syncthreads();
        if (r.visible) {
            uint32_t slot = s_prefix + local;
            const uint32_t dk = __float_as_uint(r.depth);  // z >= 0.01: float order == uint order
            depth_keys[slot] = dk;
#pragma unroll
            for (int p = 0; p < 4; p++) atomicAdd(&s_dhist[p * 256 + ((dk >> (8 * p)) & 255u)], 1u);
            gids[slot] = gid;
            counts_by_gid[gid] = r.tiles;
            row[3] = make_float4(r.pt, __uint_as_float((uint32_t)r.mask), __uint_as_float((uint32_t)(r.mask >> 32)), 0.0f);
        }
        tile = s_tile_next;
        buf ^= 1u;
        __syncthreads();  // everyone has read s_tile_next / s_prefix / this buffer before they are reused
    }
    uint32_t *hist = ctl + CTL_HIST_DEPTH;
    for (uint32_t i = threadIdx.x; i < 4 * 256; i += PROJ_THREADS) {
        const uint32_t c = s_dhist[i];
        if (c) atomicAdd(&hist[i], c);
    }
}

// int_gather(counts, sorted gid) fused with the inclusive prefix sum over the visible Gaussians.
// Single pass, decoupled look-back, 8 items per thread.  Writes cum[i] (inclusive) and
// num_intersections = cum[V-1] (clamped against the arena capacity, overflow flag set).
constexpr int SCAN_THREADS = 256, SCAN_ITEMS = 8, SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

__global__ void __launch_bounds__(SCAN_THREADS)
gather_scan_kernel(const uint32_t *__restrict__ in, const uint32_t *__restrict__ gather_idx /* nullable */,
                   uint32_t n_host, const uint32_t *__restrict__ n_dev, uint32_t *__restrict__ out,
                   uint32_t *__restrict__ total_out /* nullable */, uint32_t capacity,
                   uint32_t *__restrict__ overflow_flag /* nullable */, uint32_t *__restrict__ ticket,
                   unsigned long long *__restrict__ lb_state, const uint32_t *__restrict__ epoch_base, uint32_t epoch_off) {
    // look-back epoch = (per-context call counter kept ON THE DEVICE) * 32 + launch index inside the call: nothing
    // about it is baked into the launch, so the whole forward can be captured in a CUDA graph and replayed.
    const uint32_t epoch = ((*epoch_base) * 32u + epoch_off) & 0x3FFFFFFFu;
    __shared__ uint32_t s_scan[33];
    __shared__ uint32_t s_tile, s_prefix;
    const uint32_t n = n_dev ? min(*n_dev, n_host) : n_host;
    const uint32_t num_tiles = (n + SCAN_TILE - 1) / SCAN_TILE;
    if (num_tiles == 0) {
        if (blockIdx.x == 0 && threadIdx.x == 0 && total_out) *total_out = 0;
        return;
    }
    while (true) {
        if (threadIdx.x == 0) s_tile = atomicAdd(ticket, 1u);
        __syncthreads();
        const uint32_t tile = s_tile;
        if (tile >= num_tiles) break;
        const uint32_t base = tile * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
        uint32_t v[SCAN_ITEMS];
        uint32_t sum = 0;
#pragma unroll
        for (int i = 0; i < SCAN_ITEMS; i++) {
            uint32_t idx = base + i;
            uint32_t x = 0;
            if (idx < n) x = gather_idx ? __ldg(in + __ldg(gather_idx + idx)) : __ldg(in + idx);
            sum += x;
            v[i] = sum;  // thread-local inclusive
        }
        uint32_t total;
        uint32_t excl = block_exclusive_scan(sum, s_scan, &total);
        if (threadIdx.x < 32) {
            unsigned long long *st = lb_state + tile;
            if (threadIdx.x == 0) lb_store(st, epoch, tile == 0 ? LB_INCLUSIVE : LB_AGGREGATE, total);
            uint32_t prefix = (tile == 0) ? 0u : lb_lookback_warp(lb_state, tile, epoch);
            if (threadIdx.x == 0) {
                if (tile != 0) lb_store(st, epoch, LB_INCLUSIVE, prefix + total);
                s_prefix = prefix;
                if (tile == num_tiles - 1 && total_out) {
                    uint32_t tot = prefix + total;
                    if (tot > capacity) {
                        if (overflow_flag) *overflow_flag = tot;
                        tot = capacity;
                    }
                    *total_out = tot;
                }
            }
        }
        __syncthreads();
        const uint32_t off = s_prefix + excl;
#pragma unroll
        for (int i = 0; i < SCAN_ITEMS; i++) {
            uint32_t idx = base + i;
            if (idx < n) out[idx] = off + v[i];
        }
        __syncthreads();
    }
}

// K2 + K3.  One thread per visible Gaussian in depth order (compact gid = position in the
// depth-sorted list); WARPS are the unit of work (a ticket = 32 consecutive compact ids), so the loop has no
// block barrier.  Every lane gathers the 64-byte staged row `project_cull_kernel` wrote for its splat (the gather is
// by sorted global id, so neighbouring lanes touch unrelated rows anyway) as four 128-bit loads, copies lanes 0-12 to
// `projected[cgid]` and emits the splat's intersections; the bbox is recomputed from the row (the same inputs and
// functions as the cull), the small-bbox hits come from the mask in lanes 13-14.
// The kernel is bound by gather latency (long-scoreboard stalls on the first use of the row), hence:
//   * the NEXT ticket and its global ids are fetched at the top of an iteration, and the rows they point at are
//     pulled into L2 with cp.async.bulk.prefetch.L2 while the current splats are processed;
//   * the (tile id, compact gid) pairs of a warp -- one contiguous output range -- are gathered in shared memory
//     and written with coalesced stores; bboxes larger than the 64-bit hit mask are tested by the whole warp.
// Residency: the 22.5 KB of emission staging per 128-thread CTA allow 9 CTAs per SM; __launch_bounds__(128, 8) caps the
// kernel at 64 registers (it uses 63, no spill), and the grid is 8 CTAs per SM (api.cu).  Measured on an H100 (400 W
// limit), 1M splats at 1080p: 169 us, against 354 us for the former gather-and-recompute kernel at 6 CTAs per SM
// (DESIGN §6.8).
constexpr int VIS_THREADS = 128;

__device__ __forceinline__ void prefetch_l2_bulk(const void *p, uint32_t bytes) {  // p 16-byte aligned, bytes % 16 == 0
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}

__global__ void __launch_bounds__(VIS_THREADS, 8)
project_visible_emit_kernel(const float *__restrict__ row_by_gid, const uint32_t *__restrict__ gid_sorted,
                            const uint32_t *__restrict__ cum, uint32_t tiles_x, uint32_t tiles_y,
                            float *__restrict__ projected, uint32_t *__restrict__ tile_keys,
                            uint32_t *__restrict__ isect_vals, uint32_t isect_capacity,
                            uint32_t *__restrict__ cgid_from_gid, uint32_t *__restrict__ ctl, uint32_t tile_bits) {
    constexpr uint32_t EMIT_BUF = 1024;                  // staged (tile id, owner) pairs per warp
    __shared__ uint32_t s_emit_keys[(VIS_THREADS / 32) * EMIT_BUF];
    __shared__ uint8_t s_emit_own[(VIS_THREADS / 32) * EMIT_BUF];
    // digit histograms of the emitted tile keys for the one-sweep passes of the tile sort (<= 2 passes: < 65536 tiles)
    __shared__ uint32_t s_thist[2 * 256];
    const uint32_t hist_passes = (tile_bits <= 16u) ? (tile_bits + 7u) / 8u : 0u;   // else the sort counts itself
    const uint32_t hi_mask = (tile_bits > 8u) ? ((1u << min(8u, tile_bits - 8u)) - 1u) : 0u;
    const uint32_t lo_mask = (1u << min(8u, tile_bits)) - 1u;
    for (uint32_t i = threadIdx.x; i < 2 * 256; i += VIS_THREADS) s_thist[i] = 0;
    __syncthreads();
    auto count_key = [&](uint32_t key) {
        if (hist_passes > 0) atomicAdd(&s_thist[key & lo_mask], 1u);
        if (hist_passes > 1) atomicAdd(&s_thist[256 + ((key >> 8) & hi_mask)], 1u);
    };
    const uint32_t nvis = ctl[CTL_COUNTERS + 0];
    const uint32_t num_tickets = (nvis + 31u) / 32u;
    const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
    const uint32_t lt_mask = (1u << lane) - 1u;
    uint32_t *wkeys = s_emit_keys + wid * EMIT_BUF;
    uint8_t *wown = s_emit_own + wid * EMIT_BUF;
    auto take_ticket = [&]() {
        uint32_t t = 0;
        if (lane == 0) t = atomicAdd(&ctl[CTL_TICKETS + TK_VISIBLE], 1u);
        return __shfl_sync(0xffffffffu, t, 0);
    };
    uint32_t ticket = take_ticket();
    uint32_t gid = 0;
    if (ticket < num_tickets && ticket * 32u + lane < nvis) gid = __ldg(gid_sorted + ticket * 32u + lane);
    while (ticket < num_tickets) {
        const uint32_t cgid = ticket * 32u + lane;
        const bool active = cgid < nvis;
        // next ticket: its ids are on their way while this ticket's rows are gathered
        const uint32_t ticket_next = take_ticket();
        const bool next_active = ticket_next < num_tickets && ticket_next * 32u + lane < nvis;
        uint32_t gid_next = 0;
        if (next_active) gid_next = __ldg(gid_sorted + ticket_next * 32u + lane);

        TileBox bb;
        bb.min_x = bb.min_y = bb.max_x = bb.max_y = 0;
        uint32_t base = 0, budget = 0;
        unsigned long long hitm = 0ull;
        float e_mx = 0.f, e_my = 0.f, e_pt = 0.f;
        S2 e_conic; e_conic.c00 = e_conic.c01 = e_conic.c11 = 0.f;
        if (active) {
            const float4 *src = reinterpret_cast<const float4 *>(row_by_gid + (size_t)gid * BG_PROJECTED_STRIDE);
            const float4 q0 = __ldg(src), q1 = __ldg(src + 1), q2 = __ldg(src + 2), q3 = __ldg(src + 3);
            base = (cgid == 0) ? 0u : __ldg(cum + cgid - 1);
            budget = __ldg(cum + cgid) - base;
            float4 *dst = reinterpret_cast<float4 *>(projected + (size_t)cgid * BG_PROJECTED_STRIDE);
            dst[0] = q0;
            dst[1] = q1;
            dst[2] = q2;
            dst[3] = make_float4(q3.x, 0.0f, 0.0f, 0.0f);
            cgid_from_gid[gid] = cgid;
            hitm = (unsigned long long)__float_as_uint(q3.y) | ((unsigned long long)__float_as_uint(q3.z) << 32);
            // ---- (tile id, compact gid) pairs (map_gaussians.rs:26-79)
            e_mx = q0.x; e_my = q0.y; e_conic.c00 = q0.z; e_conic.c01 = q0.w; e_conic.c11 = q1.x; e_pt = q3.x;
            float ex, ey;
            bbox_extent(e_conic, e_pt, ex, ey);
            bb = tile_bbox(e_mx, e_my, ex, ey, tiles_x, tiles_y);
        }
        // pull the next ticket's rows towards L2 (the ids have arrived by now)
        if (next_active) prefetch_l2_bulk(row_by_gid + (size_t)gid_next * BG_PROJECTED_STRIDE, BG_PROJECTED_STRIDE * 4);
        // The output slots of a warp's 32 splats are one contiguous range [base(lane 0), end(last active lane)).
        const uint32_t warp_base = __shfl_sync(0xffffffffu, base, 0);
        uint32_t end_here = active ? base + budget : 0u;
        for (int o = 16; o > 0; o >>= 1) end_here = max(end_here, __shfl_xor_sync(0xffffffffu, end_here, o));
        const uint32_t warp_total = end_here - warp_base;
        const bool staged = warp_total <= EMIT_BUF;
        const uint32_t off = base - warp_base;
        const uint32_t bbw = bb.max_x - bb.min_x, bbh = bb.max_y - bb.min_y;
        const bool big = active && bbw * bbh > 64u;
        auto put = [&](uint32_t slot_off, uint32_t slot_base, uint32_t owner_lane, uint32_t h, uint32_t key) {
            if (staged) { wkeys[slot_off + h] = key; wown[slot_off + h] = (uint8_t)owner_lane; }
            else {
                uint32_t o = slot_base + h;
                if (o < isect_capacity) { tile_keys[o] = key; isect_vals[o] = ticket * 32u + owner_lane; count_key(key); }
            }
        };
        if (active && !big) {
            // the counting pass left the hit bits of this bbox: no tile test is repeated here
            uint32_t hits = 0;
            unsigned long long m = hitm;
            const unsigned long long row_mask = (bbw >= 64u) ? ~0ull : ((1ull << bbw) - 1ull);
            uint32_t row_key = bb.min_x + bb.min_y * tiles_x;
            for (uint32_t ry = 0; ry < bbh && hits < budget; ry++, m = (bbw >= 64u) ? 0ull : (m >> bbw), row_key += tiles_x) {
                unsigned long long rb = m & row_mask;
                while (rb && hits < budget) {
                    uint32_t rx = (uint32_t)__ffsll((long long)rb) - 1u;
                    rb &= rb - 1ull;
                    put(off, base, lane, hits, row_key + rx);
                    hits++;
                }
            }
            // same hits as the counting pass => hits == budget; keep the reference's padding so that no slot is
            // ever left unwritten.
            for (uint32_t pad = hits; pad < budget; pad++) put(off, base, lane, pad, tiles_x * tiles_y);
        }
        // bboxes beyond the 64-bit mask (0.3 % of the splats of the 1M/1080p scene, 75+ tiles each): the whole
        // warp tests 32 tiles of one such splat at a time instead of one lane walking them alone.
        uint32_t bigs = __ballot_sync(0xffffffffu, big);
        while (bigs) {
            const uint32_t L = (uint32_t)__ffs(bigs) - 1u;
            bigs &= bigs - 1u;
            const float mx = __shfl_sync(0xffffffffu, e_mx, L), my = __shfl_sync(0xffffffffu, e_my, L);
            S2 conic;
            conic.c00 = __shfl_sync(0xffffffffu, e_conic.c00, L);
            conic.c01 = __shfl_sync(0xffffffffu, e_conic.c01, L);
            conic.c11 = __shfl_sync(0xffffffffu, e_conic.c11, L);
            const float pt = __shfl_sync(0xffffffffu, e_pt, L);
            const uint32_t min_x = __shfl_sync(0xffffffffu, bb.min_x, L), min_y = __shfl_sync(0xffffffffu, bb.min_y, L);
            const uint32_t w_ = __shfl_sync(0xffffffffu, bbw, L), h_ = __shfl_sync(0xffffffffu, bbh, L);
            const uint32_t off_l = __shfl_sync(0xffffffffu, off, L), base_l = __shfl_sync(0xffffffffu, base, L);
            const uint32_t budget_l = __shfl_sync(0xffffffffu, budget, L);
            const uint32_t ntile = w_ * h_;
            uint32_t cnt = 0;
            for (uint32_t j0 = 0; j0 < ntile; j0 += 32) {
                const uint32_t j = j0 + lane;
                bool hit = false;
                uint32_t key = 0;
                if (j < ntile) {
                    const uint32_t ry = j / w_, rx = j - ry * w_;
                    hit = tile_hit(min_x + rx, min_y + ry, mx, my, conic, pt);
                    key = (min_x + rx) + (min_y + ry) * tiles_x;
                }
                const uint32_t hb = __ballot_sync(0xffffffffu, hit);
                const uint32_t pos = cnt + __popc(hb & lt_mask);
                if (hit && pos < budget_l) put(off_l, base_l, L, pos, key);
                cnt += __popc(hb);
            }
            for (uint32_t pad = min(cnt, budget_l) + lane; pad < budget_l; pad += 32) put(off_l, base_l, L, pad, tiles_x * tiles_y);
        }
        __syncwarp();
        if (staged) {
            for (uint32_t j = lane; j < warp_total; j += 32) {
                const uint32_t o = warp_base + j;
                if (o < isect_capacity) {
                    const uint32_t key = wkeys[j];
                    tile_keys[o] = key;
                    isect_vals[o] = ticket * 32u + wown[j];
                    count_key(key);
                }
            }
        }
        __syncwarp();
        ticket = ticket_next;
        gid = gid_next;
    }
    __syncthreads();
    uint32_t *hist = ctl + CTL_HIST_TILE;
    for (uint32_t i = threadIdx.x; i < hist_passes * 256; i += VIS_THREADS) {
        const uint32_t c = s_thist[i];
        if (c) atomicAdd(&hist[i], c);
    }
}

// K4.  tile_offsets must be zeroed by the caller (render.rs:232-236).
__device__ __forceinline__ void tile_boundary(uint32_t i, uint32_t tid, uint32_t prev, uint32_t n, uint32_t num_tiles,
                                              uint32_t *__restrict__ tile_offsets) {
    if (tid >= num_tiles) return;
    if (i == n - 1) tile_offsets[tid * 2 + 1] = i + 1;
    if (i == 0) {
        tile_offsets[tid * 2] = 0;
    } else if (tid != prev) {
        if (prev < num_tiles) tile_offsets[prev * 2 + 1] = i;
        tile_offsets[tid * 2] = i;
    }
}

// Four sorted ids per thread (one 128-bit load + the predecessor word): the kernel is a pure stream with a rare
// scattered store, so the only thing that matters is keeping enough loads in flight.
__global__ void __launch_bounds__(256)
tile_offsets_kernel(const uint32_t *__restrict__ tile_ids, const uint32_t *__restrict__ ctl, uint32_t num_tiles,
                    uint32_t *__restrict__ tile_offsets) {
    const uint32_t n = ctl[CTL_COUNTERS + 1];
    const uint32_t groups = (n + 3u) / 4u;
    for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += gridDim.x * blockDim.x) {
        const uint32_t i0 = g * 4u;
        uint32_t v[4];
        if (i0 + 4u <= n) {
            const uint4 q = __ldg(reinterpret_cast<const uint4 *>(tile_ids) + g);
            v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
        } else {
#pragma unroll
            for (int e = 0; e < 4; e++) v[e] = (i0 + e < n) ? __ldg(tile_ids + i0 + e) : 0xFFFFFFFFu;
        }
        uint32_t prev = (i0 == 0) ? 0xFFFFFFFFu : __ldg(tile_ids + i0 - 1);
#pragma unroll
        for (int e = 0; e < 4; e++) {
            if (i0 + e < n) tile_boundary(i0 + e, v[e], prev, n, num_tiles, tile_offsets);
            prev = v[e];
        }
    }
}

// ---- host launchers (called from api.cu) ----
template <bool MIP>
static cudaError_t launch_cull_deg(cudaStream_t s, int grid, int deg, const float *transforms, const float *sh,
                                   const float *raw_opac, uint32_t n, const BgCamera &u, uint32_t w, uint32_t h,
                                   uint32_t tx, uint32_t ty, uint32_t *depth_keys, uint32_t *gids, uint32_t *counts,
                                   float *max_radius, uint32_t *cgid_from_gid, float *row_by_gid, uint32_t *ctl,
                                   unsigned long long *lb, const uint32_t *epoch_base, uint32_t epoch_off) {
    const bool dist = u.camera_model != BG_CAMERA_PINHOLE;
#define BG_LAUNCH_CULL(D)                                                                                                  \
    if (dist) project_cull_kernel<MIP, D, true><<<grid, PROJ_THREADS, 0, s>>>(transforms, sh, raw_opac, n, u, w, h, tx, ty, \
                                       depth_keys, gids, counts, max_radius, cgid_from_gid, row_by_gid, ctl, lb, epoch_base, epoch_off); \
    else project_cull_kernel<MIP, D, false><<<grid, PROJ_THREADS, 0, s>>>(transforms, sh, raw_opac, n, u, w, h, tx, ty,      \
                                       depth_keys, gids, counts, max_radius, cgid_from_gid, row_by_gid, ctl, lb, epoch_base, epoch_off)
    switch (deg) {
        case 0: BG_LAUNCH_CULL(0); break;
        case 1: BG_LAUNCH_CULL(1); break;
        case 2: BG_LAUNCH_CULL(2); break;
        case 3: BG_LAUNCH_CULL(3); break;
        case 4: BG_LAUNCH_CULL(4); break;
        default: return cudaErrorInvalidValue;
    }
#undef BG_LAUNCH_CULL
    return cudaGetLastError();
}

cudaError_t launch_project_cull(cudaStream_t s, int grid, bool mip, int deg, const float *transforms, const float *sh,
                                const float *raw_opac, uint32_t n, const BgCamera &u, uint32_t w, uint32_t h,
                                uint32_t tx, uint32_t ty, uint32_t *depth_keys, uint32_t *gids, uint32_t *counts,
                                float *max_radius, uint32_t *cgid_from_gid, float *row_by_gid, uint32_t *ctl,
                                unsigned long long *lb, const uint32_t *epoch_base, uint32_t epoch_off) {
    if (n == 0) return cudaSuccess;
    return mip ? launch_cull_deg<true>(s, grid, deg, transforms, sh, raw_opac, n, u, w, h, tx, ty, depth_keys, gids,
                                       counts, max_radius, cgid_from_gid, row_by_gid, ctl, lb, epoch_base, epoch_off)
               : launch_cull_deg<false>(s, grid, deg, transforms, sh, raw_opac, n, u, w, h, tx, ty, depth_keys, gids,
                                        counts, max_radius, cgid_from_gid, row_by_gid, ctl, lb, epoch_base, epoch_off);
}

cudaError_t launch_gather_scan(cudaStream_t s, int grid, const uint32_t *in, const uint32_t *gather_idx,
                               uint32_t n_host, const uint32_t *n_dev, uint32_t *out, uint32_t *total_out,
                               uint32_t capacity, uint32_t *overflow_flag, uint32_t *ticket,
                               unsigned long long *lb, const uint32_t *epoch_base, uint32_t epoch_off) {
    if (n_host == 0) return cudaSuccess;
    gather_scan_kernel<<<grid, SCAN_THREADS, 0, s>>>(in, gather_idx, n_host, n_dev, out, total_out, capacity,
                                                     overflow_flag, ticket, lb, epoch_base, epoch_off);
    return cudaGetLastError();
}

cudaError_t launch_project_visible_emit(cudaStream_t s, int grid, const float *row_by_gid, const uint32_t *gid_sorted,
                                        const uint32_t *cum, uint32_t tx, uint32_t ty, float *projected,
                                        uint32_t *tile_keys, uint32_t *isect_vals, uint32_t cap,
                                        uint32_t *cgid_from_gid, uint32_t *ctl, uint32_t tile_bits) {
    project_visible_emit_kernel<<<grid, VIS_THREADS, 0, s>>>(row_by_gid, gid_sorted, cum, tx, ty, projected, tile_keys,
                                                             isect_vals, cap, cgid_from_gid, ctl, tile_bits);
    return cudaGetLastError();
}

cudaError_t launch_tile_offsets(cudaStream_t s, int grid, const uint32_t *tile_ids, const uint32_t *ctl,
                                uint32_t num_tiles, uint32_t *tile_offsets) {
    tile_offsets_kernel<<<grid, 256, 0, s>>>(tile_ids, ctl, num_tiles, tile_offsets);
    return cudaGetLastError();
}

}  // namespace bg
