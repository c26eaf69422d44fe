// sort.cu -- one-sweep LSD radix sort of (u32 key, u32 value) pairs, 8-bit digits.
//
// Replaces brush_sort::radix_argsort (brush-sort/src/lib.rs:16-125; kernels.rs:28-443), which runs
// 5 dispatches per 4-bit digit (count, reduce, scan, scan_add, scatter): 40 dispatches for the
// 32-bit depth sort and 20 for a 13-bit tile sort.  Here: digit histograms for all passes up front (one
// kernel for bg_radix_argsort_u32; inside a render the kernels that PRODUCE the keys count them, so no
// histogram pass exists), then one kernel per 8-bit digit that reads every key once and writes it once
// (chained scan with a two-level decoupled look-back): 4 launches for 32 bits, 2 for 13..16 bits.
//
// Result spec (the reference's tests, brush-sort/src/lib.rs:147-151): equal to a stable argsort on
// the low `bits` bits.  Stability comes from (a) ranking keys inside a warp in lane order (peer
// groups from per-bit ballots), (b) warps and tiles being ordered by the look-back chain.
//
// The element count may live on the device (n_dev): CTAs are persistent and pull tiles from a
// ticket, so no host readback is needed to size the grid.
#include "bg_common.cuh"
#include "bg_launch.cuh"

namespace bg {

constexpr int SORT_THREADS = 256;
constexpr int SORT_ITEMS = 16;
constexpr int SORT_TILE = SORT_THREADS * SORT_ITEMS;  // 4096 keys per tile
// Small sorts (the depth sort of ~1M visible Gaussians) run with half-size tiles: 4096-key tiles give such a sort fewer
// CTAs than the GPU holds (1.5 per SM at 1M keys), and a pass is then one latency-bound wave.
constexpr int SORT_ITEMS_SMALL = 8;
constexpr uint32_t SORT_SMALL_MAX_KEYS = 3u << 20;
constexpr int RADIX = 256;

// hist[p*256 + d] += #keys whose p-th digit is d, for p < passes.
__global__ void __launch_bounds__(SORT_THREADS)
radix_hist_kernel(const uint32_t *__restrict__ keys, uint32_t n_host, const uint32_t *__restrict__ n_dev,
                  uint32_t bits, uint32_t passes, uint32_t *__restrict__ hist) {
    __shared__ uint32_t s_hist[4 * RADIX];
    const uint32_t n = n_dev ? min(*n_dev, n_host) : n_host;
    for (uint32_t i = threadIdx.x; i < passes * RADIX; i += SORT_THREADS) s_hist[i] = 0;
    __syncthreads();
    // Pure stream + shared-memory atomics: four keys per 128-bit load keep enough loads in flight.
    // (Aggregating runs of equal digits with shuffles/ballots before the atomic measured SLOWER.)
    const uint32_t stride = gridDim.x * SORT_THREADS;
    const uint32_t tid = blockIdx.x * SORT_THREADS + threadIdx.x;
    auto add_key = [&](uint32_t k) {
        for (uint32_t p = 0; p < passes; p++) {
            uint32_t shift = p * 8, width = min(8u, bits - shift);
            atomicAdd(&s_hist[p * RADIX + ((k >> shift) & ((1u << width) - 1u))], 1u);
        }
    };
    if ((reinterpret_cast<uintptr_t>(keys) & 15u) == 0) {
        const uint32_t groups = n / 4u;
        for (uint32_t g = tid; g < groups; g += stride) {
            const uint4 q = __ldg(reinterpret_cast<const uint4 *>(keys) + g);
            add_key(q.x); add_key(q.y); add_key(q.z); add_key(q.w);
        }
        for (uint32_t i = groups * 4u + tid; i < n; i += stride) add_key(__ldg(keys + i));
    } else {
        for (uint32_t i = tid; i < n; i += stride) add_key(__ldg(keys + i));
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < passes * RADIX; i += SORT_THREADS) {
        uint32_t c = s_hist[i];
        if (c) atomicAdd(&hist[i], c);
    }
}

// One digit pass.  lb_state: [num_tiles][256] tile counts, lb_group: [ceil(num_tiles/16)][256] group totals.
template <int SORT_ITEMS>
__global__ void __launch_bounds__(SORT_THREADS, 3)
onesweep_pass_kernel(const uint32_t *__restrict__ keys_in, const uint32_t *__restrict__ vals_in,
                     uint32_t *__restrict__ keys_out, uint32_t *__restrict__ vals_out, uint32_t n_host,
                     const uint32_t *__restrict__ n_dev, uint32_t shift, uint32_t width,
                     const uint32_t *__restrict__ hist /* this pass: [256] */, uint32_t *__restrict__ ticket,
                     unsigned long long *__restrict__ lb_state, unsigned long long *__restrict__ lb_group,
                     const uint32_t *__restrict__ epoch_base, uint32_t epoch_off) {
    // look-back epoch = (per-context call counter kept ON THE DEVICE) * 32 + launch index inside the call: nothing
    // about it is baked into the launch, so the whole forward can be captured in a CUDA graph and replayed.
    const uint32_t epoch = ((*epoch_base) * 32u + epoch_off) & 0x3FFFFFFFu;
    constexpr uint32_t SORT_TILE = SORT_THREADS * SORT_ITEMS;
    __shared__ uint32_t s_keys[SORT_TILE];
    __shared__ uint32_t s_vals[SORT_TILE];
    __shared__ uint32_t s_warp_hist[(SORT_THREADS / 32) * RADIX];
    __shared__ uint32_t s_bin_start[RADIX];    // exclusive scan of the tile's digit counts
    __shared__ int64_t s_bin_dst[RADIX];       // global destination of tile-local position 0 of each bin
    __shared__ uint32_t s_digit_base[RADIX];   // exclusive scan of the global histogram
    __shared__ uint32_t s_scan[33];
    __shared__ uint32_t s_tile;
    const uint32_t n = n_dev ? min(*n_dev, n_host) : n_host;
    const uint32_t num_tiles = (n + SORT_TILE - 1) / SORT_TILE;
    const uint32_t mask = (1u << width) - 1u;
    const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
    const uint32_t lt_mask = (1u << lane) - 1u;
    if (num_tiles == 0) return;
    {   // exclusive scan of the global digit histogram (thread d owns digit d)
        uint32_t total;
        uint32_t c = __ldg(hist + threadIdx.x);
        uint32_t e = block_exclusive_scan(c, s_scan, &total);
        s_digit_base[threadIdx.x] = e;
    }
    __syncthreads();
    while (true) {
        if (threadIdx.x == 0) s_tile = atomicAdd(ticket, 1u);
        __syncthreads();
        const uint32_t tile = s_tile;
        if (tile >= num_tiles) break;
        const uint32_t tile_base = tile * SORT_TILE;
        const uint32_t tile_count = min((uint32_t)SORT_TILE, n - tile_base);
        for (uint32_t i = threadIdx.x; i < (SORT_THREADS / 32) * RADIX; i += SORT_THREADS) s_warp_hist[i] = 0;
        __syncthreads();
        // ---- load (warp-striped: warp w owns SORT_ITEMS*32 consecutive keys) and rank
        uint32_t key[SORT_ITEMS], val[SORT_ITEMS];
        uint16_t rank[SORT_ITEMS];
        const uint32_t warp_base = tile_base + wid * (SORT_ITEMS * 32);
        uint32_t *wh = s_warp_hist + wid * RADIX;
#pragma unroll
        for (int i = 0; i < SORT_ITEMS; i++) {
            uint32_t idx = warp_base + i * 32 + lane;
            bool valid = idx < n;
            key[i] = valid ? __ldg(keys_in + idx) : 0xFFFFFFFFu;
            val[i] = valid ? __ldg(vals_in + idx) : 0u;
        }
#pragma unroll
        for (int i = 0; i < SORT_ITEMS; i++) {
            // out-of-range keys are all-ones: they rank after every real key of the last digit
            // in this (final, partial) tile and are dropped at scatter time.
            // Ranking: lanes holding the same digit form a peer group (per-bit ballots); the group's lowest
            // lane bumps the warp's digit counter with ONE shared-memory atomic and broadcasts the old
            // value.  Atomics of one warp to one address retire in issue order, so item i sees exactly
            // the items before it; there is no load->store->barrier chain between the 16 items.
            uint32_t d = (key[i] >> shift) & mask;
            // peers = lanes with the same digit.  `width` ballots + masks give the same set as MATCH.ANY
            // without its shared, low-throughput unit.
            uint32_t peers = 0xffffffffu;
            for (uint32_t bit = 0; bit < width; bit++) {
                const uint32_t vote = __ballot_sync(0xffffffffu, (d >> bit) & 1u);
                peers &= ((d >> bit) & 1u) ? vote : ~vote;
            }
            uint32_t leader = (uint32_t)__ffs(peers) - 1u;
            uint32_t pre = 0;
            if (lane == leader) pre = atomicAdd(&wh[d], (uint32_t)__popc(peers));
            pre = __shfl_sync(0xffffffffu, pre, leader);
            rank[i] = (uint16_t)(pre + __popc(peers & lt_mask));
        }
        __syncthreads();
        // ---- per digit: exclusive scan over warps, tile count
        uint32_t my_count;
        {
            uint32_t d = threadIdx.x, sum = 0;
#pragma unroll
            for (int w = 0; w < SORT_THREADS / 32; w++) {
                uint32_t c = s_warp_hist[w * RADIX + d];
                s_warp_hist[w * RADIX + d] = sum;
                sum += c;
            }
            my_count = sum;
        }
        // ---- publish the aggregate (thread d serves digit d), then reorder the tile in shared memory;
        // only after that look back.  Two-level decoupled look-back: tile words only ever hold the tile's own
        // count; a tile sums the counts of the earlier tiles of its group of LB_GROUP (one batch of independent
        // loads), the group's last tile publishes the group total, and the group totals are chained with the
        // usual aggregate -> inclusive protocol.  A 1M-key sort runs all its ~230 tiles at once: with a flat chain
        // the last tile walked ~230 predecessors, 16 per L2 round trip; now any tile needs about three round trips.
        constexpr uint32_t LB_GROUP = 16;
        const uint32_t grp = tile / LB_GROUP, r = tile % LB_GROUP;
        unsigned long long *st = lb_state + (size_t)tile * RADIX + threadIdx.x;
        lb_store(st, epoch, LB_AGGREGATE, my_count);
        uint32_t bin_total;
        uint32_t bin_start = block_exclusive_scan(my_count, s_scan, &bin_total);
        s_bin_start[threadIdx.x] = bin_start;
        __syncthreads();
#pragma unroll
        for (int i = 0; i < SORT_ITEMS; i++) {
            uint32_t d = (key[i] >> shift) & mask;
            uint32_t pos = s_bin_start[d] + s_warp_hist[wid * RADIX + d] + rank[i];
            s_keys[pos] = key[i];
            s_vals[pos] = val[i];
        }
        uint32_t in_group = 0;
        {
            unsigned long long w[LB_GROUP - 1];
#pragma unroll
            for (uint32_t q = 0; q < LB_GROUP - 1; q++)
                w[q] = (q < r) ? lb_load(lb_state + (size_t)(tile - 1u - q) * RADIX + threadIdx.x) : 0ull;
#pragma unroll
            for (uint32_t q = 0; q < LB_GROUP - 1; q++) {
                if (q < r) {
                    while (lb_status(w[q], epoch) == LB_INVALID)
                        w[q] = lb_load(lb_state + (size_t)(tile - 1u - q) * RADIX + threadIdx.x);
                    in_group += lb_value(w[q]);
                }
            }
        }
        const bool closes_group = (r == LB_GROUP - 1u) || (tile == num_tiles - 1u);
        const uint32_t group_total = in_group + my_count;
        unsigned long long *gst = lb_group + (size_t)grp * RADIX + threadIdx.x;
        if (closes_group) lb_store(gst, epoch, grp == 0 ? LB_INCLUSIVE : LB_AGGREGATE, group_total);
        uint32_t gprefix = 0;
        if (grp != 0) {
            constexpr int LB_BATCH = 16;
            int64_t t = (int64_t)grp - 1;
            bool done_lb = false;
            while (!done_lb) {
                unsigned long long w[LB_BATCH];
#pragma unroll
                for (int q = 0; q < LB_BATCH; q++) {
                    int64_t tt = t - q;
                    w[q] = (tt >= 0) ? lb_load(lb_group + (size_t)tt * RADIX + threadIdx.x) : 0ull;
                }
#pragma unroll
                for (int q = 0; q < LB_BATCH; q++) {
                    if (done_lb) break;
                    int64_t tt = t - q;
                    if (tt < 0) { done_lb = true; break; }
                    uint32_t stt = lb_status(w[q], epoch);
                    while (stt == LB_INVALID) {  // not published yet: wait on this one word
                        w[q] = lb_load(lb_group + (size_t)tt * RADIX + threadIdx.x);
                        stt = lb_status(w[q], epoch);
                    }
                    gprefix += lb_value(w[q]);
                    if (stt == LB_INCLUSIVE) done_lb = true;
                }
                t -= LB_BATCH;
            }
            if (closes_group) lb_store(gst, epoch, LB_INCLUSIVE, gprefix + group_total);
        }
        const uint32_t prefix = gprefix + in_group;
        s_bin_dst[threadIdx.x] = (int64_t)s_digit_base[threadIdx.x] + (int64_t)prefix - (int64_t)bin_start;
        __syncthreads();
        // ---- coalesced scatter: consecutive positions of one bin go to consecutive addresses
        for (uint32_t j = threadIdx.x; j < tile_count; j += SORT_THREADS) {
            uint32_t k = s_keys[j];
            uint32_t d = (k >> shift) & mask;
            int64_t dst = s_bin_dst[d] + (int64_t)j;
            keys_out[dst] = k;
            vals_out[dst] = s_vals[j];
        }
        __syncthreads();
    }
}

cudaError_t launch_radix_hist(cudaStream_t s, int grid, const uint32_t *keys, uint32_t n_host, const uint32_t *n_dev,
                              uint32_t bits, uint32_t passes, uint32_t *hist) {
    radix_hist_kernel<<<grid, SORT_THREADS, 0, s>>>(keys, n_host, n_dev, bits, passes, hist);
    return cudaGetLastError();
}

cudaError_t launch_onesweep_pass(cudaStream_t s, int grid, const uint32_t *keys_in, const uint32_t *vals_in,
                                 uint32_t *keys_out, uint32_t *vals_out, uint32_t n_host, const uint32_t *n_dev,
                                 uint32_t shift, uint32_t width, const uint32_t *hist, uint32_t *ticket,
                                 unsigned long long *lb, unsigned long long *lb_group, const uint32_t *epoch_base,
                                 uint32_t epoch_off) {
    if (n_host <= SORT_SMALL_MAX_KEYS)
        onesweep_pass_kernel<SORT_ITEMS_SMALL><<<grid, SORT_THREADS, 0, s>>>(keys_in, vals_in, keys_out, vals_out, n_host, n_dev, shift,
                                                                             width, hist, ticket, lb, lb_group, epoch_base, epoch_off);
    else
        onesweep_pass_kernel<SORT_ITEMS><<<grid, SORT_THREADS, 0, s>>>(keys_in, vals_in, keys_out, vals_out, n_host, n_dev, shift, width,
                                                                       hist, ticket, lb, lb_group, epoch_base, epoch_off);
    return cudaGetLastError();
}

// number of look-back tile slots a sort of up to n keys can use (api.cu sizes the look-back words with it)
uint64_t sort_max_tiles(uint64_t n) {
    const uint64_t big = (n + SORT_TILE - 1) / SORT_TILE;
    const uint64_t small_n = n < SORT_SMALL_MAX_KEYS ? n : SORT_SMALL_MAX_KEYS;
    const uint64_t small = (small_n + SORT_THREADS * SORT_ITEMS_SMALL - 1) / (SORT_THREADS * SORT_ITEMS_SMALL);
    return (big > small ? big : small) + 1;
}

}  // namespace bg

namespace bg {
__global__ void bump_epoch_kernel(uint32_t *epoch_base) { *epoch_base = (*epoch_base + 1u) & 0x01FFFFFFu; }
cudaError_t launch_bump_epoch(cudaStream_t s, uint32_t *epoch_base) {
    bump_epoch_kernel<<<1, 1, 0, s>>>(epoch_base);
    return cudaGetLastError();
}
}  // namespace bg
