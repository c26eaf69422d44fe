// blend_fwd.cu -- per-tile front-to-back alpha blend.
// Replaces rasterize_kernel (kernels/rasterize.rs:25-190).  Semantics (rasterize.rs:116-181):
//   sigma = 0.5 (a dx^2 + c dy^2) + b dx dy at the pixel centre; alpha = min(0.999, o e^-sigma);
//   skip unless sigma >= 0 and alpha >= 1/255; T' = T (1 - alpha); if T' <= 1e-4 the pixel is done and this
//   splat is NOT blended; rgb += max(c,0) alpha T; output rgb + T bg, a = 1 - T.
// With BWD_INFO: rgba f32 output, visible[gid] = 1 for every blended splat, the tile's range end trimmed to one
// past the last blended splat (rasterize.rs:183-189), and the hand-off words of blend_common.cuh.
// SMOOTH (test-only, BWD_INFO only): the smooth alpha cutoff of blend_common.cuh, and its wider block-cull margin.
// DEPTH (BWD_INFO only): also the accumulated depth D = sum vis_i z_i ([h,w] f32, no background term; DESIGN §4.6),
// z_i = depths[compact id], the depth-sort key.  The producer lanes store z_i in the ring slot's z table; every other
// output (image, visible, trimmed ends, hand-off words) is the same as without DEPTH.
//
// Bound: instruction issue (FP32 + MUFU), not HBM.  Per warp-splat iteration (64 pixel-splat pairs) the loop is
// 3 broadcast LDS.128, 4 scalar + 9 paired (18 scalar) FMA-pipe operations, 3 colour clamps, 2 MUFU.EX2 and the pair
// tests.  The rows of a batch are staged once per tile by TMA (per-row bulk copies, blend_common.cuh) into a ring the
// four pixel warps share (below).
#include "blend_common.cuh"
#include "bg_launch.cuh"

namespace bg {

// ---- the tile's ring of staged batches.  Batch b of the tile's list lives in slot b % FWD_RING.  full[k]: the
// producer's arrive + the transaction bytes of the slot's copies; empty[k]: one arrival per pixel warp that is done
// reading the slot.  The pixel warps only read the ring (the colour clamp is applied where the colour is used), so
// every row is staged once per tile instead of once per warp.
constexpr int FWD_RING = 4;
constexpr int FWD_THREADS = RASTER_THREADS + 32;   // four pixel warps + the producer warp
struct __align__(128) BlendRing {
    float rows[FWD_RING][WB * ROW];
    float z[FWD_RING][WB];   // DEPTH: the rows' camera-space z, stored by the producer lanes
    unsigned long long full[FWD_RING], empty[FWD_RING];
};

__device__ __forceinline__ void mbar_arrive(unsigned long long *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned long long *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0u;
}

template <bool BWD_INFO, bool SMOOTH, bool DEPTH>
__global__ void __launch_bounds__(FWD_THREADS)
blend_fwd_kernel(const float *__restrict__ projected, const uint32_t *__restrict__ cgid_from_isect,
                 uint32_t *__restrict__ tile_offsets, const uint32_t *__restrict__ gid_from_cgid,
                 float4 *__restrict__ out_f32, uint32_t *__restrict__ out_packed, float *__restrict__ visible,
                 uint32_t *__restrict__ live_masks, uint32_t *__restrict__ warp_batches, BlendUniforms u,
                 const float *__restrict__ depths, float *__restrict__ out_depth) {
    __shared__ BlendRing s_ring;
    __shared__ uint32_t s_max_useful;
    __shared__ uint32_t s_live;   // bit k: pixel warp k still blends (clears when all its pixels are saturated)
    __shared__ uint32_t s_end;    // batches the producer issued; lowered from num_batches when it stops early

    const uint32_t tile = blockIdx.x;
    // (the warp index broadcast from lane 0: ptxas then knows the producer's branch is warp-uniform, so its copy
    // operands stay in uniform registers)
    const uint32_t tid = threadIdx.x, lane = tid & 31u, wid = __shfl_sync(0xffffffffu, tid >> 5, 0);
    const uint32_t tile_x0 = (tile % u.tiles_x) * TILE_W, tile_y0 = (tile / u.tiles_x) * TILE_W;
    const uint32_t range_lo = tile_offsets[tile * 2], range_hi = tile_offsets[tile * 2 + 1];
    const uint32_t num_batches = (range_hi - range_lo + WB - 1) / WB;
    if (tid < FWD_RING) { mbar_init(&s_ring.full[tid], 1); mbar_init(&s_ring.empty[tid], RASTER_WARPS); }
    if (tid == 0) {
        s_max_useful = range_lo;
        s_end = num_batches;
        // a warp whose pixels are all outside the image has nothing to blend: it counts as retired from the start
        uint32_t live = 0;
        for (uint32_t k = 0; k < RASTER_WARPS; k++)
            if (tile_x0 + 8u * (k & 1u) < u.img_w && tile_y0 + 8u * (k >> 1) < u.img_h) live |= 1u << k;
        s_live = live;
    }
    __syncthreads();   // barriers initialised before any copy is issued

    if (wid == RASTER_WARPS) {
        // ---- producer: the lanes load a batch's ids coalesced, the warp issues its copies once for all four warps
        uint32_t b = 0;
        for (; b < num_batches; b++) {
            const uint32_t slot = b % FWD_RING;
            if (b >= FWD_RING) mbar_wait(&s_ring.empty[slot], (b / FWD_RING - 1u) & 1u);
            if (__shfl_sync(0xffffffffu, *(volatile uint32_t *)&s_live, 0) == 0u) break;   // every pixel warp retired
            const uint32_t start = range_lo + b * WB;
            const uint32_t count = __shfl_sync(0xffffffffu, min((uint32_t)WB, range_hi - start), 0);
            const uint32_t id = lane < count ? __ldg(cgid_from_isect + start + lane) : 0u;
            if constexpr (DEPTH) {
                s_ring.z[slot][lane] = lane < count ? __ldg(depths + id) : 0.0f;
                __syncwarp();   // the z of the slot written before the arrive below releases it
            }
            if (lane == 0) mbar_expect_tx(&s_ring.full[slot], count * (ROW * 4u));
            issue_rows_tma(s_ring.rows[slot], id, count, projected, &s_ring.full[slot]);
        }
        if (b < num_batches && lane == 0) *(volatile uint32_t *)&s_end = b;
        // never leave a copy in flight: wait for the last batch issued into each slot
        for (uint32_t k = b > (uint32_t)FWD_RING ? b - FWD_RING : 0u; k < b; k++)
            mbar_wait(&s_ring.full[k % FWD_RING], (k / FWD_RING) & 1u);
        return;
    }

    const uint32_t blk_x0 = tile_x0 + 8u * (wid & 1u), blk_y0 = tile_y0 + 8u * (wid >> 1);
    const uint32_t pix_x = blk_x0 + (lane & 7u), pix_y0 = blk_y0 + (lane >> 3), pix_y1 = pix_y0 + 4u;
    const bool inside0 = pix_x < u.img_w && pix_y0 < u.img_h;
    const bool inside1 = pix_x < u.img_w && pix_y1 < u.img_h;
    const float px = (float)pix_x + 0.5f, py0 = (float)pix_y0 + 0.5f;
    const float2 npy2 = make_float2(-py0, -(py0 + 4.0f));
    // rectangle of this warp's pixel centres
    const float rx0 = (float)blk_x0 + 0.5f, rx1 = rx0 + 7.0f, ry0 = (float)blk_y0 + 0.5f, ry1 = ry0 + 7.0f;

    // T2: transmittance of the blended prefix (what the output uses).  Tt2: the same value while the pixel is alive;
    // the stopping splat's T' (<= 1e-4) afterwards, so that "T' > 1e-4" alone rejects every later splat.
    float2 T2 = make_float2(1.0f, 1.0f);
    float2 Tt2 = make_float2(inside0 ? 1.0f : 0.0f, inside1 ? 1.0f : 0.0f);
    float2 r2 = make_float2(0.0f, 0.0f), g2 = r2, b2 = r2, d2 = r2;
    uint32_t last_useful = range_lo;

    const size_t mbase = blend_mask_base(range_lo, tile) + wid;
    uint32_t batches_walked = 0;
    uint32_t b = 0;
    if ((s_live >> wid) & 1u) {
        for (; b < num_batches; b++) {
            const uint32_t slot = b % FWD_RING;
            const uint32_t batch_start = range_lo + b * WB;
            const uint32_t count = min((uint32_t)WB, range_hi - batch_start);
            uint32_t my_id = 0;
            if (BWD_INFO && lane < count) my_id = __ldg(cgid_from_isect + batch_start + lane);   // lands during the wait
            mbar_wait(&s_ring.full[slot], (b / FWD_RING) & 1u);
            const float *rows = s_ring.rows[slot];
            bool hit = false;
            if (lane < count) {
                const float *mine = rows + lane * ROW;
                const float4 A = *reinterpret_cast<const float4 *>(mine);
                float pt = mine[ROW_PT];
                if constexpr (SMOOTH) pt += SMOOTH_THR_EXTRA;
                hit = block_may_hit(A.x, A.y, A.z, A.w, mine[4], pt, rx0, rx1, ry0, ry1);
            }
            uint32_t bits = __ballot_sync(0xffffffffu, hit);
            uint32_t used_m = 0, acted_m = 0;
            while (bits) {
                const uint32_t s = (uint32_t)__ffs(bits) - 1u;
                bits &= bits - 1u;
                const float *row = rows + s * ROW;
                const float4 A = *reinterpret_cast<const float4 *>(row);       // mx my a b
                const float4 B = *reinterpret_cast<const float4 *>(row + 4);   // c opac r g
                const float4 C = *reinterpret_cast<const float4 *>(row + 8);   // b_col, then log2(e)-scaled c/2, a/2, b
                float2 dy2;
                const float2 sg = pair_sigma(A.x - px, A.y, C.y, C.z, C.w, npy2, dy2);
                const float2 gs = make_float2(ex2_approx(-sg.x), ex2_approx(-sg.y));
                const float2 oa = fmul2_rn(gs, bcast2(B.y));
                float a0 = fminf(0.999f, oa.x), a1 = fminf(0.999f, oa.y);   // alpha; alpha_eff under SMOOTH
                // acts: the splat passes the alpha test; a done pixel's T' stays <= 1e-4, so c is false for it
                bool act0, act1;
                if constexpr (SMOOTH) {
                    const float2 ae = smooth_alpha(make_float2(a0, a1), sg, act0, act1);
                    a0 = ae.x; a1 = ae.y;
                } else {
                    act0 = sg.x >= 0.0f && oa.x >= ALPHA_CUTOFF_MID; act1 = sg.y >= 0.0f && oa.y >= ALPHA_CUTOFF_MID;
                }
                const float2 nT = fmul2_rn(Tt2, fadd2_rn(make_float2(-a0, -a1), bcast2(1.0f)));
                const bool c0 = act0 && nT.x > 1.0e-4f, c1 = act1 && nT.y > 1.0e-4f;
                // No votes inside the splat loop: the blend runs unconditionally (weights are zero where it does
                // not apply), each lane remembers which splats touched its pixels, and "all pixels saturated" is
                // checked once per batch (saturated pixels ignore the remaining splats of the batch).
                const float2 vis = fmul2_rn(make_float2(c0 ? a0 : 0.0f, c1 ? a1 : 0.0f), T2);
                r2 = ffma2_rn(bcast2(fmaxf(B.z, 0.0f)), vis, r2);
                g2 = ffma2_rn(bcast2(fmaxf(B.w, 0.0f)), vis, g2);
                b2 = ffma2_rn(bcast2(fmaxf(C.x, 0.0f)), vis, b2);
                if constexpr (DEPTH) d2 = ffma2_rn(bcast2(s_ring.z[slot][s]), vis, d2);
                const uint32_t bit = 1u << s;
                // the hand-off needs the splats that changed a live pixel: blended it or stopped it
                const bool acted = (Tt2.x > 1.0e-4f && act0) || (Tt2.y > 1.0e-4f && act1);
                if (c0 || c1) used_m |= bit;              // per-lane masks, OR-reduced once per batch
                if (BWD_INFO && acted) acted_m |= bit;
                T2.x = c0 ? nT.x : T2.x;
                T2.y = c1 ? nT.y : T2.y;
                Tt2.x = act0 ? nT.x : Tt2.x;
                Tt2.y = act1 ? nT.y : Tt2.y;
            }
            const uint32_t used = __reduce_or_sync(0xffffffffu, used_m);   // (every lane is done reading the slot)
            if (lane == 0) mbar_arrive(&s_ring.empty[slot]);
            if (BWD_INFO) {
                const uint32_t acted = __reduce_or_sync(0xffffffffu, acted_m);
                if (lane == 0) live_masks[mbase + (size_t)b * RASTER_WARPS] = acted;
                if ((used >> lane) & 1u) {
                    visible[__ldg(gid_from_cgid + my_id)] = 1.0f;
                    last_useful = batch_start + lane + 1;
                }
            }
            batches_walked = b + 1;
            if (__all_sync(0xffffffffu, !(Tt2.x > 1.0e-4f) && !(Tt2.y > 1.0e-4f))) {
                b++;
                if (lane == 0) atomicAnd(&s_live, ~(1u << wid));
                break;
            }
        }
    }
    // retired: stop blending, but keep releasing the slots of the batches the producer still issues, until it has
    // stopped (s_end) or the list ends
    for (; b < num_batches; b++) {
        const uint32_t slot = b % FWD_RING;
        bool staged;
        while (!(staged = mbar_try_wait(&s_ring.full[slot], (b / FWD_RING) & 1u)))
            if (b >= *(volatile uint32_t *)&s_end) break;
        if (__shfl_sync(0xffffffffu, (uint32_t)staged, 0) == 0u) break;
        if (lane == 0) mbar_arrive(&s_ring.empty[slot]);
    }

    auto write_pixel = [&](float T, float r, float g, float bl, float d, uint32_t pix_y) {
        const float fr = r + T * u.bg_r, fg = g + T * u.bg_g, fb = bl + T * u.bg_b, fa = 1.0f - T;
        const size_t pix_id = (size_t)pix_x + (size_t)pix_y * u.img_w;
        if (BWD_INFO) {
            out_f32[pix_id] = make_float4(fr, fg, fb, fa);
            if constexpr (DEPTH) out_depth[pix_id] = d;
        } else {
            uint32_t r8 = (uint32_t)fminf(fmaxf(fr * 255.0f, 0.0f), 255.0f);
            uint32_t g8 = (uint32_t)fminf(fmaxf(fg * 255.0f, 0.0f), 255.0f);
            uint32_t b8 = (uint32_t)fminf(fmaxf(fb * 255.0f, 0.0f), 255.0f);
            uint32_t a8 = (uint32_t)fminf(fmaxf(fa * 255.0f, 0.0f), 255.0f);
            out_packed[pix_id] = r8 | (g8 << 8) | (b8 << 16) | (a8 << 24);
        }
    };
    if (inside0) write_pixel(T2.x, r2.x, g2.x, b2.x, d2.x, pix_y0);
    if (inside1) write_pixel(T2.y, r2.y, g2.y, b2.y, d2.y, pix_y1);
    if (BWD_INFO) {
        if (lane == 0) warp_batches[tile * RASTER_WARPS + wid] = batches_walked;
        // one barrier of the four pixel warps (named barrier 1; the producer has left), after all blending: publish
        // the trimmed range end
        uint32_t m = last_useful;
        for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (lane == 0 && m > range_lo) atomicMax(&s_max_useful, m);
        asm volatile("bar.sync 1, %0;" ::"n"(RASTER_THREADS) : "memory");
        if (tid == 0) tile_offsets[tile * 2 + 1] = s_max_useful;
    }
}

cudaError_t launch_blend_fwd(cudaStream_t s, bool bwd_info, bool smooth, uint32_t num_tiles, const float *projected,
                             const uint32_t *cgid_from_isect, uint32_t *tile_offsets, const uint32_t *gid_from_cgid, void *out_img,
                             float *visible, uint32_t *live_masks, uint32_t *warp_batches, uint32_t tiles_x, uint32_t w,
                             uint32_t h, const float *bg, const float *depths, float *out_depth) {
    BlendUniforms u;
    u.tiles_x = tiles_x; u.img_w = w; u.img_h = h; u.bg_r = bg[0]; u.bg_g = bg[1]; u.bg_b = bg[2];
#define BG_LAUNCH_FWD(B, S, D, F32, PACKED, LM, WBAT)                                                                    \
    blend_fwd_kernel<B, S, D><<<num_tiles, FWD_THREADS, 0, s>>>(projected, cgid_from_isect, tile_offsets, gid_from_cgid, \
                                                                   F32, PACKED, visible, LM, WBAT, u, depths, out_depth)
    if (!bwd_info)
        BG_LAUNCH_FWD(false, false, false, nullptr, (uint32_t *)out_img, nullptr, nullptr);
    else if (out_depth && !smooth)   // (depth with bwd_info only: the entry point rejects it for the packed pass)
        BG_LAUNCH_FWD(true, false, true, (float4 *)out_img, nullptr, live_masks, warp_batches);
    else if (out_depth)
        BG_LAUNCH_FWD(true, true, true, (float4 *)out_img, nullptr, live_masks, warp_batches);
    else if (!smooth)
        BG_LAUNCH_FWD(true, false, false, (float4 *)out_img, nullptr, live_masks, warp_batches);
    else
        BG_LAUNCH_FWD(true, true, false, (float4 *)out_img, nullptr, live_masks, warp_batches);
#undef BG_LAUNCH_FWD
    return cudaGetLastError();
}

}  // namespace bg
