// blend_fwd.cu -- per-tile front-to-back alpha blend.
// Replaces rasterize_kernel (kernels/rasterize.rs:25-190).  Semantics (rasterize.rs:116-181):
//   sigma = 0.5 (a dx^2 + c dy^2) + b dx dy at the pixel centre; alpha = min(0.999, o e^-sigma);
//   skip unless sigma >= 0 and alpha >= 1/255; T' = T (1 - alpha); if T' <= 1e-4 the pixel is done and this
//   splat is NOT blended; rgb += max(c,0) alpha T; output rgb + T bg, a = 1 - T.
// With BWD_INFO: rgba f32 output, visible[gid] = 1 for every blended splat, the tile's range end trimmed to one
// past the last blended splat (rasterize.rs:183-189), and the hand-off words of blend_common.cuh.
// SMOOTH (test-only, BWD_INFO only): the smooth alpha cutoff of blend_common.cuh, and its wider block-cull margin.
// DEPTH (BWD_INFO only): also the accumulated depth D = sum vis_i z_i ([h,w] f32, no background term; DESIGN §4.6),
// z_i = depths[compact id], the depth-sort key.  The staging lane parks z_i in pad lane 13 of the row; every other
// output (image, visible, trimmed ends, hand-off words) is the same as without DEPTH.
//
// Bound: instruction issue (FP32 + MUFU), not HBM.  Per warp-splat iteration (64 pixel-splat pairs) the loop is
// 3 broadcast LDS.128, 4 scalar + 9 paired (18 scalar) FMA-pipe operations, 2 MUFU.EX2 and the pair tests.  The rows of a
// batch are staged by TMA (per-row bulk copies, blend_common.cuh) into the warp's double buffer.
#include "blend_common.cuh"
#include "bg_launch.cuh"

namespace bg {

template <bool BWD_INFO, bool SMOOTH, bool DEPTH>
__global__ void __launch_bounds__(RASTER_THREADS)
blend_fwd_kernel(const float *__restrict__ projected, const uint32_t *__restrict__ cgid_from_isect,
                 uint32_t *__restrict__ tile_offsets, const uint32_t *__restrict__ gid_from_cgid,
                 float4 *__restrict__ out_f32, uint32_t *__restrict__ out_packed, float *__restrict__ visible,
                 uint32_t *__restrict__ live_masks, uint32_t *__restrict__ warp_batches, BlendUniforms u,
                 const float *__restrict__ depths, float *__restrict__ out_depth) {
    __shared__ BlendStage s_stage[RASTER_WARPS];   // per warp, double buffered
    __shared__ uint32_t s_max_useful;

    const uint32_t tile = blockIdx.x;
    const uint32_t tid = threadIdx.x, lane = tid & 31u, wid = tid >> 5;
    const uint32_t tile_x0 = (tile % u.tiles_x) * TILE_W, tile_y0 = (tile / u.tiles_x) * TILE_W;
    const uint32_t blk_x0 = tile_x0 + 8u * (wid & 1u), blk_y0 = tile_y0 + 8u * (wid >> 1);
    const uint32_t pix_x = blk_x0 + (lane & 7u), pix_y0 = blk_y0 + (lane >> 3), pix_y1 = pix_y0 + 4u;
    const bool inside0 = pix_x < u.img_w && pix_y0 < u.img_h;
    const bool inside1 = pix_x < u.img_w && pix_y1 < u.img_h;
    const float px = (float)pix_x + 0.5f, py0 = (float)pix_y0 + 0.5f;
    const float2 npy2 = make_float2(-py0, -(py0 + 4.0f));
    // rectangle of this warp's pixel centres
    const float rx0 = (float)blk_x0 + 0.5f, rx1 = rx0 + 7.0f, ry0 = (float)blk_y0 + 0.5f, ry1 = ry0 + 7.0f;

    const uint32_t range_lo = tile_offsets[tile * 2], range_hi = tile_offsets[tile * 2 + 1];
    if (BWD_INFO && tid == 0) s_max_useful = range_lo;
    BlendStage &st = s_stage[wid];
    if (lane == 0) { mbar_init(&st.bar[0], 1); mbar_init(&st.bar[1], 1); }
    __syncthreads();   // barriers initialised before any copy is issued
    uint32_t phase_bits = 0u;   // bit b: parity the next wait on buffer b expects

    // T2: transmittance of the blended prefix (what the output uses).  Tt2: the same value while the pixel is alive;
    // the stopping splat's T' (<= 1e-4) afterwards, so that "T' > 1e-4" alone rejects every later splat.
    float2 T2 = make_float2(1.0f, 1.0f);
    float2 Tt2 = make_float2(inside0 ? 1.0f : 0.0f, inside1 ? 1.0f : 0.0f);
    float2 r2 = make_float2(0.0f, 0.0f), g2 = r2, b2 = r2, d2 = r2;
    uint32_t last_useful = range_lo;

    const uint32_t num_batches = (range_hi - range_lo + WB - 1) / WB;
    const size_t mbase = blend_mask_base(range_lo, tile) + wid;
    uint32_t batches_walked = 0;
    uint32_t next_id = 0;
    float next_z = 0.0f;
    // stage batch b: every lane parks the id of "its" list entry, one elected lane issues the TMA copies
    auto prefetch = [&](uint32_t b) {
        const uint32_t start = range_lo + b * WB;
        const uint32_t count = min((uint32_t)WB, range_hi - start);
        const uint32_t id = lane < count ? __ldg(cgid_from_isect + start + lane) : 0u;
        next_id = id;
        if constexpr (DEPTH) next_z = lane < count ? __ldg(depths + id) : 0.0f;   // in flight during the TMA wait
        if (lane < count) st.ids[b & 1u][lane] = id;
        stage_rows_tma(st, b & 1u, count, projected, lane);
    };
    // a warp whose pixels are all outside the image has nothing to blend
    if (num_batches > 0 && __any_sync(0xffffffffu, inside0 || inside1)) {
        prefetch(0);
        for (uint32_t b = 0; b < num_batches; b++) {
            const uint32_t batch_start = range_lo + b * WB;
            const uint32_t count = min((uint32_t)WB, range_hi - batch_start);
            const uint32_t my_id = next_id;
            const float my_z = next_z;
            if (b + 1 < num_batches) prefetch(b + 1);
            mbar_wait(&st.bar[b & 1u], (phase_bits >> (b & 1u)) & 1u);
            phase_bits ^= 1u << (b & 1u);
            float *rows = st.rows[b & 1u];
            bool hit = false;
            if (lane < count) {
                float *mine = rows + lane * ROW;
                const float4 A = *reinterpret_cast<const float4 *>(mine);
                const float4 B = *reinterpret_cast<const float4 *>(mine + 4);
                const float bcol = mine[8];
                float pt = mine[ROW_PT];
                if constexpr (SMOOTH) pt += SMOOTH_THR_EXTRA;
                hit = block_may_hit(A.x, A.y, A.z, A.w, B.x, pt, rx0, rx1, ry0, ry1);
                // per-splat constants are formed once here, by the lane that staged the row: colour -> max(colour, 0)
                *reinterpret_cast<float2 *>(mine + 6) = make_float2(fmaxf(B.z, 0.0f), fmaxf(B.w, 0.0f));
                mine[8] = fmaxf(bcol, 0.0f);
                if constexpr (DEPTH) mine[ROW_Z] = my_z;
            }
            uint32_t bits = __ballot_sync(0xffffffffu, hit);   // (also orders the row fix-ups before the reads below)
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
                r2 = ffma2_rn(bcast2(B.z), vis, r2);
                g2 = ffma2_rn(bcast2(B.w), vis, g2);
                b2 = ffma2_rn(bcast2(C.x), vis, b2);
                if constexpr (DEPTH) d2 = ffma2_rn(bcast2(row[ROW_Z]), vis, d2);
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
            const uint32_t used = __reduce_or_sync(0xffffffffu, used_m);
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
                if (b + 1 < num_batches) mbar_wait(&st.bar[(b + 1) & 1u], (phase_bits >> ((b + 1) & 1u)) & 1u);   // never leave a copy in flight
                break;
            }
            __syncwarp();  // all lanes are done with this buffer before the next prefetch overwrites its twin
        }
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
        // one block barrier, after all blending: publish the trimmed range end
        uint32_t m = last_useful;
        for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
        __syncthreads();
        if (lane == 0 && m > range_lo) atomicMax(&s_max_useful, m);
        __syncthreads();
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
    blend_fwd_kernel<B, S, D><<<num_tiles, RASTER_THREADS, 0, s>>>(projected, cgid_from_isect, tile_offsets, gid_from_cgid, \
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
