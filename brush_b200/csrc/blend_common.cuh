// blend_common.cuh -- the blend kernels (blend_fwd.cu, blend_bwd.cu): shared layout, staging and the pair tests.
//
// Tile = 16x16 pixels = one CTA of 4 pixel warps (the forward adds a producer warp, blend_fwd.cu).  Warp k owns the 8x8
// pixel block with origin (8*(k&1), 8*(k>>1)); lane l owns the two pixels (l&7, l>>3) and (l&7, (l>>3)+4) of the
// block.  Every pixel warp walks the tile's depth-ordered splat list on its own, in batches of 32 splats, with no
// block-wide barrier inside the loop: a warp whose 64 pixels are saturated stops blending at once, and later batches'
// rows are staged while the current batch is blended.
//
//  * paired FP32.  The two pixels of a lane run ONE instruction stream, so all per-pixel arithmetic is
//    written on float2 (fadd2_rn / fmul2_rn / ffma2_rn of bg_common.cuh; per-splat scalars are broadcast), and
//    the per-splat work (row loads, constants, the block test) is shared by both pixels.
//  * forward -> backward hand-off.  The forward kernel records, per (tile, batch of 32, warp), the 32-bit
//    set of splats that changed any pixel of the warp's block (blended OR stopped a pixel), and per
//    (tile, warp) the number of batches it walked before all its pixels saturated.  The backward kernel
//    stages and evaluates exactly those splats: no block test, no vote, no dead iteration, no re-staging of
//    rows the forward proved irrelevant.  Both kernels evaluate the pair test below with the same
//    explicitly rounded operations, so the replayed transmittance is bit-identical to the forward's.
//
// Pair test (rasterize.rs:116-155; the backward's replay rasterize_backwards.rs:279-330), per pixel:
//   d = mean - pixel centre;  s2 = log2(e) * sigma = hx + (cy*dy)*dy + bdx*dy  with hx = (cz*dx)*dx, bdx = cw*dx
//   (cy, cz, cw = log2(e)/2*c, log2(e)/2*a, log2(e)*b are lanes 9..11 of the projected row)
//   g = ex2.approx(-s2);  oa = opac*g;  alpha = min(0.999, oa);  T' = T*(1 - alpha)
//   acts      = pixel not done  &&  s2 >= 0  &&  oa >= 1/255
//   blends    = acts && T' > 1e-4      (T <- T')
//   stops     = acts && T' <= 1e-4     (pixel done; this splat is NOT blended)
// The test-only smooth cutoff (SMOOTH, kernels/helpers.rs:20-47; rasterize.rs:132-140) blends alpha_eff =
// alpha * w(alpha) in place of alpha (T' = T*(1 - alpha_eff), vis = alpha_eff*T) and a pair acts when
// s2 >= 0 && w(alpha) > 0 (smooth_alpha below).
#pragma once
#include "bg_common.cuh"

namespace bg {

constexpr int RASTER_WARPS = 4;
constexpr int RASTER_THREADS = RASTER_WARPS * 32;
constexpr int WB = 32;                    // splats per warp batch
constexpr int ROW = BG_PROJECTED_STRIDE;  // 16 floats
constexpr int ROW_PT = 12;                // lane of ln(255 opacity), the block-cull threshold

struct BlendUniforms {
    uint32_t tiles_x, img_w, img_h;
    float bg_r, bg_g, bg_b;
};

__device__ __forceinline__ float2 bcast2(float a) { return make_float2(a, a); }

// index of the first hand-off word of a tile: one uint4-sized group (4 warps) per batch.  Tiles own disjoint
// slot ranges: floor(lo/32) + tile is strictly increasing by at least ceil(len/32) from tile to tile.
__device__ __forceinline__ size_t blend_mask_base(uint32_t range_lo, uint32_t tile) {
    return ((size_t)(range_lo >> 5) + tile) * RASTER_WARPS;
}

// ---- TMA staging of a batch of projected rows (north_star: "TMA staging of each tile's sorted Gaussian slice").
// A tile's slice is an index list, not a contiguous range, and sm_90 has no gather form of the tensor copy, so every
// 64-byte row is its own 1-D bulk copy (cp.async.bulk, SASS UBLKCP; 16-byte alignment on both sides, which the
// 64-byte rows meet -- a 2-D tensor copy would need 128-byte aligned shared destinations).  The warp issues a batch's
// copies against one mbarrier (complete_tx); nothing occupies the LSU pipe or the register file for the copy.
//
// Issues the copies of rows 0..count) into the dense rows at `dst`, completing on `bar`: lane r holds the id of row r.
// Call with the whole warp converged and `count` warp-uniform; the caller has armed `bar` with the bytes.  The id is
// broadcast with a shuffle from a constant lane (the loop is unrolled), so ptxas knows every copy operand is
// warp-uniform: the address is formed in uniform registers and the copy issues once per warp (elect.sync), with no
// per-row ELECT waterfall -- 9 instructions per row, against 14 for one lane walking ids parked in shared memory.
__device__ __forceinline__ void issue_rows_tma(float *dst, uint32_t id, uint32_t count, const float *projected,
                                               unsigned long long *bar) {
    const uint32_t d0 = smem_u32(dst), b = smem_u32(bar);
#pragma unroll
    for (uint32_t r = 0; r < WB; r++) {
        if (r >= count) break;
        const float *src = projected + (size_t)__shfl_sync(0xffffffffu, id, r) * ROW;
        asm volatile(
            "{\n.reg .pred p;\nelect.sync _|p, 0xffffffff;\n"
            "@p cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n}" ::"r"(
                d0 + r * (ROW * 4u)),
            "l"(src), "n"(ROW * 4), "r"(b)
            : "memory");
    }
}

// Per-warp staging state of the backward: two buffers of 32 dense 64-byte rows, the compacted ids of the rows in
// flight (read again by the gradient flush), the rows' camera-space z (DEPTH), each lane's constant flush factor, one
// mbarrier each.
struct __align__(128) BlendStage {
    float rows[2][WB * ROW];
    uint32_t ids[2][WB];
    float z[2][WB];
    float fconst[WB];
    unsigned long long bar[2];
};

// Issues the copy of `count` rows (ids already compacted in st.ids[buf][0..count)) into st.rows[buf].  Call with the
// whole warp converged and `count` warp-uniform.  The lanes wrote per-splat constants into the rows of this buffer
// with generic stores when it was last consumed; the async-proxy copies overwrite them, so every lane fences its
// generic writes against the async proxy before the warp issues.
__device__ __forceinline__ void stage_rows_tma(BlendStage &st, uint32_t buf, uint32_t count, const float *projected, uint32_t lane) {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncwarp();   // ids and the fenced writes visible to every lane
    if (count == 0) return;
    const uint32_t id = st.ids[buf][lane];   // (stale past count: never read)
    if (lane == 0) mbar_expect_tx(&st.bar[buf], count * (ROW * 4u));
    issue_rows_tma(st.rows[buf], id, count, projected, &st.bar[buf]);
}

// True when the splat may contribute to some pixel centre of the rectangle [x0,x1] x [y0,y1].
// sigma(p) = 0.5 (p-m)^T C (p-m) is convex for a positive definite conic; with the centre outside
// the box its minimum over the box lies on a face visible from the centre, so at most two clamped
// 1-D minimisations give the exact minimum.  A pixel passes the alpha test only if sigma <= thr
// (thr = ln(opacity / alpha_min)); the comparison carries a margin for the rounding of both sides.
__device__ __forceinline__ bool block_may_hit(float mx, float my, float a, float b, float c, float thr, float x0,
                                              float x1, float y0, float y1) {
    // anything but a positive definite conic (rounding at extreme scales, NaN): no culling
    if (!(a > 0.0f && c > 0.0f && a * c > b * b)) return true;
    const float xc = fminf(fmaxf(mx, x0), x1);
    const float yc = fminf(fmaxf(my, y0), y1);
    const bool out_x = xc != mx, out_y = yc != my;
    if (!(out_x || out_y)) return true;
    float best = 3.0e38f, err = 0.0f;
    if (out_x) {  // face x = xc, free y
        float dx = xc - mx;
        float ys = fminf(fmaxf(my - (b / c) * dx, y0), y1);
        float dy = ys - my;
        float t0 = a * dx * dx, t1 = c * dy * dy, t2 = b * dx * dy;
        float s = 0.5f * (t0 + t1) + t2;
        if (s < best) { best = s; err = fabsf(t0) + fabsf(t1) + 2.0f * fabsf(t2); }
    }
    if (out_y) {  // face y = yc, free x
        float dy = yc - my;
        float xs = fminf(fmaxf(mx - (b / a) * dy, x0), x1);
        float dx = xs - mx;
        float t0 = a * dx * dx, t1 = c * dy * dy, t2 = b * dx * dy;
        float s = 0.5f * (t0 + t1) + t2;
        if (s < best) { best = s; err = fabsf(t0) + fabsf(t1) + 2.0f * fabsf(t2); }
    }
    return !(best > thr + 0.05f + 4.0e-6f * err);  // NaN compares false -> kept
}

__device__ __forceinline__ float ex2_approx(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }

// log2(e)-scaled exponent of the pair of pixels of this lane.  npy2 = (-py0, -(py0+4)), dx = mx - px.
__device__ __forceinline__ float2 pair_sigma(float dx, float my, float cy, float cz, float cw, float2 npy2, float2 &dy2) {
    const float hx = __fmul_rn(__fmul_rn(cz, dx), dx);
    const float bdx = __fmul_rn(cw, dx);
    dy2 = fadd2_rn(bcast2(my), npy2);
    float2 t = fmul2_rn(bcast2(cy), dy2);
    t = ffma2_rn(t, dy2, bcast2(hx));
    return ffma2_rn(bcast2(bdx), dy2, t);
}

// ---- smooth alpha cutoff (test-only; kernels/helpers.rs:20-47): a smoothstep of width ALPHA_CUTOFF_BAND centred
// at ALPHA_CUTOFF_MID, explicitly rounded so that the forward and the backward's replay agree bit for bit.
__device__ __forceinline__ float cutoff_weight(float alpha) {
    const float lo = ALPHA_CUTOFF_MID - 0.5f * ALPHA_CUTOFF_BAND;
    const float t = fminf(fmaxf(__fdiv_rn(__fsub_rn(alpha, lo), ALPHA_CUTOFF_BAND), 0.0f), 1.0f);
    return __fmul_rn(__fmul_rn(t, t), __fmaf_rn(-2.0f, t, 3.0f));
}
__device__ __forceinline__ float cutoff_weight_deriv(float alpha) {
    const float low = ALPHA_CUTOFF_MID - 0.5f * ALPHA_CUTOFF_BAND, high = ALPHA_CUTOFF_MID + 0.5f * ALPHA_CUTOFF_BAND;
    bool inside = alpha > low && alpha < high;
    float t = (alpha - low) / ALPHA_CUTOFF_BAND;
    return inside ? (6.0f * t - 6.0f * t * t) / ALPHA_CUTOFF_BAND : 0.0f;
}
// ln(alpha_cutoff_mid / smallest alpha with non-zero weight): the smooth cutoff's extra block-cull margin
constexpr float SMOOTH_THR_EXTRA = 0.1365f;

// The smooth pair test, for the lane's two pixels: returns alpha_eff = alpha * w(alpha) and sets the "acts" flags.
__device__ __forceinline__ float2 smooth_alpha(float2 alpha, float2 sg, bool &act0, bool &act1) {
    const float2 w = make_float2(cutoff_weight(alpha.x), cutoff_weight(alpha.y));
    act0 = sg.x >= 0.0f && w.x > 0.0f;
    act1 = sg.y >= 0.0f && w.y > 0.0f;
    return fmul2_rn(alpha, w);
}
// d alpha_eff / d alpha = w(alpha) + alpha w'(alpha)  (rasterize_backwards.rs:349-355)
__device__ __forceinline__ float smooth_alpha_deriv(float alpha) {
    return fmaf(alpha, cutoff_weight_deriv(alpha), cutoff_weight(alpha));
}

}  // namespace bg
