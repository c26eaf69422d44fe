// blend_bwd.cu -- adjoint of the per-tile blend.
// Replaces rasterize_backwards_kernel (bwd/kernels/rasterize_backwards.rs:100-391).  SMOOTH: the test-only smooth
// alpha cutoff (blend_common.cuh), replayed from the hand-off of a smooth forward.
//
// Replay semantics (rasterize_backwards.rs:186-228, 279-383): pixel state starts at (final_rgb - T_final*bg, T = 1);
// per splat, with the forward's skip/stop rules:
//   vis = alpha*T; v_rgb += vis*v_out_rgb (gated on c >= 0); ra = 1/(1-alpha);
//   v_alpha = (sum_k (T*c_k - rem_k) v_out_k) ra + (v_out_a - bg.v_out_rgb) T_final ra;
//   v_sigma = -alpha v_alpha; if o*e^-sigma <= 0.999: v_conic += (0.5 v_sigma dx^2, v_sigma dx dy, 0.5 v_sigma dy^2),
//   v_xy += v_sigma (a dx + b dy, b dx + c dy) [dx = mean - pixel], v_opac += v_alpha e^-sigma,
//   refine += |(v_x W, v_y H)| / max(alpha_final, 1e-5);  rem -= vis*c; T <- T'.
//
// Structure.  One thread per pixel pair as in the forward (state in registers), but the walk is driven by the
// forward's hand-off (blend_common.cuh): per batch the warp reads the 32-bit set of splats that changed its block,
// stages ONLY those rows (compacted, by TMA bulk copies: blend_common.cuh), and runs a plain counted loop over them -- no block test, no vote,
// no dead iteration.  The staging lane also forms the per-splat constants once (clamped colour, -opacity, and in the
// row's free lanes 12..15 the colour gates and 1/opacity), so the loop body is per-pixel work only, written on float2
// (fadd2_rn / fmul2_rn / ffma2_rn; splat scalars broadcast).  Signs are chosen so that no negation is ever an
// instruction: the loop accumulates -vis, -v_alpha, -v_sigma and the post-reduction factors put the signs back.
// v_opac uses e^-sigma = alpha/opacity on the unsaturated pairs (the only ones that count), i.e. it is
// -(sum v_sigma)/opacity: one factor per splat instead of one FMA per pair.  This holds under SMOOTH as well: there
// v_alpha = d/d alpha already carries the factor w + alpha w'(alpha), and v_sigma = -alpha v_alpha with the raw alpha
// (not alpha_eff) on the unsaturated pairs, so -(sum v_sigma)/opacity = sum e^-sigma v_alpha (rasterize_backwards.rs:349-372).
// The loop takes two splats per iteration, in list order, and forms their 2 x 10 sums over the warp's 64 pixels with
// one 21-shuffle reduce-scatter; the twenty owning lanes flush both splats with one RED.F32 each.
//
// DEPTH: the adjoint of the accumulated depth D = sum vis_i z_i of a DEPTH forward (DESIGN §4.6).  Depth is one more
// colour channel with colour z_i (no clamp, no gate, no background): the pixel state gains rem_d (initialised to the
// final D) and v_D, the pair's v_alpha gains (T z_i - rem_d) v_D / (1 - alpha), and the 11th sum v_z_i = sum vis v_D
// (factor -1) goes to the compact-indexed v_z[]: 2 x 11 sums, 23 shuffles per pair of splats.
#include "blend_common.cuh"
#include "bg_launch.cuh"

namespace bg {

// Lanes 12..15 of a staged row, rewritten by the lane that parked its id (the projected row's lane 12, the forward's
// block-cull threshold, and its pad lanes are not read by the backward): the post-reduction factors that vary per splat.
constexpr int BROW_IOPAC = 12;    // 1/opacity: the factor of the -sum v_sigma slot (v_opacity)
constexpr int BROW_GATE = 13;     // 13..15: the colour gates, -1 where the channel's colour is >= 0, else 0
// Residency floor of the launch bounds (DESIGN §6.17: timed against the unbounded build)
constexpr int BWD_MIN_CTAS = 8;

__device__ __forceinline__ float rcp_approx_f(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float sqrt_approx_f(float x) { float r; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }

// atomicAdd (RED.F32) through a global address, for an address ptxas cannot prove global by itself
__device__ __forceinline__ void red_add_global(size_t gaddr, float v) {
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(gaddr), "f"(v) : "memory");
}

// One stage of the reduce-scatter: v (length L, padded to even length with a zero) is split in halves; lanes with `hi`
// keep the upper half, the others the lower half, and each adds its xor partner's copy of the half it keeps.
template <int L>
__device__ __forceinline__ void rs_halve(const float (&v)[L], float (&out)[(L + 1) / 2], bool hi, int lane_xor) {
    constexpr int H = (L + 1) / 2;
#pragma unroll
    for (int i = 0; i < H; i++) {
        const float lo = v[i], up = i + H < L ? v[i + H < L ? i + H : 0] : 0.0f;
        out[i] = (hi ? up : lo) + __shfl_xor_sync(0xffffffffu, hi ? lo : up, lane_xor);
    }
}

// Reduce-scatter of the 2*NS sums of a splat pair over the warp: 10+5+3+2+1 = 21 shuffles for NS = 10 (23 for 11).
// Lane l ends up with the warp total of the entry of v that rs_owner gives it, or with padding: an exact 0 + 0.
template <int L>
__device__ __forceinline__ float reduce_scatter32(const float (&v)[L], uint32_t lane) {
    constexpr int L1 = (L + 1) / 2, L2 = (L1 + 1) / 2, L3 = (L2 + 1) / 2, L4 = (L3 + 1) / 2;
    static_assert((L4 + 1) / 2 == 1, "32 lanes reduce at most 32 sums");
    float a[L1], b[L2], c[L3], d[L4], e[1];
    rs_halve(v, a, lane & 16u, 16);
    rs_halve(a, b, lane & 8u, 8);
    rs_halve(b, c, lane & 4u, 4);
    rs_halve(c, d, lane & 2u, 2);
    rs_halve(d, e, lane & 1u, 1);
    return e[0];
}
// Which entry of the L sums reduce_scatter32 leaves in `lane` (through the halving, the upper halves are the shorter
// ones).  A lane whose window runs out of real entries holds padding instead: its entry is never read, because the
// flush skips a zero sum.
template <int L>
__device__ __forceinline__ uint32_t rs_owner(uint32_t lane) {
    int len = L, idx = 0;
#pragma unroll
    for (int bit = 4; bit >= 0; bit--) {
        const int h = (len + 1) / 2;
        if ((lane >> bit) & 1u) idx += h;
        len = h;
    }
    return (uint32_t)idx;
}

// stats[0] warp-splat iterations, [1] pixel-splat pairs that blended, [2] pairs that stopped a pixel
template <bool STATS, bool SMOOTH, bool DEPTH>
__global__ void __launch_bounds__(RASTER_THREADS, SMOOTH ? 1 : DEPTH ? 7 : BWD_MIN_CTAS)
blend_bwd_kernel(const float *__restrict__ projected, const uint32_t *__restrict__ cgid_from_isect,
                 const uint32_t *__restrict__ tile_offsets, const float4 *__restrict__ out_img,
                 const float4 *__restrict__ v_output, const uint32_t *__restrict__ live_masks,
                 const uint32_t *__restrict__ warp_batches, float *__restrict__ v_combined,
                 unsigned long long *__restrict__ stats, BlendUniforms u, const float *__restrict__ depths,
                 const float *__restrict__ out_depth, const float *__restrict__ v_depth, float *__restrict__ v_z) {
    __shared__ BlendStage s_stage[RASTER_WARPS];   // per warp, double buffered rows (TMA destination)

    const uint32_t tile = blockIdx.x;
    // (warp index and batch count broadcast from lane 0: ptxas then knows the staging runs warp-converged, so the copy
    // operands stay in uniform registers)
    const uint32_t tid = threadIdx.x, lane = tid & 31u, wid = __shfl_sync(0xffffffffu, tid >> 5, 0);
    const uint32_t num_batches = __shfl_sync(0xffffffffu, __ldg(warp_batches + tile * RASTER_WARPS + wid), 0);
    BlendStage &st = s_stage[wid];
    if (lane == 0) { mbar_init(&st.bar[0], 1); mbar_init(&st.bar[1], 1); }
    __syncthreads();   // barriers initialised before any copy is issued
    if (num_batches == 0) return;
    uint32_t phase_bits = 0u;   // bit b: parity the next wait on buffer b expects
    const uint32_t range_lo = tile_offsets[tile * 2];
    const uint32_t tile_x0 = (tile % u.tiles_x) * TILE_W, tile_y0 = (tile / u.tiles_x) * TILE_W;
    const uint32_t blk_x0 = tile_x0 + 8u * (wid & 1u), blk_y0 = tile_y0 + 8u * (wid >> 1);
    const uint32_t pix_x = blk_x0 + (lane & 7u), pix_y0 = blk_y0 + (lane >> 3), pix_y1 = pix_y0 + 4u;
    const bool inside0 = pix_x < u.img_w && pix_y0 < u.img_h;
    const bool inside1 = pix_x < u.img_w && pix_y1 < u.img_h;
    const float px = (float)pix_x + 0.5f, py0 = (float)pix_y0 + 0.5f;
    const float2 npy2 = make_float2(-py0, -(py0 + 4.0f));
    const float img_wf = (float)u.img_w, img_hf = (float)u.img_h;
    const float hw = img_hf / img_wf, hw2 = hw * hw;   // |(vx W, vy H)| = W sqrt(vx^2 + (H/W)^2 vy^2)

    // ---- pixel state (load_pixel_state, rasterize_backwards.rs:186-228), as pairs
    float2 T2 = make_float2(0.0f, 0.0f);                       // 0 outside the image: nothing ever blends
    float2 rem_r = T2, rem_g = T2, rem_b = T2;                 // colour still to come (positive)
    float2 vo_r = T2, vo_g = T2, vo_b = T2, nvo_w = T2, ifa = T2;
    {
        auto load = [&](bool inside, uint32_t pix_y, float &T, float &rr, float &rg, float &rb, float &vr, float &vg,
                        float &vb, float &nvw, float &inv) {
            if (!inside) return;
            const size_t pix_id = (size_t)pix_x + (size_t)pix_y * u.img_w;
            const float4 o = __ldg(out_img + pix_id);
            const float4 vo = __ldg(v_output + pix_id);
            const float t_final = 1.0f - o.w;
            T = 1.0f;
            rr = o.x - t_final * u.bg_r; rg = o.y - t_final * u.bg_g; rb = o.z - t_final * u.bg_b;
            vr = vo.x; vg = vo.y; vb = vo.z;
            nvw = -((vo.w - (u.bg_r * vo.x + u.bg_g * vo.y + u.bg_b * vo.z)) * t_final);
            inv = img_wf / fmaxf(o.w, 1.0e-5f);
        };
        load(inside0, pix_y0, T2.x, rem_r.x, rem_g.x, rem_b.x, vo_r.x, vo_g.x, vo_b.x, nvo_w.x, ifa.x);
        load(inside1, pix_y1, T2.y, rem_r.y, rem_g.y, rem_b.y, vo_r.y, vo_g.y, vo_b.y, nvo_w.y, ifa.y);
    }
    float2 rem_d = make_float2(0.0f, 0.0f), vo_d = rem_d;   // depth still to come, v_D
    if constexpr (DEPTH) {
        const size_t pix0 = (size_t)pix_x + (size_t)pix_y0 * u.img_w, pix1 = (size_t)pix_x + (size_t)pix_y1 * u.img_w;
        if (inside0) { rem_d.x = __ldg(out_depth + pix0); vo_d.x = __ldg(v_depth + pix0); }
        if (inside1) { rem_d.y = __ldg(out_depth + pix1); vo_d.y = __ldg(v_depth + pix1); }
    }

    // ---- the flush, formed once: the NS sums of splats j and j+1 are reduce-scattered together, and the lane that
    // ends up with a real sum owns slot own_slot of splat j + own_sp (a lane left with padding holds an exact 0 and
    // never flushes).  Its output is dst[id * dst_stride].  Its factor is a shared float the lane reads at
    // f_base + j * f_step: for the colour gates and 1/opacity the row lane of its splat (f_step one row), for the
    // constant factors (signs, the 1/2 of the conic diagonal) its own entry of st.fconst (f_step 0).  Each value
    // passes through a shuffle from the lane itself: ptxas then cannot re-derive it from the lane index inside the
    // loop, which it otherwise does on every iteration to save a register.
    constexpr int NS = DEPTH ? 11 : 10;
    const uint32_t own_index = rs_owner<2 * NS>(lane);
    const uint32_t own_sp = own_index >= (uint32_t)NS ? 1u : 0u, own_slot = own_index - own_sp * NS;
    const bool fvar = own_slot >= 5u && own_slot <= 8u;
    const uint32_t own_lane = own_slot == 8u ? (uint32_t)BROW_IOPAC : BROW_GATE + own_slot - 5u;
    const uint32_t f_off = __shfl_sync(0xffffffffu, fvar ? (own_sp * ROW + own_lane) * 4u : 0u, lane);
    const uint32_t f_step = __shfl_sync(0xffffffffu, fvar ? ROW * 4u : 0u, lane);
    st.fconst[lane] = own_slot == 9u ? 1.0f : (own_slot == 2u || own_slot == 4u) ? -0.5f : -1.0f;
    const uint32_t id_off = __shfl_sync(0xffffffffu, own_sp * 4u, lane);
    const bool to_vz = DEPTH && own_slot == 10u;
    const size_t dst = __shfl_sync(
        0xffffffffu, (unsigned long long)__cvta_generic_to_global(to_vz ? v_z : v_combined + (own_slot < 10u ? own_slot : 0u)), lane);
    const uint32_t dst_stride = DEPTH ? __shfl_sync(0xffffffffu, to_vz ? 1u : BG_VCOMBINED_STRIDE, lane) : BG_VCOMBINED_STRIDE;

    const uint32_t lt_mask = (1u << lane) - 1u;
    const size_t mbase = blend_mask_base(range_lo, tile) + wid;
    auto load_mask = [&](uint32_t b) -> uint32_t {
        // (broadcast from lane 0: a mask ptxas knows is warp-uniform keeps the copy issue in uniform registers)
        return __shfl_sync(0xffffffffu, b < num_batches ? __ldg(live_masks + mbase + (size_t)b * RASTER_WARPS) : 0u, 0);
    };
    // stage the rows of batch b selected by mask m, compacted in list order, into buffer b&1: the lanes park the row
    // ids, the warp issues the TMA copies
    // (DEPTH: the same lane also starts the load of the row's z, which lands during the TMA wait)
    float z_next = 0.0f;
    auto stage = [&](uint32_t b, uint32_t m) {
        const uint32_t n = (uint32_t)__popc(m);
        if (n == 0) return;
        if ((m >> lane) & 1u) {
            const uint32_t id = __ldg(cgid_from_isect + range_lo + b * WB + lane);
            st.ids[b & 1u][__popc(m & lt_mask)] = id;
            if constexpr (DEPTH) z_next = __ldg(depths + id);
        }
        stage_rows_tma(st, b & 1u, n, projected, lane);
    };

    // ---- one splat against the lane's two pixels: advances the pixel state and returns the lane's two-pixel sums
    // g[0..NS) (-v_xy, -v_conic without the 1/2 of the diagonal, -v_rgb ungated, -v_sigma, refine; DEPTH: -v_z)
    unsigned long long st_iter = 0, st_blend = 0, st_stop = 0;
    auto splat = [&](const float *row, float z, float (&g)[NS]) {
        const float4 A = *reinterpret_cast<const float4 *>(row);       // mx my a b
        const float4 B = *reinterpret_cast<const float4 *>(row + 4);   // c -opac r+ g+
        const float4 C = *reinterpret_cast<const float4 *>(row + 8);   // b+, then log2(e)-scaled c/2, a/2, b
        const float dx = A.x - px;
        float2 dy2;
        const float2 sg = pair_sigma(dx, A.y, C.y, C.z, C.w, npy2, dy2);
        const float2 gs = make_float2(ex2_approx(-sg.x), ex2_approx(-sg.y));
        const float2 noa = fmul2_rn(gs, bcast2(B.y));                                 // -opac*g
        const float2 nal = make_float2(fmaxf(-0.999f, noa.x), fmaxf(-0.999f, noa.y));   // -alpha
        // the forward's tests (blend_common.cuh); T of a stopped pixel stays <= 1e-4, so it never blends again
        float2 nae = nal;   // -alpha_eff
        bool act0, act1;
        if constexpr (SMOOTH) {
            const float2 ae = smooth_alpha(make_float2(-nal.x, -nal.y), sg, act0, act1);
            nae = make_float2(-ae.x, -ae.y);
        } else {
            act0 = sg.x >= 0.0f && noa.x <= -ALPHA_CUTOFF_MID; act1 = sg.y >= 0.0f && noa.y <= -ALPHA_CUTOFF_MID;
        }
        const float2 oma = fadd2_rn(nae, bcast2(1.0f));
        const float2 nT = fmul2_rn(T2, oma);
        const bool c0 = act0 && nT.x > 1.0e-4f, c1 = act1 && nT.y > 1.0e-4f;
        if (STATS) {
            st_blend += __popc(__ballot_sync(0xffffffffu, c0)) + __popc(__ballot_sync(0xffffffffu, c1));
            st_stop += __popc(__ballot_sync(0xffffffffu, act0 && !c0 && T2.x > 1.0e-4f)) +
                       __popc(__ballot_sync(0xffffffffu, act1 && !c1 && T2.y > 1.0e-4f));
        }
        // -alpha_eff where the pair blends (nalc); -alpha additionally gated on "not alpha-saturated" (nals) for
        // everything but the colour terms (rasterize_backwards.rs:357-372)
        const float2 nalc = make_float2(c0 ? nae.x : 0.0f, c1 ? nae.y : 0.0f);
        const float2 nals = make_float2((c0 && noa.x >= -0.999f) ? nal.x : 0.0f, (c1 && noa.y >= -0.999f) ? nal.y : 0.0f);
        const float2 ra = make_float2(rcp_approx_f(oma.x), rcp_approx_f(oma.y));
        const float2 nvis = fmul2_rn(nalc, T2);                        // -vis
        const float2 G5 = fmul2_rn(nvis, vo_r), G6 = fmul2_rn(nvis, vo_g), G7 = fmul2_rn(nvis, vo_b);
        // u_k = rem_k - T c_k
        const float2 u_r = ffma2_rn(T2, bcast2(-B.z), rem_r);
        const float2 u_g = ffma2_rn(T2, bcast2(-B.w), rem_g);
        const float2 u_b = ffma2_rn(T2, bcast2(-C.x), rem_b);
        float2 nd = fmul2_rn(u_r, vo_r);
        nd = ffma2_rn(u_g, vo_g, nd);
        nd = ffma2_rn(u_b, vo_b, nd);                                   // -dot
        if constexpr (DEPTH) {
            const float2 u_d = ffma2_rn(T2, bcast2(-z), rem_d);          // rem_d - T z
            nd = ffma2_rn(u_d, vo_d, nd);
        }
        float2 nva = fmul2_rn(fadd2_rn(nd, nvo_w), ra);               // -v_alpha
        if constexpr (SMOOTH) nva = fmul2_rn(nva, make_float2(smooth_alpha_deriv(-nal.x), smooth_alpha_deriv(-nal.y)));
        const float2 nvs = fmul2_rn(nals, nva);                         // -v_sigma  (= alpha v_alpha)
        const float2 vsx = fmul2_rn(nvs, bcast2(dx)), vsy = fmul2_rn(nvs, dy2);
        const float2 G0 = ffma2_rn(bcast2(A.z), vsx, fmul2_rn(bcast2(A.w), vsy));   // -v_xy.x
        const float2 G1 = ffma2_rn(bcast2(A.w), vsx, fmul2_rn(bcast2(B.x), vsy));   // -v_xy.y
        const float2 G2 = fmul2_rn(vsx, bcast2(dx)), G3 = fmul2_rn(vsx, dy2), G4 = fmul2_rn(vsy, dy2);
        const float2 nn = ffma2_rn(G0, G0, fmul2_rn(fmul2_rn(G1, bcast2(hw2)), G1));
        const float2 G9 = fmul2_rn(make_float2(sqrt_approx_f(nn.x), sqrt_approx_f(nn.y)), ifa);
        // advance the pixel state
        rem_r = ffma2_rn(nvis, bcast2(B.z), rem_r);
        rem_g = ffma2_rn(nvis, bcast2(B.w), rem_g);
        rem_b = ffma2_rn(nvis, bcast2(C.x), rem_b);
        if constexpr (DEPTH) {
            const float2 G10 = fmul2_rn(nvis, vo_d);                     // -vis v_D
            g[10] = G10.x + G10.y;
            rem_d = ffma2_rn(nvis, bcast2(z), rem_d);
        }
        T2.x = act0 ? nT.x : T2.x;
        T2.y = act1 ? nT.y : T2.y;
        g[0] = G0.x + G0.y; g[1] = G1.x + G1.y; g[2] = G2.x + G2.y; g[3] = G3.x + G3.y; g[4] = G4.x + G4.y;
        g[5] = G5.x + G5.y; g[6] = G6.x + G6.y; g[7] = G7.x + G7.y; g[8] = nvs.x + nvs.y; g[9] = G9.x + G9.y;
    };

    uint32_t m_cur = load_mask(0), m_next = load_mask(1);
    stage(0, m_cur);
    for (uint32_t b = 0; b < num_batches; b++) {
        const uint32_t m = m_cur;
        const float my_z = z_next;
        m_cur = m_next;
        m_next = load_mask(b + 2);
        stage(b + 1, m_cur);   // (an all-zero mask stages nothing)
        const uint32_t n = (uint32_t)__popc(m);
        if (n == 0) continue;
        mbar_wait(&st.bar[b & 1u], (phase_bits >> (b & 1u)) & 1u);
        phase_bits ^= 1u << (b & 1u);
        float *rows = st.rows[b & 1u];
        const uint32_t *ids = st.ids[b & 1u];
        float *zs = st.z[b & 1u];
        const char *f_base = f_step ? reinterpret_cast<const char *>(rows) + f_off : reinterpret_cast<const char *>(&st.fconst[lane]);
        if ((m >> lane) & 1u) {
            // per-splat constants, formed once by the lane that parked the row's id
            const uint32_t slot_r = (uint32_t)__popc(m & lt_mask);
            float *mine = rows + slot_r * ROW;
            const float4 B = *reinterpret_cast<const float4 *>(mine + 4);   // c opac r g
            const float bcol = mine[8];
            *reinterpret_cast<float4 *>(mine + 4) = make_float4(B.x, -B.y, fmaxf(B.z, 0.0f), fmaxf(B.w, 0.0f));
            mine[8] = fmaxf(bcol, 0.0f);
            *reinterpret_cast<float4 *>(mine + BROW_IOPAC) =
                make_float4(1.0f / B.y, B.z >= 0.0f ? -1.0f : 0.0f, B.w >= 0.0f ? -1.0f : 0.0f, bcol >= 0.0f ? -1.0f : 0.0f);
            if constexpr (DEPTH) zs[slot_r] = my_z;
        }
        if (n & 1u) {
            // an odd batch ends on a null row (all zeros: -opacity 0, so no pixel acts on it) and the loop runs whole
            // pairs.  n <= 31 here, so the row exists.  With finite inputs every sum of the null row is an exact 0,
            // which never flushes; a non-finite upstream gradient makes them NaN (0 * NaN), as it makes every sum of
            // the warp's real rows.  So the null row also gets a real id, the last row's: such a NaN lands on a splat
            // the warp has already made NaN, never on a stale id from an earlier batch.
            if (lane < ROW) rows[n * ROW + lane] = 0.0f;
            if (lane == 0) st.ids[b & 1u][n] = st.ids[b & 1u][n - 1];
            if constexpr (DEPTH) if (lane == 0) zs[n] = 0.0f;
        }
        __syncwarp();
        if (STATS) st_iter += n;
        for (uint32_t j = 0; j < n; j += 2) {
            // splats j and j+1 in list order (j+1 sees the state j left), then one reduce-scatter of both
            float g0[NS], g1[NS], g[2 * NS];
            splat(rows + j * ROW, DEPTH ? zs[j] : 0.0f, g0);
            splat(rows + (j + 1) * ROW, DEPTH ? zs[j + 1] : 0.0f, g1);
#pragma unroll
            for (int i = 0; i < NS; i++) { g[i] = g0[i]; g[NS + i] = g1[i]; }
            const float d = reduce_scatter32(g, lane);
            if (d != 0.0f) {
                const uint32_t id = *reinterpret_cast<const uint32_t *>(reinterpret_cast<const char *>(ids + j) + id_off);
                const float f = *reinterpret_cast<const float *>(f_base + j * f_step);
                red_add_global(dst + (size_t)id * dst_stride * sizeof(float), d * f);
            }
        }
        __syncwarp();  // all lanes are done with this buffer before the next stage() overwrites it
    }
    if (STATS && lane == 0) {
        atomicAdd(stats + 0, st_iter); atomicAdd(stats + 1, st_blend); atomicAdd(stats + 2, st_stop);
    }
}

cudaError_t launch_blend_bwd(cudaStream_t s, bool smooth, uint32_t num_tiles, const float *projected, const uint32_t *cgid_from_isect,
                             const uint32_t *tile_offsets, const float *out_img, const float *v_output, const uint32_t *live_masks,
                             const uint32_t *warp_batches, float *v_combined, unsigned long long *stats, uint32_t tiles_x,
                             uint32_t w, uint32_t h, const float *bg, const float *depths, const float *out_depth,
                             const float *v_depth, float *v_z) {
    BlendUniforms u;
    u.tiles_x = tiles_x; u.img_w = w; u.img_h = h; u.bg_r = bg[0]; u.bg_g = bg[1]; u.bg_b = bg[2];
#define BG_LAUNCH_BWD(ST, S, D, STATS_PTR)                                                                                \
    blend_bwd_kernel<ST, S, D><<<num_tiles, RASTER_THREADS, 0, s>>>(projected, cgid_from_isect, tile_offsets, (const float4 *)out_img, \
                                                                    (const float4 *)v_output, live_masks, warp_batches, v_combined, \
                                                                    STATS_PTR, u, depths, out_depth, v_depth, v_z)
    // (test-only smooth cutoff and the depth adjoint: no counting variant)
    if (v_z) {
        if (smooth) BG_LAUNCH_BWD(false, true, true, nullptr);
        else BG_LAUNCH_BWD(false, false, true, nullptr);
    } else if (smooth) {
        BG_LAUNCH_BWD(false, true, false, nullptr);
    } else if (stats) {
        BG_LAUNCH_BWD(true, false, false, stats);
    } else {
        BG_LAUNCH_BWD(false, false, false, nullptr);
    }
#undef BG_LAUNCH_BWD
    return cudaGetLastError();
}

}  // namespace bg
