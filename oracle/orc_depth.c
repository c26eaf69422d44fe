/*
 * oracle/orc_depth.c -- TEST INFRASTRUCTURE ONLY (CPU oracle).
 *
 * Accumulated depth D = sum_i vis_i z_i of the blend (DESIGN.md section 4.6) and its adjoint.  The reference has no
 * depth output: these follow the oracle's own blend (orc_forward.c, K5) and rasterize adjoint (orc_backward.c) with
 * depth as one more colour channel whose colour is the splat's camera-space z (depths_sorted[cgid]), without the
 * colour clamp, gate or background term.  Built into liborc_depth.so by depth.mk; wrapped by oracle_depth.py.
 */
#include "orc_api.h"
#include "orc_math.h"

#include <stdlib.h>

#define TILE_WIDTH 16u
#define TILE_SIZE 256u
#define ALPHA_CUTOFF_MID (1.0f / 255.0f)

float orc_alpha_cutoff_weight(float alpha);
float orc_alpha_cutoff_weight_deriv(float alpha);

/* D [h,w] of a pass != forward render, replayed from its projected rows and depths_sorted with the pass's cutoff. */
void orc_render_depth(const OrcRender *r, float *out_depth) {
    const uint32_t w = r->w, h = r->h, tiles_x = r->tiles_x, num_tiles = r->tiles_x * r->tiles_y;
    const int smooth = r->pass == ORC_PASS_BACKWARD_SMOOTH;
#pragma omp parallel for schedule(dynamic, 4)
    for (int64_t tile = 0; tile < (int64_t)num_tiles; tile++) {
        const uint32_t range_lo = r->tile_offsets[tile * 2], range_hi = r->tile_offsets[tile * 2 + 1];
        const uint32_t ox = ((uint32_t)tile % tiles_x) * TILE_WIDTH, oy = ((uint32_t)tile / tiles_x) * TILE_WIDTH;
        for (uint32_t ly = 0; ly < TILE_WIDTH; ly++) {
            for (uint32_t lx = 0; lx < TILE_WIDTH; lx++) {
                const uint32_t px = ox + lx, py = oy + ly;
                if (!(px < w && py < h)) continue;
                const float pcx = (float)px + 0.5f, pcy = (float)py + 0.5f;
                float t_acc = 1.0f, d = 0.0f;
                for (uint32_t is = range_lo; is < range_hi; is++) {
                    const uint32_t cg = r->cgid_from_isect[is];
                    const float *p = r->projected + (size_t)cg * 9;
                    const osym2 conic = {p[2], p[3], p[4]};
                    const float sigma = orc_calc_sigma(pcx, pcy, conic, p[0], p[1]);
                    const float alpha = orc_min(0.999f, p[5] * orc_expf(-sigma));
                    const float w_cut = smooth ? orc_alpha_cutoff_weight(alpha) : (alpha >= ALPHA_CUTOFF_MID ? 1.0f : 0.0f);
                    if (!(sigma >= 0.0f && w_cut > 0.0f)) continue;
                    const float alpha_eff = alpha * w_cut;
                    const float next_t = t_acc * (1.0f - alpha_eff);
                    if (next_t <= 1.0e-4f) break;   /* the stopping splat is not blended */
                    d = fmaf(r->depths_sorted[cg], alpha_eff * t_acc, d);
                    t_acc = next_t;
                }
                out_depth[(size_t)px + (size_t)py * w] = d;
            }
        }
    }
}

/* The joint colour + depth adjoint: orc_rasterize_backward with the upstream gradient v_depth [h,w] of D (out_depth is
 * D).  v_combined [V,10] and v_z [V] (compact id), zeroed here.  Joint because the refine weight is nonlinear in v_xy. */
void orc_rasterize_backward_depth(const OrcRender *r, const float *bg3, const float *v_output, const float *out_depth,
                                  const float *v_depth, int smooth, float *v_combined, float *v_z) {
    const uint32_t w = r->w, h = r->h, tiles_x = r->tiles_x, num_tiles = r->tiles_x * r->tiles_y;
    const uint32_t V = r->num_visible, I = r->num_intersections;
    const float bg_r = bg3 ? bg3[0] : 0.0f, bg_g = bg3 ? bg3[1] : 0.0f, bg_b = bg3 ? bg3[2] : 0.0f;
    memset(v_combined, 0, sizeof(float) * 10 * (size_t)(V ? V : 1));
    memset(v_z, 0, sizeof(float) * (size_t)(V ? V : 1));
    float *partial = (float *)calloc((size_t)(I ? I : 1) * 11, sizeof(float));

#pragma omp parallel for schedule(dynamic, 4)
    for (int64_t tile = 0; tile < (int64_t)num_tiles; tile++) {
        const uint32_t range_lo = r->tile_offsets[tile * 2], range_hi = r->tile_offsets[tile * 2 + 1];
        if (range_hi <= range_lo) continue;
        const uint32_t ox = ((uint32_t)tile % tiles_x) * TILE_WIDTH, oy = ((uint32_t)tile / tiles_x) * TILE_WIDTH;
        /* pixel state: remaining colour, transmittance, remaining depth */
        float st[TILE_SIZE][5];
        for (uint32_t rank = 0; rank < TILE_SIZE; rank++) {
            uint32_t px = ox + rank % TILE_WIDTH, py = oy + rank / TILE_WIDTH;
            if (px < w && py < h) {
                const size_t pix = (size_t)px + (size_t)py * w;
                const float *o = r->out_img + pix * 4;
                float t_final = 1.0f - o[3];
                st[rank][0] = o[0] - t_final * bg_r;
                st[rank][1] = o[1] - t_final * bg_g;
                st[rank][2] = o[2] - t_final * bg_b;
                st[rank][3] = 1.0f;
                st[rank][4] = out_depth[pix];
            } else {
                st[rank][0] = st[rank][1] = st[rank][2] = st[rank][3] = st[rank][4] = 0.0f;
            }
        }
        for (uint32_t is = range_lo; is < range_hi; is++) {
            const uint32_t cg = r->cgid_from_isect[is];
            const float *sp = r->projected + (size_t)cg * 9;
            const float xy_x = sp[0], xy_y = sp[1], color_a = sp[5];
            const osym2 conic = {sp[2], sp[3], sp[4]};
            const float cr = sp[6], cgn = sp[7], cb = sp[8], z = r->depths_sorted[cg];
            const float clamped_r = orc_max(cr, 0.0f), clamped_g = orc_max(cgn, 0.0f), clamped_b = orc_max(cb, 0.0f);
            float g_xy_x = 0, g_xy_y = 0, g_cx = 0, g_cy = 0, g_cz = 0, g_r = 0, g_g = 0, g_b = 0, g_a = 0, g_ref = 0, g_z = 0;
            for (uint32_t rank = 0; rank < TILE_SIZE; rank++) {
                float state_x = st[rank][0], state_y = st[rank][1], state_z = st[rank][2], state_w = st[rank][3];
                float state_d = st[rank][4];
                if (!(state_w > 1.0e-4f)) continue;
                uint32_t px = ox + rank % TILE_WIDTH, py = oy + rank / TILE_WIDTH;
                float pcx = (float)px + 0.5f, pcy = (float)py + 0.5f;
                float dx = xy_x - pcx, dy = xy_y - pcy;
                float sigma = 0.5f * (conic.c00 * dx * dx + conic.c11 * dy * dy) + conic.c01 * dx * dy;
                float gaussian = orc_expf(-sigma);
                float alpha = orc_min(0.999f, color_a * gaussian);
                float w_cut = smooth ? orc_alpha_cutoff_weight(alpha) : (alpha >= ALPHA_CUTOFF_MID ? 1.0f : 0.0f);
                if (!(sigma >= 0.0f && w_cut > 0.0f)) continue;
                float alpha_eff = alpha * w_cut;
                float next_t = state_w * (1.0f - alpha_eff);
                if (next_t <= 1.0e-4f) { st[rank][3] = 0.0f; continue; }
                float vis = alpha_eff * state_w;
                size_t pix = (size_t)px + (size_t)py * w, pb = pix * 4;
                float v_o_x = v_output[pb], v_o_y = v_output[pb + 1], v_o_z = v_output[pb + 2], v_a = v_output[pb + 3];
                float v_d = v_depth[pix];
                float final_a = r->out_img[pb + 3];
                float t_final = 1.0f - final_a;
                float v_o_w = (v_a - (bg_r * v_o_x + bg_g * v_o_y + bg_b * v_o_z)) * t_final;
                g_r += (cr >= 0.0f) ? vis * v_o_x : 0.0f;
                g_g += (cgn >= 0.0f) ? vis * v_o_y : 0.0f;
                g_b += (cb >= 0.0f) ? vis * v_o_z : 0.0f;
                g_z += vis * v_d;
                float ra = 1.0f / (1.0f - alpha_eff);
                float dot = ((state_w * clamped_r - state_x) * v_o_x + (state_w * clamped_g - state_y) * v_o_y +
                             (state_w * clamped_b - state_z) * v_o_z + (state_w * z - state_d) * v_d) * ra;
                float nrx = state_x - vis * clamped_r, nry = state_y - vis * clamped_g, nrz = state_z - vis * clamped_b;
                float nrd = state_d - vis * z;
                float v_alpha_eff = dot + v_o_w * ra;
                float dw_dalpha = smooth ? orc_alpha_cutoff_weight_deriv(alpha) : 0.0f * alpha;
                float v_alpha = v_alpha_eff * (w_cut + alpha * dw_dalpha);
                float v_sigma = -alpha * v_alpha;
                float vxy_x = v_sigma * (conic.c00 * dx + conic.c01 * dy);
                float vxy_y = v_sigma * (conic.c01 * dx + conic.c11 * dy);
                if (color_a * gaussian <= 0.999f) {
                    g_cx += 0.5f * v_sigma * dx * dx;
                    g_cy += v_sigma * dx * dy;
                    g_cz += 0.5f * v_sigma * dy * dy;
                    g_xy_x += vxy_x;
                    g_xy_y += vxy_y;
                    g_a += v_alpha * gaussian;
                    float isx = (float)w, isy = (float)h;
                    float len = sqrtf(vxy_x * isx * vxy_x * isx + vxy_y * isy * vxy_y * isy);
                    g_ref += len / orc_max(final_a, 1.0e-5f);
                }
                st[rank][0] = nrx; st[rank][1] = nry; st[rank][2] = nrz; st[rank][3] = next_t; st[rank][4] = nrd;
            }
            float *p = partial + (size_t)is * 11;
            p[0] = g_xy_x; p[1] = g_xy_y; p[2] = g_cx; p[3] = g_cy; p[4] = g_cz;
            p[5] = g_r; p[6] = g_g; p[7] = g_b; p[8] = g_a; p[9] = g_ref; p[10] = g_z;
        }
    }
    /* partials added in intersection order, tiles ascending (one legal order of the device's atomics) */
    for (uint32_t is = 0; is < I; is++) {
        const float *p = partial + (size_t)is * 11;
        const uint32_t cg = r->cgid_from_isect[is];
        float *d = v_combined + (size_t)cg * 10;
        for (int k = 0; k < 10; k++) d[k] += p[k];
        v_z[cg] += p[10];
    }
    free(partial);
}
