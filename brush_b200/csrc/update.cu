// update.cu -- the parameter update of one training step as ONE pass over the Gaussians.
// Replaces, per step (brush-train/src/train.rs:280-416):
//   AdamScaled::step on transforms [N,10] (per-column LR), SH coefficients [N,K,3] (per-band LR, second moment =
//   row mean of g^2) and raw opacity [N]                               (adam_scaled.rs:75-165, train.rs:328-381)
//   RefineRecord::gather_stats (MAX refine weight, SUM visible, MAX radius)            (stats.rs:40-50)
//   the mean noise  means += clamp(N(0,1) (1-opacity')^150 [vis > 0] lr 50, +-median)    (train.rs:389-416)
//   (opacity' = sigmoid(raw'), or with a floor clamp(sigmoid(raw') coef(log_scales', f), 1e-6, 1-1e-6); the gate is
//   visible > 0, which for the summed counts of a multi-view step is "seen by some view")
// The reference issues ~80 generic tensor ops for this; round 1 used five kernels (3 Adam, noise draw, stats+noise).
// A warp owns 32 consecutive Gaussians: the short rows (transforms, opacity, statistics) one lane each, the SH rows as
// one contiguous span read and written with coalesced 128-bit accesses; the normal
// draws are evaluated in registers (counter-based Philox, bg_rng.cuh; only Gaussians whose noise weight is non-zero
// draw at all), nothing but the parameters, moments and the refine record touches HBM:
//   (316 + 48 K + g) N bytes, g = 44 + 12 K (dense gradient) or 48 + 12 views (factored).
//
// Multi-view steps (SURVEY.md 8e): the SH gradient of one view is rank one per Gaussian,
// v_sh[g,k,:] = Y_k(dir(mean_g, camera_v)) v_color_v[g,:]  (kernels/sh.rs:265-355), so with FACTORED the kernel takes
// the views' colour gradients (all-gathered records) and forms (1/views) sum_v Y(dir_v) v_color_v in registers -- the
// dense [N,K,3] gradient is never written or read -- and reduces the MAX statistics over the records on the way.
// View order is the global view index, so every data-parallel rank computes bit-identical updates.
//
// Compiled with -fmad=false: plain IEEE multiply / add / divide / sqrt in the order written here (the order of
// AdamScaled::step), so the update is a pure function of its inputs on any IEEE machine.
#include <algorithm>

#include "bg_common.cuh"
#include "bg_fold.cuh"
#include "bg_rng.cuh"
#include "bg_sh.cuh"
#include "bg_update.cuh"

namespace bg {

__device__ __forceinline__ float adam_m(float m, float g, const UpdateParams &P) { return P.first ? g * P.f1 : m * P.beta1 + g * P.f1; }
__device__ __forceinline__ float adam_v(float v, float gsq, const UpdateParams &P) { return P.first ? gsq * P.f2 : v * P.beta2 + gsq * P.f2; }
// The bias corrections enter as reciprocals formed once on the host (1/bc1, 1/bc2) and the denominator as ONE correctly
// rounded reciprocal per second-moment value: p -= (m/bc1) / (sqrt(v/bc2) + eps) * step  becomes
// p -= ((m * inv_bc1) * rcp(sqrt(v * inv_bc2) + eps)) * step.  An IEEE division costs ~10 instructions on its fast path
// and a subroutine call on its slow one; three of them per element made this pass instruction bound.  Each replaced
// quotient differs from the division by at most one rounding (<= 1 ulp; WGSL, which the reference's optimiser runs on, allows 2.5 ulp for a division).
__device__ __forceinline__ float adam_inv_denom(float v, const UpdateParams &P) { return __frcp_rn(__fsqrt_rn(v * P.inv_bc2) + P.eps); }
__device__ __forceinline__ float adam_p(float p, float m, float inv_denom, float step, const UpdateParams &P) {
    return p - ((m * P.inv_bc1) * inv_denom) * step;
}

constexpr int UP_THREADS = 128;   // 4 warps; a warp owns 32 consecutive Gaussians and never waits for another warp

// One lane owns one Gaussian for everything that is a row of <= 10 floats (transforms, opacity, statistics, noise).
// The SH rows (3K floats) are handled by the whole warp: the 32 rows of a warp are one contiguous span of every SH array,
// which the lanes read and write as consecutive float4 (a fully coalesced 512-byte access per instruction, 12 of them in
// flight per lane at K = 16); the gradient rows pass through shared memory once so that lane r can form row r's mean of
// g^2 (the row-reduced second moment) in column order.
// PART: 0 = the whole update; 1 = SH coefficients only; 2 = everything but the SH coefficients.  The multi-device step runs
// part 1 as soon as the gathered records are there (it needs nothing from the all-reduce) and part 2 behind the all-reduce.
template <int DEG, bool FACTORED, int PART>
__global__ void __launch_bounds__(UP_THREADS)
train_update_kernel(const UpdateParams P) {
    constexpr int K = (DEG + 1) * (DEG + 1);
    constexpr int KF = K * 3;
    constexpr int SROW = KF | 1;   // odd row stride: lane r walking row r is bank-conflict free
    constexpr uint32_t NF_FULL = 8u * KF;            // float4 in the span of a full warp (32 rows)
    constexpr int NF_LANE = (NF_FULL + 31) / 32;     // ... per lane
    __shared__ float s_g[UP_THREADS / 32][32 * SROW];
    __shared__ float s_v[UP_THREADS / 32][32];
    const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
    const uint32_t j0 = (blockIdx.x * (UP_THREADS / 32) + wid) * 32u;   // first row of this warp inside the launch's slice
    if (j0 >= P.count) return;
    const uint32_t rows = min(32u, P.count - j0);
    const uint32_t j = j0 + lane;             // this lane's row inside the slice
    const uint32_t i = P.g_begin + j;         // ... and its Gaussian
    const bool valid = lane < rows;
    float *sg = s_g[wid];

    float old_mean[3] = {0.0f, 0.0f, 0.0f};
    if (PART == 1 && valid) {   // the SH rebuild needs the (not yet updated) means only
        old_mean[0] = P.transforms[(size_t)i * 10]; old_mean[1] = P.transforms[(size_t)i * 10 + 1]; old_mean[2] = P.transforms[(size_t)i * 10 + 2];
    }
    if (PART != 1 && valid) {
        // ---- transforms row: Adam with per-column learning rates (train.rs:328-350)
        float p[10], g_opac, vis;
        {
            float g[10], m[10], v[10];
            const float2 *p2 = reinterpret_cast<const float2 *>(P.transforms + (size_t)i * 10);
            float2 *m2 = reinterpret_cast<float2 *>(P.m_t + (size_t)i * 10);
            float2 *v2 = reinterpret_cast<float2 *>(P.v_t + (size_t)i * 10);
            if (FACTORED) {   // one 48-byte row of `small`: the ten transform gradients, the opacity gradient, the visibility
                const float4 *r4 = reinterpret_cast<const float4 *>(P.small + (size_t)i * 12);
                const float4 r0 = __ldg(r4), r1 = __ldg(r4 + 1), r2 = __ldg(r4 + 2);
                g[0] = r0.x; g[1] = r0.y; g[2] = r0.z; g[3] = r0.w; g[4] = r1.x; g[5] = r1.y; g[6] = r1.z; g[7] = r1.w; g[8] = r2.x; g[9] = r2.y;
                g_opac = r2.z; vis = r2.w;
            } else {
                const float2 *g2 = reinterpret_cast<const float2 *>(P.g_t + (size_t)i * 10);
#pragma unroll
                for (int q = 0; q < 5; q++) { const float2 b = __ldg(g2 + q); g[2 * q] = b.x; g[2 * q + 1] = b.y; }
                g_opac = __ldg(P.g_o + i); vis = __ldg(P.visible + i);
            }
#pragma unroll
            for (int q = 0; q < 5; q++) {
                const float2 a = p2[q];
                p[2 * q] = a.x; p[2 * q + 1] = a.y;
                if (!P.first) { const float2 c = m2[q], d = v2[q]; m[2 * q] = c.x; m[2 * q + 1] = c.y; v[2 * q] = d.x; v[2 * q + 1] = d.y; }
                else { m[2 * q] = m[2 * q + 1] = v[2 * q] = v[2 * q + 1] = 0.0f; }
            }
            old_mean[0] = p[0]; old_mean[1] = p[1]; old_mean[2] = p[2];
#pragma unroll
            for (int c = 0; c < 10; c++) {
                const float gg = P.grad_scale == 1.0f ? g[c] : g[c] * P.grad_scale;
                m[c] = adam_m(m[c], gg, P);
                v[c] = adam_v(v[c], gg * gg, P);
                p[c] = adam_p(p[c], m[c], adam_inv_denom(v[c], P), P.lr_t[c], P);
            }
#pragma unroll
            for (int q = 0; q < 5; q++) { m2[q] = make_float2(m[2 * q], m[2 * q + 1]); v2[q] = make_float2(v[2 * q], v[2 * q + 1]); }
        }
        // ---- raw opacity
        float raw;
        {
            const float gg = P.grad_scale == 1.0f ? g_opac : g_opac * P.grad_scale;
            const float mm = adam_m(P.first ? 0.0f : P.m_o[i], gg, P);
            const float vv = adam_v(P.first ? 0.0f : P.v_o[i], gg * gg, P);
            raw = adam_p(P.raw_opac[i], mm, adam_inv_denom(vv, P), P.lr_opac, P);
            P.m_o[i] = mm; P.v_o[i] = vv; P.raw_opac[i] = raw;
        }
        // ---- refine statistics of the step (stats.rs:40-50): MAX over the views, SUM of the visibility counts
        {
            float vr, rad;
            if (FACTORED) {
                const float2 st = __ldg(reinterpret_cast<const float2 *>(P.stat) + i);
                vr = st.x; rad = st.y;
            } else {
                vr = __ldg(P.v_refine + i); rad = __ldg(P.max_radius + i);
            }
            P.refine_norm[i] = fmaxf(vr, P.refine_norm[i]);
            P.vis_weight[i] = P.vis_weight[i] + vis;
            P.max_screen[i] = fmaxf(rad, P.max_screen[i]);
        }
        // ---- mean noise on the updated means, gated by the updated opacity (train.rs:389-416).  The reference gates on
        // Splats::opacities(), which folds the floor in when there is one (gaussian_splats.rs:215-223): then the gate is
        // clamp(sigmoid(raw) coef, 1e-6, 1-1e-6) with coef from the updated log-scales.
        if (P.noisy) {
            const float opac = P.min_scale ? fold_terms(p + 7, raw, __ldg(P.min_scale + i)).opac : 1.0f / (1.0f + expf(-raw));
            const float wgt = fminf(fmaxf(powf(1.0f - opac, 150.0f), 0.0f), 1.0f) * (vis > 0.0f ? 1.0f : 0.0f);
            const float wm = wgt * P.noise_scale;
            if (wm != 0.0f) {
                const unsigned long long e0 = 3ull * i;
                const uint32_t off = (uint32_t)(e0 & 3ull);   // elements 3i..3i+2 of the stream: quad e0/4, spilling into the next
                float z[8];
                normal_quad(P.seed, P.noise_offset + e0 / 4, z);
                if (off > 1u) normal_quad(P.seed, P.noise_offset + e0 / 4 + 1, z + 4);
                else z[4] = z[5] = z[6] = z[7] = 0.0f;
#pragma unroll
                for (int c = 0; c < 3; c++) {
                    const float zc = off == 0u ? z[c] : (off == 1u ? z[c + 1] : (off == 2u ? z[c + 2] : z[c + 3]));
                    p[c] += fminf(fmaxf(zc * wm, -P.median_scale), P.median_scale);
                }
            }
        }
        float2 *p2 = reinterpret_cast<float2 *>(P.transforms + (size_t)i * 10);
#pragma unroll
        for (int q = 0; q < 5; q++) p2[q] = make_float2(p[2 * q], p[2 * q + 1]);
    }

    if (PART == 2) return;
    // ---- SH gradient rows of the warp's 32 Gaussians -> shared memory
    const size_t span0 = (size_t)P.g_begin * KF + (size_t)j0 * KF;   // first float of the warp's span in the SH arrays
    const uint32_t total = rows * KF;                                // floats in the span
    const bool vec = (total & 3u) == 0;                              // (always true for full warps)
    if (FACTORED) {
        if (valid) {
            float g[KF];
#pragma unroll
            for (int c = 0; c < KF; c++) g[c] = 0.0f;
            for (uint32_t v = 0; v < P.views; v++) {
                const uint32_t r = v / P.local, li = v - r * P.local;
                const float *vc = P.records + ((size_t)r * P.count + j) * (3u * P.local) + 3u * li;
                const float cr = __ldg(vc), cg = __ldg(vc + 1), cb = __ldg(vc + 2);
                if (cr == 0.0f && cg == 0.0f && cb == 0.0f) continue;
                const float4 cp = __ldg(reinterpret_cast<const float4 *>(P.cam_all) + v);
                const V3 u_world = sub(mk3(old_mean[0], old_mean[1], old_mean[2]), mk3(cp.x, cp.y, cp.z));
                const V3 vdir = scale(u_world, 1.0f / length(u_world));
                float Y[K];
                sh_basis<DEG>(vdir, Y);
#pragma unroll
                for (int k = 0; k < K; k++) {
                    g[3 * k] += cr * Y[k];
                    g[3 * k + 1] += cg * Y[k];
                    g[3 * k + 2] += cb * Y[k];
                }
            }
#pragma unroll
            for (int c = 0; c < KF; c++) sg[lane * SROW + c] = g[c] * P.sh_grad_scale;
        }
    } else if (rows == 32u) {   // full warp: a compile-time number of float4 per lane, all loads in flight before the first use
        const float4 *g4 = reinterpret_cast<const float4 *>(P.g_sh + span0);
        float4 t[NF_LANE];
#pragma unroll
        for (int q = 0; q < NF_LANE; q++) { const uint32_t f = lane + 32u * q; if (f < NF_FULL) t[q] = __ldg(g4 + f); }
#pragma unroll
        for (int q = 0; q < NF_LANE; q++) {
            const uint32_t f = lane + 32u * q;
            if (f < NF_FULL) {
                const uint32_t e = f * 4;
                const float tv[4] = {t[q].x, t[q].y, t[q].z, t[q].w};
#pragma unroll
                for (int c = 0; c < 4; c++) sg[((e + c) / KF) * SROW + (e + c) % KF] = tv[c];
            }
        }
    } else if (vec) {
        const float4 *g4 = reinterpret_cast<const float4 *>(P.g_sh + span0);
        for (uint32_t f = lane; f < (total >> 2); f += 32) {
            const float4 t = __ldg(g4 + f);
            const uint32_t e = f * 4;
            const float tv[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
            for (int q = 0; q < 4; q++) sg[((e + q) / KF) * SROW + (e + q) % KF] = tv[q];
        }
    } else {
        for (uint32_t e = lane; e < total; e += 32) sg[(e / KF) * SROW + e % KF] = __ldg(P.g_sh + span0 + e);
    }
    __syncwarp();
    // ---- row-mean second moment (adam_scaled.rs:152-165), in column order
    if (valid) {
        float s = 0.0f;
#pragma unroll
        for (int c = 0; c < KF; c++) { const float gv = sg[lane * SROW + c]; s += gv * gv; }
        const float vv = adam_v(P.first ? 0.0f : P.v_sh[i], s / (float)KF, P);
        P.v_sh[i] = vv;
        s_v[wid][lane] = adam_inv_denom(vv, P);   // one reciprocal per row, shared by its 3K coefficients
    }
    __syncwarp();
    // ---- element-wise update of the warp's span, coalesced
    float *ps = P.sh + span0, *ms = P.m_sh + span0;
    auto update4 = [&](float4 &pp, float4 &mm, uint32_t f) {
        float *pe = &pp.x, *me = &mm.x;
        const uint32_t e = f * 4;
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const uint32_t r = (e + q) / KF, c = (e + q) % KF;
            me[q] = adam_m(me[q], sg[r * SROW + c], P);
            pe[q] = adam_p(pe[q], me[q], s_v[wid][r], c < 3 ? P.lr_sh_dc : P.lr_sh_rest, P);
        }
    };
    if (rows == 32u) {
        float4 *p4 = reinterpret_cast<float4 *>(ps), *m4 = reinterpret_cast<float4 *>(ms);
        constexpr int GROUP = 4;   // float4 pairs in flight per lane
#pragma unroll
        for (int q0 = 0; q0 < NF_LANE; q0 += GROUP) {
            float4 pp[GROUP], mm[GROUP];
#pragma unroll
            for (int q = 0; q < GROUP; q++) {
                const uint32_t f = lane + 32u * (q0 + q);
                if (q0 + q < NF_LANE && f < NF_FULL) {
                    pp[q] = p4[f];
                    mm[q] = P.first ? make_float4(0.f, 0.f, 0.f, 0.f) : m4[f];
                }
            }
#pragma unroll
            for (int q = 0; q < GROUP; q++) {
                const uint32_t f = lane + 32u * (q0 + q);
                if (q0 + q < NF_LANE && f < NF_FULL) {
                    update4(pp[q], mm[q], f);
                    m4[f] = mm[q];
                    p4[f] = pp[q];
                }
            }
        }
    } else if (vec) {
        float4 *p4 = reinterpret_cast<float4 *>(ps), *m4 = reinterpret_cast<float4 *>(ms);
        for (uint32_t f = lane; f < (total >> 2); f += 32) {
            float4 pp = p4[f];
            float4 mm = P.first ? make_float4(0.f, 0.f, 0.f, 0.f) : m4[f];
            update4(pp, mm, f);
            m4[f] = mm;
            p4[f] = pp;
        }
    } else {
        for (uint32_t e = lane; e < total; e += 32) {
            const uint32_t r = e / KF, c = e % KF;
            const float mm = adam_m(P.first ? 0.0f : ms[e], sg[r * SROW + c], P);
            ms[e] = mm;
            ps[e] = adam_p(ps[e], mm, s_v[wid][r], c < 3 ? P.lr_sh_dc : P.lr_sh_rest, P);
        }
    }
}

template <int DEG>
static cudaError_t launch_deg(cudaStream_t s, const UpdateParams &P, bool factored, int part) {
    const unsigned grid = (P.count + UP_THREADS - 1) / UP_THREADS;   // 32 rows per warp
    if (!factored) train_update_kernel<DEG, false, 0><<<grid, UP_THREADS, 0, s>>>(P);
    else if (part == 1) train_update_kernel<DEG, true, 1><<<grid, UP_THREADS, 0, s>>>(P);
    else if (part == 2) train_update_kernel<DEG, true, 2><<<grid, UP_THREADS, 0, s>>>(P);
    else train_update_kernel<DEG, true, 0><<<grid, UP_THREADS, 0, s>>>(P);
    return cudaGetLastError();
}

cudaError_t launch_train_update(cudaStream_t s, int deg, const UpdateParams &P, bool factored, int part) {
    if (P.count == 0) return cudaSuccess;
    switch (deg) {
        case 0: return launch_deg<0>(s, P, factored, part);
        case 1: return launch_deg<1>(s, P, factored, part);
        case 2: return launch_deg<2>(s, P, factored, part);
        case 3: return launch_deg<3>(s, P, factored, part);
        case 4: return launch_deg<4>(s, P, factored, part);
    }
    return cudaErrorInvalidValue;
}

}  // namespace bg
