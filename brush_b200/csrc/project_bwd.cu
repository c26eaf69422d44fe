// project_bwd.cu -- chain the per-splat screen-space gradients back to the Gaussian parameters.
// Replaces project_backwards_kernel (bwd/kernels/project_backwards.rs:99-254) and its helpers
// (apply_normalize_vjp :18-50, quat_to_mat_vjp :53-77, inverse2x2_vjp :84-97), the SH VJPs
// (kernels/sh.rs:138-355) and the pinhole projection VJP (kernels/camera_model/pinhole.rs:58-123).
//
// The reference walks the visible splats in depth order and scatters into zero-initialised dense
// outputs (a memset of (48+12K) N bytes plus a scattered write).  Here the kernel walks ALL
// Gaussians in index order using the inverse map compact_from_global_gid written by the forward:
// parameter reads and gradient writes are fully sequential, every output row is written exactly
// once (zeros where the reference leaves the zero fill), and only the 40-byte v_combined row is
// gathered.  HBM-bound: (88+12K) V + (48+12K) N bytes (SURVEY.md 8d).
#include "bg_project.cuh"
#include "bg_sh.cuh"
#include "bg_launch.cuh"

namespace bg {

__device__ __forceinline__ Q4 normalize_vjp(Q4 q, Q4 g) {
    float lsq = dot(q, q);
    float l = sqrtf(lsq);
    float inv = 1.0f / (l * lsq);
    float cc0 = -q.w * q.x, cc1 = -q.x * q.y, cc2 = -q.y * q.w;
    float cs0 = -q.w * q.z, cs1 = -q.x * q.z, cs2 = -q.y * q.z;
    float sw = q.w * q.w, sx = q.x * q.x, sy = q.y * q.y, sz = q.z * q.z;
    Q4 r;
    r.w = ((lsq - sw) * g.w + cc0 * g.x + cc2 * g.y + cs0 * g.z) * inv;
    r.x = (cc0 * g.w + (lsq - sx) * g.x + cc1 * g.y + cs1 * g.z) * inv;
    r.y = (cc2 * g.w + cc1 * g.x + (lsq - sy) * g.y + cs2 * g.z) * inv;
    r.z = (cs0 * g.w + cs1 * g.x + cs2 * g.y + (lsq - sz) * g.z) * inv;
    return r;
}

__device__ __forceinline__ Q4 quat_to_mat_vjp(Q4 q, M3 v) {
    float w_grad = q.x * (v.c1.z - v.c2.y) + q.y * (v.c2.x - v.c0.z) + q.z * (v.c0.y - v.c1.x);
    float x_grad = -2.0f * q.x * (v.c1.y + v.c2.z) + q.y * (v.c0.y + v.c1.x) + q.z * (v.c0.z + v.c2.x) +
                   q.w * (v.c1.z - v.c2.y);
    float y_grad = q.x * (v.c0.y + v.c1.x) - 2.0f * q.y * (v.c0.x + v.c2.z) + q.z * (v.c1.z + v.c2.y) +
                   q.w * (v.c2.x - v.c0.z);
    float z_grad = q.x * (v.c0.z + v.c2.x) + q.y * (v.c1.z + v.c2.y) - 2.0f * q.z * (v.c0.x + v.c1.y) +
                   q.w * (v.c0.y - v.c1.x);
    Q4 r; r.w = 2.0f * w_grad; r.x = 2.0f * x_grad; r.y = 2.0f * y_grad; r.z = 2.0f * z_grad;
    return r;
}

__device__ __forceinline__ S2 inverse2x2_vjp(S2 minv, S2 v) {
    float t00 = -minv.c00 * v.c00 + -minv.c01 * v.c01;
    float t01 = -minv.c01 * v.c00 + -minv.c11 * v.c01;
    float t10 = -minv.c00 * v.c01 + -minv.c01 * v.c11;
    float t11 = -minv.c01 * v.c01 + -minv.c11 * v.c11;
    S2 r;
    r.c00 = t00 * minv.c00 + t10 * minv.c01;
    r.c01 = t01 * minv.c00 + t11 * minv.c01;
    r.c11 = t01 * minv.c01 + t11 * minv.c11;
    return r;
}

__device__ __forceinline__ V3 projection_vjp_pinhole(M23 jac, V3 mean_c, S3 cov_c, const BgCamera &u, S2 v_cov2d,
                                                     V2 v_mean2d) {
    float fx = u.fx, fy = u.fy;
    float mx = mean_c.x, my = mean_c.y, mz = mean_c.z;
    float inv_z = 1.0f / mz;
    float mx_raw = mx * inv_z, my_raw = my * inv_z;
    float mx_rz = clampf(mx_raw, u.lim_neg_x, u.lim_pos_x);
    float my_rz = clampf(my_raw, u.lim_neg_y, u.lim_pos_y);
    bool in_x = mx_raw <= u.lim_pos_x && mx_raw >= u.lim_neg_x;
    bool in_y = my_raw <= u.lim_pos_y && my_raw >= u.lim_neg_y;
    float inv_z2 = inv_z * inv_z, inv_z3 = inv_z2 * inv_z;
    float v_mx = fx * inv_z * v_mean2d.x;
    float v_my = fy * inv_z * v_mean2d.y;
    float v_mz = -(fx * mx * v_mean2d.x + fy * my * v_mean2d.y) * inv_z2;
    M23 tmp = mul(v_cov2d, jac);
    float vj00 = 2.0f * dot(row0(tmp), row0(cov_c));
    float vj11 = 2.0f * dot(row1(tmp), row1(cov_c));
    float vj20 = 2.0f * dot(row0(tmp), row2(cov_c));
    float vj21 = 2.0f * dot(row1(tmp), row2(cov_c));
    float tx = mz * mx_rz, ty = mz * my_rz;
    if (in_x) v_mx += -fx * inv_z2 * vj20; else v_mz += -fx * inv_z3 * vj20 * tx;
    if (in_y) v_my += -fy * inv_z2 * vj21; else v_mz += -fy * inv_z3 * vj21 * ty;
    v_mz += -fx * inv_z2 * vj00 - fy * inv_z2 * vj11 + 2.0f * fx * tx * inv_z3 * vj20 + 2.0f * fy * ty * inv_z3 * vj21;
    return mk3(v_mx, v_my, v_mz);
}

// d(colour)/d(view dir) contracted with vc; S[k] = coeff_k . vc  (kernels/sh.rs:138-259)
template <int DEG>
__device__ __forceinline__ V3 sh_viewdir_vjp(const float *S, V3 v) {
    float gx = 0.0f, gy = 0.0f, gz = 0.0f;
    const float x = v.x, y = v.y, z = v.z;
    if (DEG >= 1) {
        const float f0a = 0.4886025f;
        gx += -f0a * S[3];
        gy += -f0a * S[1];
        gz += f0a * S[2];
    }
    if (DEG >= 2) {
        const float c2 = -1.0925485f, f1a = 0.54627424f;
        gx += 2.0f * f1a * y * S[4] + c2 * z * S[7] + 2.0f * f1a * x * S[8];
        gy += 2.0f * f1a * x * S[4] + c2 * z * S[5] - 2.0f * f1a * y * S[8];
        gz += c2 * y * S[5] + 2.0f * 0.9461747f * z * S[6] + c2 * x * S[7];
    }
    const float z2 = z * z, x2 = x * x, y2 = y * y;
    if (DEG >= 3) {
        const float f2a = -0.5900436f, c1b = 1.4453057f, c0c = -2.285229f;
        float f1b = c1b * z;
        float f0c = c0c * z2 + 0.4570458f;
        float f0c_dz = 2.0f * c0c * z;
        float d12_z = 3.0f * 1.8658817f * z2 - 1.119529f;
        gx += f2a * 6.0f * x * y * S[9] + 2.0f * f1b * y * S[10] + f0c * S[13] + 2.0f * f1b * x * S[14] +
              f2a * 3.0f * (x2 - y2) * S[15];
        gy += f2a * 3.0f * (x2 - y2) * S[9] + 2.0f * f1b * x * S[10] + f0c * S[11] + (-2.0f) * f1b * y * S[14] +
              f2a * (-6.0f) * x * y * S[15];
        gz += 2.0f * c1b * x * y * S[10] + f0c_dz * y * S[11] + d12_z * S[12] + f0c_dz * x * S[13] +
              c1b * (x2 - y2) * S[14];
    }
    if (DEG >= 4) {
        float fc1 = x2 - y2, fs1 = 2.0f * x * y;
        float fc2 = x * fc1 - y * fs1, fs2 = x * fs1 + y * fc1;
        float f0d = z * (-4.683326f * z2 + 2.0071396f);
        float f0d_dz = -14.049978f * z2 + 2.0071396f;
        float f1c = 3.3116114f * z2 - 0.47308735f;
        float f1c_dz = 2.0f * 3.3116114f * z;
        const float f2b_c = -1.7701308f;
        float f2b = f2b_c * z;
        const float f3a = 0.62583575f;
        float p_sh12 = z * (1.8658817f * z2 - 1.119529f);
        float dp12 = 3.0f * 1.8658817f * z2 - 1.119529f;
        float dp6 = 2.0f * 0.9461747f * z;
        float dp20 = 1.9843135f * (p_sh12 + z * dp12) - 1.0062306f * dp6;
        gx += f3a * 4.0f * fs2 * S[16] + f2b * 3.0f * fs1 * S[17] + f1c * 2.0f * y * S[18] + f0d * S[21] +
              f1c * 2.0f * x * S[22] + f2b * 3.0f * fc1 * S[23] + f3a * 4.0f * fc2 * S[24];
        gy += f3a * 4.0f * fc2 * S[16] + f2b * 3.0f * fc1 * S[17] + f1c * 2.0f * x * S[18] + f0d * S[19] +
              f1c * (-2.0f) * y * S[22] + f2b * (-3.0f) * fs1 * S[23] + f3a * (-4.0f) * fs2 * S[24];
        gz += f2b_c * fs2 * S[17] + f1c_dz * fs1 * S[18] + f0d_dz * y * S[19] + dp20 * S[20] + f0d_dz * x * S[21] +
              f1c_dz * fc1 * S[22] + f2b_c * fc2 * S[23];
    }
    return mk3(gx, gy, gz);
}

constexpr int PB_THREADS = 128;
constexpr int PB_WARPS = PB_THREADS / 32;

// Row stride, in floats, of the per-warp SH slices in shared memory.  Rows that are a multiple of 16 bytes are
// accessed with 128-bit shared loads and stores, which run in phases of 8 lanes: an odd number of float4s per row puts
// those 8 lanes on 8 distinct 4-bank groups, so KF = 12 stays as it is and KF = 48 is padded to 52.  Odd rows
// (KF = 3, 27, 75) are accessed one float at a time, which an odd stride keeps conflict-free.
__host__ __device__ constexpr int pb_slice_stride(int kf) { return (kf % 4 != 0 || (kf / 4) % 2 == 1) ? kf : kf + 4; }

template <bool MIP, int DEG, bool DIST>
__global__ void __launch_bounds__(PB_THREADS)
project_bwd_kernel(const float *__restrict__ transforms, const float *__restrict__ sh,
                   const float *__restrict__ raw_opac, const uint32_t *__restrict__ cgid_from_gid,
                   const float *__restrict__ v_combined, uint32_t n, BgCamera u, float *__restrict__ v_transforms,
                   float *__restrict__ v_sh, float *__restrict__ v_raw_opac, float *__restrict__ v_refine,
                   float *__restrict__ v_color_out /* nullable: factored mode, see sh_grad_from_views_kernel */) {
    constexpr int K = (DEG + 1) * (DEG + 1);
    constexpr int KF = K * 3;
    // The SH rows move through a shared-memory slice of 32 rows per warp, so that neither direction makes a warp
    // touch 32 different 128-byte lines per instruction, as one row per thread straight from global memory would.
    //   in:  a row that is a multiple of 16 bytes (K = 4, 16) comes in by its own TMA bulk copy (cp.async.bulk, SASS
    //        UBLKCP), issued by one lane per warp as soon as the v_combined gather says the row is read at all, and
    //        lands while the transform row and the projection chain are worked through.  Culled and zero-gradient
    //        rows are never fetched.  Odd rows (K = 9, 25) keep the per-thread load.
    //   out: each lane leaves its SH-gradient row (zeros included) in its slot, then the warp writes its contiguous
    //        32-row span with whole-line stores (degree >= 1; a degree-0 row goes straight out).
    constexpr bool VEC4 = (KF % 4) == 0;
    constexpr bool BULK_IN = VEC4 && DEG > 0;   // degree 0 has no view-direction dependence: its row is never read
    // degree 0 rows are 12 bytes: a warp's direct stores of them already cover one contiguous 384-byte span
    constexpr bool STAGE_OUT = DEG > 0;
    constexpr int ST = pb_slice_stride(KF);
    __shared__ __align__(16) float s_vt[PB_THREADS * 10];
    __shared__ __align__(16) float s_sh[PB_THREADS * ST];
    __shared__ unsigned long long s_bar[PB_WARPS];
    const uint32_t base = blockIdx.x * PB_THREADS;
    const uint32_t rows = min((uint32_t)PB_THREADS, n - base);
    const uint32_t gid = base + threadIdx.x;
    const bool in_range = threadIdx.x < rows;
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t wbase = base + warp * 32u;   // first Gaussian of this warp's slice
    float *slice = s_sh + warp * 32u * ST;
    float *my_row = slice + lane * ST;
    if (BULK_IN) {
        if (lane == 0) mbar_init(&s_bar[warp], 1);
        __syncwarp();
    }

    uint32_t cg = 0xFFFFFFFFu;
    float rg[10];
#pragma unroll
    for (int i = 0; i < 10; i++) rg[i] = 0.0f;
    if (in_range) {
        cg = __ldg(cgid_from_gid + gid);
        if (cg != 0xFFFFFFFFu) {
            const float2 *p = reinterpret_cast<const float2 *>(v_combined + (size_t)cg * BG_VCOMBINED_STRIDE);
#pragma unroll
            for (int i = 0; i < 5; i++) { float2 t = __ldg(p + i); rg[2 * i] = t.x; rg[2 * i + 1] = t.y; }
        }
    }
    bool any = false;
#pragma unroll
    for (int i = 0; i < 10; i++) any = any || (rg[i] != 0.0f);
    if (BULK_IN) {
        const uint32_t mask = __ballot_sync(0xffffffffu, any);
        if (lane == 0 && mask != 0u) {
            const float *src = sh + (size_t)wbase * KF;
            mbar_expect_tx(&s_bar[warp], (uint32_t)__popc(mask) * (KF * 4u));
            for (uint32_t m = mask; m != 0u; m &= m - 1u) {
                const uint32_t r = (uint32_t)__ffs(m) - 1u;
                tma_bulk_g2s(slice + r * ST, src + (size_t)r * KF, KF * 4u, &s_bar[warp]);
            }
        }
    }

    float vt[10];
#pragma unroll
    for (int i = 0; i < 10; i++) vt[i] = 0.0f;
    float v_opac_out = 0.0f, v_refine_out = 0.0f;
    float Y[K];
    V3 v_color = mk3(rg[5], rg[6], rg[7]);
#pragma unroll
    for (int i = 0; i < K; i++) Y[i] = 0.0f;

    if (any) {
        const float2 *t2 = reinterpret_cast<const float2 *>(transforms + (size_t)gid * 10);
        float2 a0 = __ldg(t2), a1 = __ldg(t2 + 1), a2 = __ldg(t2 + 2), a3 = __ldg(t2 + 3), a4 = __ldg(t2 + 4);
        V3 mean = mk3(a0.x, a0.y, a1.x);
        Q4 qu; qu.w = a1.y; qu.x = a2.x; qu.y = a2.y; qu.z = a3.x;
        V3 scl = mk3(det_expf(a3.y), det_expf(a4.x), det_expf(a4.y));
        Q4 quat = normalize(qu);

        V3 u_world = sub(mean, mk3(u.cam_pos[0], u.cam_pos[1], u.cam_pos[2]));
        float u_len = length(u_world);
        V3 vdir = scale(u_world, 1.0f / u_len);
        sh_basis<DEG>(vdir, Y);

        V3 mean_c = world_to_cam(mean, u);
        M3 rm = quat_to_mat3(quat);
        M3 m = mul_diag(rm, scl);
        S2 raw_cov = calc_cov2d<DIST>(scl, quat, mean_c, u);
        float comp;
        S2 cov = compensate_cov2d<MIP>(raw_cov, comp);
        float osig = det_sigmoid(__ldg(raw_opac + gid));
        v_opac_out = comp * rg[8] * osig * (1.0f - osig);
        float rclean = is_finite(rg[9]) ? rg[9] : 0.0f;
        v_refine_out = clampf(rclean, 0.0f, 1.0e32f);

        S2 conic = inverse(cov);
        S2 v_inv; v_inv.c00 = rg[2]; v_inv.c01 = rg[3] * 0.5f; v_inv.c11 = rg[4];
        S2 v_cov2d = inverse2x2_vjp(conic, v_inv);
        S3 covar = outer_self(m);
        M3 view_rot = view_rotation(u);
        S3 cov_c = congruence(covar, view_rot);
        M23 jac = project_jacobian<DIST>(mean_c, u);
        V3 v_mean_c = DIST ? projection_vjp_distorted(jac, mean_c, cov_c, u, v_cov2d, mk2(rg[0], rg[1]))
                           : projection_vjp_pinhole(jac, mean_c, cov_c, u, v_cov2d, mk2(rg[0], rg[1]));
        S3 vcc = tcongruence(jac, v_cov2d);

        // the SH row is needed only from here on, which gives its bulk copy the whole chain above to land
        float S[K];
        if (DEG > 0) {   // S_k = coeff_k . v_color
            float row[KF];
            if (BULK_IN) {
                mbar_wait(&s_bar[warp], 0);
#pragma unroll
                for (int q = 0; q < KF / 4; q++) {
                    float4 t = reinterpret_cast<const float4 *>(my_row)[q];
                    row[4 * q] = t.x; row[4 * q + 1] = t.y; row[4 * q + 2] = t.z; row[4 * q + 3] = t.w;
                }
            } else {
                const float *src = sh + (size_t)gid * KF;
#pragma unroll
                for (int q = 0; q < KF; q++) row[q] = __ldg(src + q);
            }
#pragma unroll
            for (int k = 0; k < K; k++) S[k] = dot(mk3(row[3 * k], row[3 * k + 1], row[3 * k + 2]), v_color);
        } else {
            S[0] = 0.0f;
        }
        V3 v_v_sh = sh_viewdir_vjp<DEG>(S, vdir);
        float vdv = dot(vdir, v_v_sh);
        V3 v_mean_sh = scale(sub(v_v_sh, scale(vdir, vdv)), 1.0f / u_len);

        V3 v_mean = add(tmul(view_rot, v_mean_c), v_mean_sh);
        M3 v_m = mul(scale(tcongruence(vcc, view_rot), 2.0f), m);
        V3 v_scale = mk3(dot(rm.c0, v_m.c0) * scl.x, dot(rm.c1, v_m.c1) * scl.y, dot(rm.c2, v_m.c2) * scl.z);
        Q4 q_grad = quat_to_mat_vjp(quat, mul_diag(v_m, scl));
        Q4 v_q = normalize_vjp(qu, q_grad);
        vt[0] = v_mean.x; vt[1] = v_mean.y; vt[2] = v_mean.z;
        vt[3] = v_q.w; vt[4] = v_q.x; vt[5] = v_q.y; vt[6] = v_q.z;
        vt[7] = v_scale.x; vt[8] = v_scale.y; vt[9] = v_scale.z;
    }
    const bool factored = v_color_out != nullptr;
    if (!factored && !STAGE_OUT) {
        if (in_range) {
            float *dst = v_sh + (size_t)gid * KF;
            const float yk = any ? Y[0] : 0.0f;
            dst[0] = v_color.x * yk; dst[1] = v_color.y * yk; dst[2] = v_color.z * yk;
        }
    } else if (!factored) {
        // this lane's row of the dense gradient into its slot (a row it read above has been consumed by then), then
        // the warp's rows out as one contiguous span
        if (in_range) {
            float row[KF];
#pragma unroll
            for (int k = 0; k < K; k++) {
                float yk = any ? Y[k] : 0.0f;
                row[3 * k] = v_color.x * yk;
                row[3 * k + 1] = v_color.y * yk;
                row[3 * k + 2] = v_color.z * yk;
            }
            if (VEC4) {
#pragma unroll
                for (int q = 0; q < KF / 4; q++)
                    reinterpret_cast<float4 *>(my_row)[q] = make_float4(row[4 * q], row[4 * q + 1], row[4 * q + 2], row[4 * q + 3]);
            } else {
#pragma unroll
                for (int q = 0; q < KF; q++) my_row[q] = row[q];
            }
        }
        __syncwarp();
        if (wbase < n) {
            const uint32_t wrows = min(32u, n - wbase);
            float *dst = v_sh + (size_t)wbase * KF;
            if (VEC4) {   // 16-byte aligned: v_sh is, and the span starts 32 * KF floats into it
                constexpr uint32_t Q = KF / 4;
#pragma unroll 4
                for (uint32_t f = lane; f < wrows * Q; f += 32u) {
                    const uint32_t r = f / Q, c = f - r * Q;
                    reinterpret_cast<float4 *>(dst)[f] = *reinterpret_cast<const float4 *>(slice + r * ST + 4u * c);
                }
            } else {      // odd rows are stored unpadded: the slot layout is the span's
#pragma unroll 4
                for (uint32_t j = lane; j < wrows * KF; j += 32u) dst[j] = slice[j];
            }
        }
    } else if (in_range) {  // the SH gradient of one view is the outer product Y(dir) x v_color: ship only v_color
        float *dst = v_color_out + (size_t)gid * 3;
        dst[0] = any ? v_color.x : 0.0f; dst[1] = any ? v_color.y : 0.0f; dst[2] = any ? v_color.z : 0.0f;
    }
    if (in_range) {
#pragma unroll
        for (int i = 0; i < 10; i++) s_vt[threadIdx.x * 10 + i] = vt[i];
        v_raw_opac[gid] = v_opac_out;
        v_refine[gid] = v_refine_out;
    }
    __syncthreads();
    {   // coalesced write-out of the [rows,10] gradient block
        float *dt = v_transforms + (size_t)base * 10;
        for (uint32_t j = threadIdx.x; j < rows * 10; j += PB_THREADS) dt[j] = s_vt[j];
    }
}

// View-factored SH gradient for data-parallel training.  v_sh of ONE view is rank one per Gaussian:
// v_sh[g,k,:] = Y_k(dir(mean_g, cam_v)) * v_color_v[g,:] (kernels/sh.rs:265-355).  Instead of all-reducing
// the dense [n,K,3] tensor (192 B per Gaussian at K=16), ranks all-gather the 12-byte v_color rows of
// their views and every rank rebuilds sum_v Y_k(dir_v) v_color_v locally, in view order (so all ranks
// get bit-identical sums).  Exchange volume drops 16x for this tensor; the result equals the all-reduce
// up to f32 summation order.
struct ViewCams { float pos[16][3]; uint32_t count; };

template <int DEG>
__global__ void __launch_bounds__(PB_THREADS)
sh_grad_from_views_kernel(const float *__restrict__ transforms, const float *__restrict__ v_color_all /* [views,n,3] */,
                          uint32_t n, ViewCams cams, float out_scale, float *__restrict__ v_sh, size_t view_stride) {
    constexpr int K = (DEG + 1) * (DEG + 1);
    constexpr int KF = K * 3;
    constexpr int STRIDE = (KF % 2 == 0) ? KF + 1 : KF;
    __shared__ float s_stage[PB_THREADS * STRIDE];
    const uint32_t base = blockIdx.x * PB_THREADS;
    const uint32_t rows = min((uint32_t)PB_THREADS, n - base);
    const uint32_t gid = base + threadIdx.x;
    if (threadIdx.x < rows) {
        float acc[KF];
#pragma unroll
        for (int i = 0; i < KF; i++) acc[i] = 0.0f;
        const float *t = transforms + (size_t)gid * 10;
        const V3 mean = mk3(__ldg(t), __ldg(t + 1), __ldg(t + 2));
        for (uint32_t v = 0; v < cams.count; v++) {
            const float *vc = v_color_all + (size_t)v * view_stride + (size_t)gid * 3;
            const float cr = __ldg(vc), cg = __ldg(vc + 1), cb = __ldg(vc + 2);
            if (cr == 0.0f && cg == 0.0f && cb == 0.0f) continue;
            V3 u_world = sub(mean, mk3(cams.pos[v][0], cams.pos[v][1], cams.pos[v][2]));
            V3 vdir = scale(u_world, 1.0f / length(u_world));
            float Y[K];
            sh_basis<DEG>(vdir, Y);
#pragma unroll
            for (int k = 0; k < K; k++) {
                acc[3 * k] += cr * Y[k];
                acc[3 * k + 1] += cg * Y[k];
                acc[3 * k + 2] += cb * Y[k];
            }
        }
        float *row = s_stage + threadIdx.x * STRIDE;
#pragma unroll
        for (int i = 0; i < KF; i++) row[i] = acc[i] * out_scale;
    }
    __syncthreads();
    float *dst = v_sh + (size_t)base * KF;
    const uint32_t total = rows * KF;
    for (uint32_t j = threadIdx.x; j < total; j += PB_THREADS) {
        uint32_t r = j / KF, c = j - r * KF;
        dst[j] = s_stage[r * STRIDE + c];
    }
}

cudaError_t launch_sh_grad_from_views(cudaStream_t s, int deg, const float *transforms, const float *v_color_all,
                                      uint32_t n, const float *cam_pos_host, uint32_t views, float out_scale,
                                      float *v_sh, size_t view_stride) {
    if (n == 0) return cudaSuccess;
    if (views > 16) return cudaErrorInvalidValue;
    ViewCams cams;
    cams.count = views;
    for (uint32_t v = 0; v < views; v++)
        for (int i = 0; i < 3; i++) cams.pos[v][i] = cam_pos_host[v * 3 + i];
    const int grid = (int)((n + PB_THREADS - 1) / PB_THREADS);
    switch (deg) {
        case 0: sh_grad_from_views_kernel<0><<<grid, PB_THREADS, 0, s>>>(transforms, v_color_all, n, cams, out_scale, v_sh, view_stride); break;
        case 1: sh_grad_from_views_kernel<1><<<grid, PB_THREADS, 0, s>>>(transforms, v_color_all, n, cams, out_scale, v_sh, view_stride); break;
        case 2: sh_grad_from_views_kernel<2><<<grid, PB_THREADS, 0, s>>>(transforms, v_color_all, n, cams, out_scale, v_sh, view_stride); break;
        case 3: sh_grad_from_views_kernel<3><<<grid, PB_THREADS, 0, s>>>(transforms, v_color_all, n, cams, out_scale, v_sh, view_stride); break;
        case 4: sh_grad_from_views_kernel<4><<<grid, PB_THREADS, 0, s>>>(transforms, v_color_all, n, cams, out_scale, v_sh, view_stride); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

template <bool MIP>
static cudaError_t launch_pb_deg(cudaStream_t s, int deg, const float *transforms, const float *sh,
                                 const float *raw_opac, const uint32_t *cgid_from_gid, const float *v_combined,
                                 uint32_t n, const BgCamera &u, float *v_transforms, float *v_sh, float *v_raw_opac,
                                 float *v_refine, float *v_color_out) {
    const int grid = (int)((n + PB_THREADS - 1) / PB_THREADS);
    const bool dist = u.camera_model != BG_CAMERA_PINHOLE;
#define BG_LAUNCH_PB(D)                                                                                                 \
    if (dist) project_bwd_kernel<MIP, D, true><<<grid, PB_THREADS, 0, s>>>(transforms, sh, raw_opac, cgid_from_gid, v_combined, n, u, \
                                                           v_transforms, v_sh, v_raw_opac, v_refine, v_color_out);      \
    else project_bwd_kernel<MIP, D, false><<<grid, PB_THREADS, 0, s>>>(transforms, sh, raw_opac, cgid_from_gid, v_combined, n, u, \
                                                           v_transforms, v_sh, v_raw_opac, v_refine, v_color_out)
    switch (deg) {
        case 0: BG_LAUNCH_PB(0); break;
        case 1: BG_LAUNCH_PB(1); break;
        case 2: BG_LAUNCH_PB(2); break;
        case 3: BG_LAUNCH_PB(3); break;
        case 4: BG_LAUNCH_PB(4); break;
        default: return cudaErrorInvalidValue;
    }
#undef BG_LAUNCH_PB
    return cudaGetLastError();
}

cudaError_t launch_project_bwd(cudaStream_t s, bool mip, int deg, const float *transforms, const float *sh,
                               const float *raw_opac, const uint32_t *cgid_from_gid, const float *v_combined,
                               uint32_t n, const BgCamera &u, float *v_transforms, float *v_sh, float *v_raw_opac,
                               float *v_refine, float *v_color_out) {
    if (n == 0) return cudaSuccess;
    return mip ? launch_pb_deg<true>(s, deg, transforms, sh, raw_opac, cgid_from_gid, v_combined, n, u, v_transforms,
                                     v_sh, v_raw_opac, v_refine, v_color_out)
               : launch_pb_deg<false>(s, deg, transforms, sh, raw_opac, cgid_from_gid, v_combined, n, u, v_transforms,
                                      v_sh, v_raw_opac, v_refine, v_color_out);
}

// Depth adjoint, after project_bwd_kernel (DESIGN §4.6): z_i = R[2,:] . mean_i + t_z, so the blend's v_z[cgid] adds
// v_z R[2,:] to v_transforms[gid, 0:3].  Every Gaussian owns its row: no atomics, deterministic.  A zero v_z leaves the
// row's bits as they are (adding +0 would turn a -0 into +0).
__global__ void __launch_bounds__(256)
depth_to_means_kernel(const uint32_t *__restrict__ cgid_from_gid, const float *__restrict__ v_z, uint32_t n, float r0,
                      float r1, float r2, float *__restrict__ v_transforms) {
    const uint32_t gid = blockIdx.x * 256u + threadIdx.x;
    if (gid >= n) return;
    const uint32_t cg = __ldg(cgid_from_gid + gid);
    if (cg == 0xFFFFFFFFu) return;
    const float vz = __ldg(v_z + cg);
    if (vz == 0.0f) return;
    float *t = v_transforms + (size_t)gid * 10;
    t[0] += vz * r0;
    t[1] += vz * r1;
    t[2] += vz * r2;
}

cudaError_t launch_depth_to_means(cudaStream_t s, const uint32_t *cgid_from_gid, const float *v_z, uint32_t n,
                                  const BgCamera &u, float *v_transforms) {
    if (n == 0) return cudaSuccess;
    depth_to_means_kernel<<<(n + 255) / 256, 256, 0, s>>>(cgid_from_gid, v_z, n, u.viewmat[2], u.viewmat[5], u.viewmat[8],
                                                          v_transforms);
    return cudaGetLastError();
}

}  // namespace bg
