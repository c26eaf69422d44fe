// optim.cu -- fused optimiser kernels (pure HBM streaming).
//   adam_kernel / adam_rowreduce_kernel <- AdamScaled::step + transform (brush-train/src/adam_scaled.rs:75-165):
//       m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2  (g^2 replaced by its row mean when reduce_v,
//       adam_scaled.rs:99-104,152-165);  first step initialises m,v from g alone;
//       p -= (lr * scale[col]) * (m / bc1) / (sqrt(v / bc2) + eps).
//     The reference issues ~25 separate burn tensor ops per parameter; here one pass reads p,g,m,v
//     and writes p,m,v (28 B/element, 20 B/element + 8 B/row when v is row-reduced).
//   refine_stats_noise_kernel <- RefineRecord::gather_stats (brush-train/src/stats.rs:40-50) and the
//       mean-noise update (brush-train/src/train.rs:389-416).
//   min_scale_kernel / fold_min_scale_{fwd,bwd}_kernel <- compute_min_scale (train.rs:102-125) and
//       fold_min_scale (brush-render/src/gaussian_splats.rs:86-111): the Mip-Splatting 3D filter floor.
#include <algorithm>

#include "bg_adam.cuh"
#include "bg_common.cuh"
#include "bg_fold.cuh"
#include "bg_rng.cuh"
#include "bg_launch.cuh"

namespace bg {

// Upper bound on the CTAs of the grid-stride kernels below: 16 per SM of an H100 SXM (132 SMs).  Results do not
// depend on the grid size.
constexpr uint64_t GRID_CAP = 132ull * 16;

__global__ void __launch_bounds__(256)
adam_kernel(float *__restrict__ p, const float *__restrict__ g, float *__restrict__ m, float *__restrict__ v,
            uint64_t total, uint32_t cols, const float *__restrict__ lr_scale, AdamConsts k) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        float gg = __ldg(g + i);
        float step = lr_scale ? __ldg(lr_scale + (uint32_t)(i % cols)) * k.lr : k.lr;
        adam_element(p[i], gg, m[i], v[i], k, step);
    }
}

// Row-reduced second moment.  One CTA handles AR_ROWS rows: the g tile is staged in shared memory with
// coalesced (128-bit when the tile allows) loads, four threads per row form the row mean of g^2 in a
// fixed order (12-column partial sums in column order, then a two-step shuffle tree: deterministic, so
// data-parallel ranks stay bit-identical), then all threads update m and p element-wise.
constexpr int AR_ROWS = 64;

__global__ void __launch_bounds__(256)
adam_rowreduce_kernel(float *__restrict__ p, const float *__restrict__ g, float *__restrict__ m,
                      float *__restrict__ v, uint64_t rows, uint32_t cols, const float *__restrict__ lr_scale,
                      AdamConsts k) {
    extern __shared__ __align__(16) float s_g[];   // AR_ROWS * cols (dense copy of the tile)
    __shared__ float s_v[AR_ROWS];
    const uint64_t row0 = (uint64_t)blockIdx.x * AR_ROWS;
    const uint32_t nrows = (uint32_t)min((uint64_t)AR_ROWS, rows - row0);
    const uint64_t base = row0 * cols;
    const uint32_t total = nrows * cols;
    const bool vec = ((base | total) & 3ull) == 0;   // tile start and length are multiples of 4 floats
    if (vec) {
        const float4 *g4 = reinterpret_cast<const float4 *>(g + base);
        float4 *s4 = reinterpret_cast<float4 *>(s_g);
        for (uint32_t j = threadIdx.x; j < (total >> 2); j += blockDim.x) s4[j] = __ldg(g4 + j);
    } else {
        for (uint32_t j = threadIdx.x; j < total; j += blockDim.x) s_g[j] = __ldg(g + base + j);
    }
    __syncthreads();
    {   // 4 threads per row; partial sums over a quarter of the columns each, in column order
        const uint32_t r = threadIdx.x >> 2, part = threadIdx.x & 3u;
        float s = 0.0f;
        if (r < nrows) {
            const uint32_t per = (cols + 3u) >> 2;
            const uint32_t c0 = part * per, c1 = min(cols, c0 + per);
            const float *gr = s_g + r * cols;
            for (uint32_t c = c0; c < c1; c++) s += gr[c] * gr[c];
        }
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        if (part == 0 && r < nrows) {
            float mean_sq = s / (float)cols;
            float vv = k.first ? mean_sq * k.f2 : v[row0 + r] * k.beta2 + mean_sq * k.f2;
            v[row0 + r] = vv;
            s_v[r] = vv;
        }
    }
    __syncthreads();
    if (vec && (cols & 3u) == 0) {
        const uint32_t c4n = cols >> 2;
        float4 *p4 = reinterpret_cast<float4 *>(p + base);
        float4 *m4 = reinterpret_cast<float4 *>(m + base);
        const float4 *s4 = reinterpret_cast<const float4 *>(s_g);
        for (uint32_t j = threadIdx.x; j < (total >> 2); j += blockDim.x) {
            const uint32_t r = j / c4n, c = (j - r * c4n) << 2;
            const float4 gg = s4[j];
            float4 mm = m4[j], pp = p4[j];
            const float vv = s_v[r];
            float st[4];
#pragma unroll
            for (int q = 0; q < 4; q++) st[q] = lr_scale ? __ldg(lr_scale + c + q) * k.lr : k.lr;
            mm.x = k.first ? gg.x * k.f1 : mm.x * k.beta1 + gg.x * k.f1;
            mm.y = k.first ? gg.y * k.f1 : mm.y * k.beta1 + gg.y * k.f1;
            mm.z = k.first ? gg.z * k.f1 : mm.z * k.beta1 + gg.z * k.f1;
            mm.w = k.first ? gg.w * k.f1 : mm.w * k.beta1 + gg.w * k.f1;
            pp.x = adam_update(pp.x, gg.x, mm.x, vv, k, st[0]);
            pp.y = adam_update(pp.y, gg.y, mm.y, vv, k, st[1]);
            pp.z = adam_update(pp.z, gg.z, mm.z, vv, k, st[2]);
            pp.w = adam_update(pp.w, gg.w, mm.w, vv, k, st[3]);
            m4[j] = mm;
            p4[j] = pp;
        }
    } else {
        for (uint32_t j = threadIdx.x; j < total; j += blockDim.x) {
            uint32_t r = j / cols, c = j - r * cols;
            float gg = s_g[j];
            uint64_t i = base + j;
            float mm = k.first ? gg * k.f1 : m[i] * k.beta1 + gg * k.f1;
            m[i] = mm;
            float step = lr_scale ? __ldg(lr_scale + c) * k.lr : k.lr;
            p[i] = adam_update(p[i], gg, mm, s_v[r], k, step);
        }
    }
}

cudaError_t launch_adam(cudaStream_t s, float *p, const float *g, float *m, float *v, uint64_t rows, uint32_t cols,
                        const float *lr_scale, float lr, float beta1, float beta2, float eps, float bc1, float bc2,
                        bool first, bool reduce_v) {
    AdamConsts k;
    k.lr = lr; k.beta1 = beta1; k.beta2 = beta2; k.eps = eps; k.f1 = 1.0f - beta1; k.f2 = 1.0f - beta2;
    k.bc1 = bc1; k.bc2 = bc2; k.first = first ? 1 : 0;
    if (reduce_v && cols > 1) {
        const size_t smem = (size_t)AR_ROWS * cols * sizeof(float);
        if (smem > 48 * 1024) {
            cudaError_t e = cudaFuncSetAttribute(adam_rowreduce_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) return e;
        }
        const uint64_t grid = (rows + AR_ROWS - 1) / AR_ROWS;
        adam_rowreduce_kernel<<<(unsigned)grid, 256, smem, s>>>(p, g, m, v, rows, cols, lr_scale, k);
    } else {
        const uint64_t total = rows * cols;
        const uint64_t want = (total + 255) / 256;
        const unsigned grid = (unsigned)std::min<uint64_t>(want, GRID_CAP);
        adam_kernel<<<grid, 256, 0, s>>>(p, g, m, v, total, cols, lr_scale, k);
    }
    return cudaGetLastError();
}

__global__ void __launch_bounds__(256)
refine_stats_noise_kernel(uint32_t n, const float *__restrict__ v_refine, const float *__restrict__ visible,
                          const float *__restrict__ max_radius, float *__restrict__ refine_norm,
                          float *__restrict__ vis_weight, float *__restrict__ max_screen, float *__restrict__ transforms,
                          const float *__restrict__ raw_opac, const float *__restrict__ noise, float noise_scale,
                          float median_scale) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        float vis = __ldg(visible + i);
        refine_norm[i] = fmaxf(__ldg(v_refine + i), refine_norm[i]);   // stats.rs:47
        vis_weight[i] = vis_weight[i] + vis;                           // stats.rs:48
        max_screen[i] = fmaxf(__ldg(max_radius + i), max_screen[i]);   // stats.rs:49
        if (noise) {                                                    // train.rs:389-416
            float opac = 1.0f / (1.0f + expf(-__ldg(raw_opac + i)));
            float inv = 1.0f - opac;
            float wgt = fminf(fmaxf(powf(inv, 150.0f), 0.0f), 1.0f) * vis;
            float wm = wgt * noise_scale;
#pragma unroll
            for (int c = 0; c < 3; c++) {
                float d = fminf(fmaxf(__ldg(noise + (size_t)i * 3 + c) * wm, -median_scale), median_scale);
                transforms[(size_t)i * 10 + c] += d;
            }
        }
    }
}

cudaError_t launch_refine_stats_noise(cudaStream_t s, uint32_t n, const float *v_refine, const float *visible,
                                      const float *max_radius, float *refine_norm, float *vis_weight,
                                      float *max_screen, float *transforms, const float *raw_opac, const float *noise,
                                      float noise_scale, float median_scale) {
    const unsigned grid = (unsigned)std::min<uint64_t>(((uint64_t)n + 255) / 256, GRID_CAP);
    refine_stats_noise_kernel<<<grid, 256, 0, s>>>(n, v_refine, visible, max_radius, refine_norm, vis_weight, max_screen,
                                                   transforms, raw_opac, noise, noise_scale, median_scale);
    return cudaGetLastError();
}

// f_i = sqrt(factor) * min_v(|mean_i - cam_v| / max(focal_v, 1e-6))      (train.rs:102-125)
// cams: [views,4] = (x, y, z, focal_px) on the device.
__global__ void __launch_bounds__(256)
min_scale_kernel(uint32_t n, const float *__restrict__ transforms, const float *__restrict__ cams, uint32_t views,
                 float sqrt_factor, float *__restrict__ f_out) {
    __shared__ float4 s_cam[256];
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    float mx = 0.f, my = 0.f, mz = 0.f;
    if (i < n) { mx = __ldg(transforms + (size_t)i * 10); my = __ldg(transforms + (size_t)i * 10 + 1); mz = __ldg(transforms + (size_t)i * 10 + 2); }
    float best = 0.f;
    bool have = false;
    for (uint32_t base = 0; base < views; base += 256) {
        const uint32_t cnt = min(256u, views - base);
        __syncthreads();
        if (threadIdx.x < cnt) s_cam[threadIdx.x] = __ldg(reinterpret_cast<const float4 *>(cams) + base + threadIdx.x);
        __syncthreads();
        for (uint32_t v = 0; v < cnt; v++) {
            const float4 c = s_cam[v];
            const float dx = mx - c.x, dy = my - c.y, dz = mz - c.z;
            const float dist = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
            const float ratio = dist / fmaxf(c.w, 1e-6f);
            best = have ? fminf(best, ratio) : ratio;
            have = true;
        }
    }
    if (i < n) f_out[i] = best * sqrt_factor;
}

// transforms_out may alias transforms (bake_min_scale, gaussian_splats.rs:245-252).
__global__ void __launch_bounds__(256)
fold_min_scale_fwd_kernel(uint32_t n, const float *transforms, const float *raw_opac, const float *__restrict__ f,
                          float *transforms_out, float *raw_opac_out) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        float row[10];
#pragma unroll
        for (int c = 0; c < 10; c++) row[c] = transforms[(size_t)i * 10 + c];
        const FoldTerms t = fold_terms(row + 7, raw_opac[i], __ldg(f + i));
#pragma unroll
        for (int a = 0; a < 3; a++) row[7 + a] = 0.5f * logf(t.s2f[a]);
#pragma unroll
        for (int c = 0; c < 10; c++) transforms_out[(size_t)i * 10 + c] = row[c];
        raw_opac_out[i] = logf(t.opac / (1.0f - t.opac));
    }
}

// Chain the gradients w.r.t. the folded (log-scale, raw opacity) back to the learned ones, in place:
//   v_ls_a  = v_ls'_a * s2_a/(s2_a+f2) + v_coef * coef * f2/(s2_a+f2)
//   v_raw   = v_opac * coef * sig (1-sig),   v_opac = v_raw' / (opac (1-opac)) inside the clamp, else 0
//   v_coef  = v_opac * sig
__global__ void __launch_bounds__(256)
fold_min_scale_bwd_kernel(uint32_t n, const float *__restrict__ transforms, const float *__restrict__ raw_opac,
                          const float *__restrict__ f, float *v_transforms, float *v_raw_opac, uint32_t vt_stride,
                          uint32_t vo_stride) {   // gradient rows may be interleaved (the exchange buffer: 12-float rows)
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        float ls[3];
#pragma unroll
        for (int a = 0; a < 3; a++) ls[a] = __ldg(transforms + (size_t)i * 10 + 7 + a);
        const float fi = __ldg(f + i);
        const FoldTerms t = fold_terms(ls, __ldg(raw_opac + i), fi);
        const float v_rawf = v_raw_opac[(size_t)i * vo_stride];
        const float v_opac = t.in_range ? v_rawf / (t.opac * (1.0f - t.opac)) : 0.0f;
        const float v_coef = v_opac * t.sig;
        v_raw_opac[(size_t)i * vo_stride] = v_opac * t.coef * (t.sig * (1.0f - t.sig));
        const float f2 = fi * fi;
#pragma unroll
        for (int a = 0; a < 3; a++) {
            const float g = v_transforms[(size_t)i * vt_stride + 7 + a];
            v_transforms[(size_t)i * vt_stride + 7 + a] = g * (t.s2[a] / t.s2f[a]) + v_coef * t.coef * (f2 / t.s2f[a]);
        }
    }
}

static unsigned grid_for(uint32_t n) { return (unsigned)std::min<uint64_t>(((uint64_t)n + 255) / 256, GRID_CAP); }

cudaError_t launch_min_scale(cudaStream_t s, uint32_t n, const float *transforms, const float *cams, uint32_t views,
                             float factor, float *f_out) {
    min_scale_kernel<<<(n + 255) / 256, 256, 0, s>>>(n, transforms, cams, views, sqrtf(factor), f_out);
    return cudaGetLastError();
}
cudaError_t launch_fold_min_scale_fwd(cudaStream_t s, uint32_t n, const float *transforms, const float *raw_opac,
                                      const float *f, float *transforms_out, float *raw_opac_out) {
    fold_min_scale_fwd_kernel<<<grid_for(n), 256, 0, s>>>(n, transforms, raw_opac, f, transforms_out, raw_opac_out);
    return cudaGetLastError();
}
cudaError_t launch_fold_min_scale_bwd(cudaStream_t s, uint32_t n, const float *transforms, const float *raw_opac,
                                      const float *f, float *v_transforms, float *v_raw_opac) {
    fold_min_scale_bwd_kernel<<<grid_for(n), 256, 0, s>>>(n, transforms, raw_opac, f, v_transforms, v_raw_opac, 10, 1);
    return cudaGetLastError();
}
cudaError_t launch_fold_min_scale_bwd_strided(cudaStream_t s, uint32_t n, const float *transforms, const float *raw_opac,
                                              const float *f, float *v_transforms, float *v_raw_opac, uint32_t vt_stride,
                                              uint32_t vo_stride) {
    fold_min_scale_bwd_kernel<<<grid_for(n), 256, 0, s>>>(n, transforms, raw_opac, f, v_transforms, v_raw_opac, vt_stride, vo_stride);
    return cudaGetLastError();
}

// ---- counter-based normal noise (Philox4x32-10 + Box-Muller).  The reference draws Tensor::random(Normal) from
// burn's unseeded generator (train.rs:395-399: parity unpinned); a counter-based stream keyed by (seed, offset)
// gives every data-parallel rank the same draw without any communication, and makes a train step replayable.
__global__ void __launch_bounds__(256)
normal_noise_kernel(uint64_t seed, uint64_t offset, uint64_t count, float *__restrict__ out) {
    const uint64_t quads = (count + 3) / 4;
    for (uint64_t q = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; q < quads; q += (uint64_t)gridDim.x * blockDim.x) {
        float z[4];
        normal_quad(seed, offset + q, z);
#pragma unroll
        for (int i = 0; i < 4; i++)
            if (q * 4 + i < count) out[q * 4 + i] = z[i];
    }
}

// the loss scalar of the train step
__global__ void __launch_bounds__(256)
loss_reduce_kernel(const float *__restrict__ partials, uint32_t channels, uint32_t per_channel, float c0, float c1, float c2,
                   float c3, float *__restrict__ loss_out) {
    __shared__ float s_red[256];
    const float chain[4] = {c0, c1, c2, c3};
    float acc = 0.0f;
    for (uint32_t c = 0; c < channels; c++) {
        float s = 0.0f;
        for (uint32_t i = threadIdx.x; i < per_channel; i += 256) s += partials[(size_t)c * per_channel + i];
        acc += s * chain[c];
    }
    s_red[threadIdx.x] = acc;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) s_red[threadIdx.x] += s_red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) *loss_out = s_red[0];
}

__global__ void loss_mean_kernel(const float *__restrict__ terms, uint32_t count, float *__restrict__ out) {
    float s = 0.0f;
    for (uint32_t i = 0; i < count; i++) s += terms[i];
    *out = s * (1.0f / (float)count);
}
cudaError_t launch_loss_mean(cudaStream_t s, const float *terms, uint32_t count, float *out) {
    loss_mean_kernel<<<1, 1, 0, s>>>(terms, count, out);
    return cudaGetLastError();
}

cudaError_t launch_normal_noise(cudaStream_t s, uint64_t seed, uint64_t offset, uint64_t count, float *out) {
    if (count == 0) return cudaSuccess;
    const unsigned grid = (unsigned)std::min<uint64_t>((count / 4 + 255) / 256 + 1, GRID_CAP);
    normal_noise_kernel<<<grid, 256, 0, s>>>(seed, offset, count, out);
    return cudaGetLastError();
}
cudaError_t launch_loss_reduce(cudaStream_t s, const float *partials, uint32_t channels, uint32_t per_channel,
                               const float *chain, float *loss_out) {
    loss_reduce_kernel<<<1, 256, 0, s>>>(partials, channels, per_channel, chain[0], chain[1], chain[2], channels > 3 ? chain[3] : 0.0f, loss_out);
    return cudaGetLastError();
}

}  // namespace bg
