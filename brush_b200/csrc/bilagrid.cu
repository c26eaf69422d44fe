// bilagrid.cu -- the per-view bilateral grid of DESIGN.md section 4.11 (Wang et al., "Bilateral Guided Radiance Field
// Processing", SIGGRAPH 2024): a [L][H][W][12] lattice of 3x4 affine colour transforms, sliced per pixel at
// ((px + 0.5) / w * (W-1), (py + 0.5) / h * (H-1), clamp(gray, 0, 1) * (L-1)) and applied to the rendered colour.
//   bilagrid_slice_kernel      one pass over the pixels: 16 B in, 16 B out, the grid read through L1
//   bilagrid_slice_bwd_kernel  v_img (may alias v_out) and the grid gradient; each CTA accumulates its pixel tile's
//                              lattice nodes in shared memory (one copy per lane where it fits, so that the
//                              shared atomics of a warp's lanes never meet on one address) and flushes them with
//                              one global atomic per node
//   bilagrid_tv_kernel         one CTA per gradient slot: adds the total-variation gradient to v_grid, writes L_tv (and
//                              adds it to a loss).  In the grid update of the multi-view step the first slot of each view
//                              also sums the view's other slots first and runs the Adam step of adam_kernel after, with
//                              the bias corrections of the view's device-side step count
#include <cuda_runtime.h>

#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <cstring>

#include "bg_adam.cuh"
#include "bg_launch.cuh"

namespace bg {
namespace {

constexpr int GL = BG_BILAGRID_L, GH = BG_BILAGRID_H, GW = BG_BILAGRID_W, GC = 12;
constexpr int SLICE_THREADS = 256;
constexpr int BWD_THREADS = 256;
constexpr int BWD_TX = 32;                      // tile width in pixels: one warp per tile row
constexpr int BWD_TY = 64;                      // tile height: eight pixels per thread
constexpr int BWD_SMEM_WORDS = 28 * 1024;       // 112 KiB: two CTAs per SM
constexpr int TV_THREADS = 1024;

struct Lattice {
    int x0, y0, z0;
    float fx, fy, fz;
};

// the lattice cell and fractions of pixel (px, py) with guidance gray; x0 in [0, W-2], y0 in [0, H-2], z0 in [0, L-2]
__device__ __forceinline__ Lattice lattice(uint32_t px, uint32_t py, uint32_t w, uint32_t h, float gray) {
    Lattice t;
    const float gx = ((float)px + 0.5f) / (float)w * (float)(GW - 1);
    const float gy = ((float)py + 0.5f) / (float)h * (float)(GH - 1);
    const float gz = fminf(fmaxf(gray, 0.0f), 1.0f) * (float)(GL - 1);
    t.x0 = min((int)floorf(gx), GW - 2);
    t.y0 = min((int)floorf(gy), GH - 2);
    t.z0 = min((int)floorf(gz), GL - 2);
    t.fx = gx - (float)t.x0;
    t.fy = gy - (float)t.y0;
    t.fz = gz - (float)t.z0;
    return t;
}

__device__ __forceinline__ float luma(float4 c) { return 0.299f * c.x + 0.587f * c.y + 0.114f * c.z; }

// a[12] += wgt * the 12 coefficients of cell (z, y, x)
__device__ __forceinline__ void add_cell(float a[GC], const float4 *__restrict__ g, int z, int y, int x, float wgt) {
    const float4 *p = g + ((size_t)((z * GH + y) * GW + x)) * 3;
    const float4 q0 = __ldg(p), q1 = __ldg(p + 1), q2 = __ldg(p + 2);
    a[0] += wgt * q0.x; a[1] += wgt * q0.y; a[2] += wgt * q0.z; a[3] += wgt * q0.w;
    a[4] += wgt * q1.x; a[5] += wgt * q1.y; a[6] += wgt * q1.z; a[7] += wgt * q1.w;
    a[8] += wgt * q2.x; a[9] += wgt * q2.y; a[10] += wgt * q2.z; a[11] += wgt * q2.w;
}

// the bilinear (x, y) interpolation of level z
__device__ __forceinline__ void level(float a[GC], const float4 *__restrict__ g, const Lattice &t, int z) {
#pragma unroll
    for (int i = 0; i < GC; i++) a[i] = 0.0f;
    add_cell(a, g, z, t.y0, t.x0, (1.0f - t.fx) * (1.0f - t.fy));
    add_cell(a, g, z, t.y0, t.x0 + 1, t.fx * (1.0f - t.fy));
    add_cell(a, g, z, t.y0 + 1, t.x0, (1.0f - t.fx) * t.fy);
    add_cell(a, g, z, t.y0 + 1, t.x0 + 1, t.fx * t.fy);
}

__global__ void __launch_bounds__(SLICE_THREADS) bilagrid_slice_kernel(const float4 *__restrict__ grid,
                                                                      const float4 *__restrict__ img, uint32_t w, uint32_t h,
                                                                      float4 *__restrict__ out) {
    const uint64_t i = (uint64_t)blockIdx.x * SLICE_THREADS + threadIdx.x;
    if (i >= (uint64_t)w * h) return;
    const uint32_t py = (uint32_t)(i / w), px = (uint32_t)(i - (uint64_t)py * w);
    const float4 c = img[i];
    const Lattice t = lattice(px, py, w, h, luma(c));
    float a[GC], b[GC];
    level(a, grid, t, t.z0);
    level(b, grid, t, t.z0 + 1);
#pragma unroll
    for (int k = 0; k < GC; k++) a[k] += t.fz * (b[k] - a[k]);
    float4 o;
    o.x = a[0] * c.x + a[1] * c.y + a[2] * c.z + a[3];
    o.y = a[4] * c.x + a[5] * c.y + a[6] * c.z + a[7];
    o.z = a[8] * c.x + a[9] * c.y + a[10] * c.z + a[11];
    o.w = c.w;
    out[i] = o;
}

// CTA tile: BWD_TX x BWD_TY pixels.  The tile's lattice nodes are the box [bx, bx+nx) x [by, by+ny) x [0, L); the box
// size is the host's bound (bilagrid_bwd_shape), its origin the cell of the tile's first pixel.  `copies` interleaved
// copies of the box, lane l adding into copy l % copies, each copy nodes*12 + 1 words (the odd stride puts the same node
// of different copies in different banks).
__global__ void __launch_bounds__(BWD_THREADS) bilagrid_slice_bwd_kernel(const float4 *__restrict__ grid,
                                                                        const float4 *__restrict__ img,
                                                                        const float4 *v_out, uint32_t w, uint32_t h,
                                                                        int nx, int ny, int copies,
                                                                        float4 *v_img, float *__restrict__ v_grid) {
    extern __shared__ float s_acc[];
    const int box = nx * ny * GL * GC;
    const int stride = box + 1;
    for (int j = threadIdx.x; j < stride * copies; j += BWD_THREADS) s_acc[j] = 0.0f;
    const uint32_t tx0 = blockIdx.x * BWD_TX, ty0 = blockIdx.y * BWD_TY;
    const Lattice t0 = lattice(tx0, ty0, w, h, 0.0f);
    const int bx = t0.x0, by = t0.y0;
    __syncthreads();
    float *acc = s_acc + (threadIdx.x % 32 % copies) * stride;
    for (uint32_t j = threadIdx.x; j < BWD_TX * BWD_TY; j += BWD_THREADS) {
        const uint32_t px = tx0 + j % BWD_TX, py = ty0 + j / BWD_TX;
        if (px >= w || py >= h) continue;
        const uint64_t i = (uint64_t)py * w + px;
        const float4 c = img[i];
        const float4 v = v_out[i];
        const float gray = luma(c);
        const Lattice t = lattice(px, py, w, h, gray);
        float a[GC], b[GC];
        level(a, grid, t, t.z0);
        level(b, grid, t, t.z0 + 1);
        // dA/dgz = b - a; A = a + fz (b - a)
        float da[GC];
#pragma unroll
        for (int k = 0; k < GC; k++) {
            da[k] = b[k] - a[k];
            a[k] += t.fz * da[k];
        }
        float4 vc;
        vc.x = a[0] * v.x + a[4] * v.y + a[8] * v.z;
        vc.y = a[1] * v.x + a[5] * v.y + a[9] * v.z;
        vc.z = a[2] * v.x + a[6] * v.y + a[10] * v.z;
        vc.w = v.w;
        if (gray > 0.0f && gray < 1.0f) {
            const float dz = v.x * (da[0] * c.x + da[1] * c.y + da[2] * c.z + da[3]) +
                             v.y * (da[4] * c.x + da[5] * c.y + da[6] * c.z + da[7]) +
                             v.z * (da[8] * c.x + da[9] * c.y + da[10] * c.z + da[11]);
            const float s = dz * (float)(GL - 1);
            vc.x += s * 0.299f;
            vc.y += s * 0.587f;
            vc.z += s * 0.114f;
        }
        // dL/dA_k at this pixel: v_i c_j (j < 3), v_i (j = 3), row-major 3x4
        const float g[GC] = {v.x * c.x, v.x * c.y, v.x * c.z, v.x, v.y * c.x, v.y * c.y, v.y * c.z, v.y,
                             v.z * c.x, v.z * c.y, v.z * c.z, v.z};
        v_img[i] = vc;
        const int lx = t.x0 - bx, ly = t.y0 - by;
#pragma unroll
        for (int dz = 0; dz < 2; dz++) {
            const float wz = dz ? t.fz : 1.0f - t.fz;
#pragma unroll
            for (int dy = 0; dy < 2; dy++) {
                const float wy = dy ? t.fy : 1.0f - t.fy;
#pragma unroll
                for (int dx = 0; dx < 2; dx++) {
                    const float wgt = wz * wy * (dx ? t.fx : 1.0f - t.fx);
                    float *p = acc + (((t.z0 + dz) * ny + (ly + dy)) * nx + (lx + dx)) * GC;
#pragma unroll
                    for (int k = 0; k < GC; k++) atomicAdd(p + k, wgt * g[k]);
                }
            }
        }
    }
    __syncthreads();
    for (int j = threadIdx.x; j < box; j += BWD_THREADS) {
        float s = 0.0f;
        for (int r = 0; r < copies; r++) s += s_acc[r * stride + j];
        const int k = j % GC, node = j / GC;
        const int lx = node % nx, ly = (node / nx) % ny, z = node / (nx * ny);
        const int x = bx + lx, y = by + ly;
        if (s != 0.0f && x < GW && y < GH) atomicAdd(v_grid + ((size_t)((z * GH + y) * GW + x)) * GC + k, s);
    }
}

// TV(G) = sum over axes of (1/P_axis) sum (dG)^2; v_grid += tv_weight * dTV/dG; returns tv_weight * TV in thread 0.  One
// CTA of TV_THREADS threads in a fixed reduction order, so the value is the same bits every run; thread t handles the
// elements t + j * TV_THREADS of v_grid.  Ends after a barrier that follows the last read of grid.
__device__ __forceinline__ float bilagrid_tv(const float *grid, float *v_grid, float tv_weight) {
    constexpr float inv_pz = 1.0f / (float)(GC * (GL - 1) * GH * GW);
    constexpr float inv_py = 1.0f / (float)(GC * GL * (GH - 1) * GW);
    constexpr float inv_px = 1.0f / (float)(GC * GL * GH * (GW - 1));
    constexpr int N = GL * GH * GW * GC;
    float part = 0.0f;
    for (int i = threadIdx.x; i < N; i += TV_THREADS) {
        const int x = (i / GC) % GW, y = (i / (GC * GW)) % GH, z = i / (GC * GW * GH);
        const float g = grid[i];
        float d = 0.0f;
        if (x + 1 < GW) {
            const float e = grid[i + GC] - g;
            part += e * e * inv_px;
            d -= e * inv_px;
        }
        if (x > 0) d += (g - grid[i - GC]) * inv_px;
        if (y + 1 < GH) {
            const float e = grid[i + GC * GW] - g;
            part += e * e * inv_py;
            d -= e * inv_py;
        }
        if (y > 0) d += (g - grid[i - GC * GW]) * inv_py;
        if (z + 1 < GL) {
            const float e = grid[i + GC * GW * GH] - g;
            part += e * e * inv_pz;
            d -= e * inv_pz;
        }
        if (z > 0) d += (g - grid[i - GC * GW * GH]) * inv_pz;
        v_grid[i] += 2.0f * tv_weight * d;
    }
    __shared__ float s_part[TV_THREADS / 32];
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if (threadIdx.x % 32 == 0) s_part[threadIdx.x / 32] = part;
    __syncthreads();
    if (threadIdx.x < 32) {
        part = s_part[threadIdx.x];
        for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    }
    return tv_weight * part;
}

// CTA j: gradient slot j, a.v_slots + j * slot_stride, of view a.slot_view[j * view_stride] (view 0 when slot_view is
// null).  The first slot of a view owns it: it adds the gradients of the view's later slots to its own in slot order and
// the TV gradient of the view's grid; every slot of the view in [out_begin, out_begin + out_count) gets the TV value in
// tv_out (and added to loss, when not null).  With a.m set the owner then runs one Adam step with the view's count + 1
// (adam_kernel's arithmetic, the bias corrections formed on the device) and advances the count; without, the caller runs
// Adam itself (bg_bilagrid_update).  A view >= num_views is skipped.
struct TvArgs {
    float *grids, *m, *v;
    int32_t *steps;
    uint32_t num_views;
    float lr, tv_weight;
    float *v_slots;
    const uint32_t *slot_view;
    uint32_t slot_stride, view_stride, slots, out_begin, out_count;
    float *tv_out, *loss;
};

__global__ void __launch_bounds__(TV_THREADS) bilagrid_tv_kernel(TvArgs a) {
    constexpr int N = GL * GH * GW * GC;
    const uint32_t j = blockIdx.x;
    auto view_of = [&](uint32_t q) { return a.slot_view ? a.slot_view[(size_t)q * a.view_stride] : 0u; };
    const uint32_t view = view_of(j);
    if (view >= a.num_views) return;
    for (uint32_t q = 0; q < j; q++)
        if (view_of(q) == view) return;
    float *g = a.v_slots + (size_t)j * a.slot_stride;
    for (uint32_t q = j + 1; q < a.slots; q++) {
        if (view_of(q) != view) continue;
        const float *o = a.v_slots + (size_t)q * a.slot_stride;
        for (int i = threadIdx.x; i < N; i += TV_THREADS) g[i] += o[i];
    }
    const int32_t t = a.m ? a.steps[view] + 1 : 0;
    float *grid = a.grids + (size_t)view * N;
    const float tv = bilagrid_tv(grid, g, a.tv_weight);
    if (threadIdx.x == 0) {
        if (a.m) a.steps[view] = t;
        for (uint32_t q = j; q < a.slots; q++) {
            if (view_of(q) != view || q < a.out_begin || q - a.out_begin >= a.out_count) continue;
            a.tv_out[q - a.out_begin] = tv;
            if (a.loss) a.loss[q - a.out_begin] += tv;
        }
    }
    if (!a.m) return;
    // Adam as adam_kernel runs it for bg_bilagrid_update (betas 0.9, 0.999, eps 1e-15, no per-column scale)
    AdamConsts k;
    k.lr = a.lr; k.beta1 = 0.9f; k.beta2 = 0.999f; k.eps = 1e-15f; k.f1 = 1.0f - k.beta1; k.f2 = 1.0f - k.beta2;
    k.bc1 = adam_bias_correction(k.beta1, t); k.bc2 = adam_bias_correction(k.beta2, t); k.first = t == 1;
    float *mv = a.m + (size_t)view * N, *vv = a.v + (size_t)view * N;
    for (int i = threadIdx.x; i < N; i += TV_THREADS) adam_element(grid[i], g[i], mv[i], vv[i], k, k.lr);
}

// The CTA tile of the slice backward for an image w x h: BWD_TX x BWD_TY pixels, a shared box of nx x ny x L lattice
// nodes, `copies` copies of it.  Even the whole lattice (one copy) fits the shared-memory budget, so the tile never has
// to shrink for small images.
static_assert(GW * GH * GL * GC + 1 <= BWD_SMEM_WORDS, "one copy of the whole lattice must fit the backward's shared memory");
struct BilagridBwdShape {
    int nx, ny, copies;
};

BilagridBwdShape bilagrid_bwd_shape(uint32_t w, uint32_t h) {
    // the most lattice nodes along an axis that a tile of `span` pixels of an image `size` pixels long touches: the cells
    // of its first and last pixel differ by at most ceil((span - 1) * (cells) / size), plus one more node, plus margin
    // for rounding of the cell coordinate
    auto nodes = [](uint32_t span, uint32_t size, int cells) {
        const double d = (double)(span - 1) * cells / (double)size;
        return std::min(cells + 1, (int)std::ceil(d + 1e-3) + 2);
    };
    BilagridBwdShape s;
    s.nx = nodes(BWD_TX, w, GW - 1);
    s.ny = nodes(BWD_TY, h, GH - 1);
    s.copies = std::max(1, std::min(32, BWD_SMEM_WORDS / (s.nx * s.ny * GL * GC + 1)));
    return s;
}

}  // namespace

cudaError_t launch_bilagrid_slice(cudaStream_t s, const float *grid, const float *img, uint32_t w, uint32_t h, float *out) {
    const uint64_t px = (uint64_t)w * h;
    bilagrid_slice_kernel<<<(unsigned)((px + SLICE_THREADS - 1) / SLICE_THREADS), SLICE_THREADS, 0, s>>>(
        (const float4 *)grid, (const float4 *)img, w, h, (float4 *)out);
    return cudaGetLastError();
}

cudaError_t launch_bilagrid_slice_bwd(cudaStream_t s, const float *grid, const float *img, const float *v_out, uint32_t w,
                                      uint32_t h, float *v_img, float *v_grid) {
    cudaError_t e = cudaMemsetAsync(v_grid, 0, sizeof(float) * BG_BILAGRID_FLOATS, s);
    if (e != cudaSuccess) return e;
    const BilagridBwdShape sh = bilagrid_bwd_shape(w, h);
    const size_t smem = sizeof(float) * (size_t)(sh.nx * sh.ny * GL * GC + 1) * sh.copies;
    const dim3 blocks((w + BWD_TX - 1) / BWD_TX, (h + BWD_TY - 1) / BWD_TY);
    if (smem > 48 * 1024) {
        e = cudaFuncSetAttribute(bilagrid_slice_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    bilagrid_slice_bwd_kernel<<<blocks, BWD_THREADS, smem, s>>>((const float4 *)grid, (const float4 *)img, (const float4 *)v_out,
                                                                w, h, sh.nx, sh.ny, sh.copies, (float4 *)v_img, v_grid);
    return cudaGetLastError();
}

cudaError_t launch_bilagrid_tv(cudaStream_t s, const float *grid, float *v_grid, float tv_weight, float *tv_out, float *loss_out) {
    TvArgs a;
    memset(&a, 0, sizeof(a));
    a.grids = const_cast<float *>(grid);   // read only without a.m
    a.num_views = 1; a.tv_weight = tv_weight;
    a.v_slots = v_grid; a.slots = 1; a.out_count = 1;
    a.tv_out = tv_out; a.loss = loss_out;
    bilagrid_tv_kernel<<<1, TV_THREADS, 0, s>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_bilagrid_update_views(cudaStream_t s, float *grids, float *m, float *v, int32_t *steps, uint32_t num_views,
                                         float lr, float tv_weight, float *v_slots, uint32_t slot_stride, const uint32_t *slot_view,
                                         uint32_t view_stride, uint32_t slots, uint32_t out_begin, uint32_t out_count,
                                         float *tv_out, float *loss_terms) {
    if (slots == 0) return cudaSuccess;
    TvArgs a;
    a.grids = grids; a.m = m; a.v = v; a.steps = steps; a.num_views = num_views; a.lr = lr; a.tv_weight = tv_weight;
    a.v_slots = v_slots; a.slot_view = slot_view; a.slot_stride = slot_stride; a.view_stride = view_stride; a.slots = slots;
    a.out_begin = out_begin; a.out_count = out_count; a.tv_out = tv_out; a.loss = loss_terms;
    bilagrid_tv_kernel<<<slots, TV_THREADS, 0, s>>>(a);
    return cudaGetLastError();
}

}  // namespace bg
