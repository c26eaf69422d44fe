// depth_loss.cu -- the depth-supervision term of the training step (DESIGN.md section 4.7).
//
//   depth_loss_fused_kernel   one pass over the pixels: with a = out_img[...,3], ed = D / a and a pixel active when its
//                             target t is finite and > 0 and a >= 1/255,
//                               v_depth = c * sign(ed - t) / a          (0 on inactive pixels)
//                               v_output[...,3] += -(v_depth * ed)      (active pixels only)
//                             and per-block partial sums of |ed - t| over the active pixels.
//   depth_loss_reduce_kernel  the partials in a fixed order (the scheme of loss_reduce_kernel): c * sum -> the depth-loss
//                             scalar, also added to the step's loss scalar.
//
// No float atomics: the grid is a pure function of (h, w), every thread walks a fixed pixel sequence and both reductions
// have a fixed shape, so the value is reproducible run to run.  Compiled with -fmad=false and IEEE division, so the
// gradients are bit-identical to a float32 restatement of the formulas above.
#include <algorithm>

#include "bg_common.cuh"
#include "bg_launch.cuh"

namespace bg {

constexpr int DL_THREADS = 256;
constexpr uint32_t DL_MAX_BLOCKS = 2048;

uint32_t depth_loss_num_partials(uint32_t h, uint32_t w) {
    const uint64_t px = (uint64_t)h * w;
    return (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((px + DL_THREADS - 1) / DL_THREADS, DL_MAX_BLOCKS));
}

__global__ void __launch_bounds__(DL_THREADS)
depth_loss_fused_kernel(const float4 *__restrict__ out_img, const float *__restrict__ depth, const float *__restrict__ target,
                        uint32_t npx, float chain, float *__restrict__ v_output, float *__restrict__ v_depth,
                        float *__restrict__ partials) {
    float acc = 0.0f;
    for (uint32_t i = blockIdx.x * DL_THREADS + threadIdx.x; i < npx; i += gridDim.x * DL_THREADS) {
        const float a = __ldg(out_img + i).w;    // one 128-bit load per pixel; only alpha is used
        const float d = __ldg(depth + i), t = __ldg(target + i);
        float vd = 0.0f;
        if (t > 0.0f && t < INFINITY && a >= 1.0f / 255.0f) {
            const float ed = __fdiv_rn(d, a);
            const float diff = __fsub_rn(ed, t);
            const float s = diff > 0.0f ? 1.0f : (diff < 0.0f ? -1.0f : 0.0f);
            vd = __fdiv_rn(__fmul_rn(chain, s), a);
            float *va = v_output + (size_t)i * 4 + 3;
            *va = __fadd_rn(*va, -__fmul_rn(vd, ed));
            acc = __fadd_rn(acc, fabsf(diff));
        }
        v_depth[i] = vd;
    }
    // fixed-shape block reduction: butterfly within the warp, then the warps' sums in order
    __shared__ float s_warp[DL_THREADS / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc = __fadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, o));
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.0f;
#pragma unroll
        for (int i = 0; i < DL_THREADS / 32; i++) s = __fadd_rn(s, s_warp[i]);
        partials[blockIdx.x] = s;
    }
}

__global__ void __launch_bounds__(256)
depth_loss_reduce_kernel(const float *__restrict__ partials, uint32_t count, float chain, float *__restrict__ depth_loss_out,
                         float *__restrict__ loss_out) {
    __shared__ float s_red[256];
    float s = 0.0f;
    for (uint32_t i = threadIdx.x; i < count; i += 256) s = __fadd_rn(s, partials[i]);
    s_red[threadIdx.x] = __fmul_rn(s, chain);
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) s_red[threadIdx.x] = __fadd_rn(s_red[threadIdx.x], s_red[threadIdx.x + o]);
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        *depth_loss_out = s_red[0];
        if (loss_out) *loss_out = __fadd_rn(*loss_out, s_red[0]);
    }
}

cudaError_t launch_depth_loss_fused(cudaStream_t s, const float *out_img, const float *depth, const float *target, uint32_t h,
                                    uint32_t w, float chain, float *v_output, float *v_depth, float *partials) {
    const uint32_t npx = h * w;
    depth_loss_fused_kernel<<<depth_loss_num_partials(h, w), DL_THREADS, 0, s>>>(
        reinterpret_cast<const float4 *>(out_img), depth, target, npx, chain, v_output, v_depth, partials);
    return cudaGetLastError();
}

cudaError_t launch_depth_loss_reduce(cudaStream_t s, const float *partials, uint32_t count, float chain, float *depth_loss_out,
                                     float *loss_out) {
    depth_loss_reduce_kernel<<<1, 256, 0, s>>>(partials, count, chain, depth_loss_out, loss_out);
    return cudaGetLastError();
}

}  // namespace bg
