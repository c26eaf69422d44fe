// lod.cu -- LOD baking (brush-train/src/lod.rs): PUP 3D-GS sensitivity scores and score-ordered decimation.
//
//   pup_accumulate_kernel  <- compute_pup_scores (lod.rs:78-142): H += J J^T per view, J = (d mean, d log_scale)
//   pup_log_det_kernel     <- log_det_6x6 (lod.rs:44-69): Cholesky in f32, -inf when a pivot is <= 0
//   decimate_keys_kernel / decimate_gather_kernel <- decimate_to_count (lod.rs:13-40): the reference reads the scores
//                             back and sorts on the host; here a u32 key, the context's stable radix sort and a row gather.
//
// H is symmetric bit for bit (a*b == b*a), so only its upper triangle is stored: 21 entries, entry-major [21, n]
// (00,01,..,05,11,..,15,22,..,55), so that every access of the accumulator is coalesced.  This file is compiled with
// -fmad=false: each product and sum is rounded on its own, as in the reference's tensor ops and loops.
#include <algorithm>

#include "bg_common.cuh"
#include "bg_math.cuh"
#include "bg_launch.cuh"

namespace bg {

constexpr int PUP_ENTRIES = 21;

// index of (a, b), a <= b, in the packed upper triangle
__host__ __device__ constexpr int pup_idx(int a, int b) { return a * 6 - a * (a - 1) / 2 + (b - a); }

__global__ void __launch_bounds__(256)
pup_accumulate_kernel(uint32_t n, const float *__restrict__ v_transforms, int first, float *__restrict__ fisher) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float *row = v_transforms + (size_t)i * 10;
    const float j[6] = {__ldg(row + 0), __ldg(row + 1), __ldg(row + 2), __ldg(row + 7), __ldg(row + 8), __ldg(row + 9)};
#pragma unroll
    for (int a = 0; a < 6; a++) {
#pragma unroll
        for (int b = a; b < 6; b++) {
            float *dst = fisher + (size_t)pup_idx(a, b) * n + i;
            const float p = __fmul_rn(j[a], j[b]);
            *dst = __fadd_rn(first ? 0.0f : *dst, p);   // the first view adds to the reference's zeros
        }
    }
}

__global__ void __launch_bounds__(256)
pup_log_det_kernel(uint32_t n, const float *__restrict__ fisher, float *__restrict__ scores) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float m[PUP_ENTRIES];
#pragma unroll
    for (int e = 0; e < PUP_ENTRIES; e++) m[e] = __ldg(fisher + (size_t)e * n + i);
    float l[PUP_ENTRIES];   // lower factor, stored by (column, row) with column <= row in the same packing
    bool pd = true;
#pragma unroll
    for (int c = 0; c < 6; c++) {
        if (pd) {
            float sum = 0.0f;
#pragma unroll
            for (int k = 0; k < c; k++) sum = __fadd_rn(sum, __fmul_rn(l[pup_idx(k, c)], l[pup_idx(k, c)]));
            const float diag = __fsub_rn(m[pup_idx(c, c)], sum);
            if (diag <= 0.0f) pd = false;   // NaN passes, as in the reference, and propagates
            const float d = __fsqrt_rn(diag);
            l[pup_idx(c, c)] = d;
#pragma unroll
            for (int r = c + 1; r < 6; r++) {
                float s = 0.0f;
#pragma unroll
                for (int k = 0; k < c; k++) s = __fadd_rn(s, __fmul_rn(l[pup_idx(k, r)], l[pup_idx(k, c)]));
                l[pup_idx(c, r)] = __fdiv_rn(__fsub_rn(m[pup_idx(c, r)], s), d);
            }
        }
    }
    float log_det = 0.0f;
#pragma unroll
    for (int c = 0; c < 6; c++) log_det = __fadd_rn(log_det, det_logf(l[pup_idx(c, c)]));
    scores[i] = pd ? __fmul_rn(2.0f, log_det) : __int_as_float(0xff800000);
}

// ascending order of the key == descending score; equal scores (+0 and -0 included) give equal keys, -inf sorts below
// every finite score and NaN after everything
__global__ void __launch_bounds__(256)
decimate_keys_kernel(uint32_t n, const float *__restrict__ scores, uint32_t *__restrict__ keys, uint32_t *__restrict__ vals) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float f = __ldg(scores + i);
    if (f == 0.0f) f = 0.0f;
    const uint32_t u = __float_as_uint(f);
    keys[i] = (f != f) ? 0xFFFFFFFFu : ~(u ^ ((u >> 31) ? 0xFFFFFFFFu : 0x80000000u));
    vals[i] = i;
}

template <typename V>
__device__ __forceinline__ void gather_rows(uint32_t target, uint32_t words, const uint32_t *__restrict__ ids,
                                            const V *__restrict__ src, V *__restrict__ dst) {
    const uint64_t total = (uint64_t)target * words;
    for (uint64_t x = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t r = (uint32_t)(x / words), c = (uint32_t)(x - (uint64_t)r * words);
        dst[x] = __ldg(src + (size_t)__ldg(ids + r) * words + c);
    }
}

// blockIdx.y selects the array: 0 transforms (five 8-byte words per row), 1 SH (128-bit words when 3k is a multiple of 4,
// as in the update pass), 2 opacity, 3 the scale floor (when present)
__global__ void __launch_bounds__(256)
decimate_gather_kernel(uint32_t target, uint32_t kf, const uint32_t *__restrict__ ids, const float *transforms,
                       const float *sh, const float *raw_opac, const float *min_scale, float *transforms_out, float *sh_out,
                       float *raw_opac_out, float *min_scale_out) {
    switch (blockIdx.y) {
        case 0:
            gather_rows(target, 5u, ids, reinterpret_cast<const float2 *>(transforms), reinterpret_cast<float2 *>(transforms_out));
            break;
        case 1:
            if (kf % 4u == 0u)
                gather_rows(target, kf / 4u, ids, reinterpret_cast<const float4 *>(sh), reinterpret_cast<float4 *>(sh_out));
            else
                gather_rows(target, kf, ids, sh, sh_out);
            break;
        case 2: gather_rows(target, 1u, ids, raw_opac, raw_opac_out); break;
        default:
            if (min_scale) gather_rows(target, 1u, ids, min_scale, min_scale_out);
            break;
    }
}

// ---------------------------------------------------------------------------------------------- launchers
static unsigned lod_blocks(uint64_t n, unsigned per) {
    return (unsigned)std::min<uint64_t>(std::max<uint64_t>((n + per - 1) / per, 1), 1u << 20);
}

cudaError_t launch_pup_accumulate(cudaStream_t s, uint32_t n, const float *v_transforms, bool first, float *fisher) {
    pup_accumulate_kernel<<<lod_blocks(n, 256), 256, 0, s>>>(n, v_transforms, first ? 1 : 0, fisher);
    return cudaGetLastError();
}
cudaError_t launch_pup_log_det(cudaStream_t s, uint32_t n, const float *fisher, float *scores) {
    pup_log_det_kernel<<<lod_blocks(n, 256), 256, 0, s>>>(n, fisher, scores);
    return cudaGetLastError();
}
cudaError_t launch_decimate_keys(cudaStream_t s, uint32_t n, const float *scores, uint32_t *keys, uint32_t *vals) {
    decimate_keys_kernel<<<lod_blocks(n, 256), 256, 0, s>>>(n, scores, keys, vals);
    return cudaGetLastError();
}
cudaError_t launch_decimate_gather(cudaStream_t s, uint32_t target, uint32_t kf, const uint32_t *ids, const float *transforms,
                                   const float *sh, const float *raw_opac, const float *min_scale, float *transforms_out,
                                   float *sh_out, float *raw_opac_out, float *min_scale_out) {
    const uint32_t sh_words = kf % 4u == 0u ? kf / 4u : kf;
    const dim3 grid(lod_blocks((uint64_t)target * std::max(5u, sh_words), 256), min_scale ? 4u : 3u);
    decimate_gather_kernel<<<grid, 256, 0, s>>>(target, kf, ids, transforms, sh, raw_opac, min_scale, transforms_out, sh_out,
                                                raw_opac_out, min_scale_out);
    return cudaGetLastError();
}

}  // namespace bg
