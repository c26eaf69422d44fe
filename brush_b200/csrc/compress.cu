// compress.cu -- SuperSplat compressed PLY encoding on the device: the inverse of the importer
// (brush-serde/src/import.rs:408-600, quant.rs), which the reference only reads.  DESIGN.md section 4.8 is the
// specification; tests/compress_ref.py restates it in numpy and the tests demand equal bytes.
//
//   compress_valid_bounds_kernel  validity of every row, the kept count and the min/max of the kept means
//   compress_keys_kernel          30-bit Morton key of each kept mean over those bounds (dropped rows: 1 << 30)
//   (the context's stable radix sort on 31 bits)
//   compress_chunks_kernel        one CTA per 256 output rows: gather in Morton order, the chunk's 18 ranges, the four
//                                 packed words and the higher SH bands as bytes
//
// Compiled with -fmad=false: every product and sum is rounded on its own, as in the numpy restatement.
#include <algorithm>

#include "bg_common.cuh"
#include "bg_math.cuh"
#include "bg_launch.cuh"

namespace bg {

constexpr uint32_t CHUNK_ROWS = 256;
constexpr uint32_t DROPPED_KEY = 1u << 30;
// bounds workspace: [0] kept count, [1..3] ordered min of x y z, [4..6] ordered max
constexpr uint32_t CB_COUNT = 0, CB_MIN = 1, CB_MAX = 4, CB_WORDS = 7;

__device__ __forceinline__ bool finite_f(float x) { return ((__float_as_uint(x) >> 23) & 0xFFu) != 0xFFu; }
// monotone map of a float to u32 (ascending order preserved, -0 below +0) so atomicMin/Max reduce it
__device__ __forceinline__ uint32_t ordered(float f) {
    const uint32_t u = __float_as_uint(f);
    return u ^ ((u >> 31) ? 0xFFFFFFFFu : 0x80000000u);
}
__device__ __forceinline__ float unordered(uint32_t o) { return __uint_as_float(o ^ ((o >> 31) ? 0x80000000u : 0xFFFFFFFFu)); }
// -0 -> +0 (x + 0 is x for every other value): ranges and quantisation never see a signed zero
__device__ __forceinline__ float canon(float x) { return __fadd_rn(x, 0.0f); }

__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = fminf(v, __shfl_xor_sync(0xFFFFFFFFu, v, o));
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xFFFFFFFFu, v, o));
    return v;
}

// One CTA per 256 source rows.  A row is kept when all its 10 + 3k + 1 floats are finite and its quaternion's squared
// norm (((w*w + x*x) + y*y) + z*z) is not zero.  keys[i] = 0 (kept) or DROPPED_KEY; the bounds are reduced with
// order-independent atomics, so they do not depend on the schedule.
__global__ void __launch_bounds__(256)
compress_valid_bounds_kernel(uint32_t n, uint32_t kf, const float *__restrict__ transforms, const float *__restrict__ sh,
                             const float *__restrict__ raw_opac, uint32_t *__restrict__ keys, uint32_t *__restrict__ bounds) {
    __shared__ unsigned char bad[256];
    __shared__ float s_lo[8][3], s_hi[8][3];
    __shared__ uint32_t s_cnt[8];
    const uint32_t base = blockIdx.x * 256u, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t rows = min(256u, n - base);
    bad[tid] = 0;
    __syncthreads();
    // the block's SH rows are one contiguous span: read it coalesced, mark the rows with a non-finite coefficient
    const float *span = sh + (size_t)base * kf;
    for (uint32_t f = tid; f < rows * kf; f += 256u)
        if (!finite_f(__ldg(span + f))) bad[f / kf] = 1;
    __syncthreads();
    const uint32_t i = base + tid;
    bool keep = false;
    float m[3] = {0.0f, 0.0f, 0.0f};
    if (tid < rows) {
        const float2 *row = reinterpret_cast<const float2 *>(transforms + (size_t)i * 10);
        float t[10];
#pragma unroll
        for (int j = 0; j < 5; j++) { const float2 v = __ldg(row + j); t[2 * j] = v.x; t[2 * j + 1] = v.y; }
        keep = !bad[tid] && finite_f(__ldg(raw_opac + i));
#pragma unroll
        for (int j = 0; j < 10; j++) keep = keep && finite_f(t[j]);
        const float q2 = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(t[3], t[3]), __fmul_rn(t[4], t[4])), __fmul_rn(t[5], t[5])),
                                   __fmul_rn(t[6], t[6]));
        keep = keep && q2 != 0.0f;
        keys[i] = keep ? 0u : DROPPED_KEY;
        m[0] = canon(t[0]); m[1] = canon(t[1]); m[2] = canon(t[2]);
    }
    const uint32_t cnt = __popc(__ballot_sync(0xFFFFFFFFu, keep));
    float lo[3], hi[3];
#pragma unroll
    for (int a = 0; a < 3; a++) {
        lo[a] = warp_min(keep ? m[a] : __int_as_float(0x7f800000));
        hi[a] = warp_max(keep ? m[a] : __int_as_float(0xff800000));
    }
    if (lane == 0) {
        s_cnt[warp] = cnt;
#pragma unroll
        for (int a = 0; a < 3; a++) { s_lo[warp][a] = lo[a]; s_hi[warp][a] = hi[a]; }
    }
    __syncthreads();
    if (tid == 0) {
        uint32_t c = 0;
        float l[3], h[3];
#pragma unroll
        for (int a = 0; a < 3; a++) { l[a] = s_lo[0][a]; h[a] = s_hi[0][a]; }
        for (int w = 0; w < 8; w++) {
            c += s_cnt[w];
#pragma unroll
            for (int a = 0; a < 3; a++) { l[a] = fminf(l[a], s_lo[w][a]); h[a] = fmaxf(h[a], s_hi[w][a]); }
        }
        if (c) {
            atomicAdd(bounds + CB_COUNT, c);
#pragma unroll
            for (int a = 0; a < 3; a++) {
                atomicMin(bounds + CB_MIN + a, ordered(l[a]));
                atomicMax(bounds + CB_MAX + a, ordered(h[a]));
            }
        }
    }
}

__device__ __forceinline__ uint32_t spread3(uint32_t v) {   // 10 bits -> every third bit
    v &= 0x3FFu;
    v = (v | (v << 16)) & 0x030000FFu;
    v = (v | (v << 8)) & 0x0300F00Fu;
    v = (v | (v << 4)) & 0x030C30C3u;
    v = (v | (v << 2)) & 0x09249249u;
    return v;
}

// min(1023, floor((x - lo) / (hi - lo) * 1024)), 0 when hi == lo (and for a NaN, which needs a range that overflows f32)
__device__ __forceinline__ uint32_t morton_cell(float x, float lo, float hi) {
    if (hi == lo) return 0u;
    const float v = __fmul_rn(__fdiv_rn(__fsub_rn(x, lo), __fsub_rn(hi, lo)), 1024.0f);
    return v >= 1023.0f ? 1023u : (v >= 1.0f ? (uint32_t)v : 0u);
}

__global__ void __launch_bounds__(256)
compress_keys_kernel(uint32_t n, const float *__restrict__ transforms, const uint32_t *__restrict__ bounds,
                     uint32_t *__restrict__ keys, uint32_t *__restrict__ vals) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    vals[i] = i;
    if (keys[i]) return;   // dropped
    const float *row = transforms + (size_t)i * 10;
    uint32_t key = 0;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const float lo = unordered(__ldg(bounds + CB_MIN + a)), hi = unordered(__ldg(bounds + CB_MAX + a));
        key |= spread3(morton_cell(canon(__ldg(row + a)), lo, hi)) << (2 - a);
    }
    keys[i] = key;
}

// rint(t * (2^bits - 1)) clamped to the field, t = (v - lo) / (hi - lo); 0 when hi == lo.  fmaxf maps NaN to 0.
__device__ __forceinline__ uint32_t unorm(float v, float lo, float hi, float maxq) {
    if (hi == lo) return 0u;
    const float t = __fdiv_rn(__fsub_rn(v, lo), __fsub_rn(hi, lo));
    return (uint32_t)fminf(fmaxf(rintf(__fmul_rn(t, maxq)), 0.0f), maxq);
}
__device__ __forceinline__ uint32_t clamp_rint(float x, float lo, float hi) { return (uint32_t)fminf(fmaxf(rintf(x), lo), hi); }

__device__ __forceinline__ void block_minmax(float (&v)[9], bool active, float (*s_lo)[9], float (*s_hi)[9], float *lo,
                                             float *hi) {
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int f = 0; f < 9; f++) {
        const float a = warp_min(active ? v[f] : __int_as_float(0x7f800000));
        const float b = warp_max(active ? v[f] : __int_as_float(0xff800000));
        if (lane == 0) { s_lo[warp][f] = a; s_hi[warp][f] = b; }
    }
    __syncthreads();
    if (threadIdx.x < 9) {
        float a = s_lo[0][threadIdx.x], b = s_hi[0][threadIdx.x];
        for (int w = 1; w < 8; w++) { a = fminf(a, s_lo[w][threadIdx.x]); b = fmaxf(b, s_hi[w][threadIdx.x]); }
        lo[threadIdx.x] = a;
        hi[threadIdx.x] = b;
    }
    __syncthreads();
}

// Output rows 256c .. min(m, 256c + 256) - 1 take source rows order[r].  CTAs past m exit.
__global__ void __launch_bounds__(256)
compress_chunks_kernel(uint32_t k, const float *__restrict__ transforms, const float *__restrict__ sh,
                       const float *__restrict__ raw_opac, const uint32_t *__restrict__ bounds,
                       const uint32_t *__restrict__ order, float *__restrict__ chunks_out, uint4 *__restrict__ packed_out,
                       uint8_t *__restrict__ sh_out, uint32_t *__restrict__ order_out) {
    __shared__ float s_lo[8][9], s_hi[8][9];
    __shared__ float lo[9], hi[9];
    __shared__ uint32_t src_s[CHUNK_ROWS];
    const uint32_t m = __ldg(bounds + CB_COUNT), first = blockIdx.x * CHUNK_ROWS;
    if (first >= m) return;
    const uint32_t rows = min(CHUNK_ROWS, m - first), tid = threadIdx.x, r = first + tid;
    const bool active = tid < rows;
    const uint32_t src = active ? __ldg(order + r) : 0u;
    src_s[tid] = src;
    float t[10], v[9], op = 0.0f;
    if (active) {
        const float2 *row = reinterpret_cast<const float2 *>(transforms + (size_t)src * 10);
#pragma unroll
        for (int j = 0; j < 5; j++) { const float2 x = __ldg(row + j); t[2 * j] = x.x; t[2 * j + 1] = x.y; }
        op = __ldg(raw_opac + src);
        const float *c = sh + (size_t)src * 3 * k;
#pragma unroll
        for (int a = 0; a < 3; a++) {
            v[a] = canon(t[a]);
            v[3 + a] = canon(t[7 + a]);
            v[6 + a] = __fadd_rn(__fmul_rn(__ldg(c + a), 0.2820947917738781f), 0.5f);   // rgb = f_dc * SH_C0 + 0.5
        }
    } else {
#pragma unroll
        for (int j = 0; j < 10; j++) t[j] = 0.0f;
#pragma unroll
        for (int f = 0; f < 9; f++) v[f] = 0.0f;
    }
    block_minmax(v, active, s_lo, s_hi, lo, hi);
    if (tid < 18) chunks_out[(size_t)blockIdx.x * 18 + tid] = (tid & 1) ? hi[tid >> 1] : lo[tid >> 1];
    if (active) {
        uint32_t q[9];
#pragma unroll
        for (int f = 0; f < 9; f++) q[f] = unorm(v[f], lo[f], hi[f], f < 6 ? ((f % 3) == 1 ? 1023.0f : 2047.0f) : 255.0f);
        const uint32_t pos = q[0] << 21 | q[1] << 11 | q[2];
        const uint32_t scl = q[3] << 21 | q[4] << 11 | q[5];
        // opacity: 8 bits of the sigmoid, clamped to 1..254 so that the importer's ln(a / (1 - a)) stays finite
        const float sig = __fdiv_rn(1.0f, __fadd_rn(1.0f, det_expf(-op)));
        const uint32_t col = q[6] << 24 | q[7] << 16 | q[8] << 8 | clamp_rint(__fmul_rn(sig, 255.0f), 1.0f, 254.0f);
        // rotation: normalised as splat_to_ply does, smallest three after making the largest component positive
        const float sq = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(t[3], t[3]), __fmul_rn(t[4], t[4])), __fmul_rn(t[5], t[5])),
                                   __fmul_rn(t[6], t[6]));
        const float rn = fmaxf(__fsqrt_rn(sq), 1e-12f);
        float qn[4];
        uint32_t largest = 0;
        float best = -1.0f;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            qn[j] = __fdiv_rn(t[3 + j], rn);
            if (fabsf(qn[j]) > best) { best = fabsf(qn[j]); largest = j; }
        }
        const bool neg = qn[largest] < 0.0f;
        uint32_t rot = largest << 30;
        int sft = 20;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            if ((uint32_t)j == largest) continue;
            const float x = neg ? -qn[j] : qn[j];
            rot |= clamp_rint(__fmul_rn(__fadd_rn(__fmul_rn(x, 0.70710677f), 0.5f), 1023.0f), 0.0f, 1023.0f) << sft;
            sft -= 10;
        }
        packed_out[r] = make_uint4(pos, rot, scl, col);
        if (order_out) order_out[r] = src;
    }
    __syncthreads();   // src_s
    // higher bands: output byte j = c * (k - 1) + (i - 1) of a row is coefficient i of channel c (channel-major), written
    // as one contiguous span per chunk
    const uint32_t per = 3u * (k - 1u);
    if (per == 0) return;
    uint8_t *dst = sh_out + (size_t)first * per;
    for (uint32_t e = tid; e < rows * per; e += CHUNK_ROWS) {
        const uint32_t lr = e / per, j = e - lr * per, c = j / (k - 1u), i = j - c * (k - 1u) + 1u;
        const float x = __ldg(sh + ((size_t)src_s[lr] * k + i) * 3 + c);
        dst[e] = (uint8_t)clamp_rint(__fmul_rn(__fadd_rn(__fmul_rn(x, 0.125f), 0.5f), 254.0f), 0.0f, 255.0f);
    }
}

// ---------------------------------------------------------------------------------------------- launchers
cudaError_t launch_compress_valid_bounds(cudaStream_t s, uint32_t n, uint32_t kf, const float *transforms, const float *sh,
                                         const float *raw_opac, uint32_t *keys, uint32_t *bounds) {
    // count and maxima start at 0, minima at 0xFFFFFFFF (the top of the ordered range)
    cudaError_t e = cudaMemsetAsync(bounds, 0, CB_WORDS * sizeof(uint32_t), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(bounds + CB_MIN, 0xFF, 3 * sizeof(uint32_t), s);
    if (e != cudaSuccess) return e;
    compress_valid_bounds_kernel<<<(n + 255) / 256, 256, 0, s>>>(n, kf, transforms, sh, raw_opac, keys, bounds);
    return cudaGetLastError();
}
cudaError_t launch_compress_keys(cudaStream_t s, uint32_t n, const float *transforms, const uint32_t *bounds, uint32_t *keys,
                                 uint32_t *vals) {
    compress_keys_kernel<<<(n + 255) / 256, 256, 0, s>>>(n, transforms, bounds, keys, vals);
    return cudaGetLastError();
}
cudaError_t launch_compress_chunks(cudaStream_t s, uint32_t n, uint32_t k, const float *transforms, const float *sh,
                                   const float *raw_opac, const uint32_t *bounds, const uint32_t *order, float *chunks_out,
                                   uint32_t *packed_out, uint8_t *sh_out, uint32_t *order_out, uint32_t *count_out) {
    cudaError_t e = cudaMemcpyAsync(count_out, bounds + CB_COUNT, 4, cudaMemcpyDeviceToDevice, s);
    if (e != cudaSuccess) return e;
    compress_chunks_kernel<<<(n + CHUNK_ROWS - 1) / CHUNK_ROWS, CHUNK_ROWS, 0, s>>>(
        k, transforms, sh, raw_opac, bounds, order, chunks_out, reinterpret_cast<uint4 *>(packed_out), sh_out, order_out);
    return cudaGetLastError();
}

}  // namespace bg
