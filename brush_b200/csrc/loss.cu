// loss.cu -- fused L1 + SSIM image loss, forward map and recompute-in-backward VJP.
// Replaces image_loss_forward_kernel (brush-loss/src/lib.rs:180-359) and image_loss_backward_kernel
// (lib.rs:370-661): 11-tap sigma=1.5 separable Gaussian window, zero padding, C1=1e-4, C2=9e-4,
// sigma^2 = max(0, .), ssim clamped to [-1,1] with zero gradient where clamped, GT decoded from packed
// rgba8, optional background compositing and alpha masking, channel 3 = |pred.a - gt.a|.
//
// Differences in mechanism only: pred is addressed through (stride_c, stride_y, stride_x) so the
// rasterizer's [h,w,4] output is consumed in place (the reference permutes HWC->CHW around the op,
// lib.rs:1076,1103), and the backward uses a 16x16 tile like the forward (the reference's 8x8
// backward tile is an Apple threadgroup-memory constraint, lib.rs:75-87).  Accumulation order of the
// window sums follows the reference (symmetric pairs d=1..5, then the centre tap).
// HBM-bound: ~28 P bytes forward, ~40 P backward for C=3.
#include "bg_common.cuh"
#include "bg_launch.cuh"

namespace bg {

constexpr int LB = 16;        // tile edge
constexpr int HALO = 5;
constexpr int SH1 = LB + 2 * HALO;   // 26
constexpr int SH2 = LB + 4 * HALO;   // 36
constexpr float SSIM_C1 = 0.01f * 0.01f;
constexpr float SSIM_C2 = 0.03f * 0.03f;
constexpr float INV_255 = 1.0f / 255.0f;

struct Taps { float w[11]; };

struct LossArgs {
    const float *pred;
    const uint32_t *gt;
    uint32_t h, w;
    int64_t sc, sy, sx;
    float l1_w, ssim_w;
    float bg[3];
    int composite, mask;
};

__device__ __forceinline__ float ld_pred(const LossArgs &a, uint32_t c, int y, int x) {
    if (y < 0 || x < 0 || y >= (int)a.h || x >= (int)a.w) return 0.0f;
    return __ldg(a.pred + (int64_t)c * a.sc + (int64_t)y * a.sy + (int64_t)x * a.sx);
}
__device__ __forceinline__ float ld_gt_eff(const LossArgs &a, uint32_t c, int y, int x, float bg_c) {
    float gt_c = 0.0f, gt_a = 0.0f;
    if (!(y < 0 || x < 0 || y >= (int)a.h || x >= (int)a.w)) {
        uint32_t v = __ldg(a.gt + (size_t)y * a.w + x);
        gt_c = (float)((v >> (c * 8u)) & 0xffu) * INV_255;
        gt_a = (float)((v >> 24u) & 0xffu) * INV_255;
    }
    return a.composite ? gt_c + (1.0f - gt_a) * bg_c : gt_c;
}
__device__ __forceinline__ float ld_gt_a(const LossArgs &a, int y, int x) {
    return (float)((__ldg(a.gt + (size_t)y * a.w + x) >> 24u) & 0xffu) * INV_255;
}

// Blur of five moment images along one axis, reference accumulation order.
#define BG_BLUR5_PAIR(o, l0, l1, r0, r1, wd)          \
    o[0] += (l0 + r0) * wd;                           \
    o[1] += (l0 * l0 + r0 * r0) * wd;                 \
    o[2] += (l1 + r1) * wd;                           \
    o[3] += (l1 * l1 + r1 * r1) * wd;                 \
    o[4] += (l0 * l1 + r0 * r1) * wd;

__global__ void __launch_bounds__(LB * LB)
image_loss_fwd_kernel(LossArgs a, Taps taps, float *__restrict__ loss_map) {
    const uint32_t c = blockIdx.z;
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int tile_x0 = blockIdx.x * LB, tile_y0 = blockIdx.y * LB;
    const int pix_x = tile_x0 + tx, pix_y = tile_y0 + ty;
    const int rank = ty * LB + tx;
    if (c == 3) {  // alpha-match channel (lib.rs:215-227)
        if (pix_x < (int)a.w && pix_y < (int)a.h) {
            float ga = ld_gt_a(a, pix_y, pix_x);
            float v = fabsf(ld_pred(a, 3, pix_y, pix_x) - ga);
            if (a.mask) v = v * ga;
            loss_map[(size_t)3 * a.h * a.w + (size_t)pix_y * a.w + pix_x] = v;
        }
        return;
    }
    __shared__ float s_tile[SH1 * SH1 * 2];
    __shared__ float s_h[SH1 * LB * 5];
    const float bg_c = a.composite ? a.bg[c] : 0.0f;
    for (int i = rank; i < SH1 * SH1; i += LB * LB) {
        int ly = i / SH1, lx = i - ly * SH1;
        int gy = tile_y0 + ly - HALO, gx = tile_x0 + lx - HALO;
        s_tile[i * 2] = ld_pred(a, c, gy, gx);
        s_tile[i * 2 + 1] = ld_gt_eff(a, c, gy, gx, bg_c);
    }
    __syncthreads();
    for (int i = rank; i < SH1 * LB; i += LB * LB) {  // horizontal pass: SH1 rows x LB columns
        int ly = i / LB, ox = i - ly * LB;
        int lx = ox + HALO;
        float o[5] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
        for (int d = 1; d <= 5; d++) {
            const float wd = taps.w[5 - d];
            const float *l = &s_tile[(ly * SH1 + lx - d) * 2], *r = &s_tile[(ly * SH1 + lx + d) * 2];
            BG_BLUR5_PAIR(o, l[0], l[1], r[0], r[1], wd)
        }
        const float *cc = &s_tile[(ly * SH1 + lx) * 2];
        const float wc = taps.w[5];
        o[0] += cc[0] * wc; o[1] += cc[0] * cc[0] * wc; o[2] += cc[1] * wc; o[3] += cc[1] * cc[1] * wc;
        o[4] += cc[0] * cc[1] * wc;
#pragma unroll
        for (int k = 0; k < 5; k++) s_h[i * 5 + k] = o[k];
    }
    __syncthreads();
    float o[5] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    {
        const int ly = ty + HALO;
#pragma unroll
        for (int d = 1; d <= 5; d++) {
            const float wd = taps.w[5 - d];
            const float *t = &s_h[((ly - d) * LB + tx) * 5], *b = &s_h[((ly + d) * LB + tx) * 5];
#pragma unroll
            for (int k = 0; k < 5; k++) o[k] += (t[k] + b[k]) * wd;
        }
        const float *m = &s_h[(ly * LB + tx) * 5];
#pragma unroll
        for (int k = 0; k < 5; k++) o[k] += m[k] * taps.w[5];
    }
    if (pix_x < (int)a.w && pix_y < (int)a.h) {
        float mu1 = o[0], mu2 = o[2];
        float mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2;
        float s1 = fmaxf(0.0f, o[1] - mu1_sq), s2 = fmaxf(0.0f, o[3] - mu2_sq);
        float s12 = o[4] - mu1 * mu2;
        float A = mu1_sq + mu2_sq + SSIM_C1, B = s1 + s2 + SSIM_C2;
        float c_top = 2.0f * mu1 * mu2 + SSIM_C1, d_top = 2.0f * s12 + SSIM_C2;
        float raw = (c_top * d_top) / (A * B);
        float val = fminf(fmaxf(raw, -1.0f), 1.0f);
        const float *cc = &s_tile[((ty + HALO) * SH1 + tx + HALO) * 2];
        float loss_v = a.l1_w * fabsf(cc[0] - cc[1]) + a.ssim_w * val;
        if (a.mask) loss_v = loss_v * ld_gt_a(a, pix_y, pix_x);
        loss_map[(size_t)c * a.h * a.w + (size_t)pix_y * a.w + pix_x] = loss_v;
    }
}

__global__ void __launch_bounds__(LB * LB)
image_loss_bwd_kernel(LossArgs a, Taps taps, const float *__restrict__ dl_dmap, float *__restrict__ dl_dpred) {
    const uint32_t c = blockIdx.z;
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int tile_x0 = blockIdx.x * LB, tile_y0 = blockIdx.y * LB;
    const int pix_x = tile_x0 + tx, pix_y = tile_y0 + ty;
    const int rank = ty * LB + tx;
    const bool in_img = pix_x < (int)a.w && pix_y < (int)a.h;
    auto out_at = [&](uint32_t ch, int y, int x) -> float & {
        return dl_dpred[(int64_t)ch * a.sc + (int64_t)y * a.sy + (int64_t)x * a.sx];
    };
    if (c == 3) {  // lib.rs:393-414
        if (in_img) {
            float ga = ld_gt_a(a, pix_y, pix_x);
            float diff = ld_pred(a, 3, pix_y, pix_x) - ga;
            float sign = diff > 0.0f ? 1.0f : (diff < 0.0f ? -1.0f : 0.0f);
            float chain = __ldg(dl_dmap + (size_t)3 * a.h * a.w + (size_t)pix_y * a.w + pix_x);
            if (a.mask) chain = chain * ga;
            out_at(3, pix_y, pix_x) = sign * chain;
        }
        return;
    }
    __shared__ float s_a[SH2 * SH2 * 2];   // image tile (+2 halos), later chain*partials [SH1*SH1*3]
    __shared__ float s_b[SH2 * SH1 * 5];   // first h-blur, later second h-blur [SH1*LB*3]
    const float bg_c = a.composite ? a.bg[c] : 0.0f;
    for (int i = rank; i < SH2 * SH2; i += LB * LB) {
        int ly = i / SH2, lx = i - ly * SH2;
        int gy = tile_y0 + ly - 2 * HALO, gx = tile_x0 + lx - 2 * HALO;
        s_a[i * 2] = ld_pred(a, c, gy, gx);
        s_a[i * 2 + 1] = ld_gt_eff(a, c, gy, gx, bg_c);
    }
    __syncthreads();
    for (int i = rank; i < SH2 * SH1; i += LB * LB) {  // h-blur: SH2 rows x SH1 cols
        int ly = i / SH1, ox = i - ly * SH1;
        int lx = ox + HALO;
        float o[5] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
        for (int d = 1; d <= 5; d++) {
            const float wd = taps.w[5 - d];
            const float *l = &s_a[(ly * SH2 + lx - d) * 2], *r = &s_a[(ly * SH2 + lx + d) * 2];
            BG_BLUR5_PAIR(o, l[0], l[1], r[0], r[1], wd)
        }
        const float *cc = &s_a[(ly * SH2 + lx) * 2];
        const float wc = taps.w[5];
        o[0] += cc[0] * wc; o[1] += cc[0] * cc[0] * wc; o[2] += cc[1] * wc; o[3] += cc[1] * cc[1] * wc;
        o[4] += cc[0] * cc[1] * wc;
#pragma unroll
        for (int k = 0; k < 5; k++) s_b[i * 5 + k] = o[k];
    }
    __syncthreads();
    // centre values needed at the end are read back from global (s_a is about to be overwritten)
    float p1 = 0.0f, gt_eff_c = 0.0f;
    if (in_img) { p1 = ld_pred(a, c, pix_y, pix_x); gt_eff_c = ld_gt_eff(a, c, pix_y, pix_x, bg_c); }
    constexpr int NPART = (SH1 * SH1 + LB * LB - 1) / (LB * LB);  // 3 partial positions per thread
    float part[NPART][3];
#pragma unroll
    for (int it = 0; it < NPART; it++) {  // v-blur + SSIM partials on the SH1 x SH1 region
        const int i = rank + it * LB * LB;
        part[it][0] = part[it][1] = part[it][2] = 0.0f;
        if (i >= SH1 * SH1) continue;
        int py_ = i / SH1, px_ = i - py_ * SH1;
        int ly = py_ + HALO;
        float o[5] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
        for (int d = 1; d <= 5; d++) {
            const float wd = taps.w[5 - d];
            const float *t = &s_b[((ly - d) * SH1 + px_) * 5], *b = &s_b[((ly + d) * SH1 + px_) * 5];
#pragma unroll
            for (int k = 0; k < 5; k++) o[k] += (t[k] + b[k]) * wd;
        }
        const float *m = &s_b[(ly * SH1 + px_) * 5];
#pragma unroll
        for (int k = 0; k < 5; k++) o[k] += m[k] * taps.w[5];
        float mu1 = o[0], mu2 = o[2];
        float mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2;
        float s1 = fmaxf(0.0f, o[1] - mu1_sq), s2 = fmaxf(0.0f, o[3] - mu2_sq);
        float s12 = o[4] - mu1 * mu2;
        float A = mu1_sq + mu2_sq + SSIM_C1, B = s1 + s2 + SSIM_C2;
        float c_top = 2.0f * mu1 * mu2 + SSIM_C1, d_top = 2.0f * s12 + SSIM_C2;
        float inv_ab = 1.0f / (A * B);
        float cd = c_top * d_top * inv_ab;
        bool clamped = cd < -1.0f || cd > 1.0f;
        float dmu1 = clamped ? 0.0f : 2.0f * mu2 * inv_ab * (d_top - c_top) - 2.0f * mu1 * cd * (1.0f / A - 1.0f / B);
        float ds1 = clamped ? 0.0f : -cd / B;
        float ds12 = clamped ? 0.0f : 2.0f * c_top * inv_ab;
        int gy = tile_y0 + py_ - HALO, gx = tile_x0 + px_ - HALO;
        float chain = 0.0f;
        if (gy >= 0 && gx >= 0 && gy < (int)a.h && gx < (int)a.w) {
            chain = __ldg(dl_dmap + (size_t)c * a.h * a.w + (size_t)gy * a.w + gx);
            if (a.mask) chain = chain * ld_gt_a(a, gy, gx);
        }
        part[it][0] = dmu1 * chain; part[it][1] = ds1 * chain; part[it][2] = ds12 * chain;
    }
    __syncthreads();  // everyone done reading s_a (h-blur) and s_b (v-blur)
#pragma unroll
    for (int it = 0; it < NPART; it++) {
        const int i = rank + it * LB * LB;
        if (i < SH1 * SH1) { s_a[i * 3] = part[it][0]; s_a[i * 3 + 1] = part[it][1]; s_a[i * 3 + 2] = part[it][2]; }
    }
    __syncthreads();
    for (int i = rank; i < SH1 * LB; i += LB * LB) {  // second h-blur: SH1 rows x LB cols
        int ly = i / LB, ox = i - ly * LB;
        int lx = ox + HALO;
        float o[3] = {0.0f, 0.0f, 0.0f};
#pragma unroll
        for (int d = 1; d <= 5; d++) {
            const float wd = taps.w[5 - d];
            const float *l = &s_a[(ly * SH1 + lx - d) * 3], *r = &s_a[(ly * SH1 + lx + d) * 3];
#pragma unroll
            for (int k = 0; k < 3; k++) o[k] += (l[k] + r[k]) * wd;
        }
        const float *m = &s_a[(ly * SH1 + lx) * 3];
#pragma unroll
        for (int k = 0; k < 3; k++) o[k] += m[k] * taps.w[5];
#pragma unroll
        for (int k = 0; k < 3; k++) s_b[i * 3 + k] = o[k];
    }
    __syncthreads();
    if (in_img) {
        const int ly = ty + HALO;
        float s[3] = {0.0f, 0.0f, 0.0f};
#pragma unroll
        for (int d = 1; d <= 5; d++) {
            const float wd = taps.w[5 - d];
            const float *t = &s_b[((ly - d) * LB + tx) * 3], *b = &s_b[((ly + d) * LB + tx) * 3];
#pragma unroll
            for (int k = 0; k < 3; k++) s[k] += (t[k] + b[k]) * wd;
        }
        const float *m = &s_b[(ly * LB + tx) * 3];
#pragma unroll
        for (int k = 0; k < 3; k++) s[k] += m[k] * taps.w[5];
        float ssim_grad = s[0] + (2.0f * p1) * s[1] + gt_eff_c * s[2];
        float diff = p1 - gt_eff_c;
        float l1_sign = diff > 0.0f ? 1.0f : (diff < 0.0f ? -1.0f : 0.0f);
        float chain_c = __ldg(dl_dmap + (size_t)c * a.h * a.w + (size_t)pix_y * a.w + pix_x);
        if (a.mask) chain_c = chain_c * ld_gt_a(a, pix_y, pix_x);
        out_at(c, pix_y, pix_x) = a.ssim_w * ssim_grad + a.l1_w * l1_sign * chain_c;
    }
}

// ---------------------------------------------------------------------------------------------
// Fused train-path kernel: loss value AND dL/dpred in one pass, for the case the trainer actually
// runs (train.rs:254-260: loss = mean of the map, i.e. dL/dmap is one constant per channel).
// Equivalent to image_loss_forward + mean + image_loss_backward, without materialising the loss map and
// without re-blurring in a second kernel.  32x32 tiles: the (tile+halo)^2 / tile^2 recomputation factor of
// the separable window is 3.9 (6.3 with 16x16 tiles).
//
// The four separable passes are written as STREAMING windows on paired FP32: a thread owns a run of L
// consecutive outputs of one row (or column), keeps them as (L+1)/2 float2 accumulators -- two neighbouring
// outputs per register pair -- and walks the L+10 inputs once; input i feeds the output pair (2j, 2j+1) with
// the tap pair (w[i-2j], w[i-2j-1]), one ffma2_rn with the input broadcast.  The tap pairs are a __grid_constant__
// kernel parameter, read in place from parameter space: every index is a compile-time constant after unrolling (no
// local copy, no per-device upload, nothing for a CUDA-graph capture to trip over).
// The accumulation order is therefore by input position, not the reference's (pairs d = 1..5, then the
// centre): the same sum up to f32 rounding.  Work is cut so that each pass fills the 256 threads once:
//   P1 horizontal, 5 moments : 52 rows x 4 runs of 11      P2 vertical + SSIM partials: 42 cols x 6 runs of 7
//   P3 horizontal, 3 partials: 42 rows x 6 runs of 6       P4 vertical + L1 + store   : 32 cols x 8 runs of 4
// Per-block partial sums of the weighted map go to loss_partials (summed by the caller in a fixed
// order, so the scalar is reproducible run to run).
constexpr int FT = 32;            // tile edge
constexpr int FE = FT + 4 * HALO; // 52: staged inputs
constexpr int FP = FT + 2 * HALO; // 42: region where SSIM partials are needed
constexpr int F_BUF_A = FE * FE * 2;      // inputs (pred, gt_eff); later chain*partials [FP*FP*3]
constexpr int F_BUF_B = FE * FP * 5;      // first h-blur [FE rows][FP cols][5]; later second h-blur [FP][FT][3]
constexpr int F_THREADS = 256;

struct Chain4 { float c[4]; };
struct TapPairs { float2 p[12]; };   // p[t] = (w[t], w[t-1]) with w[-1] = w[11] = 0

// acc[jp][q] += (w[t], w[t-1]) * v[q]  for every output pair jp this input (relative index IREL) reaches
template <int NQ, int PAIRS, int IREL>
__device__ __forceinline__ void window_feed(float2 (&acc)[PAIRS][NQ], const float (&v)[NQ], const TapPairs &tp) {
#pragma unroll
    for (int jp = 0; jp < PAIRS; jp++) {
        const int t = IREL - 2 * jp;
        if (t >= 0 && t <= 11) {
#pragma unroll
            for (int q = 0; q < NQ; q++) acc[jp][q] = ffma2_rn(tp.p[t], make_float2(v[q], v[q]), acc[jp][q]);
        }
    }
}

// walks inputs 0 .. 2*PAIRS+9 of a run; load(i, v) fetches the NQ values of input i (zero beyond the staged region)
template <int NQ, int PAIRS, int IREL = 0, typename Load>
__device__ __forceinline__ void window_run(float2 (&acc)[PAIRS][NQ], const TapPairs &tp, Load load) {
    if constexpr (IREL < 2 * PAIRS + 10) {
        float v[NQ];
        load(IREL, v);
        window_feed<NQ, PAIRS, IREL>(acc, v, tp);
        window_run<NQ, PAIRS, IREL + 1>(acc, tp, load);
    }
}

__global__ void __launch_bounds__(F_THREADS, 3)
image_loss_fused_kernel(LossArgs a, Chain4 chain, const __grid_constant__ TapPairs taps, float *__restrict__ dl_dpred,
                        float *__restrict__ loss_partials) {
    extern __shared__ float f_smem[];
    float *buf_a = f_smem, *buf_b = f_smem + F_BUF_A;
    __shared__ float s_red[F_THREADS / 32];
    const uint32_t c = blockIdx.z;
    const int t = threadIdx.x;
    const int tile_x0 = blockIdx.x * FT, tile_y0 = blockIdx.y * FT;
    const int W = (int)a.w, H = (int)a.h;
    auto out_at = [&](uint32_t ch, int y, int x) -> float & {
        return dl_dpred[(int64_t)ch * a.sc + (int64_t)y * a.sy + (int64_t)x * a.sx];
    };
    float loss_acc = 0.0f;
    // (kernel parameters are selected, never indexed: a run-time index would force a local copy of the struct)
    const float chain_c = c == 0 ? chain.c[0] : (c == 1 ? chain.c[1] : (c == 2 ? chain.c[2] : chain.c[3]));
    if (c == 3) {  // alpha-match channel: |pred.a - gt.a|, no window (lib.rs:215-227, 393-414)
        for (int i = t; i < FT * FT; i += F_THREADS) {
            int y = tile_y0 + i / FT, x = tile_x0 + i % FT;
            if (x < W && y < H) {
                float ga = ld_gt_a(a, y, x);
                float diff = ld_pred(a, 3, y, x) - ga;
                float v = fabsf(diff), ch = chain_c;
                if (a.mask) { v *= ga; ch *= ga; }
                loss_acc += v;
                out_at(3, y, x) = (diff > 0.0f ? 1.0f : (diff < 0.0f ? -1.0f : 0.0f)) * ch;
            }
        }
    } else {
        const float bg_c = a.composite ? (c == 0 ? a.bg[0] : (c == 1 ? a.bg[1] : a.bg[2])) : 0.0f;
        // ---- P0: stage (pred, gt_eff) with a 2*HALO border, zero padded.  Tiles whose staged region lies inside the
        // image (all but the border tiles) skip the bounds tests and address with 32-bit offsets.
        const bool interior = tile_x0 >= 2 * HALO && tile_y0 >= 2 * HALO && tile_x0 + FT + 2 * HALO <= W && tile_y0 + FT + 2 * HALO <= H &&
                              (int64_t)H * a.sy < (1ll << 31) && a.sc < (1ll << 31);
        if (interior) {
            const float *pbase = a.pred + (int64_t)c * a.sc + (int64_t)(tile_y0 - 2 * HALO) * a.sy + (int64_t)(tile_x0 - 2 * HALO) * a.sx;
            const uint32_t *gbase = a.gt + (size_t)(tile_y0 - 2 * HALO) * a.w + (tile_x0 - 2 * HALO);
            const int sy = (int)a.sy, sx = (int)a.sx;
            const uint32_t shift = c * 8u;
            constexpr int P0_ITEMS = (FE * FE + F_THREADS - 1) / F_THREADS;   // 11 staged pixels per thread
            float pv[P0_ITEMS];
            uint32_t gv[P0_ITEMS];
#pragma unroll
            for (int k = 0; k < P0_ITEMS; k++) {   // all loads of the thread in flight before the first use
                const int i = t + k * F_THREADS;
                if (i < FE * FE) {
                    const int ly = i / FE, lx = i - ly * FE;
                    gv[k] = __ldg(gbase + ly * W + lx);
                    pv[k] = __ldg(pbase + ly * sy + lx * sx);
                }
            }
#pragma unroll
            for (int k = 0; k < P0_ITEMS; k++) {
                const int i = t + k * F_THREADS;
                if (i < FE * FE) {
                    float ge = (float)((gv[k] >> shift) & 0xffu) * INV_255;
                    if (a.composite) ge = ge + (1.0f - (float)(gv[k] >> 24u) * INV_255) * bg_c;
                    *reinterpret_cast<float2 *>(&buf_a[i * 2]) = make_float2(pv[k], ge);
                }
            }
        } else {
            for (int i = t; i < FE * FE; i += F_THREADS) {
                int ly = i / FE, lx = i - ly * FE;
                int gy = tile_y0 + ly - 2 * HALO, gx = tile_x0 + lx - 2 * HALO;
                *reinterpret_cast<float2 *>(&buf_a[i * 2]) = make_float2(ld_pred(a, c, gy, gx), ld_gt_eff(a, c, gy, gx, bg_c));
            }
        }
        __syncthreads();
        // ---- P1: horizontal window of the five moments: FE rows x 4 runs of 11 outputs (columns 0..41 of FP)
        if (t < FE * 4) {
            const int row = t >> 2, o0 = (t & 3) * 11;
            const float *src = buf_a + (row * FE + o0) * 2;
            // three windows of at most two moments each (x, x^2 | y, y^2 | x*y): one window of three moments needs 36
            // accumulator registers and pushes the kernel past its 3-CTA register budget
            {   // x, x^2
                float2 acc[6][2];
#pragma unroll
                for (int jp = 0; jp < 6; jp++)
#pragma unroll
                    for (int q = 0; q < 2; q++) acc[jp][q] = make_float2(0.0f, 0.0f);
                window_run<2, 6>(acc, taps, [&](int i, float (&v)[2]) {
                    float x = 0.0f;
                    if (o0 + i < FE) x = src[i * 2];
                    v[0] = x; v[1] = x * x;
                });
#pragma unroll
                for (int jp = 0; jp < 6; jp++) {
                    const int o = o0 + 2 * jp;
                    if (2 * jp < 11 && o < FP) { float *d = &buf_b[(row * FP + o) * 5]; d[0] = acc[jp][0].x; d[1] = acc[jp][1].x; }
                    if (2 * jp + 1 < 11 && o + 1 < FP) { float *d = &buf_b[(row * FP + o + 1) * 5]; d[0] = acc[jp][0].y; d[1] = acc[jp][1].y; }
                }
            }
            {   // y, y^2
                float2 acc[6][2];
#pragma unroll
                for (int jp = 0; jp < 6; jp++)
#pragma unroll
                    for (int q = 0; q < 2; q++) acc[jp][q] = make_float2(0.0f, 0.0f);
                window_run<2, 6>(acc, taps, [&](int i, float (&v)[2]) {
                    float y = 0.0f;
                    if (o0 + i < FE) y = src[i * 2 + 1];
                    v[0] = y; v[1] = y * y;
                });
#pragma unroll
                for (int jp = 0; jp < 6; jp++) {
                    const int o = o0 + 2 * jp;
                    if (2 * jp < 11 && o < FP) { float *d = &buf_b[(row * FP + o) * 5]; d[2] = acc[jp][0].x; d[3] = acc[jp][1].x; }
                    if (2 * jp + 1 < 11 && o + 1 < FP) { float *d = &buf_b[(row * FP + o + 1) * 5]; d[2] = acc[jp][0].y; d[3] = acc[jp][1].y; }
                }
            }
            {   // x*y
                float2 acc[6][1];
#pragma unroll
                for (int jp = 0; jp < 6; jp++) acc[jp][0] = make_float2(0.0f, 0.0f);
                window_run<1, 6>(acc, taps, [&](int i, float (&v)[1]) {
                    float2 xy = make_float2(0.0f, 0.0f);
                    if (o0 + i < FE) xy = *reinterpret_cast<const float2 *>(src + i * 2);
                    v[0] = xy.x * xy.y;
                });
#pragma unroll
                for (int jp = 0; jp < 6; jp++) {
                    const int o = o0 + 2 * jp;
                    if (2 * jp < 11 && o < FP) buf_b[(row * FP + o) * 5 + 4] = acc[jp][0].x;
                    if (2 * jp + 1 < 11 && o + 1 < FP) buf_b[(row * FP + o + 1) * 5 + 4] = acc[jp][0].y;
                }
            }
        }
        __syncthreads();
        // ---- P2: vertical window + SSIM partials on the FP x FP region: FP columns x 6 runs of 7 rows
        if (t < FP * 6) {
            const int px_ = t % FP, r0 = (t / FP) * 7;
            float2 acc[4][5];
#pragma unroll
            for (int jp = 0; jp < 4; jp++)
#pragma unroll
                for (int q = 0; q < 5; q++) acc[jp][q] = make_float2(0.0f, 0.0f);
            const float *src = buf_b + (r0 * FP + px_) * 5;
            window_run<5, 4>(acc, taps, [&](int i, float (&v)[5]) {
                if (r0 + i < FE) {
#pragma unroll
                    for (int q = 0; q < 5; q++) v[q] = src[i * FP * 5 + q];
                } else {
#pragma unroll
                    for (int q = 0; q < 5; q++) v[q] = 0.0f;
                }
            });
#pragma unroll
            for (int j = 0; j < 7; j++) {
                const int py_ = r0 + j;
                float o[5];
#pragma unroll
                for (int q = 0; q < 5; q++) o[q] = (j & 1) ? acc[j >> 1][q].y : acc[j >> 1][q].x;
                const float mu1 = o[0], mu2 = o[2];
                const float mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2;
                const float s1 = fmaxf(0.0f, o[1] - mu1_sq), s2 = fmaxf(0.0f, o[3] - mu2_sq);
                const float s12 = o[4] - mu1 * mu2;
                const float A = mu1_sq + mu2_sq + SSIM_C1, B = s1 + s2 + SSIM_C2;
                const float c_top = 2.0f * mu1 * mu2 + SSIM_C1, d_top = 2.0f * s12 + SSIM_C2;
                // two correctly rounded reciprocals serve the four quotients of lib.rs:507-520 (each within one
                // rounding of the division it replaces)
                const float inv_a = __frcp_rn(A), inv_b = __frcp_rn(B);
                const float inv_ab = inv_a * inv_b;
                const float cd = c_top * d_top * inv_ab;
                const bool clamped = cd < -1.0f || cd > 1.0f;
                const float dmu1 = clamped ? 0.0f : 2.0f * mu2 * inv_ab * (d_top - c_top) - 2.0f * mu1 * cd * (inv_a - inv_b);
                const float ds1 = clamped ? 0.0f : -cd * inv_b;
                const float ds12 = clamped ? 0.0f : 2.0f * c_top * inv_ab;
                const int gy = tile_y0 + py_ - HALO, gx = tile_x0 + px_ - HALO;
                float ch = 0.0f;
                if (gy >= 0 && gx >= 0 && gy < H && gx < W) {
                    ch = chain_c;
                    float ga = 1.0f;
                    if (a.mask) { ga = ld_gt_a(a, gy, gx); ch *= ga; }
                    // SSIM part of the loss value for the pixels this tile owns
                    if (py_ >= HALO && py_ < HALO + FT && px_ >= HALO && px_ < HALO + FT)
                        loss_acc += a.ssim_w * fminf(fmaxf(cd, -1.0f), 1.0f) * ga;
                }
                float *dst = &buf_a[(py_ * FP + px_) * 3];
                dst[0] = dmu1 * ch; dst[1] = ds1 * ch; dst[2] = ds12 * ch;
            }
        }
        __syncthreads();
        // ---- P3: second horizontal window: FP rows x 6 runs of 6 outputs (columns 0..31 of the tile)
        if (t < FP * 6) {
            const int row = t / 6, o0 = (t % 6) * 6;
            float2 acc[3][3];
#pragma unroll
            for (int jp = 0; jp < 3; jp++)
#pragma unroll
                for (int q = 0; q < 3; q++) acc[jp][q] = make_float2(0.0f, 0.0f);
            const float *src = buf_a + (row * FP + o0) * 3;
            window_run<3, 3>(acc, taps, [&](int i, float (&v)[3]) {
                if (o0 + i < FP) { v[0] = src[i * 3]; v[1] = src[i * 3 + 1]; v[2] = src[i * 3 + 2]; }
                else { v[0] = v[1] = v[2] = 0.0f; }
            });
#pragma unroll
            for (int j = 0; j < 6; j++) {
                const int o = o0 + j;
                if (o < FT) {
                    float *dst = &buf_b[(row * FT + o) * 3];
#pragma unroll
                    for (int q = 0; q < 3; q++) dst[q] = (j & 1) ? acc[j >> 1][q].y : acc[j >> 1][q].x;
                }
            }
        }
        __syncthreads();
        // ---- P4: second vertical window, L1 term, write dL/dpred: 32 columns x 8 runs of 4 rows
        {
            const int x = t & 31, y0 = (t >> 5) * 4;
            float2 acc[2][3];
#pragma unroll
            for (int jp = 0; jp < 2; jp++)
#pragma unroll
                for (int q = 0; q < 3; q++) acc[jp][q] = make_float2(0.0f, 0.0f);
            const float *src = buf_b + (y0 * FT + x) * 3;
            window_run<3, 2>(acc, taps, [&](int i, float (&v)[3]) {
                v[0] = src[i * FT * 3]; v[1] = src[i * FT * 3 + 1]; v[2] = src[i * FT * 3 + 2];   // rows y0 .. y0+13 < FP
            });
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int gy = tile_y0 + y0 + j, gx = tile_x0 + x;
                if (gy < H && gx < W) {
                    float sm[3];
#pragma unroll
                    for (int q = 0; q < 3; q++) sm[q] = (j & 1) ? acc[j >> 1][q].y : acc[j >> 1][q].x;
                    const float p1 = ld_pred(a, c, gy, gx), ge = ld_gt_eff(a, c, gy, gx, bg_c);
                    const float ssim_grad = sm[0] + (2.0f * p1) * sm[1] + ge * sm[2];
                    const float diff = p1 - ge;
                    const float l1_sign = diff > 0.0f ? 1.0f : (diff < 0.0f ? -1.0f : 0.0f);
                    float chc = chain_c, ga = 1.0f;
                    if (a.mask) { ga = ld_gt_a(a, gy, gx); chc *= ga; }
                    loss_acc += a.l1_w * fabsf(diff) * ga;
                    out_at(c, gy, gx) = a.ssim_w * ssim_grad + a.l1_w * l1_sign * chc;
                }
            }
        }
    }
    // ---- block sum of the map values (fixed order), one partial per block
    for (int o = 16; o > 0; o >>= 1) loss_acc += __shfl_xor_sync(0xffffffffu, loss_acc, o);
    if ((t & 31) == 0) s_red[t >> 5] = loss_acc;
    __syncthreads();
    if (t == 0) {
        float s = 0.0f;
        for (int i = 0; i < F_THREADS / 32; i++) s += s_red[i];
        loss_partials[(blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = s;
    }
}

static Taps make_taps() {
    // brush-loss/src/lib.rs:55-68: f32 arithmetic on the host, sigma = 1.5, normalised to sum 1.
    Taps t;
    const float sigma = 1.5f;
    float sum = 0.0f;
    for (int i = 0; i < 11; i++) {
        float x = (float)i - 5.0f;
        t.w[i] = expf(-x * x / (2.0f * sigma * sigma));
        sum += t.w[i];
    }
    for (int i = 0; i < 11; i++) t.w[i] /= sum;
    return t;
}

static LossArgs make_args(const float *pred, const uint32_t *gt, uint32_t h, uint32_t w, int64_t sc, int64_t sy,
                          int64_t sx, float l1_w, float ssim_w, const float *bg, bool mask) {
    LossArgs a;
    a.pred = pred; a.gt = gt; a.h = h; a.w = w; a.sc = sc; a.sy = sy; a.sx = sx; a.l1_w = l1_w; a.ssim_w = ssim_w;
    a.composite = bg != nullptr;
    for (int i = 0; i < 3; i++) a.bg[i] = bg ? bg[i] : 0.0f;
    a.mask = mask ? 1 : 0;
    return a;
}

cudaError_t launch_image_loss_fwd(cudaStream_t s, const float *pred, const uint32_t *gt, uint32_t c, uint32_t h,
                                  uint32_t w, int64_t sc, int64_t sy, int64_t sx, float l1_w, float ssim_w,
                                  const float *bg, bool mask, float *loss_map) {
    dim3 grid((w + LB - 1) / LB, (h + LB - 1) / LB, c), block(LB, LB);
    image_loss_fwd_kernel<<<grid, block, 0, s>>>(make_args(pred, gt, h, w, sc, sy, sx, l1_w, ssim_w, bg, mask),
                                                 make_taps(), loss_map);
    return cudaGetLastError();
}

cudaError_t launch_image_loss_bwd(cudaStream_t s, const float *pred, const uint32_t *gt, const float *dl_dmap,
                                  uint32_t c, uint32_t h, uint32_t w, int64_t sc, int64_t sy, int64_t sx, float l1_w,
                                  float ssim_w, const float *bg, bool mask, float *dl_dpred) {
    dim3 grid((w + LB - 1) / LB, (h + LB - 1) / LB, c), block(LB, LB);
    image_loss_bwd_kernel<<<grid, block, 0, s>>>(make_args(pred, gt, h, w, sc, sy, sx, l1_w, ssim_w, bg, mask),
                                                 make_taps(), dl_dmap, dl_dpred);
    return cudaGetLastError();
}

cudaError_t launch_image_loss_fused(cudaStream_t s, const float *pred, const uint32_t *gt, uint32_t c, uint32_t h,
                                    uint32_t w, int64_t sc, int64_t sy, int64_t sx, float l1_w, float ssim_w,
                                    const float *bg, bool mask, const float *chain_per_channel, float *dl_dpred,
                                    float *loss_partials) {
    dim3 grid((w + FT - 1) / FT, (h + FT - 1) / FT, c), block(F_THREADS);
    const size_t smem = (size_t)(F_BUF_A + F_BUF_B) * sizeof(float);
    cudaError_t e = cudaFuncSetAttribute(image_loss_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    Chain4 ch;
    for (uint32_t i = 0; i < 4; i++) ch.c[i] = i < c ? chain_per_channel[i] : 0.0f;
    const Taps taps = make_taps();
    TapPairs tp;
    for (int t = 0; t < 12; t++) tp.p[t] = make_float2(t <= 10 ? taps.w[t] : 0.0f, t >= 1 ? taps.w[t - 1] : 0.0f);
    image_loss_fused_kernel<<<grid, block, smem, s>>>(make_args(pred, gt, h, w, sc, sy, sx, l1_w, ssim_w, bg, mask), ch, tp,
                                                      dl_dpred, loss_partials);
    return cudaGetLastError();
}

uint32_t image_loss_fused_num_partials(uint32_t c, uint32_t h, uint32_t w) {
    return ((w + FT - 1) / FT) * ((h + FT - 1) / FT) * c;
}

}  // namespace bg
