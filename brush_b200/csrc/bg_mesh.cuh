// bg_mesh.cuh -- device functions shared by the dense (mesh.cu) and the sparse (mesh_sparse.cu) TSDF: the per-point
// integration step of one view, and the marching-tetrahedra pieces of the extraction (DESIGN.md sections 4.9, 4.10).
// Both translation units are compiled with -fmad=false, so the two grids round every product and sum alike.
#pragma once
#include <cstdint>

#include "bg_common.cuh"
#include "bg_math.cuh"
#include "bg_project.cuh"

namespace bg {

constexpr uint32_t BRICK_PTS = 512;   // 8 x 8 x 8 points, x fastest

// ------------------------------------------------------------------------------------------------------ integration
// What one view does to the lattice point at world position xw: false when the view leaves it alone; otherwise the
// truncated distance f and the un-premultiplied colour.  The sparse grid's near test is `true and f < 0`.
struct TsdfSample {
    float f, col[3];
};
template <bool DISTORTED>
__device__ __forceinline__ bool tsdf_sample(V3 xw, float trunc, const BgCamera &cam, uint32_t w, uint32_t h,
                                            const float4 *__restrict__ img, const float *__restrict__ depth, float alpha_min,
                                            TsdfSample &s) {
    const V3 xc = world_to_cam(xw, cam);
    if (!(xc.z >= 0.01f) || !isfinite(xc.z)) return false;
    float u, v;
    project_mean<DISTORTED>(xc, cam, u, v);
    if (!(u >= 0.0f && u < (float)w && v >= 0.0f && v < (float)h)) return false;   // NaN fails every comparison
    const size_t pix = (size_t)(uint32_t)v * w + (uint32_t)u;
    const float4 c = __ldg(img + pix);
    if (!(c.w >= alpha_min)) return false;
    const float ed = __fdiv_rn(__ldg(depth + pix), c.w);
    if (!(ed > 0.0f) || !isfinite(ed)) return false;
    const float sdf = ed - xc.z;
    if (sdf < -trunc) return false;
    s.f = fminf(1.0f, __fdiv_rn(sdf, trunc));
    s.col[0] = fminf(fmaxf(__fdiv_rn(c.x, c.w), 0.0f), 1.0f);
    s.col[1] = fminf(fmaxf(__fdiv_rn(c.y, c.w), 0.0f), 1.0f);
    s.col[2] = fminf(fmaxf(__fdiv_rn(c.z, c.w), 0.0f), 1.0f);
    return true;
}

// The running-mean update of point q: W' = W + 1, T' = (T W + f) / W', C' = (C W + c) / W'.
__device__ __forceinline__ void tsdf_update(float *tsdf, float *weight, float *rgb, size_t q, const TsdfSample &s) {
    const float W = weight[q], W1 = W + 1.0f;
    tsdf[q] = __fdiv_rn(tsdf[q] * W + s.f, W1);
    float *c = rgb + q * 3;
#pragma unroll
    for (int a = 0; a < 3; a++) c[a] = __fdiv_rn(c[a] * W + s.col[a], W1);
    weight[q] = W1;
}

// ------------------------------------------------------------------------------------------------------ extraction
// Edge directions in output order x, y, z, xy, xz, yz, xyz as axis bit sets (x = 1, y = 2, z = 4), one nibble each, and the
// inverse map from a bit set to its direction index.
__device__ __forceinline__ uint32_t dir_bits(uint32_t d) { return (0x7653421u >> (4 * d)) & 0xFu; }
__device__ __forceinline__ uint32_t dir_index(uint32_t bits) { return (0x6542310Fu >> (4 * bits)) & 0xFu; }
// Kuhn tetrahedra in the order xyz, xzy, yxz, yzx, zxy, zyx: corners 0, e_a, e_a + e_b, 7 (cell corner bit sets).  Even
// permutations (xyz, yzx, zxy) have positive orientation.
__device__ __forceinline__ uint32_t tet_c1(uint32_t t) { return (0x442211u >> (4 * t)) & 0xFu; }
__device__ __forceinline__ uint32_t tet_c2(uint32_t t) { return (0x656353u >> (4 * t)) & 0xFu; }
__device__ __forceinline__ bool tet_even(uint32_t t) { return (0x19u >> t) & 1u; }

// The 8 corners p + b (b = x | 2y | 4z) of the cell at p: tsdf values, and which corners lie in the grid and are observed
// (weight != 0).  Corners outside the grid are neither read nor observed.
struct Corners {
    float t[8];
    uint32_t obs, neg;
};

// Bit d of the mask: the edge p -> p + dir_bits(d) has both endpoints observed and their signs differ.
__device__ __forceinline__ uint32_t edge_mask(const Corners &c) {
    uint32_t m = 0;
    if (!(c.obs & 1u)) return 0;
#pragma unroll
    for (uint32_t d = 0; d < 7; d++) {
        const uint32_t b = dir_bits(d);
        if (((c.obs >> b) & 1u) && (((c.neg >> b) ^ c.neg) & 1u)) m |= 1u << d;
    }
    return m;
}

// The 4-bit sign pattern of tetrahedron t (bit v: corner v negative), or 0xFF when a corner is unobserved or the cell
// is not complete.
__device__ __forceinline__ uint32_t tet_signs(const Corners &c, uint32_t t) {
    const uint32_t c1 = tet_c1(t), c2 = tet_c2(t);
    const uint32_t need = 1u | (1u << c1) | (1u << c2) | 0x80u;
    if ((c.obs & need) != need) return 0xFFu;
    return (c.neg & 1u) | (((c.neg >> c1) & 1u) << 1) | (((c.neg >> c2) & 1u) << 2) | (((c.neg >> 7) & 1u) << 3);
}
__device__ __forceinline__ uint32_t tet_tris(uint32_t s) {
    if (s == 0xFFu) return 0;
    const uint32_t n = __popc(s);
    return n == 2 ? 2u : (n == 1 || n == 3) ? 1u : 0u;
}
__device__ __forceinline__ uint32_t cell_tris(const Corners &c) {
    if (c.obs != 0xFFu) return 0;   // incomplete or partly unobserved cells emit nothing (all 8 corners are in every tet)
    uint32_t n = 0;
#pragma unroll
    for (uint32_t t = 0; t < 6; t++) n += tet_tris(tet_signs(c, t));
    return n;
}

// Exclusive scan of one u32 per thread over a CTA of up to 1024 threads; *total receives the sum.
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t *s_warp, uint32_t &total) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o);
        if (lane >= (uint32_t)o) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < nw ? s_warp[lane] : 0u;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, w, o);
            if (lane >= (uint32_t)o) w += y;
        }
        if (lane < nw) s_warp[lane] = w;   // inclusive warp prefix
    }
    __syncthreads();
    total = s_warp[nw - 1];
    const uint32_t before = warp ? s_warp[warp - 1] : 0u;
    __syncthreads();   // s_warp is reused by the caller's next scan
    return before + x - v;
}

// Triangles of one tetrahedron with sign pattern s, wound so that each normal points toward the T >= 0 side.
// edge_id(ca, cb) is the vertex id of the edge between cell corners ca -> cb (ca a subset of cb).
//   one corner i apart (1 or 3 negative): triangle on edges (i,j), (i,k), (i,l), j < k < l.  det(v_j - v_i, v_k - v_i,
//     v_l - v_i) = (-1)^i times the tetrahedron's orientation; the normal points away from v_i when that is positive,
//     which is right when v_i is the negative corner.
//   two and two (negative i < j, positive k < l): the quad (i,k) (i,l) (j,l) (j,k) faces the positive side when the
//     orientation times the sign of the permutation (i, j, k, l) is positive; it is split along (i,k)-(j,l).
template <class EdgeId>
__device__ __forceinline__ uint32_t emit_tet(uint32_t t, uint32_t s, uint32_t *out, const EdgeId &edge_id) {
    const uint32_t c1 = tet_c1(t), c2 = tet_c2(t);
    const bool even = tet_even(t);
    auto cbits = [&](uint32_t v) { return v == 0 ? 0u : v == 1 ? c1 : v == 2 ? c2 : 7u; };
    auto E = [&](uint32_t a, uint32_t b) { return a < b ? edge_id(cbits(a), cbits(b)) : edge_id(cbits(b), cbits(a)); };
    const uint32_t nneg = __popc(s);
    if (nneg == 1 || nneg == 3) {
        const uint32_t i = __ffs(nneg == 1 ? s : (~s & 0xFu)) - 1;
        const uint32_t j = i == 0 ? 1u : 0u, k = i <= 1 ? 2u : 1u, l = i <= 2 ? 3u : 2u;
        const bool det_pos = ((i & 1u) == 0) == even;
        const bool keep = (nneg == 1) == det_pos;   // the apart corner is negative exactly when nneg == 1
        out[0] = E(i, j);
        out[1] = E(i, keep ? k : l);
        out[2] = E(i, keep ? l : k);
        return 1;
    }
    if (nneg == 2) {
        const uint32_t pos = ~s & 0xFu;
        const uint32_t ni = __ffs(s) - 1, nj = 31 - __clz(s), pk = __ffs(pos) - 1, pl = 31 - __clz(pos);
        const bool perm_even = !(s == 5u || s == 10u);
        const uint32_t ik = E(ni, pk), il = E(ni, pl), jl = E(nj, pl), jk = E(nj, pk);
        const bool keep = perm_even == even;
        out[0] = ik; out[1] = keep ? il : jl; out[2] = keep ? jl : il;
        out[3] = ik; out[4] = keep ? jl : jk; out[5] = keep ? jk : jl;
        return 2;
    }
    return 0;
}

}  // namespace bg
