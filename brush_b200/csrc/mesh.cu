// mesh.cu -- surface export: fuse rendered depth into a truncated signed distance field on a dense lattice and extract
// its zero level set by marching tetrahedra.  DESIGN.md section 4.9 is the specification; tests/mesh_ref.py restates it
// in numpy and the tests demand equal bits.
//
//   tsdf_integrate_kernel   one thread per lattice point: camera transform, projection (the renderer's device functions),
//                           nearest-pixel lookup, and the running-mean update of the points inside the truncation band
//   mesh_count_kernel       one CTA per 8^3 brick: the brick's vertex count (7-bit edge mask of each point) and triangle
//                           count (6 Kuhn tetrahedra of each cell), both recomputed from the 8 corners
//   mesh_scan_kernel        one CTA: exclusive scan of the brick counts, totals in 64 bits
//   mesh_vertices_kernel    one CTA per brick: each point's vertex base and mask, its vertices' positions and colours
//   mesh_faces_kernel       one CTA per brick: the triangles, each corner the owner point's base plus the popcount of
//                           its mask below the edge's direction
//
// Compiled with -fmad=false: every product and sum is rounded on its own, as in the numpy restatement.
#include <cstdint>

#include "bg_common.cuh"
#include "bg_math.cuh"
#include "bg_project.cuh"
#include "bg_launch.cuh"

namespace bg {

constexpr uint32_t BRICK_PTS = 512;   // 8 x 8 x 8 points, x fastest
// workspace header words (u64): vertex total, triangle total, the dims the counts belong to
constexpr uint32_t MH_VERTS = 0, MH_TRIS = 1, MH_DIMS = 2, MH_WORDS = 8;

// Edge directions in output order x, y, z, xy, xz, yz, xyz as axis bit sets (x = 1, y = 2, z = 4), one nibble each, and the
// inverse map from a bit set to its direction index.
__device__ __forceinline__ uint32_t dir_bits(uint32_t d) { return (0x7653421u >> (4 * d)) & 0xFu; }
__device__ __forceinline__ uint32_t dir_index(uint32_t bits) { return (0x6542310Fu >> (4 * bits)) & 0xFu; }
// Kuhn tetrahedra in the order xyz, xzy, yxz, yzx, zxy, zyx: corners 0, e_a, e_a + e_b, 7 (cell corner bit sets).  Even
// permutations (xyz, yzx, zxy) have positive orientation.
__device__ __forceinline__ uint32_t tet_c1(uint32_t t) { return (0x442211u >> (4 * t)) & 0xFu; }
__device__ __forceinline__ uint32_t tet_c2(uint32_t t) { return (0x656353u >> (4 * t)) & 0xFu; }
__device__ __forceinline__ bool tet_even(uint32_t t) { return (0x19u >> t) & 1u; }

struct Brick {
    uint32_t i, j, k;   // the thread's lattice point
    bool in;            // inside the grid
};
__device__ __forceinline__ Brick brick_point(const BgTsdfGrid &g) {
    const uint32_t nbx = (g.dims[0] + 7) / 8, nby = (g.dims[1] + 7) / 8;
    const uint32_t b = blockIdx.x, bx = b % nbx, r = b / nbx, by = r % nby, bz = r / nby;
    Brick p;
    p.i = bx * 8 + (threadIdx.x & 7);
    p.j = by * 8 + ((threadIdx.x >> 3) & 7);
    p.k = bz * 8 + (threadIdx.x >> 6);
    p.in = p.i < g.dims[0] && p.j < g.dims[1] && p.k < g.dims[2];
    return p;
}
__device__ __forceinline__ size_t lin(const BgTsdfGrid &g, uint32_t i, uint32_t j, uint32_t k) {
    return ((size_t)k * g.dims[1] + j) * g.dims[0] + i;
}

// The 8 corners p + b (b = x | 2y | 4z) of the cell at p: tsdf values, and which corners lie in the grid and are observed
// (weight != 0).  Corners outside the grid are neither read nor observed.
struct Corners {
    float t[8];
    uint32_t obs, neg;
};
__device__ __forceinline__ Corners load_corners(const BgTsdfGrid &g, const Brick &p) {
    Corners c;
    c.obs = 0;
    c.neg = 0;
#pragma unroll
    for (uint32_t b = 0; b < 8; b++) {
        const uint32_t i = p.i + (b & 1u), j = p.j + ((b >> 1) & 1u), k = p.k + (b >> 2);
        c.t[b] = 0.0f;
        if (p.in && i < g.dims[0] && j < g.dims[1] && k < g.dims[2]) {
            const size_t q = lin(g, i, j, k);
            if (__ldg(g.weight + q) != 0.0f) {
                c.t[b] = __ldg(g.tsdf + q);
                c.obs |= 1u << b;
                if (c.t[b] < 0.0f) c.neg |= 1u << b;
            }
        }
    }
    return c;
}

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

// Exclusive scan of one u32 per thread over a 512-thread CTA; *total receives the sum.
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

// ------------------------------------------------------------------------------------------------------ integration
// One thread per lattice point.  A point the view does not update is never read or written.
template <bool DISTORTED>
__global__ void __launch_bounds__(256)
tsdf_integrate_kernel(BgTsdfGrid g, BgCamera cam, uint32_t w, uint32_t h, const float4 *__restrict__ img,
                      const float *__restrict__ depth, float alpha_min) {
    const uint32_t n = g.dims[0] * g.dims[1] * g.dims[2];
    const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n) return;
    const uint32_t i = idx % g.dims[0], r = idx / g.dims[0], j = r % g.dims[1], k = r / g.dims[1];
    const V3 xw = mk3(g.origin[0] + (float)i * g.h, g.origin[1] + (float)j * g.h, g.origin[2] + (float)k * g.h);
    const V3 xc = world_to_cam(xw, cam);
    if (!(xc.z >= 0.01f) || !isfinite(xc.z)) return;
    float u, v;
    project_mean<DISTORTED>(xc, cam, u, v);
    if (!(u >= 0.0f && u < (float)w && v >= 0.0f && v < (float)h)) return;   // NaN fails every comparison
    const size_t pix = (size_t)(uint32_t)v * w + (uint32_t)u;
    const float4 c = __ldg(img + pix);
    if (!(c.w >= alpha_min)) return;
    const float ed = __fdiv_rn(__ldg(depth + pix), c.w);
    if (!(ed > 0.0f) || !isfinite(ed)) return;
    const float sdf = ed - xc.z;
    if (sdf < -g.trunc) return;
    const float f = fminf(1.0f, __fdiv_rn(sdf, g.trunc));
    const float col[3] = {fminf(fmaxf(__fdiv_rn(c.x, c.w), 0.0f), 1.0f), fminf(fmaxf(__fdiv_rn(c.y, c.w), 0.0f), 1.0f),
                          fminf(fmaxf(__fdiv_rn(c.z, c.w), 0.0f), 1.0f)};
    const float W = g.weight[idx], W1 = W + 1.0f;
    g.tsdf[idx] = __fdiv_rn(g.tsdf[idx] * W + f, W1);
    float *rgb = g.rgb + (size_t)idx * 3;
#pragma unroll
    for (int a = 0; a < 3; a++) rgb[a] = __fdiv_rn(rgb[a] * W + col[a], W1);
    g.weight[idx] = W1;
}

// ------------------------------------------------------------------------------------------------------ extraction
__global__ void __launch_bounds__(BRICK_PTS)
mesh_count_kernel(BgTsdfGrid g, uint32_t *__restrict__ brick_v, uint32_t *__restrict__ brick_t) {
    __shared__ uint32_t s_warp[32];
    const Brick p = brick_point(g);
    const Corners c = load_corners(g, p);
    uint32_t tv, tt;
    block_excl_scan(__popc(edge_mask(c)), s_warp, tv);
    block_excl_scan(cell_tris(c), s_warp, tt);
    if (threadIdx.x == 0) { brick_v[blockIdx.x] = tv; brick_t[blockIdx.x] = tt; }
}

// One CTA of 1024 threads: exclusive offsets of the bricks (u32; only meaningful when the totals fit) and the 64-bit
// totals in the header.
__global__ void __launch_bounds__(1024)
mesh_scan_kernel(uint32_t nb, uint3 dims, const uint32_t *__restrict__ brick_v, const uint32_t *__restrict__ brick_t,
                 uint32_t *__restrict__ voff, uint32_t *__restrict__ toff, unsigned long long *__restrict__ header) {
    __shared__ uint32_t s_warp[32];
    unsigned long long cv = 0, ct = 0;
    for (uint32_t base = 0; base < nb; base += 1024) {
        const uint32_t b = base + threadIdx.x;
        const uint32_t v = b < nb ? brick_v[b] : 0u, t = b < nb ? brick_t[b] : 0u;
        uint32_t sv, st;
        const uint32_t ev = block_excl_scan(v, s_warp, sv), et = block_excl_scan(t, s_warp, st);
        if (b < nb) { voff[b] = (uint32_t)(cv + ev); toff[b] = (uint32_t)(ct + et); }
        cv += sv;
        ct += st;
    }
    if (threadIdx.x == 0) {
        header[MH_VERTS] = cv;
        header[MH_TRIS] = ct;
        header[MH_DIMS] = dims.x; header[MH_DIMS + 1] = dims.y; header[MH_DIMS + 2] = dims.z;
    }
}

__global__ void __launch_bounds__(BRICK_PTS)
mesh_vertices_kernel(BgTsdfGrid g, const uint32_t *__restrict__ voff, uint32_t max_vertices, uint32_t *__restrict__ vbase,
                     uint8_t *__restrict__ vmask, float *__restrict__ verts, uint8_t *__restrict__ colors) {
    __shared__ uint32_t s_warp[32];
    const Brick p = brick_point(g);
    const Corners c = load_corners(g, p);
    const uint32_t m = edge_mask(c);
    uint32_t tot;
    uint32_t id = __ldg(voff + blockIdx.x) + block_excl_scan(__popc(m), s_warp, tot);
    if (!p.in) return;
    const size_t q0 = lin(g, p.i, p.j, p.k);
    vbase[q0] = id;
    vmask[q0] = (uint8_t)m;
    if (!m) return;
    const float x0[3] = {g.origin[0] + (float)p.i * g.h, g.origin[1] + (float)p.j * g.h, g.origin[2] + (float)p.k * g.h};
    const float *c0 = g.rgb + q0 * 3;
#pragma unroll
    for (uint32_t d = 0; d < 7; d++) {
        if (!((m >> d) & 1u)) continue;
        const uint32_t b = dir_bits(d);
        if (id >= max_vertices) break;   // only when the grid changed after bg_mesh_count: never write out of bounds
        const uint32_t e[3] = {b & 1u, (b >> 1) & 1u, b >> 2};
        const size_t q1 = lin(g, p.i + e[0], p.j + e[1], p.k + e[2]);
        const float t = __fdiv_rn(c.t[0], c.t[0] - c.t[b]);
        const uint32_t ijk[3] = {p.i, p.j, p.k};
        const float *c1 = g.rgb + q1 * 3;
#pragma unroll
        for (int a = 0; a < 3; a++) {
            const float x1 = g.origin[a] + (float)(ijk[a] + e[a]) * g.h;
            verts[(size_t)id * 3 + a] = x0[a] + t * (x1 - x0[a]);
            const float ca = __ldg(c0 + a), cb = __ldg(c1 + a);
            const float cc = fminf(fmaxf(ca + t * (cb - ca), 0.0f), 1.0f);
            colors[(size_t)id * 3 + a] = (uint8_t)rintf(cc * 255.0f);
        }
        id++;
    }
}

// Vertex id of the edge between cell corners ca -> cb (ca a subset of cb): the owner point p + ca, direction cb ^ ca.
__device__ __forceinline__ uint32_t edge_id(const BgTsdfGrid &g, const Brick &p, uint32_t ca, uint32_t cb,
                                            const uint32_t *__restrict__ vbase, const uint8_t *__restrict__ vmask) {
    const size_t q = lin(g, p.i + (ca & 1u), p.j + ((ca >> 1) & 1u), p.k + (ca >> 2));
    const uint32_t d = dir_index(cb ^ ca);
    return __ldg(vbase + q) + __popc(__ldg(vmask + q) & ((1u << d) - 1u));
}

// Triangles of one tetrahedron with sign pattern s, wound so that each normal points toward the T >= 0 side.
//   one corner i apart (1 or 3 negative): triangle on edges (i,j), (i,k), (i,l), j < k < l.  det(v_j - v_i, v_k - v_i,
//     v_l - v_i) = (-1)^i times the tetrahedron's orientation; the normal points away from v_i when that is positive,
//     which is right when v_i is the negative corner.
//   two and two (negative i < j, positive k < l): the quad (i,k) (i,l) (j,l) (j,k) faces the positive side when the
//     orientation times the sign of the permutation (i, j, k, l) is positive; it is split along (i,k)-(j,l).
__device__ __forceinline__ uint32_t emit_tet(const BgTsdfGrid &g, const Brick &p, uint32_t t, uint32_t s, uint32_t *out,
                                             const uint32_t *__restrict__ vbase, const uint8_t *__restrict__ vmask) {
    const uint32_t c1 = tet_c1(t), c2 = tet_c2(t);
    const bool even = tet_even(t);
    auto cbits = [&](uint32_t v) { return v == 0 ? 0u : v == 1 ? c1 : v == 2 ? c2 : 7u; };
    auto E = [&](uint32_t a, uint32_t b) {
        return a < b ? edge_id(g, p, cbits(a), cbits(b), vbase, vmask) : edge_id(g, p, cbits(b), cbits(a), vbase, vmask);
    };
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

__global__ void __launch_bounds__(BRICK_PTS)
mesh_faces_kernel(BgTsdfGrid g, const uint32_t *__restrict__ toff, uint32_t max_triangles, const uint32_t *__restrict__ vbase,
                  const uint8_t *__restrict__ vmask, uint32_t *__restrict__ faces) {
    __shared__ uint32_t s_warp[32];
    const Brick p = brick_point(g);
    const Corners c = load_corners(g, p);
    const uint32_t nt = cell_tris(c);
    uint32_t tot;
    const uint32_t f0 = __ldg(toff + blockIdx.x) + block_excl_scan(nt, s_warp, tot);
    if (!nt || f0 + nt > max_triangles || f0 + nt < f0) return;   // the guard only fires when the grid changed after the count
    uint32_t *out = faces + (size_t)f0 * 3;
    for (uint32_t t = 0; t < 6; t++) {
        const uint32_t s = tet_signs(c, t);
        out += 3 * emit_tet(g, p, t, s, out, vbase, vmask);
    }
}

// ---------------------------------------------------------------------------------------------- launchers
cudaError_t launch_tsdf_integrate(cudaStream_t s, const BgTsdfGrid &g, const BgCamera &cam, uint32_t w, uint32_t h,
                                  const float *img, const float *depth, float alpha_min) {
    const uint32_t n = g.dims[0] * g.dims[1] * g.dims[2];
    const uint32_t blocks = (n + 255) / 256;
    if (cam.camera_model == BG_CAMERA_PINHOLE)
        tsdf_integrate_kernel<false><<<blocks, 256, 0, s>>>(g, cam, w, h, reinterpret_cast<const float4 *>(img), depth, alpha_min);
    else
        tsdf_integrate_kernel<true><<<blocks, 256, 0, s>>>(g, cam, w, h, reinterpret_cast<const float4 *>(img), depth, alpha_min);
    return cudaGetLastError();
}

uint32_t mesh_num_bricks(const uint32_t *dims) { return ((dims[0] + 7) / 8) * ((dims[1] + 7) / 8) * ((dims[2] + 7) / 8); }

cudaError_t launch_mesh_count(cudaStream_t s, const BgTsdfGrid &g, uint32_t *brick_v, uint32_t *brick_t, uint32_t *voff,
                              uint32_t *toff, unsigned long long *header) {
    const uint32_t nb = mesh_num_bricks(g.dims);
    mesh_count_kernel<<<nb, BRICK_PTS, 0, s>>>(g, brick_v, brick_t);
    mesh_scan_kernel<<<1, 1024, 0, s>>>(nb, make_uint3(g.dims[0], g.dims[1], g.dims[2]), brick_v, brick_t, voff, toff, header);
    return cudaGetLastError();
}

cudaError_t launch_mesh_emit(cudaStream_t s, const BgTsdfGrid &g, const uint32_t *voff, const uint32_t *toff, uint32_t *vbase,
                             uint8_t *vmask, uint32_t max_vertices, uint32_t max_triangles, float *verts, uint8_t *colors,
                             uint32_t *faces) {
    const uint32_t nb = mesh_num_bricks(g.dims);
    mesh_vertices_kernel<<<nb, BRICK_PTS, 0, s>>>(g, voff, max_vertices, vbase, vmask, verts, colors);
    mesh_faces_kernel<<<nb, BRICK_PTS, 0, s>>>(g, toff, max_triangles, vbase, vmask, faces);
    return cudaGetLastError();
}

}  // namespace bg
