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

#include "bg_mesh.cuh"
#include "bg_launch.cuh"

namespace bg {

// workspace header words (u64): vertex total, triangle total, the dims the counts belong to
constexpr uint32_t MH_VERTS = 0, MH_TRIS = 1, MH_DIMS = 2, MH_WORDS = 8;

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

// The cell corners at p (bg_mesh.cuh): corners outside the grid are neither read nor observed.
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
    TsdfSample s;
    if (tsdf_sample<DISTORTED>(xw, g.trunc, cam, w, h, img, depth, alpha_min, s)) tsdf_update(g.tsdf, g.weight, g.rgb, idx, s);
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
        out += 3 * emit_tet(t, s, out, [&](uint32_t ca, uint32_t cb) { return edge_id(g, p, ca, cb, vbase, vmask); });
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
