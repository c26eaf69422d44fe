// mesh_sparse.cu -- the sparse brick TSDF: the dense grid's lattice (mesh.cu), stored only in the 8^3-point bricks that
// can hold the surface.  DESIGN.md section 4.10 is the specification and states why its mesh is bit-identical to the
// dense grid's over the same lattice; tests/sparse_mesh_ref.py restates the marking in numpy.
//
//   sparse_pyramid_base_kernel   one thread per pixel: the valid expected depth D / a of one view (min = max = D / a, or
//                                (+inf, -inf) where the dense integration would skip the pixel)
//   sparse_pyramid_reduce_kernel one thread per cell of the next level: min / max over 2 x 2 cells
//   sparse_candidate_kernel      one thread per unmarked brick: a conservative test that the view can update one of its
//                                points with f < 0; survivors are appended to a list
//   sparse_confirm_kernel        one CTA per listed brick (a persistent grid): the exact near test of every point, through
//                                the dense integration's device function; one bit per brick ORed into the bitmap
//   sparse_alloc_count_kernel    one thread per brick: allocated when a marked brick lies in its 3^3-brick neighbourhood;
//                                per-CTA counts
//   sparse_scan_kernel           one CTA: exclusive scan of per-block counts, 64-bit totals
//   sparse_assign_kernel         slots in linear brick order: brick_slot, and the brick of every slot
//   sparse_integrate_kernel      one CTA per allocated brick: the dense kernel's per-point update
//   sparse_mesh_count_kernel / sparse_mesh_vertices_kernel / sparse_mesh_faces_kernel
//                                mesh.cu's extraction, one CTA per allocated brick in slot order; points of the +1
//                                neighbour bricks are found through brick_slot, and an unallocated brick reads as
//                                unobserved
//
// Compiled with -fmad=false, like mesh.cu.
#include <cstdint>

#include "bg_mesh.cuh"
#include "bg_launch.cuh"

namespace bg {

constexpr uint32_t UNALLOCATED = 0xFFFFFFFFu;
constexpr uint32_t SCAN_BLOCK = 1024;      // bricks per CTA of the allocation kernels

// The expected-depth pyramid of a w x h view: level l is ceil(w / 2^l) x ceil(h / 2^l) float2 cells (min, max), stored one
// level after the other, up to the level of one cell.
__host__ __device__ __forceinline__ uint32_t level_w(uint32_t w, uint32_t l) { return ((w - 1) >> l) + 1; }
__host__ __device__ __forceinline__ uint64_t level_off(uint32_t w, uint32_t h, uint32_t l) {
    uint64_t off = 0;
    for (uint32_t q = 0; q < l; q++) off += (uint64_t)level_w(w, q) * level_w(h, q);
    return off;
}
static uint32_t pyramid_levels(uint32_t w, uint32_t h) {
    uint32_t l = 0;
    while (level_w(w, l) > 1 || level_w(h, l) > 1) l++;
    return l + 1;
}
uint64_t sparse_pyramid_cells(uint32_t w, uint32_t h) { return level_off(w, h, pyramid_levels(w, h)); }

__device__ __forceinline__ V3 lattice_point(const BgSparseTsdfGrid &g, uint32_t i, uint32_t j, uint32_t k) {
    return mk3(g.origin[0] + (float)i * g.h, g.origin[1] + (float)j * g.h, g.origin[2] + (float)k * g.h);
}

// The thread's point of brick b (threadIdx.x = x + 8 y + 64 z inside the brick).
struct SPoint {
    uint32_t i, j, k;
    bool in;
};
__device__ __forceinline__ SPoint sparse_point(const BgSparseTsdfGrid &g, uint32_t b) {
    const uint32_t nbx = (g.dims[0] + 7) / 8, nby = (g.dims[1] + 7) / 8;
    const uint32_t bx = b % nbx, r = b / nbx, by = r % nby, bz = r / nby;
    SPoint p;
    p.i = bx * 8 + (threadIdx.x & 7);
    p.j = by * 8 + ((threadIdx.x >> 3) & 7);
    p.k = bz * 8 + (threadIdx.x >> 6);
    p.in = p.i < g.dims[0] && p.j < g.dims[1] && p.k < g.dims[2];
    return p;
}

// ------------------------------------------------------------------------------------------------------ marking
// Level 0 of the expected-depth pyramid: exactly the ed of the dense integration's steps 4 (tsdf_sample), or an empty
// range where a pixel updates nothing.
__global__ void __launch_bounds__(256)
sparse_pyramid_base_kernel(uint32_t w, uint32_t h, const float4 *__restrict__ img, const float *__restrict__ depth,
                           float alpha_min, float2 *__restrict__ out) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= w) return;
    const size_t pix = (size_t)y * w + x;
    const float a = __ldg(img + pix).w;
    float2 m = make_float2(INFINITY, -INFINITY);
    if (a >= alpha_min) {
        const float ed = __fdiv_rn(__ldg(depth + pix), a);
        if (ed > 0.0f && isfinite(ed)) m = make_float2(ed, ed);
    }
    out[pix] = m;
}

__global__ void __launch_bounds__(256)
sparse_pyramid_reduce_kernel(uint32_t w0, uint32_t h0, const float2 *__restrict__ in, uint32_t w1, float2 *__restrict__ out) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= w1) return;
    float2 m = make_float2(INFINITY, -INFINITY);
#pragma unroll
    for (uint32_t c = 0; c < 4; c++) {
        const uint32_t xx = 2 * x + (c & 1), yy = 2 * y + (c >> 1);
        if (xx < w0 && yy < h0) {
            const float2 v = in[(size_t)yy * w0 + xx];
            m.x = fminf(m.x, v.x);
            m.y = fmaxf(m.y, v.y);
        }
    }
    out[(size_t)y * w1 + x] = m;
}

// Brick b may hold a point that the view updates with f < 0 (DESIGN.md section 4.10).  Camera-space box: the 8 corners
// through the dense kernel's world_to_cam, grown per axis by 2^-19 (sum |R| |x| + |t|).  The float transform of a corner
// or of a point is within 2^-22 (sum |R| |x| + |t|) of the exact one, so the grown box holds the float camera position of
// every point of the brick.  A box with no part at z >= 0.01 is dropped.  Pinhole, box wholly at z >= 0.01: pixel rectangle from x / z over the box's extremes with directed rounding,
// grown by 1 px for the projection's own rounding; otherwise the whole image.  Kept when a pyramid cell over the
// rectangle holds an ed range meeting [z_lo - trunc (1 + 2^-20), z_hi].
template <bool DISTORTED>
__global__ void __launch_bounds__(256)
sparse_candidate_kernel(BgSparseTsdfGrid g, BgCamera cam, uint32_t w, uint32_t h, const float2 *__restrict__ pyramid,
                        const uint32_t *__restrict__ bitmap, const unsigned long long *__restrict__ header, uint32_t nb,
                        uint32_t *__restrict__ cand, uint32_t *__restrict__ cand_count) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb || header[SPARSE_H_ALLOCATED]) return;   // marking ends with the allocation
    if ((__ldg(bitmap + (b >> 5)) >> (b & 31)) & 1u) return;   // marked by an earlier view
    const uint32_t nbx = (g.dims[0] + 7) / 8, nby = (g.dims[1] + 7) / 8;
    const uint32_t bi[3] = {b % nbx, (b / nbx) % nby, (b / nbx) / nby};
    float lo[3], hi[3], mag[3];
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const uint32_t i0 = bi[a] * 8, i1 = min(i0 + 7, g.dims[a] - 1);
        lo[a] = g.origin[a] + (float)i0 * g.h;   // the lattice formula is monotone in i: the brick's points lie in [lo, hi]
        hi[a] = g.origin[a] + (float)i1 * g.h;
        mag[a] = fmaxf(fabsf(lo[a]), fabsf(hi[a]));
    }
    V3 cmin = mk3(INFINITY, INFINITY, INFINITY), cmax = mk3(-INFINITY, -INFINITY, -INFINITY);
#pragma unroll
    for (uint32_t c = 0; c < 8; c++) {
        const V3 xc = world_to_cam(mk3((c & 1) ? hi[0] : lo[0], (c & 2) ? hi[1] : lo[1], (c & 4) ? hi[2] : lo[2]), cam);
        cmin = mk3(fminf(cmin.x, xc.x), fminf(cmin.y, xc.y), fminf(cmin.z, xc.z));
        cmax = mk3(fmaxf(cmax.x, xc.x), fmaxf(cmax.y, xc.y), fmaxf(cmax.z, xc.z));
    }
    float grow[3];
#pragma unroll
    for (int a = 0; a < 3; a++)
        grow[a] = 0x1p-19f * (fabsf(cam.viewmat[a]) * mag[0] + fabsf(cam.viewmat[3 + a]) * mag[1] +
                               fabsf(cam.viewmat[6 + a]) * mag[2] + fabsf(cam.viewmat[9 + a]));
    const float zl = __fsub_rd(cmin.z, grow[2]), zh = __fadd_ru(cmax.z, grow[2]);
    if (!(zh >= 0.01f)) return;   // no point of the brick is in front of the camera (NaN: none passes the near test either)
    uint32_t x0 = 0, x1 = w - 1, y0 = 0, y1 = h - 1;
    if (!DISTORTED && zl >= 0.01f && cam.fx > 0.0f && cam.fy > 0.0f) {
        const float xl = __fsub_rd(cmin.x, grow[0]), xh = __fadd_ru(cmax.x, grow[0]);
        const float yl = __fsub_rd(cmin.y, grow[1]), yh = __fadd_ru(cmax.y, grow[1]);
        const float ul = __fadd_rd(__fmul_rd(cam.fx, fminf(__fdiv_rd(xl, zl), __fdiv_rd(xl, zh))), cam.cx) - 1.0f;
        const float uh = __fadd_ru(__fmul_ru(cam.fx, fmaxf(__fdiv_ru(xh, zl), __fdiv_ru(xh, zh))), cam.cx) + 1.0f;
        const float vl = __fadd_rd(__fmul_rd(cam.fy, fminf(__fdiv_rd(yl, zl), __fdiv_rd(yl, zh))), cam.cy) - 1.0f;
        const float vh = __fadd_ru(__fmul_ru(cam.fy, fmaxf(__fdiv_ru(yh, zl), __fdiv_ru(yh, zh))), cam.cy) + 1.0f;
        if (isfinite(ul) && isfinite(uh) && isfinite(vl) && isfinite(vh)) {
            if (uh < 0.0f || ul >= (float)w || vh < 0.0f || vl >= (float)h) return;   // wholly off the image
            x0 = (uint32_t)fmaxf(ul, 0.0f);
            x1 = (uint32_t)fminf(uh, (float)(w - 1));
            y0 = (uint32_t)fmaxf(vl, 0.0f);
            y1 = (uint32_t)fminf(vh, (float)(h - 1));
        }
    }
    const float ed_lo = __fsub_rd(zl, __fmul_ru(g.trunc, 1.0f + 0x1p-20f)), ed_hi = zh;
    uint32_t L = 0;
    while ((x1 >> L) - (x0 >> L) > 3 || (y1 >> L) - (y0 >> L) > 3) L++;   // the top level is one cell: L stays in range
    const float2 *lv = pyramid + level_off(w, h, L);
    const uint32_t lw = level_w(w, L);
    bool hit = false;   // written so that a NaN bound keeps the brick
    for (uint32_t cy = y0 >> L; cy <= (y1 >> L); cy++)
        for (uint32_t cx = x0 >> L; cx <= (x1 >> L); cx++) {
            const float2 m = lv[(size_t)cy * lw + cx];
            hit |= !(m.x > ed_hi) && !(m.y < ed_lo);
        }
    if (hit) cand[atomicAdd(cand_count, 1u)] = b;
}

template <bool DISTORTED>
__global__ void __launch_bounds__(BRICK_PTS)
sparse_confirm_kernel(BgSparseTsdfGrid g, BgCamera cam, uint32_t w, uint32_t h, const float4 *__restrict__ img,
                      const float *__restrict__ depth, float alpha_min, const uint32_t *__restrict__ cand,
                      const uint32_t *__restrict__ cand_count, uint32_t *__restrict__ bitmap) {
    const uint32_t n = *cand_count;
    for (uint32_t c = blockIdx.x; c < n; c += gridDim.x) {
        const uint32_t b = cand[c];
        const SPoint p = sparse_point(g, b);
        TsdfSample s;
        const bool near = p.in && tsdf_sample<DISTORTED>(lattice_point(g, p.i, p.j, p.k), g.trunc, cam, w, h, img, depth,
                                                         alpha_min, s) && s.f < 0.0f;
        if (__syncthreads_or(near) && threadIdx.x == 0) atomicOr(bitmap + (b >> 5), 1u << (b & 31));
    }
}

// ------------------------------------------------------------------------------------------------------ allocation
__device__ __forceinline__ bool brick_dilated(const uint32_t *__restrict__ bitmap, uint32_t b, uint32_t nbx, uint32_t nby,
                                              uint32_t nbz) {
    const int bx = b % nbx, by = (b / nbx) % nby, bz = (b / nbx) / nby;
    for (int dz = -1; dz <= 1; dz++)
        for (int dy = -1; dy <= 1; dy++)
            for (int dx = -1; dx <= 1; dx++) {
                const int x = bx + dx, y = by + dy, z = bz + dz;
                if (x < 0 || y < 0 || z < 0 || x >= (int)nbx || y >= (int)nby || z >= (int)nbz) continue;
                const uint32_t q = ((uint32_t)z * nby + (uint32_t)y) * nbx + (uint32_t)x;
                if ((__ldg(bitmap + (q >> 5)) >> (q & 31)) & 1u) return true;
            }
    return false;
}

__global__ void __launch_bounds__(SCAN_BLOCK)
sparse_alloc_count_kernel(uint32_t nb, uint3 nbd, const uint32_t *__restrict__ bitmap, uint32_t *__restrict__ blk_cnt) {
    __shared__ uint32_t s_warp[32];
    const uint32_t b = blockIdx.x * SCAN_BLOCK + threadIdx.x;
    const uint32_t f = b < nb && brick_dilated(bitmap, b, nbd.x, nbd.y, nbd.z);
    uint32_t tot;
    block_excl_scan(f, s_warp, tot);
    if (threadIdx.x == 0) blk_cnt[blockIdx.x] = tot;
}

// One CTA of 1024 threads: exclusive u32 offsets of a[n] (and b[n] when b is not null); out[0] (out[1]) the 64-bit totals,
// out[2..5] = meta.
__global__ void __launch_bounds__(1024)
sparse_scan_kernel(uint32_t n, const uint32_t *__restrict__ a, const uint32_t *__restrict__ b, uint32_t *__restrict__ aoff,
                   uint32_t *__restrict__ boff, uint4 meta, unsigned long long *__restrict__ out) {
    __shared__ uint32_t s_warp[32];
    unsigned long long ca = 0, cb = 0;
    for (uint32_t base = 0; base < n; base += 1024) {
        const uint32_t q = base + threadIdx.x;
        const uint32_t va = q < n ? a[q] : 0u, vb = (b && q < n) ? b[q] : 0u;
        uint32_t sa, sb;
        const uint32_t ea = block_excl_scan(va, s_warp, sa), eb = block_excl_scan(vb, s_warp, sb);
        if (q < n) {
            aoff[q] = (uint32_t)(ca + ea);
            if (b) boff[q] = (uint32_t)(cb + eb);
        }
        ca += sa;
        cb += sb;
    }
    if (threadIdx.x == 0) {
        out[0] = ca;
        if (b) out[1] = cb;
        out[2] = meta.x; out[3] = meta.y; out[4] = meta.z; out[5] = meta.w;
    }
}

__global__ void __launch_bounds__(SCAN_BLOCK)
sparse_assign_kernel(uint32_t nb, uint3 nbd, const uint32_t *__restrict__ bitmap, const uint32_t *__restrict__ blk_off,
                     uint32_t *__restrict__ brick_slot, uint32_t *__restrict__ slot_brick) {
    __shared__ uint32_t s_warp[32];
    const uint32_t b = blockIdx.x * SCAN_BLOCK + threadIdx.x;
    const uint32_t f = b < nb && brick_dilated(bitmap, b, nbd.x, nbd.y, nbd.z);
    uint32_t tot;
    const uint32_t slot = __ldg(blk_off + blockIdx.x) + block_excl_scan(f, s_warp, tot);
    if (b >= nb) return;
    brick_slot[b] = f ? slot : UNALLOCATED;
    if (f) slot_brick[slot] = b;   // slot <= b < nb
}

// ------------------------------------------------------------------------------------------------------ integration
template <bool DISTORTED>
__global__ void __launch_bounds__(BRICK_PTS)
sparse_integrate_kernel(BgSparseTsdfGrid g, BgCamera cam, uint32_t w, uint32_t h, const float4 *__restrict__ img,
                        const float *__restrict__ depth, float alpha_min, const uint32_t *__restrict__ slot_brick) {
    const SPoint p = sparse_point(g, __ldg(slot_brick + blockIdx.x));
    if (!p.in) return;
    TsdfSample s;
    if (tsdf_sample<DISTORTED>(lattice_point(g, p.i, p.j, p.k), g.trunc, cam, w, h, img, depth, alpha_min, s))
        tsdf_update(g.tsdf, g.weight, g.rgb, (size_t)blockIdx.x * BRICK_PTS + threadIdx.x, s);
}

// ------------------------------------------------------------------------------------------------------ extraction
constexpr size_t NO_POINT = ~(size_t)0;

// Pool index of lattice point (i, j, k) inside the grid, or NO_POINT when its brick is unallocated.
__device__ __forceinline__ size_t pool_index(const BgSparseTsdfGrid &g, uint32_t i, uint32_t j, uint32_t k) {
    const uint32_t nbx = (g.dims[0] + 7) / 8, nby = (g.dims[1] + 7) / 8;
    const uint32_t s = __ldg(g.brick_slot + ((k >> 3) * nby + (j >> 3)) * nbx + (i >> 3));
    return s == UNALLOCATED ? NO_POINT : (size_t)s * BRICK_PTS + (((k & 7) * 8 + (j & 7)) * 8 + (i & 7));
}

// mesh.cu's load_corners over the pool: corners in the thread's own brick (slot `own`) are read directly, the others
// through brick_slot.
__device__ __forceinline__ Corners load_corners_sparse(const BgSparseTsdfGrid &g, const SPoint &p, uint32_t own) {
    Corners c;
    c.obs = 0;
    c.neg = 0;
#pragma unroll
    for (uint32_t b = 0; b < 8; b++) {
        const uint32_t i = p.i + (b & 1u), j = p.j + ((b >> 1) & 1u), k = p.k + (b >> 2);
        c.t[b] = 0.0f;
        if (p.in && i < g.dims[0] && j < g.dims[1] && k < g.dims[2]) {
            const bool same = ((i ^ p.i) | (j ^ p.j) | (k ^ p.k)) < 8;   // no carry out of the brick's low 3 bits
            const size_t q = same ? (size_t)own * BRICK_PTS + (((k & 7) * 8 + (j & 7)) * 8 + (i & 7)) : pool_index(g, i, j, k);
            if (q != NO_POINT && __ldg(g.weight + q) != 0.0f) {
                c.t[b] = __ldg(g.tsdf + q);
                c.obs |= 1u << b;
                if (c.t[b] < 0.0f) c.neg |= 1u << b;
            }
        }
    }
    return c;
}

__global__ void __launch_bounds__(BRICK_PTS)
sparse_mesh_count_kernel(BgSparseTsdfGrid g, const uint32_t *__restrict__ slot_brick, uint32_t *__restrict__ brick_v,
                         uint32_t *__restrict__ brick_t) {
    __shared__ uint32_t s_warp[32];
    const SPoint p = sparse_point(g, __ldg(slot_brick + blockIdx.x));
    const Corners c = load_corners_sparse(g, p, blockIdx.x);
    uint32_t tv, tt;
    block_excl_scan(__popc(edge_mask(c)), s_warp, tv);
    block_excl_scan(cell_tris(c), s_warp, tt);
    if (threadIdx.x == 0) { brick_v[blockIdx.x] = tv; brick_t[blockIdx.x] = tt; }
}

__global__ void __launch_bounds__(BRICK_PTS)
sparse_mesh_vertices_kernel(BgSparseTsdfGrid g, const uint32_t *__restrict__ slot_brick, const uint32_t *__restrict__ voff,
                            uint32_t max_vertices, uint32_t *__restrict__ vbase, uint8_t *__restrict__ vmask,
                            float *__restrict__ verts, uint8_t *__restrict__ colors) {
    __shared__ uint32_t s_warp[32];
    const SPoint p = sparse_point(g, __ldg(slot_brick + blockIdx.x));
    const Corners c = load_corners_sparse(g, p, blockIdx.x);
    const uint32_t m = edge_mask(c);
    uint32_t tot;
    uint32_t id = __ldg(voff + blockIdx.x) + block_excl_scan(__popc(m), s_warp, tot);
    if (!p.in) return;
    const size_t q0 = (size_t)blockIdx.x * BRICK_PTS + threadIdx.x;
    vbase[q0] = id;
    vmask[q0] = (uint8_t)m;
    if (!m) return;
    const float x0[3] = {g.origin[0] + (float)p.i * g.h, g.origin[1] + (float)p.j * g.h, g.origin[2] + (float)p.k * g.h};
    const float *c0 = g.rgb + q0 * 3;
#pragma unroll
    for (uint32_t d = 0; d < 7; d++) {
        if (!((m >> d) & 1u)) continue;
        const uint32_t b = dir_bits(d);
        if (id >= max_vertices) break;   // only when the grid changed after the count: never write out of bounds
        const uint32_t e[3] = {b & 1u, (b >> 1) & 1u, b >> 2};
        const size_t q1 = pool_index(g, p.i + e[0], p.j + e[1], p.k + e[2]);   // observed, so allocated
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

__global__ void __launch_bounds__(BRICK_PTS)
sparse_mesh_faces_kernel(BgSparseTsdfGrid g, const uint32_t *__restrict__ slot_brick, const uint32_t *__restrict__ toff,
                         uint32_t max_triangles, const uint32_t *__restrict__ vbase, const uint8_t *__restrict__ vmask,
                         uint32_t *__restrict__ faces) {
    __shared__ uint32_t s_warp[32];
    const SPoint p = sparse_point(g, __ldg(slot_brick + blockIdx.x));
    const Corners c = load_corners_sparse(g, p, blockIdx.x);
    const uint32_t nt = cell_tris(c);
    uint32_t tot;
    const uint32_t f0 = __ldg(toff + blockIdx.x) + block_excl_scan(nt, s_warp, tot);
    if (!nt || f0 + nt > max_triangles || f0 + nt < f0) return;   // the guard only fires when the grid changed after the count
    // every corner of a cell that emits is observed, so every owner below is allocated
    auto edge_id = [&](uint32_t ca, uint32_t cb) {
        const size_t q = pool_index(g, p.i + (ca & 1u), p.j + ((ca >> 1) & 1u), p.k + (ca >> 2));
        const uint32_t d = dir_index(cb ^ ca);
        return __ldg(vbase + q) + __popc(__ldg(vmask + q) & ((1u << d) - 1u));
    };
    uint32_t *out = faces + (size_t)f0 * 3;
    for (uint32_t t = 0; t < 6; t++) out += 3 * emit_tet(t, tet_signs(c, t), out, edge_id);
}

// ---------------------------------------------------------------------------------------------- launchers
static uint32_t sparse_num_bricks(const uint32_t *dims) { return ((dims[0] + 7) / 8) * ((dims[1] + 7) / 8) * ((dims[2] + 7) / 8); }
static uint3 brick_dims(const uint32_t *dims) { return make_uint3((dims[0] + 7) / 8, (dims[1] + 7) / 8, (dims[2] + 7) / 8); }

cudaError_t launch_sparse_mark(cudaStream_t s, int sm_count, const BgSparseTsdfGrid &g, const BgCamera &cam, uint32_t w, uint32_t h,
                               const float *img, const float *depth, float alpha_min, const SparseTsdfWs &ws) {
    const float4 *img4 = reinterpret_cast<const float4 *>(img);
    const uint32_t levels = pyramid_levels(w, h);
    const uint32_t nb = sparse_num_bricks(g.dims);
    cudaError_t e = cudaMemsetAsync(ws.cand_count, 0, sizeof(uint32_t), s);
    if (e != cudaSuccess) return e;
    sparse_pyramid_base_kernel<<<dim3((w + 255) / 256, h), 256, 0, s>>>(w, h, img4, depth, alpha_min, ws.pyramid);
    for (uint32_t l = 1; l < levels; l++)
        sparse_pyramid_reduce_kernel<<<dim3((level_w(w, l) + 255) / 256, level_w(h, l)), 256, 0, s>>>(
            level_w(w, l - 1), level_w(h, l - 1), ws.pyramid + level_off(w, h, l - 1), level_w(w, l), ws.pyramid + level_off(w, h, l));
    const uint32_t blocks = (nb + 255) / 256;
    if (cam.camera_model == BG_CAMERA_PINHOLE) {
        sparse_candidate_kernel<false><<<blocks, 256, 0, s>>>(g, cam, w, h, ws.pyramid, ws.bitmap, ws.header, nb, ws.list,
                                                              ws.cand_count);
        sparse_confirm_kernel<false><<<sm_count * 4, BRICK_PTS, 0, s>>>(g, cam, w, h, img4, depth, alpha_min, ws.list,
                                                                        ws.cand_count, ws.bitmap);
    } else {
        sparse_candidate_kernel<true><<<blocks, 256, 0, s>>>(g, cam, w, h, ws.pyramid, ws.bitmap, ws.header, nb, ws.list,
                                                             ws.cand_count);
        sparse_confirm_kernel<true><<<sm_count * 4, BRICK_PTS, 0, s>>>(g, cam, w, h, img4, depth, alpha_min, ws.list,
                                                                       ws.cand_count, ws.bitmap);
    }
    return cudaGetLastError();
}

cudaError_t launch_sparse_allocate(cudaStream_t s, const BgSparseTsdfGrid &g, const SparseTsdfWs &ws) {
    const uint32_t nb = sparse_num_bricks(g.dims), nblk = (nb + SCAN_BLOCK - 1) / SCAN_BLOCK;
    const uint3 nbd = brick_dims(g.dims);
    sparse_alloc_count_kernel<<<nblk, SCAN_BLOCK, 0, s>>>(nb, nbd, ws.bitmap, ws.blk_cnt);
    sparse_scan_kernel<<<1, 1024, 0, s>>>(nblk, ws.blk_cnt, nullptr, ws.blk_off, nullptr,
                                          make_uint4(1u, g.dims[0], g.dims[1], g.dims[2]), ws.header);
    sparse_assign_kernel<<<nblk, SCAN_BLOCK, 0, s>>>(nb, nbd, ws.bitmap, ws.blk_off, g.brick_slot, ws.list);
    return cudaGetLastError();
}

cudaError_t launch_sparse_integrate(cudaStream_t s, const BgSparseTsdfGrid &g, uint32_t slots, const BgCamera &cam, uint32_t w,
                                    uint32_t h, const float *img, const float *depth, float alpha_min, const SparseTsdfWs &ws) {
    const float4 *img4 = reinterpret_cast<const float4 *>(img);
    if (cam.camera_model == BG_CAMERA_PINHOLE)
        sparse_integrate_kernel<false><<<slots, BRICK_PTS, 0, s>>>(g, cam, w, h, img4, depth, alpha_min, ws.list);
    else
        sparse_integrate_kernel<true><<<slots, BRICK_PTS, 0, s>>>(g, cam, w, h, img4, depth, alpha_min, ws.list);
    return cudaGetLastError();
}

cudaError_t launch_sparse_mesh_count(cudaStream_t s, const BgSparseTsdfGrid &g, uint32_t slots, const SparseTsdfWs &ws,
                                     const SparseMeshWs &m) {
    if (slots) sparse_mesh_count_kernel<<<slots, BRICK_PTS, 0, s>>>(g, ws.list, m.brick_v, m.brick_t);
    sparse_scan_kernel<<<1, 1024, 0, s>>>(slots, m.brick_v, m.brick_t, m.voff, m.toff, make_uint4(slots, g.dims[0], g.dims[1], g.dims[2]),
                                          m.header);
    return cudaGetLastError();
}

cudaError_t launch_sparse_mesh_emit(cudaStream_t s, const BgSparseTsdfGrid &g, uint32_t slots, const SparseTsdfWs &ws,
                                    const SparseMeshWs &m, uint32_t max_vertices, uint32_t max_triangles, float *verts,
                                    uint8_t *colors, uint32_t *faces) {
    sparse_mesh_vertices_kernel<<<slots, BRICK_PTS, 0, s>>>(g, ws.list, m.voff, max_vertices, m.vbase, m.vmask, verts, colors);
    sparse_mesh_faces_kernel<<<slots, BRICK_PTS, 0, s>>>(g, ws.list, m.toff, max_triangles, m.vbase, m.vmask, faces);
    return cudaGetLastError();
}

}  // namespace bg
