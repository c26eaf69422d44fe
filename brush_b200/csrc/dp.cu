// dp.cu -- view-sharded data parallelism behind the C ABI (SURVEY.md 8e; the reference is single-device).
//
// Parameters are replicated, every rank renders its own views of the step's batch, and ONE exchange per step makes
// the gradient of the mean-over-views loss available on every rank:
//   small  [n][12]      = v_transforms (10) | v_raw_opac | visible, summed over the rank's views   -> all-reduce (SUM)
//   stat   [n][2]       = v_refine | max_radius, MAX over the rank's views (stats.rs:40-50)        -> all-reduce (MAX)
//   record [n][3 local] = v_color of each local view                                               -> all-gather
// (interleaved per Gaussian: a slice of the Gaussian range is one contiguous piece of each buffer)
// The SH gradient of one view is rank one per Gaussian (update.cu), so the views' colour gradients (12 B per
// Gaussian and view) replace the dense [n,K,3] gradient (192 B at K=16) on the wire; the optimiser pass rebuilds it in
// registers in global view order (view = rank * local + i), which makes the update bit-identical on every rank.
//
// Overlap (bg_train_step_views): the all-gather of the records and the all-reduce of `small` run back to back on the
// communicator's own stream.  The SH part of the update pass -- 70 % of its HBM traffic -- needs the gathered records only
// and runs on the caller's stream UNDER the all-reduce; the transforms / opacity / statistics part follows the all-reduce.
// (Slicing the Gaussian range into pipelined pieces was measured first: the per-collective latency ate what the overlap
// gave.)  bg_dp_exchange is the exchange on its own, optionally in slices of the Gaussian range; the receive buffer is
// laid out per slice ([world][len][3 local]) so that every all-gather lands contiguously.
//
// NCCL is bound at run time (dlopen of libnccl.so.2: the copy already loaded by the host process -- torch's in the
// Python mirror -- or the system one), so the library itself links against nothing but the CUDA runtime.
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <new>

#include "bg_common.cuh"
#include "bg_dp.cuh"

namespace bg {

// ---- minimal NCCL surface (stable since NCCL 2.x)
struct NcclApi {
    void *handle = nullptr;
    int (*GetUniqueId)(NcclUniqueId *) = nullptr;
    int (*CommInitRank)(void **, int, NcclUniqueId, int) = nullptr;
    int (*CommDestroy)(void *) = nullptr;
    int (*AllReduce)(const void *, void *, size_t, int, int, void *, cudaStream_t) = nullptr;
    int (*AllGather)(const void *, void *, size_t, int, void *, cudaStream_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    const char *(*GetErrorString)(int) = nullptr;
    bool ok = false;
};
constexpr int NCCL_FLOAT32 = 7, NCCL_SUM = 0, NCCL_MAX = 2;

static NcclApi &nccl() {
    static NcclApi api;
    static bool tried = false;
    if (tried) return api;
    tried = true;
    const char *names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char *nm : names) {
        api.handle = dlopen(nm, RTLD_NOW | RTLD_GLOBAL | RTLD_NOLOAD);   // the copy the process already holds
        if (api.handle) break;
    }
    if (!api.handle)
        for (const char *nm : names) {
            api.handle = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
            if (api.handle) break;
        }
    if (!api.handle) return api;
#define BG_SYM(field, name) *(void **)(&api.field) = dlsym(api.handle, name)
    BG_SYM(GetUniqueId, "ncclGetUniqueId");
    BG_SYM(CommInitRank, "ncclCommInitRank");
    BG_SYM(CommDestroy, "ncclCommDestroy");
    BG_SYM(AllReduce, "ncclAllReduce");
    BG_SYM(AllGather, "ncclAllGather");
    BG_SYM(GroupStart, "ncclGroupStart");
    BG_SYM(GroupEnd, "ncclGroupEnd");
    BG_SYM(GetErrorString, "ncclGetErrorString");
#undef BG_SYM
    api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllReduce && api.AllGather && api.GroupStart &&
             api.GroupEnd && api.GetErrorString;
    return api;
}

const char *dp_nccl_error(int code) {
    NcclApi &a = nccl();
    return a.ok ? a.GetErrorString(code) : "NCCL is not loaded";
}

int dp_unique_id(NcclUniqueId *out) {
    NcclApi &a = nccl();
    if (!a.ok) return -1;
    return a.GetUniqueId(out);
}

DpComm *dp_comm_create(int device, const NcclUniqueId &id, int rank, int world, int *nccl_rc) {
    *nccl_rc = 0;
    NcclApi &a = nccl();
    if (!a.ok) { *nccl_rc = -1; return nullptr; }
    DpComm *c = new (std::nothrow) DpComm();
    if (!c) return nullptr;
    c->device = device; c->rank = rank; c->world = world;
    if (cudaSetDevice(device) != cudaSuccess) { delete c; return nullptr; }
    int rc = a.CommInitRank(&c->comm, world, id, rank);
    if (rc != 0) { *nccl_rc = rc; delete c; return nullptr; }
    // highest priority: the collectives' few CTAs must be dispatched ahead of the queued CTAs of the compute grids they overlap
    int prio_lo = 0, prio_hi = 0;
    cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
    bool ok = cudaStreamCreateWithPriority(&c->stream, cudaStreamNonBlocking, prio_hi) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&c->ev_ready, cudaEventDisableTiming) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&c->ev_ready2, cudaEventDisableTiming) == cudaSuccess;
    for (int i = 0; i < DP_MAX_CHUNKS && ok; i++) ok = cudaEventCreateWithFlags(&c->ev_chunk[i], cudaEventDisableTiming) == cudaSuccess;
    if (!ok) { dp_comm_destroy(c); return nullptr; }
    return c;
}

void dp_comm_destroy(DpComm *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    NcclApi &a = nccl();
    if (c->comm && a.ok) a.CommDestroy(c->comm);
    if (c->ev_ready) cudaEventDestroy(c->ev_ready);
    if (c->ev_ready2) cudaEventDestroy(c->ev_ready2);
    for (int i = 0; i < DP_MAX_CHUNKS; i++)
        if (c->ev_chunk[i]) cudaEventDestroy(c->ev_chunk[i]);
    if (c->stream) cudaStreamDestroy(c->stream);
    delete c;
}

// Gaussian range of slice c of `chunks` (multiples of 64 rows so that every slice pointer stays 256-byte aligned).
void dp_chunk_range(uint32_t n, uint32_t chunks, uint32_t c, uint32_t *g0, uint32_t *len) {
    const uint64_t per = (((uint64_t)n + chunks - 1) / chunks + 63) / 64 * 64;
    const uint64_t a = std::min<uint64_t>(per * c, n), b = std::min<uint64_t>(per * (c + 1), n);
    *g0 = (uint32_t)a;
    *len = (uint32_t)(b - a);
}

// Enqueues slice `c` of the exchange on the communicator's stream (which must already wait on the producer of
// `small` / `record`) and records ev_chunk[c] behind it.  Returns 0 or the failing NCCL / CUDA code (negative = CUDA).
int dp_exchange_chunk(DpComm *cm, uint32_t n, uint32_t local, uint32_t chunks, uint32_t c, float *small, float *stat,
                      const float *record, float *recv) {
    NcclApi &a = nccl();
    uint32_t g0, len;
    dp_chunk_range(n, chunks, c, &g0, &len);
    const DpLayout L = dp_layout(n, local, (uint32_t)cm->world);
    int rc = 0;
    if (len > 0) {
        if ((rc = a.GroupStart()) != 0) return rc;
        rc = a.AllGather(record + (size_t)g0 * L.rec_row, recv + L.chunk_base(g0), (size_t)len * L.rec_row, NCCL_FLOAT32, cm->comm, cm->stream);
        if (rc == 0)
            rc = a.AllReduce(small + (size_t)g0 * DP_SMALL_ROW, small + (size_t)g0 * DP_SMALL_ROW, (size_t)len * DP_SMALL_ROW, NCCL_FLOAT32,
                             NCCL_SUM, cm->comm, cm->stream);
        if (rc == 0)
            rc = a.AllReduce(stat + (size_t)g0 * DP_STAT_ROW, stat + (size_t)g0 * DP_STAT_ROW, (size_t)len * DP_STAT_ROW, NCCL_FLOAT32,
                             NCCL_MAX, cm->comm, cm->stream);
        const int rc_end = a.GroupEnd();
        if (rc == 0) rc = rc_end;
        if (rc != 0) return rc;
    }
    if (cudaEventRecord(cm->ev_chunk[c], cm->stream) != cudaSuccess) return -1;
    return 0;
}

// The two halves of the exchange as separate collectives with an event behind each (the multi-view step runs the SH part of
// the update behind the all-gather, under the all-reduces): ev_chunk[0] = records gathered, ev_chunk[1] = small / stat reduced.
int dp_exchange_gather(DpComm *cm, uint32_t n, uint32_t local, const float *record, float *recv) {
    NcclApi &a = nccl();
    const DpLayout L = dp_layout(n, local, (uint32_t)cm->world);
    const int rc = a.AllGather(record, recv, L.rec_floats, NCCL_FLOAT32, cm->comm, cm->stream);
    if (rc != 0) return rc;
    return cudaEventRecord(cm->ev_chunk[0], cm->stream) == cudaSuccess ? 0 : -1;
}
int dp_exchange_reduce(DpComm *cm, uint32_t n, float *small, float *stat) {
    NcclApi &a = nccl();
    int rc = a.GroupStart();
    if (rc != 0) return rc;
    rc = a.AllReduce(small, small, (size_t)DP_SMALL_ROW * n, NCCL_FLOAT32, NCCL_SUM, cm->comm, cm->stream);
    if (rc == 0) rc = a.AllReduce(stat, stat, (size_t)DP_STAT_ROW * n, NCCL_FLOAT32, NCCL_MAX, cm->comm, cm->stream);
    const int rc_end = a.GroupEnd();
    if (rc == 0) rc = rc_end;
    if (rc != 0) return rc;
    return cudaEventRecord(cm->ev_chunk[1], cm->stream) == cudaSuccess ? 0 : -1;
}

// The views' camera positions ([local][4] floats per rank) travel once per step, ahead of the slices.
int dp_exchange_header(DpComm *cm, uint32_t local, const float *hdr, float *hdr_all) {
    NcclApi &a = nccl();
    return a.AllGather(hdr, hdr_all, (size_t)local * 4, NCCL_FLOAT32, cm->comm, cm->stream);
}

int dp_exchange_grids(DpComm *cm, size_t floats, const float *send, float *recv) {
    NcclApi &a = nccl();
    const int rc = a.AllGather(send, recv, floats, NCCL_FLOAT32, cm->comm, cm->stream);
    if (rc != 0) return rc;
    return cudaEventRecord(cm->ev_chunk[2], cm->stream) == cudaSuccess ? 0 : -1;
}

// ---- small device helpers of the multi-view step
__global__ void write_header_kernel(float *hdr, DpHeader h, uint32_t local) {
    const uint32_t i = threadIdx.x;
    if (i < local * 4) hdr[i] = (i & 3u) < 3u ? h.pos[i >> 2][i & 3u] : 0.0f;
}

__global__ void write_grid_index_kernel(float *slots, uint32_t stride, DpGridIndex idx, uint32_t local) {
    const uint32_t i = threadIdx.x;
    if (i < local) slots[(size_t)i * stride] = __uint_as_float(idx.view[i]);
}

// Folds one local view's gradients into the exchange buffers: small row (+)= (v_transforms, v_raw_opac, visible), the stat
// row keeps the running MAX of the refine weight / radius (stats.rs:40-50 over the rank's views), the record row gets the
// view's colour gradient.  The first view assigns, the others accumulate.
// DEPTH: the view also carries the depth term's v_z (bg_rasterize_backward_depth, indexed by compact id); its mean
// gradient v_z * R[2,:] is folded into the row's v_transforms[0:3] before the sum, with the rounding and the skip rules of
// depth_to_means_kernel (project_bwd.cu: multiply, then add; a culled Gaussian or a zero v_z leaves the bits alone), so
// the row equals depth_to_means followed by the plain pack bit for bit -- without a read-modify-write pass over v_t.
template <bool DEPTH>
__global__ void __launch_bounds__(256)
pack_view_kernel(uint32_t n, uint32_t rec_row, uint32_t li, int first, const float *__restrict__ v_t, const float *__restrict__ v_o,
                 const float *__restrict__ v_color, const float *__restrict__ v_refine, const float *__restrict__ visible,
                 const float *__restrict__ max_radius, float *__restrict__ small, float *__restrict__ stat, float *__restrict__ record,
                 const uint32_t *__restrict__ cgid_from_gid, const float *__restrict__ v_z, float r0, float r1, float r2) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float row[DP_SMALL_ROW];
    const float2 *t2 = reinterpret_cast<const float2 *>(v_t + (size_t)i * 10);
#pragma unroll
    for (int q = 0; q < 5; q++) { const float2 a = __ldg(t2 + q); row[2 * q] = a.x; row[2 * q + 1] = a.y; }
    if constexpr (DEPTH) {
        const uint32_t cg = __ldg(cgid_from_gid + i);
        const float vz = cg != 0xFFFFFFFFu ? __ldg(v_z + cg) : 0.0f;
        if (vz != 0.0f) {
            row[0] = __fadd_rn(row[0], __fmul_rn(vz, r0));
            row[1] = __fadd_rn(row[1], __fmul_rn(vz, r1));
            row[2] = __fadd_rn(row[2], __fmul_rn(vz, r2));
        }
    }
    row[10] = __ldg(v_o + i);
    row[11] = __ldg(visible + i);
    float4 *dst = reinterpret_cast<float4 *>(small + (size_t)i * DP_SMALL_ROW);
    float2 *sd = reinterpret_cast<float2 *>(stat + (size_t)i * DP_STAT_ROW);
    float2 st = make_float2(__ldg(v_refine + i), __ldg(max_radius + i));
    if (!first) {
#pragma unroll
        for (int q = 0; q < 3; q++) { const float4 o = dst[q]; row[4 * q] += o.x; row[4 * q + 1] += o.y; row[4 * q + 2] += o.z; row[4 * q + 3] += o.w; }
        const float2 o = *sd;
        st.x = fmaxf(st.x, o.x); st.y = fmaxf(st.y, o.y);
    }
#pragma unroll
    for (int q = 0; q < 3; q++) dst[q] = make_float4(row[4 * q], row[4 * q + 1], row[4 * q + 2], row[4 * q + 3]);
    *sd = st;
    if (v_color) {
        float *rec = record + (size_t)i * rec_row + 3 * li;
        rec[0] = __ldg(v_color + (size_t)i * 3); rec[1] = __ldg(v_color + (size_t)i * 3 + 1); rec[2] = __ldg(v_color + (size_t)i * 3 + 2);
    }
}

// The colour record of one view straight from the rasterizer's gradient rows (what project_bwd_kernel's factored mode
// writes as v_color: lanes 5..7 of the visible Gaussian's row, zero for culled ones and for all-zero rows).  It depends on
// the blend backward only, so the all-gather can start while the projection backward still runs.
__global__ void __launch_bounds__(256)
pack_color_kernel(uint32_t n, uint32_t rec_row, uint32_t li, const uint32_t *__restrict__ cgid_from_gid, const float *__restrict__ v_combined,
                  float *__restrict__ record) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t cg = __ldg(cgid_from_gid + i);
    float r = 0.0f, g = 0.0f, b = 0.0f;
    if (cg != 0xFFFFFFFFu) {
        const float2 *p = reinterpret_cast<const float2 *>(v_combined + (size_t)cg * BG_VCOMBINED_STRIDE);
        float2 t[5];
        bool any = false;
#pragma unroll
        for (int q = 0; q < 5; q++) { t[q] = __ldg(p + q); any = any || t[q].x != 0.0f || t[q].y != 0.0f; }
        if (any) { r = t[2].y; g = t[3].x; b = t[3].y; }
    }
    float *rec = record + (size_t)i * rec_row + 3 * li;
    rec[0] = r; rec[1] = g; rec[2] = b;
}

cudaError_t launch_pack_color(cudaStream_t s, uint32_t n, uint32_t local, uint32_t li, const uint32_t *cgid_from_gid,
                              const float *v_combined, float *record) {
    if (n == 0) return cudaSuccess;
    pack_color_kernel<<<(n + 255) / 256, 256, 0, s>>>(n, 3 * local, li, cgid_from_gid, v_combined, record);
    return cudaGetLastError();
}

cudaError_t launch_write_header(cudaStream_t s, float *hdr, const DpHeader &h, uint32_t local) {
    write_header_kernel<<<1, 64, 0, s>>>(hdr, h, local);
    return cudaGetLastError();
}
cudaError_t launch_write_grid_index(cudaStream_t s, float *slots, uint32_t stride, const DpGridIndex &idx, uint32_t local) {
    write_grid_index_kernel<<<1, DP_MAX_VIEWS, 0, s>>>(slots, stride, idx, local);
    return cudaGetLastError();
}
cudaError_t launch_pack_view(cudaStream_t s, uint32_t n, uint32_t local, uint32_t li, bool first, const float *v_t, const float *v_o,
                             const float *v_color, const float *v_refine, const float *visible, const float *max_radius, float *small,
                             float *stat, float *record) {
    if (n == 0) return cudaSuccess;
    pack_view_kernel<false><<<(n + 255) / 256, 256, 0, s>>>(n, 3 * local, li, first ? 1 : 0, v_t, v_o, v_color, v_refine, visible,
                                                            max_radius, small, stat, record, nullptr, nullptr, 0.0f, 0.0f, 0.0f);
    return cudaGetLastError();
}
cudaError_t launch_pack_view_depth(cudaStream_t s, uint32_t n, uint32_t local, uint32_t li, bool first, const float *v_t, const float *v_o,
                                   const float *v_refine, const float *visible, const float *max_radius, const uint32_t *cgid_from_gid,
                                   const float *v_z, const BgCamera &cam, float *small, float *stat, float *record) {
    if (n == 0) return cudaSuccess;
    pack_view_kernel<true><<<(n + 255) / 256, 256, 0, s>>>(n, 3 * local, li, first ? 1 : 0, v_t, v_o, nullptr, v_refine, visible,
                                                           max_radius, small, stat, record, cgid_from_gid, v_z, cam.viewmat[2],
                                                           cam.viewmat[5], cam.viewmat[8]);
    return cudaGetLastError();
}

}  // namespace bg
