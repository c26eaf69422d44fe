// bg_dp.cuh -- types shared by dp.cu (NCCL binding, exchange) and api.cu (the multi-view step).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bg {

constexpr int DP_MAX_CHUNKS = 16;
constexpr int DP_MAX_VIEWS = 16;

struct NcclUniqueId { char internal[128]; };

struct DpComm {
    void *comm = nullptr;          // ncclComm_t
    int device = 0, rank = 0, world = 1;
    cudaStream_t stream = nullptr;     // the exchange runs here, beside the caller's stream
    cudaEvent_t ev_ready = nullptr;    // caller's stream -> exchange stream: gradients of the step are complete
    cudaEvent_t ev_ready2 = nullptr;   // same, second hand-off of a step (the rows that follow the colour records)
    cudaEvent_t ev_chunk[DP_MAX_CHUNKS] = {};   // exchange stream -> caller's stream: slice c has arrived
};

struct DpHeader { float pos[DP_MAX_VIEWS][3]; };
// the global training-view index of each local view (its bilateral grid)
struct DpGridIndex { uint32_t view[DP_MAX_VIEWS]; };

// Exchange buffers (see dp.cu), interleaved per Gaussian so that a slice of the Gaussian range is ONE contiguous piece
// of each buffer:
//   small  [n][12]       v_transforms (10) | v_raw_opac | visible, summed over the rank's views       -> all-reduce SUM
//   stat   [n][2]        v_refine | max_radius, MAX over the rank's views (stats.rs:40-50)            -> all-reduce MAX
//   record [n][3 local]  v_color of each local view (3 each)                                          -> all-gather
//   recv   per slice (g0, len): [world][len][3 local] at float offset 3 local * world * g0
constexpr uint32_t DP_SMALL_ROW = 12, DP_STAT_ROW = 2;
struct DpLayout {
    uint32_t n, local, world, rec_row;
    size_t rec_floats, small_floats, stat_floats, recv_floats;
    __host__ __device__ size_t chunk_base(uint32_t g0) const { return (size_t)rec_row * world * g0; }
};
inline DpLayout dp_layout(uint32_t n, uint32_t local, uint32_t world) {
    DpLayout L;
    L.n = n; L.local = local; L.world = world;
    L.rec_row = 3 * local;
    L.rec_floats = (size_t)L.rec_row * n;
    L.small_floats = (size_t)DP_SMALL_ROW * n;
    L.stat_floats = (size_t)DP_STAT_ROW * n;
    L.recv_floats = L.rec_floats * world;
    return L;
}

const char *dp_nccl_error(int code);
int dp_unique_id(NcclUniqueId *out);
DpComm *dp_comm_create(int device, const NcclUniqueId &id, int rank, int world, int *nccl_rc);
void dp_comm_destroy(DpComm *c);
void dp_chunk_range(uint32_t n, uint32_t chunks, uint32_t c, uint32_t *g0, uint32_t *len);
int dp_exchange_chunk(DpComm *cm, uint32_t n, uint32_t local, uint32_t chunks, uint32_t c, float *small, float *stat,
                      const float *record, float *recv);
int dp_exchange_gather(DpComm *cm, uint32_t n, uint32_t local, const float *record, float *recv);
int dp_exchange_reduce(DpComm *cm, uint32_t n, float *small, float *stat);
int dp_exchange_header(DpComm *cm, uint32_t local, const float *hdr, float *hdr_all);
// The multi-view step's bilateral-grid slots: all-gather of `floats` per rank (each local view's grid gradient and its view
// index), ev_chunk[2] recorded behind it.
int dp_exchange_grids(DpComm *cm, size_t floats, const float *send, float *recv);
cudaError_t launch_write_header(cudaStream_t s, float *hdr, const DpHeader &h, uint32_t local);
// slots[i * stride] = the bits of idx.view[i], i < local
cudaError_t launch_write_grid_index(cudaStream_t s, float *slots, uint32_t stride, const DpGridIndex &idx, uint32_t local);
cudaError_t launch_pack_view(cudaStream_t s, uint32_t n, uint32_t local, uint32_t li, bool first, const float *v_t, const float *v_o,
                             const float *v_color, const float *v_refine, const float *visible, const float *max_radius, float *small,
                             float *stat, float *record);
// launch_pack_view with the depth term's mean gradient v_z * R[2,:] folded into v_transforms[0:3] (no colour record)
cudaError_t launch_pack_view_depth(cudaStream_t s, uint32_t n, uint32_t local, uint32_t li, bool first, const float *v_t, const float *v_o,
                                   const float *v_refine, const float *visible, const float *max_radius, const uint32_t *cgid_from_gid,
                                   const float *v_z, const BgCamera &cam, float *small, float *stat, float *record);
cudaError_t launch_pack_color(cudaStream_t s, uint32_t n, uint32_t local, uint32_t li, const uint32_t *cgid_from_gid,
                              const float *v_combined, float *record);

}  // namespace bg
