// bg_refine.cuh -- control block and pointer bundle shared by refine.cu (kernels) and api.cu (bg_refine).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bg {

// device control words of one refine (zeroed at its start, read back once at its end)
enum RefineCtlSlots : uint32_t {
    RC_NON_FINITE = 0,      // splats with a non-finite parameter
    RC_IDENTITY = 1,        // 1: nothing pruned (no splat, or every splat, matched the prune mask)
    RC_PRUNED = 2,
    RC_N = 3,               // splats after the prune
    RC_POS0 = 4,            // positive replacement weights
    RC_SPLIT_REPLACE = 5,   // splits that replace pruned splats
    RC_SPLIT_OVERSIZED = 6,
    RC_THRESHOLD_COUNT = 7,
    RC_POS1 = 8,            // positive growth weights
    RC_GROW = 9,            // growth samples requested
    RC_SPLIT_GROWTH = 10,   // new splits from the growth sample
    RC_REFINE_COUNT = 11,
    RC_N_NEW = 12,
    RC_OVERFLOW = 13,       // n_new exceeded the capacity of the destination arrays
    RC_WORDS = 16
};

struct RefinePtrs {
    const float *transforms, *sh, *raw_opac, *m_t, *v_t, *m_sh, *v_sh, *m_o, *v_o, *refine_norm, *vis_weight, *max_screen;
    float *transforms_out, *sh_out, *raw_opac_out, *m_t_out, *v_t_out, *m_sh_out, *v_sh_out, *m_o_out, *v_o_out;
    float *refine_norm_tmp, *vis_weight_tmp, *max_screen_tmp;
};

// The launchers of refine.cu, in the order bg_refine issues them.  n0: splats before the prune; n_max = n0 bounds every
// later pass, whose live count is ctl[RC_N] on the device.  kf = 3k floats per SH row.  ctl: the RC_* words above.
// keep / split / cand [n0]: 0/1 flags; *_incl: their inclusive scans.
// center: host [3]
cudaError_t launch_refine_classify(cudaStream_t s, uint32_t n0, uint32_t kf, const float *transforms, const float *sh,
                                   const float *raw_opac, const float *center, float max_allowed, uint32_t *keep, uint32_t *ctl);
cudaError_t launch_refine_plan_prune(cudaStream_t s, uint32_t n0, const uint32_t *keep_incl, uint32_t *ctl);
// the kept rows of every array of p -> its _out / _tmp arrays
cudaError_t launch_refine_compact(cudaStream_t s, uint32_t n0, uint32_t kf, const RefinePtrs &p, const uint32_t *keep,
                                  const uint32_t *keep_incl, const uint32_t *ctl);
// sampling keys for the radix sort, vals = index.  mode 0: replacement of the pruned splats, 1: growth above grad_threshold
cudaError_t launch_refine_keys(cudaStream_t s, uint32_t n_max, int mode, const RefinePtrs &p, float grad_threshold, uint64_t seed,
                               uint64_t stream_id, uint32_t *keys, uint32_t *vals, uint32_t *ctl);
cudaError_t launch_refine_plan_growth(cudaStream_t s, float fraction, uint32_t max_splats, bool enabled, uint32_t *ctl);
// marks in split the first min(ctl[k_slot], ctl[pos_slot]) of sorted_vals; counts the new marks in ctl[count_slot]
cudaError_t launch_refine_mark_topk(cudaStream_t s, uint32_t n_max, const uint32_t *sorted_vals, uint32_t k_slot, uint32_t pos_slot,
                                    uint32_t count_slot, uint32_t *split, uint32_t *ctl);
cudaError_t launch_refine_oversize_flags(cudaStream_t s, uint32_t n_max, float thr, const RefinePtrs &p, const uint32_t *split,
                                         uint32_t *cand, const uint32_t *ctl);
cudaError_t launch_refine_oversize_mark(cudaStream_t s, uint32_t n_max, uint32_t max_splats, const uint32_t *cand, const uint32_t *cand_incl,
                                        uint32_t *split, uint32_t *ctl);
cudaError_t launch_refine_plan_split(cudaStream_t s, uint32_t n_max, const uint32_t *split_incl, uint32_t capacity, uint32_t *ctl);
cudaError_t launch_refine_split(cudaStream_t s, uint32_t n_max, uint32_t kf, uint32_t capacity, float thr, const RefinePtrs &p,
                                const uint32_t *split, const uint32_t *split_incl, const uint32_t *ctl);
cudaError_t launch_refine_decay(cudaStream_t s, uint32_t cap, float minus_opac, float *raw_opac, const uint32_t *ctl);
// bg_bounds_percentile: keys = ordered bits of coordinate `axis` (non-finite ones last), *count += the finite ones;
// out2 = the lower and upper bound that hold the central `percentile` of the first *count sorted_keys
cudaError_t launch_bounds_keys(cudaStream_t s, uint32_t n, int axis, const float *transforms, uint32_t *keys, uint32_t *vals, uint32_t *count);
cudaError_t launch_bounds_pick(cudaStream_t s, const uint32_t *sorted_keys, const uint32_t *count, float percentile, float *out2);

}  // namespace bg
