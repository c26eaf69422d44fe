// bg_update.cuh -- argument block of train_update_kernel (update.cu), filled by api.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bg {

struct UpdateParams {
    uint32_t g_begin, count;         // this launch updates Gaussians [g_begin, g_begin + count)
    float *transforms, *sh, *raw_opac;
    float *m_t, *v_t, *m_sh, *v_sh, *m_o, *v_o;
    float *refine_norm, *vis_weight, *max_screen;
    const float *g_t, *g_o;          // dense: [n,10], [n].  Factored: unused (the gradients are rows of `small`)
    const float *g_sh;               // dense [n,K,3] gradient; unused when factored
    float grad_scale;                // applied to the transforms / opacity gradients (1/views)
    // factored form (multi-view steps, bg_dp.cuh): `small` [n][12] = v_transforms | v_raw_opac | visible summed over all
    // views; `stat` [n][2] = v_refine | max_radius, MAX over all views; `records` = the slice [g_begin, g_begin+count) of the
    // gathered colour gradients, [world][count][3 local]
    const float *small, *stat, *records;
    const float *cam_all;            // device [views][4]: camera positions in global view order
    uint32_t views, local, world;
    float sh_grad_scale;             // 1/views
    const float *v_refine, *max_radius;   // [n] statistics of the step when not factored
    const float *visible;            // [n] visibility of the step when not factored
    float lr_t[10];
    float lr_sh_dc, lr_sh_rest, lr_opac;
    float beta1, beta2, eps, f1, f2, inv_bc1, inv_bc2;   // 1 / (1 - beta^t), rounded once on the host
    int first;
    int noisy;
    float noise_scale, median_scale;
    unsigned long long seed, noise_offset;
    const float *min_scale;          // [n] 3D-filter floor or null: the noise gate uses the folded opacity (bg_fold.cuh)
};

cudaError_t launch_train_update(cudaStream_t s, int deg, const UpdateParams &P, bool factored, int part = 0);

}  // namespace bg
