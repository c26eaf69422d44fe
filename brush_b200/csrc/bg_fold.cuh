// bg_fold.cuh -- the terms of fold_min_scale (brush-render/src/gaussian_splats.rs:86-111), the Mip-Splatting 3D filter
// floor, shared by the fold kernels (optim.cu) and the noise gate of the update pass (update.cu), so that the folded
// opacity has one definition.
#pragma once
#include <cuda_runtime.h>

namespace bg {

// s2 = exp(2 ls), s2f = s2 + f^2, coef = sqrt(prod s2 / prod s2f), sig = sigmoid(raw),
// opac = clamp(sig * coef, 1e-6, 1 - 1e-6) (Splats::opacities with the floor folded in, gaussian_splats.rs:215-223)
struct FoldTerms { float s2[3], s2f[3], coef, sig, opac; bool in_range; };

__device__ __forceinline__ FoldTerms fold_terms(const float *ls, float raw, float f) {
    FoldTerms t;
    const float f2 = f * f;
    float det1 = 1.f, det2 = 1.f;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        t.s2[a] = expf(2.0f * ls[a]);
        t.s2f[a] = t.s2[a] + f2;
    }
    det1 = t.s2[0] * t.s2[1] * t.s2[2];
    det2 = t.s2f[0] * t.s2f[1] * t.s2f[2];
    t.coef = sqrtf(det1 / det2);
    t.sig = 1.0f / (1.0f + expf(-raw));
    const float o = t.sig * t.coef;
    t.in_range = o >= 1e-6f && o <= 1.0f - 1e-6f;
    t.opac = fminf(fmaxf(o, 1e-6f), 1.0f - 1e-6f);
    return t;
}

}  // namespace bg
