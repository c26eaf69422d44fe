// bg_adam.cuh -- the element arithmetic of one AdamScaled step (optim.cu's adam_kernel) and the bias-correction power,
// shared by the kernels that run Adam so that they round alike bit for bit.
#pragma once
#include <cuda_runtime.h>

namespace bg {

struct AdamConsts {
    float lr, beta1, beta2, eps, f1, f2, bc1, bc2;
    int first;
};

__device__ __forceinline__ float adam_update(float p, float g, float &m, float v, const AdamConsts &k, float step) {
    float m_hat = m / k.bc1;
    float v_hat = v / k.bc2;
    float upd = m_hat / (sqrtf(v_hat) + k.eps);
    return p - upd * step;
}

// one element of adam_kernel: m, v and p in place, g the gradient, step the element's learning rate
__device__ __forceinline__ void adam_element(float &p, float gg, float &m, float &v, const AdamConsts &k, float step) {
    float mm = k.first ? gg * k.f1 : m * k.beta1 + gg * k.f1;
    float gsq = gg * gg;
    float vv = k.first ? gsq * k.f2 : v * k.beta2 + gsq * k.f2;
    m = mm;
    v = vv;
    p = adam_update(p, gg, mm, vv, k, step);
}

// compiler-rt __powisf2, what Rust's f32::powi lowers to (adam_scaled.rs:135-142).  The same rounding on the host and on
// the device: every product is rounded on its own (no contraction can reach across it).
__host__ __device__ inline float powi_mul(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ inline float powi_f32(float a, int b) {
    const bool recip = b < 0;
    float r = 1.0f;
    while (true) {
        if (b & 1) r = powi_mul(r, a);
        b /= 2;
        if (b == 0) break;
        a = powi_mul(a, a);
    }
    return recip ? 1.0f / r : r;
}
// 1 - beta^t, the bias correction of Adam step t
__host__ __device__ inline float adam_bias_correction(float beta, int t) {
#ifdef __CUDA_ARCH__
    return __fsub_rn(1.0f, powi_f32(beta, t));
#else
    return 1.0f - powi_f32(beta, t);
#endif
}

}  // namespace bg
