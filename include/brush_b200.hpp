// brush_b200.hpp -- C++ host layer over the C ABI (include/brush_b200.h): the shape of the reference's own
// operator interface for this path, for callers that are compiled code (the reference is Rust; no Rust toolchain
// exists in this image, so the compiled-language host side is C++17, header only).
//
//   Camera, fov_to_focal / focal_to_fov, world_to_local, make_uniforms
//                               <- brush-render/src/camera.rs:11-254, render.rs:70-99 (ProjectUniforms)
//   Context                     <- one per logical task, like burn's per-thread stream (brush-async/src/lib.rs:1-17)
//   render                      <- SplatOps::render            brush-render/src/lib.rs:54-77, render.rs:37-315
//   rasterize_bwd / project_bwd <- SplatBwdOps                 brush-render/src/bwd/burn_glue.rs:62-92
//   render_depth, rasterize_bwd_depth, project_bwd_depth
//                               <- differentiable per-pixel depth (DESIGN.md section 4.6; no reference operator)
//   radix_argsort / prefix_sum  <- brush-sort/src/lib.rs:16, brush-prefix-sum/src/lib.rs:11
//   image_loss_forward/backward <- LossOps                     brush-loss/src/lib.rs:718-733
//   AdamScaled                  <- brush-train/src/adam_scaled.rs:64-165
//   TrainConfig, SplatTrainer   <- brush-train/src/config.rs, train.rs:138-893: step (bg_train_step), step_views
//                                  (bg_train_step_views: several views per step, one or several devices), refine (bg_refine)
//   BoundingBox, bounds_from_pos <- brush-render/src/bounding_box.rs, brush-train/src/splat_init.rs:130-160
//   Splats                      <- brush-render/src/gaussian_splats.rs:57-74 (owns the three parameter tensors)
//   DpComm                      <- no reference counterpart (SURVEY.md 8e): one NCCL rank per context, behind the ABI
//   pup_scores, decimate_to_count <- LOD baking, brush-train/src/lod.rs:13-142 (bg_pup_*, bg_decimate_to_count)
//
// Errors: the reference panics on shape / device violations (render.rs:50-64); here every non-zero ABI status
// becomes a brush_b200::Error (std::runtime_error) carrying the status and bg_last_error_string().
// Memory: outputs are freshly allocated by the callee (DeviceBuffer, cudaMalloc), inputs are borrowed device
// pointers -- the ownership convention of the reference's tensor handles (brush-cube/src/host.rs:31-57).
#pragma once
#include <cuda_runtime_api.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "brush_b200.h"

namespace brush_b200 {

struct Error : std::runtime_error {
    int32_t status;
    Error(int32_t s, const std::string &what) : std::runtime_error(what), status(s) {}
};
inline void check(int32_t status, const char *where) {
    if (status != BG_OK) {
        const char *d = bg_last_error_string();
        throw Error(status, std::string(where) + ": status " + std::to_string(status) + (d && *d ? std::string(" ") + d : ""));
    }
}
inline void check_cuda(cudaError_t e, const char *where) {
    if (e != cudaSuccess) throw Error(BG_ERR_CUDA, std::string(where) + ": " + cudaGetErrorString(e));
}

// ---------------------------------------------------------------------------------------------- camera
enum class CameraModel : uint32_t { Pinhole = 0, KannalaBrandt4 = 1, RadialTangential8 = 2, ThinPrismFisheye = 3 };

struct Camera {                      // camera.rs:11-19
    float position[3] = {0, 0, 0};
    float rotation[4] = {0, 0, 0, 1};     // glam quaternion (x, y, z, w), local -> world
    double fov_x = 0, fov_y = 0;          // radians
    float center_uv[2] = {0.5f, 0.5f};
    CameraModel model = CameraModel::Pinhole;
    float model_params[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // see BgCameraModel in brush_b200.h

    bool is_valid() const {
        bool ok = std::isfinite(fov_x) && std::isfinite(fov_y) && std::isfinite(center_uv[0]) && std::isfinite(center_uv[1]);
        for (float v : position) ok = ok && std::isfinite(v);
        for (float v : rotation) ok = ok && std::isfinite(v);
        return ok;
    }
};

namespace detail {
inline double kb4_d(double t, const float *k) {            // camera.rs:121-130
    double t2 = t * t, t3 = t2 * t, t5 = t3 * t2, t7 = t5 * t2, t9 = t7 * t2;
    return t + (double)k[0] * t3 + (double)k[1] * t5 + (double)k[2] * t7 + (double)k[3] * t9;
}
inline double kb4_dd(double t, const float *k) {
    double t2 = t * t, t4 = t2 * t2, t6 = t4 * t2, t8 = t6 * t2;
    return 1.0 + 3.0 * (double)k[0] * t2 + 5.0 * (double)k[1] * t4 + 7.0 * (double)k[2] * t6 + 9.0 * (double)k[3] * t8;
}
inline double kb4_invert_d(double target, const float *k) {   // camera.rs:146-169
    const double PI = 3.14159265358979323846;
    if (target <= 0.0) return 0.0;
    double theta = std::fmin(target, PI - 1e-6);
    for (int i = 0; i < 50; i++) {
        double f = kb4_d(theta, k) - target, fp = kb4_dd(theta, k);
        if (std::fabs(fp) < 1e-12) break;
        double next = std::fmin(std::fmax(theta - f / fp, 0.0), PI);
        if (std::fabs(next - theta) < 1e-12) { theta = next; break; }
        theta = next;
    }
    return theta;
}
inline double rt8_radial(double r, const float *p) {          // camera.rs:172-180
    double r2 = r * r, r4 = r2 * r2, r6 = r4 * r2;
    return (1.0 + (double)p[0] * r2 + (double)p[1] * r4 + (double)p[2] * r6) /
           (1.0 + (double)p[3] * r2 + (double)p[4] * r4 + (double)p[5] * r6);
}
inline double rt8_undistort_radius(double r_d, const float *p) {   // camera.rs:184-198
    double r = r_d;
    for (int i = 0; i < 30; i++) {
        double factor = rt8_radial(r, p);
        if (std::fabs(factor) < 1e-12) break;
        double r_new = r_d / factor;
        if (std::fabs(r_new - r) < 1e-12) { r = r_new; break; }
        r = r_new;
    }
    return r;
}
}  // namespace detail

inline double fov_to_focal(double fov, uint32_t pixels, CameraModel m = CameraModel::Pinhole, const float *params = nullptr) {
    static const float zeros[8] = {0};
    const float *p = params ? params : zeros;
    double half = fov / 2.0, projected;
    switch (m) {
        case CameraModel::Pinhole: projected = std::tan(half); break;
        case CameraModel::RadialTangential8: { double r = std::tan(half); projected = r * detail::rt8_radial(r, p); break; }
        default: projected = detail::kb4_d(half, p); break;     // KB4 and thin-prism fisheye share the radial polynomial
    }
    return ((double)pixels / 2.0) / projected;
}
inline double focal_to_fov(double focal, uint32_t pixels, CameraModel m = CameraModel::Pinhole, const float *params = nullptr) {
    static const float zeros[8] = {0};
    const float *p = params ? params : zeros;
    double r_norm = ((double)pixels / 2.0) / focal, half;
    switch (m) {
        case CameraModel::Pinhole: half = std::atan(r_norm); break;
        case CameraModel::RadialTangential8: half = std::atan(detail::rt8_undistort_radius(r_norm, p)); break;
        default: half = detail::kb4_invert_d(r_norm, p); break;
    }
    return 2.0 * half;
}

// camera.rs:75-81: Affine3A::from_rotation_translation(rotation, position).inverse(), top three rows, column major
// (columns c0 c1 c2, then the translation), in f32 like glam.
inline void world_to_local(const Camera &c, float out[12]) {
    const float x = c.rotation[0], y = c.rotation[1], z = c.rotation[2], w = c.rotation[3];
    const float x2 = x + x, y2 = y + y, z2 = z + z;
    const float xx = x * x2, xy = x * y2, xz = x * z2, yy = y * y2, yz = y * z2, zz = z * z2;
    const float wx = w * x2, wy = w * y2, wz = w * z2;
    const float xa[3] = {1.0f - (yy + zz), xy + wz, xz - wy};
    const float ya[3] = {xy - wz, 1.0f - (xx + zz), yz + wx};
    const float za[3] = {xz + wy, yz - wx, 1.0f - (xx + yy)};
    auto cross = [](const float *a, const float *b, float *r) {
        r[0] = a[1] * b[2] - a[2] * b[1]; r[1] = a[2] * b[0] - a[0] * b[2]; r[2] = a[0] * b[1] - a[1] * b[0];
    };
    float t0[3], t1[3], t2[3];
    cross(ya, za, t0); cross(za, xa, t1); cross(xa, ya, t2);
    const float det = za[0] * t2[0] + za[1] * t2[1] + za[2] * t2[2];
    const float inv_det = 1.0f / det;
    float m[3][3];   // m[i] = column i before the transpose
    for (int i = 0; i < 3; i++) { m[0][i] = t0[i] * inv_det; m[1][i] = t1[i] * inv_det; m[2][i] = t2[i] * inv_det; }
    float col[3][3];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) col[i][j] = m[j][i];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) out[3 * i + j] = col[i][j];
    for (int j = 0; j < 3; j++) {
        const float mt = col[0][j] * c.position[0] + col[1][j] * c.position[1] + col[2][j] * c.position[2];
        out[9 + j] = -mt;
    }
}

// render.rs:70-99 (ProjectUniforms) + calculate_jacobian_clamp_limits (camera.rs:200-254)
inline BgCamera make_uniforms(const Camera &c, uint32_t img_w, uint32_t img_h) {
    if (img_w == 0 || img_h == 0) throw Error(BG_ERR_INVALID, "Can't render images with 0 size.");
    BgCamera u;
    std::memset(&u, 0, sizeof(u));
    world_to_local(c, u.viewmat);
    const float *p = c.model_params;
    u.fx = (float)fov_to_focal(c.fov_x, img_w, c.model, p);
    u.fy = (float)fov_to_focal(c.fov_y, img_h, c.model, p);
    u.cx = c.center_uv[0] * (float)img_w;
    u.cy = c.center_uv[1] * (float)img_h;
    for (int i = 0; i < 3; i++) u.cam_pos[i] = c.position[i];
    const float wf = (float)img_w, hf = (float)img_h;
    float lpx = (1.15f * wf - u.cx) / u.fx, lpy = (1.15f * hf - u.cy) / u.fy;
    float lnx = (-0.15f * wf - u.cx) / u.fx, lny = (-0.15f * hf - u.cy) / u.fy;
    if (c.model == CameraModel::RadialTangential8) {
        auto und = [&](float e) {
            float r = (float)detail::rt8_undistort_radius(std::fabs((double)e), p);
            return r * (e > 0.0f ? 1.0f : (e < 0.0f ? -1.0f : 0.0f));
        };
        lpx = und(lpx); lpy = und(lpy); lnx = und(lnx); lny = und(lny);
    } else if (c.model != CameraModel::Pinhole) {
        lpx = lpy = lnx = lny = 0.0f;   // fisheye Jacobians are not clamped (camera.rs:244-247)
    }
    u.lim_pos_x = lpx; u.lim_pos_y = lpy; u.lim_neg_x = lnx; u.lim_neg_y = lny;
    const float hyp = (float)std::hypot((double)(float)c.fov_x, (double)(float)c.fov_y);
    const float two_pi_eps = 2.0f * 3.14159265358979323846f - 1e-6f;
    u.half_max_render_fov = std::fmin(hyp * 1.05f, two_pi_eps) * 0.5f;
    u.camera_model = (uint32_t)c.model;
    for (int i = 0; i < 8; i++) u.model_params[i] = p[i];
    return u;
}

// ---------------------------------------------------------------------------------------------- memory, context
template <typename T>
class DeviceBuffer {   // freshly allocated output, owned by the caller (like a returned tensor handle)
   public:
    DeviceBuffer() = default;
    explicit DeviceBuffer(size_t count, bool zero = false) : n_(count) {
        if (count) {
            check_cuda(cudaMalloc(&p_, count * sizeof(T)), "cudaMalloc");
            if (zero) check_cuda(cudaMemset(p_, 0, count * sizeof(T)), "cudaMemset");
        }
    }
    DeviceBuffer(const DeviceBuffer &) = delete;
    DeviceBuffer &operator=(const DeviceBuffer &) = delete;
    DeviceBuffer(DeviceBuffer &&o) noexcept : p_(o.p_), n_(o.n_) { o.p_ = nullptr; o.n_ = 0; }
    DeviceBuffer &operator=(DeviceBuffer &&o) noexcept {
        if (this != &o) { reset(); p_ = o.p_; n_ = o.n_; o.p_ = nullptr; o.n_ = 0; }
        return *this;
    }
    ~DeviceBuffer() { reset(); }
    void reset() { if (p_) cudaFree(p_); p_ = nullptr; n_ = 0; }
    T *data() { return static_cast<T *>(p_); }
    const T *data() const { return static_cast<const T *>(p_); }
    size_t size() const { return n_; }
    void upload(const T *host, size_t count, cudaStream_t s = nullptr) {
        check_cuda(cudaMemcpyAsync(p_, host, count * sizeof(T), cudaMemcpyHostToDevice, s), "upload");
    }
    void download(T *host, size_t count, cudaStream_t s = nullptr) const {
        check_cuda(cudaMemcpyAsync(host, p_, count * sizeof(T), cudaMemcpyDeviceToHost, s), "download");
        check_cuda(cudaStreamSynchronize(s), "download sync");
    }

   private:
    void *p_ = nullptr;
    size_t n_ = 0;
};

class Context {   // scratch arena; one per logical task (threading contract of brush-async)
   public:
    Context(int device, uint32_t max_splats, uint32_t max_w, uint32_t max_h, uint64_t max_intersections = 0) {
        check(bg_ctx_create(device, max_splats, max_w, max_h, max_intersections, &h_), "bg_ctx_create");
    }
    Context(const Context &) = delete;
    Context &operator=(const Context &) = delete;
    ~Context() { if (h_) bg_ctx_destroy(h_); }
    BgContext *handle() const { return h_; }
    uint64_t arena_bytes() const { return bg_ctx_arena_bytes(h_); }

   private:
    BgContext *h_ = nullptr;
};

// ---------------------------------------------------------------------------------------------- render
enum class SplatRenderMode { Default = 0, Mip = 1 };                                  // gaussian_splats.rs:12-25
enum class RasterPass { Forward = 0, Backward = 1, BackwardSmoothCutoff = 2 };        // gaussian_splats.rs:27-48

struct RenderOutput {                       // render_aux.rs:16-68
    DeviceBuffer<float> out_img_f32;        // [h,w,4] when pass != Forward
    DeviceBuffer<uint32_t> out_img_packed;  // [h,w] rgba8 when pass == Forward
    DeviceBuffer<float> visible, max_radius;   // [n]
    DeviceBuffer<float> out_depth;          // [h,w] accumulated depth sum_i vis_i z_i (render_depth only)
    BgRenderState state{};                  // device pointers into the context arena, valid until the next render
    BgCamera uniforms{};
    uint32_t w = 0, h = 0;
    // the reference awaits a readback inside render (render.rs:146-168); here the counts are read on demand
    uint32_t num_visible(cudaStream_t s = nullptr) const { sync(s); return state.counters_host[0]; }
    uint32_t num_intersections(cudaStream_t s = nullptr) const { sync(s); return state.counters_host[1]; }
    bool intersection_overflow(cudaStream_t s = nullptr) const { sync(s); return state.counters_host[2] != 0; }

   private:
    static void sync(cudaStream_t s) { check_cuda(cudaStreamSynchronize(s), "counter readback"); }
};

inline RenderOutput render(Context &ctx, cudaStream_t stream, const Camera &camera, uint32_t img_w, uint32_t img_h,
                           const float *transforms, const float *sh_coeffs, const float *raw_opacities, uint32_t n, uint32_t k,
                           SplatRenderMode mode, const float background[3], RasterPass pass) {
    RenderOutput out;
    out.w = img_w; out.h = img_h;
    out.uniforms = make_uniforms(camera, img_w, img_h);
    const bool bwd = pass != RasterPass::Forward;
    void *img = nullptr;
    if (bwd) { out.out_img_f32 = DeviceBuffer<float>((size_t)img_w * img_h * 4); img = out.out_img_f32.data(); }
    else { out.out_img_packed = DeviceBuffer<uint32_t>((size_t)img_w * img_h); img = out.out_img_packed.data(); }
    out.visible = DeviceBuffer<float>(n);
    out.max_radius = DeviceBuffer<float>(n);
    check(bg_render_forward(ctx.handle(), stream, &out.uniforms, img_w, img_h, n, k, transforms, sh_coeffs, raw_opacities,
                            mode == SplatRenderMode::Mip, background, (int32_t)pass, img, out.visible.data(),
                            out.max_radius.data(), &out.state),
          "SplatOps::render");
    return out;
}

// SplatBwdOps::rasterize_bwd: v_combined [n,10] (zero-filled by the callee, like float_zeros in render_bwd.rs:49-55)
inline DeviceBuffer<float> rasterize_bwd(Context &ctx, cudaStream_t stream, const RenderOutput &out, const float *v_output,
                                         const float background[3], bool smooth_cutoff) {
    DeviceBuffer<float> v_combined((size_t)out.state.n * BG_VCOMBINED_STRIDE);
    check(bg_rasterize_backward(ctx.handle(), stream, &out.state, out.out_img_f32.data(), v_output, background,
                                smooth_cutoff, v_combined.data(), out.state.n),
          "SplatBwdOps::rasterize_bwd");
    return v_combined;
}

struct SplatGrads { DeviceBuffer<float> v_transforms, v_coeffs, v_raw_opac, v_refine_weight; };   // bwd/burn_glue.rs:49-60

inline SplatGrads project_bwd(Context &ctx, cudaStream_t stream, const RenderOutput &out, const float *transforms,
                              const float *sh_coeffs, const float *raw_opacities, const float *v_combined) {
    const size_t n = out.state.n, k = out.state.k;
    SplatGrads g{DeviceBuffer<float>(n * 10), DeviceBuffer<float>(n * k * 3), DeviceBuffer<float>(n), DeviceBuffer<float>(n)};
    check(bg_project_backward(ctx.handle(), stream, &out.uniforms, &out.state, transforms, sh_coeffs, raw_opacities, v_combined,
                              g.v_transforms.data(), g.v_coeffs.data(), g.v_raw_opac.data(), g.v_refine_weight.data()),
          "SplatBwdOps::project_bwd");
    return g;
}

// render with the accumulated depth out_depth [h,w] (bg_render_forward_depth): pass Backward or BackwardSmoothCutoff.
// The expected depth is out_depth / alpha (out_img_f32[..., 3]).
inline RenderOutput render_depth(Context &ctx, cudaStream_t stream, const Camera &camera, uint32_t img_w, uint32_t img_h,
                                 const float *transforms, const float *sh_coeffs, const float *raw_opacities, uint32_t n,
                                 uint32_t k, SplatRenderMode mode, const float background[3], RasterPass pass) {
    RenderOutput out;
    out.w = img_w; out.h = img_h;
    out.uniforms = make_uniforms(camera, img_w, img_h);
    out.out_img_f32 = DeviceBuffer<float>((size_t)img_w * img_h * 4);
    out.out_depth = DeviceBuffer<float>((size_t)img_w * img_h);
    out.visible = DeviceBuffer<float>(n);
    out.max_radius = DeviceBuffer<float>(n);
    check(bg_render_forward_depth(ctx.handle(), stream, &out.uniforms, img_w, img_h, n, k, transforms, sh_coeffs,
                                  raw_opacities, mode == SplatRenderMode::Mip, background, (int32_t)pass,
                                  out.out_img_f32.data(), out.out_depth.data(), out.visible.data(), out.max_radius.data(),
                                  &out.state),
          "render_depth");
    return out;
}

// adjoint of render_depth with the upstream gradients v_output [h,w,4] and v_depth [h,w]:
// returns {v_combined [n,10], v_z [n]} (compact-id order, zero-filled by the callee)
inline std::pair<DeviceBuffer<float>, DeviceBuffer<float>> rasterize_bwd_depth(Context &ctx, cudaStream_t stream,
                                                                               const RenderOutput &out, const float *v_output,
                                                                               const float *v_depth, const float background[3],
                                                                               bool smooth_cutoff) {
    DeviceBuffer<float> v_combined((size_t)out.state.n * BG_VCOMBINED_STRIDE), v_z(out.state.n);
    check(bg_rasterize_backward_depth(ctx.handle(), stream, &out.state, out.out_img_f32.data(), out.out_depth.data(), v_output,
                                      v_depth, background, smooth_cutoff, v_combined.data(), out.state.n, v_z.data()),
          "rasterize_bwd_depth");
    return {std::move(v_combined), std::move(v_z)};
}

// project_bwd plus the depth chain v_transforms[:, 0:3] += v_z * R[2,:]
inline SplatGrads project_bwd_depth(Context &ctx, cudaStream_t stream, const RenderOutput &out, const float *transforms,
                                    const float *sh_coeffs, const float *raw_opacities, const float *v_combined,
                                    const float *v_z) {
    const size_t n = out.state.n, k = out.state.k;
    SplatGrads g{DeviceBuffer<float>(n * 10), DeviceBuffer<float>(n * k * 3), DeviceBuffer<float>(n), DeviceBuffer<float>(n)};
    check(bg_project_backward_depth(ctx.handle(), stream, &out.uniforms, &out.state, transforms, sh_coeffs, raw_opacities,
                                    v_combined, v_z, g.v_transforms.data(), g.v_coeffs.data(), g.v_raw_opac.data(),
                                    g.v_refine_weight.data()),
          "project_bwd_depth");
    return g;
}

// ---------------------------------------------------------------------------------------------- sort / scan / loss
inline std::pair<DeviceBuffer<uint32_t>, DeviceBuffer<uint32_t>> radix_argsort(Context &ctx, cudaStream_t stream,
                                                                              const uint32_t *keys, const uint32_t *values,
                                                                              uint32_t n, uint32_t sorting_bits) {
    if (sorting_bits > 32) throw Error(BG_ERR_INVALID, "radix_argsort: sorting_bits must be <= 32");   // brush-sort/src/lib.rs:21
    DeviceBuffer<uint32_t> ko(n), vo(n);
    check(bg_radix_argsort_u32(ctx.handle(), stream, keys, values, n, nullptr, sorting_bits, ko.data(), vo.data()), "radix_argsort");
    return {std::move(ko), std::move(vo)};
}
inline DeviceBuffer<uint32_t> prefix_sum(Context &ctx, cudaStream_t stream, const uint32_t *input, uint32_t n) {
    DeviceBuffer<uint32_t> out(n);
    check(bg_inclusive_scan_u32(ctx.handle(), stream, input, n, out.data()), "prefix_sum");
    return out;
}

struct ImageLossConfig {                     // brush-loss/src/lib.rs:698-712
    float l1_weight = 1.0f, ssim_weight = 0.0f;
    bool has_composite_bg = false;
    float composite_bg[3] = {0, 0, 0};
    bool mask = false;
};
// pred: [h,w,pred_channels] f32 (the render output, consumed in place); returns the loss map [channels,h,w]
inline DeviceBuffer<float> image_loss_forward(Context &ctx, cudaStream_t stream, const float *pred_hwc, uint32_t pred_channels,
                                              const uint32_t *gt_packed, uint32_t channels, uint32_t h, uint32_t w,
                                              const ImageLossConfig &cfg) {
    DeviceBuffer<float> map((size_t)channels * h * w);
    check(bg_image_loss_forward(ctx.handle(), stream, pred_hwc, gt_packed, channels, h, w, 1, (int64_t)w * pred_channels,
                                pred_channels, cfg.l1_weight, cfg.ssim_weight, cfg.has_composite_bg ? cfg.composite_bg : nullptr,
                                cfg.mask, map.data()),
          "LossOps::image_loss_forward");
    return map;
}
inline DeviceBuffer<float> image_loss_backward(Context &ctx, cudaStream_t stream, const float *pred_hwc, uint32_t pred_channels,
                                               const uint32_t *gt_packed, const float *dl_dmap, uint32_t channels, uint32_t h,
                                               uint32_t w, const ImageLossConfig &cfg) {
    DeviceBuffer<float> g((size_t)h * w * pred_channels, /*zero=*/true);
    check(bg_image_loss_backward(ctx.handle(), stream, pred_hwc, gt_packed, dl_dmap, channels, h, w, 1, (int64_t)w * pred_channels,
                                 pred_channels, cfg.l1_weight, cfg.ssim_weight, cfg.has_composite_bg ? cfg.composite_bg : nullptr,
                                 cfg.mask, g.data()),
          "LossOps::image_loss_backward");
    return g;
}

// ---------------------------------------------------------------------------------------------- optimiser
class AdamScaled {                           // adam_scaled.rs:64-165: one instance per parameter tensor
   public:
    AdamScaled(size_t rows, uint32_t cols, bool reduce_moment_2, float beta1 = 0.9f, float beta2 = 0.999f, float eps = 1e-15f)
        : rows_(rows), cols_(cols), reduce_(reduce_moment_2), b1_(beta1), b2_(beta2), eps_(eps),
          m_(rows * cols, true), v_(reduce_moment_2 ? rows : rows * cols, true) {}
    // p -= lr * scale (.) m_hat / (sqrt(v_hat) + eps); lr_scale_per_col: device [cols] or null
    void step(Context &ctx, cudaStream_t stream, float *param, const float *grad, float lr, const float *lr_scale_per_col = nullptr) {
        t_ += 1;
        check(bg_adam_step(ctx.handle(), stream, param, grad, m_.data(), v_.data(), rows_, cols_, lr_scale_per_col, lr, b1_, b2_,
                           eps_, t_, reduce_),
              "AdamScaled::step");
    }
    int steps() const { return t_; }

   private:
    size_t rows_;
    uint32_t cols_;
    bool reduce_;
    float b1_, b2_, eps_;
    int t_ = 0;
    DeviceBuffer<float> m_, v_;
};

// ---------------------------------------------------------------------------------------------- train step
struct TrainConfig {                         // brush-train/src/config.rs:5-132 (the fields the step uses, same defaults)
    uint32_t total_train_iters = 30000;
    double lr_mean = 2e-5, lr_mean_end = 2e-7;
    float mean_noise_weight = 50.0f;
    float lr_coeffs_dc = 2e-3f, lr_coeffs_sh_scale = 10.0f, lr_opac = 0.012f, lr_scale = 5e-3f, lr_rotation = 2e-3f;
    float ssim_weight = 0.2f, match_alpha_weight = 0.1f;
    float background[3] = {0, 0, 0};
    bool render_mip = false;
    uint64_t seed = 0;
    // refine (config.rs:47-92)
    float opac_decay = 0.004f;
    uint32_t max_splats = 10000000;
    uint32_t refine_every = 200;
    float growth_grad_threshold = 0.0025f, growth_select_fraction = 0.25f;
    uint32_t growth_stop_iter = 15000;
    float split_at_screen_size = 0.5f;
    // depth supervision (DESIGN.md section 4.7): weight of the L1 term on the expected depth; 0 = the plain step
    float depth_loss_weight = 0.0f;
};

// brush-render/src/bounding_box.rs:5-31
struct BoundingBox {
    float center[3] = {0, 0, 0};
    float extent[3] = {1, 1, 1};
    float median_size() const {   // bounding_box.rs:23-29: twice the middle extent, ordered by f32::total_cmp (NaN-safe)
        auto key = [](float f) {  // the total order of IEEE 754 (what total_cmp implements): sign-magnitude bits -> two's complement
            int32_t b;
            std::memcpy(&b, &f, 4);
            return b ^ (int32_t)((uint32_t)(b >> 31) >> 1);
        };
        float e[3] = {extent[0], extent[1], extent[2]};
        if (key(e[0]) > key(e[1])) std::swap(e[0], e[1]);
        if (key(e[1]) > key(e[2])) std::swap(e[1], e[2]);
        if (key(e[0]) > key(e[1])) std::swap(e[0], e[1]);
        return e[1] * 2.0f;
    }
    float max_extent() const { return std::fmax(extent[0], std::fmax(extent[1], extent[2])); }
};

// bounds_from_pos (splat_init.rs:130-160) on the device: per axis the ((1-p)/2, (1+p)/2) order statistics of the finite
// means.  No finite mean at all -> the unit box at the origin (splat_init.rs:141-143).  Synchronises `stream`.
inline BoundingBox bounds_from_pos(Context &ctx, cudaStream_t stream, float percentile, const float *transforms, uint32_t n) {
    BoundingBox b;
    if (n == 0) return b;
    const uint64_t need = bg_refine_workspace_bytes(n);
    DeviceBuffer<unsigned char> ws(need);
    float mm[6];
    check(bg_bounds_percentile(ctx.handle(), stream, n, transforms, percentile, ws.data(), need, mm), "bounds_from_pos");
    for (float v : mm)
        if (!std::isfinite(v)) return b;
    for (int a = 0; a < 3; a++) {
        b.center[a] = (mm[2 * a + 1] + mm[2 * a]) / 2.0f;
        b.extent[a] = (mm[2 * a + 1] - mm[2 * a]) / 2.0f;
    }
    return b;
}

// Splats (gaussian_splats.rs:57-74): owns the parameter tensors; refine replaces them (the count changes).
struct Splats {
    DeviceBuffer<float> transforms;      // [rows >= n, 10]  means 3, quaternion wxyz 4, log-scales 3
    DeviceBuffer<float> sh_coeffs;       // [rows >= n, k, 3]
    DeviceBuffer<float> raw_opacities;   // [rows >= n]
    uint32_t n = 0, k = 1;
    Splats() = default;
    Splats(const float *host_transforms, const float *host_sh, const float *host_raw_opac, uint32_t n_, uint32_t k_, cudaStream_t s = nullptr)
        : transforms((size_t)n_ * 10), sh_coeffs((size_t)n_ * k_ * 3), raw_opacities(n_), n(n_), k(k_) {
        transforms.upload(host_transforms, (size_t)n_ * 10, s);
        sh_coeffs.upload(host_sh, (size_t)n_ * k_ * 3, s);
        raw_opacities.upload(host_raw_opac, n_, s);
    }
    uint32_t num_splats() const { return n; }
};

struct RefineStats {   // brush-train/src/msg.rs RefineStats
    uint32_t num_added = 0, num_split_oversized = 0, num_split_high_grad = 0, num_pruned = 0, num_pruned_non_finite = 0, total_splats = 0;
};

// One NCCL rank bound to a context's device (bg_dp_comm_create).  Rank 0 obtains the 128-byte id with unique_id() and
// ships it to the other ranks over the host's own rendezvous; construction is collective.
class DpComm {
   public:
    static std::vector<uint8_t> unique_id() {
        std::vector<uint8_t> id(128);
        check(bg_dp_unique_id(id.data()), "bg_dp_unique_id");
        return id;
    }
    DpComm(Context &ctx, const std::vector<uint8_t> &id, int rank, int world) : rank_(rank), world_(world) {
        if (id.size() != 128) throw Error(BG_ERR_INVALID, "DpComm: the NCCL id is 128 bytes");
        check(bg_dp_comm_create(ctx.handle(), id.data(), rank, world, &h_), "bg_dp_comm_create");
    }
    DpComm(const DpComm &) = delete;
    DpComm &operator=(const DpComm &) = delete;
    ~DpComm() { if (h_) bg_dp_comm_destroy(h_); }
    BgDpComm *handle() const { return h_; }
    int rank() const { return rank_; }
    int world() const { return world_; }

   private:
    BgDpComm *h_ = nullptr;
    int rank_ = 0, world_ = 1;
};

constexpr float BOUND_PERCENTILE = 0.8f;   // train.rs:30: the bounds that drive the learning-rate scale and the prune radius

// SplatTrainer::step (train.rs:176-429) over bg_train_step.  Owns the Adam moments, the refine record and the step's
// workspace; the splat parameters stay with the caller and are updated in place.
class SplatTrainer {
   public:
    SplatTrainer(const TrainConfig &cfg, uint32_t n, uint32_t k, float median_scale)
        : cfg_(cfg), n_(n), k_(k), median_scale_(median_scale),
          m_t_((size_t)n * 10, true), v_t_((size_t)n * 10, true), m_sh_((size_t)n * k * 3, true), v_sh_(n, true), m_o_(n, true),
          v_o_(n, true), refine_norm_(n, true), vis_weight_(n, true), max_screen_(n, true), loss_(1, true) {
        decay_ = std::pow(cfg.lr_mean_end / cfg.lr_mean, 1.0 / (double)cfg.total_train_iters);
    }
    // SplatTrainer::new (train.rs:138-166) with the scene bounds: needed by refine (prune radius) and kept current by it
    SplatTrainer(const TrainConfig &cfg, uint32_t n, uint32_t k, const BoundingBox &bounds) : SplatTrainer(cfg, n, k, bounds.median_size()) {
        bounds_ = bounds;
        has_bounds_ = true;
    }
    // gt_packed: device [h,w] rgba8 (view_to_packed_data, scene.rs:97-136).  Returns the device scalar holding the loss.
    const float *step(Context &ctx, cudaStream_t stream, const Camera &camera, const uint32_t *gt_packed, uint32_t w, uint32_t h,
                      float *transforms, float *sh_coeffs, float *raw_opacities, bool has_alpha = false, bool masked_alpha = false) {
        BgTrainStepArgs a = step_args(camera, gt_packed, w, h, transforms, sh_coeffs, raw_opacities, has_alpha, masked_alpha,
                                      bg_train_step_workspace_bytes(n_, k_, w, h));
        check(bg_train_step(ctx.handle(), stream, &a), "SplatTrainer::step");
        last_state_ = a.state_out;
        return loss_.data();
    }
    // The step with depth supervision (bg_train_step_depth, DESIGN.md section 4.7): depth_target is the view's device [h,w]
    // metric camera-space z (0 = no measurement), depth_valid_count its number of valid pixels.  With
    // cfg.depth_loss_weight == 0 or no valid pixel this is the plain step.  Returns the device scalars
    // (loss = image loss + depth loss, depth loss).
    struct StepLosses {
        const float *loss;
        const float *depth_loss;
    };
    StepLosses step(Context &ctx, cudaStream_t stream, const Camera &camera, const uint32_t *gt_packed, const float *depth_target,
                    uint32_t depth_valid_count, uint32_t w, uint32_t h, float *transforms, float *sh_coeffs, float *raw_opacities,
                    bool has_alpha = false, bool masked_alpha = false) {
        BgTrainStepArgs a = step_args(camera, gt_packed, w, h, transforms, sh_coeffs, raw_opacities, has_alpha, masked_alpha,
                                      bg_train_step_depth_workspace_bytes(n_, k_, w, h));
        BgDepthSupervision d;
        d.target = depth_target;
        d.weight = cfg_.depth_loss_weight;
        d.valid_count = depth_valid_count;
        d.depth_loss_out = depth_loss_.data();
        check(bg_train_step_depth(ctx.handle(), stream, &a, &d), "SplatTrainer::step (depth)");
        last_state_ = a.state_out;
        return {loss_.data(), depth_loss_.data()};
    }

   private:
    BgTrainStepArgs step_args(const Camera &camera, const uint32_t *gt_packed, uint32_t w, uint32_t h, float *transforms,
                              float *sh_coeffs, float *raw_opacities, bool has_alpha, bool masked_alpha, uint64_t need) {
        step_ += 1;
        if (ws_.size() < need) ws_ = DeviceBuffer<unsigned char>(need);
        BgTrainStepArgs a;
        std::memset(&a, 0, sizeof(a));
        a.cam = make_uniforms(camera, w, h);
        a.w = w; a.h = h; a.n = n_; a.k = k_;
        a.mip = cfg_.render_mip;
        for (int i = 0; i < 3; i++) { a.background[i] = cfg_.background[i]; a.composite_bg[i] = cfg_.background[i]; }
        a.transforms = transforms; a.sh = sh_coeffs; a.raw_opac = raw_opacities;
        a.m_t = m_t_.data(); a.v_t = v_t_.data(); a.m_sh = m_sh_.data(); a.v_sh = v_sh_.data(); a.m_o = m_o_.data(); a.v_o = v_o_.data();
        a.refine_norm = refine_norm_.data(); a.vis_weight = vis_weight_.data(); a.max_screen = max_screen_.data();
        a.gt_packed = gt_packed;
        const bool ssim = cfg_.ssim_weight > 0.0f;
        a.l1_weight = ssim ? 1.0f - cfg_.ssim_weight : 1.0f;
        a.ssim_weight = ssim ? -cfg_.ssim_weight : 0.0f;
        const bool bg_nonzero = cfg_.background[0] != 0.0f || cfg_.background[1] != 0.0f || cfg_.background[2] != 0.0f;
        a.has_composite_bg = has_alpha && bg_nonzero;
        a.mask = masked_alpha;
        a.channels = (has_alpha && !masked_alpha && cfg_.match_alpha_weight > 0.0f) ? 4 : 3;
        a.alpha_weight = cfg_.match_alpha_weight;
        const double lr_mean = cfg_.lr_mean * std::pow(decay_, (double)(step_ - 1)) * (double)median_scale_;   // train.rs:328-333
        a.lr_mean = (float)lr_mean;
        a.lr_rotation = cfg_.lr_rotation; a.lr_scale = cfg_.lr_scale;
        a.lr_coeffs_dc = cfg_.lr_coeffs_dc; a.lr_coeffs_sh_scale = cfg_.lr_coeffs_sh_scale; a.lr_opac = cfg_.lr_opac;
        a.noise_scale = (float)lr_mean * cfg_.mean_noise_weight;
        a.median_scale = median_scale_;
        a.seed = cfg_.seed;
        a.step = step_;
        a.workspace = ws_.data(); a.workspace_bytes = need;
        a.loss_out = loss_.data();
        return a;
    }

   public:
    // One optimizer step over several views (SURVEY.md 8e, BASELINE config [4]) through bg_train_step_views: the loss is the
    // mean of the per-view losses.  `comm` == nullptr: all views on this device.  With a communicator every rank passes ITS
    // views (the same count on every rank; global view index = rank * local + i) and all ranks end with bit-identical
    // parameters.  gt_packed[i]: device [h,w] rgba8 of view i.  min_scale: optional device [n] Mip-Splatting scale floor.
    const float *step_views(Context &ctx, DpComm *comm, cudaStream_t stream, const std::vector<Camera> &cameras,
                            const std::vector<const uint32_t *> &gt_packed, uint32_t w, uint32_t h, Splats &splats,
                            const float *min_scale = nullptr, bool has_alpha = false, bool masked_alpha = false) {
        const uint32_t local = (uint32_t)cameras.size(), world = comm ? (uint32_t)comm->world() : 1u;
        if (local == 0 || gt_packed.size() != cameras.size() || local * world > 16)
            throw Error(BG_ERR_INVALID, "SplatTrainer::step_views: 1..16 views per step in total, one image per camera");
        if (splats.n != n_ || splats.k != k_) throw Error(BG_ERR_INVALID, "SplatTrainer::step_views: splat count differs from the optimizer state");
        step_ += 1;
        const uint64_t need = bg_train_step_views_workspace_bytes(n_, k_, w, h, local, world);
        if (views_ws_.size() < need) views_ws_ = DeviceBuffer<unsigned char>(need);
        std::vector<BgCamera> cams(local);
        for (uint32_t i = 0; i < local; i++) cams[i] = make_uniforms(cameras[i], w, h);
        BgTrainViewsArgs a;
        std::memset(&a, 0, sizeof(a));
        a.w = w; a.h = h; a.n = n_; a.k = k_;
        a.mip = cfg_.render_mip;
        for (int i = 0; i < 3; i++) { a.background[i] = cfg_.background[i]; a.composite_bg[i] = cfg_.background[i]; }
        a.local_views = local;
        a.cams = cams.data();
        a.gt_packed = gt_packed.data();
        a.transforms = splats.transforms.data(); a.sh = splats.sh_coeffs.data(); a.raw_opac = splats.raw_opacities.data();
        a.m_t = m_t_.data(); a.v_t = v_t_.data(); a.m_sh = m_sh_.data(); a.v_sh = v_sh_.data(); a.m_o = m_o_.data(); a.v_o = v_o_.data();
        a.refine_norm = refine_norm_.data(); a.vis_weight = vis_weight_.data(); a.max_screen = max_screen_.data();
        a.min_scale = min_scale;
        const bool ssim = cfg_.ssim_weight > 0.0f;
        a.l1_weight = ssim ? 1.0f - cfg_.ssim_weight : 1.0f;
        a.ssim_weight = ssim ? -cfg_.ssim_weight : 0.0f;
        const bool bg_nonzero = cfg_.background[0] != 0.0f || cfg_.background[1] != 0.0f || cfg_.background[2] != 0.0f;
        a.has_composite_bg = has_alpha && bg_nonzero;
        a.mask = masked_alpha;
        a.channels = (has_alpha && !masked_alpha && cfg_.match_alpha_weight > 0.0f) ? 4 : 3;
        a.alpha_weight = cfg_.match_alpha_weight;
        const double lr_mean = cfg_.lr_mean * std::pow(decay_, (double)(step_ - 1)) * (double)median_scale_;   // train.rs:328-333
        a.lr_mean = (float)lr_mean;
        a.lr_rotation = cfg_.lr_rotation; a.lr_scale = cfg_.lr_scale;
        a.lr_coeffs_dc = cfg_.lr_coeffs_dc; a.lr_coeffs_sh_scale = cfg_.lr_coeffs_sh_scale; a.lr_opac = cfg_.lr_opac;
        a.noise_scale = (float)lr_mean * cfg_.mean_noise_weight;
        a.median_scale = median_scale_;
        a.seed = cfg_.seed;
        a.step = step_;
        a.chunks = 0;
        a.workspace = views_ws_.data(); a.workspace_bytes = need;
        a.loss_out = loss_.data();
        check(bg_train_step_views(ctx.handle(), comm ? comm->handle() : nullptr, stream, &a), "SplatTrainer::step_views");
        last_state_ = a.state_out;
        return loss_.data();
    }

    // SplatTrainer::refine + refine_splats + prune_points (train.rs:431-893) through bg_refine: every decision on the
    // device, one readback of the counts.  Replaces the tensors of `splats` and the optimizer state (the count changes),
    // restarts the refine record (train.rs:442-445) and recomputes the bounds (train.rs:634).  `iteration` selects the
    // random stream and the schedules (growth stop, opacity decay).  A scale floor, if the host keeps one, must be baked
    // into the splats before the call and recomputed after it (train.rs:432-437, 641-647).
    RefineStats refine(Context &ctx, cudaStream_t stream, uint32_t iteration, Splats &splats) {
        if (!has_bounds_) throw Error(BG_ERR_INVALID, "SplatTrainer::refine: construct the trainer with the scene's BoundingBox");
        if (step_ == 0) throw Error(BG_ERR_INVALID, "Can only refine after optimizer is initialized");   // train.rs:490-492
        if (splats.n != n_ || splats.k != k_) throw Error(BG_ERR_INVALID, "SplatTrainer::refine: splat count differs from the optimizer state");
        const uint32_t n0 = n_;
        const uint64_t cap64 = std::max<uint64_t>(n0, std::min<uint64_t>(2ull * n0, std::max<uint64_t>(n0, cfg_.max_splats)));
        const uint32_t cap = (uint32_t)cap64;
        DeviceBuffer<float> t_out((size_t)cap * 10), sh_out((size_t)cap * k_ * 3), o_out(cap);
        DeviceBuffer<float> m_t((size_t)cap * 10), v_t((size_t)cap * 10), m_sh((size_t)cap * k_ * 3), v_sh(cap), m_o(cap), v_o(cap);
        const uint64_t need = bg_refine_workspace_bytes(n0);
        DeviceBuffer<unsigned char> ws(need);
        BgRefineArgs a;
        std::memset(&a, 0, sizeof(a));
        a.n = n0; a.k = k_; a.capacity = cap;
        a.transforms = splats.transforms.data(); a.sh = splats.sh_coeffs.data(); a.raw_opac = splats.raw_opacities.data();
        a.m_t = m_t_.data(); a.v_t = v_t_.data(); a.m_sh = m_sh_.data(); a.v_sh = v_sh_.data(); a.m_o = m_o_.data(); a.v_o = v_o_.data();
        a.refine_norm = refine_norm_.data(); a.vis_weight = vis_weight_.data(); a.max_screen = max_screen_.data();
        a.transforms_out = t_out.data(); a.sh_out = sh_out.data(); a.raw_opac_out = o_out.data();
        a.m_t_out = m_t.data(); a.v_t_out = v_t.data(); a.m_sh_out = m_sh.data(); a.v_sh_out = v_sh.data(); a.m_o_out = m_o.data(); a.v_o_out = v_o.data();
        for (int i = 0; i < 3; i++) a.bounds_center[i] = bounds_.center[i];
        a.max_allowed = bounds_.max_extent() * 100.0f;                                   // train.rs:485
        a.split_at_screen_size = cfg_.split_at_screen_size;
        a.growth_grad_threshold = cfg_.growth_grad_threshold;
        a.growth_select_fraction = cfg_.growth_select_fraction;
        a.max_splats = cfg_.max_splats;
        a.growth_enabled = iteration < cfg_.growth_stop_iter;
        const float train_t = std::fmin(std::fmax((float)iteration / (float)cfg_.total_train_iters, 0.0f), 1.0f);   // train.rs:809-811, in f32
        a.opac_decay_minus = cfg_.opac_decay * (1.0f - train_t);
        a.seed = cfg_.seed;
        a.refine_index = iteration;
        a.workspace = ws.data(); a.workspace_bytes = need;
        BgRefineStats rs;
        check(bg_refine(ctx.handle(), stream, &a, &rs), "SplatTrainer::refine");   // synchronises the stream once
        const uint32_t n_new = rs.total_splats;
        splats.transforms = std::move(t_out); splats.sh_coeffs = std::move(sh_out); splats.raw_opacities = std::move(o_out);
        splats.n = n_new;
        m_t_ = std::move(m_t); v_t_ = std::move(v_t); m_sh_ = std::move(m_sh); v_sh_ = std::move(v_sh); m_o_ = std::move(m_o); v_o_ = std::move(v_o);
        refine_norm_ = DeviceBuffer<float>(n_new, true); vis_weight_ = DeviceBuffer<float>(n_new, true); max_screen_ = DeviceBuffer<float>(n_new, true);
        n_ = n_new;
        bounds_ = bounds_from_pos(ctx, stream, BOUND_PERCENTILE, splats.transforms.data(), n_new);
        median_scale_ = bounds_.median_size();
        RefineStats out;
        out.num_added = rs.num_added; out.num_split_oversized = rs.num_split_oversized; out.num_split_high_grad = rs.num_split_high_grad;
        out.num_pruned = rs.num_pruned; out.num_pruned_non_finite = rs.num_pruned_non_finite; out.total_splats = n_new;
        return out;
    }
    // train_stream.rs:318-326: refine after the step with 0-based index `iter`?
    bool should_refine(uint32_t iter) const {
        const double progress = std::fmin(std::fmax((double)iter / (double)std::max(cfg_.total_train_iters, 1u), 0.0), 1.0);
        return iter > 0 && iter % cfg_.refine_every == 0 && progress <= 0.95;
    }
    uint32_t num_splats() const { return n_; }
    const BoundingBox &bounds() const { return bounds_; }
    int steps() const { return step_; }
    const BgRenderState &last_render_state() const { return last_state_; }
    const float *refine_weight_norm() const { return refine_norm_.data(); }
    const float *vis_weight() const { return vis_weight_.data(); }
    const float *max_screen_size() const { return max_screen_.data(); }

   private:
    TrainConfig cfg_;
    uint32_t n_, k_;
    float median_scale_;
    double decay_ = 1.0;
    int step_ = 0;
    DeviceBuffer<float> m_t_, v_t_, m_sh_, v_sh_, m_o_, v_o_, refine_norm_, vis_weight_, max_screen_, loss_;
    DeviceBuffer<float> depth_loss_{1, true};
    DeviceBuffer<unsigned char> ws_, views_ws_;
    BgRenderState last_state_{};
    BoundingBox bounds_;
    bool has_bounds_ = false;
};

// ---------------------------------------------------------------------------------------------- LOD baking
// One training view of pup_scores: its camera and ground truth (device [h,w] rgba8, view_to_packed_data) at the normal
// load resolution.
struct PupView {
    Camera camera;
    const uint32_t *gt_packed = nullptr;
    uint32_t w = 0, h = 0;
};

// compute_pup_scores (lod.rs:78-142): per view render (zero background, hard cutoff) -> L1 gradient of the mean over
// [h,w,3] -> rasterize / factored projection backward -> [floor fold backward] -> bg_pup_accumulate, in view order; then
// bg_pup_log_det.  min_scale: optional device [n] Mip-Splatting floor, folded into the renders.  Returns device scores [n].
inline DeviceBuffer<float> pup_scores(Context &ctx, cudaStream_t stream, const Splats &splats, const std::vector<PupView> &views,
                                      const float *min_scale = nullptr, bool mip = false) {
    const uint32_t n = splats.n, k = splats.k;
    if (n == 0 || views.empty()) throw Error(BG_ERR_INVALID, "pup_scores: needs splats and at least one view");
    DeviceBuffer<float> fisher((size_t)21 * n), scores(n), r_t, r_o;
    const float *t = splats.transforms.data(), *o = splats.raw_opacities.data();
    if (min_scale) {
        r_t = DeviceBuffer<float>((size_t)n * 10); r_o = DeviceBuffer<float>(n);
        check(bg_fold_min_scale_forward(ctx.handle(), stream, n, t, o, min_scale, r_t.data(), r_o.data()), "pup_scores: fold");
        t = r_t.data(); o = r_o.data();
    }
    DeviceBuffer<float> v_t((size_t)n * 10), v_c((size_t)n * 3), v_o(n), v_r(n), v_comb((size_t)n * BG_VCOMBINED_STRIDE), vis(n), rad(n);
    const float zero_bg[3] = {0.0f, 0.0f, 0.0f};
    for (size_t vi = 0; vi < views.size(); vi++) {
        const PupView &v = views[vi];
        BgCamera cam = make_uniforms(v.camera, v.w, v.h);
        DeviceBuffer<float> img((size_t)v.w * v.h * 4), dl((size_t)v.w * v.h * 4, /*zero=*/true);
        DeviceBuffer<float> partials(bg_image_loss_num_partials(3, v.h, v.w));
        BgRenderState st;
        check(bg_render_forward(ctx.handle(), stream, &cam, v.w, v.h, n, k, t, splats.sh_coeffs.data(), o, mip, zero_bg,
                                BG_PASS_BACKWARD, img.data(), vis.data(), rad.data(), &st), "pup_scores: render");
        const float c = (float)(1.0 / (3.0 * (double)v.w * (double)v.h));   // image_loss(..).mean() over [h, w, 3]
        const float chain[3] = {c, c, c};
        check(bg_image_loss_fused(ctx.handle(), stream, img.data(), v.gt_packed, 3, v.h, v.w, 1, (int64_t)v.w * 4, 4, 1.0f, 0.0f,
                                  nullptr, 0, chain, dl.data(), partials.data()), "pup_scores: loss");
        check(bg_rasterize_backward(ctx.handle(), stream, &st, img.data(), dl.data(), zero_bg, 0, v_comb.data(), n),
              "pup_scores: rasterize_bwd");
        check(bg_project_backward_factored(ctx.handle(), stream, &cam, &st, t, splats.sh_coeffs.data(), o, v_comb.data(),
                                           v_t.data(), v_c.data(), v_o.data(), v_r.data()), "pup_scores: project_bwd");
        if (min_scale)
            check(bg_fold_min_scale_backward(ctx.handle(), stream, n, splats.transforms.data(), splats.raw_opacities.data(),
                                             min_scale, v_t.data(), v_o.data()), "pup_scores: fold backward");
        check(bg_pup_accumulate(ctx.handle(), stream, n, v_t.data(), vi == 0, fisher.data()), "pup_scores: accumulate");
        check_cuda(cudaStreamSynchronize(stream), "pup_scores");   // the view's buffers are freed at the end of the iteration
    }
    check(bg_pup_log_det(ctx.handle(), stream, n, fisher.data(), scores.data()), "pup_scores: log_det");
    return scores;
}

// decimate_to_count (lod.rs:13-40) through bg_decimate_to_count: keeps the `target` best scores (device [n]) in
// descending score order, ties in index order, NaN last.  Replaces the tensors of `splats`; target >= n leaves them as they
// are.  min_scale: optional [n] floor, replaced by its gathered [target] rows.  kept_ids: optional, receives the
// [target] source indices.
inline void decimate_to_count(Context &ctx, cudaStream_t stream, Splats &splats, const float *scores, uint32_t target,
                              DeviceBuffer<float> *min_scale = nullptr, DeviceBuffer<uint32_t> *kept_ids = nullptr) {
    const uint32_t n = splats.n, k = splats.k;
    if (target >= n) return;
    if (target == 0) throw Error(BG_ERR_INVALID, "decimate_to_count: target must be >= 1");
    const bool floor = min_scale && min_scale->size();
    DeviceBuffer<float> t_out((size_t)target * 10), sh_out((size_t)target * k * 3), o_out(target), f_out(floor ? target : 0);
    DeviceBuffer<uint32_t> ids(kept_ids ? target : 0);
    const uint64_t need = bg_decimate_workspace_bytes(n);
    DeviceBuffer<unsigned char> ws(need);
    BgDecimateArgs a;
    std::memset(&a, 0, sizeof(a));
    a.n = n; a.k = k; a.target = target;
    a.scores = scores;
    a.transforms = splats.transforms.data(); a.sh = splats.sh_coeffs.data(); a.raw_opac = splats.raw_opacities.data();
    a.min_scale = floor ? min_scale->data() : nullptr;
    a.transforms_out = t_out.data(); a.sh_out = sh_out.data(); a.raw_opac_out = o_out.data();
    a.min_scale_out = floor ? f_out.data() : nullptr;
    a.kept_ids_out = kept_ids ? ids.data() : nullptr;
    a.workspace = ws.data(); a.workspace_bytes = need;
    check(bg_decimate_to_count(ctx.handle(), stream, &a), "decimate_to_count");
    check_cuda(cudaStreamSynchronize(stream), "decimate_to_count");   // the workspace is freed on return
    splats.transforms = std::move(t_out); splats.sh_coeffs = std::move(sh_out); splats.raw_opacities = std::move(o_out);
    splats.n = target;
    if (floor) *min_scale = std::move(f_out);
    if (kept_ids) *kept_ids = std::move(ids);
}

}  // namespace brush_b200
