// Exercises differentiable depth through the C++ host layer (include/brush_b200.hpp): render_depth +
// rasterize_bwd_depth + project_bwd_depth.
//   depth_check IN OUT   IN: u32 n k smooth, u32 length + camera line, transforms [n,10], sh [n,k,3], raw opacity [n],
//                        background [3], v_output [h,w,4], v_depth [h,w] (w, h from the camera line).
//                        OUT: image [h,w,4], depth [h,w], v_z [n], v_transforms [n,10], v_sh [n,k,3], v_raw_opac [n].
#include <cstdio>
#include <fstream>
#include <sstream>
#include <string>
#include <vector>

#include "brush_b200.hpp"

using namespace brush_b200;

template <typename T>
static std::vector<T> read_vec(std::ifstream &f, size_t n) {
    std::vector<T> v(n);
    f.read(reinterpret_cast<char *>(v.data()), n * sizeof(T));
    return v;
}
template <typename T>
static void write_dev(std::ofstream &o, const DeviceBuffer<T> &b, size_t n) {
    std::vector<T> v(n);
    b.download(v.data(), n);
    o.write(reinterpret_cast<const char *>(v.data()), n * sizeof(T));
}
static DeviceBuffer<float> to_dev(const std::vector<float> &v) {
    DeviceBuffer<float> b(v.size());
    b.upload(v.data(), v.size());
    return b;
}

int main(int argc, char **argv) {
    if (argc != 3) { std::fprintf(stderr, "usage: depth_check IN OUT\n"); return 2; }
    try {
        std::ifstream f(argv[1], std::ios::binary);
        uint32_t hdr[4];
        f.read(reinterpret_cast<char *>(hdr), sizeof(hdr));
        const uint32_t n = hdr[0], k = hdr[1], smooth = hdr[2], len = hdr[3];
        std::string line(len, ' ');
        f.read(&line[0], len);
        std::istringstream ss(line);
        Camera c;
        uint32_t model, w, h;
        ss >> c.position[0] >> c.position[1] >> c.position[2] >> c.rotation[0] >> c.rotation[1] >> c.rotation[2] >>
            c.rotation[3] >> c.fov_x >> c.fov_y >> c.center_uv[0] >> c.center_uv[1] >> model;
        c.model = (CameraModel)model;
        for (int j = 0; j < 8; j++) ss >> c.model_params[j];
        ss >> w >> h;
        auto tr = to_dev(read_vec<float>(f, (size_t)n * 10)), sh = to_dev(read_vec<float>(f, (size_t)n * k * 3));
        auto op = to_dev(read_vec<float>(f, n));
        auto bg = read_vec<float>(f, 3);
        auto v_out = to_dev(read_vec<float>(f, (size_t)w * h * 4)), v_d = to_dev(read_vec<float>(f, (size_t)w * h));
        Context ctx(0, n, w, h);
        const RasterPass pass = smooth ? RasterPass::BackwardSmoothCutoff : RasterPass::Backward;
        RenderOutput out = render_depth(ctx, nullptr, c, w, h, tr.data(), sh.data(), op.data(), n, k, SplatRenderMode::Default,
                                        bg.data(), pass);
        auto vc_vz = rasterize_bwd_depth(ctx, nullptr, out, v_out.data(), v_d.data(), bg.data(), smooth != 0);
        SplatGrads g = project_bwd_depth(ctx, nullptr, out, tr.data(), sh.data(), op.data(), vc_vz.first.data(),
                                         vc_vz.second.data());
        std::ofstream o(argv[2], std::ios::binary);
        write_dev(o, out.out_img_f32, (size_t)w * h * 4);
        write_dev(o, out.out_depth, (size_t)w * h);
        write_dev(o, vc_vz.second, n);
        write_dev(o, g.v_transforms, (size_t)n * 10);
        write_dev(o, g.v_coeffs, (size_t)n * k * 3);
        write_dev(o, g.v_raw_opac, n);
        return 0;
    } catch (const std::exception &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 1;
    }
}
