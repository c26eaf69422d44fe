// Exercises the multi-view training step with depth supervision of the C++ host layer (include/brush_b200.hpp:
// SplatTrainer::step_views with per-camera depth targets, over bg_train_step_views_depth), on one device.
//   views_depth_check IN OUT   IN: u32 n k w h steps views, f32 depth_loss_weight median_scale, transforms [n,10],
//                              sh [n,k,3], raw opacity [n], then per view: u32 length + camera line, u32 valid_count,
//                              packed ground truth [h,w] u32, and when valid_count > 0 the depth target [h,w] f32.
//                              stdout: one "loss <loss> <depth loss of view 0> ..." line per step.
//                              OUT: the parameters after the last step (transforms, sh, raw opacity, f32).
#include <cstdio>
#include <fstream>
#include <memory>
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

static Camera read_camera(std::ifstream &f) {
    uint32_t len;
    f.read(reinterpret_cast<char *>(&len), 4);
    std::string line(len, ' ');
    f.read(&line[0], len);
    std::istringstream ss(line);
    Camera c;
    uint32_t model, cw, ch;
    ss >> c.position[0] >> c.position[1] >> c.position[2] >> c.rotation[0] >> c.rotation[1] >> c.rotation[2] >> c.rotation[3] >>
        c.fov_x >> c.fov_y >> c.center_uv[0] >> c.center_uv[1] >> model;
    c.model = (CameraModel)model;
    for (int j = 0; j < 8; j++) ss >> c.model_params[j];
    ss >> cw >> ch;
    return c;
}

int main(int argc, char **argv) {
    if (argc != 3) { std::fprintf(stderr, "usage: views_depth_check IN OUT\n"); return 2; }
    try {
        std::ifstream f(argv[1], std::ios::binary);
        uint32_t hdr[6];
        float wts[2];
        f.read(reinterpret_cast<char *>(hdr), sizeof(hdr));
        f.read(reinterpret_cast<char *>(wts), sizeof(wts));
        const uint32_t n = hdr[0], k = hdr[1], w = hdr[2], h = hdr[3], steps = hdr[4], views = hdr[5];
        auto tr = read_vec<float>(f, (size_t)n * 10), sh = read_vec<float>(f, (size_t)n * k * 3), op = read_vec<float>(f, n);
        Context ctx(0, n, w, h);
        std::vector<Camera> cams;
        std::vector<std::unique_ptr<DeviceBuffer<uint32_t>>> gts;
        std::vector<std::unique_ptr<DeviceBuffer<float>>> targets;
        std::vector<const uint32_t *> gt_ptrs;
        std::vector<const float *> target_ptrs;
        std::vector<uint32_t> counts;
        for (uint32_t v = 0; v < views; v++) {
            cams.push_back(read_camera(f));
            uint32_t count;
            f.read(reinterpret_cast<char *>(&count), 4);
            auto gt = read_vec<uint32_t>(f, (size_t)w * h);
            gts.push_back(std::make_unique<DeviceBuffer<uint32_t>>(gt.size()));
            gts.back()->upload(gt.data(), gt.size());
            gt_ptrs.push_back(gts.back()->data());
            counts.push_back(count);
            if (count > 0) {
                auto t = read_vec<float>(f, (size_t)w * h);
                targets.push_back(std::make_unique<DeviceBuffer<float>>(t.size()));
                targets.back()->upload(t.data(), t.size());
                target_ptrs.push_back(targets.back()->data());
            } else {
                target_ptrs.push_back(nullptr);
            }
        }
        Splats splats(tr.data(), sh.data(), op.data(), n, k);
        TrainConfig cfg;
        cfg.total_train_iters = 1000;
        cfg.seed = 7;
        cfg.depth_loss_weight = wts[0];
        SplatTrainer trainer(cfg, n, k, wts[1]);
        for (uint32_t i = 0; i < steps; i++) {
            const SplatTrainer::ViewsLosses l = trainer.step_views(ctx, nullptr, nullptr, cams, gt_ptrs, target_ptrs, counts, w, h, splats);
            float loss;
            std::vector<float> dl(views);
            check_cuda(cudaMemcpy(&loss, l.loss, 4, cudaMemcpyDeviceToHost), "loss readback");
            check_cuda(cudaMemcpy(dl.data(), l.depth_losses, 4 * views, cudaMemcpyDeviceToHost), "depth loss readback");
            std::printf("loss %.9g", loss);
            for (float x : dl) std::printf(" %.9g", x);
            std::printf("\n");
        }
        std::ofstream o(argv[2], std::ios::binary);
        splats.transforms.download(tr.data(), tr.size());
        splats.sh_coeffs.download(sh.data(), sh.size());
        splats.raw_opacities.download(op.data(), op.size());
        o.write(reinterpret_cast<const char *>(tr.data()), tr.size() * 4);
        o.write(reinterpret_cast<const char *>(sh.data()), sh.size() * 4);
        o.write(reinterpret_cast<const char *>(op.data()), op.size() * 4);
        return 0;
    } catch (const std::exception &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 1;
    }
}
