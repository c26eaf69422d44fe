// Exercises the depth-supervised training step of the C++ host layer (include/brush_b200.hpp: SplatTrainer::step with a
// depth target, over bg_train_step_depth).
//   depth_sup_check IN   IN: u32 n k w h steps valid_count, f32 depth_loss_weight median_scale, u32 length + camera line,
//                        transforms [n,10], sh [n,k,3], raw opacity [n], packed ground truth [h,w] u32, depth target [h,w].
//                        stdout: one "loss <loss> <depth loss>" line per step.
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

int main(int argc, char **argv) {
    if (argc != 2) { std::fprintf(stderr, "usage: depth_sup_check IN\n"); return 2; }
    try {
        std::ifstream f(argv[1], std::ios::binary);
        uint32_t hdr[6];
        float wts[2];
        f.read(reinterpret_cast<char *>(hdr), sizeof(hdr));
        f.read(reinterpret_cast<char *>(wts), sizeof(wts));
        const uint32_t n = hdr[0], k = hdr[1], w = hdr[2], h = hdr[3], steps = hdr[4], valid = hdr[5];
        uint32_t len;
        f.read(reinterpret_cast<char *>(&len), 4);
        std::string line(len, ' ');
        f.read(&line[0], len);
        std::istringstream ss(line);
        Camera c;
        uint32_t model, cw, ch;
        ss >> c.position[0] >> c.position[1] >> c.position[2] >> c.rotation[0] >> c.rotation[1] >> c.rotation[2] >>
            c.rotation[3] >> c.fov_x >> c.fov_y >> c.center_uv[0] >> c.center_uv[1] >> model;
        c.model = (CameraModel)model;
        for (int j = 0; j < 8; j++) ss >> c.model_params[j];
        ss >> cw >> ch;
        auto tr = read_vec<float>(f, (size_t)n * 10), sh = read_vec<float>(f, (size_t)n * k * 3), op = read_vec<float>(f, n);
        auto gt = read_vec<uint32_t>(f, (size_t)w * h);
        auto target = read_vec<float>(f, (size_t)w * h);
        Context ctx(0, n, w, h);
        DeviceBuffer<float> d_tr(tr.size()), d_sh(sh.size()), d_op(op.size()), d_t(target.size());
        DeviceBuffer<uint32_t> d_gt(gt.size());
        d_tr.upload(tr.data(), tr.size()); d_sh.upload(sh.data(), sh.size()); d_op.upload(op.data(), op.size());
        d_gt.upload(gt.data(), gt.size()); d_t.upload(target.data(), target.size());
        TrainConfig cfg;
        cfg.total_train_iters = 1000;
        cfg.seed = 7;
        cfg.depth_loss_weight = wts[0];
        SplatTrainer trainer(cfg, n, k, wts[1]);
        for (uint32_t i = 0; i < steps; i++) {
            const SplatTrainer::StepLosses l = trainer.step(ctx, nullptr, c, d_gt.data(), d_t.data(), valid, w, h, d_tr.data(),
                                                            d_sh.data(), d_op.data());
            float loss, depth_loss;
            check_cuda(cudaMemcpy(&loss, l.loss, 4, cudaMemcpyDeviceToHost), "loss readback");
            check_cuda(cudaMemcpy(&depth_loss, l.depth_loss, 4, cudaMemcpyDeviceToHost), "depth loss readback");
            std::printf("loss %.9g %.9g\n", loss, depth_loss);
        }
        return 0;
    } catch (const std::exception &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 1;
    }
}
