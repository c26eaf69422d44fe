// Exercises the bilateral-grid training step of the C++ host layer (include/brush_b200.hpp: BilateralGrids and
// SplatTrainer::step with the grids, over bg_train_step_bilagrid).
//   bilagrid_check IN   IN: u32 n k w h steps views view, f32 median_scale, u32 length + camera line, transforms [n,10],
//                       sh [n,k,3], raw opacity [n], packed ground truth [h,w] u32.
//                       stdout: one "loss <loss> <tv loss>" line per step, then "steps <count of each view>".
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
    if (argc != 2) { std::fprintf(stderr, "usage: bilagrid_check IN\n"); return 2; }
    try {
        std::ifstream f(argv[1], std::ios::binary);
        uint32_t hdr[7];
        float median_scale;
        f.read(reinterpret_cast<char *>(hdr), sizeof(hdr));
        f.read(reinterpret_cast<char *>(&median_scale), sizeof(median_scale));
        const uint32_t n = hdr[0], k = hdr[1], w = hdr[2], h = hdr[3], steps = hdr[4], views = hdr[5], view = hdr[6];
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
        Context ctx(0, n, w, h);
        DeviceBuffer<float> d_tr(tr.size()), d_sh(sh.size()), d_op(op.size());
        DeviceBuffer<uint32_t> d_gt(gt.size());
        d_tr.upload(tr.data(), tr.size()); d_sh.upload(sh.data(), sh.size()); d_op.upload(op.data(), op.size());
        d_gt.upload(gt.data(), gt.size());
        TrainConfig cfg;
        cfg.total_train_iters = 1000;
        cfg.seed = 7;
        cfg.bilateral_grid = true;
        SplatTrainer trainer(cfg, n, k, median_scale);
        BilateralGrids grids(views);
        // the steps without grids refuse the configuration, and the multi-view step refuses grids
        int refused = 0;
        try { trainer.step(ctx, nullptr, c, d_gt.data(), w, h, d_tr.data(), d_sh.data(), d_op.data()); } catch (const Error &) { refused++; }
        Splats s;
        try { trainer.step_views(ctx, nullptr, nullptr, {c}, {d_gt.data()}, w, h, s, nullptr, false, false, &grids); } catch (const Error &) { refused++; }
        if (refused != 2 || trainer.steps() != 0) { std::fprintf(stderr, "grid refusals: %d\n", refused); return 1; }
        for (uint32_t i = 0; i < steps; i++) {
            const SplatTrainer::GridStepLosses l = trainer.step(ctx, nullptr, c, d_gt.data(), grids, view, nullptr, 0, w, h,
                                                                d_tr.data(), d_sh.data(), d_op.data());
            float loss, tv;
            check_cuda(cudaMemcpy(&loss, l.loss, 4, cudaMemcpyDeviceToHost), "loss readback");
            check_cuda(cudaMemcpy(&tv, l.tv_loss, 4, cudaMemcpyDeviceToHost), "tv loss readback");
            std::printf("loss %.9g %.9g\n", loss, tv);
        }
        std::printf("steps");
        for (uint32_t v = 0; v < views; v++) std::printf(" %d", grids.steps(v));
        std::printf("\n");
        return 0;
    } catch (const std::exception &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 1;
    }
}
