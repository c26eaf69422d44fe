// Exercises the multi-view training step with bilateral grids of the C++ host layer (include/brush_b200.hpp:
// SplatTrainer::step_views_bilagrid, over bg_train_step_views_bilagrid), on one device, without the depth term.
//   views_bilagrid_check IN OUT   IN: u32 n k w h steps views grids, f32 median_scale, transforms [n,10], sh [n,k,3], raw
//                                 opacity [n], then per view: u32 length + camera line, u32 view index, packed ground
//                                 truth [h,w] u32.
//                                 stdout: one "loss <loss> <TV term of view 0> ..." line per step, then one
//                                 "steps <count of grid 0> ..." line.
//                                 OUT: the parameters after the last step (transforms, sh, raw opacity, f32), then the
//                                 grids [grids][L,H,W,12] f32.
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
    if (argc != 3) { std::fprintf(stderr, "usage: views_bilagrid_check IN OUT\n"); return 2; }
    try {
        std::ifstream f(argv[1], std::ios::binary);
        uint32_t hdr[7];
        float median_scale;
        f.read(reinterpret_cast<char *>(hdr), sizeof(hdr));
        f.read(reinterpret_cast<char *>(&median_scale), sizeof(median_scale));
        const uint32_t n = hdr[0], k = hdr[1], w = hdr[2], h = hdr[3], steps = hdr[4], views = hdr[5], num_grids = hdr[6];
        auto tr = read_vec<float>(f, (size_t)n * 10), sh = read_vec<float>(f, (size_t)n * k * 3), op = read_vec<float>(f, n);
        Context ctx(0, n, w, h);
        std::vector<Camera> cams;
        std::vector<std::unique_ptr<DeviceBuffer<uint32_t>>> gts;
        std::vector<const uint32_t *> gt_ptrs;
        std::vector<uint32_t> view_index;
        for (uint32_t v = 0; v < views; v++) {
            cams.push_back(read_camera(f));
            uint32_t idx;
            f.read(reinterpret_cast<char *>(&idx), 4);
            view_index.push_back(idx);
            auto gt = read_vec<uint32_t>(f, (size_t)w * h);
            gts.push_back(std::make_unique<DeviceBuffer<uint32_t>>(gt.size()));
            gts.back()->upload(gt.data(), gt.size());
            gt_ptrs.push_back(gts.back()->data());
        }
        Splats splats(tr.data(), sh.data(), op.data(), n, k);
        TrainConfig cfg;
        cfg.total_train_iters = 1000;
        cfg.seed = 7;
        cfg.bilateral_grid = true;
        SplatTrainer trainer(cfg, n, k, median_scale);
        BilateralGrids grids(num_grids);
        for (uint32_t i = 0; i < steps; i++) {
            const SplatTrainer::GridViewsLosses l =
                trainer.step_views_bilagrid(ctx, nullptr, nullptr, cams, gt_ptrs, view_index, {}, {}, w, h, splats, grids);
            float loss;
            std::vector<float> tv(views);
            check_cuda(cudaMemcpy(&loss, l.loss, 4, cudaMemcpyDeviceToHost), "loss readback");
            check_cuda(cudaMemcpy(tv.data(), l.tv_losses, 4 * views, cudaMemcpyDeviceToHost), "TV readback");
            std::printf("loss %.9g", loss);
            for (float x : tv) std::printf(" %.9g", x);
            std::printf("\n");
        }
        std::printf("steps");
        for (uint32_t v = 0; v < num_grids; v++) std::printf(" %d", grids.steps(v));
        std::printf("\n");
        std::ofstream o(argv[2], std::ios::binary);
        splats.transforms.download(tr.data(), tr.size());
        splats.sh_coeffs.download(sh.data(), sh.size());
        splats.raw_opacities.download(op.data(), op.size());
        std::vector<float> g((size_t)num_grids * BG_BILAGRID_FLOATS);
        check_cuda(cudaMemcpy(g.data(), grids.grid(0), g.size() * 4, cudaMemcpyDeviceToHost), "grid readback");
        o.write(reinterpret_cast<const char *>(tr.data()), tr.size() * 4);
        o.write(reinterpret_cast<const char *>(sh.data()), sh.size() * 4);
        o.write(reinterpret_cast<const char *>(op.data()), op.size() * 4);
        o.write(reinterpret_cast<const char *>(g.data()), g.size() * 4);
        return 0;
    } catch (const std::exception &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 1;
    }
}
