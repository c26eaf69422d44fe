// Exercises the sparse mesh export through the C++ host layer (include/brush_b200.hpp).
//   sparse_mesh_check IN OUT   IN: u32 dx dy dz, f32 origin[3] h trunc, u32 views w h, then per view a BgCamera (its raw
//                              bytes), out_img [h,w,4] f32 and out_depth [h,w] f32.
//                              OUT: mesh_ply_bytes(extract_mesh(...)) after marking, allocating and integrating every view.
#include <cstdio>
#include <fstream>
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
    if (argc != 3) { std::fprintf(stderr, "usage: sparse_mesh_check IN OUT\n"); return 2; }
    try {
        std::ifstream f(argv[1], std::ios::binary);
        uint32_t dims[3], hdr[3];
        float p[5];
        f.read(reinterpret_cast<char *>(dims), sizeof(dims));
        f.read(reinterpret_cast<char *>(p), sizeof(p));
        f.read(reinterpret_cast<char *>(hdr), sizeof(hdr));
        const uint32_t views = hdr[0], w = hdr[1], h = hdr[2];
        std::vector<BgCamera> cams(views);
        std::vector<std::vector<float>> imgs(views), deps(views);
        for (uint32_t v = 0; v < views; v++) {
            f.read(reinterpret_cast<char *>(&cams[v]), sizeof(BgCamera));
            imgs[v] = read_vec<float>(f, (size_t)w * h * 4);
            deps[v] = read_vec<float>(f, (size_t)w * h);
        }
        Context ctx(0, 16, w, h);
        DeviceBuffer<float> img((size_t)w * h * 4), dep((size_t)w * h);
        SparseTsdfGrid g(p, p[3], dims, p[4], w, h);
        for (int pass = 0; pass < 2; pass++) {
            for (uint32_t v = 0; v < views; v++) {
                img.upload(imgs[v].data(), imgs[v].size());
                dep.upload(deps[v].data(), deps[v].size());
                if (pass == 0) sparse_tsdf_mark(ctx, nullptr, g, cams[v], w, h, img.data(), dep.data());
                else sparse_tsdf_integrate(ctx, nullptr, g, cams[v], w, h, img.data(), dep.data());
            }
            if (pass == 0) sparse_tsdf_allocate(ctx, nullptr, g);
        }
        const std::string bytes = mesh_ply_bytes(extract_mesh(ctx, nullptr, g));
        std::ofstream o(argv[2], std::ios::binary);
        o.write(bytes.data(), (std::streamsize)bytes.size());
        return 0;
    } catch (const std::exception &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 1;
    }
}
