// Exercises the mesh export through the C++ host layer (include/brush_b200.hpp).
//   mesh_check ply IN OUT    IN: u32 nv nf, then vertices f32 [nv,3], colors u8 [nv,3], faces u32 [nf,3].  OUT: mesh_ply_bytes.
//   mesh_check grid IN OUT   IN: u32 dx dy dz, f32 origin[3] h trunc, then tsdf [n], weight [n], rgb [n,3].
//                            OUT: mesh_ply_bytes(extract_mesh(...)) of that grid (needs a GPU).
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
    if (argc != 4) { std::fprintf(stderr, "usage: mesh_check ply|grid IN OUT\n"); return 2; }
    try {
        const std::string mode = argv[1];
        std::ifstream f(argv[2], std::ios::binary);
        std::string bytes;
        if (mode == "ply") {
            uint32_t hdr[2];
            f.read(reinterpret_cast<char *>(hdr), sizeof(hdr));
            TriangleMesh m;
            m.vertices = read_vec<float>(f, (size_t)hdr[0] * 3);
            m.colors = read_vec<uint8_t>(f, (size_t)hdr[0] * 3);
            m.faces = read_vec<uint32_t>(f, (size_t)hdr[1] * 3);
            bytes = mesh_ply_bytes(m);
        } else {
            uint32_t dims[3];
            float p[5];
            f.read(reinterpret_cast<char *>(dims), sizeof(dims));
            f.read(reinterpret_cast<char *>(p), sizeof(p));
            const size_t n = (size_t)dims[0] * dims[1] * dims[2];
            auto t = read_vec<float>(f, n), w = read_vec<float>(f, n), c = read_vec<float>(f, n * 3);
            Context ctx(0, 16, 16, 16);
            TsdfGrid g(p, p[3], dims, p[4]);
            g.tsdf.upload(t.data(), n);
            g.weight.upload(w.data(), n);
            g.rgb.upload(c.data(), n * 3);
            bytes = mesh_ply_bytes(extract_mesh(ctx, nullptr, g));
        }
        std::ofstream o(argv[3], std::ios::binary);
        o.write(bytes.data(), (std::streamsize)bytes.size());
        return 0;
    } catch (const std::exception &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 1;
    }
}
