// Exercises the compressed PLY export through the C++ host layer (include/brush_b200.hpp): compress_splats +
// compressed_ply_bytes.
//   compress_check IN OUT   IN: u32 n k mip, then transforms [n,10], sh [n,k,3], raw opacity [n].  OUT: the file bytes.
#include <cstdio>
#include <fstream>
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
    if (argc != 3) { std::fprintf(stderr, "usage: compress_check IN OUT\n"); return 2; }
    try {
        std::ifstream f(argv[1], std::ios::binary);
        uint32_t hdr[3];
        f.read(reinterpret_cast<char *>(hdr), sizeof(hdr));
        const uint32_t n = hdr[0], k = hdr[1];
        auto tr = read_vec<float>(f, (size_t)n * 10), sh = read_vec<float>(f, (size_t)n * k * 3), op = read_vec<float>(f, n);
        Context ctx(0, n, 16, 16);
        Splats splats(tr.data(), sh.data(), op.data(), n, k);
        CompressedSplats c = compress_splats(ctx, nullptr, splats.transforms.data(), splats.sh_coeffs.data(),
                                             splats.raw_opacities.data(), n, k);
        const std::string bytes = compressed_ply_bytes(c, export_comments(k, hdr[2] != 0));
        std::ofstream o(argv[2], std::ios::binary);
        o.write(bytes.data(), (std::streamsize)bytes.size());
        return 0;
    } catch (const std::exception &e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 1;
    }
}
