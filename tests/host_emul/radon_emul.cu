// CPU emulation of k_radon: runs the SAME __host__ __device__ ray body as the GPU (imageops_kernels.cuh: radon_ray) for
// every (bin, angle).
// usage: radon_emul in.bin out.bin
//   in.bin : int64 h, w, n, pad_r, pad_c, nangles ; float64 cs[nangles][2] ; float32 img[h][w]
//   out.bin: float64 out[n][nangles]
#include <cstdio>
#include <vector>
#include "../../das4whales_b200/csrc/imageops_kernels.cuh"
using namespace d4w;

template <class V>
static bool rd(FILE* f, V& v) { return fread(v.data(), sizeof(v[0]), v.size(), f) == v.size(); }

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    FILE* fi = fopen(argv[1], "rb");
    if (!fi) return 3;
    std::vector<long long> hd(6);
    if (!rd(fi, hd)) return 3;
    const int h = (int)hd[0], w = (int)hd[1], n = (int)hd[2], na = (int)hd[5];
    std::vector<double> cs(2 * (size_t)na), out((size_t)n * na);
    std::vector<float> img((size_t)h * w);
    if (!rd(fi, cs) || !rd(fi, img)) return 3;
    fclose(fi);
    RadonParams p{img.data(), h, w, n, (int)hd[3], (int)hd[4], cs.data(), na, out.data()};
    for (int b = 0; b < n; ++b)
        for (int a = 0; a < na; ++a) out[(size_t)b * na + a] = radon_ray(p, b, a);
    FILE* fo = fopen(argv[2], "wb");
    fwrite(out.data(), sizeof(double), out.size(), fo);
    fclose(fo);
    return 0;
}
