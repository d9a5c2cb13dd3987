// CPU emulation of d4w_fan_blur: the SAME __host__ __device__ bodies as the GPU (tools_kernels.cuh) run CTA by CTA and thread
// by thread, with the launch geometry of d4w_tools.cu; the global min / max pass and the normalising pass as the two launches.
// usage: fan_blur_emul in.bin out.bin
//   in.bin : int32 nx, ns ; float64 kval, fval, c_min, c_max, sigma
//   out.bin: float32 out[nx * ns]
#include <cstdio>
#include <vector>
#include "../../das4whales_b200/csrc/tools_kernels.cuh"
using namespace d4w;

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    FILE* fi = fopen(argv[1], "rb");
    if (!fi) return 3;
    int h[2];
    double d[5];
    if (fread(h, 4, 2, fi) != 2 || fread(d, 8, 5, fi) != 5) return 3;
    fclose(fi);
    const int nx = h[0], ns = h[1];
    const double sigma = d[4];
    const int r = fan_radius(sigma);
    std::vector<double> w(2 * r + 1), cw(2 * r + 2);
    std::vector<int> J(2 * (size_t)nx);
    fan_weights(sigma, r, w.data(), cw.data());                                             // k_fan_rows
    for (int i = 0; i < nx; ++i) body_fan_row(nx, ns, d[0], d[1], d[2], d[3], J.data(), i);
    FanParams p{nx, ns, r, d[0], d[1], d[2], d[3], w.data(), cw.data(), J.data()};

    std::vector<double> wz(fan_steps(r)), cws(2 * r + 2), H((size_t)fan_tile_rows(r) * kFanTJ), g((size_t)nx * ns);
    unsigned long long kmin = ~0ull, kmax = 0ull;
    for (int by = 0; by < (nx + kFanRT - 1) / kFanRT; ++by)                                // k_fan_blur, both passes
        for (int bx = 0; bx < (ns + kFanTJ - 1) / kFanTJ; ++bx) {
            const int i0 = by * kFanRT, j0 = bx * kFanTJ;
            body_fan_weights(p, wz.data(), cws.data(), 0, 1);
            body_fan_fill_tile(p, i0, j0, cws.data(), H.data(), 0, 1);
            for (int t = 0; t < kFanThreads; ++t) {
                const int lane = t % kFanTJ, gr = t / kFanTJ, j = j0 + lane;
                double acc[kFanU];
                body_fan_taps(p, wz.data(), H.data(), gr, lane, acc);
                for (int u = 0; u < kFanU; ++u) {
                    const int i = i0 + gr * kFanU + u;
                    if (i >= nx || j >= ns) continue;
                    g[(size_t)i * ns + j] = acc[u];
                    const unsigned long long k = fan_key(acc[u]);
                    if (k < kmin) kmin = k;
                    if (k > kmax) kmax = k;
                }
            }
        }
    const double mn = fan_unkey(kmin), span = fan_unkey(kmax) - mn;
    std::vector<float> out((size_t)nx * ns);
    for (size_t q = 0; q < out.size(); ++q) out[q] = (float)((g[q] - mn) / span);
    FILE* fo = fopen(argv[2], "wb");
    if (!fo) return 3;
    fwrite(out.data(), 4, out.size(), fo);
    fclose(fo);
    printf("OK\n");
    return 0;
}
