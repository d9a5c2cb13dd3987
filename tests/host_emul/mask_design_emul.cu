// CPU emulation of d4w_mask_design: the SAME __host__ __device__ bodies as the GPU (tools_kernels.cuh) run row by row, CTA by
// CTA and thread by thread with the launch geometry of d4w_mask_design.cu.  It writes the float64 values the kernels round to
// float32 on their store.
// usage: mask_design_emul in.bin out.bin
//   in.bin : int32 kind, nx, ns, col_lo, col_hi ; float64 kval, fval, cs_min, cp_min, cp_max ; float64 H[ns]
//   out.bin: float64 out[nx * ns]
#include <cstdio>
#include <vector>
#include "../../das4whales_b200/csrc/tools_kernels.cuh"
using namespace d4w;

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    FILE* fi = fopen(argv[1], "rb");
    if (!fi) return 3;
    int h[5];
    double d[5];
    if (fread(h, 4, 5, fi) != 5 || fread(d, 8, 5, fi) != 5) return 3;
    const int kind = h[0], nx = h[1], ns = h[2];
    std::vector<double> H(ns);
    if (fread(H.data(), 8, ns, fi) != (size_t)ns) return 3;
    fclose(fi);
    const int r = fan_radius(kDesignSigma);
    int h_lo = ns, h_hi = ns;
    if (kind != kDesignHybrid && !design_h_band(H.data(), ns, &h_lo, &h_hi)) return 4;
    std::vector<double> w(2 * r + 1), cw(2 * r + 2), g((size_t)nx * ns);
    std::vector<int> iv((size_t)kDesignStride * nx);
    DesignParams p{kind, nx, ns, r, d[0], d[1], d[2], d[3], d[4], h[3], h[4], h_lo, h_hi, H.data(), w.data(), cw.data(), iv.data()};
    if (kind == kDesignHybrid) {                                                            // k_design_hybrid
        for (int i = 0; i < nx; ++i)
            for (int j = 0; j < ns; ++j) g[(size_t)i * ns + j] = body_hybrid(p, i, j);
    } else {
        fan_weights(kDesignSigma, r, w.data(), cw.data());                                  // k_design_rows
        for (int i = 0; i < nx; ++i) body_design_row(p, i);
        std::vector<double> wz(fan_steps(r)), cws(2 * r + 2), T((size_t)fan_tile_rows(r) * kFanTJ);
        for (int by = 0; by < (nx + kFanRT - 1) / kFanRT; ++by)                            // k_design_blur
            for (int bx = 0; bx < (ns + kFanTJ - 1) / kFanTJ; ++bx) {
                const int i0 = by * kFanRT, j0 = bx * kFanTJ;
                body_fan_weights(p, wz.data(), cws.data(), 0, 1);
                body_fan_fill_tile(p, i0, j0, cws.data(), T.data(), 0, 1);
                for (int t = 0; t < kFanThreads; ++t) {
                    const int lane = t % kFanTJ, gr = t / kFanTJ, j = j0 + lane;
                    double acc[kFanU];
                    body_fan_taps(p, wz.data(), T.data(), gr, lane, acc);
                    for (int u = 0; u < kFanU; ++u) {
                        const int i = i0 + gr * kFanU + u;
                        if (i < nx && j < ns) g[(size_t)i * ns + j] = acc[u];
                    }
                }
            }
    }
    FILE* fo = fopen(argv[2], "wb");
    if (!fo) return 3;
    fwrite(g.data(), 8, g.size(), fo);
    fclose(fo);
    printf("OK\n");
    return 0;
}
