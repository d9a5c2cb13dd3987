// CPU emulation of the Welch PSD kernel: runs the SAME __host__ __device__ body as the GPU (welch_kernels.cuh: welch_body)
// block by block with nthr = 1, with the plan and route d4w_welch would choose (welch_config on a 227 KB shared memory).
// The workspace route's median (d4w_row_median on the GPU) is np.median's rule here: the two middle order statistics averaged.
// usage: welch_emul in.bin out.bin
//   in.bin : int32 nrows, ns, chunk, nperseg, step, nfft, detrend, median ; float64 scale ;
//            float32 x[nrows * ns] ; float32 window[nperseg]
//   out.bin: int32 mode, pairs, nseg, nbins ; float32 out[nrows * (ns / chunk) * nbins]
#include <algorithm>
#include <cstdio>
#include <string>
#include <vector>
#include "../../das4whales_b200/csrc/fft_plan.hpp"
#include "../../das4whales_b200/csrc/welch_kernels.cuh"
using namespace d4w;

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    FILE* fi = fopen(argv[1], "rb");
    if (!fi) return 3;
    int h[8];
    double scale = 0.0;
    if (fread(h, 4, 8, fi) != 8 || fread(&scale, 8, 1, fi) != 1) return 3;
    const int nrows = h[0], ns = h[1], chunk = h[2], nperseg = h[3], step = h[4], nfft = h[5], detrend = h[6], median = h[7];
    std::vector<float> x((size_t)nrows * ns), win((size_t)nperseg);
    if (fread(x.data(), 4, x.size(), fi) != x.size() || fread(win.data(), 4, win.size(), fi) != win.size()) return 3;
    fclose(fi);

    FftPlan pl{};
    std::string err;
    if (!make_plan(nfft, 25, pl, err, 128, 16)) { fprintf(stderr, "plan: %s\n", err.c_str()); return 4; }   // d4w_fft_plan_create
    const std::vector<float2> tw = make_twiddles(nfft);
    // the map of pl's own stages, as d4w_welch passes it (the plan's table, or for the prime-factor length its own)
    const std::vector<int> p2k = make_pos2freq(pl);
    std::vector<int> k2pos((size_t)nfft);
    for (int p = 0; p < nfft; ++p) k2pos[p2k[p]] = p;
    WelchParams wp;
    size_t smem = 0;
    if (welch_config(pl, ns, chunk, nperseg, step, detrend, scale, median, 227 * 1024, wp, smem)) { fprintf(stderr, "smem\n"); return 5; }
    wp.tw = tw.data(); wp.k2pos = k2pos.data();
    const long long blocks = (long long)nrows * wp.nchunks;
    std::vector<double> sm(smem / sizeof(double) + 16);
    std::vector<float> out((size_t)blocks * wp.nbins, -777.f);
    std::vector<float> ws(wp.mode == kWelchMedianWs ? (size_t)blocks * wp.nbins * wp.nseg : 1, -777.f);
    for (long long b = 0; b < blocks; ++b) welch_body(wp, x.data(), win.data(), out.data(), ws.data(), b, 0, 1, sm.data());
    if (wp.mode == kWelchMedianWs)
        for (size_t r = 0; r < (size_t)blocks * wp.nbins; ++r) {
            std::vector<float> v(ws.begin() + r * wp.nseg, ws.begin() + (r + 1) * wp.nseg);
            std::sort(v.begin(), v.end());
            out[r] = 0.5f * (v[(wp.nseg - 1) / 2] + v[wp.nseg / 2]);
        }

    FILE* fo = fopen(argv[2], "wb");
    const int info[4] = {wp.mode, wp.pairs, wp.nseg, wp.nbins};
    fwrite(info, 4, 4, fo);
    fwrite(out.data(), 4, out.size(), fo);
    fclose(fo);
    return 0;
}
