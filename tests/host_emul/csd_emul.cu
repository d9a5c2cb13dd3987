// CPU emulation of the cross-spectral density / coherence kernels: runs the SAME __host__ __device__ bodies as the GPU
// (csd_kernels.cuh: csd_body and, for the workspace median, csd_median_body) block by block with nthr = 1, with the plan
// and route d4w_csd would choose (csd_config on a 227 KB shared memory).
// usage: csd_emul csd in.bin out.bin
//   in.bin : int32 nx, ny, ns, nperseg, step, nfft, detrend, what, median ; float64 scale ;
//            float32 x[nx * ns] ; float32 y[ny * ns] ; float32 window[nperseg]       (a single row is broadcast)
//   out.bin: int32 mode, frames, nseg, nbins ; float32 out[max(nx, ny) * nbins * (what ? 1 : 2)]
// usage: csd_emul median in.bin out.bin      (the signed selection alone)
//   in.bin : int32 nrows, n ; float32 v[nrows * n]
//   out.bin: float32 median[nrows]
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include "../../das4whales_b200/csrc/fft_plan.hpp"
#include "../../das4whales_b200/csrc/csd_kernels.cuh"
using namespace d4w;

static void select_rows(const std::vector<float>& v, long long nrows, int n, float* out) {
    std::vector<int> sm(kCsdSelInts);
    for (long long b = 0; b < nrows; ++b) csd_median_body(v.data(), nrows, n, out, b, 0, 1, sm.data());
}

static int run_median(const char* fin_name, const char* fout_name) {
    FILE* fi = fopen(fin_name, "rb");
    if (!fi) return 3;
    int h[2];
    if (fread(h, 4, 2, fi) != 2) return 3;
    std::vector<float> v((size_t)h[0] * h[1]);
    if (fread(v.data(), 4, v.size(), fi) != v.size()) return 3;
    fclose(fi);
    std::vector<float> out((size_t)h[0], -777.f);
    select_rows(v, h[0], h[1], out.data());
    FILE* fo = fopen(fout_name, "wb");
    fwrite(out.data(), 4, out.size(), fo);
    fclose(fo);
    return 0;
}

int main(int argc, char** argv) {
    if (argc < 4) return 2;
    if (!strcmp(argv[1], "median")) return run_median(argv[2], argv[3]);
    FILE* fi = fopen(argv[2], "rb");
    if (!fi) return 3;
    int h[9];
    double scale = 0.0;
    if (fread(h, 4, 9, fi) != 9 || fread(&scale, 8, 1, fi) != 1) return 3;
    const int nx = h[0], ny = h[1], ns = h[2], nperseg = h[3], step = h[4], nfft = h[5], detrend = h[6], what = h[7], median = h[8];
    std::vector<float> x((size_t)nx * ns), y((size_t)ny * ns), win((size_t)nperseg);
    if (fread(x.data(), 4, x.size(), fi) != x.size() || fread(y.data(), 4, y.size(), fi) != y.size() ||
        fread(win.data(), 4, win.size(), fi) != win.size()) return 3;
    fclose(fi);

    FftPlan pl{};
    std::string err;
    if (!make_plan(nfft, 25, pl, err, 128, 16)) { fprintf(stderr, "plan: %s\n", err.c_str()); return 4; }   // d4w_fft_plan_create
    const std::vector<float2> tw = make_twiddles(nfft);
    const std::vector<int> p2k = make_pos2freq(pl);          // the map of pl's own stages, as welch_k2pos gives it
    std::vector<int> k2pos((size_t)nfft);
    for (int p = 0; p < nfft; ++p) k2pos[p2k[p]] = p;
    CsdParams cp;
    size_t smem = 0;
    if (csd_config(pl, ns, nperseg, step, detrend, scale, what, median, 227 * 1024, cp, smem)) { fprintf(stderr, "smem\n"); return 5; }
    cp.tw = tw.data(); cp.k2pos = k2pos.data();
    cp.xstride = nx == 1 ? 0 : ns;
    cp.ystride = ny == 1 ? 0 : ns;
    const int nrows = nx > ny ? nx : ny;
    std::vector<double> sm(smem / sizeof(double) + 16);
    std::vector<float> out((size_t)nrows * cp.nbins * (what ? 1 : 2), -777.f);
    std::vector<float> ws(cp.mode == kCsdMedianWs ? (size_t)nrows * cp.nbins * 2 * cp.nseg : 1, -777.f);
    for (long long b = 0; b < nrows; ++b) csd_body(cp, x.data(), y.data(), win.data(), out.data(), ws.data(), b, 0, 1, sm.data());
    if (cp.mode == kCsdMedianWs) select_rows(ws, (long long)nrows * cp.nbins * 2, cp.nseg, out.data());

    FILE* fo = fopen(argv[3], "wb");
    const int info[4] = {cp.mode, cp.frames, cp.nseg, cp.nbins};
    fwrite(info, 4, 4, fo);
    fwrite(out.data(), 4, out.size(), fo);
    fclose(fo);
    return 0;
}
