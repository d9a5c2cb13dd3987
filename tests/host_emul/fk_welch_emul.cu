// CPU emulation of the f-k Welch segment staging: runs the SAME __host__ __device__ body as k_fk_segment_stage
// (fk_welch.cuh) CTA by CTA with nthr = 1, over the grid d4w_fk_segment_stage launches (segment, row).
// usage: fk_welch_emul in.bin out.bin
//   in.bin : int32 nx, ns, c0, lx, t0, l, step, nseg, detrend, smem_row, stride_pad ;
//            float32 x[nx*ns], wx[lx], wt[l]
//   out.bin: float32 out[nseg * seg_stride], seg_stride = lx * l + stride_pad; the padding is filled with a sentinel (-7) so
//            that a write outside a segment shows
#include <cstdio>
#include <vector>
#include "../../das4whales_b200/csrc/fk_welch.cuh"
using namespace d4w;

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    FILE* fi = fopen(argv[1], "rb");
    if (!fi) return 3;
    int h[11];
    if (fread(h, 4, 11, fi) != 11) return 3;
    const int nx = h[0], ns = h[1];
    StageParams sp{};
    sp.ns = ns; sp.c0 = h[2]; sp.lx = h[3]; sp.t0 = h[4]; sp.l = h[5]; sp.step = h[6];
    const int nseg = h[7];
    sp.detrend = h[8]; sp.smem_row = h[9];
    sp.seg_stride = (size_t)sp.lx * sp.l + h[10];
    std::vector<float> x((size_t)nx * ns), wx(sp.lx), wt(sp.l);
    if (fread(x.data(), 4, x.size(), fi) != x.size() || fread(wx.data(), 4, wx.size(), fi) != wx.size() ||
        fread(wt.data(), 4, wt.size(), fi) != wt.size())
        return 3;
    fclose(fi);
    std::vector<float> out((size_t)nseg * sp.seg_stride, -7.f);
    std::vector<double> smem((fk_stage_smem_bytes(sp.l, 1, sp.smem_row) + 7) / 8);
    for (int s = 0; s < nseg; ++s)
        for (int r = 0; r < sp.lx; ++r) body_fk_segment_stage(sp, x.data(), wx.data(), wt.data(), out.data(), s, r, 0, 1, smem.data());
    FILE* fo = fopen(argv[2], "wb");
    fwrite(out.data(), 4, out.size(), fo);
    fclose(fo);
    return 0;
}
