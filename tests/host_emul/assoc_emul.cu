// CPU emulation of the association kernels: runs the SAME __host__ __device__ bodies as the GPU (assoc_kernels.cuh) with
// the host loop of d4w_loc_associate, block by block with nthr = 1 (a vote tile is still kAssocNodes nodes).  Built with
// contraction off, so every bin is the device's.
// usage: assoc_emul in.bin out.bin
//   in.bin : int64 nch, npicks, nx, ny, nz, min_picks, max_calls ; float64 fs, c0, h, r ;
//            int32 off[nch + 1], s[npicks] ; float64 pos[nch][3], gx[nx], gy[ny], gz[nz]
//   out.bin: int64 status (0, or 2 when the histogram does not fit), K, nbins ; int64 labels[npicks], node[K] ;
//            float64 t0[K] ; int64 count[K]
#include <cstdio>
#include <vector>
#include "../../das4whales_b200/csrc/assoc_kernels.cuh"
using namespace d4w;

template <class V>
static bool rd(FILE* f, V& v) { return fread(v.data(), sizeof(v[0]), v.size(), f) == v.size(); }
template <class V>
static void wr(FILE* f, const V& v) { fwrite(v.data(), sizeof(v[0]), v.size(), f); }

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    FILE* fi = fopen(argv[1], "rb");
    if (!fi) return 3;
    std::vector<long long> hd(7);
    std::vector<double> dv(4);
    if (!rd(fi, hd) || !rd(fi, dv)) return 3;
    const int nch = (int)hd[0], nx = (int)hd[2], ny = (int)hd[3], nz = (int)hd[4];
    const long long npk = hd[1];
    const int min_picks = (int)hd[5], max_calls = (int)hd[6];
    std::vector<int> off(nch + 1), s(npk);
    std::vector<double> pos(3 * (size_t)nch), gx(nx), gy(ny), gz(nz);
    if (!rd(fi, off) || !rd(fi, s) || !rd(fi, pos) || !rd(fi, gx) || !rd(fi, gy) || !rd(fi, gz)) return 3;
    fclose(fi);

    AssocParams P{};
    std::vector<double> T(npk);
    std::vector<long long> labels(npk, -1), node(max_calls), count(max_calls);
    std::vector<double> t0(max_calls);
    P.off = off.data(); P.s = s.data(); P.nch = nch; P.npicks = npk; P.fs = dv[0]; P.pos = pos.data(); P.c0 = dv[1];
    P.gx = gx.data(); P.gy = gy.data(); P.gz = gz.data(); P.nx = nx; P.ny = ny; P.nz = nz;
    P.nnodes = (long long)nx * ny * nz;
    P.ntiles = (int)((P.nnodes + kAssocNodes - 1) / kAssocNodes);
    P.h = dv[2]; P.r = dv[3]; P.min_picks = min_picks;
    P.T = T.data(); P.labels = labels.data();
    long long status = 0, K = 0, nbins = 0;
    if (npk > 0) {
        std::vector<double> sm(14);
        AssocRange rg;
        assoc_prep_body(P, 0, 1, sm.data(), &rg);
        if (rg.bad_offsets || rg.smin < 0) return 4;
        if (!assoc_bin_range((double)rg.smin / P.fs, (double)rg.smax / P.fs, rg.box, P.c0, P.r, &P.jlo, &nbins) ||
            nbins > assoc_max_bins()) {
            status = 2;
        } else {
            P.nbins = (int)nbins;
            std::vector<int> vsm(assoc_vote_smem_bytes(P.nbins, 1) / sizeof(int) + 8);
            std::vector<AssocBest> ws(P.ntiles), red(1);
            AssocBest rec;
            for (int k = 0; k < max_calls; ++k) {
                for (int t = 0; t < P.ntiles; ++t) assoc_vote_body(P, t, 0, 1, vsm.data(), ws.data());
                assoc_pick_body(P, ws.data(), k, 0, 1, red.data(), &rec, node.data(), t0.data(), count.data());
                if (rec.bad) return 5;
                if (rec.score < min_picks) break;
                for (int c = 0; c < nch; ++c) assoc_assign_body(P, &rec, k, c, 0, 1);
                K = k + 1;
            }
        }
    }
    node.resize(K); t0.resize(K); count.resize(K);
    FILE* fo = fopen(argv[2], "wb");
    std::vector<long long> head{status, K, nbins};
    wr(fo, head); wr(fo, labels); wr(fo, node); wr(fo, t0); wr(fo, count);
    fclose(fo);
    return 0;
}
