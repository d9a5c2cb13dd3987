// CPU emulation of the localisation kernels: runs the SAME __host__ __device__ bodies as the GPU (loc_kernels.cuh:
// loc_grid_body + loc_pick_body, loc_gn_body) block by block with nthr = 1 (a grid tile is then kLocGridNodes nodes).
// usage: loc_emul in.bin out.bin
//   in.bin : int64 mode (0 grid, 1 solve), ncalls, nobs, nbiter, fix_z, has_n0, nx, ny, nz ; float64 c0 ;
//            int64 off[ncalls + 1] ; float64 T[nobs], pos[nobs][3] ; float64 n0[ncalls][4] (has_n0) ;
//            float64 gx[nx], gy[ny], gz[nz] (grid)
//   out.bin: grid : int64 index[ncalls] ; float64 score[ncalls], n0[ncalls][4]
//            solve: float64 n[ncalls][4], var[ncalls], unc[ncalls][p], cinv[ncalls][p][p], cond[ncalls],
//                   traj[ncalls][nbiter][4]
#include <cstdio>
#include <vector>
#include "../../das4whales_b200/csrc/loc_kernels.cuh"
using namespace d4w;

template <class V>
static bool rd(FILE* f, V& v) { return fread(v.data(), sizeof(v[0]), v.size(), f) == v.size(); }
template <class V>
static void wr(FILE* f, const V& v) { fwrite(v.data(), sizeof(v[0]), v.size(), f); }

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    FILE* fi = fopen(argv[1], "rb");
    if (!fi) return 3;
    std::vector<long long> h(9);
    std::vector<double> c0v(1);
    if (!rd(fi, h) || !rd(fi, c0v)) return 3;
    const int mode = (int)h[0], B = (int)h[1], nbiter = (int)h[3], fix_z = (int)h[4], has_n0 = (int)h[5];
    const long long nobs = h[2];
    const int nx = (int)h[6], ny = (int)h[7], nz = (int)h[8];
    const int p = fix_z ? 3 : 4;
    std::vector<long long> off(B + 1);
    std::vector<double> T(nobs), pos(3 * nobs), n0(has_n0 ? 4 * (size_t)B : 0), gx(nx), gy(ny), gz(nz);
    if (!rd(fi, off) || !rd(fi, T) || !rd(fi, pos) || !rd(fi, n0)) return 3;
    if (mode == 0 && (!rd(fi, gx) || !rd(fi, gy) || !rd(fi, gz))) return 3;
    fclose(fi);
    FILE* fo = fopen(argv[2], "wb");
    if (mode == 0) {
        LocGridParams g{};
        g.T = T.data(); g.pos = pos.data(); g.off = off.data(); g.gx = gx.data(); g.gy = gy.data(); g.gz = gz.data();
        g.nx = nx; g.ny = ny; g.nz = nz;
        g.nnodes = (long long)nx * ny * nz;
        g.tile = kLocGridNodes;
        g.ntiles = (int)((g.nnodes + g.tile - 1) / g.tile);
        g.p = p;
        g.inv_c0 = 1.0 / c0v[0];
        std::vector<double> sm(loc_grid_smem_bytes(1) / sizeof(double) + 8);
        std::vector<LocBest> ws((size_t)B * g.ntiles);
        for (int b = 0; b < B; ++b)
            for (int t = 0; t < g.ntiles; ++t) loc_grid_body(g, t, b, 0, 1, sm.data(), ws.data());
        std::vector<long long> index(B);
        std::vector<double> score(B), nn(4 * (size_t)B);
        for (int b = 0; b < B; ++b) loc_pick_body(g, ws.data(), b, 0, 1, sm.data(), index.data(), score.data(), nn.data());
        wr(fo, index); wr(fo, score); wr(fo, nn);
    } else {
        std::vector<double> n(4 * (size_t)B), var(B), unc((size_t)B * p), cinv((size_t)B * p * p), cond(B),
            traj((size_t)B * nbiter * 4);
        LocSolveParams sp{};
        sp.T = T.data(); sp.pos = pos.data(); sp.off = off.data(); sp.n0 = has_n0 ? n0.data() : nullptr;
        sp.nbiter = nbiter; sp.fix_z = fix_z; sp.c0 = c0v[0];
        sp.n = n.data(); sp.var = var.data(); sp.unc = unc.data(); sp.cinv = cinv.data(); sp.cond = cond.data();
        sp.traj = nbiter > 0 ? traj.data() : nullptr;
        std::vector<double> sm(loc_gn_smem_bytes(1) / sizeof(double) + 8);
        for (int b = 0; b < B; ++b) loc_gn_body(sp, b, 0, 1, sm.data());
        wr(fo, n); wr(fo, var); wr(fo, unc); wr(fo, cinv); wr(fo, cond); wr(fo, traj);
    }
    fclose(fo);
    return 0;
}
