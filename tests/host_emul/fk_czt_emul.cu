// CPU emulation of the chirp-z column passes (P1 / P5 for channel counts with a prime factor > 61): runs the SAME
// __host__ __device__ bodies as the GPU (fk_kernels.cuh: body_col_fwd_czt, body_col_inv_czt) block by block with nthr = 1.
// usage: fk_czt_emul in.bin out.bin
//   in.bin : int32 nx, ns, taper, nkeep ; int32 keep[nkeep] (wavenumbers 0 <= k <= nx/2, ascending) ;
//            float32 x[nx*ns] ; complex64 w_in[nkeep*ns] (input of the inverse pass)
//   out.bin: int32 czt, m, nc, nstages ; complex64 w[nkeep*ns] (forward pass of x) ; float32 y[nx*ns] (inverse pass of w_in) ;
//            complex64 chirp[nx] ; complex64 bhat[m] ; int32 pos2k_m[m]
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../../das4whales_b200/csrc/fk_hostplan.hpp"
#include "../../das4whales_b200/csrc/fk_kernels.cuh"
using namespace d4w;

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    FILE* fi = fopen(argv[1], "rb");
    if (!fi) return 3;
    int hdr[4];
    if (fread(hdr, 4, 4, fi) != 4) return 3;
    const int nx = hdr[0], ns = hdr[1], taper = hdr[2], nkeep = hdr[3];
    std::vector<int> keep((size_t)nkeep);
    std::vector<float> x((size_t)nx * ns);
    std::vector<float2> w_in((size_t)nkeep * ns);
    if (fread(keep.data(), 4, keep.size(), fi) != keep.size() || fread(x.data(), 4, x.size(), fi) != x.size() ||
        fread(w_in.data(), 8, w_in.size(), fi) != w_in.size()) return 3;
    fclose(fi);

    FkHostPlan hp; std::string err;
    if (build_fk_hostplan(nx, ns, 227 * 1024, hp, err)) { fprintf(stderr, "plan: %s\n", err.c_str()); return 4; }
    if (!hp.czt) { fprintf(stderr, "plan: %d channels did not take the chirp-z path\n", nx); return 5; }
    CztParams cp{};
    cp.pl = hp.colpl; cp.tw = hp.tw_col.data(); cp.chirp = hp.czt_chirp.data(); cp.bhat = hp.czt_bhat.data();
    cp.nx = nx; cp.ns = ns; cp.m = hp.czt_m; cp.nc = hp.nc; cp.nc_shift = hp.nc_shift; cp.fstride = hp.fstride; cp.aligned = hp.aligned;
    // slot positions exactly as d4w_fk.cu's mask_finish_support builds them
    std::vector<int2> slot_pos((size_t)std::max(nkeep, 1));
    for (int s = 0; s < nkeep; ++s) slot_pos[s] = make_int2(hp.k2pos[keep[s]], hp.k2pos[keep[s] == 0 ? 0 : nx - keep[s]]);

    std::vector<float2> smem(hp.col_smem / sizeof(float2) + 16), w((size_t)std::max(nkeep, 1) * ns, make_float2(-777.f, -777.f));
    std::vector<float> y((size_t)nx * ns, -777.f);
    const size_t ldw = ns;
    const int ntiles = (ns + 2 * hp.nc - 1) / (2 * hp.nc);
    for (int b = 0; b < ntiles; ++b)
        body_col_fwd_czt(cp, x.data(), w.data(), ldw, slot_pos.data(), nkeep, taper ? hp.taper.data() : nullptr, b, 0, 1, smem.data());
    for (int b = 0; b < ntiles; ++b)
        body_col_inv_czt(cp, w_in.data(), ldw, slot_pos.data(), nkeep, y.data(), b, 0, 1, smem.data());

    FILE* fo = fopen(argv[2], "wb");
    const int info[4] = {hp.czt, hp.czt_m, hp.nc, hp.colpl.nstages};
    fwrite(info, 4, 4, fo);
    fwrite(w.data(), 8, (size_t)nkeep * ns, fo);
    fwrite(y.data(), 4, y.size(), fo);
    fwrite(hp.czt_chirp.data(), 8, hp.czt_chirp.size(), fo);
    fwrite(hp.czt_bhat.data(), 8, hp.czt_bhat.size(), fo);
    const std::vector<int> p2k = make_pos2freq(hp.colpl);
    fwrite(p2k.data(), 4, p2k.size(), fo);
    fclose(fo);
    return 0;
}
