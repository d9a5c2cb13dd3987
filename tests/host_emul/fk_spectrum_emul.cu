// CPU emulation of the f-k power spectrum: runs the SAME __host__ __device__ bodies as the GPU (fk_kernels.cuh,
// fk_spectrum.cuh) block by block with nthr = 1, in the order d4w_fk_spectrum_apply launches them: P1 and P2 on the
// band's half-plane rows, then the power pass.  The support is built as d4w_fk_spectrum_create builds it.
// usage: fk_spectrum_emul in.bin out.bin
//   in.bin : int32 nx, ns, taper, k_lo, k_hi, f_lo, f_hi ; float32 x[nx*ns]
//   out.bin: float32 P[(k_hi-k_lo)*(f_hi-f_lo)] ; int32 nact, all_written, accumulate_ok, scheme, t1
//            (scheme: 0 single-level, 1 single-level with dual-lane bodies, 2 two-level, 4 chirp-z; all_written: every
//            element of the band was stored; accumulate_ok: a second pass with accumulate = 1 gives exactly 2 P, so no
//            element is stored twice)
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../../das4whales_b200/csrc/fk_hostplan.hpp"
#include "../../das4whales_b200/csrc/fk_spectrum.cuh"
using namespace d4w;

template <int T1> static void split_all(float2* w, size_t ldw, int t2, const float2* twT, int nact) {
    for (int s = 0; s < nact; ++s)
        for (int t = 0; t < t2; ++t) body_row_split<T1, false>(w, ldw, t2, twT, s, t);
}
static void split_dispatch(int t1, float2* w, size_t ldw, int t2, const float2* twT, int nact) {
    switch (t1) {
#define C(T) case T: split_all<T>(w, ldw, t2, twT, nact); break;
        C(2) C(3) C(4) C(5) C(6) C(8) C(10) C(12) C(15) C(16) C(20) C(25)
#undef C
        default: fprintf(stderr, "bad t1\n"); exit(2);
    }
}
template <int X1> static void colA_all(const Col2Params& c2p, const float* x, cpd* v2, const float* taper) {
    for (int c2 = 0; c2 < c2p.x2; ++c2)
        for (int t4 = 0; t4 < c2p.tpn / 2; ++t4) body_colA_fwd<X1>(c2p, x, v2, taper, c2, t4, c2p.tpb);
}
static void colA_dispatch(const Col2Params& c2p, const float* x, cpd* v2, const float* taper) {
    switch (c2p.x1) {
        case 25: colA_all<25>(c2p, x, v2, taper); break;
        case 20: colA_all<20>(c2p, x, v2, taper); break;
        case 10: colA_all<10>(c2p, x, v2, taper); break;
        default: colA_all<16>(c2p, x, v2, taper); break;
    }
}
static bool colB_fused_emul(const FkHostPlan& hp, const Col2Params& c2p, cpd* v2, float2* w, size_t ldw, const int2* need, int pl, int tb, cpd* smem) {
#define EM_FUSED3(R0, R1, R2)                                                                                \
    if (hp.fused3 && hp.r3[0] == R0 && hp.r3[1] == R1 && hp.r3[2] == R2) {                                   \
        body_colB3_fwd<R0, R1, R2>(c2p, v2, w, ldw, need, pl, tb, 0, 1, smem, c2p.tpb, c2p.tpn);             \
        return true;                                                                                         \
    }
    EM_FUSED3(10, 10, 10) EM_FUSED3(5, 5, 4)
#undef EM_FUSED3
#define EM_FUSED(RA, RB)                                                                                     \
    if (hp.fused_ra == RA && hp.fused_rb == RB) {                                                            \
        body_colB_fwd_fused<RA, RB>(c2p, v2, w, ldw, need, pl, tb, 0, 1, smem, c2p.tpb, c2p.tpn);            \
        return true;                                                                                         \
    }
    EM_FUSED(16, 16) EM_FUSED(16, 20) EM_FUSED(16, 25) EM_FUSED(20, 16) EM_FUSED(20, 20) EM_FUSED(20, 25)
    EM_FUSED(25, 16) EM_FUSED(25, 20) EM_FUSED(25, 25)
#undef EM_FUSED
    return false;
}

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    FILE* fi = fopen(argv[1], "rb");
    if (!fi) return 3;
    int hdr[7];
    if (fread(hdr, 4, 7, fi) != 7) return 3;
    const int nx = hdr[0], ns = hdr[1], taper = hdr[2], k_lo = hdr[3], k_hi = hdr[4], f_lo = hdr[5], f_hi = hdr[6];
    std::vector<float> x((size_t)nx * ns);
    if (fread(x.data(), 4, x.size(), fi) != x.size()) return 3;
    fclose(fi);

    FkHostPlan hp; std::string err;
    if (build_fk_hostplan(nx, ns, 227 * 1024, hp, err)) { fprintf(stderr, "plan: %s\n", err.c_str()); return 4; }
    // the band's half-plane rows (d4w_fk_spectrum_create)
    const int nrows = nx / 2 + 1;
    std::vector<int> act, k2slot((size_t)nrows, -1);
    for (int k = 0; k < nrows; ++k) {
        const int rp = (k + nx / 2) % nx, rn = (nx - k + nx / 2) % nx;
        if ((rp >= k_lo && rp < k_hi) || (rn >= k_lo && rn < k_hi)) { k2slot[k] = (int)act.size(); act.push_back(k); }
    }
    const int nu = (int)act.size();
    std::vector<int> k2pos_row((size_t)hp.t2);
    for (int p = 0; p < hp.t2; ++p) k2pos_row[hp.pos2k_row[p]] = p;
    std::vector<int2> slot_pos((size_t)std::max(nu, 1));
    for (int sl = 0; sl < nu; ++sl) slot_pos[sl] = make_int2(hp.k2pos[act[sl]], hp.k2pos[act[sl] == 0 ? 0 : nx - act[sl]]);

    ColParams cp{}; cp.pl = hp.colpl; cp.tw = hp.tw_col.data(); cp.k2pos = hp.k2pos.data(); cp.pos2k = hp.pos2k.data();
    cp.nx = nx; cp.ns = ns; cp.nc = hp.nc; cp.nc_shift = hp.nc_shift; cp.fstride = hp.fstride; cp.aligned = hp.aligned;
    cp.dual = hp.dual; cp.npair = hp.npair; cp.npair_shift = hp.npair_shift; cp.aligned16 = hp.aligned16;
    CztParams cz{};
    cz.pl = hp.colpl; cz.tw = hp.tw_col.data(); cz.chirp = hp.czt_chirp.data(); cz.bhat = hp.czt_bhat.data();
    cz.nx = nx; cz.ns = ns; cz.m = hp.czt_m; cz.nc = hp.nc; cz.nc_shift = hp.nc_shift; cz.fstride = hp.fstride; cz.aligned = hp.aligned;
    RowParams rp{}; rp.pl = hp.rowpl; rp.tw = hp.tw_row.data(); rp.twT = hp.twT.data(); rp.t1 = hp.t1; rp.t2 = hp.t2; rp.dual = hp.row_dual;

    const size_t ldw = ns;
    std::vector<float2> w(std::max<size_t>((size_t)nu * ns, 1));
    std::vector<float2> smem((size_t)std::max(hp.col_smem, hp.row_smem) / sizeof(float2) + 16);
    const int tile = hp.dual ? 4 * hp.npair : 2 * hp.nc, ntiles = (ns + tile - 1) / tile;
    const bool two = hp.two_level && nu > 0;
    const float* tap = taper ? hp.taper.data() : nullptr;
    cpd* sm2 = reinterpret_cast<cpd*>(smem.data());
    // P1
    if (two) {
        Col2Params c2p{}; std::vector<int2> need2; std::vector<int> plane_ptr; std::vector<Col2Entry> ents2;
        c2p.plb = hp.plb; c2p.twb = hp.tw_x2.data(); c2p.twn = hp.tw_col.data(); c2p.nx = nx; c2p.ns = ns; c2p.x1 = hp.x1; c2p.x2 = hp.x2;
        c2p.planes = hp.planes; c2p.np = hp.np2; c2p.fstride = hp.fstride2; c2p.np_shift = hp.np2 == 8 ? 3 : hp.np2 == 4 ? 2 : hp.np2 == 2 ? 1 : 0;
        c2p.vhp = hp.chunk_pairs;
        std::vector<cpd> v2((size_t)hp.planes * hp.x2 * hp.chunk_pairs);
        std::vector<Col2EntryHost> eh; build_col2_entries(hp, k2slot, plane_ptr, eh);
        for (auto& e : eh) ents2.push_back(Col2Entry{e.pos, e.slot, e.flags, 0});
        smem.resize(std::max(smem.size(), hp.colb_smem / sizeof(float2) + 16));
        sm2 = reinterpret_cast<cpd*>(smem.data());
        if (hp.fused_ra || hp.fused3) build_col2_need(hp, k2slot, need2);
        for (int tpb = 0; tpb < ns / 2; tpb += hp.chunk_pairs) {
            c2p.tpb = tpb; c2p.tpn = std::min(hp.chunk_pairs, ns / 2 - tpb);
            colA_dispatch(c2p, x.data(), v2.data(), tap);
            const int ntb = (c2p.tpn + hp.np2 - 1) / hp.np2;
            for (int pl = 0; pl < hp.planes; ++pl)
                for (int tb = 0; tb < ntb; ++tb)
                    if (!((hp.fused_ra || hp.fused3) && colB_fused_emul(hp, c2p, v2.data(), w.data(), ldw, need2.data(), pl, tb, sm2)))
                        body_colB_fwd(c2p, v2.data(), w.data(), ldw, plane_ptr.data(), ents2.data(), pl, tb, 0, 1, sm2);
        }
    } else if (nu) {
        const int czt_tiles = (ns + 2 * hp.nc - 1) / (2 * hp.nc);
        for (int b = 0; b < (hp.czt ? czt_tiles : ntiles); ++b) {
            if (hp.czt) body_col_fwd_czt(cz, x.data(), w.data(), ldw, slot_pos.data(), nu, tap, b, 0, 1, smem.data());
            else if (hp.dual) body_col_fwd_dual(cp, x.data(), w.data(), ldw, slot_pos.data(), nu, tap, b, 0, 1, sm2);
            else body_col_fwd(cp, x.data(), w.data(), ldw, slot_pos.data(), nu, tap, b, 0, 1, smem.data());
        }
    }
    // P2
    if (hp.t1 > 1 && nu) split_dispatch(hp.t1, w.data(), ldw, hp.t2, hp.twT.data(), nu);
    // power pass: once into a sentinel-filled band, then accumulated on top of it
    const int nk = k_hi - k_lo, nf = f_hi - f_lo;
    std::vector<float> P((size_t)nk * nf, -1.f);
    SpecParams sp{};
    sp.act_k = act.data(); sp.k2pos_row = k2pos_row.data(); sp.nx = nx; sp.ns = ns;
    sp.k_lo = k_lo; sp.k_hi = k_hi; sp.f_lo = f_lo; sp.f_hi = f_hi; sp.scale = 1.f;
    std::vector<float> first;
    for (int acc = 0; acc < 2; ++acc) {
        sp.accumulate = acc;
        for (int s = 0; s < nu; ++s)
            for (int k1 = 0; k1 < hp.t1; ++k1) body_fk_power(rp, sp, w.data(), ldw, k1, s, 0, 1, smem.data(), P.data());
        if (acc == 0) first = P;
    }
    int acc_ok = 1, all_written = 1;
    for (size_t i = 0; i < P.size(); ++i) {
        all_written &= first[i] >= 0.f;
        acc_ok &= P[i] == 2.f * first[i];
    }
    FILE* fo = fopen(argv[2], "wb");
    fwrite(first.data(), 4, first.size(), fo);
    const int tail[5] = {nu, all_written, acc_ok, hp.czt ? 4 : hp.two_level ? 2 : hp.dual ? 1 : 0, hp.t1};
    fwrite(tail, 4, 5, fo);
    fclose(fo);
    return 0;
}
