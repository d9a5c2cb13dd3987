// CPU emulation of an f-k mask bank: runs the SAME __host__ __device__ bodies as the GPU (fk_kernels.cuh) block by
// block with nthr = 1, in the order d4w_fk_bank_apply launches them: P1 and P2 once on the union support U, then for
// each mask the out-of-place P3 (W -> W'), P4 on W' and P5 from W'.  Support and tables are built as d4w_fk.cu builds
// them: each mask's own kept rows at its eps, U = their union, and each bank table gathered from the mask's own table.
// usage: fk_bank_emul in.bin out.bin
//   in.bin : int32 nx, ns, taper, nmasks ; float64 eps[nmasks] ; float32 x[nx*ns] ; float32 mask[nmasks][nx*ns] (dense)
//   out.bin: float32 y[nmasks][nx*ns] ; int32 |U|, nact[nmasks], w_untouched, zero_rows_ok, scheme
//            (scheme: 0 single-level, 1 single-level with dual-lane bodies, 2 two-level, 4 chirp-z)
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../../das4whales_b200/csrc/fk_hostplan.hpp"
#include "../../das4whales_b200/csrc/fk_kernels.cuh"
using namespace d4w;

template <int T1> static void split_all(bool inv, float2* w, size_t ldw, int t2, const float2* twT, int nact) {
    for (int s = 0; s < nact; ++s)
        for (int t = 0; t < t2; ++t) {
            if (inv) body_row_split<T1, true>(w, ldw, t2, twT, s, t);
            else body_row_split<T1, false>(w, ldw, t2, twT, s, t);
        }
}
static void split_dispatch(int t1, bool inv, float2* w, size_t ldw, int t2, const float2* twT, int nact) {
    switch (t1) {
#define C(T) case T: split_all<T>(inv, w, ldw, t2, twT, nact); break;
        C(2) C(3) C(4) C(5) C(6) C(8) C(10) C(12) C(15) C(16) C(20) C(25)
#undef C
        default: fprintf(stderr, "bad t1\n"); exit(2);
    }
}
template <int X1> static void colA_all(bool inv, const Col2Params& c2p, const float* x, cpd* v2, float* y, const float* taper) {
    for (int c2 = 0; c2 < c2p.x2; ++c2)
        for (int t4 = 0; t4 < c2p.tpn / 2; ++t4) {
            if (inv) body_colA_inv<X1>(c2p, v2, y, c2, t4, c2p.tpb);
            else body_colA_fwd<X1>(c2p, x, v2, taper, c2, t4, c2p.tpb);
        }
}
static void colA_dispatch(bool inv, const Col2Params& c2p, const float* x, cpd* v2, float* y, const float* taper) {
    switch (c2p.x1) {
        case 25: colA_all<25>(inv, c2p, x, v2, y, taper); break;
        case 20: colA_all<20>(inv, c2p, x, v2, y, taper); break;
        case 10: colA_all<10>(inv, c2p, x, v2, y, taper); break;
        default: colA_all<16>(inv, c2p, x, v2, y, taper); break;
    }
}
template <bool INV>
static bool colB_fused_emul(const FkHostPlan& hp, const Col2Params& c2p, cpd* v2, float2* w, size_t ldw, const int2* need, int pl, int tb, cpd* smem) {
#define EM_FUSED3(R0, R1, R2)                                                                                \
    if (hp.fused3 && hp.r3[0] == R0 && hp.r3[1] == R1 && hp.r3[2] == R2) {                                   \
        if constexpr (!INV) body_colB3_fwd<R0, R1, R2>(c2p, v2, w, ldw, need, pl, tb, 0, 1, smem, c2p.tpb, c2p.tpn);           \
        else body_colB3_inv<R0, R1, R2>(c2p, v2, w, ldw, need, pl, tb, 0, 1, smem, c2p.tpb, c2p.tpn);                          \
        return true;                                                                                         \
    }
    EM_FUSED3(10, 10, 10) EM_FUSED3(5, 5, 4)
#undef EM_FUSED3
#define EM_FUSED(RA, RB)                                                                                     \
    if (hp.fused_ra == RA && hp.fused_rb == RB) {                                                            \
        if constexpr (!INV) body_colB_fwd_fused<RA, RB>(c2p, v2, w, ldw, need, pl, tb, 0, 1, smem, c2p.tpb, c2p.tpn);          \
        else body_colB_inv_fused<RA, RB>(c2p, v2, w, ldw, need, pl, tb, 0, 1, smem, c2p.tpb, c2p.tpn);                         \
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
    int hdr[4];
    if (fread(hdr, 4, 4, fi) != 4) return 3;
    const int nx = hdr[0], ns = hdr[1], taper = hdr[2], nm = hdr[3];
    std::vector<double> eps((size_t)nm);
    std::vector<float> x((size_t)nx * ns), dense((size_t)nm * nx * ns);
    if (fread(eps.data(), 8, eps.size(), fi) != eps.size() || fread(x.data(), 4, x.size(), fi) != x.size() ||
        fread(dense.data(), 4, dense.size(), fi) != dense.size()) return 3;
    fclose(fi);

    FkHostPlan hp; std::string err;
    if (build_fk_hostplan(nx, ns, 227 * 1024, hp, err)) { fprintf(stderr, "plan: %s\n", err.c_str()); return 4; }
    const int nrows = nx / 2 + 1;
    const double scale = 1.0 / ((double)nx * ns);
    // each mask's own support (mask_finish_support) and transform-order table (d4w_fk_mask_build)
    std::vector<std::vector<int>> act((size_t)nm);
    std::vector<std::vector<float>> own((size_t)nm);
    std::vector<char> in_union((size_t)nrows, 0);
    for (int i = 0; i < nm; ++i) {
        MaskParams mp{}; mp.kind = MASK_DENSE; mp.nx = nx; mp.ns = ns; mp.dense = dense.data() + (size_t)i * nx * ns;
        std::vector<unsigned int> rowmax((size_t)nrows, 0u);
        for (int k = 0; k < nrows; ++k) body_mask_rowmax(mp, rowmax.data(), k, 0, ns, 0, 1);
        for (int k = 0; k < nrows; ++k) { float v; memcpy(&v, &rowmax[k], 4); if (v > (float)eps[i]) { act[i].push_back(k); in_union[k] = 1; } }
        own[i].resize(std::max<size_t>(act[i].size() * ns, 1));
        for (size_t j = 0; j < act[i].size() * ns; ++j) body_mask_build(mp, own[i].data(), act[i].data(), hp.pos2k_row_tab.data(), hp.t1, hp.t2, scale, j);
    }
    // the bank: union support, row map, gathered tables (d4w_fk_bank_create / d4w_fk_bank_build)
    std::vector<int> uni, k2slot((size_t)nrows, -1);
    for (int k = 0; k < nrows; ++k) if (in_union[k]) { k2slot[k] = (int)uni.size(); uni.push_back(k); }
    const int nu = (int)uni.size();
    const size_t total = (size_t)nu * ns;
    std::vector<float> tab(std::max<size_t>((size_t)nm * total, 1));
    int zero_ok = 1;
    for (int i = 0; i < nm; ++i) {
        std::vector<int> src_row((size_t)std::max(nu, 1), -1);
        size_t j = 0;
        for (int u = 0; u < nu && j < act[i].size(); ++u) if (uni[u] == act[i][j]) src_row[u] = (int)j++;
        for (size_t idx = 0; idx < total; ++idx) body_bank_gather(own[i].data(), tab.data() + i * total, src_row.data(), ns, idx);
        for (int u = 0; u < nu; ++u)
            for (int t = 0; t < ns && src_row[u] < 0; ++t) zero_ok &= tab[i * total + (size_t)u * ns + t] == 0.f;
    }
    std::vector<int2> slot_pos((size_t)std::max(nu, 1));
    for (int sl = 0; sl < nu; ++sl) slot_pos[sl] = make_int2(hp.k2pos[uni[sl]], hp.k2pos[uni[sl] == 0 ? 0 : nx - uni[sl]]);

    ColParams cp{}; cp.pl = hp.colpl; cp.tw = hp.tw_col.data(); cp.k2pos = hp.k2pos.data(); cp.pos2k = hp.pos2k.data();
    cp.nx = nx; cp.ns = ns; cp.nc = hp.nc; cp.nc_shift = hp.nc_shift; cp.fstride = hp.fstride; cp.aligned = hp.aligned;
    cp.dual = hp.dual; cp.npair = hp.npair; cp.npair_shift = hp.npair_shift; cp.aligned16 = hp.aligned16;
    CztParams cz{};
    cz.pl = hp.colpl; cz.tw = hp.tw_col.data(); cz.chirp = hp.czt_chirp.data(); cz.bhat = hp.czt_bhat.data();
    cz.nx = nx; cz.ns = ns; cz.m = hp.czt_m; cz.nc = hp.nc; cz.nc_shift = hp.nc_shift; cz.fstride = hp.fstride; cz.aligned = hp.aligned;
    RowParams rp{}; rp.pl = hp.rowpl; rp.tw = hp.tw_row.data(); rp.twT = hp.twT.data(); rp.t1 = hp.t1; rp.t2 = hp.t2; rp.dual = hp.row_dual;

    const size_t ldw = ns;
    std::vector<float2> w(std::max<size_t>(total, 1)), w3(std::max<size_t>(total, 1));
    std::vector<float2> smem((size_t)std::max(hp.col_smem, hp.row_smem) / sizeof(float2) + 16);
    const int tile = hp.dual ? 4 * hp.npair : 2 * hp.nc, ntiles = (ns + tile - 1) / tile;
    const bool two = hp.two_level && nu > 0;
    const float* tap = taper ? hp.taper.data() : nullptr;
    Col2Params c2p{}; std::vector<int2> need2; std::vector<cpd> v2; std::vector<int> plane_ptr; std::vector<Col2Entry> ents2;
    if (two) {
        c2p.plb = hp.plb; c2p.twb = hp.tw_x2.data(); c2p.twn = hp.tw_col.data(); c2p.nx = nx; c2p.ns = ns; c2p.x1 = hp.x1; c2p.x2 = hp.x2;
        c2p.planes = hp.planes; c2p.np = hp.np2; c2p.fstride = hp.fstride2; c2p.np_shift = hp.np2 == 8 ? 3 : hp.np2 == 4 ? 2 : hp.np2 == 2 ? 1 : 0;
        c2p.vhp = hp.chunk_pairs;
        v2.resize((size_t)hp.planes * hp.x2 * hp.chunk_pairs);
        std::vector<Col2EntryHost> eh; build_col2_entries(hp, k2slot, plane_ptr, eh);
        for (auto& e : eh) ents2.push_back(Col2Entry{e.pos, e.slot, e.flags, 0});
        smem.resize(std::max(smem.size(), hp.colb_smem / sizeof(float2) + 16));
        if (hp.fused_ra || hp.fused3) build_col2_need(hp, k2slot, need2);
    }
    cpd* sm2 = reinterpret_cast<cpd*>(smem.data());
    // P1 + P2, once
    if (two) {
        for (int tpb = 0; tpb < ns / 2; tpb += hp.chunk_pairs) {
            c2p.tpb = tpb; c2p.tpn = std::min(hp.chunk_pairs, ns / 2 - tpb);
            colA_dispatch(false, c2p, x.data(), v2.data(), nullptr, tap);
            const int ntb = (c2p.tpn + hp.np2 - 1) / hp.np2;
            for (int pl = 0; pl < hp.planes; ++pl)
                for (int tb = 0; tb < ntb; ++tb)
                    if (!((hp.fused_ra || hp.fused3) && colB_fused_emul<false>(hp, c2p, v2.data(), w.data(), ldw, need2.data(), pl, tb, sm2)))
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
    if (hp.t1 > 1 && nu) split_dispatch(hp.t1, false, w.data(), ldw, hp.t2, hp.twT.data(), nu);
    const std::vector<float2> w_p2 = w;
    std::vector<float> y((size_t)nm * nx * ns, -777.f);
    for (int i = 0; i < nm; ++i) {
        const float* ti = tab.data() + i * total;
        std::fill(w3.begin(), w3.end(), make_float2(-555.f, -555.f));        // every row of W' must be written by P3
        if (hp.row_dual) {
            for (int pr = 0; pr < (nu + 1) / 2; ++pr)
                for (int k1 = 0; k1 < hp.t1; ++k1)
                    body_row_mid_dual<true>(rp, w.data(), ldw, ti, (size_t)ns, k1, pr, nu, 0, 1, sm2, w3.data());
        } else {
            for (int s = 0; s < nu; ++s)
                for (int k1 = 0; k1 < hp.t1; ++k1) {
                    if (hp.row_fused) body_row_mid_fused<float, true>(rp, w.data(), ldw, ti, (size_t)ns, k1, s, 0, 1, smem.data(), w3.data());
                    else body_row_mid<float, true>(rp, w.data(), ldw, ti, (size_t)ns, k1, s, 0, 1, smem.data(), w3.data());
                }
        }
        if (hp.t1 > 1 && nu) split_dispatch(hp.t1, true, w3.data(), ldw, hp.t2, hp.twT.data(), nu);
        float* yi = y.data() + (size_t)i * nx * ns;
        if (two) {
            for (int tpb = 0; tpb < ns / 2; tpb += hp.chunk_pairs) {
                c2p.tpb = tpb; c2p.tpn = std::min(hp.chunk_pairs, ns / 2 - tpb);
                const int ntb = (c2p.tpn + hp.np2 - 1) / hp.np2;
                for (int pl = 0; pl < hp.planes; ++pl)
                    for (int tb = 0; tb < ntb; ++tb)
                        if (!((hp.fused_ra || hp.fused3) && colB_fused_emul<true>(hp, c2p, v2.data(), w3.data(), ldw, need2.data(), pl, tb, sm2)))
                            body_colB_inv(c2p, v2.data(), w3.data(), ldw, plane_ptr.data(), ents2.data(), pl, tb, 0, 1, sm2);
                colA_dispatch(true, c2p, nullptr, v2.data(), yi, nullptr);
            }
        } else {
            const int czt_tiles = (ns + 2 * hp.nc - 1) / (2 * hp.nc);
            for (int b = 0; b < (hp.czt ? czt_tiles : ntiles); ++b) {
                if (hp.czt) body_col_inv_czt(cz, w3.data(), ldw, slot_pos.data(), nu, yi, b, 0, 1, smem.data());
                else if (hp.dual) body_col_inv_dual(cp, w3.data(), ldw, slot_pos.data(), nu, yi, b, 0, 1, sm2);
                else body_col_inv(cp, w3.data(), ldw, slot_pos.data(), nu, yi, b, 0, 1, smem.data());
            }
        }
    }
    const int w_untouched = memcmp(w.data(), w_p2.data(), w.size() * sizeof(float2)) == 0;

    FILE* fo = fopen(argv[2], "wb");
    fwrite(y.data(), 4, y.size(), fo);
    std::vector<int> tail{nu};
    for (int i = 0; i < nm; ++i) tail.push_back((int)act[i].size());
    tail.push_back(w_untouched); tail.push_back(zero_ok);
    tail.push_back(hp.czt ? 4 : hp.two_level ? 2 : hp.dual ? 1 : 0);
    fwrite(tail.data(), 4, tail.size(), fo);
    fclose(fo);
    return 0;
}
