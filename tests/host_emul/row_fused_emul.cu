// CPU checks of k_row_mid_fused's per-pair instantiation (fk_kernels.cuh, fft_smem.cuh).
// usage: row_fused_emul pairs
//          every split-row plan (T1 > 1) of every 2^a 3^b 5^c length up to 25 x 10 240, f-k and Hilbert planner settings:
//          prints "plan R0 RL" for each (first, last) radix pair with both ends in registers, "built R0 RL" for each pair
//          of D4W_ROW_FUSED_PAIRS, and "unfused ns" for a plan that has such a pair but did not get row_fused
//        row_fused_emul body ns in.bin out.bin
//          in.bin : float32 re/im of two kept rows of W (2 x ns complex), float32 mask table (2 x ns, table order),
//                   float32 re/im complex table (ns complex, table order)
//          out.bin: int32 t1, t2, r0, rl ; int32 pos2k_row_tab[t2] ;
//                   float32 W after the float table in place, W' of the out-of-place launch, W after the complex table
#include <cstdio>
#include <cstring>
#include <set>
#include <utility>
#include <vector>
#include "../../das4whales_b200/csrc/fk_hostplan.hpp"
#include "../../das4whales_b200/csrc/fk_kernels.cuh"
using namespace d4w;

static int pairs() {
    std::set<std::pair<int, int>> plan, built;
    auto inreg = [](int r) { for (int q : inreg_radices()) if (q == r) return true; return false; };
    for (int ns = 2; ns <= 25 * 10240; ++ns) {
        if (next_5smooth(ns) != ns) continue;
        for (bool fk : {true, false}) {
            FkHostPlan hp; std::string err;
            if (build_fk_hostplan(1, ns, 227 * 1024, hp, err, /*allow_row_dual=*/fk, /*row_fused_default=*/1)) continue;
            const int nst = hp.rowpl.nstages, r0 = hp.rowpl.radix[0], rl = hp.rowpl.radix[nst - 1];
            if (hp.t1 == 1 || nst < 2 || !inreg(r0) || !inreg(rl)) continue;
            plan.insert({r0, rl});
            if (!hp.row_fused) printf("unfused %d\n", ns);
        }
    }
#define D4W_LIST(A, B) built.insert({A, B});
    D4W_ROW_FUSED_PAIRS(D4W_LIST)
#undef D4W_LIST
    for (auto& p : plan) printf("plan %d %d\n", p.first, p.second);
    for (auto& p : built) printf("built %d %d\n", p.first, p.second);
    return 0;
}

static int body(int ns, const char* fin, const char* fout) {
    FkHostPlan hp; std::string err;
    if (build_fk_hostplan(1, ns, 227 * 1024, hp, err)) { fprintf(stderr, "plan: %s\n", err.c_str()); return 4; }
    const int nst = hp.rowpl.nstages, r0 = hp.rowpl.radix[0], rl = hp.rowpl.radix[nst - 1];
    if (!hp.row_fused || hp.t1 == 1) { fprintf(stderr, "plan is not fused\n"); return 5; }
    std::vector<float2> w0((size_t)2 * ns), tc((size_t)ns);
    std::vector<float> tab((size_t)2 * ns);
    FILE* fi = fopen(fin, "rb");
    if (fread(w0.data(), 8, w0.size(), fi) != w0.size() || fread(tab.data(), 4, tab.size(), fi) != tab.size() ||
        fread(tc.data(), 8, tc.size(), fi) != tc.size()) return 3;
    fclose(fi);
    RowParams rp{}; rp.pl = hp.rowpl; rp.tw = hp.tw_row.data(); rp.twT = hp.twT.data(); rp.t1 = hp.t1; rp.t2 = hp.t2;
    std::vector<float2> smem((size_t)hp.t2), a = w0, b = w0, oop((size_t)2 * ns), c = w0;
    const bool ok = with_row_fused_pair(r0, rl, [&](auto c0, auto cl) {
        constexpr int R0 = decltype(c0)::value, RL = decltype(cl)::value;
        for (int s = 0; s < 2; ++s)
            for (int k1 = 0; k1 < hp.t1; ++k1) {
                body_row_mid_fused<R0, RL>(rp, a.data(), (size_t)ns, tab.data(), (size_t)ns, k1, s, 0, 1, smem.data());
                body_row_mid_fused<R0, RL, float, true>(rp, b.data(), (size_t)ns, tab.data(), (size_t)ns, k1, s, 0, 1, smem.data(),
                                                        oop.data());
                body_row_mid_fused<R0, RL>(rp, c.data(), (size_t)ns, tc.data(), (size_t)0, k1, s, 0, 1, smem.data());
            }
    });
    if (!ok) { fprintf(stderr, "pair not built\n"); return 6; }
    if (memcmp(b.data(), w0.data(), b.size() * sizeof(float2))) { fprintf(stderr, "out-of-place pass wrote its source\n"); return 7; }
    FILE* fo = fopen(fout, "wb");
    const int info[4] = {hp.t1, hp.t2, r0, rl};
    fwrite(info, 4, 4, fo);
    fwrite(hp.pos2k_row_tab.data(), 4, (size_t)hp.t2, fo);
    fwrite(a.data(), 8, a.size(), fo);
    fwrite(oop.data(), 8, oop.size(), fo);
    fwrite(c.data(), 8, c.size(), fo);
    fclose(fo);
    return 0;
}

int main(int argc, char** argv) {
    if (argc >= 2 && std::string(argv[1]) == "pairs") return pairs();
    if (argc >= 5 && std::string(argv[1]) == "body") return body(atoi(argv[2]), argv[3], argv[4]);
    return 2;
}
