// CPU emulation of the chirp-z Hilbert rows (row lengths with no T1 x T2 split): runs the SAME __host__ __device__ bodies as
// the GPU (hilbert_czt.cuh: body_hczt_row, or body_hczt_fwd -> body_row_mid(_fused) -> body_hczt_turn -> body_row_mid(_fused)
// -> body_hczt_inv) with nthr = 1.  D4W_ROW_FUSED and D4W_HILBERT_PAIR select the route exactly as d4w_row_plan_create does.
// usage:
//   row_czt_emul plan N...          one line per N: "N direct T1 T2" | "N czt M T1 T2 fused" | "N error <message>"
//   row_czt_emul tables N out.bin   int32 m, t1, t2, fused ; complex64 chirp[N] ; complex64 bhat[m] ; int32 tab2freq[m]
//   row_czt_emul run in.bin out.bin in : int32 n, nrows, mode ; float32 x[nrows*n]
//                                   out: int32 m, t1, pair ; float32 y[nrows*n]
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../../das4whales_b200/csrc/fk_hostplan.hpp"
#include "../../das4whales_b200/csrc/hilbert_czt.cuh"
using namespace d4w;

static const size_t kSmem = 227 * 1024;

static std::vector<int> table_order(const RowCztPlan& cz) {
    const FkHostPlan& hp = cz.hp;
    const std::vector<int>& order = cz.fused ? hp.pos2k_row_tab : hp.pos2k_row;
    std::vector<int> t((size_t)cz.m);
    for (int kt1 = 0; kt1 < hp.t1; ++kt1)
        for (int pos = 0; pos < hp.t2; ++pos) t[(size_t)kt1 * hp.t2 + pos] = kt1 + hp.t1 * order[pos];
    return t;
}

template <int T1>
static void split_route(const RowCztPlan& cz, HcztParams hz, const float* x, float* y, int mode, const double* stats) {
    const FkHostPlan& hp = cz.hp;
    const int nrow = hz.pair ? (hz.nx + 1) / 2 : hz.nx;
    std::vector<float2> w((size_t)nrow * cz.m, make_float2(-777.f, -777.f)), smem((size_t)hp.t2 + 16);
    std::vector<float2> bc(cz.bhat.size());
    for (size_t i = 0; i < bc.size(); ++i) bc[i] = make_float2(cz.bhat[i].x, -cz.bhat[i].y);
    RowParams rp{};
    rp.pl = hp.rowpl; rp.tw = hp.tw_row.data(); rp.twT = hp.twT.data(); rp.t1 = hp.t1; rp.t2 = hp.t2;
    auto mid = [&](const float2* tab) {
        for (int r = 0; r < nrow; ++r)
            for (int k1 = 0; k1 < hp.t1; ++k1) {
                if (cz.fused) body_row_mid_fused(rp, w.data(), (size_t)cz.m, tab, (size_t)0, k1, r, 0, 1, smem.data());
                else body_row_mid(rp, w.data(), (size_t)cz.m, tab, (size_t)0, k1, r, 0, 1, smem.data());
            }
    };
    for (int r = 0; r < nrow; ++r) for (int t2 = 0; t2 < hp.t2; ++t2) body_hczt_fwd<T1>(hz, x, w.data(), r, t2);
    mid(cz.bhat.data());
    for (int r = 0; r < nrow; ++r) for (int t2 = 0; t2 < hp.t2; ++t2) body_hczt_turn<T1>(hz, w.data(), r, t2);
    mid(bc.data());
    for (int r = 0; r < nrow; ++r) for (int t2 = 0; t2 < hp.t2; ++t2) body_hczt_inv<T1>(hz, w.data(), x, y, mode, stats, r, t2);
}

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    const std::string cmd = argv[1];
    if (cmd == "plan") {
        for (int a = 2; a < argc; ++a) {
            const int n = std::atoi(argv[a]);
            FkHostPlan hp; std::string err;
            if (!build_fk_hostplan(1, n, kSmem, hp, err, false, 1)) { printf("%d direct %d %d\n", n, hp.t1, hp.t2); continue; }
            RowCztPlan cz;
            if (plan_czt_rows(n, kSmem, cz, err)) { printf("%d error %s\n", n, err.c_str()); continue; }
            printf("%d czt %d %d %d %d\n", n, cz.m, cz.hp.t1, cz.hp.t2, cz.fused);
        }
        return 0;
    }
    if (cmd == "tables" && argc >= 4) {
        const int n = std::atoi(argv[2]);
        RowCztPlan cz; std::string err;
        if (plan_czt_rows(n, kSmem, cz, err)) { fprintf(stderr, "plan: %s\n", err.c_str()); return 4; }
        FILE* fo = fopen(argv[3], "wb");
        const int info[4] = {cz.m, cz.hp.t1, cz.hp.t2, cz.fused};
        fwrite(info, 4, 4, fo);
        fwrite(cz.chirp.data(), 8, cz.chirp.size(), fo);
        fwrite(cz.bhat.data(), 8, cz.bhat.size(), fo);
        const std::vector<int> t = table_order(cz);
        fwrite(t.data(), 4, t.size(), fo);
        fclose(fo);
        return 0;
    }
    if (cmd == "run" && argc >= 4) {
        FILE* fi = fopen(argv[2], "rb");
        if (!fi) return 3;
        int hdr[3];
        if (fread(hdr, 4, 3, fi) != 3) return 3;
        const int n = hdr[0], nrows = hdr[1], mode = hdr[2];
        std::vector<float> x((size_t)nrows * n), y((size_t)nrows * n, -777.f);
        if (fread(x.data(), 4, x.size(), fi) != x.size()) return 3;
        fclose(fi);
        RowCztPlan cz; std::string err;
        if (plan_czt_rows(n, kSmem, cz, err)) { fprintf(stderr, "plan: %s\n", err.c_str()); return 4; }
        std::vector<double> stats((size_t)nrows * 4, 0.0);           // {mean, absmax, variance, 0} as k_row_stats
        for (int r = 0; r < nrows; ++r) {
            double s = 0.0, q = 0.0;
            for (int t = 0; t < n; ++t) { const double v = x[(size_t)r * n + t]; s += v; q += v * v; }
            const double mean = s / n;
            stats[4 * (size_t)r] = mean; stats[4 * (size_t)r + 2] = q / n - mean * mean;
        }
        HcztParams hz{};
        hz.n = n; hz.m = cz.m; hz.t2 = cz.hp.t2; hz.nx = nrows; hz.invn = (float)(1.0 / n);
        hz.pair = (cz.hp.t1 > 1 && env_int("D4W_HILBERT_PAIR", 1)) ? 1 : 0;
        hz.chirp = cz.chirp.data(); hz.twT = cz.hp.twT.data();
        if (cz.hp.t1 == 1) {
            std::vector<float2> bc(cz.bhat.size()), smem((size_t)cz.m + 16);
            for (size_t i = 0; i < bc.size(); ++i) bc[i] = make_float2(cz.bhat[i].x, -cz.bhat[i].y);
            RowParams rp{};
            rp.pl = cz.hp.rowpl; rp.tw = cz.hp.tw_row.data(); rp.twT = cz.hp.twT.data(); rp.t1 = 1; rp.t2 = cz.m;
            for (int r = 0; r < nrows; ++r)
                body_hczt_row(rp, hz, cz.bhat.data(), bc.data(), x.data(), y.data(), mode, stats.data(), r, 0, 1, smem.data());
        } else {
            switch (cz.hp.t1) {
#define D4W_HC(T) case T: split_route<T>(cz, hz, x.data(), y.data(), mode, stats.data()); break;
                D4W_HC(2) D4W_HC(3) D4W_HC(4) D4W_HC(5) D4W_HC(6) D4W_HC(8) D4W_HC(10) D4W_HC(12) D4W_HC(15) D4W_HC(16) D4W_HC(20) D4W_HC(25)
#undef D4W_HC
                default: fprintf(stderr, "split %d not built\n", cz.hp.t1); return 5;
            }
        }
        FILE* fo = fopen(argv[3], "wb");
        const int info[3] = {cz.m, cz.hp.t1, hz.pair};
        fwrite(info, 4, 3, fo);
        fwrite(y.data(), 4, y.size(), fo);
        fclose(fo);
        return 0;
    }
    return 2;
}
